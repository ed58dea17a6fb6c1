"""HL-Gauss: training the C51 network by classification (Farebrother et al., "Stop Regressing: Training Value Functions
via Classification for Scalable Deep RL", ICML 2024; the histogram loss of Imani & White, ICML 2018).

HL-Gauss trains the C51 network (c51.py) with another target.  The categorical Bellman projection is replaced by the
histogram of a Gaussian N(y, sigma^2), sigma = r * delta_z, centred on the scalar double-DQN target

  y = clamp(R + gamma^n nt sum_j p_tgt(s', a*)_j z_j, v_min, v_max)      (under value rescaling: h(R + gamma^n nt E[h^-1(Z)]))

with the bins [z_j - delta_z / 2, z_j + delta_z / 2] around the atoms, renormalised over [v_min - delta_z / 2,
v_max + delta_z / 2].  The loss is the cross-entropy -sum_j m_j log p_j(s, a), one fused kernel
(riqn_hl_gauss_loss_fwd_bwd, or riqn_hl_gauss_loss_fwd_bwd_h under value rescaling) whose gradient dq the C51 head
backward takes unchanged.  Everything else is C51's: the three passes, a*, acting, the captured step graphs and
checkpoints.
"""
from ._lib import call, ptr

def hl_gauss_loss(agent, B, log_ps, pns, actions, a_star, returns, nonterminals, loss, dq, m_out, target_out):
    """The HL-Gauss cross-entropy at ratio ``agent.hl_gauss``: riqn_hl_gauss_loss_fwd_bwd, or the transformed target
    h(R + gamma^n nt E[h^-1(Z)]) under value rescaling (riqn_hl_gauss_loss_fwd_bwd_h)."""
    args = (ptr(log_ps), ptr(pns), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals), ptr(agent.support),
            agent.gamma_n(), float(agent.Vmin), float(agent.Vmax), agent.hl_gauss)
    outs = (ptr(loss), ptr(dq), ptr(m_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_hl_gauss_loss_fwd_bwd", B, agent.action_space, agent.atoms, *args, *outs)
    else:
        call("riqn_hl_gauss_loss_fwd_bwd_h", B, agent.action_space, agent.atoms, *args, eps, *outs)
