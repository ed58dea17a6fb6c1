"""DQfD: learning from demonstrations (Hester et al., AAAI 2018) kept in the prioritized replay, for the quantile learners.

Demonstrations live permanently in the replay's last ``demo_segments`` segments and every minibatch is drawn from the one
sum-tree (DQfD's single-buffer form, as in Ape-X DQfD, Pohlen et al. 2018).  On the rows that came from demonstrations the
learner adds a large-margin supervised loss that makes the network prefer the demonstrator's action a_E = actions[b]:

  Q_a     = fl32(S_a / N),  S_a = the fp32 sum over i ascending of q_on[i*B+b, a]     (riqn_argmax_mean's mean)
  v_a     = Q_a for a = a_E,  fl32(Q_a + l) otherwise;   a_hat = the first a ascending with v_a = max_a v_a
  J[b]    = fl32(max_a v_a - Q_{a_E}) >= 0
  loss[b] = fl32(td[b] + fl32(lambda * J[b])) on a demonstration row,  td[b] on any other

on the online pass over ``states``, where td is the quantile-Huber loss the learner trains without DQfD.  Under value
rescaling the outputs, and so the margin l, are in h-space units.  One kernel forms td, its dtheta, J, a_hat and the loss
(riqn_dqfd_loss_fwd_bwd, riqn_dqfd_loss_fwd_bwd_h under value rescaling).  J's gradient, (1/N)(1{a = a_hat} - 1{a = a_E})
on every quantile row, touches a second action: at backward time riqn_dqfd_dense_grad forms the dense upstream gradient
G (N*B, A) and the head's dense backward takes it.  The replay's demonstration priority bonus eps_d (ReplayMemory,
riqn_sumtree_update_demo) keeps demonstrations sampled.  DQfD applies to IQN (risk-sensitive a* selection included) and
QR-DQN; acting, the actors' priorities and checkpoints are the plain learner's.
"""
import torch

from ._lib import call, ptr

def demo_flags(agent, demo, B):
    """The loss cores' ``demo`` argument as (B,) uint8 flags on the online network's device, or None.  A mask needs an
    agent with ``dqfd``: raises ValueError otherwise, or for a mask of another shape or type."""
    if demo is None:
        return None
    if getattr(agent, "dqfd", None) is None:
        raise ValueError("a demonstration mask needs the DQfD loss: set dqfd = 1")
    if not torch.is_tensor(demo) or demo.dtype not in (torch.uint8, torch.bool) or tuple(demo.shape) != (B,):
        raise ValueError(f"demo must be a uint8 or bool tensor of shape ({B},)")
    demo = demo.to(agent.online_net._flat.device).contiguous()
    return demo.view(torch.uint8) if demo.dtype == torch.bool else demo


def dqfd_loss(agent, B, N, Np, q_on, q_tgt, tau, actions, a_star, returns, nonterminals, demo, loss, dtheta, theta_out,
              target_out, margin_out=None):
    """The DQfD loss at ``agent.dqfd``: the quantile-Huber loss of compute_loss_iqn._quantile_loss plus lambda * J on the
    rows ``demo`` flags, by riqn_dqfd_loss_fwd_bwd (riqn_dqfd_loss_fwd_bwd_h under value rescaling).  Returns
    (td_loss (B,), a_hat (B,) int64)."""
    dev = q_on.device
    td = torch.empty(B, device=dev)
    a_hat = torch.empty(B, dtype=torch.int64, device=dev)
    margin, lam = agent.dqfd
    args = (ptr(q_on), ptr(q_tgt), ptr(tau), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals), ptr(demo),
            agent.gamma_n(), float(agent.kappa), margin, lam)
    outs = (ptr(loss), ptr(td), ptr(dtheta), ptr(margin_out), ptr(a_hat), ptr(theta_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_dqfd_loss_fwd_bwd", B, N, Np, agent.action_space, *args, *outs)
    else:
        call("riqn_dqfd_loss_fwd_bwd_h", B, N, Np, agent.action_space, *args, eps, *outs)
    return td, a_hat


def dense_grad(agent, B, N, dtheta, a_hat, actions, demo, gscale, gscale_mul):
    """G (N*B, A): the gradient of sum_b gscale[b] * gscale_mul * loss[b] with respect to the online quantiles, for the
    head's dense backward (riqn_dqfd_dense_grad)."""
    G = torch.empty(N * B, agent.action_space, device=dtheta.device)
    call("riqn_dqfd_dense_grad", B, N, agent.action_space, ptr(dtheta), ptr(a_hat), ptr(actions), ptr(demo), ptr(gscale),
         float(gscale_mul), agent.dqfd[1], ptr(G))
    return G
