"""CQL: Conservative Q-Learning (Kumar, Zhou, Tucker & Levine, NeurIPS 2020) for the quantile learners, on logged data.

On a fixed dataset the max over actions in a double-DQN target picks actions the data never took, whose values nothing
corrects.  CQL adds to each transition's distributional loss a regulariser that pushes every action's value down and the
logged action's up:

  Q_a     = fl32(S_a / N),  S_a = the fp32 sum over i ascending of q_on[i*B+b, a]     (riqn_argmax_mean's mean)
  lse     = max_a Q_a + log(sum_a exp(Q_a - max_a Q_a))                              (double, a ascending)
  pi[b,a] = fl32(exp(Q_a - lse)),   gap[b] = fl32(lse - Q_{a_t}) >= 0,   a_t = actions[b]
  loss[b] = fl32(td[b] + fl32(alpha * gap[b]))

on the online pass over ``states`` (h-space outputs under value rescaling), where td is the quantile-Huber loss the
learner trains without CQL.  The paper's Atari agent is QR-DQN plus this term.  One kernel forms td, its dtheta, pi and
the loss (riqn_cql_loss_fwd_bwd, riqn_cql_loss_fwd_bwd_h under value rescaling).  The gap's gradient,
(alpha / N) (pi[b,a] - 1{a = a_t}) on every quantile row, is dense over actions: at backward time riqn_cql_dense_grad
forms the dense upstream gradient G (N*B, A) and the head's dense backward takes it.  CQL applies to IQN (risk-sensitive
a* selection included) and QR-DQN; acting, priorities (on the CQL loss), the captured step graphs and checkpoints are the
plain learner's.
"""
import torch

from ._lib import call, ptr

def cql_loss(agent, B, N, Np, q_on, q_tgt, tau, actions, a_star, returns, nonterminals, loss, dtheta, theta_out,
             target_out, gap_out=None):
    """The CQL loss at ``agent.cql``: the quantile-Huber loss of compute_loss_iqn._quantile_loss plus alpha * gap, by
    riqn_cql_loss_fwd_bwd (riqn_cql_loss_fwd_bwd_h under value rescaling).  Returns (td_loss (B,), pi (B, A))."""
    dev = q_on.device
    td = torch.empty(B, device=dev)
    pi = torch.empty(B, agent.action_space, device=dev)
    args = (ptr(q_on), ptr(q_tgt), ptr(tau), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals),
            agent.gamma_n(), float(agent.kappa), agent.cql)
    outs = (ptr(loss), ptr(td), ptr(pi), ptr(dtheta), ptr(gap_out), ptr(theta_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_cql_loss_fwd_bwd", B, N, Np, agent.action_space, *args, *outs)
    else:
        call("riqn_cql_loss_fwd_bwd_h", B, N, Np, agent.action_space, *args, eps, *outs)
    return td, pi


def dense_grad(agent, B, N, dtheta, pi, actions, gscale, gscale_mul):
    """G (N*B, A): the gradient of sum_b gscale[b] * gscale_mul * loss[b] with respect to the online quantiles, for the
    head's dense backward (riqn_cql_dense_grad)."""
    G = torch.empty(N * B, agent.action_space, device=dtheta.device)
    call("riqn_cql_dense_grad", B, N, agent.action_space, ptr(dtheta), ptr(pi), ptr(actions), ptr(gscale),
         float(gscale_mul), agent.cql, ptr(G))
    return G
