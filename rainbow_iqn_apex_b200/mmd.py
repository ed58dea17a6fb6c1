"""MMDQN, Distributional Reinforcement Learning via Moment Matching (Nguyen-Tang, Gupta & Venkatesh, AAAI 2021).

MMDQN trains the QR-DQN network (qr.py) with another loss.  It reads the N outputs of an action as unordered particles
of the return distribution, not as quantiles at fixed fractions, and matches them to the N Bellman-target particles
T_j = R + gamma^n nt q_tgt_j(s', a*) with the squared maximum mean discrepancy under a mixture of Gaussian kernels:

  k(x, y) = sum_h exp(-(x - y)^2 / h) ,  MMD^2 = (1/N^2) sum_i sum_j [k(th_i, th_j) + k(T_i, T_j) - 2 k(th_i, T_j)]

The loss (riqn_mmd_loss_fwd_bwd, or riqn_mmd_loss_fwd_bwd_h against the transformed target under value rescaling) is
clamped at 0, since it becomes the priority loss^omega.  Everything else is QR-DQN's: the network, the three passes, a*,
the one-hot head backward (the loss writes dtheta quantile-major, as the quantile-Huber loss does), acting by the mean of
the particles, and checkpoints.  The network's second output, QR-DQN's fixed fractions, is not read.
"""
import ctypes

from ._lib import call, ptr

def mmd_loss(agent, B, N, q_on, q_tgt, actions, a_star, returns, nonterminals, loss, dtheta, theta_out, target_out):
    """The double-DQN MMD loss kernel over the bandwidths ``agent.mmd``: riqn_mmd_loss_fwd_bwd, or against the
    transformed target h(R + gamma^n nt h^-1(Z)) under value rescaling (riqn_mmd_loss_fwd_bwd_h)."""
    bw = agent.mmd
    hb = (ctypes.c_float * len(bw))(*bw)      # read by the call: a captured graph holds the values
    args = (ptr(q_on), ptr(q_tgt), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals),
            agent.gamma_n(), len(bw), hb)
    outs = (ptr(loss), ptr(dtheta), ptr(theta_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_mmd_loss_fwd_bwd", B, N, agent.action_space, *args, *outs)
    else:
        call("riqn_mmd_loss_fwd_bwd_h", B, N, agent.action_space, *args, eps, *outs)
