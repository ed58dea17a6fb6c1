"""Oracle (test infrastructure): the Munchausen-IQN target and learner step.

Vieillard, Pietquin, Geist, "Munchausen Reinforcement Learning", NeurIPS 2020, in the n-step form of the authors' M-IQN:
with the target network's quantiles Z_j over N' fractions, temperature te > 0, scale alpha >= 0 and clip l0 <= 0,

  qbar'(a) = mean_j Z_j(s_{t+n}, a)          qbar(a) = mean_j Z_j(s_t, a)
  l'(a)    = qbar'(a) - max qbar' - te ln sum_a exp((qbar'(a) - max qbar') / te)        (l from qbar likewise)
  pi'(a)   = exp((qbar'(a) - max qbar') / te) / sum_a exp(...)
  m        = alpha min(max(l(a_t), l0), 0)
  T_j      = R + m + gamma^n nt sum_a pi'(a) (Z_j(s_{t+n}, a) - l'(a))

and the quantile-Huber loss of T_j against the online network's theta_i = Z_{tau_i}(s_t, a_t), as for IQN.  The target
network runs once, over the stacked frames [next_states; states]: row j*2B + b is s_{t+n}, row j*2B + B + b is s_t.

The reference has no Munchausen term, so there is no golden fixture: tests pin this module by identities (the hard-max
limit, equal means, the sign and the clip of the bonus) and by the agreement of the float64 and torch-fp32 statements.
"""
import numpy as np
import torch

from . import losses, network as net


def _split(q_tgt, batch, n_tau_prime):
    """(N'*2B, A) stacked rows -> (Z(s_{t+n}), Z(s_t)), each (N', B, A)."""
    z = q_tgt.reshape(n_tau_prime, 2, batch, -1)
    return z[:, 0], z[:, 1]


def soft_target_np(q_tgt, returns, nonterminals, actions, gamma_n, alpha, entropy_tau, l0):
    """The target in float64.  q_tgt (N'*2B, A) in the stacked row order.  Returns (target (B, N'), bonus (B,))."""
    q_tgt = np.asarray(q_tgt, np.float64)
    batch = len(returns)
    zn, zc = _split(q_tgt, batch, q_tgt.shape[0] // (2 * batch))
    te = float(entropy_tau)

    def log_policy(qbar):
        d = qbar - qbar.max(axis=1, keepdims=True)
        s = np.exp(d / te).sum(axis=1, keepdims=True)
        return d - te * np.log(s), np.exp(d / te) / s

    lp_n, pi_n = log_policy(zn.mean(axis=0))
    lp_c, _ = log_policy(zc.mean(axis=0))
    l_at = lp_c[np.arange(batch), np.asarray(actions)]
    bonus = float(alpha) * np.minimum(np.maximum(l_at, float(l0)), 0.0)
    soft = (pi_n[None] * (zn - lp_n[None])).sum(axis=2)                     # (N', B)
    g = float(gamma_n) * np.asarray(nonterminals, np.float64)
    target = np.asarray(returns, np.float64)[None] + bonus[None] + g[None] * soft
    return target.T, bonus


def soft_target(q_tgt, returns, nonterminals, actions, gamma_n, alpha, entropy_tau, l0):
    """The same target in torch fp32 (autograd-free).  Returns (target (B, N'), bonus (B,))."""
    batch = returns.shape[0]
    zn, zc = _split(q_tgt, batch, q_tgt.shape[0] // (2 * batch))

    def log_policy(qbar):
        d = qbar - qbar.max(dim=1, keepdim=True).values
        s = torch.exp(d / entropy_tau).sum(dim=1, keepdim=True)
        return d - entropy_tau * torch.log(s), torch.exp(d / entropy_tau) / s

    lp_n, pi_n = log_policy(zn.mean(dim=0))
    lp_c, _ = log_policy(zc.mean(dim=0))
    l_at = lp_c.gather(1, actions[:, None])[:, 0]
    bonus = alpha * torch.clamp(l_at, min=l0, max=0.0)
    soft = (pi_n[None] * (zn - lp_n[None])).sum(dim=2)
    target = returns[None] + bonus[None] + (gamma_n * nonterminals)[None] * soft
    return target.t(), bonus


def pairwise_loss_np(theta, target, tau, kappa=1.0):
    """Quantile-Huber loss and its gradient in float64: theta (B, N), target (B, N'), tau (B, N).  Returns (loss (B,),
    dloss/dtheta (B, N)), the indicator detached as in losses.iqn_pairwise_loss."""
    d = np.asarray(target, np.float64)[:, :, None] - np.asarray(theta, np.float64)[:, None, :]    # (B, N', N)
    ad = np.abs(d)
    hub = np.where(ad <= kappa, 0.5 * d * d, kappa * (ad - 0.5 * kappa))
    dh = np.where(ad <= kappa, d, kappa * np.sign(d))
    w = np.abs(np.asarray(tau, np.float64)[:, None, :] - (d < 0))
    n_tp = d.shape[1]
    return (w * hub / kappa).sum(axis=2).mean(axis=1), -(w * dh / kappa).sum(axis=1) / n_tp


def miqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, taus, *, n_tau,
              n_tau_prime, discount=0.99, n_step=3, kappa=1.0, alpha=0.9, entropy_tau=0.03, l0=-1.0, keep=None, **_):
    """The Munchausen-IQN loss with injected randomness: ``noises`` = (target noise, online noise), ``taus`` = (tau'
    (N'*2B, 1) in the stacked row order, tau (N*B, 1)).  Returns loss (B,), differentiable w.r.t. p_online."""
    batch = states.shape[0]
    with torch.no_grad():
        net.apply_noise(p_target, noises[0])
        q_tgt = net.dqn_forward_iqn(p_target, torch.cat((next_states, states)), n_tau_prime, taus[0])
        target, bonus = soft_target(q_tgt, returns, nonterminals, actions, discount ** n_step, alpha, entropy_tau, l0)
    net.apply_noise(p_online, noises[1])
    q_on = net.dqn_forward_iqn(p_online, states, n_tau, taus[1], keep=keep)
    theta = q_on.gather(1, actions[:, None].repeat(n_tau, 1)).reshape(n_tau, batch).t()
    loss = losses.iqn_pairwise_loss(theta, target, taus[1].reshape(n_tau, batch).t(), kappa)
    if keep is not None:
        keep.update(target=target, bonus=bonus, theta=theta, q_tgt=q_tgt, q_on=q_on)
    return loss


def learn_step(p_online, p_target, adam, batch, weights, noises, taus, cfg, keep=None):
    """losses.learn_step with the Munchausen loss: loss -> (weights * loss).mean().backward() -> Adam.  ``cfg``:
    cases.iqn_cfg plus alpha / entropy_tau / l0.  Returns (loss (B,) detached, grads dict)."""
    states, actions, returns, next_states, nonterminals = batch
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = miqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, taus, **cfg,
                     keep=keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    adam.step(p_online, grads)
    return loss.detach(), grads
