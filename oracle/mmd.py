"""Oracle (test infrastructure): MMDQN (Nguyen-Tang, Gupta & Venkatesh, AAAI 2021) on the QR-DQN network.

The network, the double-DQN a* and the targets are oracle.qr's.  The N outputs of an action are particles; the loss of a
transition is the squared maximum mean discrepancy between the online particles theta (B, n) and the detached target
particles T (B, n) under a mixture of Gaussian kernels over the bandwidths H:

  k(x, y)  = sum_{h in H} exp(-(x - y)^2 / h) ,  k1(x, y) = d k / d x = -sum_h (2 (x - y) / h) exp(-(x - y)^2 / h)
  MMD^2[b] = (1/n^2) sum_i sum_j [k(theta_i, theta_j) + k(T_i, T_j) - 2 k(theta_i, T_j)]
  loss[b]  = max(0, MMD^2[b]) ,  dtheta_i = d MMD^2 / d theta_i = (2/n^2) sum_j [k1(theta_i, theta_j) - k1(theta_i, T_j)]

Two statements: float64 numpy (loss, clamped and unclamped, and dtheta) and a torch-fp32 learner step whose gradients
come from autograd.  There is no golden fixture (the reference has no MMD loss); tests pin the statement by identities.
"""
import numpy as np
import torch

from . import network as net, qr, value_rescaling as vr

DEFAULT_BANDWIDTHS = tuple(float(h) for h in range(1, 11))


# ------------------------------------------------------------------------------------------------ float64 statements
def _gram(x, y, bandwidths):
    """k(x_i, y_j) (B, n, m) and the per-pair sum_h (2/h) exp(-(x_i - y_j)^2 / h), for x (B, n), y (B, m)."""
    d = x[:, :, None] - y[:, None, :]
    s = d * d
    k = np.zeros_like(s)
    w = np.zeros_like(s)
    for h in bandwidths:
        e = np.exp(-s / h)
        k += e
        w += (2.0 / h) * e
    return k, w, d


def mmd2_np(theta, target, bandwidths=DEFAULT_BANDWIDTHS):
    """The unclamped MMD^2 (B,) in float64."""
    theta, target = np.asarray(theta, np.float64), np.asarray(target, np.float64)
    n = theta.shape[1]
    ktt, _, _ = _gram(theta, theta, bandwidths)
    kTT, _, _ = _gram(target, target, bandwidths)
    ktT, _, _ = _gram(theta, target, bandwidths)
    return (ktt + kTT - 2.0 * ktT).sum((1, 2)) / (n * n)


def loss_np(theta, target, bandwidths=DEFAULT_BANDWIDTHS):
    """loss (B,) = max(0, MMD^2) in float64."""
    return np.maximum(mmd2_np(theta, target, bandwidths), 0.0)


def dtheta_np(theta, target, bandwidths=DEFAULT_BANDWIDTHS):
    """d MMD^2 / d theta (B, n) in float64 (the gradient of the unclamped sum)."""
    theta, target = np.asarray(theta, np.float64), np.asarray(target, np.float64)
    n = theta.shape[1]
    _, w1, d1 = _gram(theta, theta, bandwidths)
    _, w3, d3 = _gram(theta, target, bandwidths)
    return (2.0 / (n * n)) * ((-d1 * w1) - (-d3 * w3)).sum(2)


def mmd2_torch(theta, target, bandwidths=DEFAULT_BANDWIDTHS):
    """The unclamped MMD^2 (B,) in torch, differentiable in theta (target detached), in the dtype of theta."""
    target = target.detach()
    n = theta.shape[1]

    def k(x, y):
        s = (x[:, :, None] - y[:, None, :]) ** 2
        return sum(torch.exp(-s / h) for h in bandwidths)

    return (k(theta, theta) + k(target, target) - 2.0 * k(theta, target)).sum((1, 2)) / (n * n)


def clamped(mmd2):
    """max(0, mmd2) in value, with the gradient of the unclamped mmd2 (as the kernel's dtheta)."""
    return mmd2 + (mmd2.clamp_min(0.0) - mmd2).detach()


# ------------------------------------------------------------------------------------------------ torch fp32 step
def mmd_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, *, n,
             bandwidths=DEFAULT_BANDWIDTHS, discount=0.99, n_step=3, eps=None, keep=None):
    """The MMDQN double-DQN n-step loss (B,) with injected noises (online s' pass, target pass, online s pass)."""
    B = states.shape[0]
    A = p_online["fcnoisy_z_a.bias_mu"].shape[0] // n
    with torch.no_grad():
        net.apply_noise(p_online, noises[0])
        q_sel = qr.dqn_forward_qr(p_online, next_states, A, n)
        qv = q_sel.view(n, B, A).mean(0) if eps is None else vr._mean_h_inv(q_sel, n, B, eps)
        a_star = qv.argmax(1)
        net.apply_noise(p_target, noises[1])
        q_tgt = qr.dqn_forward_qr(p_target, next_states, A, n)
        z = q_tgt.view(n, B, A)[:, torch.arange(B), a_star].t()           # (B, n)
        g = (discount ** n_step) * nonterminals[:, None]
        if eps is None:
            target = returns[:, None] + g * z
        else:
            target = vr.h_torch(returns[:, None].double() + g.double() * vr.h_inv_torch(z, eps).double(), eps).float()
    net.apply_noise(p_online, noises[2])
    q_on = qr.dqn_forward_qr(p_online, states, A, n, keep=keep)
    theta = q_on.view(n, B, A)[:, torch.arange(B), actions].t()           # (B, n)
    loss = clamped(mmd2_torch(theta, target, bandwidths))
    if keep is not None:
        keep.update(a_star=a_star, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, target=target, theta=theta.detach(), qv_next=qv)
    return loss


def learn_step(p_online, p_target, batch, weights, noises, cfg, eps=None, keep=None):
    """Loss (B,) and the gradients of (weights * loss).mean() by autograd (no optimiser step).  ``cfg`` as oracle.qr's,
    plus "bandwidths" (default: 1..10)."""
    states, actions, returns, next_states, nonterminals = batch
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = mmd_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, n=cfg["n_tau"],
                    bandwidths=cfg.get("bandwidths", DEFAULT_BANDWIDTHS), discount=cfg["discount"],
                    n_step=cfg["n_step"], eps=eps, keep=keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    return loss.detach(), grads
