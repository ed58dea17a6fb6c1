"""Oracle (test infrastructure): QR-DQN (Dabney, Rowland, Bellemare & Munos, AAAI 2018) on the reference's C51 layer set.

The network is the reference DQN's rainbow_only branch (``network.layer_shapes(A, rainbow_only=True, atoms=N)``) with its
N outputs per action read as quantile values at the fixed fractions tau_hat_i = (2i+1)/(2N):

  q_i(s, a) = v_i + a_i(a) - mean_a a_i ,  written quantile-major (N*B, A), row i*B + b ;  Q(s, a) = mean_i q_i(s, a)

The double-DQN target is R + gamma^n nt q_tgt_j(s', a*), a* = argmax_a Q_online(s', a) (under value rescaling:
h(R + gamma^n nt h^-1(q_tgt_j)), a* on mean_j h^-1(q_j)), and the loss is losses.iqn_pairwise_loss at tau_hat.

Two statements: float64 numpy (head, fractions, target, loss) and a torch-fp32 learner step whose gradients come from
autograd.  All randomness (three noise resets) is injected by the caller.
"""
import numpy as np
import torch

from . import losses, network as net, value_rescaling as vr


# ------------------------------------------------------------------------------------------------ float64 statements
def fractions_np(n):
    """tau_hat_i = (2i+1)/(2n), i = 0..n-1 (float64)."""
    return (2.0 * np.arange(n) + 1.0) / (2.0 * n)


def fractions_f32(n):
    """tau_hat_i = fl((2i+1)/(2n)): numerator and denominator exact in float32, one correctly rounded division."""
    return (2.0 * np.arange(n, dtype=np.float32) + np.float32(1)) / np.float32(2 * n)


def head_np(zv, za, action_space):
    """zv (B, n), za (B, A*n) -> q (n*B, A) in float64, quantile-major."""
    zv = np.asarray(zv, np.float64)
    B, n = zv.shape
    a = np.asarray(za, np.float64).reshape(B, action_space, n)
    q = zv[:, None, :] + a - a.mean(1, keepdims=True)                  # (B, A, n)
    return q.transpose(2, 0, 1).reshape(n * B, action_space)


def head_f32_np(zv, za, action_space):
    """The head as riqn_qr_head_fwd rounds it, in numpy float32: s_i = sum_a za (a ascending, from 0),
    q = fl(fl(zv + za) - fl(s_i / A))."""
    zv = np.asarray(zv, np.float32)
    B, n = zv.shape
    a = np.asarray(za, np.float32).reshape(B, action_space, n)
    s = np.zeros((B, n), np.float32)
    for k in range(action_space):
        s = (s + a[:, k, :]).astype(np.float32)
    mean = (s / np.float32(action_space)).astype(np.float32)
    q = ((zv[:, None, :] + a).astype(np.float32) - mean[:, None, :]).astype(np.float32)
    return q.transpose(2, 0, 1).reshape(n * B, action_space)


def q_values_np(q, batch):
    """Q (B, A) = mean_i q_i of quantile-major q (n*B, A)."""
    q = np.asarray(q, np.float64)
    return q.reshape(-1, batch, q.shape[1]).mean(0)


def target_np(q_tgt, a_star, returns, nonterminals, gamma_n, eps=None):
    """(B, n) targets R + gamma^n nt q_tgt_j(s', a*) in float64 (under value rescaling with ``eps``:
    h(R + gamma^n nt h^-1(q_tgt_j))), from the target pass q_tgt (n*B, A)."""
    q_tgt = np.asarray(q_tgt, np.float64)
    B = len(a_star)
    z = q_tgt.reshape(-1, B, q_tgt.shape[1])[:, np.arange(B), a_star].T    # (B, n)
    g = gamma_n * np.asarray(nonterminals, np.float64)[:, None]
    r = np.asarray(returns, np.float64)[:, None]
    if eps is None:
        return r + g * z
    return vr.h_np(r + g * vr.h_inv_np(z, eps), eps)


def loss_np(theta, target, kappa=1.0):
    """loss (B,) = mean_j sum_i rho^kappa_{tau_hat_i}(target_j - theta_i), theta (B, n) at the fixed fractions."""
    theta = torch.as_tensor(np.asarray(theta, np.float64))
    n = theta.shape[1]
    tau = torch.from_numpy(np.broadcast_to(fractions_np(n), theta.shape).copy())
    return losses.iqn_pairwise_loss(theta, torch.as_tensor(np.asarray(target, np.float64)), tau, kappa).numpy()


# ------------------------------------------------------------------------------------------------ torch fp32 step
def layer_shapes(action_space, n):
    return net.layer_shapes(action_space, rainbow_only=True, atoms=n)


def make_params(seed, action_space, n):
    return net.make_params(seed, action_space, rainbow_only=True, atoms=n)


def make_noises(seed, action_space, n, count=3):
    return tuple(net.make_noise(seed + 1000 * i, action_space, rainbow_only=True, atoms=n) for i in range(count))


def dqn_forward_qr(p, x, action_space, n, training=True, keep=None):
    """q (n*B, A), quantile-major, of the QR network with parameters ``p`` on frames x (B, 4, 84, 84) fp32 in [0, 1]."""
    feat = net.conv_trunk(p, x, keep)
    h_v = torch.relu(net.noisy_linear(p, "fcnoisy_h_v", feat, training))
    h_a = torch.relu(net.noisy_linear(p, "fcnoisy_h_a", feat, training))
    v = net.noisy_linear(p, "fcnoisy_z_v", h_v, training).view(-1, 1, n)
    a = net.noisy_linear(p, "fcnoisy_z_a", h_a, training).view(-1, action_space, n)
    q = v + a - a.mean(1, keepdim=True)                                # (B, A, n)
    if keep is not None:
        keep.update(feat=feat, h_v=h_v, h_a=h_a, v=v, a=a)
    return q.permute(2, 0, 1).reshape(-1, action_space)


def act_values(p, states, action_space, n, eps=None, training=True):
    """(E, A) Q = mean_i q_i (under value rescaling: mean_i h^-1(q_i)) of the online network."""
    with torch.no_grad():
        q = dqn_forward_qr(p, states, action_space, n, training)
        E = states.shape[0]
        if eps is None:
            return q.view(n, E, action_space).mean(0)
        return vr._mean_h_inv(q, n, E, eps)


def qr_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, *, n, discount=0.99,
            n_step=3, kappa=1.0, eps=None, keep=None):
    """The QR-DQN double-DQN n-step loss (B,) with injected noises (online s' pass, target pass, online s pass)."""
    B = states.shape[0]
    A = p_online["fcnoisy_z_a.bias_mu"].shape[0] // n
    with torch.no_grad():
        net.apply_noise(p_online, noises[0])
        q_sel = dqn_forward_qr(p_online, next_states, A, n)
        qv = q_sel.view(n, B, A).mean(0) if eps is None else vr._mean_h_inv(q_sel, n, B, eps)
        a_star = qv.argmax(1)
        net.apply_noise(p_target, noises[1])
        q_tgt = dqn_forward_qr(p_target, next_states, A, n)
        z = q_tgt.view(n, B, A)[:, torch.arange(B), a_star].t()           # (B, n)
        g = (discount ** n_step) * nonterminals[:, None]
        if eps is None:
            target = returns[:, None] + g * z
        else:
            target = vr.h_torch(returns[:, None].double() + g.double() * vr.h_inv_torch(z, eps).double(), eps).float()
    net.apply_noise(p_online, noises[2])
    q_on = dqn_forward_qr(p_online, states, A, n, keep=keep)
    theta = q_on.view(n, B, A)[:, torch.arange(B), actions].t()           # (B, n)
    tau = torch.from_numpy(fractions_f32(n)).expand(B, n)
    loss = losses.iqn_pairwise_loss(theta, target, tau, kappa)
    if keep is not None:
        keep.update(a_star=a_star, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, target=target, theta=theta.detach(), qv_next=qv)
    return loss


def learn_step(p_online, p_target, batch, weights, noises, cfg, eps=None, keep=None):
    """Loss (B,) and the gradients of (weights * loss).mean() by autograd (no optimiser step)."""
    states, actions, returns, next_states, nonterminals = batch
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = qr_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, n=cfg["n_tau"],
                   discount=cfg["discount"], n_step=cfg["n_step"], kappa=cfg["kappa"], eps=eps, keep=keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    return loss.detach(), grads
