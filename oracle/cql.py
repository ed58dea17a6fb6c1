"""Oracle (test infrastructure): CQL (Kumar, Zhou, Tucker & Levine, NeurIPS 2020) on the IQN and QR-DQN losses.

Per transition b, on the online pass q_on (N*B, A), quantile-major (row i*B + b), with a_t = actions[b]:

  Q_a = mean_i q_on[i*B+b, a],  lse = logsumexp_a Q_a,  pi = softmax(Q),  gap = lse - Q_{a_t} >= 0
  loss = td + alpha * gap,      d gap / d q_on[i*B+b, a] = (pi_a - 1{a = a_t}) / N

Statements: float64 numpy (gap, pi and the gap's gradient); the float32 numpy statements of the kernels (the means, the
loss and the dense upstream gradient G, every operation rounded on its own); and a torch-fp32 learner step on
losses.iqn_loss / value_rescaling.iqn_loss / qr.qr_loss whose gradients come from autograd.
"""
import numpy as np
import torch

from . import losses, qr as oq, value_rescaling as vr

F32 = np.float32


# ------------------------------------------------------------------------------------------------ float64 statements
def gap_from_means_np(Q, actions):
    """(gap (B,), pi (B, A), lse (B,)) in float64 from the action values Q (B, A): m = max_a Q_a,
    lse = m + log(sum_a exp(Q_a - m)) with the sum a ascending."""
    Q = np.asarray(Q, np.float64)
    m = Q.max(1)
    s = np.zeros(Q.shape[0])
    for a in range(Q.shape[1]):
        s = s + np.exp(Q[:, a] - m)
    lse = m + np.log(s)
    return lse - Q[np.arange(Q.shape[0]), np.asarray(actions)], np.exp(Q - lse[:, None]), lse


def gap_np(q, batch, actions):
    """gap (B,) and pi (B, A) of the quantile values q (N*B, A), Q the float64 mean."""
    q = np.asarray(q, np.float64)
    g, pi, _ = gap_from_means_np(q.reshape(-1, batch, q.shape[1]).mean(0), actions)
    return g, pi


def gap_grad_np(q, batch, actions):
    """d gap[b] / d q (N*B, A): (pi[b, a] - 1{a = a_t}) / N on every row i*B + b."""
    q = np.asarray(q, np.float64)
    n = q.shape[0] // batch
    _, pi = gap_np(q, batch, actions)
    d = pi.copy()
    d[np.arange(batch), np.asarray(actions)] -= 1.0
    return np.tile(d / n, (n, 1))


# ------------------------------------------------------------------------------------------------ float32 statements
def means_f32(q, batch):
    """Q (B, A) as the kernel forms it: the fp32 sum over i ascending, divided once by N."""
    q = np.asarray(q, F32)
    q3 = q.reshape(-1, batch, q.shape[1])
    s = np.zeros(q3.shape[1:], F32)
    for i in range(q3.shape[0]):
        s = (s + q3[i]).astype(F32)
    return (s / F32(q3.shape[0])).astype(F32)


def loss_f32(td, gap, alpha):
    """fl(td + fl(alpha * gap))."""
    return (np.asarray(td, F32) + (F32(alpha) * np.asarray(gap, F32)).astype(F32)).astype(F32)


def dense_grad_f32(dtheta, pi, actions, gscale, gscale_mul, alpha, n):
    """G (n*B, A): w_b = fl(gscale[b] * gscale_mul), c = fl(alpha / n), g = fl(c * pi); fl(w_b * g) off the action taken,
    fl(w_b * fl(dtheta + fl(g - c))) on it."""
    pi = np.asarray(pi, F32)
    B, A = pi.shape
    w = (np.asarray(gscale, F32) * F32(gscale_mul)).astype(F32)
    c = (F32(alpha) / F32(n)).astype(F32)
    g = (c * pi).astype(F32)
    G = np.tile((w[:, None] * g).astype(F32), (n, 1))
    rows = np.arange(n * B)
    at = np.tile(np.asarray(actions), n)
    on = (np.asarray(dtheta, F32) + (g[rows % B, at] - c).astype(F32)).astype(F32)
    G[rows, at] = (np.tile(w, n) * on).astype(F32)
    return G


# ------------------------------------------------------------------------------------------------ torch fp32 step
def gap_torch(q_on, n, batch, actions):
    Q = q_on.reshape(n, batch, -1).mean(0)
    return torch.logsumexp(Q, 1) - Q[torch.arange(batch), actions]


def cql_loss(kind, p_online, p_target, batch, noises, taus, cfg, alpha, eps=None, keep=None):
    """The CQL loss (B,) on the IQN (``kind`` "iqn", taus injected) or QR-DQN ("qr") double-DQN step, with keep["td"] and
    keep["gap"]; keep["qv_next"] holds the values a* was chosen on."""
    keep = {} if keep is None else keep
    states, actions, returns, next_states, nonterminals = batch
    B = states.shape[0]
    sizes = dict(discount=cfg["discount"], n_step=cfg["n_step"], kappa=cfg["kappa"])
    if kind == "qr":
        n = cfg["n_tau"]
        td = oq.qr_loss(p_online, p_target, *batch, noises, n=n, eps=eps, keep=keep, **sizes)
    else:
        n = cfg["n_tau"]
        kw = dict(n_tau=n, n_tau_prime=cfg["n_tau_prime"], n_quantile=cfg["n_quantile"], **sizes)
        if eps is None:
            td = losses.iqn_loss(p_online, p_target, *batch, noises, taus, keep=keep, **kw)
            keep["qv_next"] = keep["q_sel"].reshape(cfg["n_quantile"], B, -1).mean(0)
        else:
            td = vr.iqn_loss(p_online, p_target, *batch, noises, taus, eps=eps, keep=keep, **kw)
    gap = gap_torch(keep["q_on"], n, B, actions)
    keep.update(td=td.detach(), gap=gap.detach())
    return td + alpha * gap


def learn_step(kind, p_online, p_target, batch, weights, noises, taus, cfg, alpha, eps=None, keep=None):
    """Loss (B,) and the gradients of (weights * loss).mean() by autograd (no optimiser step)."""
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = cql_loss(kind, p_online, p_target, batch, noises, taus, cfg, alpha, eps, keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    return loss.detach(), grads
