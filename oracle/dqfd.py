"""Oracle (test infrastructure): DQfD (Hester et al., AAAI 2018) on the IQN and QR-DQN losses.

Per transition b, on the online pass q_on (N*B, A), quantile-major (row i*B + b), with a_E = actions[b], margin l and
demonstration flag d_b:

  Q_a = mean_i q_on[i*B+b, a],  v_a = Q_a + l * 1{a != a_E},  a_hat = first argmax_a v_a,  J = v_{a_hat} - Q_{a_E} >= 0
  loss = td + lambda * d_b * J,  dJ / d q_on[i*B+b, a] = (1{a = a_hat} - 1{a = a_E}) / N

Statements: float64 numpy (J, a_hat and J's gradient); the float32 numpy statements of the kernels (the loss and the dense
upstream gradient G, every operation rounded on its own; the means are oracle.cql.means_f32); the demonstration priority
bonus on top of oracle.sumtree; and a torch-fp32 learner step on losses.iqn_loss / value_rescaling.iqn_loss / qr.qr_loss
with a per-row mask, whose gradients come from autograd.
"""
import numpy as np
import torch

from . import losses, qr as oq, value_rescaling as vr
from .cql import means_f32

F32 = np.float32


# ------------------------------------------------------------------------------------------------ float64 statements
def margin_from_means_np(Q, actions, margin):
    """(J (B,), a_hat (B,)) from the action values Q (B, A): v = Q + l off a_E, a_hat the first maximum of v."""
    Q = np.asarray(Q, np.float64)
    rows, act = np.arange(Q.shape[0]), np.asarray(actions)
    v = Q + margin
    v[rows, act] = Q[rows, act]
    a_hat = np.argmax(v, 1)                      # the first of equal maxima
    return v[rows, a_hat] - Q[rows, act], a_hat


def margin_np(q, batch, actions, margin):
    """J (B,) and a_hat (B,) of the quantile values q (N*B, A), Q the float64 mean."""
    q = np.asarray(q, np.float64)
    return margin_from_means_np(q.reshape(-1, batch, q.shape[1]).mean(0), actions, margin)


def margin_grad_np(q, batch, actions, margin):
    """dJ[b] / dq (N*B, A): (1{a = a_hat} - 1{a = a_E}) / N on every row i*B + b (zero when a_hat = a_E)."""
    q = np.asarray(q, np.float64)
    n, A = q.shape[0] // batch, q.shape[1]
    _, a_hat = margin_np(q, batch, actions, margin)
    d = np.zeros((batch, A))
    d[np.arange(batch), a_hat] += 1.0
    d[np.arange(batch), np.asarray(actions)] -= 1.0
    return np.tile(d / n, (n, 1))


# ------------------------------------------------------------------------------------------------ float32 statements
def margin_f32(q, batch, actions, margin):
    """(Q (B, A), J (B,), a_hat (B,)) as the kernel forms them: v_a = fl(Q_a + l) off a_E, the first maximum, and
    J = fl(M - Q_{a_E})."""
    Q = means_f32(q, batch)
    rows, act = np.arange(batch), np.asarray(actions)
    v = (Q + F32(margin)).astype(F32)
    v[rows, act] = Q[rows, act]
    a_hat = np.argmax(v, 1)
    return Q, (v[rows, a_hat] - Q[rows, act]).astype(F32), a_hat


def loss_f32(td, J, lam, demo):
    """fl(td + fl(lambda * J)) on the flagged rows, td on the others."""
    td = np.asarray(td, F32)
    with_margin = (td + (F32(lam) * np.asarray(J, F32)).astype(F32)).astype(F32)
    return np.where(np.asarray(demo) != 0, with_margin, td)


def dense_grad_f32(dtheta, a_hat, actions, demo, gscale, gscale_mul, lam, n, A):
    """G (n*B, A), zero off the named columns: w_b = fl(gscale[b] * gscale_mul), c = fl(lambda / n); fl(w_b * dtheta) on
    a_E where demo[b] == 0 or a_hat = a_E, else fl(w_b * c) on a_hat and fl(w_b * fl(dtheta - c)) on a_E."""
    dtheta = np.asarray(dtheta, F32)
    act, a_hat = np.asarray(actions), np.asarray(a_hat)
    B = act.shape[0]
    w = (np.asarray(gscale, F32) * F32(gscale_mul)).astype(F32)
    c = (F32(lam) / F32(n)).astype(F32)
    rows = np.arange(n * B)
    b = rows % B
    ae, ah = act[b], a_hat[b]
    two = (np.asarray(demo)[b] != 0) & (ah != ae)
    G = np.zeros((n * B, A), F32)
    G[rows, ae] = np.where(two, (w[b] * (dtheta - c).astype(F32)).astype(F32), (w[b] * dtheta).astype(F32))
    G[rows[two], ah[two]] = (w[b[two]] * c).astype(F32)
    return G


# ------------------------------------------------------------------------------------------------ replay
def bonus_priorities(loss, tree_idx, exponent, demo_leaf, bonus):
    """The priorities riqn_sumtree_update_demo writes: p = fl32(loss ** omega) correctly rounded (double pow, one
    rounding), then fl32(p + eps_d) on the leaves tree_idx >= demo_leaf."""
    p = np.power(np.asarray(loss, F32).astype(np.float64), np.float64(F32(exponent))).astype(F32)
    on = np.asarray(tree_idx) >= demo_leaf
    return np.where(on, (p + F32(bonus)).astype(F32), p)


def update_priorities_demo(tree, idxs, loss, exponent, demo_leaf, bonus):
    """oracle.sumtree.SumTree.update_multiple_value on the bonus priorities (duplicates keep the reference's old-leaf
    semantics: every entry's diff is taken against the leaf before the batch).  Returns the priorities."""
    p = bonus_priorities(loss, idxs, exponent, demo_leaf, bonus)
    tree.update_multiple_value(np.asarray(idxs, np.int64), p.astype(np.float64))
    return p


# ------------------------------------------------------------------------------------------------ torch fp32 step
def margin_torch(q_on, n, batch, actions, margin):
    Q = q_on.reshape(n, batch, -1).mean(0)
    off = torch.ones_like(Q)
    off[torch.arange(batch), actions] = 0.0
    return (Q + margin * off).max(1).values - Q[torch.arange(batch), actions]


def dqfd_loss(kind, p_online, p_target, batch, noises, taus, cfg, margin, lam, demo, eps=None, keep=None):
    """The DQfD loss (B,) on the IQN (``kind`` "iqn", taus injected) or QR-DQN ("qr") double-DQN step with the (B,) 0/1
    mask ``demo``, with keep["td"] and keep["J"]; keep["qv_next"] holds the values a* was chosen on."""
    keep = {} if keep is None else keep
    states, actions, returns, next_states, nonterminals = batch
    B = states.shape[0]
    sizes = dict(discount=cfg["discount"], n_step=cfg["n_step"], kappa=cfg["kappa"])
    n = cfg["n_tau"]
    if kind == "qr":
        td = oq.qr_loss(p_online, p_target, *batch, noises, n=n, eps=eps, keep=keep, **sizes)
    else:
        kw = dict(n_tau=n, n_tau_prime=cfg["n_tau_prime"], n_quantile=cfg["n_quantile"], **sizes)
        if eps is None:
            td = losses.iqn_loss(p_online, p_target, *batch, noises, taus, keep=keep, **kw)
            keep["qv_next"] = keep["q_sel"].reshape(cfg["n_quantile"], B, -1).mean(0)
        else:
            td = vr.iqn_loss(p_online, p_target, *batch, noises, taus, eps=eps, keep=keep, **kw)
    J = margin_torch(keep["q_on"], n, B, actions, margin)
    keep.update(td=td.detach(), J=J.detach())
    return td + lam * torch.as_tensor(demo, dtype=torch.float32) * J


def learn_step(kind, p_online, p_target, batch, weights, noises, taus, cfg, margin, lam, demo, eps=None, keep=None):
    """Loss (B,) and the gradients of (weights * loss).mean() by autograd (no optimiser step)."""
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = dqfd_loss(kind, p_online, p_target, batch, noises, taus, cfg, margin, lam, demo, eps, keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    return loss.detach(), grads
