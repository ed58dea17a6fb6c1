"""Oracle (test infrastructure): FQF's fractions, its 1-Wasserstein fraction gradient and a whole FQF learner step.

Yang, Zhao, Lin, Qin, Bian & Liu, "Fully Parameterized Quantile Function for Distributional Reinforcement Learning",
NeurIPS 2019.  Per transition b, with logits l = psi(s) W_f^T + b_f over N fractions:

  P = softmax(l) ,  tau_0 = 0, tau_i = sum_{k<i} P_k, tau_N = 1 ,  tau_hat_i = (tau_i + tau_{i+1}) / 2 ,
  dtau_i = tau_{i+1} - tau_i ,  Q(s, a) = sum_i dtau_i F(s, tau_hat_i, a)

The fraction loss is the 1-Wasserstein distance W1 between the quantile function F and its step approximation
F(tau_hat_i) on [tau_i, tau_{i+1}).  With F increasing, its gradient is exact (the paper's Proposition 1):

  g_i = dW1/dtau_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1})            i = 1..N-1

and the fraction network trains on the surrogate L_f = sum_i g_i tau_i - lambda H(P) with g detached (the quantile values
carry no gradient into the fractions), whose logit gradient is
  dL/dP_k = G_k = sum_{i>k} g_i ,  dL/dl_k = P_k (G_k - sum_m P_m G_m) + lambda P_k (log P_k + H).

The learner step follows the paper's Algorithm 1 as the public implementations read it: the fractions of s' (from the
online proposal) select a* = argmax_a sum_i dtau'_i F_online(s', tau_hat'_i, a); the TARGET network is evaluated on s' at
the tau_hat of s; the quantile-Huber loss pairs F_online(s, tau_hat_i, a_t) with those N targets; the fraction loss reads
the online network at tau_hat and at the inner boundaries tau_1..tau_{N-1} with the same noise sample.

The reference has no FQF, so there is no golden fixture: tests pin this module by identities (uniform fractions at zero
logits, Proposition 1 against quadrature, the analytic backward against autograd) and by the agreement of the float64 and
torch-fp32 statements.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import losses, network as net


# ------------------------------------------------------------------------------------------------ float64 statements
def fractions_np(logits):
    """logits (B, N) -> dict(P (B, N), tau (B, N+1), tau_hat (B, N), dtau (B, N), entropy (B,)), float64."""
    lg = np.asarray(logits, np.float64)
    d = lg - lg.max(axis=1, keepdims=True)
    e = np.exp(d)
    S = e.sum(axis=1, keepdims=True)
    P = e / S
    B, N = lg.shape
    tau = np.zeros((B, N + 1))
    tau[:, 1:] = np.cumsum(P, axis=1)
    tau[:, N] = 1.0
    logP = d - np.log(S)
    return dict(P=P, tau=tau, tau_hat=0.5 * (tau[:, :-1] + tau[:, 1:]), dtau=tau[:, 1:] - tau[:, :-1],
                entropy=-(P * logP).sum(axis=1), logP=logP)


def w1_grad_np(f_bnd, f_hat):
    """g (B, N-1) from F at the inner boundaries f_bnd (B, N-1) and at the midpoints f_hat (B, N)."""
    f_bnd, f_hat = np.asarray(f_bnd, np.float64), np.asarray(f_hat, np.float64)
    return 2.0 * f_bnd - f_hat[:, 1:] - f_hat[:, :-1]


def fraction_bwd_np(logits, f_bnd, f_hat, weight, entropy_coef, tau=None):
    """The fraction loss's backward in float64.  ``tau`` (B, N+1): the fractions the surrogate is evaluated at
    (default: this module's own).  Returns (dlogits (B, N) weighted by ``weight`` (B,), loss (B,) unweighted)."""
    fr = fractions_np(logits)
    tau = fr["tau"] if tau is None else np.asarray(tau, np.float64)
    g = w1_grad_np(f_bnd, f_hat)                                     # (B, N-1): g_1..g_{N-1}
    B, N = fr["P"].shape
    G = np.zeros((B, N))
    G[:, :-1] = np.cumsum(g[:, ::-1], axis=1)[:, ::-1]              # G_k = sum_{i>k} g_i = g_{k+1} + ... + g_{N-1}
    P, H = fr["P"], fr["entropy"]
    d = P * (G - (P * G).sum(axis=1, keepdims=True)) + entropy_coef * P * (fr["logP"] + H[:, None])
    loss = (g * tau[:, 1:N]).sum(axis=1) - entropy_coef * H
    return np.asarray(weight, np.float64)[:, None] * d, loss


def w1_np(quantile_fn, tau):
    """W1 between the quantile function ``quantile_fn`` on [0, 1] and its step approximation at the midpoints of the
    fractions ``tau`` (N+1,), by adaptive quadrature in float64 (each piece split at its kink tau_hat_i)."""
    from scipy import integrate
    total = 0.0
    for lo, hi in zip(tau[:-1], tau[1:]):
        m = 0.5 * (lo + hi)
        c = quantile_fn(m)
        for a, b in ((lo, m), (m, hi)):
            if b > a:
                v, _ = integrate.quad(lambda w: abs(quantile_fn(w) - c), a, b, epsabs=1e-15, epsrel=1e-13, limit=200)
                total += v
    return total


# ------------------------------------------------------------------------------------------------ torch fp32 step
def fractions_torch(logits):
    """The fractions in torch (differentiable w.r.t. the logits).  Returns tau (B, N+1), tau_hat (B, N), dtau (B, N),
    entropy (B,)."""
    P = torch.softmax(logits, dim=1)
    logP = torch.log_softmax(logits, dim=1)
    B = logits.shape[0]
    c = torch.cumsum(P, dim=1)
    tau = torch.cat((torch.zeros(B, 1, dtype=logits.dtype), c[:, :-1], torch.ones(B, 1, dtype=logits.dtype)), dim=1)
    return tau, 0.5 * (tau[:, :-1] + tau[:, 1:]), tau[:, 1:] - tau[:, :-1], -(P * logP).sum(dim=1)


def _qmajor(t):
    """(B, N) -> (N*B, 1), row i*B + b."""
    return t.t().reshape(-1, 1).contiguous()


def fqf_step(p_online, p_target, w_f, b_f, batch, weights, noises, cfg, entropy_coef=0.0, keep=None):
    """One FQF learner step's loss and gradients in torch fp32 with injected noises (n0, n1, n2).  ``w_f`` / ``b_f``
    (leaf tensors requiring grad) are the fraction proposal.  The DQN gradients come from (weights * loss).mean(), the
    fraction gradients from (weights * L_f).mean() with the quantile values detached.  Returns (loss (B,),
    fraction loss (B,), DQN grads dict, (dW_f, db_f))."""
    states, actions, returns, next_states, nonterminals = batch
    B, N = states.shape[0], cfg["n_tau"]
    for t in list(p_online.values()) + [w_f, b_f]:
        if t.requires_grad and t.grad is not None:
            t.grad = None
    with torch.no_grad():
        net.apply_noise(p_online, noises[0])
        feat_n = net.conv_trunk(p_online, next_states)
        _, th_n, dt_n, _ = fractions_torch(F.linear(feat_n, w_f, b_f))
        q_sel = net.dqn_forward_iqn(p_online, next_states, N, _qmajor(th_n))
        A = q_sel.shape[1]
        qv = (q_sel.view(N, B, A) * dt_n.t()[:, :, None]).sum(0)
        a_star = qv.argmax(1)
        feat = net.conv_trunk(p_online, states)
    logits = F.linear(feat, w_f, b_f)
    tau, tau_hat, dtau, H = fractions_torch(logits)
    th = tau_hat.detach()
    with torch.no_grad():
        net.apply_noise(p_target, noises[1])
        q_tgt = net.dqn_forward_iqn(p_target, next_states, N, _qmajor(th))
        z = q_tgt.gather(1, a_star.repeat(N)[:, None]).reshape(N, B).t()
        target = returns[:, None] + (cfg["discount"] ** cfg["n_step"]) * nonterminals[:, None] * z
    net.apply_noise(p_online, noises[2])
    q_on = net.dqn_forward_iqn(p_online, states, N, _qmajor(th), keep=keep)
    theta = q_on.gather(1, actions[:, None].repeat(N, 1)).reshape(N, B).t()
    loss = losses.iqn_pairwise_loss(theta, target, th, cfg["kappa"])
    with torch.no_grad():
        q_bnd = net.dqn_forward_iqn(p_online, states, N - 1, _qmajor(tau[:, 1:N].detach()))
        f_bnd = q_bnd.gather(1, actions[:, None].repeat(N - 1, 1)).reshape(N - 1, B).t()
        f_hat = theta.detach()
        g = 2.0 * f_bnd - f_hat[:, 1:] - f_hat[:, :-1]
    floss = (g * tau[:, 1:N]).sum(dim=1) - entropy_coef * H
    ((weights * loss).mean() + (weights * floss).mean()).backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    if keep is not None:
        keep.update(a_star=a_star, q_sel=q_sel, q_tgt=q_tgt, q_bnd=q_bnd, logits=logits.detach(), tau=tau.detach(),
                    tau_hat=th, dtau=dtau.detach(), target=target, theta=theta.detach(), g=g, qv_next=qv)
    return loss.detach(), floss.detach(), grads, (w_f.grad.detach().clone(), b_f.grad.detach().clone())


def act_values(p_online, w_f, b_f, states, n_tau, training=True):
    """(E, A) FQF action values sum_i dtau_i F(s, tau_hat_i, a) of the online network (noise as currently applied, or
    the mu weights alone when not ``training``)."""
    with torch.no_grad():
        feat = net.conv_trunk(p_online, states)
        _, th, dt, _ = fractions_torch(F.linear(feat, w_f, b_f))
        q = net.dqn_forward_iqn(p_online, states, n_tau, _qmajor(th), training=training)
        E, A = states.shape[0], q.shape[1]
        return (q.view(n_tau, E, A) * dt.t()[:, :, None]).sum(0)
