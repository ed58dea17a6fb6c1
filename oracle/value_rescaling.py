"""Oracle (test infrastructure): value-function rescaling, the transformed Bellman operator of Pohlen et al. 2018
("Observe and Look Further: Achieving Consistent Performance on Atari", the Ape-DQfD agent; kept by R2D2):

  h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x          (odd, strictly increasing, h(0) = 0)
  T_j  = h(R + gamma^n nt h^-1(Z_j(s', a*)))

The network's outputs live in h-space.  x -> h(R + gamma^n nt h^-1(x)) is non-decreasing, so it maps the tau-quantile of
Z' to the tau-quantile of the transformed target: sample by sample it is the exact operator for IQN and FQF, and for C51
it moves the atoms before the projection.  Actions (a* in every loss and the actors' greedy actions) maximise the
expected return on the original scale, E[h^-1(Z)].

The float64 statements use cancellation-free forms (every term non-negative), in the operation order the kernels round
them in (rainbow_iqn_apex_b200/csrc/value_rescaling.cuh), so that each fp32 value the kernels store has a numpy statement
here it must equal bit for bit:

  h(x):     a = |x|;  m = a / (sqrt(a + 1) + 1);  h = copysign(m, x) + eps x
  h^-1(y):  a = |y|;  u = (a + 1) + eps;  s = sqrt(1 + (4 eps) u);  d = ((4u) a) / (((2u - 1) + s) (s + 1));
            h^-1 = copysign(d (d + 2), y)

The torch statements of the IQN, FQF and C51 learner steps restate oracle/losses.py and oracle/fqf.py with the transform.
The reference has no value rescaling, so there is no golden fixture: tests pin this module by identities (h(0) = 0, odd,
increasing, round trips, the eps = 0 closed forms, the textbook inverse, the monotone-map property).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import fqf as ofqf, losses, network as net


# ------------------------------------------------------------------------------------------------ float64 statements
def _eps64(eps):
    """eps as the kernels receive it: a float32 widened to double."""
    return float(np.float32(eps))


def h_np(x, eps):
    x = np.asarray(x, np.float64)
    eps = _eps64(eps)
    a = np.abs(x)
    m = a / (np.sqrt(a + 1.0) + 1.0)
    return np.copysign(m, x) + eps * x


def h_inv_np(y, eps):
    y = np.asarray(y, np.float64)
    eps = _eps64(eps)
    a = np.abs(y)
    u = (a + 1.0) + eps
    s = np.sqrt(1.0 + (4.0 * eps) * u)
    d = ((4.0 * u) * a) / ((((2.0 * u) - 1.0) + s) * (s + 1.0))
    return np.copysign(d * (d + 2.0), y)


def h_inv_textbook_np(y, eps):
    """sign(y) (((sqrt(1 + 4 eps (|y| + 1 + eps)) - 1) / (2 eps))^2 - 1), eps > 0: cancels catastrophically near 0."""
    y = np.asarray(y, np.float64)
    eps = _eps64(eps)
    return np.sign(y) * (((np.sqrt(1.0 + 4.0 * eps * (np.abs(y) + 1.0 + eps)) - 1.0) / (2.0 * eps)) ** 2 - 1.0)


def _g32(nonterminals, gamma_n):
    """g = fl32(gamma_n * nt), both float32, as the loss kernels form it."""
    return (np.asarray(nonterminals, np.float32) * np.float32(gamma_n)).astype(np.float32)


def target_np(z, returns, nonterminals, gamma_n, eps):
    """The IQN / FQF targets the kernel stores: z (B, N') fp32 target quantiles at a* -> fl32(h(R + g h^-1(z))), with the
    sum and the product in double."""
    g = _g32(nonterminals, gamma_n).astype(np.float64)[:, None]
    r = np.asarray(returns, np.float32).astype(np.float64)[:, None]
    return h_np(r + g * h_inv_np(z, eps), eps).astype(np.float32)


def c51_atoms_np(support, returns, nonterminals, gamma_n, eps):
    """The moved atoms tz (B, atoms) fp32 = fl32(h(R + g h^-1(support_j))), before the clamp."""
    return target_np(np.asarray(support, np.float32)[None, :], returns, nonterminals, gamma_n, eps)


def expected_np(q, batch, eps, w=None):
    """values (B, A) fp32 of h-space quantile values q (n*B, A), quantile-major: fl32(sum_k w_k h^-1(q_k)) or, w None,
    fl32((sum_k h^-1(q_k)) / n), summed in double with k ascending."""
    q = np.asarray(q, np.float32)
    n = q.shape[0] // batch
    z = h_inv_np(q.reshape(n, batch, -1), eps)
    acc = np.zeros(z.shape[1:])
    for k in range(n):
        acc = acc + (z[k] if w is None else np.asarray(w, np.float32).reshape(n, batch)[k][:, None].astype(np.float64) * z[k])
    return (acc if w is not None else acc / n).astype(np.float32)


def argmax_first(values):
    """argmax along axis 1 with the first maximal index winning (np.argmax does)."""
    return np.argmax(np.asarray(values), axis=1)


# ------------------------------------------------------------------------------------------------ torch fp32 steps
def h_torch(x, eps):
    """h of a float32 tensor, evaluated in float64 and rounded once (no gradient flows through the targets)."""
    return torch.from_numpy(h_np(x.detach().double().numpy(), eps)).to(x.dtype)


def h_inv_torch(y, eps):
    return torch.from_numpy(h_inv_np(y.detach().double().numpy(), eps)).to(y.dtype)


def _mean_h_inv(q, n, batch, eps, w=None):
    """(B, A) expected return on the original scale of q (n*B, A): mean_k h^-1(q_k), or sum_k w_k h^-1(q_k)."""
    z = h_inv_torch(q, eps).view(n, batch, -1)
    return z.mean(0) if w is None else (z * w.view(n, batch, 1)).sum(0)


def iqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, taus, *, eps, n_tau,
             n_tau_prime, n_quantile, discount=0.99, n_step=3, kappa=1.0, keep=None):
    """losses.iqn_loss under value rescaling: a* = argmax_a mean_k h^-1(Z_k(s', a)) and T_j = h(R + gamma^n nt
    h^-1(Z_j(s', a*)))."""
    batch = states.shape[0]
    with torch.no_grad():
        net.apply_noise(p_online, noises[0])
        q_sel = net.dqn_forward_iqn(p_online, next_states, n_quantile, taus[0])
        qv = _mean_h_inv(q_sel, n_quantile, batch, eps)
        a_star = qv.argmax(dim=1)
        net.apply_noise(p_target, noises[1])
        q_tgt = net.dqn_forward_iqn(p_target, next_states, n_tau_prime, taus[1])
        z = q_tgt.gather(1, a_star[:, None].repeat(n_tau_prime, 1)).reshape(n_tau_prime, batch).t()
        target = h_torch(returns[:, None] + (discount ** n_step) * nonterminals[:, None] * h_inv_torch(z, eps), eps)
    net.apply_noise(p_online, noises[2])
    q_on = net.dqn_forward_iqn(p_online, states, n_tau, taus[2], keep=keep)
    theta = q_on.gather(1, actions[:, None].repeat(n_tau, 1)).reshape(n_tau, batch).t()
    loss = losses.iqn_pairwise_loss(theta, target, taus[2].reshape(n_tau, batch).t(), kappa)
    if keep is not None:
        keep.update(a_star=a_star, target=target, theta=theta, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, qv_next=qv)
    return loss


def c51_projection(pns_a, tz, *, atoms, v_min, v_max):
    """losses.c51_projection of given (moved) atoms tz (batch, atoms), with the same index clamp."""
    batch = pns_a.shape[0]
    delta_z = (v_max - v_min) / (atoms - 1)
    tz = tz.clamp(min=v_min, max=v_max)
    b = ((tz - v_min) / delta_z).clamp(max=atoms - 1)
    lo, up = b.floor().to(torch.int64), b.ceil().to(torch.int64)
    lo[(up > 0) * (lo == up)] -= 1
    up[(lo < (atoms - 1)) * (lo == up)] += 1
    m = pns_a.new_zeros(batch, atoms)
    offset = (torch.arange(batch) * atoms)[:, None].expand(batch, atoms)
    m.view(-1).index_add_(0, (lo + offset).view(-1), (pns_a * (up.float() - b)).view(-1))
    m.view(-1).index_add_(0, (up + offset).view(-1), (pns_a * (b - lo.float())).view(-1))
    return m


def c51_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, *, eps, atoms=51,
             v_min=-10.0, v_max=10.0, discount=0.99, n_step=3, keep=None):
    """losses.c51_loss under value rescaling: a* = argmax_a sum_j p_j h^-1(z_j) and the atoms moved to
    h(R + gamma^n nt h^-1(z_j)) before the projection."""
    batch = states.shape[0]
    acts = p_online["fcnoisy_z_a.bias_mu"].shape[0] // atoms
    support = torch.linspace(v_min, v_max, atoms)
    net.apply_noise(p_online, noises[0])
    log_ps_a = net.dqn_forward_c51(p_online, states, acts, atoms, log=True)[range(batch), actions]
    with torch.no_grad():
        net.apply_noise(p_online, noises[1])
        pns = net.dqn_forward_c51(p_online, next_states, acts, atoms)
        ev = (h_inv_torch(support, eps).expand_as(pns) * pns).sum(2)
        a_star = ev.argmax(1)
        net.apply_noise(p_target, noises[2])
        pns_a = net.dqn_forward_c51(p_target, next_states, acts, atoms)[range(batch), a_star]
        tz = h_torch(returns[:, None] + (discount ** n_step) * nonterminals[:, None] * h_inv_torch(support, eps)[None],
                     eps)
        m = c51_projection(pns_a, tz, atoms=atoms, v_min=v_min, v_max=v_max)
    loss = -(m * log_ps_a).sum(1)
    if keep is not None:
        keep.update(a_star=a_star, m=m, log_ps_a=log_ps_a, ev_next=ev)
    return loss


def learn_step(p_online, p_target, adam, batch, weights, noises, taus, cfg, eps, rainbow_only=False, keep=None):
    """losses.learn_step with the rescaled IQN or C51 loss.  Returns (loss (B,) detached, grads dict)."""
    states, actions, returns, next_states, nonterminals = batch
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    if rainbow_only:
        loss = c51_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, eps=eps, **cfg,
                        keep=keep)
    else:
        loss = iqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, taus, eps=eps,
                        **cfg, keep=keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    adam.step(p_online, grads)
    return loss.detach(), grads


def fqf_step(p_online, p_target, w_f, b_f, batch, weights, noises, cfg, eps, entropy_coef=0.0, keep=None):
    """oracle.fqf.fqf_step under value rescaling: a* = argmax_a sum_i dtau'_i h^-1(F(s', tau_hat'_i, a)), targets
    h(R + gamma^n nt h^-1(F_target)); the fraction loss stays on the h-space quantile function.  Returns (loss (B,),
    fraction loss (B,), DQN grads dict, (dW_f, db_f))."""
    states, actions, returns, next_states, nonterminals = batch
    B, N = states.shape[0], cfg["n_tau"]
    for t in list(p_online.values()) + [w_f, b_f]:
        if t.requires_grad and t.grad is not None:
            t.grad = None
    qm = ofqf._qmajor
    with torch.no_grad():
        net.apply_noise(p_online, noises[0])
        feat_n = net.conv_trunk(p_online, next_states)
        _, th_n, dt_n, _ = ofqf.fractions_torch(F.linear(feat_n, w_f, b_f))
        q_sel = net.dqn_forward_iqn(p_online, next_states, N, qm(th_n))
        qv = _mean_h_inv(q_sel, N, B, eps, w=dt_n.t().contiguous())
        a_star = qv.argmax(1)
        feat = net.conv_trunk(p_online, states)
    logits = F.linear(feat, w_f, b_f)
    tau, tau_hat, dtau, H = ofqf.fractions_torch(logits)
    th = tau_hat.detach()
    with torch.no_grad():
        net.apply_noise(p_target, noises[1])
        q_tgt = net.dqn_forward_iqn(p_target, next_states, N, qm(th))
        z = q_tgt.gather(1, a_star.repeat(N)[:, None]).reshape(N, B).t()
        target = h_torch(returns[:, None] + (cfg["discount"] ** cfg["n_step"]) * nonterminals[:, None] *
                         h_inv_torch(z, eps), eps)
    net.apply_noise(p_online, noises[2])
    q_on = net.dqn_forward_iqn(p_online, states, N, qm(th), keep=keep)
    theta = q_on.gather(1, actions[:, None].repeat(N, 1)).reshape(N, B).t()
    loss = losses.iqn_pairwise_loss(theta, target, th, cfg["kappa"])
    with torch.no_grad():
        q_bnd = net.dqn_forward_iqn(p_online, states, N - 1, qm(tau[:, 1:N].detach()))
        f_bnd = q_bnd.gather(1, actions[:, None].repeat(N - 1, 1)).reshape(N - 1, B).t()
        f_hat = theta.detach()
        g = 2.0 * f_bnd - f_hat[:, 1:] - f_hat[:, :-1]
    floss = (g * tau[:, 1:N]).sum(dim=1) - entropy_coef * H
    ((weights * loss).mean() + (weights * floss).mean()).backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    if keep is not None:
        keep.update(a_star=a_star, q_sel=q_sel, q_tgt=q_tgt, target=target, theta=theta.detach(), qv_next=qv)
    return loss.detach(), floss.detach(), grads, (w_f.grad.detach().clone(), b_f.grad.detach().clone())


def act_values(p_online, states, n, taus, eps, training=True, w_f=None, b_f=None):
    """(E, A) original-scale action values of the online network: mean_k h^-1(Z_{tau_k}) at the given fractions (IQN),
    or with the FQF proposal (w_f, b_f) sum_i dtau_i h^-1(F(s, tau_hat_i))."""
    with torch.no_grad():
        E = states.shape[0]
        if w_f is None:
            q = net.dqn_forward_iqn(p_online, states, n, taus, training=training)
            return _mean_h_inv(q, n, E, eps)
        feat = net.conv_trunk(p_online, states)
        _, th, dt, _ = ofqf.fractions_torch(F.linear(feat, w_f, b_f))
        q = net.dqn_forward_iqn(p_online, states, n, ofqf._qmajor(th), training=training)
        return _mean_h_inv(q, n, E, eps, w=dt.t().contiguous())
