"""Oracle (test infrastructure): HL-Gauss (Farebrother et al., ICML 2024; the histogram loss of Imani & White, ICML 2018)
on the C51 network.

The network, the double-DQN a* and the three noisy passes are oracle.losses.c51_loss's (oracle.value_rescaling.c51_loss
under value rescaling).  The target of transition b is a histogram over the atoms' bins: the mass that a Gaussian
N(y, sigma^2) centred on the scalar target y puts in each bin, renormalised over the support's span,

  Q'  = sum_j p_tgt[b, a*, j] s_j ,  s_j = z_j  (under value rescaling h^-1(z_j))           (j ascending)
  y   = clamp(R + g Q', v_min, v_max) ,  g = fl32(nt gamma^n)  (under value rescaling clamp(h(R + g Q'), ...))
  e_i = v_min + (i - 1/2) D ,  D = (v_max - v_min) / (atoms - 1) ,  i = 0..atoms            (the bin edges)
  u_i = (e_i - y) / s ,  s = (r D) sqrt(2) ,  c_i = erfc(|u_i|) / 2                         (the tail beyond e_i)
  mass_j = c_j - c_{j+1} (u_j >= 0) | c_{j+1} - c_j (u_{j+1} <= 0) | (1/2 - c_j) + (1/2 - c_{j+1}) (the bin holding y)
  m_j = mass_j / Z ,  Z = (1/2 - c_0) + (1/2 - c_atoms)

1 - c_j - c_{j+1} is formed as (1/2 - c_j) + (1/2 - c_{j+1}): each difference is exact where c >= 1/4 (Sterbenz), so at
a wide sigma, where c_j, c_{j+1} -> 1/2 and the bin mass and Z become small, neither loses digits to a rounded 1 - c.
  loss = -sum_j m_j log p_on[b, a, j] ,  dq_j = d loss / d logit_j = -(m_j - p_on[b, a, j] sum_k m_k)

Two statements: float64 numpy, in the operation order the kernel rounds it in (target_np is the kernel's target_out bit
for bit; the histogram needs erfc, here math.erfc), and a torch-fp32 learner step whose histogram is built in float64,
cast and detached, and whose gradients come from autograd.  There is no golden fixture (the reference has no HL-Gauss);
tests pin the statement by identities.
"""
import math

import numpy as np
import torch

from . import network as net, value_rescaling as vr

SQRT2 = 1.4142135623730951
_erfc = np.frompyfunc(math.erfc, 1, 1)


# ------------------------------------------------------------------------------------------------ float64 statements
def target_np(p_tgt_a, support, returns, nonterminals, gamma_n, v_min, v_max, eps=None):
    """The scalar targets y (B,) float64, clamped, from the target network's probabilities at a* (B, atoms) float32 and
    the float32 support (h-space under value rescaling, eps not None); fl32 of it is the kernel's target_out."""
    p = np.asarray(p_tgt_a, np.float32).astype(np.float64)
    z = np.asarray(support, np.float32).astype(np.float64)
    s = z if eps is None else vr.h_inv_np(z, eps)
    prod = p * s[None, :]
    q = np.zeros(p.shape[0])
    for j in range(p.shape[1]):
        q = q + prod[:, j]
    g = vr._g32(nonterminals, gamma_n).astype(np.float64)
    y = np.asarray(returns, np.float32).astype(np.float64) + g * q
    if eps is not None:
        y = vr.h_np(y, eps)
    return np.minimum(np.maximum(y, float(np.float32(v_min))), float(np.float32(v_max)))


def edges_np(v_min, v_max, atoms):
    """e_i (atoms + 1,) and D, from the float32 v_min, v_max widened to double."""
    lo, hi = float(np.float32(v_min)), float(np.float32(v_max))
    D = (hi - lo) / float(atoms - 1)
    return lo + (np.arange(atoms + 1, dtype=np.float64) - 0.5) * D, D


def histogram_np(y, v_min, v_max, atoms, ratio):
    """m (B, atoms) float64 of targets y (B,) (inside [v_min, v_max]) at sigma = ratio * D, ratio as a float32."""
    y = np.asarray(y, np.float64).reshape(-1)
    e, D = edges_np(v_min, v_max, atoms)
    s = (float(np.float32(ratio)) * D) * SQRT2
    u = (e[None, :] - y[:, None]) / s
    c = 0.5 * _erfc(np.abs(u)).astype(np.float64)
    cj, ck, uj, uk = c[:, :-1], c[:, 1:], u[:, :-1], u[:, 1:]
    mass = np.where(uj >= 0, cj - ck, np.where(uk <= 0, ck - cj, (0.5 - cj) + (0.5 - ck)))
    Z = (0.5 - c[:, 0]) + (0.5 - c[:, -1])
    return mass / Z[:, None]


def cross_entropy_np(m, logp_a):
    """loss (B,) and dq (B, atoms) in float64 of the target m against log-probabilities logp_a (B, atoms)."""
    m, lp = np.asarray(m, np.float64), np.asarray(logp_a, np.float64)
    return -(m * lp).sum(1), -(m - np.exp(lp) * m.sum(1, keepdims=True))


# ------------------------------------------------------------------------------------------------ torch fp32 step
def hl_gauss_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, *, ratio=0.75,
                  atoms=51, v_min=-10.0, v_max=10.0, discount=0.99, n_step=3, eps=None, keep=None):
    """The HL-Gauss double-DQN n-step loss (B,) with injected noises (online s pass, online s' pass, target pass, as
    oracle.losses.c51_loss)."""
    batch = states.shape[0]
    acts = p_online["fcnoisy_z_a.bias_mu"].shape[0] // atoms
    support = torch.linspace(v_min, v_max, atoms)
    net.apply_noise(p_online, noises[0])
    log_ps_a = net.dqn_forward_c51(p_online, states, acts, atoms, log=True)[range(batch), actions]
    with torch.no_grad():
        net.apply_noise(p_online, noises[1])
        pns = net.dqn_forward_c51(p_online, next_states, acts, atoms)
        acting = support if eps is None else vr.h_inv_torch(support, eps)
        ev = (acting.expand_as(pns) * pns).sum(2)
        a_star = ev.argmax(1)
        net.apply_noise(p_target, noises[2])
        pns_a = net.dqn_forward_c51(p_target, next_states, acts, atoms)[range(batch), a_star]
        y = target_np(pns_a.numpy(), support.numpy(), returns.numpy(), nonterminals.numpy(), discount ** n_step, v_min,
                      v_max, eps)
        m = torch.from_numpy(histogram_np(y, v_min, v_max, atoms, ratio)).float()
    loss = -(m * log_ps_a).sum(1)
    if keep is not None:
        keep.update(a_star=a_star, m=m, target=torch.from_numpy(y), log_ps_a=log_ps_a.detach(), ev_next=ev,
                    pns_a=pns_a)
    return loss


def learn_step(p_online, p_target, batch, weights, noises, cfg=None, eps=None, keep=None):
    """Loss (B,) and the gradients of (weights * loss).mean() by autograd (no optimiser step).  ``cfg``: optional
    ratio, atoms, v_min, v_max, discount, n_step."""
    states, actions, returns, next_states, nonterminals = batch
    for t in p_online.values():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    loss = hl_gauss_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, eps=eps,
                         keep=keep, **(cfg or {}))
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    return loss.detach(), grads
