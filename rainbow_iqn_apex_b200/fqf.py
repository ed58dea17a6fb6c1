"""FQF, the Fully parameterized Quantile Function (Yang, Zhao, Lin, Qin, Bian & Liu, NeurIPS 2019).

FQF keeps IQN's quantile-value network (model.DQN) and replaces its uniformly drawn fractions by N per-state fractions
from a small *fraction proposal network* on the detached trunk features psi(s):

  logits = psi(s) W_f^T + b_f ,  P = softmax(logits) ,  tau_0 = 0, tau_i = sum_{k<i} P_k, tau_N = 1
  tau_hat_i = (tau_i + tau_{i+1}) / 2 ,  dtau_i = tau_{i+1} - tau_i ,  Q(s, a) = sum_i dtau_i F(s, tau_hat_i, a)

The proposal is trained on the exact gradient of the 1-Wasserstein distance between the quantile function and its
N-step approximation (the paper's Proposition 1), minus an optional entropy bonus; see riqn_fqf_fraction_bwd.

FractionProposal holds W_f (N, 3136) and b_f (N) in its own flat parameter / gradient arena, beside the DQN's: the DQN's
arena, parameter order and state_dict stay those of the reference.  It lives on the Agent (agent.fraction_net, trained
by agent.fraction_optimiser, the arena Adam; the paper used RMSProp).  There is no target copy: fractions always come
from the online proposal.
"""
import ctypes
import math
import numbers
import weakref

import torch
from torch import nn

from ._lib import call, ptr
from .model import FEAT, _ALIGN

FQF_DEFAULTS = {"fqf_fraction_lr": 2.5e-9, "fqf_entropy_coef": 0.0}   # the public FQF Atari configurations' rate
MAX_FRACTIONS = 256


def check_fqf(fqf, fraction_lr=2.5e-9, entropy_coef=0.0, rainbow_only=False, munchausen=None, risk=None,
              num_tau_samples=None):
    """Validate an FQF configuration.  Returns None when ``fqf`` is off (0 / False), else ``(fraction_lr,
    entropy_coef)``: fraction_lr > 0 and entropy_coef >= 0, both finite as float32.  FQF is IQN-only (not
    ``rainbow_only``), does not combine with Munchausen targets (``munchausen`` must be None) and is risk-neutral (``risk``
    must be None); ``num_tau_samples`` (N) must lie in 2..256.  Raises ValueError otherwise."""
    if isinstance(fqf, bool) or (isinstance(fqf, numbers.Integral) and fqf in (0, 1)):
        if not fqf:
            return None
    else:
        raise ValueError(f"fqf must be 0 or 1, got {fqf!r}")
    vals = []
    for name, v, ok, need in (("fqf_fraction_lr", fraction_lr, lambda x: x > 0.0, "> 0"),
                              ("fqf_entropy_coef", entropy_coef, lambda x: x >= 0.0, ">= 0")):
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError(f"{name} must be a real number, got {v!r}")
        f = ctypes.c_float(v).value
        if not (math.isfinite(f) and ok(f)):
            raise ValueError(f"{name} must be finite and {need} (as a float32), got {v!r}")
        vals.append(float(v))
    if rainbow_only:
        raise ValueError("FQF proposes quantile fractions for the IQN head; rainbow_only (C51) has none")
    if munchausen is not None:
        raise ValueError("FQF and Munchausen targets do not combine: set munchausen = 0 or fqf = 0")
    if risk is not None:
        raise ValueError("FQF acts on its proposed fractions: a risk measure has no fractions to distort; use the neutral "
                         "measure")
    if num_tau_samples is not None and (isinstance(num_tau_samples, bool) or not isinstance(num_tau_samples, numbers.Integral)
                                        or not 2 <= num_tau_samples <= MAX_FRACTIONS):
        raise ValueError(f"FQF needs num_tau_samples in 2..{MAX_FRACTIONS}, got {num_tau_samples!r}")
    return tuple(vals)


class FractionProposal(nn.Module):
    """The fraction proposal network: one linear layer ``weight`` (N, 3136), ``bias`` (N), views of one flat fp32 arena
    (``_flat``; gradients in ``_flat_grad``) that the arena Adam steps and data parallelism reduces in one piece.
    Xavier-uniform weights with gain 0.01 and a zero bias: the starting fractions are nearly uniform."""

    def __init__(self, num_fractions, device, feat_dim=FEAT):
        super().__init__()
        self.num_fractions, self.feat_dim = int(num_fractions), int(feat_dim)
        self.weight = nn.Parameter(torch.empty(self.num_fractions, self.feat_dim))
        self.bias = nn.Parameter(torch.zeros(self.num_fractions))
        nn.init.xavier_uniform_(self.weight.data, gain=0.01)
        self._flatten(torch.device(device))

    def _flatten(self, dev):
        nw = self.weight.numel()
        boff = (nw + _ALIGN - 1) // _ALIGN * _ALIGN
        total = (boff + self.bias.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        flat_grad = torch.zeros(total, device=dev, dtype=torch.float32)
        for p, off in ((self.weight, 0), (self.bias, boff)):
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1).float())
            p.data = flat[off:off + n].view(p.shape)
            p.grad = flat_grad[off:off + n].view(p.shape)
            p._riqn_owner = weakref.ref(self)
            p._riqn_offset = off
        self._flat, self._flat_grad = flat, flat_grad

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._flatten(self.weight.device)
        return out

    def _params_changed(self):
        """Called by the arena Adam after a step: nothing is cached from these weights."""

    def grad_view(self, p):
        return self._flat_grad[p._riqn_offset:p._riqn_offset + p.numel()].view(p.shape)

    def zero_grad(self, set_to_none=False):
        """One memset over the gradient arena; the .grad views stay bound."""
        if self._flat_grad.is_cuda:
            call("riqn_zero_f32", ptr(self._flat_grad), self._flat_grad.numel())
        else:
            self._flat_grad.zero_()
        for p in (self.weight, self.bias):
            p.grad = self.grad_view(p)

    def propose(self, feat):
        """Fractions of the states behind ``feat`` (B, 3136) fp32 (read only; nothing flows back into the trunk).
        Returns dict(logits (B, N), tau (B, N+1), tau_hat (N*B, 1), dtau (N*B,), entropy (B,)), quantile-major rows
        r = i*B + b for tau_hat / dtau as the IQN head expects (riqn_fqf_fractions)."""
        B, N, dev = feat.shape[0], self.num_fractions, feat.device
        feat = feat if feat.is_contiguous() else feat.contiguous()
        logits = torch.empty(B, N, device=dev)
        call("riqn_linear_fwd_ld", B, self.feat_dim, N, ptr(feat), self.feat_dim, ptr(self.weight), ptr(self.bias),
             ptr(logits), N, 0)
        tau = torch.empty(B, N + 1, device=dev)
        tau_hat = torch.empty(N * B, 1, device=dev)
        dtau = torch.empty(N * B, device=dev)
        entropy = torch.empty(B, device=dev)
        call("riqn_fqf_fractions", B, N, ptr(logits), ptr(tau), ptr(tau_hat), ptr(dtau), ptr(entropy))
        return dict(logits=logits, tau=tau, tau_hat=tau_hat, dtau=dtau, entropy=entropy, feat=feat)

    def backward(self, fr, q_hat, q_bnd, actions, gscale, gscale_mul, entropy_coef):
        """Accumulate the fraction loss's gradient into the arena for the proposal ``fr`` (propose()), the gradient
        pass's quantile values ``q_hat`` at tau_hat and the boundary pass's ``q_bnd`` at tau_1..tau_{N-1}.  The surrogate
        of transition b is weighted by gscale[b] * gscale_mul, like the quantile loss.  Returns (dlogits (B, N),
        fraction loss (B,) unweighted)."""
        B, N, dev = fr["logits"].shape[0], self.num_fractions, fr["logits"].device
        dlogits = torch.empty(B, N, device=dev)
        floss = torch.empty(B, device=dev)
        call("riqn_fqf_fraction_bwd", B, N, q_hat.shape[1], ptr(fr["logits"]), ptr(fr["tau"]), ptr(q_hat), ptr(q_bnd),
             ptr(actions), ptr(gscale), float(gscale_mul), float(entropy_coef), ptr(dlogits), ptr(floss))
        call("riqn_fqf_fraction_wgrad", B, N, self.feat_dim, ptr(dlogits), ptr(fr["feat"]), ptr(self.grad_view(self.weight)),
             ptr(self.grad_view(self.bias)))
        return dlogits, floss


def q_values(q, dtau, batch, num_fractions, action_space):
    """(B, A) FQF action values sum_i dtau_i F(s, tau_hat_i, a) from a head pass ``q`` (N*B, A) at tau_hat."""
    return (q.view(num_fractions, batch, action_space) * dtau.view(num_fractions, batch, 1)).sum(0)
