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
import math
import numbers

from ._lib import call, ptr

MMD_DEFAULTS = {"mmd_bandwidths": tuple(float(h) for h in range(1, 11))}
MAX_BANDWIDTHS = 16
_LOG2E = 1.4426950408889634


def _f32(x):
    return ctypes.c_float(x).value


def check_mmd(mmd, bandwidths=MMD_DEFAULTS["mmd_bandwidths"], qr_dqn=None, rainbow_only=False, munchausen=None,
              fqf=None, risk=None):
    """Validate an MMDQN configuration.  Returns None when ``mmd`` is off (0 / False), else ``bandwidths`` as a tuple of
    floats: a sequence (not a string) of 1..16 real numbers, each finite and > 0 as the float32 the kernel receives, with
    the kernel's constants log2(e)/h and 2/h finite in float32.  MMDQN trains the QR-DQN network, so it needs ``qr_dqn``
    (N, as qr.check_qr returns it, not None) and inherits QR-DQN's exclusions: ``rainbow_only``, Munchausen targets
    (``munchausen`` not None), FQF (``fqf`` not None) and a risk measure (``risk`` not None).  Raises ValueError
    otherwise."""
    if isinstance(mmd, bool) or (isinstance(mmd, numbers.Integral) and mmd in (0, 1)):
        if not mmd:
            return None
    else:
        raise ValueError(f"mmd must be 0 or 1, got {mmd!r}")
    if isinstance(bandwidths, (str, bytes)):
        raise ValueError(f"mmd_bandwidths must be a sequence of numbers, not a string: {bandwidths!r}")
    try:
        vals = tuple(bandwidths)
    except TypeError:
        raise ValueError(f"mmd_bandwidths must be a sequence of numbers, got {bandwidths!r}") from None
    if not 1 <= len(vals) <= MAX_BANDWIDTHS:
        raise ValueError(f"mmd_bandwidths needs 1..{MAX_BANDWIDTHS} bandwidths, got {len(vals)}")
    for v in vals:
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError(f"each of mmd_bandwidths must be a real number, got {v!r}")
        f = _f32(v)
        if not (math.isfinite(f) and f > 0.0 and math.isfinite(_f32(_LOG2E / f)) and math.isfinite(_f32(2.0 / f))):
            raise ValueError(f"each of mmd_bandwidths must be finite and > 0 (as a float32, with 2/h finite), got {v!r}")
    if qr_dqn is None:
        raise ValueError("mmd trains the QR-DQN network's particles: set qr_dqn = 1 as well")
    if rainbow_only:
        raise ValueError("mmd trains the QR-DQN head, and rainbow_only selects the C51 head: set one of them")
    if munchausen is not None:
        raise ValueError("MMDQN and Munchausen targets do not combine: set munchausen = 0 or mmd = 0")
    if fqf is not None:
        raise ValueError("MMDQN has no fractions for FQF to learn: set fqf = 0 or mmd = 0")
    if risk is not None:
        raise ValueError("MMDQN's particles carry no quantile fractions for a risk measure to distort; use the neutral "
                         "measure")
    return tuple(float(v) for v in vals)


def mmd_loss(agent, B, N, q_on, q_tgt, actions, a_star, returns, nonterminals, loss, dtheta, theta_out, target_out):
    """The double-DQN MMD loss kernel over the bandwidths ``agent.mmd``: riqn_mmd_loss_fwd_bwd, or against the
    transformed target h(R + gamma^n nt h^-1(Z)) under value rescaling (riqn_mmd_loss_fwd_bwd_h)."""
    bw = agent.mmd
    hb = (ctypes.c_float * len(bw))(*bw)      # read by the call: a captured graph holds the values
    args = (ptr(q_on), ptr(q_tgt), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals),
            float(agent.discount ** agent.n), len(bw), hb)
    outs = (ptr(loss), ptr(dtheta), ptr(theta_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_mmd_loss_fwd_bwd", B, N, agent.action_space, *args, *outs)
    else:
        call("riqn_mmd_loss_fwd_bwd_h", B, N, agent.action_space, *args, eps, *outs)
