"""HL-Gauss: training the C51 network by classification (Farebrother et al., "Stop Regressing: Training Value Functions
via Classification for Scalable Deep RL", ICML 2024; the histogram loss of Imani & White, ICML 2018).

HL-Gauss trains the C51 network (c51.py) with another target.  The categorical Bellman projection is replaced by the
histogram of a Gaussian N(y, sigma^2), sigma = r * delta_z, centred on the scalar double-DQN target

  y = clamp(R + gamma^n nt sum_j p_tgt(s', a*)_j z_j, v_min, v_max)      (under value rescaling: h(R + gamma^n nt E[h^-1(Z)]))

with the bins [z_j - delta_z / 2, z_j + delta_z / 2] around the atoms, renormalised over [v_min - delta_z / 2,
v_max + delta_z / 2].  The loss is the cross-entropy -sum_j m_j log p_j(s, a), one fused kernel
(riqn_hl_gauss_loss_fwd_bwd, or riqn_hl_gauss_loss_fwd_bwd_h under value rescaling) whose gradient dq the C51 head
backward takes unchanged.  Everything else is C51's: the three passes, a*, acting, the captured step graphs and
checkpoints.
"""
import ctypes
import math
import numbers

from ._lib import call, ptr

HL_GAUSS_DEFAULTS = {"hl_gauss_sigma": 0.75}
MAX_SIGMA_RATIO = 1000.0


def _f32(x):
    return ctypes.c_float(x).value


def check_hl_gauss(hl_gauss, sigma=HL_GAUSS_DEFAULTS["hl_gauss_sigma"], rainbow_only=False):
    """Validate an HL-Gauss configuration.  Returns None when ``hl_gauss`` is off (0 / False), else the ratio sigma /
    delta_z as the float32 the kernel receives: a real number (not a bool), finite, > 0 and <= 1000 in float32.  HL-Gauss
    trains the C51 head, so it needs ``rainbow_only``; that also excludes QR-DQN, MMDQN, FQF and Munchausen targets,
    which reject rainbow_only.  Raises ValueError otherwise."""
    if isinstance(hl_gauss, bool) or (isinstance(hl_gauss, numbers.Integral) and hl_gauss in (0, 1)):
        if not hl_gauss:
            return None
    else:
        raise ValueError(f"hl_gauss must be 0 or 1, got {hl_gauss!r}")
    if isinstance(sigma, bool) or not isinstance(sigma, numbers.Real):
        raise ValueError(f"hl_gauss_sigma must be a real number, got {sigma!r}")
    f = _f32(float(sigma))
    if not (math.isfinite(f) and 0.0 < f <= MAX_SIGMA_RATIO):
        raise ValueError(f"hl_gauss_sigma (sigma in bin widths) must be finite, > 0 and <= {MAX_SIGMA_RATIO:g} as a "
                         f"float32, got {sigma!r}")
    if not rainbow_only:
        raise ValueError("hl_gauss trains the C51 head's categorical output: set rainbow_only = 1 as well")
    return f


def hl_gauss_loss(agent, B, log_ps, pns, actions, a_star, returns, nonterminals, loss, dq, m_out, target_out):
    """The HL-Gauss cross-entropy at ratio ``agent.hl_gauss``: riqn_hl_gauss_loss_fwd_bwd, or the transformed target
    h(R + gamma^n nt E[h^-1(Z)]) under value rescaling (riqn_hl_gauss_loss_fwd_bwd_h)."""
    args = (ptr(log_ps), ptr(pns), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals), ptr(agent.support),
            float(agent.discount ** agent.n), float(agent.Vmin), float(agent.Vmax), agent.hl_gauss)
    outs = (ptr(loss), ptr(dq), ptr(m_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_hl_gauss_loss_fwd_bwd", B, agent.action_space, agent.atoms, *args, *outs)
    else:
        call("riqn_hl_gauss_loss_fwd_bwd_h", B, agent.action_space, agent.atoms, *args, eps, *outs)
