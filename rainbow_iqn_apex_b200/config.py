"""The agent's optional ``args`` fields: their defaults and domains, and which head and loss variants combine.

None of these fields is in the reference's namespace; a namespace without them trains the reference's agent.  ``read``
validates a whole namespace once, before the agent builds anything, and returns what the agent stores; ``read_risk``
applies the risk column of the combination table, in ``read`` and in ``Agent.set_risk``; ``read_head`` gives DQN its
head; ``read_demo`` gives ReplayMemory its demonstration fields.  Real-valued fields are checked on the float32 the
kernels receive.  Every refusal is a ValueError that names the fields at fault.
"""
import ctypes
import math
import numbers

from .model import check_risk

MAX_N = 256                # QR-DQN's quantiles and FQF's fractions (num_tau_samples)
MAX_ACTIONS = 32           # QR-DQN: riqn_argmax_mean / riqn_argmax_expected_h
MAX_BANDWIDTHS = 16        # riqn_mmd_loss_fwd_bwd
MAX_SIGMA_RATIO = 1000.0   # riqn_hl_gauss_loss_fwd_bwd
MAX_BATCH = 4096           # riqn_curl_infonce_fwd_bwd, riqn_spr_cosine_fwd_bwd
MAX_SPR_STEPS = 12         # riqn_spr_cosine_fwd_bwd; riqn_sequence_gather's history + K <= 16 at history 4
MAX_SPR_ACTIONS = 64       # riqn_spr_pack: the one-hot planes share conv1's 128 input channels with the latent's 64
_LOG2E = 1.4426950408889634


def _f32(x):
    return ctypes.c_float(x).value


def switch(name, v):
    """0 or 1 (bools and numpy integers allowed) as a bool."""
    if isinstance(v, bool) or (isinstance(v, numbers.Integral) and v in (0, 1)):
        return bool(v)
    raise ValueError(f"{name} must be 0 or 1, got {v!r}")


def real(ok, need, exact=False):
    """The domain of a real number (not a bool) that is finite and ``ok`` as the float32 a kernel receives.  Its parser
    returns that float32 as a Python float, or with ``exact`` the value itself as a Python float (a double the host
    keeps, as Adam's learning rate)."""
    def parse(name, v):
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError(f"{name} must be a real number, got {v!r}")
        f = _f32(float(v))
        if not (math.isfinite(f) and ok(f)):
            raise ValueError(f"{name} must be finite and {need} as a float32, got {v!r}")
        return float(v) if exact else f
    return parse


def integer(lo, hi):
    """The domain of an integer (not a bool) in lo..hi."""
    def parse(name, v):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not lo <= v <= hi:
            raise ValueError(f"{name} must be an integer in {lo}..{hi}, got {v!r}")
        return int(v)
    return parse


def _bandwidths(name, v):
    """1..16 bandwidths h, a sequence (not a string) of reals, each > 0 with the kernel's log2(e)/h and 2/h finite in
    float32, as a tuple of Python floats."""
    if isinstance(v, (str, bytes)):
        raise ValueError(f"{name} must be a sequence of numbers, not a string: {v!r}")
    try:
        hs = tuple(v)
    except TypeError:
        raise ValueError(f"{name} must be a sequence of numbers, got {v!r}") from None
    if not 1 <= len(hs) <= MAX_BANDWIDTHS:
        raise ValueError(f"{name} needs 1..{MAX_BANDWIDTHS} bandwidths, got {len(hs)}")
    h = real(lambda h: h > 0.0 and math.isfinite(_f32(_LOG2E / h)) and math.isfinite(_f32(2.0 / h)),
             "> 0 (with 2/h finite)", exact=True)
    return tuple(h(f"each of {name}", x) for x in hs)


# optional args field -> (default, domain).  A variant's parameters are the fields named "<its switch>_...", read only
# when the switch is on
FIELDS = {
    "qr_dqn": (0, switch),                       # N is the reference's num_tau_samples
    "munchausen": (0, switch),
    "munchausen_alpha": (0.9, real(lambda x: x >= 0.0, ">= 0", exact=True)),      # the paper's three
    "munchausen_tau": (0.03, real(lambda x: x > 0.0, "> 0", exact=True)),
    "munchausen_l0": (-1.0, real(lambda x: x <= 0.0, "<= 0", exact=True)),
    "fqf": (0, switch),
    "fqf_fraction_lr": (2.5e-9, real(lambda x: x > 0.0, "> 0", exact=True)),      # the public FQF Atari configurations'
    "fqf_entropy_coef": (0.0, real(lambda x: x >= 0.0, ">= 0", exact=True)),
    "mmd": (0, switch),
    "mmd_bandwidths": (tuple(float(h) for h in range(1, 11)), _bandwidths),
    "hl_gauss": (0, switch),
    "hl_gauss_sigma": (0.75, real(lambda x: 0.0 < x <= MAX_SIGMA_RATIO, f"in (0, {MAX_SIGMA_RATIO:g}]")),   # sigma / delta_z
    "cql": (0, switch),
    "cql_alpha": (1.0, real(lambda x: x > 0.0, "> 0")),           # this project's default, not a value from the paper
    "dqfd": (0, switch),
    "dqfd_margin": (0.8, real(lambda x: x > 0.0, "> 0")),         # Hester et al.'s two
    "dqfd_lambda": (1.0, real(lambda x: x > 0.0, "> 0")),
    "value_rescaling": (0, switch),
    "value_rescaling_eps": (1e-3, real(lambda x: x >= 0.0, ">= 0", exact=True)),  # R2D2's
    "random_shift": (0, integer(0, 83)),                          # the pad p in pixels, 0: off; DrQ uses 4
    "curl": (0, switch),
    "curl_coef": (1.0, real(lambda x: x > 0.0, "> 0")),           # this project's starting point, not tuned
    "curl_momentum": (0.001, real(lambda x: 0.0 < x <= 1.0, "in (0, 1]")),
    "spr": (0, switch),
    "spr_steps": (5, integer(1, MAX_SPR_STEPS)),                  # the paper's Atari K and lambda
    "spr_coef": (2.0, real(lambda x: x > 0.0, "> 0")),
    "reset": (0, switch),
    "reset_interval": (40000, integer(1, math.inf)),              # this project's starting point, not tuned
    "reset_shrink": (0.5, real(lambda x: 0.0 <= x <= 1.0, "in [0, 1]")),
    "target_ema": (0, switch),
    "target_ema_tau": (0.005, real(lambda x: 0.0 < x <= 1.0, "in (0, 1]")),      # BBF's two
    "adamw": (0, switch),
    "adamw_weight_decay": (0.1, real(lambda x: x >= 0.0, ">= 0")),
    "demo_segments": (0, integer(0, math.inf)),                   # at most nb_actor (read_demo)
    "demo_priority_bonus": (0.0, real(lambda x: x >= 0.0, ">= 0")),
}

HEADS = {"iqn": "the IQN head (rainbow_only = 0, qr_dqn = 0)", "qr": "the QR-DQN head (qr_dqn = 1)",
         "c51": "the C51 head (rainbow_only = 1)"}
# loss variant (at most one is on; None: the head's own loss) -> (the heads it trains, whether it takes a non-neutral
# risk measure).  A risk measure distorts the fractions the IQN head samples for a*: the other heads sample none, and
# Munchausen's soft target and FQF's proposed fractions pick no a* from them
LOSSES = {None: (("iqn", "qr", "c51"), True),
          "munchausen": (("iqn",), False),
          "fqf": (("iqn",), False),
          "cql": (("iqn", "qr"), True),
          "dqfd": (("iqn", "qr"), True),
          "mmd": (("qr",), False),
          "hl_gauss": (("c51",), False)}


def field(args, name):
    default, parse = FIELDS[name]
    return parse(name, getattr(args, name, default))


def _quantiles(args):
    return integer(2, MAX_N)("num_tau_samples", getattr(args, "num_tau_samples", None))


def read_head(args, action_space):
    """(head, N): the head ``args`` select, "iqn", "c51" (rainbow_only) or "qr" (qr_dqn), and QR-DQN's N =
    num_tau_samples, None for the other heads."""
    if not field(args, "qr_dqn"):
        return ("c51" if args.rainbow_only else "iqn"), None
    if args.rainbow_only:
        raise ValueError("qr_dqn and rainbow_only are two different heads on the same network: set one of them")
    if not 1 <= action_space <= MAX_ACTIONS:
        raise ValueError(f"qr_dqn supports 1..{MAX_ACTIONS} actions, got {action_space!r}")
    return "qr", _quantiles(args)


def read_risk(head, loss, measure, eta=None):
    """model.check_risk's value of (measure, eta), refused unless the head and the loss variant take a non-neutral
    measure (LOSSES)."""
    risk = check_risk((measure, eta))
    if risk is not None and not (head == "iqn" and LOSSES[loss][1]):
        raise ValueError(f"a non-neutral risk measure distorts the IQN head's sampled fractions: {HEADS[head]}"
                         + (f" with {loss} = 1" if loss else "") + " acts risk-neutrally")
    return risk


def read(args, action_space):
    """Validate the optional fields of ``args`` and return what the agent stores, as a dict: qr_dqn (N or None); per
    variant switch (munchausen, fqf, mmd, hl_gauss, cql, dqfd, value_rescaling, curl, spr, reset, target_ema, adamw) None
    when off, else its parameter or the tuple of its parameters; random_shift (the pad, or None); risk
    (model.check_risk's); and the "head" and the "loss" variant (or None) they select.  Resets, the EMA target
    (target_ema: tau) and AdamW (adamw: the weight decay lambda) combine with every head and variant; AdamW needs
    lr * lambda < 1 for the agent's lr and, under FQF, for fqf_fraction_lr, as the float32 values the optimiser receives."""
    head, n = read_head(args, action_space)
    v = {"qr_dqn": n}
    for name in ("munchausen", "fqf", "mmd", "hl_gauss", "cql", "dqfd", "value_rescaling", "curl", "spr", "reset",
                 "target_ema", "adamw"):
        v[name] = None
        if field(args, name):
            params = tuple(field(args, f) for f in FIELDS if f.startswith(name + "_"))
            v[name] = params if len(params) > 1 else params[0]
    on = [name for name in LOSSES if name is not None and v[name] is not None]
    if len(on) > 1:
        raise ValueError(f"{' and '.join(on)} are loss variants, of which one at most can be on")
    loss = on[0] if on else None
    heads = LOSSES[loss][0]
    if head not in heads:
        raise ValueError(f"{loss} = 1 trains {' or '.join(HEADS[h] for h in heads)}; the args select {HEADS[head]}")
    if loss == "fqf":
        _quantiles(args)
    if loss == "munchausen" and v["value_rescaling"] is not None:
        raise ValueError("value_rescaling and munchausen do not combine: Munchausen's soft target mixes log-policies of "
                         "means; set one of them to 0")
    v["random_shift"] = field(args, "random_shift") or None
    if v["curl"] is not None:
        if v["random_shift"] is None:
            raise ValueError("curl = 1 contrasts two random shifts of each state: set random_shift >= 1 (DrQ uses 4)")
        integer(2, MAX_BATCH)("batch_size", args.batch_size)      # CURL's negatives are the batch's other states
    if v["spr"] is not None:
        if v["curl"] is not None:
            raise ValueError("spr and curl are both auxiliary losses on the trunk's feature gradient, of which one at most "
                             "can be on")
        if not 1 <= action_space <= MAX_SPR_ACTIONS:
            raise ValueError(f"spr supports 1..{MAX_SPR_ACTIONS} actions (its transition model's one-hot action planes), "
                             f"got {action_space!r}")
        integer(1, MAX_BATCH)("batch_size", args.batch_size)
        history = getattr(args, "history_length", 4)
        if history + v["spr"][0] > 16:
            raise ValueError(f"spr_steps + history_length must be at most 16 (the sequence window), got "
                             f"{v['spr'][0]} + {history}")
    if v["adamw"] is not None:
        lrs = [("lr", args.lr)] + ([("fqf_fraction_lr", v["fqf"][0])] if v["fqf"] is not None else [])
        for name, lr in lrs:
            if not 0.0 <= _f32(lr) * v["adamw"] < 1.0:       # riqn_adamw_step's decay 1 - lr * lambda in (0, 1]
                raise ValueError(f"adamw_weight_decay decays by 1 - {name} * adamw_weight_decay, which must be in (0, 1]: "
                                 f"{name} = {lr!r}, adamw_weight_decay = {v['adamw']!r}")
    v["risk"] = read_risk(head, loss, getattr(args, "risk_measure", "neutral"), getattr(args, "risk_eta", None))
    return dict(v, head=head, loss=loss)


def read_demo(args):
    """ReplayMemory's (D, eps_d): D = demo_segments in 0..nb_actor, the number of segments, counted from the last, that
    hold demonstrations; eps_d the float32 demo_priority_bonus."""
    d = field(args, "demo_segments")
    if d > args.nb_actor:
        raise ValueError(f"demo_segments must be in 0..nb_actor = {args.nb_actor}, got {d}")
    return d, field(args, "demo_priority_bonus")
