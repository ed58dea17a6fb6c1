"""Periodic network resets: the reset policy, for every arena a learner trains, in one place.

Every so many updates the data-efficient Atari agents (Nikishin et al., "The Primacy Bias in Deep Reinforcement
Learning", ICML 2022; SR-SPR, D'Oro et al., ICLR 2023; BBF, Schwarzer et al., ICML 2023) redraw their last layers from
the initial distribution and pull the encoder part of the way back towards a fresh draw (shrink-and-perturb):
theta' = alpha theta + (1 - alpha) theta0.  Here, with alpha_s = reset_shrink:

  arena         segment                                                    fresh draw theta0                      alpha
  online_net    conv1-3 weight and bias                                    U(+-1/sqrt(Cin k^2))                   alpha_s
                iqn_fc weight and bias (IQN head)                          U(+-1/sqrt(quantile_embedding_dim))    0
                each NoisyLinear weight_mu, bias_mu                        U(+-1/sqrt(in))                        0
                                 weight_sigma / bias_sigma                 sigma0/sqrt(in) / sigma0/sqrt(out)     0
  fraction_net  weight / bias (FQF)                                        U(+-0.01 sqrt(6/(3136+N))) / 0         0
  curl_net      projection and bilinear                                    U(+-1/sqrt(fan_in))                    0
  spr_net       transition conv1 (fan_in (64+A) 9) and conv2               U(+-1/sqrt(fan_in))                    alpha_s
                projection and predictor q                                 U(+-1/sqrt(fan_in))                    0

i.e. each module's constructor distribution (torch's nn.Linear / nn.Conv2d init, NoisyLinear.reset_parameters, FQF's
Xavier init).  With alpha_s = 1 the trunk and the transition model are left out: only the last layers are redrawn.
One riqn_arena_reset launch per arena rewrites its segments and zeroes its Adam moments, and the optimiser restarts at
step 0, so the next step takes torch's step-1 bias corrections, eagerly and in a captured graph alike.  Afterwards CURL's
momentum projection is set to the new projection (as curl.build does at construction) and the online network's
composed weights are rebuilt, so acting right after a reset sees the new weights.

Untouched: the target network (it bootstraps from the pre-reset network until the next update_target_net; under
target_ema it follows the reset online network at rate tau from the next step on, target.py), the epsilon arenas, and CURL's momentum trunk (it keeps following the online trunk by EMA).  Each draw is keyed by
online_net._rng_seed ^ RESET_SEED with stream id (reset index) * 4 + arena index; data-parallel replicas share that seed
(parallel.make_data_parallel), so every rank draws the same reset without a collective.  Under Ape-X only the learner
rank resets; the actors receive the reset weights with the next publication.
"""
import ctypes
import math

from . import config
from ._lib import ResetSegment, call, ptr
from .model import FEAT

RESET_SEED = 0x5E5E7A            # the reset draws' key (online_net._rng_seed ^ this)
UNIFORM, CONSTANT = 0, 1         # RIQN_RESET_UNIFORM, RIQN_RESET_CONSTANT
MAX_SEGMENTS = 64                # RIQN_RESET_MAX_SEGMENTS
ARENAS = ("online_net", "fraction_net", "curl_net", "spr_net")     # the arena index of a reset's stream ids


def _f32(x):
    return ctypes.c_float(x).value


def _seg(p, kind, value, alpha):
    """(begin, end, kind, value, alpha) of parameter ``p`` (a view of its module's arena), value as its float32."""
    return (p._riqn_offset, p._riqn_offset + p.numel(), kind, _f32(value), alpha)


def _linear(w, b, fan_in, alpha):
    """A weight and its bias as nn.Linear / nn.Conv2d draw them: both U(+-1/sqrt(fan_in))."""
    bound = 1.0 / math.sqrt(fan_in)
    return [_seg(w, UNIFORM, bound, alpha)] + ([_seg(b, UNIFORM, bound, alpha)] if b is not None else [])


def shrink(agent):
    """alpha_s: the agent's reset_shrink, or its default when resets are off (reset_networks called by hand)."""
    return agent.reset[1] if agent.reset is not None else config.FIELDS["reset_shrink"][0]


def _online_segments(on, a_s):
    segs = []
    if a_s != 1.0:
        for conv in (on.conv1, on.conv2, on.conv3):
            segs += _linear(conv.weight, conv.bias, conv.weight[0].numel(), a_s)
    if on._embeds():
        segs += _linear(on.iqn_fc.weight, on.iqn_fc.bias, on.quantile_embedding_dim, 0.0)
    for _, m in on.noisy_layers():
        bound = 1.0 / math.sqrt(m.in_features)
        segs += [_seg(m.weight_mu, UNIFORM, bound, 0.0), _seg(m.bias_mu, UNIFORM, bound, 0.0),
                 _seg(m.weight_sigma, CONSTANT, m.std_init / math.sqrt(m.in_features), 0.0),
                 _seg(m.bias_sigma, CONSTANT, m.std_init / math.sqrt(m.out_features), 0.0)]
    return segs


def _fraction_segments(f, a_s):
    bound = 0.01 * math.sqrt(6.0 / (f.feat_dim + f.num_fractions))
    return [_seg(f.weight, UNIFORM, bound, 0.0), _seg(f.bias, CONSTANT, 0.0, 0.0)]


def _curl_segments(c, a_s):
    segs = _linear(c.weight_h, c.bias_h, FEAT, 0.0) + _linear(c.weight_c, c.bias_c, c.weight_c.shape[1], 0.0)
    return segs + _linear(c.bilinear, None, c.bilinear.shape[1], 0.0)


def _spr_segments(s, a_s):
    segs = _linear(s.weight_h, s.bias_h, FEAT, 0.0) + _linear(s.weight_c, s.bias_c, s.weight_c.shape[1], 0.0)
    if a_s != 1.0:
        for conv in (s.conv1, s.conv2):
            segs += _linear(conv.weight, conv.bias, conv.weight[0].numel(), a_s)
    return segs + _linear(s.weight_q, s.bias_q, s.weight_q.shape[1], 0.0)


_SEGMENTS = (_online_segments, _fraction_segments, _curl_segments, _spr_segments)    # by arena index, as ARENAS


def tables(agent):
    """[(arena index, module, optimiser, sorted segments)] of every arena ``agent`` trains: the online network's, then
    the sides'."""
    a_s = shrink(agent)
    arenas = [(0, agent.online_net, agent.optimiser)] + [(s.index, s.net, s.optimiser) for s in agent.sides]
    return [(k, net, opt, sorted(_SEGMENTS[k](net, a_s))) for k, net, opt in arenas]


def reset_arena(net, optimiser, segs, seed, stream_id):
    """One riqn_arena_reset launch over ``net``'s arena with the segment table ``segs``; restarts ``optimiser``."""
    arr = (ResetSegment * len(segs))(*(ResetSegment(*s) for s in segs))
    call("riqn_arena_reset", net._flat.numel(), ptr(net._flat), ptr(optimiser._exp_avg), ptr(optimiser._exp_avg_sq),
         len(segs), arr, seed, stream_id)
    optimiser.restart()


def reset(agent, index):
    """Reset number ``index`` of ``agent``'s networks, by the table above."""
    seed = agent.online_net._rng_seed ^ RESET_SEED
    for k, net, opt, segs in tables(agent):
        reset_arena(net, opt, segs, seed, index * len(ARENAS) + k)
    for side in agent.sides:
        if side.after_reset is not None:
            side.after_reset(agent)
    agent.online_net._params_changed()
    agent.online_net.compose_weights()
