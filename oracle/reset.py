"""Oracle (test infrastructure): riqn_arena_reset (include/riqn_b200.h) as a numpy float32 statement.

  u_i    = fl(fl((x_i >> 8) + 0.5) / 2^24), x_i word i of the Philox4x32-10 stream (riqn_fill_uniform's draw)
  theta0 = fl(value * (2 u_i - 1)) (uniform segment) or value (constant segment)
  theta' = theta0 when alpha = 0, else fl(fl(alpha * theta) + fl(fl(1 - alpha) * theta0))

Every numpy float32 operation below rounds on its own; nothing outside the segments changes.
"""
import numpy as np

UNIFORM, CONSTANT = 0, 1


def uniforms(words):
    """riqn_fill_uniform's floats of the Philox words ``words`` (uint32)."""
    m = (np.asarray(words, np.uint32) >> np.uint32(8)).astype(np.float32)
    return (m + np.float32(0.5)) * np.float32(2.0 ** -24)


def fresh(kind, value, u):
    """theta0 of a segment whose elements draw the uniforms ``u``."""
    v = np.float32(value)
    if kind == UNIFORM:
        return v * (np.float32(2.0) * u - np.float32(1.0))
    return np.full(u.shape, v, np.float32)


def arena_reset(theta, segs, words):
    """The arena ``theta`` (n,) float32 after riqn_arena_reset with the segments ``segs`` [(begin, end, kind, value,
    alpha)] under the Philox words ``words`` (at least n of them: helpers.philox_np(seed, stream_id, ceil(n / 4)))."""
    theta = np.asarray(theta, np.float32)
    out, u = theta.copy(), uniforms(words)
    for b, e, kind, value, alpha in segs:
        t0, a = fresh(kind, value, u[b:e]), np.float32(alpha)
        out[b:e] = t0 if a == 0 else a * theta[b:e] + (np.float32(1.0) - a) * t0
    return out
