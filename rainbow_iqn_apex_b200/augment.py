"""Random-shift image augmentation (DrQ: Kostrikov, Yarats & Fergus, ICLR 2021), drawn and applied on the device.

Every sample's frame stack is padded by p pixels with edge replication and cropped back to its size at a random offset,
one (dy, dx) in [-p, p]^2 per sample shared by its history frames:
    out[c, y, x] = in[c, clamp(y + dy, 0, H-1), clamp(x + dx, 0, W-1)]
Pixels stay uint8, so the trunk's pixel block matrix stays exact in bf16.  The learner (Agent.random_shift = p) shifts s_t
and s_{t+n} independently in each step; acting never shifts.  A torch loss written on net(x, N) shifts its frames with
draw_shifts and random_shift before the forward.
"""
import torch

from ._lib import call, ptr
from .model import _EAGER_STREAMS

SHIFT_SEED = 0x5D1F7     # the shift draws' key is net._rng_seed ^ SHIFT_SEED: apart from the noise and fraction draws'


def draw_shifts(net, n, pad, key=SHIFT_SEED, advance=True):
    """n shifts (dy, dx) uniform on [-pad, pad]^2, an (n, 2) int32 device tensor, from ``net``'s Philox generator
    (riqn_fill_shifts).  The stream is rank-private (net._tau_stream_offset) and counts per step like the fraction draws'
    (a static index read with the device step state in graph mode, the eager half of the id space otherwise), under a key
    of its own: a shift draw takes no stream the noise or fraction draws use.  ``key`` (xor-ed into net._rng_seed) and
    ``advance`` = False let a draw of another kind (CURL's positive view) take streams of its own without moving the
    counters the learner's shifts of s_t and s_{t+n} read."""
    out = torch.empty(n, 2, dtype=torch.int32, device=net._flat.device)
    dyn = getattr(net, "_dyn", None)
    idx = net._shift_in_step if dyn is not None else net._shift_calls
    stream_id = net._tau_stream_offset + idx + (0 if dyn is not None else _EAGER_STREAMS)
    call("riqn_fill_shifts", n, int(pad), net._rng_seed ^ key, stream_id, ptr(out), dyn.ptr() if dyn else None)
    if advance:
        net._shift_calls += 1
        net._shift_in_step += 1
    return out


def injection(learner):
    """The injection dict of the step ``learner`` is about to run: its ``_inject``, or the first of a list of them
    (peeked: the loss core pops it); an empty dict without one."""
    inj = learner._inject[0] if isinstance(learner._inject, list) and learner._inject else learner._inject
    return inj if isinstance(inj, dict) else {}


def view_shifts(learner, name, n, key):
    """n shifts (n, 2) int32 for a further view of one step's frames (CURL's positive, SPR's targets): the injection's
    ``name``, or a draw under ``key`` that moves none of the counters, so that the learner's shifts of s_t and s_{t+n}
    stay those of a learner without the view."""
    given = injection(learner).get(name)
    if given is None:
        return draw_shifts(learner.online_net, n, learner.random_shift, key=key, advance=False)
    return torch.as_tensor(given, dtype=torch.int32).reshape(n, 2).to(learner.online_net._flat.device)


def _frames(x, dev):
    """Frames the kernel reads: on ``dev``, uint8 or fp32, each sample (C, H, W)-contiguous with a 16-byte aligned start
    (replay-window views qualify as they are)."""
    x = x.to(dev)
    if x.dtype != torch.uint8:
        x = x.float()
    C, H, W = x.shape[1:]
    if (x.stride()[1:] != (H * W, W, 1) or x.stride(0) < C * H * W or x.data_ptr() % 16
            or x.stride(0) * x.element_size() % 16):
        x = x.clone(memory_format=torch.contiguous_format)
    return x


def random_shift(next_states, states, shifts):
    """Shifted copies of two batches of frame stacks (B, C, H, W), uint8 or fp32, in one launch (riqn_random_shift).
    ``shifts``: (2B, 2) int32 (dy, dx), rows [0, B) for next_states and [B, 2B) for states.  Returns the two shifted
    batches as views of one contiguous (2B, C, H, W) buffer, in that order.  ``states`` may be None: then ``shifts`` is
    (B, 2) and one shifted batch is returned."""
    dev = shifts.device if shifts.is_cuda else torch.device("cuda")
    x0 = _frames(next_states, dev)
    x1 = _frames(states, dev) if states is not None else None
    B, C, H, W = x0.shape
    if x1 is not None and (x1.dtype != x0.dtype or x1.shape != x0.shape):
        raise ValueError(f"next_states {tuple(x0.shape)} {x0.dtype} and states {tuple(x1.shape)} {x1.dtype} differ")
    n = B if x1 is None else 2 * B
    shifts = shifts.to(dev, torch.int32).contiguous()
    if tuple(shifts.shape) != (n, 2):
        raise ValueError(f"shifts must be ({n}, 2), got {tuple(shifts.shape)}")
    out = torch.empty(n, C, H, W, dtype=x0.dtype, device=dev)
    call("riqn_random_shift", B, C, H, W, ptr(x0), x0.stride(0), ptr(x1), x1.stride(0) if x1 is not None else 0,
         1 if x0.dtype == torch.uint8 else 0, ptr(shifts), ptr(out))
    return out if x1 is None else (out[:B], out[B:])
