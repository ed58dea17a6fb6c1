"""The convolution trunk's kernels, entry point by entry point, against float64 statements of the same operations
(include/riqn_b200.h): riqn_s2d_u8, riqn_conv_fwd_strip (one and two weight sets), riqn_conv_bwd_strip,
riqn_conv_fwd_tc, riqn_conv_bwd_tc, the fp32 CUDA-core path riqn_im2col_f32 / riqn_conv_fwd / riqn_conv_bwd,
riqn_split_bf16_scaled and riqn_zero_f32.

Method (as tests/test_gpu_c51_kernels.py):
* every reference is computed on the operands the kernel consumed: the bf16 block matrices and im2col images, the bf16
  weight images, and for split-bf16 x3 the three products hi.hi + hi.lo + lo.hi (conv1's split-2: pixels times
  hi + lo).  Input rounding is never part of a comparison;
* exact regime: small-integer pixels, activations and output gradients and weights that are small integers times a
  power of two keep every product and partial sum exact in fp32 (the generators assert that every sum stays below
  2^24 of its finest grid), so the kernel has to match float64 bit for bit in any summation order.  A second exact case puts a non-zero lo image on one operand, so the
  hi.lo and lo.hi products are checked bit for bit too;
* random regime: each element is held to c * K * 2^-24 * sum|a_i b_i| (K = the reduction length) plus the output
  rounding; each test prints its worst err/bound ratio;
* outputs that are one rounding (dYg, dY_hi / dYT_hi, the next layer's block images, every im2col image, the fp32 dY,
  riqn_split_bf16_scaled) are bitwise in both regimes;
* overwritten outputs start as NaN, accumulated outputs (dw, dbias) from a non-zero pattern, every buffer carries
  canaries past its end, entry points are called twice in the random regime and must agree bit for bit (no float
  atomic takes part in any sum; tests/test_gpu_fallback_paths.py pins the order of the fp32 and col2im sums),
  and every documented rejection returns cudaErrorInvalidValue and writes nothing.
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import (U, Out, assert_bits, assert_canaries, bf16, bf16_bits, check_bound, dptr, f32_bits, lib_call,
                     prefill_pattern, to_dev, to_dev_bf16)

C_BOUND = 2.0
F32 = np.float32
BF = torch.bfloat16
# (Cin, H, Cout, k, stride, pad) of the three Atari convolutions (model.py:65-67)
LAYERS = {"conv1": (4, 84, 32, 8, 4, 1), "conv2": (32, 20, 64, 4, 2, 0), "conv3": (64, 9, 64, 3, 1, 0)}
NEXT = {"conv1": "conv2", "conv2": "conv3", "conv3": None}
NAMES = list(LAYERS)


# ---------------------------------------------------------------------------------------------- float64 statements
def out_size(h, k, s, pad):
    return (h + 2 * pad - k) // s + 1


def strip_dims(cin, h, k, s, pad):
    """(OH, t, G, Kc): output edge, shifts per axis, block grid edge, block row width"""
    oh = out_size(h, k, s, pad)
    t = k // s
    return oh, t, oh + t - 1, s * s * cin


def block_matrix(x, k, s, pad, first):
    """(B*G*G, s*s*C) block matrix of the zero-padded NCHW image x: within-block order (c, iy, ix) for a first layer
    (riqn_s2d_u8), (iy, ix, c) for the block images a layer's epilogue writes for the next one"""
    B, C, H, W = x.shape
    _, _, G, _ = strip_dims(C, H, k, s, pad)
    xp = np.zeros((B, C, G * s, G * s), x.dtype)
    hh, ww = min(H, G * s - pad), min(W, G * s - pad)
    xp[:, :, pad:pad + hh, pad:pad + ww] = x[:, :, :hh, :ww]
    blk = xp.reshape(B, C, G, s, G, s)                                 # b c gy iy gx ix
    A = blk.transpose(0, 2, 4, 1, 3, 5) if first else blk.transpose(0, 2, 4, 3, 5, 1)
    return np.ascontiguousarray(A).reshape(B * G * G, C * s * s)


def strip_perm(cin, k, s, first):
    from rainbow_iqn_apex_b200.model import _strip_perm
    return _strip_perm(cin, k, s, first).numpy()


def im2col(x, k, s, pad):
    """(B*OH*OW, C*k*k) im2col matrix, k order (c, kh, kw) = the weight's; a pure gather of x"""
    B, C = x.shape[:2]
    cols = F.unfold(torch.from_numpy(np.ascontiguousarray(x)), k, padding=pad, stride=s)   # (B, C*k*k, L)
    return cols.transpose(1, 2).reshape(-1, C * k * k).numpy()


def _t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float64))


def conv64(x, w, s, pad):
    return F.conv2d(_t64(x), _t64(w), stride=s, padding=pad).numpy()


def wgrad64(x, dy, wshape, s, pad):
    return torch.nn.grad.conv2d_weight(_t64(x), tuple(wshape), _t64(dy), stride=s, padding=pad).numpy()


def dgrad64(dy, w, xshape, s, pad):
    return torch.nn.grad.conv2d_input(tuple(xshape), _t64(w), _t64(dy), stride=s, padding=pad).numpy()


def fwd_ref(pairs, bias, s, pad):
    """relu(sum over the (x, w) products + bias) in float64, the bound's sum|a b| + |bias|, and K"""
    pairs = [(x, w) for x, w in pairs if np.any(x) and np.any(w)]
    pre = sum(conv64(x, w, s, pad) for x, w in pairs) + bias.astype(np.float64)[None, :, None, None]
    mag = sum(conv64(np.abs(x), np.abs(w), s, pad) for x, w in pairs) + np.abs(bias)[None, :, None, None]
    return np.maximum(pre, 0), mag


def fwd_bound(ref, mag, K):
    return C_BOUND * (K + 1) * U * mag + U * np.abs(ref)


def assert_exact_budget(what, mag, quantum):
    """the generator's promise: every partial sum is a multiple of `quantum` below 2^24 quanta (so exact in fp32)"""
    worst = float(np.max(mag)) / quantum if np.size(mag) else 0.0
    assert worst < 2.0 ** 24, f"{what}: exact-regime sums reach {worst:.3g} quanta"


def same_f32(what, got, ref):
    """bitwise, with -0 == +0 (a ReLU or an exact zero sum may carry either sign)"""
    ref32 = np.asarray(ref, np.float64).astype(F32)
    assert np.array_equal(ref32.astype(np.float64), np.asarray(ref, np.float64)), f"{what}: reference not fp32-exact"
    assert_bits(what, f32_bits(np.asarray(got, F32) + F32(0)), f32_bits(ref32 + F32(0)))


def split_hi_lo(x):
    hi = bf16(x)
    return hi, bf16((x - hi).astype(F32))


def geom(B, cin, h, cout, k, s, pad, in_bstride=None):
    from rainbow_iqn_apex_b200.model import _geom
    return _geom(B, cin, h, cout, k, s, pad, in_bstride)


def _expect_rejected(name, args, bufs):
    """the call returns cudaErrorInvalidValue and leaves every buffer (canaries included) as it was"""
    from rainbow_iqn_apex_b200._lib import RiqnError
    bits = lambda t: t.view(torch.int16 if t.element_size() == 2 else torch.int32).clone()
    snap = [bits(b) for b in bufs]
    with pytest.raises(RiqnError, match=r"cudaError 1$"):
        lib_call(name, *args)
    torch.cuda.synchronize()
    for i, (s, b) in enumerate(zip(snap, bufs)):
        assert torch.equal(s, bits(b)), f"{name}: rejected call wrote buffer {i}"


# ---------------------------------------------------------------------------------------------- input generators
def activations(rs, shape, regime, lo=False):
    """(hi, lo) fp32 arrays of bf16 values: the two images of an activation.  exact: integers 0..7 with zeros (lo = 0,
    or l * 2^-9 with lo=True); random: relu(N(0, 1)) split into hi + lo"""
    if regime == "random":
        return split_hi_lo(np.maximum(rs.standard_normal(shape), 0).astype(F32))
    hi = rs.randint(0, 8, shape).astype(F32)
    hi[rs.uniform(size=shape) < 0.3] = 0
    lo_img = (rs.randint(-3, 4, shape) * 2.0 ** -9).astype(F32) if lo else np.zeros(shape, F32)
    return hi, lo_img


def pixels(rs, shape, regime):
    return rs.randint(0, 256 if regime == "random" else 8, shape).astype(np.uint8)


def weights(rs, cout, cin, k, regime, lo=False, div=1.0):
    """(hi, lo, bias) of a layer as the kernel reads them.  exact: hi = k * 2^-6, lo = 0 (or l * 2^-14), bias on 2^-6;
    random: N(0, 1/K) / div split into hi + lo"""
    shape = (cout, cin, k, k)
    if regime == "random":
        w = (rs.standard_normal(shape) / np.sqrt(cin * k * k) / div).astype(F32)
        return (*split_hi_lo(w), (rs.standard_normal(cout) * 0.1).astype(F32))
    hi = (rs.randint(-3, 4, shape) * 2.0 ** -6).astype(F32)
    lo_img = (rs.randint(-3, 4, shape) * 2.0 ** -14).astype(F32) if lo else np.zeros(shape, F32)
    return hi, lo_img, (rs.randint(-8, 9, cout) * 2.0 ** -6).astype(F32)


def grads(rs, shape, regime):
    """(dout, out): the output gradient and the forward output whose sign is the ReLU mask"""
    if regime == "random":
        return rs.standard_normal(shape).astype(F32), rs.standard_normal(shape).astype(F32)
    dout = rs.randint(-2, 3, shape).astype(F32)
    return dout, rs.randint(-1, 3, shape).astype(F32)


def masked(dout, out):
    return np.where(out > 0, dout, F32(0)).astype(F32)


def prefills(n, regime, rs):
    return prefill_pattern(n, 1.0, 13) if regime == "exact" else rs.standard_normal(n).astype(F32)


# ---------------------------------------------------------------------------------------------- 1. riqn_s2d_u8
S2D_GEOMS = {"atari": (4, 84, 32, 8, 4, 1), "generic": (16, 32, 32, 4, 2, 0), "generic_pad2": (4, 40, 32, 8, 4, 2)}


S2D_CASES = [(n, B, v) for n in S2D_GEOMS for B in (1, 3, 8, 512) for v in ("dense", "window") if v == "dense" or n == "atari"]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,view", S2D_CASES, ids=[f"{n}-B{b}-{v}" for n, b, v in S2D_CASES])
def test_s2d_u8(cuda_dev, name, B, view):
    """the block matrix of raw pixel values, bitwise: the byte-permute fast path (Atari conv1), the generic path, and
    the learner's (B, 7, 84, 84)[:, 3:7] replay-window view with its batch stride"""
    dev = cuda_dev
    cin, h, cout, k, s, pad = S2D_GEOMS[name]
    oh, t, G, Kc = strip_dims(cin, h, k, s, pad)
    rs = np.random.RandomState(B + len(name))
    if view == "window":
        full = rs.randint(0, 256, (B, 7, h, h)).astype(np.uint8)
        x = full[:, 3:7]
        xd = torch.from_numpy(full).to(dev)[:, 3:7]
        g = geom(B, cin, h, cout, k, s, pad, in_bstride=7 * h * h)
    else:
        x = rs.randint(0, 256, (B, cin, h, h)).astype(np.uint8)
        xd = torch.from_numpy(x).to(dev)
        g = geom(B, cin, h, cout, k, s, pad)
    want = bf16_bits(block_matrix(x.astype(F32), k, s, pad, first=True))
    for rep in range(2):                                     # no atomics: a second call is bitwise the first
        a = Out(B * G * G * Kc, dev, BF)
        lib_call("riqn_s2d_u8", g, xd.data_ptr(), a.p)
        torch.cuda.synchronize()
        assert_canaries({"a_px": a})
        assert_bits(f"a_px call {rep}", a.bits(), want.ravel())


@pytest.mark.gpu
def test_s2d_u8_rejections(cuda_dev):
    dev = cuda_dev
    buf = torch.zeros(2 * 7 * 84 * 84 + 64, dtype=torch.uint8, device=dev)
    a = Out(2 * 441 * 64, dev, BF)
    base = buf.data_ptr()
    g = geom(2, 4, 84, 32, 8, 4, 1)
    _expect_rejected("riqn_s2d_u8", (g, base + 1, a.p), [a.t])                                        # unaligned in
    _expect_rejected("riqn_s2d_u8", (geom(2, 4, 84, 32, 8, 4, 1, 4 * 84 * 84 + 8), base, a.p), [a.t])  # in_bstride % 16
    _expect_rejected("riqn_s2d_u8", (geom(2, 4, 83, 32, 8, 4, 1), base, a.p), [a.t])                   # chw % 16 (H 83)


# ---------------------------------------------------------------------------------------------- 2. riqn_conv_fwd_strip
def _strip_layer_inputs(layer, B, regime, lo_on, rs):
    """NCHW images and weights of one layer: x_hi / x_lo (conv1: raw pixels, lo = 0) and w_hi / w_lo / bias as the
    strip kernel reads them (conv1's weights already carry the 1/255)"""
    cin, h, cout, k, s, pad = LAYERS[layer]
    if layer == "conv1":
        x_hi, x_lo = pixels(rs, (B, cin, h, h), regime).astype(F32), np.zeros((B, cin, h, h), F32)
    else:
        x_hi, x_lo = activations(rs, (B, cin, h, h), regime, lo=lo_on == "a")
    w_hi, w_lo, bias = weights(rs, cout, cin, k, regime, lo=lo_on == "w", div=255.0 if layer == "conv1" else 1.0)
    return x_hi, x_lo, w_hi, w_lo, bias


def _strip_operands(layer, dev, x_hi, x_lo, w_hi, w_lo, bias):
    cin, h, cout, k, s, pad = LAYERS[layer]
    first = layer == "conv1"
    perm = strip_perm(cin, k, s, first)
    wp = lambda w: np.ascontiguousarray(w.reshape(cout, -1)[:, perm])
    return dict(a_hi=to_dev_bf16(block_matrix(x_hi, k, s, pad, first), dev),
                a_lo=None if first else to_dev_bf16(block_matrix(x_lo, k, s, pad, first), dev),
                w_hi=to_dev_bf16(wp(w_hi), dev), w_lo=to_dev_bf16(wp(w_lo), dev), bias=to_dev(bias, dev))


def _next_layout(layer):
    nxt = NEXT[layer]
    if nxt is None:
        return None
    cin, h, cout, k, s, pad = LAYERS[nxt]
    oh, t, G, Kc = strip_dims(cin, h, k, s, pad)
    return s, G, Kc, k


def _fwd_strip(dev, layer, B, ops, mode, with_out=True, two=None, share_a=0):
    """one riqn_conv_fwd_strip call; mode x3 (conv1: split-2, pixels x (hi + lo)) or single.  two = the second weight
    set's operands (stacked mode; B counts both halves)"""
    cin, h, cout, k, s, pad = LAYERS[layer]
    oh = out_size(h, k, s, pad)
    lay = _next_layout(layer)
    o = {"out": Out(B * cout * oh * oh, dev) if with_out else None}
    nargs = (None, None, 0, 0)
    if lay is not None:
        ns, nG, nKc, _ = lay
        o["next_hi"] = Out(B * nG * nG * nKc, dev, BF)
        o["next_lo"] = Out(B * nG * nG * nKc, dev, BF) if mode == "x3" else None
        nargs = (o["next_hi"].p, o["next_lo"].p if o["next_lo"] else None, ns, nG)
    a_lo = dptr(ops["a_lo"]) if mode == "x3" else None
    w_lo = (lambda d: dptr(d["w_lo"]) if mode == "x3" else None)
    w2 = (dptr(two["w_hi"]), w_lo(two), dptr(two["bias"])) if two is not None else (None, None, None)
    lib_call("riqn_conv_fwd_strip", geom(B, cin, h, cout, k, s, pad), dptr(ops["a_hi"]), a_lo, dptr(ops["w_hi"]),
             w_lo(ops), dptr(ops["bias"]), o["out"].p if with_out else None, *nargs, *w2, share_a)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _check_next_images(what, layer, o, out_img, mode):
    """next_hi / next_lo: the hi / lo split of this call's own out, laid out as the next layer's block matrix"""
    lay = _next_layout(layer)
    if lay is None:
        return
    ns, nG, nKc, nk = lay
    hi, lo = split_hi_lo(out_img)
    assert_bits(f"{what} next_hi", o["next_hi"].bits(), bf16_bits(block_matrix(hi, nk, ns, 0, False)).ravel())
    if mode == "x3":
        assert_bits(f"{what} next_lo", o["next_lo"].bits(), bf16_bits(block_matrix(lo, nk, ns, 0, False)).ravel())


FWD_STRIP_CASES = [(layer, B, mode, regime, lo)
                   for layer in NAMES for B in (1, 3, 8, 512)
                   for mode, regime, lo in [("x3", "exact", None), ("x3", "random", None), ("single", "exact", None),
                                            ("single", "random", None), ("x3", "exact", "w"), ("x3", "exact", "a")]
                   if not (lo == "a" and layer == "conv1") and not (lo and B == 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("layer,B,mode,regime,lo", FWD_STRIP_CASES,
                         ids=[f"{l}-B{b}-{m}-{r}{'-lo_' + o if o else ''}" for l, b, m, r, o in FWD_STRIP_CASES])
def test_conv_fwd_strip(cuda_dev, layer, B, mode, regime, lo):
    """out against float64 NCHW on the products the mode forms, every real output written; next_hi / next_lo bitwise
    the split of out; a second call bitwise the first; a call with out == NULL writes the same next images"""
    dev = cuda_dev
    cin, h, cout, k, s, pad = LAYERS[layer]
    K = cin * k * k
    rs = np.random.RandomState(zlib.crc32(f"{layer}{B}{mode}{regime}{lo}".encode()))
    x_hi, x_lo, w_hi, w_lo, bias = _strip_layer_inputs(layer, B, regime, lo, rs)
    ops = _strip_operands(layer, dev, x_hi, x_lo, w_hi, w_lo, bias)
    pairs = [(x_hi, w_hi)]
    if mode == "x3":
        pairs += [(x_hi, w_lo), (x_lo, w_hi)]
    ref, mag = fwd_ref(pairs, bias, s, pad)
    tag = f"{layer} B{B} {mode} {regime}"
    o = _fwd_strip(dev, layer, B, ops, mode)
    out = o["out"].f32().reshape(ref.shape)
    if regime == "exact":
        assert_exact_budget(tag, mag, 2.0 ** -15)
        same_f32(f"out {tag}", out, ref)
    else:
        check_bound(f"out {tag}", out, ref, fwd_bound(ref, mag, K))
    _check_next_images(tag, layer, o, out, mode)
    o2 = _fwd_strip(dev, layer, B, ops, mode)
    for key in o:
        if o[key] is not None:
            assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())
    o3 = _fwd_strip(dev, layer, B, ops, mode, with_out=False)
    for key in ("next_hi", "next_lo"):
        if o.get(key) is not None:
            assert_bits(f"out == NULL {key}", o3[key].bits(), o[key].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["x3", "single"])
@pytest.mark.parametrize("Bs", [256, 1024])
@pytest.mark.parametrize("layer", NAMES)
def test_conv_fwd_strip_stacked(cuda_dev, layer, Bs, mode):
    """two weight sets over one stacked batch of Bs samples (the online and the target trunk over next_states): bitwise
    two single-network calls on the halves.  conv1 shares one pixel block matrix between the halves (share_a); conv2 /
    conv3 read the stacked images.  Weights and biases differ between the halves."""
    dev = cuda_dev
    cin, h, cout, k, s, pad = LAYERS[layer]
    _, _, G, _ = strip_dims(cin, h, k, s, pad)
    half = Bs // 2
    share = layer == "conv1"
    rs = np.random.RandomState(Bs + 7 * len(mode) + cin)
    xb = half if share else Bs
    x_hi, x_lo, w_hi, w_lo, bias = _strip_layer_inputs(layer, xb, "random", None, rs)
    w2_hi, w2_lo, bias2 = weights(rs, cout, cin, k, "random", div=255.0 if share else 1.0)
    assert not np.array_equal(w_hi, w2_hi) and not np.array_equal(bias, bias2)
    one = _strip_operands(layer, dev, x_hi, x_lo, w_hi, w_lo, bias)
    two = _strip_operands(layer, dev, x_hi, x_lo, w2_hi, w2_lo, bias2)
    rows = half * G * G
    halves = []
    for i, ops in enumerate((one, two)):
        lo_rows = 0 if (share or i == 0) else rows
        sub = dict(ops, a_hi=ops["a_hi"][lo_rows:lo_rows + rows],
                   a_lo=None if ops["a_lo"] is None else ops["a_lo"][lo_rows:lo_rows + rows])
        halves.append(_fwd_strip(dev, layer, half, sub, mode))
    for with_out in (True, False):
        st = _fwd_strip(dev, layer, Bs, one, mode, with_out=with_out, two=two, share_a=1 if share else 0)
        for key in st:
            if st[key] is None:
                continue
            both = np.concatenate([halves[0][key].bits(), halves[1][key].bits()])
            assert_bits(f"stacked {key} (out {'set' if with_out else 'NULL'})", st[key].bits(), both)


@pytest.mark.gpu
def test_conv_fwd_strip_rejections(cuda_dev):
    dev = cuda_dev
    bf = lambda n: torch.zeros(n, dtype=BF, device=dev)
    f32 = lambda n: torch.zeros(n, device=dev)
    w = bf(96 * 576)
    bias = f32(96)
    a = bf(8 * 100 * 128)
    out = Out(8 * 64 * 81, dev)
    nxt = Out(8 * 81 * 96, dev, BF)
    c2 = lambda B, cout=64: geom(B, 32, 20, cout, 4, 2, 0)
    call = lambda g, w2, w2_lo, b2, w_lo=None, nx=(None, 0, 0): (
        g, a.data_ptr(), None, w.data_ptr(), w_lo, bias.data_ptr(), out.p, nx[0], None, nx[1], nx[2], w2, w2_lo, b2, 0)
    bufs = [out.t, nxt.t]
    W, B_, L = w.data_ptr(), bias.data_ptr(), w.data_ptr() + 2
    _expect_rejected("riqn_conv_fwd_strip", call(c2(3), W, None, B_), bufs)                  # odd stacked B
    _expect_rejected("riqn_conv_fwd_strip", call(c2(4), W, None, B_), bufs)                  # (B/2) G^2 % 128
    _expect_rejected("riqn_conv_fwd_strip", call(c2(256), W, None, None), bufs)              # no bias2
    _expect_rejected("riqn_conv_fwd_strip", call(c2(256), W, None, B_, w_lo=L), bufs)        # lo in one weight set only
    _expect_rejected("riqn_conv_fwd_strip", call(c2(256), W, L, B_), bufs)
    _expect_rejected("riqn_conv_fwd_strip", call(c2(8, 96), None, None, None), bufs)         # Cout > 64
    _expect_rejected("riqn_conv_fwd_strip", call(geom(8, 64, 9, 48, 3, 1, 0), None, None, None,
                                                 nx=(nxt.p, 1, 9)), bufs)                    # next images, Cout % 32
    assert_canaries({"out": out, "next": nxt})


# ---------------------------------------------------------------------------------------------- 3. riqn_conv_bwd_strip
@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B", [3, 8, 512])
@pytest.mark.parametrize("layer", NAMES)
def test_conv_bwd_strip(cuda_dev, layer, B, regime):
    """dYg bitwise on the whole strip grid (rows off the real outputs exactly +0); dbias and dw accumulated from a
    prefill (exact: bitwise at wgrad_scale 1 and 2^-8; random: bounded, conv1 at 1/255); din of conv2 / conv3 as the
    transposed strip convolution.  At B = 512, conv1's weight gradient runs as 66 splits of 54 k-blocks and dYg's
    3 528 tiles cross blocks.  No float atomics: a second call is bitwise the first."""
    dev = cuda_dev
    cin, h, cout, k, s, pad = LAYERS[layer]
    oh, t, G, Kc = strip_dims(cin, h, k, s, pad)
    K, Mg = cin * k * k, B * G * G
    first = layer == "conv1"
    rs = np.random.RandomState(B * 10 + cin + (regime == "exact"))
    x = pixels(rs, (B, cin, h, h), regime).astype(F32) if first else activations(rs, (B, cin, h, h), regime)[0]
    w_hi = weights(rs, cout, cin, k, regime)[0]
    dout, out = grads(rs, (B, cout, oh, oh), regime)
    dy = masked(dout, out)
    dyb = bf16(dy)
    grid = np.zeros((B, G, G, cout), F32)
    grid[:, :oh, :oh] = dyb.transpose(0, 2, 3, 1)
    want_dyg = bf16_bits(grid).ravel()
    S = wgrad64(x, dyb, w_hi.shape, s, pad).reshape(cout, K)
    S_mag = wgrad64(np.abs(x), np.abs(dyb), w_hi.shape, s, pad).reshape(cout, K)
    db_sum, db_mag = dy.astype(np.float64).sum((0, 2, 3)), np.abs(dy).astype(np.float64).sum((0, 2, 3))
    din_ref = din_mag = None
    if not first:
        din_ref = dgrad64(dyb, w_hi, x.shape, s, pad)
        din_mag = dgrad64(np.abs(dyb), np.abs(w_hi), x.shape, s, pad)
    d = dict(dout=to_dev(dout, dev), out=to_dev(out, dev), a_hi=to_dev_bf16(block_matrix(x, k, s, pad, first), dev),
             w_hi=to_dev_bf16(w_hi.reshape(cout, K), dev),
             perm=torch.from_numpy(strip_perm(cin, k, s, first).astype(np.int32)).to(dev))
    pre_w, pre_b = prefills(cout * K, regime, rs), prefills(cout, regime, rs)
    scales = [1.0, 2.0 ** -8] if regime == "exact" else [1.0 / 255.0 if first else 1.0]
    tag = f"{layer} B{B} {regime}"

    def run(scale):
        o = {"dYg": Out(Mg * cout, dev, BF), "dwp": Out(cout * K, dev), "dw": Out(cout * K, dev, fill=pre_w),
             "db": Out(cout, dev, fill=pre_b), "din": None if first else Out(B * cin * h * h, dev)}
        lib_call("riqn_conv_bwd_strip", geom(B, cin, h, cout, k, s, pad), dptr(d["dout"]), dptr(d["out"]),
                 dptr(d["a_hi"]), dptr(d["w_hi"]), dptr(d["perm"]), o["dYg"].p, o["dwp"].p, o["dw"].p, o["db"].p,
                 o["din"].p if o["din"] else None, float(scale))
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    for scale in scales:
        sc = np.float64(F32(scale))
        o = run(scale)
        assert_bits(f"dYg {tag}", o["dYg"].bits(), want_dyg)
        dw_ref = pre_w.astype(np.float64) + sc * S.ravel()
        db_ref = pre_b.astype(np.float64) + db_sum
        if regime == "exact":
            assert_exact_budget(f"dw {tag}", S_mag, 1.0)
            assert_exact_budget(f"dw+prefill {tag}", np.abs(pre_w) + sc * S_mag.ravel(), min(sc, 0.5))
            assert_exact_budget(f"dbias {tag}", np.abs(pre_b) + db_mag, 0.5)
            same_f32(f"dw scale {scale} {tag}", o["dw"].f32(), dw_ref)
            same_f32(f"dbias {tag}", o["db"].f32(), db_ref)
        else:
            check_bound(f"dw {tag}", o["dw"].f32(), dw_ref, C_BOUND * (Mg + 2) * U * (sc * S_mag.ravel() + np.abs(pre_w)))
            check_bound(f"dbias {tag}", o["db"].f32(), db_ref, C_BOUND * (Mg + 2) * U * (db_mag + np.abs(pre_b)))
        if not first:
            din = o["din"].f32().reshape(x.shape)
            if regime == "exact":
                assert_exact_budget(f"din {tag}", din_mag, 2.0 ** -6)
                same_f32(f"din {tag}", din, din_ref)
            else:
                check_bound(f"din {tag}", din, din_ref, C_BOUND * (cout + 1) * t * t * U * din_mag)
    if B == 512 and regime == "random":
        o2 = run(scales[-1])
        for key in o:
            if o[key] is not None and key != "dwp":
                assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())


@pytest.mark.gpu
def test_conv_bwd_strip_rejections(cuda_dev):
    dev = cuda_dev
    big = 8 * 441 * 64
    dout, out = torch.zeros(big, device=dev), torch.zeros(big, device=dev)
    a = torch.zeros(big * 2, dtype=BF, device=dev)
    w = torch.zeros(64 * 576, dtype=BF, device=dev)
    perm = torch.zeros(1024, dtype=torch.int32, device=dev)
    o = {"dYg": Out(big, dev, BF), "dwp": Out(64 * 1024, dev), "dw": Out(64 * 1024, dev, fill=prefill_pattern(64 * 1024)),
         "db": Out(64, dev, fill=prefill_pattern(64)), "din": Out(8 * 4 * 84 * 84, dev)}
    args = lambda g, din: (g, dout.data_ptr(), out.data_ptr(), a.data_ptr(), w.data_ptr(), perm.data_ptr(), o["dYg"].p,
                           o["dwp"].p, o["dw"].p, o["db"].p, din, 1.0)
    bufs = [v.t for v in o.values()]
    _expect_rejected("riqn_conv_bwd_strip", args(geom(8, 4, 84, 32, 8, 4, 1), o["din"].p), bufs)   # din with pad != 0
    _expect_rejected("riqn_conv_bwd_strip", args(geom(8, 64, 9, 60, 3, 1, 0), None), bufs)          # Cout % 8
    assert_canaries(o)


# ---------------------------------------------------------------------------------------------- 4. riqn_conv_fwd_tc
def _fwd_tc(dev, g, inp_ptr, is_u8, M, K, cout, ops, with_lo=True, with_t=True):
    o = {"col_hi": Out(M * K, dev, BF), "col_lo": Out(M * K, dev, BF) if with_lo else None,
         "colT": Out(K * M, dev, BF) if with_t else None, "out": Out(M * cout, dev)}
    lib_call("riqn_conv_fwd_tc", g, inp_ptr, is_u8, dptr(ops["w_hi"]), dptr(ops["w_lo"]), dptr(ops["bias"]),
             o["col_hi"].p, o["col_lo"].p if with_lo else None, o["colT"].p if with_t else None, o["out"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _padded_input(dev, x, bstride, offset=0):
    """x (B, ...) on the device at `offset` elements into a buffer whose samples are `bstride` elements apart"""
    B, n = x.shape[0], x[0].size
    buf = torch.zeros(offset + B * bstride + 64, dtype=torch.uint8 if x.dtype == np.uint8 else torch.float32, device=dev)
    view = buf[offset:offset + B * bstride].view(B, bstride)[:, :n]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(B, n)))
    return buf, buf.data_ptr() + offset * buf.element_size()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B", [1, 3, 8, 512])
@pytest.mark.parametrize("layer", NAMES)
def test_conv_fwd_tc(cuda_dev, layer, B, regime):
    """the im2col images col_hi / col_lo / colT_hi bitwise the bf16 split of the im2col matrix (uint8: x / 255 in fp32)
    for every input kernel: conv1 uint8 (table kernel, dense and strided), conv1 fp32 (113 KB samples: generic kernel),
    conv2 / conv3 fp32 (staged kernel; generic with the input one float off alignment; staged with a batch stride).
    All give identical bits; out (split-bf16 x3 and single) against float64"""
    dev = cuda_dev
    cin, h, cout, k, s, pad = LAYERS[layer]
    oh = out_size(h, k, s, pad)
    M, K, chw = B * oh * oh, cin * k * k, cin * h * h
    rs = np.random.RandomState(B * 3 + cin + (regime == "exact"))
    if layer == "conv1":
        px = pixels(rs, (B, cin, h, h), regime)
        x = (px.astype(F32) / F32(255)).astype(F32)
        variants = [("u8", px, chw, 0, 1), ("u8 strided", px, chw + 16, 0, 1), ("fp32", x, chw, 0, 0),
                    ("fp32 offset", x, chw, 1, 0)]
    else:
        x = np.maximum(rs.standard_normal((B, cin, h, h)), 0).astype(F32) if regime == "random" else \
            (rs.randint(0, 8, (B, cin, h, h)) + rs.randint(-1, 2, (B, cin, h, h)) * 2.0 ** -9).astype(F32)
        variants = [("staged", x, chw, 0, 0), ("generic (offset)", x, chw, 1, 0), ("staged strided", x, chw + 8, 0, 0)]
    # exact: the lo image is on the input (x = h + l * 2^-9), the weights are bf16-exact
    w = (rs.standard_normal((cout, cin, k, k)) / np.sqrt(K)).astype(F32) if regime == "random" else \
        (rs.randint(-3, 4, (cout, cin, k, k)) * 2.0 ** -6).astype(F32)
    bias = (rs.standard_normal(cout) * 0.1).astype(F32) if regime == "random" else (rs.randint(-8, 9, cout) / 64).astype(F32)
    w_hi, w_lo = split_hi_lo(w)
    ops = dict(w_hi=to_dev_bf16(w_hi.reshape(cout, K), dev), w_lo=to_dev_bf16(w_lo.reshape(cout, K), dev),
               bias=to_dev(bias, dev))
    col = im2col(x, k, s, pad)
    c_hi, c_lo = split_hi_lo(col)
    want_hi, want_lo = bf16_bits(c_hi).ravel(), bf16_bits(c_lo).ravel()
    with_t = M % 8 == 0
    x_hi, x_lo = split_hi_lo(x)
    tag = f"{layer} B{B} {regime}"
    refs = {}
    for single in (False, True):
        pairs = [(x_hi, w_hi)] if single else [(x_hi, w_hi), (x_hi, w_lo), (x_lo, w_hi)]
        refs[single] = fwd_ref(pairs, bias, s, pad)
    first = None
    for name, inp, bstride, offset, is_u8 in variants:
        buf, p = _padded_input(dev, inp, bstride, offset)
        g = geom(B, cin, h, cout, k, s, pad, bstride)
        o = _fwd_tc(dev, g, p, is_u8, M, K, cout, ops, with_t=with_t)
        assert_bits(f"col_hi {name} {tag}", o["col_hi"].bits(), want_hi)
        assert_bits(f"col_lo {name} {tag}", o["col_lo"].bits(), want_lo)
        if with_t:
            assert_bits(f"colT_hi {name} {tag}", o["colT"].bits(), want_hi.reshape(M, K).T.ravel())
        if first is None:
            first = o
            for single in (False, True):
                oo = o if not single else _fwd_tc(dev, g, p, is_u8, M, K, cout, ops, with_lo=False, with_t=False)
                ref, mag = refs[single]
                got = oo["out"].f32().reshape(B, cout, oh, oh)
                if regime == "exact" and layer != "conv1":
                    assert_exact_budget(tag, mag, 2.0 ** -15)
                    same_f32(f"out single={single} {tag}", got, ref)
                else:
                    check_bound(f"out single={single} {tag}", got, ref, fwd_bound(ref, mag, K))
        else:
            assert_bits(f"out {name} vs {variants[0][0]} {tag}", o["out"].bits(), first["out"].bits())
    if layer == "conv1" and regime == "exact":
        # integer fp32 frames: conv1's products are exact too
        xi = px.astype(F32)
        buf, p = _padded_input(dev, xi, chw)
        o = _fwd_tc(dev, geom(B, cin, h, cout, k, s, pad), p, 0, M, K, cout, ops, with_t=False)
        ref, mag = fwd_ref([(xi, w_hi), (xi, w_lo)], bias, s, pad)
        assert_exact_budget(tag, mag, 2.0 ** -6)
        same_f32(f"out integer frames {tag}", o["out"].f32().reshape(B, cout, oh, oh), ref)


@pytest.mark.gpu
def test_conv_fwd_tc_rejections(cuda_dev):
    dev = cuda_dev
    x = torch.zeros(8 * 64 * 9 * 9, device=dev)
    w = torch.zeros(64 * 576, dtype=BF, device=dev)
    bias = torch.zeros(64, device=dev)
    o = {"col_hi": Out(8 * 49 * 576, dev, BF), "col_lo": Out(8 * 49 * 576, dev, BF), "colT": Out(8 * 49 * 576, dev, BF),
         "out": Out(8 * 64 * 49, dev)}
    args = lambda g: (g, x.data_ptr(), 0, w.data_ptr(), w.data_ptr(), bias.data_ptr(), o["col_hi"].p, o["col_lo"].p,
                      o["colT"].p, o["out"].p)
    bufs = [v.t for v in o.values()]
    _expect_rejected("riqn_conv_fwd_tc", args(geom(2, 3, 9, 16, 3, 1, 0)), bufs)     # K = 27, K % 8
    _expect_rejected("riqn_conv_fwd_tc", args(geom(1, 64, 9, 64, 3, 1, 0)), bufs)    # colT_hi with M = 49
    assert_canaries(o)


# ---------------------------------------------------------------------------------------------- 5. riqn_conv_bwd_tc
# conv2 / conv3 (pad 0: fused TC_COL2IM), Cout 96 (conv_dy_bf16_kernel), pad 1 (dcol + col2im)
BWD_TC = {"conv2": (32, 20, 64, 4, 2, 0), "conv3": (64, 9, 64, 3, 1, 0), "cout96": (64, 9, 96, 3, 1, 0),
          "pad1": (32, 20, 64, 4, 2, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B", [8, 512])
@pytest.mark.parametrize("name", list(BWD_TC))
def test_conv_bwd_tc(cuda_dev, name, B, regime):
    """dY_hi / dYT_hi bitwise; dw (split over every SM, added in split order) and dbias accumulated from a prefill;
    din (dcol gathered in a fixed order) bitwise in the exact regime and bounded in the random one, where a second call
    is bitwise the first.  A call without din writes the same dYT_hi, dw and dbias and leaves dY_hi alone."""
    dev = cuda_dev
    cin, h, cout, k, s, pad = BWD_TC[name]
    oh = out_size(h, k, s, pad)
    M, K = B * oh * oh, cin * k * k
    rs = np.random.RandomState(B + cout + pad + (regime == "exact"))
    x = activations(rs, (B, cin, h, h), regime)[0]
    w_hi = weights(rs, cout, cin, k, regime)[0]
    dout, out = grads(rs, (B, cout, oh, oh), regime)
    dy = masked(dout, out)
    dyb = bf16(dy)
    dym = dyb.transpose(0, 2, 3, 1).reshape(M, cout)
    col = bf16(im2col(x, k, s, pad))                  # x is bf16 already: col is exact
    scale = 2.0 ** -8 if regime == "exact" else 1.0
    S = dym.astype(np.float64).T @ col.astype(np.float64)
    S_mag = np.abs(dym).astype(np.float64).T @ np.abs(col).astype(np.float64)
    pre_w, pre_b = prefills(cout * K, regime, rs), prefills(cout, regime, rs)
    dw_ref = pre_w.astype(np.float64) + scale * S.ravel()
    db_ref = pre_b.astype(np.float64) + dy.astype(np.float64).sum((0, 2, 3))
    db_mag = np.abs(pre_b) + np.abs(dy).astype(np.float64).sum((0, 2, 3))
    din_ref = dgrad64(dyb, w_hi, x.shape, s, pad)
    din_mag = dgrad64(np.abs(dyb), np.abs(w_hi), x.shape, s, pad)
    d = dict(dout=to_dev(dout, dev), out=to_dev(out, dev), colT=to_dev_bf16(np.ascontiguousarray(col.T), dev),
             wT=to_dev_bf16(np.ascontiguousarray(w_hi.reshape(cout, K).T), dev))
    tag = f"{name} B{B} {regime}"

    def run(with_din):
        o = {"dY": Out(M * cout, dev, BF), "dYT": Out(cout * M, dev, BF), "dcol": Out(M * K, dev),
             "dw": Out(cout * K, dev, fill=pre_w), "db": Out(cout, dev, fill=pre_b),
             "din": Out(B * cin * h * h, dev) if with_din else None}
        lib_call("riqn_conv_bwd_tc", geom(B, cin, h, cout, k, s, pad), dptr(d["dout"]), dptr(d["out"]), dptr(d["colT"]),
                 dptr(d["wT"]), o["dY"].p, o["dYT"].p, o["dcol"].p, o["dw"].p, o["db"].p,
                 o["din"].p if with_din else None, float(scale))
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = run(True)
    assert_bits(f"dY_hi {tag}", o["dY"].bits(), bf16_bits(dym).ravel())
    assert_bits(f"dYT_hi {tag}", o["dYT"].bits(), bf16_bits(np.ascontiguousarray(dym.T)).ravel())
    din = o["din"].f32().reshape(x.shape)
    if regime == "exact":
        assert_exact_budget(f"dw {tag}", S_mag, 1.0)
        assert_exact_budget(f"dw+prefill {tag}", np.abs(pre_w) + scale * S_mag.ravel(), scale)
        assert_exact_budget(f"dbias {tag}", db_mag, 0.5)
        assert_exact_budget(f"din {tag}", din_mag, 2.0 ** -6)
        same_f32(f"dw {tag}", o["dw"].f32(), dw_ref)
        same_f32(f"dbias {tag}", o["db"].f32(), db_ref)
        same_f32(f"din {tag}", din, din_ref)
    else:
        check_bound(f"dw {tag}", o["dw"].f32(), dw_ref, C_BOUND * (M + 2) * U * (S_mag.ravel() + np.abs(pre_w)))
        check_bound(f"dbias {tag}", o["db"].f32(), db_ref, C_BOUND * (M + 2) * U * db_mag)
        check_bound(f"din {tag}", din, din_ref, C_BOUND * (cout + k * k) * U * din_mag)
        again = run(True)
        for key in o:
            assert_bits(f"second call {key}", again[key].bits(), o[key].bits())
    o2 = run(False)
    assert torch.isnan(o2["dY"].t[:o2["dY"].n].float()).all(), "dY_hi written without din"
    for key in ("dYT", "dw", "db"):
        assert_bits(f"without din {key}", o2[key].bits(), o[key].bits())


@pytest.mark.gpu
def test_conv_bwd_tc_rejections(cuda_dev):
    dev = cuda_dev
    n = 8 * 64 * 81
    dout, out = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    colT, wT = torch.zeros(576 * 8 * 49, dtype=BF, device=dev), torch.zeros(576 * 64, dtype=BF, device=dev)
    o = {"dY": Out(8 * 49 * 64, dev, BF), "dYT": Out(8 * 49 * 64, dev, BF), "dcol": Out(8 * 49 * 576, dev),
         "dw": Out(64 * 576, dev, fill=prefill_pattern(64 * 576)), "db": Out(64, dev, fill=prefill_pattern(64)),
         "din": Out(8 * 64 * 81, dev)}
    args = lambda g: (g, dout.data_ptr(), out.data_ptr(), colT.data_ptr(), wT.data_ptr(), o["dY"].p, o["dYT"].p,
                      o["dcol"].p, o["dw"].p, o["db"].p, o["din"].p, 1.0)
    bufs = [v.t for v in o.values()]
    _expect_rejected("riqn_conv_bwd_tc", args(geom(1, 64, 9, 64, 3, 1, 0)), bufs)     # M = 49, M % 8
    _expect_rejected("riqn_conv_bwd_tc", args(geom(8, 64, 9, 60, 3, 1, 0)), bufs)     # Cout % 8
    no_dcol = list(args(geom(8, 64, 9, 64, 3, 1, 0)))
    no_dcol[7] = None
    _expect_rejected("riqn_conv_bwd_tc", tuple(no_dcol), bufs)                       # din without dcol
    assert_canaries(o)


# ---------------------------------------------------------------------------------------------- 6. fp32 CUDA cores
# the Atari layers (conv1 from uint8 frames in the random regime), and a 116 x 116 image whose channel plane (53 KB)
# takes the non-tile col2im_kernel
F32_GEOMS = dict(LAYERS, big=(2, 116, 8, 4, 2, 1))
F32_CASES = [(n, B, r) for n in F32_GEOMS for B in (1, 3, 8, 512) for r in ("exact", "random") if not (n == "big" and B > 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,regime", F32_CASES, ids=[f"{n}-B{b}-{r}" for n, b, r in F32_CASES])
def test_conv_fp32(cuda_dev, name, B, regime):
    """riqn_im2col_f32 and riqn_conv_fwd's col: bitwise (a gather and a correctly rounded /255); riqn_conv_fwd's out;
    riqn_conv_bwd's dY bitwise, dbias / dw accumulated (bitwise in the exact regime), din through col2im; in the random
    regime a second backward call is bitwise the first"""
    dev = cuda_dev
    cin, h, cout, k, s, pad = F32_GEOMS[name]
    oh = out_size(h, k, s, pad)
    M, K = B * oh * oh, cin * k * k
    rs = np.random.RandomState(B * 5 + cin + (regime == "exact"))
    u8 = name == "conv1" and regime == "random"
    if u8:
        px = pixels(rs, (B, cin, h, h), regime)
        xd, x = torch.from_numpy(px).to(dev), (px.astype(F32) / F32(255)).astype(F32)
    else:
        x = activations(rs, (B, cin, h, h), regime)[0]
        if regime == "random":
            x = np.maximum(rs.standard_normal((B, cin, h, h)), 0).astype(F32)
        xd = to_dev(x, dev)
    w, _, bias = weights(rs, cout, cin, k, regime)
    if regime == "random":
        w = (rs.standard_normal(w.shape) / np.sqrt(K)).astype(F32)
    wd, bd = to_dev(w, dev), to_dev(bias, dev)
    g = geom(B, cin, h, cout, k, s, pad)
    tag = f"{name} B{B} {regime}"
    want_col = f32_bits(im2col(x, k, s, pad)).ravel()
    col0 = Out(M * K, dev)
    lib_call("riqn_im2col_f32", g, xd.data_ptr(), int(u8), col0.p)
    col, fo = Out(M * K, dev), Out(B * cout * oh * oh, dev)
    lib_call("riqn_conv_fwd", g, xd.data_ptr(), int(u8), dptr(wd), dptr(bd), col.p, fo.p)
    torch.cuda.synchronize()
    assert_canaries({"col0": col0, "col": col, "out": fo})
    assert_bits(f"im2col_f32 {tag}", col0.bits(), want_col)
    assert_bits(f"conv_fwd col {tag}", col.bits(), want_col)
    ref, mag = fwd_ref([(x, w)], bias, s, pad)
    exact = regime == "exact"
    if exact:
        assert_exact_budget(tag, mag, 2.0 ** -6)
        same_f32(f"out {tag}", fo.f32().reshape(ref.shape), ref)
    else:
        check_bound(f"out {tag}", fo.f32().reshape(ref.shape), ref, fwd_bound(ref, mag, K))
    # backward on the forward's col
    dout, out = grads(rs, (B, cout, oh, oh), regime)
    dy = masked(dout, out)
    pre_w, pre_b = prefills(cout * K, regime, rs), prefills(cout, regime, rs)
    doutd, outd = to_dev(dout, dev), to_dev(out, dev)

    def bwd():
        o = {"dY": Out(M * cout, dev), "dcol": Out(M * K, dev), "dw": Out(cout * K, dev, fill=pre_w),
             "db": Out(cout, dev, fill=pre_b), "din": Out(B * cin * h * h, dev)}
        lib_call("riqn_conv_bwd", g, dptr(doutd), dptr(outd), col.p, dptr(wd), o["dY"].p, o["dcol"].p, o["dw"].p,
                 o["db"].p, o["din"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = bwd()
    assert_bits(f"dY {tag}", o["dY"].bits(), f32_bits(dy.transpose(0, 2, 3, 1)).ravel())
    dw_ref = pre_w.astype(np.float64) + wgrad64(x, dy, w.shape, s, pad).ravel()
    dw_mag = np.abs(pre_w) + wgrad64(np.abs(x), np.abs(dy), w.shape, s, pad).ravel()
    db_ref = pre_b.astype(np.float64) + dy.astype(np.float64).sum((0, 2, 3))
    db_mag = np.abs(pre_b) + np.abs(dy).astype(np.float64).sum((0, 2, 3))
    din_ref = dgrad64(dy, w, x.shape, s, pad)
    din_mag = dgrad64(np.abs(dy), np.abs(w), x.shape, s, pad)
    din = o["din"].f32().reshape(x.shape)
    if exact:
        for what, m, q in (("dw", dw_mag, 0.5), ("dbias", db_mag, 0.5), ("din", din_mag, 2.0 ** -6)):
            assert_exact_budget(f"{what} {tag}", m, q)
        same_f32(f"dw {tag}", o["dw"].f32(), dw_ref)
        same_f32(f"dbias {tag}", o["db"].f32(), db_ref)
        same_f32(f"din {tag}", din, din_ref)
    else:
        check_bound(f"dw {tag}", o["dw"].f32(), dw_ref, C_BOUND * (M + 2) * U * dw_mag)
        check_bound(f"dbias {tag}", o["db"].f32(), db_ref, C_BOUND * (M + 2) * U * db_mag)
        check_bound(f"din {tag}", din, din_ref, C_BOUND * (cout + k * k) * U * din_mag)
        again = bwd()
        for key in o:
            assert_bits(f"second call {key}", again[key].bits(), o[key].bits())


# ---------------------------------------------------------------------------------------------- 7. small helpers
@pytest.mark.gpu
@pytest.mark.parametrize("scale", [255.0, 1.0, 3.0])
@pytest.mark.parametrize("rows,cols", [(32, 256), (64, 576), (7, 13), (1, 1)])
def test_split_bf16_scaled(cuda_dev, rows, cols, scale):
    """hi = bf16(fl(src / scale)), lo = bf16(fl(src / scale) - hi), the division correctly rounded; lo == NULL writes hi
    only"""
    dev = cuda_dev
    rs = np.random.RandomState(rows * cols + int(scale))
    n = rows * cols
    src = (rs.standard_normal(n) * np.exp2(rs.randint(-20, 20, n))).astype(F32)
    special = np.array([0.0, -0.0, 255.0, -255.0, 1e-38, 2.0 ** -140, 3e38, 1.0 / 3.0], F32)
    src[:min(n, special.size)] = special[:min(n, special.size)]
    x = (src / F32(scale)).astype(F32)
    hi = bf16(x)
    o = {"hi": Out(n, dev, BF), "lo": Out(n, dev, BF)}
    sd = to_dev(src, dev)
    lib_call("riqn_split_bf16_scaled", rows, cols, dptr(sd), float(scale), o["hi"].p, o["lo"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    assert_bits("hi", o["hi"].bits(), bf16_bits(x))
    assert_bits("lo", o["lo"].bits(), bf16_bits((x - hi).astype(F32)))
    o2 = {"hi": Out(n, dev, BF), "lo": Out(n, dev, BF)}
    lib_call("riqn_split_bf16_scaled", rows, cols, dptr(sd), float(scale), o2["hi"].p, None)
    torch.cuda.synchronize()
    assert_canaries(o2)
    assert_bits("hi without lo", o2["hi"].bits(), o["hi"].bits())
    assert torch.isnan(o2["lo"].t[:n].float()).all(), "lo written though NULL"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 5, 1000, 70001])
def test_zero_f32(cuda_dev, n):
    o = Out(n, cuda_dev)
    lib_call("riqn_zero_f32", o.p, n)
    torch.cuda.synchronize()
    assert_canaries({"p": o})
    assert_bits("zeros", o.bits(), np.zeros(n, np.uint32))


# ---------------------------------------------------------------------------------------------- CPU: the statements
@pytest.mark.parametrize("layer", NAMES)
def test_reference_statements_match_conv2d(layer):
    """The numpy / float64 statements above against torch's conv2d and autograd: the block matrix with the strip
    permutation and the row shifts is the convolution; the strip weight gradient over the grid (zeros off the real
    outputs) maps back through the permutation; the next layer's block image of an output is the block matrix of that
    layer's input; im2col times the weight is the convolution; wgrad64 / dgrad64 are autograd's gradients; fp32
    arithmetic stays inside the random-regime bounds; the exact regime's inputs give fp32 results equal to float64."""
    cin, h, cout, k, s, pad = LAYERS[layer]
    first = layer == "conv1"
    oh, t, G, Kc = strip_dims(cin, h, k, s, pad)
    K = cin * k * k
    B = 2
    rs = np.random.RandomState(cin)
    x = rs.standard_normal((B, cin, h, h))
    w = rs.standard_normal((cout, cin, k, k))
    ref = conv64(x, w, s, pad)
    A = block_matrix(x, k, s, pad, first)
    assert A.shape == (B * G * G, Kc)
    perm = strip_perm(cin, k, s, first)
    wp = w.reshape(cout, K)[:, perm]
    rows = A.shape[0]
    Apad = np.concatenate([A, np.zeros((t * G + t, Kc))])                # rows past the end: TMA zero fill
    acc = np.zeros((rows, cout))
    for dy in range(t):
        for dx in range(t):
            sft = dy * t + dx
            acc += Apad[dy * G + dx: dy * G + dx + rows] @ wp[:, sft * Kc:(sft + 1) * Kc].T
    got = acc.reshape(B, G, G, cout)[:, :oh, :oh].transpose(0, 3, 1, 2)
    assert np.allclose(got, ref, rtol=1e-10, atol=1e-10)
    # weight and data gradient statements against autograd
    dy_ = rs.standard_normal(ref.shape)
    xt = torch.from_numpy(x).requires_grad_(True)
    wt = torch.from_numpy(w).requires_grad_(True)
    F.conv2d(xt, wt, stride=s, padding=pad).backward(torch.from_numpy(dy_))
    assert np.allclose(wgrad64(x, dy_, w.shape, s, pad), wt.grad.numpy(), rtol=1e-10, atol=1e-9)
    assert np.allclose(dgrad64(dy_, w, x.shape, s, pad), xt.grad.numpy(), rtol=1e-10, atol=1e-9)
    grid = np.zeros((B, G, G, cout))
    grid[:, :oh, :oh] = dy_.transpose(0, 2, 3, 1)
    dYg = grid.reshape(rows, cout)
    dwp = np.concatenate([dYg.T @ Apad[(sft // t) * G + sft % t:(sft // t) * G + sft % t + rows] for sft in range(t * t)], 1)
    dw = np.zeros((cout, K))
    dw[:, perm] += dwp
    assert np.allclose(dw, wt.grad.numpy().reshape(cout, K), rtol=1e-9, atol=1e-9)
    # im2col statement
    col = im2col(x, k, s, pad)
    assert np.allclose((col @ w.reshape(cout, K).T).reshape(B, oh, oh, cout).transpose(0, 3, 1, 2), ref, atol=1e-10)
    # the next layer's block image of this layer's output: the next layer's input in (iy, ix, c) order
    lay = _next_layout(layer)
    if lay is not None:
        ns, nG, nKc, nk = lay
        nb = block_matrix(ref, nk, ns, 0, False).reshape(B, nG, nG, ns, ns, cout)
        assert np.array_equal(nb[:, 2, 1, ns - 1, 0, 5], ref[:, 5, 2 * ns + ns - 1, 1 * ns])
    # fp32 arithmetic inside the random-regime bound; exact-regime inputs give fp32 == float64
    x32, w32 = x.astype(F32), w.astype(F32)
    conv32 = lambda a, b: (im2col(a, k, s, pad) @ b.reshape(cout, K).T).reshape(B, oh, oh, cout).transpose(0, 3, 1, 2)
    f32 = conv32(x32, w32)
    r64, mag = fwd_ref([(x32, w32)], np.zeros(cout, F32), s, pad)
    check_bound(f"fp32 conv {layer}", np.maximum(f32, 0), r64, fwd_bound(r64, mag, K))
    xe_hi, xe_lo = activations(rs, (B, cin, h, h), "exact", lo=True)
    we_hi, we_lo, be = weights(rs, cout, cin, k, "exact", lo=True)
    for xe, we in ((xe_hi, we_hi), (xe_hi, we_lo), (xe_lo, we_hi)):
        e32 = conv32(xe, we)
        assert np.array_equal(e32.astype(np.float64), conv64(xe, we, s, pad))


def test_s2d_statement_on_raw_pixels():
    """The pixel block matrix of the Atari frames holds every pixel the convolution reads exactly once per block row
    position, in (c, iy, ix) order, with zeros at the padded border; the generic geometries tile their input exactly."""
    rs = np.random.RandomState(0)
    x = rs.randint(0, 256, (2, 4, 84, 84)).astype(F32)
    A = block_matrix(x, 8, 4, 1, True).reshape(2, 21, 21, 4, 4, 4)      # b gy gx c iy ix
    assert np.all(A[:, 0, :, :, 0, :] == 0) and np.all(A[:, :, 0, :, :, 0] == 0)
    assert A[1, 3, 5, 2, 1, 2] == x[1, 2, 3 * 4 + 1 - 1, 5 * 4 + 2 - 1]
    for name, (cin, h, cout, k, s, pad) in S2D_GEOMS.items():
        oh, t, G, Kc = strip_dims(cin, h, k, s, pad)
        xg = rs.randint(0, 256, (1, cin, h, h)).astype(F32)
        Ag = block_matrix(xg, k, s, pad, True)
        assert Ag.shape == (G * G, Kc) and Kc % 64 == 0, name
        assert np.isclose(Ag.sum(), xg[:, :, :G * s - pad, :G * s - pad].sum()), name
