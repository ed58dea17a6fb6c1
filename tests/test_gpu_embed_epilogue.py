"""riqn_quantile_embed_fwd_tc's epilogue: x = feat[r // Nq] * relu(cos W_e^T + b_e) is formed in the accumulator
fragments, where a thread holds rows fr and fr + 8 of its warpgroup's 64 and the column pairs 8 j + 2 (lane % 4) + {0, 1},
and leaves through 64-row x 32-column boxes staged in the 64-byte-swizzle layout.  test_gpu_head_kernels.py holds the
images at the learner's shapes; this file covers what that indexing can get wrong elsewhere:

* rows per sample 1, 2, 8, 24, 32, 64 and 200: a thread's two rows, a warp's 16 rows and a warpgroup's 64 rows fall in
  one, two and many samples, and the feature rows of neighbouring samples differ in sign and by factors of two;
* R = B * Nq below 64, and not a multiple of 64 or 128 (the last tile's rows are clipped by the TMA store and guarded
  in the fp32 store); F = 160 ends in a 32-column tile (one chunk of four), F = 3136 with E = 72 has a k-tail;
* fp16 images with and without the bf16 image, bf16 hi with and without the residual, single and split cos operands,
  each with and without the fp32 x;
* outputs start as NaN and carry canaries, a second call must repeat every bit, and rejected calls write nothing.

Two value-only mutants the cases are aimed at (neither moves a store, both pass at the learner's shapes):
* feat indexed by row fr for both fragment rows: wrong only where rows fr and fr + 8 belong to different samples
  (rows per sample 1, 2, 8, 24 and 200 here);
* the swizzle term of the staging address taken as r & 3 instead of (r >> 1) & 3 (the term is the same for rows r and
  r + 8, so only its form can be wrong): 16-byte pieces of odd rows change places inside their 64-byte row, which the
  column-dependent bias and weights of every case show.

Expected values: the 16-bit images are the float32 statement rounded once, taken from the fp32 x the same call returned;
the fp32 x is held against float64 on the kernel's own operand images with the bound of test_gpu_head_kernels.py; in the
exact regime (tau = 0, so cos = 1 exactly; small integer weights, power-of-two features) float64 is matched bit for bit.
"""
import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, bf16, bf16_bits, check_bound, dptr, f16_bits, f32_bits,
                     lib_call, to_dev, to_dev_bf16)

C_BOUND = 2.0
# (B, Nq, F, E): R = 38, 150, 150, 200, 168, 160, 192, 600, and one 3136-wide case with a k-tail and R = 40
SHAPES = [(38, 1, 160, 64), (150, 1, 160, 64), (75, 2, 160, 64), (25, 8, 160, 64), (7, 24, 160, 64), (5, 32, 160, 64),
          (3, 64, 160, 64), (3, 200, 160, 64), (5, 8, 3136, 72)]
# (x_fp16, split cos operands, second image)
MODES = {"fp16+bf16": (1, True, True), "fp16": (1, True, False), "hi+lo": (0, True, True), "hi": (0, True, False),
         "hi+lo-single": (0, False, True), "fp16-single": (1, False, False)}


def _inputs(B, Nq, F, E, seed, exact=False):
    rs = np.random.RandomState(seed)
    R = B * Nq
    sign = np.where(np.arange(B) % 2 == 0, 1.0, -1.0)[:, None]
    if exact:
        tau = np.zeros(R, np.float32)                                    # cos(0) = 1 in every column of every row
        feat = sign * 2.0 ** (np.arange(B) % 5 - 2)[:, None] * rs.randint(1, 8, (B, F))
        w = rs.randint(-3, 4, (F, E))
        be = rs.randint(-8, 9, F) * 0.5
    else:
        tau = rs.uniform(0, 1, R)
        feat = sign * 2.0 ** (np.arange(B) % 5)[:, None] * (0.25 + np.abs(rs.standard_normal((B, F))))
        w = rs.standard_normal((F, E)) * 0.2
        be = rs.standard_normal(F) * 0.3
    tau, feat, w, be = (np.ascontiguousarray(a, np.float32) for a in (tau, feat, w, be))
    w_hi = bf16(w)
    return dict(tau=tau, feat=feat, w_hi=w_hi, w_lo=bf16(w - w_hi), be=be)


def _reference(host, cos_hi, cos_lo, Nq):
    """float64 x on the operand images, and the magnitude sum|a_i b_i| + |b_e| its bound scales with"""
    ch, wh = cos_hi.astype(np.float64), host["w_hi"].astype(np.float64)
    be = host["be"].astype(np.float64)
    pre, mag, k = ch @ wh.T + be, np.abs(ch) @ np.abs(wh).T + np.abs(be), ch.shape[1] + 2
    if cos_lo is not None:
        cl, wl = cos_lo.astype(np.float64), host["w_lo"].astype(np.float64)
        pre += ch @ wl.T + cl @ wh.T
        mag += np.abs(ch) @ np.abs(wl).T + np.abs(cl) @ np.abs(wh).T
        k = 3 * ch.shape[1] + 2
    f = host["feat"][np.arange(ch.shape[0]) // Nq].astype(np.float64)
    return f * np.maximum(pre, 0), mag * np.abs(f), k


def _images(x32, x_fp16):
    """bit patterns of the two 16-bit images of a float32 x"""
    if x_fp16:
        return f16_bits(x32), bf16_bits(x32)
    hi = bf16(x32)
    return bf16_bits(x32), bf16_bits(x32 - hi)


def test_exact_regime_is_exact_in_fp32():
    """the premise of the bitwise cases: float32 evaluation in either summation order equals float64"""
    B, Nq, F, E = 5, 8, 160, 72
    host = _inputs(B, Nq, F, E, 3, exact=True)
    ones = np.ones((B * Nq, E), np.float32)
    ref, _, _ = _reference(host, ones, np.zeros_like(ones), Nq)
    for order in (slice(None), slice(None, None, -1)):
        pre = np.zeros((B * Nq, F), np.float32)
        for k in np.arange(E)[order]:
            pre += ones[:, k:k + 1] * host["w_hi"][None, :, k]
        x = host["feat"][np.arange(B * Nq) // Nq] * np.maximum(pre + host["be"], np.float32(0))
        assert x.dtype == np.float32
        assert_bits("fp32 statement vs float64", f32_bits(x), f32_bits(ref.astype(np.float32)))
    assert np.all(ref == ref.astype(np.float32)) and np.all(host["w_lo"] == 0)
    hi_bits, lo_bits = _images(ref.astype(np.float32), 0)
    assert hi_bits.shape == lo_bits.shape == (B * Nq, F)


def _call(dev, B, Nq, F, E, mode, dev_in, with_x32):
    x_fp16, split, second = MODES[mode]
    R = B * Nq
    o = {"cos_hi": Out(R * E, dev, torch.bfloat16), "cos_lo": Out(R * E, dev, torch.bfloat16) if split else None,
         "x32": Out(R * F, dev) if with_x32 else None,
         "x_hi": Out(R * F, dev, torch.float16 if x_fp16 else torch.bfloat16),
         "x_lo": Out(R * F, dev, torch.bfloat16) if second else None}
    p = {k: (v.p if v is not None else None) for k, v in o.items()}
    lib_call("riqn_quantile_embed_fwd_tc", B, Nq, E, F, dptr(dev_in["tau"]), dptr(dev_in["feat"]), dptr(dev_in["w_hi"]),
             dptr(dev_in["w_lo"]), dptr(dev_in["be"]), p["cos_hi"], p["cos_lo"], None, p["x32"], p["x_hi"], p["x_lo"],
             None, None, x_fp16)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _to_device(host, dev):
    d = {k: to_dev(host[k], dev) for k in ("tau", "feat", "be")}
    d.update(w_hi=to_dev_bf16(host["w_hi"], dev), w_lo=to_dev_bf16(host["w_lo"], dev))
    return d


def _check(dev, B, Nq, F, E, mode, exact):
    x_fp16, split, second = MODES[mode]
    R = B * Nq
    host = _inputs(B, Nq, F, E, seed=1000 * B + Nq, exact=exact)
    dev_in = _to_device(host, dev)
    o = _call(dev, B, Nq, F, E, mode, dev_in, True)
    x32 = o["x32"].f32().reshape(R, F)
    ch = o["cos_hi"].f32().reshape(R, E)
    cl = o["cos_lo"].f32().reshape(R, E) if split else None
    ref, mag, k = _reference(host, ch, cl, Nq)
    if exact:
        assert np.all(ch == 1) and (cl is None or np.all(cl == 0))
        assert_bits(f"x32 {mode} exact", f32_bits(x32), f32_bits(ref.astype(np.float32)))
    else:
        check_bound(f"x32 {mode} Nq={Nq}", x32, ref, C_BOUND * k * U * mag + U * np.abs(ref))
    hi_bits, lo_bits = _images(x32, x_fp16)
    assert_bits(f"x_hi {mode}", o["x_hi"].bits().reshape(R, F), hi_bits)
    if second:
        assert_bits(f"x_lo {mode}", o["x_lo"].bits().reshape(R, F), lo_bits)
    again, without = _call(dev, B, Nq, F, E, mode, dev_in, True), _call(dev, B, Nq, F, E, mode, dev_in, False)
    for key, v in o.items():
        if v is not None:
            assert_bits(f"second call {key}", again[key].bits(), v.bits())
            if key != "x32":
                assert_bits(f"without x32 {key}", without[key].bits(), v.bits())


_IDS = [f"B{b}-Nq{n}-F{f}-E{e}" for b, n, f, e in SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("B,Nq,F,E", SHAPES, ids=_IDS)
def test_embed_epilogue_random(cuda_dev, B, Nq, F, E, mode):
    _check(cuda_dev, B, Nq, F, E, mode, exact=False)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp16+bf16", "hi+lo", "hi+lo-single"])
@pytest.mark.parametrize("B,Nq,F,E", SHAPES, ids=_IDS)
def test_embed_epilogue_exact(cuda_dev, B, Nq, F, E, mode):
    _check(cuda_dev, B, Nq, F, E, mode, exact=True)


@pytest.mark.gpu
def test_embed_epilogue_rejects_before_writing(cuda_dev):
    """feat or the bias off an 8-byte boundary (the epilogue reads them as column pairs), odd R and F % 32 are refused
    before the cos images are written: every output keeps its NaN fill"""
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    for B, Nq, F, shifted in [(4, 2, 96, "feat"), (4, 2, 96, "be"), (3, 3, 96, None), (4, 2, 80, None)]:
        R, E = B * Nq, 64
        host = _inputs(B, Nq, F, E, seed=R)
        dev_in = _to_device(host, dev)
        if shifted:                                   # the same values one float further on
            wide = torch.zeros(dev_in[shifted].numel() + 1, device=dev)
            wide[1:] = dev_in[shifted].reshape(-1)
            dev_in[shifted] = wide[1:]
            assert dev_in[shifted].data_ptr() % 8 == 4
        o = {"cos_hi": Out(R * E, dev, torch.bfloat16), "cos_lo": Out(R * E, dev, torch.bfloat16), "x32": Out(R * F, dev),
             "x_hi": Out(R * F, dev, torch.float16), "x_lo": Out(R * F, dev, torch.bfloat16)}
        with pytest.raises(RiqnError):
            lib_call("riqn_quantile_embed_fwd_tc", B, Nq, E, F, dptr(dev_in["tau"]), dptr(dev_in["feat"]),
                     dptr(dev_in["w_hi"]), dptr(dev_in["w_lo"]), dptr(dev_in["be"]), o["cos_hi"].p, o["cos_lo"].p, None,
                     o["x32"].p, o["x_hi"].p, o["x_lo"].p, None, None, 1)
        torch.cuda.synchronize()
        assert_canaries(o)
        for key, v in o.items():
            assert torch.isnan(v.t[:v.n].float()).all(), f"rejected call {(B, Nq, F, shifted)} wrote {key}"
