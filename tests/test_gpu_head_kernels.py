"""The IQN head's embedding and backward kernels, entry point by entry point, against float64 statements of the same
operations (include/riqn_b200.h): riqn_quantile_embed_fwd_tc, riqn_quantile_embed_bwd_tc, riqn_dueling_bwd[_bf16],
riqn_dueling_bwd_dense[_bf16], riqn_z_wgrad[_tc] and riqn_noisy_bias_grad.

Method:
* every reference is computed on the operand images the kernel consumed (its bf16 / fp16 images, and the three
  partial products hi*hi + hi*lo + lo*hi of a split-bf16 product), so the kernel's input rounding is not part of any
  comparison;
* exact regime: small integer inputs and power-of-two scales make every product and partial sum exact in fp32 in any
  summation order, so the kernel has to match float64 bit for bit -- a dropped, duplicated or shifted row, split,
  slot or sample shows up;
* random regime: Gaussian inputs with ReLU zeros; each element is held to c * K * 2^-24 * sum|a_i b_i| (K = the
  reduction length) plus the output rounding, and each test prints its worst err/bound ratio;
* where the kernel's value is one correctly rounded fp32 operation (or a chain without a multiply feeding an add: the
  library builds with FMA contraction on) it is asserted bit for bit through the rounding helpers of helpers.py;
* overwritten outputs start as NaN, accumulated outputs start from a known non-zero pattern, and every output buffer
  carries canaries past its end that must survive.
"""
import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, bf16, bf16_bits, check_bound, dptr, f16_bits, f32_bits,
                     lib_call, prefill_pattern, to_dev, to_dev_bf16)

C_BOUND = 2.0           # the constant c of the random-regime bounds
HID = 512


# ---------------------------------------------------------------------------------------------- helpers without a GPU
def _torch_bits(x, dtype):
    return torch.from_numpy(np.asarray(x, np.float32)).to(dtype).view(torch.int16).numpy().view(np.uint16)


def _special_f32(bit_patterns, values):
    a = np.array(bit_patterns, np.uint32).view(np.float32)
    return np.concatenate([a, -a, np.array(values, np.float32), -np.array(values, np.float32)])


def test_bf16_helper_matches_torch():
    x = _special_f32(
        [0x00000000, 0x00000001, 0x00007FFF, 0x00008000, 0x00008001, 0x00018000, 0x007F8000, 0x007FFFFF,  # subnormals
         0x00800000, 0x3F808000, 0x3F818000, 0x3F808001, 0x3F7F8000, 0x3F7FFFFF,                         # ties
         0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0x7F7F0000, 0x7F800000],                                    # near max, inf
        [1.0, 0.5, 3.0, 256.0, 1e-30, 3.3895314e38])
    rs = np.random.RandomState(0)
    r = rs.randint(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    x = np.concatenate([x, r[np.isfinite(r)], rs.standard_normal(10000).astype(np.float32)])
    assert_bits("bf16 bits", bf16_bits(x), _torch_bits(x, torch.bfloat16))
    assert_bits("bf16 values", f32_bits(bf16(x)), f32_bits(torch.from_numpy(x).to(torch.bfloat16).float().numpy()))


def test_fp16_helper_matches_torch():
    h = [2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11,
         65504.0, 65519.0, 65519.996, 65520.0, 1e5, 0.0, 1.0, 1e-9]
    rs = np.random.RandomState(1)
    x = np.concatenate([_special_f32([0x7F800000], h), rs.standard_normal(100000).astype(np.float32) * 100,
                        rs.standard_normal(100000).astype(np.float32) * 1e-5])
    assert_bits("fp16 bits", f16_bits(x), _torch_bits(x, torch.float16))


def test_rounding_helpers_keep_signed_zero():
    x = np.array([0.0, -0.0], np.float32)
    assert list(bf16_bits(x)) == [0x0000, 0x8000]
    assert list(f16_bits(x)) == [0x0000, 0x8000]


# ---------------------------------------------------------------------------------------------- quantile embedding forward
PI32 = np.float32(3.14159274101257324)
FWD_SHAPES = [(4, 1, 96, 64), (6, 3, 96, 72), (5, 8, 3136, 64), (4, 24, 96, 64), (2, 32, 3136, 72), (6, 33, 96, 64),
              (3, 64, 3136, 64), (2, 200, 96, 72)]           # (B, Nq, F, E); R < 128, ragged R % 128, E = 72 k-tail
FWD_MODES = ["fp16-xlo", "fp16", "bf16x3", "bf16", "bf16x3-transposed"]


def _cos_ref(tau, B, Nq, E):
    """float64 cos of the fp32 argument fl(fl(i*pi32)*tau), sample-major rows, quantile-major tau"""
    R = B * Nq
    r = np.arange(R)
    t = tau[(r % Nq) * B + r // Nq]
    ipi = (np.arange(1, E + 1, dtype=np.float32) * PI32).astype(np.float32)
    arg = (ipi[None, :] * t[:, None]).astype(np.float32)
    return np.cos(arg.astype(np.float64))


def _embed_fwd_call(dev, B, Nq, F, E, mode, inp, x32=True):
    R = B * Nq
    split = mode != "bf16"
    f16 = mode.startswith("fp16")
    trans = mode == "bf16x3-transposed"
    o = {
        "cos_hi": Out(R * E, dev, torch.bfloat16),
        "cos_lo": Out(R * E, dev, torch.bfloat16) if split else None,
        "cos_t_hi": Out(E * R, dev, torch.bfloat16) if mode != "fp16" else None,
        "x32": Out(R * F, dev) if (x32 or trans) else None,
        "x_hi": Out(R * F, dev, torch.float16 if f16 else torch.bfloat16),
        "x_lo": Out(R * F, dev, torch.bfloat16) if mode != "fp16" else None,
        "x_hi_t": Out(F * R, dev, torch.bfloat16) if trans else None,
        "x_lo_t": Out(F * R, dev, torch.bfloat16) if trans else None,
    }
    p = {k: (v.p if v is not None else None) for k, v in o.items()}
    lib_call("riqn_quantile_embed_fwd_tc", B, Nq, E, F, dptr(inp["tau"]), dptr(inp["feat"]), dptr(inp["w_hi"]),
          dptr(inp["w_lo"]), dptr(inp["be"]), p["cos_hi"], p["cos_lo"], p["cos_t_hi"], p["x32"], p["x_hi"], p["x_lo"],
          p["x_hi_t"], p["x_lo_t"], int(f16))
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _embed_fwd_inputs(dev, B, Nq, F, E, seed, zero_weight=False):
    rs = np.random.RandomState(seed)
    R = B * Nq
    tau = rs.uniform(0, 1, R).astype(np.float32)
    tau[0], tau[R // 2], tau[-1] = 0.0, 0.5, np.float32(1 - 2.0 ** -24)
    feat = np.maximum(rs.standard_normal((B, F)), 0).astype(np.float32)
    w = (rs.standard_normal((F, E)) * 0.2).astype(np.float32)
    be = (rs.standard_normal(F) * 0.3).astype(np.float32)
    if zero_weight:
        w[:] = 0
        be[:] = 1
    w_hi = bf16(w)
    w_lo = bf16(w - w_hi)
    host = dict(tau=tau, feat=feat, w=w, w_hi=w_hi, w_lo=w_lo, be=be)
    inp = dict(tau=to_dev(tau, dev), feat=to_dev(feat, dev), w=to_dev(w, dev), w_hi=to_dev_bf16(w_hi, dev),
               w_lo=to_dev_bf16(w_lo, dev), be=to_dev(be, dev))
    return host, inp


def _check_rows(R, seed):
    """rows whose float64 reference is computed: all of them, or the first and last 256 and 512 random ones"""
    if R <= 4096:
        return np.arange(R)
    return np.unique(np.concatenate([np.arange(256), np.arange(R - 256, R), np.random.RandomState(seed).randint(0, R, 512)]))


def _check_embed_fwd(dev, B, Nq, F, E, mode, seed):
    R = B * Nq
    host, inp = _embed_fwd_inputs(dev, B, Nq, F, E, seed)
    o = _embed_fwd_call(dev, B, Nq, F, E, mode, inp)
    split = o["cos_lo"] is not None
    # cos images
    c64 = _cos_ref(host["tau"], B, Nq, E)
    ch = o["cos_hi"].f32().reshape(R, E)
    cl = o["cos_lo"].f32().reshape(R, E) if split else np.zeros_like(ch)
    sp = np.spacing(np.abs(c64).astype(np.float32)).astype(np.float64)
    # CUDA's cosf: 2 ulp (CUDA C Programming Guide, maths functions); a bf16 rounding (of c, or of the residual c - hi
    # into lo) is off by at most half an ulp of its 8-bit significand, 2^-8 of the value
    cos_bound = 2 * sp + (2.0 ** -8 * np.abs(c64 - ch) if split else 2.0 ** -8 * np.abs(c64)) + sp
    check_bound(f"cos images {mode}", ch.astype(np.float64) + cl, c64, cos_bound)
    if o["cos_t_hi"] is not None:
        assert_bits("cos_t_hi", o["cos_t_hi"].bits().reshape(E, R), o["cos_hi"].bits().reshape(R, E).T)
    # x32 against feat[r // Nq] * relu(cos W_e^T + b_e) on the kernel's own cos images
    x32 = o["x32"].f32().reshape(R, F)
    rows = _check_rows(R, seed)
    chs, cls = ch[rows].astype(np.float64), cl[rows].astype(np.float64)
    wh, wl = host["w_hi"].astype(np.float64), host["w_lo"].astype(np.float64)
    pre = chs @ wh.T + host["be"].astype(np.float64)
    mag = np.abs(chs) @ np.abs(wh).T + np.abs(host["be"]).astype(np.float64)
    k = E + 2
    if split:
        pre += chs @ wl.T + cls @ wh.T
        mag += np.abs(chs) @ np.abs(wl).T + np.abs(cls) @ np.abs(wh).T
        k = 3 * E + 2
    fr = host["feat"][rows // Nq].astype(np.float64)
    ref = fr * np.maximum(pre, 0)
    check_bound(f"x32 {mode}", x32[rows], ref, C_BOUND * k * U * mag * fr + U * np.abs(ref))
    # the 16-bit images bit for bit from x32
    if mode.startswith("fp16"):
        assert_bits("x_hi = fp16(x)", o["x_hi"].bits().reshape(R, F), f16_bits(x32))
        if o["x_lo"] is not None:
            assert_bits("x_lo = bf16(x)", o["x_lo"].bits().reshape(R, F), bf16_bits(x32))
    else:
        hi = bf16(x32)
        assert_bits("x_hi = bf16(x)", o["x_hi"].bits().reshape(R, F), bf16_bits(x32))
        assert_bits("x_lo = bf16(x - hi)", o["x_lo"].bits().reshape(R, F), bf16_bits(x32 - hi))
    if o["x_hi_t"] is not None:
        assert_bits("x_hi_t", o["x_hi_t"].bits().reshape(F, R), o["x_hi"].bits().reshape(R, F).T)
        assert_bits("x_lo_t", o["x_lo_t"].bits().reshape(F, R), o["x_lo"].bits().reshape(R, F).T)
    # determinism, and the same images without the fp32 matrix
    o2 = _embed_fwd_call(dev, B, Nq, F, E, mode, inp)
    for key, v in o.items():
        if v is not None:
            assert_bits(f"second call {key}", o2[key].bits(), v.bits())
    if mode != "bf16x3-transposed":
        o3 = _embed_fwd_call(dev, B, Nq, F, E, mode, inp, x32=False)
        for key in ("cos_hi", "cos_lo", "cos_t_hi", "x_hi", "x_lo"):
            if o[key] is not None:
                assert_bits(f"x32 = NULL {key}", o3[key].bits(), o[key].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", FWD_MODES)
@pytest.mark.parametrize("B,Nq,F,E", FWD_SHAPES, ids=[f"B{b}-Nq{n}-F{f}-E{e}" for b, n, f, e in FWD_SHAPES])
def test_embed_fwd_tc(cuda_dev, B, Nq, F, E, mode):
    _check_embed_fwd(cuda_dev, B, Nq, F, E, mode, seed=B * 1000 + Nq)


@pytest.mark.gpu
def test_embed_fwd_tc_config2_rows(cuda_dev):
    """R = 512 * 64 rows (the benchmarked N = N' = 64 pass) in the default fp16 + bf16 image mode"""
    _check_embed_fwd(cuda_dev, 512, 64, 3136, 64, "fp16-xlo", seed=7)


@pytest.mark.gpu
@pytest.mark.parametrize("Nq", [1, 3, 32, 33, 200])
@pytest.mark.parametrize("mode", ["fp16-xlo", "bf16x3"])
def test_embed_fwd_tc_rows_read_their_sample(cuda_dev, Nq, mode):
    """W_e = 0, b_e = 1: every pre-activation is exactly 1, so row r must hold exactly feat[r // Nq]
    (Nq % 32 != 0 takes the epilogue's per-row feat path)."""
    B, F, E = 6, 96, 64
    host, inp = _embed_fwd_inputs(cuda_dev, B, Nq, F, E, seed=Nq, zero_weight=True)
    o = _embed_fwd_call(cuda_dev, B, Nq, F, E, mode, inp)
    assert_bits("x32 == feat[r // Nq]", f32_bits(o["x32"].f32().reshape(B * Nq, F)),
                 f32_bits(np.repeat(host["feat"], Nq, axis=0)))


@pytest.mark.gpu
def test_embed_fwd_tc_rejects_before_writing(cuda_dev):
    """Odd rows, feat_dim % 32, embed_dim % 8, transposed images without x32 or with fp16 images, and TMA operands
    that are not 16-byte aligned are rejected before the first launch: every output keeps its NaN fill."""
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    cases = [  # (B, Nq, F, E, x_fp16, x32, transposed, output passed one element past a 16-byte boundary)
        (3, 3, 96, 64, 1, True, False, None), (4, 2, 100, 64, 1, True, False, None), (4, 2, 96, 60, 1, True, False, None),
        (4, 2, 96, 64, 0, False, True, None), (4, 2, 96, 64, 1, True, True, None), (4, 2, 96, 64, 1, True, False, "cos_hi"),
        (4, 2, 96, 64, 1, True, False, "x_hi"), (4, 2, 96, 64, 0, True, False, "x_lo")]
    for B, Nq, F, E, f16, with_x32, trans, shifted in cases:
        R = B * Nq
        rs = np.random.RandomState(R)
        tau = to_dev(rs.uniform(0, 1, R).astype(np.float32), dev)
        feat = to_dev(np.abs(rs.standard_normal((B, F))).astype(np.float32), dev)
        w = to_dev_bf16(rs.standard_normal((F, E)).astype(np.float32), dev)
        be = to_dev(rs.standard_normal(F).astype(np.float32), dev)
        o = {"cos_hi": Out(R * E, dev, torch.bfloat16), "cos_lo": Out(R * E, dev, torch.bfloat16),
             "cos_t_hi": Out(E * R, dev, torch.bfloat16), "x32": Out(R * F, dev) if with_x32 else None,
             "x_hi": Out(R * F, dev, torch.float16 if f16 else torch.bfloat16),
             "x_lo": Out(R * F, dev, torch.bfloat16),
             "x_hi_t": Out(F * R, dev, torch.bfloat16) if trans else None,
             "x_lo_t": Out(F * R, dev, torch.bfloat16) if trans else None}
        p = {k: (v.p if v is not None else None) for k, v in o.items()}
        if shifted:
            p[shifted] += 2
        with pytest.raises(RiqnError):
            lib_call("riqn_quantile_embed_fwd_tc", B, Nq, E, F, dptr(tau), dptr(feat), dptr(w), dptr(w), dptr(be),
                  p["cos_hi"], p["cos_lo"], p["cos_t_hi"], p["x32"], p["x_hi"], p["x_lo"], p["x_hi_t"], p["x_lo_t"], f16)
        torch.cuda.synchronize()
        assert_canaries(o)
        for k, v in o.items():
            if v is not None:
                assert torch.isnan(v.t[:v.n].float()).all(), f"rejected call {(B, Nq, F, E, f16, with_x32, trans, shifted)} wrote {k}"


# ---------------------------------------------------------------------------------------------- quantile embedding backward
# (variant, B, Nq, F, dX bf16): tile = odd Nq; wide = even Nq with fp32 dX; wide8 = even Nq with bf16 dX.
# Nq = 66 and 130 take several 64-row passes, the last one partial.
BWD_CASES = [("tile", 8, 3, 104, False), ("tile", 8, 9, 3136, True), ("tile", 8, 9, 104, False),
             ("wide", 4, 2, 104, False), ("wide", 2, 8, 3136, False), ("wide", 2, 64, 104, False),
             ("wide", 4, 66, 3136, False), ("wide", 4, 130, 104, False),
             ("wide8", 4, 2, 104, True), ("wide8", 2, 8, 3136, True), ("wide8", 2, 64, 104, True),
             ("wide8", 4, 66, 3136, True), ("wide8", 4, 130, 104, True)]


def _embed_bwd_inputs(B, Nq, F, E, xlo, dxb, regime, seed):
    rs = np.random.RandomState(seed)
    R = B * Nq
    if regime == "exact":
        x_hi = rs.randint(-4, 9, (R, F)).astype(np.float32)
        x_hi[rs.uniform(size=(R, F)) < 0.3] = 0
        x_lo = rs.choice(np.array([0, 0, 0.5, -0.5, 0.25], np.float32), (R, F))
        dx = rs.randint(-3, 4, (R, F)).astype(np.float32)
        feat = rs.choice(np.array([0, 0, 0.5, 1, 2, 4], np.float32), (B, F))
        cos = rs.randint(-2, 3, (R, E)).astype(np.float32)
    else:
        x = rs.standard_normal((R, F)).astype(np.float32)
        x[rs.uniform(size=(R, F)) < 0.3] = 0
        x_hi = bf16(x)
        x_lo = bf16(x - x_hi)
        dx = (rs.standard_normal((R, F)) * 1e-2).astype(np.float32)
        feat = np.maximum(rs.standard_normal((B, F)), 0).astype(np.float32)
        cos = bf16(rs.uniform(-1, 1, (R, E)).astype(np.float32))
    if not xlo:
        x_lo = None
    if dxb:
        dx = bf16(dx)
    return dict(x_hi=x_hi, x_lo=x_lo, dx=dx, feat=feat, cos=cos)


def _embed_bwd_call(dev, B, Nq, F, E, dxb, d, pre_w, pre_b):
    R = B * Nq
    o = {"dpre": Out(R * F, dev, torch.bfloat16), "dfeat": Out(B * F, dev), "grad_w": Out(F * E, dev, fill=pre_w),
         "grad_b": Out(F, dev, fill=pre_b)}
    lib_call("riqn_quantile_embed_bwd_tc", B, Nq, E, F, dptr(d["x_hi"]), dptr(d["x_lo"]), dptr(d["feat"]), dptr(d["cos"]),
          dptr(d["dx"]), int(dxb), o["dpre"].p, o["dfeat"].p, o["grad_w"].p, o["grad_b"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("xlo", [True, False], ids=["xlo", "xhi"])
@pytest.mark.parametrize("variant,B,Nq,F,dxb", BWD_CASES,
                         ids=[f"{v}-B{b}-Nq{n}-F{f}-{'dxbf16' if x else 'dxf32'}" for v, b, n, f, x in BWD_CASES])
def test_embed_bwd_tc(cuda_dev, variant, B, Nq, F, dxb, xlo, regime):
    dev = cuda_dev
    E = 64 if F == 3136 else 72
    R = B * Nq
    h = _embed_bwd_inputs(B, Nq, F, E, xlo, dxb, regime, seed=R + F + (7 if regime == "exact" else 0))
    d = {"x_hi": to_dev_bf16(h["x_hi"], dev), "x_lo": to_dev_bf16(h["x_lo"], dev) if xlo else None,
         "feat": to_dev(h["feat"], dev), "cos": to_dev_bf16(h["cos"], dev),
         "dx": to_dev_bf16(h["dx"], dev) if dxb else to_dev(h["dx"], dev)}
    pre_w, pre_b = prefill_pattern(F * E), prefill_pattern(F, 0.5, 7)
    o = _embed_bwd_call(dev, B, Nq, F, E, dxb, d, pre_w, pre_b)
    # dpre = bf16(dX * feat) where fp32(x_hi + x_lo) > 0, else 0: one rounding of one product, bit for bit
    x = (h["x_hi"] + h["x_lo"]).astype(np.float32) if xlo else h["x_hi"]
    ft = np.repeat(h["feat"], Nq, axis=0)
    dp = np.where(x > 0, (h["dx"] * ft).astype(np.float32), np.float32(0)).astype(np.float32)
    assert_bits("dpre", o["dpre"].bits().reshape(R, F), bf16_bits(dp))
    # dfeat = sum_q dX * x / feat, exactly 0 where feat == 0
    dfeat = o["dfeat"].f32().reshape(B, F)
    assert np.all(dfeat[h["feat"] == 0] == 0)
    x64, dx64 = x.astype(np.float64).reshape(B, Nq, F), h["dx"].astype(np.float64).reshape(B, Nq, F)
    f64 = h["feat"].astype(np.float64)
    fpos = np.where(f64 > 0, f64, 1.0)
    ref_dfeat = np.where(f64 > 0, ((dx64 * x64).sum(1) + 0.0) / fpos, 0.0)     # (+0.0: an empty sum is +0 on the device)
    bnd_dfeat = np.where(f64 > 0, C_BOUND * (Nq + 8) * U * np.abs(dx64 * x64).sum(1) / fpos + U * np.abs(ref_dfeat), 0)
    # grad_iqn_b = prefill + sum_r of the fp32 dp (before their bf16 rounding)
    ref_b = pre_b.astype(np.float64) + dp.astype(np.float64).sum(0)
    bnd_b = C_BOUND * (R + B + 1) * U * (np.abs(dp).astype(np.float64).sum(0) + np.abs(pre_b))
    # grad_iqn_w = prefill + dpre^T cos_hi on the kernel's own dpre image
    dpre = o["dpre"].f32().reshape(R, F).astype(np.float64)
    c64 = h["cos"].astype(np.float64)
    ref_w = pre_w.reshape(F, E).astype(np.float64) + dpre.T @ c64
    bnd_w = C_BOUND * (R + 1) * U * (np.abs(dpre).T @ np.abs(c64) + np.abs(pre_w.reshape(F, E)))
    got_w = o["grad_w"].f32().reshape(F, E)
    if regime == "exact":
        assert_bits("dfeat", f32_bits(dfeat), f32_bits(ref_dfeat))
        assert_bits("grad_iqn_b", o["grad_b"].bits(), f32_bits(ref_b))
        assert_bits("grad_iqn_w", f32_bits(got_w), f32_bits(ref_w))
    else:
        check_bound(f"dfeat {variant}", dfeat, ref_dfeat, bnd_dfeat)
        check_bound(f"grad_iqn_b {variant}", o["grad_b"].f32(), ref_b, bnd_b)
        check_bound(f"grad_iqn_w {variant}", got_w, ref_w, bnd_w)
    # determinism: the same call on a fresh prefill gives the same bits everywhere
    o2 = _embed_bwd_call(dev, B, Nq, F, E, dxb, d, pre_w, pre_b)
    for key in o:
        assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())


@pytest.mark.gpu
def test_embed_bwd_tc_rejects_before_writing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    for B, Nq, F, E in [(3, 3, 104, 64), (4, 2, 100, 64), (4, 2, 104, 60)]:    # rows % 8, feat_dim % 8, embed_dim % 8
        R = B * Nq
        h = _embed_bwd_inputs(B, Nq, F, E, True, False, "random", seed=R)
        pre_w, pre_b = prefill_pattern(F * E), prefill_pattern(F)
        o = {"dpre": Out(R * F, dev, torch.bfloat16), "dfeat": Out(B * F, dev), "grad_w": Out(F * E, dev, fill=pre_w),
             "grad_b": Out(F, dev, fill=pre_b)}
        d = [to_dev_bf16(h["x_hi"], dev), to_dev_bf16(h["x_lo"], dev), to_dev(h["feat"], dev), to_dev_bf16(h["cos"], dev),
             to_dev(h["dx"], dev)]
        with pytest.raises(RiqnError):
            lib_call("riqn_quantile_embed_bwd_tc", B, Nq, E, F, *[dptr(t) for t in d[:4]], dptr(d[4]), 0, o["dpre"].p,
                  o["dfeat"].p, o["grad_w"].p, o["grad_b"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        assert torch.isnan(o["dpre"].t[:R * F].float()).all() and torch.isnan(o["dfeat"].t[:B * F]).all()
        assert_bits("grad_iqn_w untouched", o["grad_w"].bits(), f32_bits(pre_w))
        assert_bits("grad_iqn_b untouched", o["grad_b"].bits(), f32_bits(pre_b))


# ---------------------------------------------------------------------------------------------- fp32 cross-check twins
# riqn_quantile_embed_fwd / _bwd: the RIQN_*_PRECISION=fp32 modes the other arithmetic modes are judged against.
# (B, Nq, F, E): F = 98 takes the scalar epilogue of the CUDA-core GEMM, R = 4096 several split-K slices of dW_e.
F32_SHAPES = [(4, 1, 96, 64), (6, 3, 98, 72), (5, 8, 3136, 64), (6, 33, 96, 64), (2, 200, 98, 72), (64, 64, 3136, 64)]
F32_IDS = [f"B{b}-Nq{n}-F{f}-E{e}" for b, n, f, e in F32_SHAPES]


def _embed_fwd_f32_call(dev, B, Nq, F, E, inp):
    R = B * Nq
    o = {"cos": Out(R * E, dev), "x": Out(R * F, dev)}
    lib_call("riqn_quantile_embed_fwd", B, Nq, E, F, dptr(inp["tau"]), dptr(inp["feat"]), dptr(inp["w"]), dptr(inp["be"]),
          o["cos"].p, o["x"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("B,Nq,F,E", F32_SHAPES, ids=F32_IDS)
def test_embed_fwd_f32(cuda_dev, B, Nq, F, E):
    dev = cuda_dev
    R = B * Nq
    host, inp = _embed_fwd_inputs(dev, B, Nq, F, E, seed=B * 100 + Nq + 1)
    o = _embed_fwd_f32_call(dev, B, Nq, F, E, inp)
    c64 = _cos_ref(host["tau"], B, Nq, E)
    cos = o["cos"].f32().reshape(R, E)
    sp = np.spacing(np.abs(c64).astype(np.float32)).astype(np.float64)
    check_bound("cos f32", cos, c64, 3 * sp)                     # cosf: 2 ulp, plus one ulp of slack
    # x against feat[r // Nq] * relu(cos W_e^T + b_e) on the kernel's own cos values
    rows = _check_rows(R, B + Nq)
    c = cos[rows].astype(np.float64)
    w = host["w"].astype(np.float64)
    pre = c @ w.T + host["be"].astype(np.float64)
    mag = np.abs(c) @ np.abs(w).T + np.abs(host["be"]).astype(np.float64)
    fr = host["feat"][rows // Nq].astype(np.float64)
    ref = fr * np.maximum(pre, 0)
    check_bound("x f32", o["x"].f32().reshape(R, F)[rows], ref, C_BOUND * (E + 2) * U * mag * fr + U * np.abs(ref))
    o2 = _embed_fwd_f32_call(dev, B, Nq, F, E, inp)               # no atomics: deterministic
    for key in o:
        assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("Nq", [1, 3, 33, 200])
def test_embed_fwd_f32_rows_read_their_sample(cuda_dev, Nq):
    """W_e = 0, b_e = 1: row r must hold exactly feat[r // Nq]"""
    B, F, E = 6, 98, 64
    host, inp = _embed_fwd_inputs(cuda_dev, B, Nq, F, E, seed=Nq + 5, zero_weight=True)
    o = _embed_fwd_f32_call(cuda_dev, B, Nq, F, E, inp)
    assert_bits("x == feat[r // Nq]", o["x"].bits().reshape(B * Nq, F), f32_bits(np.repeat(host["feat"], Nq, axis=0)))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,Nq,F,E", F32_SHAPES, ids=F32_IDS)
def test_embed_bwd_f32(cuda_dev, B, Nq, F, E, regime):
    """dX is overwritten with dpre = dX * feat where x > 0; grad_iqn_w is accumulated from split-K partials added in
    split order: bitwise float64 on exact inputs, bounded on random ones, where a second call is bitwise the first."""
    dev = cuda_dev
    R = B * Nq
    h = _embed_bwd_inputs(B, Nq, F, E, True, False, regime, seed=R + F + (3 if regime == "exact" else 0))
    x = (h["x_hi"] + h["x_lo"]).astype(np.float32)
    pre_w, pre_b = prefill_pattern(F * E), prefill_pattern(F, 0.5, 7)
    x_d, feat_d, cos_d = to_dev(x, dev), to_dev(h["feat"], dev), to_dev(h["cos"], dev)

    def call():
        o = {"dx": Out(R * F, dev, fill=h["dx"]), "dfeat": Out(B * F, dev), "grad_w": Out(F * E, dev, fill=pre_w),
             "grad_b": Out(F, dev, fill=pre_b)}
        lib_call("riqn_quantile_embed_bwd", B, Nq, E, F, dptr(x_d), dptr(feat_d), dptr(cos_d), o["dx"].p, o["dfeat"].p,
                 o["grad_w"].p, o["grad_b"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = call()
    ft = np.repeat(h["feat"], Nq, axis=0)
    dp = np.where(x > 0, (h["dx"] * ft).astype(np.float32), np.float32(0)).astype(np.float32)
    assert_bits("dpre (in dX)", o["dx"].bits().reshape(R, F), f32_bits(dp))
    dfeat = o["dfeat"].f32().reshape(B, F)
    assert np.all(dfeat[h["feat"] == 0] == 0)
    x64, dx64 = x.astype(np.float64).reshape(B, Nq, F), h["dx"].astype(np.float64).reshape(B, Nq, F)
    f64 = h["feat"].astype(np.float64)
    fpos = np.where(f64 > 0, f64, 1.0)
    ref_dfeat = np.where(f64 > 0, ((dx64 * x64).sum(1) + 0.0) / fpos, 0.0)
    bnd_dfeat = np.where(f64 > 0, C_BOUND * (Nq + 1) * U * np.abs(dx64 * x64).sum(1) / fpos + U * np.abs(ref_dfeat), 0)
    dp64, c64 = dp.astype(np.float64), h["cos"].astype(np.float64)
    ref_b = pre_b.astype(np.float64) + dp64.sum(0)
    bnd_b = C_BOUND * (R + 2) * U * (np.abs(dp64).sum(0) + np.abs(pre_b))
    ref_w = pre_w.reshape(F, E).astype(np.float64) + dp64.T @ c64
    bnd_w = C_BOUND * (R + 2) * U * (np.abs(dp64).T @ np.abs(c64) + np.abs(pre_w.reshape(F, E)))
    got_w = o["grad_w"].f32().reshape(F, E)
    if regime == "exact":
        assert_bits("dfeat f32", f32_bits(dfeat), f32_bits(ref_dfeat))
        assert_bits("grad_iqn_b f32", o["grad_b"].bits(), f32_bits(ref_b))
        assert_bits("grad_iqn_w f32", f32_bits(got_w), f32_bits(ref_w))
    else:
        check_bound("dfeat f32", dfeat, ref_dfeat, bnd_dfeat)
        check_bound("grad_iqn_b f32", o["grad_b"].f32(), ref_b, bnd_b)
        check_bound("grad_iqn_w f32", got_w, ref_w, bnd_w)
        again = call()
        for key in o:
            assert_bits(f"second call {key}", again[key].bits(), o[key].bits())


# ---------------------------------------------------------------------------------------------- dueling backward
# (B, Nq): rows straddling samples inside a warp, R % 32 != 0, and (512, 64) = 1024 row blocks, more than the 2 * SM grid
DUEL_SHAPES = [(8, 3), (5, 8), (16, 64), (3, 200)]
DUEL_CASES = [(b, n, a) for b, n in DUEL_SHAPES for a in (1, 6, 18, 24, 25, 31)] + [(512, 64, 18), (512, 64, 31)]
DUEL_IDS = [f"B{b}-Nq{n}-A{a}" for b, n, a in DUEL_CASES]


def _duel_inputs(B, Nq, A, regime, seed):
    rs = np.random.RandomState(seed)
    R = B * Nq
    if regime == "exact":
        h = rs.randint(-2, 7, (R, 2 * HID)).astype(np.float32)
        h[rs.uniform(size=h.shape) < 0.3] = 0
        wzv = rs.randint(-8, 9, HID).astype(np.float32)
        wza = rs.randint(-2, 3, (A, HID)).astype(np.float32)
        # last row: column sums become A * c with c the rounded mean, so the mean w_bar = c is exact and |w_a - w_bar|
        # <= 2 + A/2 + 2 < 24.  With g a multiple of 1/8 and |g| <= 1, every dh value is a multiple of 1/8 below 24 in
        # magnitude, so any partial column sum over R <= 32768 rows stays below 2^20: exact in fp32 by construction
        c = np.round(wza[:A - 1].sum(0) / A) if A > 1 else rs.randint(-2, 3, HID)
        wza[A - 1] = A * c - wza[:A - 1].sum(0)
        dtheta = rs.randint(-2, 3, R).astype(np.float32)
        gscale = rs.choice(np.array([0.5, 1, 2], np.float32), B)
        gmul = 0.25
    else:
        h = np.maximum(rs.standard_normal((R, 2 * HID)), 0).astype(np.float32)
        wzv = (rs.standard_normal(HID) * 0.05).astype(np.float32)
        wza = (rs.standard_normal((A, HID)) * 0.05).astype(np.float32)
        dtheta = (rs.standard_normal(R) * 0.1).astype(np.float32)
        gscale = rs.uniform(0.5, 2, B).astype(np.float32)
        gmul = 1.0 / B
    actions = rs.randint(0, A, B).astype(np.int64)
    actions[0], actions[-1] = 0, A - 1
    wz = np.concatenate([wzv[None], wza]).astype(np.float32)
    return dict(h=h, wz=wz, dtheta=dtheta, gscale=gscale, gmul=np.float32(gmul), actions=actions)


def _duel_ref(d, B, Nq, A):
    """numpy float32 statement of the one-hot dueling backward, operation by operation as the kernels round it"""
    R = B * Nq
    r = np.arange(R)
    b, q = r // Nq, r % Nq
    g = (d["dtheta"][q * B + b] * (d["gscale"] * d["gmul"]).astype(np.float32)[b]).astype(np.float32)
    s = np.zeros(HID, np.float32)
    for k in range(A):
        s = (s + d["wz"][1 + k]).astype(np.float32)
    wbar = (s / np.float32(A)).astype(np.float32)
    act = d["actions"][b]
    h = d["h"]
    dh = np.zeros((R, 2 * HID), np.float32)
    dh[:, :HID] = np.where(h[:, :HID] > 0, (g[:, None] * d["wz"][0][None, :]).astype(np.float32), np.float32(0))
    diff = (d["wz"][1 + act] - wbar[None, :]).astype(np.float32)
    dh[:, HID:] = np.where(h[:, HID:] > 0, (g[:, None] * diff).astype(np.float32), np.float32(0))
    inv = np.float32(1) / np.float32(A)
    onehot = (np.arange(A)[None, :] == act[:, None]).astype(np.float32)
    dz = np.zeros((R, 32), np.float32)
    dz[:, 0] = g
    dz[:, 1:1 + A] = (g[:, None] * (onehot - inv).astype(np.float32)).astype(np.float32)
    return dh, dz


def _duel_dev(d, dev):
    return dict(h=to_dev(d["h"], dev), h_bf16=to_dev_bf16(d["h"], dev), wz=to_dev(d["wz"], dev), dtheta=to_dev(d["dtheta"], dev),
                gscale=to_dev(d["gscale"], dev), actions=torch.from_numpy(d["actions"]).to(dev))


def _duel_bf16_call(dev, B, Nq, A, dd, gmul, use_hb, with_t, fn="riqn_dueling_bwd_bf16"):
    R = B * Nq
    o = {"dh_hi": Out(R * 2 * HID, dev, torch.bfloat16), "dh_hi_t": Out(2 * HID * R, dev, torch.bfloat16) if with_t else None,
         "colsum": Out(2 * HID, dev), "dz": Out(R * 32, dev), "dz_bf16": Out(R * 32, dev, torch.bfloat16)}
    p = {k: (v.p if v is not None else None) for k, v in o.items()}
    hb = dptr(dd["h_bf16"]) if use_hb else None
    if fn == "riqn_dueling_bwd_bf16":
        lib_call(fn, R, B, HID, A, dptr(dd["h"]), hb, dptr(dd["wz"]), dptr(dd["dtheta"]), dptr(dd["gscale"]), float(gmul),
              dptr(dd["actions"]), p["dh_hi"], p["dh_hi_t"], p["colsum"], p["dz"], p["dz_bf16"])
    else:
        lib_call(fn, R, B, HID, A, dptr(dd["h"]), hb, dptr(dd["wz"]), dptr(dd["grad_q"]), p["dh_hi"], p["dh_hi_t"],
              p["colsum"], p["dz"], p["dz_bf16"])
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,Nq,A", DUEL_CASES, ids=DUEL_IDS)
def test_dueling_bwd_bf16(cuda_dev, B, Nq, A, regime):
    dev = cuda_dev
    R = B * Nq
    d = _duel_inputs(B, Nq, A, regime, seed=R * 32 + A)
    dd = _duel_dev(d, dev)
    dh, dz = _duel_ref(d, B, Nq, A)
    o = _duel_bf16_call(dev, B, Nq, A, dd, d["gmul"], use_hb=False, with_t=True)
    assert_bits("dh_hi", o["dh_hi"].bits().reshape(R, 2 * HID), bf16_bits(dh))
    assert_bits("dh_hi_t", o["dh_hi_t"].bits().reshape(2 * HID, R), o["dh_hi"].bits().reshape(R, 2 * HID).T)
    assert_bits("dz", o["dz"].bits().reshape(R, 32), f32_bits(dz))
    assert_bits("dz_bf16", o["dz_bf16"].bits().reshape(R, 32), bf16_bits(dz))
    ref_cs = dh.astype(np.float64).sum(0) + 0.0
    if regime == "exact":
        assert_bits("dh_colsum", o["colsum"].bits(), f32_bits(ref_cs))
    else:
        check_bound("dh_colsum", o["colsum"].f32(), ref_cs, C_BOUND * R * U * np.abs(dh).astype(np.float64).sum(0))
    # the bf16 image of h gives the same ReLU mask; without the transposed image the rest is unchanged (and the
    # kernel is deterministic)
    o2 = _duel_bf16_call(dev, B, Nq, A, dd, d["gmul"], use_hb=True, with_t=False)
    for key in ("dh_hi", "colsum", "dz", "dz_bf16"):
        assert_bits(f"h_bf16 call {key}", o2[key].bits(), o[key].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,Nq,A", DUEL_CASES, ids=DUEL_IDS)
def test_dueling_bwd_f32(cuda_dev, B, Nq, A, regime):
    dev = cuda_dev
    R = B * Nq
    d = _duel_inputs(B, Nq, A, regime, seed=R * 32 + A + 1)
    dd = _duel_dev(d, dev)
    dh, dz = _duel_ref(d, B, Nq, A)
    o = {"dh": Out(R * 2 * HID, dev), "dz": Out(R * 32, dev), "dz_bf16": Out(R * 32, dev, torch.bfloat16)}
    lib_call("riqn_dueling_bwd", R, B, HID, A, dptr(dd["h"]), dptr(dd["wz"]), dptr(dd["dtheta"]), dptr(dd["gscale"]),
          float(d["gmul"]), dptr(dd["actions"]), o["dh"].p, o["dz"].p, o["dz_bf16"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    assert_bits("dh", o["dh"].bits().reshape(R, 2 * HID), f32_bits(dh))
    assert_bits("dz", o["dz"].bits().reshape(R, 32), f32_bits(dz))
    assert_bits("dz_bf16", o["dz_bf16"].bits().reshape(R, 32), bf16_bits(dz))


DENSE_CASES = [(8, 3, 1), (5, 8, 18), (3, 200, 31), (16, 64, 6), (512, 64, 18)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["f32", "bf16"])
@pytest.mark.parametrize("B,Nq,A", DENSE_CASES, ids=[f"B{b}-Nq{n}-A{a}" for b, n, a in DENSE_CASES])
def test_dueling_bwd_dense(cuda_dev, B, Nq, A, variant):
    """Dense upstream gradient: the fmaf chain over the actions is not bit-replicable, so float64 within bounds."""
    dev = cuda_dev
    R = B * Nq
    d = _duel_inputs(B, Nq, A, "random", seed=R + A)
    rs = np.random.RandomState(A)
    G = (rs.standard_normal((R, A)) * 0.1).astype(np.float32)          # quantile-major rows q*B + b
    dd = _duel_dev(d, dev)
    dd["grad_q"] = to_dev(G, dev)
    r = np.arange(R)
    Gs = G[(r % Nq) * B + r // Nq].astype(np.float64)                   # sample-major
    wz = d["wz"].astype(np.float64)
    dv = Gs.sum(1)
    da = Gs - dv[:, None] / A
    S = np.abs(Gs).sum(1)
    mask_v, mask_a = d["h"][:, :HID] > 0, d["h"][:, HID:] > 0
    ref_dh = np.concatenate([np.where(mask_v, dv[:, None] * wz[0][None, :], 0), np.where(mask_a, da @ wz[1:], 0)], 1)
    k = A + 3
    bnd_dh = C_BOUND * k * U * np.concatenate(
        [np.where(mask_v, S[:, None] * np.abs(wz[0])[None, :], 0),
         np.where(mask_a, S[:, None] * np.abs(wz[1:]).sum(0)[None, :] + np.abs(da) @ np.abs(wz[1:]), 0)], 1)
    ref_dz = np.zeros((R, 32))
    ref_dz[:, 0], ref_dz[:, 1:1 + A] = dv, da
    bnd_dz = np.zeros((R, 32))
    bnd_dz[:, :1 + A] = C_BOUND * k * U * S[:, None]
    if variant == "f32":
        o = {"dh": Out(R * 2 * HID, dev), "dz": Out(R * 32, dev), "dz_bf16": Out(R * 32, dev, torch.bfloat16)}
        lib_call("riqn_dueling_bwd_dense", R, B, HID, A, dptr(dd["h"]), dptr(dd["wz"]), dptr(dd["grad_q"]), o["dh"].p,
              o["dz"].p, o["dz_bf16"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        check_bound("dense dh", o["dh"].f32().reshape(R, 2 * HID), ref_dh, bnd_dh)
    else:
        o = _duel_bf16_call(dev, B, Nq, A, dd, 0.0, use_hb=False, with_t=True, fn="riqn_dueling_bwd_dense_bf16")
        hi = o["dh_hi"].f32().reshape(R, 2 * HID)
        check_bound("dense dh_hi", hi, ref_dh, 2 * bnd_dh + 2.0 ** -8 * np.abs(ref_dh))
        assert_bits("dense dh_hi_t", o["dh_hi_t"].bits().reshape(2 * HID, R), o["dh_hi"].bits().reshape(R, 2 * HID).T)
        check_bound("dense dh_colsum", o["colsum"].f32(), ref_dh.sum(0),
                     bnd_dh.sum(0) + C_BOUND * R * U * np.abs(ref_dh).sum(0))
        o2 = _duel_bf16_call(dev, B, Nq, A, dd, 0.0, use_hb=True, with_t=False, fn="riqn_dueling_bwd_dense_bf16")
        for key in ("dh_hi", "colsum", "dz", "dz_bf16"):
            assert_bits(f"dense h_bf16 call {key}", o2[key].bits(), o[key].bits())
    dz = o["dz"].f32().reshape(R, 32)
    check_bound("dense dz", dz, ref_dz, bnd_dz)
    assert_bits("dense dz_bf16", o["dz_bf16"].bits().reshape(R, 32), bf16_bits(dz))


@pytest.mark.gpu
def test_dueling_bwd_rejects(cuda_dev):
    """A = 32, hidden != 512 and (bf16 variants) rows % 8 are rejected"""
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    d = _duel_inputs(8, 4, 31, "random", seed=3)
    dd = _duel_dev(d, dev)
    wz32 = torch.zeros(33 * HID, device=dev)
    for R, hid, A, wz in [(32, HID, 32, wz32), (32, 256, 6, dd["wz"]), (28, HID, 6, dd["wz"])]:
        B = 4
        o = {"dh_hi": Out(32 * 2 * HID, dev, torch.bfloat16), "dh": Out(32 * 2 * HID, dev), "colsum": Out(2 * HID, dev),
             "dz": Out(32 * 32, dev), "dz_bf16": Out(32 * 32, dev, torch.bfloat16)}
        with pytest.raises(RiqnError):
            lib_call("riqn_dueling_bwd_bf16", R, B, hid, A, dptr(dd["h"]), None, dptr(wz), dptr(dd["dtheta"]),
                  dptr(dd["gscale"]), 1.0, dptr(dd["actions"]), o["dh_hi"].p, None, o["colsum"].p, o["dz"].p,
                  o["dz_bf16"].p)
        if R % 8 == 0:
            with pytest.raises(RiqnError):
                lib_call("riqn_dueling_bwd", R, B, hid, A, dptr(dd["h"]), dptr(wz), dptr(dd["dtheta"]), dptr(dd["gscale"]),
                      1.0, dptr(dd["actions"]), o["dh"].p, o["dz"].p, o["dz_bf16"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        for k, v in o.items():
            assert torch.isnan(v.t[:v.n].float()).all(), f"rejected call wrote {k}"


# ---------------------------------------------------------------------------------------------- z-layer weight gradients
ZW_CASES = [(rows, A) for rows in (8, 40, 4104, 32768) for A in (1, 18, 31)]


def _zw_inputs(rows, A, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        dz = rs.randint(-3, 4, (rows, 32)).astype(np.float32)
        h = rs.randint(0, 7, (rows, 2 * HID)).astype(np.float32)
        h[rs.uniform(size=h.shape) < 0.3] = 0
        ch = np.array([-2, -1, -0.5, 0.5, 1, 2], np.float32)
        eps = [rs.choice(ch, n) for n in (HID, 1, A * HID, A)]
        pre = [prefill_pattern(n, 0.5, m) for n, m in ((HID, 11), (HID, 7), (1, 3), (1, 5), (A * HID, 13), (A * HID, 9),
                                                 (A, 3), (A, 5))]
    else:
        dz = (rs.standard_normal((rows, 32)) * 0.1).astype(np.float32)
        h = np.maximum(rs.standard_normal((rows, 2 * HID)), 0).astype(np.float32)
        eps = [rs.standard_normal(n).astype(np.float32) for n in (HID, 1, A * HID, A)]
        pre = [rs.standard_normal(n).astype(np.float32) for n in (HID, HID, 1, 1, A * HID, A * HID, A, A)]
    dz[:, 1 + A:] = 64 + np.arange(31 - A, dtype=np.float32)            # sentinels: must not reach any gradient
    return dz, h, eps, pre


ZW_NAMES = ["g_mu_zv", "g_sig_zv", "g_bmu_zv", "g_bsig_zv", "g_mu_za", "g_sig_za", "g_bmu_za", "g_bsig_za"]


def _zw_call(dev, variant, rows, A, dzd, dzb, hd, hb, epsd, pre, fill_scratch=float("nan")):
    o = {n: Out(p.size, dev, fill=p) for n, p in zip(ZW_NAMES, pre)}
    o["dwz"] = Out(32 * 2 * HID, dev, fill=fill_scratch)
    o["dbz"] = Out(32, dev, fill=fill_scratch)
    g = [o[n].p for n in ZW_NAMES]
    if variant == "tc":
        lib_call("riqn_z_wgrad_tc", rows, HID, A, dptr(dzb), dptr(hb), dptr(dzd), o["dwz"].p, o["dbz"].p,
              *[dptr(e) for e in epsd], *g)
    else:
        lib_call("riqn_z_wgrad", rows, HID, A, dptr(dzd), dptr(hd), o["dwz"].p, o["dbz"].p, *[dptr(e) for e in epsd], *g)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("variant", ["tc", "f32"])
@pytest.mark.parametrize("rows,A", ZW_CASES, ids=[f"rows{r}-A{a}" for r, a in ZW_CASES])
def test_z_wgrad(cuda_dev, rows, A, variant, regime):
    dev = cuda_dev
    dz, h, eps, pre = _zw_inputs(rows, A, regime, seed=rows + A)
    dzd, hd = to_dev(dz, dev), to_dev(h, dev)
    dzb, hb = to_dev_bf16(dz, dev), to_dev_bf16(h, dev)
    epsd = [to_dev(e, dev) for e in eps]
    o = _zw_call(dev, variant, rows, A, dzd, dzb, hd, hb, epsd, pre)
    # the weight half reads the operand images the product consumed, the bias half the fp32 dz
    dzi = (bf16(dz) if variant == "tc" else dz).astype(np.float64)
    hi = (bf16(h) if variant == "tc" else h).astype(np.float64)
    dwz = dzi[:, :1 + A].T @ hi
    mag = np.abs(dzi[:, :1 + A]).T @ np.abs(hi)
    dbz = dz[:, :1 + A].astype(np.float64).sum(0)
    mag_b = np.abs(dz[:, :1 + A]).astype(np.float64).sum(0)
    e_wv, e_bv, e_wa, e_ba = [e.astype(np.float64) for e in eps]
    p = [x.astype(np.float64) for x in pre]
    g_v, g_a = dwz[0, :HID], dwz[1:, HID:].ravel()
    m_v, m_a = mag[0, :HID], mag[1:, HID:].ravel()
    ref = [p[0] + g_v, p[1] + g_v * e_wv, p[2] + dbz[:1], p[3] + dbz[:1] * e_bv, p[4] + g_a, p[5] + g_a * e_wa,
           p[6] + dbz[1:], p[7] + dbz[1:] * e_ba]
    k = rows + 3
    bnd = [C_BOUND * k * U * (m_v + np.abs(p[0])), C_BOUND * k * U * (m_v * np.abs(e_wv) + np.abs(p[1])),
           C_BOUND * k * U * (mag_b[:1] + np.abs(p[2])), C_BOUND * k * U * (mag_b[:1] * np.abs(e_bv) + np.abs(p[3])),
           C_BOUND * k * U * (m_a + np.abs(p[4])), C_BOUND * k * U * (m_a * np.abs(e_wa) + np.abs(p[5])),
           C_BOUND * k * U * (mag_b[1:] + np.abs(p[6])), C_BOUND * k * U * (mag_b[1:] * np.abs(e_ba) + np.abs(p[7]))]
    for name, r_, b_ in zip(ZW_NAMES, ref, bnd):
        if regime == "exact":
            assert_bits(name, o[name].bits(), f32_bits(r_))
        else:
            check_bound(f"{name} {variant}", o[name].f32(), r_, b_)
    if variant == "tc" or regime == "random":                           # split partials added in a fixed order
        o2 = _zw_call(dev, variant, rows, A, dzd, dzb, hd, hb, epsd, pre)
        for name in ZW_NAMES:
            assert_bits(f"second call {name}", o2[name].bits(), o[name].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["tc", "f32"])
@pytest.mark.parametrize("A", [0, 32])
def test_z_wgrad_rejects_action_space(cuda_dev, variant, A):
    """dwz_scratch has 32 rows (dv + 31 advantages): A outside 1..31 is rejected before the scratch is cleared"""
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    rows = 40
    dz, h, eps, pre = _zw_inputs(rows, 31, "random", seed=A)
    eps = [np.resize(e, max(A, 1) * (HID if e.size >= HID else 1)).astype(np.float32) for e in eps]
    pre = [np.resize(x, max(A, 1) * (HID if x.size >= HID else 1)).astype(np.float32) if i >= 4 else x
           for i, x in enumerate(pre)]
    o = {n: Out(x.size, dev, fill=x) for n, x in zip(ZW_NAMES, pre)}
    scratch = Out(32 * 2 * HID, dev, fill=3.0), Out(32, dev, fill=3.0)
    args = [o[n].p for n in ZW_NAMES]
    epsd = [to_dev(e, dev) for e in eps]
    dzd, dzb, hd, hb = to_dev(dz, dev), to_dev_bf16(dz, dev), to_dev(h, dev), to_dev_bf16(h, dev)
    with pytest.raises(RiqnError):
        if variant == "tc":
            lib_call("riqn_z_wgrad_tc", rows, HID, A, dptr(dzb), dptr(hb), dptr(dzd), scratch[0].p, scratch[1].p,
                  *[dptr(e) for e in epsd], *args)
        else:
            lib_call("riqn_z_wgrad", rows, HID, A, dptr(dzd), dptr(hd), scratch[0].p, scratch[1].p,
                  *[dptr(e) for e in epsd], *args)
    torch.cuda.synchronize()
    for s in scratch:
        assert torch.all(s.t[:s.n] == 3.0), "the scratch was cleared by a rejected call"
    for n, x in zip(ZW_NAMES, pre):
        assert_bits(f"{n} untouched", o[n].bits(), f32_bits(x))


# ---------------------------------------------------------------------------------------------- NoisyLinear bias gradients
def _nbg_inputs(n, regime, rs):
    if regime == "exact":
        eps = rs.choice(np.array([-2, -1, -0.5, 0.5, 1, 2], np.float32), n)
        return eps, prefill_pattern(n, 0.5, 11), prefill_pattern(n, 0.5, 7)
    return (rs.standard_normal(n).astype(np.float32), rs.standard_normal(n).astype(np.float32),
            rs.standard_normal(n).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("rows", [0, 1, 37, 32776], ids=["colsums-given", "rows1", "rows37", "rows32776"])
def test_noisy_bias_grad(cuda_dev, rows, regime):
    """dh = NULL: the scratch already holds the column sums (riqn_dueling_bwd_bf16's dh_colsum); dh given: the
    scratch is overwritten with its column sums.  g_bmu += db, g_bsig += db * eps."""
    dev = cuda_dev
    n = 2 * HID
    rs = np.random.RandomState(rows + (1 if regime == "exact" else 0))
    eps, pre_mu, pre_sig = _nbg_inputs(n, regime, rs)
    if rows == 0:
        db = (rs.randint(-40, 41, n) * 0.25 if regime == "exact" else rs.standard_normal(n) * 10).astype(np.float32)
        dh = None
        scratch = Out(n, dev, fill=db)
        ref_db, mag = db.astype(np.float64), np.abs(db).astype(np.float64)
        k = 2
    else:
        if regime == "exact":
            dh = rs.randint(-6, 7, (rows, n)).astype(np.float32)
        else:
            dh = (rs.standard_normal((rows, n)) * 0.1).astype(np.float32)
        dh[rs.uniform(size=dh.shape) < 0.3] = 0
        scratch = Out(n, dev)
        ref_db, mag = dh.astype(np.float64).sum(0) + 0.0, np.abs(dh).astype(np.float64).sum(0)
        k = rows + 2
    g_mu, g_sig = Out(n, dev, fill=pre_mu), Out(n, dev, fill=pre_sig)
    dh_d = None if dh is None else to_dev(dh, dev)          # (held: a freed input could be reused for the next upload)
    eps_d = to_dev(eps, dev)
    lib_call("riqn_noisy_bias_grad", max(rows, 1), n, dptr(dh_d), dptr(eps_d), scratch.p, g_mu.p, g_sig.p)
    torch.cuda.synchronize()
    assert_canaries({"scratch": scratch, "g_bmu": g_mu, "g_bsig": g_sig})
    e64 = eps.astype(np.float64)
    ref_mu, ref_sig = pre_mu + ref_db, pre_sig + ref_db * e64
    if regime == "exact":
        assert_bits("db scratch", scratch.bits(), f32_bits(ref_db))
        assert_bits("g_bmu", g_mu.bits(), f32_bits(ref_mu))
        assert_bits("g_bsig", g_sig.bits(), f32_bits(ref_sig))
    else:
        check_bound("db scratch", scratch.f32(), ref_db, C_BOUND * k * U * mag)
        check_bound("g_bmu", g_mu.f32(), ref_mu, C_BOUND * k * U * (mag + np.abs(pre_mu)))
        check_bound("g_bsig", g_sig.f32(), ref_sig, C_BOUND * k * U * (mag * np.abs(e64) + np.abs(pre_sig)))
