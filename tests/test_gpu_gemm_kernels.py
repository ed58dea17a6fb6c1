"""The general wgmma / TMA GEMM (csrc/gemm_tc.cu) entry point by entry point against float64: riqn_gemm_bf16_tc and
riqn_gemm_bf16_tc_mn on 128 x {128, 64, 32} tiles (single-pass bf16 and fp16, split-2, split-bf16 x3, split-K, the
bf16 result images), the operand splitters riqn_split_bf16 and riqn_split_bf16_multi, and the argument contracts of all
four (include/riqn_b200.h).

Method (as tests/test_gpu_conv_kernels.py and tests/test_gpu_head_kernels.py):
* exact regime: the operand images are non-zero integers (hi) and integers times 2^-7 (lo), so every product is exact
  and, as the generator asserts, every partial sum of every output element stays exact in fp32 in any order; the
  output must equal float64 bit for bit (x3: A_hi B_hi^T + A_hi B_lo^T + A_lo B_hi^T, without the lo*lo term the kernel
  drops; split-2: A_hi (B_hi + B_lo)^T);
* random regime: Gaussian images, each element held to 2 * terms * K * 2^-24 * sum |a_k b_k| plus the epilogue's
  roundings (x3 also the dropped sum |a_lo b_lo|); each case prints its worst err/bound ratio;
* the bf16 images c_bf16 / c_t_bf16 equal the round-to-nearest-even bf16 of the fp32 output bit for bit;
* overwritten outputs start as NaN, accumulated ones from prefill_pattern, the padding columns of a pitch ldc > N and
  the elements past every buffer hold canaries, and every call is made twice and must agree bit for bit (split-K adds
  its partial products in split order);
* refused calls raise cudaErrorInvalidValue and leave every buffer as it was.

Each case's id names the path the tile rule of gemm_bf16_tc (gemm.h) gives it on a 132-SM H100: the tile width bn and
the number of k-splits s that remain after the clamps to one round of CTAs and to the k-block count.
The misaligned, NULL-output, internal-epilogue and short-pitch refusals live in tests whose names contain `unaligned`
or `short_pitch`: before those refusals existed such calls reached the kernel.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from helpers import CANARY, U, Out, assert_bits, assert_canaries, bf16, bf16_bits, check_bound, dptr, f16_bits, \
    f32_bits, lib_call, prefill_pattern

F32 = np.float32
LO = 2.0 ** -7          # exact regime: grid of the lo images
H100_SMS = 132          # the SM count the case ids are named for


def _riqn_error():
    from rainbow_iqn_apex_b200._lib import RiqnError
    return RiqnError


def _refused(fn):
    with pytest.raises(_riqn_error(), match=r"cudaError 1$"):      # cudaErrorInvalidValue
        fn()


# ---------------------------------------------------------------------------------------------- cases
def _case(entry, M, N, K, fmt="bf16", epi=0, split_k=1, alpha=1.0, a_is_km=1, c_bf16=False, c_t=False, pad=0):
    return SimpleNamespace(entry=entry, M=M, N=N, K=K, fmt=fmt, epi=epi, split_k=split_k, alpha=alpha, a_is_km=a_is_km,
                           c_bf16=c_bf16, c_t=c_t, ldc=N + pad)


def _cdiv(a, b):
    return -(-a // b)


def tile_path(c, sms):
    """(bn, k-splits) of gemm_bf16_tc for case c on `sms` SMs (the rule in gemm.h)"""
    single = c.fmt in ("bf16", "fp16")
    mn = c.entry == "mn"
    kb, mt = _cdiv(c.K, 64), _cdiv(c.M, 128)
    bn = None
    if single and c.N > 128 and kb >= 16 and (c.epi in (0, 3) or (c.epi == 1 and not mn and not c.c_t)):
        t128, t256 = mt * _cdiv(c.N, 128), mt * _cdiv(c.N, 256)
        unsplit = min(max(c.split_k, 1), max(sms // t128, 1), kb) == 1
        if (c.epi != 3 or unsplit) and (t256 >= sms or 2 * _cdiv(t256, sms) <= _cdiv(t128, sms)):
            bn = 256
    if bn is None:
        narrow = single and c.epi in (0, 2)
        if mn:
            bn = 64 if narrow and c.N <= 64 else 128
        else:
            bn = 32 if narrow and c.N <= 32 else 64 if narrow and c.N <= 64 else 128
    s = min(max(c.split_k, 1), max(sms // (mt * _cdiv(c.N, bn)), 1), kb)
    return bn, _cdiv(kb, _cdiv(kb, s))


def _case_id(c):
    bn, s = tile_path(c, H100_SMS)
    mode = c.fmt if c.entry == "tc" else f"{'km' if c.a_is_km else 'mk'}-{c.fmt}"
    tag = f"{c.entry}-{mode}-e{c.epi}-M{c.M}N{c.N}K{c.K}-bn{bn}-s{s}"
    if c.split_k != 1:
        tag += f"-req{c.split_k}"
    if c.alpha != 1.0:
        tag += f"-a{c.alpha:g}"
    if c.ldc != c.N:
        tag += f"-ldc{c.ldc}"
    return tag + ("-cbf16" if c.c_bf16 else "") + ("-ctbf16" if c.c_t else "")


T, MN = "tc", "mn"
CASES = [
    # bn 32: single pass, epilogue 0 / 2, N <= 32 (one element; the scalar tail with K % 64 != 0 and a padded pitch;
    # epilogue 2 through the scalar (odd ldc) and the vector accumulate; fp16 images)
    _case(T, 1, 1, 8),
    _case(T, 130, 17, 72, pad=7),
    _case(T, 257, 32, 200, epi=2, pad=3),
    _case(T, 257, 32, 200, epi=2),
    _case(T, 64, 20, 64, fmt="fp16"),
    _case(T, 33, 20, 64, pad=1),                                 # below 32 columns any pitch is taken
    # split-K on a bn 32 tile: 7 k-blocks in 1, 2 (4 + 3), 4 (2 + 2 + 2 + 1) and 7 splits
    _case(T, 64, 16, 448, epi=2, split_k=1),
    _case(T, 64, 16, 448, epi=2, split_k=2),
    _case(T, 64, 16, 448, epi=2, split_k=4),
    _case(T, 64, 16, 448, epi=2, split_k=7),
    # bn 64
    _case(T, 300, 64, 136, pad=4),
    _case(T, 129, 40, 520, epi=2, split_k=2),
    # bn 128: N = 65; N > 128 with K < 1024; wide-eligible shapes with too few tiles to go wide
    _case(T, 129, 65, 520, pad=3),
    _case(T, 200, 300, 512, pad=4),
    _case(T, 128, 256, 1024),
    _case(T, 300, 700, 3136),
    _case(T, 300, 700, 3136, fmt="x3"),
    _case(T, 128, 256, 64, fmt="x3"),
    _case(T, 128, 256, 256, fmt="x3"),
    # epilogue 1: odd M (float4 stores, the scalar tail, element stores of the transposed image), even M (warp rows,
    # 32-bit pairs of the transposed image), both images, fp16 and x3
    _case(T, 129, 200, 256, epi=1),
    _case(T, 129, 200, 256, epi=1, c_t=True, pad=4),
    _case(T, 256, 256, 320, epi=1, c_bf16=True, c_t=True),
    _case(T, 254, 100, 64, epi=1, c_t=True),
    _case(T, 254, 96, 64, epi=1, c_bf16=True),
    _case(T, 66, 20, 64, epi=1, c_t=True, pad=3),               # N < 32: scalar stores only
    _case(T, 131, 96, 64, fmt="x3", epi=1, c_t=True),
    _case(T, 1000, 1024, 3136, epi=1),
    _case(T, 1000, 1024, 3136, fmt="x3", epi=1),
    # split-2 (B split, A exact in bf16), epilogue 0
    _case(T, 200, 150, 264, fmt="split2", pad=2),
    # x3 with epilogues 2 and 3, split and unsplit
    _case(T, 100, 200, 640, fmt="x3", epi=2, split_k=2),
    _case(T, 1024, 3136, 4096, fmt="x3", epi=2, split_k=4),     # 200 tiles: the split clamps to one
    _case(T, 200, 300, 512, fmt="x3", epi=3, pad=1),
    _case(T, 256, 512, 8000, fmt="x3", epi=3, split_k=7),        # 125 k-blocks: 6 splits of 18 and one of 17
    _case(T, 200, 300, 512, epi=3, split_k=2),
    # split_k above the k-block count (4) and above one round of CTAs (16 tiles: 8 splits)
    _case(T, 130, 150, 200, epi=2, split_k=9),
    _case(T, 512, 512, 4096, epi=3, split_k=20),
    # MN-major: a_is_km = 1 (A (K, M), any K) and 0 (A (M, K)), B (K, N)
    _case(MN, 96, 64, 203),
    _case(MN, 64, 64, 72, c_bf16=True),
    _case(MN, 48, 32, 80, fmt="fp16", epi=2, split_k=2, alpha=2.0 ** -8),
    _case(MN, 200, 48, 136, epi=2, alpha=0.5),
    _case(MN, 200, 48, 136, epi=2, split_k=2, alpha=2.0 ** -8),
    _case(MN, 136, 200, 400, epi=2, split_k=3),
    _case(MN, 136, 200, 400, epi=2, alpha=2.0 ** -8, pad=3),
    _case(MN, 77, 56, 96, epi=2, split_k=2, alpha=0.5, a_is_km=0),
    _case(MN, 256, 192, 333, epi=3, pad=1),
    _case(MN, 256, 192, 1000, epi=3, split_k=4),
    _case(MN, 100, 72, 64, epi=3, a_is_km=0),
]
# Products that run through several shapes in one test each (see the tests at the end of the product section)
MANY_TILES = [
    _case(T, 4096, 2048, 1024),                   # 512 tiles: every CTA walks several (wide tiles on 132 SMs)
    _case(T, 8192, 1024, 512, fmt="x3", epi=1),   # 512 x3 tiles with bias + ReLU
]
MN_MAJOR = [
    _case(MN, 128, 256, 64),                      # one tile, one k-block
    _case(MN, 128, 256, 512),
    _case(MN, 64, 64, 200),                       # narrow tile, ragged reduction
    _case(MN, 1024, 3136, 4096, epi=3, split_k=4),   # NoisyLinear weight gradient shape (wide tiles: the split clamps)
    _case(MN, 32, 576, 2000, epi=2, split_k=5, alpha=0.5),   # conv weight gradient shape: 4 splits of 7 k-blocks, one of 4
    _case(MN, 300, 3136, 1024, a_is_km=0),        # dX = dY W from the untransposed weight
    _case(MN, 128, 256, 64, a_is_km=0),
    _case(MN, 300, 3136, 1024, a_is_km=0, c_bf16=True),   # the same product written as bf16 instead of fp32
]
FP16_OPERANDS = [
    _case(T, 300, 1024, 3136, fmt="fp16", epi=1),   # the fp16 head forward
    _case(MN, 1024, 3136, 512, fmt="fp16"),
    _case(MN, 300, 3136, 1024, fmt="fp16", a_is_km=0),
]


# ---------------------------------------------------------------------------------------------- operands and reference
def exact_ints(shape, gen, dev, top=3):
    """non-zero integers in [-top, top] (float32)"""
    mag = torch.randint(1, top + 1, shape, generator=gen, device=dev)
    sgn = torch.randint(0, 2, shape, generator=gen, device=dev) * 2 - 1
    return (mag * sgn).float()


def make_images(c, regime, dev, seed):
    """Operand images as the entry point takes them: (a_hi, a_lo, b_hi, b_lo) (lo may be None), 16-bit device tensors.
    Exact regime: hi = non-zero integers in [-3, 3], lo = the same times 2^-7."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    if c.entry == "tc":
        a_shape, b_shape = (c.M, c.K), (c.N, c.K)
    else:
        a_shape, b_shape = ((c.K, c.M) if c.a_is_km else (c.M, c.K)), (c.K, c.N)
    hi_t = torch.float16 if c.fmt == "fp16" else torch.bfloat16
    a_split, b_split = c.fmt == "x3", c.fmt in ("x3", "split2")

    def one(shape, split):
        if regime == "exact":
            hi = exact_ints(shape, gen, dev).to(hi_t)
            return hi, (exact_ints(shape, gen, dev) * LO).to(torch.bfloat16) if split else None
        x = torch.randn(shape, generator=gen, device=dev)
        hi = x.to(hi_t)
        return hi, (x - hi.float()).to(torch.bfloat16) if split else None

    return (*one(a_shape, a_split), *one(b_shape, b_split))


def product_ref(c, ims, exact):
    """float64 (M, N) product of the images, sum |terms| and the random regime's extra bound (the dropped lo*lo)"""
    a_hi, a_lo, b_hi, b_lo = (None if t is None else t.double() for t in ims)
    if c.entry == "mn":
        a_hi = a_hi.t() if c.a_is_km else a_hi
        b_hi = b_hi.t()
    P, S, terms, extra = a_hi @ b_hi.t(), a_hi.abs() @ b_hi.abs().t(), 1, 0.0
    if b_lo is not None:
        P += a_hi @ b_lo.t()
        S += a_hi.abs() @ b_lo.abs().t()
        terms = 2
    if a_lo is not None:
        P += a_lo @ b_hi.t()
        S += a_lo.abs() @ b_hi.abs().t()
        terms = 3
        if not exact:
            P += a_lo @ b_lo.t()
            extra = a_lo.abs() @ b_lo.abs().t()
    if exact:       # every term is a multiple of g and their absolute sum fits 24 bits: any partial sum is exact in fp32
        g = LO if b_lo is not None else 1.0
        assert float(S.max()) <= 2.0 ** 24 * g, "exact-regime sum exceeds 24 bits"
    return P, S, terms, extra


def epilogue_inputs(c, P, exact, dev, seed):
    """bias (epilogue 1), C and out2 prefills and eps (epilogue 3); the exact regime puts row M // 2 at the ReLU edge"""
    rs = np.random.RandomState(seed)
    M, N = c.M, c.N
    bias = c0 = e0 = eps = None
    if c.epi == 1:
        if exact:
            bias = rs.randint(-64, 65, N).astype(np.float64) / 8
            edge = -P[M // 2].cpu().numpy()
            bias[::2] = edge[::2]                     # acc + bias == 0 exactly at the even columns of that row
        else:
            bias = rs.standard_normal(N)
        bias = bias.astype(F32)
    if c.epi in (2, 3):
        c0 = prefill_pattern(M * N).reshape(M, N)
    if c.epi == 3:
        e0 = prefill_pattern(M * N, scale=0.5, mod=7).reshape(M, N)
        eps = (rs.choice([-1.0, -0.5, -0.25, 0.25, 0.5, 1.0], (M, N)) if exact else rs.standard_normal((M, N))).astype(F32)
    return bias, c0, e0, eps


def expected(c, P, S, terms, extra, splits, bias, c0, e0, eps, dev):
    """float64 outputs {name: (value, bound)} of the epilogue"""
    bP = 2 * terms * c.K * U * S + extra + 2 * splits * U * S
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(dev)
    out = {}
    if c.epi == 0:
        out["C"] = (P, bP + U * P.abs())
    elif c.epi == 1:
        pre = P + t(bias)
        out["C"] = (pre.clamp(min=0), bP + U * pre.abs())
    elif c.epi == 2:
        v = t(c0) + c.alpha * P
        out["C"] = (v, c.alpha * bP + U * c.alpha * P.abs() + U * v.abs())
    else:
        v, te = t(c0) + P, t(eps)
        w = t(e0) + P * te
        out["C"] = (v, bP + U * v.abs())
        out["out2"] = (w, te.abs() * bP + U * (P * te).abs() + U * w.abs())
    return out


# ---------------------------------------------------------------------------------------------- buffers and calls
def pitched(M, N, ldc, dev, init=None):
    """(M, ldc) fp32 buffer: the body NaN (or init), canaries in the padding columns and past the end"""
    body = np.full((M, ldc), CANARY, F32)
    body[:, :N] = np.nan if init is None else init
    return Out(M * ldc, dev, fill=body)


def body(o, M, N, ldc):
    """(M, N) body of a pitched buffer; asserts the padding columns and the canaries past the end are untouched"""
    a = o.f32().reshape(M, ldc)
    assert np.all(a[:, N:] == CANARY), "write into the padding columns of the pitch"
    assert_canaries({"pitched": o})
    return a[:, :N]


def gemm_call(c, ims, bufs, bias_d, eps_o, split_k=None):
    a_hi, a_lo, b_hi, b_lo = ims
    C, out2, cb, ct = (bufs.get(k) for k in ("C", "out2", "cb", "ct"))
    p = lambda o: None if o is None else o.p
    sk = c.split_k if split_k is None else split_k
    if c.entry == "tc":
        lib_call("riqn_gemm_bf16_tc", c.M, c.N, c.K, dptr(a_hi), dptr(a_lo), dptr(b_hi), dptr(b_lo), p(C), c.ldc, c.epi,
                 dptr(bias_d), p(out2), p(eps_o), sk, p(ct), p(cb), 3 if c.fmt == "fp16" else 0)
    else:
        lib_call("riqn_gemm_bf16_tc_mn", c.M, c.N, c.K, dptr(a_hi), dptr(b_hi), c.a_is_km, p(C), c.ldc, c.epi, p(out2),
                 p(eps_o), c.alpha, sk, p(cb), 3 if c.fmt == "fp16" else 0)
    torch.cuda.synchronize()


def run_case(c, ims, dev, bias, c0, e0, eps):
    """Call the entry point on fresh buffers; returns {name: Out}"""
    M, N, ldc = c.M, c.N, c.ldc
    only_bf16 = c.entry == "mn" and c.c_bf16               # the result goes to c_bf16 INSTEAD of C
    bufs = {}
    if not only_bf16:
        bufs["C"] = pitched(M, N, ldc, dev, c0)
    if c.epi == 3:
        bufs["out2"] = pitched(M, N, ldc, dev, e0)
    if c.c_bf16:
        bufs["cb"] = Out(M * N, dev, torch.bfloat16)
    if c.c_t:
        bufs["ct"] = Out(N * M, dev, torch.bfloat16)
    eps_o = pitched(M, N, ldc, dev, eps) if c.epi == 3 else None
    bias_d = None if bias is None else torch.from_numpy(bias).to(dev)
    gemm_call(c, ims, bufs, bias_d, eps_o)
    return bufs


def bits_of(bufs):
    return {k: o.bits() for k, o in bufs.items()}


def check_case(dev, c):
    """Both regimes: the outputs against float64 (bitwise / within the bound), the pitch padding and canaries, the bf16
    images against the bf16 of the fp32 output, and a second call bit for bit equal to the first."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    bn, splits = tile_path(c, sms)
    print(f"path on {sms} SMs: bn {bn}, {splits} k-splits")
    for regime in ("exact", "random"):
        exact = regime == "exact"
        seed = (c.M * 7919 + c.N * 31 + c.K) % 100003 + exact
        ims = make_images(c, regime, dev, seed)
        P, S, terms, extra = product_ref(c, ims, exact)
        bias, c0, e0, eps = epilogue_inputs(c, P, exact, dev, seed)
        want = expected(c, P, S, terms, extra, splits, bias, c0, e0, eps, dev)
        bufs = run_case(c, ims, dev, bias, c0, e0, eps)
        again = run_case(c, ims, dev, bias, c0, e0, eps)
        first, second = bits_of(bufs), bits_of(again)
        for k in first:
            assert_bits(f"{regime} {k}: second call", second[k], first[k])
        got = {k: body(bufs[k], c.M, c.N, c.ldc) for k in ("C", "out2") if k in bufs}
        if "C" not in got:
            # c_bf16 instead of C: the image must be the bf16 of the fp32 result of the same product
            assert_canaries(bufs)
            plain = SimpleNamespace(**{**vars(c), "c_bf16": False})
            got["C"] = body(run_case(plain, ims, dev, bias, c0, e0, eps)["C"], c.M, c.N, c.ldc)
        for k, g in got.items():
            ref, bnd = want[k]
            if exact:
                ref = ref.cpu().numpy()
                ref = np.where(ref == 0, 0.0, ref)
                assert np.array_equal(ref.astype(F32).astype(np.float64), ref), f"{k}: exact reference not in fp32"
                g = np.where(g == 0, F32(0), g)                      # +0 and -0 alike
                assert_bits(f"exact {k} (float64)", f32_bits(g), f32_bits(ref))
            else:
                check_bound(f"{_case_id(c)} {k}", g, ref.cpu().numpy(), bnd.cpu().numpy())
        if c.epi == 1 and exact:
            assert np.all(got["C"][c.M // 2, ::2] == 0), "ReLU edge"
        if "cb" in bufs:
            assert_canaries({"c_bf16": bufs["cb"]})
            assert_bits(f"{regime} c_bf16", bufs["cb"].bits().reshape(c.M, c.N), bf16_bits(got["C"]))
        if "ct" in bufs:
            assert_canaries({"c_t_bf16": bufs["ct"]})
            assert_bits(f"{regime} c_t_bf16", bufs["ct"].bits().reshape(c.N, c.M), bf16_bits(got["C"].T))


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_gemm(cuda_dev, c):
    check_case(cuda_dev, c)


@pytest.mark.gpu
def test_gemm_many_tiles_persistent(cuda_dev):
    """Products with more tiles than SMs, so that every persistent CTA walks several (check_case on each shape)."""
    for c in MANY_TILES:
        print(_case_id(c))
        check_case(cuda_dev, c)


@pytest.mark.gpu
def test_gemm_mn_major(cuda_dev):
    """riqn_gemm_bf16_tc_mn at the weight- and data-gradient shapes of the head and the convolutions, K-major and
    MN-major A, with split-K, alpha and the bf16 output (check_case on each shape)."""
    for c in MN_MAJOR:
        print(_case_id(c))
        check_case(cuda_dev, c)


@pytest.mark.gpu
def test_gemm_fp16_operands(cuda_dev):
    """fp16 x fp16 single-pass products (the head forward's arithmetic), K-major and MN-major (check_case on each
    shape); mixing fp16 and bf16 images is refused in test_gemm_refusals."""
    for c in FP16_OPERANDS:
        print(_case_id(c))
        check_case(cuda_dev, c)


# ---------------------------------------------------------------------------------------------- operand splitters
SPECIALS = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.1754942e-38, 3.4028235e38, -3.4028235e38, 3.3961776e38,
                     1.00390625, 1.01171875, -1.00390625, 65504.0, 65520.0, 7e4, 6e-8, 2e-8, 1e-9, 1.0, -2.5],
                    dtype=F32)
# 1.00390625 / 1.01171875: bf16 ties (to even: down / up); FLT_MAX and 3.3961776e38 round up to bf16 infinity;
# 65520 and 7e4 overflow fp16; 6e-8, 2e-8: fp16 subnormal / underflow


def split_input(rows, cols, seed):
    """Gaussian values over 2^-30 .. 2^30, with the specials at the start and the end"""
    rs = np.random.RandomState(seed)
    x = (rs.standard_normal(rows * cols) * np.exp2(rs.randint(-30, 31, rows * cols))).astype(F32)
    k = min(len(SPECIALS), x.size)
    x[:k] = SPECIALS[:k]
    x[-k:] = SPECIALS[::-1][:k]
    return x.reshape(rows, cols)


def split_statement(x):
    """hi = bf16(x) and lo = bf16(x - hi) as bit patterns (x - hi is exact in fp32 unless hi overflowed)"""
    hi = bf16_bits(x)
    with np.errstate(over="ignore", invalid="ignore"):
        lo = bf16_bits(np.asarray(x, F32) - (hi.astype(np.uint32) << 16).view(F32))
    return hi, lo


SPLIT_SHAPES = [(1, 1), (33, 65), (1000, 3136)]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", SPLIT_SHAPES, ids=[f"{r}x{c}" for r, c in SPLIT_SHAPES])
@pytest.mark.parametrize("outs", ["hi,lo,hi_t,lo_t", "hi", "lo,hi_t", "hi_t,lo_t", "fp16:hi,lo", "fp16:hi"])
def test_split_bf16(cuda_dev, rows, cols, outs):
    """riqn_split_bf16: hi, lo, hi_t, lo_t bit for bit against the numpy statement (fp16 mode: hi = fp16(x), lo = bf16(x)),
    with +-0, subnormals, bf16 ties and values that round to infinity; the outputs not asked for are NULL."""
    dev = cuda_dev
    fp16 = outs.startswith("fp16:")
    want = set(outs.split(":")[-1].split(","))
    x = split_input(rows, cols, rows + cols)
    xd = torch.from_numpy(x).to(dev)
    hi, lo = split_statement(x)
    ref = {"hi": f16_bits(x) if fp16 else hi, "lo": bf16_bits(x) if fp16 else lo, "hi_t": hi.T, "lo_t": lo.T}

    def call():
        o = {k: Out(rows * cols, dev, torch.float16 if (fp16 and k == "hi") else torch.bfloat16) for k in want}
        lib_call("riqn_split_bf16", rows, cols, xd.data_ptr(), *(o[k].p if k in o else None for k in ("hi", "lo", "hi_t", "lo_t")),
                 1 if fp16 else 0)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o, o2 = call(), call()
    for k in want:
        assert_bits(f"{k} second call", o2[k].bits(), o[k].bits())
        shape = (cols, rows) if k.endswith("_t") else (rows, cols)
        assert_bits(k, o[k].bits().reshape(shape), np.ascontiguousarray(ref[k]))


# (rows, cols, div, perm, lo, hi_t): element counts below, at and above one 256-element block, and not multiples of it
MULTI_JOBS = [(1, 1, 1.0, False, True, True), (1, 255, 255.0, True, True, False), (16, 16, 1.0, True, False, True),
              (3, 100, 3.0, False, True, True), (8, 64, 1.0, True, True, False), (7, 73, 255.0, True, True, True),
              (3136, 1, 1.0, False, True, False), (1, 257, 1.0, False, False, False), (32, 256, 255.0, True, True, False),
              (64, 576, 1.0, False, True, True), (2, 3, 7.0, True, True, True), (5, 51, 1.0, True, True, True)]


@pytest.mark.gpu
def test_split_bf16_multi(cuda_dev):
    """riqn_split_bf16_multi with 12 jobs against numpy: x = fl32(src[r, perm[c]] / div), hi / lo / hi_t as above (the
    last job's permutation included), and equal to riqn_split_bf16 / riqn_split_bf16_scaled on the permuted source."""
    from rainbow_iqn_apex_b200._lib import SplitJob
    dev = cuda_dev
    rs = np.random.RandomState(12)
    jobs, arr = [], (SplitJob * len(MULTI_JOBS))()
    for i, (rows, cols, div, with_perm, with_lo, with_t) in enumerate(MULTI_JOBS):
        src = split_input(rows, cols, 100 + i)
        perm = rs.permutation(cols).astype(np.int32) if with_perm else None
        jobs.append(dict(src=src, perm=perm, div=div, src_d=torch.from_numpy(src).to(dev),
                         perm_d=None if perm is None else torch.from_numpy(perm).to(dev)))

    def call():
        outs = []
        for j, J, spec in zip(arr, jobs, MULTI_JOBS):
            rows, cols, _, _, with_lo, with_t = spec
            o = {"hi": Out(rows * cols, dev, torch.bfloat16)}
            if with_lo:
                o["lo"] = Out(rows * cols, dev, torch.bfloat16)
            if with_t:
                o["hi_t"] = Out(rows * cols, dev, torch.bfloat16)
            j.src, j.perm, j.rows, j.cols, j.div = J["src_d"].data_ptr(), dptr(J["perm_d"]), rows, cols, J["div"]
            j.hi, j.lo, j.hi_t = o["hi"].p, o["lo"].p if with_lo else None, o["hi_t"].p if with_t else None
            outs.append(o)
        lib_call("riqn_split_bf16_multi", len(MULTI_JOBS), arr)
        torch.cuda.synchronize()
        for o in outs:
            assert_canaries(o)
        return outs

    first, second = call(), call()
    for i, (J, spec, o, o2) in enumerate(zip(jobs, MULTI_JOBS, first, second)):
        rows, cols = spec[:2]
        x = J["src"][:, J["perm"]] if J["perm"] is not None else J["src"]
        if J["div"] != 1.0:
            x = (x / F32(J["div"])).astype(F32)
        hi, lo = split_statement(np.ascontiguousarray(x, F32))
        ref = {"hi": hi, "lo": lo, "hi_t": hi.T}
        for k in o:
            assert_bits(f"job {i} {k} second call", o2[k].bits(), o[k].bits())
            shape = (cols, rows) if k == "hi_t" else (rows, cols)
            assert_bits(f"job {i} {k}", o[k].bits().reshape(shape), np.ascontiguousarray(ref[k]))
        # the single-call splitters on the permuted source write the same images
        xs = torch.from_numpy(np.ascontiguousarray(J["src"][:, J["perm"]] if J["perm"] is not None else J["src"])).to(dev)
        rh = torch.empty(rows, cols, dtype=torch.bfloat16, device=dev)
        rl = torch.empty_like(rh)
        if J["div"] != 1.0:
            lib_call("riqn_split_bf16_scaled", rows, cols, xs.data_ptr(), J["div"], rh.data_ptr(), rl.data_ptr())
        else:
            lib_call("riqn_split_bf16", rows, cols, xs.data_ptr(), rh.data_ptr(), rl.data_ptr(), None, None, 0)
        torch.cuda.synchronize()
        assert_bits(f"job {i} hi vs single call", o["hi"].bits(), rh.view(torch.int16).cpu().numpy().view(np.uint16).ravel())
        if "lo" in o:
            assert_bits(f"job {i} lo vs single call", o["lo"].bits(), rl.view(torch.int16).cpu().numpy().view(np.uint16).ravel())


# ---------------------------------------------------------------------------------------------- refusals
class Rig:
    """Small valid operands and outputs for the refusal tests: every buffer is snapshotted and must be unchanged after a
    refused call.  tc(**over) / mn(**over) call the entry points with the defaults replaced by `over`."""

    def __init__(self, dev, M=64, N=64, K=256):
        self.dev = dev
        self.M, self.N, self.K = M, N, K
        gen = torch.Generator(device=dev).manual_seed(5)
        rnd = lambda *sh: torch.randn(*sh, generator=gen, device=dev)
        kk = max(K, 64)
        self.a_hi, self.a_lo = rnd(M, kk).bfloat16(), rnd(M, kk).bfloat16()
        self.b_hi, self.b_lo = rnd(max(N, 64), kk).bfloat16(), rnd(max(N, 64), kk).bfloat16()
        self.a_km = rnd(kk, max(M, 64)).bfloat16()
        self.b_kn = rnd(kk, max(N, 64)).bfloat16()
        n = M * (N + 8) + 64
        self.bias = Out(N + 64, dev, fill=np.linspace(-1, 1, N + 64).astype(F32))
        self.C = Out(n, dev)
        self.C2 = Out(n, dev, fill=prefill_pattern(n))
        self.out2 = Out(n, dev, fill=prefill_pattern(n, 0.5, 7))
        self.eps = Out(n, dev, fill=prefill_pattern(n, 0.125, 5))
        self.cb = Out(M * N + 64, dev, torch.bfloat16)
        self.ct = Out(M * N + 64, dev, torch.bfloat16)
        self.outs = [self.C, self.C2, self.out2, self.cb, self.ct]

    def tc(self, **over):
        d = dict(M=self.M, N=self.N, K=self.K, a_hi=self.a_hi.data_ptr(), a_lo=None, b_hi=self.b_hi.data_ptr(), b_lo=None,
                 c=self.C.p, ldc=self.N, epi=0, bias=self.bias.p, out2=None, eps=None, split_k=1, c_t=None, c_bf16=None,
                 fmt=0)
        d.update(over)
        lib_call("riqn_gemm_bf16_tc", *d.values())

    def mn(self, **over):
        d = dict(M=self.M, N=self.N, K=self.K, a=self.a_km.data_ptr(), b=self.b_kn.data_ptr(), a_is_km=1, c=self.C.p,
                 ldc=self.N, epi=0, out2=None, eps=None, alpha=1.0, split_k=1, c_bf16=None, fmt=0)
        d.update(over)
        lib_call("riqn_gemm_bf16_tc_mn", *d.values())

    def refused(self, tag, fn):
        torch.cuda.synchronize()
        before = [o.t.clone() for o in self.outs]
        _refused(fn)
        torch.cuda.synchronize()
        for o, b in zip(self.outs, before):
            w = torch.int16 if o.t.element_size() == 2 else torch.int32
            assert torch.equal(o.t.view(w), b.view(w)), f"refused call ({tag}) wrote an output"

    def accum(self, **over):
        """epilogue 2 / 3 arguments (prefilled C, out2, eps)"""
        return dict(dict(c=self.C2.p, out2=self.out2.p, eps=self.eps.p), **over)


def _lo(r):
    return r.a_lo.data_ptr()


def _blo(r):
    return r.b_lo.data_ptr()


def _fp16_pair(r):
    return r.a_hi.half().data_ptr(), r.b_hi.half().data_ptr()


@pytest.mark.gpu
def test_gemm_refusals(cuda_dev):
    """Refusals that predate the argument checks of the entry points: K % 8, mixed fmt, fp16 split products, split-2 with
    an epilogue other than 0, split_k > 1 with epilogue 0 / 1 on a product small enough to keep its splits, the c_bf16
    conditions, and the MN-major M / N / K and epilogue rules.  The unmodified calls run."""
    r = Rig(cuda_dev)
    r.tc()
    r.tc(epi=1, c_t=r.ct.p, c_bf16=r.cb.p)
    r.mn()
    r.mn(**r.accum(epi=3))
    bad = [("K % 8", lambda: r.tc(K=12)),
           ("fmt 1", lambda: r.tc(fmt=1)), ("fmt 2", lambda: r.tc(fmt=2)), ("mn fmt 1", lambda: r.mn(fmt=1)),
           ("mn fmt 2", lambda: r.mn(fmt=2)),
           ("fp16 x3", lambda: r.tc(a_lo=_lo(r), b_lo=_blo(r), fmt=3)), ("fp16 split-2", lambda: r.tc(b_lo=_blo(r), fmt=3)),
           ("split-2 epilogue 1", lambda: r.tc(b_lo=_blo(r), epi=1)),
           ("split-2 epilogue 2", lambda: r.tc(b_lo=_blo(r), **r.accum(epi=2))),
           ("split-2 epilogue 3", lambda: r.tc(b_lo=_blo(r), **r.accum(epi=3))),
           ("split_k epilogue 0, small", lambda: r.tc(split_k=2)),
           ("split_k epilogue 1, small", lambda: r.tc(epi=1, split_k=2)),
           ("c_bf16 epilogue 0", lambda: r.tc(c_bf16=r.cb.p)), ("c_bf16 epilogue 2", lambda: r.tc(c_bf16=r.cb.p, **r.accum(epi=2))),
           ("c_bf16 odd M", lambda: r.tc(M=63, epi=1, c_bf16=r.cb.p)), ("c_bf16 N % 32", lambda: r.tc(N=48, epi=1, c_bf16=r.cb.p)),
           ("mn c_bf16 epilogue 2", lambda: r.mn(c_bf16=r.cb.p, **r.accum(epi=2))),
           ("mn c_bf16 N % 32", lambda: r.mn(N=48, c=None, c_bf16=r.cb.p)),
           ("mn a_is_km M % 8", lambda: r.mn(M=60)), ("mn N % 8", lambda: r.mn(N=60)),
           ("mn a_is_km 0 K % 8", lambda: r.mn(a_is_km=0, a=r.a_hi.data_ptr(), K=60)),
           ("mn epilogue 1", lambda: r.mn(epi=1))]
    for tag, fn in bad:
        r.refused(tag, fn)


NEW_REFUSALS = ["alpha_not_epi2", "a_lo_without_b_lo", "c_t_bf16_not_epi1", "split_k_epi01_large", "split2_epi2_split",
                "lo_t_without_hi_t"]


@pytest.mark.gpu
@pytest.mark.parametrize("what", NEW_REFUSALS)
def test_gemm_refusals_mistaken_arguments(cuda_dev, what):
    """Arguments the entry points used to reinterpret silently: alpha on epilogues 0 / 3 (ignored), a_lo without b_lo
    (a single-pass product), c_t_bf16 on epilogues 0 / 2 / 3 (never written), split_k > 1 with epilogue 0 / 1 on a product
    with more tiles than SMs (clamped to one split instead of refused), split-2 with epilogue 2 and split_k > 1 (run
    through the store epilogue's partials), and riqn_split_bf16 with lo_t but no hi_t (lo_t never written).  The
    in-range neighbours run."""
    if what == "alpha_not_epi2":
        r = Rig(cuda_dev)
        r.refused("alpha epilogue 3", lambda: r.mn(alpha=0.5, **r.accum(epi=3)))
        r.refused("alpha epilogue 0", lambda: r.mn(alpha=0.5))
        r.mn(alpha=0.5, **r.accum(epi=2))
    elif what == "a_lo_without_b_lo":
        r = Rig(cuda_dev)
        r.refused("a_lo alone", lambda: r.tc(a_lo=_lo(r)))
        r.tc(a_lo=_lo(r), b_lo=_blo(r))
    elif what == "c_t_bf16_not_epi1":
        r = Rig(cuda_dev)
        r.refused("c_t_bf16 epilogue 0", lambda: r.tc(c_t=r.ct.p))
        r.refused("c_t_bf16 epilogue 2", lambda: r.tc(c_t=r.ct.p, **r.accum(epi=2)))
        r.refused("c_t_bf16 epilogue 3", lambda: r.tc(c_t=r.ct.p, **r.accum(epi=3)))
        r.tc(c_t=r.ct.p, epi=1)
    elif what == "split_k_epi01_large":
        sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
        r = Rig(cuda_dev, M=1024, N=128 * _cdiv(sms + 1, 8), K=256)     # more 128 x 128 tiles than SMs
        r.refused("split_k epilogue 0", lambda: r.tc(split_k=4))
        r.refused("split_k epilogue 1", lambda: r.tc(split_k=4, epi=1))
        r.tc(split_k=4, **r.accum(epi=2))
    elif what == "split2_epi2_split":
        r = Rig(cuda_dev)
        r.refused("split-2 epilogue 2 split", lambda: r.tc(b_lo=_blo(r), split_k=2, **r.accum(epi=2)))
        r.tc(b_lo=_blo(r))
    else:
        r = Rig(cuda_dev)
        src = torch.randn(r.M, r.N, device=cuda_dev)
        split = lambda *ims: lib_call("riqn_split_bf16", r.M, r.N, src.data_ptr(), *ims, 0)
        r.refused("lo_t without hi_t", lambda: split(r.cb.p, None, None, r.ct.p))
        r.refused("lo, lo_t without hi_t", lambda: split(None, r.cb.p, None, r.ct.p))
        split(None, None, r.cb.p, r.ct.p)


UNSAFE = ["c_offset_e0", "ldc_odd_e0", "c_offset_e1", "ldc_odd_e1", "bias_offset", "c_bf16_offset", "c_t_bf16_offset",
          "mn_c_offset", "mn_ldc_odd", "mn_c_bf16_offset", "null_c", "null_bias", "null_out2_eps", "epilogue_codes"]


@pytest.mark.gpu
@pytest.mark.parametrize("what", UNSAFE)
def test_gemm_refusals_unaligned_null_or_internal(cuda_dev, what):
    """Calls that would send misaligned 16-byte (C on epilogues 0 / 1, c_bf16, the bias read) or 32-bit (c_t_bf16)
    accesses, NULL pointers or an internal epilogue code (4..8, e.g. 5 with a NULL feature pointer) into the kernel are
    refused and write nothing; the aligned neighbours run."""
    r = Rig(cuda_dev)
    f4, h2 = 4, 2             # bytes per fp32 / bf16 element
    cases = {
        "c_offset_e0": [lambda: r.tc(c=r.C.p + f4)],
        "ldc_odd_e0": [lambda: r.tc(ldc=r.N + 1), lambda: r.tc(ldc=r.N + 2)],
        "c_offset_e1": [lambda: r.tc(c=r.C.p + 2 * f4, epi=1), lambda: r.tc(c=r.C.p + f4, epi=1, M=63)],
        "ldc_odd_e1": [lambda: r.tc(ldc=r.N + 2, epi=1), lambda: r.tc(ldc=r.N + 1, epi=1, M=63)],
        "bias_offset": [lambda: r.tc(bias=r.bias.p + f4, epi=1), lambda: r.tc(bias=r.bias.p + 2 * f4, epi=1, M=63)],
        "c_bf16_offset": [lambda: r.tc(epi=1, c_bf16=r.cb.p + 4 * h2)],
        "c_t_bf16_offset": [lambda: r.tc(epi=1, c_t=r.ct.p + h2)],
        "mn_c_offset": [lambda: r.mn(c=r.C.p + f4)],
        "mn_ldc_odd": [lambda: r.mn(ldc=r.N + 1), lambda: r.mn(ldc=r.N + 2, a_is_km=0, a=r.a_hi.data_ptr())],
        "mn_c_bf16_offset": [lambda: r.mn(c=None, c_bf16=r.cb.p + 4 * h2)],
        "null_c": [lambda: r.tc(c=None), lambda: r.tc(c=None, epi=1), lambda: r.tc(**r.accum(c=None, epi=2)),
                   lambda: r.mn(c=None), lambda: r.mn(**r.accum(c=None, epi=3))],
        "null_bias": [lambda: r.tc(bias=None, epi=1)],
        "null_out2_eps": [lambda: r.tc(**r.accum(out2=None, epi=3)), lambda: r.tc(**r.accum(eps=None, epi=3)),
                          lambda: r.mn(**r.accum(out2=None, epi=3)), lambda: r.mn(**r.accum(eps=None, epi=3))],
        "epilogue_codes": [(lambda e=e: r.tc(epi=e)) for e in (-1, 4, 5, 6, 7, 8, 9)]
                          + [(lambda e=e: r.mn(epi=e)) for e in (-1, 1, 4, 5, 8)],
    }
    for i, fn in enumerate(cases[what]):
        r.refused(f"{what} #{i}", fn)
    r.tc(ldc=r.N + 4)
    r.tc(epi=1, ldc=r.N + 4, c_bf16=r.cb.p, c_t=r.ct.p + 2 * h2)
    r.tc(**r.accum(epi=2, ldc=r.N + 1, c=r.C2.p + f4))         # epilogue 2 takes any pitch and alignment
    r.mn(c=None, c_bf16=r.cb.p)
    s = Rig(cuda_dev, N=24)                                    # narrower than one 32-column chunk: scalar stores only
    s.tc(ldc=25, c=s.C.p + f4)
    s.tc(epi=1, ldc=27, c=s.C.p + f4, bias=s.bias.p + f4, c_t=s.ct.p + h2)
    s.mn(ldc=25, c=s.C.p + f4)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["tc", "mn"])
def test_gemm_refusals_short_pitch(cuda_dev, entry):
    """ldc < N (rows would overlap and the last one run past the buffer) is refused on every epilogue that writes C."""
    r = Rig(cuda_dev)
    call = r.tc if entry == "tc" else r.mn
    for epi in ((0, 1, 2, 3) if entry == "tc" else (0, 2, 3)):
        kw = r.accum(epi=epi) if epi >= 2 else dict(epi=epi)
        r.refused(f"{entry} epilogue {epi} ldc N - 4", lambda: call(ldc=r.N - 4, **kw))
        r.refused(f"{entry} epilogue {epi} ldc N - 1", lambda: call(ldc=r.N - 1, **kw))
    call(ldc=r.N)


@pytest.mark.gpu
def test_split_refusals(cuda_dev):
    """riqn_split_bf16 in fp16 mode with hi_t, lo_t or without hi, and riqn_split_bf16_multi with 0 or 13 jobs, no job
    table, a NULL src or hi, or rows / cols < 1 are refused and write nothing."""
    from rainbow_iqn_apex_b200._lib import SplitJob
    dev = cuda_dev
    src = torch.randn(32, 48, device=dev)
    outs = [Out(32 * 48, dev, torch.bfloat16) for _ in range(4)]
    o16 = Out(32 * 48, dev, torch.float16)
    keep = [o.t.clone() for o in outs + [o16]]

    def untouched(tag):
        torch.cuda.synchronize()
        for o, k in zip(outs + [o16], keep):
            assert torch.equal(o.t.view(torch.int16), k.view(torch.int16)), f"refused call ({tag}) wrote an output"

    split = lambda hi, lo, ht, lt, f: lib_call("riqn_split_bf16", 32, 48, src.data_ptr(), hi, lo, ht, lt, f)
    for tag, args in (("fp16 hi_t", (o16.p, outs[0].p, outs[1].p, None)), ("fp16 lo_t", (o16.p, None, None, outs[1].p)),
                      ("fp16 no hi", (None, outs[0].p, None, None))):
        _refused(lambda: split(*args, 1))
        untouched(tag)

    def jobs(n, **over):
        arr = (SplitJob * max(n, 1))()
        for j, o in zip(arr, (outs * 4)[:n]):
            j.src, j.perm, j.rows, j.cols, j.div, j.hi, j.lo, j.hi_t = src.data_ptr(), None, 32, 48, 1.0, o.p, None, None
        for k, v in over.items():
            setattr(arr[n - 1], k, v)
        return arr

    for tag, n, over in (("0 jobs", 0, {}), ("13 jobs", 13, {}), ("NULL src", 3, dict(src=None)),
                         ("NULL hi", 3, dict(hi=None)), ("rows 0", 3, dict(rows=0)), ("cols 0", 3, dict(cols=0)),
                         ("rows -1", 2, dict(rows=-1))):
        arr = jobs(n, **over)
        _refused(lambda: lib_call("riqn_split_bf16_multi", n, arr))
        untouched(tag)
    _refused(lambda: lib_call("riqn_split_bf16_multi", 1, None))
    untouched("no job table")
    lib_call("riqn_split_bf16_multi", 1, jobs(1))


# ---------------------------------------------------------------------------------------------- CPU: the statements
@pytest.mark.parametrize("fmt,K", [("bf16", 8), ("bf16", 3136), ("x3", 4096), ("x3", 8000), ("split2", 264), ("fp16", 3136)])
def test_exact_regime_sums_are_exact(fmt, K):
    """The exact-regime images keep every partial sum exact: sum |terms| fits 24 bits of the terms' grid (the assertion
    in product_ref), and float32 sums of the terms of sampled elements in several orders equal float64."""
    c = _case(T, 24, 20, K, fmt=fmt)
    ims = make_images(c, "exact", torch.device("cpu"), seed=K)
    P, S, _, _ = product_ref(c, ims, exact=True)
    a_hi, a_lo, b_hi, b_lo = (None if t is None else t.double().numpy() for t in ims)
    rs = np.random.RandomState(K)
    for m, n in zip(rs.randint(0, c.M, 6), rs.randint(0, c.N, 6)):
        terms = [a_hi[m] * b_hi[n]]
        if b_lo is not None:
            terms.append(a_hi[m] * b_lo[n])
        if a_lo is not None:
            terms.append(a_lo[m] * b_hi[n])
        t = np.concatenate(terms).astype(F32)
        assert np.array_equal(t.astype(np.float64), np.concatenate(terms)), "a product is not exact in fp32"
        sums = [np.cumsum(t[o], dtype=F32)[-1] for o in (np.arange(t.size), np.arange(t.size)[::-1], rs.permutation(t.size))]
        for s in sums + [t.sum(dtype=F32), t.reshape(-1, 8).sum(0, dtype=F32).sum(dtype=F32)]:
            assert float(s) == float(P[m, n]), (fmt, K, m, n)
        assert abs(float(P[m, n])) <= float(S[m, n])


def test_split_statements_match_torch():
    """The numpy bf16 / fp16 statements the splitter tests use agree with torch's round-to-nearest-even conversions,
    including +-0, subnormals, ties and values that round to infinity."""
    x = split_input(40, 50, 3)
    t = torch.from_numpy(x)
    hi, lo = split_statement(x)
    th = t.bfloat16()
    assert_bits("hi", hi, th.view(torch.int16).numpy().view(np.uint16))
    assert_bits("lo", lo, (t - th.float()).bfloat16().view(torch.int16).numpy().view(np.uint16))
    assert_bits("fp16", f16_bits(x), t.half().view(torch.int16).numpy().view(np.uint16))
    assert_bits("bf16()", f32_bits(bf16(x)), f32_bits(th.float().numpy()))
    assert np.isinf(bf16(SPECIALS[7:10])).all() and np.all((f16_bits(SPECIALS[13:16]) & 0x7FFF) == [0x7BFF, 0x7C00, 0x7C00])
