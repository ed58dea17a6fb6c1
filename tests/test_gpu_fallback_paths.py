"""The backward paths the network takes at shapes, alignments and precisions the main path does not cover: the fp32
CUDA-core trunk backward (B % 8 != 0, riqn_conv_bwd), the fp32 head backward (B * N % 8 != 0, riqn_z_wgrad and
riqn_quantile_embed_bwd), the im2col tensor-core trunk (frames the strip convolution refuses, e.g. history 3,
riqn_conv_bwd_tc) and the fp32 cross-check arm.  They must obey the rule of csrc/common.cuh: no float atomic takes part in
a sum that crosses blocks, because losses become priorities and a last-bit difference changes which transitions later
steps draw.

* The compiled library holds no float add atomic or reduction at all (CPU, cuobjdump).
* Each entry point against its ordered-sum statement, bit for bit, on Gaussian inputs where the order matters:
  - a split-K weight gradient is, per split, one fp32 fmaf chain over k ascending from 0 (the k range of split z is
    gemm_f32_kchunk's cut), the split partials are added in split order from 0, and that sum is added once onto the
    prefill (sum_slots_add);
  - din is, per input pixel, an fp32 sum over (kh, kw) ascending from 0 of the dcol the same call wrote.
  Each entry point is called three times and must give identical bits; the values also stay inside float64 bounds.
* Learner steps on these paths (two learners from one seed, eager and replayed from the step graph) draw the same
  samples and compute identical losses and parameters.
"""
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from helpers import U, Out, assert_bits, assert_canaries, bf16, check_bound, dptr, f32_bits, lib_call, to_dev, to_dev_bf16
from test_gpu_conv_kernels import C_BOUND, dgrad64, geom, grads, im2col, masked, out_size
from test_gpu_learn import _assert_steps_bitwise_reproducible, precision  # noqa: F401 (fixture)

F32 = np.float32
HID = 512
GEOMS = {"conv1": (4, 84, 32, 8, 4, 1), "conv2": (32, 20, 64, 4, 2, 0), "conv3": (64, 9, 64, 3, 1, 0),
         "big": (2, 116, 8, 4, 2, 1), "pad1": (32, 20, 64, 4, 2, 1)}


# ---------------------------------------------------------------------------------------------- the statements (CPU)
def fmaf(a, b, c):
    """fl32(a * b + c) with a single rounding, elementwise on float32 arrays.  a * b is exact in float64; the float64 sum
    is made round-to-odd (its error term from TwoSum decides the last bit), which makes the final rounding to fp32 that of
    the exact value (53 >= 24 + 2 bits)."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bv = s - p
    e = (p - (s - bv)) + (c - bv)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def kchunk(K, split):
    """gemm_f32_kchunk: rows of K per split, ceil(K / split) rounded up to whole 16-row k-slabs"""
    split = max(split, 1)
    kc = -(-K // split)
    return 16 if kc < 16 else -(-kc // 16) * 16


def split_k_sum(a, b, split):
    """sum_k a[k, m] * b[k, n] as the split-K statement: split z is an fmaf chain over its k rows ascending from 0, the
    partials are added in split order from 0.  a (K, m), b (K, n) float32 -> (m, n) float32"""
    K = a.shape[0]
    kc = kchunk(K, split)
    S = -(-K // kc)
    pad = lambda x: np.concatenate([x, np.zeros((S * kc - K, x.shape[1]), F32)]).reshape(S, kc, x.shape[1])
    a3, b3 = pad(np.asarray(a, F32)), pad(np.asarray(b, F32))
    acc = np.zeros((S, a.shape[1], b.shape[1]), F32)
    for j in range(kc):              # rows past K: fmaf(0, 0, acc) = acc (an fmaf chain from +0 never holds -0)
        acc = fmaf(a3[:, j, :, None], b3[:, j, None, :], acc)
    tot = np.zeros(acc.shape[1:], F32)
    for z in range(S):
        tot = tot + acc[z]
    return tot


def col2im_sum(dcol, B, cin, h, k, s, pad):
    """din[b, c, ih, iw] = sum over (kh, kw) ascending, from 0, of dcol[(b, oh, ow), (c, kh, kw)] (fp32 adds)"""
    oh = out_size(h, k, s, pad)
    d = np.asarray(dcol, F32).reshape(B, oh, oh, cin, k, k)
    din = np.zeros((B, cin, h, h), F32)
    for kh in range(k):
        ih = np.arange(oh) * s + kh - pad
        vh = (ih >= 0) & (ih < h)
        for kw in range(k):
            iw = np.arange(oh) * s + kw - pad
            vw = (iw >= 0) & (iw < h)
            src = d[:, vh][:, :, vw][..., kh, kw].transpose(0, 3, 1, 2)          # (B, cin, oh', ow')
            idx = np.ix_(np.arange(B), np.arange(cin), ih[vh], iw[vw])
            din[idx] = din[idx] + src
    return din


def _round_exact(x):
    """correctly rounded fp32 of a Fraction (ties to even)"""
    r = F32(float(x))
    cands = [np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))]
    best = min(abs(Fraction(float(c)) - x) for c in cands)
    ties = [c for c in cands if abs(Fraction(float(c)) - x) == best]
    return ties[0] if len(ties) == 1 else [c for c in ties if (int(np.array(c, F32).view(np.uint32)) & 1) == 0][0]


def test_fmaf_statement_rounds_once():
    """fmaf() against exact rational arithmetic, including a case where rounding the float64 sum to fp32 would round
    twice: 1 + 2^-23 + (1 + 2^-15) * (1 - 2^-15) * 2^-24 lies just below a midpoint that float64 rounds onto."""
    a, b, c = F32(1 + 2.0 ** -15), F32((1 - 2.0 ** -15) * 2.0 ** -24), F32(1 + 2.0 ** -23)
    naive = F32(np.float64(a) * np.float64(b) + np.float64(c))
    want = _round_exact(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))
    assert naive != want and fmaf(a, b, c) == want
    rs = np.random.RandomState(3)
    n = 3000
    a = rs.standard_normal(n).astype(F32)
    b = (rs.standard_normal(n) * np.exp2(rs.randint(-30, 30, n))).astype(F32)
    c = (rs.standard_normal(n) * np.exp2(rs.randint(-30, 30, n))).astype(F32)
    got = fmaf(a, b, c)
    want = [_round_exact(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)]
    assert_bits("fmaf", f32_bits(got), f32_bits(np.array(want, F32)))


def test_statements_match_float64():
    """split_k_sum is the product and col2im_sum the data gradient of the convolution, to fp32 accuracy."""
    rs = np.random.RandomState(4)
    a, b = rs.standard_normal((300, 3)).astype(F32), rs.standard_normal((300, 5)).astype(F32)
    for split in (1, 3, 40):
        ref = a.astype(np.float64).T @ b
        check_bound(f"split_k_sum split {split}", split_k_sum(a, b, split), ref,
                    C_BOUND * 302 * U * (np.abs(a).astype(np.float64).T @ np.abs(b)))
    assert np.array_equal(split_k_sum(a[:16], b[:16], 1), split_k_sum(a[:16], b[:16], 7))    # one k-slab: one split
    for name in ("conv1", "conv3", "big"):
        cin, h, cout, k, s, pad = GEOMS[name]
        oh = out_size(h, k, s, pad)
        dy = rs.standard_normal((2, cout, oh, oh)).astype(F32)
        w = rs.standard_normal((cout, cin, k, k)).astype(F32)
        dcol = dy.transpose(0, 2, 3, 1).reshape(-1, cout).astype(np.float64) @ w.reshape(cout, -1)
        din = col2im_sum(dcol.astype(F32), 2, cin, h, k, s, pad)
        check_bound(f"col2im_sum {name}", din, dgrad64(dy, w, (2, cin, h, h), s, pad),
                    C_BOUND * (cout + k * k) * U * dgrad64(np.abs(dy), np.abs(w), (2, cin, h, h), s, pad))


# ---------------------------------------------------------------------------------------------- a. SASS guard (CPU)
FLOAT_ADD_ATOMIC = re.compile(r"\b(RED|ATOM)G?\.E\.ADD\.F32|\bATOMS\.CAST\.SPIN")


def test_library_has_no_float_add_atomics():
    """No kernel of the library contains a float add atomic or reduction: a global one (REDG / ATOMG ...ADD.F32) or the
    compare-and-swap loop a shared-memory float atomicAdd compiles to (ATOMS.CAST.SPIN).  Integer counters are fine."""
    from rainbow_iqn_apex_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(tool) and os.path.exists(nvcc) and os.path.exists(_lib.LIB_PATH)):
        pytest.skip("cuobjdump, nvcc or the built library is missing")
    if "release 12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("the instruction names were checked with CUDA 12.9")
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    blocks = re.split(r"\n\s*Function : ", sass)[1:]
    assert blocks, "no kernels in the library's SASS"
    bad = [b.split("\n", 1)[0].strip() for b in blocks if FLOAT_ADD_ATOMIC.search(b.split("\n", 1)[1])]
    assert bad == [], f"kernels with float add atomics: {bad}"


# ---------------------------------------------------------------------------------------------- b. entry points (GPU)
def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _rows(n, seed, k=4):
    """a row subsample: the first and last rows and a few random ones"""
    return np.unique(np.concatenate([[0, n - 1], np.random.RandomState(seed).randint(0, n, k)]))


def _three_calls(call):
    """the call three times; every output bitwise the first call's"""
    outs = [call() for _ in range(3)]
    for o in outs[1:]:
        for key, v in o.items():
            if v is not None:
                assert_bits(f"repeated call {key}", v.bits(), outs[0][key].bits())
    return outs[0]


ZW_ROWS = [40, 64, 169, 2048, 32771]          # 40, 64: one split (the statement is today's single-split product)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ZW_ROWS)
def test_z_wgrad_is_the_ordered_split_k_sum(cuda_dev, rows):
    """riqn_z_wgrad's (32, 2 * hid) scratch product dz^T h: up to 32 splits of whole k-slabs, added in split order onto
    the cleared scratch, bit for bit on a row subsample; the z-layer gradients from it identical over three calls."""
    dev = cuda_dev
    A = 18
    rs = np.random.RandomState(rows)
    dz = rs.standard_normal((rows, 32)).astype(F32)
    h = np.maximum(rs.standard_normal((rows, 2 * HID)), 0).astype(F32)
    eps = [rs.standard_normal(n).astype(F32) for n in (HID, 1, A * HID, A)]
    pre = [rs.standard_normal(n).astype(F32) for n in (HID, HID, 1, 1, A * HID, A * HID, A, A)]
    dzd, hd, epsd = to_dev(dz, dev), to_dev(h, dev), [to_dev(e, dev) for e in eps]
    names = ["g_mu_zv", "g_sig_zv", "g_bmu_zv", "g_bsig_zv", "g_mu_za", "g_sig_za", "g_bmu_za", "g_bsig_za"]

    def call():
        o = {n: Out(p.size, dev, fill=p) for n, p in zip(names, pre)}
        o["dwz"], o["dbz"] = Out(32 * 2 * HID, dev), Out(32, dev)
        lib_call("riqn_z_wgrad", rows, HID, A, dptr(dzd), dptr(hd), o["dwz"].p, o["dbz"].p, *[dptr(e) for e in epsd],
                 *[o[n].p for n in names])
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = _three_calls(call)
    sel = _rows(32, rows)
    dwz = o["dwz"].f32().reshape(32, 2 * HID)[sel]
    split = min(32, -(-rows // 64))
    want = F32(0) + split_k_sum(dz[:, sel], h, split)
    assert_bits(f"dwz rows {list(sel)} ({-(-rows // kchunk(rows, split))} splits)", f32_bits(dwz), f32_bits(want))
    ref = dz[:, sel].astype(np.float64).T @ h
    check_bound("dwz", dwz, ref, C_BOUND * (rows + 2) * U * (np.abs(dz[:, sel]).astype(np.float64).T @ h))


EMB_SHAPES = [(4, 16), (13, 13), (37, 33), (512, 64)]        # R = 64: one split


@pytest.mark.gpu
@pytest.mark.parametrize("B,Nq", EMB_SHAPES, ids=[f"B{b}-Nq{n}" for b, n in EMB_SHAPES])
def test_quantile_embed_bwd_is_the_ordered_split_k_sum(cuda_dev, B, Nq):
    """riqn_quantile_embed_bwd's grad_iqn_w += dpre^T cos: splits of whole k-slabs over the B * Nq rows (3 per SM over
    the 128-row tiles), added in split order, then once onto the prefill; bit for bit on a row subsample, on the dpre
    the call wrote into dX.  Every output identical over three calls."""
    dev = cuda_dev
    F, E, R = 3136, 64, B * Nq
    rs = np.random.RandomState(R)
    x = rs.standard_normal((R, F)).astype(F32)
    x[rs.uniform(size=x.shape) < 0.3] = 0
    feat = np.maximum(rs.standard_normal((B, F)), 0).astype(F32)
    cos = rs.uniform(-1, 1, (R, E)).astype(F32)
    dx = (rs.standard_normal((R, F)) * 1e-2).astype(F32)
    pre_w, pre_b = rs.standard_normal(F * E).astype(F32), rs.standard_normal(F).astype(F32)
    xd, fd, cd = to_dev(x, dev), to_dev(feat, dev), to_dev(cos, dev)

    def call():
        o = {"dx": Out(R * F, dev, fill=dx), "dfeat": Out(B * F, dev), "grad_w": Out(F * E, dev, fill=pre_w),
             "grad_b": Out(F, dev, fill=pre_b)}
        lib_call("riqn_quantile_embed_bwd", B, Nq, E, F, dptr(xd), dptr(fd), dptr(cd), o["dx"].p, o["dfeat"].p,
                 o["grad_w"].p, o["grad_b"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = _three_calls(call)
    dpre = o["dx"].f32().reshape(R, F)
    sel = _rows(F, R)
    split = min(-(-3 * _sms(dev) // -(-F // 128)), -(-R // 64))
    got = o["grad_w"].f32().reshape(F, E)[sel]
    want = pre_w.reshape(F, E)[sel] + split_k_sum(dpre[:, sel], cos, split)
    assert_bits(f"grad_iqn_w rows {list(sel)} ({-(-R // kchunk(R, split))} splits)", f32_bits(got), f32_bits(want))
    d64 = dpre[:, sel].astype(np.float64)
    check_bound("grad_iqn_w", got, pre_w.reshape(F, E)[sel] + d64.T @ cos,
                C_BOUND * (R + 2) * U * (np.abs(d64).T @ np.abs(cos) + np.abs(pre_w.reshape(F, E)[sel])))


def _conv_inputs(name, B, rs):
    cin, h, cout, k, s, pad = GEOMS[name]
    oh = out_size(h, k, s, pad)
    x = np.maximum(rs.standard_normal((B, cin, h, h)), 0).astype(F32)
    w = (rs.standard_normal((cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(F32)
    dout, out = grads(rs, (B, cout, oh, oh), "random")
    return x, w, masked(dout, out), dout, out


def _check_din(what, din, dcol, dy, w, B, name, samples):
    """din of the sample subset: bitwise the ordered gather of the call's own dcol, and inside the float64 bound"""
    cin, h, cout, k, s, pad = GEOMS[name]
    oh = out_size(h, k, s, pad)
    rows = dcol.reshape(B, oh * oh, -1)[samples].reshape(-1, dcol.shape[-1])
    want = col2im_sum(rows, len(samples), cin, h, k, s, pad)
    got = din.reshape(B, cin, h, h)[samples]
    assert_bits(f"{what} din samples {list(samples)}", f32_bits(got + F32(0)), f32_bits(want + F32(0)))
    shape = (len(samples), cin, h, h)
    check_bound(f"{what} din", got, dgrad64(dy[samples], w, shape, s, pad),
                C_BOUND * (cout + k * k) * U * dgrad64(np.abs(dy[samples]), np.abs(w), shape, s, pad))


CONV_CASES = [(n, B) for n in ("conv1", "conv2", "conv3", "big") for B in (3, 13, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", CONV_CASES, ids=[f"{n}-B{b}" for n, b in CONV_CASES])
def test_conv_bwd_is_the_ordered_statement(cuda_dev, name, B):
    """riqn_conv_bwd: dW += dY^T col as splits of whole k-slabs over the B * OH * OW rows (2 per SM over the 128 x 128
    tiles, at least 64 rows each), added in split order, then once onto the prefill; din the ordered gather of dcol.
    Bit for bit on a subsample of dW rows and samples; every output identical over three calls."""
    dev = cuda_dev
    cin, h, cout, k, s, pad = GEOMS[name]
    oh = out_size(h, k, s, pad)
    M, K = B * oh * oh, cin * k * k
    rs = np.random.RandomState(M + K)
    x, w, dy, dout, out = _conv_inputs(name, B, rs)
    pre_w, pre_b = rs.standard_normal(cout * K).astype(F32), rs.standard_normal(cout).astype(F32)
    g = geom(B, cin, h, cout, k, s, pad)
    xd, wd, doutd, outd = to_dev(x, dev), to_dev(w, dev), to_dev(dout, dev), to_dev(out, dev)
    col = Out(M * K, dev)
    lib_call("riqn_im2col_f32", g, dptr(xd), 0, col.p)

    def call():
        o = {"dY": Out(M * cout, dev), "dcol": Out(M * K, dev), "dw": Out(cout * K, dev, fill=pre_w),
             "db": Out(cout, dev, fill=pre_b), "din": Out(B * cin * h * h, dev)}
        lib_call("riqn_conv_bwd", g, dptr(doutd), dptr(outd), col.p, dptr(wd), o["dY"].p, o["dcol"].p, o["dw"].p,
                 o["db"].p, o["din"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = _three_calls(call)
    dym = dy.transpose(0, 2, 3, 1).reshape(M, cout)
    colh = col.f32().reshape(M, K)
    assert_bits("col", f32_bits(colh), f32_bits(im2col(x, k, s, pad)))
    tiles = -(-cout // 128) * -(-K // 128)
    split = min(-(-2 * _sms(dev) // tiles), -(-M // 64))
    sel = _rows(cout, M)
    got = o["dw"].f32().reshape(cout, K)[sel]
    want = pre_w.reshape(cout, K)[sel] + split_k_sum(dym[:, sel], colh, split)
    tag = f"{name} B{B}"
    assert_bits(f"{tag} dw rows {list(sel)} ({-(-M // kchunk(M, split))} splits)", f32_bits(got), f32_bits(want))
    d64 = dym[:, sel].astype(np.float64)
    check_bound(f"{tag} dw", got, pre_w.reshape(cout, K)[sel] + d64.T @ colh,
                C_BOUND * (M + 2) * U * (np.abs(d64).T @ np.abs(colh) + np.abs(pre_w.reshape(cout, K)[sel])))
    _check_din(tag, o["din"].f32(), o["dcol"].f32().reshape(M, K), dy, w, B, name, _rows(B, B, 1))


TC_CASES = [(n, B) for n in ("conv2", "conv3", "pad1") for B in (8, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", TC_CASES, ids=[f"{n}-B{b}" for n, b in TC_CASES])
def test_conv_bwd_tc_din_is_the_ordered_gather(cuda_dev, name, B):
    """riqn_conv_bwd_tc writes dcol = dY W on the tensor cores at every padding, and din is its ordered gather, bit for
    bit; dcol and dw inside float64 bounds on the bf16 operands; every output identical over three calls."""
    dev = cuda_dev
    cin, h, cout, k, s, pad = GEOMS[name]
    oh = out_size(h, k, s, pad)
    M, K = B * oh * oh, cin * k * k
    rs = np.random.RandomState(M + K + pad)
    x, w, dy, dout, out = _conv_inputs(name, B, rs)
    x, w = bf16(x), bf16(w)
    dyb = bf16(dy)
    dym = dyb.transpose(0, 2, 3, 1).reshape(M, cout)
    col = im2col(x, k, s, pad)
    pre_w, pre_b = rs.standard_normal(cout * K).astype(F32), rs.standard_normal(cout).astype(F32)
    d = dict(dout=to_dev(dout, dev), out=to_dev(out, dev), colT=to_dev_bf16(np.ascontiguousarray(col.T), dev),
             wT=to_dev_bf16(np.ascontiguousarray(w.reshape(cout, K).T), dev))
    g = geom(B, cin, h, cout, k, s, pad)

    def call():
        o = {"dY": Out(M * cout, dev, torch.bfloat16), "dYT": Out(cout * M, dev, torch.bfloat16), "dcol": Out(M * K, dev),
             "dw": Out(cout * K, dev, fill=pre_w), "db": Out(cout, dev, fill=pre_b), "din": Out(B * cin * h * h, dev)}
        lib_call("riqn_conv_bwd_tc", g, dptr(d["dout"]), dptr(d["out"]), dptr(d["colT"]), dptr(d["wT"]), o["dY"].p,
                 o["dYT"].p, o["dcol"].p, o["dw"].p, o["db"].p, o["din"].p, 1.0)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = _three_calls(call)
    tag = f"{name} B{B}"
    samples = _rows(B, B, 1)
    dcol = o["dcol"].f32().reshape(M, K)
    rows = (np.arange(M).reshape(B, -1)[samples]).ravel()
    w2 = w.reshape(cout, K).astype(np.float64)
    check_bound(f"{tag} dcol", dcol[rows], dym[rows].astype(np.float64) @ w2,
                C_BOUND * (cout + 1) * U * (np.abs(dym[rows]).astype(np.float64) @ np.abs(w2)))
    dw = o["dw"].f32().reshape(cout, K)
    check_bound(f"{tag} dw", dw, pre_w.reshape(cout, K) + dym.astype(np.float64).T @ col,
                C_BOUND * (M + 2) * U * (np.abs(dym).astype(np.float64).T @ np.abs(col) + np.abs(pre_w.reshape(cout, K))))
    _check_din(tag, o["din"].f32(), dcol, dyb, w, B, name, samples)


# ---------------------------------------------------------------------------------------------- c. learner steps (GPU)
IQN_ODD = dict(batch_size=13, num_tau_samples=13, num_tau_prime_samples=11, num_quantile_samples=7)
STEP_CASES = {"iqn-B13-N13": (0, IQN_ODD, None),                  # the fp32 trunk and head backwards
              "c51-B13": (1, dict(batch_size=13), None),           # the fp32 trunk backward
              "iqn-history3-B32": (0, dict(batch_size=32, history_length=3), None),   # the im2col tensor-core trunk
              "iqn-fp32-B32": (0, dict(batch_size=32), ("fp32", "fp32"))}


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_fallback_learner_steps_are_bitwise_reproducible(cuda_dev, precision, case, graph):  # noqa: F811
    """Two learners from the same seed, four steps each on a backward path the benchmarked size does not take: the same
    sampled indices, losses and parameter arena, bit for bit, eagerly and replayed from the step graph."""
    rainbow_only, fields, mode = STEP_CASES[case]
    if mode is not None:
        precision(*mode)
    _assert_steps_bitwise_reproducible(cuda_dev, graph, rainbow_only=rainbow_only, cap=1 << 14, steps=4, **fields)
