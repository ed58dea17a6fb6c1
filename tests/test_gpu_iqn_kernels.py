"""The IQN learner's forward and loss path below the hidden layer, entry point by entry point, against float64 statements
of the same operations (include/riqn_b200.h): riqn_dueling_fwd (the register kernel, the streamed kernel from 4096 rows
and the A > 24 kernel), riqn_argmax_mean and the quantile-Huber loss riqn_iqn_loss_fwd_bwd, with the argument contracts
of these and of riqn_iqn_loss_fwd_bwd_h / riqn_miqn_loss_fwd_bwd.

Method (as tests/test_gpu_head_kernels.py):
* exact regime: small integers and dyadic values make every product and partial sum exact in fp32 in any order (the
  test asserts the condition on the host), so the kernel has to match float64 bit for bit;
* random regime: each element is held to a first-order bound of the kernel's roundings, and each test prints its worst
  err/bound ratio;
* single-rounding outputs (the targets, theta, a*) must equal a numpy float32 statement bit for bit in both regimes;
* overwritten outputs start as NaN (a_star as an int64 sentinel), every buffer carries canaries past its end, every call
  is made twice and must agree bit for bit, and refused calls raise and write nothing.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

from helpers import PAD, U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, load_params, \
    make_args, rel_err, to_dev
from oracle import cases, losses, network as net

HID = 512
F32 = np.float32
A_SENTINEL = -5         # int64 prefill of a_star


def _riqn_error():
    from rainbow_iqn_apex_b200._lib import RiqnError
    return RiqnError


# ---------------------------------------------------------------------------------------------- dueling forward
def _dueling_call(dev, rows, B, A, hd, wzd, bzd, hidden=HID):
    q = Out(rows * A, dev)
    lib_call("riqn_dueling_fwd", rows, B, hidden, A, dptr(hd), dptr(wzd), dptr(bzd), q.p)
    torch.cuda.synchronize()
    assert_canaries({"q": q})
    return q


_H = {}


def _hidden(dev, rows, regime):
    """h (rows, 1024) >= 0 as the ReLU leaves it, host and device copies; kept for the A values of one row count"""
    if (rows, regime) not in _H:
        if any(k[0] != rows for k in _H):
            _H.clear()
        g = torch.Generator().manual_seed(rows * 2 + (regime == "exact"))
        if regime == "exact":       # small integers times 2^-2, 30 % zeros
            h = torch.randint(0, 8, (rows, 2 * HID), generator=g).float().mul_(0.25)
            h.mul_(torch.rand(rows, 2 * HID, generator=g) >= 0.3)
        else:
            h = torch.randn(rows, 2 * HID, generator=g).clamp_(min=0)
        _H[(rows, regime)] = (h, h.to(dev))
    return _H[(rows, regime)]


def _zero_sum_columns(rs, A):
    """A x HID integers in [-3, 3] whose every column sums to 0: then sum_a a_a = sum_a bz_a for every row"""
    if A == 1:
        return np.zeros((1, HID), np.int64)
    w = rs.randint(-3, 4, (A, HID))
    cols = np.arange(HID)
    for _ in range(10000):
        s = w.sum(0)
        if not s.any():
            return w
        k = rs.randint(0, A, HID)
        cand = w[k, cols] - np.sign(s)
        ok = (s != 0) & (np.abs(cand) <= 3)
        w[k[ok], cols[ok]] = cand[ok]
    raise AssertionError("no zero-sum weight columns")


def _z_weights(A, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        # w in [-3, 3] * 2^-6 (the advantage columns summing to 0), b on the 2^-8 grid with sum_a b_a = A * t * 2^-8:
        # the advantage sum is then a multiple of A on the grid, and its mean exact
        wz = np.concatenate([rs.randint(-3, 4, (1, HID)), _zero_sum_columns(rs, A)]).astype(F32) / 64
        ba = rs.randint(-256, 257, A)
        ba[-1] = A * rs.choice([-3, -2, -1, 1, 2, 3]) - ba[:-1].sum()
        bz = np.concatenate([[rs.randint(-256, 257)], ba]).astype(F32) / 256
    else:
        wz = (rs.standard_normal((1 + A, HID)) * 0.05).astype(F32)
        bz = rs.standard_normal(1 + A).astype(F32)
    return wz, bz


def _dueling_ref(h, wz, bz, B, exact):
    """float64 q in quantile-major rows and its first-order error bound: each dot within 512 u sum|h_i w_i| plus the bias
    add, the action sum within A u sum|a_k| plus the dots' errors, one rounding each for the mean, v + a and the
    subtraction.  exact: assert (units of 2^-8) that every partial sum fits in 24 bits and the mean is exact."""
    R, A = h.shape[0], wz.shape[0] - 1
    w64, b64 = torch.from_numpy(wz).double(), torch.from_numpy(bz).double()
    q, bnd = np.empty((R, A)), np.empty((R, A))
    for lo in range(0, R, 8192):
        hc = h[lo:lo + 8192].double()
        sv, sa = hc[:, :HID] @ w64[0].abs(), hc[:, HID:] @ w64[1:].abs().t()          # h >= 0
        v = hc[:, :HID] @ w64[0] + b64[0]
        a = hc[:, HID:] @ w64[1:].t() + b64[1:]
        asum = a.sum(1)
        mean = asum / A
        qq = v[:, None] + a - mean[:, None]
        if exact:
            lim = 2.0 ** 24 / 256
            assert float((sv + b64[0].abs()).max()) < lim and float((sa + b64[1:].abs()).max()) < lim
            assert float(a.abs().sum(1).max()) < lim
            assert bool(torch.all(torch.remainder(asum * 256, A) == 0)), "advantage sum not a multiple of A"
            assert float((v.abs()[:, None] + a.abs() + mean.abs()[:, None]).max()) < lim
        e_v = 512 * U * sv + U * v.abs()
        e_a = 512 * U * sa + U * a.abs()
        e_mean = (e_a.sum(1) + A * U * a.abs().sum(1)) / A + U * mean.abs()
        e_q = e_v[:, None] + e_a + e_mean[:, None] + U * (v[:, None] + a).abs() + U * qq.abs()
        q[lo:lo + 8192], bnd[lo:lo + 8192] = qq.numpy(), e_q.numpy()
    nq = R // B
    perm = (np.arange(R) % nq) * B + np.arange(R) // nq         # sample-major row r -> quantile-major row
    out_q, out_b = np.empty_like(q), np.empty_like(bnd)
    out_q[perm], out_b[perm] = q, bnd
    if exact:
        assert np.array_equal(out_q.astype(F32).astype(np.float64), out_q), "q not representable in fp32"
    return out_q, out_b


def _register_slices(dev, hd, wzd, bzd, rows, B, A):
    """riqn_dueling_fwd on < 4096-row slices (the register kernel), mapped back to the quantile-major rows of one call
    over all rows: slices of rows for B = 1 (the row map is the identity), of whole samples otherwise"""
    out = torch.empty(rows, A, device=dev)
    nq = rows // B
    if B == 1:
        for lo in range(0, rows, 4000):
            n = min(4000, rows - lo)
            out[lo:lo + n] = _dueling_call(dev, n, 1, A, hd[lo:lo + n], wzd, bzd).t[:n * A].view(n, A)
    else:
        per = 4095 // nq
        assert per >= 1
        for b0 in range(0, B, per):
            nb = min(per, B - b0)
            qs = _dueling_call(dev, nb * nq, nb, A, hd[b0 * nq:(b0 + nb) * nq], wzd, bzd)
            out.view(nq, B, A)[:, b0:b0 + nb] = qs.t[:nb * nq * A].view(nq, nb, A)
    return out


# (rows, B): single rows, a ragged last 4-row group below and above 4096, a ragged final bulk copy, B > 1 with Nq > 1
DUEL_ROWS = [(1, 1), (3, 3), (4095, 5), (4096, 64), (4097, 17), (8197, 7), (8203, 1), (32768, 512), (65536, 512)]
DUEL_A = [1, 2, 3, 9, 17, 18, 23, 24, 25, 31]
DUEL_CASES = [(r, b, a) for r, b in DUEL_ROWS for a in DUEL_A]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,B,A", DUEL_CASES, ids=[f"R{r}-B{b}-A{a}" for r, b, a in DUEL_CASES])
def test_dueling_fwd(cuda_dev, rows, B, A):
    """A <= 24: the register kernel below 4096 rows, the streamed kernel from 4096 rows (odd A runs its unpaired last
    action); A = 25, 31: the warp-per-row kernel.  Exact regime bitwise against float64, random regime within the bound;
    the streamed kernel bitwise equal to the register kernel over slices."""
    dev = cuda_dev
    for regime in ("exact", "random"):
        h, hd = _hidden(dev, rows, regime)
        wz, bz = _z_weights(A, regime, seed=rows * 40 + A)
        wzd, bzd = to_dev(wz, dev), to_dev(bz, dev)
        q = _dueling_call(dev, rows, B, A, hd, wzd, bzd)
        assert_bits(f"second call {regime}", _dueling_call(dev, rows, B, A, hd, wzd, bzd).bits(), q.bits())
        ref, bnd = _dueling_ref(h, wz, bz, B, regime == "exact")
        got = q.f32().reshape(rows, A)
        if regime == "exact":
            assert_bits("q (float64)", f32_bits(got), f32_bits(ref))
        else:
            check_bound(f"q R{rows} B{B} A{A}", got, ref, bnd)
        if A <= 24 and rows >= 4096:
            sl = _register_slices(dev, hd, wzd, bzd, rows, B, A)
            assert_bits(f"streamed vs register kernel {regime}", q.bits(),
                        sl.reshape(-1).view(torch.int32).cpu().numpy().view(np.uint32))


@pytest.mark.gpu
def test_dueling_fwd_refusals(cuda_dev):
    """Refused before any launch, q untouched: misaligned h or wz (register, streamed and A > 24 paths), rows not whole
    samples, batch 0, A outside 1..31, hidden != 512.  The in-range neighbours run."""
    dev = cuda_dev
    rows_max = 4096
    hbuf = torch.rand(rows_max * 2 * HID + 4, device=dev)
    wbuf = torch.rand(32 * HID + 4, device=dev)
    bz = torch.rand(32, device=dev)
    h, wz = hbuf[:-4], wbuf[:-4]
    bad = [(8, 1, HID, 18, hbuf[1:], wz, "h misaligned"), (4096, 1, HID, 18, hbuf[1:], wz, "h misaligned, streamed"),
           (8, 1, HID, 25, hbuf[1:], wz, "h misaligned, A > 24"), (8, 1, HID, 18, h, wbuf[1:], "wz misaligned"),
           (4096, 1, HID, 9, h, wbuf[1:], "wz misaligned, streamed"), (8, 1, HID, 31, h, wbuf[1:], "wz misaligned, A > 24"),
           (11, 5, HID, 18, h, wz, "rows % batch"), (8, 0, HID, 18, h, wz, "batch 0"), (8, 1, HID, 0, h, wz, "A = 0"),
           (8, 1, HID, 32, h, wz, "A = 32"), (8, 1, 256, 18, h, wz, "hidden 256")]
    for rows, B, hidden, A, hh, ww, tag in bad:
        q = Out(rows * max(A, 1), dev)
        with pytest.raises(_riqn_error()):
            lib_call("riqn_dueling_fwd", rows, B, hidden, A, dptr(hh), dptr(ww), dptr(bz), q.p)
        torch.cuda.synchronize()
        assert q.canaries_ok() and bool(torch.isnan(q.t[:q.n]).all()), f"refused call ({tag}) wrote q"
    for rows, B, A in ((10, 5, 18), (8, 1, 1), (8, 1, 31), (4096, 1, 9)):
        q = _dueling_call(dev, rows, B, A, h, wz, bz)
        assert bool(torch.isfinite(q.t[:q.n]).all())


# ---------------------------------------------------------------------------------------------- argmax of the mean
def _argmax_statement(q, K, B, A):
    """numpy float32: s = ((q_0 + q_1) + ...) / K with k ascending, then the first maximal index"""
    q3 = q.reshape(K, B, A)
    s = np.zeros((B, A), F32)
    for k in range(K):
        s = s + q3[k]
    s = s / F32(K)
    return s, s.argmax(1)


def _argmax_data(K, B, A, seed):
    """Gaussian q (K*B, A) with constructed ties: {row: tied best actions}"""
    rs = np.random.RandomState(seed)
    q = torch.randn(K, B, A, generator=torch.Generator().manual_seed(seed)).numpy()
    ties = {}

    def tie(b, acts):
        if b < B and len(set(acts)) == len(acts) and max(acts) < A and b not in ties:
            q[:, b, acts[0]] += 50.0
            for a in acts[1:]:
                q[:, b, a] = q[:, b, acts[0]]
            ties[b] = sorted(acts)
    if A >= 2:
        i = rs.randint(0, A - 1)
        tie(0, [i, rs.randint(i + 1, A)])                          # a copied column
        tie(1, [A - 1, 0])                                         # lanes 0 and A - 1 (31 at A = 32)
        tie(2, [A - 1, 1, A // 2])                                 # three-way
        if B > 3:
            q[:, 3, :] = q[:, 3, :1]                               # all equal
            ties[3] = list(range(A))
        if K >= 2:                                                 # +0 against -0 means: -2^-149 / K rounds to -0
            for b, (neg, pos) in ((4, (0, A - 1)), (5, (A - 1, 0))):
                if b < B - 1:
                    q[:, b, :] = -1.0
                    q[:, b, pos] = 0.0
                    q[:, b, neg] = 0.0
                    q[0, b, neg] = -(2.0 ** -149)
                    ties[b] = sorted((neg, pos))
        tie(B - 1, [A - 1, A // 3])                                # the last row: the ragged last block
    return np.ascontiguousarray(q.reshape(K * B, A), F32), ties


def _argmax_call(dev, B, K, A, qd):
    a = torch.full((B + PAD,), A_SENTINEL, dtype=torch.int64, device=dev)
    lib_call("riqn_argmax_mean", B, K, A, dptr(qd), a.data_ptr())
    torch.cuda.synchronize()
    assert bool(torch.all(a[B:] == A_SENTINEL)), "a_star written past the batch"
    return a[:B].cpu().numpy()


@pytest.mark.gpu
def test_argmax_mean_gaussian(cuda_dev):
    """Gaussian q (no ties) at B = 37, K = 32, A = 18: a* equals torch's mean-then-argmax, the reference's statement
    (compute_loss_iqn.py:238-245), and the numpy float32 statement."""
    rs = np.random.RandomState(1)
    B, K, A = 37, 32, 18
    q = rs.standard_normal((K * B, A)).astype(F32)
    got = _argmax_call(cuda_dev, B, K, A, to_dev(q, cuda_dev))
    assert np.array_equal(got, torch.from_numpy(q).reshape(K, B, A).mean(0).argmax(1).numpy())
    assert np.array_equal(got, _argmax_statement(q, K, B, A)[1])


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 7, 32, 64, 200, 256])
@pytest.mark.parametrize("A", [1, 2, 17, 31, 32])
def test_argmax_mean_grid(cuda_dev, A, K):
    """a* equals the numpy float32 statement on every row (one warp per row: several blocks and a ragged last one),
    and the first of equal maxima wins on copied columns, lanes 0 and A - 1, three-way ties, all-equal rows and
    +0 / -0 means."""
    dev = cuda_dev
    for B in (1, 37, 512, 4096, 12345):
        q, ties = _argmax_data(K, B, A, seed=K * 1000 + A * 10 + B)
        s, want = _argmax_statement(q, K, B, A)
        for b, acts in ties.items():
            assert np.all(s[b, acts] == s[b, acts[0]]) and s[b, acts[0]] == s[b].max(), f"row {b}: not a tie"
            assert want[b] == acts[0]
        for b in (4, 5):
            if b in ties:
                # the device adds the subnormal -2^-149 and divides by K: an exact mean in (-2^-150, 0] rounds to -0.
                # Checked in float64, where the value is normal, so that no host flush-to-zero setting matters.
                m = q.reshape(K, B, A)[:, b].astype(np.float64).sum(0) / K
                assert np.sum((m < 0) & (m >= -2.0 ** -150)) == 1 and np.sum(m == 0) == 1, "no +0 / -0 pair"
        qd = to_dev(q, dev)
        got = _argmax_call(dev, B, K, A, qd)
        assert np.array_equal(got, want), \
            f"B{B}: a* differs at rows {np.flatnonzero(got != want)[:6]}: {got[got != want][:6]} want {want[got != want][:6]}"
        assert np.array_equal(_argmax_call(dev, B, K, A, qd), got), "second call differs"


@pytest.mark.gpu
def test_argmax_mean_refusals(cuda_dev):
    dev = cuda_dev
    qd = torch.randn(8 * 4 * 33, device=dev)
    for B, K, A in ((0, 8, 4), (4, 0, 4), (4, 8, 0), (4, 8, 33)):
        a = torch.full((4 + PAD,), A_SENTINEL, dtype=torch.int64, device=dev)
        with pytest.raises(_riqn_error()):
            lib_call("riqn_argmax_mean", B, K, A, dptr(qd), a.data_ptr())
        torch.cuda.synchronize()
        assert bool(torch.all(a == A_SENTINEL)), f"refused call (B {B}, K {K}, A {A}) wrote a_star"


# ---------------------------------------------------------------------------------------------- quantile-Huber loss
def huber_statement(T, th, ta, kappa):
    """float64 statement of the loss and its theta gradient (include/riqn_b200.h), T (B, N'), th and ta (B, N):
    loss[b] = (1/N') sum_{j,i} |ta_i - 1{d<0}| huber(d) / kappa, dth[b, i] = -(1/N') sum_j |ta_i - 1{d<0}| dh(d) / kappa,
    d = T_j - th_i.  Also returns the per-pair terms t and g, d and w for the bounds."""
    d = np.asarray(T, np.float64)[:, :, None] - np.asarray(th, np.float64)[:, None, :]
    ad = np.abs(d)
    quad = ad <= kappa
    hub = np.where(quad, 0.5 * d * d, kappa * (ad - 0.5 * kappa))
    dh = np.where(quad, d, np.copysign(kappa, d))
    w = np.abs(np.asarray(ta, np.float64)[:, None, :] - (d < 0))
    t, g = w * hub / kappa, w * dh / kappa
    Np = d.shape[1]
    return t.sum((1, 2)) / Np, (0.0 - g.sum(1)) / Np, t, g, d, w          # 0 - sum: +0 as the kernel's chain


def _f32_quotient(num, n):
    """fl32(num / n), correctly rounded, for exact float64 num: the float64 quotient rounds once more only where it
    lands on an fp32 midpoint, and there the exact quotient decides"""
    x = num / n
    f = x.astype(F32)
    m = f.astype(np.float64)
    other = np.nextafter(f, np.where(x > m, np.inf, -np.inf).astype(F32)).astype(np.float64)
    for i in np.flatnonzero((x != m) & (x == (m + other) / 2)):
        e, xm = Fraction(float(num.flat[i])) / n, Fraction(float(x.flat[i]))
        if e != xm and (e > xm) == (other.flat[i] > m.flat[i]):
            f.flat[i] = F32(other.flat[i])
    return f


def _loss_inputs(B, N, Np, A, kappa, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        # theta, T on the grid kappa/4 within +-2 kappa (both Huber regions, d == 0 and |d| == kappa), gamma^n = 1/2 on
        # even targets, tau in {0, 1/4, 1/2, 3/4}: every term is a multiple of kappa/128, every gradient term of 1/16
        s = kappa / 4
        q_on = (rs.randint(-4, 5, (N * B, A)) * s).astype(F32)
        q_tg = (rs.randint(-2, 3, (Np * B, A)) * 2 * s).astype(F32)
        ret = (rs.randint(-2, 3, B) * s).astype(F32)
        tau = (rs.randint(0, 4, N * B) / 4).astype(F32)
        gamma_n = 0.5
    else:
        q_on = (rs.standard_normal((N * B, A)) * kappa).astype(F32)
        q_tg = (rs.standard_normal((Np * B, A)) * kappa).astype(F32)
        ret = (rs.standard_normal(B) * kappa / 2).astype(F32)
        tau = rs.uniform(0, 1, N * B).astype(F32)
        edges = np.array([0.0, 2.0 ** -24, 1 - 2.0 ** -24], F32)
        pick = rs.choice(N * B, min(N * B, 3 * max(1, B // 4)), replace=False)
        tau[pick] = edges[np.arange(len(pick)) % 3]
        gamma_n = 0.99 ** 3
    nt = (rs.uniform(size=B) < 0.8).astype(F32)
    nt[0] = 0.0                                                    # a terminal row
    act = rs.randint(0, A, B).astype(np.int64)
    ast = rs.randint(0, A, B).astype(np.int64)
    if A > 1:
        ast[0] = (act[0] + 1) % A                                  # a* != the taken action
    return dict(q_on=q_on, q_tg=q_tg, tau=tau, act=act, ast=ast, ret=ret, nt=nt), gamma_n


def _loss_statements(h, B, N, Np, A, gamma_n):
    """the kernel's targets fl(R + fl(fl(gamma^n nt) Z)) and theta as numpy float32, tau as (B, N)"""
    rows = np.arange(B)
    g = (F32(gamma_n) * h["nt"]).astype(F32)
    z = h["q_tg"].reshape(Np, B, A)[:, rows, h["ast"]].T
    T = (h["ret"][:, None] + (g[:, None] * z).astype(F32)).astype(F32)
    th = h["q_on"].reshape(N, B, A)[:, rows, h["act"]].T
    return T, np.ascontiguousarray(th), h["tau"].reshape(N, B).T


def _loss_dev(h, dev):
    return {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}


def _loss_call(dev, d, B, N, Np, A, gamma_n, kappa, debug_out=True):
    o = {"loss": Out(B, dev), "dth": Out(N * B, dev), "theta": Out(B * N, dev) if debug_out else None,
         "target": Out(B * Np, dev) if debug_out else None}
    lib_call("riqn_iqn_loss_fwd_bwd", B, N, Np, A, *[dptr(d[k]) for k in ("q_on", "q_tg", "tau", "act", "ast", "ret", "nt")],
             float(gamma_n), float(kappa), o["loss"].p, o["dth"].p, o["theta"].p if debug_out else None,
             o["target"].p if debug_out else None)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _check_loss_rows(B, N, Np):
    """the rows held to float64: all of them, or the first, the last and a spread sample where B N N' is large"""
    n = max(2, min(B, (1 << 22) // (N * Np)))
    return np.unique(np.concatenate([[0, B - 1], np.linspace(0, B - 1, n).astype(np.int64)]))


LOSS_SHAPES = [(1, 1), (8, 8), (33, 64), (64, 64), (16, 40), (100, 9), (256, 256), (1500, 64), (64, 2000)]
KAPPAS = [1.0, 0.5, 2.0, 2.0 ** -10, 64.0]


@pytest.mark.gpu
@pytest.mark.parametrize("kappa", KAPPAS, ids=[f"k{k:g}" for k in KAPPAS])
@pytest.mark.parametrize("N,Np", LOSS_SHAPES, ids=[f"N{n}-Np{p}" for n, p in LOSS_SHAPES])
def test_iqn_loss(cuda_dev, N, Np, kappa):
    """target_out and theta_out bitwise against the numpy float32 statement; loss and dtheta bitwise against float64 in
    the exact regime (d == 0 and |d| == kappa both occur) and within the per-element bound in the random regime; NULL
    theta_out / target_out give the same bits; a second call is bitwise the first."""
    dev = cuda_dev
    n_zero = n_kappa = 0
    big = 4096 if max(N, Np) * 4096 * 32 <= (1 << 25) else 512
    for A, B in ((1, 1), (18, 512), (32, big)):
        threads = min(1024, max(32, (max(N, Np) + 31) // 32 * 32))
        per_thread = -(-N // threads)
        for regime in ("exact", "random"):
            h, gamma_n = _loss_inputs(B, N, Np, A, kappa, regime, seed=N * 7 + Np * 13 + A + B + int(kappa * 1024))
            d = _loss_dev(h, dev)
            tag = f"A{A} B{B} {regime}"
            o = _loss_call(dev, d, B, N, Np, A, gamma_n, kappa)
            T, th, ta = _loss_statements(h, B, N, Np, A, gamma_n)
            assert_bits(f"target {tag}", o["target"].bits(), f32_bits(T).ravel())
            assert_bits(f"theta {tag}", o["theta"].bits(), f32_bits(th).ravel())
            o2 = _loss_call(dev, d, B, N, Np, A, gamma_n, kappa, debug_out=False)
            o3 = _loss_call(dev, d, B, N, Np, A, gamma_n, kappa)
            for k in ("loss", "dth"):
                assert_bits(f"{k} without theta_out / target_out {tag}", o2[k].bits(), o[k].bits())
                assert_bits(f"{k} second call {tag}", o3[k].bits(), o[k].bits())
            for k in ("theta", "target"):
                assert_bits(f"{k} second call {tag}", o3[k].bits(), o[k].bits())
            rows = _check_loss_rows(B, N, Np)
            loss, dth, t, g, dd, w = huber_statement(T[rows], th[rows], ta[rows], kappa)
            S, G = t.sum((1, 2)), 0.0 - g.sum(1)                   # exact in float64 in the exact regime
            got_loss = o["loss"].f32()[rows]
            got_dth = o["dth"].f32().reshape(N, B).T[rows]
            if regime == "exact":
                qt, qg = kappa / 128, 1.0 / 16
                assert np.all(np.mod(t / qt, 1) == 0) and np.all(np.mod(g / qg, 1) == 0), "terms off the grid"
                assert float(np.abs(t).sum((1, 2)).max()) / qt < 2 ** 24, "loss sum beyond 24 bits"
                assert float(np.abs(g).sum(1).max()) / qg < 2 ** 24, "gradient sum beyond 24 bits"
                n_zero += int((dd == 0).sum())
                n_kappa += int((np.abs(dd) == kappa).sum())
                assert_bits(f"loss {tag}", f32_bits(got_loss), f32_bits(_f32_quotient(S, Np)))
                assert_bits(f"dtheta {tag}", f32_bits(got_dth), f32_bits(_f32_quotient(G, Np)))
            else:
                ad = np.abs(dd)
                e_t = U * (w * ad * np.minimum(ad, kappa) / kappa + 6 * np.abs(t)) + 2.0 ** -126
                e_loss = (e_t.sum((1, 2)) + (Np + per_thread + 10) * U * np.abs(t).sum((1, 2))) / Np + U * np.abs(loss)
                check_bound(f"loss N{N} N'{Np} k{kappa:g} {tag}", got_loss, loss, e_loss)
                e_g = U * (w * ad * (ad <= kappa) / kappa + 4 * np.abs(g)) + 2.0 ** -126
                e_dth = (e_g.sum(1) + Np * U * np.abs(g).sum(1)) / Np + U * np.abs(dth)
                check_bound(f"dtheta N{N} N'{Np} k{kappa:g} {tag}", got_dth, dth, e_dth)
    assert n_zero > 0 and n_kappa > 0, f"the exact grids gave d == 0 {n_zero} times and |d| == kappa {n_kappa} times"


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,Np,kappa", [(7, 8, 8, 1.0), (33, 64, 64, 1.0), (4, 16, 40, 0.5), (3, 100, 9, 2.0)])
def test_iqn_loss_vs_autograd(cuda_dev, B, N, Np, kappa):
    """The kernel against torch autograd of oracle.losses.iqn_pairwise_loss under per-transition weights: dtheta * w
    is dL/dq_online at the taken action."""
    rs = np.random.RandomState(B)
    A = 18
    q_on = torch.from_numpy(rs.standard_normal((N * B, A)).astype(F32)).requires_grad_(True)
    q_tg = torch.from_numpy(rs.standard_normal((Np * B, A)).astype(F32))
    tau = torch.from_numpy(rs.uniform(0, 1, (N * B, 1)).astype(F32))
    actions = torch.from_numpy(rs.randint(0, A, B).astype(np.int64))
    a_star = torch.from_numpy(rs.randint(0, A, B).astype(np.int64))
    returns = torch.from_numpy(rs.standard_normal(B).astype(F32))
    nt = torch.from_numpy((rs.uniform(size=B) < 0.8).astype(F32))
    g = 0.99 ** 3
    target = (returns[:, None].repeat(Np, 1) + (g * nt[:, None]).repeat(Np, 1)
              * q_tg.gather(1, a_star[:, None].repeat(Np, 1))).reshape(Np, B).t()
    theta = q_on.gather(1, actions[:, None].repeat(N, 1)).reshape(N, B).t()
    ref = losses.iqn_pairwise_loss(theta, target, tau.reshape(N, B).t(), kappa)
    w = torch.from_numpy(rs.uniform(0.1, 1, B).astype(F32))
    (w * ref).sum().backward()
    d = {k: t.detach().to(cuda_dev) for k, t in (("q_on", q_on), ("q_tg", q_tg), ("tau", tau), ("act", actions),
                                                 ("ast", a_star), ("ret", returns), ("nt", nt))}
    o = _loss_call(cuda_dev, d, B, N, Np, A, g, kappa)
    assert np.array_equal(o["target"].f32().reshape(B, Np), target.numpy())      # same fp32 op order as the reference
    assert np.array_equal(o["theta"].f32().reshape(B, N), theta.detach().numpy())
    assert rel_err(o["loss"].f32(), ref.detach().numpy()) < 1e-5
    gref = q_on.grad.gather(1, actions[:, None].repeat(N, 1)).reshape(N, B)
    got = torch.from_numpy(o["dth"].f32()).reshape(N, B) * w[None, :]
    assert rel_err(got.numpy(), gref.numpy()) < 1e-5


def test_huber_statement_matches_autograd():
    """CPU: the float64 statement above equals float64 autograd of oracle.losses.iqn_pairwise_loss, loss and d/dtheta,
    including d == 0, |d| == kappa and tau at 0 and 1 - 2^-24."""
    rs = np.random.RandomState(3)
    for kappa in KAPPAS:
        B, N, Np = 6, 9, 11
        th = rs.standard_normal((B, N)) * kappa
        T = rs.standard_normal((B, Np)) * kappa
        T[0, 0], T[0, 1], T[0, 2] = th[0, 0], th[0, 1] + kappa, th[0, 2] - kappa
        ta = rs.uniform(0, 1, (B, N))
        ta[1, 0], ta[1, 1] = 0.0, 1 - 2.0 ** -24
        tht = torch.from_numpy(th).requires_grad_(True)
        ref = losses.iqn_pairwise_loss(tht, torch.from_numpy(T), torch.from_numpy(ta), kappa)
        ref.sum().backward()
        loss, dth = huber_statement(T, th, ta, kappa)[:2]
        assert np.max(np.abs(loss - ref.detach().numpy()) / np.abs(ref.detach().numpy())) < 1e-12
        assert np.max(np.abs(dth - tht.grad.numpy())) <= 1e-12 * np.max(np.abs(tht.grad.numpy()))


@pytest.mark.gpu
def test_loss_refusals(cuda_dev):
    """riqn_iqn_loss_fwd_bwd, riqn_iqn_loss_fwd_bwd_h and riqn_miqn_loss_fwd_bwd refuse batch, n_tau or n_tau_prime
    below 1, A outside 1..32, kappa <= 0 or non-finite, and targets beyond the 48 KB of shared memory, writing nothing.
    At the shared-memory limit the calls run."""
    dev = cuda_dev
    B, N, Np, A = 2, 4, 4, 4
    NP_MAX = 48 * 1024 // 4 - 32                                   # 12256 staged targets
    NP_MAX_M = NP_MAX - 1024 // 4                                  # M-IQN: less its 1 KB of static shared memory
    rs = np.random.RandomState(5)
    big = 2 * B * 33 * (NP_MAX + 1)
    d = dict(q_on=to_dev(rs.standard_normal(B * 33 * 64).astype(F32), dev),
             q_tg=to_dev(rs.standard_normal(big).astype(F32), dev), tau=to_dev(rs.uniform(0, 1, B * 64).astype(F32), dev),
             act=torch.zeros(B, dtype=torch.int64, device=dev), ast=torch.zeros(B, dtype=torch.int64, device=dev),
             ret=to_dev(np.ones(B, F32), dev), nt=to_dev(np.ones(B, F32), dev))
    p = {k: dptr(v) for k, v in d.items()}

    def call(entry, b, n, np_, a, kappa):
        o = {"loss": Out(max(b, 1), dev), "dth": Out(max(n, 1) * max(b, 1), dev),
             "theta": Out(max(b, 1) * max(n, 1), dev), "target": Out(max(b, 1) * max(np_, 1), dev),
             "bonus": Out(max(b, 1), dev)}
        outs = [o["loss"].p, o["dth"].p, o["theta"].p, o["target"].p]
        try:
            if entry == "riqn_iqn_loss_fwd_bwd":
                lib_call(entry, b, n, np_, a, p["q_on"], p["q_tg"], p["tau"], p["act"], p["ast"], p["ret"], p["nt"],
                         0.9, float(kappa), *outs)
            elif entry == "riqn_iqn_loss_fwd_bwd_h":
                lib_call(entry, b, n, np_, a, p["q_on"], p["q_tg"], p["tau"], p["act"], p["ast"], p["ret"], p["nt"],
                         0.9, float(kappa), 1e-3, *outs)
            else:
                lib_call(entry, b, n, np_, a, p["q_on"], p["q_tg"], p["tau"], p["act"], p["ret"], p["nt"], 0.9,
                         float(kappa), 0.9, 0.03, -1.0, *outs, o["bonus"].p)
            refused = False
        except _riqn_error():
            refused = True
        torch.cuda.synchronize()
        assert_canaries(o)
        if entry != "riqn_miqn_loss_fwd_bwd":
            del o["bonus"]
        return refused, o

    for entry in ("riqn_iqn_loss_fwd_bwd", "riqn_iqn_loss_fwd_bwd_h", "riqn_miqn_loss_fwd_bwd"):
        bad = [(0, N, Np, A, 1.0), (B, 0, Np, A, 1.0), (B, N, 0, A, 1.0), (B, N, Np, 0, 1.0), (B, N, Np, 33, 1.0),
               (B, N, Np, A, 0.0), (B, N, Np, A, -1.0), (B, N, Np, A, float("inf")), (B, N, Np, A, float("nan")),
               (B, N, NP_MAX + 1, A, 1.0)]
        if entry == "riqn_miqn_loss_fwd_bwd":
            bad.append((B, N, NP_MAX_M + 1, A, 1.0))
        for args in bad:
            refused, o = call(entry, *args)
            assert refused, f"{entry} accepted {args}"
            for k, v in o.items():
                assert bool(torch.isnan(v.t[:v.n]).all()), f"{entry} refused {args} but wrote {k}"
        for args in ((B, N, Np, A, 1.0), (1, 1, NP_MAX_M if entry == "riqn_miqn_loss_fwd_bwd" else NP_MAX, 1, 1.0)):
            refused, o = call(entry, *args)
            assert not refused, f"{entry} refused {args}"
            assert bool(torch.isfinite(o["loss"].t[:o["loss"].n]).all()), (entry, args)
            assert bool(torch.isfinite(o["dth"].t[:o["dth"].n]).all()), (entry, args)


# ---------------------------------------------------------------------------------------------- one learner step, A = 9
@pytest.mark.gpu
def test_learner_step_nine_actions_vs_oracle(cuda_dev):
    """An IQN learner at an odd action count (A = 9: MsPacman, Enduro, Asterix) at B = 512, N = N' = 64, K = 32, where
    every network pass runs the streamed dueling kernel's unpaired last action, against the torch-fp32 oracle under
    injected noises and fractions: the loss within the default arithmetic's tolerance (near-tie argmaxes masked), every
    gradient at cosine >= 0.999 (0.98 upstream of a ReLU unit the two put on opposite sides of 0, or of a near tie)."""
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch, _loss_tol, _tie_mask
    A, B = 9, 512
    cfg = cases.iqn_cfg(64, 64, 32)
    seed = 909
    params = net.make_params(seed, action_space=A)
    lr = Learner(make_args(cuda_dev, B, cfg), A, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, B, action_space=A)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg))
    noises = cases.make_noises(seed + 3, action_space=A)
    lr._inject = dict(noises=noises, taus=taus)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]),
                                        noises, taus, cfg, keep=keep)
    ties = _tie_mask(keep, dbg["a_star"].cpu().numpy())
    ok = ~ties
    assert ties.sum() <= 2
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    err = np.abs(lg[ok] - lo[ok]) / np.abs(lo[ok])
    assert np.max(err) < _loss_tol(), float(np.max(err))
    gk = dbg["keep"]
    hq = gk["h"].cpu().reshape(B, -1, 2 * HID).transpose(0, 1).reshape(-1, 2 * HID)      # quantile-major rows
    fl = [int(((x.cpu() > 0) != (y > 0)).sum()) for x, y in
          ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
           (hq[:, :HID], keep["h_v"]), (hq[:, HID:], keep["h_a"]))]
    relaxed = set()
    if fl[3] + fl[4] or ties.any():
        relaxed |= {"conv1", "conv2", "conv3", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a", "iqn_fc"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    worst = 1.0
    for k, g_ref in o_grads.items():
        a, r = grads[k].double().ravel(), g_ref.double().ravel()
        c = float((a * r).sum() / (a.norm() * r.norm() + 1e-300))
        worst = min(worst, c)
        assert c > (0.98 if k.split(".")[0] in relaxed else 0.999), (k, c, fl)
    print(f"A=9 B=512: max loss rel err {np.max(err):.3g}, min cos {worst:.6f}, ReLU flips {fl}, ties {int(ties.sum())}")
