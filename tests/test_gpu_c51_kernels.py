"""The Rainbow-only (C51) head, loss and linear-layer kernels, entry point by entry point, against float64 statements of
the same operations (include/riqn_b200.h): riqn_c51_head_fwd, riqn_c51_loss_fwd_bwd, riqn_c51_head_bwd,
riqn_linear_fwd_ld, riqn_linear_dgrad_ld, riqn_noisy_wgrad_ld, riqn_noisy_linear_fwd / _dgrad / _wgrad and
riqn_relu_mask.

Method (as tests/test_gpu_head_kernels.py):
* every reference is computed on the operands the kernel read: the dueling logits q and the projection indices are
  restated in numpy float32, operation by operation as the kernels round them, and the rest is float64 on top;
* exact regime: small integers and dyadic values make every product and partial sum exact in fp32 in any order, so the
  kernel has to match float64 bit for bit -- a dropped split, row, slab, warp or atom shows up;
* random regime: each element is held to c * K * 2^-24 * sum|a_i b_i| (K = the reduction length) plus the output
  rounding, and each test prints its worst err/bound ratio;
* overwritten outputs start as NaN, accumulated outputs from a non-zero pattern, every output buffer carries canaries
  past its end, strided outputs carry sentinels in the columns they must not write, entry points without atomics are
  called twice and must agree bit for bit, and rejected calls must write nothing.
"""
import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, prefill_pattern,
                     to_dev)
from oracle.losses import c51_projection

C_BOUND = 2.0           # the constant c of the random-regime bounds
HID = 512
FEAT = 3136
SENTINEL = 12345.0      # exact in fp32; marks memory an entry point must neither write nor read
F32 = np.float32


def _support(v_min, v_max, atoms):
    """the support the learner hands the kernels (Agent.support: torch.linspace in fp32)"""
    return torch.linspace(v_min, v_max, atoms).numpy()


# ---------------------------------------------------------------------------------------------- head forward
def _head_q(zv, za, A):
    """q = (zv + za) - mean_a za as the kernel rounds it: the mean is a fp32 sum over a ascending, divided by A"""
    B, atoms = zv.shape
    za3 = za.reshape(B, A, atoms)
    s = np.zeros((B, atoms), F32)
    for a in range(A):
        s = (s + za3[:, a]).astype(F32)
    amean = (s / F32(A)).astype(F32)
    return ((zv[:, None, :] + za3).astype(F32) - amean[:, None, :]).astype(F32)


def _head_ref(q, support):
    """float64 softmax / log-softmax of the fp32 logits, their bounds, the expected values and their error bounds"""
    q = q.astype(np.float64)
    d = q - q.max(2, keepdims=True)
    e = np.exp(d)
    s = e.sum(2, keepdims=True)
    p = e / s
    logp = d - np.log(s)
    spread = (p * np.abs(d)).sum(2, keepdims=True)
    # expf: 2 ulp; fl(q - max): U |d| of argument; the warp sum of <= 64 positive terms: 7 U; the division or the
    # subtraction: U; logf: 1 ulp of lse.  Tiny p may come out subnormal (or flushed), hence the absolute term.
    bnd_p = C_BOUND * p * (12 * U + U * np.abs(d) + U * spread) + 2.0 ** -126
    bnd_logp = C_BOUND * (U * np.abs(d) + U * np.abs(logp) + 2 * U * np.abs(np.log(s)) + 12 * U + U * spread)
    z = support.astype(np.float64)
    ev = (p * z).sum(2)
    bnd_ev = (np.abs(z) * bnd_p).sum(2) + C_BOUND * (q.shape[2] + 2) * U * (np.abs(z) * p).sum(2)
    return p, logp, bnd_p, bnd_logp, ev, bnd_ev


def _head_call(dev, B, A, atoms, zvd, zad, supd, want_p, want_logp, want_a):
    o = {"p": Out(B * A * atoms, dev) if want_p else None, "logp": Out(B * A * atoms, dev) if want_logp else None}
    a_star = torch.full((B + 64,), -5, dtype=torch.int64, device=dev) if want_a else None
    lib_call("riqn_c51_head_fwd", B, A, atoms, dptr(zvd), dptr(zad), dptr(supd), o["p"].p if want_p else None,
             o["logp"].p if want_logp else None, dptr(a_star))
    torch.cuda.synchronize()
    assert_canaries(o)
    if a_star is not None:
        assert torch.all(a_star[B:] == -5), "a_star written past the batch"
        a_star = a_star[:B].cpu().numpy()
    return o, a_star


def _check_a_star(what, a_star, ev, bnd_ev):
    """a_star exactly where the top two expected values are separated by more than both their error bounds;
    elsewhere within that margin of the maximum"""
    B, A = ev.shape
    assert np.all((a_star >= 0) & (a_star < A)), f"{what}: a_star out of range"
    best = ev.argmax(1)
    margin = 2 * bnd_ev.max(1)
    if A > 1:
        top2 = np.sort(ev, 1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > margin
    else:
        clear = np.ones(B, bool)
    bad = clear & (a_star != best)
    assert not bad.any(), f"{what}: a_star {a_star[bad][:4]} want {best[bad][:4]} at rows {np.flatnonzero(bad)[:4]}"
    got_ev = ev[np.arange(B), a_star]
    assert np.all(got_ev >= ev.max(1) - margin), f"{what}: a_star picks an action below the maximum"
    return int(clear.sum())


HEAD_B, HEAD_A, HEAD_ATOMS = (1, 5, 512), (1, 2, 8, 9, 18), (2, 31, 32, 33, 51, 64)


@pytest.mark.gpu
@pytest.mark.parametrize("atoms", HEAD_ATOMS)
@pytest.mark.parametrize("A", HEAD_A)
def test_c51_head_fwd(cuda_dev, A, atoms):
    """Every batch size, then the four output combinations the library uses (log p for the loss, p for the target,
    p + a_star for action selection, a_star alone for acting); the combinations agree bit for bit."""
    dev = cuda_dev
    for B in HEAD_B:
        rs = np.random.RandomState(B * 1000 + A * 70 + atoms)
        scale = 3.0 if B != 5 else 60.0                 # B = 5: logits of magnitude ~100
        zv = (rs.standard_normal((B, atoms)) * scale).astype(F32)
        za = (rs.standard_normal((B, A * atoms)) * scale).astype(F32)
        support = _support(-10.0, 10.0, atoms)
        zvd, zad, supd = to_dev(zv, dev), to_dev(za, dev), to_dev(support, dev)
        q = _head_q(zv, za, A)
        p, logp, bnd_p, bnd_logp, ev, bnd_ev = _head_ref(q, support)
        tag = f"B{B}-A{A}-atoms{atoms}"
        o, _ = _head_call(dev, B, A, atoms, zvd, zad, supd, True, False, False)
        check_bound(f"p {tag}", o["p"].f32().reshape(B, A, atoms), p, bnd_p)
        o2, _ = _head_call(dev, B, A, atoms, zvd, zad, supd, False, True, False)
        check_bound(f"logp {tag}", o2["logp"].f32().reshape(B, A, atoms), logp, bnd_logp)
        o3, a3 = _head_call(dev, B, A, atoms, zvd, zad, supd, True, False, True)
        assert_bits(f"p with a_star {tag}", o3["p"].bits(), o["p"].bits())
        n_clear = _check_a_star(f"a_star {tag}", a3, ev, bnd_ev)
        _, a4 = _head_call(dev, B, A, atoms, zvd, zad, supd, False, False, True)
        assert np.array_equal(a4, a3), f"a_star alone differs from a_star with p {tag}"
        o5, a5 = _head_call(dev, B, A, atoms, zvd, zad, supd, True, True, True)
        assert_bits(f"p second call {tag}", o5["p"].bits(), o["p"].bits())
        assert_bits(f"logp second call {tag}", o5["logp"].bits(), o2["logp"].bits())
        assert np.array_equal(a5, a3)
        print(f"{tag}: a_star checked exactly on {n_clear} of {B} rows")


@pytest.mark.gpu
@pytest.mark.parametrize("atoms", [2, 33, 51, 64])
@pytest.mark.parametrize("first,second", [(0, 1), (0, 17), (3, 9), (16, 17)])
def test_c51_head_fwd_first_maximum_wins(cuda_dev, first, second, atoms):
    """Small-integer logits; actions `first` < `second` identical and clearly the best (+30 on the last atom, -30 on the
    others): their expected values are the same fp32 computation, so the tie is exact, and the first index must win."""
    dev = cuda_dev
    B, A = 9, 18
    rs = np.random.RandomState(first * 100 + second + atoms)
    zv = rs.randint(-3, 4, (B, atoms)).astype(F32)
    za = rs.randint(-3, 4, (B, A, atoms)).astype(F32)
    za[:, first] = -30
    za[:, first, -1] = 30                          # all the mass on v_max: the largest expected value
    za[:, second] = za[:, first]
    za = za.reshape(B, A * atoms)
    support = _support(-10.0, 10.0, atoms)
    zvd, zad, supd = to_dev(zv, dev), to_dev(za, dev), to_dev(support, dev)
    o, a_star = _head_call(dev, B, A, atoms, zvd, zad, supd, True, False, True)
    p = o["p"].f32().reshape(B, A, atoms)
    assert_bits("identical actions give identical p", f32_bits(p[:, first]), f32_bits(p[:, second]))
    assert np.all(a_star == first), f"a_star {a_star}, want {first}"
    _, a_only = _head_call(dev, B, A, atoms, zvd, zad, supd, False, False, True)
    assert np.all(a_only == first), f"a_star alone {a_only}, want {first}"


@pytest.mark.gpu
def test_c51_head_fwd_rejects_more_than_64_atoms(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    B, A, atoms = 3, 4, 65
    rs = np.random.RandomState(65)
    zvd = to_dev(rs.standard_normal((B, atoms)).astype(F32), dev)
    zad = to_dev(rs.standard_normal((B, A * atoms)).astype(F32), dev)
    supd = to_dev(_support(-10.0, 10.0, atoms), dev)
    o = {"p": Out(B * A * atoms, dev), "logp": Out(B * A * atoms, dev)}
    a_star = torch.full((B,), -5, dtype=torch.int64, device=dev)
    with pytest.raises(RiqnError):
        lib_call("riqn_c51_head_fwd", B, A, atoms, dptr(zvd), dptr(zad), dptr(supd), o["p"].p, o["logp"].p, dptr(a_star))
    torch.cuda.synchronize()
    assert_canaries(o)
    for k, v in o.items():
        assert torch.isnan(v.t[:v.n]).all(), f"rejected call wrote {k}"
    assert torch.all(a_star == -5), "rejected call wrote a_star"


# ---------------------------------------------------------------------------------------------- projection + loss
def project_indices(returns, nonterminals, gamma_n, v_min, v_max, atoms, support, clamp=True):
    """numpy float32 statement of the kernel's projection indices: fl(nt * gamma_n), fl(r + fl(g * z_j)), the clamp to
    [v_min, v_max], b_j = fl(fl(tz - v_min) / delta_z) (clamped to atoms - 1), l / u with the l == u fix.
    Returns (b, l, u, the b before its clamp)."""
    delta_z = F32((v_max - v_min) / (atoms - 1))
    g = (np.asarray(nonterminals, F32) * F32(gamma_n)).astype(F32)
    tz = (np.asarray(returns, F32)[:, None] + (g[:, None] * support[None, :]).astype(F32)).astype(F32)
    tz = np.minimum(np.maximum(tz, F32(v_min)), F32(v_max))
    b_raw = ((tz - F32(v_min)).astype(F32) / delta_z).astype(F32)
    b = np.minimum(b_raw, F32(atoms - 1)) if clamp else b_raw
    lo, up = np.floor(b).astype(np.int64), np.ceil(b).astype(np.int64)
    lo[(up > 0) & (lo == up)] -= 1               # agent.py:119
    up[(lo < atoms - 1) & (lo == up)] += 1       # agent.py:120
    return b, lo, up, b_raw


def _loss_ref(logp, p_target, actions, a_star, returns, nonterm, gamma_n, v_min, v_max, atoms, support):
    B = logp.shape[0]
    rows = np.arange(B)
    pa = p_target[rows, a_star]                                       # (B, atoms) fp32
    b, lo, up, _ = project_indices(returns, nonterm, gamma_n, v_min, v_max, atoms, support)
    wl = (pa * (up.astype(F32) - b).astype(F32)).astype(F32)
    wu = (pa * (b - lo.astype(F32)).astype(F32)).astype(F32)
    # m as the kernel adds it (fp32, all l-adds in j order, then all u-adds) and in float64
    m32 = np.zeros((B, atoms), F32)
    for j in range(atoms):
        m32[rows, lo[:, j]] = (m32[rows, lo[:, j]] + wl[:, j]).astype(F32)
    for j in range(atoms):
        m32[rows, up[:, j]] = (m32[rows, up[:, j]] + wu[:, j]).astype(F32)
    m64 = np.zeros((B, atoms))
    np.add.at(m64, (rows[:, None], lo), wl.astype(np.float64))
    np.add.at(m64, (rows[:, None], up), wu.astype(np.float64))
    bnd_m = C_BOUND * 2 * atoms * U * m64
    return pa, m32, m64, bnd_m


def _loss_call(dev, B, A, atoms, d, gamma_n, v_min, v_max, with_m=True):
    o = {"loss": Out(B, dev), "dq": Out(B * atoms, dev), "m": Out(B * atoms, dev) if with_m else None}
    delta_z = (v_max - v_min) / (atoms - 1)
    lib_call("riqn_c51_loss_fwd_bwd", B, A, atoms, dptr(d["logp"]), dptr(d["pt"]), dptr(d["act"]), dptr(d["astar"]),
             dptr(d["ret"]), dptr(d["nt"]), dptr(d["sup"]), float(gamma_n), float(v_min), float(v_max), float(delta_z),
             o["loss"].p, o["dq"].p, o["m"].p if with_m else None)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _loss_inputs(B, A, atoms, v_min, v_max, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        # delta_z = 1 and integer support: returns on a 1/4 grid, gamma_n in {3/4, 1} and p_target in k/256 keep tz, b,
        # the weights and every partial sum of m on dyadic grids far inside 24 bits; log p on a 1/8 grid
        returns = rs.randint(-80, 81, B).astype(F32) / 4
        p_target = (rs.randint(0, 17, (B, A, atoms)) / 256).astype(F32)
        logp = (-rs.randint(0, 64, (B, A, atoms)) / 8).astype(F32)
    else:
        returns = rs.uniform(-1.5, 1.5, B).astype(F32) * (v_max - v_min) / 2
        p_target = rs.dirichlet(np.ones(atoms), (B, A)).astype(F32)
        logp = np.log(rs.dirichlet(np.ones(atoms), (B, A))).astype(F32)
    nonterm = (rs.uniform(size=B) > 0.1).astype(F32)
    actions = rs.randint(0, A, B).astype(np.int64)
    a_star = rs.randint(0, A, B).astype(np.int64)
    # edge rows: a terminal transition, returns beyond both ends (both branches of the l == u fix), tz on the atoms,
    # actions and a_star at 0 and A - 1
    mid = (v_min + v_max) / 2
    edges = [(mid + 0.25, 0.0), (v_max + 7, 1.0), (v_min - 7, 1.0), (v_max + 7, 0.0), (v_min - 7, 0.0), (v_max, 0.0),
             (v_min, 0.0), (float(np.floor(mid)), 1.0)]
    for i, (r, n) in enumerate(edges[:B]):
        returns[i], nonterm[i] = r, n
    actions[0], a_star[0], actions[-1], a_star[-1] = 0, A - 1, A - 1, 0
    if B > 2:
        actions[1], a_star[1] = A - 1, A - 1
    return dict(logp=logp, pt=p_target, act=actions, astar=a_star, ret=returns, nt=nonterm)


def _loss_dev(h, dev, support):
    d = {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}
    d["sup"] = to_dev(support, dev)
    return d


# (v_min, v_max, atoms, gamma_n, regime): the exact grid, the shipped support, atoms 2 / 64, and (-1, 1, 62), where fp32
# rounding takes b above atoms - 1 at tz = v_max
LOSS_CASES = [(-16.0, 16.0, 33, 0.75, "exact"), (-16.0, 16.0, 33, 1.0, "exact"), (-10.0, 10.0, 51, 0.99 ** 3, "random"),
              (-10.0, 10.0, 51, 1.0, "random"), (-1.0, 1.0, 62, 0.99 ** 3, "random"), (-1.0, 1.0, 62, 1.0, "random"),
              (-5.0, 5.0, 64, 0.99 ** 3, "random"), (-10.0, 10.0, 2, 0.99 ** 3, "random"),
              (-10.0, 10.0, 31, 0.9, "random")]


@pytest.mark.gpu
@pytest.mark.parametrize("B,A", [(1, 1), (9, 18), (37, 4), (512, 18)])
@pytest.mark.parametrize("v_min,v_max,atoms,gamma_n,regime", LOSS_CASES,
                         ids=[f"{a}atoms-{lo:g}..{hi:g}-g{g:.3g}-{r}" for lo, hi, a, g, r in LOSS_CASES])
def test_c51_loss(cuda_dev, B, A, v_min, v_max, atoms, gamma_n, regime):
    dev = cuda_dev
    support = _support(v_min, v_max, atoms)
    h = _loss_inputs(B, A, atoms, v_min, v_max, regime, seed=B * 100 + A + atoms)
    d = _loss_dev(h, dev, support)
    o = _loss_call(dev, B, A, atoms, d, gamma_n, v_min, v_max)
    pa, m32, m64, bnd_m = _loss_ref(h["logp"], h["pt"], h["act"], h["astar"], h["ret"], h["nt"], gamma_n, v_min, v_max,
                                    atoms, support)
    m = o["m"].f32().reshape(B, atoms)
    # m: bit for bit the fp32 statement of the kernel's add order, and within float64 bounds of the exact sum
    assert_bits("m (fp32 statement)", f32_bits(m), f32_bits(m32))
    if regime == "exact":
        assert_bits("m (float64)", f32_bits(m), f32_bits(m64))
    else:
        check_bound("m", m, m64, bnd_m)
    # mass conservation: sum_j m_j = sum_j p_target[b, a*, j]
    msum = m.astype(np.float64).sum(1)
    psum = pa.astype(np.float64).sum(1)
    if regime == "exact":
        assert np.array_equal(msum, psum), "mass not conserved"
    else:
        check_bound("sum m", msum, psum, C_BOUND * 3 * atoms * U * psum)
    # loss = -sum_j m_j logp[b, act, j] and dq = -(m - exp(logp) sum m), on the kernel's own m
    lp = h["logp"][np.arange(B), h["act"]].astype(np.float64)
    m_d = m.astype(np.float64)
    ref_loss = -(m_d * lp).sum(1)
    mt = m_d.sum(1, keepdims=True)
    e = np.exp(lp)
    ref_dq = -(m_d - e * mt)
    bnd_dq = C_BOUND * (6 * U * e * mt + e * (atoms + 2) * U * mt + U * np.abs(ref_dq))
    if regime == "exact":
        assert_bits("loss", o["loss"].bits(), f32_bits(ref_loss))
    else:
        check_bound("loss", o["loss"].f32(), ref_loss, C_BOUND * (atoms + 2) * U * np.abs(m_d * lp).sum(1))
    check_bound("dq", o["dq"].f32().reshape(B, atoms), ref_dq, bnd_dq)
    # m_out = NULL computes the same loss and dq; no atomics: a second call is bitwise the first
    o2 = _loss_call(dev, B, A, atoms, d, gamma_n, v_min, v_max, with_m=False)
    assert_bits("loss without m_out", o2["loss"].bits(), o["loss"].bits())
    assert_bits("dq without m_out", o2["dq"].bits(), o["dq"].bits())
    o3 = _loss_call(dev, B, A, atoms, d, gamma_n, v_min, v_max)
    for k in o:
        assert_bits(f"second call {k}", o3[k].bits(), o[k].bits())


@pytest.mark.gpu
def test_c51_loss_index_clamp_at_vmax(cuda_dev):
    """(-1, 1, 62): tz = v_max gives b = 61.0000038 in fp32.  With the index clamped, b = 61 puts every weight on the
    last atom (l = 60 gets exactly 0), so m[b, 61] is the fp32 sum of p_target[b, a*, :] in j order.  Without the
    clamp u = 62 = atoms and a 3.8e-6 share of the mass is written past m."""
    dev = cuda_dev
    B, A, atoms, v_min, v_max = 4, 3, 62, -1.0, 1.0
    support = _support(v_min, v_max, atoms)
    rs = np.random.RandomState(62)
    h = dict(logp=np.log(rs.dirichlet(np.ones(atoms), (B, A))).astype(F32),
             pt=rs.dirichlet(np.ones(atoms), (B, A)).astype(F32), act=np.array([0, 1, 2, 0], np.int64),
             astar=np.array([1, 2, 0, 1], np.int64), ret=np.array([5.0, 0.3, 5.0, -5.0], F32),
             nt=np.array([0.0, 1.0, 1.0, 0.0], F32))
    o = _loss_call(dev, B, A, atoms, _loss_dev(h, dev, support), 0.99 ** 3, v_min, v_max)
    m = o["m"].f32().reshape(B, atoms)
    pa = h["pt"][np.arange(B), h["astar"]].astype(np.float64)
    for b in (0, 2):                                   # every tz = v_max
        assert np.all(m[b, :-1] == 0), f"sample {b}: mass below the last atom"
        s = F32(0)
        for v in h["pt"][b, h["astar"][b]]:
            s = F32(s + v)
        assert_bits(f"m[{b}, -1]", f32_bits(m[b, -1:]), f32_bits(np.array([s])))
    assert np.all(m[3, 1:] == 0)                       # tz = v_min
    check_bound("sum m", m.astype(np.float64).sum(1), pa.sum(1), C_BOUND * 3 * atoms * U * pa.sum(1))


# ---------------------------------------------------------------------------------------------- CPU: the clamp
def test_projection_index_exceeds_last_atom_in_fp32():
    """The fp32 statement of the kernel's index reaches b > atoms - 1 at (-1, 1, 62) for tz = v_max, and not for the
    shipped (-10, 10, 51)."""
    for v_min, v_max, atoms, over in [(-1.0, 1.0, 62, True), (-10.0, 10.0, 51, False)]:
        support = _support(v_min, v_max, atoms)
        b, lo, up, b_raw = project_indices(np.array([v_max + 3], F32), np.array([0.0], F32), 0.99 ** 3, v_min, v_max,
                                           atoms, support)
        assert (b_raw.max() > atoms - 1) == over, (v_min, v_max, atoms, float(b_raw.max()))
        assert b.max() <= atoms - 1 and up.max() <= atoms - 1 and lo.min() >= 0


def test_oracle_projection_conserves_mass_at_the_rounding_edge():
    """oracle.losses.c51_projection at (-1, 1, 62): samples whose every tz is v_max keep all their mass on the last atom
    (the reference's index_add_ moves it to the next sample's atom 0, or past the end for the last sample)."""
    B, atoms, v_min, v_max = 6, 62, -1.0, 1.0
    rs = np.random.RandomState(3)
    pns_a = torch.from_numpy(rs.dirichlet(np.ones(atoms), B).astype(F32))
    returns = torch.tensor([5.0, 0.1, 5.0, -0.4, -5.0, 5.0])
    nonterm = torch.tensor([0.0, 1.0, 1.0, 1.0, 0.0, 0.0])
    m = c51_projection(pns_a, returns, nonterm, atoms=atoms, v_min=v_min, v_max=v_max, gamma_n=0.99 ** 3).double()
    p = pns_a.double()
    assert torch.allclose(m.sum(1), p.sum(1), rtol=1e-6, atol=0)
    for b in (0, 2, 5):
        assert torch.allclose(m[b, -1], p[b].sum(), rtol=1e-6) and float(m[b, :-1].abs().max()) == 0.0
    assert torch.allclose(m[4, 0], p[4].sum(), rtol=1e-6)
    # the emulation of the kernel's indices agrees with the oracle's projection on these rows
    support = _support(v_min, v_max, atoms)
    b_, lo, up, _ = project_indices(returns.numpy(), nonterm.numpy(), 0.99 ** 3, v_min, v_max, atoms, support)
    m_np = np.zeros((B, atoms))
    pn = pns_a.numpy()
    np.add.at(m_np, (np.arange(B)[:, None], lo), (pn * (up.astype(F32) - b_).astype(F32)).astype(F32))
    np.add.at(m_np, (np.arange(B)[:, None], up), (pn * (b_ - lo.astype(F32)).astype(F32)).astype(F32))
    assert np.allclose(m_np, m.numpy(), rtol=1e-6, atol=1e-9)


# ---------------------------------------------------------------------------------------------- head backward
HB_CASES = [(1, 1, 2), (5, 18, 51), (7, 9, 33), (3, 2, 64), (509, 18, 51)]      # B * A * atoms % 256 != 0


@pytest.mark.gpu
@pytest.mark.parametrize("B,A,atoms", HB_CASES, ids=[f"B{b}-A{a}-atoms{n}" for b, a, n in HB_CASES])
def test_c51_head_bwd(cuda_dev, B, A, atoms):
    """dzv = g, dza[a] = g * (1{a == act} - 1/A), g = dq * fl(gscale * gmul): each a chain of correctly rounded fp32
    operations without a multiply feeding an add, so bit for bit"""
    dev = cuda_dev
    assert (B * A * atoms) % 256
    rs = np.random.RandomState(B + A + atoms)
    dq = rs.standard_normal((B, atoms)).astype(F32)
    gscale = rs.uniform(0.1, 2, B).astype(F32)
    gmul = F32(1.0 / 3.0)
    actions = rs.randint(0, A, B).astype(np.int64)
    actions[0], actions[-1] = 0, A - 1
    o = {"dzv": Out(B * atoms, dev), "dza": Out(B * A * atoms, dev)}
    dqd, gsd, actd = to_dev(dq, dev), to_dev(gscale, dev), torch.from_numpy(actions).to(dev)
    lib_call("riqn_c51_head_bwd", B, A, atoms, dptr(dqd), dptr(gsd), float(gmul), dptr(actd), o["dzv"].p, o["dza"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    g = (dq * (gscale * gmul).astype(F32)[:, None]).astype(F32)
    inv = F32(1) / F32(A)
    onehot = (np.arange(A)[None, :] == actions[:, None]).astype(F32)
    dza = (g[:, None, :] * (onehot - inv).astype(F32)[:, :, None]).astype(F32)
    assert_bits("dzv", o["dzv"].bits(), f32_bits(g).ravel())
    assert_bits("dza", o["dza"].bits(), f32_bits(dza).ravel())


# ---------------------------------------------------------------------------------------------- z-layer products
LD_ROWS = (1, 5, 64, 65, 128, 129, 512, 1000, 4096)
LD_OUT = (51, 918)                  # z_v reads h[:, :hid], z_a reads h[:, hid:] (c51.py)


def _ld_inputs(rows, out, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        h = rs.randint(0, 7, (rows, 2 * HID)).astype(F32)
        h[rs.uniform(size=h.shape) < 0.3] = 0
        w = rs.randint(-3, 4, (out, HID)).astype(F32)
        bias = rs.randint(-40, 41, out).astype(F32)
        dy = rs.randint(-3, 4, (rows, out)).astype(F32)
        eps = rs.choice(np.array([-2, -1, -0.5, 0.5, 1, 2], F32), (out, HID))
        pre_mu, pre_sig = prefill_pattern(out * HID, 0.5, 11), prefill_pattern(out * HID, 0.5, 7)
    else:
        h = np.maximum(rs.standard_normal((rows, 2 * HID)), 0).astype(F32)
        w = (rs.standard_normal((out, HID)) * 0.05).astype(F32)
        bias = (rs.standard_normal(out) * 0.1).astype(F32)
        dy = (rs.standard_normal((rows, out)) * 0.1).astype(F32)
        eps = rs.standard_normal((out, HID)).astype(F32)
        pre_mu, pre_sig = rs.standard_normal(out * HID).astype(F32), rs.standard_normal(out * HID).astype(F32)
    off = 0 if out == 51 else HID
    h_in = h.copy()
    h_in[:, HID - off:2 * HID - off] = SENTINEL          # the other half: must not be read
    return dict(h=h_in, x=h[:, off:off + HID], off=off, w=w, bias=bias, dy=dy, eps=eps, pre_mu=pre_mu, pre_sig=pre_sig)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("out", LD_OUT)
@pytest.mark.parametrize("rows", LD_ROWS)
def test_linear_fwd_ld(cuda_dev, rows, out, regime):
    """y (rows, out) [ldy] = x [ldx = 2 hid, at the layer's half of h] w^T + bias, with and without ReLU; the ldy gaps
    keep their sentinels"""
    dev = cuda_dev
    d = _ld_inputs(rows, out, regime, seed=rows * 7 + out)
    hd, wd, bd = to_dev(d["h"], dev), to_dev(d["w"], dev), to_dev(d["bias"], dev)
    ldy = out + 3
    x64, w64 = d["x"].astype(np.float64), d["w"].astype(np.float64)
    pre = x64 @ w64.T + d["bias"]
    mag = np.abs(x64) @ np.abs(w64).T + np.abs(d["bias"])
    first = None
    for relu in (0, 1):
        y = Out(rows * ldy, dev, fill=np.full(rows * ldy, SENTINEL, F32))
        y.t[:rows * ldy].view(rows, ldy)[:, :out] = float("nan")
        lib_call("riqn_linear_fwd_ld", rows, HID, out, hd.data_ptr() + 4 * d["off"], 2 * HID, dptr(wd), dptr(bd), y.p,
                 ldy, relu)
        torch.cuda.synchronize()
        assert_canaries({"y": y})
        got = y.f32().reshape(rows, ldy)
        assert np.all(got[:, out:] == SENTINEL), "the ldy gap was written"
        ref = np.maximum(pre, 0) if relu else pre
        if regime == "exact":
            assert_bits(f"y relu={relu}", f32_bits(got[:, :out]), f32_bits(ref))
        else:
            check_bound(f"y relu={relu}", got[:, :out], ref, C_BOUND * (HID + 1) * U * mag + U * np.abs(ref))
        if relu == 0:
            first = y
    y2 = Out(rows * ldy, dev, fill=np.full(rows * ldy, SENTINEL, F32))
    lib_call("riqn_linear_fwd_ld", rows, HID, out, hd.data_ptr() + 4 * d["off"], 2 * HID, dptr(wd), dptr(bd), y2.p, ldy, 0)
    torch.cuda.synchronize()
    assert_bits("second call", y2.bits(), first.bits())


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("out", LD_OUT)
@pytest.mark.parametrize("rows", LD_ROWS)
def test_linear_dgrad_ld(cuda_dev, rows, out, regime):
    """dx = dy w written into the layer's half of dh (lddx = 2 hid); the other half keeps its sentinels"""
    dev = cuda_dev
    d = _ld_inputs(rows, out, regime, seed=rows * 11 + out)
    dyd, wd = to_dev(d["dy"], dev), to_dev(d["w"], dev)
    ref = d["dy"].astype(np.float64) @ d["w"].astype(np.float64)
    mag = np.abs(d["dy"]).astype(np.float64) @ np.abs(d["w"]).astype(np.float64)
    off = d["off"]
    dh = Out(rows * 2 * HID, dev, fill=np.full(rows * 2 * HID, SENTINEL, F32))
    dh.t[:rows * 2 * HID].view(rows, 2 * HID)[:, off:off + HID] = float("nan")
    lib_call("riqn_linear_dgrad_ld", rows, HID, out, dptr(dyd), out, dptr(wd), dh.p + 4 * off, 2 * HID)
    torch.cuda.synchronize()
    assert_canaries({"dh": dh})
    got = dh.f32().reshape(rows, 2 * HID)
    assert np.all(got[:, HID - off:2 * HID - off] == SENTINEL), "the other half of dh was written"
    if regime == "exact":
        assert_bits("dx", f32_bits(got[:, off:off + HID]), f32_bits(ref))
    else:
        check_bound("dx", got[:, off:off + HID], ref, C_BOUND * (out + 1) * U * mag)
    dh2 = Out(rows * 2 * HID, dev, fill=np.full(rows * 2 * HID, SENTINEL, F32))
    lib_call("riqn_linear_dgrad_ld", rows, HID, out, dptr(dyd), out, dptr(wd), dh2.p + 4 * off, 2 * HID)
    torch.cuda.synchronize()
    assert_bits("second call", dh2.bits().reshape(rows, 2 * HID)[:, off:off + HID],
                dh.bits().reshape(rows, 2 * HID)[:, off:off + HID])


def _wgrad_ld_call(dev, rows, out, d, dyd, hd, epsd):
    o = {"g_mu": Out(out * HID, dev, fill=d["pre_mu"]), "g_sig": Out(out * HID, dev, fill=d["pre_sig"])}
    lib_call("riqn_noisy_wgrad_ld", rows, HID, out, dptr(dyd), out, hd.data_ptr() + 4 * d["off"], 2 * HID, dptr(epsd),
             o["g_mu"].p, o["g_sig"].p)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("out", LD_OUT)
@pytest.mark.parametrize("rows", LD_ROWS)
def test_noisy_wgrad_ld(cuda_dev, rows, out, regime):
    """grad_mu += dy^T x, grad_sigma += (dy^T x) * eps from a non-zero prefill, x the layer's half of h.  rows 65 / 129 /
    1000 / 4096 take 2, 3, 5 and up to 32 row splits (the last one shorter); two calls must agree bit for bit."""
    dev = cuda_dev
    d = _ld_inputs(rows, out, regime, seed=rows * 13 + out)
    dyd, hd, epsd = to_dev(d["dy"], dev), to_dev(d["h"], dev), to_dev(d["eps"], dev)
    o = _wgrad_ld_call(dev, rows, out, d, dyd, hd, epsd)
    dy64, x64 = d["dy"].astype(np.float64), d["x"].astype(np.float64)
    s = (dy64.T @ x64).ravel()
    mag = (np.abs(dy64).T @ np.abs(x64)).ravel()
    e64 = d["eps"].astype(np.float64).ravel()
    pm, ps = d["pre_mu"].astype(np.float64), d["pre_sig"].astype(np.float64)
    ref_mu, ref_sig = pm + s, ps + s * e64
    k = rows + 2
    if regime == "exact":
        assert_bits("grad_mu", o["g_mu"].bits(), f32_bits(ref_mu))
        assert_bits("grad_sigma", o["g_sig"].bits(), f32_bits(ref_sig))
    else:
        check_bound("grad_mu", o["g_mu"].f32(), ref_mu, C_BOUND * k * U * (mag + np.abs(pm)))
        check_bound("grad_sigma", o["g_sig"].f32(), ref_sig, C_BOUND * (k + 1) * U * (mag * np.abs(e64) + np.abs(ps)))
    o2 = _wgrad_ld_call(dev, rows, out, d, dyd, hd, epsd)
    for key in o:
        assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())


# ---------------------------------------------------------------------------------------------- hidden NoisyLinear (fp32)
NL_OUT = 2 * HID


def _nl_inputs(rows, regime, seed):
    rs = np.random.RandomState(seed)
    if regime == "exact":
        x = rs.randint(0, 5, (rows, FEAT)).astype(F32)
        x[rs.uniform(size=x.shape) < 0.4] = 0
        w = rs.randint(-2, 3, (NL_OUT, FEAT)).astype(F32)
        b = rs.randint(-20, 21, NL_OUT).astype(F32)
        dh = rs.randint(-3, 4, (rows, NL_OUT)).astype(F32)
        dh[rs.uniform(size=dh.shape) < 0.3] = 0
        ch = np.array([-2, -1, -0.5, 0.5, 1, 2], F32)
        eps_w, eps_b = rs.choice(ch, (NL_OUT, FEAT)), rs.choice(ch, NL_OUT)
        pre = [prefill_pattern(NL_OUT * FEAT, 0.5, 11), prefill_pattern(NL_OUT * FEAT, 0.5, 7),
               prefill_pattern(NL_OUT, 0.5, 5), prefill_pattern(NL_OUT, 0.5, 3)]
    else:
        x = np.maximum(rs.standard_normal((rows, FEAT)), 0).astype(F32)
        w = (rs.standard_normal((NL_OUT, FEAT)) * 0.02).astype(F32)
        b = (rs.standard_normal(NL_OUT) * 0.1).astype(F32)
        dh = (rs.standard_normal((rows, NL_OUT)) * 0.1).astype(F32)
        dh[rs.uniform(size=dh.shape) < 0.3] = 0
        eps_w, eps_b = rs.standard_normal((NL_OUT, FEAT)).astype(F32), rs.standard_normal(NL_OUT).astype(F32)
        pre = [rs.standard_normal(n).astype(F32) for n in (NL_OUT * FEAT, NL_OUT * FEAT, NL_OUT, NL_OUT)]
    return dict(x=x, w=w, b=b, dh=dh, eps_w=eps_w, eps_b=eps_b, pre=pre)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("rows", [1, 3, 5, 7])
def test_noisy_linear_fp32(cuda_dev, rows, regime):
    """The hidden layers of the C51 head when B % 8 != 0 (the actor acts at B = 1) and in fp32 mode:
    h = relu(x w^T + b), dx = dh w, and the four weight / bias gradients accumulated from a prefill"""
    dev = cuda_dev
    d = _nl_inputs(rows, regime, seed=rows + (50 if regime == "exact" else 0))
    xd, wd, bd, dhd = to_dev(d["x"], dev), to_dev(d["w"], dev), to_dev(d["b"], dev), to_dev(d["dh"], dev)
    ewd, ebd = to_dev(d["eps_w"], dev), to_dev(d["eps_b"], dev)
    x64, w64, dh64 = d["x"].astype(np.float64), d["w"].astype(np.float64), d["dh"].astype(np.float64)

    def run():
        o = {"h": Out(rows * NL_OUT, dev), "dx": Out(rows * FEAT, dev), "db": Out(NL_OUT, dev)}
        o.update({n: Out(p.size, dev, fill=p) for n, p in zip(("g_wmu", "g_wsig", "g_bmu", "g_bsig"), d["pre"])})
        lib_call("riqn_noisy_linear_fwd", rows, FEAT, NL_OUT, dptr(xd), dptr(wd), dptr(bd), o["h"].p)
        lib_call("riqn_noisy_linear_dgrad", rows, FEAT, NL_OUT, dptr(dhd), dptr(wd), o["dx"].p)
        lib_call("riqn_noisy_linear_wgrad", rows, FEAT, NL_OUT, dptr(dhd), dptr(xd), dptr(ewd), dptr(ebd), o["db"].p,
                 o["g_wmu"].p, o["g_wsig"].p, o["g_bmu"].p, o["g_bsig"].p)
        torch.cuda.synchronize()
        assert_canaries(o)
        return o

    o = run()
    pre = np.maximum(x64 @ w64.T + d["b"], 0)
    mag_h = np.abs(x64) @ np.abs(w64).T + np.abs(d["b"])
    dx = dh64 @ w64
    mag_dx = np.abs(dh64) @ np.abs(w64)
    s = (dh64.T @ x64).ravel()
    mag_s = (np.abs(dh64).T @ np.abs(x64)).ravel()
    db = dh64.sum(0) + 0.0
    mag_db = np.abs(dh64).sum(0)
    ew, eb = d["eps_w"].astype(np.float64).ravel(), d["eps_b"].astype(np.float64)
    p = [x.astype(np.float64) for x in d["pre"]]
    refs = {"h": (pre, C_BOUND * (FEAT + 1) * U * mag_h + U * pre),
            "dx": (dx, C_BOUND * (NL_OUT + 1) * U * mag_dx),
            "db": (db, C_BOUND * (rows + 1) * U * mag_db),
            "g_wmu": (p[0] + s, C_BOUND * (rows + 2) * U * (mag_s + np.abs(p[0]))),
            "g_wsig": (p[1] + s * ew, C_BOUND * (rows + 3) * U * (mag_s * np.abs(ew) + np.abs(p[1]))),
            "g_bmu": (p[2] + db, C_BOUND * (rows + 2) * U * (mag_db + np.abs(p[2]))),
            "g_bsig": (p[3] + db * eb, C_BOUND * (rows + 3) * U * (mag_db * np.abs(eb) + np.abs(p[3])))}
    for name, (ref, bnd) in refs.items():
        got = o[name].f32().reshape(np.shape(ref))
        if regime == "exact":
            assert_bits(name, f32_bits(got), f32_bits(ref))
        else:
            check_bound(name, got, ref, bnd)
    o2 = run()                          # split 1 and ordered column sums: deterministic
    for key in o:
        assert_bits(f"second call {key}", o2[key].bits(), o[key].bits())


# ---------------------------------------------------------------------------------------------- ReLU mask
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 257, 1000, 70001])
def test_relu_mask(cuda_dev, n):
    """grad[i] = 0 unless act[i] > 0: +0, -0, NaN, negative and positive subnormals, negatives and infinities"""
    dev = cuda_dev
    rs = np.random.RandomState(n)
    special = np.array([0.0, -0.0, np.nan, -np.nan, 1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149), -1.0, 1.0, np.inf,
                        -np.inf, 3e38, -3e38], F32)
    act = rs.standard_normal(n).astype(F32)
    act[:min(n, special.size)] = special[:min(n, special.size)]
    act[rs.uniform(size=n) < 0.1] = -0.0
    grad = rs.standard_normal(n).astype(F32)
    grad[-1] = np.nan if n > 1 else grad[-1]
    g = Out(n, dev, fill=grad)
    actd = to_dev(act, dev)
    lib_call("riqn_relu_mask", n, dptr(actd), g.p)
    torch.cuda.synchronize()
    assert_canaries({"grad": g})
    want = np.where(act > 0, grad, F32(0)).astype(F32)
    assert_bits("masked grad", g.bits(), f32_bits(want))
