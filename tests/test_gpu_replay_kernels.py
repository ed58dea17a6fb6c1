"""The prioritized replay's kernels (csrc/sumtree.cu) entry point by entry point: riqn_sumtree_stratified,
riqn_sumtree_sample, riqn_sumtree_is_weights, riqn_sumtree_update, riqn_replay_append and riqn_frame_gather, and the
resample loop of ReplayMemory.sample_indices.

Statements: the stratified sampler is float64 arithmetic on Philox words (stratified_np, with the Philox statement of
helpers.philox_np); the descent is "the first leaf, left to right, whose inclusive prefix sum is >= the value"
(prefix_leaf), pinned here against oracle.sumtree.retrieve on integer trees; the rest are oracle.sumtree and
oracle.replay.  Every output starts as NaN (-7 for int64, 0xAB for uint8), has canaries past its end, is written twice
with the same bits, and every refused call raises RiqnError leaving outputs, tree, store and max_priority untouched."""
import functools
from fractions import Fraction

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, make_args, philox_np
from oracle import replay as orep, sumtree as osum

F32 = np.float32
FRAME = 84 * 84
KEY_XOR = 0x5BD1E995
I64_FILL = -7


# ------------------------------------------------------------------------------------------------ statements (numpy)
def stratified_np(seed, stream, total, n, fused=True):
    """riqn_sumtree_stratified: (values, u, order) with values[j] = v[order[j]].  v_s = fl(a + fl(d u_s)), a = fl(s seg),
    seg = total / n, u_s = (((x << 32 | y) >> 11) + 0.5) 2^-53 of the words x, y of draw s; the keys are word x of the
    draws at stream ^ 0x5bd1e995, ranked by (key, s).  d = fl((s+1) seg - a) with the exact product, as the kernel's
    b - a is compiled (one DFMA); fused=False gives CPython's random.uniform, d = fl(fl((s+1) seg) - a)."""
    keys = philox_np(seed, stream ^ KEY_XOR, n).reshape(n, 4)[:, 0]
    order = np.lexsort((np.arange(n), keys))              # order[j]: the stratum at output slot j
    w = philox_np(seed, stream, n).reshape(n, 4).astype(np.uint64)
    m = ((w[:, 0] << np.uint64(32)) | w[:, 1]) >> np.uint64(11)
    u = (m.astype(np.float64) + 0.5) * 2.0 ** -53
    seg = np.float64(total) / np.float64(n)
    s = np.arange(n, dtype=np.float64)
    a, b = s * seg, (s + 1) * seg
    if fused:
        fs = Fraction(float(seg))
        d = np.array([float(Fraction(k + 1) * fs - Fraction(float(ak))) for k, ak in enumerate(a)])
    else:
        d = b - a
    v = a + d * u
    return v[order], u, order


def leaf_order(cap):
    """Data indices of the leaves of a 2 cap - 1 node heap in left-to-right order (deeper level projected)."""
    from test_gpu_replay import _heap_leaf_rank
    return np.argsort(_heap_leaf_rank(cap, "cpu").numpy())


def prefix_leaf(leaves, values):
    """Data index of the first leaf, left to right, whose inclusive prefix sum is >= value (values <= total)."""
    order = leaf_order(len(leaves))
    prefix = np.cumsum(leaves[order])
    return order[np.searchsorted(prefix, values, side="left")]


def right_spine_leaf(cap):
    i = 0
    while 2 * i + 1 < 2 * cap - 1:
        i = 2 * i + 2
    return i - cap + 1


def build_tree(leaves):
    """A float64 heap whose every parent is left + right (bottom-up, one numpy op per run of nodes)."""
    C = len(leaves)
    t = np.zeros(2 * C - 1, np.float64)
    t[C - 1:] = leaves
    hi = C - 1
    while hi > 0:
        i = np.arange(hi // 2, hi)
        t[i] = t[2 * i + 1] + t[2 * i + 2]
        hi //= 2
    return t


def int_leaves(rs, C):
    """Integer priorities 0..4, about a quarter of them zero, a zero at both ends."""
    p = rs.randint(0, 5, C).astype(np.float64)
    p[0] = p[-1] = 0.0
    if C > 2:
        p[1] = 3.0
    return p


def is_weights_ref(p, total, capacity, beta):
    """oracle.sumtree.importance_weights with the reference's fallback: priorities <= 0 become 1 / capacity."""
    p = np.where(np.asarray(p, np.float64) <= 0, 1.0 / np.float64(capacity), p)
    return osum.importance_weights(p, total, capacity, beta)


def ulp_diff32(a, b):
    a = np.asarray(a, F32).view(np.int32).astype(np.int64)
    b = np.asarray(b, F32).view(np.int32).astype(np.int64)
    return int(np.max(np.abs(a - b))) if a.size else 0


# ------------------------------------------------------------------------------------------------ statements (CPU)
@pytest.mark.parametrize("cap,nb", [(1, 1), (2, 1), (3, 1), (5, 1), (8, 1), (13, 1), (32, 1), (11, 3), (33, 1),
                                    (25, 4), (100, 1)])
def test_retrieve_is_the_first_leaf_whose_prefix_reaches_the_value(cap, nb):
    """oracle.sumtree.retrieve on integer trees with zeros: every half-integer in [0, total] (so every exact prefix sum)
    goes to the first leaf whose inclusive prefix sum is >= it; values above the total follow the all-right path."""
    C = cap * nb
    rs = np.random.RandomState(C)
    leaves = int_leaves(rs, C)
    ot = osum.SumTree(cap, nb)
    ot.tree = build_tree(leaves)
    total = ot.total()
    assert total == leaves.sum()
    values = np.arange(int(2 * total) + 1) / 2.0
    got = ot.retrieve(values) - C + 1
    assert np.array_equal(got, prefix_leaf(leaves, values))
    prefixes = np.cumsum(leaves[leaf_order(C)])
    assert np.isin(prefixes, values).all()
    above = np.array([np.nextafter(total, np.inf), total + 1, 2 * total + 7])
    assert np.all(ot.retrieve(above) - C + 1 == right_spine_leaf(C))
    assert right_spine_leaf(C) == leaf_order(C)[-1]
    # the descent's tie rule: '<' instead of '<=' moves some exact prefix sum to a later leaf
    if C > 1 and total > 0:
        lt = [int(np.searchsorted(prefixes, v, side="right")) for v in values]
        assert any(leaf_order(C)[min(k, C - 1)] != g for k, g in zip(lt, got))


@pytest.mark.parametrize("n", [1, 3, 1023, 1024, 1025, 12000])
def test_stratified_statement(n):
    """One value per stratum [a_s, b_s]; with CPython's b - a, oracle.sumtree.stratified_samples given the statement's u
    and permutation bit for bit, and the kernel's fused b - a within one ulp of it."""
    seed, stream = 0x1234_5678_9ABC_DEF, (1 << 39) + 17
    for total in (1.0, 12345.678, 2.0 ** 40 / 3):
        v, u, order = stratified_np(seed, stream, total, n)
        assert np.all((u > 0) & (u < 1))
        plain = stratified_np(seed, stream, total, n, fused=False)[0]
        assert_bits("oracle.stratified_samples", plain.view(np.uint64),
                    osum.stratified_samples(total, n, u, order).view(np.uint64))
        # the fused b - a moves a value by at most one ulp from random.uniform's
        assert np.all(np.abs(v - plain) <= np.spacing(np.abs(plain)))
        seg = total / n
        assert np.all(v >= order * seg) and np.all(v <= (order + 1) * seg)
        assert sorted(order.tolist()) == list(range(n))
    if n >= 1023:
        assert not np.array_equal(order, np.arange(n))
        # keys on the value stream, or u from one word, give other values
        w = philox_np(seed, stream, n).reshape(n, 4)
        assert not np.array_equal(np.lexsort((np.arange(n), w[:, 0])), order)
        u_x = ((w[:, 0].astype(np.uint64) >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
        assert not np.array_equal(u_x, u)


def test_fallback_weights_statement():
    """is_weights_ref: every priority <= 0 (0 and -0 included) weighs as 1 / capacity; equal priorities weigh alike."""
    p = np.array([0.0, -0.0, -3.0, 0.25, 0.25, 1.0])
    w = is_weights_ref(p, 10.0, 8, 0.4)
    assert w[0] == w[1] == w[2] and w[3] == w[4] and w.max() == 1.0
    assert w[0] == is_weights_ref([1 / 8, 0.25, 1.0], 10.0, 8, 0.4)[0]


# ------------------------------------------------------------------------------------------------ GPU helpers
def _err():
    from rainbow_iqn_apex_b200._lib import RiqnError
    return RiqnError


def _i64_bits(o):
    return o.t[:o.n].view(torch.int64).cpu().numpy()


def _f64(o):
    return o.t[:o.n].cpu().numpy()


def _f64_bits(o):
    return _f64(o).view(np.uint64)


def _dyn(dev, capacity=1.0, beta=0.0, writes=3):
    from rainbow_iqn_apex_b200.dynstate import DynState
    d = DynState(dev)
    for _ in range(writes):                 # rng_offset = 64 (writes - 1)
        d.write(0.0, 1.0, capacity, beta)
    torch.cuda.synchronize()
    return d


# ------------------------------------------------------------------------------------------------ stratified (GPU)
def _stratified(dev, n, seed, stream, tree, dyn=None):
    outs = []
    for _ in range(2):
        o = Out(n, dev, torch.float64)
        lib_call("riqn_sumtree_stratified", n, seed, stream, dptr(tree), o.p, dyn.ptr() if dyn else None)
        torch.cuda.synchronize()
        assert_canaries({"values": o})
        outs.append(_f64_bits(o))
    assert np.array_equal(outs[0], outs[1])
    return outs[0]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 1023, 1024, 1025, 2560, 12000])
def test_stratified_vs_statement(cuda_dev, n):
    """Bit for bit against stratified_np, without and with a riqn_dyn_state (then the stream moves by rng_offset)."""
    seed, stream = 0x0F1E_2D3C_4B5A_6978, (1 << 39) + 3
    for total in (1.0, 12345.678, 2.0 ** 40 / 3):
        tree = torch.tensor([total, 1.0, 2.0], dtype=torch.float64, device=cuda_dev)
        got = _stratified(cuda_dev, n, seed, stream, tree)
        assert_bits("stratified", got, stratified_np(seed, stream, total, n)[0].view(np.uint64))
        dyn = _dyn(cuda_dev)
        got_d = _stratified(cuda_dev, n, seed, stream, tree, dyn)
        assert_bits("stratified with dyn", got_d, stratified_np(seed, stream + 128, total, n)[0].view(np.uint64))
        assert_bits("dyn = plain call at stream + rng_offset", got_d, _stratified(cuda_dev, n, seed, stream + 128, tree))


@pytest.mark.gpu
def test_stratified_refusals(cuda_dev):
    tree = torch.tensor([5.0], dtype=torch.float64, device=cuda_dev)
    o = Out(12001, cuda_dev, torch.float64)
    for n, t, v in ((0, tree, o.p), (12001, tree, o.p), (-1, tree, o.p), (8, None, o.p), (8, tree, None)):
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_stratified", n, 1, 2, dptr(t), v, None)
    torch.cuda.synchronize()
    assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ sample (GPU)
SAMPLE_CAPS = [1, 2, 3, 5, 31, 32, 33, 48, 63, 64, 65, 1023, 1024, 1025, 1500, (1 << 15) + 1]
SAMPLE_HN = [(4, 3), (1, 1), (12, 4), (0, 0)]


@functools.lru_cache(maxsize=4)
def _sample_case(ac, nb):
    """An integer tree with zeros, and sample values: every exact prefix sum (a subset on the largest trees), 0, the
    total, the total + 1 ulp, random interior values; 4096 of them, 12000 on trees above 4000 leaves."""
    C = ac * nb
    rs = np.random.RandomState(ac * 7 + nb)
    leaves = int_leaves(rs, C)
    tree = build_tree(leaves)
    total = tree[0]
    N = 4096 if C <= 4000 else 12000
    prefixes = np.unique(np.cumsum(leaves[leaf_order(C)]))
    if prefixes.size > N // 2:
        prefixes = rs.choice(prefixes, N // 2, replace=False)
    special = np.array([0.0, total, np.nextafter(total, np.inf)])
    interior = rs.uniform(0, total, N - prefixes.size - special.size)
    values = np.concatenate([special, prefixes, interior])
    values = values[np.r_[0:3, 3 + rs.permutation(values.size - 3)]]
    ot = osum.SumTree(ac, nb)
    ot.tree = tree
    return tree, values, ot.retrieve(values)


def _sample(dev, tree_d, values_d, q, C, ac, heads_d, h, n):
    outs = []
    for _ in range(2):
        ti, di = Out(q, dev, torch.int64, I64_FILL), Out(q, dev, torch.int64, I64_FILL)
        pr = Out(q, dev, torch.float64)
        lib_call("riqn_sumtree_sample", q, C, ac, dptr(tree_d), dptr(values_d), dptr(heads_d), h, n, ti.p, di.p, pr.p)
        torch.cuda.synchronize()
        assert_canaries({"tree_idx": ti, "data_idx": di, "priorities": pr})
        outs.append((_i64_bits(ti), _i64_bits(di), _f64_bits(pr)))
    for a, b in zip(*outs):
        assert np.array_equal(a, b), "two calls differ"
    return outs[0]


def _check_sample(dev, tree, values, retrieved, ac, nb, heads, h, n, rows, q_list):
    C = ac * nb
    ot = osum.SumTree(ac, nb)
    ot.tree = tree
    ot.index_actor = np.asarray(heads, np.int64)
    want_t = ot.transform_to_valid(retrieved[rows], h, n)
    want = (want_t, want_t - C + 1, tree[want_t].view(np.uint64))
    tree_d = torch.from_numpy(tree).to(dev)
    vals_d = torch.from_numpy(np.ascontiguousarray(values[rows])).to(dev)
    heads_d = torch.tensor(heads, dtype=torch.int64, device=dev)
    for q in q_list:
        got = _sample(dev, tree_d, vals_d, q, C, ac, heads_d, h, n)
        for what, g, w in zip(("tree_idx", "data_idx", "priorities"), got, want):
            assert_bits(f"{what} (q {q}, heads {list(heads)})", g, w[:q])
    return want[1]


@pytest.mark.gpu
@pytest.mark.parametrize("hn", SAMPLE_HN, ids=[f"h{h}n{n}" for h, n in SAMPLE_HN])
@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("ac", SAMPLE_CAPS)
def test_sample_vs_oracle(cuda_dev, ac, nb, hn):
    """tree_idx, data_idx and priorities bit for bit against oracle retrieve + transform_to_valid: ties at every exact
    prefix sum, 0, the total and above, random interior values; query counts 1, 3 (a partial block of four warps) and
    all; write heads at 0, at cap - 1, random, and at every distance -n-1 .. history+1 from a sampled slot."""
    h, n = hn
    C = ac * nb
    tree, values, retrieved = _sample_case(ac, nb)
    rs = np.random.RandomState(C + 31 * h + n)
    allrows = np.arange(values.size)
    heads = rs.randint(0, ac, nb)
    _check_sample(cuda_dev, tree, values, retrieved, ac, nb, heads, h, n, allrows, (1, 3, values.size))
    # the head sweep on 96 rows that include, per segment, a row whose leaf is the target slot
    data = retrieved - C + 1
    targets, rows = [], list(range(64))
    for a in range(nb):
        in_a = np.nonzero(data // ac == a)[0]
        if in_a.size:
            r = int(in_a[np.argmin(np.abs(data[in_a] % ac - ac // 2))])
            rows.append(r)
            targets.append(int(data[r] % ac))
        else:
            targets.append(ac // 2)
    rows = np.array(rows + list(range(64, 96 - len(rows) + 64)))
    settings = [np.zeros(nb, np.int64), np.full(nb, ac - 1)]
    settings += [np.array([(p - dist) % ac for p in targets]) for dist in range(-n - 1, h + 2)]
    moved = 0
    for heads in settings:
        got = _check_sample(cuda_dev, tree, values, retrieved, ac, nb, heads, h, n, rows, (rows.size,))
        moved += int((got != data[rows]).sum())
    assert moved > 0 or ac <= 2


@pytest.mark.gpu
def test_sample_refusals(cuda_dev):
    tree = torch.from_numpy(build_tree(np.arange(1.0, 13.0))).to(cuda_dev)
    vals = torch.tensor([1.0, 5.0, 70.0], dtype=torch.float64, device=cuda_dev)
    heads = torch.zeros(3, dtype=torch.int64, device=cuda_dev)
    ti, di = Out(3, cuda_dev, torch.int64, I64_FILL), Out(3, cuda_dev, torch.int64, I64_FILL)
    pr = Out(3, cuda_dev, torch.float64)
    ok = [3, 12, 4, dptr(tree), dptr(vals), dptr(heads), 4, 3, ti.p, di.p, pr.p]
    bad = [(1, 0), (1, -12), (2, 0), (2, -4), (2, 5), (2, 7), (6, -1), (7, -1)] + [(k, None) for k in (3, 4, 5, 8, 9, 10)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_sample", *args)
    torch.cuda.synchronize()
    assert bool((ti.t[:3] == I64_FILL).all() and (di.t[:3] == I64_FILL).all() and torch.isnan(pr.t[:3]).all())
    assert_canaries({"ti": ti, "di": di, "pr": pr})
    lib_call("riqn_sumtree_sample", *ok)            # the accepted call writes
    torch.cuda.synchronize()
    assert bool((ti.t[:3] >= 11).all())


# ------------------------------------------------------------------------------------------------ IS weights (GPU)
IS_N = [1, 2, 31, 32, 33, 1023, 1024, 1025, 4096, 12000]


def _is_weights(dev, p, total, capacity, beta, dyn=None, count=True):
    n = len(p)
    tree = torch.tensor([total], dtype=torch.float64, device=dev)
    pd = torch.from_numpy(np.ascontiguousarray(p, np.float64)).to(dev)
    outs = []
    for _ in range(2):
        w64, w32 = Out(n, dev, torch.float64), Out(n, dev, torch.float32)
        cnt = Out(1, dev, torch.int32, I64_FILL) if count else None
        lib_call("riqn_sumtree_is_weights", n, dptr(tree), dptr(pd), float(capacity), float(beta), w64.p, w32.p,
                 cnt.p if count else None, dyn.ptr() if dyn else None)
        torch.cuda.synchronize()
        assert_canaries({"w64": w64, "w32": w32, "count": cnt})
        outs.append((_f64(w64), w32.bits(), int(cnt.t[0].item()) if count else None))
    assert np.array_equal(outs[0][0].view(np.uint64), outs[1][0].view(np.uint64))
    assert np.array_equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
    return outs[0]


def _priorities(rs, n, total, with_nonpositive):
    p = rs.uniform(0, 1, n) ** 3 * total / 4 + 1e-9 * total
    if n >= 8:
        p[rs.randint(0, n, max(1, n // 50))] = p[0]                       # equal priorities
    if with_nonpositive and n >= 4:
        k = rs.permutation(n)[:max(3, n // 40)]
        p[k[0::3]], p[k[1::3]], p[k[2::3]] = 0.0, -0.0, -rs.uniform(0, 1, k[2::3].size)
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("n", IS_N)
def test_is_weights_vs_oracle(cuda_dev, n):
    """w64 within the pow bound of the oracle with the <= 0 fallback; max(w64) == 1 exactly and every w64 <= 1;
    w32 == fl32(w64); beta 0 -> 1.0; equal priorities -> equal bits; n_nonpositive counts 0, -0 and negatives; NULL
    count accepted.  Bound: the device pow is within 2 ulp (CUDA's documented double pow), numpy's within 1 ulp, one
    rounding per division on each side, so |w - w_ref| <= w_ref ((2 + 2) + (1 + 1) + 1) 2^-52 (1 + 2^-40)."""
    rs = np.random.RandomState(n)
    worst = 0.0
    for total, capacity, beta, nonpos in ((1234.5, 5000, 0.4, True), (3.0, 17, 1.0, False), (1e6, 1 << 20, 0.73, True)):
        p = _priorities(rs, n, total, nonpos)
        w64, w32, cnt = _is_weights(cuda_dev, p, total, capacity, beta)
        ref = is_weights_ref(p, total, capacity, beta)
        bound = ref * 7 * 2.0 ** -52 * (1 + 2.0 ** -40)
        worst = max(worst, check_bound(f"w64 n={n} beta={beta}", w64, ref, bound))
        assert w64.max() == 1.0 and np.all(w64 <= 1.0)
        assert_bits("w32 = fl32(w64)", w32, f32_bits(w64.astype(F32)))
        assert cnt == int((p <= 0).sum())
        eq = p == p[0]
        assert np.unique(w64[eq].view(np.uint64)).size == 1
        if nonpos and n >= 4:
            assert cnt > 0 and np.unique(w64[p <= 0].view(np.uint64)).size == 1
        w64n, w32n, _ = _is_weights(cuda_dev, p, total, capacity, beta, count=False)
        assert np.array_equal(w64n.view(np.uint64), w64.view(np.uint64))
    w64, w32, _ = _is_weights(cuda_dev, _priorities(rs, n, 10.0, True), 10.0, 64, 0.0)
    assert np.all(w64 == 1.0) and np.all(w32 == f32_bits(np.ones(n, F32)))
    print(f"is_weights n={n}: worst err/bound {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_is_weights_dyn_overrides(cuda_dev, n):
    """With a riqn_dyn_state the device capacity and beta are used, and the by-value ones (even invalid) ignored."""
    rs = np.random.RandomState(n + 1)
    p = _priorities(rs, n, 50.0, True)
    plain = _is_weights(cuda_dev, p, 50.0, 300, 0.6)
    dyn = _dyn(cuda_dev, capacity=300, beta=0.6)
    for cap, beta in ((17, 0.1), (float("nan"), -1.0), (0.0, float("inf"))):
        got = _is_weights(cuda_dev, p, 50.0, cap, beta, dyn)
        assert np.array_equal(got[0].view(np.uint64), plain[0].view(np.uint64)) and got[2] == plain[2]


@pytest.mark.gpu
def test_is_weights_refusals(cuda_dev):
    n = 8
    tree = torch.tensor([4.0], dtype=torch.float64, device=cuda_dev)
    p = torch.full((n,), 0.5, dtype=torch.float64, device=cuda_dev)
    w64, w32, cnt = Out(n, cuda_dev, torch.float64), Out(n, cuda_dev), Out(1, cuda_dev, torch.int32, I64_FILL)
    ok = [n, dptr(tree), dptr(p), 16.0, 0.4, w64.p, w32.p, cnt.p, None]
    bad = [(0, 0), (0, -3), (1, None), (2, None), (5, None), (6, None)]
    bad += [(3, v) for v in (-1e-300, -1.0, float("nan"), float("inf"))] + [(4, v) for v in (-0.1, float("nan"), float("inf"))]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_is_weights", *args)
    torch.cuda.synchronize()
    assert bool(torch.isnan(w64.t[:n]).all() and torch.isnan(w32.t[:n]).all()) and int(cnt.t[0].item()) == I64_FILL
    assert_canaries({"w64": w64, "w32": w32, "cnt": cnt})



@pytest.mark.gpu
def test_is_weights_zero_capacity_is_the_references_nan(cuda_dev):
    """Capacity 0 (a tree filled without the fill count) is accepted and gives what the reference's numpy gives:
    (0 * p)^-beta = inf for p > 0 and 0 * inf for the fallback's 1/0, so every weight is NaN; the count still holds."""
    p = np.array([0.5, 2.0, 0.0, -0.0, 1.0])
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = is_weights_ref(p, 4.0, 0.0, 0.4)
    assert np.all(np.isnan(ref))
    w64, w32, cnt = _is_weights(cuda_dev, p, 4.0, 0.0, 0.4)
    assert np.all(np.isnan(w64)) and np.all(np.isnan(w32.view(F32))) and cnt == 2

# ------------------------------------------------------------------------------------------------ update (GPU)
def _update(dev, tree64, idx, loss, exponent, apply_pow=1, max_priority=1.0):
    C = (tree64.size + 1) // 2
    n = idx.size
    idx_d = torch.from_numpy(idx.astype(np.int64)).to(dev)
    loss_d = torch.from_numpy(np.ascontiguousarray(loss, F32)).to(dev)
    res = []
    for _ in range(2):
        tree = torch.from_numpy(tree64.copy()).to(dev)
        new = Out(n, dev)
        diff = torch.empty(n, dtype=torch.float64, device=dev)
        mx = torch.full((1,), max_priority, dtype=torch.float64, device=dev)
        lib_call("riqn_sumtree_update", n, C, dptr(tree), dptr(idx_d), dptr(loss_d), float(exponent), apply_pow, new.p,
                 dptr(diff), dptr(mx))
        torch.cuda.synchronize()
        assert_canaries({"new": new})
        res.append((tree.cpu().numpy(), new.f32(), float(mx.item())))
    assert np.array_equal(res[0][0].view(np.uint64), res[1][0].view(np.uint64))
    assert np.array_equal(f32_bits(res[0][1]), f32_bits(res[1][1])) and res[0][2] == res[1][2]
    return res[0]


def _update_indices(rs, C, n, kind):
    lo, hi = C - 1, 2 * C - 1
    if kind == "one_leaf":
        return np.full(n, rs.randint(lo, hi), np.int64)
    idx = rs.randint(lo, hi, n)
    if kind == "slices" and n > 64:
        # duplicates across the eight propagate slices: entry j and j + 64 k name the same leaf
        for j in range(0, min(n, 64), 5):
            idx[j::64] = idx[j]
    if kind == "depths":
        # leaves at both depths of a non-power-of-two tree under shared ancestors: neighbours of the depth boundary
        d = int(np.floor(np.log2(2 * C - 1)))
        first_deep = (1 << d) - 1
        near = np.r_[np.arange(max(lo, first_deep - 40), first_deep), np.arange(max(lo, first_deep), min(hi, first_deep + 40)),
                     np.arange(max(lo, hi - 40), hi)]
        idx = near[rs.randint(0, near.size, n)]
    return idx.astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "slices", "depths", "one_leaf"])
@pytest.mark.parametrize("n", [1, 7, 8, 127, 128, 129, 4096])
def test_update_vs_oracle(cuda_dev, n, kind):
    """Tree and max_priority bit for bit against oracle update_multiple_value on the device's own priorities (within 1
    ulp of numpy's float32 power); the pairwise root sum at its block boundaries; apply_pow 0, exponent 0, loss 0."""
    for cap, nb in ((1000, 3), (1024, 1)):
        C = cap * nb
        rs = np.random.RandomState(n * 7 + C + len(kind))
        # full float64 leaves: with float32-valued leaves every diff and node sum would be exact, and the order of the
        # adds (pairwise root, shallower leaves first) would not show in the bits
        base = build_tree(rs.uniform(0.05, 1.5, C))
        idx = _update_indices(rs, C, n, kind)
        assert idx.min() >= C - 1 and idx.max() <= 2 * C - 2
        loss = (rs.uniform(0.01, 3.0, n) * 10.0 ** -rs.randint(0, 3, n) * 8).astype(F32)
        loss[rs.randint(0, n)] = F32(0.0)
        if n > 1:
            loss[-1] = F32(40.0)                                            # raises max_priority
        for omega, apply_pow in ((0.2, 1), (0.5, 1), (0.0, 1), (0.2, 0)):
            t, new, mx = _update(cuda_dev, base, idx, loss, omega, apply_pow)
            if apply_pow:
                assert ulp_diff32(new, np.power(loss, F32(omega))) <= 1
                if omega == 0.0:
                    assert np.all(new == 1.0)
                assert np.all(new[loss == 0] == 0.0) or omega == 0.0
            else:
                assert_bits("apply_pow 0 passes the priorities through", f32_bits(new), f32_bits(loss))
            ot = osum.SumTree(cap, nb)
            ot.tree = base.copy()
            ot.update_multiple_value(idx, new.astype(np.float64))
            assert_bits(f"tree (omega {omega}, apply_pow {apply_pow})", t.view(np.uint64), ot.tree.view(np.uint64))
            assert mx == ot.max_priority


@pytest.mark.gpu
def test_update_refusals(cuda_dev):
    C = 64
    base = build_tree(np.linspace(0.1, 1.0, C))
    tree = torch.from_numpy(base.copy()).to(cuda_dev)
    idx = torch.arange(C - 1, C + 4096, dtype=torch.int64, device=cuda_dev) % C + C - 1
    loss = torch.full((4097,), 0.5, device=cuda_dev)
    new = Out(4097, cuda_dev)
    diff = torch.empty(4097, dtype=torch.float64, device=cuda_dev)
    mx = torch.full((1,), 0.25, dtype=torch.float64, device=cuda_dev)
    ok = [10, C, dptr(tree), dptr(idx), dptr(loss), 0.5, 1, new.p, dptr(diff), dptr(mx)]
    bad = [(0, 4097), (1, 0), (1, -5)] + [(k, None) for k in (2, 3, 4, 7, 8, 9)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_update", *args)
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_update_demo", *args, C - 1, 0.0)
    torch.cuda.synchronize()
    assert np.array_equal(tree.cpu().numpy().view(np.uint64), base.view(np.uint64)) and float(mx.item()) == 0.25
    assert bool(torch.isnan(new.t[:new.n]).all()) and new.canaries_ok()


# ------------------------------------------------------------------------------------------------ frame store (GPU)
class _Store:
    """The device frame store (flat buffers with canaries past their ends) beside an oracle ReplayStore holding the
    same transitions."""

    def __init__(self, dev, rs, cap, nb, p_start=0.0, p_term=0.0):
        self.cap, self.nb, self.dev = cap, nb, dev
        C = cap * nb
        self.o = orep.ReplayStore(cap, nb)
        ts = rs.randint(1, 50, C)
        ts[rs.uniform(size=C) < p_start] = 0
        dn = rs.uniform(size=C) < p_term
        fr = rs.randint(0, 256, (C, 84, 84)).astype(np.uint8)
        ac = rs.randint(0, 18, C)
        rw = (rs.randint(-80000, 80001, C) / 8).astype(F32)          # exact in fp32, |r| <= 10^4
        for a in range(nb):
            seg = slice(a * cap, (a + 1) * cap)
            self.o.write(a, 0, ts[seg], fr[seg], ac[seg], rw[seg], dn[seg])
        P = 4096

        def buf(x, dt, canary):
            t = torch.full((x.size + P,), canary, dtype=dt, device=dev)
            t[:x.size] = torch.from_numpy(np.ascontiguousarray(x).ravel()).to(dev, dt)
            return t
        self.frames = buf(fr, torch.uint8, 0x5C)
        self.timestep = buf(ts, torch.int32, -77)
        self.action = buf(ac, torch.int32, -77)
        self.reward = buf(rw, torch.float32, -77.0)
        self.nonterminal = buf((~dn).astype(np.uint8), torch.uint8, 0x5C)
        self.C = C

    def ptrs(self):
        return [dptr(t) for t in (self.frames, self.timestep, self.action, self.reward, self.nonterminal)]

    def snapshot(self):
        return [t.cpu().numpy().copy() for t in (self.frames, self.timestep, self.action, self.reward, self.nonterminal)]

    def assert_matches_oracle(self):
        C, o = self.C, self.o
        fr, ts, ac, rw, nt = self.snapshot()
        assert np.array_equal(fr[:C * FRAME], o.frame.ravel()) and np.all(fr[C * FRAME:] == 0x5C)
        assert np.array_equal(ts[:C], o.timestep) and np.all(ts[C:] == -77)
        assert np.array_equal(ac[:C], o.action) and np.all(ac[C:] == -77)
        assert np.array_equal(f32_bits(rw[:C]), f32_bits(o.reward.astype(F32))) and np.all(rw[C:] == -77.0)
        assert np.array_equal(nt[:C], o.nonterminal.astype(np.uint8)) and np.all(nt[C:] == 0x5C)


@pytest.mark.gpu
@pytest.mark.parametrize("id_actor,start,n", [(0, 0, 1), (2, 63, 1), (1, 0, 64), (2, 61, 64), (1, 60, 9), (0, 17, 40)])
def test_append_vs_oracle(cuda_dev, id_actor, start, n):
    """The whole store after riqn_replay_append (frames and the four metadata arrays of every segment, canaries past
    each) equals ReplayStore.write bit for bit, wrapping the ring where start + n passes its end; a repeated call
    leaves the same store."""
    rs = np.random.RandomState(id_actor * 1000 + start * 10 + n)
    cap, nb = 64, 3
    st = _Store(cuda_dev, rs, cap, nb, 0.1, 0.1)
    ts, fr = rs.randint(0, 9, n), rs.randint(0, 256, (n, 84, 84)).astype(np.uint8)
    ac, rw, dn = rs.randint(0, 18, n), (rs.randint(-80000, 80001, n) / 8).astype(F32), rs.uniform(size=n) < 0.3
    src = [torch.from_numpy(np.ascontiguousarray(x)).to(cuda_dev, dt) for x, dt in
           ((fr.reshape(n, FRAME), torch.uint8), (ts, torch.int32), (ac, torch.int32), (rw, torch.float32),
            ((~dn).astype(np.uint8), torch.uint8))]
    st.o.write(id_actor, start, ts, fr, ac, rw, dn)
    for _ in range(2):
        lib_call("riqn_replay_append", n, cap, id_actor, start, *[dptr(t) for t in src], *st.ptrs())
        torch.cuda.synchronize()
        st.assert_matches_oracle()


@pytest.mark.gpu
def test_append_refusals(cuda_dev):
    rs = np.random.RandomState(3)
    cap, nb = 16, 2
    st = _Store(cuda_dev, rs, cap, nb)
    n = cap + 1
    src = [torch.from_numpy(np.ascontiguousarray(x)).to(cuda_dev) for x in
           (np.full(n * FRAME, 9, np.uint8), np.full(n, 5, np.int32), np.full(n, 3, np.int32), np.full(n, 2.5, F32),
            np.zeros(n, np.uint8))]
    before = st.snapshot()
    ok = [4, cap, 1, 3, *[dptr(t) for t in src], *st.ptrs()]
    bad = [(0, cap + 1), (1, 0), (1, -2), (2, -1), (3, -1), (3, cap), (3, cap + 5)] + [(k, None) for k in range(4, 14)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_replay_append", *args)
    torch.cuda.synchronize()
    for a, b in zip(st.snapshot(), before):
        assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("device_side", [False, True])
def test_segment_tree_append_refuses_before_the_tree(cuda_dev, device_side):
    """SegmentTree.append_arrays / append_device refuse n > actor_capacity, a start outside the ring and a segment
    outside the store before the priorities reach the tree: tree, max_priority and store stay as they were."""
    from rainbow_iqn_apex_b200 import ReplayMemory
    mem = ReplayMemory(make_args(cuda_dev, 8, nb_actor=2, actor_capacity=16), None)
    tr = mem.transitions
    tr.append_arrays(0, 0, np.arange(16), np.zeros((16, 84, 84), np.uint8), np.zeros(16), np.zeros(16, F32),
                     np.zeros(16, bool), np.full(16, 0.5, F32))
    snap = [t.clone() for t in (tr.tree, tr.max_priority, tr.frames, tr.timestep, tr.index_actor)]
    for a, start, n in ((0, 0, 17), (1, 16, 4), (1, -1, 4), (2, 0, 4), (-1, 0, 4)):
        pri = np.full(n, 7.0, F32)
        with pytest.raises(ValueError):
            if device_side:
                tr.append_device(a, start, torch.zeros(n, device=cuda_dev), torch.full((n, FRAME), 3, dtype=torch.uint8,
                                 device=cuda_dev), torch.zeros(n, device=cuda_dev), torch.zeros(n, device=cuda_dev),
                                 torch.ones(n, device=cuda_dev), torch.from_numpy(pri).to(cuda_dev))
            else:
                tr.append_arrays(a, start, np.arange(n), np.full((n, 84, 84), 3, np.uint8), np.zeros(n), np.zeros(n, F32),
                                 np.zeros(n, bool), pri)
    torch.cuda.synchronize()
    for a, b in zip((tr.tree, tr.max_priority, tr.frames, tr.timestep, tr.index_actor), snap):
        assert torch.equal(a, b)


GATHER_HN = [(1, 1), (2, 5), (4, 1), (4, 3), (4, 12), (8, 8), (12, 4)]


def _gather(dev, st, data_idx, h, n, gamma_pow):
    B, L = data_idx.size, h + n
    d = torch.from_numpy(data_idx).to(dev)
    g = torch.tensor(gamma_pow, dtype=torch.float64, device=dev)
    outs = []
    for _ in range(2):
        win = torch.full((B * L * FRAME + 4096,), 0x5C, dtype=torch.uint8, device=dev)
        win[:B * L * FRAME] = 0xAB
        act, ret, nt = Out(B, dev, torch.int64, I64_FILL), Out(B, dev), Out(B, dev)
        lib_call("riqn_frame_gather", B, st.cap, h, n, dptr(d), *st.ptrs(), dptr(g), dptr(win), act.p, ret.p, nt.p)
        torch.cuda.synchronize()
        assert bool((win[B * L * FRAME:] == 0x5C).all())
        assert_canaries({"actions": act, "returns": ret, "nonterminals": nt})
        outs.append((win[:B * L * FRAME].cpu().numpy().reshape(B, L, 84, 84), _i64_bits(act), ret.bits(), nt.bits()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b), "two calls differ"
    return outs[0]


@pytest.mark.gpu
@pytest.mark.parametrize("hn", GATHER_HN, ids=[f"h{h}n{n}" for h, n in GATHER_HN])
def test_frame_gather_vs_oracle(cuda_dev, hn):
    """Window, actions, returns and nonterminals bit for bit against ReplayStore.assemble, discounts 0.99 and 0.5,
    rewards up to 10^4; an episode start and a terminal at every offset of the window; ring positions 0 and cap - 1 of
    segments > 0; B = 4096.  Window frame k >= history is assemble's last next-state frame at n_step = k - history + 1."""
    h, n = hn
    L = h + n
    cap, nb = 64, 3
    rs = np.random.RandomState(10 * h + n)
    st = _Store(cuda_dev, rs, cap, nb, 0.12, 0.12)
    B = 4096
    d = rs.randint(0, cap * nb, B).astype(np.int64)
    d[:cap * nb] = np.arange(cap * nb)
    d[-4:] = [cap, 2 * cap - 1, 2 * cap, 3 * cap - 1]
    for k in range(L):                   # the store puts an episode start and a terminal at every window offset
        slots = np.array([st.o.window_slots(int(x), h, n)[k] for x in d[:cap * nb]])
        assert (st.o.timestep[slots] == 0).any() and (~st.o.nonterminal[slots]).any(), k
    for disc in (0.99, 0.5):
        gp = [disc ** k for k in range(n)]
        win, act, ret, nt = _gather(cuda_dev, st, d, h, n, gp)
        s, a, r, nx, t = st.o.assemble(d, h, n, disc)
        assert np.array_equal(win[:, :h], s) and np.array_equal(win[:, n:n + h], nx)
        assert np.array_equal(act, a)
        assert_bits("returns", ret, f32_bits(r))
        assert_bits("nonterminals", nt, f32_bits(t))
        assert (t == 0).any() and (t == 1).any() and np.abs(r).max() > 1000
    for k in range(h, L):
        nxk = st.o.assemble(d, h, k - h + 1, 0.99)[3]
        assert np.array_equal(win[:, k], nxk[:, h - 1]), k


@pytest.mark.gpu
def test_frame_gather_refusals(cuda_dev):
    rs = np.random.RandomState(4)
    st = _Store(cuda_dev, rs, 16, 2)
    d = torch.arange(4, dtype=torch.int64, device=cuda_dev)
    g = torch.ones(16, dtype=torch.float64, device=cuda_dev)
    win = torch.full((4 * 17 * FRAME,), 0xAB, dtype=torch.uint8, device=cuda_dev)
    act, ret, nt = Out(4, cuda_dev, torch.int64, I64_FILL), Out(4, cuda_dev), Out(4, cuda_dev)
    ok = [4, 16, 4, 3, dptr(d), *st.ptrs(), dptr(g), dptr(win), act.p, ret.p, nt.p]
    bad = [(1, 0), (1, -16), (2, 0), (2, -1), (3, 0), (3, -2), (3, 13)] + [(k, None) for k in range(4, 15)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_frame_gather", *args)
    torch.cuda.synchronize()
    assert bool((win == 0xAB).all()) and bool((act.t[:4] == I64_FILL).all())
    assert bool(torch.isnan(ret.t[:4]).all() and torch.isnan(nt.t[:4]).all())
    assert_canaries({"act": act, "ret": ret, "nt": nt})


# ------------------------------------------------------------------------------------------------ ReplayMemory (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("filled", [1, 2, 3])
def test_resample_loop_draws_eleven_times_then_falls_back(cuda_dev, filled):
    """A segment written only at positions 0 .. h-1 (h <= n_step): every sample shifts to slot cap + h - n - 1, which is
    unwritten, so every draw has priority 0.  sample_indices draws 11 times, as the reference (one draw and up to 10
    more), then applies the fallback: all weights exactly 1, last_nonpositive == B.  A filled segment draws once."""
    from rainbow_iqn_apex_b200 import ReplayMemory
    B, cap = 32, 64
    mem = ReplayMemory(make_args(cuda_dev, B, nb_actor=1, actor_capacity=cap), None)
    tr = mem.transitions
    h = filled
    tr.append_arrays(0, 0, np.arange(1, h + 1), np.zeros((h, 84, 84), np.uint8), np.zeros(h), np.ones(h, F32),
                     np.zeros(h, bool), np.ones(h, F32))
    d0 = tr._draws
    tree_idx, data_idx, pri, w64, w32 = mem.sample_indices(B)
    torch.cuda.synchronize()
    assert tr._draws - d0 == 11
    assert np.all(data_idx.cpu().numpy() == cap + h - mem.n - 1)
    assert np.all(pri.cpu().numpy() == 0.0)
    assert np.all(w64.cpu().numpy() == 1.0) and np.all(w32.cpu().numpy() == 1.0)
    assert int(mem.last_nonpositive.item()) == B
    tr.append_arrays(0, h, np.arange(cap - h), np.zeros((cap - h, 84, 84), np.uint8), np.zeros(cap - h),
                     np.ones(cap - h, F32), np.zeros(cap - h, bool), np.ones(cap - h, F32))
    d0 = tr._draws
    mem.sample_indices(B)
    assert tr._draws - d0 == 1 and int(mem.last_nonpositive.item()) == 0
