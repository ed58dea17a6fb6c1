"""DQfD (Hester et al., AAAI 2018): the quantile-Huber loss plus lambda times the large-margin imitation loss on the rows
flagged as demonstrations (riqn_dqfd_loss_fwd_bwd, riqn_dqfd_loss_fwd_bwd_h), its dense upstream gradient
(riqn_dqfd_dense_grad), the demonstration priority bonus of the replay (riqn_sumtree_update_demo), behind the optional Agent
fields dqfd, dqfd_margin, dqfd_lambda and the ReplayMemory fields demo_segments, demo_priority_bonus.

The unmarked tests pin the float64 statement (oracle/dqfd.py) by identities, against float64 autograd and central
differences, check the torch-fp32 step against it and check the host-side validation.  The gpu tests hold the entry points
to their statements with the method of test_gpu_cql.py (NaN prefills, canaries, two calls alike, rejected calls write
nothing): td_loss, dtheta, theta_out and target_out bit for bit those of riqn_iqn_loss_fwd_bwd[_h]; Q, a_hat, J, loss and
G bit for bit against their numpy float32 statements; the tree update bit for bit against the numpy tree.  Value-only
mutants of those statements, and the cases that reject them (test_kernel_vs_float64 and test_tree_update_vs_oracle assert
it): the margin added on a_E as well (every case with a row whose a_E leads the others and absorbs no l), the last of equal maxima winning (the "equal" regime at A >= 3), c =
lambda instead of lambda / N (N > 1, a flagged row with a_hat != a_E), the mask ignored in the loss (the zero and
alternating masks, where an unflagged row has J > 0) or in the dense gradient (the same, where a_hat != a_E), the bonus
applied below demo_leaf and the bonus added before the power (the tree cases).  These are checked as numpy statements
against the kernels' outputs, not as rebuilt libraries.  At the learner level: the step against the torch oracle,
autograd, the replay's flags, reproducibility eagerly and from the replay and batch graphs, data parallelism, the actors,
launch counts, configuration errors, and that a namespace without the fields runs exactly as before."""
import math

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, assert_canaries, dptr, f32_bits, lib_call, load_params, make_args, to_dev
from oracle import cases, dqfd as od, network as net, qr as oq, sumtree as ost

F32 = np.float32
MARGINS = [0.8, 2.0 ** -10, 3.0, 100.0]
LAMBDAS = [1.0, 0.5, 4.0, 2.0 ** -10]


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def _q(rs, N, B, A, scale=1.0):
    return rs.standard_normal((N * B, A)) * scale


def test_margin_identities():
    rs = np.random.RandomState(1)
    for N, B, A in ((1, 5, 1), (8, 16, 4), (64, 32, 18), (3, 7, 32)):
        q = _q(rs, N, B, A, 3.0)
        act = rs.randint(0, A, B)
        for l in (0.8, 0.05, 5.0):
            J, a_hat = od.margin_np(q, B, act, l)
            Q = q.reshape(N, B, A).mean(0)
            Qe = Q[np.arange(B), act]
            others = np.where(np.arange(A)[None, :] == act[:, None], -np.inf, Q).max(1)
            assert np.all(J >= 0)
            zero = Qe >= others + l                     # J = 0 exactly when a_E leads every other action by l
            assert np.all((J == 0) == zero)
            assert np.allclose(J[~zero], (l + others - Qe)[~zero], rtol=0, atol=1e-12)
            if A == 1:
                assert np.all(J == 0) and np.all(a_hat == 0)
            # a constant on every quantile of every action changes neither J nor its gradient
            for c in (-7.5, 1e3):
                assert np.max(np.abs(od.margin_np(q + c, B, act, l)[0] - J)) <= 1e-9
                assert np.array_equal(od.margin_grad_np(q + c, B, act, l), od.margin_grad_np(q, B, act, l))
            d = od.margin_grad_np(q, B, act, l).reshape(N, B, A)
            assert np.max(np.abs(d.sum((0, 2)))) == 0.0     # the gradient sums to zero per transition
            assert np.all(d[:, a_hat == act] == 0)


def test_margin_gradient_vs_autograd_and_differences():
    rs = np.random.RandomState(2)
    for N, B, A in ((1, 3, 2), (8, 4, 18), (64, 2, 32)):
        q = _q(rs, N, B, A, 2.0)
        act = rs.randint(0, A, B)
        l = 0.8
        qt = torch.tensor(q, dtype=torch.float64, requires_grad=True)
        od.margin_torch(qt, N, B, torch.from_numpy(act), l).sum().backward()
        d = od.margin_grad_np(q, B, act, l)
        assert np.max(np.abs(d - qt.grad.numpy())) <= 1e-15
        h = 1e-6
        v = q.reshape(N, B, A).mean(0) + l
        v[np.arange(B), act] -= l
        gap2 = np.sort(v, 1)[:, -2:] if A > 1 else np.zeros((B, 2))
        for r, a in zip(rs.randint(0, N * B, 12), rs.randint(0, A, 12)):
            if A > 1 and gap2[r % B, 1] - gap2[r % B, 0] < 1e-3:
                continue                                # a near-tie of the maximum: J is not differentiable there
            qp, qm = q.copy(), q.copy()
            qp[r, a] += h
            qm[r, a] -= h
            num = (od.margin_np(qp, B, act, l)[0] - od.margin_np(qm, B, act, l)[0]) / (2 * h)
            assert abs(num[r % B] - d[r, a]) <= 1e-6


@pytest.mark.parametrize("kind,eps", [("iqn", None), ("iqn", 1e-3), ("qr", None), ("qr", 1e-3)])
def test_float64_and_torch_fp32_statements_agree(kind, eps):
    B, N, A, l, lam = 4, 8, 6, 0.8, 2.0
    cfg = cases.iqn_cfg(N, N, 8)
    b = cases.make_batch(40, B, action_space=A)
    st, ac, rt, nx, nt = cases.batch_to_torch(b)
    if eps is not None:
        rt = rt * 40
    if kind == "qr":
        params, noises, taus = oq.make_params(41, A, N), oq.make_noises(42, A, N), None
    else:
        params, noises = net.make_params(41, A), cases.make_noises(42, action_space=A)
        taus = tuple(torch.from_numpy(t) for t in cases.make_taus(43, B, cfg))
    demo = np.array([1, 0, 1, 1], np.uint8)
    keep = {}
    loss = od.dqfd_loss(kind, net.to_torch(params, requires_grad=True), net.to_torch(params), (st, ac, rt, nx, nt),
                        noises, taus, cfg, l, lam, demo, eps, keep)
    J64, _ = od.margin_np(keep["q_on"].detach().numpy(), B, b["actions"], l)
    assert np.all(J64 >= 0)
    l64 = keep["td"].numpy().astype(np.float64) + lam * demo * J64
    assert np.max(np.abs(loss.detach().numpy() - l64) / np.abs(l64)) < 1e-6


def test_bonus_priorities_on_the_oracle_tree():
    """With the bonus, a leaf's priority is the plain one plus eps_d at and above demo_leaf; a duplicate's diff is taken
    against the leaf before the batch (the reference's old-leaf semantics), so it ends as p1 + p2 - old."""
    rs = np.random.RandomState(3)
    cap, nb = 64, 4
    base = ost.SumTree(cap, nb)
    for a in range(nb):
        base.append_priorities(0, a, rs.uniform(0.1, 1.0, cap).astype(F32).astype(np.float64))
    C = base.full_capacity
    leaf = (nb - 1) * cap + C - 1
    idx = np.array([C - 1, leaf - 1, leaf, leaf, C + 3 * cap + 10, 2 * C - 2])
    loss = rs.uniform(0.1, 2.0, idx.size).astype(F32)
    plain = od.bonus_priorities(loss, idx, 0.5, leaf, 0.0)
    p = od.bonus_priorities(loss, idx, 0.5, leaf, 0.25)
    on = idx >= leaf
    assert np.array_equal(p[~on], plain[~on]) and np.array_equal(p[on], (plain[on] + F32(0.25)).astype(F32))
    t = ost.SumTree(cap, nb)
    t.tree = base.tree.copy()
    old = t.tree[idx].copy()
    got = od.update_priorities_demo(t, idx, loss, 0.5, leaf, 0.25)
    assert np.array_equal(got, p)
    assert t.tree[leaf] == old[2] + (p[2] - old[2]) + (p[3] - old[3])
    assert t.tree[idx[0]] == float(p[0]) and t.max_priority == max(1.0, float(p.max()))
    assert t.check() < 1e-12


# ------------------------------------------------------------------------------------------------ kernels (GPU)
# (B, A, N, N'): the CQL kernel tests' shapes
KERNEL_SHAPES = [(1, 1, 1, 1), (7, 4, 8, 5), (32, 18, 64, 64), (512, 18, 64, 64), (4096, 4, 32, 32), (32, 32, 200, 200),
                 (7, 32, 1500, 64), (32, 1, 64, 2000), (512, 32, 64, 2000)]
REGIMES = ["gauss", "equal", "ahead", "large"]
MASKS = ["null", "zero", "one", "alternating"]


def _kernel_inputs(B, A, N, Np, regime, seed):
    rs = np.random.RandomState(seed)
    q_on = rs.standard_normal((N * B, A))
    if regime == "equal":        # every Q within 1e-6; columns with the same offset are equal bit for bit: exact ties
        off = np.tile(rs.randint(0, 2, (1, B, A)) * 1e-6, (N, 1, 1)).reshape(N * B, A)
        q_on = np.tile(rs.standard_normal((N * B, 1)), (1, A)) + off
    elif regime == "large":
        q_on = q_on * 1e4
    h = dict(q_on=q_on.astype(F32), q_tg=rs.standard_normal((Np * B, A)).astype(F32),
             tau=rs.uniform(0, 1, N * B).astype(F32), act=rs.randint(0, A, B).astype(np.int64),
             ast=rs.randint(0, A, B).astype(np.int64), ret=(rs.standard_normal(B) * 3).astype(F32),
             nt=(rs.uniform(size=B) > 0.1).astype(F32))
    if A > 1:
        h["ast"][0] = (h["act"][0] + 1) % A
    if regime == "ahead":        # a_E ahead of every other action by 200 on half the rows: J = 0 there
        q = h["q_on"].reshape(N, B, A)
        q[:, np.arange(B // 2 + 1)[:B], h["act"][: B // 2 + 1]] += F32(200.0)
    return h


def _mask(kind, B):
    if kind == "null":
        return None
    return {"zero": np.zeros(B, np.uint8), "one": np.ones(B, np.uint8),
            "alternating": (np.arange(B) % 2).astype(np.uint8)}[kind]


def _dqfd_call(dev, d, demo_d, B, A, N, Np, margin, lam, eps, outs=True):
    o = {"loss": Out(B, dev), "td": Out(B, dev), "dth": Out(N * B, dev), "J": Out(B, dev) if outs else None,
         "a_hat": Out(B, dev, dtype=torch.int64, fill=-5), "theta": Out(B * N, dev) if outs else None,
         "target": Out(B * Np, dev) if outs else None}
    args = ([B, N, Np, A] + [dptr(d[k]) for k in ("q_on", "q_tg", "tau", "act", "ast", "ret", "nt")] + [dptr(demo_d)]
            + [0.99 ** 3, 1.0, float(margin), float(lam)])
    ptrs = [o[k].p if o[k] is not None else None for k in ("loss", "td", "dth", "J", "a_hat", "theta", "target")]
    if eps is None:
        lib_call("riqn_dqfd_loss_fwd_bwd", *args, *ptrs)
    else:
        lib_call("riqn_dqfd_loss_fwd_bwd_h", *args, float(eps), *ptrs)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def _plain_call(dev, d, B, A, N, Np, eps):
    o = {"loss": Out(B, dev), "dth": Out(N * B, dev), "theta": Out(B * N, dev), "target": Out(B * Np, dev)}
    args = [B, N, Np, A] + [dptr(d[k]) for k in ("q_on", "q_tg", "tau", "act", "ast", "ret", "nt")] + [0.99 ** 3, 1.0]
    ptrs = [o[k].p for k in ("loss", "dth", "theta", "target")]
    if eps is None:
        lib_call("riqn_iqn_loss_fwd_bwd", *args, *ptrs)
    else:
        lib_call("riqn_iqn_loss_fwd_bwd_h", *args, float(eps), *ptrs)
    torch.cuda.synchronize()
    return o


def _grad_call(dev, B, A, N, dth, a_hat, act, demo_d, gs, gmul, lam):
    G = Out(N * B * A, dev)
    lib_call("riqn_dqfd_dense_grad", B, N, A, dptr(dth), dptr(a_hat), dptr(act), dptr(demo_d), dptr(gs), float(gmul),
             float(lam), G.p)
    torch.cuda.synchronize()
    assert_canaries({"G": G})
    return G


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("B,A,N,Np", KERNEL_SHAPES, ids=[f"B{b}-A{a}-N{n}-Np{p}" for b, a, n, p in KERNEL_SHAPES])
def test_kernel_vs_float64(cuda_dev, B, A, N, Np, regime):
    dev = cuda_dev
    h = _kernel_inputs(B, A, N, Np, regime, B * 7 + A * 3 + N + Np + REGIMES.index(regime))
    d = {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}
    rows = np.arange(B)
    rs = np.random.RandomState(B + A)
    gs = rs.uniform(0.1, 1.0, B).astype(F32)
    gs_d = to_dev(gs, dev)
    gmul = 1.0 / B
    seen = dict(ties=0, two_col=0, same_col=0)
    for k, eps in enumerate((None, 0.0, 1e-3)):
        margin = MARGINS[(k + REGIMES.index(regime)) % 4]
        lam = LAMBDAS[(k + 2 * REGIMES.index(regime)) % 4]
        p = _plain_call(dev, d, B, A, N, Np, eps)
        Q, J, a_hat = od.margin_f32(h["q_on"], B, h["act"], margin)
        v = (Q + F32(margin)).astype(F32)
        v[rows, h["act"]] = Q[rows, h["act"]]
        last = A - 1 - np.argmax(v[:, ::-1], 1)
        seen["ties"] += int((last != a_hat).sum())
        for mk in MASKS:
            demo = _mask(mk, B)
            demo_d = None if demo is None else torch.from_numpy(demo).to(dev)
            flags = np.zeros(B, np.uint8) if demo is None else demo
            o = _dqfd_call(dev, d, demo_d, B, A, N, Np, margin, lam, eps)
            what = f"(eps {eps}, mask {mk})"
            for a, b_ in (("td", "loss"), ("dth", "dth"), ("theta", "theta"), ("target", "target")):
                assert_bits(f"{a} vs the quantile-Huber kernel {what}", o[a].bits(), p[b_].bits())
            assert np.array_equal(o["a_hat"].t[:B].cpu().numpy(), a_hat), what
            assert_bits(f"J vs its float32 statement {what}", o["J"].bits(), f32_bits(J))
            assert np.all(J >= 0) and (A > 1 or np.all(J == 0))
            td = o["td"].f32()
            want = od.loss_f32(td, J, lam, flags)
            assert_bits(f"loss vs its float32 statement {what}", o["loss"].bits(), f32_bits(want))
            if not flags.any():
                assert_bits(f"loss without flags vs the plain loss {what}", o["loss"].bits(), p["loss"].bits())
            G = _grad_call(dev, B, A, N, o["dth"].t[:N * B], o["a_hat"].t[:B], d["act"], demo_d, gs_d, gmul, lam)
            dth = o["dth"].f32()
            Gw = od.dense_grad_f32(dth, a_hat, h["act"], flags, gs, gmul, lam, N, A)
            assert_bits(f"G vs its float32 statement {what}", G.bits(), f32_bits(Gw).ravel())
            two = (flags != 0) & (a_hat != h["act"])
            seen["two_col"] += int(two.sum())
            seen["same_col"] += int(((flags != 0) & ~two).sum())
            # the value-only mutants of the statements; each would fail the checks above
            Jm = ((Q + F32(margin)).astype(F32).max(1) - Q[rows, h["act"]]).astype(F32)
            Qe = Q[rows, h["act"]]
            lead = (Qe > np.where(np.arange(A)[None, :] == h["act"][:, None], -np.inf, Q).max(1)) & \
                ((Qe + F32(margin)).astype(F32) != Qe)
            if lead.any():                  # a_E strictly ahead and the margin not absorbed by its rounding
                assert not np.array_equal(f32_bits(Jm), f32_bits(J)), "margin on a_E as well"
            if mk in ("zero", "alternating") and np.any((flags == 0) & (J > 0)):
                lm = od.loss_f32(td, J, lam, np.ones(B))
                if np.any(lm[flags == 0] != want[flags == 0]):
                    assert not np.array_equal(f32_bits(lm), f32_bits(want)), "mask ignored in the loss"
            if mk in ("zero", "alternating") and np.any((flags == 0) & (a_hat != h["act"])):
                Gm = od.dense_grad_f32(dth, a_hat, h["act"], np.ones(B), gs, gmul, lam, N, A)
                assert not np.array_equal(f32_bits(Gm), f32_bits(Gw)), "mask ignored in G"
            if N > 1 and two.any():
                Gm = od.dense_grad_f32(dth, a_hat, h["act"], flags, gs, gmul, lam * N, N, A)
                assert not np.array_equal(f32_bits(Gm), f32_bits(Gw)), "c = lambda"
            again = _dqfd_call(dev, d, demo_d, B, A, N, Np, margin, lam, eps)
            for key in o:
                assert_bits(f"second call {key}", again[key].bits(), o[key].bits())
            bare = _dqfd_call(dev, d, demo_d, B, A, N, Np, margin, lam, eps, outs=False)
            for key in ("loss", "td", "dth", "a_hat"):
                assert_bits(f"{key} without the optional outputs", bare[key].bits(), o[key].bits())
    if regime == "equal" and A >= 3:
        assert seen["ties"] > 0, "the last of equal maxima is not told apart from the first"
    print(f"B={B} A={A} N={N} N'={Np} {regime}: rows with ties {seen['ties']}, flagged rows with a_hat != a_E "
          f"{seen['two_col']}, with a_hat = a_E {seen['same_col']}")


@pytest.mark.gpu
def test_entry_points_reject_invalid_calls_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    src = torch.full((64 * 64 * 33,), 0.5, device=dev)
    idx = torch.zeros(64, dtype=torch.int64, device=dev)
    mask = torch.ones(64, dtype=torch.uint8, device=dev)
    outs = [Out(64 * 64 * 33, dev) for _ in range(7)]
    bad = [dict(B=0), dict(B=-1), dict(N=0), dict(Np=0), dict(A=0), dict(A=33), dict(kappa=0.0), dict(kappa=math.nan),
           dict(margin=0.0), dict(margin=-0.8), dict(margin=math.nan), dict(margin=math.inf), dict(lam=0.0),
           dict(lam=-1.0), dict(lam=math.nan), dict(lam=math.inf), dict(Np=12 * 1024), dict(null=0), dict(null=1),
           dict(null=2), dict(null=4)]
    for kw in bad:
        B, N, Np, A = kw.get("B", 4), kw.get("N", 8), kw.get("Np", 8), kw.get("A", 4)
        ptrs = [o.p for o in outs]
        if "null" in kw:
            ptrs[kw["null"]] = None
        args = [B, N, Np, A, dptr(src), dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src), dptr(src), dptr(mask),
                0.97, kw.get("kappa", 1.0), kw.get("margin", 0.8), kw.get("lam", 1.0)]
        for fn, extra in (("riqn_dqfd_loss_fwd_bwd", []), ("riqn_dqfd_loss_fwd_bwd_h", [1e-3])):
            with pytest.raises(RiqnError):
                lib_call(fn, *args, *extra, *ptrs)
    for eps in (-1e-3, math.nan, math.inf):
        with pytest.raises(RiqnError):
            lib_call("riqn_dqfd_loss_fwd_bwd_h", 4, 8, 8, 4, dptr(src), dptr(src), dptr(src), dptr(idx), dptr(idx),
                     dptr(src), dptr(src), dptr(mask), 0.97, 1.0, 0.8, 1.0, eps, *(o.p for o in outs))
    for kw in (dict(B=0), dict(N=0), dict(A=0), dict(A=33), dict(lam=0.0), dict(lam=math.nan), dict(lam=-2.0),
               dict(lam=math.inf), dict(null=0), dict(null=1), dict(null=2), dict(null=3)):
        p = [dptr(src), dptr(idx), dptr(idx), dptr(src)]
        if "null" in kw:
            p[kw["null"]] = None
        with pytest.raises(RiqnError):
            lib_call("riqn_dqfd_dense_grad", kw.get("B", 4), kw.get("N", 8), kw.get("A", 4), p[0], p[1], p[2],
                     dptr(mask), p[3], 1.0, kw.get("lam", 1.0), outs[0].p)
    with pytest.raises(RiqnError):
        lib_call("riqn_dqfd_dense_grad", 4, 8, 4, dptr(src), dptr(idx), dptr(idx), dptr(mask), dptr(src), 1.0, 1.0, None)
    torch.cuda.synchronize()
    for o in outs:
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ tree update (GPU)
def _tree_case(seed, cap, nb):
    rs = np.random.RandomState(seed)
    t = ost.SumTree(cap, nb)
    for a in range(nb):
        t.append_priorities(0, a, rs.uniform(0.05, 1.5, cap).astype(F32).astype(np.float64))
    return rs, t


def _tree_update(dev, tree64, idx, loss, exponent, leaf=None, bonus=None):
    tree = torch.from_numpy(tree64.copy()).to(dev)
    C = (tree64.size + 1) // 2
    n = idx.size
    idx_d = torch.from_numpy(idx.astype(np.int64)).to(dev)
    loss_d = to_dev(loss, dev)
    new = Out(n, dev)
    diff = torch.empty(n, dtype=torch.float64, device=dev)
    mx = torch.ones(1, dtype=torch.float64, device=dev)
    if leaf is None:
        lib_call("riqn_sumtree_update", n, C, dptr(tree), dptr(idx_d), dptr(loss_d), float(exponent), 1, new.p,
                 dptr(diff), dptr(mx))
    else:
        lib_call("riqn_sumtree_update_demo", n, C, dptr(tree), dptr(idx_d), dptr(loss_d), float(exponent), 1, new.p,
                 dptr(diff), dptr(mx), int(leaf), float(bonus))
    torch.cuda.synchronize()
    assert_canaries({"new": new})
    return tree.cpu().numpy(), new.f32(), float(mx.item())


@pytest.mark.gpu
@pytest.mark.parametrize("cap,nb,n,D", [(64, 4, 48, 1), (1000, 3, 512, 2), (2500, 4, 4096, 1), (7, 3, 30, 2)])
def test_tree_update_vs_oracle(cuda_dev, cap, nb, n, D):
    """riqn_sumtree_update_demo against the numpy tree: duplicates, leaves on both sides of demo_leaf, max_priority; at
    eps_d = 0 it is riqn_sumtree_update bit for bit."""
    rs, base = _tree_case(cap * 3 + nb + n, cap, nb)
    C = base.full_capacity
    leaf = (nb - D) * cap + C - 1
    idx = rs.randint(C - 1, 2 * C - 1, n)
    idx[: n // 4] = idx[n // 4: 2 * (n // 4)]                        # duplicates
    idx[-1], idx[-2], idx[-3] = leaf, leaf - 1, 2 * C - 2            # both sides of demo_leaf
    assert np.any(idx >= leaf) and np.any(idx < leaf)
    loss = rs.uniform(0.01, 3.0, n).astype(F32)
    loss[0] = F32(40.0)                                              # raises max_priority
    for omega in (0.2, 0.5):
        tp, newp, mxp = _tree_update(cuda_dev, base.tree, idx, loss, omega)
        t0, new0, mx0 = _tree_update(cuda_dev, base.tree, idx, loss, omega, leaf, 0.0)
        assert np.array_equal(tp, t0) and np.array_equal(f32_bits(newp), f32_bits(new0)) and mxp == mx0
        for bonus in (1e-3, 0.25, 7.0):
            t1, new1, mx1 = _tree_update(cuda_dev, base.tree, idx, loss, omega, leaf, bonus)
            on = idx >= leaf
            want = np.where(on, (newp + F32(bonus)).astype(F32), newp)
            assert_bits(f"priorities at eps_d {bonus}", f32_bits(new1), f32_bits(want))
            o = ost.SumTree(cap, nb)
            o.tree = base.tree.copy()
            o.update_multiple_value(idx, want.astype(np.float64))
            assert np.array_equal(t1.view(np.uint64), o.tree.view(np.uint64)), "tree vs the numpy tree"
            assert mx1 == max(1.0, float(np.float64(want.max())))
            again = _tree_update(cuda_dev, base.tree, idx, loss, omega, leaf, bonus)
            assert np.array_equal(again[0], t1) and np.array_equal(again[1], new1)
            # the value-only mutants: the bonus below demo_leaf too, the bonus before the power
            everywhere = (newp + F32(bonus)).astype(F32)
            assert not np.array_equal(f32_bits(everywhere), f32_bits(want)), "bonus below demo_leaf"
            before = np.where(on, np.power((loss + F32(bonus)).astype(F32).astype(np.float64), omega).astype(F32), newp)
            assert not np.array_equal(f32_bits(before), f32_bits(want)), "bonus before the power"


@pytest.mark.gpu
def test_tree_update_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    _, base = _tree_case(5, 64, 2)
    tree = torch.from_numpy(base.tree.copy()).to(cuda_dev)
    idx = torch.arange(100, 110, device=cuda_dev)
    loss = torch.full((10,), 0.5, device=cuda_dev)
    new = Out(10, cuda_dev)
    diff = torch.empty(10, dtype=torch.float64, device=cuda_dev)
    mx = torch.ones(1, dtype=torch.float64, device=cuda_dev)
    for leaf, bonus in ((100, -1e-3), (100, math.nan), (100, math.inf), (100, -math.inf), (-1, 0.1)):
        with pytest.raises(RiqnError):
            lib_call("riqn_sumtree_update_demo", 10, 128, dptr(tree), dptr(idx), dptr(loss), 0.5, 1, new.p, dptr(diff),
                     dptr(mx), leaf, bonus)
    torch.cuda.synchronize()
    assert np.array_equal(tree.cpu().numpy(), base.tree) and bool(torch.isnan(new.t[:10]).all()) and new.canaries_ok()
    assert float(mx.item()) == 1.0


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def _args(dev, B, kind, N, **kw):
    a = make_args(dev, B, cases.iqn_cfg(N, N, 32))
    if kind == "qr":
        a.qr_dqn = 1
    elif kind == "cvar":
        a.risk_measure, a.risk_eta = "cvar", 0.25
    a.dqfd = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _dqfd_learner(dev, B, kind, N, params, **kw):
    from rainbow_iqn_apex_b200 import Learner
    lr = Learner(_args(dev, B, kind, N, **kw), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    return lr


def _flips(dbg, keep, B, kind):
    gk = dbg["keep"]
    h = gk["h"]
    if kind != "qr":
        from test_gpu_learn import _qmajor
        h = _qmajor(h, B)
    h = h.cpu()
    pairs = [(gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
             (h[:, :512], keep["h_v"]), (h[:, 512:], keep["h_a"])]
    return [int(((x.cpu() > 0) != (y > 0)).sum()) for x, y in pairs]


STEP_CASES = [(k, B, N) for k in ("iqn", "cvar", "qr") for B, N in ((32, 64), (512, 64), (32, 200))]


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("kind,B,N", STEP_CASES)
def test_learner_step_vs_oracle(cuda_dev, kind, B, N, eps):
    """Learner.compute_gradients with half the rows flagged, under injected noises (and fractions), against the torch-fp32
    DQfD step: loss within 1e-3 relative and every gradient at cosine >= 0.999, 0.98 upstream of a flipped ReLU or a
    near-tie a_hat or a*."""
    from test_gpu_learn import _dev_batch
    cfg, seed, l, lam = cases.iqn_cfg(N, N, 32), 16100 + B + N + len(kind), 0.8, 2.0
    kw = dict(dqfd_lambda=lam)
    if eps is not None:
        kw.update(value_rescaling=1, value_rescaling_eps=eps)
    params = oq.make_params(seed, 18, N) if kind == "qr" else net.make_params(seed)
    torch.manual_seed(seed)
    lr = _dqfd_learner(cuda_dev, B, kind, N, params, **kw)
    assert lr.dqfd == (float(F32(l)), lam) and lr.value_rescaling == eps
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    if eps is not None:
        b["returns"] = (b["returns"] * 40).astype(F32)
    taus = None
    if kind == "qr":
        noises = oq.make_noises(seed + 3, 18, N)
        lr._inject = dict(noises=noises)
    else:
        noises = cases.make_noises(seed + 3)
        t_sel, t_tgt, t_on = (torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg))
        lr._inject = dict(noises=noises, taus=(None if kind == "cvar" else t_sel, t_tgt, t_on))
    demo = (np.arange(B) % 2).astype(np.uint8)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg, demo=torch.from_numpy(demo).to(cuda_dev))
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    _, J32, ah32 = od.margin_f32(dbg["q_on"].cpu().numpy(), B, b["actions"], lr.dqfd[0])
    assert_bits("J", f32_bits(dbg["margin"].cpu().numpy()), f32_bits(J32))
    assert np.array_equal(dbg["a_hat"].cpu().numpy(), ah32)
    assert_bits("loss", f32_bits(loss.detach().cpu().numpy()),
                f32_bits(od.loss_f32(dbg["td_loss"].cpu().numpy(), J32, lam, demo)))
    if kind != "qr":
        taus = (dbg["tau_sel"].cpu(), t_tgt, t_on)
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_grads = od.learn_step("qr" if kind == "qr" else "iqn", p_on, p_tg, cases.batch_to_torch(b),
                                    torch.from_numpy(b["weights"]), noises, taus, cfg, l, lam, demo, eps, keep=keep)
    qv = keep["qv_next"].numpy()
    top2 = np.sort(qv, axis=1)[:, -2:]
    tie = (top2[:, 1] - top2[:, 0]) < (1e-4 if eps is None else 1e-3)
    ok = dbg["a_star"].cpu().numpy() == keep["a_star"].numpy()
    assert np.all(ok | tie)
    # a near-tie of the margin's maximum: a_hat may differ from the oracle's, J does not by more than the tie
    Qo = keep["q_on"].detach().reshape(N, B, -1).mean(0).numpy().astype(np.float64)
    vo = Qo + l
    vo[np.arange(B), b["actions"]] -= l
    t2 = np.sort(vo, 1)[:, -2:]
    near = (t2[:, 1] - t2[:, 0]) < 1e-4
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    err = np.abs(lg - lo) / np.abs(lo)
    assert np.max(err[ok]) < 1e-3, float(np.max(err[ok]))
    fl = _flips(dbg, keep, B, kind)
    relaxed = set()
    if fl[3] + fl[4] or not ok.all() or np.any(near & (demo != 0)):
        relaxed |= {"conv1", "conv2", "conv3", "iqn_fc", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    worst = 1.0
    for k, g_ref in o_grads.items():
        c = _cos(grads[k], g_ref)
        worst = min(worst, c)
        assert c > (0.98 if k.split(".")[0] in relaxed else 0.999), (k, c, fl)
    print(f"{kind} B={B} N={N} eps={eps}: max loss rel err {np.max(err[ok]):.3g}, min cos {worst:.6f}, flips {fl}, "
          f"ties {int((~ok).sum())}, margin near-ties {int(near.sum())}, mean J {float(dbg['margin'].mean()):.4g}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "qr"])
def test_autograd_through_the_loss_node_equals_compute_gradients(cuda_dev, kind):
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    params = oq.make_params(77, 18, N) if kind == "qr" else net.make_params(77)
    b = cases.make_batch(78, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    demo = torch.from_numpy((np.arange(B) % 3 == 0)).to(cuda_dev)          # bool flags
    if kind == "qr":
        inj = dict(noises=oq.make_noises(80, 18, N))
    else:
        inj = dict(noises=cases.make_noises(80),
                   taus=tuple(torch.from_numpy(t) for t in cases.make_taus(81, B, cases.iqn_cfg(N, N, 32))))
    out = []
    for mode in ("learner", "autograd"):
        torch.manual_seed(79)
        lr = _dqfd_learner(cuda_dev, B, kind, N, params)
        lr._inject = dict(inj)
        if mode == "learner":
            loss = lr.compute_gradients(st, ac, rt, nx, nt, w, demo=demo)
        else:
            lr.online_net.zero_grad()
            loss = lr.compute_loss_actor_or_learner(st, ac, rt, nx, nt, demo=demo)
            (w * loss).mean().backward()
        torch.cuda.synchronize()
        out.append((loss.detach().clone(), lr.online_net._flat_grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def _demo_args(dev, fields, cap=1 << 14, nb=4):
    import bench
    a = bench.make_args(dev, cap)
    a.nb_actor, a.actor_capacity = nb, cap // nb
    a.demo_segments, a.demo_priority_bonus = 1, 1e-3
    for k, v in fields.items():
        setattr(a, k, v)
    return a


def _demo_run(dev, kind, fields, steps=2, seed=5, count=False):
    """Steps of a bench-sized learner (B = 512) whose replay holds four segments, the last of them demonstrations, eagerly
    ("eager") or replayed from the replay or batch graph; returns per-step (idxs, loss, library launches, kernels) and the
    final parameters."""
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib
    torch.manual_seed(seed)
    a = _demo_args(dev, fields)
    lr = Learner(a, bench.ACTIONS, None)
    lr.train()
    mem = ReplayMemory(a, None)
    bench.fill_replay_segments(mem, dev, 7)
    out = []
    if kind == "batch":
        lr.enable_cuda_graph(mem)
        lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(a.batch_size)))
    elif kind == "replay":
        lr.enable_cuda_graph(mem)
    for _ in range(steps):
        c0, kernels = _lib.launch_count(), None
        if kind == "batch":
            h = tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(a.batch_size))
            idxs, loss = h[0], lr.learn_on_host_batch(h)
        elif count:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                idxs, loss = lr.learn_and_update(mem)
                torch.cuda.synchronize()
            kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                          and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
        else:
            idxs, loss = lr.learn_and_update(mem)
        out.append((torch.as_tensor(idxs).clone(), loss.clone(), _lib.launch_count() - c0, kernels))
    torch.cuda.synchronize()
    return out, lr.online_net._flat.detach().clone(), lr, mem


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eager", "replay", "batch"])
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_steps_are_bitwise_reproducible(cuda_dev, kind, head):
    """Two consecutive B = 512 steps on a replay with demonstrations, eagerly and from the replay and batch graphs,
    twice alike; some rows of every step are demonstrations and some are not."""
    fields = dict(dqfd=1, **(dict(qr_dqn=1) if head == "qr" else {}))
    (o1, p1, lr, mem), (o2, p2, _, _) = _demo_run(cuda_dev, kind, fields), _demo_run(cuda_dev, kind, fields)
    for (i1, l1, _, _), (i2, l2, _, _) in zip(o1, o2):
        assert torch.equal(i1, i2) and torch.equal(l1, l2) and bool(torch.isfinite(l1).all()) and bool((l1 >= 0).all())
        flags = mem.demo_mask(i1)
        assert 0 < int(flags.sum()) < flags.numel()
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_learn_graph_refuses_dqfd(cuda_dev):
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_qr import _graph_batch
    lr = Learner(_args(cuda_dev, 32, "iqn", 64), 18, None)
    with pytest.raises(RuntimeError):
        lr.enable_learn_graph(_graph_batch(cuda_dev, 32, 4))
    assert not lr._graphs


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_dqfd_step_makes_two_more_launches_than_its_plain_twin(cuda_dev, head):
    """On the same replay with demonstrations, the eager DQfD step launches two more kernels than the plain one: the
    mask (a torch comparison) and the dense gradient (a library launch).  The profiler's kernel counts are compared from
    the second step on: its first window can miss the first kernels it traces."""
    base = dict(qr_dqn=1) if head == "qr" else {}
    (s1, p1, _, _), (s2, _, _, _) = (_demo_run(cuda_dev, "eager", f, steps=3, count=True)
                                     for f in (base, dict(base, dqfd=1)))
    lib1, lib2 = [c for _, _, c, _ in s1], [c for _, _, c, _ in s2]
    k1, k2 = [k for _, _, _, k in s1], [k for _, _, _, k in s2]
    print(f"{head}: eager library launches per step, plain {lib1}, DQfD {lib2}; kernels plain {k1}, DQfD {k2}")
    assert {b - a for a, b in zip(lib1, lib2)} == {1}
    assert {b - a for a, b in zip(k1[1:], k2[1:])} == {2}
    assert torch.equal(s1[0][0], s2[0][0])          # the same sampled rows


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_replay_of_demonstrations_flags_every_row(cuda_dev, head):
    """A replay whose only filled segment is its demonstration segment: every sampled row is flagged, with and without
    random shifts, and the step's loss is td + lambda * J on every row."""
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    B, cap, nb = 32, 1000, 4
    for shift in (0, 4):
        a = _args(cuda_dev, B, head, 64, actor_capacity=cap, nb_actor=nb, demo_segments=1, demo_priority_bonus=1e-2,
                  random_shift=shift, dqfd_lambda=3.0)
        torch.manual_seed(3)
        lr = Learner(a, 18, None)
        lr.train()
        mem = ReplayMemory(a, None)
        assert mem.demo_leaf == (nb - 1) * cap + nb * cap - 1
        rs = np.random.RandomState(4)
        ts = np.arange(cap) % 250
        mem.transitions.append_arrays(nb - 1, 0, ts, rs.randint(0, 256, (cap, 84, 84)).astype(np.uint8),
                                      rs.randint(0, 18, cap), rs.randint(-1, 2, cap).astype(np.float32), ts == 249,
                                      np.ones(cap, np.float32))
        for _ in range(3):
            idxs, st, ac, rt, nx, nt, w = mem.sample(B)
            flags = mem.demo_mask(idxs)
            assert flags.dtype == torch.uint8 and bool((flags == 1).all())
            dbg = {}
            loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg, demo=flags)
            want = od.loss_f32(dbg["td_loss"].cpu().numpy(), dbg["margin"].cpu().numpy(), 3.0, np.ones(B))
            assert_bits("loss", f32_bits(loss.cpu().numpy()), f32_bits(want))
            idxs, loss = lr.learn(mem, None)
            new = mem.update_priorities(idxs, loss)
            plain = np.power(loss.detach().cpu().numpy().astype(np.float64), np.float64(F32(0.2))).astype(F32)
            assert np.all(new.cpu().numpy() >= plain)          # every leaf got the bonus
        assert mem.transitions.check_sumtree_correct() < 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "qr"])
def test_data_parallel_half_batches_equal_one_learner(cuda_dev, kind):
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    cfg = cases.iqn_cfg(N, N, 32)
    b = cases.make_batch(12, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    demo = torch.from_numpy((np.arange(B) % 2).astype(np.uint8)).to(cuda_dev)
    params = oq.make_params(12, 18, N) if kind == "qr" else net.make_params(12)
    noises = oq.make_noises(13, 18, N) if kind == "qr" else cases.make_noises(13)
    taus = [torch.from_numpy(t) for t in cases.make_taus(14, B, cfg)]

    def grads_of(sl, scale):
        torch.manual_seed(1)
        lr = _dqfd_learner(cuda_dev, sl.stop - sl.start, kind, N, params)
        inj = dict(noises=noises)
        if kind != "qr":
            inj["taus"] = tuple(t.view(-1, B)[:, sl].reshape(-1, 1).contiguous() for t in taus)
        lr._inject = inj
        lr.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl] * scale, demo=demo[sl])
        torch.cuda.synchronize()
        return lr.online_net._flat_grad.clone()

    full = grads_of(slice(0, B), 1.0)
    halves = grads_of(slice(0, B // 2), 0.5) + grads_of(slice(B // 2, B), 0.5)
    err = float((halves - full).abs().max() / full.abs().max())
    c = _cos(halves, full)
    print(f"{kind} data parallel: max |sum of half-batch grads - full| / max |full| = {err:.3g}, cos {c:.8f}")
    assert err < 2e-3 and c > 0.99999


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_without_a_mask_the_dqfd_agent_is_the_plain_agent(cuda_dev, head):
    """A DQfD learner given no mask, its actors' values and actions, and compute_priorities: bit for bit the plain
    agent's."""
    from rainbow_iqn_apex_b200 import Actor
    from test_gpu_learn import _dev_batch
    B, N, seed = 32, 32, 16300
    cfg = cases.iqn_cfg(N, N, 8)
    params = oq.make_params(seed, 18, N) if head == "qr" else net.make_params(seed)
    b = cases.make_batch(seed + 1, B)
    batch = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    res = []
    for on in (1, 0):
        lr = _dqfd_learner(cuda_dev, B, head, N, params, dqfd=on, num_quantile_samples=8)
        if head == "qr":
            lr._inject = dict(noises=oq.make_noises(seed + 3, 18, N))
        else:
            lr._inject = dict(noises=cases.make_noises(seed + 3),
                              taus=tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg)))
        loss = lr.compute_gradients(*batch, w)
        torch.cuda.synchronize()
        res.append((loss.clone(), lr.online_net._flat_grad.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    actors = []
    for on in (1, 0):
        torch.manual_seed(seed)
        a = Actor(_args(cuda_dev, 8, head, N, dqfd=on, num_quantile_samples=8), 18, None)
        load_params(a.online_net, params)
        a.update_target_net()
        actors.append(a)
    dq, plain = actors
    assert dq.dqfd is not None and plain.dqfd is None
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (8, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    vals = []
    for a in actors:
        a.eval()
        torch.manual_seed(1)
        vals.append(a.act_batch_values(su8))
    assert torch.equal(vals[0], vals[1])
    L, hist = 14, 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    pri = []
    for a in actors:
        a.train()
        torch.manual_seed(2)
        pri.append(a.compute_priorities(tab_state, tab_action, tab_reward, [1.0] * L, 0.2))
    assert np.array_equal(pri[0], pri[1]) and np.all(np.isfinite(pri[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("base", [{}, dict(rainbow_only=1), dict(qr_dqn=1)])
def test_namespace_without_the_fields_is_unchanged(cuda_dev, base):
    """IQN, C51 and QR-DQN learners from a namespace without the DQfD and demonstration fields, with them at 0, and with
    demonstration segments but no bonus and dqfd = 0, run the same launches per step and give bit-identical sampled
    indices, losses and parameters."""
    from test_gpu_qr import _bench_learner
    variants = (base, dict(base, dqfd=0, dqfd_margin=0.5, dqfd_lambda=3.0, demo_segments=0, demo_priority_bonus=0.0),
                dict(base, demo_segments=1, demo_priority_bonus=0.0))
    runs = [_bench_learner(cuda_dev, 1 << 14, False, 2, f) for f in variants]
    (s1, p1, l1, m1) = runs[0]
    assert l1.dqfd is None and m1.demo_leaf is None and m1.demo_segments == 0
    assert runs[2][3].demo_leaf == (1 << 14) - 1 + 0
    for s2, p2, l2, _ in runs[1:]:
        assert l2.dqfd is None
        for k, ((i1, x1, c1), (i2, x2, c2)) in enumerate(zip(s1, s2)):
            assert torch.equal(i1, i2) and torch.equal(x1, x2), k
            assert c1 == c2, (k, c1, c2)
        assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner, ReplayMemory
    B = 32
    for kind, kw in (("iqn", dict(dqfd=2)), ("iqn", dict(dqfd="1")), ("iqn", dict(dqfd_margin=0.0)),
                     ("iqn", dict(dqfd_margin=-1.0)), ("iqn", dict(dqfd_lambda=math.nan)),
                     ("iqn", dict(dqfd_lambda=math.inf)), ("iqn", dict(dqfd_margin="1")), ("iqn", dict(rainbow_only=1)),
                     ("iqn", dict(rainbow_only=1, hl_gauss=1)), ("iqn", dict(munchausen=1)), ("iqn", dict(fqf=1)),
                     ("qr", dict(mmd=1)), ("iqn", dict(cql=1)), ("qr", dict(cql=1))):
        with pytest.raises(ValueError):
            Agent(_args(cuda_dev, B, kind, 64, **kw), 18, None)
    for kw in (dict(demo_segments=-1), dict(demo_segments=3), dict(demo_segments=1.0), dict(demo_priority_bonus=-1.0),
               dict(demo_priority_bonus=math.nan), dict(demo_priority_bonus=True)):
        with pytest.raises(ValueError):
            ReplayMemory(_args(cuda_dev, B, "iqn", 64, nb_actor=2, actor_capacity=100, **kw), None)
    ag = Learner(_args(cuda_dev, B, "cvar", 64, value_rescaling=1, random_shift=4, dqfd_margin=np.float32(0.5)), 18, None)
    assert ag.dqfd == (0.5, 1.0) and ag.value_rescaling == 1e-3 and ag.random_shift == 4 and ag.risk is not None
    ag.set_risk("wang", 0.5)
    plain = Learner(_args(cuda_dev, B, "iqn", 64, dqfd=0), 18, None)
    c51 = Learner(_args(cuda_dev, B, "iqn", 64, dqfd=0, rainbow_only=1), 18, None)
    from test_gpu_qr import _graph_batch
    st, ac, rt, nx, nt, w = _graph_batch(cuda_dev, B, 4)
    mask = torch.ones(B, dtype=torch.uint8, device=cuda_dev)
    for lr in (plain, c51):                               # a mask needs a DQfD learner
        with pytest.raises(ValueError):
            lr.compute_gradients(st, ac, rt, nx, nt, w, demo=mask)
    for bad in (torch.ones(B + 1, dtype=torch.uint8, device=cuda_dev), torch.ones(B, device=cuda_dev)):
        with pytest.raises(ValueError):
            ag.compute_gradients(st, ac, rt, nx, nt, w, demo=bad)
