"""CQL (Kumar, Zhou, Tucker & Levine, NeurIPS 2020): the quantile-Huber loss plus alpha times the log-sum-exp gap of the
online pass (riqn_cql_loss_fwd_bwd, riqn_cql_loss_fwd_bwd_h) and its dense upstream gradient (riqn_cql_dense_grad),
behind the optional Agent fields cql and cql_alpha, for the IQN and QR-DQN learners.

The unmarked tests pin the float64 statement (oracle/cql.py) by identities, against float64 autograd and central
differences, check the torch-fp32 step against it and check the host-side validation.  The gpu tests hold the entry points
to float64 with the method of test_gpu_iqn_kernels.py (NaN prefills, canaries, two calls alike, rejected calls write
nothing): td_loss, dtheta, theta_out and target_out bit for bit those of riqn_iqn_loss_fwd_bwd[_h]; pi and gap within one
float ulp of the float64 statement on the kernel's float32 means; loss and G bit for bit against their numpy float32
statements on the kernel's own intermediates.  Value-only mutants of those statements, each of which the kernel cases
reject (test_kernel_vs_float64 asserts it): the mean over N - 1 and the gap taken at a* (every case with N > 1, resp.
any N, and A > 1 outside the nearly-equal regime; row 0 has a* != a_t), c = alpha instead of alpha / N (every case with
N > 1 and A > 1), the - c on a_t dropped (every case), w read at row i instead of b (every case with N > 1 and B > 1).
These are checked as numpy statements against the kernel's outputs, not as rebuilt libraries.  At the learner level: the step
against the torch oracle, autograd, reproducibility eagerly and from each captured graph, data parallelism, augmentation,
the actors and priorities, launch counts, checkpoints, configuration errors, the offline recipe, and that a namespace
without the field runs exactly as before."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, assert_canaries, dptr, f32_bits, lib_call, load_params, make_args, rel_err, to_dev
from oracle import cases, cql as oc, network as net, qr as oq

F32 = np.float32
ALPHAS = [2.0 ** -10, 1.0, 4.0, 100.0]


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def _q(rs, N, B, A, scale=1.0):
    return rs.standard_normal((N * B, A)) * scale


def test_gap_identities():
    rs = np.random.RandomState(1)
    for N, B, A in ((1, 5, 1), (8, 16, 4), (64, 32, 18), (3, 7, 32)):
        q = _q(rs, N, B, A, 3.0)
        act = rs.randint(0, A, B)
        gap, pi = oc.gap_np(q, B, act)
        assert np.all(gap >= 0) and np.allclose(pi.sum(1), 1.0, rtol=0, atol=1e-15)
        # equal Q: the gap is ln A
        flat = np.tile(rs.standard_normal((1, B, 1)), (N, 1, A)).reshape(N * B, A)
        assert np.max(np.abs(oc.gap_np(flat, B, act)[0] - math.log(A))) <= 1e-15
        # the action taken ahead of every other by 50: the gap vanishes
        ahead = q.copy().reshape(N, B, A)
        ahead[:, np.arange(B), act] += 50.0 + 2 * np.abs(q).max()
        if A > 1:
            assert np.max(oc.gap_np(ahead.reshape(N * B, A), B, act)[0]) < 1e-20
        # a constant on every quantile of every action changes neither the gap nor its gradient
        for c in (-7.5, 1e3):
            assert np.max(np.abs(oc.gap_np(q + c, B, act)[0] - gap)) <= 1e-11
            assert np.max(np.abs(oc.gap_grad_np(q + c, B, act) - oc.gap_grad_np(q, B, act))) <= 1e-13
        # the gradient sums to zero per transition
        d = oc.gap_grad_np(q, B, act).reshape(N, B, A)
        assert np.max(np.abs(d.sum((0, 2)))) <= 1e-15


def test_gap_gradient_vs_autograd_and_differences():
    rs = np.random.RandomState(2)
    for N, B, A in ((1, 3, 2), (8, 4, 18), (64, 2, 32)):
        q = _q(rs, N, B, A, 2.0)
        act = rs.randint(0, A, B)
        qt = torch.tensor(q, dtype=torch.float64, requires_grad=True)
        oc.gap_torch(qt, N, B, torch.from_numpy(act)).sum().backward()
        d = oc.gap_grad_np(q, B, act)
        assert np.max(np.abs(d - qt.grad.numpy())) <= 1e-12
        h = 1e-6
        for r, a in zip(rs.randint(0, N * B, 12), rs.randint(0, A, 12)):
            qp, qm = q.copy(), q.copy()
            qp[r, a] += h
            qm[r, a] -= h
            num = (oc.gap_np(qp, B, act)[0] - oc.gap_np(qm, B, act)[0]) / (2 * h)
            assert abs(num[r % B] - d[r, a]) <= 1e-6


@pytest.mark.parametrize("kind,eps", [("iqn", None), ("iqn", 1e-3), ("qr", None), ("qr", 1e-3)])
def test_float64_and_torch_fp32_statements_agree(kind, eps):
    B, N, A, alpha = 4, 8, 6, 4.0
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
    keep = {}
    loss = oc.cql_loss(kind, net.to_torch(params, requires_grad=True), net.to_torch(params), (st, ac, rt, nx, nt), noises,
                       taus, cfg, alpha, eps, keep)
    gap64, _ = oc.gap_np(keep["q_on"].detach().numpy(), B, b["actions"])
    assert np.all(gap64 >= 0)
    l64 = keep["td"].numpy().astype(np.float64) + alpha * gap64
    assert np.max(np.abs(loss.detach().numpy() - l64) / np.abs(l64)) < 1e-6


# ------------------------------------------------------------------------------------------------ kernels (GPU)
# (B, A, N, N'): N, N' from 1 up to the IQN kernel tests' (1500, 64) and (64, 2000)
KERNEL_SHAPES = [(1, 1, 1, 1), (7, 4, 8, 5), (32, 18, 64, 64), (512, 18, 64, 64), (4096, 4, 32, 32), (32, 32, 200, 200),
                 (7, 32, 1500, 64), (32, 1, 64, 2000), (512, 32, 64, 2000)]
REGIMES = ["gauss", "equal", "ahead", "large"]


def _kernel_inputs(B, A, N, Np, regime, seed):
    rs = np.random.RandomState(seed)
    q_on = rs.standard_normal((N * B, A))
    if regime == "equal":                                    # all Q within a few ulp of each other
        q_on = np.tile(rs.standard_normal((N * B, 1)), (1, A)) + rs.standard_normal((N * B, A)) * 1e-6
    elif regime == "large":
        q_on = q_on * 1e4
    h = dict(q_on=q_on.astype(F32), q_tg=rs.standard_normal((Np * B, A)).astype(F32),
             tau=rs.uniform(0, 1, N * B).astype(F32), act=rs.randint(0, A, B).astype(np.int64),
             ast=rs.randint(0, A, B).astype(np.int64), ret=(rs.standard_normal(B) * 3).astype(F32),
             nt=(rs.uniform(size=B) > 0.1).astype(F32))
    if A > 1:
        h["ast"][0] = (h["act"][0] + 1) % A                 # a* differs from the action taken
    if regime == "ahead":                                    # one action ahead by >= 100: the others' pi underflow
        lead = rs.randint(0, A, B)
        lead[: B // 2] = h["act"][: B // 2]
        q = h["q_on"].reshape(N, B, A)
        q[:, np.arange(B), lead] += F32(200.0)
    return h


def _cql_call(dev, d, B, A, N, Np, alpha, eps, outs=True):
    o = {"loss": Out(B, dev), "td": Out(B, dev), "pi": Out(B * A, dev), "dth": Out(N * B, dev),
         "gap": Out(B, dev) if outs else None, "theta": Out(B * N, dev) if outs else None,
         "target": Out(B * Np, dev) if outs else None}
    args = [B, N, Np, A] + [dptr(d[k]) for k in ("q_on", "q_tg", "tau", "act", "ast", "ret", "nt")] + [0.99 ** 3, 1.0,
                                                                                                        float(alpha)]
    ptrs = [o[k].p if o[k] is not None else None for k in ("loss", "td", "pi", "dth", "gap", "theta", "target")]
    if eps is None:
        lib_call("riqn_cql_loss_fwd_bwd", *args, *ptrs)
    else:
        lib_call("riqn_cql_loss_fwd_bwd_h", *args, float(eps), *ptrs)
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


def _grad_call(dev, B, A, N, dth, pi, act, gs, gmul, alpha):
    G = Out(N * B * A, dev)
    lib_call("riqn_cql_dense_grad", B, N, A, dptr(dth), dptr(pi), dptr(act), dptr(gs), float(gmul), float(alpha), G.p)
    torch.cuda.synchronize()
    assert_canaries({"G": G})
    return G


def _ulps(a, b):
    return np.abs(f32_bits(a).astype(np.int64) - f32_bits(b).astype(np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("B,A,N,Np", KERNEL_SHAPES, ids=[f"B{b}-A{a}-N{n}-Np{p}" for b, a, n, p in KERNEL_SHAPES])
def test_kernel_vs_float64(cuda_dev, B, A, N, Np, regime):
    dev = cuda_dev
    h = _kernel_inputs(B, A, N, Np, regime, B * 7 + A * 3 + N + Np + REGIMES.index(regime))
    d = {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}
    rows = np.arange(B)
    Q = oc.means_f32(h["q_on"], B)
    gap64, pi64, _ = oc.gap_from_means_np(Q, h["act"])
    rs = np.random.RandomState(B + A)
    gs = rs.uniform(0.1, 1.0, B).astype(F32)
    gs_d = to_dev(gs, dev)
    exact = [0, 0, 0]
    for k, eps in enumerate((None, 0.0, 1e-3)):
        alpha = ALPHAS[(k + REGIMES.index(regime)) % 4]
        o = _cql_call(dev, d, B, A, N, Np, alpha, eps)
        p = _plain_call(dev, d, B, A, N, Np, eps)
        for a, b_ in (("td", "loss"), ("dth", "dth"), ("theta", "theta"), ("target", "target")):
            assert_bits(f"{a} vs the quantile-Huber kernel (eps {eps})", o[a].bits(), p[b_].bits())
        pi, gap = o["pi"].f32().reshape(B, A), o["gap"].f32()
        up, ug = _ulps(pi, pi64.astype(F32)), _ulps(gap, gap64.astype(F32))
        assert np.max(up) <= 1 and np.max(ug) <= 1, (int(np.max(up)), int(np.max(ug)))
        exact[0] += int((up == 0).sum()) + int((ug == 0).sum())
        exact[1] += up.size + ug.size
        assert np.all(gap >= 0) and np.all(o["loss"].f32() >= 0)
        td = o["td"].f32()
        assert_bits("loss vs its float32 statement", o["loss"].bits(), f32_bits(oc.loss_f32(td, gap, alpha)))
        if A == 1:
            assert_bits("loss at A = 1 vs the plain loss", o["loss"].bits(), p["loss"].bits())
        gmul = 1.0 / B
        G = _grad_call(dev, B, A, N, o["dth"].t[:N * B], o["pi"].t[:B * A], d["act"], gs_d, gmul, alpha)
        dth = o["dth"].f32()
        want = oc.dense_grad_f32(dth, pi, h["act"], gs, gmul, alpha, N)
        assert_bits("G vs its float32 statement", G.bits(), f32_bits(want).ravel())
        if A == 1:       # no off-action part: G is the one-hot gradient w_b * dtheta
            assert np.array_equal(G.f32(), (np.tile((gs * F32(gmul)).astype(F32), N) * dth).astype(F32))
        # the value-only mutants of the statements; each would fail the checks above
        if N > 1 and A > 1 and regime != "equal":
            Qm = (oc.means_f32(h["q_on"], B) * F32(N) / F32(N - 1)).astype(F32)
            assert np.any(_ulps(gap, oc.gap_from_means_np(Qm, h["act"])[0].astype(F32)) > 1), "mean over N - 1"
        if A > 1 and regime != "equal":
            assert np.any(_ulps(gap, oc.gap_from_means_np(Q, h["ast"])[0].astype(F32)) > 1), "gap at a*"
        mutants = {"- c dropped": _g_mutant(dth, pi, h["act"], gs, gmul, alpha, N, drop_c=True)}
        if N > 1:
            if A > 1:    # at A = 1, pi = 1 and g - c = 0 whatever c is
                mutants["c = alpha"] = _g_mutant(dth, pi, h["act"], gs, gmul, alpha * N, N)
            if B > 1:
                mutants["w at row i"] = _g_mutant(dth, pi, h["act"], gs, gmul, alpha, N, w_row=True)
        for what, Gm in mutants.items():
            assert not np.array_equal(f32_bits(want), f32_bits(Gm)), what
        again = _cql_call(dev, d, B, A, N, Np, alpha, eps)
        for key in o:
            assert_bits(f"second call {key}", again[key].bits(), o[key].bits())
        bare = _cql_call(dev, d, B, A, N, Np, alpha, eps, outs=False)
        for key in ("loss", "td", "pi", "dth"):
            assert_bits(f"{key} without the optional outputs", bare[key].bits(), o[key].bits())
    print(f"B={B} A={A} N={N} N'={Np} {regime}: pi and gap exact {exact[0]} of {exact[1]}")


def _g_mutant(dth, pi, act, gs, gmul, alpha, N, drop_c=False, w_row=False):
    """oc.dense_grad_f32 (alpha * N as ``alpha``: c = alpha) with the - c on the action taken dropped (``drop_c``) or
    w read at quantile row i instead of transition b (``w_row``)."""
    B, A = pi.shape
    c = (F32(alpha) / F32(N)).astype(F32)
    g = (c * pi).astype(F32)
    rows = np.arange(N * B)
    at = np.tile(act, N)
    X = np.tile(g, (N, 1))
    X[rows, at] = (dth + (g[rows % B, at] if drop_c else (g[rows % B, at] - c).astype(F32))).astype(F32)
    w = (gs * F32(gmul)).astype(F32)
    wr = w[np.minimum(rows // B, B - 1)] if w_row else w[rows % B]
    return (wr[:, None] * X).astype(F32)


@pytest.mark.gpu
def test_entry_points_reject_invalid_calls_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    src = torch.full((64 * 64 * 33,), 0.5, device=dev)
    idx = torch.zeros(64, dtype=torch.int64, device=dev)
    outs = [Out(64 * 64 * 33, dev) for _ in range(7)]
    bad = [dict(B=0), dict(B=-1), dict(N=0), dict(Np=0), dict(A=0), dict(A=33), dict(kappa=0.0), dict(kappa=math.nan),
           dict(alpha=0.0), dict(alpha=-1.0), dict(alpha=math.nan), dict(alpha=math.inf), dict(Np=12 * 1024),
           dict(null=0), dict(null=1), dict(null=2), dict(null=3)]
    for kw in bad:
        B, N, Np, A = kw.get("B", 4), kw.get("N", 8), kw.get("Np", 8), kw.get("A", 4)
        ptrs = [o.p for o in outs]
        if "null" in kw:
            ptrs[kw["null"]] = None
        args = [B, N, Np, A, dptr(src), dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src), dptr(src), 0.97,
                kw.get("kappa", 1.0), kw.get("alpha", 1.0)]
        for fn, extra in (("riqn_cql_loss_fwd_bwd", []), ("riqn_cql_loss_fwd_bwd_h", [1e-3])):
            with pytest.raises(RiqnError):
                lib_call(fn, *args, *extra, *ptrs)
    for eps in (-1e-3, math.nan, math.inf):
        with pytest.raises(RiqnError):
            lib_call("riqn_cql_loss_fwd_bwd_h", 4, 8, 8, 4, dptr(src), dptr(src), dptr(src), dptr(idx), dptr(idx),
                     dptr(src), dptr(src), 0.97, 1.0, 1.0, eps, *(o.p for o in outs))
    for kw in (dict(B=0), dict(N=0), dict(A=0), dict(A=33), dict(alpha=0.0), dict(alpha=math.nan), dict(alpha=-2.0),
               dict(alpha=math.inf), dict(null=True)):
        with pytest.raises(RiqnError):
            lib_call("riqn_cql_dense_grad", kw.get("B", 4), kw.get("N", 8), kw.get("A", 4), dptr(src), dptr(src),
                     dptr(idx), None if "null" in kw else dptr(src), 1.0, kw.get("alpha", 1.0), outs[0].p)
    torch.cuda.synchronize()
    for o in outs:
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


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
    a.cql = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _cql_learner(dev, B, kind, N, params, **kw):
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


STEP_CASES = [(k, B, N) for k in ("iqn", "cvar", "qr") for B, N in ((32, 64), (512, 64), (32, 200))] + [("qr", 512, 200)]


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("kind,B,N", STEP_CASES)
def test_learner_step_vs_oracle(cuda_dev, kind, B, N, eps):
    """Learner.compute_gradients under injected noises (and fractions) against the torch-fp32 CQL step: loss within 1e-3
    relative and every gradient at cosine >= 0.999, 0.98 upstream of a flipped ReLU or a near-tie argmax."""
    from test_gpu_learn import _dev_batch
    cfg, seed, alpha = cases.iqn_cfg(N, N, 32), 15100 + B + N + len(kind), 4.0
    kw = dict(cql_alpha=alpha)
    if eps is not None:
        kw.update(value_rescaling=1, value_rescaling_eps=eps)
    params = oq.make_params(seed, 18, N) if kind == "qr" else net.make_params(seed)
    torch.manual_seed(seed)
    lr = _cql_learner(cuda_dev, B, kind, N, params, **kw)
    assert lr.cql == alpha and lr.value_rescaling == eps
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
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    for k in ("td_loss", "gap", "pi"):
        assert bool(torch.isfinite(dbg[k]).all()), k
    # the kernel's gap on the product's own online pass, and the loss it forms
    gap64 = oc.gap_from_means_np(oc.means_f32(dbg["q_on"].cpu().numpy(), B), b["actions"])[0]
    assert np.max(_ulps(dbg["gap"].cpu().numpy(), gap64.astype(F32))) <= 1
    assert_bits("loss", f32_bits(loss.detach().cpu().numpy()),
                f32_bits(oc.loss_f32(dbg["td_loss"].cpu().numpy(), dbg["gap"].cpu().numpy(), alpha)))
    if kind != "qr":
        taus = (dbg["tau_sel"].cpu(), t_tgt, t_on)
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_grads = oc.learn_step("qr" if kind == "qr" else "iqn", p_on, p_tg, cases.batch_to_torch(b),
                                    torch.from_numpy(b["weights"]), noises, taus, cfg, alpha, eps, keep=keep)
    qv = keep["qv_next"].numpy()
    top2 = np.sort(qv, axis=1)[:, -2:]
    tie = (top2[:, 1] - top2[:, 0]) < (1e-4 if eps is None else 1e-3)
    a_gpu = dbg["a_star"].cpu().numpy()
    ok = a_gpu == keep["a_star"].numpy()
    assert np.all(ok | tie)
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    err = np.abs(lg - lo) / np.abs(lo)
    assert np.max(err[ok]) < 1e-3, float(np.max(err[ok]))
    fl = _flips(dbg, keep, B, kind)
    relaxed = set()
    if fl[3] + fl[4] or not ok.all():
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
          f"ties {int((~ok).sum())}, mean gap {float(dbg['gap'].mean()):.4g}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "qr"])
def test_autograd_through_the_loss_node_equals_compute_gradients(cuda_dev, kind):
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    params = oq.make_params(77, 18, N) if kind == "qr" else net.make_params(77)
    b = cases.make_batch(78, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    if kind == "qr":
        inj = dict(noises=oq.make_noises(80, 18, N))
    else:
        inj = dict(noises=cases.make_noises(80),
                   taus=tuple(torch.from_numpy(t) for t in cases.make_taus(81, B, cases.iqn_cfg(N, N, 32))))
    out = []
    for mode in ("learner", "autograd"):
        torch.manual_seed(79)
        lr = _cql_learner(cuda_dev, B, kind, N, params)
        lr._inject = dict(inj)
        if mode == "learner":
            loss = lr.compute_gradients(st, ac, rt, nx, nt, w)
        else:
            lr.online_net.zero_grad()
            loss = lr.compute_loss_actor_or_learner(st, ac, rt, nx, nt)
            (w * loss).mean().backward()
        torch.cuda.synchronize()
        out.append((loss.detach().clone(), lr.online_net._flat_grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.gpu
def test_autograd_of_a_torch_written_cql_loss(cuda_dev):
    """A CQL loss written in torch on net(x) of the QR-DQN network goes through the dense head backward and matches the
    oracle's autograd."""
    from rainbow_iqn_apex_b200.model import DQN
    B, N, A, alpha = 32, 64, 18, 2.0
    params = oq.make_params(81, A, N)
    a = _args(cuda_dev, B, "qr", N)
    d = DQN(a, A).to(cuda_dev)
    load_params(d, params)
    d.train()
    noise = oq.make_noises(82, A, N, count=1)[0]
    d.reset_noise({k: tuple(t.to(cuda_dev) for t in v) for k, v in noise.items()})
    b = cases.make_batch(83, B)
    x = torch.from_numpy(b["states"]).to(cuda_dev)
    target = torch.from_numpy(np.random.RandomState(84).standard_normal((B, N)).astype(F32))
    acts = torch.from_numpy(b["actions"])

    def torch_loss(q, tau):
        th = q.view(N, B, A)[:, torch.arange(B, device=q.device), acts.to(q.device)].t()
        dl = target.to(q.device)[:, :, None] - th[:, None, :]
        t = tau.view(N, B).t()[:, None, :]
        hub = torch.where(dl.abs() <= 1.0, 0.5 * dl * dl, dl.abs() - 0.5)
        td = ((t - (dl.detach() < 0).float()).abs() * hub).sum(2).mean(1)
        return (td + alpha * oc.gap_torch(q, N, B, acts.to(q.device))).mean()

    d.zero_grad()
    q, tau = d(x)
    torch_loss(q, tau).backward()
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().clone() for k, p in d.named_parameters()}
    p = net.to_torch(params, requires_grad=True)
    net.apply_noise(p, noise)
    q_o = oq.dqn_forward_qr(p, cases.batch_to_torch(b)[0], A, N)
    torch_loss(q_o, torch.from_numpy(oq.fractions_f32(N)).repeat_interleave(B)).backward()
    for k, t in p.items():
        if t.requires_grad:
            assert _cos(got[k], t.grad) > 0.999, k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eager", "replay", "batch", "learn"])
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_steps_are_bitwise_reproducible(cuda_dev, kind, head):
    """Two consecutive B = 512 steps, eagerly and from each of the three captured graphs, twice alike."""
    from test_gpu_augment import _bench_run
    fields = dict(cql=1, **(dict(qr_dqn=1) if head == "qr" else {}))
    (o1, p1), (o2, p2) = _bench_run(cuda_dev, kind, fields, steps=2), _bench_run(cuda_dev, kind, fields, steps=2)
    for (_, l1), (_, l2) in zip(o1, o2):
        assert torch.equal(l1, l2) and bool(torch.isfinite(l1).all()) and bool((l1 >= 0).all())
    assert torch.equal(p1, p2)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "qr"])
def test_data_parallel_half_batches_equal_one_learner(cuda_dev, kind):
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    cfg = cases.iqn_cfg(N, N, 32)
    b = cases.make_batch(12, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    params = oq.make_params(12, 18, N) if kind == "qr" else net.make_params(12)
    noises = oq.make_noises(13, 18, N) if kind == "qr" else cases.make_noises(13)
    taus = [torch.from_numpy(t) for t in cases.make_taus(14, B, cfg)]

    def grads_of(sl, scale):
        torch.manual_seed(1)
        lr = _cql_learner(cuda_dev, sl.stop - sl.start, kind, N, params)
        inj = dict(noises=noises)
        if kind != "qr":   # the fractions of the half batch: rows i*B + b of the quantile-major draws
            inj["taus"] = tuple(t.view(-1, B)[:, sl].reshape(-1, 1).contiguous() for t in taus)
        lr._inject = inj
        lr.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl] * scale)
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
def test_zero_shifts_equal_the_unshifted_learner(cuda_dev, head):
    from test_gpu_augment import _learner, _step, _assert_same, _window_batch
    B = 32
    fields = dict(cql=1, **(dict(qr_dqn=1) if head == "qr" else {}))
    win_np, win, b, rest = _window_batch(cuda_dev, B, 900)
    plain = _learner(cuda_dev, B, fields, seed=11)
    aug = _learner(cuda_dev, B, fields, shift=4, seed=11)
    assert plain.cql == 1.0 and aug.cql == 1.0 and aug.random_shift == 4
    z = np.zeros((B, 2), np.int32)
    aug._inject = dict(shifts=(z, z))
    _assert_same(_step(aug, win[:, :4], win[:, 3:7], rest), _step(plain, win[:, :4], win[:, 3:7], rest), head)


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_actors_equal_the_plain_agent_and_priorities_match_the_oracle(cuda_dev, head):
    from rainbow_iqn_apex_b200 import Actor
    N, E, seed, alpha = 32, 8, 15300, 2.0
    cfg = cases.iqn_cfg(N, N, 8)
    params = oq.make_params(seed, 18, N) if head == "qr" else net.make_params(seed)
    actors = []
    for on in (1, 0):
        torch.manual_seed(seed)
        a = Actor(_args(cuda_dev, 8, head, N, cql=on, cql_alpha=alpha, num_quantile_samples=8), 18, None)
        load_params(a.online_net, params)
        a.update_target_net()
        actors.append(a)
    cq, plain = actors
    assert cq.cql == alpha and plain.cql is None
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    for a in actors:
        a.eval()
    torch.manual_seed(1)
    v1 = cq.act_batch_values(su8)
    torch.manual_seed(1)
    v2 = plain.act_batch_values(su8)
    assert torch.equal(v1, v2)
    torch.manual_seed(2)
    a1 = cq.act(list(states[0]))
    torch.manual_seed(2)
    assert a1 == plain.act(list(states[0]))
    cq.train()
    bs, L, n, hist = 8, 14, cfg["n_step"], 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    if head == "qr":
        inj = [dict(noises=oq.make_noises(seed + 10 * c, 18, N)) for c in range(chunks)]
    else:
        inj = []
        for c in range(chunks):
            m = min(bs, L - n - c * bs)
            inj.append(dict(noises=cases.make_noises(seed + 10 * c),
                            taus=tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 10 * c + 1, m, cfg))))
    cq._inject = list(inj)
    pri = cq.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not cq._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(cfg["discount"] ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        loss = oc.cql_loss(head, net.to_torch(params, requires_grad=True), net.to_torch(params),
                           (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx,
                            torch.ones(hi - lo)), inj[c]["noises"], inj[c].get("taus"), cfg, alpha)
        out.append(loss.detach().numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    rel = np.abs(pri - ref_p) / ref_p
    print(f"{head} priorities rel err median {np.median(rel):.3g} max {np.max(rel):.3g}")
    assert np.median(rel) < 1e-3 and np.max(rel) < 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_cql_step_makes_one_more_launch_than_its_plain_twin(cuda_dev, head):
    from test_gpu_qr import _bench_learner
    base = dict(qr_dqn=1) if head == "qr" else {}
    (s1, _, _, _), (s2, _, _, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f) for f in (base, dict(base, cql=1)))
    c1, c2 = [c for _, _, c in s1], [c for _, _, c in s2]
    print(f"{head}: eager launches per step, plain {c1}, CQL {c2}")
    diff = {b - a for a, b in zip(c1, c2)}
    assert len(diff) == 1 and 1 <= diff.pop() <= 3


@pytest.mark.gpu
@pytest.mark.parametrize("base", [{}, dict(rainbow_only=1), dict(qr_dqn=1)])
def test_namespace_without_the_field_is_unchanged(cuda_dev, base):
    """IQN, C51 and QR-DQN learners from a namespace without cql and with cql = 0 run the same launches per step and give
    bit-identical sampled indices, losses and parameters."""
    from test_gpu_qr import _bench_learner
    (s1, p1, l1, _), (s2, p2, l2, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f)
                                        for f in (base, dict(base, cql=0, cql_alpha=3.0)))
    assert l1.cql is None and l2.cql is None
    for k, ((i1, x1, c1), (i2, x2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(x1, x2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_checkpoints_round_trip_between_cql_and_plain(cuda_dev, tmp_path, head):
    from rainbow_iqn_apex_b200 import Agent, Learner
    from test_gpu_qr import _graph_batch
    B, N = 32, 64
    batch = _graph_batch(cuda_dev, B, 4)
    for src, dst in ((dict(cql=1), dict(cql=0)), (dict(cql=0), dict(cql=1, cql_alpha=5.0))):
        lr = Learner(_args(cuda_dev, B, head, N, **src), 18, None)
        lr.train()
        lr.learn_on_batch(*batch)
        lr.save(str(tmp_path), 0, 1, "ck.pth")
        path = os.path.join(tmp_path, "ck.pth")
        ck = torch.load(path, map_location="cpu")
        assert not any("cql" in k for k in ck)
        back = Agent(_args(cuda_dev, B, head, N, model=path, **dst), 18, None)
        assert torch.equal(back.online_net._flat, lr.online_net._flat) and back.optimiser._step == 1
        assert back.cql == (None if not dst["cql"] else 5.0)


@pytest.mark.gpu
def test_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    for kind, kw in (("iqn", dict(cql=2)), ("iqn", dict(cql="1")), ("iqn", dict(cql_alpha=0.0)),
                     ("iqn", dict(cql_alpha=-1.0)), ("iqn", dict(cql_alpha=math.nan)), ("iqn", dict(cql_alpha=math.inf)),
                     ("iqn", dict(cql_alpha="1")), ("iqn", dict(rainbow_only=1)), ("iqn", dict(rainbow_only=1, hl_gauss=1)),
                     ("iqn", dict(munchausen=1)), ("iqn", dict(fqf=1)), ("qr", dict(mmd=1))):
        with pytest.raises(ValueError):
            Agent(_args(cuda_dev, B, kind, 64, **kw), 18, None)
    ag = Learner(_args(cuda_dev, B, "cvar", 64, value_rescaling=1, random_shift=4, cql_alpha=np.float32(0.5)), 18, None)
    assert ag.cql == 0.5 and ag.value_rescaling == 1e-3 and ag.random_shift == 4 and ag.risk is not None


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "qr"])
def test_offline_recipe(cuda_dev, head):
    """The offline recipe: a replay filled only by append_arrays (timesteps from 0 at each episode start, priorities 1),
    priority_exponent = 0, Learner.learn with update_target_net every target_update steps and no actors: every IS
    weight is 1 and every loss is finite."""
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    B, steps, target_update = 32, 20, 8
    a = _args(cuda_dev, B, head, 64, actor_capacity=2000, nb_actor=1, priority_exponent=0.0)
    torch.manual_seed(3)
    lr = Learner(a, 18, None)
    lr.train()
    mem = ReplayMemory(a, None)
    rs = np.random.RandomState(4)
    n, ep = 2000, 250
    ts = np.arange(n) % ep
    dones = (ts == ep - 1)
    mem.transitions.append_arrays(0, 0, ts, rs.randint(0, 256, (n, 84, 84)).astype(np.uint8), rs.randint(0, 18, n),
                                  rs.randint(-1, 2, n).astype(np.float32), dones, np.ones(n, np.float32))
    for t in range(steps):
        assert bool((mem.sample(B)[-1] == 1).all())
        idxs, loss = lr.learn(mem, None)
        mem.update_priorities(idxs, loss)
        assert bool(torch.isfinite(loss).all()) and bool((loss >= 0).all())
        if (t + 1) % target_update == 0:
            lr.update_target_net()
    assert bool(torch.isfinite(lr.online_net._flat).all())
