"""MMDQN (Nguyen-Tang, Gupta & Venkatesh, AAAI 2021): the moment-matching loss on the QR-DQN particle network
(riqn_mmd_loss_fwd_bwd, riqn_mmd_loss_fwd_bwd_h) behind the optional Agent fields mmd and mmd_bandwidths.

The unmarked tests pin the oracle (oracle/mmd.py) by identities, check its float64 and torch-fp32 statements against each
other, and check the host-side validation.  The gpu tests check both entry points against float64 on the particles and
targets they read, with the kernel's per-term error model (the method of test_gpu_c51_kernels.py: NaN prefills,
canaries, two calls alike, rejected calls write nothing), a learner step, autograd and the actors against the torch
oracle, reproducibility eagerly and from each captured step graph, data parallelism, augmentation, checkpoints, and that
a namespace without the field runs exactly as before."""
import ctypes
import math

import numpy as np
import pytest
import torch

from helpers import U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, load_params, make_args, \
    rel_err, to_dev
from oracle import cases, mmd as om, network as net, qr as oq

F32 = np.float32
BW_DEFAULT = tuple(float(h) for h in range(1, 11))
BW_WIDE = tuple(float(x) for x in np.logspace(-3, 3, 16).astype(np.float32))


def _mmd_args(dev, B, N=64, **kw):
    a = make_args(dev, B, cases.iqn_cfg(N, N, 32))
    a.qr_dqn, a.mmd = 1, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def test_large_bandwidth_limit_is_the_squared_mean_gap():
    """One bandwidth h -> infinity: exp(-d^2/h) = 1 - d^2/h + O(h^-2), so h MMD^2 -> 2 (mean theta - mean T)^2."""
    rs = np.random.RandomState(1)
    th, T = rs.standard_normal((6, 9)), rs.standard_normal((6, 9)) + 0.5
    want = 2.0 * (th.mean(1) - T.mean(1)) ** 2
    errs = []
    for h in (1e2, 1e3, 1e4):
        errs.append(np.max(np.abs(h * om.mmd2_np(th, T, (h,)) - want)))
    assert errs[2] < 1e-3 * np.max(want) and errs[0] > errs[1] > errs[2]


def test_sign_zero_and_positive():
    rs = np.random.RandomState(2)
    for scale in (1.0, 1e-4):
        th = rs.standard_normal((50, 16))
        T = th + scale * rs.standard_normal((50, 16))
        m = om.mmd2_np(th, T)
        assert np.all(m >= 0) and np.all(m > 0)
        assert np.array_equal(om.loss_np(th, T), np.maximum(m, 0))
    th = rs.standard_normal((20, 12))
    perm = np.stack([rs.permutation(th[b]) for b in range(20)])
    assert np.max(np.abs(om.mmd2_np(th, perm))) <= 1e-15
    assert np.max(np.abs(om.mmd2_np(th, perm, BW_WIDE))) <= 1e-15
    assert np.all(om.mmd2_np(th, th + 1e-2) > 0)
    dup = th.copy()
    dup[:, 0] = dup[:, 1]                                           # another multiset with the same support size
    assert np.all(om.mmd2_np(th, dup) > 0)


def test_translation_and_permutation_invariance():
    rs = np.random.RandomState(3)
    th, T = rs.standard_normal((8, 10)), rs.standard_normal((8, 10))
    for bw in (BW_DEFAULT, (1.0,), BW_WIDE):
        l0, g0 = om.mmd2_np(th, T, bw), om.dtheta_np(th, T, bw)
        assert np.allclose(om.mmd2_np(th + 3.25, T + 3.25, bw), l0, rtol=1e-12, atol=1e-15)
        assert np.allclose(om.dtheta_np(th + 3.25, T + 3.25, bw), g0, rtol=1e-12, atol=1e-15)
        p = rs.permutation(10)
        assert np.allclose(om.mmd2_np(th[:, p], T, bw), l0, rtol=1e-12, atol=1e-15)
        assert np.allclose(om.dtheta_np(th[:, p], T, bw), g0[:, p], rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("bw", [BW_DEFAULT, (1.0,), BW_WIDE])
def test_gradient_vs_autograd_and_central_differences(bw):
    rs = np.random.RandomState(4)
    th, T = rs.standard_normal((5, 7)) * 2, rs.standard_normal((5, 7)) * 2
    g = om.dtheta_np(th, T, bw)
    t = torch.tensor(th, dtype=torch.float64, requires_grad=True)
    om.mmd2_torch(t, torch.tensor(T, dtype=torch.float64), bw).sum().backward()
    assert np.max(np.abs(t.grad.numpy() - g)) <= 1e-12 * max(1.0, np.abs(g).max())
    h = 1e-5
    fd = np.zeros_like(th)
    for i in range(th.shape[1]):
        e = np.zeros_like(th)
        e[:, i] = h
        fd[:, i] = (om.mmd2_np(th + e, T, bw) - om.mmd2_np(th - e, T, bw)) / (2 * h)
    assert np.max(np.abs(fd - g)) <= 1e-6 * max(1.0, np.abs(g).max())
    # the clamp: value max(0, MMD^2), gradient of the unclamped sum
    m = torch.tensor([-1e-9, 2.0], dtype=torch.float64, requires_grad=True)
    c = om.clamped(m)
    c.sum().backward()
    assert c.tolist() == [0.0, 2.0] and m.grad.tolist() == [1.0, 1.0]


@pytest.mark.parametrize("eps", [None, 1e-3])
def test_float64_and_torch_fp32_statements_agree(eps):
    B, A, n = 4, 4, 8
    cfg = cases.iqn_cfg(n, n, 8)
    params = oq.make_params(31, A, n)
    b = cases.make_batch(32, B, action_space=A)
    st, ac, rt, nx, nt = cases.batch_to_torch(b)
    noises = oq.make_noises(33, A, n)
    keep = {}
    loss, _ = om.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params), (st, ac, rt, nx, nt),
                            torch.from_numpy(b["weights"]), noises, cfg, eps=eps, keep=keep)
    tgt = oq.target_np(keep["q_tgt"].numpy(), keep["a_star"].numpy(), b["returns"], b["nonterminals"], 0.99 ** 3, eps)
    assert rel_err(keep["target"].numpy(), tgt) < 1e-6
    ref = om.loss_np(keep["theta"].numpy(), tgt)
    assert np.max(np.abs(loss.numpy() - ref)) <= 1e-6 * np.max(np.abs(ref))
    th = keep["theta"].clone().requires_grad_(True)
    om.mmd2_torch(th, keep["target"]).sum().backward()
    g = om.dtheta_np(keep["theta"].numpy(), tgt)
    assert np.max(np.abs(th.grad.numpy() - g)) <= 1e-6 * np.max(np.abs(g))


def test_check_mmd():
    from rainbow_iqn_apex_b200.mmd import MMD_DEFAULTS, check_mmd
    assert MMD_DEFAULTS["mmd_bandwidths"] == BW_DEFAULT
    assert check_mmd(0) is None and check_mmd(False) is None and check_mmd(0, "x", rainbow_only=True) is None
    assert check_mmd(1, qr_dqn=64) == BW_DEFAULT
    assert check_mmd(True, [2, 0.5], qr_dqn=8) == (2.0, 0.5) and check_mmd(np.int64(1), np.float32([3]), qr_dqn=2) == (3.0,)
    assert check_mmd(1, BW_WIDE, qr_dqn=200) == BW_WIDE
    bad = [dict(mmd=2), dict(mmd=-1), dict(mmd=0.5), dict(mmd=1.0), dict(mmd="1"), dict(mmd=None),
           dict(bandwidths="1,2"), dict(bandwidths=b"12"), dict(bandwidths=3.0), dict(bandwidths=None),
           dict(bandwidths=(1.0, True)), dict(bandwidths=(False,)), dict(bandwidths=(1.0, float("nan"))),
           dict(bandwidths=(float("inf"),)), dict(bandwidths=(-float("inf"),)), dict(bandwidths=(0.0,)),
           dict(bandwidths=(1.0, -2.0)), dict(bandwidths=(1e-50,)), dict(bandwidths=(1e-39,)), dict(bandwidths=(1e39,)),
           dict(bandwidths=("1",)), dict(bandwidths=(1.0,) * 17), dict(bandwidths=()), dict(bandwidths=[]),
           dict(qr_dqn=None), dict(rainbow_only=1), dict(munchausen=(0.9, 0.03, -1.0)), dict(fqf=(2.5e-9, 0.0)),
           dict(risk=("cvar", 0.25))]
    for kw in bad:
        kw = dict(dict(mmd=1, bandwidths=BW_DEFAULT, qr_dqn=64), **kw)
        with pytest.raises(ValueError):
            check_mmd(**kw)
    assert check_mmd(1, (1.0,) * 16, qr_dqn=2) == (1.0,) * 16


# ------------------------------------------------------------------------------------------------ kernels (GPU)
KERNEL_CASES = [(1, 1, 2, BW_DEFAULT), (5, 4, 7, (1.0,)), (33, 32, 64, BW_WIDE), (512, 18, 200, BW_DEFAULT),
                (64, 18, 256, BW_DEFAULT), (4096, 4, 7, BW_DEFAULT), (7, 1, 256, BW_WIDE), (100, 32, 2, BW_WIDE),
                (3000, 18, 1, (1.0,)), (128, 4, 200, (1.0,))]
CHECK_ROWS = 48          # rows held to float64 per case (all rows are checked bitwise against the second call)


def _hb(bw):
    return (ctypes.c_float * len(bw))(*bw)


def _operands(B, A, n, regime, seed):
    """q_on, q_tgt (n*B, A), actions, a_star, returns, nonterminals, gamma_n."""
    rs = np.random.RandomState(seed)
    q_on = rs.standard_normal((n * B, A)).astype(F32)
    q_tgt = rs.standard_normal((n * B, A)).astype(F32)
    acts = rs.randint(0, A, B).astype(np.int64)
    ast = rs.randint(0, A, B).astype(np.int64)
    R = rs.standard_normal(B).astype(F32)
    nt = (rs.uniform(size=B) < 0.8).astype(F32)
    g = 0.97
    if regime == "gap":                     # targets >= 3000 away from every particle (also as h(R + ...) under rescaling):
        R = (R + 1e7).astype(F32)           # every cross term underflows, even at h = 1e3
    elif regime == "near":                  # T_j = theta_j + 1e-3 noise
        cols = q_on.reshape(n, B, A)[:, np.arange(B), acts]
        q3 = q_tgt.reshape(n, B, A)
        q3[:, np.arange(B), ast] = (cols + 1e-3 * rs.standard_normal(cols.shape)).astype(F32)
        R, nt, g = np.zeros(B, F32), np.ones(B, F32), 1.0
    return q_on, q_tgt, acts, ast, R, nt, g


def _call(dev, B, A, n, ops, bw, eps=None, outs=True):
    q_on, q_tgt, acts, ast, R, nt, g = ops
    d = [to_dev(q_on, dev), to_dev(q_tgt, dev), to_dev(acts, dev, torch.int64), to_dev(ast, dev, torch.int64),
         to_dev(R, dev), to_dev(nt, dev)]
    loss, dth = Out(B, dev), Out(n * B, dev)
    th, tg = (Out(B * n, dev), Out(B * n, dev)) if outs else (None, None)
    args = [B, n, A, *(dptr(t) for t in d), float(g), len(bw), _hb(bw)]
    o = [loss.p, dth.p, th.p if th else None, tg.p if tg else None]
    if eps is None:
        lib_call("riqn_mmd_loss_fwd_bwd", *args, *o)
    else:
        lib_call("riqn_mmd_loss_fwd_bwd_h", *args, float(eps), *o)
    torch.cuda.synchronize()
    assert_canaries({"loss": loss, "dtheta": dth, "theta": th, "target": tg})
    return loss, dth, th, tg


def _iqn_outs(dev, B, A, n, ops, eps):
    """theta_out / target_out of riqn_iqn_loss_fwd_bwd[_h] on the same inputs."""
    q_on, q_tgt, acts, ast, R, nt, g = ops
    d = [to_dev(q_on, dev), to_dev(q_tgt, dev), torch.full((n * B,), 0.5, device=dev), to_dev(acts, dev, torch.int64),
         to_dev(ast, dev, torch.int64), to_dev(R, dev), to_dev(nt, dev)]
    loss, dth, th, tg = Out(B, dev), Out(n * B, dev), Out(B * n, dev), Out(B * n, dev)
    args = [B, n, n, A, *(dptr(t) for t in d), float(g), 1.0]
    if eps is None:
        lib_call("riqn_iqn_loss_fwd_bwd", *args, loss.p, dth.p, th.p, tg.p)
    else:
        lib_call("riqn_iqn_loss_fwd_bwd_h", *args, float(eps), loss.p, dth.p, th.p, tg.p)
    torch.cuda.synchronize()
    return th, tg


def _bounds(th, T, bw):
    """float64 loss (unclamped), dtheta, and their error bounds from the kernel's per-term model, for rows th, T (R, n)."""
    R_, n = th.shape
    H = len(bw)
    ln2 = math.log(2.0)
    lb, gb = np.zeros(R_), np.zeros((R_, n))
    tiny = 2.0 ** -126
    c_acc = (H + n + 64) * U          # the sums over h, over j and the reduction over i, generously
    for x, y, wt, grad_sign in ((th, th, 1.0, -1.0), (T, T, 1.0, 0.0), (th, T, 2.0, 1.0)):
        d = x[:, :, None] - y[:, None, :]
        s = d * d
        for h in bw:
            a = s / h / ln2                                   # the exponent in log2 units
            e = np.exp(-s / h)
            per = e * ((8 + 6 * ln2 * a) * U + c_acc) + tiny
            lb += wt * per.sum((1, 2))
            if grad_sign:
                gb += (np.abs(d) * (2.0 / h) * (per + 2 * U * e)).sum(2)
    return lb / (n * n), 2.0 * gb / (n * n)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 0.0, 1e-3])
@pytest.mark.parametrize("regime", ["gauss", "gap", "near"])
@pytest.mark.parametrize("B,A,n,bw", KERNEL_CASES)
def test_mmd_loss_vs_float64(cuda_dev, B, A, n, bw, regime, eps):
    ops = _operands(B, A, n, regime, B + 3 * A + 7 * n + len(bw))
    loss, dth, tho, tgo = _call(cuda_dev, B, A, n, ops, bw, eps)
    # the particles and targets the kernel read are those riqn_iqn_loss_fwd_bwd[_h] reads, bit for bit
    ith, itg = _iqn_outs(cuda_dev, B, A, n, ops, eps)
    assert_bits("theta_out vs iqn", tho.bits(), ith.bits())
    assert_bits("target_out vs iqn", tgo.bits(), itg.bits())
    th = tho.f32().reshape(B, n).astype(np.float64)
    T = tgo.f32().reshape(B, n).astype(np.float64)
    L, G = loss.f32(), dth.f32().reshape(n, B).T
    assert np.all(L >= 0), "a negative loss"
    rows = np.unique(np.concatenate([np.arange(min(B, CHECK_ROWS // 2)),
                                     np.random.RandomState(B).randint(0, B, CHECK_ROWS // 2), [B - 1]]))
    ref_l, ref_g = om.mmd2_np(th[rows], T[rows], bw), om.dtheta_np(th[rows], T[rows], bw)
    lb, gb = _bounds(th[rows], T[rows], bw)
    r1 = check_bound("loss", L[rows], np.maximum(ref_l, 0), lb + 2 * U * np.abs(ref_l))
    r2 = check_bound("dtheta", G[rows], ref_g, gb + 2 * U * np.abs(ref_g) + 1e-40)
    print(f"B={B} A={A} n={n} H={len(bw)} {regime} eps={eps}: worst err/bound loss {r1:.3g}, dtheta {r2:.3g}")
    if regime == "gap":                  # no cross term survives: the loss is the theta-theta and T-T sums, >= 2 H / n
        assert np.all(L >= F32(0.999 * 2 * len(bw) / n))
    l2, g2, _, _ = _call(cuda_dev, B, A, n, ops, bw, eps, outs=False)
    assert_bits("second call loss", l2.bits(), loss.bits())
    assert_bits("second call dtheta", g2.bits(), dth.bits())


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("B,A,n,bw", KERNEL_CASES)
def test_equal_targets_give_exact_zero(cuda_dev, B, A, n, bw, eps):
    """R = 0, gamma^n = 1, nt = 1 and the target column equal to the online column: T_j = theta_j (fl(h(h^-1(z))) = z
    under rescaling), so every bracket and gradient pair cancels exactly."""
    q_on, _, acts, _, _, _, _ = _operands(B, A, n, "gauss", 11 * B + n)
    ops = (q_on, q_on.copy(), acts, acts.copy(), np.zeros(B, F32), np.ones(B, F32), 1.0)
    loss, dth, tho, tgo = _call(cuda_dev, B, A, n, ops, bw, eps)
    assert_bits("targets equal the particles", tgo.bits(), tho.bits())
    assert_bits("loss", loss.bits(), np.zeros(B, np.uint32))
    assert_bits("dtheta", dth.bits(), np.zeros(n * B, np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("B,A,n,bw", KERNEL_CASES)
def test_translation_is_bitwise_invariant(cuda_dev, B, A, n, bw):
    """Particles and targets on a dyadic grid (k 2^-6, |k| < 2^10), shifted together by c = 37.5: every shifted value
    and every difference is exact, so the loss and dtheta keep their bits."""
    rs = np.random.RandomState(B * n)
    q_on = (rs.randint(-1024, 1024, (n * B, A)) * 2.0 ** -6).astype(F32)
    q_tgt = (rs.randint(-1024, 1024, (n * B, A)) * 2.0 ** -6).astype(F32)
    acts, ast = rs.randint(0, A, B).astype(np.int64), rs.randint(0, A, B).astype(np.int64)
    base = (q_on, q_tgt, acts, ast, np.zeros(B, F32), np.ones(B, F32), 1.0)
    moved = ((q_on + F32(37.5)).astype(F32), (q_tgt + F32(37.5)).astype(F32), acts, ast, np.zeros(B, F32),
             np.ones(B, F32), 1.0)
    l0, g0, _, _ = _call(cuda_dev, B, A, n, base, bw)
    l1, g1, _, _ = _call(cuda_dev, B, A, n, moved, bw)
    assert_bits("loss", l1.bits(), l0.bits())
    assert_bits("dtheta", g1.bits(), g0.bits())
    assert np.all(l0.f32() >= 0)


@pytest.mark.gpu
def test_entry_points_reject_invalid_calls_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    src = torch.zeros(300 * 300 * 4, device=dev)
    idx = torch.zeros(300, dtype=torch.int64, device=dev)
    outs = [Out(300 * 300 * 4, dev) for _ in range(4)]
    bad = [dict(n=0), dict(n=257), dict(n=-1), dict(B=0), dict(B=-2), dict(A=33), dict(A=0), dict(bw=()),
           dict(bw=(1.0,) * 17), dict(bw=(float("nan"),)), dict(bw=(1.0, float("inf"))), dict(bw=(-float("inf"),)),
           dict(bw=(0.0,)), dict(bw=(1.0, -1.0)), dict(bw=(1e-40,)), dict(nbw=17), dict(nbw=0), dict(nbw=-1)]
    for kw in bad:
        B, A, n, bw = kw.get("B", 4), kw.get("A", 4), kw.get("n", 8), kw.get("bw", BW_DEFAULT)
        nbw = kw.get("nbw", len(bw))
        hb = _hb(bw if len(bw) >= max(nbw, 0) else bw + (1.0,) * (nbw - len(bw)))
        args = [B, n, A, dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src), dptr(src), 0.97, nbw, hb]
        for fn, extra in (("riqn_mmd_loss_fwd_bwd", []), ("riqn_mmd_loss_fwd_bwd_h", [1e-3])):
            with pytest.raises(RiqnError):
                lib_call(fn, *args, *extra, *(o.p for o in outs))
    for eps in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(RiqnError):
            lib_call("riqn_mmd_loss_fwd_bwd_h", 4, 8, 4, dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src),
                     dptr(src), 0.97, 10, _hb(BW_DEFAULT), eps, *(o.p for o in outs))
    torch.cuda.synchronize()
    for o in outs:
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _mmd_learner(dev, B, N, params, **kw):
    from rainbow_iqn_apex_b200 import Learner
    lr = Learner(_mmd_args(dev, B, N, **kw), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    return lr


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("B,N", [(32, 64), (512, 64), (32, 200), (512, 200)])
def test_learner_step_vs_oracle(cuda_dev, B, N, eps):
    """Under injected noises, against the torch-fp32 oracle step.  The gradients are held to QR-DQN's bounds.  The loss
    is held per transition to 1e-3 relative, or, where MMD^2 is small against its three terms, to a floor derived from
    the kernel bound and the forward passes' error (below)."""
    from test_gpu_learn import _dev_batch
    cfg, seed = cases.iqn_cfg(N, N, 32), 9800 + B + N
    params = oq.make_params(seed, 18, N)
    torch.manual_seed(seed)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    lr = _mmd_learner(cuda_dev, B, N, params, **kw)
    assert lr.qr_dqn == N and lr.mmd == BW_DEFAULT and lr.value_rescaling == eps
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    if eps is not None:
        b["returns"] = (b["returns"] * 40).astype(F32)
    noises = oq.make_noises(seed + 3, 18, N)
    lr._inject = dict(noises=noises)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    q_on = dbg["q_on"].cpu().numpy()
    th = dbg["theta"].cpu().numpy()
    assert np.array_equal(th, q_on.reshape(N, B, 18)[:, np.arange(B), b["actions"]].T)
    tgt = oq.target_np(dbg["q_tgt"].cpu().numpy(), dbg["a_star"].cpu().numpy(), b["returns"], b["nonterminals"],
                       cfg["discount"] ** cfg["n_step"], eps)
    assert rel_err(dbg["target"].cpu().numpy(), tgt) < 1e-6
    T = dbg["target"].cpu().numpy().astype(np.float64)
    th = th.astype(np.float64)
    lb, _ = _bounds(th, T, BW_DEFAULT)
    check_bound("loss vs float64 on its own operands", loss.detach().cpu().numpy(),
                om.loss_np(th, T), lb + 2 * U * np.abs(om.mmd2_np(th, T)))
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_grads = om.learn_step(p_on, p_tg, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises, cfg,
                                    eps=eps, keep=keep)
    # the loss: 1e-3 relative, or the floor of the forward's error carried to first order through the loss (MMD^2 is
    # symmetric, so dL/dT is dtheta_np with the roles swapped), doubled, plus the kernel bound for each of the two fp32
    # evaluations
    d_th = np.abs(th - keep["theta"].numpy())
    d_T = np.abs(T - keep["target"].numpy())
    fwd = (np.abs(om.dtheta_np(th, T)) * d_th).sum(1) + (np.abs(om.dtheta_np(T, th)) * d_T).sum(1)
    floor = 2.0 * fwd + 2.0 * lb
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    qv = keep["qv_next"].numpy()
    top2 = np.sort(qv, axis=1)[:, -2:]
    tie = (top2[:, 1] - top2[:, 0]) < (1e-4 if eps is None else 1e-3)
    ok = dbg["a_star"].cpu().numpy() == keep["a_star"].numpy()
    assert np.all(ok | tie)
    tol = 1e-3 * np.abs(lo) + floor
    err = np.abs(lg - lo)
    assert np.all((err <= tol)[ok]), float(np.max((err / tol)[ok]))
    print(f"loss: worst err / (1e-3 rel + floor) {np.max((err / tol)[ok]):.3g}, rows beyond 1e-3 relative "
          f"{int(np.sum(err[ok] > 1e-3 * np.abs(lo[ok])))} of {int(ok.sum())}")
    _check_grads(dbg, grads, o_grads, keep, ok)


def _check_grads(dbg, grads, o_grads, keep, ok):
    """QR-DQN's gradient bounds: cosine >= 0.999, relaxed to 0.98 upstream of a flipped ReLU or a near-tie argmax."""
    from test_gpu_qr import _relu_flips
    fl = _relu_flips(dbg["keep"], keep)
    relaxed = set()
    if fl[3] + fl[4] or not ok.all():
        relaxed |= {"conv1", "conv2", "conv3", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    worst = 1.0
    for k, g_ref in o_grads.items():
        c = _cos(grads[k], g_ref)
        worst = min(worst, c)
        assert c > (0.98 if k.split(".")[0] in relaxed else 0.999), (k, c, fl)
    print(f"min cos {worst:.6f}, ReLU flips {fl}, ties {int((~ok).sum())}")


@pytest.mark.gpu
def test_autograd_of_a_torch_written_mmd_loss(cuda_dev):
    """A torch-written MMD loss on net(x), back-propagated through riqn_qr_head_bwd_dense into the layer backwards,
    matches the oracle's autograd with QR-DQN's dense-backward tolerances."""
    from rainbow_iqn_apex_b200.model import DQN
    B, N, A = 32, 64, 18
    params = oq.make_params(77, A, N)
    torch.manual_seed(77)
    d = DQN(_mmd_args(cuda_dev, B, N), A).to(cuda_dev)
    load_params(d, params)
    d.train()
    noise = oq.make_noises(78, A, N, count=1)[0]
    d.reset_noise({k: tuple(t.to(cuda_dev) for t in v) for k, v in noise.items()})
    b = cases.make_batch(79, B)
    x = torch.from_numpy(b["states"]).to(cuda_dev)
    rs = np.random.RandomState(80)
    target = torch.from_numpy(rs.standard_normal((B, N)).astype(F32))
    acts = torch.from_numpy(b["actions"] % A)

    def torch_loss(q):
        th = q.view(N, B, A)[:, torch.arange(B, device=q.device), acts.to(q.device)].t()
        return om.clamped(om.mmd2_torch(th, target.to(q.device))).mean()

    d.zero_grad()
    q, _ = d(x)
    torch_loss(q).backward()
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().clone() for k, p in d.named_parameters()}
    p = net.to_torch(params, requires_grad=True)
    net.apply_noise(p, noise)
    q_o = oq.dqn_forward_qr(p, cases.batch_to_torch(b)[0], A, N)
    torch_loss(q_o).backward()
    assert rel_err(q.detach().cpu().numpy(), q_o.detach().numpy()) < 2e-3
    for k, t in p.items():
        if t.requires_grad:
            c = _cos(got[k], t.grad)
            assert c > 0.999, (k, c)


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_mmd_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    from test_gpu_qr import _bench_learner
    runs = [_bench_learner(cuda_dev, 1 << 14, graph, 2, dict(qr_dqn=1, mmd=1)) for _ in range(2)]
    (s1, p1, l1, _), (s2, p2, _, _) = runs
    assert l1.mmd == BW_DEFAULT and l1.batch_size == 512
    for k, ((i1, x1, _), (i2, x2, _)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(x1, x2), k
        assert bool(torch.isfinite(x1).all()) and bool((x1 >= 0).all())
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_batch_and_learn_graphs_are_bitwise_reproducible(cuda_dev):
    import bench
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_qr import _bench_learner, _graph_batch
    B = 512
    batches = [_graph_batch(cuda_dev, B, s) for s in (61, 62)]

    def batch_graph_run():
        _, _, lr, mem = _bench_learner(cuda_dev, 1 << 14, True, 1, dict(qr_dqn=1, mmd=1))
        lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(B)))
        hosts = [tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(B)) for _ in range(2)]
        out = [lr.learn_on_host_batch(h).clone() for h in hosts]
        torch.cuda.synchronize()
        return out, lr.online_net._flat.clone()

    def learn_graph_run():
        torch.manual_seed(9)
        a = bench.make_args(cuda_dev, 1 << 14)
        a.qr_dqn, a.mmd = 1, 1
        lr = Learner(a, bench.ACTIONS, None)
        lr.train()
        lr.enable_learn_graph(batches[0])
        out = [lr.learn_on_graph(bt).clone() for bt in batches]
        torch.cuda.synchronize()
        return out, lr.online_net._flat.clone()

    for run in (batch_graph_run, learn_graph_run):
        (o1, p1), (o2, p2) = run(), run()
        assert all(torch.equal(x, y) and bool(torch.isfinite(x).all()) for x, y in zip(o1, o2))
        assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_data_parallel_half_batches_equal_one_learner(cuda_dev):
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    b = cases.make_batch(12, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    params = oq.make_params(12, 18, N)
    noises = oq.make_noises(13, 18, N)

    def grads_of(sl, scale):
        torch.manual_seed(1)
        lr = _mmd_learner(cuda_dev, sl.stop - sl.start, N, params)
        lr._inject = dict(noises=noises)
        lr.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl] * scale)
        torch.cuda.synchronize()
        return lr.online_net._flat_grad.clone()

    full = grads_of(slice(0, B), 1.0)
    halves = grads_of(slice(0, B // 2), 0.5) + grads_of(slice(B // 2, B), 0.5)
    err = float((halves - full).abs().max() / full.abs().max())
    print(f"data parallel: max |sum of half-batch grads - full| / max |full| = {err:.3g}")
    assert err < 2e-3 and _cos(halves, full) > 0.99999


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_shifted_step_equals_the_plain_step_on_shifted_frames(cuda_dev, B):
    from test_gpu_augment import _learner, _step, _assert_same, _window_batch, shift_np
    fields = dict(qr_dqn=1, mmd=1)
    win_np, win, b, rest = _window_batch(cuda_dev, B, 500 + B)
    rs = np.random.RandomState(B + 1)
    s_st = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_nx = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_st[0], s_nx[0] = (3, -2), (-4, 1)
    aug = _learner(cuda_dev, B, fields, shift=4, seed=12)
    assert aug.mmd == BW_DEFAULT and aug.random_shift == 4
    aug._inject = dict(shifts=(s_st, s_nx))
    got = _step(aug, win[:, :4], win[:, 3:7], rest)
    st = torch.from_numpy(shift_np(win_np[:, :4], s_st)).to(cuda_dev)
    nx = torch.from_numpy(shift_np(win_np[:, 3:7], s_nx)).to(cuda_dev)
    plain = _learner(cuda_dev, B, fields, seed=12)
    _assert_same(got, _step(plain, st, nx, rest), "mmd")


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
def test_actors_equal_qr_dqn_and_priorities_match_the_oracle(cuda_dev, eps):
    from rainbow_iqn_apex_b200 import Actor
    N, E, seed = 32, 8, 9900
    cfg = cases.iqn_cfg(N, N, 8)
    params = oq.make_params(seed, 18, N)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    actors = []
    for fields in (dict(mmd=1), dict(mmd=0)):
        torch.manual_seed(seed)
        a = Actor(_mmd_args(cuda_dev, 8, N, **kw, **fields), 18, None)
        load_params(a.online_net, params)
        a.update_target_net()
        actors.append(a)
    mm, qr = actors
    assert mm.mmd == BW_DEFAULT and qr.mmd is None
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    for mode in ("eval", "train"):
        for a in actors:
            getattr(a, mode)()
        noise = oq.make_noises(seed + 5, 18, N, count=1)[0]
        for a in actors:
            a.online_net.reset_noise({k: tuple(t.to(cuda_dev) for t in v) for k, v in noise.items()})
        assert torch.equal(mm.act_batch_values(su8), qr.act_batch_values(su8))
        assert torch.equal(mm.act_batch(su8), qr.act_batch(su8))
        assert mm.act(list(states[0])) == qr.act(list(states[0]))
    mm.train()
    bs, L, n, hist = 8, 14, cfg["n_step"], 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    inj = [dict(noises=oq.make_noises(seed + 10 * c, 18, N)) for c in range(chunks)]
    mm._inject = list(inj)
    pri = mm.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not mm._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(cfg["discount"] ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        loss, _ = om.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params),
                                (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx,
                                 torch.ones(hi - lo)), torch.ones(hi - lo), inj[c]["noises"], cfg, eps=eps)
        out.append(loss.numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    print("priorities rel err median / max", np.median(np.abs(pri - ref_p) / ref_p), np.max(np.abs(pri - ref_p) / ref_p))
    assert np.median(np.abs(pri - ref_p) / ref_p) < 2e-3 and np.max(np.abs(pri - ref_p) / ref_p) < 2e-2


@pytest.mark.gpu
def test_checkpoint_round_trip_either_loss(cuda_dev, tmp_path):
    import os
    from rainbow_iqn_apex_b200 import Agent, Learner
    from test_gpu_qr import _graph_batch
    B, N = 32, 51
    batch = _graph_batch(cuda_dev, B, 4)
    lr = Learner(_mmd_args(cuda_dev, B, N), 18, None)
    lr.train()
    lr.learn_on_batch(*batch)
    lr.save(str(tmp_path), 0, 1, "mmd.pth")
    path = os.path.join(tmp_path, "mmd.pth")
    ck = torch.load(path, map_location="cpu")
    assert ck["qr_dqn_quantiles"] == N and set(ck) == {"T_actors", "T_learner", "model_state_dict",
                                                      "optimiser_state_dict", "qr_dqn_quantiles"}
    for fields in (dict(), dict(mmd=0)):          # MMD checkpoint, fine-tuned as MMDQN or as QR-DQN
        back = Agent(_mmd_args(cuda_dev, B, N, model=path, **fields), 18, None)
        assert torch.equal(back.online_net._flat, lr.online_net._flat) and back.optimiser._step == 1
    with pytest.raises(ValueError, match="qr_dqn_quantiles = 51.*64"):
        Agent(_mmd_args(cuda_dev, B, 64, model=path), 18, None)


@pytest.mark.gpu
def test_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    for kw in (dict(mmd=2), dict(qr_dqn=0), dict(mmd_bandwidths="1 2"), dict(mmd_bandwidths=()),
               dict(mmd_bandwidths=(1.0, 0.0)), dict(mmd_bandwidths=(1.0,) * 17), dict(rainbow_only=1),
               dict(munchausen=1), dict(fqf=1), dict(risk_measure="cvar", risk_eta=0.25), dict(num_tau_samples=1)):
        with pytest.raises(ValueError):
            Agent(_mmd_args(cuda_dev, B, **kw), 18, None)
    ag = Learner(_mmd_args(cuda_dev, B, value_rescaling=1, random_shift=4, mmd_bandwidths=[0.5, 4]), 18, None)
    assert ag.mmd == (0.5, 4.0) and ag.value_rescaling == 1e-3 and ag.random_shift == 4 and ag.qr_dqn == 64
    for m, e in (("cvar", 0.25), ("wang", 0.5)):
        with pytest.raises(ValueError):
            ag.set_risk(m, e)
    assert ag.risk is None


@pytest.mark.gpu
def test_mmd_step_makes_the_qr_dqn_launches(cuda_dev):
    """An MMD learner step makes exactly QR-DQN's launches (one loss entry point in place of another)."""
    from test_gpu_qr import _bench_learner
    (s1, _, _, _), (s2, _, _, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f)
                                    for f in (dict(qr_dqn=1), dict(qr_dqn=1, mmd=1)))
    assert [c for _, _, c in s1] == [c for _, _, c in s2]


@pytest.mark.gpu
@pytest.mark.parametrize("base", [{}, dict(rainbow_only=1), dict(qr_dqn=1)])
def test_namespace_without_the_field_is_unchanged(cuda_dev, base):
    """IQN, C51 and QR-DQN learners from a namespace without mmd and with mmd = 0 run the same launches per step and
    give bit-identical sampled indices, losses and parameters."""
    from test_gpu_qr import _bench_learner
    (s1, p1, l1, _), (s2, p2, l2, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f)
                                        for f in (base, dict(base, mmd=0)))
    assert l1.mmd is None and l2.mmd is None
    for k, ((i1, x1, c1), (i2, x2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(x1, x2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)
