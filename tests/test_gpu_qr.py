"""QR-DQN (Dabney, Rowland, Bellemare & Munos, AAAI 2018): the fixed-fraction quantile head on the C51 network
(riqn_qr_head_fwd, riqn_qr_head_bwd, riqn_qr_head_bwd_dense) behind the optional Agent field qr_dqn.

The unmarked tests pin the oracle (oracle/qr.py) by identities, check its float64 and torch-fp32 statements against each
other, and check the host-side validation and the QR network's layout.  The gpu tests check every entry point against
float64 and against its numpy float32 statement on the operands it read (the method of test_gpu_c51_kernels.py), a
learner step, autograd and the actors against the torch oracle, reproducibility eagerly and from each captured step graph,
data parallelism, checkpoints, and that a namespace without the field runs exactly as before."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, load_params, make_args,
                     rel_err, to_dev)
from oracle import cases, network as net, qr as oq

F32 = np.float32


def _qr_args(dev, B, N=64, **kw):
    a = make_args(dev, B, cases.iqn_cfg(N, N, 32))
    a.qr_dqn = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("n,A", [(2, 1), (7, 4), (64, 18), (200, 18)])
def test_head_identities(n, A):
    """mean_a (q_i(., a) - v_i) = 0 for every i, Q is the mean of the quantiles, and the float32 statement of the head
    is within two roundings of float64."""
    rs = np.random.RandomState(n + A)
    B = 5
    zv, za = rs.standard_normal((B, n)), rs.standard_normal((B, A * n))
    q = oq.head_np(zv, za, A)
    qi = q.reshape(n, B, A)
    assert np.max(np.abs((qi - zv.T[:, :, None]).mean(2))) < 1e-14
    a3 = za.reshape(B, A, n)
    Q = zv.mean(1)[:, None] + a3.mean(2) - a3.mean(1).mean(1)[:, None]
    assert np.allclose(oq.q_values_np(q, B), Q, rtol=0, atol=1e-13)
    q32 = oq.head_f32_np(zv.astype(F32), za.astype(F32), A)
    q64 = oq.head_np(zv.astype(F32), za.astype(F32), A)
    assert np.all(np.abs(q32 - q64) <= 4 * U * (np.abs(zv).max() + (A + 2) * np.abs(za).max()))


@pytest.mark.parametrize("n", [2, 7, 64, 200, 256])
def test_fixed_fractions(n):
    """tau_hat_i = fl((2i+1)/(2N)) in the oracle and in the product's (N*B, 1) quantile-major array."""
    from rainbow_iqn_apex_b200 import qr
    from rainbow_iqn_apex_b200.model import DQN
    t32 = oq.fractions_f32(n)
    assert np.array_equal(t32, oq.fractions_np(n).astype(F32))
    assert np.all(np.diff(t32) > 0) and t32[0] > 0 and t32[-1] < 1
    d = DQN(_qr_args(torch.device("cpu"), 3, n), 4)
    t = qr.fractions(d, 3)
    assert t.shape == (3 * n, 1) and not t.requires_grad
    assert_bits("tau_hat", f32_bits(t.numpy().reshape(n, 3)), f32_bits(np.repeat(t32[:, None], 3, 1)))
    assert qr.fractions(d, 3) is t


@pytest.mark.parametrize("n,k", [(4, 1), (4, 2), (5, 3), (16, 4)])
def test_loss_subgradient_contains_zero_at_the_selected_order_statistics(n, k):
    """Against a target of N' = N*k equally weighted atoms and kappa -> 0, the loss is minimised quantile by quantile
    at the order statistic z_(m), m = ceil(tau_hat_i N'): 0 lies between the left and right derivatives there, and not
    below it; above it only where tau_hat_i N' is an integer, where [z_(m), z_(m+1)] minimises the loss."""
    rs = np.random.RandomState(n * 10 + k)
    Np = n * k
    z = np.sort(rs.uniform(-5, 5, Np))
    tau = oq.fractions_np(n)
    kappa, h = 2.0 ** -60, 1e-6          # kappa exact in float32 (the oracle loss rounds it there), far below h
    gap = np.min(np.diff(z))
    assert gap > 10 * h

    def d_i(i, x, side):
        th = np.zeros((1, n))
        th[0, i] = x
        base = oq.loss_np(th, z[None, :], kappa)[0]
        th[0, i] = x + side * h
        return side * (oq.loss_np(th, z[None, :], kappa)[0] - base) / h

    for i in range(n):
        m = int(math.ceil(tau[i] * Np - 1e-12))          # 1-indexed order statistic
        x = z[m - 1]
        left, right = d_i(i, x, -1), d_i(i, x, +1)
        assert left <= 1e-6 and right >= -1e-6, (i, m, left, right)
        if m >= 2:
            assert d_i(i, 0.5 * (z[m - 2] + z[m - 1]), +1) < -1e-3 / Np
        if m < Np:      # tau_hat_i N' an integer (k even): the loss is flat up to z_(m+1), which also minimises it
            flat = abs(tau[i] * Np - m) < 1e-9
            right_of = d_i(i, 0.5 * (z[m - 1] + z[m]), +1)
            assert abs(right_of) < 1e-6 if flat else right_of > 1e-3 / Np


@pytest.mark.parametrize("eps", [None, 1e-3])
def test_float64_and_torch_fp32_statements_agree(eps):
    B, A, n = 4, 4, 8
    cfg = cases.iqn_cfg(n, n, 8)
    params = oq.make_params(31, A, n)
    b = cases.make_batch(32, B, action_space=A)
    st, ac, rt, nx, nt = cases.batch_to_torch(b)
    noises = oq.make_noises(33, A, n)
    keep = {}
    loss, _ = oq.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params), (st, ac, rt, nx, nt),
                            torch.from_numpy(b["weights"]), noises, cfg, eps=eps, keep=keep)
    # the head on the torch statement's own z-layer outputs
    v, a = keep["v"].detach().numpy().reshape(B, n), keep["a"].detach().numpy().reshape(B, A * n)
    assert rel_err(keep["q_on"].detach().numpy(), oq.head_np(v, a, A)) < 1e-6
    assert np.array_equal(keep["a_star"].numpy(), oq.q_values_np(keep["q_sel"].numpy(), B).argmax(1)) or eps is not None
    tgt = oq.target_np(keep["q_tgt"].numpy(), keep["a_star"].numpy(), b["returns"], b["nonterminals"], 0.99 ** 3, eps)
    assert rel_err(keep["target"].numpy(), tgt) < 1e-6
    assert rel_err(loss.numpy(), oq.loss_np(keep["theta"].numpy(), tgt)) < 1e-6


@pytest.mark.parametrize("n", [64, 200])
def test_qr_state_dict_layout(n):
    """Host logic on CPU tensors only: the C51 layer set with z-layer widths N and A*N, the C51 parameter order, the
    arena views and [h_v | h_a] adjacency; fixed-fraction arguments are refused before any launch."""
    from rainbow_iqn_apex_b200.model import DQN
    d = DQN(_qr_args(torch.device("cpu"), 32, n), 18)
    sd = d.state_dict()
    shapes = oq.layer_shapes(18, n)
    assert set(sd) == set(shapes) and "iqn_fc.weight" not in sd
    for k, s in shapes.items():
        assert tuple(sd[k].shape) == s, k
    names = [nm for nm, _ in d.named_parameters()]
    expect = ["conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias"]
    for l in ("fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"):
        expect += [f"{l}.{p}" for p in ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma")]
    assert names == expect
    assert d.num_quantiles == n and d.qr_dqn and d._w_eff_z.shape == (19 * n, 512)
    hv, ha = d.fcnoisy_h_v.weight_mu, d.fcnoisy_h_a.weight_mu
    assert ha.data_ptr() == hv.data_ptr() + 4 * hv.numel()
    zv, za = d.fcnoisy_z_v.weight_mu, d.fcnoisy_z_a.weight_mu
    assert za.data_ptr() == zv.data_ptr() + 4 * zv.numel()
    d.zero_grad()
    assert all(p.grad.data_ptr() == d._flat_grad.data_ptr() + 4 * p._riqn_offset for p in d.parameters())
    p0 = d.conv1.weight.data_ptr()
    d.load_state_dict({k: torch.randn(s) for k, s in shapes.items()})
    assert d.conv1.weight.data_ptr() == p0 == d._flat.data_ptr() + 4 * d.conv1.weight._riqn_offset
    x = torch.zeros(2, 4, 84, 84, dtype=torch.uint8)
    for kw in (dict(tau=torch.full((2 * n, 1), 0.5)), dict(risk=("cvar", 0.5)), dict(log=True), dict(num_quantiles=8)):
        with torch.no_grad(), pytest.raises(ValueError):
            d(x, **kw)
    c51 = DQN(make_args(torch.device("cpu"), 32, rainbow_only=True), 18)
    assert [nm for nm, _ in c51.named_parameters()] == expect and not c51.qr_dqn and c51.num_quantiles is None


# ------------------------------------------------------------------------------------------------ kernels (GPU)
KERNEL_CASES = [(1, 1, 2), (5, 4, 7), (33, 32, 64), (512, 18, 200), (64, 18, 256), (4096, 4, 256), (7, 1, 200),
                (100, 32, 2), (1, 18, 64), (3000, 18, 7)]


def _operands(B, A, n, regime, seed):
    """zv (B, n), za (B, A*n).  "exact": multiples of 2^-4 below 2^6, with za's last action column chosen so that every
    sum over the actions is a multiple of A * 2^-4: each head operation is exact in fp32.  "random": normal values."""
    rs = np.random.RandomState(seed)
    if regime == "random":
        return rs.standard_normal((B, n)).astype(F32), (rs.standard_normal((B, A * n)) * 2).astype(F32)
    zv = (rs.randint(-512, 512, (B, n)) * 2.0 ** -4).astype(F32)
    za = rs.randint(-256, 256, (B, A, n)).astype(np.float64)
    if A > 1:
        target = rs.randint(-8, 8, (B, n)) * A
        za[:, A - 1, :] = target - za[:, :A - 1, :].sum(1)
    return zv, (za.reshape(B, A * n) * 2.0 ** -4).astype(F32)


def _fwd(dev, B, A, n, zv, za):
    o = Out(n * B * A, dev)
    zvd, zad = to_dev(zv, dev), to_dev(za, dev)         # held until the kernel has read them
    lib_call("riqn_qr_head_fwd", B, A, n, dptr(zvd), dptr(zad), o.p)
    torch.cuda.synchronize()
    assert_canaries({"q": o})
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,A,n", KERNEL_CASES)
def test_qr_head_fwd(cuda_dev, B, A, n, regime):
    zv, za = _operands(B, A, n, regime, B * 7 + A * 3 + n)
    o = _fwd(cuda_dev, B, A, n, zv, za)
    got = o.f32().reshape(n * B, A)
    assert_bits("q vs float32 statement", o.bits(), f32_bits(oq.head_f32_np(zv, za, A)).ravel())
    ref = oq.head_np(zv, za, A)
    if regime == "exact":
        assert_bits("q vs float64", f32_bits(got), f32_bits(ref.astype(F32)))
    else:
        a = np.abs(za.reshape(B, A, n).astype(np.float64))
        scale = np.abs(zv.astype(np.float64)).T[:, :, None] + a.transpose(2, 0, 1) + a.transpose(2, 0, 1).mean(2, keepdims=True)
        check_bound("q", got, ref, 2.0 * (A + 3) * U * scale.reshape(n * B, A))
    assert_bits("second call", _fwd(cuda_dev, B, A, n, zv, za).bits(), o.bits())


def _bwd_operands(B, A, n, regime, seed):
    rs = np.random.RandomState(seed)
    acts = rs.randint(0, A, B).astype(np.int64)
    if regime == "random":
        return (rs.standard_normal(n * B).astype(F32), rs.uniform(0.1, 1, B).astype(F32), acts,
                rs.standard_normal((n * B, A)).astype(F32))
    dth = (rs.randint(-64, 64, n * B) * 2.0 ** -8).astype(F32)
    gs = (rs.randint(1, 16, B) * 2.0 ** -4).astype(F32)
    G = rs.randint(-128, 128, (n * B, A)).astype(np.float64)
    if A > 1:
        G[:, A - 1] = rs.randint(-8, 8, n * B) * A - G[:, :A - 1].sum(1)
    return dth, gs, acts, (G * 2.0 ** -6).astype(F32)


def _bwd(dev, B, A, n, dth, gs, gmul, acts, G=None):
    dzv, dza = Out(B * n, dev), Out(B * A * n, dev)
    if G is None:
        # operands held in locals until the kernel has read them
        dthd, gsd, actd = to_dev(dth, dev), None if gs is None else to_dev(gs, dev), to_dev(acts, dev, torch.int64)
        lib_call("riqn_qr_head_bwd", B, A, n, dptr(dthd), dptr(gsd), float(gmul), dptr(actd), dzv.p, dza.p)
    else:
        Gd = to_dev(G, dev)
        lib_call("riqn_qr_head_bwd_dense", B, A, n, dptr(Gd), dzv.p, dza.p)
    torch.cuda.synchronize()
    assert_canaries({"dzv": dzv, "dza": dza})
    return dzv, dza


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,A,n", KERNEL_CASES)
def test_qr_head_bwd_one_hot(cuda_dev, B, A, n, regime):
    """Against float64 (bit for bit in the exact regime, where 1/A is a power of two), bit for bit against
    riqn_c51_head_bwd on dq = dtheta^T, and twice alike."""
    dth, gs, acts, _ = _bwd_operands(B, A, n, regime, B + 5 * A + n)
    gmul = 1.0 / 32 if regime == "exact" else 1.0 / B
    dzv, dza = _bwd(cuda_dev, B, A, n, dth, gs, gmul, acts)
    w = gs.astype(np.float64) * F32(gmul)
    g = dth.reshape(n, B).T.astype(np.float64) * w[:, None]                           # (B, n)
    onehot = (np.arange(A)[None, :] == acts[:, None]).astype(np.float64)               # (B, A)
    ref_za = (g[:, None, :] * (onehot[:, :, None] - 1.0 / A)).reshape(B, A * n)
    if regime == "exact":
        assert_bits("dzv vs float64", dzv.bits(), f32_bits(g.astype(F32)).ravel())
        if A & (A - 1) == 0:
            assert_bits("dza vs float64", dza.bits(), f32_bits(ref_za.astype(F32)).ravel())
    check_bound("dzv", dzv.f32(), g.ravel(), 2 * U * np.abs(g).ravel())
    check_bound("dza", dza.f32(), ref_za.ravel(), 4 * U * np.abs(np.repeat(g, A, 0).reshape(B, A * n)).ravel() + 1e-45)
    # riqn_c51_head_bwd on dq (B, n) = dtheta^T: the same bits
    cz, ca = Out(B * n, cuda_dev), Out(B * A * n, cuda_dev)
    dqd = to_dev(np.ascontiguousarray(dth.reshape(n, B).T), cuda_dev)
    gsd, actd = to_dev(gs, cuda_dev), to_dev(acts, cuda_dev, torch.int64)
    lib_call("riqn_c51_head_bwd", B, A, n, dptr(dqd), dptr(gsd), float(gmul), dptr(actd), cz.p, ca.p)
    torch.cuda.synchronize()
    assert_bits("dzv vs c51", dzv.bits(), cz.bits())
    assert_bits("dza vs c51", dza.bits(), ca.bits())
    d2v, d2a = _bwd(cuda_dev, B, A, n, dth, gs, gmul, acts)
    assert_bits("second call dzv", d2v.bits(), dzv.bits())
    assert_bits("second call dza", d2a.bits(), dza.bits())


@pytest.mark.gpu
def test_qr_head_bwd_without_gscale_uses_gscale_mul(cuda_dev):
    B, A, n = 9, 4, 7
    dth, gs, acts, _ = _bwd_operands(B, A, n, "exact", 3)
    a = _bwd(cuda_dev, B, A, n, dth, None, 0.25, acts)
    b = _bwd(cuda_dev, B, A, n, dth, np.ones(B, F32), 0.25, acts)
    assert_bits("dzv", a[0].bits(), b[0].bits())
    assert_bits("dza", a[1].bits(), b[1].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "random"])
@pytest.mark.parametrize("B,A,n", KERNEL_CASES)
def test_qr_head_bwd_dense(cuda_dev, B, A, n, regime):
    _, _, _, G = _bwd_operands(B, A, n, regime, 3 * B + A + 11 * n)
    dzv, dza = _bwd(cuda_dev, B, A, n, None, None, 1.0, None, G)
    G3 = G.reshape(n, B, A).astype(np.float64)
    ref_v = G3.sum(2).T                                                                 # (B, n)
    ref_a = (G3.transpose(1, 2, 0) - ref_v[:, None, :] / A).reshape(B, A * n)
    # numpy float32 statement: fp32 adds over a ascending from 0, then G - fl(s / A)
    s = np.zeros((n, B), F32)
    for k in range(A):
        s = (s + G.reshape(n, B, A)[:, :, k]).astype(F32)
    st_a = (G.reshape(n, B, A).transpose(1, 2, 0) - (s.T / F32(A)).astype(F32)[:, None, :]).astype(F32)
    assert_bits("dzv vs float32 statement", dzv.bits(), f32_bits(s.T).ravel())
    assert_bits("dza vs float32 statement", dza.bits(), f32_bits(st_a).ravel())
    if regime == "exact":
        assert_bits("dzv vs float64", dzv.bits(), f32_bits(ref_v.astype(F32)).ravel())
        assert_bits("dza vs float64", dza.bits(), f32_bits(ref_a.astype(F32)).ravel())
    else:
        absum = np.abs(G3).sum(2).T
        check_bound("dzv", dzv.f32(), ref_v.ravel(), 2 * A * U * absum.ravel())
        check_bound("dza", dza.f32(), ref_a.ravel(),
                    (4 * U * (np.abs(G3.transpose(1, 2, 0)) + absum[:, None, :]) + 2 * U * absum[:, None, :]).ravel())
    d2v, d2a = _bwd(cuda_dev, B, A, n, None, None, 1.0, None, G)
    assert_bits("second call dzv", d2v.bits(), dzv.bits())
    assert_bits("second call dza", d2a.bits(), dza.bits())


@pytest.mark.gpu
def test_entry_points_reject_invalid_shapes_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    src = torch.zeros(300 * 300 * 4, device=dev)
    act = torch.zeros(64, dtype=torch.int64, device=dev)
    big = Out(300 * 300 * 4, dev)
    big2 = Out(300 * 300 * 4, dev)
    for B, A, n in ((4, 4, 1), (4, 4, 0), (4, 4, 257), (4, 4, -2), (4, 0, 8), (4, 33, 8), (4, -1, 8), (0, 4, 8),
                    (-3, 4, 8)):
        with pytest.raises(RiqnError):
            lib_call("riqn_qr_head_fwd", B, A, n, dptr(src), dptr(src), big.p)
        with pytest.raises(RiqnError):
            lib_call("riqn_qr_head_bwd", B, A, n, dptr(src), dptr(src), 1.0, dptr(act), big.p, big2.p)
        with pytest.raises(RiqnError):
            lib_call("riqn_qr_head_bwd_dense", B, A, n, dptr(src), big.p, big2.p)
    torch.cuda.synchronize()
    for o in (big, big2):
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def _qr_learner(dev, B, N, params, **kw):
    from rainbow_iqn_apex_b200 import Learner
    lr = Learner(_qr_args(dev, B, N, **kw), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    return lr


def _relu_flips(gk, keep):
    """ReLU units that the product and the oracle put on opposite sides of 0: conv1-3, then h_v, h_a."""
    h = gk["h"].cpu()
    return [int(((x.cpu() > 0) != (y > 0)).sum()) for x, y in
            ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
             (h[:, :512], keep["h_v"]), (h[:, 512:], keep["h_a"]))]


def _check_step(loss, dbg, grads, o_loss, o_grads, keep, B, tie_tol=1e-4):
    """Per-transition loss within 1e-3 relative and every gradient at cosine >= 0.999, except where the double-DQN argmax
    is a near tie (the oracle's top-2 Q within tie_tol) or a ReLU kink flips, which relax the parameters upstream of it."""
    qv = keep["qv_next"].numpy()
    top2 = np.sort(qv, axis=1)[:, -2:]
    tie = (top2[:, 1] - top2[:, 0]) < tie_tol
    a_gpu = dbg["a_star"].cpu().numpy()
    ok = a_gpu == keep["a_star"].numpy()
    assert np.all(ok | tie)
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    err = np.abs(lg - lo) / np.abs(lo)
    assert np.max(err[ok]) < 1e-3, float(np.max(err[ok]))
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
    print(f"B={B}: max loss rel err {np.max(err[ok]):.3g}, min cos {worst:.6f}, ReLU flips {fl}, ties {int(tie.sum())}")


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("B,N", [(32, 64), (512, 64), (32, 200), (512, 200)])
def test_learner_step_vs_oracle(cuda_dev, B, N, eps):
    from test_gpu_learn import _dev_batch
    cfg, seed = cases.iqn_cfg(N, N, 32), 9500 + B + N
    params = oq.make_params(seed, 18, N)
    torch.manual_seed(seed)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    lr = _qr_learner(cuda_dev, B, N, params, **kw)
    assert lr.qr_dqn == N and lr.value_rescaling == eps
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    if eps is not None:
        b["returns"] = (b["returns"] * 40).astype(F32)              # unclipped-scale returns
    noises = oq.make_noises(seed + 3, 18, N)
    lr._inject = dict(noises=noises)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    for k in ("a_star", "theta", "target", "q_sel", "q_tgt", "q_on"):
        assert k in dbg and bool(torch.isfinite(dbg[k].float()).all()), k
    # the product's loss kernel on its own operands: theta, target and the quantile-major tau_hat
    q_on = dbg["q_on"].cpu().numpy()
    assert np.array_equal(dbg["theta"].cpu().numpy(), q_on.reshape(N, B, 18)[:, np.arange(B), b["actions"]].T)
    tgt = oq.target_np(dbg["q_tgt"].cpu().numpy(), dbg["a_star"].cpu().numpy(), b["returns"], b["nonterminals"],
                       cfg["discount"] ** cfg["n_step"], eps)
    assert rel_err(dbg["target"].cpu().numpy(), tgt) < 1e-6
    assert rel_err(loss.detach().cpu().numpy(), oq.loss_np(dbg["theta"].cpu().numpy(), tgt)) < 1e-5
    assert_bits("tau_hat", f32_bits(dbg["tau"].cpu().numpy().reshape(N, B)),
                f32_bits(np.repeat(oq.fractions_f32(N)[:, None], B, 1)))
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_grads = oq.learn_step(p_on, p_tg, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises, cfg,
                                    eps=eps, keep=keep)
    _check_step(loss, dbg, grads, o_loss, o_grads, keep, B, tie_tol=1e-4 if eps is None else 1e-3)


@pytest.mark.gpu
def test_autograd_of_a_torch_written_loss(cuda_dev):
    """net(x) returns (q, tau) as one autograd node; .backward() of a quantile loss written in torch on q goes through
    riqn_qr_head_bwd_dense into the layer backwards and matches the oracle's autograd."""
    from rainbow_iqn_apex_b200.model import DQN
    B, N, A = 32, 64, 18
    params = oq.make_params(77, A, N)
    torch.manual_seed(77)
    d = DQN(_qr_args(cuda_dev, B, N), A).to(cuda_dev)
    load_params(d, params)
    d.train()
    noise = oq.make_noises(78, A, N, count=1)[0]
    d.reset_noise({k: tuple(t.to(cuda_dev) for t in v) for k, v in noise.items()})
    b = cases.make_batch(79, B)
    x = torch.from_numpy(b["states"]).to(cuda_dev)
    rs = np.random.RandomState(80)
    target = torch.from_numpy(rs.standard_normal((B, N)).astype(F32))
    acts = torch.from_numpy(b["actions"] % A)

    def torch_loss(q, tau):
        th = q.view(N, B, A)[:, torch.arange(B, device=q.device), acts.to(q.device)].t()
        dl = target.to(q.device)[:, :, None] - th[:, None, :]
        t = tau.view(N, B).t()[:, None, :]
        hub = torch.where(dl.abs() <= 1.0, 0.5 * dl * dl, dl.abs() - 0.5)
        return ((t - (dl.detach() < 0).float()).abs() * hub).sum(2).mean(1).mean()

    d.zero_grad()
    q, tau = d(x)
    assert q.grad_fn is not None and not tau.requires_grad and q.shape == (N * B, A)
    torch_loss(q, tau).backward()
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().clone() for k, p in d.named_parameters()}
    p = net.to_torch(params, requires_grad=True)
    net.apply_noise(p, noise)
    keep = {}
    q_o = oq.dqn_forward_qr(p, cases.batch_to_torch(b)[0], A, N, keep=keep)
    torch_loss(q_o, torch.from_numpy(oq.fractions_f32(N)).repeat_interleave(B)).backward()
    assert rel_err(q.detach().cpu().numpy(), q_o.detach().numpy()) < 2e-3
    for k, t in p.items():
        if t.requires_grad:
            c = _cos(got[k], t.grad)
            assert c > 0.999, (k, c)


def _bench_learner(dev, cap, graph, steps, fields=None):
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib
    torch.manual_seed(5)
    a = bench.make_args(dev, cap)
    for k, v in (fields or {}).items():
        setattr(a, k, v)
    learner = Learner(a, bench.ACTIONS, None)
    learner.train()
    mem = ReplayMemory(a, None)
    bench.fill_replay(mem, cap, dev, 7)
    if graph:
        learner.enable_cuda_graph(mem)
    out = []
    for _ in range(steps):
        c0 = _lib.launch_count()
        idxs, loss = learner.learn_and_update(mem)
        out.append((idxs.clone(), loss.clone(), _lib.launch_count() - c0))
    torch.cuda.synchronize()
    return out, learner.online_net._flat.detach().clone(), learner, mem


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_qr_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    """Two consecutive steps at B = 512 (the benchmark's learner with qr_dqn = 1), eagerly and replayed from the step
    graph, twice alike."""
    runs = [_bench_learner(cuda_dev, 1 << 14, graph, 2, dict(qr_dqn=1)) for _ in range(2)]
    (s1, p1, l1, _), (s2, p2, _, _) = runs
    assert l1.qr_dqn == 64 and l1.batch_size == 512
    for k, ((i1, x1, _), (i2, x2, _)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(x1, x2), k
        assert bool(torch.isfinite(x1).all())
    assert torch.equal(p1, p2)


def _graph_batch(dev, B, seed):
    b = cases.make_batch(seed, B)
    return tuple(torch.from_numpy(b[k]).to(dev) for k in
                 ("states", "actions", "returns", "next_states", "nonterminals", "weights"))


@pytest.mark.gpu
def test_batch_and_learn_graphs_are_bitwise_reproducible(cuda_dev):
    """Two steps replayed from the batch graph (host minibatches) and from the learn graph (Ape-X), twice alike."""
    import bench
    B = 512
    batches = [_graph_batch(cuda_dev, B, s) for s in (61, 62)]

    def batch_graph_run():
        _, _, lr, mem = _bench_learner(cuda_dev, 1 << 14, True, 1, dict(qr_dqn=1))
        lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(B)))
        hosts = [tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(B)) for _ in range(2)]
        out = [lr.learn_on_host_batch(h).clone() for h in hosts]
        torch.cuda.synchronize()
        return out, lr.online_net._flat.clone()

    def learn_graph_run():
        torch.manual_seed(9)
        a = bench.make_args(cuda_dev, 1 << 14)
        a.qr_dqn = 1
        from rainbow_iqn_apex_b200 import Learner
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


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_half_batches_equal_one_learner(cuda_dev):
    """Two half-batch replicas, each scaled by grad_scale = 1/2, sum to the gradients of one learner on the concatenated
    batch; and a one-rank process group takes the all-reduce path with the same bits as no group."""
    import torch.distributed as dist
    from test_gpu_learn import _dev_batch
    B, N = 64, 64
    b = cases.make_batch(12, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    params = oq.make_params(12, 18, N)
    noises = oq.make_noises(13, 18, N)

    def grads_of(sl, scale):
        torch.manual_seed(1)
        lr = _qr_learner(cuda_dev, sl.stop - sl.start, N, params)
        lr._inject = dict(noises=noises)
        lr.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl] * scale)
        torch.cuda.synchronize()
        return lr.online_net._flat_grad.clone()

    full = grads_of(slice(0, B), 1.0)
    halves = grads_of(slice(0, B // 2), 0.5) + grads_of(slice(B // 2, B), 0.5)
    err = float((halves - full).abs().max() / full.abs().max())
    print(f"data parallel: max |sum of half-batch grads - full| / max |full| = {err:.3g}")
    assert err < 2e-3
    cos = _cos(halves, full)
    assert cos > 0.99999, cos
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        out = []
        for dp in (False, True):
            torch.manual_seed(1)
            lr = _qr_learner(cuda_dev, B, N, params)
            if dp:
                from rainbow_iqn_apex_b200 import parallel
                parallel.make_data_parallel(lr)
                lr.process_group = dist.group.WORLD
            losses_ = [lr.learn_on_batch(st, ac, rt, nx, nt, w).clone() for _ in range(2)]
            torch.cuda.synchronize()
            out.append((losses_, lr.online_net._flat.clone()))
        assert all(torch.equal(x, y) for x, y in zip(out[0][0], out[1][0]))
        assert torch.equal(out[0][1], out[1][1])
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
def test_actor_paths_vs_oracle(cuda_dev, eps):
    """act / act_batch / act_batch_values act on mean_i q_i (under value rescaling mean_i h^-1(q_i)), and
    compute_priorities runs the QR loss."""
    from rainbow_iqn_apex_b200 import Actor
    N, E, seed = 32, 8, 9700
    cfg = cases.iqn_cfg(N, N, 8)
    params = oq.make_params(seed, 18, N)
    torch.manual_seed(seed)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    actor = Actor(_qr_args(cuda_dev, 8, N, **kw), 18, None)
    load_params(actor.online_net, params)
    actor.update_target_net()
    actor.eval()                      # eval: the mu weights alone, so the oracle needs no noise
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    qv = actor.act_batch_values(su8).cpu().numpy()
    ref = oq.act_values(net.to_torch(params), torch.from_numpy(states).float().div_(255), 18, N, eps=eps,
                        training=False).numpy()
    assert rel_err(qv, ref) < 5e-3
    with pytest.raises(ValueError):
        actor.act_batch_values(su8, tau=torch.full((N * E, 1), 0.5, device=cuda_dev))
    a = actor.act_batch(su8).cpu().numpy()
    top2 = np.sort(ref, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-3 * max(1.0, float(np.abs(ref).max()))
    assert np.array_equal(a[clear], ref.argmax(1)[clear]) and np.array_equal(a, qv.argmax(1))
    assert clear.sum() >= E // 2
    for e in range(E):
        if clear[e]:
            assert actor.act(list(states[e])) == int(a[e])
            break
    actor.train()
    bs, L, n, hist = 8, 14, cfg["n_step"], 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    inj = [dict(noises=oq.make_noises(seed + 10 * c, 18, N)) for c in range(chunks)]
    actor._inject = list(inj)
    pri = actor.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not actor._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(cfg["discount"] ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        loss, _ = oq.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params),
                                (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx,
                                 torch.ones(hi - lo)), torch.ones(hi - lo), inj[c]["noises"], cfg, eps=eps)
        out.append(loss.numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    assert np.median(np.abs(pri - ref_p) / ref_p) < 1e-3 and np.max(np.abs(pri - ref_p) / ref_p) < 2e-2


@pytest.mark.gpu
def test_checkpoint_round_trip_and_mismatches(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B, N = 32, 51
    batch = _graph_batch(cuda_dev, B, 4)
    lr = Learner(_qr_args(cuda_dev, B, N), 18, None)
    lr.train()
    lr.learn_on_batch(*batch)
    lr.save(str(tmp_path), 0, 1, "qr.pth")
    path = os.path.join(tmp_path, "qr.pth")
    ck = torch.load(path, map_location="cpu")
    assert ck["qr_dqn_quantiles"] == N and set(ck["model_state_dict"]) == set(oq.layer_shapes(18, N))
    back = Agent(_qr_args(cuda_dev, B, N, model=path), 18, None)
    assert torch.equal(back.online_net._flat, lr.online_net._flat) and back.optimiser._step == 1
    # N = atoms = 51: the QR network has the C51 network's shapes; the checkpoint field tells them apart
    c51_args = make_args(cuda_dev, B, rainbow_only=True)
    c51_args.model = path
    with pytest.raises(ValueError, match="qr_dqn_quantiles = 51.*None"):
        Agent(c51_args, 18, None)
    with pytest.raises(ValueError, match="qr_dqn_quantiles = 51.*64"):
        Agent(_qr_args(cuda_dev, B, 64, model=path), 18, None)
    c51_args.model = None
    Agent(c51_args, 18, None).save(str(tmp_path), 0, 1, "c51.pth")
    assert "qr_dqn_quantiles" not in torch.load(os.path.join(tmp_path, "c51.pth"), map_location="cpu")
    with pytest.raises(ValueError, match="qr_dqn_quantiles = None.*51"):
        Agent(_qr_args(cuda_dev, B, N, model=os.path.join(tmp_path, "c51.pth")), 18, None)


@pytest.mark.gpu
def test_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    for kw in (dict(qr_dqn=2), dict(num_tau_samples=1), dict(num_tau_samples=257), dict(rainbow_only=1),
               dict(munchausen=1), dict(fqf=1), dict(risk_measure="cvar", risk_eta=0.25), dict(munchausen=1,
                                                                                                value_rescaling=1)):
        with pytest.raises(ValueError):
            Agent(_qr_args(cuda_dev, B, **kw), 18, None)
    with pytest.raises(ValueError):
        Agent(_qr_args(cuda_dev, B), 33, None)
    ag = Learner(_qr_args(cuda_dev, B, value_rescaling=1), 18, None)
    assert ag.qr_dqn == 64 and ag.value_rescaling == 1e-3 and ag.num_tau_samples == 64
    ag.set_risk("neutral")
    for m, e in (("cvar", 0.25), ("wang", 0.5)):
        with pytest.raises(ValueError):
            ag.set_risk(m, e)
    assert ag.risk is None
    a = make_args(cuda_dev, B)
    del a.num_tau_prime_samples, a.num_quantile_samples, a.quantile_embedding_dim
    a.qr_dqn, a.atoms, a.V_min, a.V_max = 1, None, None, None          # not read under QR-DQN
    assert Agent(a, 18, None).qr_dqn == 64


@pytest.mark.gpu
@pytest.mark.parametrize("c51", [False, True])
def test_namespace_without_the_field_is_unchanged(cuda_dev, c51):
    """IQN and C51 learners from a namespace without qr_dqn and with qr_dqn = 0 run the same launches per step and give
    bit-identical sampled indices, losses and parameters."""
    base = dict(rainbow_only=1) if c51 else {}
    (s1, p1, _, _), (s2, p2, _, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f) for f in (base, dict(base, qr_dqn=0)))
    for k, ((i1, l1, c1), (i2, l2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(l1, l2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)
