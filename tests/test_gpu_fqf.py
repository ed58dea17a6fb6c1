"""FQF (Yang et al., NeurIPS 2019): a learned fraction proposal network and its 1-Wasserstein fraction loss
(riqn_fqf_fractions, riqn_fqf_fraction_bwd, riqn_fqf_fraction_wgrad, riqn_argmax_weighted) behind the optional Agent
fields fqf, fqf_fraction_lr and fqf_entropy_coef.

The unmarked tests pin the float64 oracle (oracle/fqf.py) by identities, check the torch-fp32 oracle against it, and check
the host-side validation and the unchanged DQN layout.  The gpu tests check every entry point against float64 on the
operands it read, a learner step and the actors against the torch oracle, reproducibility eagerly and from the captured
step graph, data parallelism, checkpoints, and that a namespace without the fields issues exactly the launches of plain
IQN."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from helpers import load_params, make_args, rel_err
from oracle import cases, fqf as of, network as net

PAD = 64
CANARY = -77.0


def _fqf_args(dev, B, cfg, **kw):
    a = make_args(dev, B, cfg)
    a.fqf = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("N", [2, 7, 64, 256])
def test_zero_logits_give_uniform_fractions(N):
    fr = of.fractions_np(np.zeros((3, N)))
    i = np.arange(N + 1)
    assert np.allclose(fr["tau"], i / N, rtol=0, atol=1e-15)
    assert np.allclose(fr["tau_hat"], (2 * np.arange(N) + 1) / (2 * N), rtol=0, atol=1e-15)
    assert np.allclose(fr["dtau"], 1.0 / N, rtol=0, atol=1e-15)
    assert np.allclose(fr["entropy"], math.log(N), rtol=1e-15)
    q = np.random.RandomState(N).standard_normal((3, N, 5))
    assert np.allclose((fr["dtau"][:, :, None] * q).sum(1), q.mean(1), rtol=0, atol=1e-14)


@pytest.mark.parametrize("fn", ["cubic", "probit"])
def test_w1_gradient_is_proposition_1(fn):
    """Central differences of the quadrature W1 in each inner fraction match 2F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1})."""
    from scipy.stats import norm
    F = {"cubic": lambda t: t ** 3 + t, "probit": lambda t: norm.ppf(0.01 + 0.98 * t)}[fn]
    rs = np.random.RandomState(3)
    N = 8
    tau = of.fractions_np(rs.standard_normal((1, N)))["tau"][0]
    th = 0.5 * (tau[:-1] + tau[1:])
    g = 2 * F(tau[1:N]) - F(th[1:]) - F(th[:-1])
    h = 1e-5
    for i in range(1, N):
        tp, tm = tau.copy(), tau.copy()
        tp[i] += h
        tm[i] -= h
        fd = (of.w1_np(F, tp) - of.w1_np(F, tm)) / (2 * h)
        assert abs(fd - g[i - 1]) <= 1e-6 * abs(g[i - 1]), (i, fd, g[i - 1])


@pytest.mark.parametrize("lam", [0.0, 0.01, 1.0])
def test_analytic_fraction_backward_is_autograd_of_the_surrogate(lam):
    rs = np.random.RandomState(5)
    B, N = 6, 12
    logits = rs.standard_normal((B, N)) * 2
    f_bnd, f_hat = rs.standard_normal((B, N - 1)), rs.standard_normal((B, N))
    w = rs.uniform(0.1, 1, B)
    d, loss = of.fraction_bwd_np(logits, f_bnd, f_hat, w, lam)
    lt = torch.tensor(logits, dtype=torch.float64, requires_grad=True)
    tau, _, _, H = of.fractions_torch(lt)
    g = torch.tensor(of.w1_grad_np(f_bnd, f_hat))
    L = (g * tau[:, 1:N]).sum(1) - lam * H
    (torch.tensor(w) * L).sum().backward()
    assert np.max(np.abs(d - lt.grad.numpy())) <= 1e-12 * max(1.0, np.max(np.abs(d)))
    assert np.max(np.abs(loss - L.detach().numpy())) <= 1e-12 * max(1.0, np.max(np.abs(loss)))


def test_torch_fp32_fractions_agree_with_float64():
    rs = np.random.RandomState(6)
    logits = (rs.standard_normal((16, 64)) * 3).astype(np.float32)
    fr = of.fractions_np(logits)
    tau, th, dt, H = of.fractions_torch(torch.from_numpy(logits))
    for a, b in ((tau, fr["tau"]), (th, fr["tau_hat"]), (dt, fr["dtau"])):
        assert np.max(np.abs(a.numpy() - b)) < 1e-6
    assert rel_err(H.numpy(), fr["entropy"]) < 1e-6


def test_dqn_layout_is_unchanged_under_fqf():
    """The DQN's state_dict keys, parameter order and census do not see the fraction proposal, which has its own arena."""
    from rainbow_iqn_apex_b200.fqf import FractionProposal
    from rainbow_iqn_apex_b200.model import DQN
    args = _fqf_args(torch.device("cpu"), 32, None)
    d = DQN(args, 18)
    shapes = net.layer_shapes(18)
    assert set(d.state_dict()) == set(shapes)
    assert sum(p.numel() for p in d.parameters()) == 6725894
    assert [n for n, _ in d.named_parameters()][:2] == ["conv1.weight", "conv1.bias"]
    torch.manual_seed(0)
    f = FractionProposal(64, "cpu")
    assert set(f.state_dict()) == {"weight", "bias"} and f.weight.shape == (64, 3136)
    bound = 0.01 * math.sqrt(6.0 / (3136 + 64))
    wmax = float(f.weight.detach().abs().max())
    assert 0.5 * bound < wmax <= bound and float(f.bias.detach().abs().max()) == 0.0
    assert all(p.data_ptr() == f._flat.data_ptr() + 4 * p._riqn_offset for p in f.parameters())
    assert f._flat.data_ptr() != d._flat.data_ptr()


# ------------------------------------------------------------------------------------------------ kernels (GPU)
def _buf(dev, n, fill=math.nan, dtype=torch.float32):
    """A device buffer of n elements prefilled with ``fill`` and followed by PAD canaries; returns (full, view)."""
    full = torch.full((n + PAD,), fill, dtype=dtype, device=dev)
    full[n:] = CANARY if dtype.is_floating_point else -7
    return full, full[:n]


def _canaries_ok(full, n):
    c = full[n:].cpu()
    return bool((c == (CANARY if c.dtype.is_floating_point else -7)).all())


def _fractions(dev, logits):
    from rainbow_iqn_apex_b200._lib import call, ptr
    B, N = logits.shape
    lg = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).to(dev)
    bufs = [_buf(dev, B * (N + 1)), _buf(dev, N * B), _buf(dev, N * B), _buf(dev, B)]
    call("riqn_fqf_fractions", B, N, ptr(lg), *(ptr(v) for _, v in bufs))
    torch.cuda.synchronize()
    for (full, v) in bufs:
        assert _canaries_ok(full, v.numel())
    tau, th, dt, H = (v.cpu().numpy() for _, v in bufs)
    return tau.reshape(B, N + 1), th.reshape(N, B).T, dt.reshape(N, B).T, H


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,scale", [(512, 64, 1.0), (3, 2, 5.0), (37, 256, 0.3), (33, 7, 20.0)])
def test_fractions_vs_float64(cuda_dev, B, N, scale):
    logits = (np.random.RandomState(B + N).standard_normal((B, N)) * scale).astype(np.float32)
    tau, th, dt, H = _fractions(cuda_dev, logits)
    for a in (tau, th, dt, H):
        assert np.all(np.isfinite(a))
    assert np.all(tau[:, 0] == 0.0) and np.all(tau[:, N] == 1.0)                # bitwise
    assert np.all(np.diff(tau, axis=1) >= 0) and np.all(dt >= 0)
    assert np.all((th >= 0) & (th <= 1))
    eps32 = np.finfo(np.float32).eps
    assert np.all(np.abs(dt.astype(np.float64).sum(1) - 1.0) <= N * eps32)      # sum of dtau = 1 within N ulp
    ref = of.fractions_np(logits)
    # tau_i = fl(c_i / S) with c_i, S in double: one rounding of a value <= 1 (plus double error far below it)
    assert np.all(np.abs(tau - ref["tau"]) <= 0.5 * eps32 * np.maximum(ref["tau"], 2.0 ** -126) + 1e-15)
    assert np.all(np.abs(th - ref["tau_hat"]) <= 2 * eps32 * ref["tau_hat"] + 1e-15)
    assert np.all(np.abs(dt - ref["dtau"]) <= 2 * eps32 + 1e-15)
    assert rel_err(H, ref["entropy"]) < 1e-6
    again = _fractions(cuda_dev, logits)
    for a, b in zip((tau, th, dt, H), again):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_fractions_extreme_logits_are_finite(cuda_dev):
    """Logits of +-80 and one dominant entry: the other P_k underflow float, giving dtau == 0 and no NaN."""
    B, N = 8, 32
    lg = np.zeros((B, N), np.float32)
    lg[0] = np.where(np.arange(N) % 2, 80.0, -80.0)
    lg[1] = -80.0
    lg[1, 5] = 80.0
    lg[2] = -80.0
    lg[3, -1] = 200.0
    lg[4] = np.linspace(-80, 80, N)
    tau, th, dt, H = _fractions(cuda_dev, lg)
    for a in (tau, th, dt, H):
        assert np.all(np.isfinite(a))
    assert np.all(tau[:, -1] == 1.0) and np.all(tau[:, 0] == 0.0) and np.all(np.diff(tau, axis=1) >= 0)
    assert dt[1, 5] == 1.0 and np.all(np.delete(dt[1], 5) == 0.0)
    assert dt[3, -1] == 1.0 and abs(H[3]) < 1e-6
    assert np.allclose(dt[2], 1.0 / N) and abs(H[2] - math.log(N)) < 1e-6


def _bwd_case(seed, B, N, A):
    rs = np.random.RandomState(seed)
    return dict(logits=(rs.standard_normal((B, N)) * 2).astype(np.float32),
                q_hat=rs.standard_normal((N * B, A)).astype(np.float32),
                q_bnd=rs.standard_normal(((N - 1) * B, A)).astype(np.float32),
                actions=rs.randint(0, A, B).astype(np.int64), gscale=rs.uniform(0.1, 1, B).astype(np.float32))


def _bwd(dev, c, B, N, A, mul, lam, tau=None, prefill=math.nan):
    from rainbow_iqn_apex_b200._lib import call, ptr
    d = {k: torch.from_numpy(v).to(dev) for k, v in c.items()}
    if tau is None:
        tau = torch.from_numpy(_fractions(dev, c["logits"])[0]).to(dev)
    dl, loss = _buf(dev, B * N, prefill), _buf(dev, B, prefill)
    call("riqn_fqf_fraction_bwd", B, N, A, ptr(d["logits"]), ptr(tau), ptr(d["q_hat"]), ptr(d["q_bnd"]), ptr(d["actions"]),
         ptr(d["gscale"]), float(mul), float(lam), ptr(dl[1]), ptr(loss[1]))
    torch.cuda.synchronize()
    assert _canaries_ok(dl[0], B * N) and _canaries_ok(loss[0], B)
    return dl[1].cpu().numpy().reshape(B, N), loss[1].cpu().numpy(), tau.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,A,lam", [(512, 64, 18, 0.0), (5, 2, 4, 0.5), (9, 256, 32, 0.01), (17, 33, 1, 1.0)])
def test_fraction_bwd_vs_float64(cuda_dev, B, N, A, lam):
    c = _bwd_case(B + N + A, B, N, A)
    mul = 1.0 / B
    dl, loss, tau = _bwd(cuda_dev, c, B, N, A, mul, lam)
    ai = c["actions"]
    f_hat = c["q_hat"].reshape(N, B, A)[:, np.arange(B), ai].T
    f_bnd = c["q_bnd"].reshape(N - 1, B, A)[:, np.arange(B), ai].T
    ref_d, ref_l = of.fraction_bwd_np(c["logits"], f_bnd, f_hat, c["gscale"].astype(np.float64) * mul, lam, tau=tau)
    assert np.all(np.isfinite(dl)) and np.all(np.isfinite(loss))
    assert rel_err(dl, ref_d) < 1e-5, rel_err(dl, ref_d)
    assert rel_err(loss, ref_l) < 1e-5, rel_err(loss, ref_l)
    dl2, loss2, _ = _bwd(cuda_dev, c, B, N, A, mul, lam, tau=torch.from_numpy(tau).to(cuda_dev))
    assert np.array_equal(dl, dl2) and np.array_equal(loss, loss2)


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,F", [(512, 64, 3136), (3, 2, 5), (40, 100, 130)])
def test_fraction_wgrad_is_exact(cuda_dev, B, N, F):
    """Small-integer operands with power-of-two scales: every sum is exact, so the result matches bit for bit, accumulated
    onto a non-zero prefill."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    rs = np.random.RandomState(B + N)
    dl = (rs.randint(-8, 9, (B, N)) * 2.0 ** -6).astype(np.float32)
    ft = (rs.randint(0, 9, (B, F)) * 2.0 ** -3).astype(np.float32)
    pre_w = (rs.randint(-4, 5, N * F) * 0.5).astype(np.float32)
    pre_b = (rs.randint(-4, 5, N) * 0.5).astype(np.float32)
    dl_d, ft_d = torch.from_numpy(dl).to(cuda_dev), torch.from_numpy(ft).to(cuda_dev)
    outs = []
    for _ in range(2):
        gw, gb = _buf(cuda_dev, N * F, 0.0), _buf(cuda_dev, N, 0.0)
        gw[1].copy_(torch.from_numpy(pre_w))
        gb[1].copy_(torch.from_numpy(pre_b))
        call("riqn_fqf_fraction_wgrad", B, N, F, ptr(dl_d), ptr(ft_d), ptr(gw[1]), ptr(gb[1]))
        torch.cuda.synchronize()
        assert _canaries_ok(gw[0], N * F) and _canaries_ok(gb[0], N)
        outs.append((gw[1].cpu().numpy(), gb[1].cpu().numpy()))
    ref_w = pre_w.astype(np.float64) + (dl.astype(np.float64).T @ ft.astype(np.float64)).ravel()
    ref_b = pre_b.astype(np.float64) + dl.astype(np.float64).sum(0)
    assert np.array_equal(outs[0][0], ref_w.astype(np.float32)) and np.array_equal(outs[0][1], ref_b.astype(np.float32))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,A", [(512, 64, 18), (3, 2, 1), (70, 256, 32)])
def test_argmax_weighted_vs_numpy(cuda_dev, B, N, A):
    from rainbow_iqn_apex_b200._lib import call, ptr
    rs = np.random.RandomState(B + A)
    q = rs.standard_normal((N * B, A)).astype(np.float32)
    w = rs.uniform(0, 1, (N * B,)).astype(np.float32)
    qv = q.reshape(N, B, A).astype(np.float64)
    # exact ties: copy each sample's best column onto a lower and a higher index
    for b in range(0, B, 3):
        if A > 1:
            best = int((qv[:, b] * w.reshape(N, B)[:, b, None]).sum(0).argmax())
            lo = rs.randint(0, A)
            q.reshape(N, B, A)[:, b, lo] = q.reshape(N, B, A)[:, b, best]
    ref_sum = (q.reshape(N, B, A).astype(np.float64) * w.reshape(N, B, 1)).sum(0)
    ref = ref_sum.argmax(1)
    q_d, w_d = torch.from_numpy(q).to(cuda_dev), torch.from_numpy(w).to(cuda_dev)
    outs = []
    for _ in range(2):
        a = _buf(cuda_dev, B, -7, torch.int64)
        call("riqn_argmax_weighted", B, N, A, ptr(q_d), ptr(w_d), ptr(a[1]))
        torch.cuda.synchronize()
        assert _canaries_ok(a[0], B)
        outs.append(a[1].cpu().numpy())
    top2 = np.sort(ref_sum, axis=1)[:, -2:] if A > 1 else None
    ties = np.zeros(B, bool) if A == 1 else (top2[:, 1] - top2[:, 0] == 0)
    clear = np.ones(B, bool) if A == 1 else ((top2[:, 1] - top2[:, 0] > 1e-4) | ties)
    assert np.array_equal(outs[0][clear], ref[clear])                          # numpy's argmax: first maximal index
    assert np.array_equal(outs[0], outs[1])
    assert ties.sum() >= B // 6 if A > 1 else True


@pytest.mark.gpu
def test_entry_points_reject_invalid_arguments_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError, call, ptr
    dev = cuda_dev
    B = 4
    nan = lambda n: torch.full((n,), math.nan, device=dev)
    big = nan(300 * 300)
    lg = torch.zeros(B * 300, device=dev)
    act = torch.zeros(B, dtype=torch.int64, device=dev)
    for N in (1, 0, -3, 257):
        with pytest.raises(RiqnError):
            call("riqn_fqf_fractions", B, N, ptr(lg), ptr(big), ptr(big), ptr(big), ptr(big))
        with pytest.raises(RiqnError):
            call("riqn_fqf_fraction_bwd", B, N, 4, ptr(lg), ptr(lg), ptr(lg), ptr(lg), ptr(act), None, 1.0, 0.0, ptr(big),
                 ptr(big))
        with pytest.raises(RiqnError):
            call("riqn_fqf_fraction_wgrad", B, N, 16, ptr(lg), ptr(lg), ptr(big), ptr(big))
        a = torch.full((B,), -7, dtype=torch.int64, device=dev)
        with pytest.raises(RiqnError):
            call("riqn_argmax_weighted", B, N, 4, ptr(lg), ptr(lg), ptr(a))
    for kw in (dict(A=33), dict(A=0), dict(lam=-0.1), dict(lam=math.nan), dict(lam=math.inf), dict(mul=math.nan),
               dict(mul=math.inf), dict(B=0)):
        p = dict(B=B, A=4, lam=0.0, mul=1.0)
        p.update(kw)
        with pytest.raises(RiqnError):
            call("riqn_fqf_fraction_bwd", p["B"], 8, p["A"], ptr(lg), ptr(lg), ptr(lg), ptr(lg), ptr(act), None, p["mul"],
                 p["lam"], ptr(big), ptr(big))
    for A in (0, 33):
        with pytest.raises(RiqnError):
            call("riqn_argmax_weighted", B, 8, A, ptr(lg), ptr(lg), ptr(a))
    with pytest.raises(RiqnError):
        call("riqn_fqf_fraction_wgrad", B, 8, 0, ptr(lg), ptr(lg), ptr(big), ptr(big))
    torch.cuda.synchronize()
    assert bool(torch.isnan(big).all()) and bool((a == -7).all())


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _oracle_fraction_params(lr):
    return (lr.fraction_net.weight.detach().cpu().clone().requires_grad_(True),
            lr.fraction_net.bias.detach().cpu().clone().requires_grad_(True))


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_learner_step_vs_oracle(cuda_dev, B):
    """compute_gradients under FQF with injected noises against the torch-fp32 FQF step.

    Bounds.  The product's trunk and head run on bf16/fp16 operands (relative error ~4e-3 per element, mostly averaging
    out), so the quantile values F agree with the oracle to ~1e-3 relative.  The fractions come from an fp32 GEMM of the
    same features (the trunk's split-bf16 x3 products are fp32-faithful): logits and tau agree to well below 1e-4.  The fraction gradient
    g_i = 2F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}) is a difference of nearby quantile values: its magnitude is
    ~|dF/dtau| * dtau^2-ish while the forward's error is ~1e-3 |F|, so its relative error can reach several percent on
    individual rows.  dW_f = dlogits^T psi sums these over the batch; it is compared with cosine >= 0.99 (0.999 when the
    oracle's own g dominates the error), and the product's dlogits are checked exactly against the float64 statement of
    the quantile values the product itself computed."""
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch, _qmajor
    N = 64
    cfg, seed = cases.iqn_cfg(N, N, 32), 9100 + B
    params = net.make_params(seed)
    torch.manual_seed(seed)
    lr = Learner(_fqf_args(cuda_dev, B, cfg, fqf_entropy_coef=0.01), 18, None)
    assert lr.fqf == (2.5e-9, 0.01)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    # fractions away from uniform, so that g is not ~0 everywhere
    with torch.no_grad():
        lr.fraction_net.weight.mul_(30.0)
        lr.fraction_net.bias.copy_(torch.from_numpy(np.random.RandomState(seed).standard_normal(N).astype(np.float32)))
    wf, bf = _oracle_fraction_params(lr)
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    noises = cases.make_noises(seed + 3)
    lr._inject = dict(noises=noises)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    gw, gb = (lr.fraction_net.grad_view(p).detach().cpu().clone() for p in (lr.fraction_net.weight, lr.fraction_net.bias))
    for k in ("tau", "tau_hat", "dtau", "q_bnd", "a_star", "dlogits", "fraction_loss"):
        assert k in dbg and bool(torch.isfinite(dbg[k].float()).all()), k
    # the product's own fraction backward against float64 on the operands it read
    q_on, q_bnd = dbg["q_on"].cpu().numpy(), dbg["q_bnd"].cpu().numpy()
    f_hat = q_on.reshape(N, B, 18)[:, np.arange(B), b["actions"]].T
    f_bnd = q_bnd.reshape(-1, B, 18)[:N - 1, np.arange(B), b["actions"]].T
    ref_d, ref_l = of.fraction_bwd_np(dbg["logits"].cpu().numpy(), f_bnd, f_hat, b["weights"].astype(np.float64) / B, 0.01,
                                      tau=dbg["tau"].cpu().numpy())
    assert rel_err(dbg["dlogits"].cpu().numpy(), ref_d) < 1e-5
    assert rel_err(dbg["fraction_loss"].cpu().numpy(), ref_l) < 1e-5

    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_floss, o_grads, (o_gw, o_gb) = of.fqf_step(
        p_on, p_tg, wf, bf, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises, cfg, 0.01, keep=keep)
    dt_max = float(np.max(np.abs(dbg["tau"].cpu().numpy() - keep["tau"].numpy())))
    dth_max = float(np.max(np.abs(dbg["tau_hat"].cpu().numpy().reshape(N, B).T - keep["tau_hat"].numpy())))
    print(f"B={B}: max |tau - tau_oracle| = {dt_max:.3g}, tau_hat {dth_max:.3g}")
    assert dt_max < 1e-4 and dth_max < 1e-4
    # argmax near-ties (the oracle's top-2 dtau-weighted means within 1e-4) may resolve differently
    qv = keep["qv_next"].numpy()
    top2 = np.sort(qv, axis=1)[:, -2:]
    tie = (top2[:, 1] - top2[:, 0]) < 1e-4
    a_gpu = dbg["a_star"].cpu().numpy()
    assert np.all((a_gpu == keep["a_star"].numpy()) | tie)
    ok = a_gpu == keep["a_star"].numpy()
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max((np.abs(lg - lo) / np.abs(lo))[ok]) < 1e-3
    # ReLU kinks that the product and the oracle round to opposite sides of 0 relax the parameters upstream of them
    gk = dbg["keep"]
    h = _qmajor(gk["h"], B).cpu()
    fl = [int(((x.cpu() > 0) != (y > 0)).sum()) for x, y in
          ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
           (h[:, :512], keep["h_v"]), (h[:, 512:], keep["h_a"]))]
    relaxed = set()
    if fl[3] + fl[4] or not ok.all():
        relaxed |= {"conv1", "conv2", "conv3", "iqn_fc", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    for k, g_ref in o_grads.items():
        c = _cos(grads[k], g_ref)
        assert c > (0.98 if k.split(".")[0] in relaxed else 0.999), (k, c, fl)
    cw, cb = _cos(gw, o_gw), _cos(gb, o_gb)
    print(f"B={B}: cos(dW_f) = {cw:.6f}, cos(db_f) = {cb:.6f}, ReLU flips {fl}, ties {int(tie.sum())}")
    assert cw >= 0.99 and cb >= 0.99, (cw, cb)


@pytest.mark.gpu
def test_actor_paths_vs_oracle(cuda_dev):
    """Actor.act / act_batch / act_batch_values act on sum_i dtau_i F(s, tau_hat_i, a) over the proposed fractions, and
    compute_priorities runs the FQF loss."""
    from rainbow_iqn_apex_b200 import Actor
    N, E, seed = 16, 8, 9300
    cfg = cases.iqn_cfg(N, N, 8)
    params = net.make_params(seed)
    torch.manual_seed(seed)
    actor = Actor(_fqf_args(cuda_dev, 8, cfg), 18, None)
    load_params(actor.online_net, params)
    actor.update_target_net()
    actor.eval()                      # eval: the mu weights alone, so the oracle needs no noise
    with torch.no_grad():
        actor.fraction_net.weight.mul_(50.0)
    wf, bf = (t.detach() for t in _oracle_fraction_params(actor))
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    qv = actor.act_batch_values(su8).cpu().numpy()
    # eval mode: the noisy layers use mu alone
    ref = of.act_values(net.to_torch(params), wf, bf, torch.from_numpy(states).float().div_(255), N, training=False).numpy()
    assert rel_err(qv, ref) < 5e-3
    a = actor.act_batch(su8).cpu().numpy()
    top2 = np.sort(ref, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-3
    assert np.array_equal(a[clear], ref.argmax(1)[clear]) and np.array_equal(a[clear], qv.argmax(1)[clear])
    if clear[0]:
        assert actor.act(list(states[0])) == int(a[0])
    # priorities: compute_priorities goes through the FQF loss core
    actor.train()
    bs, L, n, hist = 8, 14, cfg["n_step"], 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    inj = [dict(noises=cases.make_noises(seed + 10 * c)) for c in range(chunks)]
    actor._inject = list(inj)
    pri = actor.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not actor._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(cfg["discount"] ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
        wl, bl = wf.clone().requires_grad_(True), bf.clone().requires_grad_(True)
        loss, _, _, _ = of.fqf_step(p_on, p_tg, wl, bl, (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]),
                                                       nx, torch.ones(hi - lo)), torch.ones(hi - lo), inj[c]["noises"], cfg)
        out.append(loss.numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    assert np.median(np.abs(pri - ref_p) / ref_p) < 1e-3 and np.max(np.abs(pri - ref_p) / ref_p) < 2e-2


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
    frac = learner.fraction_net._flat.detach().clone() if learner.fraction_net is not None else None
    return out, learner.online_net._flat.detach().clone(), frac, learner


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_fqf_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    runs = [_bench_learner(cuda_dev, 1 << 14, graph, 3, dict(fqf=1, fqf_fraction_lr=1e-4)) for _ in range(2)]
    (s1, p1, f1, l1), (s2, p2, f2, _) = runs
    for k, ((i1, x1, _), (i2, x2, _)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2), f"step {k}: sampled indices differ"
        assert torch.equal(x1, x2), f"step {k}: losses differ"
        assert bool(torch.isfinite(x1).all())
    assert torch.equal(p1, p2) and torch.equal(f1, f2)
    assert l1.fraction_optimiser._step == l1.optimiser._step
    (s0, _, _, _) = _bench_learner(cuda_dev, 1 << 14, graph, 1)
    assert not torch.equal(s0[0][1], s1[0][1])


@pytest.mark.gpu
def test_replayed_step_moves_the_fraction_arena_by_one_adam_step_at_its_own_rate(cuda_dev):
    """After a replay, the fraction arena is exactly one Adam step (the fraction optimiser's rate and step count, as the
    dyn struct beside the DQN's carries them) from its state before the replay, on the gradients the replay left."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    from rainbow_iqn_apex_b200.dynstate import DynState
    _, _, _, lr = _bench_learner(cuda_dev, 1 << 14, True, 1, dict(fqf=1, fqf_fraction_lr=1e-4))
    fo = lr.fraction_optimiser
    p0, m0, v0 = (t.clone() for t in (fo._flat, fo._exp_avg, fo._exp_avg_sq))
    lr.learn_and_update(lr._graphs["replay"].mem)
    torch.cuda.synchronize()
    g = lr.fraction_net._flat_grad.clone()
    assert bool(g.abs().sum() > 0)
    d = DynState(cuda_dev)
    d.write(*fo.bias_corrections(fo._step), 1.0, 0.0)
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    grp = fo.param_groups[0]
    call("riqn_adam_step", p.numel(), ptr(p), ptr(g), ptr(m), ptr(v), fo._step, float(grp["lr"]), float(grp["betas"][0]),
         float(grp["betas"][1]), float(grp["eps"]), 1.0, d.ptr())
    torch.cuda.synchronize()
    assert torch.equal(p, fo._flat) and torch.equal(m, fo._exp_avg) and torch.equal(v, fo._exp_avg_sq)
    assert not torch.equal(p0, fo._flat)


@pytest.mark.gpu
def test_plain_learner_is_unchanged(cuda_dev):
    """A namespace without the new fields and one with fqf=0 run the same launches per step and give bit-identical
    sampled indices, losses and parameters."""
    (s1, p1, f1, _), (s2, p2, f2, _) = (_bench_learner(cuda_dev, 1 << 14, False, 3, f) for f in (None, dict(fqf=0)))
    assert f1 is None and f2 is None
    for k, ((i1, l1, c1), (i2, l2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(l1, l2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_learn_graph_and_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    cfg = cases.iqn_cfg(8, 8, 8)
    lr = Learner(_fqf_args(cuda_dev, B, cfg, fqf_fraction_lr=1e-4, fqf_entropy_coef=0.1), 18, None)
    b = cases.make_batch(3, B)
    ex = tuple(torch.from_numpy(b[k]).to(cuda_dev) for k in
               ("states", "actions", "returns", "next_states", "nonterminals", "weights"))
    lr.enable_learn_graph(ex)
    f0 = lr.fraction_net._flat.clone()
    for _ in range(2):
        loss = lr.learn_on_graph(ex)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss).all())
    assert not torch.equal(f0, lr.fraction_net._flat) and lr.fraction_optimiser._step == lr.optimiser._step
    with pytest.raises(ValueError):
        Agent(_fqf_args(cuda_dev, B, cfg, risk_measure="cvar", risk_eta=0.25), 18, None)
    with pytest.raises(ValueError):
        Agent(_fqf_args(cuda_dev, B, cfg, munchausen=1), 18, None)
    a = make_args(cuda_dev, B, cfg, rainbow_only=True)
    a.fqf = 1
    with pytest.raises(ValueError):
        Agent(a, 18, None)
    for kw in (dict(fqf_fraction_lr=0.0), dict(fqf_entropy_coef=-1.0), dict(fqf=2), dict(num_tau_samples=1),
               dict(num_tau_samples=300)):
        with pytest.raises(ValueError):
            Agent(_fqf_args(cuda_dev, B, cfg, **kw), 18, None)
    ag = Agent(_fqf_args(cuda_dev, B, cfg), 18, None)
    ag.set_risk("neutral")
    with pytest.raises(ValueError):
        ag.set_risk("cvar", 0.25)
    assert ag.risk is None


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_replica_runs_the_fqf_step(cuda_dev):
    """A learner in a one-rank process group takes the data-parallel path (both arenas all-reduced) and computes the same
    bits as the plain FQF learner, fraction arena included."""
    import torch.distributed as dist
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch
    B, cfg = 32, cases.iqn_cfg(8, 8, 8)
    b = cases.make_batch(12, B)
    batch = (*_dev_batch(b, cuda_dev), torch.from_numpy(b["weights"]).to(cuda_dev))
    params = net.make_params(12)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        out = []
        for dp in (False, True):
            torch.manual_seed(1)
            lr = Learner(_fqf_args(cuda_dev, B, cfg, fqf_fraction_lr=1e-4), 18, None)
            load_params(lr.online_net, params)
            lr.update_target_net()
            lr.train()
            if dp:
                lr.process_group = dist.group.WORLD
            losses_ = [lr.learn_on_batch(*batch).clone() for _ in range(2)]
            torch.cuda.synchronize()
            assert lr._dp_tail is None
            out.append((losses_, lr.online_net._flat.clone(), lr.fraction_net._flat.clone()))
        for l1, l2 in zip(out[0][0], out[1][0]):
            assert torch.equal(l1, l2)
        assert torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_checkpoint_round_trip(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B, cfg = 32, cases.iqn_cfg(8, 8, 8)
    b = cases.make_batch(4, B)
    batch = tuple(torch.from_numpy(b[k]).to(cuda_dev) for k in
                  ("states", "actions", "returns", "next_states", "nonterminals", "weights"))
    lr = Learner(_fqf_args(cuda_dev, B, cfg, fqf_fraction_lr=1e-4), 18, None)
    lr.train()
    lr.learn_on_batch(*batch)
    lr.save(str(tmp_path), 0, 1, "fqf.pth")
    ck = torch.load(os.path.join(tmp_path, "fqf.pth"), map_location="cpu")
    assert {"fraction_net_state_dict", "fraction_optimiser_state_dict"} <= set(ck)
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    back = Agent(_fqf_args(cuda_dev, B, cfg, fqf_fraction_lr=1e-4, model=os.path.join(tmp_path, "fqf.pth")), 18, None)
    assert torch.equal(back.fraction_net._flat, lr.fraction_net._flat)
    fo, bo = lr.fraction_optimiser, back.fraction_optimiser
    assert bo._step == fo._step == 1
    assert torch.equal(bo._exp_avg, fo._exp_avg) and torch.equal(bo._exp_avg_sq, fo._exp_avg_sq)
    assert torch.equal(back.online_net._flat, lr.online_net._flat)
    plain_args = make_args(cuda_dev, B, cfg)
    plain_args.model = os.path.join(tmp_path, "fqf.pth")
    plain = Agent(plain_args, 18, None)
    assert plain.fqf is None and plain.fraction_net is None
    assert torch.equal(plain.online_net._flat, lr.online_net._flat)
    # a plain IQN checkpoint gives an FQF agent a fresh proposal network
    plain.save(str(tmp_path), 0, 1, "iqn.pth")
    assert "fraction_net_state_dict" not in torch.load(os.path.join(tmp_path, "iqn.pth"), map_location="cpu")
    fresh = Agent(_fqf_args(cuda_dev, B, cfg, model=os.path.join(tmp_path, "iqn.pth")), 18, None)
    assert fresh.fraction_optimiser._step == 0 and float(fresh.fraction_net.bias.detach().abs().max()) == 0.0
