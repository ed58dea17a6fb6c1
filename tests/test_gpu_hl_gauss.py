"""HL-Gauss (Farebrother et al., ICML 2024; Imani & White, ICML 2018): the cross-entropy of the C51 head against the
Gaussian histogram of the scalar double-DQN target (riqn_hl_gauss_loss_fwd_bwd, riqn_hl_gauss_loss_fwd_bwd_h) behind the
optional Agent fields hl_gauss and hl_gauss_sigma.

The unmarked tests pin the float64 statement (oracle/hl_gauss.py) by identities, check the torch-fp32 statement against
it and check the host-side validation.  The gpu tests hold both entry points to the float64 statement (the method of
test_gpu_c51_kernels.py: NaN prefills, canaries, two calls alike, rejected calls write nothing): target_out bit for bit,
m_out within one float ulp, loss and dq bit for bit against the numpy float32 statement of the cross-entropy tail on the
kernel's own m.  Value-only kernel mutants and the cases that catch them: Z not applied, edges at the atoms, or
sigma = r instead of r * D -- m_out in every test_kernel_vs_float64 case; the target read at actions[b] instead of a* --
target_out in every case with A > 1; g without the nonterminal -- target_out of the terminal row 0 in every case;
h^-1 skipped on the atoms -- target_out in every rescaled case (eps = 0 included).  At the learner level: the step
against the torch oracle, autograd, reproducibility eagerly and from each captured graph, data parallelism,
augmentation, the actors, launch counts, checkpoints, and that a namespace without the field runs exactly as before."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, assert_canaries, dptr, f32_bits, lib_call, load_params, make_args, rel_err, to_dev
from oracle import cases, hl_gauss as oh, network as net

F32 = np.float32
RATIOS = [0.01, 0.75, 2.0, 100.0, 1000.0]


def _hl_args(dev, B, **kw):
    a = make_args(dev, B, rainbow_only=True)
    a.hl_gauss = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("atoms", [2, 51, 64])
def test_histogram_is_a_distribution(ratio, atoms):
    """sum_j m_j = 1 to 1e-13 and every m_j >= 0 for y over all of [v_min, v_max], both ends included."""
    for v_min, v_max in ((-10.0, 10.0), (-3.0, 40.0)):
        y = np.concatenate((np.linspace(v_min, v_max, 2001), [np.nextafter(v_max, 0), np.nextafter(v_min, 0)]))
        m = oh.histogram_np(y, v_min, v_max, atoms, ratio)
        assert np.max(np.abs(m.sum(1) - 1.0)) <= 1e-13
        assert np.all(m >= 0)


@pytest.mark.parametrize("ratio,tol", [(0.75, 1e-5), (2.0, 1e-8)])
def test_histogram_mean_is_the_target(ratio, tol):
    """|sum_j z_j m_j - y| <= tol * D for y at least 6 sigma inside the support (51 atoms on +-10)."""
    atoms, v_min, v_max = 51, -10.0, 10.0
    e, D = oh.edges_np(v_min, v_max, atoms)
    z = v_min + np.arange(atoms) * D
    s = ratio * D
    y = np.linspace(v_min + 6 * s, v_max - 6 * s, 2001)
    m = oh.histogram_np(y, v_min, v_max, atoms, ratio)
    err = np.max(np.abs(m @ z - y)) / D
    print(f"ratio {ratio}: max |mean - y| / D = {err:.3g}")
    assert err <= tol


def test_narrow_sigma_is_one_hot():
    """ratio = 0.01: the histogram is one-hot (to 1e-12) on the nearest atom for y at least 0.1 D from a bin edge."""
    atoms, v_min, v_max = 51, -10.0, 10.0
    e, D = oh.edges_np(v_min, v_max, atoms)
    y = np.linspace(v_min, v_max, 4001)
    d_edge = np.min(np.abs(y[:, None] - e[None, :]), 1)
    y = y[d_edge >= 0.1 * D]
    m = oh.histogram_np(y, v_min, v_max, atoms, 0.01)
    near = np.rint((y - v_min) / D).astype(np.int64)
    want = np.zeros_like(m)
    want[np.arange(y.size), near] = 1.0
    assert y.size > 3000 and np.max(np.abs(m - want)) <= 1e-12


@pytest.mark.parametrize("ratio", RATIOS)
def test_mirror_symmetry(ratio):
    """On a symmetric support, y -> -y reverses m: to 1e-14, plus the edges' own rounding (e_i and -e_(atoms-i) differ
    by up to 2 ulp of 10) carried through the Gaussian's peak density 1 / (sigma sqrt(2 pi)), which only counts at
    narrow sigma."""
    for atoms in (2, 21, 51, 64):
        y = np.linspace(-10.0, 10.0, 1001)
        m, mm = oh.histogram_np(y, -10.0, 10.0, atoms, ratio), oh.histogram_np(-y, -10.0, 10.0, atoms, ratio)
        _, D = oh.edges_np(-10.0, 10.0, atoms)
        tol = 1e-14 + 2 * 2.0 * np.spacing(10.0) / (ratio * D * math.sqrt(2 * math.pi))
        assert np.max(np.abs(mm - m[:, ::-1])) <= tol


@pytest.mark.parametrize("eps", [None, 1e-3])
def test_targets_beyond_the_support_clamp(eps):
    """Every target y >= v_max gives m(v_max) bit for bit (and y <= v_min gives m(v_min))."""
    atoms, v_min, v_max = 51, -10.0, 10.0
    support = torch.linspace(v_min, v_max, atoms).numpy()
    rs = np.random.RandomState(3)
    p = rs.dirichlet(np.ones(atoms), 64).astype(F32)
    R = np.concatenate((10.0 ** rs.uniform(2, 6, 32), -(10.0 ** rs.uniform(2, 6, 32)))).astype(F32)
    y = oh.target_np(p, support, R, np.ones(64, F32), 0.99 ** 3, v_min, v_max, eps)
    assert np.all(y[:32] == v_max) and np.all(y[32:] == v_min)
    for ratio in RATIOS:
        m = oh.histogram_np(y, v_min, v_max, atoms, ratio)
        top, bot = oh.histogram_np([v_max, v_min], v_min, v_max, atoms, ratio)
        assert np.array_equal(m[:32], np.repeat(top[None], 32, 0)) and np.array_equal(m[32:], np.repeat(bot[None], 32, 0))


def test_dq_is_the_autograd_of_the_cross_entropy():
    rs = np.random.RandomState(5)
    for atoms in (2, 51, 64):
        logits = torch.tensor(rs.standard_normal((16, atoms)) * 3, dtype=torch.float64, requires_grad=True)
        m = oh.histogram_np(rs.uniform(-10, 10, 16), -10.0, 10.0, atoms, 0.75)
        lp = torch.log_softmax(logits, 1)
        loss = -(torch.from_numpy(m) * lp).sum(1)
        loss.sum().backward()
        l64, dq = oh.cross_entropy_np(m, lp.detach().numpy())
        assert np.max(np.abs(l64 - loss.detach().numpy())) <= 1e-12
        assert np.max(np.abs(dq - logits.grad.numpy())) <= 1e-12


@pytest.mark.parametrize("eps", [None, 1e-3])
def test_float64_and_torch_fp32_statements_agree(eps):
    B, A = 4, 4
    params = net.make_params(31, A, rainbow_only=True)
    b = cases.make_batch(32, B, action_space=A)
    st, ac, rt, nx, nt = cases.batch_to_torch(b)
    if eps is not None:
        rt = rt * 40
    noises = cases.make_noises(33, action_space=A, rainbow_only=True)
    keep = {}
    loss, _ = oh.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params), (st, ac, rt, nx, nt),
                            torch.from_numpy(b["weights"]), noises, eps=eps, keep=keep)
    support = torch.linspace(-10.0, 10.0, 51).numpy()
    y = oh.target_np(keep["pns_a"].numpy(), support, rt.numpy(), b["nonterminals"], 0.99 ** 3, -10.0, 10.0, eps)
    assert np.array_equal(keep["target"].numpy(), y)
    m64 = oh.histogram_np(y, -10.0, 10.0, 51, 0.75)
    l64, _ = oh.cross_entropy_np(m64, keep["log_ps_a"].numpy())
    assert rel_err(keep["m"].numpy(), m64) < 1e-6
    assert np.max(np.abs(loss.numpy() - l64) / l64) < 1e-6


# ------------------------------------------------------------------------------------------------ kernels (GPU)
KERNEL_CASES = [(1, 1, 2, -10.0, 10.0), (7, 4, 21, -3.0, 40.0), (32, 18, 51, -10.0, 10.0), (512, 32, 64, -3.0, 40.0),
                (4096, 18, 51, -10.0, 10.0), (32, 1, 64, -10.0, 10.0), (512, 4, 21, -10.0, 10.0), (7, 32, 2, -3.0, 40.0)]


def _inputs(B, A, atoms, seed):
    rs = np.random.RandomState(seed)
    h = dict(logp=np.log(rs.dirichlet(np.ones(atoms), (B, A))).astype(F32),
             pt=rs.dirichlet(np.ones(atoms), (B, A)).astype(F32), act=rs.randint(0, A, B).astype(np.int64),
             astar=rs.randint(0, A, B).astype(np.int64),
             ret=(rs.standard_normal(B) * rs.choice([0.5, 5.0, 1e4], B)).astype(F32),
             nt=(rs.uniform(size=B) > 0.1).astype(F32))
    h["nt"][0] = 0.0                                               # a terminal row: y = clamp(R) (h(R))
    if A > 1:                                                      # a* differs from the action taken
        h["astar"][0] = (h["act"][0] + 1) % A
    return h


def _call(dev, B, A, atoms, h, support, gamma_n, v_min, v_max, ratio, eps=None, outs=True):
    d = {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}
    sup = to_dev(support, dev)
    o = {"loss": Out(B, dev), "dq": Out(B * atoms, dev), "m": Out(B * atoms, dev) if outs else None,
         "target": Out(B, dev) if outs else None}
    args = [B, A, atoms] + [dptr(d[k]) for k in ("logp", "pt", "act", "astar", "ret", "nt")] + [
        dptr(sup), float(gamma_n), float(v_min), float(v_max), float(ratio)]
    ptrs = [o[k].p if o[k] is not None else None for k in ("loss", "dq", "m", "target")]
    if eps is None:
        lib_call("riqn_hl_gauss_loss_fwd_bwd", *args, *ptrs)
    else:
        lib_call("riqn_hl_gauss_loss_fwd_bwd_h", *args, float(eps), *ptrs)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


def tail_np(m, lp):
    """numpy float32 statement of the kernel's cross-entropy tail on m (B, atoms), lp = logp[b, act] (B, atoms): the
    two-warp reductions of fl(m_j lp_j) and m_j, loss = -tot and dq = -fl(m - fl(p mt)) with p = fl32(exp(lp)) for
    the two float32 neighbours a float64 exp within 2^-50 relative can round to (equal unless exp(lp) lies that close to
    a float32 rounding boundary).  Returns loss, dq at the lower and at the upper p, and the count of such p."""
    from test_gpu_value_rescaling import _warp_sum_np
    B, atoms = m.shape
    part, ms = np.zeros((B, 64), F32), np.zeros((B, 64), F32)
    part[:, :atoms] = (m * lp).astype(F32)
    ms[:, :atoms] = m
    tot = ((F32(0) + _warp_sum_np(part[:, :32])).astype(F32) + _warp_sum_np(part[:, 32:])).astype(F32)
    mt = ((F32(0) + _warp_sum_np(ms[:, :32])).astype(F32) + _warp_sum_np(ms[:, 32:])).astype(F32)
    e = np.exp(lp.astype(np.float64))
    p_lo, p_hi = (e * (1 - 2.0 ** -50)).astype(F32), (e * (1 + 2.0 ** -50)).astype(F32)
    dq = [-((m - (p * mt[:, None]).astype(F32)).astype(F32)) for p in (p_lo, p_hi)]
    return -tot, dq[0], dq[1], int(np.sum(p_lo != p_hi))


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 0.0, 1e-3])
@pytest.mark.parametrize("ratio", [0.01, 0.75, 2.0, 100.0])
@pytest.mark.parametrize("B,A,atoms,v_min,v_max", KERNEL_CASES)
def test_kernel_vs_float64(cuda_dev, B, A, atoms, v_min, v_max, ratio, eps):
    support = torch.linspace(v_min, v_max, atoms).numpy()
    gamma_n = 0.99 ** 3
    h = _inputs(B, A, atoms, B * 7 + A * 3 + atoms)
    o = _call(cuda_dev, B, A, atoms, h, support, gamma_n, v_min, v_max, ratio, eps)
    rows = np.arange(B)
    y = oh.target_np(h["pt"][rows, h["astar"]], support, h["ret"], h["nt"], gamma_n, v_min, v_max, eps)
    assert_bits("target_out", o["target"].bits(), f32_bits(y.astype(F32)))
    if B >= 32:                                       # the clamp binds at both ends somewhere
        assert np.any(y == float(F32(v_max))) and np.any(y == float(F32(v_min)))
    m = o["m"].f32().reshape(B, atoms)
    want = oh.histogram_np(y, v_min, v_max, atoms, ratio).astype(F32)
    ulps = np.abs(f32_bits(m).astype(np.int64) - f32_bits(want).astype(np.int64))
    assert np.max(ulps) <= 1, f"m_out: {int(np.sum(ulps > 1))} elements beyond one ulp, worst {int(np.max(ulps))}"
    assert np.all(m >= 0)
    loss32, dq_lo, dq_hi, amb = tail_np(m, h["logp"][rows, h["act"]])
    assert_bits("loss vs float32 tail", o["loss"].bits(), f32_bits(loss32))
    dq = o["dq"].f32().reshape(B, atoms)
    assert np.all((f32_bits(dq) == f32_bits(dq_lo)) | (f32_bits(dq) == f32_bits(dq_hi))), "dq vs float32 tail"
    assert np.all(o["loss"].f32() >= 0)
    print(f"B={B} A={A} atoms={atoms} [{v_min}, {v_max}] r={ratio} eps={eps}: m exact {int(np.sum(ulps == 0))} of "
          f"{ulps.size}, near-boundary exp {amb}")
    again = _call(cuda_dev, B, A, atoms, h, support, gamma_n, v_min, v_max, ratio, eps)
    for k in o:
        assert_bits(f"second call {k}", again[k].bits(), o[k].bits())
    bare = _call(cuda_dev, B, A, atoms, h, support, gamma_n, v_min, v_max, ratio, eps, outs=False)
    assert_bits("loss without m_out, target_out", bare["loss"].bits(), o["loss"].bits())
    assert_bits("dq without m_out, target_out", bare["dq"].bits(), o["dq"].bits())


@pytest.mark.gpu
def test_entry_points_reject_invalid_calls_and_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    src = torch.full((64 * 64 * 8,), 0.5, device=dev)
    idx = torch.zeros(64, dtype=torch.int64, device=dev)
    outs = [Out(64 * 64 * 8, dev) for _ in range(4)]
    bad = [dict(B=0), dict(B=-1), dict(A=0), dict(A=-3), dict(atoms=1), dict(atoms=0), dict(atoms=65),
           dict(v_min=math.nan), dict(v_max=math.inf), dict(v_min=-math.inf), dict(v_min=10.0), dict(v_min=11.0),
           dict(r=0.0), dict(r=-0.75), dict(r=math.nan), dict(r=math.inf), dict(r=1000.001), dict(r=1e-46)]
    for kw in bad:
        B, A, atoms = kw.get("B", 4), kw.get("A", 4), kw.get("atoms", 51)
        args = [B, A, atoms, dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src), dptr(src), dptr(src), 0.97,
                kw.get("v_min", -10.0), kw.get("v_max", 10.0), kw.get("r", 0.75)]
        for fn, extra in (("riqn_hl_gauss_loss_fwd_bwd", []), ("riqn_hl_gauss_loss_fwd_bwd_h", [1e-3])):
            with pytest.raises(RiqnError):
                lib_call(fn, *args, *extra, *(o.p for o in outs))
    for eps in (-1e-3, math.nan, math.inf):
        with pytest.raises(RiqnError):
            lib_call("riqn_hl_gauss_loss_fwd_bwd_h", 4, 4, 51, dptr(src), dptr(src), dptr(idx), dptr(idx), dptr(src),
                     dptr(src), dptr(src), 0.97, -10.0, 10.0, 0.75, eps, *(o.p for o in outs))
    torch.cuda.synchronize()
    for o in outs:
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _hl_learner(dev, B, params, **kw):
    from rainbow_iqn_apex_b200 import Learner
    lr = Learner(_hl_args(dev, B, **kw), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    return lr


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("B", [32, 512])
def test_learner_step_vs_oracle(cuda_dev, B, eps):
    """Learner.compute_gradients under injected noises against the torch-fp32 oracle step (51 atoms, r = 0.75)."""
    from test_gpu_learn import _dev_batch
    from test_gpu_value_rescaling import _check_grads, _near_ties
    seed = 13100 + B
    params = net.make_params(seed, rainbow_only=True)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    lr = _hl_learner(cuda_dev, B, params, **kw)
    assert lr.hl_gauss == 0.75 and lr.value_rescaling == eps
    b = cases.make_batch(seed + 1, B)
    if eps is not None:
        b["returns"] = (b["returns"] * 40).astype(F32)
    noises = cases.make_noises(seed + 3, rainbow_only=True)
    lr._inject = dict(noises=noises)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    a_gpu = dbg["a_star"].cpu().numpy()
    support = lr.support.cpu().numpy()
    # the kernel's target is the float64 statement of the probabilities the product computed, bit for bit
    pt = dbg["p_target"].cpu().numpy()[np.arange(B), a_gpu]
    y = oh.target_np(pt, support, b["returns"], b["nonterminals"], 0.99 ** 3, -10.0, 10.0, eps)
    assert_bits("target", f32_bits(dbg["target"].cpu().numpy()), f32_bits(y.astype(F32)))
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, o_grads = oh.learn_step(p_on, p_tg, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises,
                                    eps=eps, keep=keep)
    tie = _near_ties(keep["ev_next"].numpy(), 1e-4 if eps is None else 1e-3)
    ok = a_gpu == keep["a_star"].numpy()
    assert np.all(ok | tie)
    t_err = rel_err(dbg["target"].cpu().numpy()[ok], keep["target"].numpy()[ok])
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    l_err = np.max((np.abs(lg - lo) / np.abs(lo))[ok])
    print(f"B={B} eps={eps}: target rel err {t_err:.3g}, max loss rel err {l_err:.3g}, ties {int((~ok).sum())}")
    assert t_err < 1e-5 and l_err < 1e-3
    _check_grads(grads, o_grads, [1, 1, 1, 0, 0], not ok.all())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 64, 512])
def test_head_loss_autograd_equals_compute_gradients(cuda_dev, B):
    """(w * loss).mean().backward() through the agent's loss node equals Learner.compute_gradients bit for bit (B a power
    of two, so w / B is exact either way)."""
    from test_gpu_learn import _dev_batch
    params = net.make_params(77 + B, rainbow_only=True)
    b = cases.make_batch(78 + B, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    noises = cases.make_noises(79 + B, rainbow_only=True)
    lr1, lr2 = _hl_learner(cuda_dev, B, params), _hl_learner(cuda_dev, B, params)
    lr1._inject = dict(noises=noises)
    l1 = lr1.compute_gradients(st, ac, rt, nx, nt, w)
    lr2._inject = dict(noises=noises)
    lr2.online_net.zero_grad()
    l2 = lr2.compute_loss_actor_or_learner(st, ac, rt, nx, nt)
    (w * l2).mean().backward()
    torch.cuda.synchronize()
    assert torch.equal(l1, l2.detach())
    assert torch.equal(lr1.online_net._flat_grad, lr2.online_net._flat_grad)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eager", "replay", "batch", "learn"])
def test_steps_are_bitwise_reproducible(cuda_dev, kind):
    """Two consecutive B = 512 steps, eagerly and from each of the three captured graphs, twice alike."""
    from test_gpu_augment import _bench_run
    fields = dict(rainbow_only=1, hl_gauss=1)
    (o1, p1), (o2, p2) = _bench_run(cuda_dev, kind, fields, steps=2), _bench_run(cuda_dev, kind, fields, steps=2)
    for (_, l1), (_, l2) in zip(o1, o2):
        assert torch.equal(l1, l2) and bool(torch.isfinite(l1).all()) and bool((l1 >= 0).all())
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_data_parallel_half_batches_equal_one_learner(cuda_dev):
    from test_gpu_learn import _dev_batch
    B = 64
    b = cases.make_batch(12, B)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    params = net.make_params(12, rainbow_only=True)
    noises = cases.make_noises(13, rainbow_only=True)

    def grads_of(sl, scale):
        lr = _hl_learner(cuda_dev, sl.stop - sl.start, params)
        lr._inject = dict(noises=noises)
        lr.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl] * scale)
        torch.cuda.synchronize()
        return lr.online_net._flat_grad.clone()

    full = grads_of(slice(0, B), 1.0)
    halves = grads_of(slice(0, B // 2), 0.5) + grads_of(slice(B // 2, B), 0.5)
    err = float((halves - full).abs().max() / full.abs().max())
    c = float((halves.double() * full.double()).sum() / (halves.double().norm() * full.double().norm()))
    print(f"data parallel: max |sum of half-batch grads - full| / max |full| = {err:.3g}, cos {c:.8f}")
    assert err < 2e-3 and c > 0.99999


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_shifted_step_equals_the_plain_step_on_shifted_frames(cuda_dev, B):
    from test_gpu_augment import _learner, _step, _assert_same, _window_batch, shift_np
    fields = dict(rainbow_only=1, hl_gauss=1)
    win_np, win, b, rest = _window_batch(cuda_dev, B, 700 + B)
    rs = np.random.RandomState(B + 2)
    s_st = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_nx = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_st[0], s_nx[0] = (3, -2), (-4, 1)
    aug = _learner(cuda_dev, B, fields, shift=4, seed=14)
    assert aug.hl_gauss == 0.75 and aug.random_shift == 4
    aug._inject = dict(shifts=(s_st, s_nx))
    got = _step(aug, win[:, :4], win[:, 3:7], rest)
    st = torch.from_numpy(shift_np(win_np[:, :4], s_st)).to(cuda_dev)
    nx = torch.from_numpy(shift_np(win_np[:, 3:7], s_nx)).to(cuda_dev)
    plain = _learner(cuda_dev, B, fields, seed=14)
    _assert_same(got, _step(plain, st, nx, rest), "hl_gauss")


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [None, 1e-3])
def test_actors_equal_c51_and_priorities_match_the_oracle(cuda_dev, eps):
    from rainbow_iqn_apex_b200 import Actor
    E, seed = 8, 13300
    params = net.make_params(seed, rainbow_only=True)
    kw = dict(value_rescaling=1, value_rescaling_eps=eps) if eps is not None else {}
    actors = []
    for fields in (dict(hl_gauss=1), dict(hl_gauss=0)):
        torch.manual_seed(seed)
        a = Actor(_hl_args(cuda_dev, 8, **kw, **fields), 18, None)
        load_params(a.online_net, params)
        a.update_target_net()
        actors.append(a)
    hl, c51 = actors
    assert hl.hl_gauss == 0.75 and c51.hl_gauss is None
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    for mode in ("eval", "train"):
        for a in actors:
            getattr(a, mode)()
        noise = cases.make_noises(seed + 5, count=1, rainbow_only=True)[0]
        for a in actors:
            a.online_net.reset_noise({k: tuple(t.to(cuda_dev) for t in v) for k, v in noise.items()})
        assert torch.equal(hl.online_net(su8), c51.online_net(su8))
        assert torch.equal(hl.act_batch(su8), c51.act_batch(su8))
        assert hl.act(list(states[0])) == c51.act(list(states[0]))
    hl.train()
    bs, L, n, hist = 8, 14, 3, 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    inj = [dict(noises=cases.make_noises(seed + 10 * c, rainbow_only=True)) for c in range(chunks)]
    hl._inject = list(inj)
    pri = hl.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not hl._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(0.99 ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        loss, _ = oh.learn_step(net.to_torch(params, requires_grad=True), net.to_torch(params),
                                (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx,
                                 torch.ones(hi - lo)), torch.ones(hi - lo), inj[c]["noises"], eps=eps)
        out.append(loss.numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    rel = np.abs(pri - ref_p) / ref_p
    print(f"priorities rel err median {np.median(rel):.3g} max {np.max(rel):.3g}")
    assert np.median(rel) < 1e-3 and np.max(rel) < 2e-2


@pytest.mark.gpu
def test_hl_gauss_step_makes_the_c51_launches(cuda_dev):
    from test_gpu_qr import _bench_learner
    (s1, _, _, _), (s2, _, _, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f)
                                    for f in (dict(rainbow_only=1), dict(rainbow_only=1, hl_gauss=1)))
    assert [c for _, _, c in s1] == [c for _, _, c in s2]
    assert not torch.equal(s1[0][1], s2[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize("base", [{}, dict(rainbow_only=1), dict(qr_dqn=1)])
def test_namespace_without_the_field_is_unchanged(cuda_dev, base):
    """IQN, C51 and QR-DQN learners from a namespace without hl_gauss and with hl_gauss = 0 run the same launches per
    step and give bit-identical sampled indices, losses and parameters."""
    from test_gpu_qr import _bench_learner
    (s1, p1, l1, _), (s2, p2, l2, _) = (_bench_learner(cuda_dev, 1 << 14, False, 2, f)
                                        for f in (base, dict(base, hl_gauss=0)))
    assert l1.hl_gauss is None and l2.hl_gauss is None
    for k, ((i1, x1, c1), (i2, x2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(x1, x2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_checkpoints_round_trip_between_c51_and_hl_gauss(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent, Learner
    from test_gpu_qr import _graph_batch
    B = 32
    batch = _graph_batch(cuda_dev, B, 4)
    for src, dst in ((dict(hl_gauss=1), dict(hl_gauss=0)), (dict(hl_gauss=0), dict(hl_gauss=1, hl_gauss_sigma=2.0))):
        lr = Learner(_hl_args(cuda_dev, B, **src), 18, None)
        lr.train()
        lr.learn_on_batch(*batch)
        lr.save(str(tmp_path), 0, 1, "ck.pth")
        path = os.path.join(tmp_path, "ck.pth")
        ck = torch.load(path, map_location="cpu")
        assert set(ck) == {"T_actors", "T_learner", "model_state_dict", "optimiser_state_dict"}
        back = Agent(_hl_args(cuda_dev, B, model=path, **dst), 18, None)
        assert torch.equal(back.online_net._flat, lr.online_net._flat) and back.optimiser._step == 1
        assert back.hl_gauss == (None if not dst["hl_gauss"] else 2.0)


@pytest.mark.gpu
def test_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    for kw in (dict(hl_gauss=2), dict(hl_gauss="1"), dict(rainbow_only=0), dict(hl_gauss_sigma=0.0),
               dict(hl_gauss_sigma=-1.0), dict(hl_gauss_sigma=math.nan), dict(hl_gauss_sigma=math.inf),
               dict(hl_gauss_sigma=1001.0), dict(hl_gauss_sigma="0.75"), dict(qr_dqn=1), dict(munchausen=1),
               dict(fqf=1), dict(qr_dqn=1, mmd=1), dict(risk_measure="cvar", risk_eta=0.25)):
        with pytest.raises(ValueError):
            Agent(_hl_args(cuda_dev, B, **kw), 18, None)
    ag = Learner(_hl_args(cuda_dev, B, value_rescaling=1, random_shift=4, hl_gauss_sigma=np.float32(1.5)), 18, None)
    assert ag.hl_gauss == 1.5 and ag.value_rescaling == 1e-3 and ag.random_shift == 4 and ag.rainbow_only
