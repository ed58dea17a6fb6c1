"""Munchausen-IQN (Vieillard, Pietquin & Geist 2020): a soft double-expectation target with a clipped log-policy bonus,
fused into one device loss kernel (riqn_miqn_loss_fwd_bwd) behind the optional Agent fields munchausen,
munchausen_alpha, munchausen_tau and munchausen_l0.

The unmarked tests pin the float64 oracle (oracle/munchausen.py) by identities, check the torch-fp32 oracle against it and
check the host-side validation.  The gpu tests check the kernel against the float64 oracle, a learner step and the actors'
priorities against the torch oracle, reproducibility in the eager and the captured step, and that a namespace without
the fields issues exactly the launches of plain IQN."""
import math
import socket

import numpy as np
import pytest
import torch

from helpers import load_params, make_args, rel_err
from oracle import cases, losses, munchausen as om, network as net

DEFAULTS = dict(alpha=0.9, entropy_tau=0.03, l0=-1.0)


def _case(seed, B, Np, A, spread=1.0, N=None):
    """Random inputs of the loss: q_tgt (N'*2B, A) in the stacked row order, returns, nonterminals, actions (+ q_on, tau
    when N is given)."""
    rs = np.random.RandomState(seed)
    c = dict(q_tgt=(spread * rs.standard_normal((Np * 2 * B, A))).astype(np.float32),
             returns=rs.standard_normal(B).astype(np.float32),
             nonterminals=(rs.uniform(size=B) < 0.8).astype(np.float32),
             actions=rs.randint(0, A, B).astype(np.int64))
    if N is not None:
        c["q_on"] = rs.standard_normal((N * B, A)).astype(np.float32)
        c["tau"] = rs.uniform(0, 1, (N * B, 1)).astype(np.float32)
    return c


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def test_oracle_hard_max_limit_is_the_iqn_target():
    """alpha = 0 and a small temperature: the soft expectation is Z_j(s', argmax qbar') when the max is unique by >= 1e-2."""
    B, Np, A, g = 16, 13, 6, 0.99 ** 3
    c = _case(1, B, Np, A)
    q = c["q_tgt"].astype(np.float64).reshape(Np, 2, B, A)
    best = np.random.RandomState(2).randint(0, A, B)
    q[:, 0, np.arange(B), best] += 3.0
    qbar = q[:, 0].mean(0)
    top2 = np.sort(qbar, axis=1)[:, -2:]
    assert np.all(top2[:, 1] - top2[:, 0] >= 1e-2) and np.array_equal(qbar.argmax(1), best)
    t, bonus = om.soft_target_np(q.reshape(-1, A), c["returns"], c["nonterminals"], c["actions"], g, 0.0, 1e-4, -1.0)
    r, nt = c["returns"].astype(np.float64), c["nonterminals"].astype(np.float64)
    iqn = r[:, None] + g * nt[:, None] * q[:, 0, np.arange(B), best].T
    assert np.max(np.abs(t - iqn)) < 1e-8
    assert np.all(bonus == 0.0)


@pytest.mark.parametrize("l0", [-1.0, -0.05])
def test_oracle_equal_means_give_the_uniform_log_policy(l0):
    B, Np, A, te, alpha = 8, 5, 18, 0.03, 0.9
    c = _case(3, B, Np, A)
    q = c["q_tgt"].reshape(Np, 2, B, A)
    q[:, 1] = q[:, 1, :, :1]                       # Z_j(s_t, a) equal across actions
    t, bonus = om.soft_target_np(q.reshape(-1, A), c["returns"], c["nonterminals"], c["actions"], 0.97, alpha, te, l0)
    assert np.all(bonus == alpha * max(-te * np.log(A), l0))


def test_oracle_bonus_is_never_positive_and_a_dispreferred_action_hits_the_clip():
    for seed in range(5):
        for alpha, te in ((0.9, 0.03), (2.0, 1.0), (0.1, 1e-3)):
            c = _case(10 + seed, 32, 8, 18, spread=3.0)
            _, bonus = om.soft_target_np(c["q_tgt"], c["returns"], c["nonterminals"], c["actions"], 0.97, alpha, te, -1.0)
            assert np.all(bonus <= 0.0) and np.all(bonus >= -alpha)
    B, Np, A = 8, 4, 18
    c = _case(20, B, Np, A)
    q = c["q_tgt"].reshape(Np, 2, B, A)
    q[:, 1, np.arange(B), c["actions"]] -= 50.0
    _, bonus = om.soft_target_np(q.reshape(-1, A), c["returns"], c["nonterminals"], c["actions"], 0.97, 0.9, 0.03, -1.0)
    assert np.all(bonus == 0.9 * -1.0)


@pytest.mark.parametrize("spread", [0.1, 1.0, 30.0])
def test_torch_oracle_agrees_with_float64(spread):
    B, Np, A, g = 16, 13, 18, 0.99 ** 3
    c = _case(30, B, Np, A, spread=spread)
    t64, b64 = om.soft_target_np(c["q_tgt"], c["returns"], c["nonterminals"], c["actions"], g, **DEFAULTS)
    t32, b32 = om.soft_target(*(torch.from_numpy(c[k]) for k in ("q_tgt", "returns", "nonterminals", "actions")), g,
                              **DEFAULTS)
    assert rel_err(t32.numpy(), t64) < 1e-6
    assert rel_err(b32.numpy(), b64) < 1e-6 and np.all(np.isfinite(t32.numpy()))


# ------------------------------------------------------------------------------------------------ kernel (GPU)
def _kernel(c, B, N, Np, A, g, kappa, alpha, entropy_tau, l0, outs=None):
    from rainbow_iqn_apex_b200._lib import call, ptr
    dev = torch.device("cuda")
    d = {k: torch.from_numpy(v).to(dev) for k, v in c.items()}
    o = outs or dict(loss=torch.empty(B, device=dev), dtheta=torch.empty(N * B, device=dev),
                     theta=torch.empty(B, N, device=dev), target=torch.empty(B, Np, device=dev),
                     bonus=torch.empty(B, device=dev))
    call("riqn_miqn_loss_fwd_bwd", B, N, Np, A, ptr(d["q_on"]), ptr(d["q_tgt"]), ptr(d["tau"]), ptr(d["actions"]),
         ptr(d["returns"]), ptr(d["nonterminals"]), float(g), float(kappa), alpha, entropy_tau, l0, ptr(o["loss"]),
         ptr(o["dtheta"]), ptr(o["theta"]), ptr(o["target"]), ptr(o["bonus"]))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _oracle(c, B, N, Np, g, kappa, alpha, entropy_tau, l0):
    target, bonus = om.soft_target_np(c["q_tgt"], c["returns"], c["nonterminals"], c["actions"], g, alpha, entropy_tau,
                                      l0)
    theta = c["q_on"][np.arange(N * B), np.tile(c["actions"], N)].reshape(N, B).T
    loss, dth = om.pairwise_loss_np(theta, target, c["tau"].reshape(N, B).T, kappa)
    return dict(loss=loss, dtheta=dth.T.reshape(-1), theta=theta, target=target, bonus=bonus)


def _check(got, ref, tol=1e-5):
    for k in ("loss", "dtheta", "target", "bonus"):
        assert np.all(np.isfinite(got[k])), k
        assert rel_err(got[k], ref[k]) < tol, (k, rel_err(got[k], ref[k]))
    assert np.array_equal(got["theta"], ref["theta"])


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,Np,A,kappa", [(512, 64, 64, 18, 1.0), (3, 8, 13, 4, 1.0), (3, 8, 13, 32, 0.5)])
def test_kernel_matches_float64_oracle(cuda_dev, B, N, Np, A, kappa):
    g = 0.99 ** 3
    c = _case(100 + B + A, B, Np, A, N=N)
    got = _kernel(c, B, N, Np, A, g, kappa, **DEFAULTS)
    _check(got, _oracle(c, B, N, Np, g, kappa, **DEFAULTS))
    again = _kernel(c, B, N, Np, A, g, kappa, **DEFAULTS)
    for k in got:
        assert np.array_equal(got[k], again[k]), k                      # bitwise reproducible
    assert np.any(got["bonus"] < 0) and np.all(got["bonus"] <= 0)


@pytest.mark.gpu
def test_kernel_underflowing_policy_is_finite(cuda_dev):
    """Action means 5 apart at te = 0.03: pi' underflows for all but the best action and l(a_t) sits far below l0."""
    B, N, Np, A, g = 64, 16, 24, 18, 0.99 ** 3
    c = _case(7, B, Np, A, N=N)
    c["q_tgt"] = (c["q_tgt"] * 0.01 + 5.0 * np.arange(A, dtype=np.float32)[None, :]).astype(np.float32)
    got = _kernel(c, B, N, Np, A, g, 1.0, **DEFAULTS)
    ref = _oracle(c, B, N, Np, g, 1.0, **DEFAULTS)
    _check(got, ref)
    worst = c["actions"] < A - 1
    assert np.all(got["bonus"][worst] == np.float32(0.9) * np.float32(-1.0))


@pytest.mark.gpu
def test_kernel_hard_max_limit_equals_the_iqn_loss(cuda_dev):
    """alpha = 0, te = 1e-6: the M-IQN kernel computes riqn_iqn_loss_fwd_bwd's loss with a* = argmax of the target mean."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    B, N, Np, A, g = 128, 32, 40, 18, 0.99 ** 3
    c = _case(8, B, Np, A, N=N)
    q = c["q_tgt"].reshape(Np, 2, B, A)
    q[:, 0, np.arange(B), np.random.RandomState(9).randint(0, A, B)] += 3.0
    got = _kernel(c, B, N, Np, A, g, 1.0, 0.0, 1e-6, -1.0)
    dev = cuda_dev
    q_next = torch.from_numpy(np.ascontiguousarray(q[:, 0].reshape(Np * B, A))).to(dev)
    a_star = torch.empty(B, dtype=torch.int64, device=dev)
    call("riqn_argmax_mean", B, Np, A, ptr(q_next), ptr(a_star))
    d = {k: torch.from_numpy(c[k]).to(dev) for k in ("q_on", "tau", "actions", "returns", "nonterminals")}
    o = dict(loss=torch.empty(B, device=dev), dtheta=torch.empty(N * B, device=dev), target=torch.empty(B, Np, device=dev))
    call("riqn_iqn_loss_fwd_bwd", B, N, Np, A, ptr(d["q_on"]), ptr(q_next), ptr(d["tau"]), ptr(d["actions"]), ptr(a_star),
         ptr(d["returns"]), ptr(d["nonterminals"]), float(g), 1.0, ptr(o["loss"]), ptr(o["dtheta"]), None, ptr(o["target"]))
    for k, v in o.items():
        ref = v.cpu().numpy()
        assert np.max(np.abs(got[k] - ref) / np.maximum(np.abs(ref), 1e-30)) < 1e-6, k
    assert np.all(got["bonus"] == 0.0)


@pytest.mark.gpu
def test_kernel_rejects_invalid_arguments_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    B, N, Np = 4, 8, 8
    nan = lambda *s: torch.full(s, math.nan, device=cuda_dev)
    outs = dict(loss=nan(B), dtheta=nan(N * B), theta=nan(B, N), target=nan(B, Np), bonus=nan(B))
    bad = [dict(A=33), dict(te=0.0), dict(te=-0.03), dict(te=math.nan), dict(te=math.inf), dict(l0=0.5),
           dict(l0=math.nan), dict(l0=-math.inf), dict(alpha=-0.1), dict(alpha=math.nan), dict(alpha=math.inf)]
    for kw in bad:
        p = dict(A=18, alpha=0.9, te=0.03, l0=-1.0)
        p.update(kw)
        c = _case(11, B, Np, p["A"], N=N)
        with pytest.raises(RiqnError):
            _kernel(c, B, N, Np, p["A"], 0.97, 1.0, p["alpha"], p["te"], p["l0"], outs=outs)
    torch.cuda.synchronize()
    assert all(bool(torch.isnan(v).all()) for v in outs.values())


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _munchausen_args(dev, B, cfg, **kw):
    a = make_args(dev, B, cfg)
    a.munchausen = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("B,n", [(32, 8), (512, 64)])
def test_learner_step_vs_oracle(cuda_dev, B, n):
    """compute_gradients under Munchausen with injected noises and fractions against the torch oracle's learner step."""
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch, _qmajor
    cfg, seed = cases.iqn_cfg(n, n, 32), 7700 + B
    params = net.make_params(seed)
    lr = Learner(_munchausen_args(cuda_dev, B, cfg), 18, None)
    assert lr.munchausen == (0.9, 0.03, -1.0)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    rs = np.random.RandomState(seed + 2)
    t_tgt = torch.from_numpy(rs.uniform(0, 1, (n * 2 * B, 1)).astype(np.float32))
    t_on = torch.from_numpy(rs.uniform(0, 1, (n * B, 1)).astype(np.float32))
    noises = cases.make_noises(seed + 3, count=2)
    lr._inject = dict(noises=noises, taus=(t_tgt, t_on))
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    assert dbg["bonus"].shape == (B,) and dbg["q_tgt"].shape == (n * 2 * B, 18) and torch.equal(dbg["tau"].cpu(), t_on)
    # the kernel's targets and bonus are the float64 statement of its own target-network quantiles
    t64, b64 = om.soft_target_np(dbg["q_tgt"].cpu().numpy(), b["returns"], b["nonterminals"], b["actions"],
                                 cfg["discount"] ** cfg["n_step"], **DEFAULTS)
    assert rel_err(dbg["target"].cpu().numpy(), t64) < 1e-5 and rel_err(dbg["bonus"].cpu().numpy(), b64) < 1e-5

    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = om.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises,
                                    (t_tgt, t_on), dict(cfg, **DEFAULTS), keep=keep)
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max(np.abs(lg - lo) / np.abs(lo)) < 1e-3
    # ReLU kinks that the product and the oracle round to opposite sides of 0 relax the parameters upstream of them
    gk = dbg["keep"]
    h = _qmajor(gk["h"], B).cpu()
    fl = [int(((a.cpu() > 0) != (b_ > 0)).sum()) for a, b_ in
          ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
           (h[:, :512], keep["h_v"]), (h[:, 512:], keep["h_a"]))]
    relaxed = set()
    if fl[3] + fl[4]:
        relaxed |= {"conv1", "conv2", "conv3", "iqn_fc", "fcnoisy_h_v", "fcnoisy_h_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    for k, g_ref in o_grads.items():
        gg = grads[k]
        cos = float((gg * g_ref).sum() / (gg.norm() * g_ref.norm() + 1e-30))
        rel = float((gg - g_ref).norm() / (g_ref.norm() + 1e-30))
        if k.split(".")[0] in relaxed:
            assert cos > 0.98 and rel < 0.2, (k, cos, rel, fl)
        else:
            assert cos >= 0.999 and rel < 3e-2, (k, cos, rel, fl)


@pytest.mark.gpu
def test_actor_priorities_vs_oracle(cuda_dev):
    """Actor.compute_priorities runs the Munchausen loss per chunk of batch_size transitions (and so the Ape-X actors'
    initial priorities, which come from it)."""
    from rainbow_iqn_apex_b200 import Actor
    bs, L, seed, cfg = 8, 22, 8100, cases.iqn_cfg(8, 8, 8)
    n, hist = cfg["n_step"], 4
    rs = np.random.RandomState(seed)
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(a) for a in rs.randint(0, 18, L)]
    tab_reward = [float(r) for r in rs.randint(-1, 2, L)]
    tab_nonterminal = [1.0] * L
    tab_nonterminal[9] = 0.0
    params = net.make_params(seed)
    actor = Actor(_munchausen_args(cuda_dev, bs, cfg), 18, None)
    load_params(actor.online_net, params)
    actor.update_target_net()
    actor.train()
    chunks = math.ceil((L - n) / bs)
    inj = []
    for c in range(chunks):
        m = min(bs, L - n - c * bs)
        inj.append(dict(noises=cases.make_noises(seed + 10 * c, count=2),
                        taus=(torch.from_numpy(rs.uniform(0, 1, (8 * 2 * m, 1)).astype(np.float32)),
                              torch.from_numpy(rs.uniform(0, 1, (8 * m, 1)).astype(np.float32)))))
    actor._inject = list(inj)
    pri = actor.compute_priorities(tab_state, tab_action, tab_reward, tab_nonterminal, 0.2)
    assert not actor._inject and pri.shape == (L - n,)
    # the oracle: the reference's buffer arithmetic (actor.py:41-124) around the Munchausen loss
    nonterm = np.float32(tab_nonterminal[n:])
    for i in np.where(nonterm == 0)[0]:
        nonterm[i + 1:i + n + 1] = 0
    returns = np.float32([sum(cfg["discount"] ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    p_on, p_tg = net.to_torch(params), net.to_torch(params)
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        with torch.no_grad():
            loss = om.miqn_loss(p_on, p_tg, st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx,
                                torch.from_numpy(nonterm[lo:hi]), inj[c]["noises"], inj[c]["taus"], **cfg, **DEFAULTS)
        out.append(loss.numpy())
    ref = np.power(np.concatenate(out), 0.2)
    assert np.max(np.abs(pri - ref) / ref) < 1e-3


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
    return out, learner.online_net._flat.detach().clone()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_munchausen_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    """Two learners built from the same seed compute bit-identical sampled indices, losses and parameters, eagerly and
    replayed from the step's CUDA graph; the steps differ from plain IQN's."""
    runs = [_bench_learner(cuda_dev, 1 << 14, graph, 3, dict(munchausen=1)) for _ in range(2)]
    (s1, p1), (s2, p2) = runs
    for k, ((i1, l1, _), (i2, l2, _)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2), f"step {k}: sampled indices differ"
        assert torch.equal(l1, l2), f"step {k}: losses differ"
        assert bool(torch.isfinite(l1).all())
    assert torch.equal(p1, p2)
    (s0, p0) = _bench_learner(cuda_dev, 1 << 14, graph, 1)
    assert not torch.equal(s0[0][1], s1[0][1])


@pytest.mark.gpu
def test_plain_learner_is_unchanged(cuda_dev):
    """A namespace without the new fields and one with munchausen=0 run the same launches per step and give bit-identical
    sampled indices, losses and parameters."""
    (s1, p1), (s2, p2) = (_bench_learner(cuda_dev, 1 << 14, False, 3, f) for f in (None, dict(munchausen=0)))
    for k, ((i1, l1, c1), (i2, l2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(l1, l2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_learn_graph_and_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B = 32
    cfg = cases.iqn_cfg(8, 8, 8)
    lr = Learner(_munchausen_args(cuda_dev, B, cfg, munchausen_alpha=0.5, munchausen_tau=0.1, munchausen_l0=-2.0), 18, None)
    assert lr.munchausen == (0.5, 0.1, -2.0)
    b = cases.make_batch(3, B)
    ex = tuple(torch.from_numpy(b[k]).to(cuda_dev) for k in
               ("states", "actions", "returns", "next_states", "nonterminals", "weights"))
    lr.enable_learn_graph(ex)
    for _ in range(2):
        loss = lr.learn_on_graph(ex)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss).all())
    # rejected combinations, at construction and in set_risk
    with pytest.raises(ValueError):
        Agent(_munchausen_args(cuda_dev, B, cfg, risk_measure="cvar", risk_eta=0.25), 18, None)
    a = make_args(cuda_dev, B, cfg, rainbow_only=True)
    a.munchausen = 1
    with pytest.raises(ValueError):
        Agent(a, 18, None)
    for kw in (dict(munchausen_tau=0.0), dict(munchausen_alpha=-1.0), dict(munchausen_l0=0.5), dict(munchausen=2)):
        with pytest.raises(ValueError):
            Agent(_munchausen_args(cuda_dev, B, cfg, **kw), 18, None)
    ag = Agent(_munchausen_args(cuda_dev, B, cfg), 18, None)
    ag.set_risk("neutral")
    with pytest.raises(ValueError):
        ag.set_risk("wang", -0.75)
    assert ag.risk is None


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_replica_runs_the_munchausen_step(cuda_dev):
    """A learner in a one-rank process group takes the data-parallel path (the gradient all-reduce started inside the
    backward, then the rest before Adam) and computes the same bits as the plain learner."""
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
            lr = Learner(_munchausen_args(cuda_dev, B, cfg), 18, None)
            load_params(lr.online_net, params)
            lr.update_target_net()
            lr.train()
            if dp:
                lr.process_group = dist.group.WORLD
            losses_ = [lr.learn_on_batch(*batch).clone() for _ in range(2)]
            torch.cuda.synchronize()
            assert lr._dp_tail is None
            out.append((losses_, lr.online_net._flat.clone()))
        for l1, l2 in zip(out[0][0], out[1][0]):
            assert torch.equal(l1, l2)
        assert torch.equal(out[0][1], out[1][1])
    finally:
        dist.destroy_process_group()
