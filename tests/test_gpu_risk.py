"""Risk-sensitive IQN policies: distorted quantile fractions beta(tau) (Dabney et al. 2018, section 3.1) drawn on the
device by riqn_fill_tau_distorted, and the places they apply -- acting (Actor.act / act_batch / act_batch_values) and
the double-DQN action a* of the loss -- while the N and N' fractions of the quantile-Huber loss stay uniform.

The unmarked tests check the float64 oracle (oracle/risk.py) by the identities of the distortion functions, and the
host-side argument checks.  The gpu tests check the kernel against that oracle applied to riqn_fill_uniform's draw,
the network, the actors and one learner step against the torch oracle, reproducibility, and that the risk-neutral
default issues exactly the launches it issued before the feature existed."""
import math
import struct

import numpy as np
import pytest
import torch

from helpers import load_params, make_args, rel_err
from oracle import cases, losses, network as net, risk as orisk

GRID = np.linspace(0.0, 1.0, 20001)[1:-1]
MEASURES = {                                    # (measure, eta) pairs the device is checked at
    "cvar": [0.1, 0.25, 0.5, 1.0],
    "wang": [-0.75, -0.25, 0.0, 0.5, 2.0],
    "cpw": [0.5, 0.71, 1.0, 1.5],
    "pow": [-2.0, -0.5, 0.0, 0.5, 2.0],
    "norm": [1, 2, 3, 32],
}


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("measure,eta", [("cvar", 1.0), ("pow", 0.0), ("wang", 0.0), ("cpw", 1.0), ("norm", 1),
                                         ("neutral", 0.0)])
def test_oracle_identity_parameters(measure, eta):
    assert np.allclose(orisk.distort(measure, eta, GRID), GRID, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("measure", ["cvar", "wang", "cpw", "pow"])
def test_oracle_monotone(measure):
    for eta in MEASURES[measure]:
        b = orisk.distort(measure, eta, GRID)
        assert np.all(np.isfinite(b)) and np.all(np.diff(b) >= 0), (measure, eta)
        assert b.min() >= 0.0 and b.max() <= 1.0, (measure, eta)


def test_oracle_orderings():
    for eta in MEASURES["cvar"]:
        assert np.all(orisk.distort("cvar", eta, GRID) <= eta)
    averse = [("wang", -0.75), ("wang", -0.25), ("pow", -2.0), ("pow", -0.5), ("cvar", 0.1), ("cvar", 0.5)]
    seeking = [("wang", 0.5), ("wang", 2.0), ("pow", 0.5), ("pow", 2.0)]
    for m, eta in averse:
        assert np.all(orisk.distort(m, eta, GRID) <= GRID), (m, eta)
    for m, eta in seeking:
        assert np.all(orisk.distort(m, eta, GRID) >= GRID), (m, eta)


def test_oracle_norm_is_a_mean():
    u = np.random.RandomState(0).uniform(size=(200000, 4))
    b = orisk.distort("norm", 4, u.ravel())
    assert np.array_equal(b, orisk.distort("norm", 4, u))
    assert np.allclose(b, u.mean(1), rtol=1e-15, atol=1e-15)
    assert abs(b.mean() - 0.5) < 3e-3 and abs(b.var() - 1 / 48) < 1e-3      # Var(mean of 4 uniforms) = 1/(12*4)


# ------------------------------------------------------------------------------------------------ host checks (CPU)
def test_check_risk_domain():
    from rainbow_iqn_apex_b200.model import check_risk
    assert check_risk(None) is None and check_risk(("neutral", None)) is None and check_risk(("NEUTRAL", 3)) is None
    assert check_risk(("CVaR", 1)) == ("cvar", 1.0) and check_risk(("norm", np.int64(4))) == ("norm", 4.0)
    assert check_risk(("wang", np.float32(-0.75))) == ("wang", -0.75)
    bad = [("cvar", 0.0), ("cvar", 1.5), ("cvar", -0.1), ("cvar", math.nan), ("cvar", None), ("cvar", 1e-50),
           ("cpw", 0.0), ("cpw", -1.0), ("cpw", math.inf), ("wang", math.inf), ("wang", math.nan), ("pow", -math.inf),
           ("pow", 1e39), ("norm", 0), ("norm", 33), ("norm", 2.5), ("wang", True), ("wang", "0.5"), ("var", 0.5),
           ("cvar",), "cvar", 0.5]
    for r in bad:
        with pytest.raises(ValueError):
            check_risk(r)


def test_c51_and_invalid_risk_rejected_before_any_launch():
    """Host tensors: the checks raise before a kernel could be reached."""
    from rainbow_iqn_apex_b200.model import DQN
    x = torch.zeros(1, 4, 84, 84, dtype=torch.uint8)
    c51 = DQN(make_args(torch.device("cpu"), rainbow_only=True), 18)
    for call in (lambda: c51(x, risk=("cvar", 0.5)), lambda: c51.forward(x, risk=("wang", -0.75))):
        with pytest.raises(ValueError):
            call()
    iqn = DQN(make_args(torch.device("cpu")), 18)
    with pytest.raises(ValueError):
        iqn(x, 8, risk=("cvar", 2.0))


# ------------------------------------------------------------------------------------------------ kernel (GPU)
SEED, STREAM = 0x1234_5678_9ABC_DEF1, 77


def _fill_uniform(n, stream_id=STREAM, dyn=None):
    from rainbow_iqn_apex_b200._lib import call, ptr
    out = torch.empty(n, device="cuda")
    call("riqn_fill_uniform", n, SEED, stream_id, ptr(out), dyn)
    return out


def _fill_distorted(n, measure, eta, stream_id=STREAM, dyn=None, out=None):
    from rainbow_iqn_apex_b200._lib import call, ptr
    from rainbow_iqn_apex_b200.model import RISK_MEASURES
    out = torch.empty(n, device="cuda") if out is None else out
    code = RISK_MEASURES[measure] if isinstance(measure, str) else measure
    call("riqn_fill_tau_distorted", n, SEED, stream_id, code, eta, ptr(out), dyn)
    return out


def _within_one_ulp(dev, ref64):
    ref32 = ref64.astype(np.float32)
    err = np.abs(dev.astype(np.float64) - ref32.astype(np.float64))
    return err <= np.spacing(np.abs(ref32)).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("measure", list(MEASURES))
def test_kernel_matches_oracle_on_the_plain_draw(cuda_dev, measure):
    n = (1 << 20) + 3
    for eta in MEASURES[measure]:
        eta32 = float(np.float32(eta))                  # eta crosses the C-ABI as a float
        m = int(eta) if measure == "norm" else 1
        u = _fill_uniform(n * m).cpu().numpy()
        dev = _fill_distorted(n, measure, eta).cpu().numpy()
        ref = orisk.distort(measure, eta32, u)
        ok = _within_one_ulp(dev, ref)
        assert np.all(np.isfinite(dev)), (measure, eta)
        assert ok.all(), (measure, eta, int((~ok).sum()), dev[~ok][:4], ref[~ok][:4])
        if measure == "cvar":
            assert np.all(dev <= eta32)


@pytest.mark.gpu
def test_kernel_identities_dyn_offset_and_errors(cuda_dev):
    n = (1 << 20) + 3
    u = _fill_uniform(n)
    for measure, eta in (("cvar", 1.0), ("pow", 0.0), ("pow", -0.0), ("neutral", 0.5), ("norm", 1)):
        assert torch.equal(_fill_distorted(n, measure, eta), u), (measure, eta)
    # the dyn struct's rng_offset is added to the stream id, as in riqn_fill_uniform
    k = 12345
    dyn = torch.tensor(list(struct.pack("<Qffdd", k, 0.0, 0.0, 0.0, 0.0)), dtype=torch.uint8, device=cuda_dev)
    for measure, eta in (("wang", -0.75), ("norm", 4)):
        a = _fill_distorted(n, measure, eta, dyn=dyn.data_ptr())
        assert torch.equal(a, _fill_distorted(n, measure, eta, stream_id=STREAM + k)), measure
        assert not torch.equal(a, _fill_distorted(n, measure, eta)), measure
    assert torch.equal(_fill_uniform(n, dyn=dyn.data_ptr()), _fill_uniform(n, stream_id=STREAM + k))
    # an unknown measure or an eta outside its domain: an error, and nothing written
    from rainbow_iqn_apex_b200._lib import RiqnError
    out = torch.full((4096,), -7.0, device=cuda_dev)
    bad = [(6, 0.5), (-1, 0.5), ("cvar", 0.0), ("cvar", -0.25), ("cvar", 1.5), ("cvar", math.nan), ("cpw", 0.0),
           ("cpw", -1.0), ("cpw", math.inf), ("wang", math.inf), ("wang", -math.inf), ("wang", math.nan),
           ("pow", math.inf), ("pow", math.nan), ("norm", 0.0), ("norm", 33.0), ("norm", 2.5), ("norm", math.nan)]
    for measure, eta in bad:
        with pytest.raises(RiqnError):
            _fill_distorted(4096, measure, eta, out=out)
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())


# ------------------------------------------------------------------------------------------------ network (GPU)
def _next_fractions(d, n, measure, eta):
    """What the network's next eager quantile draw returns under (measure, eta)."""
    from rainbow_iqn_apex_b200 import model
    from rainbow_iqn_apex_b200._lib import call, ptr
    out = torch.empty(n, 1, device=d._flat.device)
    call("riqn_fill_tau_distorted", n, d._rng_seed ^ 0x7A75, d._tau_stream_offset + d._tau_calls + model._EAGER_STREAMS,
         model.RISK_MEASURES[measure], eta, ptr(out), None)
    return out


def _dqn(dev, seed, batch=8):
    from rainbow_iqn_apex_b200.model import DQN
    d = DQN(make_args(dev, batch), 18).to(dev)
    load_params(d, net.make_params(seed))
    d.reset_noise(net.make_noise(seed + 1))
    d.zero_grad()
    return d


@pytest.mark.gpu
def test_network_draws_distorted_fractions(cuda_dev):
    from rainbow_iqn_apex_b200 import _lib
    B, K = 8, 32
    d = _dqn(cuda_dev, 4242, B)
    x = torch.from_numpy(cases.make_batch(4243, B)["states"]).to(cuda_dev)
    with torch.no_grad():
        expect = _next_fractions(d, K * B, "cvar", 0.25)
        q, tau = d(x, K, risk=("cvar", 0.25))
        assert torch.equal(tau, expect) and bool((tau <= 0.25).all())
        q2, tau2 = d(x, K, tau=tau)
        assert torch.equal(q, q2) and torch.equal(tau2, tau)
        # an explicit tau wins over risk
        q3, tau3 = d(x, K, tau=tau, risk=("wang", 1.0))
        assert torch.equal(q3, q) and torch.equal(tau3, tau)
        # neutral is the plain uniform draw; every variant issues one draw launch
        counts = []
        for r in (None, ("neutral", None), ("cvar", 0.25)):
            c0 = _lib.launch_count()
            d(x, K, risk=r)
            counts.append(_lib.launch_count() - c0)
        assert counts[0] == counts[1] == counts[2], counts
        from rainbow_iqn_apex_b200.model import _EAGER_STREAMS
        plain = torch.empty(K * B, 1, device=cuda_dev)
        _lib.call("riqn_fill_uniform", K * B, d._rng_seed ^ 0x7A75, d._tau_stream_offset + d._tau_calls + _EAGER_STREAMS,
                  _lib.ptr(plain), None)
        _, tau_n = d(x, K, risk=("neutral", 0.7))
        assert torch.equal(tau_n, plain)


@pytest.mark.gpu
def test_autograd_call_with_risk_equals_injected_tau(cuda_dev):
    B, K = 8, 32
    d = _dqn(cuda_dev, 5151, B)
    x = torch.from_numpy(cases.make_batch(5152, B)["states"]).to(cuda_dev)
    G = torch.from_numpy(np.random.RandomState(5153).standard_normal((K * B, 18)).astype(np.float32)).to(cuda_dev)
    expect = _next_fractions(d, K * B, "wang", -0.75)
    q1, t1 = d(x, K, risk=("wang", -0.75))
    assert q1.grad_fn is not None and not t1.requires_grad and torch.equal(t1, expect)
    (q1 * G).sum().backward()
    g1 = d._flat_grad.clone()
    d.zero_grad()
    q2, t2 = d(x, K, tau=t1)
    (q2 * G).sum().backward()
    assert torch.equal(q1.detach(), q2.detach()) and torch.equal(t2, t1)
    assert torch.equal(g1, d._flat_grad)
    assert float(g1.norm()) > 0


# ------------------------------------------------------------------------------------------------ actors (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("measure,eta", [("wang", -0.75), ("cvar", 0.25)])
def test_actor_acts_on_q_beta(cuda_dev, measure, eta):
    from rainbow_iqn_apex_b200 import Actor
    E, K, seed = 64, 32, 7300
    args = make_args(cuda_dev, 32, cases.iqn_cfg(64, 64, K))
    args.risk_measure, args.risk_eta = measure, eta
    actor = Actor(args, 18, None)
    assert actor.risk == (measure, float(eta))
    params, noise = net.make_params(seed), net.make_noise(seed + 1)
    load_params(actor.online_net, params)
    actor.train()
    actor.online_net.reset_noise(noise)
    states = np.random.RandomState(seed).randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    sd = torch.from_numpy(states).to(cuda_dev)
    p_on = net.apply_noise(net.to_torch(params), noise)

    def oracle_means(tau):
        with torch.no_grad():
            q = net.dqn_forward_iqn(p_on, torch.from_numpy(states).float().div_(255), K, tau.cpu())
        return q.reshape(K, E, 18).mean(0).numpy()

    tau_v = _next_fractions(actor.online_net, K * E, measure, eta)
    qm = actor.act_batch_values(sd).cpu().numpy()
    assert rel_err(qm, oracle_means(tau_v)) < 1e-3
    tau_a = _next_fractions(actor.online_net, K * E, measure, eta)
    a = actor.act_batch(sd).cpu().numpy()
    qo = oracle_means(tau_a)
    ao = qo.argmax(1)
    for e in np.where(a != ao)[0]:                                      # only numerical ties may differ
        assert abs(qo[e, ao[e]] - qo[e, a[e]]) < 1e-4
    assert (a != ao).sum() <= 1
    # act() on one frame stack: the same draw as act_batch on a batch of one
    tau_1 = _next_fractions(actor.online_net, K, measure, eta)
    a1 = actor.act([states[0, i] for i in range(4)])
    actor._inject_act_tau = tau_1
    assert a1 == int(actor.act_batch(sd[:1])[0])


# ------------------------------------------------------------------------------------------------ learner (GPU)
@pytest.mark.gpu
def test_learner_step_vs_oracle_with_distorted_action_selection(cuda_dev):
    """IQN config-1 shape (B=32, N=N'=8, K=32): injected noises and N / N' fractions; the K pass draws under Wang(-0.75)
    and the oracle is handed the same fractions."""
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch, _qmajor, _tie_mask
    B, cfg, seed = 32, cases.iqn_cfg(8, 8, 32), 6100
    params = net.make_params(seed)
    args = make_args(cuda_dev, B, cfg)
    args.risk_measure, args.risk_eta = "wang", -0.75
    lr = Learner(args, 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    _, t_tgt, t_on = (torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg))
    noises = cases.make_noises(seed + 3)
    lr._inject = dict(noises=noises, taus=(None, t_tgt, t_on))
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    tau_sel = dbg["tau_sel"].cpu()
    assert tau_sel.shape == (32 * B, 1)
    assert bool(((tau_sel > 0) & (tau_sel < 1)).all()) and float(tau_sel.mean()) < 0.4   # E = Phi(-0.75/sqrt 2) = 0.30
    assert torch.equal(dbg["tau"].cpu(), t_on)                         # the N fractions stay as injected (uniform)

    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]),
                                        noises, (tau_sel, t_tgt, t_on), cfg, keep=keep)
    ties = _tie_mask(keep, dbg["a_star"].cpu().numpy(), tol=1e-4)
    ok = ~ties
    assert ties.sum() <= 1
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max(np.abs(lg[ok] - lo[ok]) / np.abs(lo[ok])) < 1e-3
    if ties.any():
        return
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


def _bench_learner(dev, cap, graph, steps, risk=None, record_tau_sel=None):
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib
    torch.manual_seed(5)
    a = bench.make_args(dev, cap)
    if risk is not None:
        a.risk_measure, a.risk_eta = risk
    learner = Learner(a, bench.ACTIONS, None)
    learner.train()
    mem = ReplayMemory(a, None)
    bench.fill_replay(mem, cap, dev, 7)
    drawn = []
    if record_tau_sel is not None:               # keep the K-pass fraction buffers (the captured one is the last)
        on, draw = learner.online_net, learner.online_net.draw_quantiles

        def recording(n, risk=None):
            t = draw(n, risk)
            if risk is not None:
                drawn.append(t)
            return t
        on.draw_quantiles = recording
    if graph:
        learner.enable_cuda_graph(mem)
    out = []
    for _ in range(steps):
        c0 = _lib.launch_count()
        idxs, loss = learner.learn_and_update(mem)
        launches = _lib.launch_count() - c0
        if record_tau_sel is not None:
            record_tau_sel.append(drawn[-1].clone())
        out.append((idxs.clone(), loss.clone(), launches))
    torch.cuda.synchronize()
    return out, learner.online_net._flat.detach().clone()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_risk_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    """Two learners built from the same seed under CVaR(0.1) compute bit-identical sampled indices, losses and
    parameters, eagerly and replayed from the step's CUDA graph (where the dyn offset advances the K-pass fractions)."""
    taus = []
    (s1, p1), (s2, p2) = (_bench_learner(cuda_dev, 1 << 14, graph, 3, ("cvar", 0.1), taus) for _ in range(2))
    for k, ((i1, l1, _), (i2, l2, _)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2), f"step {k}: sampled indices differ"
        assert torch.equal(l1, l2), f"step {k}: losses differ"
    assert torch.equal(p1, p2)
    first = taus[:3]
    assert all(bool((t <= 0.1).all()) for t in first)
    assert not torch.equal(first[0], first[1]) and not torch.equal(first[1], first[2])
    assert all(torch.equal(a, b) for a, b in zip(first, taus[3:]))


@pytest.mark.gpu
def test_neutral_learner_is_unchanged(cuda_dev):
    """A namespace without the new fields and one with risk_measure="neutral" run the same launches per step and give
    bit-identical sampled indices, losses and parameters."""
    (s1, p1), (s2, p2) = (_bench_learner(cuda_dev, 1 << 14, False, 3, risk) for risk in (None, ("neutral", None)))
    for k, ((i1, l1, c1), (i2, l2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(l1, l2), k
        assert c1 == c2, (k, c1, c2)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_risk_configuration_errors(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    args = make_args(cuda_dev, 8, rainbow_only=True)
    args.risk_measure, args.risk_eta = "cvar", 0.5
    with pytest.raises(ValueError):
        Agent(args, 18, None)
    args.risk_measure = "neutral"
    c51 = Agent(args, 18, None)
    with pytest.raises(ValueError):
        c51.set_risk("wang", -0.75)
    for measure, eta in (("cvar", 1.5), ("cvar", None), ("norm", 2.5), ("mean-variance", 0.5)):
        a = make_args(cuda_dev, 8, cases.iqn_cfg(8, 8, 8))
        a.risk_measure, a.risk_eta = measure, eta
        with pytest.raises(ValueError):
            Learner(a, 18, None)
    # a captured step graph holds the measure: set_risk refuses until the graphs are released
    B = 32
    lr = Learner(make_args(cuda_dev, B, cases.iqn_cfg(8, 8, 8)), 18, None)
    lr.set_risk("cpw", 0.71)
    assert lr.risk == ("cpw", 0.71)
    b = cases.make_batch(3, B)
    ex = tuple(torch.from_numpy(b[k]).to(cuda_dev) for k in
               ("states", "actions", "returns", "next_states", "nonterminals", "weights"))
    lr.enable_learn_graph(ex)
    with pytest.raises(RuntimeError, match="recapture"):
        lr.set_risk("cvar", 0.25)
    assert lr.risk == ("cpw", 0.71)
    lr.release_graphs()
    lr.set_risk("cvar", 0.25)
    lr.enable_learn_graph(ex)
    loss = lr.learn_on_graph(ex)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss).all())
