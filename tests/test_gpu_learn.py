"""GPU: end-to-end parity of the learner step (Learner.learn / Agent.compute_loss_actor_or_learner) against
(a) the golden fixtures recorded from the unmodified reference and (b) the CPU oracle on fresh seeded inputs.

Tolerances (BASELINE.json north_star): per-transition fp32 IQN loss within 1e-3 relative; here the fp32 CUDA
path is held to 2e-4, gradients to cosine >= 0.999 and 1e-3 norm-relative (SURVEY.md section 8d)."""
import os

import numpy as np
import pytest
import torch

from helpers import digest, load_params, make_args, rel_err
from oracle import cases, losses, network as net

pytestmark = pytest.mark.gpu
LOSS_TOL = 2e-4      # fp32 / split-bf16x3 forward products; the north_star bound is 1e-3


def _loss_tol():
    """Per-transition loss tolerance of the current forward arithmetic: the single-pass fp16 head (the default) measured
    max 1.6e-4 at B=512 (tests/test_gpu_parity_full.py, forward table), split-bf16x3 / fp32 3e-6."""
    from rainbow_iqn_apex_b200 import model
    return {"fp16": 5e-4, "bf16": 1e-3}.get(model.PRECISION["fwd"], LOSS_TOL)


def _grad_tol():
    """Norm-relative gradient tolerance of the current backward arithmetic (model.PRECISION)."""
    from rainbow_iqn_apex_b200 import model
    return 1e-3 if model.PRECISION["bwd"] in ("fp32", "bf16x3") else 1e-2


@pytest.fixture
def precision():
    from rainbow_iqn_apex_b200 import model
    old = dict(model.PRECISION)
    yield model.set_precision
    model.PRECISION.update(old)


def _cfg(g):
    return cases.iqn_cfg(int(g["cfg_n_tau"]), int(g["cfg_n_tau_prime"]), int(g["cfg_n_quantile"]),
                         float(g["cfg_discount"]), int(g["cfg_n_step"]), float(g["cfg_kappa"]))


class FakeMem:
    def __init__(self, sample):
        self.sample = sample

    def get_sample_from_mp_queue(self, q):
        return self.sample


def _learner(dev, batch, cfg, params):
    from rainbow_iqn_apex_b200 import Learner
    lr = Learner(make_args(dev, batch, cfg), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    return lr


def _dev_batch(b, dev, fp32_frames=False):
    st, nx = torch.from_numpy(b["states"]).to(dev), torch.from_numpy(b["next_states"]).to(dev)
    if fp32_frames:  # the reference's own input format (fp32 / 255)
        st, nx = st.float().div_(255), nx.float().div_(255)
    return (st, torch.from_numpy(b["actions"]).to(dev), torch.from_numpy(b["returns"]).to(dev), nx,
            torch.from_numpy(b["nonterminals"]).to(dev))


@pytest.mark.parametrize("name", ["iqn_small", "iqn_cfg1"])
def test_learn_matches_reference_golden(cuda_dev, golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    seed, batch, steps = int(g["seed"]), int(g["batch"]), int(g["steps"])
    cfg = _cfg(g)
    params_np = net.make_params(seed)
    lr = _learner(cuda_dev, batch, cfg, params_np)
    p_or = net.to_torch(params_np)
    for s in range(steps):
        b = cases.make_batch(seed + 10 + s, batch, n_step=cfg["n_step"], discount=cfg["discount"])
        taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 20 + s, batch, cfg))
        lr._inject = dict(noises=cases.make_noises(seed + 30 + s), taus=taus)
        st, ac, rt, nx, nt = _dev_batch(b, cuda_dev, fp32_frames=(s == 1))
        w = torch.from_numpy(b["weights"]).to(cuda_dev)
        dbg = {}
        loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
        lr.apply_gradients()
        assert rel_err(loss.cpu().numpy(), g[f"loss_{s}"]) < _loss_tol()
        assert np.max(np.abs(loss.cpu().numpy() - g[f"loss_{s}"]) / np.abs(g[f"loss_{s}"])) < 1e-3  # per transition
        # ReLU kinks: with 4..32 samples a single pre-activation that rounds to opposite sides of 0 on the CPU and the
        # GPU moves the conv1/conv2 gradients by percents.  Count them against the oracle's activations (the oracle
        # equals the reference on these inputs -- asserted by make_golden.py): no flip -> the tight tolerance holds for
        # every parameter; k flips -> the parameters upstream of them get 5% each.
        keep_o = {}
        with torch.no_grad():
            losses.iqn_loss(p_or, net.to_torch(params_np), *cases.batch_to_torch(b), lr._inject["noises"],
                            lr._inject["taus"], **cfg, keep=keep_o)
        gk = dbg["keep"]
        fl = [int(((a.cpu() > 0) != (b_ > 0)).sum()) for a, b_ in ((gk["out"][0], keep_o["o1"]), (gk["out"][1], keep_o["o2"]),
                                                                   (gk["out"][2], keep_o["o3"]))]
        upstream = {"conv1": sum(fl), "conv2": fl[1] + fl[2], "conv3": fl[2]}
        for k, p in lr.online_net.named_parameters():
            gd = digest(p.grad)
            ref = g[f"grad_{s}_{k}"]
            nfl = upstream.get(k.split(".")[0], 0)
            gtol = _grad_tol() if nfl == 0 else min(0.25, 5e-2 * nfl)
            assert abs(gd[2] - ref[2]) <= gtol * ref[2] + 1e-9, (k, gd[:3], ref[:3], fl)       # l2 norm
            assert np.allclose(gd[3:], ref[3:], rtol=2 * gtol, atol=2 * gtol * ref[2] / np.sqrt(p.numel()) + 1e-9), (k, fl)
            pd, pref = digest(p), g[f"param_{s}_{k}"]
            if nfl or _grad_tol() > 1e-3:   # l2 norm and leading elements (the signed sum over a tensor amplifies a kink
                # flip, and with the bf16 backward the 1e-2 gradient noise of elements Adam normalises by sqrt(v))
                assert np.allclose(pd[2:], pref[2:], rtol=1e-5, atol=5e-6), k
            else:
                assert np.allclose(pd, pref, rtol=1e-5, atol=1e-6), k
        # the oracle's parameters follow the reference's (param digests above): advance them for the next step's flip count
        for k, p in lr.online_net.named_parameters():
            p_or[k] = p.detach().cpu().clone()


def _qmajor(t, batch):
    """head-internal rows are sample-major (b*Nq + q); the oracle's are quantile-major (q*B + b)."""
    nq = t.shape[0] // batch
    return t.reshape(batch, nq, -1).transpose(0, 1).reshape(batch * nq, -1)


def _tie_mask(keep_oracle, a_star_gpu, tol=1e-5):
    """Samples whose double-DQN argmax differs only because the top-2 oracle Q-means are within tol."""
    a_ref = keep_oracle["a_star"].numpy()
    diff = a_star_gpu != a_ref
    if not diff.any():
        return diff
    K = keep_oracle["q_sel"].shape[0] // len(a_ref)
    qm = keep_oracle["q_sel"].reshape(K, len(a_ref), -1).mean(0).numpy()
    for b in np.where(diff)[0]:
        assert abs(qm[b, a_ref[b]] - qm[b, a_star_gpu[b]]) < tol, "argmax differs beyond a numerical tie"
    return diff


@pytest.mark.parametrize("mode", [("fp32", "fp32"), ("bf16x3", "bf16x3"), ("bf16x3", "bf16"), ("bf16", "bf16"), ("fp16", "bf16")])
# (13, N = 13, N' = 11, K = 7): odd B and B * N, the fp32 trunk and head backwards behind every forward arithmetic
@pytest.mark.parametrize("batch,cfg", [(16, cases.iqn_cfg(64, 64, 32)), (5, cases.iqn_cfg(16, 24, 8, kappa=0.5)),
                                       (13, cases.iqn_cfg(13, 11, 7))])
def test_loss_api_and_autograd_vs_oracle(cuda_dev, precision, batch, cfg, mode):
    """Agent.compute_loss_actor_or_learner + (weights*loss).mean().backward() + optimiser.step(), the exact
    call sequence of learner.py:18-24, against the oracle (autograd on CPU)."""
    from rainbow_iqn_apex_b200 import Agent
    precision(*mode)
    loss_tol = _loss_tol()                                  # bf16 operands: the north_star bound itself
    act_tol = {"bf16": 2e-3, "fp16": 3e-4}.get(mode[0], 1e-4)
    seed = 900 + batch
    params = net.make_params(seed)
    ag = Agent(make_args(cuda_dev, batch, cfg), 18, None)
    load_params(ag.online_net, params)
    ag.update_target_net()
    b = cases.make_batch(seed + 1, batch, n_step=cfg["n_step"], discount=cfg["discount"])
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, batch, cfg))
    noises = cases.make_noises(seed + 3)
    ag._inject = dict(noises=noises, taus=taus)
    dbg = {}
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    loss = ag.compute_loss_actor_or_learner(st, ac, rt, nx, nt, debug=dbg)
    assert loss.requires_grad
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    ag.online_net.zero_grad()
    (w * loss).mean().backward()
    grads_gpu = {k: p.grad.detach().cpu().clone() for k, p in ag.online_net.named_parameters()}
    ag.optimiser.step()

    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]),
                                        noises, taus, cfg, keep=keep)
    ties = _tie_mask(keep, dbg["a_star"].cpu().numpy(), tol={"bf16": 1e-3, "fp16": 1e-4}.get(mode[0], 1e-5))
    ok = ~ties
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max(np.abs(lg[ok] - lo[ok]) / np.abs(lo[ok])) < loss_tol
    assert rel_err(dbg["theta"].cpu().numpy(), keep["theta"].detach().numpy()) < act_tol
    assert rel_err(dbg["target"].cpu().numpy()[ok], keep["target"].numpy()[ok]) < act_tol
    # ReLU-kink flips between the CPU and GPU activations (see the golden test) relax the gradient check
    gk = dbg["keep"]
    flips = sum(int(((a.cpu() > 0) != (b_ > 0)).sum()) for a, b_ in
                ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
                 (_qmajor(gk["h"], batch)[:, :512], keep["h_v"]), (_qmajor(gk["h"], batch)[:, 512:], keep["h_a"])))
    if not ties.any():
        for k, g_ref in o_grads.items():
            gg = grads_gpu[k]
            cos = float((gg * g_ref).sum() / (gg.norm() * g_ref.norm() + 1e-30))
            rel = float((gg - g_ref).norm() / (g_ref.norm() + 1e-30))
            if flips == 0:
                assert cos > 0.999 and rel < (3e-2 if mode[0] in ("bf16", "fp16") else _grad_tol()), (k, cos, rel)   # SURVEY 8d gate: cos
                assert np.allclose(dict(ag.online_net.named_parameters())[k].detach().cpu().numpy(),
                                   p_on[k].detach().numpy(), rtol=0, atol=1e-6 if _grad_tol() < 5e-3 else 5e-6), k
            else:
                assert cos > 0.98 and rel < 0.2, (k, cos, rel, flips)     # many ReLU kinks flip when the forward is bf16


def test_no_grad_path_and_native_rng(cuda_dev):
    """Actor-style use (no optimiser, device RNG): loss is finite, positive and differs between calls because
    noise / quantiles are resampled (compute_loss_iqn.py:234,255,289; model.py:131-134)."""
    from rainbow_iqn_apex_b200 import Agent
    cfg = cases.iqn_cfg(16, 16, 8)
    ag = Agent(make_args(cuda_dev, 8, cfg), 18, None)
    b = cases.make_batch(5, 8)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    with torch.no_grad():
        l1 = ag.compute_loss_actor_or_learner(st, ac, rt, nx, nt)
        l2 = ag.compute_loss_actor_or_learner(st, ac, rt, nx, nt)
    assert not l1.requires_grad and torch.isfinite(l1).all() and (l1 > 0).all()
    assert not torch.equal(l1, l2)
    # online and target nets must not share a noise stream
    assert not torch.equal(ag.online_net.fcnoisy_h_v.weight_epsilon, ag.target_net.fcnoisy_h_v.weight_epsilon)
    assert not torch.equal(ag.online_net.fcnoisy_h_v.bias_epsilon[:8], ag.online_net.fcnoisy_h_a.bias_epsilon[:8])


def test_checkpoint_roundtrip(cuda_dev, tmp_path):
    """Agent.save schema (agent.py:150-160) and reload through args.model (agent.py:26-34,45-47)."""
    from rainbow_iqn_apex_b200 import Learner
    cfg = cases.iqn_cfg(8, 8, 4)
    lr = _learner(cuda_dev, 4, cfg, net.make_params(41))
    b = cases.make_batch(6, 4)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    lr.learn(FakeMem((np.arange(4), st, ac, rt, nx, nt, w)), None)
    lr.save(str(tmp_path), 123, 45, "ckpt.pth")
    ck = torch.load(os.path.join(str(tmp_path), "ckpt.pth"), map_location="cpu")
    assert set(ck) == {"T_actors", "T_learner", "model_state_dict", "optimiser_state_dict"}
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    assert len(ck["optimiser_state_dict"]["state"]) == 24
    # a stock torch Adam over a reference-shaped parameter list accepts the optimiser state
    ref_params = [torch.nn.Parameter(torch.zeros_like(p)) for p in lr.online_net.parameters()]
    torch.optim.Adam(ref_params, lr=5e-5, eps=3.125e-4).load_state_dict(ck["optimiser_state_dict"])
    args = make_args(cuda_dev, 4, cfg)
    args.model = os.path.join(str(tmp_path), "ckpt.pth")
    lr2 = Learner(args, 18, None)
    assert torch.equal(lr2.online_net._flat, lr.online_net._flat)
    assert torch.equal(lr2.optimiser._exp_avg, lr.optimiser._exp_avg) and lr2.optimiser._step == 1
    # both continue identically under identical injected randomness
    inj = dict(noises=cases.make_noises(77), taus=tuple(torch.from_numpy(t) for t in cases.make_taus(78, 4, cfg)))
    lr._inject = lr2._inject = inj
    lr2.update_target_net(); lr.update_target_net()
    _, la = lr.learn(FakeMem((np.arange(4), st, ac, rt, nx, nt, w)), None)
    _, lb = lr2.learn(FakeMem((np.arange(4), st, ac, rt, nx, nt, w)), None)
    assert torch.equal(la, lb)                      # the forward passes are deterministic
    # and so are the backward passes (B = 4: the fp32 trunk backward; every cross-block sum in a fixed order)
    assert torch.equal(lr2.online_net._flat, lr.online_net._flat)


@pytest.mark.parametrize("batch", [512])
def test_full_size_config2_vs_oracle(cuda_dev, batch):
    """BASELINE config 2 (B=512, N=N'=64, K=32): one full learner step against the CPU oracle."""
    cfg = cases.iqn_cfg(64, 64, 32)
    seed = 5150
    params = net.make_params(seed)
    lr = _learner(cuda_dev, batch, cfg, params)
    b = cases.make_batch(seed + 1, batch)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, batch, cfg))
    noises = cases.make_noises(seed + 3)
    lr._inject = dict(noises=noises, taus=taus)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    from rainbow_iqn_apex_b200 import compute_loss_iqn
    loss, _ = compute_loss_iqn.loss_core(lr, st, ac, rt, nx, nt, keep_graph=False, debug=dbg)
    p_on, p_tg = net.to_torch(params), net.to_torch(params)
    keep = {}
    with torch.no_grad():
        o_loss = losses.iqn_loss(p_on, p_tg, *cases.batch_to_torch(b), noises, taus, **cfg, keep=keep)
    ties = _tie_mask(keep, dbg["a_star"].cpu().numpy())
    ok = ~ties
    assert ties.sum() <= 2
    lg, lo = loss.cpu().numpy(), o_loss.numpy()
    assert np.max(np.abs(lg[ok] - lo[ok]) / np.abs(lo[ok])) < 1e-3          # north_star tolerance
    assert np.max(np.abs(lg[ok] - lo[ok]) / np.abs(lo[ok])) < _loss_tol()   # what the default arithmetic achieves


# ----------------------------------------------------------------------------------------------- C51 (rainbow_only)
def test_c51_learn_matches_reference_golden(cuda_dev, golden_dir):
    """BASELINE config 3 path: categorical loss (agent.py:77-141) + backward + Adam against the fixtures recorded from
    the unmodified reference (two consecutive Learner.learn calls)."""
    from rainbow_iqn_apex_b200 import Learner
    g = np.load(os.path.join(golden_dir, "c51_small.npz"))
    seed, batch, steps = int(g["seed"]), int(g["batch"]), int(g["steps"])
    lr = Learner(make_args(cuda_dev, batch, rainbow_only=True), 18, None)
    load_params(lr.online_net, net.make_params(seed, rainbow_only=True))
    lr.update_target_net()
    lr.train()
    for s in range(steps):
        b = cases.make_batch(seed + 10 + s, batch)
        lr._inject = dict(noises=cases.make_noises(seed + 30 + s, rainbow_only=True), taus=None)
        st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
        w = torch.from_numpy(b["weights"]).to(cuda_dev)
        _, loss = lr.learn(FakeMem((np.arange(batch), st, ac, rt, nx, nt, w)), None)
        assert np.max(np.abs(loss.cpu().numpy() - g[f"loss_{s}"]) / np.abs(g[f"loss_{s}"])) < LOSS_TOL
        for k, p in lr.online_net.named_parameters():
            gd, ref = digest(p.grad), g[f"grad_{s}_{k}"]
            gtol = 5e-2 if k.startswith(("conv1", "conv2")) else 2e-3
            assert abs(gd[2] - ref[2]) <= gtol * ref[2] + 1e-9, (k, gd[:3], ref[:3])
            pd, pref = digest(p), g[f"param_{s}_{k}"]
            assert np.allclose(pd[2:], pref[2:], rtol=1e-5, atol=5e-6), k


def test_c51_loss_api_vs_oracle(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent
    batch, seed = 16, 777
    params = net.make_params(seed, rainbow_only=True)
    ag = Agent(make_args(cuda_dev, batch, rainbow_only=True), 18, None)
    load_params(ag.online_net, params)
    ag.update_target_net()
    b = cases.make_batch(seed + 1, batch)
    noises = cases.make_noises(seed + 3, rainbow_only=True)
    ag._inject = dict(noises=noises, taus=None)
    dbg = {}
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    loss = ag.compute_loss_actor_or_learner(st, ac, rt, nx, nt, debug=dbg)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    ag.online_net.zero_grad()
    (w * loss).mean().backward()
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss = losses.c51_loss(p_on, p_tg, *cases.batch_to_torch(b), noises, keep=keep)
    (torch.from_numpy(b["weights"]) * o_loss).mean().backward()
    assert torch.equal(dbg["a_star"].cpu(), keep["a_star"])
    assert rel_err(dbg["m"].cpu().numpy(), keep["m"].numpy()) < 1e-4
    assert np.max(np.abs(loss.detach().cpu().numpy() - o_loss.detach().numpy()) / np.abs(o_loss.detach().numpy())) < LOSS_TOL
    for k in ("fcnoisy_z_a.weight_mu", "fcnoisy_z_v.weight_sigma", "fcnoisy_h_a.weight_mu", "fcnoisy_h_v.bias_sigma", "conv3.weight"):
        gg, gr = dict(ag.online_net.named_parameters())[k].grad.cpu(), p_on[k].grad
        cos = float((gg * gr).sum() / (gg.norm() * gr.norm() + 1e-30))
        assert cos > 0.999, (k, cos)
    # Actor.act on the categorical head (actor.py:19-21) agrees with the oracle's expected-value argmax
    from rainbow_iqn_apex_b200 import Actor
    actor = Actor(make_args(cuda_dev, batch, rainbow_only=True), 18, None)
    load_params(actor.online_net, params)
    actor.eval()
    frames = [b["states"][0, i] for i in range(4)]
    a = actor.act(frames)
    p_eval = net.dqn_forward_c51(net.to_torch(params), torch.from_numpy(b["states"][:1]).float().div_(255), 18, 51, training=False)
    assert a == int((p_eval * torch.linspace(-10, 10, 51)).sum(2).argmax(1))


def _assert_steps_bitwise_reproducible(dev, graph, rainbow_only, cap, steps=6, **fields):
    """``fields``: arguments that replace the benchmark's (batch_size, history_length, ...)."""
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory

    def run():
        torch.manual_seed(5)
        a = bench.make_args(dev, cap, rainbow_only=rainbow_only)
        if rainbow_only:
            a.lr, a.adam_eps = 6.25e-5, 1.5e-4                     # bench.c51_leg
        for k, v in fields.items():
            setattr(a, k, v)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        if graph:
            learner.enable_cuda_graph(mem)
        out = []
        for _ in range(steps):
            idxs, loss = learner.learn_and_update(mem)
            out.append((idxs.clone(), loss.clone()))
        torch.cuda.synchronize()
        return out, learner.online_net._flat.detach().clone()

    (s1, p1), (s2, p2) = run(), run()
    for k, ((i1, l1), (i2, l2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2), f"step {k}: sampled indices differ"
        assert torch.equal(l1, l2), f"step {k}: losses differ"
    assert torch.equal(p1, p2), "parameters differ"


@pytest.mark.parametrize("graph", [False, True])
def test_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    """Two learners built from the same seed draw the same prioritized samples and compute bit-identical losses and
    parameters over several steps at the benchmarked size, eagerly and replayed from the step's CUDA graph.  The losses become the next steps' priorities, so any
    order-dependent rounding (a float atomic in a cross-block sum) would change which transitions are drawn later."""
    _assert_steps_bitwise_reproducible(cuda_dev, graph, rainbow_only=0, cap=1 << 14)


@pytest.mark.parametrize("graph", [False, True])
def test_c51_learner_steps_are_bitwise_reproducible(cuda_dev, graph):
    """The same for the Rainbow-only (C51) learner at B = 512 (bench.c51_leg's learning rate and Adam epsilon): its
    z-layer weight gradients are split-K products over the batch rows, whose partials must be added in a fixed order."""
    _assert_steps_bitwise_reproducible(cuda_dev, graph, rainbow_only=1, cap=1 << 14)
