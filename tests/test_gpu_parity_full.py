"""GPU: parity at the BENCHMARKED configuration and beyond one step (VERDICT round 1, "What's weak" 1-5):

  (a) full Learner.learn at B=512, N=N'=64, K=32 against the CPU oracle: per-parameter gradient cosine / norm-relative
      error, post-Adam parameter displacement, argmax-tie and ReLU-kink aware;
  (b) 20-step trajectories at B=32 (injected noise / quantiles): loss parity and parameter drift per arithmetic mode;
  (c) data-parallel equivalence on ONE GPU: two half-batch replicas + arena sum + grad_scale = 1/2 == one learner on the
      concatenated batch (SURVEY 8e);
  (d) forward arithmetic table at B=512: per-transition relative loss error (max / p99) of every forward mode;
  (e) C51 (config 3) at B=512 against the oracle;
  (f) IQN Actor.act / act_batch / compute_priorities / buffer flush against the reference fixture (actor_small.npz,
      recorded from the unmodified reference by oracle/make_golden.py) and the oracle.

Each test prints its numbers as one JSON line (visible with pytest -s).
"""
import json
import os

import numpy as np
import pytest
import torch

from helpers import load_params, make_args, rel_err
from oracle import actor as oactor, cases, losses, network as net
from test_gpu_learn import FakeMem, _dev_batch, _learner, _qmajor, _tie_mask, precision  # noqa: F401
from test_oracle_golden import actor_case

pytestmark = pytest.mark.gpu


def _rel_loss(lg, lo, ok):
    r = np.abs(lg - lo) / np.abs(lo)
    r = np.sort(r[ok])
    return dict(max=float(r[-1]), p99=float(r[int(0.99 * (len(r) - 1))]), median=float(np.median(r)))


def _flips(gk, keep, batch):
    pairs = ((gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
             (_qmajor(gk["h"], batch)[:, :512], keep["h_v"]), (_qmajor(gk["h"], batch)[:, 512:], keep["h_a"]))
    return [int(((a.cpu() > 0) != (b_ > 0)).sum()) for a, b_ in pairs]


# ------------------------------------------------------------------------------------------------ shared B=512 case
class Case512:
    cfg = cases.iqn_cfg(64, 64, 32)
    seed, batch = 6160, 512

    def __init__(self):
        self.params = net.make_params(self.seed)
        self.b = cases.make_batch(self.seed + 1, self.batch)
        self.taus = tuple(torch.from_numpy(t) for t in cases.make_taus(self.seed + 2, self.batch, self.cfg))
        self.noises = cases.make_noises(self.seed + 3)
        self.keep = {}
        p_on, p_tg = net.to_torch(self.params), net.to_torch(self.params)
        with torch.no_grad():
            self.o_loss = losses.iqn_loss(p_on, p_tg, *cases.batch_to_torch(self.b), self.noises, self.taus, **self.cfg,
                                          keep=self.keep).numpy()


@pytest.fixture(scope="module")
def case512():
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    return Case512()


def _gpu_forward(dev, c, mode=None):
    from rainbow_iqn_apex_b200 import compute_loss_iqn, model
    old = dict(model.PRECISION)
    if mode is not None:
        model.set_precision(*mode)
    try:
        lr = _learner(dev, c.batch, c.cfg, c.params)
        lr._inject = dict(noises=c.noises, taus=c.taus)
        st, ac, rt, nx, nt = _dev_batch(c.b, dev)
        dbg = {}
        loss, _ = compute_loss_iqn.loss_core(lr, st, ac, rt, nx, nt, keep_graph=False, debug=dbg)
        return lr, loss.cpu().numpy(), dbg["a_star"].cpu().numpy()
    finally:
        model.PRECISION.update(old)


def test_forward_arithmetic_table_b512(cuda_dev, case512):
    """(d) Every forward mode at the benchmarked size: the per-transition relative loss error distribution decides
    the default (the cheapest mode whose MAX stays 3x inside the north_star bound of 1e-3)."""
    from rainbow_iqn_apex_b200 import model
    c = case512
    table = {}
    for mode in (("bf16x3", "bf16"), ("fp16", "bf16"), ("bf16", "bf16")):
        _, lg, a_star = _gpu_forward(cuda_dev, c, mode)
        ties = _tie_mask(c.keep, a_star, tol=2e-3 if mode[0] == "bf16" else 1e-4)
        table[mode[0]] = dict(_rel_loss(lg, c.o_loss, ~ties), ties=int(ties.sum()))
    print("forward arithmetic vs oracle at B=512:", json.dumps(table))
    assert table["bf16x3"]["max"] < 2e-4
    assert table["fp16"]["max"] < 3.4e-4                      # 3x margin to the north_star tolerance
    assert table[model.PRECISION["fwd"]]["max"] < 1e-3        # the default, against the north_star bound itself


def test_full_size_learn_step_gradients_vs_oracle(cuda_dev, case512):
    """(a) Config 2 in the DEFAULT arithmetic: loss, every parameter's gradient and the Adam step against the oracle."""
    from rainbow_iqn_apex_b200 import model
    c = case512
    lr, lg0, a_star = _gpu_forward(cuda_dev, c)
    ties = _tie_mask(c.keep, a_star, tol=1e-4)
    assert ties.sum() <= 2
    w_np = c.b["weights"].copy()
    w_np[ties] = 0.0                                          # a flipped double-DQN action changes that transition's target
    w = torch.from_numpy(w_np)
    lr._inject = dict(noises=c.noises, taus=c.taus)
    dbg = {}
    st, ac, rt, nx, nt = _dev_batch(c.b, cuda_dev)
    p0 = lr.online_net._flat.clone()
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w.to(cuda_dev), debug=dbg)
    lr.apply_gradients()
    grads_gpu = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    p_on, p_tg = net.to_torch(c.params, requires_grad=True), net.to_torch(c.params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(c.b), w, c.noises, c.taus, c.cfg, keep=keep)
    ok = ~ties
    lrel = _rel_loss(loss.cpu().numpy(), o_loss.numpy(), ok)
    assert lrel["max"] < 1e-3, lrel
    flips = _flips(dbg["keep"], keep, c.batch)
    report = dict(precision=dict(model.PRECISION), loss=lrel, ties=int(ties.sum()), relu_flips=dict(zip(
        ("conv1", "conv2", "conv3", "h_v", "h_a"), flips)), grads={})
    named = dict(lr.online_net.named_parameters())
    lr_, eps_ = 5e-5, 3.125e-4
    for k, g_ref in o_grads.items():
        gg = grads_gpu[k]
        cos = float((gg * g_ref).sum() / (gg.norm() * g_ref.norm() + 1e-30))
        rel = float((gg - g_ref).norm() / (g_ref.norm() + 1e-30))
        # Adam displacement against the oracle's, on elements whose gradient dominates adam_eps (step 1: |dp| = lr*|g|/(|g|+eps))
        dp_gpu = (named[k].detach().cpu() - torch.from_numpy(c.params[k])).reshape(-1)
        dp_ref = (p_on[k].detach() - torch.from_numpy(c.params[k])).reshape(-1)
        big = g_ref.reshape(-1).abs() > 10 * eps_
        dperr = float((dp_gpu - dp_ref).abs().max() / lr_)
        dperr_big = float((dp_gpu - dp_ref)[big].abs().max() / lr_) if big.any() else 0.0
        report["grads"][k] = dict(cos=cos, rel=rel, adam_step_err_over_lr=dperr, adam_step_err_over_lr_big_g=dperr_big,
                                  n_big=int(big.sum()))
    print("B=512 learn step vs oracle:", json.dumps(report))
    for k, r in report["grads"].items():
        assert r["cos"] >= 0.999, (k, r)                       # SURVEY 8d gate
        assert r["rel"] < (2e-3 if model.PRECISION["bwd"] != "bf16" else 2e-2), (k, r)
        # a wrong bias correction / grad_scale would show as O(1) in both; elements with |g| << adam_eps amplify noise
        assert r["adam_step_err_over_lr"] < 0.15 and r["adam_step_err_over_lr_big_g"] < 0.01, (k, r)


@pytest.mark.parametrize("mode", [("fp32", "fp32"), ("bf16x3", "bf16x3"), ("bf16x3", "bf16"), ("fp16", "bf16")])
def test_trajectory_20_steps_vs_oracle(cuda_dev, precision, mode):
    """(b) 20 consecutive learner steps at B=32 with injected randomness: per-step loss parity and parameter drift
    relative to the distance travelled.  ("fp32", "fp32") = CUDA-core fp32 GEMMs, i.e. the reference's own arithmetic in a
    different summation order: it is the yardstick for how fast two fp32 implementations separate (Adam divides
    by sqrt(v), so elements with tiny gradients amplify last-bit differences) -- round 2 measured a loss gap of up to
    1.3e-3 on single small-loss transitions after 12 steps even for the fp32-faithful bf16x3 arithmetic."""
    precision(*mode)
    batch, steps, seed = 32, 20, 7300
    cfg = cases.iqn_cfg(64, 64, 32)
    params = net.make_params(seed)
    lr = _learner(cuda_dev, batch, cfg, params)
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    from rainbow_iqn_apex_b200 import compute_loss_iqn
    named = dict(lr.online_net.named_parameters())
    hist = []
    for s in range(steps):
        b = cases.make_batch(seed + 10 + s, batch)
        taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 100 + s, batch, cfg))
        noises = cases.make_noises(seed + 200 + s)
        st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
        # forward-only pass on both sides to mask argmax near-ties (a flip would fork the trajectories)
        lr._inject = dict(noises=noises, taus=taus)
        dbg = {}
        compute_loss_iqn.loss_core(lr, st, ac, rt, nx, nt, keep_graph=False, debug=dbg)
        keep = {}
        with torch.no_grad():
            losses.iqn_loss({k: v.detach().clone() for k, v in p_on.items()}, {k: v.clone() for k, v in p_tg.items()},
                            *cases.batch_to_torch(b), noises, taus, **cfg, keep=keep)
        ties = _tie_mask(keep, dbg["a_star"].cpu().numpy(), tol=1e-4)
        w_np = b["weights"].copy()
        w_np[ties] = 0.0
        w = torch.from_numpy(w_np)
        lr._inject = dict(noises=noises, taus=taus)
        _, loss = lr.learn(FakeMem((np.arange(batch), st, ac, rt, nx, nt, w.to(cuda_dev))), None)
        o_loss, _ = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), w, noises, taus, cfg)
        lrel = _rel_loss(loss.cpu().numpy(), o_loss.numpy(), ~ties)
        num = den = 0.0
        maxabs = 0.0
        for k in p_on:
            if not net.is_trainable(k):
                continue
            pg, pr, p0 = named[k].detach().cpu(), p_on[k].detach(), torch.from_numpy(params[k])
            num += float(((pg - pr) ** 2).sum())
            den += float(((pr - p0) ** 2).sum())
            maxabs = max(maxabs, float((pg - pr).abs().max()))
        hist.append(dict(step=s, loss_max_rel=lrel["max"], loss_p99_rel=lrel["p99"], loss_median_rel=lrel["median"], drift=float(np.sqrt(num / den)), max_abs_over_lr=maxabs / 5e-5,
                         ties=int(ties.sum())))
    print("trajectory", mode, json.dumps(hist[-1]), "worst loss", max(h["loss_max_rel"] for h in hist))
    assert hist[0]["loss_max_rel"] < 1e-3                                        # same parameters: the north_star bound
    assert max(h["loss_median_rel"] for h in hist) < 1e-4 and max(h["loss_max_rel"] for h in hist) < 1e-2
    assert hist[-1]["drift"] < 0.02, hist[-1]                                    # distance to the oracle / distance travelled


def test_data_parallel_equivalence_one_gpu(cuda_dev):
    """(c) SURVEY 8e: two replicas on half batches, gradient arenas summed (what the all-reduce does), grad_scale = 1/2,
    identical noise on both replicas == ONE learner on the concatenated batch, up to fp32 reduction-order noise."""
    B, cfg, seed = 32, cases.iqn_cfg(16, 16, 8), 8400
    params = net.make_params(seed)
    full = _learner(cuda_dev, 2 * B, cfg, params)
    halves = [_learner(cuda_dev, B, cfg, params) for _ in range(2)]
    b = cases.make_batch(seed + 1, 2 * B)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, 2 * B, cfg))
    noises = cases.make_noises(seed + 3)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    full._inject = dict(noises=noises, taus=taus)
    loss_full = full.compute_gradients(st, ac, rt, nx, nt, w).clone()
    g_full = full.online_net._flat_grad.clone()
    losses_h = []
    for h, lrn in enumerate(halves):
        sl = slice(h * B, (h + 1) * B)
        th = tuple(t.view(-1, 2 * B)[:, sl].reshape(-1, 1).contiguous() for t in taus)   # rows are quantile-major
        lrn._inject = dict(noises=noises, taus=th)
        losses_h.append(lrn.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl]).clone())
    assert torch.equal(torch.cat(losses_h), loss_full)               # per-transition work is independent of the sharding
    g_sum = halves[0].online_net._flat_grad + halves[1].online_net._flat_grad
    assert float((0.5 * g_sum - g_full).norm() / g_full.norm()) < 1e-5
    for lrn in halves:                                               # every rank applies the same reduced gradient
        lrn.online_net._flat_grad.copy_(g_sum)
        lrn.optimiser.grad_scale = 0.5
        lrn.optimiser.step()
    full.optimiser.step()
    assert torch.equal(halves[0].online_net._flat, halves[1].online_net._flat)
    dp = (halves[0].online_net._flat - full.online_net._flat).abs().max().item()
    assert dp < 3e-8, dp                                             # a few ulp of a 0.06-sized weight (6e-4 of one Adam step); observed 1 ulp
    # the native noise path: replicas sharing the Philox seed and counters draw identical epsilons (parallel.py)
    n0, n1 = halves[0].online_net, halves[1].online_net
    n1._rng_seed = n0._rng_seed
    for (_, m0), (_, m1) in zip(n0.noisy_layers(), n1.noisy_layers()):
        m0._noise_calls = m1._noise_calls = 0
    n0.reset_noise()
    n1.reset_noise()
    assert torch.equal(n0._eps_flat, n1._eps_flat) and float(n0._eps_flat.abs().sum()) > 0


def test_c51_full_size_vs_oracle(cuda_dev):
    """(e) BASELINE config 3 (rainbow_only, B=512): categorical loss, gradients and Adam against the oracle."""
    from rainbow_iqn_apex_b200 import Learner
    batch, seed = 512, 9100
    params = net.make_params(seed, rainbow_only=True)
    lr = Learner(make_args(cuda_dev, batch, rainbow_only=True), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, batch)
    noises = cases.make_noises(seed + 3, rainbow_only=True)
    lr._inject = dict(noises=noises, taus=None)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"])
    _, loss = lr.learn(FakeMem((np.arange(batch), st, ac, rt, nx, nt, w.to(cuda_dev))), None)
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=6.25e-5, eps=1.5e-4)
    ocfg = dict(atoms=51, v_min=-10.0, v_max=10.0, discount=0.99, n_step=3)
    keep = {}
    o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), w, noises, None, ocfg, rainbow_only=True,
                                        keep=keep)
    lg, lo = loss.cpu().numpy(), o_loss.numpy()
    rel = np.abs(lg - lo) / np.abs(lo)
    # a flipped double-DQN action (near-tie of two expected values) changes the projected target of that transition
    bad = rel > 1e-3
    assert bad.sum() <= 2, (int(bad.sum()), float(rel.max()))
    report = dict(loss_max_rel=float(rel[~bad].max()), flipped=int(bad.sum()), grads={})
    for k, g_ref in o_grads.items():
        gg = dict(lr.online_net.named_parameters())[k].grad.cpu()
        cos = float((gg * g_ref).sum() / (gg.norm() * g_ref.norm() + 1e-30))
        report["grads"][k] = dict(cos=cos, rel=float((gg - g_ref).norm() / (g_ref.norm() + 1e-30)))
    print("C51 B=512 vs oracle:", json.dumps(report))
    if not bad.any():
        for k, r in report["grads"].items():
            assert r["cos"] >= 0.999, (k, r)


# ------------------------------------------------------------------------------------------------ actor side
def test_actor_matches_reference_golden(cuda_dev, golden_dir):
    """(f) Actor.act / compute_priorities / flush (actor.py:15-25, 41-124; launch_actor.py:116-140) against the outputs
    recorded from the unmodified reference."""
    from rainbow_iqn_apex_b200 import Actor, ReplayMemory
    g = np.load(os.path.join(golden_dir, "actor_small.npz"))
    cfg, seed, bs, tab_state, tab_action, tab_reward, tab_nonterminal, noises, taus = actor_case(g)
    actor = Actor(make_args(cuda_dev, bs, cfg, actor_capacity=64), 18, None)
    load_params(actor.online_net, net.make_params(seed))
    actor.update_target_net()
    actor.train()
    # act: reset_noise (launch_actor.py:76-77) then the greedy action of the K-quantile mean
    actor.online_net.reset_noise(net.make_noise(seed + 1))
    actor._inject_act_tau = torch.from_numpy(g["act_tau"])
    assert actor.act(tab_state[:4]) == int(g["act_action"])
    actor._inject_act_tau = torch.from_numpy(g["act_tau"])
    qm = actor.act_batch_values(torch.from_numpy(np.stack(tab_state[:4]))[None].to(cuda_dev))
    assert rel_err(qm.cpu().numpy()[0], g["act_q_mean"]) < 1e-3
    # compute_priorities: one injection per chunk of batch_size transitions
    actor._inject = [dict(noises=noises[c], taus=taus[c]) for c in range(len(noises))]
    pri = actor.compute_priorities(tab_state, tab_action, tab_reward, tab_nonterminal, 0.2)
    assert pri.shape == g["priorities"].shape and not actor._inject
    assert np.max(np.abs(pri - g["priorities"]) / g["priorities"]) < 1e-3
    # tail rule + append: the last n steps enter with the shard's max priority
    mem = ReplayMemory(make_args(cuda_dev, bs, cfg, actor_capacity=64), None)
    mem.transitions.max_priority.fill_(1.25)
    fl = actor.flush_priorities(g["priorities"], mem)
    assert np.array_equal(fl, g["flushed"])
    n = cfg["n_step"]
    buf = [[i, tab_state[i + 3], tab_action[i], tab_reward[i], not tab_nonterminal[i]] for i in range(len(tab_action))]
    actor._inject = [dict(noises=noises[c], taus=taus[c]) for c in range(len(noises))]
    nxt = actor.flush_buffer(mem, buf, 50, 0, tab_state, tab_action, tab_reward, tab_nonterminal, T_actor=22)
    assert nxt == (50 + len(buf)) % 64 and mem.transitions.actor_full
    C = mem.transitions.full_capacity
    pos = (np.arange(50, 50 + len(buf)) % 64) + C - 1
    leaves = mem.transitions.tree.cpu().numpy()[pos]
    assert np.all(leaves[-n:] == 1.25)
    assert np.max(np.abs(leaves[:-n] - g["priorities"]) / g["priorities"]) < 1e-3
    assert mem.transitions.check_sumtree_correct() < 1e-12


def test_act_batch_vs_oracle(cuda_dev):
    """(f) batched greedy actions (many environments per launch) == the oracle's per-state argmax of the K-quantile mean."""
    from rainbow_iqn_apex_b200 import Actor
    E, seed, cfg = 48, 9900, cases.iqn_cfg(64, 64, 32)
    params = net.make_params(seed)
    actor = Actor(make_args(cuda_dev, 32, cfg), 18, None)
    load_params(actor.online_net, params)
    actor.train()
    noise = net.make_noise(seed + 1)
    actor.online_net.reset_noise(noise)
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    tau = rs.uniform(0, 1, (32 * E, 1)).astype(np.float32)
    actor._inject_act_tau = torch.from_numpy(tau)
    a = actor.act_batch(torch.from_numpy(states).to(cuda_dev)).cpu().numpy()
    actor._inject_act_tau = torch.from_numpy(tau)
    qm = actor.act_batch_values(torch.from_numpy(states).to(cuda_dev)).cpu().numpy()
    p_on = net.apply_noise(net.to_torch(params), noise)
    with torch.no_grad():
        q = net.dqn_forward_iqn(p_on, torch.from_numpy(states).float().div_(255), 32, torch.from_numpy(tau))
    qo = q.reshape(32, E, 18).mean(0).numpy()
    assert rel_err(qm, qo) < 1e-3
    ao = qo.argmax(1)
    for e in np.where(a != ao)[0]:                                      # only numerical ties may differ
        assert abs(qo[e, ao[e]] - qo[e, a[e]]) < 1e-4
    assert (a != ao).sum() <= 1
    # eval mode uses the mean weights (model.py:48-53); a single state through act() agrees with the batch
    actor._inject_act_tau = torch.from_numpy(tau[:32 * 1].copy())
    one = actor.act_batch(torch.from_numpy(states[:1]).to(cuda_dev))
    assert one.shape == (1,)
