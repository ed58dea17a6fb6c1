"""The whole BBF agent at once (Schwarzer et al., ICML 2023): SPR (K = 5), random shifts, periodic resets, the EMA target,
AdamW and the update-horizon / discount annealing, all on together, for the IQN, QR-DQN and C51 heads.

Each feature has its own tests; these check where they meet.  A learner with every field on is, bit for bit, a twin
without AdamW and resets that applies the decay (oracle/bbf.py) and the resets by hand, over a run that reaches the
schedule's end, is reset mid-run and passes a second reset; at every reset the arenas are oracle/reset.py's statement on
Philox words, every optimiser restarts, the target is left alone, SPR's EMA projection is the new online projection and
the schedule restarts.  One step at a mid-schedule position is checked against a float64 statement built from the step's
device weights: the n-step returns and discounts of oracle/replay.py, the head loss with gamma^n = 1 and the discounts
in the nonterminals' place, SPR's loss on the EMA target trunk and projection, the gradients of both trained arenas and
the AdamW step.  Captured graphs (with a reset deferred out of the warm-up), checkpoints (at a reset boundary and mid
schedule) and a data-parallel replica are checked against eager twins, bit for bit."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_bits, check_bound, f32_bits, philox_np
from oracle import bbf, cases, losses, network as net, qr as oq, replay as orep, reset as ors, spr as osp
from test_gpu_reset import _args, _assert_same, _setup, _state
from test_horizon_config import horizon_schedule

F32 = lambda x: ctypes.c_float(x).value
N0, G0, N1, G1 = 10, 0.97, 3, 0.997
HEADS = {"iqn": {}, "qr": dict(qr_dqn=1), "c51": dict(rainbow_only=1)}
# random_shift = 4 comes with test_gpu_reset._setup; reset_interval and horizon_anneal_steps are set per test
BBF = dict(spr=1, reset=1, target_ema=1, target_ema_tau=0.25, adamw=1, adamw_weight_decay=0.5, horizon_anneal=1,
           horizon_anneal_n=N0, horizon_anneal_gamma=G0, multi_step=N1, discount=G1)
BBF_DEFAULTS = dict(spr=1, reset=1, target_ema=1, adamw=1, horizon_anneal=1, multi_step=N1, discount=G1)


def _bbf(head, P, R, defaults=False, **more):
    return dict(BBF_DEFAULTS if defaults else BBF, **HEADS[head], horizon_anneal_steps=P, reset_interval=R, **more)


def _full_state(lr, mem):
    """test_gpu_reset._state (every arena and moment arena, each optimiser's step, the target, the epsilons, updates,
    resets and the tree) with SPR's EMA projection and the replay's max priority."""
    return _state(lr, mem) + [lr.spr_ema_projection.clone(), mem.transitions.max_priority.clone()]


def _words(seed, stream, n):
    return philox_np(seed, stream, (n + 3) // 4)[:n]


def _check_reset(a, before, target_before, index):
    """``a`` right after reset number ``index``, against the statement on the pre-reset arenas ``before``."""
    from rainbow_iqn_apex_b200 import reset as rs_mod
    seed = a.online_net._rng_seed ^ rs_mod.RESET_SEED
    tables = rs_mod.tables(a)
    assert [k for k, *_ in tables] == [0, 3]
    for k, net_, opt, segs in tables:
        want = ors.arena_reset(before[k], segs, _words(seed, index * len(rs_mod.ARENAS) + k, net_._flat.numel()))
        assert_bits(f"reset {index} arena {k}", f32_bits(net_._flat.cpu().numpy()), f32_bits(want))
        assert opt._step == 0 and not opt._exp_avg.any() and not opt._exp_avg_sq.any()
    assert torch.equal(a.target_net._flat, target_before)
    assert torch.equal(a.spr_ema_projection, a.spr_net._flat[:a.spr_net.proj_numel])
    assert a.horizon() == (N0, G0)


# ------------------------------------------------------------------------------------------------ the trajectory
def _twin_step(b, mem, decays):
    """One step of the twin without AdamW and resets: its own sample and gradient, every trained arena replaced by
    fl32(theta * d) at its optimiser's (lr, weight decay) in ``decays``, the Adam steps (and the SPR projection's and
    the target's EMA), then the priorities."""
    b._horizon.write(*b.horizon())
    idxs, loss = b._step_pre(mem)
    for net_, (lr_, wd) in zip(b._trained_nets(), decays):
        net_._flat.copy_(torch.from_numpy(bbf.decayed_f32(net_._flat.cpu().numpy(), lr_, wd)))
    b._step_optimisers()
    b._count_updates(1)
    mem.update_priorities(idxs, loss)
    return idxs, loss


@pytest.mark.gpu
@pytest.mark.parametrize("head,B,defaults", [("iqn", 32, False), ("qr", 32, False), ("c51", 32, False),
                                              ("iqn", 512, False), ("iqn", 32, True)],
                         ids=["iqn-32", "qr-32", "c51-32", "iqn-512", "iqn-32-bbf-defaults"])
def test_trajectory_is_the_statement(cuda_dev, head, B, defaults):
    """13 steps at P = 4, R = 6: the schedule's end at u = 4, resets after updates 6 and 12."""
    P, R = 4, 6
    fields = _bbf(head, P, R, defaults)
    a, mem_a = _setup(cuda_dev, fields, seed=17, B=B)
    b, mem_b = _setup(cuda_dev, dict(fields, adamw=0), seed=17, B=B, reset=0)
    assert a.adamw is not None and b.adamw is None and b.reset is None and a.spr[0] == 5
    decays = [(o.param_groups[0]["lr"], o.param_groups[0]["weight_decay"]) for o in a._optimisers()]
    assert len(decays) == 2 and all(wd == F32(a.adamw) for _, wd in decays)        # SPR's arena is decayed too
    u, seen = 0, []
    for step in range(1, 14):
        ia, la = a.learn_and_update(mem_a)
        ib, lb = _twin_step(b, mem_b, decays)
        torch.cuda.synchronize()
        assert a._horizon.value == b._horizon.value == horizon_schedule(N0, G0, P, N1, G1, u), step
        seen.append(a._horizon.value)
        assert torch.equal(ia, ib) and torch.equal(la.view(torch.int32), lb.view(torch.int32)), step
        assert bool(torch.isfinite(la).all())
        u += 1
        if step % R == 0:
            before = {0: b.online_net._flat.cpu().numpy(), 3: b.spr_net._flat.cpu().numpy()}
            target_before = b.target_net._flat.clone()
            b.reset_networks()
            torch.cuda.synchronize()
            _check_reset(a, before, target_before, step // R - 1)
            u = 0
        _assert_same(_full_state(a, mem_a), _full_state(b, mem_b), (head, step))
    assert a.updates == 13 and a.resets == 2
    assert seen[0] == seen[6] == seen[12] == (N0, G0) and seen[4] == seen[5] == (N1, G1)
    assert N1 < seen[1][0] < N0 and G0 < seen[1][1] < G1


# ------------------------------------------------------------------------------------------------ float64 statement
def _store_twin(mem):
    """oracle/replay.py's store holding what test_gpu_reset._setup wrote into ``mem`` (the same RandomState stream)."""
    tr = mem.transitions
    ref = orep.ReplayStore(tr.actor_capacity, 2)
    rs = np.random.RandomState(1)
    for a, n in enumerate((512 + 100, 300)):
        for s0 in range(0, n, 512):
            e = min(n, s0 + 512)
            k = e - s0
            frames = rs.randint(0, 256, (k, 84, 84)).astype(np.uint8)
            actions, rewards = rs.randint(0, 18, k), rs.randint(-1, 2, k).astype(np.float32)
            dones = rs.uniform(size=k) < 0.03
            rs.uniform(0.1, 1, k)
            ref.write(a, s0 % 512, np.arange(s0, e) % 97, frames, actions, rewards, dones)
    return ref


def _d(x):
    return torch.as_tensor(x).detach().cpu().double()


def _noises(head, seed):
    if head == "iqn":
        return cases.make_noises(seed)
    if head == "c51":
        return cases.make_noises(seed, rainbow_only=True)
    return oq.make_noises(seed, 18, 64)


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def _flips(x, y):
    return int(((x.cpu() > 0) != (y > 0)).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("head,B", [("iqn", 32), ("iqn", 512), ("qr", 32), ("c51", 32)])
def test_step_vs_float64_oracle(cuda_dev, head, B):
    """P = 4, R = 3: the fifth step runs at u = 1 after the reset (n = 7), the second AdamW step of both restarted
    optimisers.  Its sample, loss, gradients and AdamW step against float64, with injected noises, quantile fractions
    and shifts."""
    from test_gpu_augment import shift_np
    from test_gpu_learn import _grad_tol, _loss_tol, _qmajor
    P, R = 4, 3
    lr, mem = _setup(cuda_dev, _bbf(head, P, R), seed=23, B=B)
    for _ in range(4):
        lr.learn_and_update(mem)
    assert lr.resets == 1 and lr.optimiser._step == lr.spr_optimiser._step == 1
    n_u, g_u = lr.horizon()
    assert (n_u, g_u) == horizon_schedule(N0, G0, P, N1, G1, 1) and N1 < n_u < N0
    K, coef = lr.spr
    # the step's device weights, moments and injected randomness
    before = [(n_._flat.cpu().numpy().copy(), o._exp_avg.cpu().numpy().copy(), o._exp_avg_sq.cpu().numpy().copy())
              for n_, o in zip(lr._trained_nets(), lr._optimisers())]
    p_on = {k: _d(v).requires_grad_(net.is_trainable(k)) for k, v in lr.online_net.state_dict().items()}
    p_tg = {k: _d(v) for k, v in lr.target_net.state_dict().items()}
    sp = {k: _d(lr.spr_net.get_parameter(k)).requires_grad_(True) for k in osp.NAMES}
    sp_ema = dict(zip(("weight_h", "bias_h", "weight_c", "bias_c"), (_d(x) for x in lr.spr_net.views(lr.spr_ema_projection))))
    rs = np.random.RandomState(B)
    s_st, s_nx = (rs.randint(-4, 5, (B, 2)).astype(np.int32) for _ in range(2))
    s_t = rs.randint(-4, 5, (K * B, 2)).astype(np.int32)
    noises = _noises(head, 31 + B)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(41 + B, B, cases.iqn_cfg(64, 64, 32))) if head == "iqn" else None
    lr._inject = dict(noises=noises, taus=taus, shifts=(s_st, s_nx), spr_shifts=s_t)
    # the step, as learn_and_update runs it, with its sample and intermediates kept
    lr._horizon.write(n_u, g_u)
    lr._reset_step_streams(mem)
    idxs, st, ac, rt, nx, disc, w = lr._sample(mem, None)
    seq = lr._sequence(mem, idxs)
    dbg = {}
    with lr._feeding_discounts():
        loss = lr.compute_gradients(st, ac, rt, nx, disc, w, debug=dbg, sequence=seq)
    grads = [n_._flat_grad.cpu().numpy().copy() for n_ in lr._trained_nets()]
    g_on = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    g_sp = {k: lr.spr_net.get_parameter(k).grad.detach().cpu().clone() for k in osp.NAMES}
    lr.apply_gradients()
    lr._count_updates(1)
    mem.update_priorities(idxs, loss)
    torch.cuda.synchronize()
    lr._inject = None
    assert lr._horizon.value == (n_u, g_u)
    # the sample: ReplayStore.assemble at (n_u, gamma_u), discounts fl32(gamma_u^n_u) nt
    data_idx = (idxs - (mem.capacity - 1)).cpu().numpy()
    s_ref, a_ref, r_ref, nx_ref, nt_ref = _store_twin(mem).assemble(data_idx, 4, n_u, g_u)
    assert np.array_equal(st.cpu().numpy(), s_ref) and np.array_equal(nx.cpu().numpy(), nx_ref)
    assert np.array_equal(ac.cpu().numpy(), a_ref)
    assert_bits("returns", f32_bits(rt.cpu().numpy()), f32_bits(r_ref))
    assert_bits("discounts", f32_bits(disc.cpu().numpy()), f32_bits(np.float32(F32(g_u ** n_u)) * nt_ref))
    win, acts, valid = (t.cpu() for t in seq)
    w_ref, acts_ref, valid_ref = osp.sequence(_store_twin(mem), data_idx, mem.transitions.index_actor.cpu().numpy(), 4, K)
    assert np.array_equal(win.numpy(), w_ref) and np.array_equal(acts.numpy(), acts_ref)
    assert np.array_equal(valid.numpy(), valid_ref)
    # the shifted frames are the statement's, exactly
    x_np, nx_np = shift_np(s_ref, s_st), shift_np(nx_ref, s_nx)
    assert np.array_equal(dbg["shifted_states"].cpu().numpy(), x_np)
    assert np.array_equal(dbg["shifted_next_states"].cpu().numpy(), nx_np)
    xt_np = np.concatenate([shift_np(w_ref[:, k + 1:k + 5], s_t[k * B:(k + 1) * B]) for k in range(K)])
    x, xn, xt = (torch.from_numpy(v).double().div_(255) for v in (x_np, nx_np, xt_np))
    # float64: the head loss at gamma^n = 1 with the discounts as nonterminals, and SPR's on the EMA target encoder
    nz = tuple({k: (_d(e_in), _d(e_out)) for k, (e_in, e_out) in nse.items()} for nse in noises)
    acts_t, r64, d64 = torch.from_numpy(a_ref), _d(r_ref), _d(np.float32(F32(g_u ** n_u)) * nt_ref)
    keep, trunk, gk = {}, {}, dbg.get("keep")
    if head == "iqn":
        o_loss = losses.iqn_loss(p_on, p_tg, x, acts_t, r64, xn, d64, nz, tuple(_d(t) for t in taus), n_tau=64,
                                 n_tau_prime=64, n_quantile=32, discount=1.0, n_step=1, kappa=1.0, keep=keep)
        q_next = keep["q_sel"].reshape(32, B, 18).mean(0)
        h = _qmajor(gk["h"], B).cpu()
        hidden = (keep["h_v"], keep["h_a"])
    elif head == "qr":
        o_loss = oq.qr_loss(p_on, p_tg, x, acts_t, r64, xn, d64, nz, n=64, discount=1.0, n_step=1, keep=keep)
        q_next, h, hidden = keep["qv_next"], gk["h"].cpu(), (keep["h_v"], keep["h_a"])
    else:
        o_loss = losses.c51_loss(p_on, p_tg, x, acts_t, r64, xn, d64, nz, discount=1.0, n_step=1, keep=keep)
        with torch.no_grad():
            p = dict(p_on)
            pns = net.dqn_forward_c51(net.apply_noise(p, nz[1]), xn, 18, 51)
            q_next = (torch.linspace(-10, 10, 51).double() * pns).sum(2)
            pre = [F.conv2d(x, p["conv1.weight"], p["conv1.bias"], stride=4, padding=1)]
            pre.append(F.conv2d(torch.relu(pre[0]), p["conv2.weight"], p["conv2.bias"], stride=2))
            pre.append(F.conv2d(torch.relu(pre[1]), p["conv3.weight"], p["conv3.bias"]))
            feat = torch.relu(pre[2]).reshape(B, -1)
            net.apply_noise(p, nz[0])
            pre += [net.noisy_linear(p, k, feat) for k in ("fcnoisy_h_v", "fcnoisy_h_a")]
    seq_acts = torch.from_numpy(acts_ref)
    rows, _, t = bbf.spr_loss_ema(p_on, p_tg, sp, sp_ema, x, seq_acts, valid_ref, xt, 18)
    ((_d(w) * o_loss).mean() + coef * rows.mean()).backward()
    # near-ties of the double-DQN argmax and ReLU kinks the device and the statement put on opposite sides of 0
    a_gpu, a_ref_ = dbg["a_star"].cpu().numpy(), keep["a_star"].numpy()
    ok = a_gpu == a_ref_
    qn = q_next.detach().numpy()
    for b_ in np.flatnonzero(~ok):
        assert abs(qn[b_, a_gpu[b_]] - qn[b_, a_ref_[b_]]) < 1e-4, "the argmax differs beyond a numerical tie"
    lg, lo = loss.cpu().numpy(), o_loss.detach().numpy()
    err = np.abs(lg - lo) / np.abs(lo)
    assert np.max(err[ok]) < _loss_tol(), float(np.max(err[ok]))
    with torch.no_grad():
        net.conv_trunk(p_on, x, trunk)
        z, zs = trunk["o3"].reshape(B, 64, 7, 7), []
        for k in range(K):
            z = osp.transition(sp, z, seq_acts[:, k], 18)
            zs.append(z)
    if gk is not None:
        fl = [_flips(gk["out"][i], trunk[f"o{i + 1}"]) for i in range(3)]
        fl += [_flips(h[:, :512], hidden[0]), _flips(h[:, 512:], hidden[1])]
    else:        # the C51 loss core keeps no activations: count the pre-activations within 1e-5 of a layer's scale
        fl = [int((q.abs() < 1e-5 * q.abs().max()).sum()) for q in pre]
    fl.append(_flips(dbg["spr_latents"], torch.stack(zs)))
    relaxed = set()
    if fl[3] + fl[4] or not ok.all():
        relaxed |= {"conv1", "conv2", "conv3", "iqn_fc", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)} | {"spr"}
    if fl[5]:
        relaxed |= {"conv1", "conv2", "conv3", "spr"}
    assert _cos(dbg["spr_targets"].cpu(), t) >= 0.9999
    gtol = _grad_tol()
    worst = 1.0
    for group, got, ref in (("online", g_on, {k: v.grad for k, v in p_on.items() if v.grad is not None}),
                            ("spr", g_sp, {k: sp[k].grad for k in osp.NAMES})):
        assert set(ref) <= set(got)
        for k, g_ref in ref.items():
            c, rel = _cos(got[k], g_ref), float((got[k].double() - g_ref).norm() / (g_ref.norm() + 1e-300))
            worst = min(worst, c)
            if (k.split(".")[0] if group == "online" else "spr") in relaxed:
                assert c > 0.98 and rel < 0.2, (group, k, c, rel, fl)
            else:
                assert c >= 0.999 and rel <= gtol, (group, k, c, rel, fl)
    print(f"{head} B={B} n={n_u}: max loss rel err {np.max(err[ok]):.3g}, min cos {worst:.6f}, flips {fl}, "
          f"ties {int((~ok).sum())}")
    # AdamW on both arenas: within test_gpu_adamw_ema's bound of the float64 step on the device's gradients
    for (th0, m0, v0), g, n_, o in zip(before, grads, lr._trained_nets(), lr._optimisers()):
        grp = o.param_groups[0]
        want, _, _ = bbf.adamw_step_np(th0, g, m0, v0, o._step, grp["lr"], grp["weight_decay"], *grp["betas"], grp["eps"])
        assert o._step == 2 and grp["weight_decay"] > 0
        bound = (8 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-5 * np.abs(want - th0)
                 + 1e-6 * grp["lr"])
        check_bound(f"AdamW {type(n_).__name__}", n_._flat.cpu().numpy(), want, bound)


# ------------------------------------------------------------------------------------------------ graphs
def _eager_twin(b, mem, plan):
    """Eager steps of ``b`` through the device step state, as a capture's warm-up and replays run them (plan:
    "step" / "capture" / "reset"), each step's horizon from the updates counted so far; per step (loss, idxs,
    horizon, state)."""
    from rainbow_iqn_apex_b200.dynstate import DynState
    b._dyn = DynState(b.online_net._flat.device, slots=len(b._optimisers()))
    out = []
    with b._attached(mem):
        for what in plan:
            if what == "capture":
                b._dyn.epoch += 1
            elif what == "reset":
                b.reset_networks()
                out[-1] = out[-1][:3] + (_full_state(b, mem),)
            else:
                b._write_dyn(mem)
                idx, loss = b._step_pre(mem)
                b._step_post(mem, idx, loss)
                b.updates += 1
                out.append((loss.clone(), idx.clone(), b._horizon.value, _full_state(b, mem)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("head", ["iqn", "c51"])
def test_graph_replays_equal_eager_steps(cuda_dev, head):
    """warm-up 3, R = 2, P = 1: the reset due after update 2 is deferred to the capture's end (after update 3), so warm-up
    step 3 still runs at schedule position 2 (the schedule's end); the replays then reset after every even update, at
    positions 0, 0, 1, 0, 1, ... ((n0, gamma0) and the end)."""
    P, R, W, steps = 1, 2, 3, 8
    fields = _bbf(head, P, R)
    a, mem_a = _setup(cuda_dev, fields, seed=19, B=32)
    b, mem_b = _setup(cuda_dev, fields, seed=19, B=32)
    a.enable_cuda_graph(mem_a, warmup=W)
    assert a.updates == W and a.resets == 1 and a.horizon() == (N0, G0)
    plan = []
    for u in range(1, W + steps + 1):
        plan.append("step")
        if u == W:
            plan += ["capture", "reset"]
        elif u > W and u % R == 0:
            plan.append("reset")
    want = _eager_twin(b, mem_b, plan)
    assert [h for _, _, h, _ in want[:W]] == [horizon_schedule(N0, G0, P, N1, G1, u) for u in range(W)]
    torch.cuda.synchronize()
    _assert_same(_full_state(a, mem_a), want[W - 1][3], "after the capture")
    seen = []
    for k, (lb, ib, hb, sb) in enumerate(want[W:]):
        u = a.updates - a._horizon_base
        ia, la = a.learn_and_update(mem_a)
        torch.cuda.synchronize()
        assert a._horizon.value == hb == horizon_schedule(N0, G0, P, N1, G1, u), k
        assert torch.equal(la.view(torch.int32), lb.view(torch.int32)) and torch.equal(ia, ib), k
        assert bool(torch.isfinite(la).all())
        _assert_same(_full_state(a, mem_a), sb, k)
        seen.append(hb)
    assert a.updates == W + steps and a.resets == 1 + steps // R
    assert seen == [horizon_schedule(N0, G0, P, N1, G1, u) for u in (0, 0, 1, 0, 1, 0, 1, 0)]


# ------------------------------------------------------------------------------------------------ checkpoints
def _resume(dev, src, fields, path):
    """A learner built from the checkpoint ``path`` of ``src``, given what a checkpoint does not carry: the epsilon
    arenas, the noise seeds and the Philox call counters."""
    from rainbow_iqn_apex_b200 import Learner
    torch.manual_seed(321)
    back = Learner(_args(dev, 32, fields, model=path), 18, None)
    back.train()
    back.target_net._eps_flat.copy_(src.target_net._eps_flat)
    back.online_net._eps_flat.copy_(src.online_net._eps_flat)
    for x, y in ((back.online_net, src.online_net), (back.target_net, src.target_net)):
        x._rng_seed, x._tau_calls, x._shift_calls = y._rng_seed, y._tau_calls, y._shift_calls
        for (_, m), (_, n_) in zip(x.noisy_layers(), y.noisy_layers()):
            m._noise_calls = n_._noise_calls
        x.compose_weights()
    return back


@pytest.mark.gpu
def test_checkpoint_resume(cuda_dev, tmp_path):
    """R = 4, P = 3.  Saved at the first reset (update 4) and resumed, the run equals the uninterrupted one bit for bit
    for the next R steps, across the second reset.  Saved mid-schedule (update 9), it resumes at (n0, gamma0) with
    every arena, moment, step count, the target, the EMA projection, updates and resets as saved."""
    P, R = 3, 4
    fields = _bbf("iqn", P, R)
    run, mem_run = _setup(cuda_dev, fields, seed=29, B=32)
    src, mem_src = _setup(cuda_dev, fields, seed=29, B=32)
    for _ in range(R):
        run.learn_and_update(mem_run)
        src.learn_and_update(mem_src)
    assert (src.updates, src.resets) == (R, 1) and src.optimiser._step == 0
    src.save(str(tmp_path), 0, R, "bbf.pth")
    path = os.path.join(tmp_path, "bbf.pth")
    ck = torch.load(path, map_location="cpu")
    assert tuple(ck["reset_state"]) == (R, 1) and "target_state_dict" in ck and "spr_ema_projection" in ck
    back = _resume(cuda_dev, src, fields, path)
    torch.cuda.synchronize()
    assert (back.updates, back.resets) == (R, 1) and back.horizon() == run.horizon() == (N0, G0)
    _assert_same(_full_state(back, mem_src), _full_state(run, mem_run), "restored at a reset")
    for step in range(R + 1, 2 * R + 1):
        ia, la = run.learn_and_update(mem_run)
        ib, lb = back.learn_and_update(mem_src)
        torch.cuda.synchronize()
        assert run._horizon.value == back._horizon.value, step
        assert torch.equal(ia, ib) and torch.equal(la.view(torch.int32), lb.view(torch.int32)), step
        _assert_same(_full_state(back, mem_src), _full_state(run, mem_run), step)
    assert run.resets == back.resets == 2 and run.horizon() == (N0, G0)
    # mid schedule: the resumed learner starts the schedule again, everything else as saved
    run.learn_and_update(mem_run)
    assert run.horizon() != (N0, G0) and run.optimiser._step == 1
    run.save(str(tmp_path), 0, 2 * R + 1, "mid.pth")
    mid = _resume(cuda_dev, run, fields, os.path.join(tmp_path, "mid.pth"))
    torch.cuda.synchronize()
    assert mid.horizon() == (N0, G0) and (mid.updates, mid.resets) == (run.updates, run.resets)
    _assert_same(_full_state(mid, mem_run), _full_state(run, mem_run), "restored mid schedule")
    mid.learn_and_update(mem_run)
    assert mid._horizon.value == (N0, G0)


# ------------------------------------------------------------------------------------------------ data parallel
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_replica(cuda_dev):
    """A gloo world of one: with process_group set (the all-reduce of every gradient arena), the BBF learner equals the
    plain one bit for bit over 7 steps at R = 3, P = 2 (the schedule's end at u = 2, resets after 3 and 6)."""
    import torch.distributed as dist
    P, R = 2, 3
    fields = _bbf("iqn", P, R)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        runs = []
        for dp in (False, True):
            lr, mem = _setup(cuda_dev, fields, seed=37, B=32)
            if dp:
                lr.process_group = dist.group.WORLD
            out = []
            for _ in range(7):
                idx, loss = lr.learn_and_update(mem)
                torch.cuda.synchronize()
                out.append((idx.clone(), loss.clone(), lr._horizon.value, _full_state(lr, mem)))
            runs.append(out)
            assert lr.resets == 2
        for k, ((i0, l0, h0, s0), (i1, l1, h1, s1)) in enumerate(zip(*runs)):
            assert h0 == h1 and torch.equal(i0, i1) and torch.equal(l0.view(torch.int32), l1.view(torch.int32)), k
            _assert_same(s0, s1, k)
        assert [h for _, _, h, _ in runs[0]] == [horizon_schedule(N0, G0, P, N1, G1, u) for u in (0, 1, 2, 0, 1, 2, 0)]
    finally:
        dist.destroy_process_group()
