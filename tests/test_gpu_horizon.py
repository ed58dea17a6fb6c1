"""Update-horizon and discount annealing (BBF) on the device: riqn_frame_gather_horizon and riqn_sumtree_sample_horizon
(csrc/sumtree.cu) against their fixed-n siblings and oracle/replay.py, bit for bit, with their refusals; and the
annealing learner (horizon.py, Learner under horizon_anneal), whose step u is, bit for bit, a fixed learner's step at
(multi_step, discount) = (n_u, gamma_u) for every head and loss variant, eagerly and replayed from one captured graph
across the whole schedule, restarted at a reset, and refused by the entry points that take batches assembled at a fixed
n."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, assert_canaries, dptr, f32_bits, lib_call, make_args
from oracle import cases, replay as orep

FRAME = 84 * 84
I64_FILL = -7
F32 = lambda x: ctypes.c_float(x).value


def _err():
    from rainbow_iqn_apex_b200._lib import RiqnError
    return RiqnError


def _hz(dev, n_max, n, gamma):
    from rainbow_iqn_apex_b200.dynstate import HorizonState
    hz = HorizonState(dev, n_max)
    hz.write(n, gamma)
    return hz


# ------------------------------------------------------------------------------------------------ the gather
def _store(dev, ac=64, nb=3, seed=0):
    """A device frame store and its oracle twin: three segments, one written past its end (the ring wraps), one
    partly; episodes of random lengths (timestep 0 at each start, terminals inside every window length)."""
    from rainbow_iqn_apex_b200.replay_memory import SegmentTree
    rs = np.random.RandomState(seed)
    tr = SegmentTree(ac, nb, dev)
    ref = orep.ReplayStore(ac, nb)
    # segment 0 is written past its end (positions 50..63 then 0..15), segment 1 up to its middle
    for a, s0, k in ((0, 0, ac), (0, 50, 30), (1, 0, ac // 2), (2, 0, ac)):
        dones = rs.uniform(size=k) < 0.12
        ts = np.zeros(k, np.int64)
        for i in range(1, k):
            ts[i] = 0 if dones[i - 1] else ts[i - 1] + 1
        ts[0] = rs.randint(0, 3)
        frames = rs.randint(0, 256, (k, 84, 84)).astype(np.uint8)
        actions = rs.randint(0, 18, k)
        rewards = rs.uniform(-2, 2, k).astype(np.float32)
        tr.append_arrays(a, s0, ts, frames, actions, rewards, dones, np.ones(k, np.float32))
        ref.write(a, s0, ts, frames, actions, rewards, dones)
    return tr, ref


def _gather(dev, tr, di, history, n, gamma):
    B = di.numel()
    gp = torch.tensor([gamma ** k for k in range(n)], dtype=torch.float64, device=dev)
    win = torch.full((B, history + n, 84, 84), 0xAB, dtype=torch.uint8, device=dev)
    act, ret, nt = Out(B, dev, torch.int64, I64_FILL), Out(B, dev), Out(B, dev)
    lib_call("riqn_frame_gather", B, tr.actor_capacity, history, n, dptr(di), dptr(tr.frames), dptr(tr.timestep),
             dptr(tr.action), dptr(tr.reward), dptr(tr.nonterminal), dptr(gp), dptr(win), act.p, ret.p, nt.p)
    return win, act, ret, nt


def _gather_horizon(dev, tr, di, history, n_max, hz):
    B = di.numel()
    fr = torch.full((B, 2 * history, 84, 84), 0xAB, dtype=torch.uint8, device=dev)
    act, ret, nt, disc = Out(B, dev, torch.int64, I64_FILL), Out(B, dev), Out(B, dev), Out(B, dev)
    lib_call("riqn_frame_gather_horizon", B, tr.actor_capacity, history, n_max, dptr(di), dptr(tr.frames),
             dptr(tr.timestep), dptr(tr.action), dptr(tr.reward), dptr(tr.nonterminal), hz.ptr(), dptr(fr), act.p, ret.p,
             nt.p, disc.p)
    return fr, act, ret, nt, disc


@pytest.mark.gpu
@pytest.mark.parametrize("gamma", [0.97, 0.5])
def test_gather_horizon_is_frame_gather_at_n(cuda_dev, gamma):
    """Every sample of a wrapped, partly filled three-segment store, every n in 1..12 at history 4, with n_max = n and
    n_max = 12: frames, actions, returns and nonterminals are riqn_frame_gather's at n, the next states its window[:,
    n:n+4], all equal to oracle/replay.py, and discounts = fl32(gamma^n) * nt.  One horizon state is rewritten between
    the calls: the kernel reads n on the device."""
    history = 4
    tr, ref = _store(cuda_dev)
    C = tr.full_capacity
    di = torch.arange(C, dtype=torch.int64, device=cuda_dev)
    from rainbow_iqn_apex_b200.dynstate import HorizonState
    hz12 = HorizonState(cuda_dev, 12)
    for n in range(1, 13):
        win, act, ret, nt = _gather(cuda_dev, tr, di, history, n, gamma)
        s_ref, a_ref, r_ref, nx_ref, nt_ref = ref.assemble(np.arange(C), history, n, gamma)
        hz12.write(n, gamma)
        for hz, n_max in ((_hz(cuda_dev, n, n, gamma), n), (hz12, 12)):
            outs = []
            for _ in range(2):                                           # every call: the same bits
                fr, act_h, ret_h, nt_h, disc = _gather_horizon(cuda_dev, tr, di, history, n_max, hz)
                torch.cuda.synchronize()
                assert_canaries({"actions": act_h, "returns": ret_h, "nonterminals": nt_h, "discounts": disc})
                outs.append((fr.cpu().numpy(), act_h.t[:C].cpu().numpy(), ret_h.bits(), nt_h.bits(), disc.bits()))
            for x, y in zip(outs[0], outs[1]):
                assert np.array_equal(x, y)
            fr, a_h, r_h, nt_bits, d_bits = outs[0]
            w = win.cpu().numpy()
            assert np.array_equal(fr[:, :history], w[:, :history]), n
            assert np.array_equal(fr[:, history:], w[:, n:n + history]), n
            assert np.array_equal(fr[:, :history], s_ref) and np.array_equal(fr[:, history:], nx_ref), n
            assert np.array_equal(a_h, act.t[:C].cpu().numpy()) and np.array_equal(a_h, a_ref)
            assert_bits(f"returns n={n}", r_h, ret.bits())
            assert_bits(f"returns vs oracle n={n}", r_h, f32_bits(r_ref))
            assert_bits(f"nonterminals n={n}", nt_bits, nt.bits())
            assert_bits(f"nonterminals vs oracle n={n}", nt_bits, f32_bits(nt_ref))
            g = np.float32(F32(gamma ** n))
            assert_bits(f"discounts n={n}", d_bits, f32_bits(g * nt_ref))
        assert 0 < nt_ref.sum() < C and (r_ref != 0).any()                   # terminals and rewards in the windows


@pytest.mark.gpu
def test_gather_horizon_refusals(cuda_dev):
    tr, _ = _store(cuda_dev)
    di = torch.arange(8, dtype=torch.int64, device=cuda_dev)
    hz = _hz(cuda_dev, 12, 3, 0.9)
    fr = torch.full((8, 8, 84, 84), 0xAB, dtype=torch.uint8, device=cuda_dev)
    outs = [Out(8, cuda_dev, torch.int64, I64_FILL), Out(8, cuda_dev), Out(8, cuda_dev), Out(8, cuda_dev)]
    ok = [8, tr.actor_capacity, 4, 12, dptr(di), dptr(tr.frames), dptr(tr.timestep), dptr(tr.action), dptr(tr.reward),
          dptr(tr.nonterminal), hz.ptr(), dptr(fr)] + [o.p for o in outs]
    bad = [(1, 0), (2, 0), (3, 0), (3, 13), (2, 13)] + [(k, None) for k in range(4, 16)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_frame_gather_horizon", *args)
    torch.cuda.synchronize()
    assert bool((fr == 0xAB).all()) and bool((outs[0].t[:8] == I64_FILL).all())
    assert all(bool(torch.isnan(o.t[:8]).all()) for o in outs[1:]) and all(o.canaries_ok() for o in outs)
    lib_call("riqn_frame_gather_horizon", *ok)
    torch.cuda.synchronize()
    assert not bool(torch.isnan(outs[3].t[:8]).any())


@pytest.mark.gpu
def test_horizon_state_writer_refuses_out_of_range(cuda_dev):
    from rainbow_iqn_apex_b200.dynstate import HorizonState
    hz = HorizonState(cuda_dev, 10)
    for n in (0, 11, -1, 3.0, True):
        with pytest.raises(ValueError):
            hz.write(n, 0.9)
    for n_max in (0, 17):
        with pytest.raises(ValueError):
            HorizonState(cuda_dev, n_max)
    hz.write(10, 0.9)
    torch.cuda.synchronize()
    raw = hz.dev.cpu().numpy().tobytes()
    import struct
    from rainbow_iqn_apex_b200.dynstate import HORIZON_FMT
    got = struct.unpack(HORIZON_FMT, raw)
    assert got[0] == 10 and got[1] == F32(0.9 ** 10) and list(got[2:12]) == [0.9 ** k for k in range(10)]


# ------------------------------------------------------------------------------------------------ the sampler
@pytest.mark.gpu
@pytest.mark.parametrize("ac, nb", [(40, 3), (64, 1), (33, 2)])
def test_sample_horizon_is_sumtree_sample_at_n(cuda_dev, ac, nb):
    """tree_idx, data_idx and priorities bit for bit against riqn_sumtree_sample at every n in 1..12 (n_max 12 and n),
    with 4096 values that reach every leaf, write heads at 0, at the end and in mid-segment, so that samples next to a
    write head on both sides are shifted."""
    C = ac * nb
    rs = np.random.RandomState(C)
    leaves = rs.randint(1, 5, C).astype(np.float64)
    from test_gpu_replay_kernels import build_tree
    tree = torch.from_numpy(build_tree(leaves)).to(cuda_dev)
    total = float(tree[0])
    vals = torch.from_numpy(np.concatenate([np.linspace(0, total, 3000), rs.uniform(0, total, 1096)])).to(cuda_dev)
    q = vals.numel()
    moved = 0
    for heads in (np.zeros(nb, np.int64), np.full(nb, ac - 1), rs.randint(0, ac, nb)):
        heads_d = torch.tensor(heads, dtype=torch.int64, device=cuda_dev)
        data = {}
        for n in range(1, 13):
            want = [Out(q, cuda_dev, torch.int64, I64_FILL), Out(q, cuda_dev, torch.int64, I64_FILL),
                    Out(q, cuda_dev, torch.float64)]
            lib_call("riqn_sumtree_sample", q, C, ac, dptr(tree), dptr(vals), dptr(heads_d), 4, n, *[o.p for o in want])
            for n_max in (n, 12):
                hz = _hz(cuda_dev, n_max, n, 0.97)
                got = [Out(q, cuda_dev, torch.int64, I64_FILL), Out(q, cuda_dev, torch.int64, I64_FILL),
                       Out(q, cuda_dev, torch.float64)]
                lib_call("riqn_sumtree_sample_horizon", q, C, ac, dptr(tree), dptr(vals), dptr(heads_d), 4, n_max,
                         hz.ptr(), *[o.p for o in got])
                torch.cuda.synchronize()
                assert_canaries(dict(zip(("ti", "di", "pr"), got)))
                for g, w in zip(got, want):
                    assert torch.equal(g.t[:q], w.t[:q]), (n, n_max, heads)
            data[n] = want[1].t[:q].clone()
        moved += int((data[1] != data[12]).sum())         # rows next to a write head: their shift depends on n
    assert moved > 0


@pytest.mark.gpu
def test_sample_horizon_refusals(cuda_dev):
    from test_gpu_replay_kernels import build_tree
    tree = torch.from_numpy(build_tree(np.arange(1.0, 13.0))).to(cuda_dev)
    vals = torch.tensor([1.0, 5.0, 70.0], dtype=torch.float64, device=cuda_dev)
    heads = torch.zeros(3, dtype=torch.int64, device=cuda_dev)
    hz = _hz(cuda_dev, 3, 3, 0.9)
    ti, di = Out(3, cuda_dev, torch.int64, I64_FILL), Out(3, cuda_dev, torch.int64, I64_FILL)
    pr = Out(3, cuda_dev, torch.float64)
    ok = [3, 12, 4, dptr(tree), dptr(vals), dptr(heads), 4, 3, hz.ptr(), ti.p, di.p, pr.p]
    bad = [(1, 0), (2, 0), (2, 5), (6, -1), (7, 0), (7, 17)] + [(k, None) for k in (3, 4, 5, 8, 9, 10, 11)]
    for k, v in bad:
        args = list(ok)
        args[k] = v
        with pytest.raises(_err()):
            lib_call("riqn_sumtree_sample_horizon", *args)
    torch.cuda.synchronize()
    assert bool((ti.t[:3] == I64_FILL).all() and (di.t[:3] == I64_FILL).all() and torch.isnan(pr.t[:3]).all())
    assert_canaries({"ti": ti, "di": di, "pr": pr})
    lib_call("riqn_sumtree_sample_horizon", *ok)
    torch.cuda.synchronize()
    assert bool((ti.t[:3] >= 11).all())


# ------------------------------------------------------------------------------------------------ learners
ANNEAL = dict(horizon_anneal=1, horizon_anneal_n=10, horizon_anneal_gamma=0.97, horizon_anneal_steps=8, multi_step=3,
              discount=0.997)


def _setup(dev, fields, seed=0, B=32):
    """A seeded learner with ``fields`` and a replay of 612 + 300 transitions in two segments (the first wraps)."""
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    torch.manual_seed(seed)
    args = make_args(dev, B, cases.iqn_cfg(64, 64, 32), rainbow_only=bool(fields.get("rainbow_only")), nb_actor=2,
                     actor_capacity=512)
    for k, v in fields.items():
        setattr(args, k, v)
    lr = Learner(args, 18, None)
    lr.train()
    mem = ReplayMemory(args, None)
    rs = np.random.RandomState(1)
    for a, n in enumerate((512 + 100, 300)):
        for s0 in range(0, n, 512):
            e = min(n, s0 + 512)
            k = e - s0
            mem.transitions.append_arrays(a, s0 % 512, np.arange(s0, e) % 97,
                                          rs.randint(0, 256, (k, 84, 84)).astype(np.uint8), rs.randint(0, 18, k),
                                          rs.randint(-1, 2, k).astype(np.float32), rs.uniform(size=k) < 0.03,
                                          (rs.uniform(0.1, 1, k) ** 0.2).astype(np.float32))
    for obj, sd in ((lr.online_net, 11), (lr.target_net, 12), (mem.transitions, 13)):
        obj._rng_seed = sd
    return lr, mem


def _state(lr, mem):
    out = []
    for net, opt in zip(lr._trained_nets(), lr._optimisers()):
        out += [net._flat, opt._exp_avg, opt._exp_avg_sq]
    out += [lr.target_net._flat, lr.online_net._eps_flat, mem.transitions.tree, mem.transitions.max_priority]
    return [t.clone() for t in out]


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y), (what, k)


def _annealed_vs_fixed(dev, fields, u, B=32, seed=3):
    """One eager learn_and_update of an annealing learner at schedule position u (its updates count set to u; resets
    off) and of a fixed learner built at (multi_step, discount) = (n_u, gamma_u): losses, indices, every arena and
    moment, the target, the tree and max priority, bit for bit."""
    a, mem_a = _setup(dev, dict(ANNEAL, **fields), seed, B)
    a.updates = u
    n_u, g_u = a.horizon()
    f, mem_f = _setup(dev, dict(fields, multi_step=n_u, discount=g_u), seed, B)
    assert f.horizon_anneal is None
    ia, la = a.learn_and_update(mem_a)
    i_f, lf = f.learn_and_update(mem_f)
    torch.cuda.synchronize()
    assert a._horizon.value == (n_u, g_u)
    assert torch.equal(ia, i_f) and torch.equal(la.view(torch.int32), lf.view(torch.int32)), (fields, u)
    assert bool(torch.isfinite(la).all())
    _assert_same(_state(a, mem_a), _state(f, mem_f), (fields, u))
    return n_u, g_u


@pytest.mark.gpu
@pytest.mark.parametrize("head", [dict(), dict(qr_dqn=1), dict(rainbow_only=1)], ids=["iqn", "qr", "c51"])
def test_step_u_is_a_fixed_horizon_step(cuda_dev, head):
    seen = [_annealed_vs_fixed(cuda_dev, head, u) for u in (0, 4, 9)]
    assert seen[0] == (10, 0.97) and seen[2] == (3, 0.997) and 3 < seen[1][0] < 10 and 0.97 < seen[1][1] < 0.997


VARIANTS = [dict(munchausen=1), dict(fqf=1), dict(cql=1), dict(qr_dqn=1, cql=1), dict(dqfd=1, demo_segments=1),
            dict(qr_dqn=1, mmd=1), dict(rainbow_only=1, hl_gauss=1), dict(value_rescaling=1),
            dict(rainbow_only=1, value_rescaling=1), dict(random_shift=4), dict(curl=1, random_shift=4), dict(spr=1),
            dict(target_ema=1, adamw=1)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in v))
def test_variants_at_a_mid_schedule_step(cuda_dev, variant):
    _annealed_vs_fixed(cuda_dev, variant, 3)


def _attached_steps(b, mem, n_warm, n_steps):
    """Eager steps of ``b`` through the device step state, as a capture's warm-up and replays run them, counting
    updates after each (the schedule advances as the replays'), with the horizon each step read."""
    from rainbow_iqn_apex_b200.dynstate import DynState
    b._dyn = DynState(b.online_net._flat.device, slots=len(b._optimisers()))
    out = []
    with b._attached(mem):
        for k in range(n_warm + n_steps):
            if k == n_warm:
                b._dyn.epoch += 1
            b._write_dyn(mem)
            idx, loss = b._step_pre(mem)
            b._step_post(mem, idx, loss)
            b._count_updates(1)
            out.append((loss.clone(), idx.clone(), b._horizon.value, _state(b, mem)))
    return out[n_warm:]


@pytest.mark.gpu
@pytest.mark.parametrize("head", [dict(), dict(rainbow_only=1)], ids=["iqn", "c51"])
def test_one_graph_follows_the_schedule(cuda_dev, head):
    """One capture (P = 8, n0 = 10, multi_step = 3), replayed across the whole schedule and past it: every replay equals
    the eager annealing learner's step through the same device state, bit for bit, at the schedule's (n, gamma)."""
    from test_horizon_config import horizon_schedule
    a, mem_a = _setup(cuda_dev, dict(ANNEAL, **head), 5, 32)
    b, mem_b = _setup(cuda_dev, dict(ANNEAL, **head), 5, 32)
    a.enable_cuda_graph(mem_a, warmup=3)
    assert a.updates == 3
    want = _attached_steps(b, mem_b, 3, 9)
    seen = []
    for k, (lb, ib, hb, sb) in enumerate(want):
        u = a.updates
        ia, la = a.learn_and_update(mem_a)
        torch.cuda.synchronize()
        assert a._horizon.value == hb == horizon_schedule(10, 0.97, 8, 3, 0.997, u)
        assert torch.equal(la.view(torch.int32), lb.view(torch.int32)) and torch.equal(ia, ib), k
        _assert_same(_state(a, mem_a), sb, k)
        seen.append(hb[0])
    assert seen[0] > 3 and seen[-1] == 3 and len(set(seen)) > 2


@pytest.mark.gpu
def test_reset_restarts_the_schedule(cuda_dev):
    """reset = 1, reset_interval = 3: the step after each reset (eager, then replayed from a graph) runs at (n0, gamma0),
    and reset_networks() called by hand restarts it too."""
    lr, mem = _setup(cuda_dev, dict(ANNEAL, reset=1, reset_interval=3), 6, 32)
    hs = []
    for _ in range(4):
        lr.learn_and_update(mem)
        hs.append(lr._horizon.value)
    assert lr.resets == 1 and hs[0] == hs[3] == (10, 0.97) and hs[1][0] < 10 and hs[2][0] < hs[1][0] + 1
    lr.enable_cuda_graph(mem, warmup=2)          # updates 6: the deferred reset restarts the schedule
    assert lr.resets == 2 and lr.horizon() == (10, 0.97)
    hs = []
    for _ in range(4):
        lr.learn_and_update(mem)
        hs.append(lr._horizon.value)
    assert lr.resets == 3 and hs[0] == hs[3] == (10, 0.97) and hs[1] != (10, 0.97)
    lr.learn_and_update(mem)
    lr.reset_networks()
    assert lr.horizon() == (10, 0.97)
    lr.learn_and_update(mem)
    assert lr._horizon.value == (10, 0.97)


@pytest.mark.gpu
def test_learn_on_batch_trains_at_the_horizon(cuda_dev):
    """A batch the caller assembles at horizon() trains as the fixed learner's learn_on_batch at (n_u, gamma_u)."""
    a, mem_a = _setup(cuda_dev, ANNEAL, 8, 32)
    a.updates = 5
    n_u, g_u = a.horizon()
    f, mem_f = _setup(cuda_dev, dict(multi_step=n_u, discount=g_u), 8, 32)
    batch = mem_f.sample(32)
    la = a.learn_on_batch(*batch[1:])
    lf = f.learn_on_batch(*batch[1:])
    torch.cuda.synchronize()
    assert torch.equal(la.view(torch.int32), lf.view(torch.int32))
    assert torch.equal(a.online_net._flat, f.online_net._flat)


@pytest.mark.gpu
def test_fixed_n_entry_points_refuse(cuda_dev):
    from rainbow_iqn_apex_b200 import apex
    lr, mem = _setup(cuda_dev, ANNEAL, 9, 32)
    example = mem.sample(32)
    with pytest.raises(ValueError, match="horizon_anneal"):
        lr.enable_learn_graph(example[1:])
    lr.enable_cuda_graph(mem, warmup=1)
    with pytest.raises(ValueError, match="horizon_anneal"):
        lr.enable_batch_graph(mem, example)
    with pytest.raises(ValueError, match="horizon_anneal"):
        lr.learn(mem, _Queue(example))
    topo = object.__new__(apex.ApexTopology)     # the refusal comes before any collective
    with pytest.raises(ValueError, match="horizon_anneal"):
        topo.maybe_publish(lr)
    lr.learn_and_update(mem)                      # the learner still steps


class _Queue:
    def __init__(self, item):
        self.item = item

    def get(self):
        return self.item
