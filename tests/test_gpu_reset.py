"""Periodic network resets: riqn_arena_reset (rainbow_iqn_apex_b200/csrc/reset.cu), the reset policy (reset.py) and the
learner's schedule (Learner.reset_networks, Learner.updates).

Kernel: bit for bit against the numpy statement of oracle/reset.py on Philox words of helpers.philox_np, over a
synthetic arena of 2^20 + 3 elements with gaps, uniform and constant segments, several bounds and alpha in {0, 0.25,
0.8}; untouched elements (NaN and inf among them) keep their bits, both moments are zero, canaries survive, and every
refused call returns cudaErrorInvalidValue with nothing written.  Policy: the segment tables cover every parameter of
every arena exactly once for the IQN, C51, QR-DQN, FQF, CURL and SPR agents, with each module's constructor bound or
constant, and a reset is the statement applied to every arena.  Learner: the schedule (eager, replayed and deferred past
a capture's warm-up) against a learner that calls reset_networks() by hand, Adam's restart against a fresh Adam, what a
reset leaves alone, acting right after a reset, checkpoints and data-parallel replicas."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, f32_bits, make_args, philox_np
from oracle import cases, reset as ors

RESET_SEED_TEST = 0x1234_5678_9ABC_DEF1
CONFIGS = {"iqn": {}, "c51": dict(rainbow_only=1), "qr": dict(qr_dqn=1), "fqf": dict(fqf=1), "curl": dict(curl=1),
           "spr": dict(spr=1)}
U, C = ors.UNIFORM, ors.CONSTANT


def _words(seed, stream, n):
    return philox_np(seed, stream, (n + 3) // 4)[:n]


def _raw(n, params, m, v, segs, seed=RESET_SEED_TEST, sid=5, nseg=None):
    """riqn_arena_reset's return code (no raise)."""
    from rainbow_iqn_apex_b200 import _lib
    arr = None
    if segs is not None:
        arr = (_lib.ResetSegment * max(len(segs), 1))(*(_lib.ResetSegment(*s) for s in segs))
    nseg = len(segs) if nseg is None else nseg
    return _lib.load().riqn_arena_reset(n, params, m, v, nseg, arr, seed, sid, _lib.stream())


# ------------------------------------------------------------------------------------------------ kernel
N_BIG = (1 << 20) + 3
SEGS = [(0, 1, U, 0.5, 0.0), (5, 1000, U, 1 / 56, 0.25), (1000, 1003, C, 0.1 / 56, 0.0), (1027, 70000, U, 3.0, 0.8),
        (70001, 70002, C, -2.5, 0.25), (70002, 500000, C, 0.0, 0.8), (500003, 1048000, U, 1e-3, 0.0),
        (1048001, N_BIG, U, 7.0, 0.25)]


def _f32_segs(segs):
    return [(b, e, k, ctypes.c_float(v).value, ctypes.c_float(a).value) for b, e, k, v, a in segs]


def _theta(n, segs, seed=0):
    """A random arena with NaN, inf and -0 in the gaps and in the alpha = 0 segments (alpha > 0 reads finite values)."""
    rs = np.random.RandomState(seed)
    th = rs.standard_normal(n).astype(np.float32) * np.float32(3.0)
    free = np.ones(n, bool)
    for b, e, _, _, a in segs:
        free[b:e] = a == 0
    idx = np.flatnonzero(free)
    pick = rs.choice(idx, min(300, idx.size), replace=False)
    th[pick[:100]] = np.nan
    th[pick[100:200]] = np.inf
    th[pick[200:]] = -0.0
    th.view(np.uint32)[pick[:50]] |= np.uint32(0x12345)          # NaN payloads the kernel must not touch outside segments
    return th


@pytest.mark.gpu
@pytest.mark.parametrize("moments", [True, False])
def test_kernel_vs_statement_bit_for_bit(cuda_dev, moments):
    n, segs = N_BIG, _f32_segs(SEGS)
    th = _theta(n, segs)
    p = Out(n, cuda_dev, fill=th)
    m = Out(n, cuda_dev, fill=np.full(n, 0.75, np.float32)) if moments else None
    v = Out(n, cuda_dev, fill=np.full(n, -3.5, np.float32)) if moments else None
    seed, sid = RESET_SEED_TEST, (7 << 36) + 9
    for rep in range(2):                       # the same bits every call (a second call resets the reset arena again)
        src = th if rep == 0 else want
        assert _raw(n, p.p, m.p if m else None, v.p if v else None, segs, seed, sid) == 0
        torch.cuda.synchronize()
        want = ors.arena_reset(src, segs, _words(seed, sid, n))
        assert_bits("arena", p.bits(), f32_bits(want))
        assert p.canaries_ok()
        for o in (m, v):
            if o is not None:
                assert not o.bits().any() and o.canaries_ok()
    # the statement's uniforms are riqn_fill_uniform's, and the draws are those of the whole arena's positions
    u = Out(n, cuda_dev)
    from rainbow_iqn_apex_b200._lib import call
    call("riqn_fill_uniform", n, seed, sid, u.p, None)
    torch.cuda.synchronize()
    assert_bits("uniforms", u.bits(), f32_bits(ors.uniforms(_words(seed, sid, n))))
    # a segment table of one arena, split into two calls' tables, draws the same values
    th2 = _theta(n, segs, seed=1)
    q = Out(n, cuda_dev, fill=th2)
    assert _raw(n, q.p, None, None, segs[:3], seed, sid) == 0
    assert _raw(n, q.p, None, None, segs[3:], seed, sid) == 0
    torch.cuda.synchronize()
    assert_bits("split table", q.bits(), f32_bits(ors.arena_reset(th2, segs, _words(seed, sid, n))))
    # an arena that is not 16-byte aligned takes the element-wise path: the same bits
    r = Out(n + 1, cuda_dev, fill=np.concatenate([np.float32([5.0]), th2]))
    assert _raw(n, r.p + 4, None, None, segs, seed, sid) == 0
    torch.cuda.synchronize()
    assert_bits("unaligned", r.bits()[1:], f32_bits(ors.arena_reset(th2, segs, _words(seed, sid, n))))
    assert r.f32()[0] == 5.0 and r.canaries_ok()
    # alpha = 0 is theta0 itself; fresh constant segments hold the constant
    b, e = 1000, 1003
    assert np.all(p.f32()[b:e] == np.float32(0.1 / 56))


@pytest.mark.gpu
def test_rejected_calls_write_nothing(cuda_dev):
    n = 4099
    ok = [(0, 10, U, 0.5, 0.0), (20, 30, C, 1.0, 0.5)]
    th = _theta(n, ok, seed=3)
    p, m, v = Out(n, cuda_dev, fill=th), Out(n, cuda_dev, fill=np.ones(n, np.float32)), Out(n, cuda_dev, fill=np.ones(n, np.float32))
    before = [o.t.clone() for o in (p, m, v)]
    inf, nan = math.inf, math.nan
    bad_tables = [[(10, 20, U, 1.0, 0.0), (0, 5, U, 1.0, 0.0)],          # unsorted
                  [(0, 10, U, 1.0, 0.0), (9, 20, U, 1.0, 0.0)],          # overlapping
                  [(n - 1, n + 1, U, 1.0, 0.0)], [(-1, 3, U, 1.0, 0.0)], [(5, 5, U, 1.0, 0.0)], [(7, 3, U, 1.0, 0.0)],
                  [(0, 3, 2, 1.0, 0.0)], [(0, 3, -1, 1.0, 0.0)],
                  [(0, 3, U, 0.0, 0.0)], [(0, 3, U, -1.0, 0.0)], [(0, 3, U, inf, 0.0)], [(0, 3, U, nan, 0.0)],
                  [(0, 3, C, inf, 0.0)], [(0, 3, C, -inf, 0.0)], [(0, 3, C, nan, 0.0)],
                  [(0, 3, U, 1.0, -0.1)], [(0, 3, U, 1.0, 1.0)], [(0, 3, U, 1.0, 1.5)], [(0, 3, U, 1.0, nan)],
                  [(k, k + 1, U, 1.0, 0.0) for k in range(65)]]              # 65 segments
    calls = [dict(segs=t) for t in bad_tables]
    calls += [dict(n=0), dict(n=-1), dict(nseg=0), dict(nseg=65), dict(params=None), dict(m=None), dict(v=None),
              dict(segs=None, nseg=1), dict(n=25)]                            # n = 25 puts segment (20, 30) outside
    for c in calls:
        args = dict(n=n, params=p.p, m=m.p, v=v.p, segs=ok, nseg=None)
        args.update(c)
        rc = _raw(args["n"], args["params"], args["m"], args["v"], args["segs"], nseg=args["nseg"])
        assert rc == 1, (c, rc)                      # cudaErrorInvalidValue
    torch.cuda.synchronize()
    for o, t in zip((p, m, v), before):
        assert torch.equal(o.t.view(torch.int32), t.view(torch.int32))
    # the same table is accepted as it stands, with both moments or with neither
    assert _raw(n, p.p, m.p, v.p, ok) == 0 and _raw(n, p.p, None, None, ok) == 0
    torch.cuda.synchronize()
    assert p.canaries_ok() and m.canaries_ok() and v.canaries_ok()


# ------------------------------------------------------------------------------------------------ learners
def _args(dev, B, fields, **more):
    a = make_args(dev, B, cases.iqn_cfg(64, 64, 32), rainbow_only=bool(fields.get("rainbow_only")), nb_actor=2,
                  actor_capacity=512)
    for k, v in dict(fields, random_shift=4, **more).items():
        setattr(a, k, v)
    return a


def _setup(dev, fields, seed=0, B=32, **more):
    """A seeded learner with ``fields`` (resets on unless ``more`` says otherwise) and a replay of 612 + 300 transitions."""
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    torch.manual_seed(seed)
    args = _args(dev, B, fields, **dict(dict(reset=1), **more))
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


def _state(lr, mem=None):
    """Every arena and moment arena, each optimiser's step, and the replay tree: clones."""
    out = []
    for net, opt in zip(lr._trained_nets(), lr._optimisers()):
        out += [net._flat.clone(), opt._exp_avg.clone(), opt._exp_avg_sq.clone(), opt._step]
    out += [lr.target_net._flat.clone(), lr.online_net._eps_flat.clone(), lr.updates, lr.resets]
    if mem is not None:
        out.append(mem.transitions.tree.clone())
    return out


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        if torch.is_tensor(x):
            assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                               y.view(torch.int32) if y.dtype == torch.float32 else y), (what, k)
        else:
            assert x == y, (what, k, x, y)


def _torch_bound(t, gain_kind):
    """The largest value torch's constructor init could draw for ``t``: kaiming_uniform_(a=sqrt(5)) of nn.Linear /
    nn.Conv2d weights, 1/sqrt(fan_in) of their biases, FQF's xavier_uniform_(gain=0.01)."""
    if gain_kind == "xavier":
        fan_in, fan_out = torch.nn.init._calculate_fan_in_and_fan_out(t)
        return math.sqrt(3.0) * 0.01 * math.sqrt(2.0 / float(fan_in + fan_out))
    if gain_kind == "kaiming":
        fan_in, _ = torch.nn.init._calculate_fan_in_and_fan_out(t)
        return math.sqrt(3.0) * torch.nn.init.calculate_gain("leaky_relu", math.sqrt(5)) / math.sqrt(fan_in)
    return 1.0 / math.sqrt(gain_kind)


def _expected(lr):
    """Per arena index, parameter name -> ("U", the largest value its constructor could draw), ("C", the double its
    constructor fills in) or ("S", that bound) for the shrink-and-perturb segments."""
    on = lr.online_net
    exp = {0: {}}
    for name, p in on.named_parameters():
        mod, attr = name.rsplit(".", 1)
        m = on.get_submodule(mod)
        if mod.startswith("conv"):
            exp[0][name] = ("S", _torch_bound(m.weight, "kaiming") if attr == "weight" else 1 / math.sqrt(m.weight[0].numel()))
        elif mod == "iqn_fc":
            exp[0][name] = ("U", _torch_bound(p, "kaiming") if attr == "weight" else 1 / math.sqrt(m.in_features))
        elif attr in ("weight_mu", "bias_mu"):
            exp[0][name] = ("U", 1 / math.sqrt(m.in_features))
        elif attr == "weight_sigma":
            exp[0][name] = ("C", m.std_init / math.sqrt(m.in_features))
        else:
            exp[0][name] = ("C", m.std_init / math.sqrt(m.out_features))
    if lr.fraction_net is not None:
        f = lr.fraction_net
        exp[1] = {"weight": ("U", _torch_bound(f.weight, "xavier")), "bias": ("C", 0.0)}
    for k, net in ((2, lr.curl_net), (3, lr.spr_net)):
        if net is None:
            continue
        exp[k] = {}
        for name in net.NAMES:
            p = net.get_parameter(name)
            kind = "S" if name.startswith("conv") else "U"
            if p.dim() > 1:
                exp[k][name] = (kind, _torch_bound(p, "kaiming"))
            else:
                w = net.get_parameter(name.replace("bias", "weight"))
                exp[k][name] = (kind, 1 / math.sqrt(w[0].numel()))
    return exp


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_tables_cover_the_arenas_and_reset_is_the_statement(cuda_dev, cfg):
    from rainbow_iqn_apex_b200 import reset as rs_mod
    for shrink in (0.0, 0.5):
        lr, mem = _setup(cuda_dev, CONFIGS[cfg], seed=4, reset_shrink=shrink)
        lr.learn_and_update(mem)                       # moments and weights away from their construction values
        tables = rs_mod.tables(lr)
        exp = _expected(lr)
        assert [k for k, *_ in tables] == sorted(exp)
        before = {k: net._flat.cpu().numpy().copy() for k, net, _, _ in tables}
        lr.reset_networks()
        torch.cuda.synchronize()
        seed = lr.online_net._rng_seed ^ rs_mod.RESET_SEED
        for k, net, opt, segs in tables:
            assert 1 <= len(segs) <= 64 and opt._step == 0 and not opt.state
            assert not opt._exp_avg.any() and not opt._exp_avg_sq.any()
            got = net._flat.cpu().numpy()
            want = ors.arena_reset(before[k], segs, _words(seed, k, net._flat.numel()))
            assert_bits(f"{cfg} arena {k}", f32_bits(got), f32_bits(want))
            by_begin = {s[0]: s for s in segs}
            covered = 0
            for name, p in net.named_parameters():
                s = by_begin.pop(p._riqn_offset)           # every parameter is exactly one segment
                assert s[1] == p._riqn_offset + p.numel(), name
                covered += p.numel()
                kind, val = exp[k][name]
                assert s[4] == (ctypes.c_float(shrink).value if kind == "S" else 0.0), name
                x = got[s[0]:s[1]]
                if kind == "C":
                    assert s[2] == C and s[3] == ctypes.c_float(val).value, name
                    assert np.all(f32_bits(x) == f32_bits(np.float32(val))), name
                    continue
                b = ctypes.c_float(val).value
                assert s[2] == U and s[3] == b, (name, s[3], b)
                if s[4] == 0.0:
                    assert np.all(np.abs(x) <= np.float32(b)), name
                    if x.size >= 4096:
                        x64, nn_ = x.astype(np.float64), x.size
                        assert abs(x64.mean()) <= 6 * b / math.sqrt(3 * nn_), name
                        assert abs((x64 ** 2).mean() - b * b / 3) <= 6 * b * b * math.sqrt(4 / 45 / nn_), name
            assert not by_begin                                 # nothing else is in a segment
            assert covered == sum(s[1] - s[0] for s in segs)
        assert lr.resets == 1


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["spr", "fqf", "curl"])
def test_schedule_equals_reset_by_hand(cuda_dev, cfg):
    """reset_interval = 3: seven eager learn_and_update steps equal seven steps of a learner that resets by hand after
    steps 3 and 6 (every arena, moment, optimiser step, loss and priority)."""
    a, mem_a = _setup(cuda_dev, CONFIGS[cfg], seed=6, reset_interval=3)
    b, mem_b = _setup(cuda_dev, CONFIGS[cfg], seed=6, reset_interval=10 ** 9)
    for step in range(1, 8):
        ia, la = a.learn_and_update(mem_a)
        ib, lb = b.learn_and_update(mem_b)
        if step % 3 == 0:
            b.reset_networks()
        torch.cuda.synchronize()
        assert torch.equal(ia, ib) and torch.equal(la, lb), step
        _assert_same(_state(a, mem_a), _state(b, mem_b), (cfg, step))
    assert a.updates == 7 and a.resets == 2


def _eager_attached(b, mem_b, plan):
    """Eager steps of ``b`` through the device step state, as a capture's warm-up and replays run them: ``plan`` a list
    of "step" / "reset" / "capture" (the epoch a capture writes without running a step)."""
    from rainbow_iqn_apex_b200.dynstate import DynState
    b._dyn = DynState(b.online_net._flat.device, slots=len(b._optimisers()))
    losses = []
    with b._attached(mem_b):
        for what in plan:
            if what == "capture":
                b._dyn.epoch += 1
            elif what == "reset":
                b.reset_networks()
            else:
                b._write_dyn(mem_b)
                idx, loss = b._step_pre(mem_b)
                b._step_post(mem_b, idx, loss)
                b.updates += 1
                losses.append(loss.clone())
    return losses


@pytest.mark.gpu
@pytest.mark.parametrize("interval,warmup,resets_after", [(3, 3, (3, 6)), (2, 3, (3, 4, 6))])
def test_replayed_schedule_and_deferred_reset(cuda_dev, interval, warmup, resets_after):
    """Through enable_cuda_graph: the warm-up steps count, a reset due inside them runs when enable_cuda_graph returns
    (interval 2, warm-up 3: after update 3, then 4 and 6), and the replays equal eager steps with resets by hand."""
    a, mem_a = _setup(cuda_dev, CONFIGS["spr"], seed=3, reset_interval=interval)
    b, mem_b = _setup(cuda_dev, CONFIGS["spr"], seed=3, reset_interval=10 ** 9)
    a.enable_cuda_graph(mem_a, warmup=warmup)
    assert a.updates == warmup and a.resets == 1
    plan = []
    for u in range(1, 8):
        plan.append("step")
        if u == warmup:
            plan.append("capture")
        if u in resets_after:
            plan.append("reset")
    lb = _eager_attached(b, mem_b, plan)
    la = [a.learn_and_update(mem_a)[1].clone() for _ in range(7 - warmup)]
    torch.cuda.synchronize()
    for x, y in zip(la, lb[warmup:]):
        assert torch.equal(x, y) and bool(torch.isfinite(x).all())
    assert a.updates == 7 and a.resets == len(resets_after)
    _assert_same(_state(a, mem_a), _state(b, mem_b), "graph vs eager")


@pytest.mark.gpu
def test_adam_restart_equals_a_fresh_adam(cuda_dev):
    from rainbow_iqn_apex_b200.model import DQN
    from rainbow_iqn_apex_b200.optim import Adam
    from rainbow_iqn_apex_b200.spr import SprNet
    lr, mem = _setup(cuda_dev, CONFIGS["spr"], seed=9)
    for _ in range(2):
        lr.learn_and_update(mem)
    lr.reset_networks()
    idxs, st, ac, rt, nx, nt, w = mem.sample(32)
    seq = mem.sample_sequence(idxs, lr.spr[0])
    lr.compute_gradients(st, ac, rt, nx, nt, w, sequence=seq)
    pairs = []
    for net, fresh in ((lr.online_net, DQN(_args(cuda_dev, 32, {}), 18).to(cuda_dev)), (lr.spr_net, SprNet(18, cuda_dev))):
        fresh._flat.copy_(net._flat)
        fresh._flat_grad.copy_(net._flat_grad)
        pairs.append((net, fresh, Adam(fresh.parameters(), lr=lr.optimiser.param_groups[0]["lr"],
                                       eps=lr.optimiser.param_groups[0]["eps"])))
    lr.apply_gradients()
    for net, fresh, opt in pairs:
        opt.step()
    torch.cuda.synchronize()
    for (net, fresh, opt), mine in zip(pairs, (lr.optimiser, lr.spr_optimiser)):
        assert torch.equal(net._flat, fresh._flat) and mine._step == opt._step == 1
        assert torch.equal(mine._exp_avg, opt._exp_avg) and torch.equal(mine._exp_avg_sq, opt._exp_avg_sq)
        assert float(mine.state_dict()["state"][0]["step"]) == 1.0


@pytest.mark.gpu
def test_policy_leaves_target_epsilons_and_momentum_trunk(cuda_dev):
    from rainbow_iqn_apex_b200 import curl
    from rainbow_iqn_apex_b200.model import DQN
    lr, mem = _setup(cuda_dev, CONFIGS["curl"], seed=2)
    for _ in range(2):
        lr.learn_and_update(mem)
    keep = [lr.target_net._flat.clone(), lr.target_net._eps_flat.clone(), lr.online_net._eps_flat.clone(),
            lr.momentum_net._flat.clone()]
    lr.reset_networks()
    torch.cuda.synchronize()
    for x, y in zip(keep, (lr.target_net._flat, lr.target_net._eps_flat, lr.online_net._eps_flat, lr.momentum_net._flat)):
        assert torch.equal(x, y)
    assert torch.equal(lr.momentum_projection, lr.curl_net._flat[:lr.curl_net.proj_numel])
    n = curl.trunk_numel(lr.online_net)
    assert not torch.equal(lr.online_net._flat[:n], lr.momentum_net._flat[:n])
    # acting right after the reset reads the reset weights: a network loaded with the reset arena acts the same
    states = mem.sample(8)[1]
    tau = torch.rand(32 * 8, 1, device=cuda_dev)
    ref = DQN(_args(cuda_dev, 8, {}), 18).to(cuda_dev)
    ref.load_state_dict(lr.online_net.state_dict())
    ref.train()
    with torch.no_grad():
        q_act, _ = lr.online_net(states, 32, tau=tau, fresh_weights=True)
        q_ref, _ = ref(states, 32, tau=tau)
    torch.cuda.synchronize()
    assert torch.equal(q_act, q_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["iqn", "spr"])
def test_shrink_one_keeps_the_trunk(cuda_dev, cfg):
    from rainbow_iqn_apex_b200 import curl
    lr, mem = _setup(cuda_dev, CONFIGS[cfg], seed=5, reset_shrink=1.0)
    lr.learn_and_update(mem)
    n = curl.trunk_numel(lr.online_net)
    trunk = lr.online_net._flat[:n].clone()
    head = lr.online_net._flat[n:].clone()
    spr = None
    if lr.spr_net is not None:
        s = lr.spr_net
        b, e = s.conv1.weight._riqn_offset, s.conv2.bias._riqn_offset + s.conv2.bias.numel()
        spr = (b, e, s._flat[b:e].clone())
    lr.reset_networks()
    torch.cuda.synchronize()
    assert torch.equal(lr.online_net._flat[:n], trunk) and not torch.equal(lr.online_net._flat[n:], head)
    assert not lr.optimiser._exp_avg.any()
    if spr is not None:
        b, e, t = spr
        assert torch.equal(lr.spr_net._flat[b:e], t)


@pytest.mark.gpu
def test_checkpoint_between_resets_resumes_bit_for_bit(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Learner
    lr, mem = _setup(cuda_dev, CONFIGS["spr"], seed=8, reset_interval=3)
    batches = []
    for _ in range(8):
        idxs, st, ac, rt, nx, nt, w = mem.sample(32)
        batches.append((st, ac, rt, nx, nt, w, mem.sample_sequence(idxs, lr.spr[0])))
    for bt in batches[:4]:
        lr.learn_on_batch(*bt[:6], sequence=bt[6])
    assert (lr.updates, lr.resets) == (4, 1)
    lr.save(str(tmp_path), 0, 4, "reset.pth")
    path = os.path.join(tmp_path, "reset.pth")
    ck = torch.load(path, map_location="cpu")
    assert tuple(ck["reset_state"]) == (4, 1)
    torch.manual_seed(123)
    back = Learner(_args(cuda_dev, 32, CONFIGS["spr"], reset=1, reset_interval=3, model=path), 18, None)
    back.train()
    assert (back.updates, back.resets) == (4, 1) and back.optimiser._step == lr.optimiser._step == 1
    back.target_net._flat.copy_(lr.target_net._flat)
    back.target_net._eps_flat.copy_(lr.target_net._eps_flat)
    back.online_net._eps_flat.copy_(lr.online_net._eps_flat)
    for x, y in ((back.online_net, lr.online_net), (back.target_net, lr.target_net)):
        x._rng_seed, x._tau_calls, x._shift_calls = y._rng_seed, y._tau_calls, y._shift_calls
        for (_, m), (_, n_) in zip(x.noisy_layers(), y.noisy_layers()):
            m._noise_calls = n_._noise_calls
        x.compose_weights()
    _assert_same(_state(back), _state(lr), "restored")
    for step, bt in enumerate(batches[4:], 5):
        l1 = lr.learn_on_batch(*bt[:6], sequence=bt[6])
        l2 = back.learn_on_batch(*bt[:6], sequence=bt[6])
        torch.cuda.synchronize()
        assert torch.equal(l1, l2), step
        _assert_same(_state(back), _state(lr), step)
    assert lr.resets == back.resets == 2
    # resets off: no reset_state, and model_state_dict keeps the reference schema
    from oracle import network as net
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    plain, _ = _setup(cuda_dev, {}, seed=8, reset=0)
    plain.save(str(tmp_path), 0, 0, "plain.pth")
    assert "reset_state" not in torch.load(os.path.join(tmp_path, "plain.pth"), map_location="cpu")


@pytest.mark.gpu
def test_data_parallel_replicas_draw_identical_resets(cuda_dev):
    """Two learners whose arenas and noise seed are rank 0's (what make_data_parallel broadcasts) reset identically."""
    r0, m0 = _setup(cuda_dev, CONFIGS["spr"], seed=31)
    r1, m1 = _setup(cuda_dev, CONFIGS["spr"], seed=32)
    assert not torch.equal(r0.online_net._flat, r1.online_net._flat)
    for x, y in ((r1.online_net, r0.online_net), (r1.target_net, r0.target_net)):
        x._flat.copy_(y._flat)
        x._eps_flat.copy_(y._eps_flat)
        x._rng_seed = y._rng_seed
        x.compose_weights()
    r1.spr_net._flat.copy_(r0.spr_net._flat)
    for r in (r0, r1):
        r.reset_networks()
        r.reset_networks()
    torch.cuda.synchronize()
    _assert_same(_state(r0), _state(r1), "replicas")
    assert r0.resets == 2
