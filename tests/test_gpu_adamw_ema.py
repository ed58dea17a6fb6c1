"""AdamW and the EMA target network (BBF): riqn_adamw_step (rainbow_iqn_apex_b200/csrc/iqn_ops.cu), optim.Adam's
weight_decay, target.py and SPR's EMA target encoder.

Kernel: bit for bit against riqn_adam_step applied to numpy's fl32(theta * d) (oracle/bbf.py), eagerly and through a
riqn_dyn_state, at n in {1, 3, 255, 256, 257, 2^20 + 3} and grad_scale in {1, 1/2}; at lambda = 0 it is riqn_adam_step;
non-zero moment prefills, canaries, every call twice with the same bits, refused calls write nothing; and within a
stated bound of torch.optim.AdamW on the CPU.  Learner: every step of a learner with either switch or both is, bit for
bit, a plain learner's gradient followed by the statement by hand (theta * d, Adam, the numpy EMA of oracle/bbf.py, and
a forced rebuild of the target's images), for the IQN, C51 and QR-DQN heads at B = 32 and 512 over three steps; SPR's
targets come from the EMA target's trunk and the EMA projection (against the torch oracle); captured graphs reproduce
eager steps bit for bit; a changed lr under AdamW refuses a replay; checkpoints, resets and data-parallel replicas; and
namespaces with the fields at 0 run the same launches and bits as without them."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, check_bound, f32_bits
from oracle import bbf
from test_gpu_reset import _assert_same, _setup

F32 = lambda x: ctypes.c_float(x).value
SIZES = [1, 3, 255, 256, 257, (1 << 20) + 3]
B1, B2 = 0.9, 0.999


def _raw(name, n, p, g, m, v, step, lr, eps, wd, gs, dyn=None):
    """The return code of riqn_adam_step / riqn_adamw_step (no raise)."""
    from rainbow_iqn_apex_b200 import _lib
    lib = _lib.load()
    mid = [wd] if name == "riqn_adamw_step" else []
    return getattr(lib, name)(n, p, g, m, v, step, lr, B1, B2, eps, *mid, gs, dyn, _lib.stream())


def _inputs(n, seed):
    rs = np.random.RandomState(seed)
    theta = (rs.standard_normal(n) * 10.0 ** rs.uniform(-4, 1, n)).astype(np.float32)
    g = (rs.standard_normal(n) * 10.0 ** rs.uniform(-6, 0, n)).astype(np.float32)
    m = (rs.standard_normal(n) * 1e-3).astype(np.float32)                # non-zero moment prefills
    v = (rs.uniform(0, 1e-5, n)).astype(np.float32)
    return theta, g, m, v


def _run(name, dev, theta, g, m, v, step, lr, eps, wd, gs, dyn=None):
    n = theta.size
    P, M, V = Out(n, dev, fill=theta), Out(n, dev, fill=m), Out(n, dev, fill=v)
    G = Out(n, dev, fill=g)
    assert _raw(name, n, P.p, G.p, M.p, V.p, step, lr, eps, wd, gs, dyn) == 0
    torch.cuda.synchronize()
    for o in (P, M, V, G):
        assert o.canaries_ok()
    assert_bits("grads untouched", G.bits(), f32_bits(g))
    return P.bits(), M.bits(), V.bits()


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("gs", [1.0, 0.5])
def test_adamw_is_adam_on_the_decayed_params(cuda_dev, n, gs):
    from rainbow_iqn_apex_b200.dynstate import DynState
    theta, g, m, v = _inputs(n, n % 1000)
    lr, eps, step = F32(1e-3), F32(1.5e-4), 3
    dyn = DynState(cuda_dev)
    for wd in (0.0, 0.1, 2.5, 999.0):
        d = bbf.decay_f32(lr, wd)
        decayed = bbf.decayed_f32(theta, lr, wd)
        assert wd > 0 or np.array_equal(decayed.view(np.uint32), theta.view(np.uint32))
        for use_dyn in (False, True):
            ptr = None
            if use_dyn:       # bias corrections of another step than the by-value one: the kernel must read the struct
                dyn.write(-(lr / (1 - B1 ** 7)), (1 - B2 ** 7) ** 0.5, 1.0, 0.0)
                ptr = dyn.ptr()
            want = _run("riqn_adam_step", cuda_dev, decayed, g, m, v, step, lr, eps, 0.0, gs, ptr)
            for _ in range(2):                                           # every call: the same bits
                got = _run("riqn_adamw_step", cuda_dev, theta, g, m, v, step, lr, eps, wd, gs, ptr)
                for what, x, y in zip(("theta", "m", "v"), got, want):
                    assert_bits(f"{what} n={n} wd={wd} dyn={use_dyn}", x, y)
        assert 0.0 < d <= 1.0


@pytest.mark.gpu
def test_refused_calls_write_nothing(cuda_dev):
    n = 1000
    theta, g, m, v = _inputs(n, 7)
    P, G, M, V = (Out(n, cuda_dev, fill=x) for x in (theta, g, m, v))
    before = [o.t.clone() for o in (P, G, M, V)]
    lr, eps = F32(1e-3), F32(1e-8)
    calls = [dict(n=0), dict(n=-5), dict(p=None), dict(g=None), dict(m=None), dict(v=None), dict(wd=-1e-9),
             dict(wd=-math.inf), dict(wd=math.inf), dict(wd=math.nan), dict(wd=1000.0),      # lr wd = 1: d = 0
             dict(wd=2000.0), dict(lr=-1e-3, wd=0.1),                                        # d > 1
             dict(lr=math.nan, wd=0.1), dict(lr=math.inf, wd=0.1),
             dict(step=0), dict(step=-1), dict(step=0, wd=0.0)]                              # bc1 = 1 - b1^step <= 0
    for c in calls:
        a = dict(n=n, p=P.p, g=G.p, m=M.p, v=V.p, lr=lr, wd=0.1, step=1)
        a.update(c)
        rc = _raw("riqn_adamw_step", a["n"], a["p"], a["g"], a["m"], a["v"], a["step"], a["lr"], eps, a["wd"], 1.0)
        assert rc == 1, (c, rc)                                            # cudaErrorInvalidValue
    torch.cuda.synchronize()
    for o, t in zip((P, G, M, V), before):
        assert torch.equal(o.t.view(torch.int32), t.view(torch.int32))
    assert _raw("riqn_adamw_step", n, P.p, G.p, M.p, V.p, 1, lr, eps, 999.0, 1.0) == 0    # lr wd just below 1
    torch.cuda.synchronize()
    assert all(o.canaries_ok() for o in (P, G, M, V))


@pytest.mark.gpu
@pytest.mark.parametrize("wd", [0.1, 3.0])
def test_within_bound_of_torch_adamw(cuda_dev, wd):
    """Three steps against torch.optim.AdamW (foreach=False) in float32 on the CPU.  Bound per element:
    8 ulp(theta) + 1e-5 |theta_t - theta_0| + 1e-6 lr.  The update formulas are torch's, but its step size, decay factor
    and 1 - beta1 are formed in double where the kernel receives float32 values."""
    n = (1 << 16) + 5
    theta, _, _, _ = _inputs(n, 11)
    lr, eps = 1e-3, 1e-8
    p = torch.from_numpy(theta.copy()).requires_grad_(True)
    opt = torch.optim.AdamW([p], lr=lr, eps=eps, weight_decay=wd, foreach=False)
    P, M, V = Out(n, cuda_dev, fill=theta), Out(n, cuda_dev, fill=np.zeros(n, np.float32)), Out(n, cuda_dev, fill=np.zeros(n, np.float32))
    rs = np.random.RandomState(12)
    for t in range(1, 4):
        g = (rs.standard_normal(n) * 10.0 ** rs.uniform(-6, 0, n)).astype(np.float32)
        p.grad = torch.from_numpy(g)
        opt.step()
        G = Out(n, cuda_dev, fill=g)
        assert _raw("riqn_adamw_step", n, P.p, G.p, M.p, V.p, t, lr, eps, wd, 1.0) == 0
    torch.cuda.synchronize()
    ref = p.detach().numpy().astype(np.float64)
    bound = 8 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-5 * np.abs(ref - theta) + 1e-6 * lr
    check_bound(f"AdamW wd={wd}", P.f32(), ref, bound)


# ------------------------------------------------------------------------------------------------ learners
HEADS = {"iqn": {}, "c51": dict(rainbow_only=1), "qr": dict(qr_dqn=1)}
SWITCHES = {"ema": dict(target_ema=1, target_ema_tau=0.25), "adamw": dict(adamw=1, adamw_weight_decay=0.5),
            "both": dict(target_ema=1, target_ema_tau=0.25, adamw=1, adamw_weight_decay=0.5)}


def _pair(dev, head, switches, B, seed=5):
    """A learner with ``switches`` and a plain one, both seeded alike (resets off)."""
    a, mem_a = _setup(dev, dict(HEADS[head], **switches), seed=seed, B=B, reset=0)
    b, mem_b = _setup(dev, HEADS[head], seed=seed, B=B, reset=0)
    return a, mem_a, b, mem_b


def _by_hand(b, mem, tau, wd):
    """One step of the plain learner ``b`` with the statement applied by hand: its gradient, theta <- fl32(theta d),
    Adam, then xi <- the numpy EMA and the target's images rebuilt."""
    idxs, loss = b._step_pre(mem)
    if wd is not None:
        d = bbf.decay_f32(b.optimiser.param_groups[0]["lr"], wd)
        b.online_net._flat.mul_(float(d))
    b.optimiser.step()
    mem.update_priorities(idxs, loss)
    if tau is not None:
        on, tg = b.online_net._flat.cpu().numpy(), b.target_net._flat.cpu().numpy()
        b.target_net._flat.copy_(torch.from_numpy(bbf.ema_f32(on, tg, tau)))
        b.target_net.compose_weights()
    return idxs, loss


@pytest.mark.gpu
@pytest.mark.parametrize("head", list(HEADS))
@pytest.mark.parametrize("sw", list(SWITCHES))
@pytest.mark.parametrize("B", [32, 512])
def test_learner_steps_are_the_statement(cuda_dev, head, sw, B):
    a, mem_a, b, mem_b = _pair(cuda_dev, head, SWITCHES[sw], B)
    tau, wd = a.target_ema, a.adamw
    xi = a.target_net._flat.cpu().numpy()
    assert np.array_equal(xi, a.online_net._flat.cpu().numpy())
    for step in range(3):
        ia, la = a.learn_and_update(mem_a)
        ib, lb = _by_hand(b, mem_b, tau, wd)
        torch.cuda.synchronize()
        assert torch.equal(ia, ib) and torch.equal(la, lb), step
        for x, y in ((a.online_net._flat, b.online_net._flat), (a.target_net._flat, b.target_net._flat),
                     (a.optimiser._exp_avg, b.optimiser._exp_avg), (a.optimiser._exp_avg_sq, b.optimiser._exp_avg_sq),
                     (mem_a.transitions.tree, mem_b.transitions.tree)):
            assert torch.equal(x, y), step
        if tau is not None:             # k EMA updates on the online arenas the steps produced, in numpy
            xi = bbf.ema_f32(a.online_net._flat.cpu().numpy(), xi, tau)
            assert_bits(f"target after step {step}", f32_bits(a.target_net._flat.cpu().numpy()), f32_bits(xi))
        else:                           # AdamW alone: the target stays the hard copy
            assert np.array_equal(a.target_net._flat.cpu().numpy(), xi)


@pytest.mark.gpu
def test_spr_targets_come_from_the_ema_encoder(cuda_dev):
    """SPR with target_ema, no random shift: the step's t_k against the torch oracle on the EMA target's trunk and the
    EMA projection, and the EMA projection after the step is the numpy statement."""
    from oracle import curl as ocurl, network as onet
    B = 32
    lr, mem = _setup(cuda_dev, dict(spr=1, target_ema=1, target_ema_tau=0.3, adamw=1), seed=4, B=B, reset=0)
    lr.random_shift = None
    K = lr.spr[0]
    for step in range(3):
        idxs, st, ac, rt, nx, nt, w = mem.sample(B)
        seq = mem.sample_sequence(idxs, K)
        p_tg = {k: v.detach().cpu().clone() for k, v in lr.target_net.state_dict().items() if k.startswith("conv")}
        sp_ema = dict(zip(("weight_h", "bias_h", "weight_c", "bias_c"),
                          (x.cpu().clone() for x in lr.spr_net.views(lr.spr_ema_projection))))
        proj_before = lr.spr_ema_projection.cpu().numpy()
        dbg = {}
        loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg, sequence=seq)
        lr._step_post(mem, idxs, loss)
        torch.cuda.synchronize()
        win = seq[0].cpu()
        xt = torch.cat([win[:, k + 1:k + 5] for k in range(K)]).float().div_(255)
        t = ocurl.project(sp_ema, onet.conv_trunk(p_tg, xt))
        got = dbg["spr_targets"].cpu()
        a, b_ = got.double(), t.double()
        assert float((a * b_).sum() / (a.norm() * b_.norm())) >= 0.9999, step
        assert float((got - t).abs().max()) <= 1e-3 * float(t.abs().max()), step
        want = bbf.ema_f32(lr.spr_net._flat[:lr.spr_net.proj_numel].cpu().numpy(), proj_before, lr.target_ema)
        assert_bits("EMA projection", f32_bits(lr.spr_ema_projection.cpu().numpy()), f32_bits(want))


def _attached_steps(b, mem, n_warm, n_steps):
    """Eager steps of ``b`` through the device step state, as a capture's warm-up and replays run them."""
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
            out.append(loss.clone())
    return out[n_warm:]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [dict(target_ema=1, adamw=1), dict(spr=1, target_ema=1, adamw=1)], ids=["iqn", "spr"])
def test_replay_graph_reproduces_eager_steps(cuda_dev, cfg):
    B = 512 if "spr" not in cfg else 32
    a, mem_a = _setup(cuda_dev, cfg, seed=7, B=B, reset=0)
    b, mem_b = _setup(cuda_dev, cfg, seed=7, B=B, reset=0)
    a.enable_cuda_graph(mem_a)
    la = [a.learn_and_update(mem_a)[1].clone() for _ in range(2)]
    lb = _attached_steps(b, mem_b, 3, 2)
    torch.cuda.synchronize()
    for x, y in zip(la, lb):
        assert torch.equal(x, y) and bool(torch.isfinite(x).all())
    nets = [(a.online_net._flat, b.online_net._flat), (a.target_net._flat, b.target_net._flat),
            (a.optimiser._exp_avg, b.optimiser._exp_avg)]
    if a.spr_ema_projection is not None:
        nets.append((a.spr_ema_projection, b.spr_ema_projection))
    for x, y in nets:
        assert torch.equal(x, y)
    assert not torch.equal(a.target_net._flat, a.online_net._flat)


@pytest.mark.gpu
def test_learn_graph_reproduces_eager_steps(cuda_dev):
    B = 512
    cfg = dict(target_ema=1, adamw=1)
    a, mem_a = _setup(cuda_dev, cfg, seed=8, B=B, reset=0)
    b, mem_b = _setup(cuda_dev, cfg, seed=8, B=B, reset=0)
    batches = [tuple(t.clone() for t in mem_a.sample(B)[1:]) for _ in range(4)]
    a.enable_learn_graph(batches[0])
    la = [a.learn_on_graph(bt).clone() for bt in batches[2:]]
    from rainbow_iqn_apex_b200.dynstate import DynState
    b._dyn = DynState(cuda_dev, slots=len(b._optimisers()))
    lb = []
    with b._attached(None):
        for k, bt in enumerate([batches[0], batches[0]] + batches[2:]):
            if k == 2:
                b._dyn.epoch += 1
            b._write_dyn(None)
            b._reset_step_streams()
            loss = b.compute_gradients(*bt)
            b._step_post(None, None, loss)
            lb.append(loss.clone())
    torch.cuda.synchronize()
    for x, y in zip(la, lb[2:]):
        assert torch.equal(x, y)
    assert torch.equal(a.online_net._flat, b.online_net._flat) and torch.equal(a.target_net._flat, b.target_net._flat)


@pytest.mark.gpu
def test_changed_lr_after_capture_refuses_a_replay(cuda_dev):
    a, mem = _setup(cuda_dev, dict(adamw=1), seed=9, B=32, reset=0)
    a.enable_cuda_graph(mem)
    a.learn_and_update(mem)
    for o, key, f in ((a.optimiser, "lr", 2.0), (a.optimiser, "weight_decay", 0.5)):
        old = o.param_groups[0][key]
        o.param_groups[0][key] = old * f
        with pytest.raises(RuntimeError, match="release_graphs"):
            a.learn_and_update(mem)
        o.param_groups[0][key] = old
        a.learn_and_update(mem)                      # the captured values again: replays
    a.optimiser.param_groups[0]["lr"] *= 2
    a.release_graphs()
    a.learn_and_update(mem)                          # eager
    a.enable_cuda_graph(mem)
    a.learn_and_update(mem)
    # without AdamW an lr change reaches the graph through the device step state, as before
    p, mem_p = _setup(cuda_dev, {}, seed=9, B=32, reset=0)
    p.enable_cuda_graph(mem_p)
    p.optimiser.param_groups[0]["lr"] *= 2
    p.learn_and_update(mem_p)


@pytest.mark.gpu
def test_half_batch_replicas_agree_with_one_learner_given_its_gradient(cuda_dev):
    """Two replicas that each compute a half batch's gradient and then step at grad_scale 1/2 on the summed arenas (what
    the all-reduce leaves) hold the same parameters and target, bit for bit, with no collective for the EMA; and a
    learner at grad_scale 1 stepping on half that sum holds them too."""
    cfg = dict(target_ema=1, adamw=1)
    reps = [_setup(cuda_dev, cfg, seed=10, B=32, reset=0) for _ in range(2)]
    one = _setup(cuda_dev, cfg, seed=10, B=32, reset=0)[0]
    grads = []
    idxs, st, ac, rt, nx, nt, w = reps[0][1].sample(64)
    for (r, _), sl in zip(reps, (slice(0, 32), slice(32, 64))):
        r.compute_gradients(st[sl], ac[sl], rt[sl], nx[sl], nt[sl], w[sl])
        grads.append(r.online_net._flat_grad.clone())
    total = grads[0] + grads[1]
    for r, _ in reps:
        r.online_net._flat_grad.copy_(total)
        r.optimiser.grad_scale = 0.5
        r._step_optimisers()
    one.online_net._flat_grad.copy_(total * 0.5)
    one._step_optimisers()
    torch.cuda.synchronize()
    for r, _ in reps[1:] + reps[:1]:
        assert torch.equal(r.online_net._flat, one.online_net._flat)
        assert torch.equal(r.target_net._flat, one.target_net._flat)
    assert not torch.equal(one.target_net._flat, one.online_net._flat)


@pytest.mark.gpu
def test_checkpoint_restores_target_projection_and_adamw(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_reset import _args
    cfg = dict(spr=1, target_ema=1, adamw=1, adamw_weight_decay=0.2)
    lr, mem = _setup(cuda_dev, cfg, seed=12, B=32, reset=0)
    for _ in range(2):
        lr.learn_and_update(mem)
    lr.save(str(tmp_path), 0, 2, "bbf.pth")
    path = os.path.join(tmp_path, "bbf.pth")
    ck = torch.load(path, map_location="cpu")
    from oracle import network as net
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    assert ck["optimiser_state_dict"]["param_groups"][0]["weight_decay"] == F32(0.2)
    back = Learner(_args(cuda_dev, 32, cfg, reset=0, model=path), 18, None)
    for x, y in ((back.online_net._flat, lr.online_net._flat), (back.target_net._flat, lr.target_net._flat),
                 (back.spr_ema_projection, lr.spr_ema_projection), (back.spr_net._flat, lr.spr_net._flat),
                 (back.optimiser._exp_avg, lr.optimiser._exp_avg), (back.spr_optimiser._exp_avg_sq, lr.spr_optimiser._exp_avg_sq)):
        assert torch.equal(x, y)
    assert not torch.equal(back.target_net._flat, back.online_net._flat)
    assert back.optimiser._step == 2 and back.optimiser.decay() == lr.optimiser.decay() is not None
    # a checkpoint without the EMA entries (saved with the switch off) starts xi = theta and g_xi = g_theta
    del ck["target_state_dict"], ck["spr_ema_projection"]
    torch.save(ck, os.path.join(tmp_path, "old.pth"))
    old = Learner(_args(cuda_dev, 32, cfg, reset=0, model=os.path.join(tmp_path, "old.pth")), 18, None)
    assert torch.equal(old.target_net._flat, old.online_net._flat)
    assert torch.equal(old.spr_ema_projection, old.spr_net._flat[:old.spr_net.proj_numel])


@pytest.mark.gpu
def test_reset_leaves_the_target_which_then_follows_the_reset_network(cuda_dev):
    lr, mem = _setup(cuda_dev, dict(spr=1, target_ema=1), seed=13, B=32, reset=0)
    for _ in range(2):
        lr.learn_and_update(mem)
    xi = lr.target_net._flat.clone()
    lr.reset_networks()
    torch.cuda.synchronize()
    assert torch.equal(lr.target_net._flat, xi)
    assert torch.equal(lr.spr_ema_projection, lr.spr_net._flat[:lr.spr_net.proj_numel])    # set to the new projection
    lr.learn_and_update(mem)
    torch.cuda.synchronize()
    want = bbf.ema_f32(lr.online_net._flat.cpu().numpy(), xi.cpu().numpy(), lr.target_ema)
    assert_bits("target after reset", f32_bits(lr.target_net._flat.cpu().numpy()), f32_bits(want))


# Extra launches per eager step: target_ema adds the EMA and the target's conv / iqn_fc image rebuild
# (riqn_split_bf16_multi), and under SPR the EMA of the projection; adamw adds none (riqn_adamw_step replaces
# riqn_adam_step).
EXTRA_LAUNCHES = {"ema": 2, "adamw": 0, "both": 2}


@pytest.mark.gpu
@pytest.mark.parametrize("head", list(HEADS))
def test_fields_at_zero_run_the_same_launches_and_bits(cuda_dev, head):
    from rainbow_iqn_apex_b200 import _lib
    runs = {}
    for name, extra in (("absent", {}), ("zero", dict(target_ema=0, adamw=0, target_ema_tau=0.5,
                                                      adamw_weight_decay=0.3)),
                        ("ema", SWITCHES["ema"]), ("adamw", SWITCHES["adamw"]), ("both", SWITCHES["both"])):
        lr, mem = _setup(cuda_dev, dict(HEADS[head], **extra), seed=14, B=32, reset=0)
        lr.learn_and_update(mem)                     # first step: every image built once
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        _, loss = lr.learn_and_update(mem)
        torch.cuda.synchronize()
        runs[name] = (_lib.launch_count() - n0, loss.clone(), lr.online_net._flat.clone(), lr.target_net._flat.clone())
    assert runs["absent"][0] == runs["zero"][0]
    _assert_same(runs["absent"][1:], runs["zero"][1:], "fields at 0")
    for name, extra in EXTRA_LAUNCHES.items():
        assert runs[name][0] - runs["absent"][0] == extra, (name, runs[name][0], runs["absent"][0])
