"""GPU: the CUDA-graph learner step (Learner.enable_cuda_graph) equals the eager step driven by the same device-resident
per-step state (Philox offsets, Adam bias corrections, beta / capacity), and advances its randomness every replay."""
import numpy as np
import pytest
import torch

from helpers import load_params, make_args
from oracle import cases, network as net

pytestmark = pytest.mark.gpu


def _setup(dev, seed):
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    torch.manual_seed(seed)
    cfg = cases.iqn_cfg(16, 16, 8)
    args = make_args(dev, 16, cfg, nb_actor=1, actor_capacity=512)
    lr = Learner(args, 18, None)
    load_params(lr.online_net, net.make_params(5))
    lr.update_target_net()
    mem = ReplayMemory(args, None)
    rs = np.random.RandomState(1)
    n = 512
    mem.transitions.append_arrays(0, 0, np.arange(n) % 97, rs.randint(0, 256, (n, 84, 84)).astype(np.uint8),
                                  rs.randint(0, 18, n), rs.randint(-1, 2, n).astype(np.float32), rs.uniform(size=n) < 0.03,
                                  (rs.uniform(0.1, 1, n) ** 0.2).astype(np.float32))
    for obj, sd in ((lr.online_net, 11), (lr.target_net, 12), (mem.transitions, 13)):
        obj._rng_seed = sd
    return lr, mem


def test_graph_replay_matches_eager_through_the_attached_step_state(cuda_dev):
    from rainbow_iqn_apex_b200.dynstate import DynState
    a, mem_a = _setup(cuda_dev, 0)
    b, mem_b = _setup(cuda_dev, 0)
    a.enable_cuda_graph(mem_a, warmup=2)              # 2 eager warm-up steps, then capture
    # b: the same steps, all eager, through the same body / dyn protocol
    b._dyn = DynState(cuda_dev)

    def eager_step():
        nss, sbc = b.optimiser.bias_corrections(b.optimiser._step + 1)
        b._dyn.write(nss, sbc, mem_b.transitions.get_current_capacity(), mem_b.priority_weight)
        idxs, loss = b._step_pre(mem_b)
        b._step_post(mem_b, idxs, loss)
        return idxs, loss

    losses = []
    with b._attached(mem_b):
        for _ in range(2):
            eager_step()
        b._dyn.epoch += 1                              # the write issued right before the capture
        for i in range(3):
            ia, la = a.learn_and_update(mem_a)
            ib, lb = eager_step()
            assert torch.equal(ia, ib)                 # same prioritized sample (device RNG driven by the same state)
            # fp32 atomics (split-K / col2im accumulation order) differ run to run: last-bits noise in the gradients,
            # occasionally one ReLU-kink flip in a later step (see below)
            assert torch.allclose(la, lb, rtol=2e-3, atol=1e-6)
            losses.append(la.clone())
    assert a.optimiser._step == b.optimiser._step == 5
    # The two runs differ by the order of fp32 atomics (split-K / col2im / strip weight gradients): ~1e-8 on the weights
    # after a step.  That noise can push a hidden activation across its ReLU kink in one run only, which changes ONE
    # row of the next weight gradient (dh[r, o] * x[r, :]); Adam turns it into a difference of at most lr per step on
    # that row.  So: all but a handful of rows agree to 1e-5, and nothing differs by more than 3 steps * lr.
    d = (a.online_net._flat - b.online_net._flat).abs()
    assert float(d.max()) <= 3 * 5e-5 + 1e-6
    assert int((d > 1e-5).sum()) <= 5 * 3136
    assert torch.allclose(mem_a.transitions.tree, mem_b.transitions.tree, rtol=1e-4, atol=0)
    assert not torch.equal(losses[0], losses[1])       # fresh noise / quantiles / samples every replay
    assert torch.isfinite(torch.stack(losses)).all()
    assert not torch.equal(a.online_net._flat, a.target_net._flat)
    # after the capture the dyn state is detached: eager calls use their by-value arguments and the host counters again
    assert a.optimiser._dyn is None and mem_a.transitions._dyn is None and a.online_net._dyn is None
    step_before = a.optimiser._step
    s1, s2 = mem_a.sample(16), mem_a.sample(16)
    assert not torch.equal(s1[0], s2[0])               # fresh stratified draws (the eager counter advances)
    from rainbow_iqn_apex_b200 import ReplayMemory
    other = ReplayMemory(make_args(cuda_dev, 16, cases.iqn_cfg(16, 16, 8), nb_actor=1, actor_capacity=512), None)
    other.transitions.append_arrays(0, 0, np.arange(512) % 97, np.zeros((512, 84, 84), np.uint8), np.zeros(512, np.int64),
                                    np.ones(512, np.float32), np.zeros(512, bool), np.full(512, 0.5, np.float32))
    p_before = a.online_net._flat.clone()
    a.learn_and_update(other)                          # eager fall-through on a memory the graph was not captured for
    assert a.optimiser._step == step_before + 1 and not torch.equal(p_before, a.online_net._flat)


def test_host_batch_graph(cuda_dev):
    lr, mem = _setup(cuda_dev, 1)
    lr.enable_cuda_graph(mem, warmup=2)
    lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(16)))
    host = tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(16))
    before = lr.online_net._flat.clone()
    l1 = lr.learn_on_host_batch(host).clone()
    l2 = lr.learn_on_host_batch(host).clone()
    assert torch.isfinite(l1).all() and not torch.equal(l1, l2)
    assert not torch.equal(before, lr.online_net._flat)
    new_pri = mem.transitions.tree[host[0].to(cuda_dev)]
    assert torch.allclose(new_pri.float(), l2.pow(0.2), rtol=1e-5)      # priorities of the batch were updated
    # prefetched path: same batch through the side-stream staging gives a valid step too
    lr.prefetch_host_batch(host)
    l3 = lr.learn_on_host_batch().clone()
    lr.prefetch_host_batch(host)
    l4 = lr.learn_on_host_batch().clone()
    assert torch.isfinite(l3).all() and torch.isfinite(l4).all() and not torch.equal(l3, l4)


def test_learn_graph_reads_the_live_step_state_after_a_later_capture(cuda_dev):
    """A learner that captures its learn graph and then its replay-resident step keeps one device step state for both:
    later learn-graph replays draw fresh noise and step Adam with the current bias corrections."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    from rainbow_iqn_apex_b200.dynstate import DynState
    lr, mem = _setup(cuda_dev, 2)
    ex = tuple(t.contiguous() for t in mem.sample(16)[1:])
    lr.enable_learn_graph(ex)
    lr.enable_cuda_graph(mem)
    eps = lr.online_net.fcnoisy_h_v._eps_in
    lr.learn_on_graph(ex)
    torch.cuda.synchronize()
    eps1 = eps.clone()
    o = lr.optimiser
    p0, m0, v0 = (t.clone() for t in (o._flat, o._exp_avg, o._exp_avg_sq))
    lr.learn_on_graph(ex)
    torch.cuda.synchronize()
    assert not torch.equal(eps1, eps)                  # fresh noise every replay
    g = lr.online_net._flat_grad.clone()
    d = DynState(cuda_dev)
    d.write(*o.bias_corrections(o._step), 1.0, 0.0)
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    grp = o.param_groups[0]
    call("riqn_adam_step", p.numel(), ptr(p), ptr(g), ptr(m), ptr(v), o._step, float(grp["lr"]), float(grp["betas"][0]),
         float(grp["betas"][1]), float(grp["eps"]), float(o.grad_scale), d.ptr())
    torch.cuda.synchronize()
    assert torch.equal(p, o._flat) and torch.equal(m, o._exp_avg) and torch.equal(v, o._exp_avg_sq)
    assert not torch.equal(p0, o._flat)


def test_data_parallel_graphs_with_the_collective_outside(cuda_dev):
    """A learner in a one-rank process group that keeps the all-reduce eager between two graphs per step computes the
    bits of the same learner without a process group, and its host-batch graph is split the same way."""
    import bench
    import torch.distributed as dist
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    from test_gpu_fqf import _free_port
    cap = 1 << 14
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        runs = []
        for dp in (False, True):
            torch.manual_seed(5)
            a = bench.make_args(cuda_dev, cap)
            lr = Learner(a, bench.ACTIONS, None)
            lr.train()
            mem = ReplayMemory(a, None)
            bench.fill_replay(mem, cap, cuda_dev, 7)
            if dp:
                lr.process_group = dist.group.WORLD
            lr.enable_cuda_graph(mem, warmup=2, capture_collectives=False)
            assert (lr._graphs["replay"].post is not None) == dp
            steps = [tuple(t.clone() for t in lr.learn_and_update(mem)) for _ in range(3)]
            torch.cuda.synchronize()
            runs.append((steps, lr.online_net._flat.detach().clone()))
        (s1, p1), (s2, p2) = runs
        for k, ((i1, l1), (i2, l2)) in enumerate(zip(s1, s2)):
            assert torch.equal(i1, i2), f"step {k}: sampled indices differ"
            assert torch.equal(l1, l2), f"step {k}: losses differ"
        assert torch.equal(p1, p2)
        lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(bench.B)))
        assert lr._graphs["batch"].post is not None
        host = tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(bench.B))
        l1 = lr.learn_on_host_batch(host).clone()
        l2 = lr.learn_on_host_batch(host).clone()
        assert torch.isfinite(l1).all() and torch.isfinite(l2).all() and not torch.equal(l1, l2)
        new_pri = mem.transitions.tree[host[0].to(cuda_dev)]
        assert torch.allclose(new_pri.float(), l2.pow(0.2), rtol=1e-5)      # priorities of the batch were updated
    finally:
        dist.destroy_process_group()
