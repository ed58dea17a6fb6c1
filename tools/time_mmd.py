"""Cost of MMDQN at the benchmark size (B=512).  (1) One learner step (prioritized sample, loss, backward, Adam, priority
update) replayed from its CUDA graph, for QR-DQN and MMDQN (bandwidths 1..10) at N = 64 and N = 200, in alternating
rounds of 50 steps from one 2^18-transition replay each.  (2) The loss kernel alone, riqn_mmd_loss_fwd_bwd at
n in {64, 200} and H in {1, 10}, against QR-DQN's quantile-Huber kernel riqn_iqn_loss_fwd_bwd (n = n' = N) at the same
sizes, on Gaussian operands, each timed over many launches between CUDA events.  Prints one JSON line with the card's
name and power limit."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib  # noqa: E402

ARMS = (("qr64", dict(qr_dqn=1, num_tau_samples=64)), ("mmd64", dict(qr_dqn=1, mmd=1, num_tau_samples=64)),
        ("qr200", dict(qr_dqn=1, num_tau_samples=200)), ("mmd200", dict(qr_dqn=1, mmd=1, num_tau_samples=200)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_us(B=512, A=bench.ACTIONS, reps=200):
    """Microseconds per launch of the MMD and quantile-Huber loss kernels (median of 5 blocks of ``reps`` launches)."""
    dev = torch.device("cuda")
    out = {}
    for n in (64, 200):
        g = torch.Generator(device=dev).manual_seed(n)
        q_on = torch.randn(n * B, A, device=dev, generator=g)
        q_tgt = torch.randn(n * B, A, device=dev, generator=g)
        acts = torch.randint(0, A, (B,), device=dev, generator=g)
        ast = torch.randint(0, A, (B,), device=dev, generator=g)
        R, nt = torch.randn(B, device=dev, generator=g), torch.ones(B, device=dev)
        tau = torch.rand(n * B, device=dev, generator=g)
        loss, dth = torch.empty(B, device=dev), torch.empty(n * B, device=dev)
        p = _lib.ptr
        calls = {"huber": lambda: _lib.call("riqn_iqn_loss_fwd_bwd", B, n, n, A, p(q_on), p(q_tgt), p(tau), p(acts),
                                            p(ast), p(R), p(nt), 0.97, 1.0, p(loss), p(dth), None, None)}
        for H in (1, 10):
            hb = (ctypes.c_float * H)(*[float(h) for h in range(1, H + 1)])
            calls[f"mmd_h{H}"] = (lambda hb=hb, H=H: _lib.call(
                "riqn_mmd_loss_fwd_bwd", B, n, A, p(q_on), p(q_tgt), p(acts), p(ast), p(R), p(nt), 0.97, H, hb, p(loss),
                p(dth), None, None))
        for name, fn in calls.items():
            timed(fn, 20)
            out[f"kernel_us_{name}_n{n}"] = round(1e3 * float(np.median([timed(fn, reps) for _ in range(5)])), 2)
    return out


def main(cap=1 << 18, steps=50, rounds=5):
    dev = torch.device("cuda")
    arms = {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        for k, v in fields.items():
            setattr(a, k, v)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        c0 = _lib.launch_count()
        learner.learn_and_update(mem)                    # one eager step: the launches it makes
        launches = _lib.launch_count() - c0
        learner.enable_cuda_graph(mem)
        for _ in range(5):
            learner.learn_and_update(mem)
        arms[name] = (learner, mem, launches)
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (learner, mem, _) in arms.items():
            step_ms[name].append(timed(lambda: learner.learn_and_update(mem), steps))
    for learner, _, _ in arms.values():
        learner.release_graphs()
    ker = kernel_us()

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **ker}))


if __name__ == "__main__":
    main()
