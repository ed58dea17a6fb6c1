"""Cost of HL-Gauss at the benchmark size (B=512, 51 atoms).  (1) One learner step (prioritized sample, loss, backward,
Adam, priority update) replayed from its CUDA graph, for C51, HL-Gauss (r = 0.75), rescaled C51 and rescaled HL-Gauss,
in alternating rounds of 50 steps from one 2^18-transition replay each.  (2) The loss kernels alone,
riqn_hl_gauss_loss_fwd_bwd[_h] against C51's projection riqn_c51_loss_fwd_bwd at B = 512 and 4096 (A = 18), on random
categorical operands, each the median of 5 blocks of 200 launches between CUDA events.  Prints one JSON line with the
card's name, power limit and SM clocks."""
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

ARMS = (("c51", dict(rainbow_only=1)), ("hl_gauss", dict(rainbow_only=1, hl_gauss=1)),
        ("c51_vr", dict(rainbow_only=1, value_rescaling=1)),
        ("hl_gauss_vr", dict(rainbow_only=1, hl_gauss=1, value_rescaling=1)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_us(A=bench.ACTIONS, atoms=51, reps=200):
    """Microseconds per launch of the HL-Gauss and C51 loss kernels (median of 5 blocks of ``reps`` launches)."""
    dev = torch.device("cuda")
    out = {}
    for B in (512, 4096):
        g = torch.Generator(device=dev).manual_seed(B)
        logp = torch.log_softmax(torch.randn(B, A, atoms, device=dev, generator=g), 2)
        pt = torch.softmax(torch.randn(B, A, atoms, device=dev, generator=g), 2)
        acts = torch.randint(0, A, (B,), device=dev, generator=g)
        ast = torch.randint(0, A, (B,), device=dev, generator=g)
        R, nt = 3 * torch.randn(B, device=dev, generator=g), torch.ones(B, device=dev)
        support = torch.linspace(-10.0, 10.0, atoms, device=dev)
        loss, dq = torch.empty(B, device=dev), torch.empty(B, atoms, device=dev)
        p = _lib.ptr
        ops = (p(logp), p(pt), p(acts), p(ast), p(R), p(nt), p(support), 0.97, -10.0, 10.0)
        calls = {"c51": lambda: _lib.call("riqn_c51_loss_fwd_bwd", B, A, atoms, *ops, 20.0 / (atoms - 1), p(loss), p(dq),
                                          None),
                 "hl_gauss": lambda: _lib.call("riqn_hl_gauss_loss_fwd_bwd", B, A, atoms, *ops, 0.75, p(loss), p(dq),
                                               None, None),
                 "hl_gauss_h": lambda: _lib.call("riqn_hl_gauss_loss_fwd_bwd_h", B, A, atoms, *ops, 0.75, 1e-3, p(loss),
                                                 p(dq), None, None)}
        for name, fn in calls.items():
            timed(fn, 20)
            out[f"kernel_us_{name}_b{B}"] = round(1e3 * float(np.median([timed(fn, reps) for _ in range(5)])), 2)
    return out


def main(cap=1 << 18, steps=50, rounds=5):
    dev = torch.device("cuda")
    arms = {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        a.lr, a.adam_eps = 6.25e-5, 1.5e-4
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

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **ker}))


if __name__ == "__main__":
    main()
