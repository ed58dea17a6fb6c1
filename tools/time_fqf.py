"""Cost of FQF at the benchmark size (B=512, N=64): one learner step (prioritized sample, loss, fraction loss, backward,
both Adam steps, priority update) replayed from its CUDA graph, for a plain IQN learner (K=32, N'=64) and an FQF learner,
in alternating rounds of 50 steps.  The FQF step runs 191 no-grad head rows per transition (N for a*, N for the target,
N-1 inner boundaries) against IQN's 96 (K + N'), plus the fraction proposal (two logits products, the fractions, the
fraction backward and weight gradient).  Device time from CUDA events; prints one JSON line with the card's name and
power limit."""
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


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main(cap=1 << 18, steps=50, rounds=5):
    dev = torch.device("cuda")
    arms = {}
    for name, fqf in (("iqn", 0), ("fqf", 1)):
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        a.fqf = fqf
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

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "n_tau": bench.N_TAU, "n_tau_prime": bench.N_TAU_P, "n_quantile": bench.K_Q,
                      "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()}}))


if __name__ == "__main__":
    main()
