"""Cost of value rescaling (the transformed Bellman operator) at the benchmark size (B=512, N=N'=64, K=32; C51 with 51
atoms): one learner step (prioritized sample, loss, backward, Adam, priority update) replayed from its CUDA graph, for
IQN against rescaled IQN and C51 against rescaled C51, in alternating rounds of 50 steps.  The rescaled step swaps the
argmax and loss kernels for their _h twins (the same launch count): a few double-precision square roots per target value
(B*N' = 32 768 for IQN) and per K-pass element.  Device time from CUDA events; prints one JSON line with the card's name
and power limit."""
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
    for name, rainbow_only, rescale in (("iqn", False, 0), ("iqn_h", False, 1), ("c51", True, 0), ("c51_h", True, 1)):
        torch.manual_seed(0)
        a = bench.make_args(dev, cap, rainbow_only=rainbow_only)
        if rainbow_only:
            a.lr, a.adam_eps = 6.25e-5, 1.5e-4                     # bench.c51_leg
        a.value_rescaling = rescale
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
