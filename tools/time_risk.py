"""Cost of risk-sensitive action selection at the benchmark size (B=512, N=N'=64, K=32).
  step    one learner step (prioritized sample, loss, backward, Adam, priority update) replayed from its CUDA graph, for a
          risk-neutral learner and a CVaR(0.25) learner, in alternating blocks
  kernel  the K-pass draw alone at n = K*B = 16384: riqn_fill_uniform against riqn_fill_tau_distorted (CVaR, Wang)
Device time from CUDA events; prints one JSON line with the card's name and power limit."""
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
from rainbow_iqn_apex_b200.model import RISK_MEASURES  # noqa: E402


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main(cap=1 << 18, steps=50, rounds=5, kernel_reps=2000):
    dev = torch.device("cuda")
    arms = {}
    for name, risk in (("neutral", None), ("cvar0.25", ("cvar", 0.25))):
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        if risk is not None:
            a.risk_measure, a.risk_eta = risk
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        learner.enable_cuda_graph(mem)
        for _ in range(5):
            learner.learn_and_update(mem)
        arms[name] = (learner, mem)
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (learner, mem) in arms.items():
            step_ms[name].append(timed(lambda: learner.learn_and_update(mem), steps))

    n = bench.K_Q * bench.B
    out = torch.empty(n, device=dev)
    seed = 12345
    kern = {"fill_uniform": lambda: _lib.call("riqn_fill_uniform", n, seed, 1, _lib.ptr(out), None),
            "distorted_cvar0.25": lambda: _lib.call("riqn_fill_tau_distorted", n, seed, 1, RISK_MEASURES["cvar"], 0.25,
                                                    _lib.ptr(out), None),
            "distorted_wang-0.75": lambda: _lib.call("riqn_fill_tau_distorted", n, seed, 1, RISK_MEASURES["wang"], -0.75,
                                                     _lib.ptr(out), None)}
    kern_us = {k: [] for k in kern}
    for fn in kern.values():
        timed(fn, 100)
    for _ in range(rounds):
        for name, fn in kern.items():
            kern_us[name].append(1e3 * timed(fn, kernel_reps))

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "n_tau": bench.N_TAU, "n_quantile": bench.K_Q, "replay_capacity": cap,
                      "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **{f"kernel_us_{k}": [round(t, 2) for t in v] for k, v in kern_us.items()},
                      **{f"kernel_median_us_{k}": round(float(np.median(v)), 2) for k, v in kern_us.items()}}))


if __name__ == "__main__":
    main()
