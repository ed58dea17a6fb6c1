"""Cost of update-horizon and discount annealing (horizon.py) at the benchmark size (B = 512, A = 18, N = N' = 64, IQN).
The gathers from CUDA events around 200 launches each, in 5 alternating rounds: riqn_frame_gather_horizon against
riqn_frame_gather at n in {3, 10}, with the frame bytes each writes (the horizon gather writes 2 * history = 8 frames per
sample, the fixed one history + n).  Then the graph-replayed step (learn_and_update after enable_cuda_graph), annealing
off and on (BBF's schedule, which stays near n = 10 over the timed steps), alternating.  Prints one JSON line with the
card's name, power limit and SM clocks, read in the same call."""
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
from rainbow_iqn_apex_b200._lib import call, ptr  # noqa: E402
from rainbow_iqn_apex_b200.dynstate import HorizonState  # noqa: E402

FRAME = 84 * 84
ARMS = (("fixed", {}), ("anneal", dict(horizon_anneal=1)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps          # microseconds


def main(cap=1 << 18, reps=200, steps=50, rounds=5):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    a = bench.make_args(dev, cap)
    B, h = bench.B, a.history_length
    mem = ReplayMemory(a, None)
    bench.fill_replay(mem, cap, dev, 7)
    tr = mem.transitions
    di = torch.randint(0, cap, (B,), device=dev)
    act, ret, nt, disc = (torch.empty(B, dtype=dt, device=dev) for dt in (torch.int64, torch.float32, torch.float32,
                                                                           torch.float32))
    frames = torch.empty(B, 2 * h, 84, 84, dtype=torch.uint8, device=dev)
    stores = (ptr(tr.frames), ptr(tr.timestep), ptr(tr.action), ptr(tr.reward), ptr(tr.nonterminal))
    launches, nbytes = {}, {}
    for n in (3, 10):
        gp = torch.tensor([a.discount ** k for k in range(n)], dtype=torch.float64, device=dev)
        win = torch.empty(B, h + n, 84, 84, dtype=torch.uint8, device=dev)
        hz = HorizonState(dev, 10)
        hz.write(n, a.discount)
        launches[f"gather_n{n}"] = (lambda n=n, gp=gp, win=win: call(
            "riqn_frame_gather", B, tr.actor_capacity, h, n, ptr(di), *stores, ptr(gp), ptr(win), ptr(act), ptr(ret),
            ptr(nt)))
        launches[f"gather_horizon_n{n}"] = (lambda hz=hz: call(
            "riqn_frame_gather_horizon", B, tr.actor_capacity, h, 10, ptr(di), *stores, hz.ptr(), ptr(frames), ptr(act),
            ptr(ret), ptr(nt), ptr(disc)))
        nbytes[f"gather_n{n}"] = B * (h + n) * FRAME
        nbytes[f"gather_horizon_n{n}"] = B * 2 * h * FRAME
    for fn in launches.values():
        fn()
    torch.cuda.synchronize()
    launch_us = {k: [] for k in launches}
    for _ in range(rounds):
        for k, fn in launches.items():
            launch_us[k].append(timed(fn, reps))
    del mem, tr
    arms = {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        for k, val in fields.items():
            setattr(a, k, val)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        learner.learn_and_update(mem)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        learner.learn_and_update(mem)                    # one eager step: the library launches it makes
        count = _lib.launch_count() - c0
        learner.enable_cuda_graph(mem)
        for _ in range(5):
            learner.learn_and_update(mem)
        arms[name] = (learner, mem, count)
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (learner, mem, _) in arms.items():
            step_ms[name].append(timed(lambda: learner.learn_and_update(mem), steps) / 1e3)
    horizon_end = arms["anneal"][0].horizon()
    for learner, _, _ in arms.values():
        learner.release_graphs()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    med = {k: float(np.median(t)) for k, t in launch_us.items()}
    print(json.dumps({"batch": B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"{k}_frame_bytes": b for k, b in nbytes.items()},
                      **{f"{k}_us": [round(t, 2) for t in ts] for k, ts in launch_us.items()},
                      **{f"{k}_median_us": round(t, 2) for k, t in med.items()},
                      **{f"launches_per_step_{k}": arm[2] for k, arm in arms.items()},
                      "anneal_horizon_after_timing": list(horizon_end),
                      **{f"step_ms_{k}": [round(t, 4) for t in ts] for k, ts in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(ts)), 4) for k, ts in step_ms.items()}}))


if __name__ == "__main__":
    main()
