"""Cost of AdamW and the EMA target network (optim.py, target.py) at the benchmark size (B = 512, A = 18, N = N' = 64,
IQN).  Launches on the online DQN arena, from CUDA events around 200 launches each, in 5 alternating rounds:
riqn_adamw_step against riqn_adam_step, and riqn_ema_f32 into the target arena.  Beside each, the bytes it must move:
Adam and AdamW read theta, g, m, v and write theta, m, v (28 bytes per element), the EMA reads theta and xi and writes
xi (12).  Then the whole graph-replayed step (learn_and_update after enable_cuda_graph), plain, with target_ema, with
both switches, and SPR (random_shift = 4, K = 5) plain and with both, alternating.  Prints one JSON line with the card's
name, power limit and SM clocks, read in the same call."""
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

ARMS = (("iqn", {}), ("iqn_ema", dict(target_ema=1)), ("iqn_ema_adamw", dict(target_ema=1, adamw=1)),
        ("spr", dict(spr=1, random_shift=4)), ("spr_ema_adamw", dict(spr=1, random_shift=4, target_ema=1, adamw=1)))


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
    base = Learner(a, bench.ACTIONS, None)
    on, tg, opt = base.online_net, base.target_net, base.optimiser
    n = on._flat.numel()
    g = torch.randn(n, device=dev) * 1e-3
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    lr, eps = float(a.lr), float(a.adam_eps)
    launches = {
        "adam": lambda: call("riqn_adam_step", n, ptr(on._flat), ptr(g), ptr(m), ptr(v), 1, lr, 0.9, 0.999, eps, 1.0,
                             None),
        "adamw": lambda: call("riqn_adamw_step", n, ptr(on._flat), ptr(g), ptr(m), ptr(v), 1, lr, 0.9, 0.999, eps, 0.1,
                              1.0, None),
        "ema": lambda: call("riqn_ema_f32", n, ptr(on._flat), ptr(tg._flat), 0.005),
    }
    nbytes = {"adam": 28 * n, "adamw": 28 * n, "ema": 12 * n}
    for fn in launches.values():
        fn()
    torch.cuda.synchronize()
    launch_us = {k: [] for k in launches}
    for _ in range(rounds):
        for k, fn in launches.items():
            launch_us[k].append(timed(fn, reps))
    del base, opt
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
    for learner, _, _ in arms.values():
        learner.release_graphs()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    med = {k: float(np.median(t)) for k, t in launch_us.items()}
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      "arena_elements": n, **{f"{k}_bytes": b for k, b in nbytes.items()},
                      **{f"{k}_us": [round(t, 2) for t in ts] for k, ts in launch_us.items()},
                      **{f"{k}_median_us": round(t, 2) for k, t in med.items()},
                      **{f"{k}_GBps": round(nbytes[k] / (t * 1e3), 1) for k, t in med.items()},
                      **{f"launches_per_step_{k}": arm[2] for k, arm in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in ts] for k, ts in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(ts)), 4) for k, ts in step_ms.items()}}))


if __name__ == "__main__":
    main()
