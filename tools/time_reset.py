"""Cost of one periodic network reset (reset.py) at the benchmark size (B = 512, A = 18, N = N' = 64, IQN), without and
with SPR (random_shift = 4, K = 5).  Per arena: the riqn_arena_reset launch alone, from CUDA events around 200 launches
(a reset rewrites the same segments each time, so every launch does the same work), in 5 alternating rounds; and the
whole Learner.reset_networks() (every arena's launch, the optimiser restarts and the recomposed online weights), timed
the same way.  Beside each launch, the bytes it must move: every segment element written, the kept share of each
shrink-and-perturb segment read, and both moment arenas written.  Prints one JSON line with the card's name, power limit
and SM clocks."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rainbow_iqn_apex_b200 import Learner, reset  # noqa: E402

ARMS = (("iqn", {}), ("spr_iqn", dict(spr=1, random_shift=4)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps          # microseconds


def main(reps=200, rounds=5):
    dev = torch.device("cuda")
    jobs, out = {}, {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, 1 << 12)
        a.reset = 1
        for k, v in fields.items():
            setattr(a, k, v)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        seed = learner.online_net._rng_seed ^ reset.RESET_SEED
        for k, net, opt, segs in reset.tables(learner):
            arena = reset.ARENAS[k]
            n = net._flat.numel()
            written = sum(e - b for b, e, *_ in segs)
            kept = sum(e - b for b, e, _, _, alpha in segs if alpha != 0.0)
            out[f"{name}_{arena}_elements"] = n
            out[f"{name}_{arena}_bytes"] = 4 * (written + kept) + 8 * n
            jobs[f"{name}_{arena}"] = (lambda net=net, opt=opt, segs=segs, k=k:
                                      reset.reset_arena(net, opt, segs, seed, k))
        jobs[f"{name}_reset_networks"] = learner.reset_networks
    for fn in jobs.values():                            # warm-up: module load, first launches
        fn()
    torch.cuda.synchronize()
    us = {k: [] for k in jobs}
    for _ in range(rounds):
        for k, fn in jobs.items():
            us[k].append(timed(fn, reps))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    med = {k: float(np.median(v)) for k, v in us.items()}
    print(json.dumps({"batch": bench.B, "gpu": q[0] if q else torch.cuda.get_device_name(), **out,
                      **{f"{k}_us": [round(t, 2) for t in v] for k, v in us.items()},
                      **{f"{k}_median_us": round(t, 2) for k, t in med.items()},
                      **{f"{k}_GBps": round(out[f"{k}_bytes"] / (med[k] * 1e3), 1) for k in med if f"{k}_bytes" in out}}))


if __name__ == "__main__":
    main()
