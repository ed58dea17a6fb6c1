"""Microbenchmark of riqn_quantile_embed_fwd_tc (the embedding producer): CUDA-event time per launch and achieved GB/s on the
algorithmic bytes of SURVEY 8d for the three launch shapes of a learner step (fp16 mode: K=32 one image, N'=64 one image,
N=64 two images) and the bf16 hi + lo mode.  Each case runs --rounds rounds of --reps back-to-back launches after
--warmup, rotating between two output sets larger than L2; prints one JSON line per case with the median and the range.

    python tools/time_embed.py [--root TREE] [--reps 200] [--rounds 5]

--root imports the package from another checkout (built in place), so two builds can be timed in one session."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--reps", type=int, default=200)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from rainbow_iqn_apex_b200._lib import call, ptr, require_device  # noqa: E402

require_device()
dev = torch.device("cuda")
B, E, F = 512, 64, 3136
PEAK_GBS = 3350.0      # H100 SXM data sheet, HBM3


def bf(*s):
    return torch.empty(*s, device=dev, dtype=torch.bfloat16)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def run(nq, images, fp16):
    R = B * nq
    tau = torch.rand(R, device=dev)
    feat = torch.rand(B, F, device=dev)
    w = torch.randn(F, E, device=dev) * 0.1
    w_hi = w.to(torch.bfloat16)
    w_lo = (w - w_hi.float()).to(torch.bfloat16)
    bias = torch.randn(F, device=dev) * 0.1
    cos_hi, cos_lo = bf(R, E), bf(R, E)
    sets = [(bf(R, F), bf(R, F) if images == 2 else None) for _ in range(2)]       # rotate outputs (> L2)

    def go(i):
        x_hi, x_lo = sets[i & 1]
        call("riqn_quantile_embed_fwd_tc", B, nq, E, F, ptr(tau), ptr(feat), ptr(w_hi), ptr(w_lo), ptr(bias), ptr(cos_hi),
             ptr(cos_lo), None, None, ptr(x_hi), ptr(x_lo), None, None, 1 if fp16 else 0)
    for i in range(args.warmup):
        go(i)
    times = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.reps):
            go(i)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / args.reps)
    times.sort()
    us = times[len(times) // 2]
    nbytes = 2.0 * images * R * F + 4.0 * R + 4.0 * B * F + 4.0 * (E * F + F)
    print(json.dumps({"case": f"nq={nq} images={images} {'fp16' if fp16 else 'bf16 hi/lo'}", "us_median": round(us, 1),
                      "us_range": [round(times[0], 1), round(times[-1], 1)], "note": "cos kernel included",
                      "algorithmic_mb": round(nbytes / 1e6), "gbs": round(nbytes / us / 1e3),
                      "frac_of_3350_gbs": round(nbytes / us / 1e3 / PEAK_GBS, 3), "root": os.path.abspath(args.root),
                      "gpu": info}), flush=True)


info = gpu_info()
run(32, 1, True)
run(64, 1, True)
run(64, 2, True)
run(64, 2, False)
