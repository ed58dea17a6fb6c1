"""Device time of the NoisyLinear head's products through their entry points, at the learner's shapes (B=512,
N=N'=64, K=32): the no-grad forward (R=16384, fp16 operands, bias+ReLU into fp32 h), the gradient-pass forward
(R=32768, plus the bf16 image h_hi), the data gradient (32768x3136x1024, MN-major weight, bf16 dx) and the weight
gradient (1024x3136x32768, both operands MN-major, dmu / dsigma accumulated).  CUDA events around --reps back-to-back
launches after --warmup, --rounds times; prints one JSON line per product with the median and the range.

    python tools/time_head_gemm.py [--root TREE] [--reps 30] [--rounds 5]

--root imports the package from another checkout (built in place), so two builds can be timed in one session."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from rainbow_iqn_apex_b200._lib import call, ptr, require_device  # noqa: E402

require_device()
dev = torch.device("cuda")
FEAT, HID2 = 3136, 1024
gen = torch.Generator(device=dev).manual_seed(0)


def rnd(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, generator=gen, device=dev) * scale).to(dtype)


def forward(R, image):
    x, w, bias = rnd(R, FEAT, dtype=torch.float16), rnd(HID2, FEAT, scale=0.02, dtype=torch.float16), rnd(HID2, dtype=torch.float32)
    h = torch.empty(R, HID2, device=dev)
    h_hi = torch.empty(R, HID2, dtype=torch.bfloat16, device=dev) if image else None
    return (2.0 * R * HID2 * FEAT, lambda: call("riqn_gemm_bf16_tc", R, HID2, FEAT, ptr(x), None, ptr(w), None, ptr(h), HID2, 1,
                                                ptr(bias), None, None, 1, None, ptr(h_hi), 3))


def dgrad(R):
    dh, w = rnd(R, HID2), rnd(HID2, FEAT, scale=0.02)
    dx = torch.empty(R, FEAT, dtype=torch.bfloat16, device=dev)
    return (2.0 * R * FEAT * HID2, lambda: call("riqn_gemm_bf16_tc_mn", R, FEAT, HID2, ptr(dh), ptr(w), 0, None, FEAT, 0, None,
                                                None, 1.0, 1, ptr(dx), 0))


def wgrad(R):
    dh, x = rnd(R, HID2, scale=0.01), rnd(R, FEAT)
    mu, sigma, eps = torch.zeros(HID2, FEAT, device=dev), torch.zeros(HID2, FEAT, device=dev), rnd(HID2, FEAT, dtype=torch.float32)
    return (2.0 * R * FEAT * HID2, lambda: call("riqn_gemm_bf16_tc_mn", HID2, FEAT, R, ptr(dh), ptr(x), 1, ptr(mu), FEAT, 3,
                                                ptr(sigma), ptr(eps), 1.0, 4, None, 0))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


cases = {"forward R=16384": forward(16384, False), "forward R=32768 +h_hi": forward(32768, True),
         "dgrad 32768x3136x1024 bf16": dgrad(32768), "wgrad 1024x3136x32768": wgrad(32768)}
info = gpu_info()
for name, (flop, fn) in cases.items():
    for _ in range(args.warmup):
        fn()
    times = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / args.reps)
    times.sort()
    us = times[len(times) // 2]
    print(json.dumps({"product": name, "us_median": round(us, 1), "us_range": [round(times[0], 1), round(times[-1], 1)],
                      "tflops": round(flop / us / 1e6, 1), "root": os.path.abspath(args.root), "gpu": info}), flush=True)
