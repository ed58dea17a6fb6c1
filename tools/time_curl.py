"""Cost of CURL at the benchmark size (B = 512, A = 18, N = N' = 64, K = 32, random_shift = 4).  (1) One learner step
(prioritized sample, shifts, loss, backward, Adam, momentum update, priority update) replayed from its CUDA graph, for IQN
and C51 with and without CURL, in alternating rounds of 50 steps from one 2^18-transition replay each.  (2) The launches
of one eager step of each arm.  (3) The new kernels alone at B = 512 (riqn_curl_infonce_fwd_bwd, riqn_layernorm_fwd /
_bwd at widths 512 and 128, riqn_ema_f32 over the trunk and over the projection, riqn_add_f32 over the features,
riqn_colsum_add, and the 3136-wide products on the tensor cores: riqn_split_bf16 of the features and riqn_gemm_bf16_tc in
split-bf16 x3 mode for the forward, the weight gradient and the data gradient) on random operands.  Each kernel time is
the median of 5 replays of a CUDA graph of 200 launches between CUDA events, so no host call is in the timed window.
Prints one JSON line with the card's name, power limit and SM clocks."""
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

ARMS = (("iqn", {}), ("curl_iqn", dict(curl=1)), ("c51", dict(rainbow_only=1)), ("curl_c51", dict(rainbow_only=1, curl=1)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_us(B=bench.B, reps=200):
    dev = torch.device("cuda")
    p = _lib.ptr
    g = torch.Generator(device=dev).manual_seed(0)
    za, zk = (torch.randn(B, 128, device=dev, generator=g) for _ in range(2))
    w = torch.randn(128, 128, device=dev, generator=g) / 11.3
    rows, dz, dw = torch.empty(B, device=dev), torch.empty(B, 128, device=dev), torch.zeros(128, 128, device=dev)
    x512, y512 = torch.randn(B, 512, device=dev, generator=g), torch.empty(B, 512, device=dev)
    x128, y128 = torch.randn(B, 128, device=dev, generator=g), torch.empty(B, 128, device=dev)
    feat, feat2 = torch.randn(B, 3136, device=dev, generator=g), torch.randn(B, 3136, device=dev, generator=g)
    theta, xi = torch.randn(80000, device=dev, generator=g), torch.randn(80000, device=dev, generator=g)
    ptheta, pxi = torch.randn(1672000, device=dev, generator=g), torch.randn(1672000, device=dev, generator=g)
    gw, gb = torch.zeros(512, 3136, device=dev), torch.zeros(512, device=dev)
    bf = lambda *sh: torch.empty(*sh, dtype=torch.bfloat16, device=dev)
    x_hi, x_lo, x_hiT, x_loT = bf(B, 3136), bf(B, 3136), bf(3136, B), bf(3136, B)
    w_hi, w_lo, w_hiT, w_loT = bf(512, 3136), bf(512, 3136), bf(3136, 512), bf(3136, 512)
    d_hi, d_lo, d_hiT, d_loT = bf(B, 512), bf(B, 512), bf(512, B), bf(512, B)
    for src, r, c, ims in ((feat, B, 3136, (x_hi, x_lo, x_hiT, x_loT)), (gw, 512, 3136, (w_hi, w_lo, w_hiT, w_loT)),
                           (y512, B, 512, (d_hi, d_lo, d_hiT, d_loT))):
        _lib.call("riqn_split_bf16", r, c, p(src), *(p(t) for t in ims), 0)
    calls = {"infonce": lambda: _lib.call("riqn_curl_infonce_fwd_bwd", B, 128, p(za), p(zk), p(w), 1.0, p(rows), p(dz),
                                          p(dw), None),
             "layernorm_fwd_512": lambda: _lib.call("riqn_layernorm_fwd", B, 512, p(x512), p(gb), 1, p(y512)),
             "layernorm_bwd_512": lambda: _lib.call("riqn_layernorm_bwd", B, 512, p(x512), p(gb), p(x512), 1, p(y512)),
             "layernorm_fwd_128": lambda: _lib.call("riqn_layernorm_fwd", B, 128, p(x128), None, 0, p(y128)),
             "layernorm_bwd_128": lambda: _lib.call("riqn_layernorm_bwd", B, 128, p(x128), None, p(x128), 0, p(y128)),
             "ema_trunk": lambda: _lib.call("riqn_ema_f32", theta.numel(), p(theta), p(xi), 0.001),
             "ema_projection": lambda: _lib.call("riqn_ema_f32", ptheta.numel(), p(ptheta), p(pxi), 0.001),
             "colsum_512": lambda: _lib.call("riqn_colsum_add", B, 512, p(y512), p(gb)),
             "split_feat_bf16x2_with_transpose": lambda: _lib.call("riqn_split_bf16", B, 3136, p(feat), p(x_hi), p(x_lo),
                                                                   p(x_hiT), p(x_loT), 0),
             "gemm_tc_fwd_512x3136": lambda: _lib.call("riqn_gemm_bf16_tc", B, 512, 3136, p(x_hi), p(x_lo), p(w_hi),
                                                       p(w_lo), p(y512), 512, 0, None, None, None, 1, None, None, 0),
             "gemm_tc_wgrad_512x3136": lambda: _lib.call("riqn_gemm_bf16_tc", 512, 3136, B, p(d_hiT), p(d_loT), p(x_hiT),
                                                         p(x_loT), p(gw), 3136, 2, None, None, None, 1, None, None, 0),
             "gemm_tc_dgrad_512x3136": lambda: _lib.call("riqn_gemm_bf16_tc", B, 3136, 512, p(d_hi), p(d_lo), p(w_hiT),
                                                         p(w_loT), p(feat2), 3136, 0, None, None, None, 1, None, None, 0),
             "add_feat": lambda: _lib.call("riqn_add_f32", feat.numel(), p(feat), p(feat2), p(feat2)),
             "linear_wgrad_512x3136": lambda: _lib.call("riqn_linear_wgrad", B, 512, 3136, p(y512), p(feat), p(gw), p(gb)),
             "linear_fwd_512x3136": lambda: _lib.call("riqn_linear_fwd_ld", B, 3136, 512, p(feat), 3136, p(gw), p(gb),
                                                      p(y512), 512, 0),
             "linear_dgrad_512x3136": lambda: _lib.call("riqn_linear_dgrad_ld", B, 3136, 512, p(y512), 512, p(gw), p(feat2),
                                                        3136)}
    out = {}
    for name, fn in calls.items():
        fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(reps):
                fn()
        graph.replay()
        torch.cuda.synchronize()
        out[f"kernel_us_{name}"] = round(1e3 * float(np.median([timed(graph.replay, 1) / reps for _ in range(5)])), 2)
    return out


def main(cap=1 << 18, steps=50, rounds=5):
    dev = torch.device("cuda")
    arms = {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        a.random_shift = 4
        for k, v in fields.items():
            setattr(a, k, v)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        learner.learn_and_update(mem)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        learner.learn_and_update(mem)                    # one eager step: the library launches it makes
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
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "random_shift": 4,
                      "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **ker}))


if __name__ == "__main__":
    main()
