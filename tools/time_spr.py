"""Cost of SPR at the benchmark size (B = 512, A = 18, N = N' = 64, random_shift = 4, K = 5).  (1) One learner step
(prioritized sample, sequence gather, shifts, target trunk pass over the K*B shifted states, loss, backward through the
transition model, Adam, priority update) replayed from its CUDA graph, for IQN and C51 with and without SPR, in
alternating rounds of 50 steps from one 2^18-transition replay each.  (2) The launches of one eager step of each arm.
(3) Per entry point, the summed device time of its calls in one eager SPR step (CUDA events around every call,
_lib.time_entry_points), median of 5 steps.  Prints one JSON line with the card's name, power limit and SM clocks."""
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

ARMS = (("iqn", {}), ("spr_iqn", dict(spr=1)), ("c51", dict(rainbow_only=1)), ("spr_c51", dict(rainbow_only=1, spr=1)))
ENTRY_POINTS = ("riqn_sequence_gather", "riqn_random_shift", "riqn_s2d_u8", "riqn_conv_fwd_strip", "riqn_conv_bwd_strip",
                "riqn_spr_pack", "riqn_spr_unpack_grad", "riqn_spr_weight_images", "riqn_spr_weight_grad_add",
                "riqn_spr_cosine_fwd_bwd", "riqn_split_bf16", "riqn_gemm_bf16_tc", "riqn_layernorm_fwd",
                "riqn_layernorm_bwd", "riqn_linear_fwd_ld", "riqn_linear_wgrad", "riqn_linear_dgrad_ld", "riqn_colsum_add")


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def entry_point_ms(learner, mem, steps=5):
    """Summed event time per entry point over one eager step, median over ``steps`` steps (a profiling run of its own:
    the events add host work, so these steps are not the timed ones)."""
    per = {n: [] for n in ENTRY_POINTS}
    for _ in range(steps):
        timers = _lib.time_entry_points(ENTRY_POINTS)
        learner.learn_and_update(mem)
        torch.cuda.synchronize()
        for n, evs in timers.items():
            per[n].append(sum(e0.elapsed_time(e1) for e0, e1, _ in evs))
        _lib.time_entry_points(None)
    return {f"eager_spr_step_ms_{n}": round(float(np.median(v)), 4) for n, v in per.items() if any(v)}


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
        prof = entry_point_ms(learner, mem) if fields.get("spr") else {}
        learner.enable_cuda_graph(mem)
        for _ in range(5):
            learner.learn_and_update(mem)
        arms[name] = (learner, mem, launches, prof)
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (learner, mem, _, _) in arms.items():
            step_ms[name].append(timed(lambda: learner.learn_and_update(mem), steps))
    for learner, _, _, _ in arms.values():
        learner.release_graphs()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "random_shift": 4, "spr_steps": 5,
                      "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **{f"{k}_{n}": t for k, v in arms.items() for n, t in v[3].items()}}))


if __name__ == "__main__":
    main()
