"""Cost of random-shift augmentation at the benchmark size (B=512): one learner step (prioritized sample, shift draw and
shift, loss, backward, Adam, priority update) replayed from its CUDA graph, for IQN (N=N'=64, K=32) and C51 (51 atoms),
each with random_shift 0 and 4, in alternating rounds of 50 steps from one 2^18-transition replay each; and
riqn_random_shift alone on the learner's operands (s_{t+n} and s_t as views of a replay window, 2B = 1024 uint8 images),
timed over many launches with CUDA events, with the bytes it must move (read and write the 2B C H W pixels once).
Prints one JSON line with the card's name and power limit."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib, augment  # noqa: E402

ARMS = (("iqn", {}), ("iqn_shift4", dict(random_shift=4)), ("c51", dict(rainbow_only=1)),
        ("c51_shift4", dict(rainbow_only=1, random_shift=4)))
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_us(B=512, n_step=3, reps=2000):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    win = torch.randint(0, 256, (B, 4 + n_step, 84, 84), dtype=torch.uint8, device=dev, generator=g)
    shifts = torch.randint(-4, 5, (2 * B, 2), dtype=torch.int32, device=dev, generator=g)
    nx, st = win[:, n_step:n_step + 4], win[:, :4]
    for _ in range(20):
        augment.random_shift(nx, st, shifts)
    out = torch.empty(2 * B, 4, 84, 84, dtype=torch.uint8, device=dev)
    args = (B, 4, 84, 84, nx.data_ptr(), nx.stride(0), st.data_ptr(), st.stride(0), 1, shifts.data_ptr(), out.data_ptr())
    ms = timed(lambda: _lib.call("riqn_random_shift", *args), reps)
    moved = 2 * out.numel()                                 # bytes read + bytes written
    return ms * 1e3, moved


def main(cap=1 << 18, steps=50, rounds=5):
    dev = torch.device("cuda")
    arms = {}
    for name, fields in ARMS:
        torch.manual_seed(0)
        a = bench.make_args(dev, cap)
        for k, v in fields.items():
            setattr(a, k, v)
        learner = Learner(a, bench.ACTIONS, None)
        learner.train()
        mem = ReplayMemory(a, None)
        bench.fill_replay(mem, cap, dev, 7)
        learner.learn_and_update(mem)
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
    us, moved = kernel_us()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    med = {k: float(np.median(v)) for k, v in step_ms.items()}
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(m, 4) for k, m in med.items()},
                      "shift_cost_iqn": round(med["iqn_shift4"] / med["iqn"] - 1, 4),
                      "shift_cost_c51": round(med["c51_shift4"] / med["c51"] - 1, 4),
                      "random_shift_us": round(us, 2), "random_shift_bytes": moved,
                      "random_shift_bytes_per_s": round(moved / (us * 1e-6), -9),
                      "random_shift_share_of_hbm_peak": round(moved / (us * 1e-6) / HBM_BYTES_PER_S, 3)}))


if __name__ == "__main__":
    main()
