"""Cost of QR-DQN at the benchmark size (B=512): one learner step (prioritized sample, loss, backward, Adam, priority
update) replayed from its CUDA graph, for IQN (N=N'=64, K=32), C51 (51 atoms), QR-DQN at N=64 and QR-DQN at N=200, in
alternating rounds of 50 steps from one 2^18-transition replay each.  QR-DQN's head runs on B rows like C51's (z-layers of
width N and A*N), IQN's on N*B rows.  Also the share of the step that the fp32 SIMT z-layer products take
(riqn_linear_fwd_ld, riqn_linear_dgrad_ld, riqn_noisy_wgrad_ld) take, each call of one eager step timed on its own.
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

Z_LAYER_OPS = ("riqn_linear_fwd_ld", "riqn_linear_dgrad_ld", "riqn_noisy_wgrad_ld")
ARMS = (("iqn", {}), ("c51", dict(rainbow_only=1)), ("qr64", dict(qr_dqn=1, num_tau_samples=64)),
        ("qr200", dict(qr_dqn=1, num_tau_samples=200)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def z_layer_ms(learner, mem, reps=20):
    """Device time per step of the fp32 SIMT z-layer products: the calls one eager step makes, each replayed ``reps``
    times between CUDA events on the operands it was given.  Run last: the replays write into buffers the step has
    released."""
    timers = _lib.time_entry_points(Z_LAYER_OPS)
    try:
        learner.learn_and_update(mem)
    finally:
        _lib.time_entry_points(None)
    torch.cuda.synchronize()
    calls = [(name, args) for name, v in timers.items() for _, _, args in v]
    return sum(timed(lambda: _lib.call(name, *args), reps) for name, args in calls)


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
    z_ms = {}
    for name, (learner, mem, _) in arms.items():
        learner.release_graphs()
        if name != "iqn":
            z_ms[name] = z_layer_ms(learner, mem)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **{f"z_layer_ms_{k}": round(z, 4) for k, z in z_ms.items()},
                      **{f"z_layer_share_{k}": round(z / float(np.median(step_ms[k])), 4) for k, z in z_ms.items()}}))


if __name__ == "__main__":
    main()
