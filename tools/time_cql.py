"""Cost of CQL at the benchmark size (B = 512, A = 18).  (1) One learner step (prioritized sample, loss, backward, Adam,
priority update) replayed from its CUDA graph, for IQN, CQL-IQN, and QR-DQN and CQL-QR-DQN at N = 64 and 200, in
alternating rounds of 50 steps from one 2^18-transition replay each.  (2) The kernels alone against the quantile-Huber
loss riqn_iqn_loss_fwd_bwd: riqn_cql_loss_fwd_bwd and riqn_cql_dense_grad at N = N' = 64 and 200, on random operands,
each the median of 5 blocks of 200 launches between CUDA events.  Prints one JSON line with the card's name, power limit
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
from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib  # noqa: E402

ARMS = (("iqn", {}), ("cql_iqn", dict(cql=1)),
        ("qr64", dict(qr_dqn=1)), ("cql_qr64", dict(qr_dqn=1, cql=1)),
        ("qr200", dict(qr_dqn=1, num_tau_samples=200)), ("cql_qr200", dict(qr_dqn=1, num_tau_samples=200, cql=1)))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_us(B=bench.B, A=bench.ACTIONS, reps=200):
    """Microseconds per launch of the quantile-Huber loss, the CQL loss and the dense gradient (median of 5 blocks)."""
    dev = torch.device("cuda")
    out = {}
    p = _lib.ptr
    for N in (64, 200):
        g = torch.Generator(device=dev).manual_seed(N)
        q_on, q_tg = (torch.randn(N * B, A, device=dev, generator=g) for _ in range(2))
        tau = torch.rand(N * B, device=dev, generator=g)
        acts, ast = (torch.randint(0, A, (B,), device=dev, generator=g) for _ in range(2))
        R, nt, gs = 3 * torch.randn(B, device=dev, generator=g), torch.ones(B, device=dev), torch.rand(B, device=dev)
        loss, td, pi, dth = (torch.empty(B, device=dev), torch.empty(B, device=dev), torch.empty(B, A, device=dev),
                             torch.empty(N * B, device=dev))
        G = torch.empty(N * B, A, device=dev)
        ops = (p(q_on), p(q_tg), p(tau), p(acts), p(ast), p(R), p(nt), 0.97, 1.0)
        calls = {"iqn_loss": lambda: _lib.call("riqn_iqn_loss_fwd_bwd", B, N, N, A, *ops, p(loss), p(dth), None, None),
                 "cql_loss": lambda: _lib.call("riqn_cql_loss_fwd_bwd", B, N, N, A, *ops, 1.0, p(loss), p(td), p(pi),
                                               p(dth), None, None, None),
                 "cql_dense_grad": lambda: _lib.call("riqn_cql_dense_grad", B, N, A, p(dth), p(pi), p(acts), p(gs),
                                                     1.0 / B, 1.0, p(G))}
        for name, fn in calls.items():
            timed(fn, 20)
            out[f"kernel_us_{name}_n{N}"] = round(1e3 * float(np.median([timed(fn, reps) for _ in range(5)])), 2)
    return out


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
    for learner, _, _ in arms.values():
        learner.release_graphs()
    ker = kernel_us()

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": bench.B, "replay_capacity": cap, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"launches_per_step_{k}": v[2] for k, v in arms.items()},
                      **{f"step_ms_{k}": [round(t, 4) for t in v] for k, v in step_ms.items()},
                      **{f"step_median_ms_{k}": round(float(np.median(v)), 4) for k, v in step_ms.items()},
                      **ker}))


if __name__ == "__main__":
    main()
