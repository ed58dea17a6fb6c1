"""Gradient pass of one IQN learner step at the benchmark size (B=512, N=N'=64, K=32), two ways, alternating:
  fused     Learner.compute_gradients: three forwards + the fused loss kernel + the one-hot head backward
  autograd  the same loss written with net(...) calls and torch ops (oracle.losses.iqn_pairwise_loss), then
            (w * loss).mean().backward() through DQN.forward's autograd node and the dense head backward
Device time per step from CUDA events; prints one JSON line with the card's name and power limit."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import make_args  # noqa: E402
from oracle import cases, losses  # noqa: E402
from rainbow_iqn_apex_b200 import Learner  # noqa: E402

B, N, NP, K, A = 512, 64, 64, 32, 18


def autograd_step(lr, st, ac, rt, nx, nt, w):
    on, tg = lr.online_net, lr.target_net
    on.reset_noise()
    with torch.no_grad():
        q_sel, _ = on(nx, K)
        a_star = q_sel.view(K, B, A).mean(0).argmax(1)
        tg.reset_noise()
        q_tgt, _ = tg(nx, NP)
        target = (rt[:, None].repeat(NP, 1) + lr.discount ** lr.n * nt[:, None].repeat(NP, 1)
                  * q_tgt.gather(1, a_star[:, None].repeat(NP, 1))).view(NP, B).t()
    on.reset_noise()
    q, tau = on(st, N)
    theta = q.gather(1, ac[:, None].repeat(N, 1)).view(N, B).t()
    loss = losses.iqn_pairwise_loss(theta, target, tau.view(N, B).t(), lr.kappa)
    on.zero_grad()
    (w * loss).mean().backward()
    return loss


def main(reps=30, rounds=4):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    lr = Learner(make_args(dev, B, cases.iqn_cfg(N, NP, K)), A, None)
    lr.train()
    b = cases.make_batch(1, B)
    st, nx = torch.from_numpy(b["states"]).to(dev), torch.from_numpy(b["next_states"]).to(dev)
    ac, rt = torch.from_numpy(b["actions"]).to(dev), torch.from_numpy(b["returns"]).to(dev)
    nt, w = torch.from_numpy(b["nonterminals"]).to(dev), torch.from_numpy(b["weights"]).to(dev)
    arms = {"fused": lambda: lr.compute_gradients(st, ac, rt, nx, nt, w),
            "autograd": lambda: autograd_step(lr, st, ac, rt, nx, nt, w)}
    times = {k: [] for k in arms}
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / reps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": B, "n_tau": N, "gpu": q[0] if q else torch.cuda.get_device_name(),
                      **{f"{k}_ms_per_step": [round(t, 3) for t in v] for k, v in times.items()},
                      **{f"{k}_median_ms": round(float(np.median(v)), 3) for k, v in times.items()}}))


if __name__ == "__main__":
    main()
