"""Oracle (test infrastructure): SPR (Schwarzer et al., ICLR 2021) as this project states it
(rainbow_iqn_apex_b200/spr.py), written from the paper: the K-step sequence gather in numpy on top of replay.py's rules,
and the transition model, projection, predictor and masked cosine loss in torch on the CPU, composed with
``losses.learn_step``.

  z_0 = f(s_t) ,  z_k = ReLU(conv2(ReLU(conv1([z_{k-1} ; onehot(a_{t+k-1})]))))  (3x3, padding 1)
  y_k = q(g(z_k)) ,  t_k = g(f(s'_{t+k})) (no gradient) ,  g(feat) = LN(W_c ReLU(LN(W_h feat + b_h)) + b_c)
  L_SPR = (1/B) sum_b sum_k valid_{b,k} (-cos(y_{b,k}, t_{b,k}))  (F.normalize, eps 1e-12)
  objective (1/B) sum_b w_b L_RL,b + lambda L_SPR
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import losses, network as net
from .curl import project

NAMES = ("weight_h", "bias_h", "weight_c", "bias_c", "conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias",
         "weight_q", "bias_q")


def sequence(store, data_indexes, heads, history=4, K=5):
    """The sequence gather over a replay.ReplayStore: (window u8 (B, history+K, 84, 84), actions i64 (B, K), valid u8
    (B, K)).  The window's slots and blank frames are replay.ReplayStore.assemble's at n_step = K; valid[b, k-1] needs
    the last frame of s_{t+k} not blank and the walk p+1 .. p+k not to reach the segment's write head ``heads[actor]``."""
    cap = store.actor_capacity
    wins, acts, vals = [], [], []
    for d in data_indexes:
        d = int(d)
        slots = store.window_slots(d, history, K)
        ts = [int(store.timestep[s]) for s in slots]
        nt = [bool(store.nonterminal[s]) for s in slots]
        blank = [False] * len(slots)
        for t in range(history - 2, -1, -1):
            if ts[t + 1] == 0:
                ts[t], nt[t], blank[t] = 0, False, True
        for t in range(history, history + K):
            if not nt[t - 1]:
                ts[t], nt[t], blank[t] = 0, False, True
        wins.append(np.stack([np.zeros((84, 84), np.uint8) if b else store.frame[s] for s, b in zip(slots, blank)]))
        acts.append([int(store.action[slots[history - 1 + k]]) for k in range(K)])
        dist = (int(heads[d // cap]) - d % cap) % cap
        vals.append([int(not blank[history - 1 + k] and not 1 <= dist <= k) for k in range(1, K + 1)])
    return np.stack(wins), np.array(acts, np.int64), np.array(vals, np.uint8)


def transition(p, z, a, num_actions):
    """T(z, a) for z (B, 64, 7, 7) and actions a (B,)."""
    B, _, H, W = z.shape
    planes = F.one_hot(a, num_actions).to(z.dtype)[:, :, None, None].expand(B, num_actions, H, W)
    h = torch.relu(F.conv2d(torch.cat([z, planes], 1), p["conv1.weight"], p["conv1.bias"], padding=1))
    return torch.relu(F.conv2d(h, p["conv2.weight"], p["conv2.bias"], padding=1))


def spr_loss(p_online, sp, x, actions, valid, x_targets, num_actions, keep=None):
    """(per-sample terms (B,), whose mean is L_SPR; predictions (K*B, 128); targets (K*B, 128)).  ``x``: the learner's
    shifted s_t (B, 4, 84, 84) fp32 / 255; ``x_targets``: the shifted s_{t+1} .. s_{t+K} stacked step-major (K*B, ...);
    ``actions`` (B, K) int64, ``valid`` (B, K)."""
    B, K = actions.shape
    z = net.conv_trunk(p_online, x).reshape(B, 64, 7, 7)
    if keep is not None:
        keep["z0"] = z
    zs = []
    for k in range(K):
        z = transition(sp, z, actions[:, k], num_actions)
        zs.append(z)
    y = F.linear(project(sp, torch.stack(zs).reshape(K * B, -1)), sp["weight_q"], sp["bias_q"])
    with torch.no_grad():
        t = project({k: v.detach() for k, v in sp.items()},
                    net.conv_trunk({k: v.detach() for k, v in p_online.items()}, x_targets))
    cos = (F.normalize(y, dim=1, eps=1e-12) * F.normalize(t, dim=1, eps=1e-12)).sum(1).reshape(K, B)
    rows = -(torch.as_tensor(valid, dtype=y.dtype).t() * cos).sum(0)
    return rows, y, t


class _Recorder:
    """A stand-in optimiser for losses.learn_step: keeps the RL gradients, steps nothing."""

    def step(self, params, grads):
        self.grads = grads


def learn_step(p_online, p_target, adam, batch, weights, noises, taus, cfg, sp, spr_adam, actions, valid, x_targets,
               num_actions, coef, rainbow_only=False, keep=None):
    """Learner.compute_gradients + apply_gradients of an SPR learner.  ``batch``: the shifted frames as losses.learn_step
    takes them; ``sp``: leaf tensors with requires_grad (NAMES), stepped by ``spr_adam``.  Returns (RL loss (B,), online
    grads, SPR grads, dict(rows, y, t))."""
    rec = _Recorder()
    loss, _ = losses.learn_step(p_online, p_target, rec, batch, weights, noises, taus, cfg, rainbow_only=rainbow_only,
                                keep=keep)
    for t in sp.values():
        t.grad = None
    rows, y, t = spr_loss(p_online, sp, batch[0], actions, valid, x_targets, num_actions)
    (coef * rows.mean()).backward()               # adds onto the RL gradients left in the online parameters' .grad
    grads = {k: v.grad.detach().clone() for k, v in p_online.items() if v.requires_grad and v.grad is not None}
    sgrads = {k: sp[k].grad.detach().clone() for k in NAMES}
    adam.step(p_online, grads)
    spr_adam.step(sp, sgrads)
    return loss, grads, sgrads, dict(rows=rows.detach(), y=y.detach(), t=t)
