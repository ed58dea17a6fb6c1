"""Oracle (test infrastructure): BBF's update rule as this project states it (rainbow_iqn_apex_b200/optim.py, target.py):
AdamW's decoupled weight decay and the EMA (Polyak) target network, written from torch.optim.AdamW's documented update and
the BBF paper (Schwarzer et al., ICML 2023).

  AdamW (non-amsgrad), step t, lr, lambda:   theta <- theta * (1 - lr lambda)
                                             m <- b1 m + (1 - b1) g ,  v <- b2 v + (1 - b2) g^2
                                             theta <- theta - lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
  EMA target, tau:                           xi <- xi + tau (theta - xi)
  SPR's targets under the EMA target:        t_k = g_xi(f_xi(s'_{t+k}))
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import network as net
from . import spr as ospr
from .curl import project

F32 = np.float32


def adamw_step_np(theta, g, m, v, t, lr, wd, b1=0.9, b2=0.999, eps=1e-8):
    """One AdamW step in float64 numpy; returns (theta, m, v)."""
    theta, g, m, v = (np.asarray(x, np.float64) for x in (theta, g, m, v))
    theta = theta * (1.0 - lr * wd)
    m = b1 * m + (1.0 - b1) * g
    v = b2 * v + (1.0 - b2) * g * g
    theta = theta - (lr / (1.0 - b1 ** t)) * m / (np.sqrt(v) / np.sqrt(1.0 - b2 ** t) + eps)
    return theta, m, v


def decay_f32(lr, wd):
    """d = fl32(1 - lr wd) from the float32 lr and wd, the product and difference in double (riqn_adamw_step)."""
    return F32(1.0 - float(F32(lr)) * float(F32(wd)))


def decayed_f32(theta, lr, wd):
    """fl32(theta * d): the decay half of riqn_adamw_step."""
    return (np.asarray(theta, F32) * decay_f32(lr, wd)).astype(F32)


def ema_f32(theta, xi, tau):
    """riqn_ema_f32's statement: fl(xi + fl(tau * fl(theta - xi))), every operation rounded to float32 on its own."""
    theta, xi, tau = np.asarray(theta, F32), np.asarray(xi, F32), F32(tau)
    return (xi + (tau * (theta - xi)).astype(F32)).astype(F32)


class AdamW:
    """torch.optim.AdamW over a dict of leaf tensors, with losses.Adam's step(params, grads) interface: the torch-fp32
    learner step's optimiser (lr, eps and lambda as the agent's)."""

    def __init__(self, params, keys, lr, eps, weight_decay, betas=(0.9, 0.999)):
        self.keys = list(keys)
        self.opt = torch.optim.AdamW([params[k] for k in self.keys], lr=lr, eps=eps, betas=betas,
                                     weight_decay=weight_decay, foreach=False)

    def step(self, params, grads):
        for k in self.keys:
            params[k].grad = grads[k].clone()
        self.opt.step()


def polyak(p_online, p_target, tau):
    """The torch-fp32 EMA of every trainable parameter of the target dict (xi + tau (theta - xi), each op in fp32)."""
    with torch.no_grad():
        for k, t in p_target.items():
            if net.is_trainable(k):
                t.copy_(t + tau * (p_online[k].detach() - t))


def spr_loss_ema(p_online, p_target, sp, sp_ema, x, actions, valid, x_targets, num_actions):
    """oracle.spr.spr_loss with BBF's target encoder: the targets from the EMA target network's trunk ``p_target`` and
    the EMA projection ``sp_ema`` (weight_h, bias_h, weight_c, bias_c)."""
    B, K = actions.shape
    z = net.conv_trunk(p_online, x).reshape(B, 64, 7, 7)
    zs = []
    for k in range(K):
        z = ospr.transition(sp, z, actions[:, k], num_actions)
        zs.append(z)
    y = F.linear(project(sp, torch.stack(zs).reshape(K * B, -1)), sp["weight_q"], sp["bias_q"])
    with torch.no_grad():
        t = project({k: v.detach() for k, v in sp_ema.items()},
                    net.conv_trunk({k: v.detach() for k, v in p_target.items()}, x_targets))
    cos = (F.normalize(y, dim=1, eps=1e-12) * F.normalize(t, dim=1, eps=1e-12)).sum(1).reshape(K, B)
    rows = -(torch.as_tensor(valid, dtype=y.dtype).t() * cos).sum(0)
    return rows, y, t
