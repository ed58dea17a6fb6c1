"""Oracle (test infrastructure): CURL (Srinivas, Laskin & Abbeel, ICML 2020) as this project states it
(rainbow_iqn_apex_b200/curl.py), in torch fp32 on the CPU, composed with ``losses.learn_step``.

  g(feat) = LN(W_c ReLU(LN(W_h feat + b_h)) + b_c) ,  logits_ij = z_a,i^T W z_k,j ,
  L_CURL = (1/B) sum_i [logsumexp_j logits_ij - logits_ii] ,  objective (1/B) sum_b w_b L_RL,b + lambda L_CURL ,
  xi <- xi + tau (theta - xi) after the Adam steps (float32, each operation rounded on its own).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import losses, network as net

NAMES = ("weight_h", "bias_h", "weight_c", "bias_c", "bilinear")
PROJ = NAMES[:4]
CONV = ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias")


def layer_norm(x, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], eps=eps)


def project(p, feat):
    """z = g(feat) for the projection parameters ``p`` (weight_h, bias_h, weight_c, bias_c)."""
    r = torch.relu(layer_norm(F.linear(feat, p["weight_h"], p["bias_h"])))
    return layer_norm(F.linear(r, p["weight_c"], p["bias_c"]))


def infonce(z_a, z_k, w):
    """(per-row terms (B,), logits (B, B)): logsumexp_j l_ij - l_ii, row-max shifted."""
    logits = z_a @ w @ z_k.t()
    m = logits.max(dim=1, keepdim=True).values.detach()
    rows = (m[:, 0] + torch.log(torch.exp(logits - m).sum(1))) - logits.diagonal()
    return rows, logits


def ema(theta, xi, tau):
    """riqn_ema_f32 in numpy float32: xi + tau * (theta - xi), each operation rounded on its own."""
    theta, xi = np.asarray(theta, np.float32), np.asarray(xi, np.float32)
    return xi + np.float32(tau) * (theta - xi)


class _Recorder:
    """A stand-in optimiser for losses.learn_step: keeps the RL gradients, steps nothing."""

    def step(self, params, grads):
        self.grads = grads


def learn_step(p_online, p_target, adam, batch, weights, noises, taus, cfg, curl_p, curl_adam, mom_conv, mom_proj, x_k,
               coef, tau_m, rainbow_only=False, keep=None):
    """Learner.compute_gradients + apply_gradients of a CURL learner.  ``batch``: the anchor-view (shifted) frames as
    losses.learn_step takes them; ``x_k``: the positive view (B, 4, 84, 84) fp32 / 255.  ``curl_p``: leaf tensors with
    requires_grad (NAMES), stepped by ``curl_adam``; ``mom_conv`` (CONV) and ``mom_proj`` (PROJ): the momentum copies,
    updated in place.  Returns (RL loss (B,), online grads, CURL grads, dict(rows, z_a, z_k, logits))."""
    rec = _Recorder()
    loss, _ = losses.learn_step(p_online, p_target, rec, batch, weights, noises, taus, cfg, rainbow_only=rainbow_only,
                                keep=keep)
    for t in curl_p.values():
        t.grad = None
    z_a = project(curl_p, net.conv_trunk(p_online, batch[0]))
    with torch.no_grad():
        z_k = project(mom_proj, net.conv_trunk(mom_conv, x_k))
    rows, logits = infonce(z_a, z_k, curl_p["bilinear"])
    (coef * rows.mean()).backward()               # adds onto the RL gradients left in the online parameters' .grad
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    cgrads = {k: curl_p[k].grad.detach().clone() for k in NAMES}
    adam.step(p_online, grads)
    curl_adam.step(curl_p, cgrads)
    for src, dst, keys in ((p_online, mom_conv, CONV), (curl_p, mom_proj, PROJ)):
        for k in keys:
            dst[k] = torch.from_numpy(ema(src[k].detach().numpy(), dst[k].numpy(), tau_m))
    return loss, grads, cgrads, dict(rows=rows.detach(), z_a=z_a.detach(), z_k=z_k, logits=logits.detach())
