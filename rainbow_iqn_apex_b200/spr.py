"""SPR: Self-Predictive Representations (Schwarzer et al., "Data-Efficient Reinforcement Learning with Self-Predictive
Representations", ICLR 2021), an auxiliary loss on the convolution trunk of every learner.

From the trunk's latent of s_t, a transition model predicts the latents of the next K states from the logged actions,
and each prediction should point where the encoder maps the state actually reached.  With f the conv trunk, s_t the
learner's (shifted) state, a_t .. a_{t+K-1} the logged actions and valid_k the mask of ReplayMemory.sample_sequence:

  z_0 = f_theta(s_t)                       the gradient pass's kept conv3 output (B, 64, 7, 7): no extra trunk pass
  z_k = T(z_{k-1}, a_{t+k-1}),  k = 1..K,  T(z, a) = ReLU(conv2(ReLU(conv1([z ; onehot(a)]))))   (3x3, padding 1, 64)
  y_k = q(g(z_k))                          q: Linear(128, 128) with bias (the predictor)
  t_k = g(f_theta(s'_{t+k}))               no gradient; s'_{t+k} an independent random shift of s_{t+k}
  g(feat) = LN(W_c ReLU(LN(W_h feat + b_h)) + b_c)          (3136 -> 512 -> 128, curl.project, SPR's own parameters)
  L_SPR = (1/B) sum_b sum_k valid_{b,k} (-cos(y_{b,k}, t_{b,k}))   (F.normalize's eps 1e-12 on both norms)

and the step minimises (1/B) sum_b w_b L_RL,b + lambda L_SPR.  The target encoder and projection are the online ones
under stop-gradient (the paper's Atari setting, tau = 0).  Priorities and the returned loss stay the RL loss; L_SPR is
not importance-weighted.  Defaults K = 5, lambda = 2 (the paper's Atari values).

This project's choices, not tuned:
  - the projection g is a separate LayerNorm MLP, not the Q head's first layer: the IQN head's first layer reads
    quantile-embedded features and the C51 and QR-DQN heads differ, so one projection serves every head;
  - the transition model has no BatchNorm (batch statistics couple the rows, running statistics add state) and the
    latents are not min-max renormalised (the min / max subgradients tie massively after a ReLU);
  - the one-hot action planes are zero-padded to 128 input channels for conv1, because the strip convolution needs
    stride^2 * Cin % 64 == 0: so at most 64 actions.

The transition convolutions have conv3's geometry on the zero-bordered 9x9 latent (3x3, stride 1, pad 0) and run on
riqn_conv_fwd_strip (split-bf16 x3, fp32-faithful) and riqn_conv_bwd_strip (the trunk's bf16 backward, data gradient
included); riqn_spr_pack writes their A operands and riqn_spr_unpack_grad crops the data gradients back.  The learner arms
DQN._trunk_addend for one backward: the addend reads the kept conv3 output, unrolls T, projects, predicts, runs
riqn_spr_cosine_fwd_bwd and backpropagates through the predictor, the projection and the K steps (weight gradients
accumulated k = K .. 1), and returns dfeat_RL + dfeat_SPR, so no loss core changes.  SPR runs only in
Learner.compute_gradients on a minibatch sampled with its sequence: not in acting, the actors, compute_priorities or the
autograd path.

Modules, built after every existing one (so that both DQNs initialise as a plain agent's from the same seed):
  agent.spr_net        SprNet: the projection, the transition model and the predictor in one flat arena, trained by
                       agent.spr_optimiser (the arena Adam with the agent's lr and adam_eps)
"""
import torch
from torch import nn

from . import augment
from ._lib import call, ptr
from .arena import Side
from .curl import DIM, HIDDEN, ProjectionArena, project, project_backward
from .model import FEAT, _geom, _strip_perm

SPR_SHIFT_SEED = 0x59E2          # the target views' draw key (net._rng_seed ^ this)
CH, EDGE, GRID = 64, 7, 9        # latent channels and edge, zero-bordered edge
CPAD = 128                       # conv1's input channels: the latent, the one-hot action planes, zeros


class SprNet(ProjectionArena):
    """SPR's trained parameters, views of one flat fp32 arena laid out weight_h (512, 3136) | bias_h | weight_c
    (128, 512) | bias_c | conv1.weight (64, 64 + A, 3, 3) | conv1.bias | conv2.weight (64, 64, 3, 3) | conv2.bias |
    weight_q (128, 128) | bias_q, the projection first so that curl.project / curl.project_backward serve it.  Initialised
    as nn.Linear / nn.Conv2d are."""

    NAMES = ("weight_h", "bias_h", "weight_c", "bias_c", "conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias",
             "weight_q", "bias_q")

    def __init__(self, action_space, device):
        super().__init__()
        h, c = nn.Linear(FEAT, HIDDEN), nn.Linear(HIDDEN, DIM)
        self.conv1 = nn.Conv2d(CH + action_space, CH, 3, padding=1)
        self.conv2 = nn.Conv2d(CH, CH, 3, padding=1)
        q = nn.Linear(DIM, DIM)
        for name, t in zip(("weight_h", "bias_h", "weight_c", "bias_c", "weight_q", "bias_q"),
                           (h.weight, h.bias, c.weight, c.bias, q.weight, q.bias)):
            setattr(self, name, nn.Parameter(t.detach().clone()))
        self.action_space = action_space
        self._flatten(torch.device(device))

    def images(self):
        """The transition convolutions' bf16 weight images, rebuilt from the arena (riqn_spr_weight_images): per layer
        (strip-ordered hi, lo, original-order hi, the strip permutation).  Called inside every step, so that a captured
        graph reads the weights of the step it replays."""
        dev = self._flat.device
        if getattr(self, "_perm", None) is None or self._perm[CPAD].device != dev:
            self._perm = {c: _strip_perm(c, 3, 1, False).to(dev, torch.int32) for c in (CPAD, CH)}
        out = []
        for conv, cpad in ((self.conv1, CPAD), (self.conv2, CH)):
            hi, lo, hio = (torch.empty(CH, 9 * cpad, dtype=torch.bfloat16, device=dev) for _ in range(3))
            call("riqn_spr_weight_images", CH, conv.weight.shape[1], cpad, ptr(conv.weight), ptr(hi), ptr(lo), ptr(hio))
            out.append((hi, lo, hio, self._perm[cpad]))
        return out


def build(agent, args, checkpoint):
    """agent.spr_net and agent.spr_optimiser (after every other module), restored from ``checkpoint`` when it holds
    them.  Returns SPR's Side."""
    from .optim import Adam
    net = agent.spr_net = SprNet(agent.action_space, args.device)
    opt = agent.spr_optimiser = Adam(net.parameters(), lr=args.lr, eps=args.adam_eps)
    if checkpoint is not None and "spr_state_dict" in checkpoint:
        net.load_state_dict(checkpoint["spr_state_dict"])
        opt.load_state_dict(checkpoint["spr_optimiser_state_dict"])
    return Side(3, net, opt, lambda: {"spr_state_dict": net.state_dict(), "spr_optimiser_state_dict": opt.state_dict()},
                broadcast=(net._flat,), trunk_term=trunk_term)


def _bf(rows, cols, dev):
    return torch.empty(rows, cols, dtype=torch.bfloat16, device=dev)


def transition_forward(net, ims, z, actions, out):
    """One step of T: ``z`` (B, 64, 7, 7) fp32, ``actions`` a (B,) int64 view (any stride), ``out`` (B, 64, 7, 7)
    receives T(z, a).  Returns the backward's operands (conv1's A image, conv1's output, conv2's A image)."""
    B, dev = z.shape[0], z.device
    (w1h, w1l, _, _), (w2h, w2l, _, _) = ims
    a1h, a1l = _bf(B * GRID * GRID, CPAD, dev), _bf(B * GRID * GRID, CPAD, dev)
    call("riqn_spr_pack", B, CPAD, ptr(z), ptr(actions), actions.stride(0), net.action_space, ptr(a1h), ptr(a1l))
    h = torch.empty(B, CH, EDGE, EDGE, device=dev)
    call("riqn_conv_fwd_strip", _geom(B, CPAD, GRID, CH, 3, 1, 0), ptr(a1h), ptr(a1l), ptr(w1h), ptr(w1l),
         ptr(net.conv1.bias), ptr(h), None, None, 0, 0, None, None, None, 0)
    a2h, a2l = _bf(B * GRID * GRID, CH, dev), _bf(B * GRID * GRID, CH, dev)
    call("riqn_spr_pack", B, CH, ptr(h), None, 1, 0, ptr(a2h), ptr(a2l))
    call("riqn_conv_fwd_strip", _geom(B, CH, GRID, CH, 3, 1, 0), ptr(a2h), ptr(a2l), ptr(w2h), ptr(w2l),
         ptr(net.conv2.bias), ptr(out), None, None, 0, 0, None, None, None, 0)
    return a1h, h, a2h


def transition_backward(net, ims, saved, out, dout, gw1_pad):
    """Backward of one step of T for the upstream ``dout`` (B, 64, 7, 7) of its output ``out``: conv2's weight and bias
    gradients and conv1's bias gradient accumulate into net's arena, conv1's (zero-padded, (64, 128*9)) weight gradient
    into ``gw1_pad``.  Returns the data gradient of conv1's input (B, 128, 9, 9)."""
    B, dev = dout.shape[0], dout.device
    (_, _, w1o, p1), (_, _, w2o, p2) = ims
    a1h, h, a2h = saved
    gv = net.grad_view
    dYg = _bf(B * GRID * GRID, CH, dev)
    din2 = torch.empty(B, CH, GRID, GRID, device=dev)
    call("riqn_conv_bwd_strip", _geom(B, CH, GRID, CH, 3, 1, 0), ptr(dout), ptr(out), ptr(a2h), ptr(w2o), ptr(p2),
         ptr(dYg), ptr(torch.empty(CH * CH * 9, device=dev)), ptr(gv(net.conv2.weight)), ptr(gv(net.conv2.bias)),
         ptr(din2), 1.0)
    dh = torch.empty(B, CH, EDGE, EDGE, device=dev)
    call("riqn_spr_unpack_grad", B, CH, ptr(din2), None, ptr(dh))
    din1 = torch.empty(B, CPAD, GRID, GRID, device=dev)
    call("riqn_conv_bwd_strip", _geom(B, CPAD, GRID, CH, 3, 1, 0), ptr(dh), ptr(h), ptr(a1h), ptr(w1o), ptr(p1),
         ptr(dYg), ptr(torch.empty(CH * CPAD * 9, device=dev)), ptr(gw1_pad), ptr(gv(net.conv1.bias)), ptr(din1), 1.0)
    return din1


def targets(learner, window, debug=None):
    """t_k of one step, (K*B, 128) with rows k*B + b: the online trunk (no gradient) over independent shifts of
    s_{t+1} .. s_{t+K} = window[:, k:k+history] (drawn after the step's shifts of s_t and s_{t+n}, under SPR_SHIFT_SEED
    and without moving the shift counters, or the parity hook's ``"spr_shifts"`` (K*B, 2) int32), then g."""
    on, K, H = learner.online_net, learner.spr[0], learner.history
    B, dev = window.shape[0], on._flat.device
    x = torch.empty(K * B, H, 84, 84, dtype=torch.uint8, device=dev)
    shifts = None
    if learner.random_shift is not None:
        shifts = augment.view_shifts(learner, "spr_shifts", K * B, SPR_SHIFT_SEED)
        for k in range(K):
            v = window[:, k + 1:k + 1 + H]
            call("riqn_random_shift", B, H, 84, 84, ptr(v), v.stride(0), None, 0, 1, ptr(shifts[k * B:]), ptr(x[k * B:]))
    else:
        for k in range(K):
            x[k * B:(k + 1) * B].copy_(window[:, k + 1:k + 1 + H])
    if getattr(on, "_strip_ops", None) is None or getattr(on, "_static_ops_dirty", True):
        on._refresh_tc_operands(h_done=True)         # the trunk's images, as the loss core would build them
    net = learner.spr_net
    t = project(net.views(net._flat), on.trunk(x))
    if debug is not None:
        debug.update(spr_shifts=shifts, spr_targets=t)
    return t


def trunk_term(learner, raw_states, sequence, debug=None):
    """SPR's term of one step on its ``sequence`` ((window, actions (B, K), valid (B, K)) of
    ReplayMemory.sample_sequence): the targets, computed now, and the one-shot addend DQN.backward_trunk applies
    (DQN._trunk_addend): from the gradient pass's kept conv3 output, unroll T over the sequence's actions, project and
    predict, run the masked cosine and backpropagate (the SPR gradients land in spr_net's arena); return
    dfeat + dfeat_SPR."""
    t = targets(learner, sequence[0], debug)
    net, (K, coef) = learner.spr_net, learner.spr
    _, actions, valid = sequence

    def addend(keep, dfeat):
        B, dev = dfeat.shape[0], dfeat.device
        ims = net.images()
        Z = torch.empty(K, B, CH, EDGE, EDGE, device=dev)
        saved, z = [], keep["out"][2]
        for k in range(K):
            saved.append(transition_forward(net, ims, z, actions[:, k], Z[k]))
            z = Z[k]
        pk = {}
        zp = project(net.views(net._flat), Z.view(K * B, FEAT), pk)
        y = torch.empty(K * B, DIM, device=dev)
        call("riqn_linear_fwd_ld", K * B, DIM, DIM, ptr(zp), DIM, ptr(net.weight_q), ptr(net.bias_q), ptr(y), DIM, 0)
        rows, dy = torch.empty(B, device=dev), torch.empty(K * B, DIM, device=dev)
        call("riqn_spr_cosine_fwd_bwd", B, K, DIM, ptr(y), ptr(t), ptr(valid), coef, ptr(rows), ptr(dy))
        call("riqn_linear_wgrad", K * B, DIM, DIM, ptr(dy), ptr(zp), ptr(net.grad_view(net.weight_q)),
             ptr(net.grad_view(net.bias_q)))
        dzp = torch.empty(K * B, DIM, device=dev)
        call("riqn_linear_dgrad_ld", K * B, DIM, DIM, ptr(dy), DIM, ptr(net.weight_q), ptr(dzp), DIM)
        dZ = project_backward(net, pk, dzp).view(K, B, CH, EDGE, EDGE)
        gw1 = torch.empty(CH, CPAD * 9, device=dev)
        call("riqn_zero_f32", ptr(gw1), gw1.numel())
        din1 = None
        for k in range(K - 1, -1, -1):                # dz_k = the projection's gradient + step k+1's data gradient
            if din1 is not None:
                call("riqn_spr_unpack_grad", B, CPAD, ptr(din1), ptr(dZ[k]), ptr(dZ[k]))
            din1 = transition_backward(net, ims, saved[k], Z[k], dZ[k], gw1)
        w1 = net.conv1.weight
        call("riqn_spr_weight_grad_add", CH, w1.shape[1], CPAD, ptr(gw1), ptr(net.grad_view(w1)))
        dfeat_spr = torch.empty(B, FEAT, device=dev)
        call("riqn_spr_unpack_grad", B, CPAD, ptr(din1), None, ptr(dfeat_spr))
        out = torch.empty_like(dfeat)
        call("riqn_add_f32", dfeat.numel(), ptr(dfeat), ptr(dfeat_spr), ptr(out))
        if debug is not None:
            debug.update(spr_latents=Z, spr_pred=y, spr_loss=rows, dfeat_spr=dfeat_spr)
        return out
    return addend
