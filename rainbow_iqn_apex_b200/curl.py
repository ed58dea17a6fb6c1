"""CURL: Contrastive Unsupervised Representations for Reinforcement Learning (Srinivas, Laskin & Abbeel, ICML 2020), an
auxiliary loss on the convolution trunk of every learner.

Two augmentations of the same state should map to nearby features.  The anchor x_a is the randomly shifted s_t that the
gradient pass already reads (Agent.random_shift); the positive x_k is a second, independent random shift of the same
unshifted s_t, drawn under a Philox key of its own that moves none of the shift counters, so that the shifts of s_t and
s_{t+n} stay those of a learner without CURL in every step, eager or replayed.  With f the conv trunk and this project's projection head

  g(feat) = LN(W_c ReLU(LN(W_h feat + b_h)) + b_c)       (3136 -> 512 -> 128; LN: row LayerNorm without affine, eps 1e-5)

  z_a = g_theta(f_theta(x_a)) ,  z_k = g_xi(f_xi(x_k))  (no gradient) ,  logits_ij = z_a,i^T W z_k,j   (B x B)
  L_CURL = (1/B) sum_i [logsumexp_j logits_ij - logits_ii]

and the step minimises (1/B) sum_b w_b L_RL,b + lambda L_CURL (the CURL term is not importance-weighted).  xi, the key
encoder, is a momentum copy of the trunk and of the projection (not of W): after the Adam steps
xi <- xi + tau (theta - xi), each operation rounded on its own (riqn_ema_f32).  Priorities and the returned loss stay the
RL loss.  The projection sizes, the LayerNorms and the defaults lambda = 1, tau = 0.001 are this project's starting
point, not tuned and not the paper's settings.

The anchor needs no extra trunk pass: the learner arms DQN._trunk_addend for one backward, and DQN.backward_trunk hands
it the gradient pass's kept features and the loss core's dfeat; it returns dfeat_RL + dfeat_CURL (riqn_add_f32), so no
loss core changes.  CURL runs only in Learner.compute_gradients: not in acting, the actors, compute_priorities or the
autograd path of Agent.compute_loss_actor_or_learner.

Modules, all built after every existing one (so that both DQNs initialise as a plain agent's from the same seed):
  agent.curl_net        CurlProjection: W_h, b_h, W_c, b_c and W in one flat arena, trained by agent.curl_optimiser
                        (the arena Adam with the agent's lr and adam_eps)
  agent.momentum_net    a DQN whose trunk alone ever runs (f_xi), and agent.momentum_projection, the untrained
                        buffer arena of g_xi (the projection prefix of curl_net's arena layout)
"""
import torch
from torch import nn

from . import augment
from ._lib import call, ptr
from .arena import ArenaModule, Side
from .model import DQN, FEAT

HIDDEN, DIM = 512, 128                                         # projection widths
CURL_SHIFT_SEED = 0xC0A1                                       # the positive view's draw key (net._rng_seed ^ this)


class ProjectionArena(ArenaModule):
    """An arena whose first four groups are a projection g (weight_h, bias_h, weight_c, bias_c): the prefix
    [0, proj_numel) that project and project_backward read.  CURL's and SPR's arenas."""

    @property
    def proj_numel(self):
        return self.get_parameter(self.NAMES[4])._riqn_offset

    def views(self, arena):
        """(weight_h, bias_h, weight_c, bias_c) of the projection laid out in ``arena`` (this arena, or a copy of its
        projection prefix)."""
        params = [self.get_parameter(name) for name in self.NAMES[:4]]
        return tuple(arena[p._riqn_offset:p._riqn_offset + p.numel()].view(p.shape) for p in params)


class CurlProjection(ProjectionArena):
    """The online projection g_theta and the bilinear W, views of one flat fp32 arena laid out weight_h (512, 3136) |
    bias_h | weight_c (128, 512) | bias_c | bilinear (128, 128).  Initialised like nn.Linear (uniform in
    +-1/sqrt(fan_in)), W like a bias-free nn.Linear(128, 128)."""

    NAMES = ("weight_h", "bias_h", "weight_c", "bias_c", "bilinear")

    def __init__(self, device):
        super().__init__()
        h, c, w = nn.Linear(FEAT, HIDDEN), nn.Linear(HIDDEN, DIM), nn.Linear(DIM, DIM, bias=False)
        for name, t in zip(self.NAMES, (h.weight, h.bias, c.weight, c.bias, w.weight)):
            setattr(self, name, nn.Parameter(t.detach().clone()))
        self._flatten(torch.device(device))


def _tc(B):
    """Whether the 3136-wide products of a batch of B run on the tensor cores (split-bf16 x3, fp32-faithful): every
    reduction length there is a multiple of 8 (the weight gradient's is B).  Otherwise they run on the fp32 SIMT GEMM."""
    return B % 8 == 0


def _split(x, rows, cols, transposed=False):
    """bf16 (hi, lo) images of the fp32 matrix x (rows, cols), and with ``transposed`` those of x^T (riqn_split_bf16)."""
    bf = lambda *sh: torch.empty(*sh, dtype=torch.bfloat16, device=x.device)
    hi, lo = bf(rows, cols), bf(rows, cols)
    hiT, loT = (bf(cols, rows), bf(cols, rows)) if transposed else (None, None)
    call("riqn_split_bf16", rows, cols, ptr(x), ptr(hi), ptr(lo), ptr(hiT), ptr(loT), 0)
    return hi, lo, hiT, loT


def project(views, feat, keep=None):
    """z = g(feat) for the projection ``views`` (CurlProjection.views) and features ``feat`` (B, 3136) fp32.  The
    3136 -> 512 product runs on riqn_gemm_bf16_tc in split-bf16 x3 mode when _tc(B) (its bias joins in the LayerNorm),
    else on the fp32 SIMT GEMM; the 512 -> 128 product on the SIMT GEMM.  ``keep``: dict that receives the backward's
    operands."""
    B, dev = feat.shape[0], feat.device
    wh, bh, wc, bc = views
    h = torch.empty(B, HIDDEN, device=dev)
    if _tc(B):
        x_hi, x_lo, x_hiT, x_loT = _split(feat, B, FEAT, transposed=keep is not None)
        w_hi, w_lo, w_hiT, w_loT = _split(wh, HIDDEN, FEAT, transposed=keep is not None)
        call("riqn_gemm_bf16_tc", B, HIDDEN, FEAT, ptr(x_hi), ptr(x_lo), ptr(w_hi), ptr(w_lo), ptr(h), HIDDEN, 0, None,
             None, None, 1, None, None, 0)
        h_bias = bh
    else:
        call("riqn_linear_fwd_ld", B, FEAT, HIDDEN, ptr(feat), FEAT, ptr(wh), ptr(bh), ptr(h), HIDDEN, 0)
        h_bias = None
    r = torch.empty(B, HIDDEN, device=dev)
    call("riqn_layernorm_fwd", B, HIDDEN, ptr(h), ptr(h_bias), 1, ptr(r))
    c = torch.empty(B, DIM, device=dev)
    call("riqn_linear_fwd_ld", B, HIDDEN, DIM, ptr(r), HIDDEN, ptr(wc), ptr(bc), ptr(c), DIM, 0)
    z = torch.empty(B, DIM, device=dev)
    call("riqn_layernorm_fwd", B, DIM, ptr(c), None, 0, ptr(z))
    if keep is not None:
        keep.update(feat=feat, h=h, h_bias=h_bias, r=r, c=c)
        if _tc(B):
            keep.update(x_T=(x_hiT, x_loT), w_T=(w_hiT, w_loT))
    return z


def project_backward(net, keep, dz):
    """Accumulate dL/d(weight_h, bias_h, weight_c, bias_c) into ``net``'s gradient arena for the forward in ``keep`` and
    the upstream ``dz`` (B, 128); returns dL/dfeat (B, 3136).  The two 3136-wide products (dW_h += dh^T feat and
    dfeat = dh W_h) take the path the forward took; on the tensor cores the weight gradient is one split, so each
    element gets one add, and b_h's gradient is riqn_colsum_add's fixed-order column sum."""
    B, dev = dz.shape[0], dz.device
    wh, _, wc, _ = net.views(net._flat)
    gwh, gbh, gwc, gbc = net.views(net._flat_grad)
    dc = torch.empty(B, DIM, device=dev)
    call("riqn_layernorm_bwd", B, DIM, ptr(keep["c"]), None, ptr(dz), 0, ptr(dc))
    call("riqn_linear_wgrad", B, DIM, HIDDEN, ptr(dc), ptr(keep["r"]), ptr(gwc), ptr(gbc))
    dr = torch.empty(B, HIDDEN, device=dev)
    call("riqn_linear_dgrad_ld", B, HIDDEN, DIM, ptr(dc), DIM, ptr(wc), ptr(dr), HIDDEN)
    dh = torch.empty(B, HIDDEN, device=dev)
    call("riqn_layernorm_bwd", B, HIDDEN, ptr(keep["h"]), ptr(keep["h_bias"]), ptr(dr), 1, ptr(dh))
    dfeat = torch.empty(B, FEAT, device=dev)
    if "x_T" in keep:
        d_hi, d_lo, d_hiT, d_loT = _split(dh, B, HIDDEN, transposed=True)
        (x_hiT, x_loT), (w_hiT, w_loT) = keep["x_T"], keep["w_T"]
        call("riqn_gemm_bf16_tc", HIDDEN, FEAT, B, ptr(d_hiT), ptr(d_loT), ptr(x_hiT), ptr(x_loT), ptr(gwh), FEAT, 2, None,
             None, None, 1, None, None, 0)
        call("riqn_colsum_add", B, HIDDEN, ptr(dh), ptr(gbh))
        call("riqn_gemm_bf16_tc", B, FEAT, HIDDEN, ptr(d_hi), ptr(d_lo), ptr(w_hiT), ptr(w_loT), ptr(dfeat), FEAT, 0, None,
             None, None, 1, None, None, 0)
    else:
        call("riqn_linear_wgrad", B, HIDDEN, FEAT, ptr(dh), ptr(keep["feat"]), ptr(gwh), ptr(gbh))
        call("riqn_linear_dgrad_ld", B, FEAT, HIDDEN, ptr(dh), HIDDEN, ptr(wh), ptr(dfeat), FEAT)
    return dfeat


def build(agent, args, checkpoint):
    """The CURL modules of ``agent`` (after both DQNs and the fraction proposal): curl_net, curl_optimiser, momentum_net
    and momentum_projection, with xi = theta, or all four restored from ``checkpoint`` when it holds them.  Returns
    CURL's Side."""
    net = agent.curl_net = CurlProjection(args.device)
    from .optim import Adam
    opt = agent.curl_optimiser = Adam(net.parameters(), lr=args.lr, eps=args.adam_eps)
    agent.momentum_net = DQN(args, agent.action_space).to(device=args.device)
    agent.momentum_projection = torch.empty(net.proj_numel, device=net._flat.device)
    if checkpoint is not None and "curl_state_dict" in checkpoint:
        net.load_state_dict(checkpoint["curl_state_dict"])
        opt.load_state_dict(checkpoint["curl_optimiser_state_dict"])
        mom = checkpoint["curl_momentum_state_dict"]
        for name in ("conv1", "conv2", "conv3"):
            conv = getattr(agent.momentum_net, name)
            conv.weight.data.copy_(mom[name + ".weight"])
            conv.bias.data.copy_(mom[name + ".bias"])
        for v, name in zip(net.views(agent.momentum_projection), CurlProjection.NAMES):
            v.copy_(mom[name])
    else:
        n = trunk_numel(agent.online_net)
        agent.momentum_net._flat[:n].copy_(agent.online_net._flat[:n])
        copy_projection(agent)
    agent.momentum_net._params_changed()
    return Side(2, net, opt,
                lambda: {"curl_state_dict": net.state_dict(), "curl_optimiser_state_dict": opt.state_dict(),
                         "curl_momentum_state_dict": momentum_state_dict(agent)},
                broadcast=(net._flat, agent.momentum_net._flat, agent.momentum_projection),
                after_step=momentum_update, after_reset=copy_projection, trunk_term=trunk_term)


def copy_projection(agent):
    """g_xi <- g_theta: the momentum projection set to the online one (at construction and after a reset)."""
    agent.momentum_projection.copy_(agent.curl_net._flat[:agent.curl_net.proj_numel])


def momentum_state_dict(agent):
    """curl_momentum_state_dict of a checkpoint: the key encoder's conv1-3 and projection, by name (on the CPU)."""
    out = {}
    for name in ("conv1", "conv2", "conv3"):
        conv = getattr(agent.momentum_net, name)
        out[name + ".weight"], out[name + ".bias"] = conv.weight.detach().cpu().clone(), conv.bias.detach().cpu().clone()
    for v, name in zip(agent.curl_net.views(agent.momentum_projection), CurlProjection.NAMES):
        out[name] = v.detach().cpu().clone()
    return out


def trunk_numel(net):
    """Length of the conv1-3 prefix of a DQN's parameter arena (the first groups of _param_groups_in_arena_order)."""
    return net._offsets[id(net.conv3.bias)] + net.conv3.bias.numel()


def positives(learner, states, debug=None):
    """The key view of one step: an independent shift of the unshifted ``states`` (drawn after the step's shifts of s_t
    and s_{t+n}, under CURL_SHIFT_SEED, or the parity hook's ``"curl_shifts"`` (B, 2) int32), through the momentum trunk
    and projection.
    Returns z_k (B, 128)."""
    mom = learner.momentum_net
    shifts = augment.view_shifts(learner, "curl_shifts", states.shape[0], CURL_SHIFT_SEED)
    x_k = augment.random_shift(states, None, shifts)
    # the EMA rewrites the key trunk every step: its operand images are rebuilt here, inside every captured replay
    mom._refresh_tc_operands(force=True, h_done=True)
    z_k = project(learner.curl_net.views(learner.momentum_projection), mom.trunk(x_k))
    if debug is not None:
        debug.update(curl_shifts=shifts, z_k=z_k)
    return z_k


def trunk_term(learner, raw_states, sequence, debug=None):
    """CURL's term of one step on the unshifted ``raw_states``: the positives, drawn now, and the one-shot addend
    DQN.backward_trunk applies (DQN._trunk_addend): given the gradient pass's kept operands and the loss core's dfeat,
    run the anchor projection on the kept features, the InfoNCE and the projection backward (the CURL gradients land in
    curl_net's arena) and return dfeat + dfeat_CURL."""
    z_k = positives(learner, raw_states, debug)
    net, coef = learner.curl_net, learner.curl[0]

    def addend(keep, dfeat):
        B = dfeat.shape[0]
        feat = keep["out"][2].view(B, FEAT)
        pk = {}
        z_a = project(net.views(net._flat), feat, pk)
        rows = torch.empty(B, device=dfeat.device)
        dz_a = torch.empty(B, DIM, device=dfeat.device)
        logits = torch.empty(B, B, device=dfeat.device) if debug is not None else None
        call("riqn_curl_infonce_fwd_bwd", B, DIM, ptr(z_a), ptr(z_k), ptr(net.bilinear), coef, ptr(rows), ptr(dz_a),
             ptr(net.grad_view(net.bilinear)), ptr(logits))
        dfeat_curl = project_backward(net, pk, dz_a)
        out = torch.empty_like(dfeat)
        call("riqn_add_f32", dfeat.numel(), ptr(dfeat), ptr(dfeat_curl), ptr(out))
        if debug is not None:
            debug.update(z_a=z_a, logits=logits, curl_loss=rows, dfeat_curl=dfeat_curl)
        return out
    return addend


def momentum_update(learner):
    """xi <- xi + tau (theta - xi) over the trunk's arena prefix and the projection (after the Adam steps)."""
    on, mom, net, tau = learner.online_net, learner.momentum_net, learner.curl_net, learner.curl[1]
    call("riqn_ema_f32", trunk_numel(on), ptr(on._flat), ptr(mom._flat), tau)
    call("riqn_ema_f32", net.proj_numel, ptr(net._flat), ptr(learner.momentum_projection), tau)
