"""Rainbow-only (C51) branch of the reference: DQN.forward (model.py:120-129) and the categorical loss
(agent.py:77-141), on the same CUDA trunk / NoisyLinear ops as the IQN path plus csrc/c51.cu.  HL-Gauss (agent.hl_gauss,
hl_gauss.py) runs the same step with the Gaussian-histogram loss kernel in place of the projection."""
import torch

from . import hl_gauss
from ._lib import call, ptr
from .compute_loss_iqn import _loss_inputs
from .model import FEAT


def _tc_mode(B):
    """Hidden NoisyLinear products on the wgmma path (same arithmetic modes as the IQN head, model.PRECISION)."""
    from .model import PRECISION
    return PRECISION["fwd"] != "fp32" and PRECISION["bwd"] == "bf16" and B % 8 == 0


def forward(net, x, log=False, keep=None, fresh_weights=False, want_argmax=None, support=None):
    """Returns probabilities (or log-probabilities) (B, A, atoms).  model.py:120-129"""
    if not fresh_weights:
        net._compose_weights()
    zv, za = hidden_z(net, x, keep=keep)
    B, A, atoms = zv.shape[0], net.action_space, net.atoms
    out = torch.empty(B, A, atoms, device=zv.device)
    if support is None:
        support = net._support(zv.device)
    call("riqn_c51_head_fwd", B, A, atoms, ptr(zv), ptr(za), ptr(support), None if log else ptr(out),
         ptr(out) if log else None, ptr(want_argmax))
    return out


def hidden_z(net, x, keep=None, col_cache=None, feat=None):
    """Trunk, noisy hidden layers [h_v | h_a] and z-layers of the C51-shaped network (C51 and QR-DQN heads): returns
    zv (B, zv width), za (B, za width), the widths those of fcnoisy_z_v / fcnoisy_z_a.  ``feat``: trunk features computed
    by the caller (trunk_pair) for a no-grad pass.  ``keep``: dict that receives the backward's operands."""
    from .model import PRECISION
    if feat is None:
        feat = net.trunk(x, keep, col_cache)
    B = feat.shape[0]
    dev = feat.device
    hid = net.hidden
    nzv, nza = net.fcnoisy_z_v.out_features, net.fcnoisy_z_a.out_features
    h = torch.empty(B, 2 * hid, device=dev)
    x_bf = None
    if _tc_mode(B):
        # features -> 16-bit operand images (fp16 forward: fp16(x) for this product + bf16(x) for the weight gradient)
        fwd = PRECISION["fwd"]
        f16, x3 = fwd == "fp16", fwd == "bf16x3"
        x_hi = torch.empty(B, FEAT, dtype=torch.float16 if f16 else torch.bfloat16, device=dev)
        x_lo = torch.empty(B, FEAT, dtype=torch.bfloat16, device=dev) if (x3 or (f16 and keep is not None)) else None
        call("riqn_split_bf16", B, FEAT, ptr(feat), ptr(x_hi), ptr(x_lo), None, None, 1 if f16 else 0)
        call("riqn_gemm_bf16_tc", B, 2 * hid, FEAT, ptr(x_hi), ptr(x_lo) if x3 else None, ptr(net._w_hi),
             ptr(net._w_lo) if x3 else None, ptr(h), 2 * hid, 1, ptr(net._b_eff_h), None, None, 1, None, None, 3 if f16 else 0)
        x_bf = x_lo if f16 else x_hi
    else:
        call("riqn_noisy_linear_fwd", B, FEAT, 2 * hid, ptr(feat), ptr(net._w_eff_h), ptr(net._b_eff_h), ptr(h))
    zv = torch.empty(B, nzv, device=dev)
    za = torch.empty(B, nza, device=dev)
    wz, bz = net._w_eff_z, net._b_eff_z          # rows [0, nzv) = z_v, rows [nzv, nzv + nza) = z_a
    hv, ha = h[:, :hid], h[:, hid:]
    call("riqn_linear_fwd_ld", B, hid, nzv, ptr(hv), 2 * hid, ptr(wz), ptr(bz), ptr(zv), nzv, 0)
    wza, bza = wz[nzv:], bz[nzv:]
    call("riqn_linear_fwd_ld", B, hid, nza, ptr(ha), 2 * hid, ptr(wza), ptr(bza), ptr(za), nza, 0)
    if keep is not None:
        keep.update(feat=feat, h=h, B=B, x_bf=x_bf)
    return zv, za


def loss_core(agent, states, actions, returns, next_states, nonterminals, debug=None, keep_graph=True, demo=None):
    """agent.py:77-141.  Returns the loss (B,) and its backward(gscale, gscale_mul=1.0), which accumulates into the online
    network's gradient arena the gradient of sum_b gscale[b] * gscale_mul * loss[b]; None without ``keep_graph``.

    The reference runs online(states) first (:82-83), then the two no-grad passes over next_states (:95-104), each after
    its own reset_noise.  The passes are independent, so they are evaluated here as 2, 3, 1 -- every pass still with its own
    noise sample (injected noises keep their reference slot) -- which leaves the gradient pass's weights and epsilons LIVE
    when the backward runs: no 50 MB of weight / epsilon snapshots per step.  ``demo`` must be None: DQfD's margin loss
    is not defined on the categorical head."""
    if demo is not None:
        raise ValueError("the C51 and HL-Gauss losses take no demonstration mask: DQfD applies to IQN and QR-DQN")
    (states, actions, returns, next_states, nonterminals), inj = _loss_inputs(
        agent, states, actions, returns, next_states, nonterminals)
    on, tg = agent.online_net, agent.target_net
    B, A, atoms = states.shape[0], agent.action_space, agent.atoms
    dev = states.device
    noises = inj.get("noises", (None, None, None))   # a dict may carry only "shifts"
    on.reset_noise(noises[1])                                              # :95
    a_star = torch.empty(B, dtype=torch.int64, device=dev)
    forward(on, next_states, fresh_weights=True, want_argmax=a_star, support=agent.acting_support)  # :97-102
    tg.reset_noise(noises[2])                                              # :103
    pns = forward(tg, next_states, fresh_weights=True, support=agent.support)                      # :104
    on.reset_noise(noises[0])                                              # agent.py:82
    keep = {} if keep_graph else None
    log_ps = forward(on, states, log=True, keep=keep, fresh_weights=True, support=agent.support)   # :83
    loss = torch.empty(B, device=dev)
    dq = torch.empty(B, atoms, device=dev)
    m_out = torch.empty(B, atoms, device=dev) if debug is not None else None
    target_out = None
    if getattr(agent, "hl_gauss", None) is not None:   # HL-Gauss: the histogram of the scalar target (hl_gauss.py)
        target_out = torch.empty(B, device=dev) if debug is not None else None
        hl_gauss.hl_gauss_loss(agent, B, log_ps, pns, actions, a_star, returns, nonterminals, loss, dq, m_out,
                               target_out)
    else:
        args = (ptr(log_ps), ptr(pns), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals), ptr(agent.support),
                agent.gamma_n(), float(agent.Vmin), float(agent.Vmax), float(agent.delta_z))
        eps = getattr(agent, "value_rescaling", None)
        if eps is None:
            call("riqn_c51_loss_fwd_bwd", B, A, atoms, *args, ptr(loss), ptr(dq), ptr(m_out))
        else:   # the atoms move to h(R + gamma^n nt h^-1(z_j)) before the projection
            call("riqn_c51_loss_fwd_bwd_h", B, A, atoms, *args, eps, ptr(loss), ptr(dq), ptr(m_out))
    if debug is not None:
        debug.update(a_star=a_star, m=m_out, log_ps=log_ps)
        if target_out is not None:                     # HL-Gauss: the scalar targets and the probabilities they came from
            debug.update(target=target_out, p_target=pns)
    if keep is None:
        return loss, None
    version = getattr(on, "_noise_version", 0)       # bumped by every DQN.reset_noise()

    def backward(gscale, gscale_mul=1.0):
        if getattr(on, "_noise_version", 0) != version:
            raise RuntimeError("the online network's noise was resampled between the C51 loss and its backward")
        gscale = gscale.contiguous().float()
        dzv = torch.empty(B, atoms, device=dev)
        dza = torch.empty(B, A * atoms, device=dev)
        call("riqn_c51_head_bwd", B, A, atoms, ptr(dq), ptr(gscale), float(gscale_mul), ptr(actions), ptr(dzv), ptr(dza))
        _backward_below_head(on, keep, dzv, dza, on.grad_view)

    return loss, backward


def backward_dense(on, keep, out, grad_out, log, gv):
    """Parameter gradients of a forward recorded in ``keep`` given the dense dL/dout ``grad_out`` (B, A, atoms) of its
    output ``out`` (probabilities, or log-probabilities when ``log``); ``gv(param)`` is each parameter's gradient buffer."""
    B, A, atoms = out.shape
    dzv = torch.empty(B, atoms, device=out.device)
    dza = torch.empty(B, A * atoms, device=out.device)
    call("riqn_c51_head_bwd_dense", B, A, atoms, ptr(out), ptr(grad_out), 1 if log else 0, ptr(dzv), ptr(dza))
    _backward_below_head(on, keep, dzv, dza, gv)


def _backward_below_head(on, keep, dzv, dza, gv):
    """From the z-layer data gradients dzv (B, zv width), dza (B, za width) down to the trunk: z-layer and hidden-layer
    NoisyLinear gradients, then the convolutions.  The widths are fcnoisy_z_v's and fcnoisy_z_a's (C51: atoms and
    A*atoms; QR-DQN: N and A*N)."""
    B, dev = keep["B"], dzv.device
    hid = on.hidden
    hvL, haL, zvL, zaL = on.fcnoisy_h_v, on.fcnoisy_h_a, on.fcnoisy_z_v, on.fcnoisy_z_a
    h = keep["h"]
    dh = torch.empty(B, 2 * hid, device=dev)
    dhv, dha = dh[:, :hid], dh[:, hid:]
    hv, ha = h[:, :hid], h[:, hid:]
    nzv, nza = zvL.out_features, zaL.out_features
    w_z = on._w_eff_z
    wzv, wza = w_z[:nzv], w_z[nzv:]
    call("riqn_linear_dgrad_ld", B, hid, nzv, ptr(dzv), nzv, ptr(wzv), ptr(dhv), 2 * hid)
    call("riqn_linear_dgrad_ld", B, hid, nza, ptr(dza), nza, ptr(wza), ptr(dha), 2 * hid)
    call("riqn_relu_mask", dh.numel(), ptr(h), ptr(dh))
    scratch = torch.empty(max(nza, 2 * hid), device=dev)
    for layer, d, xin in ((zvL, dzv, hv), (zaL, dza, ha)):
        call("riqn_noisy_wgrad_ld", B, hid, layer.out_features, ptr(d), layer.out_features, ptr(xin), 2 * hid,
             ptr(layer.weight_epsilon), ptr(gv(layer.weight_mu)), ptr(gv(layer.weight_sigma)))
        call("riqn_noisy_bias_grad", B, layer.out_features, ptr(d), ptr(layer.bias_epsilon), ptr(scratch),
             ptr(gv(layer.bias_mu)), ptr(gv(layer.bias_sigma)))
    # hidden layers: [h_v | h_a] adjacent in every arena (parameters, gradients, epsilons)
    dfeat = torch.empty(B, FEAT, device=dev)
    if keep.get("x_bf") is not None:
        # tensor cores: dW = dh^T x straight from the row-major bf16 images (MN-major operands), dx = dh W from W itself
        from .model import PRECISION
        dh_bf = torch.empty(B, 2 * hid, dtype=torch.bfloat16, device=dev)
        call("riqn_split_bf16", B, 2 * hid, ptr(dh), ptr(dh_bf), None, None, None, 0)
        w_bf = on._w_lo if PRECISION["fwd"] == "fp16" else on._w_hi
        call("riqn_gemm_bf16_tc_mn", 2 * hid, FEAT, B, ptr(dh_bf), ptr(keep["x_bf"]), 1, ptr(gv(hvL.weight_mu)), FEAT, 3,
             ptr(gv(hvL.weight_sigma)), ptr(hvL.weight_epsilon), 1.0, 1, None, 0)
        call("riqn_noisy_bias_grad", B, 2 * hid, ptr(dh), ptr(hvL.bias_epsilon), ptr(scratch), ptr(gv(hvL.bias_mu)),
             ptr(gv(hvL.bias_sigma)))
        call("riqn_gemm_bf16_tc_mn", B, FEAT, 2 * hid, ptr(dh_bf), ptr(w_bf), 0, ptr(dfeat), FEAT, 0, None, None, 1.0, 1,
             None, 0)
    else:
        call("riqn_noisy_linear_wgrad", B, FEAT, 2 * hid, ptr(dh), ptr(keep["feat"]), ptr(hvL.weight_epsilon),
             ptr(hvL.bias_epsilon), ptr(scratch), ptr(gv(hvL.weight_mu)), ptr(gv(hvL.weight_sigma)), ptr(gv(hvL.bias_mu)),
             ptr(gv(hvL.bias_sigma)))
        call("riqn_noisy_linear_dgrad", B, FEAT, 2 * hid, ptr(dh), ptr(on._w_eff_h), ptr(dfeat))
    on.backward_trunk(keep, dfeat)
