"""QR-DQN, Distributional Reinforcement Learning with Quantile Regression (Dabney, Rowland, Bellemare & Munos, AAAI 2018).

QR-DQN keeps the C51 network (conv trunk, noisy hidden layers [h_v | h_a], z-layers) but reads the N outputs of each
action as quantile values at the fixed fractions tau_hat_i = (2i+1)/(2N), i = 0..N-1, instead of logits over a fixed
support:

  q_i(s, a) = v_i(s) + a_i(s, a) - mean_a' a_i(s, a') ,   Q(s, a) = mean_i q_i(s, a)

The head (riqn_qr_head_fwd) writes q quantile-major, (N*B, A) with row i*B + b, like the IQN head, so the quantile-Huber
loss, the argmax kernels and value rescaling are IQN's own.  There is no support: with value rescaling, QR-DQN learns
unclipped returns at the cost of a C51 step.

The learner step runs the IQN path's three passes, each after its own noise reset: online(s') -> a* = argmax_a mean_i q_i,
target(s') (both trunks in one stacked trunk_pair), online(s) with the backward's operands; then the quantile-Huber loss
against R + gamma^n nt q_tgt[a*] at the N x N fraction pairs, and riqn_qr_head_bwd below it.  MMDQN (agent.mmd, mmd.py)
runs the same step with the MMD loss kernel in place of the quantile-Huber one; CQL (agent.cql, cql.py) adds alpha times
the log-sum-exp gap to the quantile-Huber loss and takes riqn_qr_head_bwd_dense.
"""
import numbers

import torch

from . import c51, cql, mmd
from ._lib import call, ptr
from .compute_loss_iqn import _loss_inputs, _quantile_loss, greedy_actions

MAX_QUANTILES = 256
MAX_ACTIONS = 32       # riqn_argmax_mean / riqn_argmax_expected_h


def check_qr(qr_dqn, num_tau_samples=None, action_space=None, rainbow_only=False, munchausen=None, fqf=None, risk=None):
    """Validate a QR-DQN configuration.  Returns None when ``qr_dqn`` is off (0 / False), else N = ``num_tau_samples``,
    an integer in 2..256.  ``action_space`` must not exceed 32; QR-DQN does not combine with ``rainbow_only``, Munchausen
    targets (``munchausen`` not None) or FQF (``fqf`` not None), and acts risk-neutrally (``risk`` None, as
    model.check_risk returns it for the neutral measure).  Raises ValueError otherwise."""
    if isinstance(qr_dqn, bool) or (isinstance(qr_dqn, numbers.Integral) and qr_dqn in (0, 1)):
        if not qr_dqn:
            return None
    else:
        raise ValueError(f"qr_dqn must be 0 or 1, got {qr_dqn!r}")
    if (isinstance(num_tau_samples, bool) or not isinstance(num_tau_samples, numbers.Integral)
            or not 2 <= num_tau_samples <= MAX_QUANTILES):
        raise ValueError(f"QR-DQN needs num_tau_samples (its N) in 2..{MAX_QUANTILES}, got {num_tau_samples!r}")
    if action_space is not None and not 1 <= action_space <= MAX_ACTIONS:
        raise ValueError(f"QR-DQN supports 1..{MAX_ACTIONS} actions, got {action_space!r}")
    if rainbow_only:
        raise ValueError("qr_dqn and rainbow_only are two different heads on the same network: set one of them")
    if munchausen is not None:
        raise ValueError("QR-DQN and Munchausen targets do not combine: set munchausen = 0 or qr_dqn = 0")
    if fqf is not None:
        raise ValueError("QR-DQN has fixed fractions and FQF learned ones: set fqf = 0 or qr_dqn = 0")
    if risk is not None:
        raise ValueError("QR-DQN has fixed quantile fractions: a risk measure has nothing to distort; use the neutral "
                         "measure")
    return int(num_tau_samples)


def fractions(net, batch):
    """The fixed fractions tau_hat_i = fl((2i+1)/(2N)) as an (N*batch, 1) array, quantile-major (row i*batch + b); built
    once per batch size and cached on ``net``."""
    N, dev = net.num_quantiles, net._flat.device
    cache = net.__dict__.setdefault("_qr_tau", {})
    t = cache.get(batch)
    if t is None or t.device != dev:
        i = torch.arange(N, dtype=torch.float32)
        tau = (2.0 * i + 1.0) / float(2 * N)           # exact numerator and denominator, one IEEE division
        t = tau.repeat_interleave(batch).reshape(N * batch, 1).to(dev)
        cache[batch] = t
    return t


def forward(net, x, keep=None, fresh_weights=False, col_cache=None, feat=None):
    """Quantile values q (N*B, A), quantile-major, of the QR network ``net`` on frames ``x`` (or on the trunk features
    ``feat`` a trunk_pair computed)."""
    if not fresh_weights:
        net._compose_weights()
    zv, za = c51.hidden_z(net, x, keep=keep, col_cache=col_cache, feat=feat)
    B, A, N = zv.shape[0], net.action_space, net.num_quantiles
    q = torch.empty(N * B, A, device=zv.device)
    call("riqn_qr_head_fwd", B, A, N, ptr(zv), ptr(za), ptr(q))
    return q


def backward_dense(on, keep, grad_q, gv):
    """Parameter gradients of a forward recorded in ``keep`` given the dense dL/dq ``grad_q`` (N*B, A); ``gv(param)`` is
    each parameter's gradient buffer."""
    B, N = keep["B"], on.num_quantiles
    dzv = torch.empty(B, N, device=grad_q.device)
    dza = torch.empty(B, on.action_space * N, device=grad_q.device)
    call("riqn_qr_head_bwd_dense", B, on.action_space, N, ptr(grad_q), ptr(dzv), ptr(dza))
    c51._backward_below_head(on, keep, dzv, dza, gv)


def loss_core(agent, states, actions, returns, next_states, nonterminals, debug=None, keep_graph=True):
    """The QR-DQN loss (B,) and its backward(gscale, gscale_mul=1.0), which accumulates into the online network's
    gradient arena the gradient of sum_b gscale[b] * gscale_mul * loss[b]; None without ``keep_graph``.  Injection hook:
    ``agent._inject = {"noises": (n0, n1, n2)}`` (or a list of them, one per call), the noises of the three passes in
    their order."""
    (states, actions, returns, next_states, nonterminals), inj = _loss_inputs(
        agent, states, actions, returns, next_states, nonterminals)
    on, tg = agent.online_net, agent.target_net
    B, A, N = states.shape[0], agent.action_space, agent.num_tau_samples
    dev = states.device
    noises = inj.get("noises", (None, None, None))   # a dict may carry only "shifts"
    on.reset_noise(noises[0])
    cache = {}   # conv1's pixel block matrix of next_states, shared by the two no-grad passes when they run one by one
    pair = on.trunk_pair(tg, next_states)
    f_on, f_tg = pair if pair is not None else (None, None)
    q_sel = forward(on, next_states, fresh_weights=True, col_cache=cache, feat=f_on)
    a_star = greedy_actions(agent, B, N, q_sel)
    tg.reset_noise(noises[1])
    q_tgt = forward(tg, next_states, fresh_weights=True, col_cache=cache, feat=f_tg)
    on.reset_noise(noises[2])
    keep = {} if keep_graph else None
    q_on = forward(on, states, keep=keep, fresh_weights=True)
    tau_hat = fractions(on, B)
    loss = torch.empty(B, device=dev)
    dtheta = torch.empty(N * B, device=dev)
    theta_out = target_out = None
    if debug is not None:
        theta_out = torch.empty(B, N, device=dev)
        target_out = torch.empty(B, N, device=dev)
    pi = None
    if getattr(agent, "cql", None) is not None:       # CQL: the same loss plus alpha * gap (cql.py)
        gap = torch.empty(B, device=dev) if debug is not None else None
        td, pi = cql.cql_loss(agent, B, N, N, q_on, q_tgt, tau_hat, actions, a_star, returns, nonterminals, loss, dtheta,
                              theta_out, target_out, gap)
        if debug is not None:
            debug.update(td_loss=td, gap=gap, pi=pi)
    elif getattr(agent, "mmd", None) is None:
        _quantile_loss(agent, B, N, N, q_on, q_tgt, tau_hat, actions, a_star, returns, nonterminals, loss, dtheta,
                       theta_out, target_out)
    else:                                              # MMDQN: the same particles under the MMD loss (mmd.py)
        mmd.mmd_loss(agent, B, N, q_on, q_tgt, actions, a_star, returns, nonterminals, loss, dtheta, theta_out,
                     target_out)
    if debug is not None:
        debug.update(a_star=a_star, theta=theta_out, target=target_out, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on,
                     tau=tau_hat, keep=keep)
    if keep is None:
        return loss, None
    version = getattr(on, "_noise_version", 0)

    def backward(gscale, gscale_mul=1.0):
        if getattr(on, "_noise_version", 0) != version:
            raise RuntimeError("the online network's noise was resampled between the QR-DQN loss and its backward")
        gscale = gscale.contiguous().float()
        if pi is not None:                             # CQL: the gap's gradient is dense over actions
            backward_dense(on, keep, cql.dense_grad(agent, B, N, dtheta, pi, actions, gscale, gscale_mul), on.grad_view)
            return
        dzv = torch.empty(B, N, device=dev)
        dza = torch.empty(B, A * N, device=dev)
        call("riqn_qr_head_bwd", B, A, N, ptr(dtheta), ptr(gscale), float(gscale_mul), ptr(actions), ptr(dzv), ptr(dza))
        c51._backward_below_head(on, keep, dzv, dza, on.grad_view)

    return loss, backward
