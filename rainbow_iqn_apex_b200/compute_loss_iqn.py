"""IQN loss for actor or learner -- mirror of the reference ``rainbowiqn/compute_loss_iqn.py:216-358``.

``loss_core(agent, states, actions, returns, next_states, nonterminals) -> (loss (B,), backward)`` is the contract of
every loss core (c51.loss_core, qr.loss_core).  Agent.compute_loss_actor_or_learner runs the agent's core as one autograd
node, so ``(weights * loss).mean().backward()`` (learner.py:23) runs the CUDA backward and leaves the gradients in the
parameters' ``.grad`` (views of the gradient arena), exactly where the reference leaves them.

Three network passes, in the reference's order and with a fresh noise sample before each
(:234, :255, :289): online(next_states, K) -> a*; target(next_states, N') -> targets; online(states, N).
Under a risk measure (Agent.set_risk) only the K pass draws distorted fractions beta(tau).

Munchausen-IQN (Agent.munchausen, Vieillard, Pietquin & Geist 2020) replaces the double-DQN target by a soft one with a
clipped log-policy bonus (riqn_miqn_loss_fwd_bwd).  It needs no a*, so it runs two passes: target([next_states; states], N')
as one stacked batch, then online(states, N).

FQF (Agent.fqf, Yang et al. 2019; see fqf.py) takes every fraction from the online fraction proposal instead of drawing
them: online(next_states, N at the proposed tau_hat') -> a* by the dtau'-weighted mean; target(next_states, N at the
tau_hat of states); online(states, N at tau_hat) and, without a reset, online(states, at tau_1..tau_{N-1}) for the fraction
loss (_fqf_core; its gradient is part of loss_core's backward).  num_quantile_samples and num_tau_prime_samples are not
read under FQF.

CQL (Agent.cql, cql.py) adds alpha times the log-sum-exp gap of the online pass to the plain IQN loss; its backward runs
the head's dense backward on the gradient riqn_cql_dense_grad forms.
"""
import ctypes
import math
import numbers

import torch

from . import cql
from ._lib import call, ptr

MUNCHAUSEN_DEFAULTS = {"munchausen_alpha": 0.9, "munchausen_tau": 0.03, "munchausen_l0": -1.0}   # the paper's


def check_munchausen(munchausen, alpha=0.9, entropy_tau=0.03, l0=-1.0, rainbow_only=False, risk=None):
    """Validate a Munchausen configuration.  Returns None when ``munchausen`` is off (0 / False), else the float triple
    ``(alpha, entropy_tau, l0)``: scale alpha >= 0, temperature entropy_tau > 0 and clip l0 <= 0, all finite as the kernel
    receives them (float32).  Munchausen is IQN-only (not ``rainbow_only``) and risk-neutral (``risk`` must be None, as
    model.check_risk returns it for the neutral measure).  Raises ValueError otherwise."""
    if isinstance(munchausen, bool) or (isinstance(munchausen, numbers.Integral) and munchausen in (0, 1)):
        if not munchausen:
            return None
    else:
        raise ValueError(f"munchausen must be 0 or 1, got {munchausen!r}")
    vals = []
    for name, v, ok, need in (("munchausen_alpha", alpha, lambda x: x >= 0.0, ">= 0"),
                              ("munchausen_tau", entropy_tau, lambda x: x > 0.0, "> 0"),
                              ("munchausen_l0", l0, lambda x: x <= 0.0, "<= 0")):
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError(f"{name} must be a real number, got {v!r}")
        f = ctypes.c_float(v).value
        if not (math.isfinite(f) and ok(f)):
            raise ValueError(f"{name} must be finite and {need} (as a float32), got {v!r}")
        vals.append(float(v))
    if rainbow_only:
        raise ValueError("Munchausen targets are implemented for the IQN loss; rainbow_only (C51) does not take them")
    if risk is not None:
        raise ValueError("Munchausen targets have no target action a* to act risk-sensitively on: use the neutral measure")
    return tuple(vals)


VALUE_RESCALING_DEFAULTS = {"value_rescaling_eps": 1e-3}   # R2D2's epsilon


def check_value_rescaling(value_rescaling, eps=1e-3, munchausen=None):
    """Validate a value-rescaling configuration (the transformed Bellman operator, Pohlen et al. 2018).  Returns None when
    ``value_rescaling`` is off (0 / False), else eps: finite and >= 0 as the kernels receive it (float32).  It applies to
    the IQN, FQF and C51 losses and does not combine with Munchausen targets (``munchausen`` must be None), whose soft
    target mixes log-policies of means.  Raises ValueError otherwise."""
    if isinstance(value_rescaling, bool) or (isinstance(value_rescaling, numbers.Integral) and value_rescaling in (0, 1)):
        if not value_rescaling:
            return None
    else:
        raise ValueError(f"value_rescaling must be 0 or 1, got {value_rescaling!r}")
    if isinstance(eps, bool) or not isinstance(eps, numbers.Real):
        raise ValueError(f"value_rescaling_eps must be a real number, got {eps!r}")
    f = ctypes.c_float(eps).value
    if not (math.isfinite(f) and f >= 0.0):
        raise ValueError(f"value_rescaling_eps must be finite and >= 0 (as a float32), got {eps!r}")
    if munchausen is not None:
        raise ValueError("value rescaling and Munchausen targets do not combine: set value_rescaling = 0 or munchausen = 0")
    return float(eps)


def greedy_actions(agent, batch, n, q, w=None):
    """a* (batch,) int64: the greedy actions of quantile values q (n*batch, A), quantile-major, on the mean over the n
    fractions (``w`` None, IQN) or the w-weighted sum (FQF: w = dtau).  Under value rescaling (agent.value_rescaling) q
    lives in h-space and the expectation is taken of h^-1(q), the original scale (riqn_argmax_expected_h); otherwise
    riqn_argmax_mean / riqn_argmax_weighted."""
    A = agent.action_space
    a_star = torch.empty(batch, dtype=torch.int64, device=q.device)
    eps = getattr(agent, "value_rescaling", None)
    if eps is not None:
        call("riqn_argmax_expected_h", batch, n, A, ptr(q), ptr(w), eps, None, ptr(a_star))
    elif w is None:
        call("riqn_argmax_mean", batch, n, A, ptr(q), ptr(a_star))
    else:
        call("riqn_argmax_weighted", batch, n, A, ptr(q), ptr(w), ptr(a_star))
    return a_star


def _quantile_loss(agent, B, N, Np, q_on, q_tgt, tau, actions, a_star, returns, nonterminals, loss, dtheta, theta_out,
                   target_out):
    """The double-DQN quantile-Huber loss kernel: riqn_iqn_loss_fwd_bwd, or against the transformed target
    h(R + gamma^n nt h^-1(Z)) under value rescaling (riqn_iqn_loss_fwd_bwd_h)."""
    args = (ptr(q_on), ptr(q_tgt), ptr(tau), ptr(actions), ptr(a_star), ptr(returns), ptr(nonterminals),
            float(agent.discount ** agent.n), float(agent.kappa))
    outs = (ptr(loss), ptr(dtheta), ptr(theta_out), ptr(target_out))
    eps = getattr(agent, "value_rescaling", None)
    if eps is None:
        call("riqn_iqn_loss_fwd_bwd", B, N, Np, agent.action_space, *args, *outs)
    else:
        call("riqn_iqn_loss_fwd_bwd_h", B, N, Np, agent.action_space, *args, eps, *outs)


def _loss_inputs(agent, states, actions, returns, next_states, nonterminals):
    """Every loss core's prologue.  Returns the batch on the online network's device (frames uint8 or fp32, actions int64,
    returns and nonterminals fp32) and the injection dict of this call: ``agent._inject``, or the next entry popped from it
    when it is a queue (one per call, as Actor.compute_priorities chunks), or {} without one."""
    dev = agent.online_net._flat.device

    def frames(x):
        x = x.to(dev)
        return x if x.dtype == torch.uint8 else x.float()

    inj = getattr(agent, "_inject", None)
    if isinstance(inj, list):
        inj = inj.pop(0) if inj else None
    return ((frames(states), actions.to(dev, torch.int64).contiguous(), returns.to(dev, torch.float32).contiguous(),
             frames(next_states), nonterminals.to(dev, torch.float32).contiguous()), inj or {})


def loss_core(agent, states, actions, returns, next_states, nonterminals, debug=None, keep_graph=True):
    """Forward passes + fused loss kernel.  Returns the loss (B,) and its backward(gscale, gscale_mul=1.0), which
    accumulates the gradient of sum_b gscale[b] * gscale_mul * loss[b] into the online network's gradient arena and, under
    FQF, the fraction loss's into agent.fraction_net's; None without ``keep_graph``."""
    (states, actions, returns, next_states, nonterminals), inj = _loss_inputs(
        agent, states, actions, returns, next_states, nonterminals)
    noises = inj.get("noises", (None, None, None))   # a dict may carry only "shifts"
    taus = inj.get("taus", (None, None, None))       # FQF's hook has no fractions
    batch = (agent, states, actions, returns, next_states, nonterminals)
    if getattr(agent, "munchausen", None) is not None:
        loss, dtheta, keep = _munchausen_core(*batch, noises, taus, keep_graph, debug)
    elif getattr(agent, "fqf", None) is not None:
        loss, dtheta, keep = _fqf_core(*batch, noises, keep_graph, debug)
    else:
        loss, dtheta, keep = _iqn_core(*batch, noises, taus, keep_graph, debug)
    if keep is None:
        return loss, None

    def backward(gscale, gscale_mul=1.0):
        gscale = gscale.contiguous().float()
        pi = keep.get("cql_pi")
        if pi is None:
            agent.online_net.backward_iqn(keep, dtheta, gscale, actions, gscale_mul)
        else:                 # CQL: the gap's gradient is dense over actions
            agent.online_net.check_live(keep)
            B = actions.shape[0]
            G = cql.dense_grad(agent, B, dtheta.shape[0] // B, dtheta, pi, actions, gscale, gscale_mul)
            agent.online_net.backward_iqn_dense(keep, G)
        fk = keep.get("fqf")
        if fk is not None:   # the fraction loss's surrogate of transition b is weighted like its quantile loss
            dlogits, floss = agent.fraction_net.backward(fk["fr"], fk["q_hat"], fk["q_bnd"], actions, gscale, gscale_mul,
                                                         agent.fqf[1])
            if debug is not None:
                debug.update(dlogits=dlogits, fraction_loss=floss)

    return loss, backward


def _iqn_core(agent, states, actions, returns, next_states, nonterminals, noises, taus, keep_graph, debug):
    """loss_core of plain IQN: (loss (B,), dtheta (N*B,), keep-dict for the backward or None)."""
    on, tg = agent.online_net, agent.target_net
    B = states.shape[0]
    K, Np, N = agent.num_quantile_samples, agent.num_tau_prime_samples, agent.num_tau_samples
    dev = states.device
    on.reset_noise(noises[0])                                                       # :234
    cache = {}   # conv1's pixel block matrix of next_states is shared by the online and the target pass
    # both no-grad passes read next_states: their conv trunks (noise-free weights) run as ONE stacked batch, three launches
    pair = on.trunk_pair(tg, next_states) if not on.rainbow_only else None
    f_on, f_tg = pair if pair is not None else (None, None)
    # the action selection alone acts under the agent's risk measure (IQN paper, section 3.1): a* = argmax_a Q_beta(x', a)
    q_sel, tau_sel = on.forward(next_states, K, tau=taus[0], fresh_weights=True, col_cache=cache, feat=f_on,
                                risk=getattr(agent, "risk", None))                                        # :235-237
    a_star = greedy_actions(agent, B, K, q_sel)                                     # :238-245
    tg.reset_noise(noises[1])                                                       # :255
    q_tgt, _ = tg.forward(next_states, Np, tau=taus[1], fresh_weights=True, col_cache=cache, feat=f_tg)  # :256-258
    on.reset_noise(noises[2])                                                       # :289
    keep = {} if keep_graph else None
    q_on, tau = on.forward(states, N, tau=taus[2], keep=keep, fresh_weights=True)   # :290

    loss = torch.empty(B, device=dev)
    dtheta = torch.empty(N * B, device=dev)
    theta_out = target_out = None
    if debug is not None:
        theta_out = torch.empty(B, N, device=dev)
        target_out = torch.empty(B, Np, device=dev)
    if getattr(agent, "cql", None) is None:
        _quantile_loss(agent, B, N, Np, q_on, q_tgt, tau, actions, a_star, returns, nonterminals, loss, dtheta, theta_out,
                       target_out)                                                  # :262-357
    else:                                                                           # CQL (cql.py)
        gap = torch.empty(B, device=dev) if debug is not None else None
        td, pi = cql.cql_loss(agent, B, N, Np, q_on, q_tgt, tau, actions, a_star, returns, nonterminals, loss, dtheta,
                              theta_out, target_out, gap)
        if keep is not None:
            keep["cql_pi"] = pi
        if debug is not None:
            debug.update(td_loss=td, gap=gap, pi=pi)
    if debug is not None:
        debug.update(a_star=a_star, theta=theta_out, target=target_out, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, tau=tau,
                     keep=keep, tau_sel=tau_sel)
    return loss, dtheta, keep


def _munchausen_core(agent, states, actions, returns, next_states, nonterminals, noises, taus, keep_graph, debug):
    """loss_core under Munchausen.  Injection hook: ``agent._inject = {"noises": (target, online), "taus": (tau_target
    (N'*2B, 1) over the stacked rows j*2B + [next_states; states], tau_online (N*B, 1))}``."""
    on, tg = agent.online_net, agent.target_net
    B, A = states.shape[0], agent.action_space
    Np, N = agent.num_tau_prime_samples, agent.num_tau_samples
    alpha, entropy_tau, l0 = agent.munchausen
    dev = states.device
    tg.reset_noise(noises[0])
    # one target pass over both frame sets: a 2B-sample copy, which keeps uint8 frames on the strip convolution
    q_tgt, _ = tg.forward(torch.cat((next_states, states)), Np, tau=taus[0], fresh_weights=True)
    on.reset_noise(noises[1])
    keep = {} if keep_graph else None
    q_on, tau = on.forward(states, N, tau=taus[1], keep=keep, fresh_weights=True)

    loss = torch.empty(B, device=dev)
    dtheta = torch.empty(N * B, device=dev)
    theta_out = target_out = bonus_out = None
    if debug is not None:
        theta_out = torch.empty(B, N, device=dev)
        target_out = torch.empty(B, Np, device=dev)
        bonus_out = torch.empty(B, device=dev)
    call("riqn_miqn_loss_fwd_bwd", B, N, Np, A, ptr(q_on), ptr(q_tgt), ptr(tau), ptr(actions), ptr(returns),
         ptr(nonterminals), float(agent.discount ** agent.n), float(agent.kappa), alpha, entropy_tau, l0, ptr(loss),
         ptr(dtheta), ptr(theta_out), ptr(target_out), ptr(bonus_out))
    if debug is not None:
        debug.update(bonus=bonus_out, theta=theta_out, target=target_out, q_tgt=q_tgt, q_on=q_on, tau=tau, keep=keep)
    return loss, dtheta, keep


def _fqf_core(agent, states, actions, returns, next_states, nonterminals, noises, keep_graph, debug):
    """loss_core under FQF (agent.fqf, the fraction proposal agent.fraction_net).  Injection hook: ``agent._inject =
    {"noises": (n0, n1, n2)}``; FQF draws no random fractions.

    The double-DQN step of the FQF paper's Algorithm 1, as its public implementations read it: fractions of s' from the
    online proposal select a* = argmax_a sum_i dtau'_i F(s', tau_hat'_i, a); the target network is evaluated on s' at the
    tau_hat of s; the online network at tau_hat (gradient pass) and, with the same composed weights, at the inner
    boundaries tau_1..tau_{N-1} (no-grad) for the fraction loss's W1 gradient.  With ``keep_graph`` the fraction state
    goes into ``keep["fqf"]`` for the fraction backward."""
    on, tg, fnet = agent.online_net, agent.target_net, agent.fraction_net
    B, N = states.shape[0], agent.num_tau_samples
    dev = states.device
    on.reset_noise(noises[0])
    cache = {}
    pair = on.trunk_pair(tg, next_states)
    f_on, f_tg = pair if pair is not None else (on.trunk(next_states, col_cache=cache), None)
    fr_n = fnet.propose(f_on)                                                         # fractions of s'
    q_sel, _ = on.forward(next_states, N, tau=fr_n["tau_hat"], fresh_weights=True, col_cache=cache, feat=f_on)
    a_star = greedy_actions(agent, B, N, q_sel, fr_n["dtau"])
    # the conv trunk is noise-free: the gradient pass's trunk runs here, once, and its features propose the fractions of s
    keep = {} if keep_graph else None
    feat = on.trunk(states, keep)
    fr = fnet.propose(feat)
    tg.reset_noise(noises[1])
    q_tgt, _ = tg.forward(next_states, N, tau=fr["tau_hat"], fresh_weights=True, col_cache=cache, feat=f_tg)
    on.reset_noise(noises[2])
    q_on, tau_hat = on.forward(states, N, tau=fr["tau_hat"], keep=keep, fresh_weights=True, feat=feat)
    # the inner boundaries tau_1..tau_{N-1}, quantile-major; one more row block (tau_N = 1) keeps the row count even where
    # the tensor-core embedding needs it
    nb = N - 1 if (N - 1) * B % 2 == 0 else N
    q_bnd, _ = on.forward(states, nb, tau=fr["tau"][:, 1:nb + 1].t().contiguous(), fresh_weights=True, feat=feat)

    loss = torch.empty(B, device=dev)
    dtheta = torch.empty(N * B, device=dev)
    theta_out = target_out = None
    if debug is not None:
        theta_out = torch.empty(B, N, device=dev)
        target_out = torch.empty(B, N, device=dev)
    _quantile_loss(agent, B, N, N, q_on, q_tgt, tau_hat, actions, a_star, returns, nonterminals, loss, dtheta, theta_out,
                   target_out)
    if keep is not None:
        keep["fqf"] = dict(fr=fr, q_hat=q_on, q_bnd=q_bnd)
    if debug is not None:
        debug.update(a_star=a_star, theta=theta_out, target=target_out, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, q_bnd=q_bnd,
                     tau=fr["tau"], tau_hat=fr["tau_hat"], dtau=fr["dtau"], logits=fr["logits"], entropy=fr["entropy"],
                     tau_next=fr_n["tau"], dtau_next=fr_n["dtau"], keep=keep)
    return loss, dtheta, keep
