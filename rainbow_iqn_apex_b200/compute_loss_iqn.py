"""IQN loss for actor or learner -- mirror of the reference ``rainbowiqn/compute_loss_iqn.py:216-358``.

Same call signature ``compute_loss_actor_or_learner_iqn(agent, states, actions, returns, next_states,
nonterminals) -> loss (B,)``; the returned tensor is differentiable w.r.t. the online network: calling
``(weights * loss).mean().backward()`` (learner.py:23) runs the CUDA backward and leaves the gradients in
the parameters' ``.grad`` (views of the gradient arena), exactly where the reference leaves them.

Three network passes, in the reference's order and with a fresh noise sample before each
(:234, :255, :289): online(next_states, K) -> a*; target(next_states, N') -> targets; online(states, N).
Under a risk measure (Agent.set_risk) only the K pass draws distorted fractions beta(tau).

Munchausen-IQN (Agent.munchausen, Vieillard, Pietquin & Geist 2020) replaces the double-DQN target by a soft one with a
clipped log-policy bonus (riqn_miqn_loss_fwd_bwd).  It needs no a*, so it runs two passes: target([next_states; states], N')
as one stacked batch, then online(states, N).
"""
import ctypes
import math
import numbers

import torch

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


def _as_device_inputs(agent, states, actions, returns, next_states, nonterminals):
    dev = agent.online_net._flat.device

    def frames(x):
        x = x.to(dev)
        return x if x.dtype == torch.uint8 else x.float()

    return (frames(states), actions.to(dev, torch.int64).contiguous(), returns.to(dev, torch.float32).contiguous(),
            frames(next_states), nonterminals.to(dev, torch.float32).contiguous())


def loss_core(agent, states, actions, returns, next_states, nonterminals, keep_graph=True, debug=None):
    """Forward passes + fused loss kernel.  Returns (loss (B,), dtheta (N*B,), keep-dict for backward)."""
    states, actions, returns, next_states, nonterminals = _as_device_inputs(
        agent, states, actions, returns, next_states, nonterminals)
    on, tg = agent.online_net, agent.target_net
    B = states.shape[0]
    A = agent.action_space
    K, Np, N = agent.num_quantile_samples, agent.num_tau_prime_samples, agent.num_tau_samples
    inj = getattr(agent, "_inject", None)
    if isinstance(inj, list):            # a queue of injections: one per call (Actor.compute_priorities chunks)
        inj = inj.pop(0) if inj else None
    noises = inj["noises"] if inj else (None, None, None)
    taus = inj["taus"] if inj else (None, None, None)
    dev = states.device
    if getattr(agent, "munchausen", None) is not None:
        return _munchausen_core(agent, states, actions, returns, next_states, nonterminals, noises, taus, keep_graph, debug)

    on.reset_noise(noises[0])                                                       # :234
    cache = {}   # conv1's pixel block matrix of next_states is shared by the online and the target pass
    # both no-grad passes read next_states: their conv trunks (noise-free weights) run as ONE stacked batch, three launches
    pair = on.trunk_pair(tg, next_states) if not on.rainbow_only else None
    f_on, f_tg = pair if pair is not None else (None, None)
    # the action selection alone acts under the agent's risk measure (IQN paper, section 3.1): a* = argmax_a Q_beta(x', a)
    q_sel, tau_sel = on.forward(next_states, K, tau=taus[0], fresh_weights=True, col_cache=cache, feat=f_on,
                                risk=getattr(agent, "risk", None))                                        # :235-237
    a_star = torch.empty(B, dtype=torch.int64, device=dev)
    call("riqn_argmax_mean", B, K, A, ptr(q_sel), ptr(a_star))                      # :238-245
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
    call("riqn_iqn_loss_fwd_bwd", B, N, Np, A, ptr(q_on), ptr(q_tgt), ptr(tau), ptr(actions), ptr(a_star),
         ptr(returns), ptr(nonterminals), float(agent.discount ** agent.n), float(agent.kappa), ptr(loss),
         ptr(dtheta), ptr(theta_out), ptr(target_out))                              # :262-357
    if debug is not None:
        debug.update(a_star=a_star, theta=theta_out, target=target_out, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on, tau=tau,
                     keep=keep, tau_sel=tau_sel)
    return loss, dtheta, keep, actions


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
    return loss, dtheta, keep, actions


class _IQNLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, agent, states, actions, returns, next_states, nonterminals, debug, *params):
        loss, dtheta, keep, actions = loss_core(agent, states, actions, returns, next_states, nonterminals,
                                                keep_graph=True, debug=debug)
        ctx.agent, ctx.keep, ctx.dtheta, ctx.actions = agent, keep, dtheta, actions
        ctx.n_params = len(params)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        ctx.agent.online_net.backward_iqn(ctx.keep, ctx.dtheta, grad_loss.contiguous().float(), ctx.actions)
        ctx.keep = None
        # gradients were accumulated straight into the arena behind every parameter's .grad
        return (None,) * (7 + ctx.n_params)


def compute_loss_actor_or_learner_iqn(agent, states, actions, returns, next_states, nonterminals, debug=None):
    if torch.is_grad_enabled():
        params = [p for p in agent.online_net.parameters() if p.requires_grad]
        return _IQNLoss.apply(agent, states, actions, returns, next_states, nonterminals, debug, *params)
    loss, _, _, _ = loss_core(agent, states, actions, returns, next_states, nonterminals, keep_graph=False, debug=debug)
    return loss
