"""IQN loss for actor or learner -- mirror of the reference ``rainbowiqn/compute_loss_iqn.py:216-358``.

Same call signature ``compute_loss_actor_or_learner_iqn(agent, states, actions, returns, next_states,
nonterminals) -> loss (B,)``; the returned tensor is differentiable w.r.t. the online network: calling
``(weights * loss).mean().backward()`` (learner.py:23) runs the CUDA backward and leaves the gradients in
the parameters' ``.grad`` (views of the gradient arena), exactly where the reference leaves them.

Three network passes, in the reference's order and with a fresh noise sample before each
(:234, :255, :289): online(next_states, K) -> a*; target(next_states, N') -> targets; online(states, N).
Under a risk measure (Agent.set_risk) only the K pass draws distorted fractions beta(tau).
"""
import torch

from ._lib import call, ptr


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
