"""Oracle (test infrastructure): restatement of the reference losses and learner step.

Follows
  * ``compute_loss_actor_or_learner_iqn``   /root/reference/rainbowiqn/compute_loss_iqn.py:216-358
  * C51 branch of ``Agent.compute_loss_actor_or_learner``   rainbowiqn/agent.py:77-141
  * ``Learner.learn`` (loss -> zero_grad -> (w*loss).mean().backward() -> Adam)  rainbowiqn/learner.py:14-26
  * ``torch.optim.Adam`` update rule with the reference's (lr, eps)   rainbowiqn/agent.py:43

All randomness (3 noise resets, 3 quantile draws per loss) is injected by the caller.
"""
import math

import torch

from . import network as net


def iqn_pairwise_loss(theta, target, tau, kappa=1.0):
    """Quantile-Huber loss over all (tau_i, tau'_j) pairs.      compute_loss_iqn.py:314-357

    theta (B,N) current quantile values, target (B,N') target values, tau (B,N).
    Returns loss (B,) = mean_j sum_i |tau_i - 1{delta<0}| * huber_k(delta) / kappa,
    delta[b,j,i] = target[b,j] - theta[b,i].
    """
    delta = target[:, :, None] - theta[:, None, :]  # (B, N', N)
    absd = torch.abs(delta)
    huber = (absd <= kappa).float() * 0.5 * delta ** 2 + (absd > kappa).float() * kappa * (absd - 0.5 * kappa)
    indicator = (delta < 0).float().detach()
    rho = torch.abs(tau[:, None, :] - indicator) * huber / kappa
    return rho.sum(dim=2).mean(dim=1)


def iqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals,
             noises, taus, *, n_tau, n_tau_prime, n_quantile, discount=0.99, n_step=3, kappa=1.0,
             keep=None):
    """compute_loss_actor_or_learner_iqn with injected randomness.  compute_loss_iqn.py:216-358

    ``noises`` = (online noise for the action-selection pass, target-net noise, online noise for
    the gradient pass); ``taus`` = (tau_K (K*B,1), tau' (N'*B,1), tau (N*B,1)).  The parameter
    dicts are mutated (their epsilon buffers are overwritten), as the reference's nets are.
    """
    batch = states.shape[0]
    acts = p_online["fcnoisy_z_a.bias_mu"].shape[0]
    with torch.no_grad():
        # (1) double-DQN action from the online net, K quantiles      :234-250
        net.apply_noise(p_online, noises[0])
        q_sel = net.dqn_forward_iqn(p_online, next_states, n_quantile, taus[0])
        a_star = q_sel.reshape(n_quantile, batch, acts).mean(dim=0).argmax(dim=1)
        # (2) target-net quantiles at a*, n-step target               :255-287
        net.apply_noise(p_target, noises[1])
        q_tgt = net.dqn_forward_iqn(p_target, next_states, n_tau_prime, taus[1])
        q_tgt_a = q_tgt.gather(1, a_star[:, None].repeat(n_tau_prime, 1))
        gamma_nt = ((discount ** n_step) * nonterminals[:, None]).repeat(n_tau_prime, 1)
        full = returns[:, None].repeat(n_tau_prime, 1) + gamma_nt * q_tgt_a
        target = full.reshape(n_tau_prime, batch).t()  # (B, N')
    # (3) online quantiles of the taken action (grad)                 :289-310
    net.apply_noise(p_online, noises[2])
    q_on = net.dqn_forward_iqn(p_online, states, n_tau, taus[2], keep=keep)
    theta = q_on.gather(1, actions[:, None].repeat(n_tau, 1)).reshape(n_tau, batch).t()  # (B, N)
    tau_bn = taus[2].reshape(n_tau, batch).t()
    loss = iqn_pairwise_loss(theta, target, tau_bn, kappa)
    if keep is not None:
        keep.update(a_star=a_star, target=target, theta=theta, q_sel=q_sel, q_tgt=q_tgt, q_on=q_on)
    return loss


def c51_projection(pns_a, returns, nonterminals, *, atoms=51, v_min=-10.0, v_max=10.0, gamma_n=0.99 ** 3):
    """Bellman projection of the target distributions pns_a (batch, atoms) onto the support.   agent.py:105-133

    Departs from the reference in one place: the index b is clamped to atoms - 1.  Clamping tz to [v_min, v_max] does
    not bound b = (tz - v_min) / delta_z in fp32 (v_min = -1, v_max = 1, 62 atoms: tz = v_max gives b = 61.0000038),
    and there the reference's u = atoms makes index_add_ put the mass on the next sample's atom 0, or out of range
    for the last sample.  Every b <= atoms - 1 is unchanged.
    """
    batch = pns_a.shape[0]
    support = torch.linspace(v_min, v_max, atoms)
    delta_z = (v_max - v_min) / (atoms - 1)
    tz = returns.unsqueeze(1) + nonterminals.unsqueeze(1) * gamma_n * support.unsqueeze(0)
    tz = tz.clamp(min=v_min, max=v_max)
    b = ((tz - v_min) / delta_z).clamp(max=atoms - 1)
    lo, up = b.floor().to(torch.int64), b.ceil().to(torch.int64)
    lo[(up > 0) * (lo == up)] -= 1            # agent.py:119
    up[(lo < (atoms - 1)) * (lo == up)] += 1  # agent.py:120
    m = pns_a.new_zeros(batch, atoms)
    offset = (torch.arange(batch) * atoms)[:, None].expand(batch, atoms)
    m.view(-1).index_add_(0, (lo + offset).view(-1), (pns_a * (up.float() - b)).view(-1))
    m.view(-1).index_add_(0, (up + offset).view(-1), (pns_a * (b - lo.float())).view(-1))
    return m


def c51_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, *,
             atoms=51, v_min=-10.0, v_max=10.0, discount=0.99, n_step=3, keep=None):
    """Categorical (C51) double-DQN n-step loss.                      agent.py:77-141

    ``noises`` = (online noise for log p(s,.), online noise for action selection, target noise).
    """
    batch = states.shape[0]
    acts = p_online["fcnoisy_z_a.bias_mu"].shape[0] // atoms
    support = torch.linspace(v_min, v_max, atoms)
    net.apply_noise(p_online, noises[0])
    log_ps = net.dqn_forward_c51(p_online, states, acts, atoms, log=True)
    log_ps_a = log_ps[range(batch), actions]
    with torch.no_grad():
        net.apply_noise(p_online, noises[1])
        pns = net.dqn_forward_c51(p_online, next_states, acts, atoms)
        a_star = (support.expand_as(pns) * pns).sum(2).argmax(1)
        net.apply_noise(p_target, noises[2])
        pns_a = net.dqn_forward_c51(p_target, next_states, acts, atoms)[range(batch), a_star]
        m = c51_projection(pns_a, returns, nonterminals, atoms=atoms, v_min=v_min, v_max=v_max,
                           gamma_n=discount ** n_step)
    loss = -(m * log_ps_a).sum(1)
    if keep is not None:
        keep.update(a_star=a_star, m=m, log_ps_a=log_ps_a)
    return loss


class Adam:
    """torch.optim.Adam (amsgrad=False, weight_decay=0) restated.    agent.py:43, learner.py:24

    m <- b1 m + (1-b1) g ; v <- b2 v + (1-b2) g^2 ;
    p <- p - (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
    """

    def __init__(self, keys, lr, eps, betas=(0.9, 0.999)):
        self.lr, self.eps, self.b1, self.b2 = lr, eps, betas[0], betas[1]
        self.step_count = 0
        self.m = {k: None for k in keys}
        self.v = {k: None for k in keys}

    def step(self, params, grads):
        self.step_count += 1
        bc1 = 1.0 - self.b1 ** self.step_count
        bc2 = 1.0 - self.b2 ** self.step_count
        step_size = self.lr / bc1
        for k, g in grads.items():
            if self.m[k] is None:
                self.m[k] = torch.zeros_like(g)
                self.v[k] = torch.zeros_like(g)
            self.m[k].lerp_(g, 1.0 - self.b1)
            self.v[k].mul_(self.b2).addcmul_(g, g, value=1.0 - self.b2)
            denom = (self.v[k].sqrt() / math.sqrt(bc2)).add_(self.eps)
            with torch.no_grad():
                params[k].addcdiv_(self.m[k], denom, value=-step_size)


def learn_step(p_online, p_target, adam, batch, weights, noises, taus, cfg, rainbow_only=False, keep=None):
    """Learner.learn on an already-assembled minibatch.               learner.py:14-26

    ``p_online`` must hold leaf tensors with requires_grad for trainable keys.  Returns
    (loss (B,) detached, grads dict) after applying the Adam update in place.
    """
    states, actions, returns, next_states, nonterminals = batch
    for k, t in p_online.items():
        if t.requires_grad and t.grad is not None:
            t.grad = None
    if rainbow_only:
        loss = c51_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises,
                        **cfg, keep=keep)
    else:
        loss = iqn_loss(p_online, p_target, states, actions, returns, next_states, nonterminals, noises, taus,
                        **cfg, keep=keep)
    (weights * loss).mean().backward()
    grads = {k: t.grad.detach().clone() for k, t in p_online.items() if t.requires_grad and t.grad is not None}
    adam.step(p_online, grads)
    return loss.detach(), grads
