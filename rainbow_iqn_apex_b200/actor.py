"""Actor -- mirror of the reference ``rainbowiqn/actor.py:11-124`` (act, act_e_greedy,
load_weight_from_redis, compute_priorities), computed by the CUDA path."""
import io
import math
import random

import numpy as np
import torch

from . import fqf
from ._lib import call, ptr
from .agent import Agent
from .compute_loss_iqn import greedy_actions
from .learner import MODEL_WEIGHT_STR


class Actor(Agent):
    _inject_act_tau = None   # parity hook: quantile fractions for the NEXT act / act_batch call (consumed once)

    def _pop_tau(self):
        tau, self._inject_act_tau = self._inject_act_tau, None
        return tau

    def _fqf_pass(self, states_u8):
        """FQF acting: fractions proposed on the trunk features, one head pass at their tau_hat.  Returns (q (N*E, A),
        dtau (N*E,)); Q = sum_i dtau_i q_i.  num_quantile_samples is not read."""
        on = self.online_net
        on._compose_weights()                  # what forward() does first; the trunk reads the refreshed images
        feat = on.trunk(states_u8)
        fr = self.fraction_net.propose(feat)
        q, _ = on.forward(states_u8, self.num_tau_samples, tau=fr["tau_hat"], fresh_weights=True, feat=feat)
        return q, fr["dtau"]

    def _fqf_argmax(self, states_u8):
        q, dtau = self._fqf_pass(states_u8)
        return greedy_actions(self, states_u8.shape[0], self.num_tau_samples, q, dtau)

    def act(self, state_buffer):
        """actor.py:15-25: greedy action from the mean over K sampled quantiles (IQN; distorted by ``self.risk``), the
        dtau-weighted mean over the proposed fractions (FQF), the mean over the N fixed-fraction quantiles (QR-DQN) or the
        expected value of the categorical distribution (C51).
        Under value rescaling each of them is the expectation of h^-1 of the network's h-space values, the return's own
        scale.  Frames go to the device as uint8; the /255 of the reference happens inside the conv kernel."""
        state = torch.from_numpy(np.stack(state_buffer).astype(np.uint8)).to(self.online_net._flat.device)
        with torch.no_grad():
            if self.rainbow_only:
                p = self.online_net(state.unsqueeze(0))
                return (p * self.acting_support).sum(2).argmax(1).item()
            if self.fqf is not None:
                return int(self._fqf_argmax(state.unsqueeze(0)).item())
            if self.qr_dqn is not None:
                q, _ = self.online_net(state.unsqueeze(0))
                return int(greedy_actions(self, 1, self.qr_dqn, q).item())
            quantile_values, _ = self.online_net(state.unsqueeze(0), self.num_quantile_samples, tau=self._pop_tau(),
                                                  risk=self.risk)
            return int(greedy_actions(self, 1, self.num_quantile_samples, quantile_values).item())

    def act_batch(self, states_u8):
        """Batched greedy actions for many environments at once: states (E, history, 84, 84) uint8 -> (E,)."""
        with torch.no_grad():
            if self.rainbow_only:
                return (self.online_net(states_u8) * self.acting_support).sum(2).argmax(1)
            if self.fqf is not None:
                return self._fqf_argmax(states_u8)
            if self.qr_dqn is not None:
                q, _ = self.online_net(states_u8)
                return greedy_actions(self, states_u8.shape[0], self.qr_dqn, q)
            q, _ = self.online_net(states_u8, self.num_quantile_samples, tau=self._pop_tau(), risk=self.risk)
            return greedy_actions(self, states_u8.shape[0], self.num_quantile_samples, q)

    def act_batch_values(self, states_u8, tau=None):
        """(E, A) mean quantile values behind act_batch (the argmax input; parity tests and epsilon schedules): Q_beta
        under ``self.risk``, the mean over K fractions beta(tau) unless ``tau`` is given.  FQF: sum_i dtau_i F(s, tau_hat_i, a)
        over the proposed fractions (``tau`` is not taken).  QR-DQN: mean_i q_i(s, a) over its N fixed fractions (``tau`` is
        not taken).  Under value rescaling: the same expectations of h^-1 of the
        quantile values, on the return's scale (riqn_argmax_expected_h)."""
        with torch.no_grad():
            E = states_u8.shape[0]
            if self.fqf is not None:
                if tau is not None:
                    raise ValueError("FQF acts on its proposed fractions: act_batch_values takes no tau")
                q, w = self._fqf_pass(states_u8)
                n = self.num_tau_samples
            elif self.qr_dqn is not None:
                if tau is not None:
                    raise ValueError("QR-DQN acts on its N fixed fractions: act_batch_values takes no tau")
                q, _ = self.online_net(states_u8)
                w, n = None, self.qr_dqn
            else:
                q, _ = self.online_net(states_u8, self.num_quantile_samples,
                                       tau=tau if tau is not None else self._pop_tau(), risk=self.risk)
                w, n = None, self.num_quantile_samples
            if self.value_rescaling is not None:
                values = torch.empty(E, self.action_space, device=q.device)
                call("riqn_argmax_expected_h", E, n, self.action_space, ptr(q), ptr(w), self.value_rescaling, ptr(values),
                     None)
                return values
            if w is not None:
                return fqf.q_values(q, w, E, n, self.action_space)
            # q rows are quantile-major (k*E + e), like the reference (model.py:149)
            return q.view(n, E, self.action_space).mean(0)

    def act_e_greedy(self, state_buffer, epsilon=0.001):
        """actor.py:27-34"""
        return random.randrange(self.action_space) if random.random() < epsilon else self.act(state_buffer)

    def load_weight_from_redis(self):
        """actor.py:36-39"""
        load_bytesIO = io.BytesIO(self.redis_servor.get(MODEL_WEIGHT_STR))
        self.online_net.load_state_dict(torch.load(load_bytesIO, map_location="cpu"))
        self.online_net.compose_weights()

    def compute_priorities(self, tab_state, tab_action, tab_reward, tab_nonterminal, priority_exponent):
        """actor.py:41-124: initial priorities = loss ** exponent for a buffer of consecutive steps."""
        len_buffer = len(tab_action)
        assert len(tab_action) == len(tab_reward) == len(tab_nonterminal) == len(tab_state) - self.history + 1
        tab_nonterminal = np.float32(tab_nonterminal[self.n:])
        for indice in np.where(tab_nonterminal == 0)[0]:                       # actor.py:67-69
            tab_nonterminal[indice + 1:(indice + self.n + 1)] = 0
        dev = self.online_net._flat.device
        actions = torch.tensor(tab_action[: len_buffer - self.n], dtype=torch.int64, device=dev)
        tab_returns = [sum(self.discount ** n * tab_reward[n + indice] for n in range(self.n))
                       for indice in range(0, len_buffer - self.n)]
        returns = torch.tensor(tab_returns, dtype=torch.float32, device=dev)
        nonterminals = torch.tensor(tab_nonterminal, dtype=torch.float32, device=dev)
        frames = torch.from_numpy(np.stack(tab_state).astype(np.uint8)).to(dev)  # (len+history-1, 84, 84)
        tab_priorities = []
        with torch.no_grad():
            for indice in range(math.ceil(len(actions) / self.batch_size)):
                lo = indice * self.batch_size
                hi = min((indice + 1) * self.batch_size, len(actions))
                idx = torch.arange(lo, hi, device=dev)[:, None] + torch.arange(self.history, device=dev)[None, :]
                states = frames[idx]                        # (b, history, 84, 84)
                next_states = frames[idx + self.n]
                loss = self.compute_loss_actor_or_learner(states, actions[lo:hi], returns[lo:hi], next_states,
                                                          nonterminals[lo:hi])
                tab_priorities.append(loss.detach().cpu().numpy())
        return np.power(np.concatenate(tab_priorities), priority_exponent)

    def flush_priorities(self, priorities_buffer, mem):
        """launch_actor.py:127-133: the last n steps of a flushed buffer have no next_state yet; they enter the replay
        with the shard's current max priority (the reference reads MAX_PRIORITY_STR from Redis; here one 8-byte
        device->host read of the tree's max_priority)."""
        max_priority = np.float64(mem.transitions.max_priority.item())
        return np.concatenate((np.asarray(priorities_buffer, np.float64), np.ones(self.n) * max_priority))

    def flush_buffer(self, mem, actor_buffer, index_actor_in_memory, id_actor, tab_state, tab_action, tab_reward,
                     tab_nonterminal, T_actor=0):
        """The buffer flush of the actor loop (launch_actor.py:116-140) against a device-resident shard: initial
        priorities from compute_priorities, max_priority tail, append.  Returns the next write index."""
        tr = mem.transitions
        if (not tr.actor_full) and (index_actor_in_memory + len(actor_buffer)) >= tr.actor_capacity:
            tr.actor_full = True                                                  # launch_actor.py:117-121
        pri = self.compute_priorities(tab_state, tab_action, tab_reward, tab_nonterminal, mem.priority_exponent)
        tr.append_actor_buffer(actor_buffer, index_actor_in_memory, id_actor, self.flush_priorities(pri, mem), T_actor)
        return (index_actor_in_memory + len(actor_buffer)) % tr.actor_capacity
