"""Actor -- mirror of the reference ``rainbowiqn/actor.py:11-124`` (act, act_e_greedy,
load_weight_from_redis, compute_priorities), computed by the CUDA path."""
import io
import math
import random

import numpy as np
import torch

from ._lib import call, ptr
from .agent import Agent
from .learner import MODEL_WEIGHT_STR


class Actor(Agent):
    _inject_act_tau = None   # parity hook: quantile fractions for the NEXT act / act_batch call (consumed once)

    def _pop_tau(self):
        tau, self._inject_act_tau = self._inject_act_tau, None
        return tau

    def act(self, state_buffer):
        """actor.py:15-25: greedy action from the mean over K sampled quantiles (IQN; distorted by ``self.risk``) or the
        expected value of the categorical distribution (C51).  Frames go to the device as uint8; the /255 of the
        reference happens inside the conv kernel."""
        state = torch.from_numpy(np.stack(state_buffer).astype(np.uint8)).to(self.online_net._flat.device)
        with torch.no_grad():
            if self.rainbow_only:
                p = self.online_net(state.unsqueeze(0))
                return (p * self.support).sum(2).argmax(1).item()
            quantile_values, _ = self.online_net(state.unsqueeze(0), self.num_quantile_samples, tau=self._pop_tau(),
                                                  risk=self.risk)
            a = torch.empty(1, dtype=torch.int64, device=state.device)
            call("riqn_argmax_mean", 1, self.num_quantile_samples, self.action_space, ptr(quantile_values), ptr(a))
            return int(a.item())

    def act_batch(self, states_u8):
        """Batched greedy actions for many environments at once: states (E, history, 84, 84) uint8 -> (E,)."""
        with torch.no_grad():
            if self.rainbow_only:
                return (self.online_net(states_u8) * self.support).sum(2).argmax(1)
            E = states_u8.shape[0]
            q, _ = self.online_net(states_u8, self.num_quantile_samples, tau=self._pop_tau(), risk=self.risk)
            a = torch.empty(E, dtype=torch.int64, device=q.device)
            call("riqn_argmax_mean", E, self.num_quantile_samples, self.action_space, ptr(q), ptr(a))
            return a

    def act_batch_values(self, states_u8, tau=None):
        """(E, A) mean quantile values behind act_batch (the argmax input; parity tests and epsilon schedules): Q_beta
        under ``self.risk``, the mean over K fractions beta(tau) unless ``tau`` is given."""
        with torch.no_grad():
            E = states_u8.shape[0]
            q, _ = self.online_net(states_u8, self.num_quantile_samples, tau=tau if tau is not None else self._pop_tau(),
                                   risk=self.risk)
            # q rows are quantile-major (k*E + e), like the reference (model.py:149)
            return q.view(self.num_quantile_samples, E, self.action_space).mean(0)

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
