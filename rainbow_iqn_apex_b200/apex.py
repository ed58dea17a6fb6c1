"""Ape-X topology on the GPUs of one box (BASELINE configs[3], SURVEY.md section 8e): ONE learner rank, every other
rank an actor GPU that owns a replay shard.

The reference runs this over Redis/TCP: actor processes append 1000-step buffers with initial priorities
(launch_actor.py:64-176), a single Redis server holds the whole prioritized replay (redis_memory.py), the learner
samples from it (launch_learner.py:24-50, 173-197) and publishes its weights through a Redis key every 400 steps
(learner.py:28-36, actor.py:36-39).  Here the replay is SHARDED over the actor GPUs (frames + a float64 sum-tree per
shard, the per-actor segments of redis_memory.py:160-165 become per-environment segments of the shard), and the three
exchanges ride the collective fabric (NCCL over NVLink/NVSwitch; gloo in the CPU tests):

  sample      every actor rank draws counts[s] ~ B/S transitions from its own shard (device tree descent + 7-frame window
              gather) and the windows / metadata are gathered to the learner: 3.6 MB per shard per step at B = 512;
  priorities  the learner broadcasts the B new losses; each shard applies its slice (float32 power + diff-propagating
              update, bit-exact tree arithmetic) to the leaves it sampled;
  parameters  the learner broadcasts its flat 26.9 MB parameter arena every ``publish_every`` steps (parallel.publish_parameters).

Sampling scheme (SURVEY 8e, the "simpler" variant): a fixed number of transitions per shard instead of one stratified
draw over the concatenated totals.  The probability of drawing transition i of shard s is then
P(i) = (counts[s] / B) * p_i / total_s, and the importance weights w_i = (N * P(i))^-beta / max_j w_j use exactly that
probability (N = filled capacity over all shards), so the estimator stays unbiased for any imbalance between shard totals.
With ONE shard this reduces to the reference's formula (redis_memory.py:465-475).
"""
import numpy as np
import torch
import torch.distributed as dist

from . import parallel
from .replay_memory import FRAME


def shard_counts(batch, n_shards):
    """Transitions drawn from each shard per learner step: B = sum(counts), counts differ by at most one."""
    if n_shards < 1 or batch < n_shards:
        raise ValueError("need at least one transition per shard")
    return [batch // n_shards + (1 if s < batch % n_shards else 0) for s in range(n_shards)]


def sharded_is_weights(pri, shard_of, totals, counts, filled_capacity, beta):
    """Importance weights of a batch assembled from several shards (float64, like the reference's numpy).

    pri (B,) sampled priorities, shard_of (B,) shard index of each sample, totals (S,) shard tree roots, counts (S,)
    per-shard draw counts, filled_capacity = transitions currently stored over all shards.  Non-positive priorities take
    the reference's fallback probability 1/capacity (redis_memory.py:446-456)."""
    pri = pri.to(torch.float64)
    totals = torch.as_tensor(totals, dtype=torch.float64, device=pri.device)
    counts = torch.as_tensor(counts, dtype=torch.float64, device=pri.device)
    batch = counts.sum()
    cap = torch.as_tensor(filled_capacity, dtype=torch.float64, device=pri.device)     # may be a device scalar: no host sync
    prob = (counts[shard_of] / batch) * pri / totals[shard_of]
    prob = torch.where(pri > 0, prob, (1.0 / cap).expand_as(prob))
    w = (cap * prob) ** (-float(beta))
    return w / w.max()


class ShardSample:
    """What one shard contributes to a learner batch (device tensors; fixed, padded row count n_max)."""
    FIELDS = ("tree_idx", "pri", "window", "actions", "returns", "nonterminals")

    @staticmethod
    def empty(n_max, device, history=4, n_step=3):
        L = history + n_step
        return dict(tree_idx=torch.zeros(n_max, dtype=torch.int64, device=device),
                    pri=torch.zeros(n_max, dtype=torch.float64, device=device),
                    window=torch.zeros(n_max, L, 84, 84, dtype=torch.uint8, device=device),
                    actions=torch.zeros(n_max, dtype=torch.int64, device=device),
                    returns=torch.zeros(n_max, dtype=torch.float32, device=device),
                    nonterminals=torch.zeros(n_max, dtype=torch.float32, device=device))


def packed_bytes(n_max, history=4, n_step=3):
    return n_max * ((history + n_step) * FRAME + 8 + 8 + 8 + 4 + 4) + 16


def pack(sample, stat, n_max):
    """One contiguous uint8 record per shard -- [windows | tree_idx | pri | actions | returns | nonterminals | shard total,
    filled capacity] -- so that a learner batch costs ONE gather instead of eight (every section starts 8-byte aligned)."""
    parts = [sample[k].reshape(n_max, -1).contiguous().view(torch.uint8).reshape(-1) for k in ShardSample.FIELDS]
    return torch.cat(parts + [stat.contiguous().view(torch.uint8)])


def unpack(buf, n_max, history=4, n_step=3):
    """Views into a packed record (no copies).  Returns (sample dict, stat (2,) float64)."""
    L = history + n_step
    sizes = (("window", n_max * L * FRAME, torch.uint8), ("tree_idx", n_max * 8, torch.int64), ("pri", n_max * 8, torch.float64),
             ("actions", n_max * 8, torch.int64), ("returns", n_max * 4, torch.float32), ("nonterminals", n_max * 4, torch.float32))
    out, off = {}, 0
    by_name = dict((n, (sz, dt)) for n, sz, dt in sizes)
    for k in ShardSample.FIELDS:
        sz, dt = by_name[k]
        v = buf[off:off + sz].view(dt)
        out[k] = v.view(n_max, L, 84, 84) if k == "window" else v
        off += sz
    return out, buf[off:off + 16].view(torch.float64)


def sample_shard(mem, count, n_max, samples=None):
    """Actor-rank half of a learner sample: ``count`` prioritized transitions of this shard, padded to n_max rows."""
    tr = mem.transitions
    out = ShardSample.empty(n_max, mem.device, mem.history, mem.n)
    pri, data_idx, tree_idx = tr.find_multiple_values(mem.history, mem.n, count, samples)
    window, actions, returns, nonterminals = mem.assemble_window(data_idx)
    out["tree_idx"][:count] = tree_idx
    out["pri"][:count] = pri
    out["window"][:count] = window
    out["actions"][:count] = actions
    out["returns"][:count] = returns
    out["nonterminals"][:count] = nonterminals
    return out


def assemble_batch(parts, counts, totals, filled_capacity, beta, history=4, n_step=3):
    """Learner half: concatenate the valid rows of every shard's contribution (shard-major order) and attach the
    importance weights.  Returns (shard_of, tree_idx, states, actions, returns, next_states, nonterminals, weights fp32)."""
    dev = parts[0]["pri"].device
    cat = {k: torch.cat([p[k][:c] for p, c in zip(parts, counts)]) for k in ShardSample.FIELDS}
    shard_of = torch.cat([torch.full((c,), s, dtype=torch.int64, device=dev) for s, c in enumerate(counts)])
    w = sharded_is_weights(cat["pri"], shard_of, totals, counts, filled_capacity, beta).to(torch.float32)
    win = cat["window"]
    return (shard_of, cat["tree_idx"], win[:, :history], cat["actions"], cat["returns"], win[:, n_step:n_step + history],
            cat["nonterminals"], w)


def route_priorities(mem, shard, counts, sample, loss):
    """Actor-rank half of the priority update: this shard's slice of the broadcast loss vector goes to the leaves it
    sampled (redis_memory.py:557-573 on the shard's own tree)."""
    lo = sum(counts[:shard])
    c = counts[shard]
    return mem.update_priorities(sample["tree_idx"][:c], loss[lo:lo + c])


# ------------------------------------------------------------------------------------------------ actor side
class ActorPool:
    """E environments stepped in lockstep on one actor GPU (the reference runs one environment per actor process,
    launch_actor.py:64-176; an actor GPU batches many).  Environment e owns segment e of the rank's replay shard.

      act(states)      reset_noise + batched greedy actions          launch_actor.py:76-84, actor.py:15-25
      observe(...)     append one step of every environment to the device-side rolling buffers   :97-108
      flush()          initial priorities of the buffered steps (batched loss-only passes, actor.py:41-124), max_priority
                       tail for the last n steps (launch_actor.py:127-133), append to the shard (:135-140)
    """

    def __init__(self, actor, mem, n_envs, buffer_len, replay_frequency=4):
        tr = mem.transitions
        if tr.nb_actor != n_envs:
            raise ValueError("the shard needs one segment per environment (nb_actor == n_envs)")
        self.actor, self.mem, self.E, self.L = actor, mem, n_envs, buffer_len
        dev = actor.online_net._flat.device
        h = actor.history
        self.frames = torch.zeros(n_envs, buffer_len + h - 1, 84, 84, dtype=torch.uint8, device=dev)
        self.actions = torch.zeros(n_envs, buffer_len, dtype=torch.int64, device=dev)
        self.rewards = torch.zeros(n_envs, buffer_len, dtype=torch.float32, device=dev)
        self.nonterminal = torch.ones(n_envs, buffer_len, dtype=torch.bool, device=dev)
        self.timestep = torch.zeros(n_envs, buffer_len, dtype=torch.int32, device=dev)
        self.t_env = torch.zeros(n_envs, dtype=torch.int32, device=dev)     # step inside the running episode
        self.fill = 0
        self.replay_frequency = replay_frequency
        self.write_index = np.zeros(n_envs, np.int64)                        # ring position of each segment
        self.steps = 0

    def act(self, states_u8):
        if (self.steps // self.E) % self.replay_frequency == 0:      # launch_actor.py:76-77: a new set of noisy weights
            self.actor.reset_noise()
        return self.actor.act_batch(states_u8)

    def observe(self, states_u8, actions, rewards, dones):
        """states_u8 (E, history, 84, 84): the stacks the actions were chosen from; their LAST frame is the step's frame
        (launch_actor.py:97: actor_buffer.append([timestep, state_buffer[-1], action, reward, done]))."""
        i, h = self.fill, self.actor.history
        if i == 0:
            self.frames[:, :h] = states_u8                                   # launch_actor.py:99-101
        else:
            self.frames[:, i + h - 1] = states_u8[:, -1]
        self.actions[:, i] = actions
        self.rewards[:, i] = rewards
        self.nonterminal[:, i] = ~dones
        self.timestep[:, i] = self.t_env
        self.t_env = torch.where(dones, torch.zeros_like(self.t_env), self.t_env + 1)
        self.fill += 1
        self.steps += self.E
        return self.fill >= self.L

    def initial_priorities(self):
        """actor.py:41-124 for every environment at once: (E, fill - n) initial priorities = loss ** omega."""
        a = self.actor
        n, h, L, E = a.n, a.history, self.fill, self.E
        dev = self.frames.device
        nt = self.nonterminal[:, n:L].clone()                                # actor.py:63-69: an episode end taints the
        term = ~nt                                                           # next n transitions as well
        for k in range(1, n + 1):
            nt[:, k:] &= ~term[:, :-k]
        gam = torch.tensor([a.discount ** k for k in range(n)], dtype=torch.float64, device=dev)
        rw = self.rewards[:, :L].to(torch.float64)
        T = L - n
        returns = sum(gam[k] * rw[:, k:k + T] for k in range(n)).to(torch.float32)
        e_idx, t_idx = torch.meshgrid(torch.arange(E, device=dev), torch.arange(T, device=dev), indexing="ij")
        e_idx, t_idx = e_idx.reshape(-1), t_idx.reshape(-1)
        off = torch.arange(h, device=dev)[None, :]
        pri = torch.empty(E * T, dtype=torch.float32, device=dev)
        bs = a.batch_size
        with torch.no_grad():
            for lo in range(0, E * T, bs):
                sl = slice(lo, min(lo + bs, E * T))
                e, t = e_idx[sl, None], t_idx[sl, None]
                states = self.frames[e, t + off]
                nexts = self.frames[e, t + off + n]
                loss = a.compute_loss_actor_or_learner(states, self.actions[e_idx[sl], t_idx[sl]], returns[e_idx[sl], t_idx[sl]],
                                                       nexts, nt[e_idx[sl], t_idx[sl]].to(torch.float32))
                pri[sl] = loss.detach().pow(self.mem.priority_exponent)
        return pri.view(E, T)

    def flush(self, T_actor=0):
        """launch_actor.py:116-140 for every environment; returns the number of transitions appended."""
        if self.fill <= self.actor.n:
            return 0
        tr = self.mem.transitions
        L, n, h = self.fill, self.actor.n, self.actor.history
        pri = self.initial_priorities()
        max_pri = tr.max_priority.to(torch.float32).expand(self.E, n)          # launch_actor.py:130-133
        allp = torch.cat([pri, max_pri], 1)
        for e in range(self.E):
            start = int(self.write_index[e])
            tr.append_device(e, start, self.timestep[e, :L], self.frames[e, h - 1:h - 1 + L].reshape(L, FRAME),
                             self.actions[e, :L], self.rewards[e, :L], self.nonterminal[e, :L], allp[e])
            self.write_index[e] = (start + L) % tr.actor_capacity
        tr.step_actor[:] = T_actor
        self.fill = 0
        return L * self.E


# ------------------------------------------------------------------------------------------------ collectives
class ApexTopology:
    """Rank 0 = learner, ranks 1..W-1 = actor GPUs with one shard each.  All methods are collective: every rank of the
    group calls them in the same order (lock-step learner iterations, as the reference's synchronize_actors_with_learner
    mode keeps actors and learner in step, launch_actor.py:143-153)."""

    def __init__(self, batch, group=None, publish_every=100):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if self.world < 2:
            raise ValueError("the Ape-X topology needs a learner rank and at least one actor rank")
        self.n_shards = self.world - 1
        self.counts = shard_counts(batch, self.n_shards)
        self.n_max = max(self.counts)
        self.batch = batch
        self.publish_every = publish_every
        self.is_learner = self.rank == 0
        self.shard = self.rank - 1
        self.steps = 0

    def presample(self, mem):
        """Actor ranks: draw this shard's part of the NEXT learner batch now (tree descent + window gather + packing), so that
        the collective at the start of the next step finds it ready.  Called before route() (bench.py) the draw is one step
        stale -- the reference's sampler queue holds five batches, launch_learner.py:24-50 -- and the learner never waits for
        the shards; called after route() it already sees the priorities of the step that just finished."""
        mine = sample_shard(mem, self.counts[self.shard], self.n_max)
        stat = torch.stack([mem.transitions.tree[0], torch.tensor(float(mem.transitions.get_current_capacity()),
                                                                  dtype=torch.float64, device=mem.device)])
        self._ready = (mine, pack(mine, stat, self.n_max))

    def sample_begin(self, mem=None, device=None, history=4, n_step=3):
        """First half of a learner sample: ONE gather of the packed per-shard records (on the current stream; the shards'
        parts come from presample(), or are drawn here).  Returns a ticket for sample_end()."""
        nbytes = packed_bytes(self.n_max, history, n_step)
        if self.is_learner:
            mine, dev = None, device
            if getattr(self, "_zero_rec", None) is None:
                self._zero_rec = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
            rec = self._zero_rec
        else:
            if getattr(self, "_ready", None) is None:
                self.presample(mem)
            (mine, rec), self._ready, dev = self._ready, None, mem.device
        # ONE all-gather of the packed records (ring / NVLS over NVLink: 29 MB at B = 512 on 8 ranks).  A gather to the learner
        # alone would move 1/8 of the bytes, but torch's NCCL gather is built from point-to-point sends that measured
        # 3-27 GB/s on this box (10.5 ms per step on 8 GPUs) where the collective runs at NVLink speed.
        if getattr(self, "_recv", None) is None:
            self._recv = [torch.empty(self.world * nbytes, dtype=torch.uint8, device=dev) for _ in range(2)]   # ping-pong
            self._recv_i = 0
        self._recv_i ^= 1
        flat = self._recv[self._recv_i]
        dist.all_gather_into_tensor(flat, rec, group=self.group)
        out = [flat[r * nbytes:(r + 1) * nbytes] for r in range(self.world)] if self.is_learner else None
        return dict(mine=mine, out=out, history=history, n_step=n_step)

    def sample_end(self, ticket, beta=0.4):
        """Learner: the assembled batch (see assemble_batch).  Actor ranks: their own ShardSample (kept for route())."""
        if not self.is_learner:
            return ticket["mine"]
        h, n = ticket["history"], ticket["n_step"]
        plist, stats = [], []
        for s in range(self.n_shards):
            smp, stat = unpack(ticket["out"][s + 1], self.n_max, h, n)
            plist.append(smp)
            stats.append(stat)
        st = torch.stack(stats)                            # (S, 2) on the device: shard totals and filled capacities --
        return assemble_batch(plist, self.counts, st[:, 0], st[:, 1].sum(), beta, h, n)   # the learner's host never waits

    def sample(self, mem=None, beta=0.4, device=None, history=4, n_step=3):
        return self.sample_end(self.sample_begin(mem, device, history, n_step), beta)

    def route(self, loss, mem=None, sample=None):
        """Broadcast the learner's per-transition losses; each actor rank updates the leaves it sampled."""
        dist.broadcast(loss, src=0, group=self.group)
        if not self.is_learner:
            route_priorities(mem, self.shard, self.counts, sample, loss)

    def maybe_publish(self, agent):
        """learner.py:28-36 / actor.py:36-39 every ``publish_every`` learner steps, as one broadcast of the flat arena.
        Refuses an agent under horizon_anneal on every rank, before the collective: the shards assemble their
        transitions at the fixed multi_step and discount, which an annealing learner does not train at."""
        if getattr(agent, "horizon_anneal", None) is not None:
            raise ValueError("horizon_anneal = 1 anneals the learner's update horizon n, but the Ape-X shards assemble "
                             "every transition at the fixed multi_step: train an annealing learner from its own replay "
                             "(Learner.learn / learn_and_update)")
        self.steps += 1
        if self.steps % self.publish_every == 0:
            parallel.publish_parameters(agent, src=0, group=self.group)
            return True
        return False
