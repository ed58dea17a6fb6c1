"""Device-resident prioritized replay -- mirror of ``rainbowiqn/redis_memory.py`` of the reference.

The reference keeps the sum-tree as Redis string keys and the transitions as Redis hashes, and pays a TCP
round trip per tree level (RedisSegmentTree, redis_memory.py:15-390).  Here the float64 tree, the uint8 frame
ring and the per-slot metadata live in HBM, and sampling / priority updates / transition assembly are CUDA
kernels (csrc/sumtree.cu) that reproduce the reference arithmetic bit for bit.

Class / method names follow the reference so ``launch_learner``-style loops read the same:
  ReplayMemory (= ReplayRedisMemory)      .sample_byte / .get_sample_from_mp_queue / .update_priorities
  SegmentTree  (= RedisSegmentTree)       .initialize_redis_database / .append_actor_buffer / .total /
                                          .find_multiple_values / .get_current_capacity / .check_sumtree_correct
"""
import numpy as np
import torch

from . import _lib, config
from ._lib import call, ptr

FRAME = 84 * 84


class SegmentTree:
    def __init__(self, actor_capacity, nb_actor, device, store_frames=True):
        _lib.require_device()
        self.actor_capacity = int(actor_capacity)
        self.nb_actor = int(nb_actor)
        self.full_capacity = self.actor_capacity * self.nb_actor
        self.actor_full = False
        self.memory_full = False
        if self.actor_capacity < 1 or self.nb_actor < 1:
            raise ValueError(f"actor_capacity {actor_capacity} and nb_actor {nb_actor} must be >= 1")
        self.device = torch.device(device)
        self.store_frames = store_frames
        self._rng_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        self._draws = 0
        self._draws_in_step = 0
        self._dyn = None
        self.initialize_redis_database()

    # -------------------------------------------------------------- init / bookkeeping
    def initialize_redis_database(self):
        """redis_memory.py:61-92: all priorities 0, write heads 0, max_priority 1."""
        C, dev = self.full_capacity, self.device
        self.tree = torch.zeros(2 * C - 1, dtype=torch.float64, device=dev)
        self.index_actor = torch.zeros(self.nb_actor, dtype=torch.int64, device=dev)
        self.index_actor_host = np.zeros(self.nb_actor, np.int64)
        self.is_full_actor = np.zeros(self.nb_actor, np.int64)
        self.step_actor = np.zeros(self.nb_actor, np.int64)
        self.max_priority = torch.ones(1, dtype=torch.float64, device=dev)
        if self.store_frames:
            self.frames = torch.zeros(C, FRAME, dtype=torch.uint8, device=dev)
        self.timestep = torch.zeros(C, dtype=torch.int32, device=dev)
        self.action = torch.zeros(C, dtype=torch.int32, device=dev)
        self.reward = torch.zeros(C, dtype=torch.float32, device=dev)
        self.nonterminal = torch.zeros(C, dtype=torch.uint8, device=dev)

    def get_current_capacity(self):
        """redis_memory.py:371-390"""
        if self.memory_full:
            return self.full_capacity
        capacity, full = 0, True
        for a in range(self.nb_actor):
            if int(self.is_full_actor[a]):
                capacity += self.actor_capacity
            else:
                capacity += int(self.index_actor_host[a])
                full = False
        self.memory_full = full
        return capacity

    def total(self):
        """redis_memory.py:333-335 (device -> host read of the root)."""
        return float(self.tree[0].item())

    def check_sumtree_correct(self):
        """redis_memory.py:107-136: max |left + right - parent|."""
        C = self.full_capacity
        t = self.tree
        return float((t[1:2 * C - 1:2] + t[2:2 * C - 1:2] - t[:C - 1]).abs().max().item()) if C > 1 else 0.0

    # -------------------------------------------------------------- writes
    def update_multiple_value(self, tree_idx, values, apply_pow=False, exponent=0.0):
        """redis_memory.py:139-151 (+ the np.power of :560 when apply_pow).  tree_idx int64, values fp32."""
        n = tree_idx.numel()
        if n > 4096:
            # The reference reads ALL old leaves before it applies one batch (duplicates see the same old value); the
            # kernel holds one batch of <= 4096 entries.  Splitting silently would change the result for duplicates that
            # straddle a chunk boundary, so larger batches are the caller's decision (bench.py's fill loops over chunks).
            raise ValueError("update_multiple_value takes at most 4096 entries per call (one reference batch)")
        new_pri = torch.empty(n, dtype=torch.float32, device=self.device)
        diff = torch.empty(n, dtype=torch.float64, device=self.device)
        tree_idx, values = tree_idx.contiguous(), values.contiguous()
        call("riqn_sumtree_update", n, self.full_capacity, ptr(self.tree), ptr(tree_idx), ptr(values),
             float(exponent), 1 if apply_pow else 0, ptr(new_pri), ptr(diff), ptr(self.max_priority))
        return new_pri

    def _check_append(self, id_actor, start, n):
        """Refuse, before the tree is touched, an append the frame store would refuse: n steps of segment ``id_actor``
        at ring position ``start`` must fit the segment once (more would write one slot twice in one launch)."""
        if not 0 <= int(id_actor) < self.nb_actor or not 0 <= int(start) < self.actor_capacity \
                or n > self.actor_capacity:
            raise ValueError(f"append of {n} steps at position {start} of segment {id_actor}: needs 0 <= segment < "
                             f"{self.nb_actor}, 0 <= position < {self.actor_capacity} and at most "
                             f"{self.actor_capacity} steps")

    def append_arrays(self, id_actor, start, timesteps, frames, actions, rewards, dones, priorities, T_actor=0):
        """append_actor_buffer (redis_memory.py:153-202) on arrays: n consecutive steps of actor ``id_actor``
        written at ring position ``start``; priorities (n,) already exponentiated (launch_actor.py:123-133)."""
        dev = self.device
        n = len(actions)
        cap = self.actor_capacity
        if not self.store_frames:
            raise RuntimeError("this SegmentTree was built with store_frames=False (tree only): no transition store")
        self._check_append(id_actor, start, n)
        pos = (np.arange(start, start + n) % cap) + id_actor * cap
        tree_idx = torch.from_numpy(pos + self.full_capacity - 1).to(dev)
        pri = torch.as_tensor(np.asarray(priorities, np.float32)).to(dev)
        self.update_multiple_value(tree_idx, pri)

        def dv(x, dt):
            return torch.as_tensor(np.ascontiguousarray(x)).to(dev, dt).contiguous()

        fr = frames if torch.is_tensor(frames) else torch.from_numpy(np.ascontiguousarray(frames))
        fr = fr.to(dev, torch.uint8).reshape(n, FRAME).contiguous()
        # device staging buffers are bound to names so they outlive the (asynchronous) kernel launch
        nonterminal = dv(~np.asarray(dones, np.bool_), torch.uint8)
        ts_d, ac_d, rw_d = dv(timesteps, torch.int32), dv(actions, torch.int32), dv(rewards, torch.float32)
        call("riqn_replay_append", n, cap, id_actor, int(start), ptr(fr), ptr(ts_d), ptr(ac_d), ptr(rw_d),
             ptr(nonterminal), ptr(self.frames), ptr(self.timestep), ptr(self.action), ptr(self.reward),
             ptr(self.nonterminal))
        if start + n >= cap:
            self.is_full_actor[id_actor] = 1                 # launch_actor.py:117-121
        self.index_actor_host[id_actor] = (start + n) % cap  # redis_memory.py:197
        self.index_actor[id_actor] = int(self.index_actor_host[id_actor])
        self.step_actor[id_actor] = T_actor

    def append_device(self, id_actor, start, timesteps, frames, actions, rewards, nonterminals, priorities, T_actor=None):
        """append_actor_buffer (redis_memory.py:153-202) for buffers that already live on the device (actor GPUs,
        apex.ActorPool): n consecutive steps of segment ``id_actor`` at ring position ``start``; no host staging."""
        if not self.store_frames:
            raise RuntimeError("this SegmentTree was built with store_frames=False (tree only): no transition store")
        dev, cap = self.device, self.actor_capacity
        n = int(actions.numel())
        self._check_append(id_actor, start, n)
        pos = (torch.arange(start, start + n, device=dev) % cap) + id_actor * cap
        self.update_multiple_value(pos + self.full_capacity - 1, priorities.to(dev, torch.float32).contiguous())
        fr = frames.to(dev, torch.uint8).reshape(n, FRAME).contiguous()
        nt = nonterminals.to(dev, torch.uint8).contiguous()
        ts_d, ac_d = timesteps.to(dev, torch.int32).contiguous(), actions.to(dev, torch.int32).contiguous()
        rw_d = rewards.to(dev, torch.float32).contiguous()
        call("riqn_replay_append", n, cap, id_actor, int(start), ptr(fr), ptr(ts_d), ptr(ac_d), ptr(rw_d), ptr(nt),
             ptr(self.frames), ptr(self.timestep), ptr(self.action), ptr(self.reward), ptr(self.nonterminal))
        if start + n >= cap:
            self.is_full_actor[id_actor] = 1
        self.index_actor_host[id_actor] = (start + n) % cap
        self.index_actor[id_actor] = int(self.index_actor_host[id_actor])
        if T_actor is not None:
            self.step_actor[id_actor] = T_actor

    def append_actor_buffer(self, actor_buffer, actor_index_in_replay_memory, id_actor, priorities, T_actor):
        """redis_memory.py:153-202 with the reference's list-of-[timestep, frame, action, reward, done] buffer."""
        ts = np.array([b[0] for b in actor_buffer], np.int64)
        fr = np.stack([np.asarray(b[1], np.uint8).reshape(84, 84) for b in actor_buffer])
        ac = np.array([b[2] for b in actor_buffer], np.int64)
        rw = np.array([b[3] for b in actor_buffer], np.float32)
        dn = np.array([bool(b[4]) for b in actor_buffer])
        self.append_arrays(id_actor, actor_index_in_replay_memory, ts, fr, ac, rw, dn, priorities, T_actor)

    # -------------------------------------------------------------- sampling
    def find_multiple_values(self, history_length, n_step_length, batch_size, samples=None, hz=None):
        """redis_memory.py:267-331.  Returns device tensors (priorities f64, data_idx, tree_idx) and the
        device-resident total is read by the weights kernel; ``samples`` (float64) injects the stratified
        values, otherwise they are drawn on the device.  ``hz``: a dynstate.HorizonState whose n the valid-index shift
        reads on the device in place of ``n_step_length`` (riqn_sumtree_sample_horizon), or None."""
        dev = self.device
        if samples is None:
            samples = torch.empty(batch_size, dtype=torch.float64, device=dev)
            dyn = self._dyn
            idx = self._draws_in_step if dyn is not None else self._draws
            call("riqn_sumtree_stratified", batch_size, self._rng_seed, idx + (0 if dyn is not None else 1 << 39), ptr(self.tree), ptr(samples),
                 dyn.ptr() if dyn else None)
            self._draws += 1
            self._draws_in_step += 1
        else:
            samples = torch.as_tensor(samples, dtype=torch.float64).to(dev).contiguous()
        tree_idx = torch.empty(batch_size, dtype=torch.int64, device=dev)
        data_idx = torch.empty(batch_size, dtype=torch.int64, device=dev)
        pri = torch.empty(batch_size, dtype=torch.float64, device=dev)
        if hz is None:
            call("riqn_sumtree_sample", batch_size, self.full_capacity, self.actor_capacity, ptr(self.tree), ptr(samples),
                 ptr(self.index_actor), history_length, n_step_length, ptr(tree_idx), ptr(data_idx), ptr(pri))
        else:
            call("riqn_sumtree_sample_horizon", batch_size, self.full_capacity, self.actor_capacity, ptr(self.tree),
                 ptr(samples), ptr(self.index_actor), history_length, hz.n_max, hz.ptr(), ptr(tree_idx), ptr(data_idx),
                 ptr(pri))
        return pri, data_idx, tree_idx


class ReplayMemory:
    """ReplayRedisMemory (redis_memory.py:393-573) with the Redis server replaced by HBM."""

    def __init__(self, args, redis_servor=None, store_frames=True):
        self.device = args.device
        self.capacity = args.actor_capacity * args.nb_actor
        self.history = args.history_length
        self.discount = args.discount
        self.n = args.multi_step
        self.priority_weight = args.priority_weight      # beta, annealed by the caller (launch_learner.py:167-169)
        self.priority_exponent = args.priority_exponent
        self.batch_size = getattr(args, "batch_size", 32)
        self.t = 0
        self.transitions = SegmentTree(args.actor_capacity, args.nb_actor, args.device, store_frames)
        self._gamma_pow = torch.tensor([self.discount ** k for k in range(self.n)], dtype=torch.float64,
                                       device=self.device)
        self.last_nonpositive = None
        # DQfD demonstrations: optional args fields (absent from the reference's namespace: none).  The last D segments,
        # data indices >= (nb_actor - D) * actor_capacity, hold them; the sampler's valid-index shift never leaves a
        # segment, so a sampled row is a demonstration exactly when its tree index is >= demo_leaf.  update_priorities
        # adds demo_priority_bonus (DQfD's eps_d) to their new priorities
        self.demo_segments, self.demo_priority_bonus = config.read_demo(args)
        self.demo_leaf = None
        if self.demo_segments > 0:
            self.demo_leaf = (args.nb_actor - self.demo_segments) * args.actor_capacity + self.capacity - 1

    def sample_indices(self, batch_size, samples=None, hz=None):
        """find_multiple_values + importance weights (redis_memory.py:424-475), including the reference's resample loop:
        while some sampled priority is <= 0 (a slot next to a write head of a partially filled segment) the batch is
        drawn again, up to 10 more times, 11 draws in all (:432-438); after that -- and always inside a captured CUDA
        graph or with injected ``samples``, where a host-side retry is impossible -- the reference's final fallback
        applies (:446-456: those probabilities become 1/capacity).  The count of such samples is left in
        ``last_nonpositive`` (device int).  ``hz``: see SegmentTree.find_multiple_values."""
        tr = self.transitions
        retry = samples is None and tr._dyn is None and not torch.cuda.is_current_stream_capturing()
        for attempt in range(11 if retry else 1):
            pri, data_idx, tree_idx = tr.find_multiple_values(self.history, self.n, batch_size, samples, hz)
            w64 = torch.empty(batch_size, dtype=torch.float64, device=self.device)
            w32 = torch.empty(batch_size, dtype=torch.float32, device=self.device)
            self.last_nonpositive = torch.empty(1, dtype=torch.int32, device=self.device)    # written (not accumulated) by the kernel
            call("riqn_sumtree_is_weights", batch_size, ptr(tr.tree), ptr(pri), float(tr.get_current_capacity()),
                 float(self.priority_weight), ptr(w64), ptr(w32), ptr(self.last_nonpositive),
                 tr._dyn.ptr() if tr._dyn is not None else None)
            if not retry or int(self.last_nonpositive.item()) == 0:       # one 4-byte read per eager sample
                break
        return tree_idx, data_idx, pri, w64, w32

    def assemble(self, data_idx):
        """get_byte_multiple_transition + get_torch_tensor_from_byte_transition (:347-369, :479-541)."""
        window, actions, returns, nonterminals = self.assemble_window(data_idx)
        return window[:, :self.history], actions, returns, window[:, self.n:self.n + self.history], nonterminals

    def assemble_window(self, data_idx):
        """The (B, history + n, 84, 84) uint8 frame window itself (states = window[:, :history], next_states =
        window[:, n:n+history]) with actions / returns / nonterminals: what a replay shard ships to the learner rank."""
        tr = self.transitions
        if not tr.store_frames:
            raise RuntimeError("this replay was built with store_frames=False (tree only): nothing to assemble")
        B = data_idx.numel()
        L = self.history + self.n
        window = torch.empty(B, L, 84, 84, dtype=torch.uint8, device=self.device)
        actions = torch.empty(B, dtype=torch.int64, device=self.device)
        returns = torch.empty(B, dtype=torch.float32, device=self.device)
        nonterminals = torch.empty(B, dtype=torch.float32, device=self.device)
        call("riqn_frame_gather", B, tr.actor_capacity, self.history, self.n, ptr(data_idx), ptr(tr.frames),
             ptr(tr.timestep), ptr(tr.action), ptr(tr.reward), ptr(tr.nonterminal), ptr(self._gamma_pow), ptr(window),
             ptr(actions), ptr(returns), ptr(nonterminals))
        return window, actions, returns, nonterminals

    def assemble_horizon(self, data_idx, hz):
        """assemble_window at the n of the dynstate.HorizonState ``hz``, read on the device (riqn_frame_gather_horizon):
        frames (B, 2 * history, 84, 84) uint8, states = frames[:, :history] and next_states = frames[:, history:], with
        actions, returns, the 0/1 nonterminals and discounts = fl32(gamma^n) * nonterminals."""
        tr = self.transitions
        if not tr.store_frames:
            raise RuntimeError("this replay was built with store_frames=False (tree only): nothing to assemble")
        B = data_idx.numel()
        frames = torch.empty(B, 2 * self.history, 84, 84, dtype=torch.uint8, device=self.device)
        actions = torch.empty(B, dtype=torch.int64, device=self.device)
        returns, nonterminals, discounts = (torch.empty(B, dtype=torch.float32, device=self.device) for _ in range(3))
        call("riqn_frame_gather_horizon", B, tr.actor_capacity, self.history, hz.n_max, ptr(data_idx), ptr(tr.frames),
             ptr(tr.timestep), ptr(tr.action), ptr(tr.reward), ptr(tr.nonterminal), hz.ptr(), ptr(frames), ptr(actions),
             ptr(returns), ptr(nonterminals), ptr(discounts))
        return frames, actions, returns, nonterminals, discounts

    def sample_horizon(self, batch_size, hz):
        """sample() at the update horizon the dynstate.HorizonState ``hz`` holds on the device (a learner under
        horizon_anneal): (tree_idxs, states u8, actions, returns, next_states u8, discounts, weights), the sampler's shift
        and the transitions at hz's n, and discounts = fl32(gamma^n) * nonterminal in place of the nonterminals."""
        tree_idx, data_idx, _, _, w32 = self.sample_indices(batch_size, hz=hz)
        frames, actions, returns, _, discounts = self.assemble_horizon(data_idx, hz)
        h = self.history
        return tree_idx, frames[:, :h], actions, returns, frames[:, h:], discounts, w32

    def sample_sequence(self, tree_idx, K):
        """SPR's K-step sequence of the sampled tree indices ``tree_idx`` (data index tree_idx - capacity + 1), as device
        tensors (riqn_sequence_gather): window (B, history + K, 84, 84) uint8 whose first history frames are the
        sample's states bit for bit, actions (B, K) int64 a_t .. a_{t+K-1} (actions[:, 0] is the sample's), and valid
        (B, K) uint8, valid[:, k-1] = 0 where s_{t+k} crosses a terminal or the segment's write head.  The sampler is not
        changed: steps it did not guarantee are masked, never resampled."""
        tr = self.transitions
        if not tr.store_frames:
            raise RuntimeError("this replay was built with store_frames=False (tree only): nothing to assemble")
        data_idx = (torch.as_tensor(tree_idx).to(self.device, torch.int64) - (self.capacity - 1)).contiguous()
        B = data_idx.numel()
        window = torch.empty(B, self.history + K, 84, 84, dtype=torch.uint8, device=self.device)
        actions = torch.empty(B, K, dtype=torch.int64, device=self.device)
        valid = torch.empty(B, K, dtype=torch.uint8, device=self.device)
        call("riqn_sequence_gather", B, tr.actor_capacity, self.history, K, ptr(data_idx), ptr(tr.index_actor),
             ptr(tr.frames), ptr(tr.timestep), ptr(tr.action), ptr(tr.nonterminal), ptr(window), ptr(actions), ptr(valid))
        return window, actions, valid

    def sample(self, batch_size, samples=None):
        """Everything Learner.learn needs, as device tensors:
        (tree_idxs, states u8, actions, returns, next_states u8, nonterminals, weights)."""
        tree_idx, data_idx, _, _, w32 = self.sample_indices(batch_size, samples)
        states, actions, returns, next_states, nonterminals = self.assemble(data_idx)
        return tree_idx, states, actions, returns, next_states, nonterminals, w32

    def sample_byte(self, batch_size):
        """redis_memory.py:465-475.  The reference returns raw Redis bytes for a subprocess queue; the device
        path returns (tree_idxs, data_idx, weights) -- ``get_sample_from_mp_queue`` assembles from data_idx."""
        tree_idx, data_idx, _, w64, _ = self.sample_indices(batch_size)
        return tree_idx, data_idx, w64

    def get_sample_from_mp_queue(self, mp_queue):
        """redis_memory.py:545-554.  ``mp_queue`` may be None (sample on the device now), or yield either an
        assembled 7-tuple or a (tree_idxs, data_idx, weights) triple from ``sample_byte``."""
        if mp_queue is None:
            return self.sample(self.batch_size)
        item = mp_queue.get()
        if len(item) == 7:
            return tuple(item)
        tree_idxs, data_idx, weights = item
        assert len(tree_idxs) == len(weights)
        states, actions, returns, next_states, nonterminals = self.assemble(torch.as_tensor(data_idx).to(self.device))
        weights = torch.as_tensor(weights).to(self.device, torch.float32)
        return tree_idxs, states, actions, returns, next_states, nonterminals, weights

    def demo_mask(self, tree_idx):
        """The (B,) uint8 demonstration flags of the sampled tree indices: 1 where tree_idx >= demo_leaf.  None when the
        memory holds no demonstration segments."""
        if self.demo_leaf is None:
            return None
        return torch.ge(torch.as_tensor(tree_idx).to(self.device), self.demo_leaf).view(torch.uint8)

    def update_priorities(self, idxs, priorities):
        """redis_memory.py:557-573: priorities = loss ** priority_exponent, then the diff-propagating update; with
        demonstration segments and a bonus eps_d > 0, the demonstrations' priorities are fl32(loss ** omega + eps_d)
        (riqn_sumtree_update_demo)."""
        idxs = torch.as_tensor(idxs).to(self.device, torch.int64).contiguous()
        priorities = torch.as_tensor(priorities).detach().to(self.device, torch.float32).contiguous()
        tr = self.transitions
        if self.demo_leaf is None or self.demo_priority_bonus == 0.0:
            return tr.update_multiple_value(idxs, priorities, apply_pow=True, exponent=self.priority_exponent)
        n = idxs.numel()
        if n > 4096:
            raise ValueError("update_priorities takes at most 4096 entries per call (one reference batch)")
        new_pri = torch.empty(n, dtype=torch.float32, device=self.device)
        diff = torch.empty(n, dtype=torch.float64, device=self.device)
        call("riqn_sumtree_update_demo", n, tr.full_capacity, ptr(tr.tree), ptr(idxs), ptr(priorities),
             float(self.priority_exponent), 1, ptr(new_pri), ptr(diff), ptr(tr.max_priority), self.demo_leaf,
             self.demo_priority_bonus)
        return new_pri


# reference spellings
ReplayRedisMemory = ReplayMemory
RedisSegmentTree = SegmentTree
