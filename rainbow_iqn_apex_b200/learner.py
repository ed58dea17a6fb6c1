"""Learner -- mirror of the reference ``rainbowiqn/learner.py:8-36``.

``learn(mem, mp_queue) -> (idxs, loss)`` performs the reference's sequence
sample -> loss -> zero_grad -> (weights*loss).mean().backward() -> Adam.step (learner.py:14-26) with the
backward driven directly (no autograd graph) and the IS weights folded into the upstream gradient
gscale[b] = weights[b] / B.  ``north_star`` spellings Agent.learn / Agent.update_target are aliased.

Every step also zeroes, fills, (all-reduces) and steps the arena of each side network (Agent.sides).  A user's own loop
around ``loss.backward()`` gets FQF's fraction gradients from that backward too, and must zero and step that arena itself.
Under CURL (curl.py) the step also contrasts the gradient pass's trunk features with a momentum encoder's, and after the
Adam steps moves the momentum encoder towards the online trunk and projection.  Under SPR (spr.py) it gathers the sampled
transitions' K-step sequences (ReplayMemory.sample_sequence) and predicts their latents; entry points that receive an
already assembled minibatch without its sequence (learn_on_batch without ``sequence``, the batch and learn graphs,
learn_on_host_batch) refuse.  Each rank contrasts or predicts its own local batch.

Under resets (reset.py) ``updates`` counts the optimiser steps this learner has run, and after every reset_interval-th
update the step entry points (learn_on_batch and learn through it, learn_and_update eager or replayed, learn_on_graph,
learn_on_host_batch) call reset_networks() before they return: one eager launch per arena between two steps, never
inside a captured graph.  The warm-up steps of a capture count; a reset that falls due during them runs when the
enable_* call returns (one, however many fell due).  reset_networks() is public, for a schedule of one's own or a loop
of one's own around loss.backward().

Under target_ema (target.py) every step ends with the EMA of the target network, after the optimisers and the sides'
after_step hooks, eagerly and in every captured graph.  Under adamw every optimiser is AdamW; a captured graph holds
each one's decay 1 - lr * weight_decay by value, so a replay after an lr or weight_decay change raises.

Under horizon_anneal (horizon.py) the learner anneals its update horizon n and discount gamma over the updates since the
last reset (or construction; a resumed run starts the schedule again).  Before every step that samples from a replay
(learn(mem, None) and learn_and_update, eager, warmed up or replayed from enable_cuda_graph's graph) it writes that
step's (n, gamma) into its device horizon state, and the step samples through ReplayMemory.sample_horizon and hands the
loss core the per-transition discounts with gamma^n = 1.  horizon() gives the next step's (n, gamma); learn_on_batch on
a batch the caller assembled at horizon() trains at gamma^n of horizon() with the batch's own nonterminals.  The batch and
learn graphs and a queued batch (learn with an mp_queue) take batches assembled at a fixed n, and refuse.
"""
import contextlib
import io
from typing import NamedTuple

import torch

from . import augment, horizon, reset, target
from .agent import Agent
from .dynstate import DynState, HorizonState

MODEL_WEIGHT_STR = "model_weight"      # rainbowiqn/constants.py:18
STEP_LEARNER_STR = "step_learner:"     # rainbowiqn/constants.py:14


class _StepGraph(NamedTuple):
    """A captured learner step."""
    graph: object        # torch.cuda.CUDAGraph of the step, or of its part before the all-reduce when that stays eager
    post: object         # the graph of Adam and the priority update after an eager all-reduce, or None
    mem: object          # the replay memory whose fill and beta every replay writes into the struct, or None
    inputs: tuple        # the static input buffers a replay copies its batch into, or None (the step samples them)
    out: object          # the static outputs, overwritten by every replay
    decay: tuple         # every optimiser's AdamW decay factor (Adam.decay) that the graph holds by value


class Learner(Agent):
    def __init__(self, args, action_space, redis_servor):
        self._graphs = {}          # captured step graphs by kind: "replay", "batch", "learn"
        super().__init__(args, action_space, redis_servor)
        self.process_group = None  # set by parallel.make_data_parallel
        self._dp_stream = self._dp_tail = None
        self.overlap_allreduce = True   # data parallel: start the NoisyLinear-gradient all-reduce inside the backward
        self.capture_collectives = True  # data parallel: capture the all-reduces in the step graphs (enable_cuda_graph)
        self._dyn = None           # the riqn_dyn_state every step graph of this learner reads (built at the first capture)
        self._dyn_on = False       # the struct is attached: a step is being warmed up or captured
        self._horizon = self._horizon_base = None
        if self.horizon_anneal is not None:
            # the riqn_horizon_state every annealed step reads, and the updates count at the schedule's start
            self._horizon = HorizonState(self.online_net._flat.device, max(self.horizon_anneal[0], self.n))
            self._horizon_base = self.updates

    def learn(self, mem_redis, mp_queue):
        if self._horizon is not None:
            if mp_queue is not None:
                self._refuse_anneal("learn with an mp_queue")
            self._horizon.write(*self.horizon())
        sample = self._sample(mem_redis, mp_queue)
        idxs, states, actions, returns, next_states, nonterminals, weights = sample
        with self._feeding_discounts():
            loss = self.learn_on_batch(states, actions, returns, next_states, nonterminals, weights,
                                       demo=self._demo_mask(mem_redis, idxs), sequence=self._sequence(mem_redis, idxs))
        return idxs, loss

    def _sample(self, mem, mp_queue):
        """The step's sample: ReplayMemory.get_sample_from_mp_queue, or under horizon_anneal ReplayMemory.sample_horizon at
        the horizon state's (n, gamma), with the discounts in the nonterminals' place."""
        if self._horizon is None:
            return mem.get_sample_from_mp_queue(mp_queue)
        return mem.sample_horizon(mem.batch_size, self._horizon)

    @contextlib.contextmanager
    def _feeding_discounts(self):
        """Under horizon_anneal, the loss cores run inside this with gamma^n = 1 (Agent.gamma_n): the step's sample carries
        the per-transition discounts in the nonterminals' place."""
        self._discounts_fed = self._horizon is not None
        try:
            yield
        finally:
            self._discounts_fed = False

    def horizon(self):
        """(n, gamma) of the next step: under horizon_anneal the schedule's (horizon.py) at the updates since the last
        reset, otherwise (multi_step, discount).  For logging, and for callers that assemble learn_on_batch's batch."""
        return self._horizon_at(0)

    def _horizon_at(self, ahead):
        """(n, gamma) of the step ``ahead`` steps after the next (a capture's warm-up steps count updates only at its
        end)."""
        if self._horizon is None:
            return super().horizon()
        return horizon.schedule(self.horizon_anneal, self.n, self.discount, self.updates - self._horizon_base + ahead)

    def _refuse_anneal(self, what):
        if self._horizon is not None:
            raise ValueError(f"horizon_anneal = 1 anneals the update horizon n from step to step: {what} takes batches "
                             "assembled at a fixed n; step the learner with learn(mem, None) / learn_and_update (and "
                             "enable_cuda_graph), or pass learn_on_batch a batch assembled at horizon()")

    def _demo_mask(self, mem, idxs):
        """Under DQfD, the demonstration flags of the sampled tree indices ``idxs`` (ReplayMemory.demo_mask: None when the
        memory holds no demonstrations); None otherwise."""
        return mem.demo_mask(idxs) if self.dqfd is not None else None

    def _sequence(self, mem, idxs):
        """Under SPR, the K-step sequences of the sampled tree indices ``idxs`` (ReplayMemory.sample_sequence); None
        otherwise."""
        return mem.sample_sequence(idxs, self.spr[0]) if self.spr is not None else None

    def _refuse_spr(self, what):
        if self.spr is not None:
            raise ValueError(f"spr = 1 predicts the K states after each sampled one: {what} receives an assembled "
                             "minibatch without its sequences; step an SPR learner with learn / learn_and_update (and "
                             "enable_cuda_graph), or pass learn_on_batch the sequence= of ReplayMemory.sample_sequence")

    def learn_on_batch(self, states, actions, returns, next_states, nonterminals, weights, demo=None, sequence=None):
        """learner.py:18-24 on an already assembled minibatch.  Returns the per-transition loss (B,).  ``demo``: the
        DQfD demonstration flags (B,), or None.  ``sequence``: under SPR (required there), the minibatch's
        ReplayMemory.sample_sequence."""
        if sequence is None:
            self._refuse_spr("learn_on_batch without sequence=")
        loss = self.compute_gradients(states, actions, returns, next_states, nonterminals, weights, demo=demo,
                                      sequence=sequence)
        self.apply_gradients()
        self._count_updates(1)
        return loss

    def reset_networks(self):
        """Reset the networks now (reset.py): redraw the last layers, shrink and perturb the trunk and SPR's transition
        model by reset_shrink (its default, 0.5, when reset = 0), restart every optimiser of a reset arena, and count
        the reset (the next one draws from the next streams)."""
        reset.reset(self, self.resets)
        self.resets += 1
        if self._horizon is not None:
            self._horizon_base = self.updates        # the horizon schedule starts again

    def _count_updates(self, n):
        """Count ``n`` optimiser steps; under resets, reset once if one of them completed a reset_interval."""
        before = self.updates
        self.updates += n
        if self.reset is not None and self.updates // self.reset[0] > before // self.reset[0]:
            self.reset_networks()

    def _start_tail_allreduce(self, offset):
        """Called by DQN.backward_iqn once the NoisyLinear gradients (arena[offset:], 25.8 of 26.9 MB) are final: their
        all-reduce runs on a side stream under the rest of the backward (head data gradient, embedding and trunk backward)."""
        if self.process_group is None:
            return
        if getattr(self, "_dp_stream", None) is None:
            self._dp_stream = torch.cuda.Stream()
        self._dp_stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._dp_stream):
            torch.distributed.all_reduce(self.online_net._flat_grad[offset:], group=self.process_group)
        self._dp_tail = offset

    def apply_gradients(self):
        """Gradient all-reduce (data-parallel replicas) + Adam.  learner.py:24"""
        if self.process_group is not None:
            self._allreduce_all_grads()
        self._step_optimisers()

    def _allreduce_all_grads(self):
        """Every gradient arena, one all-reduce each, in _trained_nets order (FQF: the fraction arena, 0.8 MB at N = 64,
        after the DQN's).  When the backward already started the online arena's tail (_start_tail_allreduce), only its
        head is left: reduce it, then join the side stream."""
        for net in self._trained_nets():
            if net is self.online_net and self._dp_tail is not None:
                torch.distributed.all_reduce(net._flat_grad[:self._dp_tail], group=self.process_group)
                torch.cuda.current_stream().wait_stream(self._dp_stream)
                self._dp_tail = None
            else:
                torch.distributed.all_reduce(net._flat_grad, group=self.process_group)

    def _trained_nets(self):
        """The networks whose gradient arenas a step fills: the online network, then the sides'."""
        return (self.online_net,) + tuple(side.net for side in self.sides)

    def _optimisers(self):
        return (self.optimiser,) + tuple(side.optimiser for side in self.sides)

    def _step_optimisers(self):
        for o in self._optimisers():
            o.step()
        for side in self.sides:
            if side.after_step is not None:
                side.after_step(self)
        target.update(self)

    def _write_dyn(self, mem, ahead=0):
        """Stage the next step's device scalars: the Adam bias corrections of every optimiser, and the fill and beta of the
        replay memory ``mem`` ((1, 0) for a step without one); under horizon_anneal, the (n, gamma) of the step ``ahead``
        steps after the next (_horizon_at)."""
        nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
        more = tuple(o.bias_corrections(o._step + 1) for o in self._optimisers()[1:])
        capacity, beta = (1.0, 0.0) if mem is None else (mem.transitions.get_current_capacity(), mem.priority_weight)
        self._dyn.write(nss, sbc, capacity, beta, *more)
        if self._horizon is not None:
            self._horizon.write(*self._horizon_at(ahead))

    def compute_gradients(self, states, actions, returns, next_states, nonterminals, weights, debug=None, demo=None,
                          sequence=None):
        """loss -> zero_grad -> backward of (weights*loss).mean()   (learner.py:18-23); gradients land in the arenas.
        ``debug``: dict that receives the loss core's intermediates (self.loss_core), with random_shift the shifts and
        the shifted frames (_shift_frames), under CURL curl_shifts, z_a, z_k, logits, curl_loss (the per-row InfoNCE
        terms, (B,)) and dfeat_curl, and under SPR spr_shifts, spr_targets, spr_latents, spr_pred, spr_loss (the
        per-sample sums of the masked negative cosines, (B,)) and dfeat_spr.  ``demo``: the DQfD demonstration flags (B,)
        uint8 / bool, or None.  ``sequence``: under SPR (required there), ReplayMemory.sample_sequence of the batch."""
        on = self.online_net
        if sequence is None:
            self._refuse_spr("compute_gradients without sequence=")
        weights = weights.to(on._flat.device, torch.float32)
        raw_states = states
        if self.random_shift is not None:
            states, next_states = self._shift_frames(states, next_states, debug)
        # CURL's or SPR's feature gradient joins the loss core's in the trunk backward (config.read allows one of them)
        terms = [side.trunk_term(self, raw_states, sequence, debug) for side in self.sides if side.trunk_term is not None]
        assert len(terms) <= 1, "at most one side network adds a trunk term"
        loss, bw = self.loss_core(self, states, actions, returns, next_states, nonterminals, debug=debug, demo=demo)
        for net in self._trained_nets():                                        # learner.py:22
            net.zero_grad()
        # data parallel: DQN.backward_iqn starts the all-reduce of the NoisyLinear gradients as soon as they are final
        on._grads_ready_hook = self._start_tail_allreduce if (self.process_group is not None and self.overlap_allreduce) else None
        if terms:
            on._trunk_addend = terms[0]
        try:
            bw(weights, 1.0 / weights.shape[0])                                 # learner.py:23 (.mean())
        finally:
            on._grads_ready_hook = on._trunk_addend = None
        return loss

    def _shift_frames(self, states, next_states, debug=None):
        """Random-shift augmentation of one step's frames (DrQ with K = M = 1): independent shifts of s_t and s_{t+n}, one
        per sample, drawn on the device (augment.draw_shifts) or taken from the step's injection dict (``"shifts":
        (shifts_states, shifts_next_states)``; a list of dicts is peeked, the loss pops it), and ONE riqn_random_shift
        launch into a [s_{t+n}; s_t] buffer.  Every pass of the loss over a frame set then reads the same shifted frames.
        The shifts of the last step stay in self._shifts ((2B, 2): rows [0, B) for s_{t+n}; a graph's static buffer)."""
        on = self.online_net
        B = states.shape[0]
        given = augment.injection(self).get("shifts")
        if given is None:
            shifts = augment.draw_shifts(on, 2 * B, self.random_shift)
        else:
            shifts = torch.cat([torch.as_tensor(s, dtype=torch.int32).reshape(B, 2) for s in (given[1], given[0])])
            shifts = shifts.to(on._flat.device)
        next_states, states = augment.random_shift(next_states, states, shifts)
        self._shifts = shifts
        if debug is not None:
            debug.update(shifts=(shifts[B:], shifts[:B]), shifted_states=states, shifted_next_states=next_states)
        return states, next_states

    # ------------------------------------------------------------------ whole step: sample -> learn -> priority update
    def learn_and_update(self, mem):
        """One learner iteration against a device-resident ReplayMemory: prioritized sample, Learner.learn and
        ReplayMemory.update_priorities of the sampled leaves (launch_learner.py:173-197 without the host queues).
        Replays the captured CUDA graph when enable_cuda_graph(mem) was called.  Returns (tree_idxs, loss); in graph
        mode these are static buffers that the next call overwrites."""
        g = self._graphs.get("replay")
        if g is not None and mem is g.mem:
            return self._replay(g)
        idxs, loss = self.learn(mem, None)
        mem.update_priorities(idxs, loss)
        return idxs, loss

    def _reset_step_streams(self, mem=None):
        """Start a step: reset the per-step Philox stream indices of both networks (and of ``mem``'s stratified draws),
        which read the attached riqn_dyn_state, or their by-value arguments when none is attached."""
        dyn = self._dyn if self._dyn_on else None
        self.online_net.begin_step(dyn)
        self.target_net.begin_step(dyn)
        if mem is not None:
            mem.transitions._draws_in_step = 0

    @contextlib.contextmanager
    def _attached(self, mem):
        """Route the per-step scalars (Philox offsets, Adam bias corrections, beta / capacity) through the device-resident
        riqn_dyn_state -- ONLY while a step is being warmed up / captured.  A captured graph keeps the struct's address in its
        kernel arguments; eager calls made after the capture, or after a capture that raised (learn_and_update on another
        memory, mem.sample(), optimiser.step(), reset_noise()), must read their by-value arguments again, not the
        last-written struct."""
        def route(dyn):
            self._dyn_on = dyn is not None
            self.optimiser._dyn = dyn
            for k, o in enumerate(self._optimisers()[1:], 1):     # the sides' optimisers, in Agent.sides order
                o._dyn = dyn.slot(k) if dyn is not None else None
            if mem is not None:
                mem.transitions._dyn = dyn
            self._reset_step_streams()

        route(self._dyn)
        try:
            yield
        finally:
            route(None)

    def _step_pre(self, mem):
        """sample -> three forwards -> loss -> backward (gradients in the arena)."""
        self._reset_step_streams(mem)
        idxs, states, actions, returns, next_states, nonterminals, weights = self._sample(mem, None)
        with self._feeding_discounts():
            loss = self.compute_gradients(states, actions, returns, next_states, nonterminals, weights,
                                          demo=self._demo_mask(mem, idxs), sequence=self._sequence(mem, idxs))
        return idxs, loss

    def _step_post(self, mem, idxs, loss, allreduce=True):
        """(all-reduce) -> Adam -> priority update of ``mem``'s sampled leaves (none without a memory)."""
        if allreduce:
            self.apply_gradients()
        else:
            self._step_optimisers()
        if mem is not None:
            mem.update_priorities(idxs, loss)

    def _capture(self, kind, pre, post, warmup, mem, inputs=None):
        """Capture one learner step as the graph of ``kind``.  ``pre()`` runs the sample or input copy, the loss and the
        backward and returns the step's outputs; ``post(out, allreduce)`` runs the (all-reduce and) Adam and the priority
        update.  ``mem``: the replay memory whose fill and beta the struct carries, or None.  Data parallel with
        capture_collectives False: pre and post become two graphs, with the all-reduce left eager between them."""
        if self._dyn is None:      # one struct for every graph of this learner: no captured address can go stale
            self._dyn = DynState(self.online_net._flat.device, slots=len(self._optimisers()))
        split = self.process_group is not None and not self.capture_collectives
        step0 = [o._step for o in self._optimisers()]
        with self._attached(mem):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for k in range(warmup):                  # eager warm-up on a side stream (allocator, attributes)
                    self._write_dyn(mem, k)
                    post(pre(), True)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self._write_dyn(mem)
            self.online_net._static_ops_dirty = True     # the captured step must rebuild the conv / iqn_fc operand images
            if self.target_ema is not None:              # and, as the EMA rewrites it every step, the target's
                self.target_net._static_ops_dirty = True
            if split:
                self.overlap_allreduce = False
            graph, post_graph = torch.cuda.CUDAGraph(), None
            with torch.cuda.graph(graph):
                out = pre()
                if not split:
                    post(out, True)
            if split:
                post_graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(post_graph, pool=graph.pool()):
                    post(out, False)
        # the capture itself does not execute the step: undo the host-side counters it advanced
        for o, s0 in zip(self._optimisers(), step0):
            o._step = s0 + warmup
        self._graphs[kind] = _StepGraph(graph, post_graph, mem, inputs, out, self._decays())
        self._count_updates(warmup)     # after the counters are set: a reset here restarts them for good

    def _replay(self, g, batch=None):
        """One step through the captured graph ``g``: ``batch`` (if given) into its static inputs, the struct written from
        the memory it was captured on, the replay (with an eager all-reduce: then the collective and the post graph).
        Returns the static outputs."""
        if self._decays() != g.decay:
            raise RuntimeError("this learner's step is captured in a CUDA graph that holds each optimiser's AdamW decay "
                               "1 - lr * weight_decay, and an lr or weight_decay has changed since: call release_graphs(), "
                               "then recapture (enable_cuda_graph / enable_batch_graph / enable_learn_graph)")
        if batch is not None:
            for d, src in zip(g.inputs, batch):
                d.copy_(src, non_blocking=True)
        self._write_dyn(g.mem)
        g.graph.replay()
        if g.post is not None:
            self._allreduce_all_grads()
            g.post.replay()
        for o in self._optimisers():        # advance the host step counters the replayed Adam launches stand for
            o._step += 1
        self._count_updates(1)
        return g.out

    def _decays(self):
        return tuple(o.decay() for o in self._optimisers())

    def enable_cuda_graph(self, mem, warmup=3, capture_collectives=True):
        """Capture learn_and_update(mem) in a CUDA graph (shapes are static: batch_size, N, N', K).  Everything that
        changes between steps lives on the device: Philox stream offsets, Adam bias corrections, beta and the replay
        fill are read from a riqn_dyn_state struct that is refreshed by one 32-byte async copy per step.
        Data parallel: the two NCCL all-reduces are captured too (ONE graph launch per step on every rank; the big bucket
        overlaps the backward on a side stream inside the graph); capture_collectives=False keeps them eager between two
        graphs, in this capture and in the batch and learn graphs captured after it."""
        self.capture_collectives = bool(capture_collectives)
        self._capture("replay", lambda: self._step_pre(mem), lambda out, allreduce: self._step_post(mem, *out, allreduce),
                      warmup, mem)
        return self

    def enable_batch_graph(self, mem, example):
        """Second captured graph for minibatches that arrive from the HOST (the reference's mp-queue hand-off,
        learner.py:16): static device input buffers, filled by async copies from pinned host tensors, then
        learn_on_batch + update_priorities replayed.  ``example`` = (idxs, states, actions, returns, next_states,
        nonterminals, weights) device tensors defining the shapes.  Requires enable_cuda_graph(mem) first.  Not under
        SPR: the host batch carries no sequences."""
        self._refuse_spr("enable_batch_graph")
        self._refuse_anneal("enable_batch_graph")
        g = self._graphs.get("replay")
        assert g is not None and mem is g.mem
        inputs = tuple(t.clone() for t in example)

        def pre():
            self._reset_step_streams()
            return self.compute_gradients(*inputs[1:], demo=self._demo_mask(mem, inputs[0]))

        self._capture("batch", pre, lambda loss, allreduce: self._step_post(mem, inputs[0], loss, allreduce), 2, mem,
                      inputs)
        return self

    def enable_learn_graph(self, example):
        """CUDA graph of learn_on_batch alone (no replay on this rank): the Ape-X learner, whose minibatch is gathered from
        the actor GPUs' shards (apex.ApexTopology.sample).  ``example`` = (states, actions, returns, next_states,
        nonterminals, weights) device tensors defining the shapes; learn_on_graph(batch) copies a batch into the static
        inputs and replays.  Returns self.  Not under DQfD: a gathered batch carries no demonstration flags."""
        if self.dqfd is not None:
            raise RuntimeError("the learn graph takes batches gathered from the actor shards, which carry no demonstration "
                               "flags: a DQfD learner steps from its own replay (enable_cuda_graph / enable_batch_graph)")
        self._refuse_spr("enable_learn_graph")
        self._refuse_anneal("enable_learn_graph")
        inputs = tuple(t.contiguous().clone() for t in example)

        def pre():
            self._reset_step_streams()
            return self.compute_gradients(*inputs)

        self._capture("learn", pre, lambda loss, allreduce: self._step_post(None, None, loss, allreduce), 2, None, inputs)
        return self

    def learn_on_graph(self, batch):
        """One learner step on ``batch`` (same shapes as enable_learn_graph's example) through the captured graph; returns
        the per-transition loss (static buffer, overwritten by the next call)."""
        return self._replay(self._graphs["learn"], batch)

    def prefetch_host_batch(self, host_batch):
        """Start the H2D copy of a FUTURE minibatch on a side stream (double-buffered device staging), so that it
        overlaps the current step -- what the reference's sampler subprocess + mp queue achieve on the host
        (launch_learner.py:24-50).  The next learn_on_host_batch() consumes it."""
        if not hasattr(self, "_pf_stream"):
            self._pf_stream = torch.cuda.Stream()
            self._pf_buf = [tuple(torch.empty_like(t) for t in self._graphs["batch"].inputs) for _ in range(2)]
            self._pf_slot, self._pf_event = 0, None
            self._pf_read_done = [None, None]
            self._pf_stream.wait_stream(torch.cuda.current_stream())   # fresh staging memory: order after its last user
        slot = self._pf_slot ^ 1
        # the staging slot must no longer be read by the (older) step that consumed it: wait for THAT step's
        # device-to-device copies only, not for the compute enqueued since -- the H2D overlaps the current step
        ev_read = self._pf_read_done[slot]
        if ev_read is not None:
            self._pf_stream.wait_event(ev_read)
        with torch.cuda.stream(self._pf_stream):
            for d, h in zip(self._pf_buf[slot], host_batch):
                d.copy_(h, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        self._pf_slot, self._pf_event = slot, ev

    def learn_on_host_batch(self, host_batch=None):
        """host_batch: pinned host tensors (idxs, states u8, actions, returns, next_states u8, nonterminals, weights),
        or None to consume the batch started by prefetch_host_batch().  H2D copies + one graph replay; returns the
        device loss (B,) (static buffer)."""
        self._refuse_spr("learn_on_host_batch")
        g = self._graphs["batch"]
        if host_batch is None:
            torch.cuda.current_stream().wait_event(self._pf_event)
            for d, src in zip(g.inputs, self._pf_buf[self._pf_slot]):
                d.copy_(src, non_blocking=True)                          # device-to-device, 29 MB
            ev = torch.cuda.Event()
            ev.record()
            self._pf_read_done[self._pf_slot] = ev                       # this staging slot may be refilled from here on
        return self._replay(g, host_batch)

    def set_risk(self, measure, eta=None):
        """Agent.set_risk.  A captured step graph holds the measure and eta as kernel arguments, so it refuses once one
        is captured: release_graphs(), set the risk, then capture again."""
        if self._graphs:
            raise RuntimeError("this learner's step is captured in a CUDA graph that holds the current risk measure: "
                               "call release_graphs(), set the risk, then recapture (enable_cuda_graph / "
                               "enable_batch_graph / enable_learn_graph)")
        super().set_risk(measure, eta)

    def release_graphs(self):
        """Drop every captured step graph; learn_and_update runs eagerly again until the next capture.  The device step
        state stays: the next capture reads the same struct."""
        self._graphs.clear()

    # north_star spellings
    update_target = Agent.update_target_net

    def save_to_redis(self, T_learner):
        """learner.py:28-36 (kept for wire compatibility; needs a redis-like object with pipeline())."""
        save_bytesIO = io.BytesIO()
        torch.save(self.online_net.state_dict(), save_bytesIO)
        pipe = self.redis_servor.pipeline()
        pipe.set(MODEL_WEIGHT_STR, save_bytesIO.getvalue())
        pipe.set(STEP_LEARNER_STR, T_learner)
        pipe.execute()
