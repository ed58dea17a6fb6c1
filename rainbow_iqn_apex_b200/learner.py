"""Learner -- mirror of the reference ``rainbowiqn/learner.py:8-36``.

``learn(mem, mp_queue) -> (idxs, loss)`` performs the reference's sequence
sample -> loss -> zero_grad -> (weights*loss).mean().backward() -> Adam.step (learner.py:14-26) with the
backward driven directly (no autograd graph) and the IS weights folded into the upstream gradient
gscale[b] = weights[b] / B.  ``north_star`` spellings Agent.learn / Agent.update_target are aliased.
"""
import io

import torch

from . import compute_loss_iqn
from .agent import Agent

MODEL_WEIGHT_STR = "model_weight"      # rainbowiqn/constants.py:18
STEP_LEARNER_STR = "step_learner:"     # rainbowiqn/constants.py:14


class Learner(Agent):
    def __init__(self, args, action_space, redis_servor):
        super().__init__(args, action_space, redis_servor)
        self.process_group = None  # set by parallel.make_data_parallel
        self._dp_stream = self._dp_tail = None
        self.overlap_allreduce = True   # data parallel: start the NoisyLinear-gradient all-reduce inside the backward
        self._graph = None         # CUDA-graph mode (enable_cuda_graph)
        self._graph_post = None

    def learn(self, mem_redis, mp_queue):
        sample = mem_redis.get_sample_from_mp_queue(mp_queue)
        idxs, states, actions, returns, next_states, nonterminals, weights = sample
        loss = self.learn_on_batch(states, actions, returns, next_states, nonterminals, weights)
        return idxs, loss

    def learn_on_batch(self, states, actions, returns, next_states, nonterminals, weights):
        """learner.py:18-24 on an already assembled minibatch.  Returns the per-transition loss (B,)."""
        loss = self.compute_gradients(states, actions, returns, next_states, nonterminals, weights)
        self.apply_gradients()
        return loss

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
            tail = getattr(self, "_dp_tail", None)
            if tail is not None:             # the big bucket is already in flight: reduce the rest, then join
                torch.distributed.all_reduce(self.online_net._flat_grad[:tail], group=self.process_group)
                torch.cuda.current_stream().wait_stream(self._dp_stream)
                self._dp_tail = None
            else:
                torch.distributed.all_reduce(self.online_net._flat_grad, group=self.process_group)
        self.optimiser.step()

    def compute_gradients(self, states, actions, returns, next_states, nonterminals, weights, debug=None):
        """loss -> zero_grad -> backward of (weights*loss).mean()   (learner.py:18-23); gradients land in the arena.
        ``debug``: dict that receives the IQN loss's intermediates (compute_loss_iqn.loss_core)."""
        on = self.online_net
        dev = on._flat.device
        weights = weights.to(dev, torch.float32)
        if self.rainbow_only:
            from . import c51
            loss, bw = c51.loss_core(self, states, actions, returns, next_states, nonterminals)
            on.zero_grad()
            bw(weights, 1.0 / weights.shape[0])
        else:
            loss, dtheta, keep, actions = compute_loss_iqn.loss_core(
                self, states, actions, returns, next_states, nonterminals, keep_graph=True, debug=debug)
            if getattr(self, "_debug", None) is not None:                       # parity tests: the pass's activations
                self._debug.update(keep=keep)
            on.zero_grad()                                                      # learner.py:22
            on._grads_ready_hook = self._start_tail_allreduce if (self.process_group is not None and self.overlap_allreduce) else None
            on.backward_iqn(keep, dtheta, weights.contiguous(), actions, 1.0 / weights.shape[0])  # learner.py:23 (.mean())
            on._grads_ready_hook = None
        return loss

    # ------------------------------------------------------------------ whole step: sample -> learn -> priority update
    def learn_and_update(self, mem):
        """One learner iteration against a device-resident ReplayMemory: prioritized sample, Learner.learn and
        ReplayMemory.update_priorities of the sampled leaves (launch_learner.py:173-197 without the host queues).
        Replays the captured CUDA graph when enable_cuda_graph(mem) was called.  Returns (tree_idxs, loss); in graph
        mode these are static buffers that the next call overwrites."""
        if self._graph is not None and mem is self._graph_mem:
            dyn = self._dyn
            nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
            dyn.write(nss, sbc, mem.transitions.get_current_capacity(), mem.priority_weight)
            self._graph.replay()
            if self._graph_post is not None:          # data parallel: the collective stays outside the graphs
                torch.distributed.all_reduce(self.online_net._flat_grad, group=self.process_group)
                self._graph_post.replay()
            self.optimiser._step += 1
            return self._graph_out
        idxs, loss = self.learn(mem, None)
        mem.update_priorities(idxs, loss)
        return idxs, loss

    def _attach_dyn(self, mem, on):
        """Route the per-step scalars (Philox offsets, Adam bias corrections, beta / capacity) through the device-resident
        riqn_dyn_state -- ONLY while a step is being warmed up / captured.  A captured graph keeps the struct's address in its
        kernel arguments; eager calls made after the capture (learn_and_update on another memory, mem.sample(),
        optimiser.step(), reset_noise()) must read their by-value arguments again, not the last-written struct."""
        dyn = self._dyn if on else None
        self._dyn_on = bool(on)
        self.optimiser._dyn = dyn
        if mem is not None:
            mem.transitions._dyn = dyn
        self.online_net.begin_step(dyn)
        self.target_net.begin_step(dyn)

    def _step_pre(self, mem):
        """sample -> three forwards -> loss -> backward (gradients in the arena)."""
        dyn = self._dyn if getattr(self, "_dyn_on", False) else None
        self.online_net.begin_step(dyn)
        self.target_net.begin_step(dyn)
        mem.transitions._draws_in_step = 0
        idxs, states, actions, returns, next_states, nonterminals, weights = mem.get_sample_from_mp_queue(None)
        loss = self.compute_gradients(states, actions, returns, next_states, nonterminals, weights)
        return idxs, loss

    def _step_post(self, mem, idxs, loss, allreduce=True):
        """(all-reduce) -> Adam -> priority update."""
        if allreduce:
            self.apply_gradients()
        else:
            self.optimiser.step()
        mem.update_priorities(idxs, loss)

    def _step_body(self, mem):
        idxs, loss = self._step_pre(mem)
        self._step_post(mem, idxs, loss)
        return idxs, loss

    def enable_cuda_graph(self, mem, warmup=3, capture_collectives=True):
        """Capture learn_and_update(mem) in a CUDA graph (shapes are static: batch_size, N, N', K).  Everything that
        changes between steps lives on the device: Philox stream offsets, Adam bias corrections, beta and the replay
        fill are read from a riqn_dyn_state struct that is refreshed by one 32-byte async copy per step.
        Data parallel: the two NCCL all-reduces are captured too (ONE graph launch per step on every rank; the big bucket
        overlaps the backward on a side stream inside the graph); capture_collectives=False keeps them eager between two
        graphs (the round-1 scheme)."""
        self._capture_collectives = bool(capture_collectives)
        from .dynstate import DynState
        dev = self.online_net._flat.device
        self._dyn = DynState(dev)
        self._attach_dyn(mem, True)
        step0 = self.optimiser._step
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(warmup):                      # eager warm-up on the capture stream (allocator, attributes)
                nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
                self._dyn.write(nss, sbc, mem.transitions.get_current_capacity(), mem.priority_weight)
                self._step_body(mem)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
        self._dyn.write(nss, sbc, mem.transitions.get_current_capacity(), mem.priority_weight)
        self.online_net._static_ops_dirty = True     # the captured step must rebuild the conv / iqn_fc operand images
        post = None
        if self.process_group is None or self._capture_collectives:
            with torch.cuda.graph(graph):
                out = self._step_body(mem)
        else:
            # data parallel, eager collective: two graphs around one all-reduce of the whole arena
            self.overlap_allreduce = False
            with torch.cuda.graph(graph):
                out = self._step_pre(mem)
            post = torch.cuda.CUDAGraph()
            with torch.cuda.graph(post, pool=graph.pool()):
                self._step_post(mem, out[0], out[1], allreduce=False)
        # the capture itself does not execute the step: undo the host-side counter it advanced
        self.optimiser._step = step0 + warmup
        self._graph, self._graph_post, self._graph_mem, self._graph_out = graph, post, mem, out
        self._attach_dyn(mem, False)           # eager calls from here on use their by-value arguments again
        return self

    def enable_batch_graph(self, mem, example):
        """Second captured graph for minibatches that arrive from the HOST (the reference's mp-queue hand-off,
        learner.py:16): static device input buffers, filled by async copies from pinned host tensors, then
        learn_on_batch + update_priorities replayed.  ``example`` = (idxs, states, actions, returns, next_states,
        nonterminals, weights) device tensors defining the shapes.  Requires enable_cuda_graph(mem) first."""
        assert self._graph is not None and mem is self._graph_mem
        self._bg_in = tuple(t.clone() for t in example)
        self._attach_dyn(mem, True)

        def pre():
            self.online_net.begin_step(self._dyn)
            self.target_net.begin_step(self._dyn)
            idxs, st, ac, rt, nx, nt, w = self._bg_in
            return self.compute_gradients(st, ac, rt, nx, nt, w)

        def body():
            loss = pre()
            self._step_post(mem, self._bg_in[0], loss)
            return loss

        step0 = self.optimiser._step
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
                self._dyn.write(nss, sbc, mem.transitions.get_current_capacity(), mem.priority_weight)
                body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        self.online_net._static_ops_dirty = True
        post = None
        if self.process_group is None or getattr(self, "_capture_collectives", True):
            with torch.cuda.graph(graph):
                out = body()
        else:
            with torch.cuda.graph(graph):
                out = pre()
            post = torch.cuda.CUDAGraph()
            with torch.cuda.graph(post, pool=graph.pool()):
                self._step_post(mem, self._bg_in[0], out, allreduce=False)
        self.optimiser._step = step0 + 2
        self._bgraph, self._bgraph_post, self._bg_out = graph, post, out
        self._attach_dyn(mem, False)
        return self

    def enable_learn_graph(self, example):
        """CUDA graph of learn_on_batch alone (no replay on this rank): the Ape-X learner, whose minibatch is gathered from
        the actor GPUs' shards (apex.ApexTopology.sample).  ``example`` = (states, actions, returns, next_states,
        nonterminals, weights) device tensors defining the shapes; learn_on_graph(batch) copies a batch into the static
        inputs and replays.  Returns self."""
        from .dynstate import DynState
        if getattr(self, "_dyn", None) is None:
            self._dyn = DynState(self.online_net._flat.device)
        self._lg_in = tuple(t.contiguous().clone() for t in example)

        def body():
            self.online_net.begin_step(self._dyn)
            self.target_net.begin_step(self._dyn)
            loss = self.compute_gradients(*self._lg_in)
            self.apply_gradients()
            return loss

        self._attach_dyn(None, True)
        step0 = self.optimiser._step
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
                self._dyn.write(nss, sbc, 1.0, 0.0)
                body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
        self._dyn.write(nss, sbc, 1.0, 0.0)
        self.online_net._static_ops_dirty = True
        with torch.cuda.graph(graph):
            out = body()
        self.optimiser._step = step0 + 2
        self._lgraph, self._lg_out = graph, out
        self._attach_dyn(None, False)
        return self

    def learn_on_graph(self, batch):
        """One learner step on ``batch`` (same shapes as enable_learn_graph's example) through the captured graph; returns
        the per-transition loss (static buffer, overwritten by the next call)."""
        for d, src in zip(self._lg_in, batch):
            d.copy_(src, non_blocking=True)
        nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
        self._dyn.write(nss, sbc, 1.0, 0.0)
        self._lgraph.replay()
        self.optimiser._step += 1
        return self._lg_out

    def prefetch_host_batch(self, host_batch):
        """Start the H2D copy of a FUTURE minibatch on a side stream (double-buffered device staging), so that it
        overlaps the current step -- what the reference's sampler subprocess + mp queue achieve on the host
        (launch_learner.py:24-50).  The next learn_on_host_batch() consumes it."""
        if not hasattr(self, "_pf_stream"):
            self._pf_stream = torch.cuda.Stream()
            self._pf_buf = [tuple(torch.empty_like(t) for t in self._bg_in) for _ in range(2)]
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
        if host_batch is None:
            torch.cuda.current_stream().wait_event(self._pf_event)
            for d, src in zip(self._bg_in, self._pf_buf[self._pf_slot]):
                d.copy_(src, non_blocking=True)                          # device-to-device, 29 MB
            ev = torch.cuda.Event()
            ev.record()
            self._pf_read_done[self._pf_slot] = ev                       # this staging slot may be refilled from here on
        else:
            for d, h in zip(self._bg_in, host_batch):
                d.copy_(h, non_blocking=True)
        mem = self._graph_mem
        nss, sbc = self.optimiser.bias_corrections(self.optimiser._step + 1)
        self._dyn.write(nss, sbc, mem.transitions.get_current_capacity(), mem.priority_weight)
        self._bgraph.replay()
        if self._bgraph_post is not None:
            torch.distributed.all_reduce(self.online_net._flat_grad, group=self.process_group)
            self._bgraph_post.replay()
        self.optimiser._step += 1
        return self._bg_out

    def set_risk(self, measure, eta=None):
        """Agent.set_risk.  A captured step graph holds the measure and eta as kernel arguments, so it refuses once one
        is captured: release_graphs(), set the risk, then capture again."""
        if any(getattr(self, g, None) is not None for g in ("_graph", "_bgraph", "_lgraph")):
            raise RuntimeError("this learner's step is captured in a CUDA graph that holds the current risk measure: "
                               "call release_graphs(), set the risk, then recapture (enable_cuda_graph / "
                               "enable_batch_graph / enable_learn_graph)")
        super().set_risk(measure, eta)

    def release_graphs(self):
        """Drop every captured step graph; learn_and_update runs eagerly again until the next capture."""
        self._graph = self._graph_post = self._graph_mem = self._graph_out = None
        self._bgraph = self._bgraph_post = self._bg_out = None
        self._lgraph = self._lg_out = None

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
