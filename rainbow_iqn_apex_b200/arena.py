"""Flat parameter arenas: the layout every arena shares, and the side networks an agent trains beside its DQN, each in
an arena of its own (FQF's fraction proposal, CURL's projection, SPR's networks).  Each side's ``build`` returns its Side;
Agent.sides lists them, and Agent.save, the Learner's step, parallel.py and reset.py walk that list."""
import weakref
from typing import Callable, NamedTuple, Optional

import torch
from torch import nn

from ._lib import call, ptr

_ALIGN = 64  # floats; arena groups start on 256-byte boundaries


def layout(groups):
    """The arena layout of ``groups`` (lists of element counts): every member's offset, members in order, each group
    starting on an _ALIGN boundary; and the total length, rounded up to one."""
    total, offsets = 0, []
    for group in groups:
        total = (total + _ALIGN - 1) // _ALIGN * _ALIGN
        for n in group:
            offsets.append(total)
            total += n
    return offsets, (total + _ALIGN - 1) // _ALIGN * _ALIGN


class ArenaModule(nn.Module):
    """Parameters ``NAMES`` (dotted names allowed) as views of one flat fp32 arena (``_flat``; gradients in
    ``_flat_grad``) that the arena Adam steps and data parallelism reduces in one piece, one group each, in NAMES order.
    A subclass assigns its parameters, then calls _flatten."""

    NAMES = ()

    def _flatten(self, dev):
        params = [self.get_parameter(name) for name in self.NAMES]
        offsets, total = layout([[p.numel()] for p in params])
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        flat_grad = torch.zeros(total, device=dev, dtype=torch.float32)
        for p, off in zip(params, offsets):
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1).float())
            p.data = flat[off:off + n].view(p.shape)
            p.grad = flat_grad[off:off + n].view(p.shape)
            p._riqn_owner = weakref.ref(self)
            p._riqn_offset = off
        self._flat, self._flat_grad = flat, flat_grad

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._flatten(self.get_parameter(self.NAMES[0]).device)
        return out

    def _params_changed(self):
        """Called by the arena Adam after a step: nothing is cached from these weights."""

    def grad_view(self, p):
        return self._flat_grad[p._riqn_offset:p._riqn_offset + p.numel()].view(p.shape)

    def zero_grad(self, set_to_none=False):
        """One memset over the gradient arena; the .grad views stay bound."""
        if self._flat_grad.is_cuda:
            call("riqn_zero_f32", ptr(self._flat_grad), self._flat_grad.numel())
        else:                       # CPU arenas exist only for the host-logic tests; nothing computes there
            self._flat_grad.zero_()
        for p in self.parameters():
            p.grad = self.grad_view(p)


class Side(NamedTuple):
    """One side network of an agent: what the walkers of Agent.sides need to know of it."""
    index: int                           # its arena index in reset.ARENAS: the stream ids of its resets
    net: ArenaModule
    optimiser: object                    # the arena Adam over net
    checkpoint: Callable[[], dict]       # the entries it adds to a saved checkpoint (its build restores them)
    broadcast: tuple                     # the tensors a data-parallel replica takes from rank 0
    publish: bool = False                # Ape-X publication sends net._flat to the actors, who act on it
    after_step: Optional[Callable] = None     # (learner): after every optimiser's step
    after_reset: Optional[Callable] = None    # (agent): after the arenas' resets
    trunk_term: Optional[Callable] = None     # (learner, raw_states, sequence, debug) -> the step's DQN._trunk_addend
