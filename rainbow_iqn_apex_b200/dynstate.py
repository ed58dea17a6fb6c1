"""Device-resident per-step scalars (riqn_dyn_state, include/riqn_b200.h) so that a learner step can be captured in a
CUDA graph once and replayed: the host rewrites this 32-byte struct with one async copy before each replay.

A learner keeps one slot per Learner._optimisers() entry, in that order, written by the same copy: each slot's Adam
fields are that optimiser's bias corrections (its own learning rate), and every rng_offset repeats the first one's."""
import struct

import torch

_FMT = "<Qffdd"          # rng_offset, adam_neg_step_size, adam_sqrt_bc2, is_capacity, is_beta
_SIZE = struct.calcsize(_FMT)
_RING = 16


class _Slot:
    def __init__(self, state, index):
        self._state, self._index = state, index

    def ptr(self):
        return self._state.ptr() + _SIZE * self._index


class DynState:
    def __init__(self, device, slots=1):
        assert _SIZE == 32
        self.slots = slots
        self.dev = torch.zeros(_SIZE * slots, dtype=torch.uint8, device=device)
        self._host = [torch.zeros(_SIZE * slots, dtype=torch.uint8).pin_memory() for _ in range(_RING)]
        self._events = [None] * _RING
        self._i = 0
        self.epoch = 0       # learner steps issued; Philox streams advance by 64 per epoch

    def ptr(self):
        return self.dev.data_ptr()

    def slot(self, index):
        """An object whose ptr() is the address of struct ``index`` (what the entry points taking `dyn` read)."""
        assert 0 <= index < self.slots
        return _Slot(self, index)

    def write(self, neg_step_size, sqrt_bc2, capacity, beta, *more_adam):
        """Stage the values of the NEXT step and enqueue the copy on the current stream.  ``more_adam``: the
        (neg_step_size, sqrt_bc2) pairs of the further slots."""
        slot = self._i % _RING
        if self._events[slot] is not None:
            self._events[slot].synchronize()          # the copy that last used this pinned slot has completed
        buf = self._host[slot]
        struct.pack_into(_FMT, buf.numpy(), 0, 64 * self.epoch, float(neg_step_size), float(sqrt_bc2), float(capacity),
                         float(beta))
        for k, (nss, sbc) in enumerate(more_adam[:self.slots - 1]):
            struct.pack_into(_FMT, buf.numpy(), _SIZE * (k + 1), 64 * self.epoch, float(nss), float(sbc), float(capacity),
                             float(beta))
        self.dev.copy_(buf, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        self._i += 1
        self.epoch += 1
