"""Device-resident per-step scalars (riqn_dyn_state, include/riqn_b200.h) so that a learner step can be captured in a
CUDA graph once and replayed: the host rewrites this 32-byte struct with one async copy before each replay.

A learner keeps one slot per Learner._optimisers() entry, in that order, written by the same copy: each slot's Adam
fields are that optimiser's bias corrections (its own learning rate), and every rng_offset repeats the first one's.

Under horizon_anneal (horizon.py) the learner also keeps one riqn_horizon_state (HorizonState), the step's n and gamma,
written by one async copy before every step, eager or replayed."""
import ctypes
import numbers
import struct

import torch

_FMT = "<Qffdd"          # rng_offset, adam_neg_step_size, adam_sqrt_bc2, is_capacity, is_beta
_SIZE = struct.calcsize(_FMT)
_RING = 16
MAX_HORIZON = 16         # RIQN_MAX_HORIZON
HORIZON_FMT = f"<if{MAX_HORIZON}d"   # n_step, gamma_n, gamma_pow[16]


class _Slot:
    def __init__(self, state, index):
        self._state, self._index = state, index

    def ptr(self):
        return self._state.ptr() + _SIZE * self._index


class _Staged:
    """A device buffer of ``nbytes`` and a ring of pinned host buffers: each write packs one host buffer and enqueues its
    copy on the current stream, so the host never overwrites a buffer whose copy is still pending."""

    def __init__(self, device, nbytes):
        self.dev = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self._host = [torch.zeros(nbytes, dtype=torch.uint8).pin_memory() for _ in range(_RING)]
        self._events = [None] * _RING
        self._i = 0

    def ptr(self):
        return self.dev.data_ptr()

    def _next_host(self):
        slot = self._i % _RING
        if self._events[slot] is not None:
            self._events[slot].synchronize()          # the copy that last used this pinned slot has completed
        return self._host[slot]

    def _copy(self, buf):
        self.dev.copy_(buf, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[self._i % _RING] = ev
        self._i += 1


class DynState(_Staged):
    def __init__(self, device, slots=1):
        assert _SIZE == 32
        super().__init__(device, _SIZE * slots)
        self.slots = slots
        self.epoch = 0       # learner steps issued; Philox streams advance by 64 per epoch

    def slot(self, index):
        """An object whose ptr() is the address of struct ``index`` (what the entry points taking `dyn` read)."""
        assert 0 <= index < self.slots
        return _Slot(self, index)

    def write(self, neg_step_size, sqrt_bc2, capacity, beta, *more_adam):
        """Stage the values of the NEXT step and enqueue the copy on the current stream.  ``more_adam``: the
        (neg_step_size, sqrt_bc2) pairs of the further slots."""
        buf = self._next_host()
        struct.pack_into(_FMT, buf.numpy(), 0, 64 * self.epoch, float(neg_step_size), float(sqrt_bc2), float(capacity),
                         float(beta))
        for k, (nss, sbc) in enumerate(more_adam[:self.slots - 1]):
            struct.pack_into(_FMT, buf.numpy(), _SIZE * (k + 1), 64 * self.epoch, float(nss), float(sbc), float(capacity),
                             float(beta))
        self._copy(buf)
        self.epoch += 1


class HorizonState(_Staged):
    """The riqn_horizon_state that riqn_sumtree_sample_horizon and riqn_frame_gather_horizon read, and its one writer.
    ``n_max``: the largest n it may hold (the entry points' n_max)."""

    def __init__(self, device, n_max):
        if not 1 <= n_max <= MAX_HORIZON:
            raise ValueError(f"n_max must be in 1..{MAX_HORIZON}, got {n_max!r}")
        super().__init__(device, struct.calcsize(HORIZON_FMT))
        self.n_max = n_max
        self.value = None      # the (n, gamma) last written

    def write(self, n, gamma):
        """Stage the next step's n and gamma and enqueue the copy on the current stream: n_step = n, gamma_n =
        fl32(gamma ** n) and gamma_pow[k] = gamma ** k for k < n, every power taken in double as ReplayMemory's."""
        if isinstance(n, bool) or not isinstance(n, numbers.Integral) or not 1 <= n <= self.n_max:
            raise ValueError(f"the update horizon n must be an integer in 1..{self.n_max}, got {n!r}")
        n, gamma = int(n), float(gamma)
        pows = [gamma ** k for k in range(n)] + [0.0] * (MAX_HORIZON - n)
        buf = self._next_host()
        struct.pack_into(HORIZON_FMT, buf.numpy(), 0, n, ctypes.c_float(gamma ** n).value, *pows)
        self._copy(buf)
        self.value = (n, gamma)
