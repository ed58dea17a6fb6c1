"""Adam over the flat parameter arena (one kernel launch per step).

Drop-in for ``torch.optim.Adam(online_net.parameters(), lr=..., eps=...)`` as the reference uses it
(rainbowiqn/agent.py:43, learner.py:24): same update rule, and ``state_dict()`` / ``load_state_dict()``
keep torch's layout (per-parameter ``step``, ``exp_avg``, ``exp_avg_sq``) so reference checkpoints
(agent.py:150-160, :45-47) round-trip.  With ``weight_decay`` > 0 it is ``torch.optim.AdamW`` (decoupled decay,
riqn_adamw_step); the moments have the same layout, so Adam and AdamW checkpoints load into each other.
"""
import ctypes

import torch

from ._lib import call, ptr


class Adam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        params = list(params)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._weight_decay = weight_decay
        self._bind()
        self._step = 0
        self.grad_scale = 1.0  # set to 1/world_size by the data-parallel learner
        self._dyn = None       # DynState in CUDA-graph mode

    def _bind(self):
        ps = [p for g in self.param_groups for p in g["params"]]
        owner = getattr(ps[0], "_riqn_owner", None)
        owner = owner() if owner is not None else None
        if owner is None or any(getattr(p, "_riqn_owner", lambda: None)() is not owner for p in ps):
            raise ValueError("Adam expects the parameters of a rainbow_iqn_apex_b200 DQN (views of one flat arena)")
        self._net = owner
        self._flat = owner._flat
        self._exp_avg = torch.zeros_like(self._flat)
        self._exp_avg_sq = torch.zeros_like(self._flat)
        self._params = ps

    def _views(self, p):
        off, n = p._riqn_offset, p.numel()
        return self._exp_avg[off:off + n].view(p.shape), self._exp_avg_sq[off:off + n].view(p.shape)

    def _publish_state(self):
        for p in self._params:
            m, v = self._views(p)
            self.state[p] = {"step": torch.tensor(float(self._step)), "exp_avg": m, "exp_avg_sq": v}

    @torch.no_grad()
    def step(self, closure=None):
        if self._flat is not self._net._flat:       # the module was moved / re-flattened after construction
            self._rebind_after_move()
        grad_flat = self._net._flat_grad
        base = grad_flat.data_ptr()
        for p in self._params:
            if p.grad is None:
                raise RuntimeError("a parameter has no gradient; call online_net.zero_grad() (arena memset) "
                                   "instead of setting grads to None")
            if p.grad.data_ptr() != base + 4 * p._riqn_offset:   # foreign gradient tensor: stage it into the arena
                self._net.grad_view(p).copy_(p.grad)
        self._step += 1
        g = self.param_groups[0]
        head = (self._flat.numel(), ptr(self._flat), ptr(grad_flat), ptr(self._exp_avg), ptr(self._exp_avg_sq),
                self._step, float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]))
        tail = (float(self.grad_scale), self._dyn.ptr() if self._dyn is not None else None)
        if g["weight_decay"] > 0:
            call("riqn_adamw_step", *head, float(g["weight_decay"]), *tail)
        else:
            call("riqn_adam_step", *head, *tail)
        self._net._params_changed()             # conv / iqn_fc operand images are rebuilt by the next reset_noise()

    def restart(self):
        """Become a freshly constructed optimiser once the caller has zeroed the moment arenas (riqn_arena_reset): step
        0, no per-parameter state, so that the next step takes the step-1 bias corrections."""
        self._step = 0
        self.state.clear()

    def decay(self):
        """AdamW's decay factor d = fl32(1 - lr * weight_decay) as riqn_adamw_step forms it, or None without decay.  A
        captured step holds it by value (Learner._replay compares it)."""
        g = self.param_groups[0]
        if not g["weight_decay"] > 0:
            return None
        f32 = lambda x: ctypes.c_float(x).value
        return f32(1.0 - f32(g["lr"]) * f32(g["weight_decay"]))

    def bias_corrections(self, step):
        """(-(lr / (1 - b1^t)), sqrt(1 - b2^t)) of step t, as torch.optim.Adam computes them."""
        g = self.param_groups[0]
        b1, b2 = g["betas"]
        return -(g["lr"] / (1.0 - b1 ** step)), (1.0 - b2 ** step) ** 0.5

    def _rebind_after_move(self):
        old_m, old_v = self._exp_avg, self._exp_avg_sq
        self._bind()
        if old_m.numel() == self._exp_avg.numel():
            self._exp_avg.copy_(old_m)
            self._exp_avg_sq.copy_(old_v)

    def state_dict(self):
        if self._step > 0:
            self._publish_state()
        return super().state_dict()

    def load_state_dict(self, state_dict):
        """torch's load, except that weight_decay stays this optimiser's: the update rule (Adam or AdamW) is chosen at
        construction, and a state saved by the other one restores the step and the moments only."""
        super().load_state_dict(state_dict)
        for g in self.param_groups:
            g["weight_decay"] = self._weight_decay
        step = 0
        for p in self._params:
            st = self.state.get(p)
            if not st:
                continue
            m, v = self._views(p)
            m.copy_(st["exp_avg"])
            v.copy_(st["exp_avg_sq"])
            step = int(float(st["step"]))
        self._step = step
        if step > 0:
            self._publish_state()
