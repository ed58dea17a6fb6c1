"""Adam over the flat parameter arena (one kernel launch per step).

Drop-in for ``torch.optim.Adam(online_net.parameters(), lr=..., eps=...)`` as the reference uses it
(rainbowiqn/agent.py:43, learner.py:24): same update rule, and ``state_dict()`` / ``load_state_dict()``
keep torch's layout (per-parameter ``step``, ``exp_avg``, ``exp_avg_sq``) so reference checkpoints
(agent.py:150-160, :45-47) round-trip.
"""
import torch

from ._lib import call, ptr


class Adam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        params = list(params)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
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
        call("riqn_adam_step", self._flat.numel(), ptr(self._flat), ptr(grad_flat), ptr(self._exp_avg),
             ptr(self._exp_avg_sq), self._step, float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]),
             float(g["eps"]), float(self.grad_scale), self._dyn.ptr() if self._dyn is not None else None)
        self._net._params_changed()             # conv / iqn_fc operand images are rebuilt by the next reset_noise()

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
        super().load_state_dict(state_dict)
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
