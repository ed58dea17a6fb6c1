"""Agent -- mirror of the reference ``rainbowiqn/agent.py:10-166`` (shared by Learner and Actor).

Same constructor ``Agent(args, action_space, redis_servor)`` reading the same ``args`` fields, same public attributes
(online_net, target_net, optimiser, n, history, discount, device, batch_size, kappa, num_tau_samples,
num_tau_prime_samples, num_quantile_samples, support, ...) and methods (reset_noise, update_target_net,
compute_loss_actor_or_learner, save, train, eval), plus ``loss_core`` for the loss the agent trains (c51.loss_core,
qr.loss_core or compute_loss_iqn.loss_core), ``risk`` / ``set_risk`` for risk-sensitive acting and ``munchausen`` for
Munchausen-IQN targets, ``fqf`` for FQF fractions (fqf.py), ``value_rescaling`` (and, for C51, ``acting_support``) for
the transformed Bellman operator on unclipped rewards, and ``qr_dqn`` for QR-DQN's fixed-fraction quantile head, ``mmd``
for MMDQN's moment-matching loss on that head (mmd.py), ``hl_gauss`` for HL-Gauss's Gaussian-histogram loss on the C51
head (hl_gauss.py), ``cql`` for the conservative regulariser of the IQN and QR-DQN losses (cql.py), ``dqfd`` for DQfD's
large-margin loss on demonstrations (dqfd.py), ``random_shift`` for the learner's random-shift augmentation
(augment.py), ``curl`` for CURL's contrastive loss on the trunk (curl.py), ``spr`` for SPR's self-predictive loss on the
trunk (spr.py), ``reset`` (reset_interval, reset_shrink) with ``updates`` / ``resets`` for the learner's periodic
network resets (reset.py), ``target_ema`` (tau) for the learner's EMA target network (target.py) and ``adamw`` (the
weight decay) for AdamW in every optimiser the agent builds, ``horizon_anneal`` (n0, gamma0, steps) for the learner's
update-horizon and discount annealing (horizon.py), and ``horizon()`` / ``gamma_n()`` for the (n, gamma) the loss cores
train at.  The networks FQF, CURL and SPR train beside the DQN and
their optimisers are set by those modules' ``build`` (None when off), and ``sides`` lists them (arena.Side).  The
networks are
rainbow_iqn_apex_b200.model.DQN (CUDA) and the optimiser is the arena Adam; checkpoints keep the reference schema
{T_actors, T_learner, model_state_dict, optimiser_state_dict} (agent.py:150-160), plus, under resets, reset_state and
each side's entries.
"""
import os

import torch

from . import _lib
from . import c51, compute_loss_iqn, config, curl, fqf, qr, spr
from .model import DQN
from .optim import Adam


class Agent:
    # public attribute <- args field (agent.py:13-63; read by the loss code, the actors and the launch scripts)
    _ARG_FIELDS = (("n", "multi_step"), ("history", "history_length"), ("discount", "discount"), ("device", "device"),
                   ("batch_size", "batch_size"), ("rainbow_only", "rainbow_only"))
    _C51_FIELDS = (("atoms", "atoms"), ("Vmin", "V_min"), ("Vmax", "V_max"))
    _IQN_FIELDS = ("kappa", "num_tau_samples", "num_tau_prime_samples", "num_quantile_samples")

    def __init__(self, args, action_space, redis_servor):
        _lib.require_device()
        self.action_space, self.redis_servor = action_space, redis_servor
        for attr, field in self._ARG_FIELDS:
            setattr(self, attr, getattr(args, field))
        self.length_actor_buffer = getattr(args, "length_actor_buffer", 1000)

        # online network (+ optional checkpoint, agent.py:26-34), noisy target copy with frozen parameters (:37-41), Adam (:43)
        checkpoint = self._read_checkpoint(getattr(args, "model", None))
        # the head and loss variants and their optional args fields (absent from the reference's namespace: off), read
        # once (config.py).  Each is fixed for the agent's life, so that a captured step graph stays valid; only the risk
        # measure has a setter
        v = config.read(args, action_space)
        self._head, self._loss = v.pop("head"), v.pop("loss")
        for attr, value in v.items():
            setattr(self, attr, value)
        # both checked before any weights load: a QR network with N = atoms has the C51 network's shapes
        if checkpoint is not None and checkpoint.get("qr_dqn_quantiles") != self.qr_dqn:
            raise ValueError(f"the checkpoint was trained with qr_dqn_quantiles = {checkpoint.get('qr_dqn_quantiles')} "
                             f"(None: not QR-DQN), the args ask for {self.qr_dqn}: the z-layers hold other quantities")
        if checkpoint is not None and checkpoint.get("value_rescaling_eps") != self.value_rescaling:
            raise ValueError(f"the checkpoint was trained with value_rescaling_eps = {checkpoint.get('value_rescaling_eps')} "
                             f"(None: off), the args ask for {self.value_rescaling}: a network trained in h-space acts "
                             "differently on the linear scale")
        self.online_net = DQN(args, action_space).to(device=args.device)
        if checkpoint is not None:
            self.online_net.load_state_dict(checkpoint["model_state_dict"])
        self.target_net = DQN(args, action_space).to(device=args.device)
        self.update_target_net()
        if self.target_ema is not None and checkpoint is not None and "target_state_dict" in checkpoint:
            self.target_net.load_state_dict(checkpoint["target_state_dict"])     # an EMA target is not the online net
            self.target_net.compose_weights()
        for net in (self.online_net, self.target_net):
            net.train()                                  # the target stays in train mode: it is noisy too
        for p in self.target_net.parameters():
            p.requires_grad = False
        self.optimiser = Adam(self.online_net.parameters(), lr=args.lr, eps=args.adam_eps, weight_decay=self.adamw or 0.0)
        if checkpoint is not None:
            self.optimiser.load_state_dict(checkpoint["optimiser_state_dict"])

        # the head's sizes and the loss core this agent trains (every core returns (loss, backward))
        if self._head == "c51":                          # categorical support (agent.py:49-57)
            for attr, field in self._C51_FIELDS:
                setattr(self, attr, getattr(args, field))
            self.support = torch.linspace(self.Vmin, self.Vmax, self.atoms).to(device=args.device)
            self.delta_z = (self.Vmax - self.Vmin) / (self.atoms - 1)
            self.loss_core = c51.loss_core
        elif self._head == "qr":                         # QR-DQN: N fixed fractions, nothing sampled
            self.kappa, self.num_tau_samples = args.kappa, self.qr_dqn
            self.loss_core = qr.loss_core
        else:                                            # IQN sampling sizes (agent.py:58-63)
            for field in self._IQN_FIELDS:
                setattr(self, field, getattr(args, field))
            self.loss_core = compute_loss_iqn.loss_core
        self._inject = None  # parity hook: {"noises": (n0, n1, n2), "taus": (t0, t1, t2)}; Munchausen: two of each;
        #                      FQF and QR-DQN: {"noises": (n0, n1, n2)}; with random_shift, any of these may also carry
        #                      "shifts": (shifts_states, shifts_next_states), int32 (B, 2) (dy, dx), in place of the draw
        if self.rainbow_only:
            # the support the C51 head takes expectations over when it acts: h^-1 of the h-space support under rescaling
            self.acting_support = self.support
            if self.value_rescaling is not None:
                self.acting_support = torch.empty_like(self.support)
                _lib.call("riqn_value_rescale", self.atoms, _lib.ptr(self.support), self.value_rescaling, 1,
                          _lib.ptr(self.acting_support))
        # random_shift: only Learner.compute_gradients shifts; acting and the actors' priorities see the stored frames.
        # The side networks (arena.py), set by their modules' build (None when off), come after both DQNs in the fixed
        # order FQF, CURL, SPR: every network initialises from a seed as it would without the later ones
        self.fraction_net = self.fraction_optimiser = None
        self.curl_net = self.curl_optimiser = self.momentum_net = self.momentum_projection = None
        self.spr_net = self.spr_optimiser = self.spr_ema_projection = None
        self.sides = tuple(module.build(self, args, checkpoint)
                           for on, module in ((self.fqf, fqf), (self.curl, curl), (self.spr, spr)) if on is not None)
        # optimiser steps run and resets done (Learner.reset_networks): a resumed run resets at the same updates with the
        # same draws
        self.updates = self.resets = 0
        if self.reset is not None and checkpoint is not None and "reset_state" in checkpoint:
            self.updates, self.resets = (int(x) for x in checkpoint["reset_state"])
        self._discounts_fed = False   # the loss cores' nonterminals are per-transition discounts (Learner, horizon_anneal)

    def horizon(self):
        """(n, gamma) of the agent's updates: multi_step and discount (a Learner anneals them under horizon_anneal)."""
        return self.n, self.discount

    def gamma_n(self):
        """The gamma^n every loss core hands its kernel, which multiplies the nonterminals by it: 1.0 while a step feeds
        the per-transition discounts fl32(gamma^n) * nt in their place (Learner under horizon_anneal), otherwise
        gamma ** n of horizon()."""
        if self._discounts_fed:
            return 1.0
        n, gamma = self.horizon()
        return float(gamma ** n)

    def set_risk(self, measure, eta=None):
        """Act, and pick the double-DQN target action a*, under a distortion risk measure (IQN paper, section 3.1):
        ``measure`` is "neutral", "cvar", "wang", "cpw", "pow" or "norm" (model.RISK_MEASURES), ``eta`` its parameter.
        The K quantile fractions of those passes become beta(tau); the N and N' fractions of the loss stay uniform."""
        self.risk = config.read_risk(self._head, self._loss, measure, eta)

    @staticmethod
    def _read_checkpoint(path):
        """agent.py:26-34: a given but missing checkpoint is an error (bare Exception, like the reference)."""
        if not path:
            return None
        if not os.path.isfile(path):
            print("We didn't fint the model you gave as input!")
            raise Exception
        print("We loaded model ", path)
        return torch.load(path, map_location="cpu")

    def reset_noise(self):
        """agent.py:66-67"""
        self.online_net.reset_noise()

    def update_target_net(self):
        """agent.py:69-70 -- parameters AND epsilon buffers, as load_state_dict(state_dict()) copies them;
        here two flat device copies instead of 32 tensor copies."""
        self.target_net._flat.copy_(self.online_net._flat)
        self.target_net._eps_flat.copy_(self.online_net._eps_flat)
        self.target_net.compose_weights()

    def compute_loss_actor_or_learner(self, states, actions, returns, next_states, nonterminals, debug=None, demo=None):
        """agent.py:72-147: the loss (B,) of self.loss_core, differentiable with respect to the online network (and,
        under FQF, the fraction proposal) when grad mode is on.  ``debug``: dict that receives the core's intermediates.
        ``demo``: None, or the (B,) demonstration flags of a DQfD agent (dqfd.py).  CURL's auxiliary loss is not part of
        it, nor SPR's: only Learner.compute_gradients adds those terms."""
        if torch.is_grad_enabled():
            params = [p for p in self.online_net.parameters() if p.requires_grad]
            return _Loss.apply(self, states, actions, returns, next_states, nonterminals, debug, demo, *params)
        loss, _ = self.loss_core(self, states, actions, returns, next_states, nonterminals, debug=debug, keep_graph=False,
                                 demo=demo)
        return loss

    def save(self, path, T_actors, T_learner, name):
        """agent.py:150-160.  Under value rescaling the checkpoint also holds value_rescaling_eps, under QR-DQN
        qr_dqn_quantiles (N), under resets reset_state = (updates, resets), under target_ema target_state_dict (the EMA
        target, which the online network no longer determines; a checkpoint without it starts the target at the online
        network), and each side network's entries (Side.checkpoint); model_state_dict keeps the reference schema either
        way."""
        ckpt = {
            "T_actors": T_actors,
            "T_learner": T_learner,
            "model_state_dict": self.online_net.state_dict(),
            "optimiser_state_dict": self.optimiser.state_dict(),
        }
        if self.value_rescaling is not None:
            ckpt["value_rescaling_eps"] = self.value_rescaling
        if self.qr_dqn is not None:
            ckpt["qr_dqn_quantiles"] = self.qr_dqn
        if self.reset is not None:
            ckpt["reset_state"] = (self.updates, self.resets)
        if self.target_ema is not None:
            ckpt["target_state_dict"] = self.target_net.state_dict()
        for side in self.sides:
            ckpt.update(side.checkpoint())
        torch.save(ckpt, os.path.join(path, name))

    def train(self):
        self.online_net.train()

    def eval(self):
        self.online_net.eval()


class _Loss(torch.autograd.Function):
    """The agent's loss core as one autograd node.  The online network's parameters are inputs only so that the loss
    requires grad: the core's backward accumulates straight into the gradient arenas behind every parameter's .grad."""

    @staticmethod
    def forward(ctx, agent, states, actions, returns, next_states, nonterminals, debug, demo, *params):
        loss, ctx.bw = agent.loss_core(agent, states, actions, returns, next_states, nonterminals, debug=debug, demo=demo)
        ctx.n_params = len(params)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        ctx.bw(grad_loss)
        ctx.bw = None
        return (None,) * (8 + ctx.n_params)
