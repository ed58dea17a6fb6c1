"""Agent -- mirror of the reference ``rainbowiqn/agent.py:10-166`` (shared by Learner and Actor).

Same constructor ``Agent(args, action_space, redis_servor)`` reading the same ``args`` fields, same public
attributes (online_net, target_net, optimiser, n, history, discount, device, batch_size, kappa, num_tau_samples,
num_tau_prime_samples, num_quantile_samples, support, ...) and methods (reset_noise, update_target_net,
compute_loss_actor_or_learner, save, train, eval), plus ``loss_core`` for the loss the agent trains (c51.loss_core,
qr.loss_core or compute_loss_iqn.loss_core), ``risk`` / ``set_risk`` for risk-sensitive acting and
``munchausen`` for Munchausen-IQN targets, ``fqf`` / ``fraction_net`` / ``fraction_optimiser`` for FQF fractions,
``value_rescaling`` (and, for C51, ``acting_support``) for the transformed Bellman operator on unclipped rewards, and
``qr_dqn`` for QR-DQN's fixed-fraction quantile head, ``mmd`` for MMDQN's moment-matching loss on that head (mmd.py),
``hl_gauss`` for HL-Gauss's Gaussian-histogram loss on the C51 head (hl_gauss.py), ``cql`` for the conservative
regulariser of the IQN and QR-DQN losses (cql.py), ``dqfd`` for DQfD's large-margin loss on demonstrations (dqfd.py),
``random_shift`` for the
learner's random-shift augmentation (augment.py), and ``curl`` / ``curl_net`` / ``curl_optimiser`` / ``momentum_net`` /
``momentum_projection`` for CURL's contrastive loss on the trunk (curl.py).  The networks are rainbow_iqn_apex_b200.model.DQN (CUDA) and the
optimiser is the arena Adam; checkpoints keep the reference schema {T_actors, T_learner, model_state_dict,
optimiser_state_dict} (agent.py:150-160), plus the fraction network's two entries under FQF and CURL's three.
"""
import os

import torch

from . import _lib
from . import augment, c51, compute_loss_iqn, cql, curl, dqfd, fqf, hl_gauss, mmd, qr
from .model import DQN, check_risk
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
        # QR-DQN: optional args field (absent from the reference's namespace: off).  None, or N of qr.check_qr; checked
        # against the checkpoint before its weights load (a QR network with N = atoms has the C51 network's shapes)
        self.qr_dqn = qr.check_qr(getattr(args, "qr_dqn", 0), getattr(args, "num_tau_samples", None), action_space,
                                  rainbow_only=self.rainbow_only)
        if checkpoint is not None and checkpoint.get("qr_dqn_quantiles") != self.qr_dqn:
            raise ValueError(f"the checkpoint was trained with qr_dqn_quantiles = {checkpoint.get('qr_dqn_quantiles')} "
                             f"(None: not QR-DQN), the args ask for {self.qr_dqn}: the z-layers hold other quantities")
        self.online_net = DQN(args, action_space).to(device=args.device)
        if checkpoint is not None:
            self.online_net.load_state_dict(checkpoint["model_state_dict"])
        self.target_net = DQN(args, action_space).to(device=args.device)
        self.update_target_net()
        for net in (self.online_net, self.target_net):
            net.train()                                  # the target stays in train mode: it is noisy too
        for p in self.target_net.parameters():
            p.requires_grad = False
        self.optimiser = Adam(self.online_net.parameters(), lr=args.lr, eps=args.adam_eps)
        if checkpoint is not None:
            self.optimiser.load_state_dict(checkpoint["optimiser_state_dict"])

        # the head's sizes and the loss core this agent trains (every core returns (loss, backward))
        if self.rainbow_only:                            # categorical support (agent.py:49-57)
            for attr, field in self._C51_FIELDS:
                setattr(self, attr, getattr(args, field))
            self.support = torch.linspace(self.Vmin, self.Vmax, self.atoms).to(device=args.device)
            self.delta_z = (self.Vmax - self.Vmin) / (self.atoms - 1)
            self.loss_core = c51.loss_core
        elif self.qr_dqn is not None:                    # QR-DQN: N fixed fractions, nothing sampled
            self.kappa, self.num_tau_samples = args.kappa, self.qr_dqn
            self.loss_core = qr.loss_core
        else:                                            # IQN sampling sizes (agent.py:58-63)
            for field in self._IQN_FIELDS:
                setattr(self, field, getattr(args, field))
            self.loss_core = compute_loss_iqn.loss_core
        self._inject = None  # parity hook: {"noises": (n0, n1, n2), "taus": (t0, t1, t2)}; Munchausen: two of each;
        #                      FQF and QR-DQN: {"noises": (n0, n1, n2)}; with random_shift, any of these may also carry
        #                      "shifts": (shifts_states, shifts_next_states), int32 (B, 2) (dy, dx), in place of the draw
        # Munchausen-IQN targets: optional args fields (absent from the reference's namespace: plain IQN).
        # None, or (alpha, entropy_tau, l0) of compute_loss_iqn.check_munchausen
        self.munchausen = compute_loss_iqn.check_munchausen(
            getattr(args, "munchausen", 0),
            *(getattr(args, f, v) for f, v in compute_loss_iqn.MUNCHAUSEN_DEFAULTS.items()), rainbow_only=self.rainbow_only)
        # FQF fraction proposal: optional args fields (absent from the reference's namespace: plain IQN).
        # None, or (fraction_lr, entropy_coef) of fqf.check_fqf
        self.fqf = fqf.check_fqf(getattr(args, "fqf", 0), *(getattr(args, f, v) for f, v in fqf.FQF_DEFAULTS.items()),
                                 rainbow_only=self.rainbow_only, munchausen=self.munchausen,
                                 num_tau_samples=getattr(args, "num_tau_samples", None))
        if self.qr_dqn is not None:
            qr.check_qr(1, self.qr_dqn, munchausen=self.munchausen, fqf=self.fqf)
        # MMDQN: optional args fields (absent from the reference's namespace: off).  None, or the bandwidths of
        # mmd.check_mmd; fixed for the agent's life, so that a captured step graph stays valid
        self.mmd = mmd.check_mmd(getattr(args, "mmd", 0),
                                 getattr(args, "mmd_bandwidths", mmd.MMD_DEFAULTS["mmd_bandwidths"]),
                                 qr_dqn=self.qr_dqn, rainbow_only=self.rainbow_only, munchausen=self.munchausen,
                                 fqf=self.fqf)
        # HL-Gauss: optional args fields (absent from the reference's namespace: off).  None, or the float32 ratio
        # sigma / delta_z of hl_gauss.check_hl_gauss; fixed for the agent's life, since a captured step graph holds it
        self.hl_gauss = hl_gauss.check_hl_gauss(
            getattr(args, "hl_gauss", 0), getattr(args, "hl_gauss_sigma", hl_gauss.HL_GAUSS_DEFAULTS["hl_gauss_sigma"]),
            rainbow_only=self.rainbow_only)
        # CQL: optional args fields (absent from the reference's namespace: off).  None, or the float32 alpha of
        # cql.check_cql; fixed for the agent's life, since a captured step graph holds it
        self.cql = cql.check_cql(getattr(args, "cql", 0), getattr(args, "cql_alpha", cql.CQL_DEFAULTS["cql_alpha"]),
                                 rainbow_only=self.rainbow_only, munchausen=self.munchausen, fqf=self.fqf, mmd=self.mmd)
        # DQfD: optional args fields (absent from the reference's namespace: off).  None, or the float32 (margin, lambda)
        # of dqfd.check_dqfd; fixed for the agent's life, since a captured step graph holds them
        self.dqfd = dqfd.check_dqfd(getattr(args, "dqfd", 0),
                                    *(getattr(args, f, v) for f, v in dqfd.DQFD_DEFAULTS.items()),
                                    rainbow_only=self.rainbow_only, munchausen=self.munchausen, fqf=self.fqf, mmd=self.mmd,
                                    cql=self.cql)
        self.fraction_net = self.fraction_optimiser = None
        if self.fqf is not None:
            # drawn after both DQNs, so that their initialisation is that of a plain IQN agent from the same seed
            self.fraction_net = fqf.FractionProposal(self.num_tau_samples, args.device)
            self.fraction_optimiser = Adam(self.fraction_net.parameters(), lr=self.fqf[0], eps=args.adam_eps)
            if checkpoint is not None and "fraction_net_state_dict" in checkpoint:
                self.fraction_net.load_state_dict(checkpoint["fraction_net_state_dict"])
                self.fraction_optimiser.load_state_dict(checkpoint["fraction_optimiser_state_dict"])
        # value rescaling (the transformed Bellman operator): optional args fields (absent from the reference's namespace:
        # off).  None, or eps of compute_loss_iqn.check_value_rescaling; fixed for the agent's life, so that a captured
        # step graph stays valid
        self.value_rescaling = compute_loss_iqn.check_value_rescaling(
            getattr(args, "value_rescaling", 0),
            *(getattr(args, f, v) for f, v in compute_loss_iqn.VALUE_RESCALING_DEFAULTS.items()), munchausen=self.munchausen)
        if checkpoint is not None and checkpoint.get("value_rescaling_eps") != self.value_rescaling:
            raise ValueError(f"the checkpoint was trained with value_rescaling_eps = {checkpoint.get('value_rescaling_eps')} "
                             f"(None: off), the args ask for {self.value_rescaling}: a network trained in h-space acts "
                             "differently on the linear scale")
        if self.rainbow_only:
            # the support the C51 head takes expectations over when it acts: h^-1 of the h-space support under rescaling
            self.acting_support = self.support
            if self.value_rescaling is not None:
                self.acting_support = torch.empty_like(self.support)
                _lib.call("riqn_value_rescale", self.atoms, _lib.ptr(self.support), self.value_rescaling, 1,
                          _lib.ptr(self.acting_support))
        # random-shift augmentation of the learner's frames: optional args field (absent from the reference's namespace:
        # off).  None, or the pad p of augment.check_random_shift; fixed for the agent's life, so that a captured step graph
        # stays valid.  Only Learner.compute_gradients shifts; acting and the actors' priorities see the stored frames
        self.random_shift = augment.check_random_shift(getattr(args, "random_shift", 0))
        # CURL's contrastive auxiliary loss on the trunk: optional args fields (absent from the reference's namespace: off).
        # None, or the float32 (lambda, tau) of curl.check_curl; its modules are built last, so that both DQNs (and the
        # fraction proposal) initialise as a plain agent's from the same seed
        self.curl = curl.check_curl(getattr(args, "curl", 0),
                                    *(getattr(args, f, v) for f, v in curl.CURL_DEFAULTS.items()),
                                    random_shift=self.random_shift, batch_size=self.batch_size)
        self.curl_net = self.curl_optimiser = self.momentum_net = self.momentum_projection = None
        if self.curl is not None:
            curl.build(self, args, checkpoint)
        # risk-sensitive acting: optional args fields (absent from the reference's namespace: risk-neutral)
        self.risk = None
        self.set_risk(getattr(args, "risk_measure", "neutral"), getattr(args, "risk_eta", None))

    def set_risk(self, measure, eta=None):
        """Act, and pick the double-DQN target action a*, under a distortion risk measure (IQN paper, section 3.1):
        ``measure`` is "neutral", "cvar", "wang", "cpw", "pow" or "norm" (model.RISK_MEASURES), ``eta`` its parameter.
        The K quantile fractions of those passes become beta(tau); the N and N' fractions of the loss stay uniform."""
        risk = check_risk((measure, eta))
        if risk is not None and self.rainbow_only:
            raise ValueError("risk measures distort the IQN quantile fractions; rainbow_only (C51) acts risk-neutrally")
        if self.munchausen is not None:
            compute_loss_iqn.check_munchausen(1, *self.munchausen, risk=risk)
        if getattr(self, "fqf", None) is not None:
            fqf.check_fqf(1, *self.fqf, risk=risk)
        if getattr(self, "qr_dqn", None) is not None:
            qr.check_qr(1, self.qr_dqn, risk=risk)
        if getattr(self, "mmd", None) is not None:
            mmd.check_mmd(1, self.mmd, qr_dqn=self.qr_dqn, risk=risk)
        if getattr(self, "dqfd", None) is not None:
            dqfd.check_dqfd(1, *self.dqfd, rainbow_only=self.rainbow_only, munchausen=self.munchausen, fqf=self.fqf,
                            mmd=self.mmd, cql=self.cql)
        self.risk = risk

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
        it: only Learner.compute_gradients adds that term."""
        if torch.is_grad_enabled():
            params = [p for p in self.online_net.parameters() if p.requires_grad]
            return _Loss.apply(self, states, actions, returns, next_states, nonterminals, debug, demo, *params)
        loss, _ = self.loss_core(self, states, actions, returns, next_states, nonterminals, debug=debug, keep_graph=False,
                                 demo=demo)
        return loss

    def save(self, path, T_actors, T_learner, name):
        """agent.py:150-160.  Under FQF the checkpoint also holds fraction_net_state_dict and
        fraction_optimiser_state_dict, under value rescaling value_rescaling_eps, under QR-DQN qr_dqn_quantiles (N), under CURL
        curl_state_dict, curl_optimiser_state_dict and curl_momentum_state_dict; model_state_dict keeps the reference schema either way."""
        ckpt = {
            "T_actors": T_actors,
            "T_learner": T_learner,
            "model_state_dict": self.online_net.state_dict(),
            "optimiser_state_dict": self.optimiser.state_dict(),
        }
        if self.fqf is not None:
            ckpt["fraction_net_state_dict"] = self.fraction_net.state_dict()
            ckpt["fraction_optimiser_state_dict"] = self.fraction_optimiser.state_dict()
        if self.value_rescaling is not None:
            ckpt["value_rescaling_eps"] = self.value_rescaling
        if self.qr_dqn is not None:
            ckpt["qr_dqn_quantiles"] = self.qr_dqn
        if self.curl is not None:
            ckpt["curl_state_dict"] = self.curl_net.state_dict()
            ckpt["curl_optimiser_state_dict"] = self.curl_optimiser.state_dict()
            ckpt["curl_momentum_state_dict"] = curl.momentum_state_dict(self)
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
