"""FQF, the Fully parameterized Quantile Function (Yang, Zhao, Lin, Qin, Bian & Liu, NeurIPS 2019).

FQF keeps IQN's quantile-value network (model.DQN) and replaces its uniformly drawn fractions by N per-state fractions
from a small *fraction proposal network* on the detached trunk features psi(s):

  logits = psi(s) W_f^T + b_f ,  P = softmax(logits) ,  tau_0 = 0, tau_i = sum_{k<i} P_k, tau_N = 1
  tau_hat_i = (tau_i + tau_{i+1}) / 2 ,  dtau_i = tau_{i+1} - tau_i ,  Q(s, a) = sum_i dtau_i F(s, tau_hat_i, a)

The proposal is trained on the exact gradient of the 1-Wasserstein distance between the quantile function and its
N-step approximation (the paper's Proposition 1), minus an optional entropy bonus; see riqn_fqf_fraction_bwd.

FractionProposal holds W_f (N, 3136) and b_f (N) in its own flat parameter / gradient arena, beside the DQN's: the DQN's
arena, parameter order and state_dict stay those of the reference.  It lives on the Agent (agent.fraction_net, trained
by agent.fraction_optimiser, the arena Adam; the paper used RMSProp).  There is no target copy: fractions always come
from the online proposal.
"""
import torch
from torch import nn

from ._lib import call, ptr
from .arena import ArenaModule, Side
from .model import FEAT


class FractionProposal(ArenaModule):
    """The fraction proposal network: one linear layer ``weight`` (N, 3136), ``bias`` (N), views of one flat fp32 arena.
    Xavier-uniform weights with gain 0.01 and a zero bias: the starting fractions are nearly uniform."""

    NAMES = ("weight", "bias")

    def __init__(self, num_fractions, device, feat_dim=FEAT):
        super().__init__()
        self.num_fractions, self.feat_dim = int(num_fractions), int(feat_dim)
        self.weight = nn.Parameter(torch.empty(self.num_fractions, self.feat_dim))
        self.bias = nn.Parameter(torch.zeros(self.num_fractions))
        nn.init.xavier_uniform_(self.weight.data, gain=0.01)
        self._flatten(torch.device(device))

    def propose(self, feat):
        """Fractions of the states behind ``feat`` (B, 3136) fp32 (read only; nothing flows back into the trunk).
        Returns dict(logits (B, N), tau (B, N+1), tau_hat (N*B, 1), dtau (N*B,), entropy (B,)), quantile-major rows
        r = i*B + b for tau_hat / dtau as the IQN head expects (riqn_fqf_fractions)."""
        B, N, dev = feat.shape[0], self.num_fractions, feat.device
        feat = feat if feat.is_contiguous() else feat.contiguous()
        logits = torch.empty(B, N, device=dev)
        call("riqn_linear_fwd_ld", B, self.feat_dim, N, ptr(feat), self.feat_dim, ptr(self.weight), ptr(self.bias),
             ptr(logits), N, 0)
        tau = torch.empty(B, N + 1, device=dev)
        tau_hat = torch.empty(N * B, 1, device=dev)
        dtau = torch.empty(N * B, device=dev)
        entropy = torch.empty(B, device=dev)
        call("riqn_fqf_fractions", B, N, ptr(logits), ptr(tau), ptr(tau_hat), ptr(dtau), ptr(entropy))
        return dict(logits=logits, tau=tau, tau_hat=tau_hat, dtau=dtau, entropy=entropy, feat=feat)

    def backward(self, fr, q_hat, q_bnd, actions, gscale, gscale_mul, entropy_coef):
        """Accumulate the fraction loss's gradient into the arena for the proposal ``fr`` (propose()), the gradient
        pass's quantile values ``q_hat`` at tau_hat and the boundary pass's ``q_bnd`` at tau_1..tau_{N-1}.  The surrogate
        of transition b is weighted by gscale[b] * gscale_mul, like the quantile loss.  Returns (dlogits (B, N),
        fraction loss (B,) unweighted)."""
        B, N, dev = fr["logits"].shape[0], self.num_fractions, fr["logits"].device
        dlogits = torch.empty(B, N, device=dev)
        floss = torch.empty(B, device=dev)
        call("riqn_fqf_fraction_bwd", B, N, q_hat.shape[1], ptr(fr["logits"]), ptr(fr["tau"]), ptr(q_hat), ptr(q_bnd),
             ptr(actions), ptr(gscale), float(gscale_mul), float(entropy_coef), ptr(dlogits), ptr(floss))
        call("riqn_fqf_fraction_wgrad", B, N, self.feat_dim, ptr(dlogits), ptr(fr["feat"]), ptr(self.grad_view(self.weight)),
             ptr(self.grad_view(self.bias)))
        return dlogits, floss


def build(agent, args, checkpoint):
    """agent.fraction_net and agent.fraction_optimiser (learning rate agent.fqf[0]), restored from ``checkpoint`` when it
    holds them.  Returns FQF's Side: the actors act on the learner's fractions, so Ape-X publishes its arena."""
    from .optim import Adam
    net = agent.fraction_net = FractionProposal(agent.num_tau_samples, args.device)
    opt = agent.fraction_optimiser = Adam(net.parameters(), lr=agent.fqf[0], eps=args.adam_eps)
    if checkpoint is not None and "fraction_net_state_dict" in checkpoint:
        net.load_state_dict(checkpoint["fraction_net_state_dict"])
        opt.load_state_dict(checkpoint["fraction_optimiser_state_dict"])
    return Side(1, net, opt,
                lambda: {"fraction_net_state_dict": net.state_dict(), "fraction_optimiser_state_dict": opt.state_dict()},
                broadcast=(net._flat,), publish=True)


def q_values(q, dtau, batch, num_fractions, action_space):
    """(B, A) FQF action values sum_i dtau_i F(s, tau_hat_i, a) from a head pass ``q`` (N*B, A) at tau_hat."""
    return (q.view(num_fractions, batch, action_space) * dtau.view(num_fractions, batch, 1)).sum(0)
