"""GPU: DQN.forward / NoisyLinear.forward under torch autograd.  A scalar built from the network's output by ordinary
torch code, then .backward(), leaves every parameter gradient in param.grad: the dense head backward
(riqn_dueling_bwd_dense[_bf16], riqn_c51_head_bwd_dense) feeds the same z-layer / hidden-layer / embedding / trunk
backward as the fused learner loss.  Everything is checked against the oracle (torch fp32 autograd) with injected
noise and quantiles, at the tolerances of tests/test_gpu_learn.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_params, make_args
from oracle import cases, losses, network as net
from test_gpu_learn import _dev_batch, _grad_tol, _learner, _loss_tol, precision  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
MODES = [("fp32", "fp32"), ("bf16x3", "bf16x3"), ("bf16x3", "bf16"), ("bf16", "bf16"), ("fp16", "bf16")]


def _oracle_params(params, noise, dev, requires_grad=True):
    p = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in params.items()}
    net.apply_noise(p, {k: (a.to(dev), b.to(dev)) for k, (a, b) in noise.items()})
    for k, t in p.items():
        if requires_grad and net.is_trainable(k):
            t.requires_grad_(True)
    return p


def _net(dev, params, noise, batch=32, rainbow_only=False):
    from rainbow_iqn_apex_b200.model import DQN
    d = DQN(make_args(dev, batch, rainbow_only=rainbow_only), 18).to(dev)
    load_params(d, params)
    d.reset_noise(noise)
    d.zero_grad()
    return d


def _cmp_grads(d, p_or, strict_rel, relaxed=()):
    """cosine >= 0.999 for every parameter and norm-relative error below ``strict_rel``; parameters whose names start
    with one of ``relaxed`` (upstream of a ReLU kink that rounds to opposite sides of 0 in the product and the oracle)
    get test_gpu_learn's bound for that case, cosine > 0.98 and relative error < 0.2."""
    errs = []
    for k, p in d.named_parameters():
        gg, gr = p.grad.detach().double(), p_or[k].grad.detach().double().to(p.device)
        errs.append((k, float((gg * gr).sum() / (gg.norm() * gr.norm() + 1e-30)),
                     float((gg - gr).norm() / (gr.norm() + 1e-30))))
    for k, cos, rel in errs:
        print(f"  {k}: cos {cos:.6f} rel {rel:.2e}")
    for k, cos, rel in errs:
        if k.startswith(tuple(relaxed)):
            assert cos > 0.98 and rel < 0.2, (k, cos, rel)
        else:
            assert cos >= 0.999 and rel < strict_rel, (k, cos, rel)


def _oracle_no_tf32():
    """The C51 and NoisyLinear oracles run on the device: no TF32 in their products."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    return old


def _restore_tf32(old):
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _rel_tol(mode):
    """Norm-relative gradient bound: test_gpu_learn's 3e-2 for bf16 / fp16 forward operands; 1e-2 for the other
    tensor-core backwards, whose z-layer weight gradient (riqn_z_wgrad_tc) is one bf16 product even in bf16x3 mode."""
    if mode[0] in ("bf16", "fp16"):
        return 3e-2
    return _grad_tol() if mode[1] == "fp32" else 1e-2


# ----------------------------------------------------------------------------------------------------------------- IQN
_IQN_ORACLE = {}


def _iqn_case(batch, nq):
    """Seeded inputs and the oracle's q and gradients of (q * G).sum() (on the host: the oracle's cosine embedding
    builds host tensors), computed once per shape and shared by the precision modes."""
    if (batch, nq) not in _IQN_ORACLE:
        seed = 31 + batch
        params, noise = net.make_params(seed), net.make_noise(seed + 1)
        x = torch.from_numpy(cases.make_batch(seed + 2, batch)["states"])
        tau = torch.from_numpy(np.random.RandomState(seed + 3).uniform(0, 1, (nq * batch, 1)).astype(np.float32))
        G = torch.from_numpy(np.random.RandomState(seed + 4).standard_normal((nq * batch, 18)).astype(np.float32))
        p_or, keep = _oracle_params(params, noise, "cpu"), {}
        q_ref = net.dqn_forward_iqn(p_or, x.float() / 255, nq, tau, keep=keep)
        (q_ref * G).sum().backward()
        acts = [keep[k].detach() > 0 for k in ("o1", "o2", "o3", "h_v", "h_a")]
        _IQN_ORACLE[(batch, nq)] = (params, noise, x, tau, G, q_ref.detach(), p_or, acts)
    return _IQN_ORACLE[(batch, nq)]


def _relu_flips(d, x, nq, tau, acts):
    """ReLU kinks on opposite sides of 0 in the product and the oracle: (conv1-3, hidden layers)."""
    k = {}
    with torch.no_grad():
        d.forward(x, nq, tau=tau, keep=k, fresh_weights=True)
    B = x.shape[0]
    h = k["h"].reshape(B, nq, -1).transpose(0, 1).reshape(B * nq, -1).cpu() > 0     # sample-major -> quantile-major
    mine = [o.cpu() > 0 for o in k["out"]] + [h[:, :512], h[:, 512:]]
    n = [int((a != b).sum()) for a, b in zip(mine, acts)]
    return sum(n[:3]), sum(n[3:])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch,nq", [(32, 8), (512, 64), (13, 13)])     # 13 x 13: the fp32 trunk and head backwards
def test_iqn_dense_upstream_gradient_vs_oracle(cuda_dev, precision, batch, nq, mode):
    precision(*mode)
    params, noise, x, tau, G, q_ref, p_or, acts = _iqn_case(batch, nq)
    d = _net(cuda_dev, params, noise, batch)
    xd, td = x.to(cuda_dev), tau.to(cuda_dev)
    q, tau_out = d(xd, nq, tau=td)
    assert q.grad_fn is not None and not tau_out.requires_grad
    (q * G.to(cuda_dev)).sum().backward()
    q = q.detach().cpu()
    err = float((q - q_ref).abs().max() / q_ref.abs().max())
    trunk_flips, head_flips = _relu_flips(d, xd, nq, td, acts)
    print(f"mode {mode} B={batch} N={nq}: q rel err {err:.2e}, ReLU flips trunk {trunk_flips} head {head_flips}")
    assert err < {"bf16": 2e-3}.get(mode[0], _loss_tol()), err      # test_gpu_learn's activation bound for bf16
    # the z-layers are upstream of no kink: they always take the strict bound
    relaxed = (("conv",) if trunk_flips or head_flips else ()) + (("iqn_fc", "fcnoisy_h_") if head_flips else ())
    _cmp_grads(d, p_or, _rel_tol(mode), relaxed)


def test_reference_iqn_loss_by_hand_matches_learner(cuda_dev):
    """compute_loss_iqn.py:216-358 written with net(...) calls and the oracle's pairwise loss on device tensors, then
    (w * loss).mean().backward(): the same losses and gradients as the fused Learner.compute_gradients."""
    batch, cfg, seed = 32, cases.iqn_cfg(64, 64, 32), 4242
    K, Np, N = cfg["n_quantile"], cfg["n_tau_prime"], cfg["n_tau"]
    params = net.make_params(seed)
    b = cases.make_batch(seed + 1, batch)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, batch, cfg))
    noises = cases.make_noises(seed + 3)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)

    lr = _learner(cuda_dev, batch, cfg, params)
    lr._inject = dict(noises=noises, taus=taus)
    loss_fused = lr.compute_gradients(st, ac, rt, nx, nt, w)
    g_fused = {k: p.grad.detach().clone() for k, p in lr.online_net.named_parameters()}

    lr2 = _learner(cuda_dev, batch, cfg, params)
    on, tg = lr2.online_net, lr2.target_net
    dev_t = [t.to(cuda_dev) for t in taus]
    on.reset_noise(noises[0])
    with torch.no_grad():
        q_sel, _ = on(nx, K, tau=dev_t[0])
        a_star = q_sel.view(K, batch, 18).mean(0).argmax(1)
        tg.reset_noise(noises[1])
        q_tgt, _ = tg(nx, Np, tau=dev_t[1])
        q_tgt_a = q_tgt.gather(1, a_star[:, None].repeat(Np, 1))
        gamma_n = cfg["discount"] ** cfg["n_step"]
        target = (rt[:, None].repeat(Np, 1) + gamma_n * nt[:, None].repeat(Np, 1) * q_tgt_a).view(Np, batch).t()
    on.reset_noise(noises[2])
    q_on, tau = on(st, N, tau=dev_t[2])
    theta = q_on.gather(1, ac[:, None].repeat(N, 1)).view(N, batch).t()
    loss = losses.iqn_pairwise_loss(theta, target, tau.view(N, batch).t(), cfg["kappa"])
    on.zero_grad()
    (w * loss).mean().backward()

    lf, lh = loss_fused.detach(), loss.detach()
    assert float(((lf - lh).abs() / lh.abs()).max()) < _loss_tol()
    for k, p in on.named_parameters():
        gg, gr = p.grad.double(), g_fused[k].double()
        cos = float((gg * gr).sum() / (gg.norm() * gr.norm() + 1e-30))
        rel = float((gg - gr).norm() / (gr.norm() + 1e-30))
        assert cos >= 0.999 and rel < _grad_tol(), (k, cos, rel)


# ----------------------------------------------------------------------------------------------------------------- C51
@pytest.mark.parametrize("log", [True, False])
@pytest.mark.parametrize("batch", [32, 512, 13])                        # 13: the fp32 trunk backward
def test_c51_dense_upstream_gradient_vs_oracle(cuda_dev, batch, log):
    seed = 77 + batch
    params, noise = net.make_params(seed, rainbow_only=True), net.make_noise(seed + 1, rainbow_only=True)
    x = torch.from_numpy(cases.make_batch(seed + 2, batch)["states"]).to(cuda_dev)
    G = torch.from_numpy(np.random.RandomState(seed + 4).standard_normal((batch, 18, 51)).astype(np.float32)).to(cuda_dev)
    d = _net(cuda_dev, params, noise, batch, rainbow_only=True)
    out = d(x, log=log)
    assert out.grad_fn is not None
    (out * G).sum().backward()
    old = _oracle_no_tf32()
    try:
        p_or = _oracle_params(params, noise, cuda_dev)
        ref = net.dqn_forward_c51(p_or, x.float() / 255, 18, 51, log=log)
        (ref * G).sum().backward()
    finally:
        _restore_tf32(old)
    err = float((out.detach() - ref.detach()).abs().max() / ref.detach().abs().max())
    assert err < _loss_tol(), err
    _cmp_grads(d, p_or, _rel_tol(("fp16", "bf16")))


# ------------------------------------------------------------------------------------------------------- accumulation
def _two_forwards(d, x1, x2, tau1, tau2, G1, G2, together):
    d.zero_grad()
    if together:
        q1, _ = d(x1, 8, tau=tau1)
        q2, _ = d(x2, 8, tau=tau2)
        ((q1 * G1).sum() + (q2 * G2).sum()).backward()
    else:
        q1, _ = d(x1, 8, tau=tau1)
        (q1 * G1).sum().backward()
        q2, _ = d(x2, 8, tau=tau2)
        (q2 * G2).sum().backward()
    return d._flat_grad.clone()


def test_forwards_accumulate_and_repeat_bitwise(cuda_dev):
    params, noise = net.make_params(5), net.make_noise(6)
    d = _net(cuda_dev, params, noise)
    rs = np.random.RandomState(7)
    x1, x2 = (torch.from_numpy(rs.randint(0, 256, (32, 4, 84, 84)).astype(np.uint8)).to(cuda_dev) for _ in range(2))
    tau1, tau2 = (torch.from_numpy(rs.uniform(0, 1, (256, 1)).astype(np.float32)).to(cuda_dev) for _ in range(2))
    G1, G2 = (torch.from_numpy(rs.standard_normal((256, 18)).astype(np.float32)).to(cuda_dev) for _ in range(2))
    g_sum = _two_forwards(d, x1, x2, tau1, tau2, G1, G2, together=True)
    g_sep = _two_forwards(d, x1, x2, tau1, tau2, G1, G2, together=False)
    assert float((g_sum - g_sep).norm() / g_sep.norm()) < 1e-5
    g_again = _two_forwards(d, x1, x2, tau1, tau2, G1, G2, together=True)
    assert torch.equal(g_sum, g_again)


# ------------------------------------------------------------------------------------------------------------ errors
def test_stale_or_repeated_backward_and_input_grad_raise(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent
    params, noise = net.make_params(8), net.make_noise(9)
    ag = Agent(make_args(cuda_dev, 8), 18, None)
    load_params(ag.online_net, params)
    d = ag.online_net
    d.reset_noise(noise)
    x = torch.from_numpy(cases.make_batch(10, 8)["states"]).to(cuda_dev)

    def fwd():
        return d(x, 8)[0].sum()

    sd = {k: v.clone() for k, v in d.state_dict().items()}
    for change in (lambda: d.reset_noise(noise), lambda: ag.optimiser.step(), lambda: d.load_state_dict(sd),
                   lambda: d.compose_weights()):
        d.zero_grad()
        loss = fwd()
        change()
        with pytest.raises(RuntimeError, match="changed between this forward and its backward"):
            loss.backward()
    d.reset_noise(noise)
    loss = fwd()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already ran"):
        loss.backward()
    xf = (x.float() / 255).requires_grad_(True)
    with pytest.raises(RuntimeError, match="not for its inputs"):
        d(xf, 8)
    with torch.no_grad():                               # no autograd node: the input's requires_grad does not matter
        q, _ = d(xf, 8)
    assert q.grad_fn is None


@pytest.mark.parametrize("rainbow_only", [False, True])
def test_eval_mode_leaves_sigma_gradients_alone(cuda_dev, rainbow_only):
    seed = 12
    params = net.make_params(seed, rainbow_only=rainbow_only)
    noise = net.make_noise(seed + 1, rainbow_only=rainbow_only)
    d = _net(cuda_dev, params, noise, rainbow_only=rainbow_only)
    d.eval()
    x = torch.from_numpy(cases.make_batch(seed + 2, 32)["states"]).to(cuda_dev)
    sig = {k: p for k, p in d.named_parameters() if "sigma" in k}
    for p in sig.values():
        p.grad.fill_(0.25)
    if rainbow_only:
        G = torch.from_numpy(np.random.RandomState(seed + 4).standard_normal((32, 18, 51)).astype(np.float32)).to(cuda_dev)
        (d(x, log=True) * G).sum().backward()
    else:
        tau = torch.from_numpy(np.random.RandomState(seed + 3).uniform(0, 1, (256, 1)).astype(np.float32)).to(cuda_dev)
        G = torch.from_numpy(np.random.RandomState(seed + 4).standard_normal((256, 18)).astype(np.float32)).to(cuda_dev)
        (d(x, 8, tau=tau)[0] * G).sum().backward()
    for k, p in sig.items():
        assert torch.equal(p.grad, torch.full_like(p.grad, 0.25)), k
    p_or = _oracle_params(params, noise, "cpu")           # on the host (the IQN oracle builds host tensors)
    xf = x.cpu().float() / 255
    if rainbow_only:
        ref = net.dqn_forward_c51(p_or, xf, 18, 51, log=True, training=False)
    else:
        ref = net.dqn_forward_iqn(p_or, xf, 8, tau.cpu(), training=False)
    (ref * G.cpu()).sum().backward()
    for k, p in d.named_parameters():
        if k not in sig:
            gg, gr = p.grad.double().cpu(), p_or[k].grad.double()
            cos = float((gg * gr).sum() / (gg.norm() * gr.norm() + 1e-30))
            assert cos >= 0.999, (k, cos)


# ------------------------------------------------------------------------------------------------------- NoisyLinear
@pytest.mark.parametrize("training", [True, False])
def test_noisy_linear_gradients_vs_f_linear(cuda_dev, training):
    from rainbow_iqn_apex_b200.model import NoisyLinear
    torch.manual_seed(3)
    layer = NoisyLinear(256, 96, 0.5).to(cuda_dev)
    layer.reset_noise(seed=11)
    layer.train(training)
    x = torch.randn(40, 256, device=cuda_dev, requires_grad=True)
    G = torch.randn(40, 96, device=cuda_dev)
    y = layer(x)
    (y * G).sum().backward()
    old = _oracle_no_tf32()
    try:
        ref = {k: t.detach().clone().requires_grad_(True) for k, t in
               (("weight_mu", layer.weight_mu), ("weight_sigma", layer.weight_sigma), ("bias_mu", layer.bias_mu),
                ("bias_sigma", layer.bias_sigma))}
        xr = x.detach().clone().requires_grad_(True)
        if training:
            yr = F.linear(xr, ref["weight_mu"] + ref["weight_sigma"] * layer.weight_epsilon,
                          ref["bias_mu"] + ref["bias_sigma"] * layer.bias_epsilon)
        else:
            yr = F.linear(xr, ref["weight_mu"], ref["bias_mu"])
        (yr * G).sum().backward()
    finally:
        _restore_tf32(old)
    assert torch.allclose(y.detach(), yr.detach(), rtol=1e-5, atol=1e-5)
    assert torch.allclose(x.grad, xr.grad, rtol=1e-4, atol=1e-5)
    for k, t in ref.items():
        p = getattr(layer, k)
        if t.grad is None:                      # eval mode: sigma is not in the graph
            assert p.grad is None, k
        else:
            assert torch.allclose(p.grad, t.grad, rtol=1e-4, atol=1e-5), k
