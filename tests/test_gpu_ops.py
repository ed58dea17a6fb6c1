"""GPU: per-op parity of the CUDA kernels (through the C-ABI) against the CPU oracle."""
import numpy as np
import pytest
import torch

from helpers import load_params, make_args, rel_err
from oracle import cases, network as net

pytestmark = pytest.mark.gpu


def _call():
    from rainbow_iqn_apex_b200._lib import call, ptr
    return call, ptr


@pytest.mark.parametrize("M,N,K,ta,tb", [(130, 70, 33, False, False), (257, 129, 64, True, False),
                                         (64, 300, 1000, False, True), (19, 1024, 777, True, True)])
def test_gemm_f32_strided(cuda_dev, M, N, K, ta, tb):
    call, ptr = _call()
    rs = np.random.RandomState(0)
    A = rs.standard_normal((M, K)).astype(np.float32)
    B = rs.standard_normal((N, K)).astype(np.float32)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    a = torch.from_numpy(A.T.copy() if ta else A).to(cuda_dev)
    b = torch.from_numpy(B.T.copy() if tb else B).to(cuda_dev)
    c = torch.empty(M, N, device=cuda_dev)
    sa = (1, M) if ta else (K, 1)
    sb = (1, N) if tb else (K, 1)
    call("riqn_gemm_f32", M, N, K, ptr(a), sa[0], sa[1], ptr(b), sb[0], sb[1], ptr(c), N)
    assert rel_err(c.cpu().numpy(), ref) < 1e-5


@pytest.fixture(scope="module")
def nets(cuda_dev):
    from rainbow_iqn_apex_b200.model import DQN
    params = net.make_params(7)
    d = DQN(make_args(cuda_dev), 18).to(cuda_dev)
    load_params(d, params)
    return d, params


def test_trunk_u8_and_f32(cuda_dev, nets):
    d, params = nets
    b = cases.make_batch(3, 6)
    p = net.to_torch(params)
    ref = net.conv_trunk(p, torch.from_numpy(b["states"]).float().div_(255)).numpy()
    got_u8 = d.trunk(torch.from_numpy(b["states"]).to(cuda_dev)).cpu().numpy()
    got_f32 = d.trunk(torch.from_numpy(b["states"]).float().div_(255).to(cuda_dev)).cpu().numpy()
    assert rel_err(got_u8, ref) < 3e-5      # split-bf16x3 tensor-core convolution
    # uint8 ingest folds the /255 into the weights (pixel values are exact bf16 operands); fp32 ingest splits x/255
    assert rel_err(got_u8, got_f32) < 1e-5
    # strided window view (B, 7, 84, 84)[:, 3:7]
    win = torch.from_numpy(np.concatenate([b["states"][:, :3], b["next_states"]], axis=1)).to(cuda_dev)
    got_view = d.trunk(win[:, 3:7]).cpu().numpy()
    ref2 = net.conv_trunk(p, torch.from_numpy(b["next_states"]).float().div_(255)).numpy()
    assert rel_err(got_view, ref2) < 3e-5


def test_trunk_u8_im2col_fallback(cuda_dev):
    """uint8 frames the strip convolution does not take (history 3: conv1's block width 16*3 is not a multiple of 64) run
    the explicit im2col on the tensor cores: riqn_conv_fwd_tc forward, riqn_conv_bwd_tc backward."""
    from rainbow_iqn_apex_b200 import DQN
    B = 8                        # im2col row counts B*400, B*81, B*49 are multiples of 8: the backward stays on the tensor cores
    args = make_args(cuda_dev)
    args.history_length = 3
    d = DQN(args, 18).to(cuda_dev)
    params = net.make_params(17, history=3)
    load_params(d, params)
    rs = np.random.RandomState(8)
    frames = rs.randint(0, 256, (B, 3, 84, 84)).astype(np.uint8)
    x = torch.from_numpy(frames).to(cuda_dev)
    xf = torch.from_numpy(frames.astype(np.float32) / np.float32(255))      # correctly rounded x / 255, as the kernels do
    p = net.to_torch(params, requires_grad=True)
    ref = net.conv_trunk(p, xf)
    got = d.trunk(x)
    assert rel_err(got.cpu().numpy(), ref.detach().numpy()) < 3e-5
    # the uint8 im2col splits x / 255 into the same bf16 hi / lo operands as the fp32 im2col of x / 255
    assert torch.equal(got, d.trunk(xf.to(cuda_dev)))
    keep = {}
    d.zero_grad()
    d.trunk(x, keep)
    assert keep["bwd_tc"] and keep["strip_bwd"] is None
    dfeat = torch.from_numpy(rs.standard_normal((B, 3136)).astype(np.float32))
    d.backward_trunk(keep, dfeat.to(cuda_dev))
    ref.backward(dfeat)
    for name in ("conv1", "conv2", "conv3"):
        for part in ("weight", "bias"):
            g_ref = p[f"{name}.{part}"].grad
            g = d.grad_view(getattr(getattr(d, name), part)).cpu()
            assert float((g - g_ref).norm() / g_ref.norm()) < 1e-2, (name, part)   # bf16 backward


def test_forward_injected(cuda_dev, nets):
    d, params = nets
    B, Nq = 5, 8
    b = cases.make_batch(4, B)
    noise = net.make_noise(11)
    tau = torch.from_numpy(np.random.RandomState(5).uniform(0, 1, (Nq * B, 1)).astype(np.float32))
    p = net.apply_noise(net.to_torch(params), noise)
    keep = {}
    ref = net.dqn_forward_iqn(p, torch.from_numpy(b["states"]).float().div_(255), Nq, tau, keep=keep)
    d.train()
    d.reset_noise(noise)
    k2 = {}
    q, tau_out = d.forward(torch.from_numpy(b["states"]).to(cuda_dev), Nq, tau=tau, keep=k2, fresh_weights=True)
    assert torch.equal(tau_out.cpu(), tau)
    tc = k2["tc"]

    def qmajor(t):   # head-internal rows are sample-major (b*Nq + q); the oracle's are quantile-major (q*B + b)
        return t.reshape(B, Nq, -1).transpose(0, 1).reshape(B * Nq, -1)

    cos_gpu = qmajor(tc["cos_hi"].float() + tc["cos_lo"].float()).cpu().numpy()    # bf16 hi + lo images
    assert rel_err(cos_gpu, keep["cos"].numpy()) < 2e-5
    if tc["f16"]:     # default arithmetic: x leaves as fp16(x) (head forward operand) + bf16(x) (backward operand)
        assert tc["x_hi"].dtype == torch.float16
        assert rel_err(qmajor(tc["x_hi"].float()).cpu().numpy(), keep["x"].numpy()) < 5e-4
        assert rel_err(qmajor(tc["x_lo"].float()).cpu().numpy(), keep["x"].numpy()) < 4e-3
        htol = 3e-4
    else:
        x_gpu = qmajor(tc["x_hi"].float() + tc["x_lo"].float()).cpu().numpy()
        assert rel_err(x_gpu, keep["x"].numpy()) < 3e-5
        htol = 1e-4                                                              # split-bf16x3 tensor-core products
    h_gpu = qmajor(k2["h"])
    assert rel_err(h_gpu[:, :512].cpu().numpy(), keep["h_v"].numpy()) < htol
    assert rel_err(h_gpu[:, 512:].cpu().numpy(), keep["h_a"].numpy()) < htol
    assert rel_err(q.cpu().numpy(), ref.numpy()) < htol
    # stored epsilons == outer product of the injected factors (model.py:39-43), bit for bit
    assert torch.equal(d.fcnoisy_h_a.weight_epsilon.cpu(), torch.outer(noise["fcnoisy_h_a"][1], noise["fcnoisy_h_a"][0]))
    # eval mode uses mu only (model.py:52-53)
    d.eval()
    q_eval, _ = d.forward(torch.from_numpy(b["states"]).to(cuda_dev), Nq, tau=tau)
    ref_eval = net.dqn_forward_iqn(p, torch.from_numpy(b["states"]).float().div_(255), Nq, tau, training=False)
    assert rel_err(q_eval.cpu().numpy(), ref_eval.numpy()) < htol
    d.train()


def test_adam_matches_torch(cuda_dev):
    call, ptr = _call()
    rs = np.random.RandomState(2)
    n = 10007
    p0 = rs.standard_normal(n).astype(np.float32)
    p_ref = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([p_ref], lr=5e-5, eps=3.125e-4)
    p = torch.from_numpy(p0.copy()).to(cuda_dev)
    m = torch.zeros(n, device=cuda_dev)
    v = torch.zeros(n, device=cuda_dev)
    for step in range(1, 4):
        g = (rs.standard_normal(n) * 10.0 ** rs.randint(-6, 1, n)).astype(np.float32)
        p_ref.grad = torch.from_numpy(g.copy())
        opt.step()
        gd = torch.from_numpy(g).to(cuda_dev)
        call("riqn_adam_step", n, ptr(p), ptr(gd), ptr(m), ptr(v), step, 5e-5, 0.9, 0.999, 3.125e-4, 1.0, None)
        assert np.allclose(p.cpu().numpy(), p_ref.detach().numpy(), rtol=0, atol=2.5e-7)   # <= 1 fp32 ulp of |p| < 4
        upd, upd_ref = p.cpu().numpy() - p0, p_ref.detach().numpy() - p0
        assert rel_err(upd, upd_ref) < 5e-3
    assert rel_err(m.cpu().numpy(), opt.state[p_ref]["exp_avg"].numpy()) < 1e-6


def test_device_rng_statistics(cuda_dev):
    call, ptr = _call()
    n = 1 << 20
    u = torch.empty(n, device=cuda_dev)
    call("riqn_fill_uniform", n, 1234, 0, ptr(u), None)
    u2 = torch.empty(n, device=cuda_dev)
    call("riqn_fill_uniform", n, 1234, 1, ptr(u2), None)
    a = u.cpu().numpy().astype(np.float64)
    assert 0 < a.min() and a.max() < 1 and abs(a.mean() - 0.5) < 2e-3 and abs(a.var() - 1 / 12) < 1e-3
    assert abs(np.corrcoef(a, u2.cpu().numpy())[0, 1]) < 5e-3
    z = torch.empty(n, device=cuda_dev)
    call("riqn_noisy_sample", n, 99, 0, ptr(z), None)
    f = z.cpu().numpy().astype(np.float64)
    x = np.sign(f) * f * f                      # invert f(x) = sign(x) sqrt|x|  -> N(0,1)
    assert abs(x.mean()) < 5e-3 and abs(x.var() - 1) < 1e-2 and abs((x ** 4).mean() - 3) < 0.1


def test_noisy_reset_net_matches_per_layer_calls(cuda_dev):
    """riqn_noisy_reset_net (two launches per network) draws and composes exactly what riqn_noisy_sample +
    riqn_noisy_compose produce layer by layer on the same seed / stream ids (model.py:32-43,159-162)."""
    from rainbow_iqn_apex_b200._lib import NoisyLayer
    call, ptr = _call()
    shapes = [(512, 3136), (512, 3136), (1, 512), (18, 512)]
    seed, g = 4242, torch.Generator().manual_seed(5)
    keep, desc = [], (NoisyLayer * len(shapes))()
    for k, (o, i) in enumerate(shapes):
        t = dict(mu=torch.randn(o, i, generator=g), sg=torch.rand(o, i, generator=g), bmu=torch.randn(o, generator=g),
                 bsg=torch.rand(o, generator=g))
        t = {n: v.to(cuda_dev) for n, v in t.items()}
        for n, shp in (("eps", (o, i)), ("beps", (o,)), ("ein", (i,)), ("eout", (o,)), ("w", (o, i)), ("b", (o,))):
            t[n] = torch.zeros(*shp, device=cuda_dev)
            t[n + "_ref"] = torch.zeros(*shp, device=cuda_dev)
        keep.append(t)
        d = desc[k]
        d.out_features, d.in_features = o, i
        d.weight_mu, d.weight_sigma, d.weight_epsilon = ptr(t["mu"]), ptr(t["sg"]), ptr(t["eps"])
        d.bias_mu, d.bias_sigma, d.bias_epsilon = ptr(t["bmu"]), ptr(t["bsg"]), ptr(t["beps"])
        d.eps_in, d.eps_out, d.w_eff, d.b_eff = ptr(t["ein"]), ptr(t["eout"]), ptr(t["w"]), ptr(t["b"])
        d.stream_in, d.stream_out = (k << 40) + 6, (k << 40) + 7
    call("riqn_noisy_reset_net", len(shapes), desc, seed, 1, 1, None)
    for k, (o, i) in enumerate(shapes):
        t = keep[k]
        call("riqn_noisy_sample", i, seed, (k << 40) + 6, ptr(t["ein_ref"]), None)
        call("riqn_noisy_sample", o, seed, (k << 40) + 7, ptr(t["eout_ref"]), None)
        call("riqn_noisy_compose", o, i, ptr(t["mu"]), ptr(t["sg"]), ptr(t["eps_ref"]), ptr(t["ein_ref"]),
             ptr(t["eout_ref"]), ptr(t["bmu"]), ptr(t["bsg"]), ptr(t["beps_ref"]), ptr(t["w_ref"]), ptr(t["b_ref"]), 1)
        for n in ("ein", "eout", "eps", "beps", "w", "b"):
            assert torch.equal(t[n], t[n + "_ref"]), (k, n)
        # and it is the reference formula: W = mu + sigma * (eps_out (x) eps_in)
        assert torch.equal(t["w"], t["mu"] + t["sg"] * torch.outer(t["eout"], t["ein"]))
    # eval mode: the effective weights are the means; sample = 0 keeps the given factor vectors
    ein0 = keep[0]["ein"].clone()
    call("riqn_noisy_reset_net", len(shapes), desc, seed + 1, 0, 0, None)
    assert torch.equal(keep[0]["ein"], ein0) and torch.equal(keep[0]["w"], keep[0]["mu"])
    assert torch.equal(keep[3]["b"], keep[3]["bmu"])


def test_trunk_pair_equals_two_trunks(cuda_dev):
    """Online + target conv trunks over the same frames as ONE stacked batch (three launches, two weight sets selected by
    m-tile) == the two trunks run one after the other, bit for bit."""
    from rainbow_iqn_apex_b200 import DQN
    B = 128
    a, b_ = DQN(make_args(cuda_dev), 18).to(cuda_dev), DQN(make_args(cuda_dev), 18).to(cuda_dev)
    load_params(a, net.make_params(31))
    load_params(b_, net.make_params(32))
    x = torch.from_numpy(np.random.RandomState(9).randint(0, 256, (B, 7, 84, 84)).astype(np.uint8)).to(cuda_dev)[:, 3:7]
    pair = a.trunk_pair(b_, x)
    assert pair is not None
    fa, fb = pair
    assert torch.equal(fa, a.trunk(x)) and torch.equal(fb, b_.trunk(x))
    assert not torch.equal(fa, fb)
    ref = net.conv_trunk(net.to_torch(net.make_params(32)), x.cpu().float().div_(255)).numpy()
    assert rel_err(fb.cpu().numpy(), ref) < 3e-5
    assert a.trunk_pair(b_, x[:5]) is None                      # rows per network must fill whole 128-row tiles
