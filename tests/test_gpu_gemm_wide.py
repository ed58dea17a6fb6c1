"""GPU: the 128x256-tile path of the wgmma GEMM (csrc/gemm_tc.cu, rule in gemm.h) at the NoisyLinear head's shapes --
forward (fp16, bias + ReLU, bf16 image of h), data gradient (MN-major weight, bf16 or fp32 out) and weight gradient
(both operands MN-major, one k-split accumulated into dmu / dsigma) -- against float64 host products of the rounded
operands on a subsample of the output rows, and bitwise-repeatable from call to call."""
import numpy as np
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu

FEAT, HID2 = 3136, 1024


def _randn(dev, gen, *shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, generator=gen, device=dev) * scale).to(dtype)


def _rows(M, n, seed):
    return np.sort(np.random.RandomState(seed).choice(M, size=min(n, M), replace=False))


def _forward(dev, M, N, K, fp16, seed):
    from rainbow_iqn_apex_b200._lib import call, ptr
    gen = torch.Generator(device=dev).manual_seed(seed)
    dt = torch.float16 if fp16 else torch.bfloat16
    a, b = _randn(dev, gen, M, K, dtype=dt), _randn(dev, gen, N, K, scale=0.05, dtype=dt)
    bias = torch.randn(N, generator=gen, device=dev)
    outs = []
    for _ in range(2):
        c = torch.full((M, N), float("nan"), device=dev)
        h = torch.zeros(M, N, dtype=torch.bfloat16, device=dev) if M % 2 == 0 and N % 32 == 0 else None
        call("riqn_gemm_bf16_tc", M, N, K, ptr(a), None, ptr(b), None, ptr(c), N, 1, ptr(bias), None, None, 1, None,
             ptr(h), 3 if fp16 else 0)
        outs.append((c, h))
    torch.cuda.synchronize()
    (c, h), (c2, h2) = outs
    assert torch.equal(c, c2) and (h is None or torch.equal(h, h2)), "two calls differ"
    r = _rows(M, 256, seed)
    ref = np.maximum(a[r].double().cpu().numpy() @ b.double().cpu().numpy().T + bias.double().cpu().numpy(), 0)
    assert rel_err(c[r].cpu().numpy(), ref) < 1e-5, rel_err(c[r].cpu().numpy(), ref)
    if h is not None:
        assert torch.equal(h, c.to(torch.bfloat16))


def _dgrad(dev, M, N, K, bf16_out, seed):
    """dx (M, N) = dh (M, K) @ W (K, N): K-major A, MN-major B."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    gen = torch.Generator(device=dev).manual_seed(seed)
    a, b = _randn(dev, gen, M, K), _randn(dev, gen, K, N, scale=0.05)
    outs = []
    for _ in range(2):
        if bf16_out:
            o = torch.zeros(M, N, dtype=torch.bfloat16, device=dev)
            call("riqn_gemm_bf16_tc_mn", M, N, K, ptr(a), ptr(b), 0, None, N, 0, None, None, 1.0, 1, ptr(o), 0)
        else:
            o = torch.full((M, N), float("nan"), device=dev)
            call("riqn_gemm_bf16_tc_mn", M, N, K, ptr(a), ptr(b), 0, ptr(o), N, 0, None, None, 1.0, 1, None, 0)
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "two calls differ"
    r = _rows(M, 256, seed)
    ref = a[r].double().cpu().numpy() @ b.double().cpu().numpy()
    got = outs[0][r].double().cpu().numpy()
    assert rel_err(got, ref) < (4e-3 if bf16_out else 1e-5), rel_err(got, ref)


def _wgrad(dev, M, N, K, split_k, seed):
    """dmu (M, N) += dh^T x, dsigma += (dh^T x) * eps with dh (K, M), x (K, N) row-major: both operands MN-major."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    gen = torch.Generator(device=dev).manual_seed(seed)
    a, b = _randn(dev, gen, K, M, scale=0.1), _randn(dev, gen, K, N)
    c0 = torch.randn(M, N, generator=gen, device=dev)
    s0 = torch.randn(M, N, generator=gen, device=dev)
    eps = torch.randn(M, N, generator=gen, device=dev)
    outs = []
    for _ in range(2):
        c, s = c0.clone(), s0.clone()
        call("riqn_gemm_bf16_tc_mn", M, N, K, ptr(a), ptr(b), 1, ptr(c), N, 3, ptr(s), ptr(eps), 1.0, split_k, None, 0)
        outs.append((c, s))
    torch.cuda.synchronize()
    (c, s), (c2, s2) = outs
    assert torch.equal(c, c2) and torch.equal(s, s2), "two calls differ"
    r = _rows(M, 48, seed)
    prod = a[:, r].double().cpu().numpy().T @ b.double().cpu().numpy()
    dc = (c - c0)[r].double().cpu().numpy()
    ds = (s - s0)[r].double().cpu().numpy()
    # one fp32 accumulator chain over all K rows: its rounding grows with K (4e-5 of the largest entry at K = 32768)
    tol = 1e-5 if K <= 8192 else 1e-4
    assert rel_err(dc, prod) < tol, rel_err(dc, prod)
    assert rel_err(ds, prod * eps[r].double().cpu().numpy()) < tol


@pytest.mark.parametrize("fp16", [True, False])
def test_wide_head_forward(cuda_dev, fp16):
    _forward(cuda_dev, 16384, HID2, FEAT, fp16, seed=1)


def test_wide_head_forward_ragged(cuda_dev):
    _forward(cuda_dev, 32768, HID2, FEAT, True, seed=2)
    _forward(cuda_dev, 8301, 1000, FEAT, True, seed=3)      # odd M (lane-per-row stores), last n-tile 232 wide


@pytest.mark.parametrize("bf16_out", [True, False])
def test_wide_head_data_gradient(cuda_dev, bf16_out):
    _dgrad(cuda_dev, 32768, FEAT, HID2, bf16_out, seed=4)   # last n-tile: 64 of 256 columns


def test_wide_head_data_gradient_ragged(cuda_dev):
    _dgrad(cuda_dev, 4200, FEAT, HID2, False, seed=5)       # partial last m-tile


@pytest.mark.parametrize("M,K", [(HID2, 32768), (HID2, 4000), (2048, 8192)])
def test_wide_head_weight_gradient(cuda_dev, M, K):
    # split_k = 4 as the learner asks: one round of 128-wide CTAs cannot hold a split here, so the product runs unsplit
    # on 104 (208) wide tiles; K = 4000 ends in a partial k-block
    _wgrad(cuda_dev, M, FEAT, K, 4, seed=M + K)
