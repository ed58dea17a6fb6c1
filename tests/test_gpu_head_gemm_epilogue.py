"""GPU: the NoisyLinear head's three products on 128x256 tiles (csrc/gemm_tc.cu), through their entry points, at the
learner's row counts and at ragged shapes -- forward (bias + ReLU into fp32 h, with and without the bf16 image h_hi;
TMA-store epilogue), data gradient (bf16 dx through the TMA-store epilogue, fp32 dx through the slab epilogue) and
weight gradient (dmu / dsigma accumulated).

Method:
* exact regime: small integers with power-of-two scales make every product and partial sum exact in fp32 in any
  order, so every output element must equal the float64 product bit for bit (the bf16 image: the rounding of it);
* random regime: Gaussian operands, held to the bounds of test_gpu_gemm_wide.py on a subsample of rows;
* overwritten outputs start as NaN, every output buffer carries canaries past its end (and in the padding columns of a
  row pitch wider than N), so a row or column written past a clipped edge shows up;
* every product runs twice and the two results must agree bit for bit;
* outputs the 16-byte vector stores cannot serve (an unaligned base or row pitch) are refused before any launch.
"""
import numpy as np
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu

FEAT, HID2 = 3136, 1024
ROWS = [16384, 32768, 32256, 65536]   # K and N' passes, gradient pass, FQF boundary pass (63 x 512), Munchausen target
CANARY = 256
CAN_F32, CAN_BF16 = 1234.5, -77.0


def _call(*args):
    from rainbow_iqn_apex_b200._lib import call
    call(*args)


def _ptr(t):
    from rainbow_iqn_apex_b200._lib import ptr
    return ptr(t)


def _operand(dev, gen, shape, exact, scale, dtype):
    if exact:   # integers in [-3, 3] times a power of two: exact in fp16 and bf16
        return (torch.randint(-3, 4, shape, generator=gen, device=dev).float() * scale).to(dtype)
    return (torch.randn(*shape, generator=gen, device=dev) * scale).to(dtype)


class _Out:
    """(M, N) output with row pitch ld inside a flat buffer: the (M, N) part is prefilled (NaN unless given), the
    padding columns and CANARY elements past the end hold a canary value."""

    def __init__(self, dev, M, N, ld, dtype, init=None):
        can = CAN_F32 if dtype == torch.float32 else CAN_BF16
        self.buf = torch.full((M * ld + CANARY,), can, dtype=dtype, device=dev)
        self.M, self.N, self.ld, self.can = M, N, ld, can
        self.view[:] = float("nan") if init is None else init

    @property
    def view(self):
        return self.buf[:self.M * self.ld].view(self.M, self.ld)[:, :self.N]

    def check_canaries(self):
        pad = self.buf[:self.M * self.ld].view(self.M, self.ld)[:, self.N:]
        assert bool((self.buf[self.M * self.ld:] == self.can).all()), "write past the end of the output"
        assert bool((pad == self.can).all()), "write into the padding columns"


def _twice(run):
    a, b = run(), run()
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x.buf, y.buf), "two calls differ"
            x.check_canaries()
    return a


def _forward(dev, M, N, K, image, exact, seed, fp16=True, ldc=None):
    gen = torch.Generator(device=dev).manual_seed(seed)
    dt = torch.float16 if fp16 else torch.bfloat16
    a = _operand(dev, gen, (M, K), exact, 1.0, dt)
    b = _operand(dev, gen, (N, K), exact, 2.0 ** -4 if exact else 0.05, dt)
    bias = _operand(dev, gen, (N,), exact, 2.0 ** -4 if exact else 1.0, torch.float32)
    ldc = ldc or N

    def run():
        c = _Out(dev, M, N, ldc, torch.float32)
        h = _Out(dev, M, N, N, torch.bfloat16) if image else None
        _call("riqn_gemm_bf16_tc", M, N, K, _ptr(a), None, _ptr(b), None, _ptr(c.buf), ldc, 1, _ptr(bias), None, None, 1,
              None, _ptr(h.buf) if h else None, 3 if fp16 else 0)
        return c, h

    c, h = _twice(run)
    if exact:
        ref = torch.relu(a.double() @ b.double().T + bias.double()).float()
        assert torch.equal(c.view, ref), "forward differs from the exact product"
    else:
        r = torch.from_numpy(np.sort(np.random.RandomState(seed).choice(M, 256, replace=False))).to(dev)
        ref = torch.relu(a[r].double() @ b.double().T + bias.double())
        assert rel_err(c.view[r].cpu().numpy(), ref.cpu().numpy()) < 1e-5
    if h is not None:
        assert torch.equal(h.view, c.view.to(torch.bfloat16)), "h_hi is not the bf16 rounding of h"


def _dgrad(dev, M, N, K, bf16_out, exact, seed):
    """dx (M, N) = dh (M, K) @ W (K, N): K-major A, MN-major B."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    a = _operand(dev, gen, (M, K), exact, 1.0, torch.bfloat16)
    b = _operand(dev, gen, (K, N), exact, 2.0 ** -4 if exact else 0.05, torch.bfloat16)

    def run():
        o = _Out(dev, M, N, N, torch.bfloat16 if bf16_out else torch.float32)
        _call("riqn_gemm_bf16_tc_mn", M, N, K, _ptr(a), _ptr(b), 0, None if bf16_out else _ptr(o.buf), N, 0, None, None,
              1.0, 1, _ptr(o.buf) if bf16_out else None, 0)
        return (o,)

    (o,) = _twice(run)
    if exact:
        ref = (a.double() @ b.double()).float()
        assert torch.equal(o.view, ref.to(torch.bfloat16) if bf16_out else ref), "data gradient differs from the exact product"
    else:
        r = torch.from_numpy(np.sort(np.random.RandomState(seed).choice(M, 256, replace=False))).to(dev)
        ref = a[r].double() @ b.double()
        assert rel_err(o.view[r].double().cpu().numpy(), ref.cpu().numpy()) < (4e-3 if bf16_out else 1e-5)


def _wgrad(dev, M, N, K, exact, seed):
    """dmu (M, N) += dh^T x, dsigma += (dh^T x) * eps with dh (K, M), x (K, N) row-major: both operands MN-major."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    a = _operand(dev, gen, (K, M), exact, 1.0 if exact else 0.1, torch.bfloat16)
    b = _operand(dev, gen, (K, N), exact, 2.0 ** -4 if exact else 1.0, torch.bfloat16)
    c0 = _operand(dev, gen, (M, N), exact, 2.0 ** -4 if exact else 1.0, torch.float32)
    s0 = _operand(dev, gen, (M, N), exact, 2.0 ** -4 if exact else 1.0, torch.float32)
    if exact:    # +-1/2, +-1, +-2: the product times eps stays exact
        eps = torch.randint(-1, 2, (M, N), generator=gen, device=dev).float().exp2() * (
            torch.randint(0, 2, (M, N), generator=gen, device=dev).float() * 2 - 1)
    else:
        eps = torch.randn(M, N, generator=gen, device=dev)

    def run():
        c, s = _Out(dev, M, N, N, torch.float32, c0), _Out(dev, M, N, N, torch.float32, s0)
        _call("riqn_gemm_bf16_tc_mn", M, N, K, _ptr(a), _ptr(b), 1, _ptr(c.buf), N, 3, _ptr(s.buf), _ptr(eps), 1.0, 4,
              None, 0)
        return c, s

    c, s = _twice(run)
    if exact:
        prod = a.double().T @ b.double()
        assert torch.equal(c.view, (c0.double() + prod).float()), "dmu differs from the exact product"
        assert torch.equal(s.view, (s0.double() + prod * eps.double()).float()), "dsigma differs from the exact product"
    else:
        r = torch.from_numpy(np.sort(np.random.RandomState(seed).choice(M, 48, replace=False))).to(dev)
        prod = (a[:, r].double().T @ b.double()).cpu().numpy()
        assert rel_err((c.view - c0)[r].double().cpu().numpy(), prod) < 1e-4
        assert rel_err((s.view - s0)[r].double().cpu().numpy(), prod * eps[r].double().cpu().numpy()) < 1e-4


@pytest.mark.parametrize("image", [False, True])
@pytest.mark.parametrize("M", ROWS)
def test_head_forward_exact(cuda_dev, M, image):
    _forward(cuda_dev, M, HID2, FEAT, image, True, seed=M + image)


def test_head_forward_bf16_operands_exact(cuda_dev):
    _forward(cuda_dev, 32768, HID2, FEAT, True, True, seed=11, fp16=False)


def test_head_forward_ragged_exact(cuda_dev):
    _forward(cuda_dev, 8301, 1000, 4000, False, True, seed=12)    # odd M, last n-tile 232 wide, partial last k-block
    _forward(cuda_dev, 8302, HID2, 4000, True, True, seed=13)
    _forward(cuda_dev, 8301, 1000, 4000, False, True, seed=14, ldc=1004)   # row pitch wider than N


def test_head_forward_random(cuda_dev):
    _forward(cuda_dev, 32768, HID2, FEAT, True, False, seed=15)


@pytest.mark.parametrize("M", ROWS)
def test_head_data_gradient_exact(cuda_dev, M):
    _dgrad(cuda_dev, M, FEAT, HID2, True, True, seed=M + 1)


def test_head_data_gradient_fp32_exact(cuda_dev):
    _dgrad(cuda_dev, 32768, FEAT, HID2, False, True, seed=21)


def test_head_data_gradient_ragged_exact(cuda_dev):
    _dgrad(cuda_dev, 8301, FEAT, 4000, True, True, seed=22)     # odd M: clipped last m-tile of the bf16 TMA stores
    _dgrad(cuda_dev, 8301, 1000, 4000, False, True, seed=23)


@pytest.mark.parametrize("bf16_out", [True, False])
def test_head_data_gradient_random(cuda_dev, bf16_out):
    _dgrad(cuda_dev, 32768, FEAT, HID2, bf16_out, False, seed=24 + bf16_out)


@pytest.mark.parametrize("K", ROWS)
def test_head_weight_gradient_exact(cuda_dev, K):
    _wgrad(cuda_dev, HID2, FEAT, K, True, seed=K + 2)


def test_head_weight_gradient_ragged_exact(cuda_dev):
    _wgrad(cuda_dev, 1000, 1000, 4000, True, seed=31)


def test_head_weight_gradient_random(cuda_dev):
    _wgrad(cuda_dev, HID2, FEAT, 32768, False, seed=32)


def test_head_unaligned_outputs_are_refused(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    dev = cuda_dev
    M, N, K = 16384, HID2, FEAT
    a = torch.zeros(M, K, dtype=torch.float16, device=dev)
    b = torch.zeros(N, K, dtype=torch.float16, device=dev)
    bias = torch.zeros(N, device=dev)
    c = _Out(dev, M, N, N + 1, torch.float32)
    with pytest.raises(RiqnError):       # odd row pitch
        _call("riqn_gemm_bf16_tc", M, N, K, _ptr(a), None, _ptr(b), None, _ptr(c.buf), N + 1, 1, _ptr(bias), None, None,
              1, None, None, 3)
    buf = torch.full((M * N + 4,), float("nan"), device=dev)
    with pytest.raises(RiqnError):       # base 4 bytes past a 16-byte boundary
        _call("riqn_gemm_bf16_tc", M, N, K, _ptr(a), None, _ptr(b), None, _ptr(buf) + 4, N, 1, _ptr(bias), None, None,
              1, None, None, 3)
    o = torch.full((M * FEAT + 8,), float("nan"), dtype=torch.bfloat16, device=dev)
    dh, w = torch.zeros(M, HID2, dtype=torch.bfloat16, device=dev), torch.zeros(HID2, FEAT, dtype=torch.bfloat16, device=dev)
    with pytest.raises(RiqnError):       # bf16 data gradient 2 bytes past a 16-byte boundary
        _call("riqn_gemm_bf16_tc_mn", M, FEAT, HID2, _ptr(dh), _ptr(w), 0, None, FEAT, 0, None, None, 1.0, 1, _ptr(o) + 2, 0)
    torch.cuda.synchronize()
    assert bool(c.view.isnan().all()) and bool(buf.isnan().all()) and bool(o.isnan().all()), "a refused call wrote"
    c.check_canaries()
