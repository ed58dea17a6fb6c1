"""GPU: the data gradient of the strip convolution (riqn_conv_bwd_strip) at the learner's batch, computed as a transposed
strip convolution on the block grid: against float64 conv_transpose2d of the same bf16 operands, bitwise reproducible,
written once everywhere, and with no term crossing a sample boundary."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_err

pytestmark = pytest.mark.gpu

# (Cin, H, Cout, k, stride) of conv2 and conv3 (the layers with a data gradient); pad 0
LAYERS = {"conv2": (32, 20, 64, 4, 2), "conv3": (64, 9, 64, 3, 1)}


def _setup(dev, name, batch, seed):
    from rainbow_iqn_apex_b200._lib import ConvGeom
    from rainbow_iqn_apex_b200.model import _strip_perm
    cin, h, cout, k, s = LAYERS[name]
    oh = (h - k) // s + 1
    G, kc = oh + k // s - 1, s * s * cin
    g = torch.Generator().manual_seed(seed)
    K = cin * k * k
    w = torch.randn(cout, K, generator=g) / K ** 0.5
    t = dict(
        geom=ConvGeom(batch, cin, h, h, cout, k, k, s, 0, oh, oh, cin * h * h), G=G, K=K, k=k, s=s,
        dout=torch.randn(batch, cout, oh, oh, generator=g),
        out=torch.randn(batch, cout, oh, oh, generator=g),                          # ReLU mask: out > 0
        a_hi=torch.randn(batch * G * G, kc, generator=g).to(torch.bfloat16),        # block matrix of the weight gradient
        w_hi=w.to(torch.bfloat16),                                                   # (Cout, K), original k order
        perm=_strip_perm(cin, k, s, False).to(torch.int32))
    return {key: (v.to(dev) if torch.is_tensor(v) else v) for key, v in t.items()}


def _din(t, fill=0.0):
    from rainbow_iqn_apex_b200._lib import call, ptr
    gm, dev = t["geom"], t["dout"].device
    din = torch.full((gm.B, gm.Cin, gm.H, gm.W), fill, device=dev)
    dYg = torch.empty(gm.B * t["G"] ** 2, gm.Cout, dtype=torch.bfloat16, device=dev)
    dwp = torch.empty(gm.Cout, t["K"], device=dev)
    dw = torch.zeros(gm.Cout, t["K"], device=dev)
    db = torch.zeros(gm.Cout, device=dev)
    call("riqn_conv_bwd_strip", gm, ptr(t["dout"]), ptr(t["out"]), ptr(t["a_hi"]), ptr(t["w_hi"]), ptr(t["perm"]), ptr(dYg),
         ptr(dwp), ptr(dw), ptr(db), ptr(din), 1.0)
    torch.cuda.synchronize()
    return din


def _reference(t):
    """float64 conv_transpose2d of the operands the kernel multiplies: bf16(dout * (out > 0)) and the bf16 weight."""
    gm = t["geom"]
    dy = torch.where(t["out"] > 0, t["dout"], torch.zeros_like(t["dout"])).to(torch.bfloat16).double().cpu()
    w = t["w_hi"].double().cpu().reshape(gm.Cout, gm.Cin, t["k"], t["k"])
    return F.conv_transpose2d(dy, w, stride=t["s"]).numpy()


@pytest.mark.parametrize("name", ["conv2", "conv3"])
def test_strip_dgrad_learner_batch(cuda_dev, name):
    """B = 512: within fp32 accumulation of the exact float64 result, bitwise equal over two calls, and every element
    written (din pre-filled with NaN comes back finite)."""
    t = _setup(cuda_dev, name, 512, seed=1)
    d1 = _din(t)
    d2 = _din(t, fill=float("nan"))
    assert torch.isfinite(d2).all()
    assert torch.equal(d1.view(torch.int32), d2.view(torch.int32))
    err = rel_err(d1.cpu().numpy(), _reference(t))
    assert err < 1e-5, (name, err)


@pytest.mark.parametrize("name", ["conv2", "conv3"])
def test_strip_dgrad_sample_boundaries(cuda_dev, name):
    """Only the first and the last sample carry a (large) gradient: the samples between get exactly zero, so no shift
    reads a neighbouring sample's outputs, and sample 0 (whose top-left blocks take rows before the start of dYg) and
    the last sample match the reference."""
    B = 6
    t = _setup(cuda_dev, name, B, seed=2)
    t["dout"][1:B - 1] = 0.0
    t["dout"][0] *= 1e4
    t["dout"][B - 1] *= 1e4
    t["out"].abs_()                                     # every output active: the whole sample feeds its neighbours' rows
    din = _din(t, fill=float("nan")).cpu().numpy()
    assert np.all(din[1:B - 1] == 0.0)
    ref = _reference(t)
    for b in (0, B - 1):
        assert rel_err(din[b], ref[b]) < 1e-5, (name, b, rel_err(din[b], ref[b]))
