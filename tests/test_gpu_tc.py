"""GPU: the strip convolution's forward and backward chain (csrc/gemm_tc.cu, csrc/conv.cu) against float64 conv2d and
autograd.  The general GEMM entry points and the operand splitters are tested in tests/test_gpu_gemm_kernels.py."""
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu


def _strip_layers():
    # (Cin, H, Cout, k, stride, pad, first) of the three Atari convolutions (model.py:65-67)
    return [(4, 84, 32, 8, 4, 1, True), (32, 20, 64, 4, 2, 0, False), (64, 9, 64, 3, 1, 0, False)]


@pytest.mark.parametrize("batch", [3, 8])
def test_strip_convolution_forward_and_backward(cuda_dev, batch):
    """riqn_s2d_u8 + riqn_conv_fwd_strip (x3 products) against float64 conv2d, layer by layer through the block matrices
    each epilogue writes for the next layer; riqn_conv_bwd_strip (bf16 products) against autograd.  batch = 3 makes
    the strip grids ragged (B*G*G not a multiple of 8 / 128)."""
    import torch.nn.functional as F
    from rainbow_iqn_apex_b200._lib import call, ptr, ConvGeom
    from rainbow_iqn_apex_b200.model import _strip_perm
    dev = cuda_dev
    g = torch.Generator().manual_seed(11 + batch)
    x = torch.randint(0, 256, (batch, 4, 84, 84), generator=g, dtype=torch.uint8)
    bf = lambda *sh: torch.zeros(*sh, dtype=torch.bfloat16, device=dev)
    xd = x.to(dev)
    ws, bs, outs_ref, geoms = [], [], [], []
    inp = x.double() / 255.0
    for (cin, h, cout, k, s, pad, first) in _strip_layers():
        w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).float()
        b = (torch.randn(cout, generator=g) * 0.1).float()
        ws.append(w); bs.append(b)
        inp = F.relu(F.conv2d(inp, w.double(), b.double(), stride=s, padding=pad))
        outs_ref.append(inp)
        oh = (h + 2 * pad - k) // s + 1
        geoms.append(ConvGeom(batch, cin, h, h, cout, k, k, s, pad, oh, oh, cin * h * h))
    grids = [gm.OH + gm.KH // gm.stride - 1 for gm in geoms]            # 21, 10, 9
    kcs = [gm.stride * gm.stride * gm.Cin for gm in geoms]              # 64, 128, 64
    a_hi = [bf(batch * G * G, kc) for G, kc in zip(grids, kcs)]
    a_lo = [None] + [bf(batch * G * G, kc) for G, kc in zip(grids[1:], kcs[1:])]
    call("riqn_s2d_u8", geoms[0], ptr(xd), ptr(a_hi[0]))
    outs, w_ops, perms = [], [], []
    for i, (gm, w, b) in enumerate(zip(geoms, ws, bs)):
        cin, h, cout, k, s, pad, first = _strip_layers()[i]
        perm = _strip_perm(cin, k, s, first)
        perms.append(perm.to(torch.int32).to(dev))
        wp = w.reshape(cout, -1)[:, perm].contiguous().to(dev)
        K = wp.shape[1]
        w_hi, w_lo = bf(cout, K), bf(cout, K)
        if i == 0:
            call("riqn_split_bf16_scaled", cout, K, ptr(wp), 255.0, ptr(w_hi), ptr(w_lo))
        else:
            call("riqn_split_bf16", cout, K, ptr(wp), ptr(w_hi), ptr(w_lo), None, None, 0)
        w_ops.append((wp, w_hi, w_lo))
        out = torch.zeros(batch, cout, gm.OH, gm.OH, device=dev)
        bd = b.to(dev)
        nxt = (ptr(a_hi[i + 1]), ptr(a_lo[i + 1]), geoms[i + 1].stride, grids[i + 1]) if i < 2 else (None, None, 0, 0)
        call("riqn_conv_fwd_strip", gm, ptr(a_hi[i]), ptr(a_lo[i]), ptr(w_hi), ptr(w_lo), ptr(bd), ptr(out), *nxt, None, None, None, 0)
        torch.cuda.synchronize()
        outs.append(out)
        assert rel_err(out.cpu().numpy(), outs_ref[i].numpy()) < 2e-5, (i, rel_err(out.cpu().numpy(), outs_ref[i].numpy()))
    # the block matrix written for layer 2 holds hi + lo == out1 in (iy, ix, c) order
    G2 = grids[1]
    blk = (a_hi[1].float() + a_lo[1].float()).view(batch, G2, G2, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(batch, 32, 20, 20)
    assert rel_err(blk.cpu().numpy(), outs[0].cpu().numpy()) < 2e-5

    # ---- backward of the last two layers (pad == 0: data gradient) and of the first (weight gradient only)
    xin = [x.double() / 255.0, outs_ref[0], outs_ref[1]]
    for i in (2, 1, 0):
        cin, h, cout, k, s, pad, first = _strip_layers()[i]
        gm = geoms[i]
        w64 = ws[i].double().requires_grad_(True)
        b64 = bs[i].double().requires_grad_(True)
        xi = xin[i].clone().requires_grad_(i > 0)
        y = F.relu(F.conv2d(xi, w64, b64, stride=s, padding=pad))
        dout = torch.randn(y.shape, generator=g).double()
        y.backward(dout)
        K = cin * k * k
        G = grids[i]
        w_hi_orig = bf(cout, K)
        call("riqn_split_bf16", cout, K, ptr(ws[i].reshape(cout, K).contiguous().to(dev)), ptr(w_hi_orig), None, None, None, 0)
        dYg = bf(batch * G * G, cout)
        dwp = torch.zeros(cout, K, device=dev)
        dw = torch.zeros(cout, K, device=dev)
        db = torch.zeros(cout, device=dev)
        din = torch.zeros(batch, cin, h, h, device=dev) if i > 0 else None
        doutd = dout.float().to(dev)
        a_in = a_hi[i]
        out_mask = y.detach().float().to(dev)          # the reference's activations: identical ReLU masks on both sides
        call("riqn_conv_bwd_strip", gm, ptr(doutd), ptr(out_mask), ptr(a_in), ptr(w_hi_orig), ptr(perms[i]), ptr(dYg), ptr(dwp),
             ptr(dw), ptr(db), ptr(din), 1.0 / 255.0 if i == 0 else 1.0)
        torch.cuda.synchronize()
        assert rel_err(db.cpu().numpy(), b64.grad.numpy()) < 1e-4, i
        assert rel_err(dw.cpu().numpy(), w64.grad.reshape(cout, K).numpy()) < 1e-2, (i, rel_err(dw.cpu().numpy(), w64.grad.reshape(cout, K).numpy()))
        if i > 0:
            assert rel_err(din.cpu().numpy(), xi.grad.numpy()) < 1e-2, i
