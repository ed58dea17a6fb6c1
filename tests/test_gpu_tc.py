"""GPU: the wgmma/TMA GEMM (csrc/gemm_tc.cu) against float64 products computed on the host."""
import numpy as np
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu


def _bf16_round(x):
    return torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()


def _run(dev, M, N, K, split3, epi=0, split_k=1, seed=0):
    from rainbow_iqn_apex_b200._lib import call, ptr
    rs = np.random.RandomState(seed)
    A = rs.standard_normal((M, K)).astype(np.float32)
    B = (rs.standard_normal((N, K)) * 0.05).astype(np.float32)
    a, b = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
    a_hi = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
    b_hi = torch.empty(N, K, dtype=torch.bfloat16, device=dev)
    a_lo = torch.empty_like(a_hi) if split3 else None
    b_lo = torch.empty_like(b_hi) if split3 else None
    call("riqn_split_bf16", M, K, ptr(a), ptr(a_hi), ptr(a_lo), None, None, 0)
    call("riqn_split_bf16", N, K, ptr(b), ptr(b_hi), ptr(b_lo), None, None, 0)
    assert np.array_equal(a_hi.float().cpu().numpy(), _bf16_round(A))
    bias = torch.from_numpy(rs.standard_normal(N).astype(np.float32)).to(dev)
    c = torch.zeros(M, N, device=dev)
    eps = torch.from_numpy(rs.standard_normal((M, N)).astype(np.float32)).to(dev)
    c2 = torch.zeros(M, N, device=dev)
    call("riqn_gemm_bf16_tc", M, N, K, ptr(a_hi), ptr(a_lo), ptr(b_hi), ptr(b_lo), ptr(c), N, epi, ptr(bias), ptr(c2),
         ptr(eps), split_k, None, None, 0)
    torch.cuda.synchronize()
    if split3:
        ref = A.astype(np.float64) @ B.astype(np.float64).T
        tol = 2e-5
    else:
        ref = _bf16_round(A).astype(np.float64) @ _bf16_round(B).astype(np.float64).T
        tol = 1e-5      # fp32 accumulation inside the tensor core over up to 8000 products
    got = c.cpu().numpy()
    if epi == 1:
        ref = np.maximum(ref + bias.cpu().numpy().astype(np.float64), 0)
    assert rel_err(got, ref) < tol, (M, N, K, split3, epi, split_k, rel_err(got, ref))
    if epi == 3:
        assert rel_err(c2.cpu().numpy(), ref * eps.cpu().numpy().astype(np.float64)) < max(tol, 1e-5)


@pytest.mark.parametrize("split3", [False, True])
def test_tc_gemm_single_tile(cuda_dev, split3):
    _run(cuda_dev, 128, 256, 64, split3)
    _run(cuda_dev, 128, 256, 256, split3, seed=1)


@pytest.mark.parametrize("split3", [False, True])
def test_tc_gemm_multi_tile_ragged(cuda_dev, split3):
    _run(cuda_dev, 300, 700, 3136, split3, seed=2)            # partial M, N tiles; 49 k-blocks
    _run(cuda_dev, 1000, 1024, 3136, split3, epi=1, seed=3)   # head forward shape (rows x 1024 x 3136) + bias/relu


@pytest.mark.parametrize("split3", [False, True])
def test_tc_gemm_splitk_atomic(cuda_dev, split3):
    _run(cuda_dev, 1024, 3136, 4096, split3, epi=2, split_k=4, seed=4)     # wgrad shape, K = rows
    _run(cuda_dev, 256, 512, 1000 * 8, split3, epi=3, split_k=7, seed=5)   # uneven split + dsigma output


def test_tc_gemm_many_tiles_persistent(cuda_dev):
    _run(cuda_dev, 4096, 2048, 1024, False, seed=6)           # 512 tiles > 132 SMs: every CTA walks several tiles
    _run(cuda_dev, 8192, 1024, 512, True, epi=1, seed=7)


def _run_mn(dev, M, N, K, epi=0, split_k=1, alpha=1.0, seed=0, a_is_km=1):
    """C (+)= alpha * A^T B with A (K, M), B (K, N) row-major bf16 -- the MN-major operand mode; a_is_km = 0:
    C (+)= alpha * A B with A (M, K) row-major (K-major A, MN-major B: a data gradient from the untransposed weight)."""
    from rainbow_iqn_apex_b200._lib import call, ptr
    rs = np.random.RandomState(seed)
    A = _bf16_round(rs.standard_normal((K, M) if a_is_km else (M, K)).astype(np.float32))
    B = _bf16_round((rs.standard_normal((K, N)) * 0.05).astype(np.float32))
    a = torch.from_numpy(A).to(dev).to(torch.bfloat16)
    b = torch.from_numpy(B).to(dev).to(torch.bfloat16)
    c0 = rs.standard_normal((M, N)).astype(np.float32) if epi else np.zeros((M, N), np.float32)
    c = torch.from_numpy(c0).to(dev)
    eps = torch.from_numpy(rs.standard_normal((M, N)).astype(np.float32)).to(dev)
    c2 = torch.zeros(M, N, device=dev)
    call("riqn_gemm_bf16_tc_mn", M, N, K, ptr(a), ptr(b), a_is_km, ptr(c), N, epi, ptr(c2), ptr(eps), alpha, split_k, None, 0)
    torch.cuda.synchronize()
    prod = (A.astype(np.float64).T if a_is_km else A.astype(np.float64)) @ B.astype(np.float64)
    ref = prod if epi == 0 else c0 + alpha * prod
    assert rel_err(c.cpu().numpy(), ref) < 1e-5, (M, N, K, epi, split_k, rel_err(c.cpu().numpy(), ref))
    if epi == 3:
        assert rel_err(c2.cpu().numpy(), alpha * prod * eps.cpu().numpy().astype(np.float64)) < 1e-5


def test_tc_gemm_mn_major(cuda_dev):
    _run_mn(cuda_dev, 128, 256, 64)                                   # one tile, one k-block
    _run_mn(cuda_dev, 128, 256, 512, seed=1)
    _run_mn(cuda_dev, 64, 64, 200, seed=2)                            # narrow tile, ragged reduction
    _run_mn(cuda_dev, 1024, 3136, 4096, epi=3, split_k=4, seed=3)     # NoisyLinear weight gradient shape
    _run_mn(cuda_dev, 32, 576, 2000, epi=2, split_k=5, alpha=0.5, seed=4)   # conv weight gradient shape (Cout x K)
    # mixed majors: A (M, K) K-major, B (K, N) MN-major -- dX = dY W from the untransposed weight
    _run_mn(cuda_dev, 300, 3136, 1024, seed=5, a_is_km=0)
    _run_mn(cuda_dev, 128, 256, 64, seed=6, a_is_km=0)
    # the same product written as bf16 instead of fp32 (the head data gradient feeding the embedding backward)
    from rainbow_iqn_apex_b200._lib import call, ptr
    rs = np.random.RandomState(7)
    A, B = _bf16_round(rs.standard_normal((300, 1024)).astype(np.float32)), _bf16_round(rs.standard_normal((1024, 3136)).astype(np.float32) * 0.05)
    a, b = torch.from_numpy(A).to(cuda_dev).to(torch.bfloat16), torch.from_numpy(B).to(cuda_dev).to(torch.bfloat16)
    cb = torch.zeros(300, 3136, dtype=torch.bfloat16, device=cuda_dev)
    call("riqn_gemm_bf16_tc_mn", 300, 3136, 1024, ptr(a), ptr(b), 0, None, 3136, 0, None, None, 1.0, 1, ptr(cb), 0)
    torch.cuda.synchronize()
    ref = A.astype(np.float64) @ B.astype(np.float64)
    assert rel_err(cb.float().cpu().numpy(), ref) < 4e-3          # one bf16 rounding of the result


def test_tc_gemm_fp16_operands(cuda_dev):
    """fp16 x fp16 single-pass products (the head forward's arithmetic), K-major and MN-major; a product mixing fp16 and
    bf16 images is refused (wgmma takes one 16-bit format for both operands)."""
    from rainbow_iqn_apex_b200._lib import RiqnError, call, ptr
    rs = np.random.RandomState(43)
    M, N, K = 300, 1024, 3136
    a = torch.from_numpy(rs.standard_normal((M, K)).astype(np.float32)).to(cuda_dev).half()
    b = torch.from_numpy((rs.standard_normal((N, K)) * 0.05).astype(np.float32)).to(cuda_dev).half()
    bias = torch.from_numpy(rs.standard_normal(N).astype(np.float32)).to(cuda_dev)
    c = torch.zeros(M, N, device=cuda_dev)
    call("riqn_gemm_bf16_tc", M, N, K, ptr(a), None, ptr(b), None, ptr(c), N, 1, ptr(bias), None, None, 1, None, None, 3)
    ref = np.maximum(a.float().cpu().numpy().astype(np.float64) @ b.float().cpu().numpy().astype(np.float64).T
                     + bias.cpu().numpy(), 0)
    assert rel_err(c.cpu().numpy(), ref) < 1e-5
    for a_is_km in (0, 1):
        Mm, Nn, Kk = (300, 3136, 1024) if not a_is_km else (1024, 3136, 512)
        a2 = torch.from_numpy(rs.standard_normal((Kk, Mm) if a_is_km else (Mm, Kk)).astype(np.float32)).to(cuda_dev).half()
        b2 = torch.from_numpy((rs.standard_normal((Kk, Nn)) * 0.05).astype(np.float32)).to(cuda_dev).half()
        c2 = torch.zeros(Mm, Nn, device=cuda_dev)
        call("riqn_gemm_bf16_tc_mn", Mm, Nn, Kk, ptr(a2), ptr(b2), a_is_km, ptr(c2), Nn, 0, None, None, 1.0, 1, None, 3)
        af = a2.float().cpu().numpy().astype(np.float64)
        ref2 = (af.T if a_is_km else af) @ b2.float().cpu().numpy().astype(np.float64)
        assert rel_err(c2.cpu().numpy(), ref2) < 1e-5, a_is_km
    for fmt in (1, 2):
        with pytest.raises(RiqnError):
            call("riqn_gemm_bf16_tc", M, N, K, ptr(a), None, ptr(b), None, ptr(c), N, 1, ptr(bias), None, None, 1, None, None, fmt)
    # fp16(x) + bf16(x) images from one split call (the compose_weights path of the fp16 forward)
    src = torch.from_numpy(rs.standard_normal((64, 96)).astype(np.float32)).to(cuda_dev)
    h, l = torch.empty(64, 96, dtype=torch.float16, device=cuda_dev), torch.empty(64, 96, dtype=torch.bfloat16, device=cuda_dev)
    call("riqn_split_bf16", 64, 96, ptr(src), ptr(h), ptr(l), None, None, 1)
    assert torch.equal(h, src.half()) and torch.equal(l, src.bfloat16())


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
