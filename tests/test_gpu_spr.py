"""SPR (Schwarzer et al., ICLR 2021): riqn_sequence_gather, riqn_spr_pack / _unpack_grad / _weight_images /
_weight_grad_add, riqn_spr_cosine_fwd_bwd and the learner fields spr, spr_steps, spr_coef (rainbow_iqn_apex_b200/spr.py).

Kernels: the sequence gather bit for bit against the numpy oracle (oracle/spr.py) over wrapped and unwrapped segments,
terminals at every offset, write heads at every distance 0..K+1, demonstration segments and K = 1, 5, 12, and against
riqn_frame_gather's states and actions; the packing, its adjoint and the weight images bit for bit; the cosine against
float64 over batch sizes 1..4096 and K = 1..12 with masked, near-zero-norm and (anti)parallel rows; one transition step
against float64 at the trunk's strip-convolution tolerances.  Learner: the SPR term against the torch oracle over three
steps for IQN, C51 and QR-DQN; an SPR learner against a plain one (sampled indices, weights, shifts, loss, priorities and
every head gradient bit for bit); the replay graph against eager steps; reproducibility, checkpoints, refusals and data
parallelism."""
import os
import socket

import numpy as np
import pytest
import torch

from helpers import Out, assert_bits, dptr, f32_bits, make_args, to_dev
from oracle import cases, network as net, replay as orep, spr as osp

D = 128


# ------------------------------------------------------------------------------------------------ sequence gather
def _store(rs, cap, nb, fill, p_term):
    """A replay.ReplayStore and the device memory holding the same transitions: ``fill[a]`` steps written into segment a
    from position 0 (more than cap wraps)."""
    from rainbow_iqn_apex_b200 import ReplayMemory
    args = make_args(torch.device("cuda"), 8, nb_actor=nb, actor_capacity=cap)
    mem = ReplayMemory(args, None)
    st = orep.ReplayStore(cap, nb)
    for a, n in enumerate(fill):
        ts = np.arange(n) % 37
        fr = rs.randint(0, 256, (n, 84, 84)).astype(np.uint8)
        ac = rs.randint(0, 18, n)
        rw = rs.randint(-1, 2, n).astype(np.float32)
        dn = rs.uniform(size=n) < p_term
        for s0 in range(0, n, cap):          # a wrap writes the ring twice
            e = min(n, s0 + cap)
            st.write(a, s0 % cap, ts[s0:e], fr[s0:e], ac[s0:e], rw[s0:e], dn[s0:e])
            mem.transitions.append_arrays(a, s0 % cap, ts[s0:e], fr[s0:e], ac[s0:e], rw[s0:e], dn[s0:e],
                                          np.ones(e - s0, np.float32))
    return st, mem


def _gather(mem, data_idx, K):
    tree = torch.as_tensor(data_idx, dtype=torch.int64).cuda() + mem.capacity - 1
    return tuple(t.cpu().numpy() for t in mem.sample_sequence(tree, K))


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 5, 12])
@pytest.mark.parametrize("wrapped", [False, True])
def test_sequence_gather_vs_oracle(cuda_dev, K, wrapped):
    rs = np.random.RandomState(K + 10 * wrapped)
    cap, nb = 64, 3
    fill = [cap + 23, cap + 5, 2 * cap + 9] if wrapped else [40, 50, 30]
    st, mem = _store(rs, cap, nb, fill, 0.08)
    heads = mem.transitions.index_actor_host.copy()
    idx = []
    for a in range(nb):
        h = int(heads[a])
        idx += [a * cap + (h - dd) % cap for dd in range(0, K + 2)]          # the write head at every distance 0..K+1
        idx += list(a * cap + rs.randint(0, fill[a] if not wrapped else cap, 12))
    idx = np.array(idx, np.int64)
    w, ac, va = _gather(mem, idx, K)
    ow, oa, ov = osp.sequence(st, idx, heads, 4, K)
    assert np.array_equal(w, ow) and np.array_equal(ac, oa) and np.array_equal(va, ov)
    assert va.any() and not va.all()
    # window[:, :4] and actions[:, 0] are riqn_frame_gather's states and actions
    s, a, _, _, _ = mem.assemble(torch.from_numpy(idx).cuda())
    assert np.array_equal(w[:, :4], s.cpu().numpy()) and np.array_equal(ac[:, 0], a.cpu().numpy())


@pytest.mark.gpu
def test_sequence_gather_terminals_at_every_offset(cuda_dev):
    """A terminal at each offset j of the window from the sampled index: steps past it are blank and invalid."""
    from rainbow_iqn_apex_b200 import ReplayMemory
    K, cap = 5, 64
    args = make_args(torch.device("cuda"), 8, nb_actor=2, actor_capacity=cap)
    args.demo_segments = 1                                         # the last segment holds demonstrations
    mem = ReplayMemory(args, None)
    st = orep.ReplayStore(cap, 2)
    rs = np.random.RandomState(5)
    for a in range(2):
        n = cap - 3
        ts, fr = np.arange(1, n + 1), rs.randint(0, 256, (n, 84, 84)).astype(np.uint8)
        ac, rw = rs.randint(0, 18, n), np.zeros(n, np.float32)
        dn = np.zeros(n, bool)
        dn[10 + np.arange(0, 7 * 8, 8)] = True                         # terminals 10, 18, 26, ...
        st.write(a, 0, ts, fr, ac, rw, dn)
        mem.transitions.append_arrays(a, 0, ts, fr, ac, rw, dn, np.ones(n, np.float32))
    idx = np.array([a * cap + 10 - j for a in range(2) for j in range(-1, K + 1)], np.int64)
    w, ac_, va = _gather(mem, idx, K)
    ow, oa, ov = osp.sequence(st, idx, mem.transitions.index_actor_host, 4, K)
    assert np.array_equal(w, ow) and np.array_equal(ac_, oa) and np.array_equal(va, ov)
    for r, j in enumerate(list(range(-1, K + 1)) * 2):           # sample at 10 - j: the terminal is j steps ahead
        want = [int(k <= j or j < 0) for k in range(1, K + 1)]            # j = -1: the terminal lies past the window
        assert list(va[r]) == want, (r, j, va[r])
    assert mem.demo_mask(torch.from_numpy(idx).cuda() + mem.capacity - 1).any()


@pytest.mark.gpu
def test_sequence_gather_rejected_calls_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError, call
    rs = np.random.RandomState(1)
    _, mem = _store(rs, 64, 1, [40], 0.0)
    tr = mem.transitions
    idx = torch.arange(4, dtype=torch.int64, device=cuda_dev) + 10
    win = Out(4 * 17 * 84 * 84 // 4, cuda_dev)
    acts, val = Out(4 * 13 * 2, cuda_dev), Out(4 * 13 // 4 + 1, cuda_dev)
    common = (ptr_ := dptr(idx), dptr(tr.index_actor), dptr(tr.frames), dptr(tr.timestep), dptr(tr.action),
              dptr(tr.nonterminal), win.p, acts.p, val.p)
    for bad in ((4, 64, 4, 13), (4, 64, 4, 0), (0, 64, 4, 5), (4, 0, 4, 5), (4, 64, 0, 5)):
        with pytest.raises(RiqnError):
            call("riqn_sequence_gather", *bad, *common)
    with pytest.raises(RiqnError):
        call("riqn_sequence_gather", 4, 64, 4, 5, ptr_, None, *common[2:])
    torch.cuda.synchronize()
    for o in (win, acts, val):
        assert bool(torch.isnan(o.t[:o.n]).all()) and o.canaries_ok()


# ------------------------------------------------------------------------------------------------ pack / unpack
def _pack_np(z, a, C, A):
    B = z.shape[0]
    out = np.zeros((B, 9, 9, C), np.float32)
    out[:, 1:8, 1:8, :64] = z.transpose(0, 2, 3, 1)
    if a is not None:
        for b in range(B):
            if 0 <= a[b] < A:
                out[b, 1:8, 1:8, 64 + a[b]] = 1.0
    return out.reshape(B * 81, C)


def _bf16_split(x):
    x = torch.from_numpy(np.ascontiguousarray(x))
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize("C,A", [(64, 0), (128, 1), (128, 18), (128, 64)])
def test_pack_and_unpack_grad_bit_for_bit(cuda_dev, C, A):
    from rainbow_iqn_apex_b200._lib import call
    rs = np.random.RandomState(C + A)
    B, K = 5, 3
    z = rs.standard_normal((B, 64, 7, 7)).astype(np.float32)
    acts = rs.randint(-1, A + 2, (B, K)).astype(np.int64) if A else None        # out-of-range actions set no plane
    hi = torch.empty(B * 81, C, dtype=torch.bfloat16, device=cuda_dev)
    lo = torch.empty_like(hi)
    ad = to_dev(acts, cuda_dev, torch.int64) if A else None
    zd = to_dev(z, cuda_dev)                   # bound to names: the buffers must outlive the launch
    call("riqn_spr_pack", B, C, dptr(zd), dptr(ad[:, 1]) if A else None, K if A else 1, A, dptr(hi), dptr(lo))
    want = _pack_np(z, acts[:, 1] if A else None, C, A)
    whi, wlo = _bf16_split(want)
    assert torch.equal(hi.cpu().view(torch.int16), whi.view(torch.int16))
    assert torch.equal(lo.cpu().view(torch.int16), wlo.view(torch.int16))
    din = rs.standard_normal((B, C, 9, 9)).astype(np.float32)
    acc = rs.standard_normal((B, 64, 7, 7)).astype(np.float32)
    for with_acc in (False, True):
        out = torch.empty(B, 64, 7, 7, device=cuda_dev)
        a_d, din_d = to_dev(acc, cuda_dev), to_dev(din, cuda_dev)
        call("riqn_spr_unpack_grad", B, C, dptr(din_d), dptr(a_d) if with_acc else None, dptr(out))
        crop = din[:, :64, 1:8, 1:8]
        assert_bits("unpack", f32_bits(out.cpu().numpy()), f32_bits(acc + crop if with_acc else crop))


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cpad", [(64, 64), (82, 128), (65, 128), (128, 128)])
def test_weight_images_and_grad_add_bit_for_bit(cuda_dev, cin, cpad):
    from rainbow_iqn_apex_b200._lib import call
    from rainbow_iqn_apex_b200.model import _strip_perm
    rs = np.random.RandomState(cin)
    w = rs.standard_normal((64, cin, 3, 3)).astype(np.float32)
    wp = np.zeros((64, cpad, 3, 3), np.float32)
    wp[:, :cin] = w
    hi, lo, hio = (torch.empty(64, 9 * cpad, dtype=torch.bfloat16, device=cuda_dev) for _ in range(3))
    wd = to_dev(w, cuda_dev)
    call("riqn_spr_weight_images", 64, cin, cpad, dptr(wd), dptr(hi), dptr(lo), dptr(hio))
    perm = _strip_perm(cpad, 3, 1, False).numpy()
    shi, slo = _bf16_split(wp.reshape(64, -1)[:, perm])
    ohi, _ = _bf16_split(wp.reshape(64, -1))
    for got, want in ((hi, shi), (lo, slo), (hio, ohi)):
        assert torch.equal(got.cpu().view(torch.int16), want.view(torch.int16))
    gpad = rs.standard_normal((64, cpad, 9)).astype(np.float32)
    gw = rs.standard_normal((64, cin, 9)).astype(np.float32)
    gd, gpd = to_dev(gw, cuda_dev), to_dev(gpad, cuda_dev)
    call("riqn_spr_weight_grad_add", 64, cin, cpad, dptr(gpd), dptr(gd))
    assert_bits("grad add", f32_bits(gd.cpu().numpy()), f32_bits(gw + gpad[:, :cin]))


# ------------------------------------------------------------------------------------------------ cosine
def _cosine64(p, t, v, coef):
    """float64 statement: rows[b] = sum_k v (-cos), dpred = -(coef/B) v d cos / dp with F.normalize's eps."""
    K, B, _ = p.shape
    p, t = p.astype(np.float64), t.astype(np.float64)
    lp = np.linalg.norm(p, axis=2, keepdims=True)
    npn, nt = np.maximum(lp, 1e-12), np.maximum(np.linalg.norm(t, axis=2, keepdims=True), 1e-12)
    ph, th = p / npn, t / nt
    cos = (ph * th).sum(2)
    vv = v.T.astype(np.float64)
    rows = -(vv * cos).sum(0)
    g = np.where(lp > 1e-12, (th - cos[..., None] * ph) / npn, th / npn)
    return rows, -(coef / B) * vv[..., None] * g


def _cos_inputs(rs, K, B, regime):
    p = rs.standard_normal((K, B, D)).astype(np.float32)
    t = rs.standard_normal((K, B, D)).astype(np.float32)
    v = (rs.uniform(size=(B, K)) < 0.7).astype(np.uint8)
    if regime == "masked":
        v[: B // 2] = 0
    elif regime == "tiny":
        p[:, ::3] *= np.float32(1e-14)                       # norms below the eps: the clamped branch
        t[:, 1::3] *= np.float32(1e-20)
    elif regime == "parallel":
        t[:, ::2] = p[:, ::2] * np.float32(3.0)
        t[:, 1::2] = -p[:, 1::2]
    return p, t, v


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["plain", "masked", "tiny", "parallel"])
@pytest.mark.parametrize("K,B", [(1, 1), (5, 7), (12, 33), (5, 512), (3, 4096), (12, 4096)])
def test_cosine_vs_float64(cuda_dev, K, B, regime):
    from rainbow_iqn_apex_b200._lib import call
    rs = np.random.RandomState(K * 7919 + B)
    p, t, v = _cos_inputs(rs, K, B, regime)
    coef = 2.0
    rows = Out(B, cuda_dev)
    dp = Out(K * B * D, cuda_dev)
    pd, td, vd = to_dev(p, cuda_dev), to_dev(t, cuda_dev), to_dev(v, cuda_dev, torch.uint8)
    call("riqn_spr_cosine_fwd_bwd", B, K, D, dptr(pd), dptr(td), dptr(vd), coef, rows.p, dp.p)
    torch.cuda.synchronize()
    assert rows.canaries_ok() and dp.canaries_ok()
    r64, g64 = _cosine64(p, t, v, coef)
    r, g = rows.f32()[:B], dp.f32()[:K * B * D].reshape(K, B, D)
    # |cos| <= 1 per term: the sum of K terms is off by O(K * 8u); the gradient by a few ulps of its terms' scale
    assert np.max(np.abs(r - r64)) <= K * 64 * 2.0 ** -24 + 1e-30
    scale = (coef / B) * (np.abs(t / np.maximum(np.linalg.norm(t.astype(np.float64), axis=2, keepdims=True), 1e-12))
                          + np.abs(p) / np.maximum(np.linalg.norm(p.astype(np.float64), axis=2, keepdims=True),
                                                   1e-12)) / np.maximum(
        np.linalg.norm(p.astype(np.float64), axis=2, keepdims=True), 1e-12)
    assert np.all(np.abs(g - g64) <= 64 * 2.0 ** -24 * scale + 1e-38), float(np.max(np.abs(g - g64) / (scale + 1e-300)))
    masked = v.T == 0
    assert np.all(g[masked] == 0)


@pytest.mark.gpu
def test_cosine_rejected_calls_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError, call
    big = Out(4096 * 13 * D, cuda_dev)
    src = to_dev(np.ones(13 * 4096 * D, np.float32), cuda_dev)
    s = dptr(src)
    p = big.p
    for a in ((0, 5, D), (4097, 5, D), (8, 0, D), (8, 13, D), (8, 5, 64)):
        with pytest.raises(RiqnError):
            call("riqn_spr_cosine_fwd_bwd", *a, s, s, s, 1.0, p, p)
    for a in ((8, 5, D, s, s, s, float("nan"), p, p), (8, 5, D, None, s, s, 1.0, p, p),
              (8, 5, D, s, s, None, 1.0, p, p), (8, 5, D, s, s, s, 1.0, None, p)):
        with pytest.raises(RiqnError):
            call("riqn_spr_cosine_fwd_bwd", *a)
    for name, a in (("riqn_spr_pack", (4, 96, s, None, 1, 0, p, p)), ("riqn_spr_pack", (4, 128, s, None, 1, 18, p, p)),
                    ("riqn_spr_pack", (4, 128, s, s, 1, 65, p, p)), ("riqn_spr_pack", (4, 64, s, s, 1, 18, p, p)),
                    ("riqn_spr_pack", (0, 64, s, None, 1, 0, p, p)), ("riqn_spr_unpack_grad", (4, 96, s, None, p)),
                    ("riqn_spr_unpack_grad", (4, 64, None, None, p)), ("riqn_spr_weight_images", (64, 82, 96, s, p, p, p)),
                    ("riqn_spr_weight_images", (64, 130, 128, s, p, p, p)),
                    ("riqn_spr_weight_grad_add", (64, 130, 128, s, p))):
        with pytest.raises(RiqnError):
            call(name, *a)
    torch.cuda.synchronize()
    assert bool(torch.isnan(big.t[:big.n]).all()) and big.canaries_ok()


# ------------------------------------------------------------------------------------------------ one transition step
C_BOUND = 2.0          # the trunk's strip-convolution tests' constant


def _check_layer(tag, x, w, b, out, dout, dw, db, din):
    """One 3x3 / padding 1 layer + ReLU against float64 with the trunk's strip-convolution test bounds: the forward
    (split-bf16 x3) against the fp32 operands, the backward (bf16) against float64 sums of the bf16-rounded operands.
    ``din``: the device's (B, Cpad, 9, 9) data gradient, compared on its interior and the real channels."""
    from helpers import check_bound
    from torch.nn.grad import conv2d_input, conv2d_weight
    d = lambda t: t.detach().cpu().double()
    bf = lambda t: t.detach().cpu().to(torch.bfloat16).double()
    x64, w64, b64 = d(x), d(w), d(b)
    pre = torch.nn.functional.conv2d(x64, w64, b64, padding=1)
    ref = torch.relu(pre)
    mag = torch.nn.functional.conv2d(x64.abs(), w64.abs(), b64.abs(), padding=1)
    K = w.shape[1] * 9
    check_bound(f"out {tag}", d(out).numpy(), ref.numpy(), (C_BOUND * (K + 1) * 2.0 ** -24 * mag + 2.0 ** -24 * ref.abs()).numpy())
    dy = bf(dout * (out > 0))
    xb, wb = bf(x), bf(w)
    B = x.shape[0]
    dw_ref = conv2d_weight(xb, w.shape, dy, padding=1)
    dw_mag = conv2d_weight(xb.abs(), w.shape, dy.abs(), padding=1)
    check_bound(f"dw {tag}", d(dw).numpy(), dw_ref.numpy(), (C_BOUND * (B * 81 + 2) * 2.0 ** -24 * dw_mag).numpy())
    dyf = d(dout * (out > 0))                                     # the bias gradient sums the fp32 dY
    check_bound(f"db {tag}", d(db).numpy(), dyf.sum((0, 2, 3)).numpy(),
                (C_BOUND * (B * 81 + 2) * 2.0 ** -24 * dyf.abs().sum((0, 2, 3))).numpy())
    din_ref = conv2d_input(x.shape, wb, dy, padding=1)
    din_mag = conv2d_input(x.shape, wb.abs(), dy.abs(), padding=1)
    got = d(din)[:, :x.shape[1], 1:8, 1:8]
    check_bound(f"din {tag}", got.numpy(), din_ref.numpy(), (C_BOUND * (w.shape[0] + 1) * 9 * 2.0 ** -24 * din_mag).numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [3, 32])
def test_transition_step_vs_float64(cuda_dev, B):
    """Both layers of one step of T, forward and weight, bias and data gradients, against float64, each layer on the
    device's own input."""
    from rainbow_iqn_apex_b200 import spr
    from rainbow_iqn_apex_b200._lib import call
    torch.manual_seed(B)
    A = 18
    sn = spr.SprNet(A, cuda_dev)
    rs = np.random.RandomState(B)
    z = np.maximum(rs.standard_normal((B, 64, 7, 7)), 0).astype(np.float32)
    a = rs.randint(0, A, B).astype(np.int64)
    zd, ad = to_dev(z, cuda_dev), to_dev(a, cuda_dev, torch.int64)
    out = torch.empty(B, 64, 7, 7, device=cuda_dev)
    ims = sn.images()
    saved = spr.transition_forward(sn, ims, zd, ad, out)
    h = saved[1]
    dout = to_dev(rs.standard_normal((B, 64, 7, 7)).astype(np.float32), cuda_dev)
    sn.zero_grad()
    gw1 = torch.zeros(64, 128 * 9, device=cuda_dev)
    # the data gradient of conv2 is what conv1's backward reads: capture it from riqn_spr_unpack_grad's input
    from rainbow_iqn_apex_b200 import _lib
    seen = {}
    real = _lib.call

    def spy(name, *args):
        if name == "riqn_spr_unpack_grad" and args[1] == 64:
            seen["din2"] = torch.empty(B, 64, 9, 9, device=cuda_dev)
            real("riqn_add_f32", seen["din2"].numel(), args[2], args[2], seen["din2"].data_ptr())
        return real(name, *args)
    spr.call = spy
    try:
        din1 = spr.transition_backward(sn, ims, saved, out, dout, gw1)
    finally:
        spr.call = real
    call("riqn_spr_weight_grad_add", 64, 64 + A, 128, dptr(gw1), dptr(sn.grad_view(sn.conv1.weight)))
    torch.cuda.synchronize()
    seen["din2"] *= 0.5                                            # the spy stored 2 * din2 (an exact doubling)
    dh = torch.empty(B, 64, 7, 7, device=cuda_dev)
    call("riqn_spr_unpack_grad", B, 64, dptr(seen["din2"]), None, dptr(dh))
    x1 = torch.cat([zd, torch.nn.functional.one_hot(ad, A).float()[:, :, None, None].expand(B, A, 7, 7)], 1)
    _check_layer("conv1", x1, sn.conv1.weight, sn.conv1.bias, h, dh, sn.conv1.weight.grad, sn.conv1.bias.grad, din1)
    _check_layer("conv2", h, sn.conv2.weight, sn.conv2.bias, out, dout, sn.conv2.weight.grad, sn.conv2.bias.grad,
                 seen["din2"])


# ------------------------------------------------------------------------------------------------ learner (GPU)
CONFIGS = {"iqn": {}, "cvar": dict(risk_measure="cvar", risk_eta=0.25), "cql": dict(cql=1), "dqfd": dict(dqfd=1),
           "iqn_vr": dict(value_rescaling=1), "miqn": dict(munchausen=1), "fqf": dict(fqf=1), "qr": dict(qr_dqn=1),
           "mmd": dict(qr_dqn=1, mmd=1), "c51": dict(rainbow_only=1), "hl_gauss": dict(rainbow_only=1, hl_gauss=1)}


def _args(dev, B, fields, spr=True, **more):
    a = make_args(dev, B, cases.iqn_cfg(64, 64, 32), rainbow_only=bool(fields.get("rainbow_only")), nb_actor=2,
                  actor_capacity=512)
    for k, v in dict(fields, random_shift=4, **more).items():
        setattr(a, k, v)
    if spr:
        a.spr = 1
    return a


def _setup(dev, B, fields, spr=True, seed=0, **more):
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    torch.manual_seed(seed)
    args = _args(dev, B, fields, spr, **more)
    lr = Learner(args, 18, None)
    lr.train()
    mem = ReplayMemory(args, None)
    rs = np.random.RandomState(1)
    for a, n in enumerate((512 + 100, 300)):                          # one wrapped segment, one partly filled
        for s0 in range(0, n, 512):
            e = min(n, s0 + 512)
            m = e - s0
            mem.transitions.append_arrays(a, s0 % 512, np.arange(s0, e) % 97,
                                          rs.randint(0, 256, (m, 84, 84)).astype(np.uint8), rs.randint(0, 18, m),
                                          rs.randint(-1, 2, m).astype(np.float32), rs.uniform(size=m) < 0.03,
                                          (rs.uniform(0.1, 1, m) ** 0.2).astype(np.float32))
    for obj, sd in ((lr.online_net, 11), (lr.target_net, 12), (mem.transitions, 13)):
        obj._rng_seed = sd
    return lr, mem


class _TrunkSpy:
    def __init__(self, net_):
        self.net, self.orig, self.calls = net_, net_.backward_trunk, []

        def spy(keep, dfeat):
            self.calls.append((keep, dfeat.clone()))
            return self.orig(keep, dfeat)
        net_.backward_trunk = spy


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_spr_learner_equals_plain_learner_past_the_trunk(cuda_dev, cfg):
    B = 32
    runs = {}
    for on in (False, True):
        lr, mem = _setup(cuda_dev, B, CONFIGS[cfg], spr=on, seed=21)
        spy = _TrunkSpy(lr.online_net)
        outs = []
        for _ in range(2):                  # two eager steps: the second samples the tree the first's priorities updated
            dbg = {}
            idxs, st, ac, rt, nx, nt, w = mem.sample(B)
            seq = mem.sample_sequence(idxs, lr.spr[0]) if on else None
            loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg, demo=lr._demo_mask(mem, idxs), sequence=seq)
            grad = lr.online_net._flat_grad.clone()
            mem.update_priorities(idxs, loss)      # no Adam: SPR's trunk gradient would move the next step's features
            outs.append((idxs.clone(), w.clone(), loss.clone(), dbg, grad, mem.transitions.tree.clone()))
        torch.cuda.synchronize()
        runs[on] = (lr, spy, outs)
    (pl, pspy, pouts), (sl, sspy, souts) = runs[False], runs[True]
    n = sl.online_net._offsets[id(sl.online_net.conv3.bias)] + sl.online_net.conv3.bias.numel()
    for (i0, w0, l0, d0, g0, t0), (i1, w1, l1, d1, g1, t1) in zip(pouts, souts):
        assert torch.equal(i0, i1) and torch.equal(w0, w1) and torch.equal(l0, l1) and torch.equal(t0, t1)
        for s0, s1 in zip(d0["shifts"], d1["shifts"]):
            assert torch.equal(s0, s1)
        assert torch.equal(g0[n:], g1[n:]) and not torch.equal(g0[:n], g1[:n])
    (_, dfeat_p), (keep, dfeat_rl) = pspy.calls[-1], sspy.calls[-1]
    assert torch.equal(dfeat_p, dfeat_rl)
    # the trunk gradient is a standalone trunk backward of dfeat_RL + dfeat_SPR
    dbg = souts[-1][3]
    total = torch.from_numpy(dfeat_rl.cpu().numpy() + dbg["dfeat_spr"].cpu().numpy()).to(cuda_dev)
    on = sl.online_net
    on.zero_grad()
    sspy.orig(keep, total)
    torch.cuda.synchronize()
    assert torch.equal(on._flat_grad[:n], souts[-1][4][:n])
    assert on._shift_calls == pl.online_net._shift_calls
    assert not torch.equal(dbg["spr_shifts"][:B], dbg["shifts"][0])


def _to_torch_spr(lr):
    return {k: lr.spr_net.get_parameter(k).detach().cpu().clone().requires_grad_(True) for k in osp.NAMES}


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "c51", "qr"])
def test_spr_term_vs_torch_oracle(cuda_dev, kind):
    """Three eager steps; at each, L_SPR's per-sample terms, the SPR arena's gradients and dfeat_SPR against the torch
    fp32 oracle on the step's device weights, frames and shifts (the RL part is the plain learner's, bit for bit, above)."""
    from test_gpu_augment import shift_np
    B = 32
    fields = {"iqn": {}, "c51": dict(rainbow_only=1), "qr": dict(qr_dqn=1)}[kind]
    lr, mem = _setup(cuda_dev, B, fields, seed=5)
    K, coef = lr.spr
    for step in range(3):
        idxs, st, ac, rt, nx, nt, w = mem.sample(B)
        seq = mem.sample_sequence(idxs, K)
        rs = np.random.RandomState(step)
        s_st, s_nx = (rs.randint(-4, 5, (B, 2)).astype(np.int32) for _ in range(2))
        s_t = rs.randint(-4, 5, (K * B, 2)).astype(np.int32)
        p_on = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in lr.online_net.state_dict().items()
                if k.startswith("conv")}
        sp = _to_torch_spr(lr)
        lr._inject = dict(shifts=(s_st, s_nx), spr_shifts=s_t)
        dbg = {}
        loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg, sequence=seq)
        torch.cuda.synchronize()
        lr._inject = None
        win, acts, valid = (t.cpu() for t in seq)
        x = torch.from_numpy(shift_np(st.cpu().numpy(), s_st)).float().div_(255)
        xt = np.concatenate([shift_np(win[:, k + 1:k + 5].numpy(), s_t[k * B:(k + 1) * B]) for k in range(K)])
        okeep = {}
        rows, y, t = osp.spr_loss(p_on, sp, x, acts, valid.numpy(), torch.from_numpy(xt).float().div_(255), 18, okeep)
        okeep["z0"].retain_grad()
        (coef * rows.mean()).backward()
        got = dbg["spr_loss"].cpu()
        assert float((got - rows.detach()).abs().max()) <= 2e-3 * K, (step, float((got - rows.detach()).abs().max()))
        assert _cos(dbg["spr_targets"].cpu(), t) >= 0.9999
        for k in osp.NAMES:
            c = _cos(lr.spr_net.get_parameter(k).grad.cpu(), sp[k].grad)
            assert c >= (0.99 if k.startswith("conv") else 0.999), (step, k, c)
        c = _cos(dbg["dfeat_spr"].cpu(), okeep["z0"].grad.reshape(B, -1))
        assert c >= 0.99, (step, c)
        lr._step_post(mem, idxs, loss)


@pytest.mark.gpu
def test_replay_graph_equals_eager_steps_and_runs_reproduce(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent
    from rainbow_iqn_apex_b200.dynstate import DynState
    B = 32
    (a, mem_a), (b, mem_b) = (_setup(cuda_dev, B, {}, seed=3) for _ in range(2))
    a.enable_cuda_graph(mem_a)
    b._dyn = DynState(cuda_dev, slots=len(b._optimisers()))
    la, lb = [], []
    with b._attached(mem_b):
        for _ in range(3):
            b._write_dyn(mem_b)
            b._step_post(mem_b, *b._step_pre(mem_b))
        b._dyn.epoch += 1
        for _ in range(3):
            _, l1 = a.learn_and_update(mem_a)
            b._write_dyn(mem_b)
            idx, l2 = b._step_pre(mem_b)
            b._step_post(mem_b, idx, l2)
            torch.cuda.synchronize()
            la.append(l1.clone())
            lb.append(l2.clone())
    for x, y in zip(la, lb):
        assert torch.equal(x, y) and bool(torch.isfinite(x).all())
    assert not torch.equal(la[0], la[1])
    for x, y in ((a.online_net._flat, b.online_net._flat), (a.spr_net._flat, b.spr_net._flat),
                 (a.spr_optimiser._exp_avg, b.spr_optimiser._exp_avg), (mem_a.transitions.tree, mem_b.transitions.tree)):
        assert torch.equal(x, y)
    # two seeded eager runs
    res = []
    for _ in range(2):
        lr, mem = _setup(cuda_dev, B, {}, seed=8)
        ls = [lr.learn_and_update(mem)[1].clone() for _ in range(2)]
        torch.cuda.synchronize()
        res.append((lr, mem, ls))
    (l1, m1, a1), (l2, m2, a2) = res
    assert all(torch.equal(x, y) for x, y in zip(a1, a2))
    assert torch.equal(l1.spr_net._flat, l2.spr_net._flat) and torch.equal(l1.online_net._flat, l2.online_net._flat)
    # checkpoint round trip: a restored learner resumes bit for bit
    l1.save(str(tmp_path), 0, 2, "spr.pth")
    path = os.path.join(tmp_path, "spr.pth")
    ck = torch.load(path, map_location="cpu")
    assert {"spr_state_dict", "spr_optimiser_state_dict"} <= set(ck)
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    from rainbow_iqn_apex_b200 import Learner
    back = Learner(_args(cuda_dev, B, {}, model=path), 18, None)
    back.train()
    plain = Agent(_args(cuda_dev, B, {}, spr=False, model=path), 18, None)           # an SPR checkpoint, plain agent
    assert plain.spr_net is None and torch.equal(plain.online_net._flat, back.online_net._flat)
    assert torch.equal(back.spr_net._flat, l1.spr_net._flat) and back.spr_optimiser._step == 2
    assert torch.equal(back.spr_optimiser._exp_avg_sq, l1.spr_optimiser._exp_avg_sq)
    back.target_net._flat.copy_(l1.target_net._flat)
    back.target_net._eps_flat.copy_(l1.target_net._eps_flat)
    back.online_net._eps_flat.copy_(l1.online_net._eps_flat)
    for x, y in ((back.online_net, l1.online_net), (back.target_net, l1.target_net)):
        x._rng_seed, x._tau_calls, x._shift_calls = y._rng_seed, y._tau_calls, y._shift_calls
        for (_, m), (_, n_) in zip(x.noisy_layers(), y.noisy_layers()):
            m._noise_calls = n_._noise_calls
        x.compose_weights()
    idxs, st, ac, rt, nx, nt, w = m1.sample(B)
    seq = m1.sample_sequence(idxs, 5)
    l_back = back.learn_on_batch(st, ac, rt, nx, nt, w, sequence=seq)
    l_orig = l1.learn_on_batch(st, ac, rt, nx, nt, w, sequence=seq)
    torch.cuda.synchronize()
    assert torch.equal(l_back, l_orig)
    assert torch.equal(back.spr_net._flat, l1.spr_net._flat) and torch.equal(back.online_net._flat, l1.online_net._flat)


@pytest.mark.gpu
def test_construction_and_refusals(cuda_dev):
    from rainbow_iqn_apex_b200 import Learner
    torch.manual_seed(4)
    plain = Learner(_args(cuda_dev, 32, {}, spr=False), 18, None)
    torch.manual_seed(4)
    lr = Learner(_args(cuda_dev, 32, {}), 18, None)
    assert lr.spr == (5, 2.0) and plain.spr is None and plain.spr_net is None
    assert torch.equal(lr.online_net._flat, plain.online_net._flat)
    assert lr.spr_net.conv1.weight.shape == (64, 82, 3, 3) and lr.spr_net.weight_q.shape == (128, 128)
    assert lr.spr_optimiser.param_groups[0]["lr"] == 5e-5 and lr.spr_optimiser in lr._optimisers()
    for bad in (dict(curl=1), dict(spr_steps=0), dict(spr_steps=13), dict(spr_coef=0.0), dict(spr=2)):
        a = _args(cuda_dev, 32, {})
        for k, v in bad.items():
            setattr(a, k, v)
        with pytest.raises(ValueError):
            Learner(a, 18, None)
    with pytest.raises(ValueError):
        Learner(_args(cuda_dev, 32, {}), 65, None)
    batch = tuple(torch.from_numpy(cases.make_batch(1, 32)[k]).to(cuda_dev) for k in
                  ("states", "actions", "returns", "next_states", "nonterminals", "weights"))
    with pytest.raises(ValueError, match="sequence"):
        lr.learn_on_batch(*batch)
    with pytest.raises(ValueError, match="sequence"):
        lr.enable_learn_graph(batch)
    with pytest.raises(ValueError, match="sequence"):
        lr.enable_batch_graph(None, (None,) + batch)
    with pytest.raises(ValueError, match="sequence"):
        lr.learn_on_host_batch()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_replica_runs_the_spr_step(cuda_dev):
    import torch.distributed as dist
    from rainbow_iqn_apex_b200 import parallel
    B = 32
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        out = []
        for dp in (False, True):
            lr, mem = _setup(cuda_dev, B, {}, seed=1)
            if dp:
                lr.process_group = dist.group.WORLD
                assert lr.spr_net in lr._trained_nets() and lr.spr_optimiser in lr._optimisers()
            ls = [lr.learn_and_update(mem)[1].clone() for _ in range(2)]
            torch.cuda.synchronize()
            out.append((ls, lr.online_net._flat.clone(), lr.spr_net._flat.clone()))
        for l1, l2 in zip(out[0][0], out[1][0]):
            assert torch.equal(l1, l2)
        for x, y in zip(out[0][1:], out[1][1:]):
            assert torch.equal(x, y)
        lr, _ = _setup(cuda_dev, B, {}, seed=1)
        before = lr.spr_net._flat.clone()
        real = parallel.dist.get_world_size
        parallel.dist.get_world_size = lambda group=None: 2
        try:
            assert parallel.make_data_parallel(lr) is lr
        finally:
            parallel.dist.get_world_size = real
        assert lr.optimiser.grad_scale == lr.spr_optimiser.grad_scale == 0.5
        assert torch.equal(before, lr.spr_net._flat)
    finally:
        dist.destroy_process_group()
