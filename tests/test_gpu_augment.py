"""Random-shift augmentation (DrQ; Kostrikov, Yarats & Fergus 2021): riqn_fill_shifts, riqn_random_shift and the learner
field random_shift.

The statement of the shift is numpy on clipped index arrays (shift_np), and of the draw integer arithmetic on the 24-bit
integers behind riqn_fill_uniform's floats (draw_from_m of a numpy Philox4x32-10, philox_np).  The unmarked tests pin both by identities: against np.pad(edge)
and torch's replicate pad followed by a crop, composition on the interior, and the draw's end points and frequencies.
The gpu tests check both entry points bit for bit against those statements (NaN / 0xAB prefills, canaries past every
buffer, two calls alike, rejected calls write nothing), the strip trunk's pixel block matrix of the shifted frames, and the
learner: zero shifts reproduce the plain learner bit for bit; non-zero shifts equal the plain learner on numpy-shifted
frames bit for bit, for every loss; IQN, C51 and QR-DQN against the torch-fp32 oracles on shifted frames; the captured
graphs, data parallelism, the actors, the launch counts and the validation."""
import socket

import numpy as np
import pytest
import torch

from helpers import assert_bits, dptr, f32_bits, lib_call, load_params, make_args, philox_np
from oracle import cases, losses, network as net, qr as oq

HW = 84
PAD = 256          # canary bytes past every output buffer
CANARY = 0x5C


# ------------------------------------------------------------------------------------------------ statements (numpy)
def shift_np(x, shifts):
    """out[i, c, y, x] = x[i, c, clip(y + dy_i, 0, H-1), clip(x + dx_i, 0, W-1)] for x (B, C, H, W), shifts (B, 2)."""
    B, C, H, W = x.shape
    s = np.asarray(shifts, np.int64).reshape(B, 2)
    yi = np.clip(np.arange(H)[None, :] + s[:, :1], 0, H - 1)
    xi = np.clip(np.arange(W)[None, :] + s[:, 1:], 0, W - 1)
    out = np.empty_like(x)
    for i in range(B):
        out[i] = x[i][:, yi[i]][:, :, xi[i]]
    return out


def draw_from_m(m, pad):
    """The shift of the 24-bit integer m: floor(m (2p+1) / 2^24) - p, in integers."""
    return ((np.asarray(m, np.int64) * (2 * pad + 1)) >> 24) - pad


def uniform_of_m(m):
    """riqn_fill_uniform's float of the 24-bit integer m: fl32(m + 0.5) 2^-24 (m + 0.5 rounds to even from m = 2^23 on)."""
    return (np.asarray(m).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)


def _frames(seed, shape, dtype=np.uint8):
    rs = np.random.RandomState(seed)
    if dtype == np.uint8:
        return rs.randint(0, 256, shape).astype(np.uint8)
    return rs.standard_normal(shape).astype(np.float32)


def _all_shifts(p, extra=True):
    s = [(dy, dx) for dy in range(-p, p + 1) for dx in range(-p, p + 1)]
    if extra:
        s += [(83, -83), (-83, 83), (1000, -1000), (-1000, 1000), (0, 1000), (-1000, 0), (2 ** 31 - 1, -2 ** 31)]
    return np.array(s, np.int64)


# ------------------------------------------------------------------------------------------------ statements (CPU)
def test_zero_shift_is_the_identity():
    x = _frames(1, (3, 4, HW, HW))
    assert np.array_equal(shift_np(x, np.zeros((3, 2))), x)


@pytest.mark.parametrize("p", [1, 4, 8, 83, 1000])
def test_statement_is_edge_pad_and_crop(p):
    """np.pad(mode="edge") by P and a crop at (dy + P, dx + P), and torch's replicate pad of fp32 frames and the same crop,
    for every (dy, dx) in [-p, p]^2 (p = 1, 4, 8) or at the extremes +-p and 0 (p = 83, 1000)."""
    x = _frames(p, (1, 2, HW, HW))
    xf = torch.from_numpy(x.astype(np.float32))
    vals = range(-p, p + 1) if p <= 8 else (-p, -1, 0, 1, p)
    P = p
    xp = np.pad(x, ((0, 0), (0, 0), (P, P), (P, P)), mode="edge")
    tp = torch.nn.functional.pad(xf, (P, P, P, P), mode="replicate").numpy() if p < HW else None
    for dy in vals:
        for dx in vals:
            got = shift_np(x, [(dy, dx)])
            want = xp[:, :, P + dy:P + dy + HW, P + dx:P + dx + HW]
            assert np.array_equal(got, want), (dy, dx)
            if tp is not None:
                assert np.array_equal(shift_np(x.astype(np.float32), [(dy, dx)]),
                                      tp[:, :, P + dy:P + dy + HW, P + dx:P + dx + HW]), (dy, dx)


def test_two_shifts_compose_on_the_interior():
    p = 4
    x = _frames(3, (1, 2, HW, HW))
    rs = np.random.RandomState(4)
    inner = slice(2 * p, HW - 2 * p)
    for _ in range(50):
        a, b = rs.randint(-p, p + 1, 2), rs.randint(-p, p + 1, 2)
        two = shift_np(shift_np(x, [a]), [b])
        one = shift_np(x, [a + b])
        assert np.array_equal(two[:, :, inner, inner], one[:, :, inner, inner])


@pytest.mark.parametrize("p", [0, 1, 4, 8, 83])
def test_draw_statement_end_points_and_frequencies(p):
    assert draw_from_m(0, p) == -p and draw_from_m(2 ** 24 - 1, p) == p
    counts = np.bincount(draw_from_m(np.arange(2 ** 24), p) + p, minlength=2 * p + 1)
    assert counts.size == 2 * p + 1 and counts.min() > 0
    assert np.all(np.abs(counts / 2.0 ** 24 - 1.0 / (2 * p + 1)) <= 2.0 ** -24)
    # below 2^23 the float riqn_fill_uniform writes determines m (m = u 2^24 - 0.5 exactly); from 2^23 on, m + 0.5 rounds
    # to even in fp32, so the statement reads m from the Philox word itself
    m = np.arange(0, 2 ** 23)
    assert np.array_equal(uniform_of_m(m).astype(np.float64) * 2 ** 24 - 0.5, m)
    assert uniform_of_m(2 ** 23 + 1) == uniform_of_m(2 ** 23 + 2)


def test_philox_statement_known_answers():
    """Random123's known-answer vector of Philox4x32-10 at counter 0 and key 0."""
    assert list(philox_np(0, 0, 1)) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


# ------------------------------------------------------------------------------------------------ kernels (GPU)
def _u8_out(n, dev):
    t = torch.full((n + PAD,), CANARY, dtype=torch.uint8, device=dev)
    t[:n] = 0xAB
    return t


def _f32_out(n, dev):
    t = torch.full((n + PAD // 4,), -77.0, device=dev)
    t[:n] = float("nan")
    return t


def _canaries_ok(t, n):
    return bool((t[n:] == (CANARY if t.dtype == torch.uint8 else -77.0)).all())


@pytest.mark.gpu
@pytest.mark.parametrize("with_dyn", [False, True])
def test_fill_shifts_vs_statement(cuda_dev, with_dyn):
    """At n = 2^20 + 3: the numpy Philox statement reproduces riqn_fill_uniform(2n) at the same seed / stream bit for bit,
    and riqn_fill_shifts equals the draw statement on its words bit for bit (and on m = u 2^24 - 0.5 of the floats
    themselves wherever u < 1/2, where u determines m); the 81 outcomes of p = 4 within a chi-square bound; two calls
    alike."""
    from scipy.stats import chi2
    from rainbow_iqn_apex_b200.dynstate import DynState
    n, seed, stream = (1 << 20) + 3, 0x1234_5678_9ABC, 77
    dyn = None
    if with_dyn:
        dyn = DynState(cuda_dev)
        for _ in range(3):
            dyn.write(0.0, 1.0, 1.0, 0.0)                   # rng_offset = 64 * 2
    got = {}
    for p in (0, 1, 4, 83):
        u = _f32_out(2 * n, cuda_dev)
        lib_call("riqn_fill_uniform", 2 * n, seed, stream, dptr(u), dyn.ptr() if dyn else None)
        outs = []
        for _ in range(2):
            o = torch.full((2 * n + PAD,), -0x54545455, dtype=torch.int32, device=cuda_dev)   # 0xABABABAB
            lib_call("riqn_fill_shifts", n, p, seed, stream, dptr(o), dyn.ptr() if dyn else None)
            torch.cuda.synchronize()
            assert bool((o[2 * n:] == -0x54545455).all())
            outs.append(o[:2 * n].cpu().numpy())
        assert np.array_equal(outs[0], outs[1])
        uh = u[:2 * n].cpu().numpy()
        m = philox_np(seed, stream + (128 if dyn else 0), (2 * n + 3) // 4)[:2 * n] >> 8
        assert_bits("fill_uniform vs Philox statement", f32_bits(uh), f32_bits(uniform_of_m(m)))
        assert np.array_equal(outs[0].reshape(n, 2), draw_from_m(m, p).reshape(n, 2)), p
        low = uh < 0.5
        assert np.array_equal(outs[0][low], draw_from_m(uh[low].astype(np.float64) * 2 ** 24 - 0.5, p))
        got[p] = outs[0]
        if p == 4:
            s = outs[0].reshape(n, 2) + 4
            counts = np.bincount(s[:, 0] * 9 + s[:, 1], minlength=81)
            stat = float(((counts - n / 81) ** 2 / (n / 81)).sum())
            print(f"p=4: chi2 {stat:.1f} over 80 dof")
            assert counts.size == 81 and stat < chi2.ppf(1 - 1e-6, 80)
    if with_dyn:      # the dyn offset moves the stream: the by-value call draws other shifts
        o2 = torch.empty(2 * n, dtype=torch.int32, device=cuda_dev)
        lib_call("riqn_fill_shifts", n, 4, seed, stream, dptr(o2), None)
        assert not np.array_equal(o2.cpu().numpy(), got[4])


def _shift_call(x0, x1, shifts, dev):
    """riqn_random_shift of device views x0, x1 (x1 may be None) into a prefilled, canary-guarded buffer."""
    u8 = x0.dtype == torch.uint8
    B, C, H, W = x0.shape
    nimg = B if x1 is None else 2 * B
    n = nimg * C * H * W
    out = _u8_out(n, dev) if u8 else _f32_out(n, dev)
    sh = torch.from_numpy(np.ascontiguousarray(shifts, np.int32)).to(dev)
    lib_call("riqn_random_shift", B, C, H, W, dptr(x0), x0.stride(0), dptr(x1), x1.stride(0) if x1 is not None else 0,
             1 if u8 else 0, dptr(sh), dptr(out))
    torch.cuda.synchronize()
    assert _canaries_ok(out, n)
    return out[:n].view(nimg, C, H, W)


def _bits(t):
    a = t.cpu().numpy()
    return a if a.dtype == np.uint8 else a.view(np.uint32)


def _shifts_for(nimg, p, seed):
    pool = _all_shifts(p)
    rs = np.random.RandomState(seed)
    if nimg >= len(pool):
        return np.concatenate([pool, rs.randint(-p, p + 1, (nimg - len(pool), 2))])[rs.permutation(nimg)]
    return pool[rs.choice(len(pool), nimg, replace=False)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["u8", "f32"])
@pytest.mark.parametrize("B", [1, 2, 7, 32, 512, 1024])
def test_random_shift_vs_statement(cuda_dev, B, dtype):
    """Contiguous batches, both halves; then the replay window's views (s at offset 0, s' at offset n frames) for
    n = 1, 3, 5; in1 = NULL; distinct batch strides for in0 and in1.  Shifts cover [-4, 4]^2 and the extremes."""
    npdt = np.uint8 if dtype == "u8" else np.float32
    tdt = torch.uint8 if dtype == "u8" else torch.float32
    for n_step in (1, 3, 5):
        win_np = _frames(B * 10 + n_step, (B, 4 + n_step, HW, HW), npdt)
        win = torch.from_numpy(win_np).to(cuda_dev)
        s, s2 = win[:, :4], win[:, n_step:n_step + 4]
        sh = _shifts_for(2 * B, 4, B + n_step)
        got = _shift_call(s2, s, sh, cuda_dev)
        want = shift_np(np.concatenate([win_np[:, n_step:n_step + 4], win_np[:, :4]]), sh)
        assert_bits(f"window n={n_step}", _bits(got).ravel(), (want if dtype == "u8" else want.view(np.uint32)).ravel())
        assert_bits("second call", _bits(_shift_call(s2, s, sh, cuda_dev)).ravel(), _bits(got).ravel())
        if n_step == 3:
            one = _shift_call(s2, None, sh[:B], cuda_dev)                                   # in1 = NULL
            assert_bits("in1 NULL", _bits(one).ravel(), _bits(got[:B]).ravel())
            other = torch.from_numpy(_frames(B + 99, (B, 4, HW, HW), npdt)).to(cuda_dev, tdt)   # stride C*H*W
            mixed = _shift_call(s2, other, sh, cuda_dev)
            want2 = shift_np(np.concatenate([win_np[:, 3:7], other.cpu().numpy()]), sh)
            assert_bits("distinct strides", _bits(mixed).ravel(),
                        (want2 if dtype == "u8" else want2.view(np.uint32)).ravel())


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,W", [(1, 4, 4), (3, 8, 6), (2, 16, 3), (1, 1, 16), (5, 32, 32)])
def test_random_shift_small_planes(cuda_dev, C, H, W):
    """Planes whose rows are not multiples of 4 bytes: words that run into the next row and clamped columns."""
    B = 5
    x_np = _frames(C * H * W, (B, C, H, W))
    x = torch.from_numpy(x_np).to(cuda_dev)
    sh = np.array([(0, 0), (1, -1), (-H - 3, W + 2), (2, 3), (-1, -W)])
    assert_bits("u8", _shift_call(x, None, sh, cuda_dev).cpu().numpy().ravel(), shift_np(x_np, sh).ravel())
    xf_np = _frames(7, (B, C, H, W), np.float32)
    got = _shift_call(torch.from_numpy(xf_np).to(cuda_dev), None, sh, cuda_dev)
    assert_bits("f32", _bits(got).ravel(), shift_np(xf_np, sh).view(np.uint32).ravel())


@pytest.mark.gpu
def test_random_shift_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    B, chw = 4, 4 * HW * HW
    x = torch.zeros(B + 1, 4, HW, HW, dtype=torch.uint8, device=cuda_dev)
    sh = torch.zeros(2 * B, 2, dtype=torch.int32, device=cuda_dev)
    out = _u8_out(2 * B * chw, cuda_dev)
    p0, ps, po = dptr(x), dptr(sh), dptr(out)
    bad = [(0, 4, HW, HW, p0, chw, p0, chw, 1, ps, po), (B, 0, HW, HW, p0, chw, p0, chw, 1, ps, po),
           (B, 4, 0, HW, p0, chw, p0, chw, 1, ps, po), (B, 4, HW, -1, p0, chw, p0, chw, 1, ps, po),
           (B, 4, HW, HW, None, chw, p0, chw, 1, ps, po), (B, 4, HW, HW, p0, chw, p0, chw, 1, None, po),
           (B, 4, HW, HW, p0, chw, p0, chw, 1, ps, None), (B, 4, HW, HW, p0, chw - 16, p0, chw, 1, ps, po),
           (B, 4, HW, HW, p0, chw, p0, chw - 16, 1, ps, po), (B, 4, HW, HW, p0 + 1, chw, p0, chw, 1, ps, po),
           (B, 4, HW, HW, p0, chw, p0 + 8, chw, 1, ps, po), (B, 4, HW, HW, p0, chw, p0, chw, 1, ps, po + 4),
           (B, 4, HW, HW, p0, chw + 1, p0, chw, 1, ps, po), (B, 4, HW, HW, p0, chw, p0, chw + 4, 1, ps, po),
           (B, 4, 3, 3, p0, chw, p0, chw, 1, ps, po), (B, 4, HW, HW, p0, chw, p0, chw, 2, ps, po),
           (B, 1, 256, 256, p0, chw, None, 0, 0, ps, po)]
    for args in bad:
        with pytest.raises(RiqnError):
            lib_call("riqn_random_shift", *args)
    o = torch.full((64,), -0x54545455, dtype=torch.int32, device=cuda_dev)
    for n, p in ((-1, 4), (4, -1), (4, 1 << 30)):
        with pytest.raises(RiqnError):
            lib_call("riqn_fill_shifts", n, p, 1, 2, dptr(o), None)
    torch.cuda.synchronize()
    assert bool((out[:2 * B * chw] == 0xAB).all()) and _canaries_ok(out, 2 * B * chw)
    assert bool((o == -0x54545455).all())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_strip_pixel_blocks_of_shifted_frames(cuda_dev, B):
    """riqn_s2d_u8 (conv1's pixel block matrix) of each half of the kernel's output equals that of the numpy-shifted
    frames, bit for bit: the halves satisfy the strip trunk's layout."""
    from rainbow_iqn_apex_b200 import augment
    from rainbow_iqn_apex_b200.model import _geom, _strip_block
    win_np = _frames(B, (B, 7, HW, HW))
    win = torch.from_numpy(win_np).to(cuda_dev)
    sh_np = _shifts_for(2 * B, 4, 5)
    nx, st = augment.random_shift(win[:, 3:7], win[:, :4], torch.from_numpy(sh_np.astype(np.int32)).to(cuda_dev))
    assert nx.is_contiguous() and st.is_contiguous() and st.data_ptr() % 16 == 0
    ref = shift_np(np.concatenate([win_np[:, 3:7], win_np[:, :4]]), sh_np)
    for half, r in ((nx, ref[:B]), (st, ref[B:])):
        blocks = []
        for x in (half, torch.from_numpy(np.ascontiguousarray(r)).to(cuda_dev)):
            g = _geom(B, 4, HW, 32, 8, 4, 1, x.stride(0))
            G, width = _strip_block(g)
            a = torch.full((B * G * G, width), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
            lib_call("riqn_s2d_u8", g, dptr(x), dptr(a))
            blocks.append(a)
        torch.cuda.synchronize()
        assert torch.equal(blocks[0].view(torch.int16), blocks[1].view(torch.int16))


# ------------------------------------------------------------------------------------------------ learner (GPU)
CONFIGS = {"iqn": {}, "cvar": dict(risk_measure="cvar", risk_eta=0.25), "miqn": dict(munchausen=1), "fqf": dict(fqf=1),
           "c51": dict(rainbow_only=1), "qr": dict(qr_dqn=1), "iqn_vr": dict(value_rescaling=1),
           "c51_vr": dict(rainbow_only=1, value_rescaling=1)}


def _args(dev, B, fields, shift=None):
    a = make_args(dev, B, cases.iqn_cfg(64, 64, 32), rainbow_only=bool(fields.get("rainbow_only")))
    for k, v in fields.items():
        setattr(a, k, v)
    if shift is not None:
        a.random_shift = shift
    return a


def _learner(dev, B, fields, shift=None, seed=0):
    from rainbow_iqn_apex_b200 import Learner
    torch.manual_seed(seed)
    lr = Learner(_args(dev, B, fields, shift), 18, None)
    lr.train()
    return lr


def _window_batch(dev, B, seed):
    """A replay-window-like batch: s and s' are views of one (B, 7, 84, 84) uint8 tensor (n = 3)."""
    b = cases.make_batch(seed, B)
    win_np = _frames(seed, (B, 7, HW, HW))
    win = torch.from_numpy(win_np).to(dev)
    rest = tuple(torch.from_numpy(b[k]).to(dev) for k in ("actions", "returns", "nonterminals", "weights"))
    return win_np, win, b, rest


def _step(lr, st, nx, rest, debug=None):
    ac, rt, nt, w = rest
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=debug)
    torch.cuda.synchronize()
    g = [lr.online_net._flat_grad.clone()]
    if lr.fraction_net is not None:
        g.append(lr.fraction_net._flat_grad.clone())
    return loss.detach().clone(), g


def _assert_same(a, b, what):
    (la, ga), (lb, gb) = a, b
    assert bool(torch.isfinite(la).all())
    assert torch.equal(la, lb), what
    for x, y in zip(ga, gb):
        assert torch.equal(x, y), what


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_zero_shifts_reproduce_the_plain_learner(cuda_dev, cfg, B):
    """Injected zero shifts into a learner with random_shift = 4: loss (the priorities it hands the update) and every
    gradient equal a learner without the field bit for bit, drawing noises and fractions natively from the same seeds."""
    win_np, win, b, rest = _window_batch(cuda_dev, B, 300 + B)
    plain = _learner(cuda_dev, B, CONFIGS[cfg], seed=11)
    aug = _learner(cuda_dev, B, CONFIGS[cfg], shift=4, seed=11)
    assert plain.random_shift is None and aug.random_shift == 4
    z = np.zeros((B, 2), np.int32)
    aug._inject = dict(shifts=(z, z))
    ref = _step(plain, win[:, :4], win[:, 3:7], rest)
    dbg = {}
    got = _step(aug, win[:, :4], win[:, 3:7], rest, debug=dbg)
    _assert_same(got, ref, cfg)
    assert torch.equal(dbg["shifted_states"].cpu(), win[:, :4].cpu())
    assert torch.equal(dbg["shifted_next_states"].cpu(), win[:, 3:7].cpu())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_shifted_step_equals_the_plain_step_on_shifted_frames(cuda_dev, cfg, B):
    """Asymmetric non-zero shifts, injected, and then drawn: the step equals a plain learner's on the numpy-shifted frames
    (s_t by the states' shifts, s_{t+n} by the next states'), bit for bit."""
    win_np, win, b, rest = _window_batch(cuda_dev, B, 400 + B)
    rs = np.random.RandomState(B)
    s_st = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_nx = rs.randint(-4, 5, (B, 2)).astype(np.int32)
    s_st[0], s_nx[0] = (3, -2), (-4, 1)                               # asymmetric: the two sets differ everywhere here
    for drawn in (False, True):
        aug = _learner(cuda_dev, B, CONFIGS[cfg], shift=4, seed=12)
        if not drawn:
            aug._inject = dict(shifts=(s_st, s_nx))
        dbg = {}
        got = _step(aug, win[:, :4], win[:, 3:7], rest, debug=dbg)
        sh_st, sh_nx = (t.cpu().numpy() for t in dbg["shifts"])
        if not drawn:
            assert np.array_equal(sh_st, s_st) and np.array_equal(sh_nx, s_nx)
        else:
            assert np.abs(np.concatenate([sh_st, sh_nx])).max() <= 4 and not np.array_equal(sh_st, sh_nx)
        st = torch.from_numpy(shift_np(win_np[:, :4], sh_st)).to(cuda_dev)
        nx = torch.from_numpy(shift_np(win_np[:, 3:7], sh_nx)).to(cuda_dev)
        assert torch.equal(dbg["shifted_states"], st) and torch.equal(dbg["shifted_next_states"], nx)
        plain = _learner(cuda_dev, B, CONFIGS[cfg], seed=12)
        _assert_same(got, _step(plain, st, nx, rest), (cfg, drawn))


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,B", [("iqn", 32), ("iqn", 512), ("c51", 32), ("c51", 512), ("qr", 32)])
def test_shifted_step_vs_torch_oracle(cuda_dev, kind, B):
    """Injected shifts, noises (and IQN fractions) against the torch-fp32 oracle step on numpy-shifted frames: loss within
    1e-3 relative off near-ties of a*, every gradient at cosine >= 0.999 (0.98 upstream of a ReLU kink or a tie)."""
    seed = 9800 + B
    cfg = cases.iqn_cfg(64, 64, 32)
    rainbow = kind == "c51"
    params = (oq.make_params(seed, 18, 64) if kind == "qr" else net.make_params(seed, rainbow_only=rainbow))
    fields = dict(qr_dqn=1) if kind == "qr" else (dict(rainbow_only=1) if rainbow else {})
    lr = _learner(cuda_dev, B, fields, shift=4, seed=seed)
    load_params(lr.online_net, params)
    lr.update_target_net()
    b = cases.make_batch(seed + 1, B)
    rs = np.random.RandomState(seed)
    s_st, s_nx = rs.randint(-4, 5, (B, 2)).astype(np.int32), rs.randint(-4, 5, (B, 2)).astype(np.int32)
    if kind == "qr":
        noises = oq.make_noises(seed + 3, 18, 64)
        lr._inject = dict(noises=noises, shifts=(s_st, s_nx))
    elif rainbow:
        noises = cases.make_noises(seed + 3, rainbow_only=True)
        lr._inject = dict(noises=noises, taus=None, shifts=(s_st, s_nx))
    else:
        noises = cases.make_noises(seed + 3)
        taus = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg))
        lr._inject = dict(noises=noises, taus=taus, shifts=(s_st, s_nx))
    dev_b = {k: torch.from_numpy(v).to(cuda_dev) for k, v in b.items()}
    dbg = {}
    loss = lr.compute_gradients(dev_b["states"], dev_b["actions"], dev_b["returns"], dev_b["next_states"],
                                dev_b["nonterminals"], dev_b["weights"], debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    bs = dict(b, states=shift_np(b["states"], s_st), next_states=shift_np(b["next_states"], s_nx))
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    w = torch.from_numpy(b["weights"])
    if kind == "qr":
        o_loss, o_grads = oq.learn_step(p_on, p_tg, cases.batch_to_torch(bs), w, noises, cfg, keep=keep)
        qv = keep["qv_next"].numpy()
    else:
        adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
        ocfg = dict(atoms=51, v_min=-10.0, v_max=10.0, discount=0.99, n_step=3) if rainbow else cfg
        o_loss, o_grads = losses.learn_step(p_on, p_tg, adam, cases.batch_to_torch(bs), w, noises,
                                            None if rainbow else taus, ocfg, rainbow_only=rainbow, keep=keep)
        qv = None
        if not rainbow:
            qv = keep["q_sel"].detach().reshape(32, B, -1).mean(0).numpy()
    lg, lo = loss.detach().cpu().numpy(), o_loss.detach().numpy()
    rel = np.abs(lg - lo) / np.abs(lo)
    if qv is not None:
        top2 = np.sort(qv, axis=1)[:, -2:]
        tie = (top2[:, 1] - top2[:, 0]) < 1e-4
    else:
        tie = rel > 1e-3                          # C51: a flipped a* of a near-tie changes the projected target
        assert tie.sum() <= 2, (int(tie.sum()), float(rel.max()))
    assert np.max(rel[~tie]) < 1e-3, float(np.max(rel[~tie]))
    relaxed = bool(tie.any())
    worst = 1.0
    for k, g_ref in o_grads.items():
        c = _cos(grads[k], g_ref)
        worst = min(worst, c)
        assert c > (0.98 if relaxed or k.startswith("conv") else 0.999), (k, c)
    print(f"{kind} B={B}: max loss rel err {np.max(rel[~tie]):.3g}, min cos {worst:.6f}, ties {int(tie.sum())}")


def _bench_run(dev, kind, fields, steps=3, seed=5):
    """Steps of a bench-sized learner (B = 512) eagerly ("eager") or replayed from a captured graph ("replay", "batch",
    "learn"); returns per-step (shifts, loss) and the final parameters."""
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    torch.manual_seed(seed)
    cap = 1 << 14
    a = bench.make_args(dev, cap)
    for k, v in fields.items():
        setattr(a, k, v)
    lr = Learner(a, bench.ACTIONS, None)
    lr.train()
    mem = ReplayMemory(a, None)
    bench.fill_replay(mem, cap, dev, 7)
    B = a.batch_size
    out = []
    if kind in ("eager", "replay"):
        if kind == "replay":
            lr.enable_cuda_graph(mem)
        for _ in range(steps):
            _, loss = lr.learn_and_update(mem)
            out.append((lr._shifts.clone() if lr.random_shift else None, loss.clone()))
    elif kind == "batch":
        lr.enable_cuda_graph(mem)
        lr.enable_batch_graph(mem, tuple(t.contiguous() for t in mem.sample(B)))
        for _ in range(steps):
            h = tuple(t.contiguous().cpu().pin_memory() for t in mem.sample(B))
            loss = lr.learn_on_host_batch(h)
            out.append((lr._shifts.clone() if lr.random_shift else None, loss.clone()))
    else:
        batches = []
        for s in range(steps):
            b = cases.make_batch(60 + s, B)
            batches.append(tuple(torch.from_numpy(b[k]).to(dev) for k in
                                 ("states", "actions", "returns", "next_states", "nonterminals", "weights")))
        lr.enable_learn_graph(batches[0])
        for bt in batches:
            loss = lr.learn_on_graph(bt)
            out.append((lr._shifts.clone() if lr.random_shift else None, loss.clone()))
    torch.cuda.synchronize()
    return out, lr.online_net._flat.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eager", "replay", "batch", "learn"])
@pytest.mark.parametrize("c51", [False, True])
def test_steps_draw_new_shifts_and_are_bitwise_reproducible(cuda_dev, kind, c51):
    fields = dict(random_shift=4, **(dict(rainbow_only=1) if c51 else {}))
    (o1, p1), (o2, p2) = _bench_run(cuda_dev, kind, fields), _bench_run(cuda_dev, kind, fields)
    for (s1, l1), (s2, l2) in zip(o1, o2):
        assert torch.equal(s1, s2) and torch.equal(l1, l2) and bool(torch.isfinite(l1).all())
        assert s1.shape == (1024, 2) and int(s1.abs().max()) == 4
    for (sa, _), (sb, _) in zip(o1, o1[1:]):
        assert not torch.equal(sa, sb)
    assert torch.equal(p1, p2)


@pytest.mark.gpu
def test_launch_counts(cuda_dev):
    """An eager learner step makes the plain step's launches plus two (draw, shift), or plus one with injected shifts;
    a namespace with random_shift = 0 makes exactly the plain step's launches."""
    from rainbow_iqn_apex_b200 import _lib
    B = 64
    win_np, win, b, rest = _window_batch(cuda_dev, B, 5)
    counts = {}
    for name, shift, inj in (("plain", None, False), ("zero", 0, False), ("drawn", 4, False), ("injected", 4, True)):
        lr = _learner(cuda_dev, B, {}, shift=shift, seed=1)
        if inj:
            z = np.zeros((B, 2), np.int32)
            lr._inject = dict(shifts=(z, z))
        _step(lr, win[:, :4], win[:, 3:7], rest)
        c0 = _lib.launch_count()
        _step(lr, win[:, :4], win[:, 3:7], rest)
        counts[name] = _lib.launch_count() - c0
    print("launches per step:", counts)
    assert counts["zero"] == counts["plain"]
    assert counts["drawn"] == counts["plain"] + 2 and counts["injected"] == counts["plain"] + 1


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel(cuda_dev):
    """Two half-batch replicas with injected shifts at grad_scale 1/2 sum to the one-learner gradient; two ranks' shift
    streams (parallel.make_data_parallel's rank-private offset) differ."""
    B = 64
    win_np, win, b, rest = _window_batch(cuda_dev, B, 21)
    ac, rt, nt, w = rest
    rs = np.random.RandomState(22)
    s_st, s_nx = rs.randint(-4, 5, (B, 2)).astype(np.int32), rs.randint(-4, 5, (B, 2)).astype(np.int32)
    noises = cases.make_noises(23)
    taus = tuple(torch.from_numpy(t) for t in cases.make_taus(24, B, cases.iqn_cfg(64, 64, 32)))

    def grads_of(sl, scale):
        lr = _learner(cuda_dev, sl.stop - sl.start, {}, shift=4, seed=1)
        q = cases.iqn_cfg(64, 64, 32)
        t = tuple(x.reshape(n, B)[:, sl].reshape(-1, 1) for x, n in zip(taus, (q["n_quantile"], q["n_tau_prime"],
                                                                                q["n_tau"])))
        lr._inject = dict(noises=noises, taus=t, shifts=(s_st[sl], s_nx[sl]))
        lr.compute_gradients(win[sl, :4], ac[sl], rt[sl], win[sl, 3:7], nt[sl], w[sl] * scale)
        torch.cuda.synchronize()
        return lr.online_net._flat_grad.clone()

    full = grads_of(slice(0, B), 1.0)
    halves = grads_of(slice(0, B // 2), 0.5) + grads_of(slice(B // 2, B), 0.5)
    err = float((halves - full).abs().max() / full.abs().max())
    print(f"data parallel: max |sum of half-batch grads - full| / max |full| = {err:.3g}")
    assert err < 2e-3 and _cos(halves, full) > 0.99999
    from rainbow_iqn_apex_b200 import augment
    draws = []
    for rank in (0, 1):
        lr = _learner(cuda_dev, B, {}, shift=4, seed=1)
        lr.online_net._tau_stream_offset = rank << 40                # what parallel.make_data_parallel sets
        draws.append(augment.draw_shifts(lr.online_net, 2 * B, 4).cpu())
    assert not torch.equal(draws[0], draws[1])


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["iqn", "fqf", "c51", "qr"])
def test_actors_never_shift(cuda_dev, cfg):
    """act, act_batch, act_batch_values (not C51's) and compute_priorities of an agent with random_shift = 4 equal those of one
    without, bit for bit (same seeds, native draws)."""
    from rainbow_iqn_apex_b200 import Actor
    rs = np.random.RandomState(3)
    states = rs.randint(0, 256, (8, 4, HW, HW)).astype(np.uint8)
    L = 14
    tab_state = [rs.randint(0, 256, (HW, HW)).astype(np.uint8) for _ in range(L + 3)]
    tab_action = [int(x) for x in rs.randint(0, 18, L)]
    tab_reward = [float(x) for x in rs.randint(-1, 2, L)]
    out = []
    for shift in (None, 4):
        torch.manual_seed(31)
        actor = Actor(_args(cuda_dev, 8, CONFIGS[cfg], shift), 18, None)
        actor.train()
        su8 = torch.from_numpy(states).to(cuda_dev)
        r = [actor.act_batch(su8).cpu(), torch.tensor(actor.act(list(states[0])))]
        if cfg != "c51":                                            # the categorical actor has no act_batch_values
            r.append(actor.act_batch_values(su8).cpu())
        r.append(torch.from_numpy(actor.compute_priorities(tab_state, tab_action, tab_reward, [1.0] * L, 0.2)))
        out.append(r)
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_configuration(cuda_dev):
    from rainbow_iqn_apex_b200 import Agent, Learner
    for v in (True, 1.5, -1, 84, float("nan")):
        with pytest.raises(ValueError):
            Agent(_args(cuda_dev, 32, {}, v), 18, None)
    for fields in CONFIGS.values():                                  # combines with every other option
        assert Learner(_args(cuda_dev, 32, fields, 83), 18, None).random_shift == 83
    assert Agent(_args(cuda_dev, 32, {}, 0), 18, None).random_shift is None
    assert Agent(_args(cuda_dev, 32, {}), 18, None).random_shift is None
