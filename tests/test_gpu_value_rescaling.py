"""Value-function rescaling (Pohlen et al. 2018, the transformed Bellman operator) for training on unclipped rewards:
riqn_value_rescale, riqn_iqn_loss_fwd_bwd_h, riqn_argmax_expected_h and riqn_c51_loss_fwd_bwd_h behind the optional Agent
fields value_rescaling and value_rescaling_eps.

The unmarked tests pin the float64 oracle (oracle/value_rescaling.py) by identities, check the host-side validation and
check that the existing loss kernels' instantiations compile to the SASS they had before the rescaled ones were added.
The gpu tests hold every entry point bitwise to its numpy statement (NaN prefills, canaries, repeated calls, rejected
calls that write nothing), the IQN (also under CVaR), FQF and C51 learner steps and the actors against the torch oracle,
reproducibility eagerly and from the captured step graph, and the checkpoint key."""
import hashlib
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, load_params, make_args,
                     rel_err, to_dev)
from oracle import cases, losses, munchausen as om, network as net, value_rescaling as vr

EPS = [0.0, 1e-3, 1e-2]
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def _magnitudes():
    m = np.logspace(-12, 6, 2000)
    return np.concatenate((-m[::-1], m))


@pytest.mark.parametrize("eps", EPS)
def test_h_is_odd_increasing_and_zero_at_zero(eps):
    x = _magnitudes()
    assert vr.h_np(0.0, eps) == 0.0 and vr.h_inv_np(0.0, eps) == 0.0
    assert np.array_equal(vr.h_np(-x, eps), -vr.h_np(x, eps))
    assert np.array_equal(vr.h_inv_np(-x, eps), -vr.h_inv_np(x, eps))
    assert np.all(np.diff(vr.h_np(x, eps)) > 0) and np.all(np.diff(vr.h_inv_np(x, eps)) > 0)


@pytest.mark.parametrize("eps", EPS)
def test_round_trips(eps):
    x = _magnitudes()
    for f, g in ((vr.h_np, vr.h_inv_np), (vr.h_inv_np, vr.h_np)):
        r = g(f(x, eps), eps)
        assert np.max(np.abs(r - x) / np.abs(x)) < 1e-14


def test_closed_forms_and_sample_values():
    # eps = 0: h = sqrt(a + 1) - 1 and h^-1 = (a + 1)^2 - 1, compared where those forms do not cancel; the
    # cancellation-free forms reduce to a / (sqrt(a + 1) + 1) and a (a + 2)
    x = np.abs(_magnitudes())
    big = x >= 1
    assert np.array_equal(vr.h_np(x, 0.0), x / (np.sqrt(x + 1) + 1))
    assert np.max(np.abs(vr.h_inv_np(x, 0.0) / (x * (x + 2)) - 1)) < 1e-15
    assert np.max(np.abs(vr.h_np(x[big], 0.0) / (np.sqrt(x[big] + 1) - 1) - 1)) < 1e-15
    assert np.max(np.abs(vr.h_inv_np(x[big], 0.0) / ((x[big] + 1) ** 2 - 1) - 1)) < 1e-15
    assert abs(vr.h_np(1000.0, 1e-3) - 31.6) < 0.05 and abs(vr.h_inv_np(10.0, 1e-3) - 117) < 0.5


@pytest.mark.parametrize("eps", [1e-3, 1e-2])
def test_textbook_inverse_agrees_where_it_does_not_cancel(eps):
    y = _magnitudes()
    y = y[np.abs(y) >= 1]
    assert np.max(np.abs(vr.h_inv_np(y, eps) / vr.h_inv_textbook_np(y, eps) - 1)) < 1e-12


@pytest.mark.parametrize("eps", EPS)
def test_target_map_is_monotone(eps):
    """Sorting the target network's quantiles before or after the transform gives the same targets: the transformed
    target of the tau-quantile is the tau-quantile of the transformed target."""
    rs = np.random.RandomState(4)
    B, Np = 64, 33
    z = (rs.standard_normal((B, Np)) * rs.choice([0.1, 3.0, 40.0], (B, 1))).astype(F32)
    r = (rs.standard_normal(B) * 300).astype(F32)
    nt = (rs.uniform(size=B) < 0.8).astype(F32)
    t1 = np.sort(vr.target_np(z, r, nt, 0.99 ** 3, eps), axis=1)
    t2 = vr.target_np(np.sort(z, axis=1), r, nt, 0.99 ** 3, eps)
    assert np.array_equal(t1, t2)


# The existing instantiations of the two loss kernels compile to the SASS they had before the rescaled instantiations
# were added: normalized `cuobjdump -sass` (symbol names and column alignment aside), CUDA 12.9, sm_90a.
SASS_DIGESTS = {"iqn_loss_kernel": "51ff206e68935cde47f787404dacf0220602e77c4ef41e242d2676b58a226b59",
                "c51_loss_kernel": "b58fefbcc4712205698071483505fe44c10ada17739a3c555767e8b580a30a40"}


def test_existing_loss_kernels_compile_to_unchanged_sass():
    from rainbow_iqn_apex_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(tool) and os.path.exists(nvcc) and os.path.exists(_lib.LIB_PATH)):
        pytest.skip("cuobjdump, nvcc or the built library is missing")
    if "release 12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("the digests were taken with CUDA 12.9")
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = block.split("\n", 1)
        m = re.match(r"_ZN4riqn15(iqn_loss_kernel|c51_loss_kernel)ILb0EE", name.strip())
        if m:
            body = body.split("\n\t\t..........")[0]
            norm = "\n".join(re.sub(r"\s+", " ", ln).strip() for ln in body.splitlines() if ln.strip())
            found[m.group(1)] = hashlib.sha256(norm.encode()).hexdigest()
    assert found == SASS_DIGESTS


# ------------------------------------------------------------------------------------------------ entry points (GPU)
def _rescale(dev, x, eps, inverse):
    xd = to_dev(x, dev)
    o = Out(x.size, dev)
    lib_call("riqn_value_rescale", x.size, dptr(xd), eps, inverse, o.p)
    torch.cuda.synchronize()
    assert_canaries({"out": o})
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("inverse", [0, 1])
def test_value_rescale_is_the_numpy_statement(cuda_dev, eps, inverse):
    rs = np.random.RandomState(11 + inverse)
    mags = np.concatenate(([0.0, 1e-45, 1e-40, 1e-30, 1e-12, 1e-7, 0.5, 1.0, 117.0, 1e6, 1e19, 1e30, 3.4e38],
                           10.0 ** rs.uniform(-40, 38, 3000)))
    x = np.concatenate((mags, -mags)).astype(F32)
    o = _rescale(cuda_dev, x, eps, inverse)
    with np.errstate(over="ignore"):
        want = (vr.h_inv_np if inverse else vr.h_np)(x, eps).astype(F32)
    assert_bits("h^-1" if inverse else "h", o.bits(), f32_bits(want))
    assert np.signbit(o.f32()[x.size // 2]) and not np.signbit(o.f32()[0])          # -0 -> -0, +0 -> +0
    if inverse:
        assert np.isinf(o.f32()[np.abs(x) == F32(3.4e38)]).all()                    # overflow to +-inf
    assert_bits("second call", _rescale(cuda_dev, x, eps, inverse).bits(), o.bits())


@pytest.mark.gpu
def test_value_rescale_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    x = to_dev(np.ones(16, F32), cuda_dev)
    o = Out(16, cuda_dev)
    for eps, inv, out in ((-1e-3, 0, o.p), (math.nan, 0, o.p), (math.inf, 1, o.p), (1e-3, 2, o.p), (1e-3, 0, None)):
        with pytest.raises(RiqnError):
            lib_call("riqn_value_rescale", 16, dptr(x), eps, inv, out)
    torch.cuda.synchronize()
    assert np.isnan(o.f32()).all() and o.canaries_ok()


def _iqn_case(seed, B, N, Np, A, scale=1.0):
    rs = np.random.RandomState(seed)
    c = dict(q_on=(scale * rs.standard_normal((N * B, A))).astype(F32),
             q_tgt=(scale * rs.standard_normal((Np * B, A))).astype(F32),
             tau=rs.uniform(0, 1, (N * B, 1)).astype(F32), actions=rs.randint(0, A, B).astype(np.int64),
             a_star=rs.randint(0, A, B).astype(np.int64), returns=(rs.standard_normal(B) * 50).astype(F32),
             nonterminals=(rs.uniform(size=B) < 0.8).astype(F32))
    c["nonterminals"][0] = 0.0
    return c


def _iqn_call(dev, c, B, N, Np, A, g, kappa, eps=None):
    d = {k: torch.from_numpy(v).to(dev) for k, v in c.items()}
    o = dict(loss=Out(B, dev), dtheta=Out(N * B, dev), theta=Out(B * N, dev), target=Out(B * Np, dev))
    args = [B, N, Np, A] + [dptr(d[k]) for k in ("q_on", "q_tgt", "tau", "actions", "a_star", "returns",
                                                  "nonterminals")] + [float(g), float(kappa)]
    outs = [o[k].p for k in ("loss", "dtheta", "theta", "target")]
    if eps is None:
        lib_call("riqn_iqn_loss_fwd_bwd", *args, *outs)
    else:
        lib_call("riqn_iqn_loss_fwd_bwd_h", *args, eps, *outs)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("B,N,Np,A,kappa,scale", [(512, 64, 64, 18, 1.0, 1.0), (3, 8, 13, 32, 0.5, 30.0),
                                                    (37, 5, 40, 1, 1.0, 0.01)])
def test_iqn_loss_h(cuda_dev, eps, B, N, Np, A, kappa, scale):
    g = 0.99 ** 3
    c = _iqn_case(B + N + A, B, N, Np, A, scale)
    o = _iqn_call(cuda_dev, c, B, N, Np, A, g, kappa, eps)
    z = c["q_tgt"].reshape(Np, B, A)[:, np.arange(B), c["a_star"]].T                     # (B, N')
    want = vr.target_np(z, c["returns"], c["nonterminals"], g, eps)
    target = o["target"].f32().reshape(B, Np)
    assert_bits("target", f32_bits(target), f32_bits(want))
    term = c["nonterminals"] == 0
    assert term.any()
    hr = vr.h_np(c["returns"][term], eps).astype(F32)
    assert_bits("terminal targets", f32_bits(target[term]), f32_bits(np.repeat(hr[:, None], Np, 1)))
    theta = c["q_on"][np.arange(N * B), np.tile(c["actions"], N)].reshape(N, B).T
    assert np.array_equal(o["theta"].f32().reshape(B, N), theta)
    loss, dth = om.pairwise_loss_np(theta, target, c["tau"].reshape(N, B).T, kappa)
    assert rel_err(o["loss"].f32(), loss) < 1e-5 and rel_err(o["dtheta"].f32(), dth.T.reshape(-1)) < 1e-5
    again = _iqn_call(cuda_dev, c, B, N, Np, A, g, kappa, eps)
    for k in o:
        assert_bits(f"second call {k}", again[k].bits(), o[k].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
def test_iqn_loss_h_identity_is_the_plain_loss(cuda_dev, eps):
    """R = 0, gamma^n = 1, nt = 1: fl32(h(h^-1(z))) = z for every float z, so every output is riqn_iqn_loss_fwd_bwd's."""
    B, N, Np, A = 128, 32, 48, 18
    c = _iqn_case(3, B, N, Np, A, 5.0)
    rs = np.random.RandomState(5)
    c["q_tgt"] = (c["q_tgt"] * 10.0 ** rs.uniform(-6, 6, c["q_tgt"].shape)).astype(F32)
    c["returns"][:] = 0
    c["nonterminals"][:] = 1
    h = _iqn_call(cuda_dev, c, B, N, Np, A, 1.0, 1.0, eps)
    p = _iqn_call(cuda_dev, c, B, N, Np, A, 1.0, 1.0)
    for k in h:
        assert_bits(k, h[k].bits(), p[k].bits())


@pytest.mark.gpu
def test_iqn_loss_h_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    B, N, Np = 4, 8, 8
    for A, eps in ((18, -1e-3), (18, math.nan), (18, math.inf), (33, 1e-3)):
        c = _iqn_case(1, B, N, Np, A)
        d = {k: torch.from_numpy(v).to(cuda_dev) for k, v in c.items()}
        o = dict(loss=Out(B, cuda_dev), dtheta=Out(N * B, cuda_dev), theta=Out(B * N, cuda_dev), target=Out(B * Np, cuda_dev))
        with pytest.raises(RiqnError):
            lib_call("riqn_iqn_loss_fwd_bwd_h", B, N, Np, A, *[dptr(d[k]) for k in ("q_on", "q_tgt", "tau", "actions",
                     "a_star", "returns", "nonterminals")], 0.97, 1.0, eps, *[o[k].p for k in ("loss", "dtheta", "theta",
                                                                                             "target")])
        torch.cuda.synchronize()
        assert all(np.isnan(v.f32()).all() and v.canaries_ok() for v in o.values())


def _expected_call(dev, q, w, B, n, A, eps, want_values=True, want_a=True):
    qd, wd = to_dev(q, dev), (to_dev(w, dev) if w is not None else None)
    v = Out(B * A, dev) if want_values else None
    a = torch.full((B + 64,), -5, dtype=torch.int64, device=dev) if want_a else None
    lib_call("riqn_argmax_expected_h", B, n, A, dptr(qd), dptr(wd), eps, v.p if v else None, dptr(a))
    torch.cuda.synchronize()
    if v is not None:
        assert v.canaries_ok()
    if a is not None:
        assert torch.all(a[B:] == -5)
    return v, (a[:B].cpu().numpy() if a is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("B,n,A,weighted", [(512, 32, 18, False), (512, 64, 18, True), (3, 1, 1, False),
                                            (70, 256, 32, True), (33, 7, 5, False)])
def test_argmax_expected_h(cuda_dev, eps, B, n, A, weighted):
    rs = np.random.RandomState(B + n + A)
    q = (rs.standard_normal((n * B, A)) * 10.0 ** rs.uniform(-2, 2, (1, A))).astype(F32)
    w = rs.dirichlet(np.ones(n), B).T.reshape(-1).astype(F32) if weighted else None
    # a duplicated best column in sample 0: the first of the two identical actions wins
    if A > 2:
        q.reshape(n, B, A)[:, 0, A - 1] = q.reshape(n, B, A)[:, 0, 1] = np.abs(q.reshape(n, B, A)[:, 0]).max() + 1
    want = vr.expected_np(q, B, eps, w)
    v, a = _expected_call(cuda_dev, q, w, B, n, A, eps)
    assert_bits("values", v.bits(), f32_bits(want.reshape(-1)))
    assert np.array_equal(a, vr.argmax_first(want))
    if A > 2:
        assert a[0] == 1
    v2, _ = _expected_call(cuda_dev, q, w, B, n, A, eps, want_a=False)
    _, a2 = _expected_call(cuda_dev, q, w, B, n, A, eps, want_values=False)
    assert_bits("values alone", v2.bits(), v.bits())
    assert np.array_equal(a2, a)


@pytest.mark.gpu
def test_argmax_expected_h_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    B, n = 4, 8
    for A, eps, nulls in ((18, -1.0, False), (18, math.nan, False), (18, math.inf, False), (33, 1e-3, False),
                          (18, 1e-3, True)):
        q = to_dev(np.ones((n * B, A), F32), cuda_dev)
        v = Out(B * A, cuda_dev)
        a = torch.full((B,), -5, dtype=torch.int64, device=cuda_dev)
        with pytest.raises(RiqnError):
            lib_call("riqn_argmax_expected_h", B, n, A, dptr(q), None, eps, None if nulls else v.p,
                     None if nulls else dptr(a))
        torch.cuda.synchronize()
        assert np.isnan(v.f32()).all() and v.canaries_ok() and torch.all(a == -5)


def _warp_sum_np(v):
    """common.cuh warp_sum over 32 lanes (B, 32) fp32: xor butterfly, lane 0's value."""
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, idx ^ o]).astype(F32)
    return v[:, 0]


def _c51_statement(h, support, gamma_n, v_min, v_max, atoms, eps):
    """numpy fp32 statement of riqn_c51_loss_fwd_bwd_h: the moved atoms, the projection indices and weights, m in the
    kernel's add order and the loss through its two-warp reduction."""
    B = h["ret"].shape[0]
    rows = np.arange(B)
    delta_z = F32((v_max - v_min) / (atoms - 1))
    tz = vr.c51_atoms_np(support, h["ret"], h["nt"], gamma_n, eps)
    tz = np.minimum(np.maximum(tz, F32(v_min)), F32(v_max))
    b = np.minimum(((tz - F32(v_min)).astype(F32) / delta_z).astype(F32), F32(atoms - 1))
    lo, up = np.floor(b).astype(np.int64), np.ceil(b).astype(np.int64)
    lo[(up > 0) & (lo == up)] -= 1
    up[(lo < atoms - 1) & (lo == up)] += 1
    pa = h["pt"][rows, h["astar"]]
    wl = (pa * (up.astype(F32) - b).astype(F32)).astype(F32)
    wu = (pa * (b - lo.astype(F32)).astype(F32)).astype(F32)
    m = np.zeros((B, atoms), F32)
    for j in range(atoms):
        m[rows, lo[:, j]] = (m[rows, lo[:, j]] + wl[:, j]).astype(F32)
    for j in range(atoms):
        m[rows, up[:, j]] = (m[rows, up[:, j]] + wu[:, j]).astype(F32)
    part = np.zeros((B, 64), F32)
    part[:, :atoms] = (m * h["logp"][rows, h["act"]]).astype(F32)
    tot = ((F32(0) + _warp_sum_np(part[:, :32])).astype(F32) + _warp_sum_np(part[:, 32:])).astype(F32)
    return m, -tot, pa


def _c51_inputs(B, A, atoms, seed, v_max):
    rs = np.random.RandomState(seed)
    h = dict(logp=np.log(rs.dirichlet(np.ones(atoms), (B, A))).astype(F32),
             pt=rs.dirichlet(np.ones(atoms), (B, A)).astype(F32), act=rs.randint(0, A, B).astype(np.int64),
             astar=rs.randint(0, A, B).astype(np.int64),
             ret=(rs.standard_normal(B) * rs.choice([0.5, 30.0, 3000.0], B)).astype(F32),
             nt=(rs.uniform(size=B) > 0.1).astype(F32))
    h["nt"][0], h["ret"][0] = 0.0, F32(v_max / 3)
    return h


def _c51_call(dev, B, A, atoms, h, support, gamma_n, v_min, v_max, eps=None):
    d = {k: (torch.from_numpy(v).to(dev) if v.dtype == np.int64 else to_dev(v, dev)) for k, v in h.items()}
    sup = to_dev(support, dev)
    o = {"loss": Out(B, dev), "dq": Out(B * atoms, dev), "m": Out(B * atoms, dev)}
    args = [B, A, atoms] + [dptr(d[k]) for k in ("logp", "pt", "act", "astar", "ret", "nt")] + [
        dptr(sup), float(gamma_n), float(v_min), float(v_max), float((v_max - v_min) / (atoms - 1))]
    outs = [o["loss"].p, o["dq"].p, o["m"].p]
    if eps is None:
        lib_call("riqn_c51_loss_fwd_bwd", *args, *outs)
    else:
        lib_call("riqn_c51_loss_fwd_bwd_h", *args, eps, *outs)
    torch.cuda.synchronize()
    assert_canaries(o)
    return o


C51_CASES = [(-16.0, 16.0, 33, 0.75), (-10.0, 10.0, 51, 0.99 ** 3), (-50.0, 50.0, 64, 0.99 ** 3), (-10.0, 10.0, 2, 1.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("B,A", [(1, 1), (37, 4), (512, 18)])
@pytest.mark.parametrize("v_min,v_max,atoms,gamma_n", C51_CASES)
def test_c51_loss_h(cuda_dev, eps, B, A, v_min, v_max, atoms, gamma_n):
    support = torch.linspace(v_min, v_max, atoms).numpy()
    h = _c51_inputs(B, A, atoms, B * 7 + atoms, v_max)
    o = _c51_call(cuda_dev, B, A, atoms, h, support, gamma_n, v_min, v_max, eps)
    m32, loss32, pa = _c51_statement(h, support, gamma_n, v_min, v_max, atoms, eps)
    m = o["m"].f32().reshape(B, atoms)
    assert_bits("m", f32_bits(m), f32_bits(m32))
    assert_bits("loss", o["loss"].bits(), f32_bits(loss32))
    psum = pa.astype(np.float64).sum(1)
    check_bound("sum m", m.astype(np.float64).sum(1), psum, 2.0 * 3 * atoms * U * psum)
    lp = h["logp"][np.arange(B), h["act"]].astype(np.float64)
    mt = m.astype(np.float64).sum(1, keepdims=True)
    e = np.exp(lp)
    ref_dq = -(m.astype(np.float64) - e * mt)
    check_bound("dq", o["dq"].f32().reshape(B, atoms), ref_dq, 2.0 * (6 * U * e * mt + e * (atoms + 2) * U * mt +
                                                                      U * np.abs(ref_dq)))
    again = _c51_call(cuda_dev, B, A, atoms, h, support, gamma_n, v_min, v_max, eps)
    for k in o:
        assert_bits(f"second call {k}", again[k].bits(), o[k].bits())


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
def test_c51_loss_h_identity_is_the_plain_loss(cuda_dev, eps):
    B, A, atoms, v_min, v_max = 64, 18, 51, -10.0, 10.0
    support = torch.linspace(v_min, v_max, atoms).numpy()
    h = _c51_inputs(B, A, atoms, 9, v_max)
    h["ret"][:] = 0
    hh = _c51_call(cuda_dev, B, A, atoms, h, support, 1.0, v_min, v_max, eps)
    pp = _c51_call(cuda_dev, B, A, atoms, h, support, 1.0, v_min, v_max)
    for k in hh:
        assert_bits(k, hh[k].bits(), pp[k].bits())


@pytest.mark.gpu
def test_c51_loss_h_rejects_and_writes_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError
    B, A = 4, 3
    for atoms, eps in ((51, -1e-3), (51, math.nan), (51, math.inf), (65, 1e-3)):
        support = torch.linspace(-10, 10, atoms).numpy()
        h = _c51_inputs(B, A, atoms, 1, 10.0)
        d = {k: (torch.from_numpy(v).to(cuda_dev) if v.dtype == np.int64 else to_dev(v, cuda_dev)) for k, v in h.items()}
        sup = to_dev(support, cuda_dev)
        o = {"loss": Out(B, cuda_dev), "dq": Out(B * atoms, cuda_dev), "m": Out(B * atoms, cuda_dev)}
        with pytest.raises(RiqnError):
            lib_call("riqn_c51_loss_fwd_bwd_h", B, A, atoms, *[dptr(d[k]) for k in ("logp", "pt", "act", "astar", "ret",
                     "nt")], dptr(sup), 0.97, -10.0, 10.0, 20.0 / (atoms - 1), eps, o["loss"].p, o["dq"].p, o["m"].p)
        torch.cuda.synchronize()
        assert all(np.isnan(v.f32()).all() and v.canaries_ok() for v in o.values())


# ------------------------------------------------------------------------------------------------ learner (GPU)
def _vr_args(dev, B, cfg=None, rainbow_only=False, **kw):
    a = make_args(dev, B, cfg, rainbow_only=rainbow_only)
    a.value_rescaling = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def _flips(dbg, keep, B):
    """ReLU kinks that the product and the oracle round to opposite sides of 0: conv1..3, h_v, h_a."""
    from test_gpu_learn import _qmajor
    gk = dbg["keep"]
    h = _qmajor(gk["h"], B).cpu()
    pairs = [(gk["out"][0], keep["o1"]), (gk["out"][1], keep["o2"]), (gk["out"][2], keep["o3"]),
             (h[:, :512], keep["h_v"]), (h[:, 512:], keep["h_a"])]
    return [int(((x.cpu() > 0) != (y > 0)).sum()) for x, y in pairs]


def _check_grads(grads, o_grads, fl, ties):
    relaxed = set()
    if sum(fl[3:]) or ties:
        relaxed |= {"conv1", "conv2", "conv3", "iqn_fc", "fcnoisy_h_v", "fcnoisy_h_a", "fcnoisy_z_v", "fcnoisy_z_a"}
    for i in range(3):
        if fl[i]:
            relaxed |= {f"conv{j + 1}" for j in range(i + 1)}
    for k, g_ref in o_grads.items():
        c = _cos(grads[k], g_ref)
        assert c > (0.98 if k.split(".")[0] in relaxed else 0.999), (k, c, fl)


def _near_ties(values, tol):
    top2 = np.sort(values, axis=1)[:, -2:]
    return (top2[:, 1] - top2[:, 0]) < tol


@pytest.mark.gpu
@pytest.mark.parametrize("B,risk", [(32, None), (512, None), (32, ("cvar", 0.25))])
def test_iqn_learner_step_vs_oracle(cuda_dev, B, risk):
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch
    n = 8 if B == 32 else 64
    cfg, seed, eps = cases.iqn_cfg(n, n, 32), 12100 + B, 1e-3
    params = net.make_params(seed)
    args = _vr_args(cuda_dev, B, cfg)
    if risk is not None:
        args.risk_measure, args.risk_eta = risk
    lr = Learner(args, 18, None)
    assert lr.value_rescaling == eps
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    b["returns"] = (b["returns"] * 40).astype(F32)                     # unclipped-scale returns
    t_sel, t_tgt, t_on = (torch.from_numpy(t) for t in cases.make_taus(seed + 2, B, cfg))
    noises = cases.make_noises(seed + 3)
    lr._inject = dict(noises=noises, taus=(None if risk else t_sel, t_tgt, t_on))
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    tau_sel = dbg["tau_sel"].cpu()
    if risk is not None:
        assert float(tau_sel.max()) <= 0.25
    # the kernel's a* and targets are the numpy statements of the quantile values the product computed
    q_sel, q_tgt = dbg["q_sel"].cpu().numpy(), dbg["q_tgt"].cpu().numpy()
    a_gpu = dbg["a_star"].cpu().numpy()
    assert np.array_equal(a_gpu, vr.argmax_first(vr.expected_np(q_sel, B, eps)))
    z = q_tgt.reshape(n, B, 18)[:, np.arange(B), a_gpu].T
    assert_bits("targets", f32_bits(dbg["target"].cpu().numpy()),
                f32_bits(vr.target_np(z, b["returns"], b["nonterminals"], cfg["discount"] ** cfg["n_step"], eps)))

    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=5e-5, eps=3.125e-4)
    keep = {}
    o_loss, o_grads = vr.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises,
                                    (tau_sel, t_tgt, t_on), cfg, eps, keep=keep)
    tie = _near_ties(keep["qv_next"].numpy(), 1e-4)
    ok = (a_gpu == keep["a_star"].numpy())
    assert np.all(ok | tie)
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max((np.abs(lg - lo) / np.abs(lo))[ok]) < 1e-3
    _check_grads(grads, o_grads, _flips(dbg, keep, B), not ok.all())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_fqf_learner_step_vs_oracle(cuda_dev, B):
    from rainbow_iqn_apex_b200 import Learner
    from test_gpu_learn import _dev_batch
    N, eps = 32, 1e-2
    cfg, seed = cases.iqn_cfg(N, N, 32), 12300 + B
    params = net.make_params(seed)
    torch.manual_seed(seed)
    lr = Learner(_vr_args(cuda_dev, B, cfg, fqf=1, value_rescaling_eps=eps), 18, None)
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    with torch.no_grad():
        lr.fraction_net.weight.mul_(30.0)
    wf, bf = (t.detach().cpu().clone().requires_grad_(True) for t in (lr.fraction_net.weight, lr.fraction_net.bias))
    b = cases.make_batch(seed + 1, B, n_step=cfg["n_step"], discount=cfg["discount"])
    b["returns"] = (b["returns"] * 40).astype(F32)
    noises = cases.make_noises(seed + 3)
    lr._inject = dict(noises=noises)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_gradients(st, ac, rt, nx, nt, w, debug=dbg)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    a_gpu = dbg["a_star"].cpu().numpy()
    qv = vr.expected_np(dbg["q_sel"].cpu().numpy(), B, eps, dbg["dtau_next"].cpu().numpy())
    assert np.array_equal(a_gpu, vr.argmax_first(qv))
    z = dbg["q_tgt"].cpu().numpy().reshape(N, B, 18)[:, np.arange(B), a_gpu].T
    assert_bits("targets", f32_bits(dbg["target"].cpu().numpy()),
                f32_bits(vr.target_np(z, b["returns"], b["nonterminals"], cfg["discount"] ** cfg["n_step"], eps)))
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    keep = {}
    o_loss, _, o_grads, _ = vr.fqf_step(p_on, p_tg, wf, bf, cases.batch_to_torch(b), torch.from_numpy(b["weights"]),
                                        noises, cfg, eps, keep=keep)
    tie = _near_ties(keep["qv_next"].numpy(), 1e-4)
    ok = a_gpu == keep["a_star"].numpy()
    assert np.all(ok | tie)
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max((np.abs(lg - lo) / np.abs(lo))[ok]) < 1e-3
    _check_grads(grads, o_grads, _flips(dbg, keep, B), not ok.all())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [32, 512])
def test_c51_learner_step_vs_oracle(cuda_dev, B):
    """The C51 loss through the Agent API (compute_loss_actor_or_learner + (w * loss).mean().backward(), the reference
    learner's call sequence), whose debug dict carries a* and m."""
    from rainbow_iqn_apex_b200 import Agent
    from test_gpu_learn import _dev_batch
    seed, eps = 12500 + B, 1e-3
    params = net.make_params(seed, rainbow_only=True)
    lr = Agent(_vr_args(cuda_dev, B, rainbow_only=True), 18, None)
    assert torch.equal(lr.acting_support.cpu(), torch.from_numpy(vr.h_inv_np(lr.support.cpu().numpy(), eps).astype(F32)))
    load_params(lr.online_net, params)
    lr.update_target_net()
    lr.train()
    b = cases.make_batch(seed + 1, B)
    b["returns"] = (b["returns"] * 40).astype(F32)
    noises = cases.make_noises(seed + 3, rainbow_only=True)
    lr._inject = dict(noises=noises, taus=None)
    st, ac, rt, nx, nt = _dev_batch(b, cuda_dev)
    w = torch.from_numpy(b["weights"]).to(cuda_dev)
    dbg = {}
    loss = lr.compute_loss_actor_or_learner(st, ac, rt, nx, nt, debug=dbg)
    lr.online_net.zero_grad()
    (w * loss).mean().backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=6.25e-5, eps=1.5e-4)
    keep = {}
    o_loss, o_grads = vr.learn_step(p_on, p_tg, adam, cases.batch_to_torch(b), torch.from_numpy(b["weights"]), noises,
                                    None, dict(atoms=51, v_min=-10.0, v_max=10.0), eps, rainbow_only=True, keep=keep)
    a_gpu = dbg["a_star"].cpu().numpy()
    tie = _near_ties(keep["ev_next"].numpy(), 1e-4)
    ok = a_gpu == keep["a_star"].numpy()
    assert np.all(ok | tie)
    assert rel_err(dbg["m"].cpu().numpy()[ok], keep["m"].numpy()[ok]) < 1e-3
    lg, lo = loss.detach().cpu().numpy(), o_loss.numpy()
    assert np.max((np.abs(lg - lo) / np.abs(lo))[ok]) < 1e-3
    # the C51 forward keeps no trunk activations to count ReLU-kink flips on: the convolutions take the relaxed bound
    _check_grads(grads, o_grads, [1, 1, 1, 0, 0], not ok.all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "fqf", "c51"])
def test_actor_paths_vs_oracle(cuda_dev, kind):
    """act, act_batch and act_batch_values act on the original-scale expectation; compute_priorities runs the rescaled
    loss."""
    from rainbow_iqn_apex_b200 import Actor
    E, seed, eps, K = 8, 12700, 1e-3, 16
    cfg = cases.iqn_cfg(16, 16, K)
    c51 = kind == "c51"
    params = net.make_params(seed, rainbow_only=c51)
    torch.manual_seed(seed)
    actor = Actor(_vr_args(cuda_dev, 8, None if c51 else cfg, rainbow_only=c51, **({"fqf": 1} if kind == "fqf" else {})),
                  18, None)
    load_params(actor.online_net, params)
    actor.update_target_net()
    actor.eval()
    rs = np.random.RandomState(seed)
    states = rs.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8)
    su8 = torch.from_numpy(states).to(cuda_dev)
    x = torch.from_numpy(states).float().div_(255)
    p_ev = net.to_torch(params)
    if c51:
        p = net.dqn_forward_c51(p_ev, x, 18, 51, training=False)
        ref = (p * torch.from_numpy(vr.h_inv_np(np.linspace(-10, 10, 51), eps)).float()).sum(2).numpy()
    else:
        if kind == "fqf":
            with torch.no_grad():
                actor.fraction_net.weight.mul_(50.0)
            wf, bf = actor.fraction_net.weight.detach().cpu(), actor.fraction_net.bias.detach().cpu()
            ref = vr.act_values(p_ev, x, 16, None, eps, training=False, w_f=wf, b_f=bf).numpy()
            qv = actor.act_batch_values(su8).cpu().numpy()
        else:
            tau = torch.from_numpy(rs.uniform(0, 1, (K * E, 1)).astype(F32))
            ref = vr.act_values(p_ev, x, K, tau, eps, training=False).numpy()
            qv = actor.act_batch_values(su8, tau=tau.to(cuda_dev)).cpu().numpy()
            actor._inject_act_tau = tau.to(cuda_dev)
        assert rel_err(qv, ref) < 5e-3
    a = actor.act_batch(su8).cpu().numpy()
    clear = ~_near_ties(ref, 1e-3)
    assert np.array_equal(a[clear], ref.argmax(1)[clear])
    if kind == "iqn":
        actor._inject_act_tau = torch.from_numpy(rs.uniform(0, 1, (K, 1)).astype(F32)).to(cuda_dev)
        with torch.no_grad():
            v1 = vr.expected_np(net.dqn_forward_iqn(p_ev, x[:1], K, actor._inject_act_tau.cpu(), training=False).numpy(),
                                1, eps)
        a1 = actor.act(list(states[0]))
        assert a1 == int(vr.argmax_first(v1)[0]) or _near_ties(v1, 1e-3)[0]
    elif clear[0]:
        assert actor.act(list(states[0])) == int(a[0])
    # priorities: compute_priorities runs the rescaled loss
    actor.train()
    bs, L, n, hist = 8, 14, 3, 4
    tab_state = [rs.randint(0, 256, (84, 84)).astype(np.uint8) for _ in range(L + hist - 1)]
    tab_action = [int(v) for v in rs.randint(0, 18, L)]
    tab_reward = [float(v) for v in rs.randint(-30, 31, L)]
    tab_nt = [1.0] * L
    chunks = math.ceil((L - n) / bs)
    rsm = [min(bs, L - n - c * bs) for c in range(chunks)]
    inj = []
    for c in range(chunks):
        d = dict(noises=cases.make_noises(seed + 10 * c, rainbow_only=c51))
        if kind == "iqn":
            d["taus"] = tuple(torch.from_numpy(t) for t in cases.make_taus(seed + 10 * c + 1, rsm[c], cfg))
        inj.append(d)
    actor._inject = list(inj)
    pri = actor.compute_priorities(tab_state, tab_action, tab_reward, tab_nt, 0.2)
    assert not actor._inject and pri.shape == (L - n,) and np.all(np.isfinite(pri))
    returns = np.float32([sum(0.99 ** k * tab_reward[k + i] for k in range(n)) for i in range(L - n)])
    out = []
    for c in range(chunks):
        lo, hi = c * bs, min((c + 1) * bs, L - n)
        st = torch.from_numpy(np.stack([np.stack(tab_state[i:i + hist]) for i in range(lo, hi)])).float().div_(255)
        nx = torch.from_numpy(np.stack([np.stack(tab_state[i + n:i + n + hist]) for i in range(lo, hi)])).float().div_(255)
        bt = (st, torch.tensor(tab_action[lo:hi]), torch.from_numpy(returns[lo:hi]), nx, torch.ones(hi - lo))
        p_on, p_tg = net.to_torch(params), net.to_torch(params)
        with torch.no_grad():
            if kind == "iqn":
                loss = vr.iqn_loss(p_on, p_tg, *bt, inj[c]["noises"], inj[c]["taus"], eps=eps, **cfg)
            elif kind == "c51":
                loss = vr.c51_loss(p_on, p_tg, *bt, inj[c]["noises"], eps=eps)
        if kind == "fqf":
            p_on = net.to_torch(params, requires_grad=True)
            loss, _, _, _ = vr.fqf_step(p_on, p_tg, wf.clone().requires_grad_(True), bf.clone().requires_grad_(True),
                                        bt, torch.ones(hi - lo), inj[c]["noises"], cfg, eps)
        out.append(loss.detach().numpy())
    ref_p = np.power(np.concatenate(out), 0.2)
    assert np.median(np.abs(pri - ref_p) / ref_p) < 1e-3 and np.max(np.abs(pri - ref_p) / ref_p) < 2e-2


def _bench_learner(dev, cap, graph, steps, rainbow_only, fields=None):
    import bench
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory, _lib
    torch.manual_seed(5)
    a = bench.make_args(dev, cap, rainbow_only=rainbow_only)
    if rainbow_only:
        a.lr, a.adam_eps = 6.25e-5, 1.5e-4
    for k, v in (fields or {}).items():
        setattr(a, k, v)
    learner = Learner(a, bench.ACTIONS, None)
    learner.train()
    mem = ReplayMemory(a, None)
    bench.fill_replay(mem, cap, dev, 7)
    if graph:
        learner.enable_cuda_graph(mem)
    out = []
    for _ in range(steps):
        c0 = _lib.launch_count()
        idxs, loss = learner.learn_and_update(mem)
        out.append((idxs.clone(), loss.clone(), _lib.launch_count() - c0))
    torch.cuda.synchronize()
    return out, learner.online_net._flat.detach().clone()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("rainbow_only", [False, True])
def test_rescaled_learner_steps_are_bitwise_reproducible(cuda_dev, graph, rainbow_only):
    fields = dict(value_rescaling=1)
    (s1, p1), (s2, p2) = (_bench_learner(cuda_dev, 1 << 14, graph, 3, rainbow_only, fields) for _ in range(2))
    for k, ((i1, l1, c1), (i2, l2, c2)) in enumerate(zip(s1, s2)):
        assert torch.equal(i1, i2) and torch.equal(l1, l2), k
        assert bool(torch.isfinite(l1).all())
    assert torch.equal(p1, p2)
    (s0, _) = _bench_learner(cuda_dev, 1 << 14, graph, 1, rainbow_only, dict(value_rescaling=0))
    assert not torch.equal(s0[0][1], s1[0][1])
    if not graph:
        assert s0[0][2] == s1[0][2]                    # the same launches: each entry point swapped for its _h twin


@pytest.mark.gpu
def test_checkpoint_key_and_mismatched_load(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent, Learner
    B, cfg = 32, cases.iqn_cfg(8, 8, 8)
    lr = Learner(_vr_args(cuda_dev, B, cfg, value_rescaling_eps=0.01), 18, None)
    lr.save(str(tmp_path), 0, 1, "vr.pth")
    ck = torch.load(os.path.join(tmp_path, "vr.pth"), map_location="cpu")
    assert ck["value_rescaling_eps"] == 0.01 and set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    back = Agent(_vr_args(cuda_dev, B, cfg, value_rescaling_eps=0.01, model=os.path.join(tmp_path, "vr.pth")), 18, None)
    assert back.value_rescaling == 0.01 and torch.equal(back.online_net._flat, lr.online_net._flat)
    plain = make_args(cuda_dev, B, cfg)
    plain.model = os.path.join(tmp_path, "vr.pth")
    with pytest.raises(ValueError, match="0.01"):
        Agent(plain, 18, None)
    with pytest.raises(ValueError):
        Agent(_vr_args(cuda_dev, B, cfg, model=os.path.join(tmp_path, "vr.pth")), 18, None)   # eps 1e-3 != 0.01
    Agent(make_args(cuda_dev, B, cfg), 18, None).save(str(tmp_path), 0, 1, "plain.pth")
    assert "value_rescaling_eps" not in torch.load(os.path.join(tmp_path, "plain.pth"), map_location="cpu")
    with pytest.raises(ValueError, match="None"):
        Agent(_vr_args(cuda_dev, B, cfg, model=os.path.join(tmp_path, "plain.pth")), 18, None)
    # rejected configurations
    for kw in (dict(munchausen=1), dict(value_rescaling_eps=-1.0), dict(value_rescaling_eps=math.nan),
               dict(value_rescaling=2)):
        with pytest.raises(ValueError):
            Agent(_vr_args(cuda_dev, B, cfg, **kw), 18, None)
