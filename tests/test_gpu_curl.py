"""CURL (Srinivas, Laskin & Abbeel, ICML 2020): riqn_curl_infonce_fwd_bwd, riqn_layernorm_fwd / _bwd, riqn_ema_f32,
riqn_add_f32, riqn_linear_wgrad and the learner fields curl, curl_coef, curl_momentum (rainbow_iqn_apex_b200/curl.py).

Kernels: the InfoNCE against float64 numpy over batch sizes 2 .. 4096 in three logit regimes (small, saturating, tied rows)
within fp32 bounds propagated from the statement, dW accumulated onto a prefill; the LayerNorm at widths 128 and 512 with
and without ReLU against float64; the EMA and the sum bit for bit against their numpy float32 statements; canaries past
every output and rejected calls that write nothing.  Learner: IQN and C51 against the torch-fp32 oracle (oracle/curl.py)
over three steps; a CURL learner against a plain one for every loss core (the loss, the shifts, every gradient past the
conv prefix bit for bit, and the conv gradient equal to a standalone trunk backward of dfeat_RL + dfeat_CURL); the
replay, batch and learn graphs against eager steps on the same device step state (momentum weights and operand images
included); reproducibility, checkpoints, validation and data parallelism.  Value-only mutants of the statements (the
softmax gradient without its identity term, W transposed, tau and 1 - tau swapped, the CURL term weighted by the IS
weights, the positive drawn before the existing shifts) are each rejected by the checks aimed at them."""
import os
import socket

import numpy as np
import pytest
import torch

from helpers import (U, Out, assert_bits, assert_canaries, check_bound, dptr, f32_bits, lib_call, load_params,
                     make_args, prefill_pattern, to_dev)
from oracle import cases, curl as oc, losses, network as net

D = 128


# ------------------------------------------------------------------------------------------------ statements (numpy)
def _ln(x):
    z = np.asarray(x, np.float64)
    d = z - z.mean(1, keepdims=True)
    return d / np.sqrt((d * d).mean(1, keepdims=True) + 1e-5)


def _infonce64(za, zk, w, coef, transpose_w=False, drop_identity=False):
    """float64 statement: rows, logits, dz_a, dW and the abs-value magnitudes the bounds are built from."""
    za, zk, w = (np.asarray(a, np.float64) for a in (za, zk, w))
    B = za.shape[0]
    W = w.T if transpose_w else w
    L = za @ W @ zk.T
    m = L.max(1, keepdims=True)
    e = np.exp(L - m)
    s = e.sum(1, keepdims=True)
    p = e / s
    rows = m[:, 0] + np.log(s[:, 0]) - np.diag(L)
    scale = np.float64(np.float32(coef) / np.float32(B))
    dl = scale * (p - (0 if drop_identity else np.eye(B)))
    g = dl @ zk
    dz = g @ W.T
    dW = za.T @ g
    if transpose_w:
        dW = dW.T
    A = np.abs(za) @ np.abs(w) @ np.abs(zk).T
    return dict(rows=rows, L=L, p=p, m=m[:, 0], s=s[:, 0], dl=dl, g=g, dz=dz, dW=dW, A=A, scale=scale)


def _bounds(r, za, zk, w, B):
    za, zk, w = (np.abs(np.asarray(a, np.float64)) for a in (za, zk, w))
    E = 300 * U * r["A"].max(1)                                       # logits error per row
    rel = 2 * E[:, None] + (B / 32 + 16) * U
    ddl = r["scale"] * (r["p"] * rel + 2 * U * (r["p"] + np.eye(B))) + U * np.abs(r["dl"])
    dg = ddl @ zk + (B + 2) * U * (np.abs(r["dl"]) @ zk)
    bz = dg @ w.T + 130 * U * (np.abs(r["g"]) @ w.T) + 1e-30
    bW = za.T @ dg + (B + 2) * U * (za.T @ np.abs(r["g"])) + 1e-30
    brow = 3 * E + (B / 32 + 16) * U + 2 * U * (np.abs(r["m"]) + np.abs(np.log(r["s"])) + np.abs(np.diag(r["L"])))
    return dict(L=300 * U * r["A"] + 1e-30, rows=brow, dz=bz, dW=bW)


def _inputs(B, regime, seed):
    rs = np.random.RandomState(seed)
    za = _ln(rs.standard_normal((B, D))).astype(np.float32)
    zk = _ln(rs.standard_normal((B, D))).astype(np.float32)
    w = (rs.uniform(-1, 1, (D, D)) / np.sqrt(D)).astype(np.float32)
    if regime == "saturating":
        w = (w * 40).astype(np.float32)                               # logits ~ 1e2 .. 1e3: exp underflows off the max
    elif regime == "tied":
        zk[:] = zk[0]                                                 # every row's logits tie
    return za, zk, w


def _run_infonce(dev, za, zk, w, coef, logits=True):
    B = za.shape[0]
    o = dict(rows=Out(B, dev), dz=Out(B * D, dev), dW=Out(D * D, dev, fill=prefill_pattern(D * D, 1e-3)),
             L=Out(B * B, dev) if logits else None)
    ins = [to_dev(a, dev) for a in (za, zk, w)]           # held until the launch has run
    lib_call("riqn_curl_infonce_fwd_bwd", B, D, *(dptr(t) for t in ins), coef, o["rows"].p, o["dz"].p, o["dW"].p,
             o["L"].p if logits else None)
    torch.cuda.synchronize()
    assert_canaries(o)
    return {k: (v.f32() if v is not None else None) for k, v in o.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["small", "saturating", "tied"])
@pytest.mark.parametrize("B", [2, 3, 31, 128, 512, 1000, 4096])
def test_infonce_vs_float64(cuda_dev, B, regime):
    za, zk, w = _inputs(B, regime, 100 + B)
    coef = 0.7
    got = _run_infonce(cuda_dev, za, zk, w, coef, logits=B <= 1000)
    r = _infonce64(za, zk, w, coef)
    bd = _bounds(r, za, zk, w, B)
    pre = prefill_pattern(D * D, 1e-3).astype(np.float64)
    if got["L"] is not None:
        check_bound("logits", got["L"].reshape(B, B), r["L"], bd["L"])
    check_bound("rows", got["rows"], r["rows"], bd["rows"])
    check_bound("dz_a", got["dz"].reshape(B, D), r["dz"], bd["dz"])
    check_bound("dW", got["dW"].reshape(D, D), pre.reshape(D, D) + r["dW"], bd["dW"] + U * np.abs(pre.reshape(D, D) + r["dW"]))
    again = _run_infonce(cuda_dev, za, zk, w, coef, logits=False)
    for k in ("rows", "dz", "dW"):
        assert_bits(k, f32_bits(again[k]), f32_bits(got[k]))
    if regime == "small" and B in (31, 512):
        # the value-only mutants of the statement, each rejected by the checks above
        for kw, key in ((dict(drop_identity=True), "dz"), (dict(transpose_w=True), "rows")):
            m = _infonce64(za, zk, w, coef, **kw)
            with pytest.raises(AssertionError):
                if key == "dz":
                    check_bound("dz_a (mutant)", got["dz"].reshape(B, D), m["dz"], bd["dz"])
                else:
                    check_bound("rows (mutant)", got["rows"], m["rows"], bd["rows"])


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("width", [128, 512])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("rows", [1, 7, 512])
def test_layernorm_vs_float64(cuda_dev, rows, width, relu, bias):
    rs = np.random.RandomState(rows * width + relu)
    x0 = (rs.standard_normal((rows, width)) * 3 + rs.standard_normal((rows, 1)) * 5).astype(np.float32)
    bv = rs.standard_normal(width).astype(np.float32) if bias else None
    dy = rs.standard_normal((rows, width)).astype(np.float32)
    y, dx = Out(rows * width, cuda_dev), Out(rows * width, cuda_dev)
    xd, dyd = to_dev(x0, cuda_dev), to_dev(dy, cuda_dev)
    bd = to_dev(bv, cuda_dev) if bias else None
    lib_call("riqn_layernorm_fwd", rows, width, dptr(xd), dptr(bd), relu, y.p)
    lib_call("riqn_layernorm_bwd", rows, width, dptr(xd), dptr(bd), dptr(dyd), relu, dx.p)
    torch.cuda.synchronize()
    assert_canaries(dict(y=y, dx=dx))
    x = x0 + bv if bias else x0                       # the row the kernels normalise: fl32(x + bias)
    xh = _ln(x)
    ref_y = np.maximum(xh, 0) if relu else xh
    d = x.astype(np.float64) - x.astype(np.float64).mean(1, keepdims=True)
    rstd = 1 / np.sqrt((d * d).mean(1, keepdims=True) + 1e-5)
    g = np.where(xh > 0, dy, 0.0) if relu else dy.astype(np.float64)
    ref_dx = rstd * (g - g.mean(1, keepdims=True) - xh * (g * xh).mean(1, keepdims=True))
    # x_hat is within ~(width + 8) u relative of |x - mean| rstd plus the mean's rounding; the backward adds its own sums
    by = (width + 16) * U * (np.abs(xh) + np.abs(x.astype(np.float64) - d).max(1, keepdims=True) * rstd + 1)
    check_bound("layernorm y", y.f32().reshape(rows, width), ref_y, by)
    mag = rstd * (np.abs(g) + np.abs(g).mean(1, keepdims=True) + np.abs(xh) * np.abs(g * xh).mean(1, keepdims=True))
    bdx = 4 * (width + 16) * U * (mag + rstd * np.abs(g).max(1, keepdims=True) * (1 + np.abs(xh)))
    if relu:      # a kink flip of a value within the forward's error of 0 moves its gradient: excluded from the bound
        near = np.abs(xh) <= by
        bdx = bdx + np.abs(near.astype(np.float64) * dy) * rstd * 2 + near.any(1, keepdims=True) * rstd * np.abs(dy).max() * 2 / width
    check_bound("layernorm dx", dx.f32().reshape(rows, width), ref_dx, bdx)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 1000, 1 << 20])
def test_ema_and_add_bit_for_bit(cuda_dev, n):
    rs = np.random.RandomState(n)
    theta = rs.standard_normal(n).astype(np.float32)
    xi0 = rs.standard_normal(n).astype(np.float32)
    th, x0 = to_dev(theta, cuda_dev), to_dev(xi0, cuda_dev)
    for tau in (0.001, 0.3, 1.0):
        xi = Out(n, cuda_dev, fill=xi0)
        lib_call("riqn_ema_f32", n, dptr(th), xi.p, tau)
        torch.cuda.synchronize()
        assert_canaries(dict(xi=xi))
        assert_bits(f"ema tau={tau}", f32_bits(xi.f32()), f32_bits(oc.ema(theta, xi0, tau)))
        if tau != 1.0:   # mutant: tau and 1 - tau swapped
            assert not np.array_equal(f32_bits(xi.f32()), f32_bits(oc.ema(theta, xi0, np.float32(1) - np.float32(tau))))
    out = Out(n, cuda_dev)
    lib_call("riqn_add_f32", n, dptr(th), dptr(x0), out.p)
    torch.cuda.synchronize()
    assert_canaries(dict(out=out))
    assert_bits("add", f32_bits(out.f32()), f32_bits(theta + xi0))


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,F", [(3, 512, 3136), (64, 128, 512), (5, 1, 7)])
def test_linear_wgrad_is_the_fraction_wgrad_statement(cuda_dev, B, n, F):
    """grad_w += dy^T x, grad_b += sum_b dy: one fmaf chain over b ascending per element, then added once."""
    rs = np.random.RandomState(B * n)
    dy = rs.standard_normal((B, n)).astype(np.float32)
    x = rs.standard_normal((B, F)).astype(np.float32)
    gw0, gb0 = prefill_pattern(n * F), prefill_pattern(n)
    gw, gb = Out(n * F, cuda_dev, fill=gw0), Out(n, cuda_dev, fill=gb0)
    dyd, xd = to_dev(dy, cuda_dev), to_dev(x, cuda_dev)
    lib_call("riqn_linear_wgrad", B, n, F, dptr(dyd), dptr(xd), gw.p, gb.p)
    torch.cuda.synchronize()
    assert_canaries(dict(gw=gw, gb=gb))
    acc = np.zeros((n, F), np.float32)
    accb = np.zeros(n, np.float32)
    for b in range(B):
        acc = (acc.astype(np.float64) + dy[b][:, None].astype(np.float64) * x[b][None, :]).astype(np.float32)  # fmaf
        accb = accb + dy[b]
    assert_bits("grad_w", f32_bits(gw.f32()), f32_bits(gw0 + acc.ravel()))
    assert_bits("grad_b", f32_bits(gb.f32()), f32_bits(gb0 + accb))


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(1, 1), (32, 512), (513, 512), (4096, 7)])
def test_colsum_add(cuda_dev, rows, cols):
    """out += the column sums, fp32 within the sum's chain-length bound, onto a prefill, and bit for bit again."""
    x = np.random.RandomState(rows + cols).standard_normal((rows, cols)).astype(np.float32)
    xd = to_dev(x, cuda_dev)
    pre = prefill_pattern(cols)
    outs = []
    for _ in range(2):
        o = Out(cols, cuda_dev, fill=pre)
        lib_call("riqn_colsum_add", rows, cols, dptr(xd), o.p)
        torch.cuda.synchronize()
        assert_canaries(dict(o=o))
        outs.append(o.f32())
    ref = pre.astype(np.float64) + x.astype(np.float64).sum(0)
    check_bound("colsum", outs[0], ref, (rows + 2) * U * (np.abs(x).sum(0) + np.abs(pre)) + 1e-30)
    assert_bits("colsum again", f32_bits(outs[1]), f32_bits(outs[0]))


@pytest.mark.gpu
def test_rejected_calls_write_nothing(cuda_dev):
    from rainbow_iqn_apex_b200._lib import RiqnError, call
    big = Out(4096 * 4096 // 16, cuda_dev)
    src = to_dev(np.ones(8 * 512, np.float32), cuda_dev)
    p, s = big.p, dptr(src)
    bad = [("riqn_curl_infonce_fwd_bwd", (1, D, s, s, s, 1.0, p, p, p, p)),
           ("riqn_curl_infonce_fwd_bwd", (4097, D, s, s, s, 1.0, p, p, p, p)),
           ("riqn_curl_infonce_fwd_bwd", (8, 64, s, s, s, 1.0, p, p, p, p)),
           ("riqn_curl_infonce_fwd_bwd", (8, D, s, s, s, float("nan"), p, p, p, p)),
           ("riqn_curl_infonce_fwd_bwd", (8, D, None, s, s, 1.0, p, p, p, p)),
           ("riqn_curl_infonce_fwd_bwd", (8, D, s, s, s, 1.0, p, None, p, p)),
           ("riqn_layernorm_fwd", (0, 128, s, None, 0, p)), ("riqn_layernorm_fwd", (4, 256, s, s, 0, p)),
           ("riqn_layernorm_fwd", (4, 128, None, s, 0, p)), ("riqn_layernorm_bwd", (4, 512, s, None, s, 1, None)),
           ("riqn_layernorm_bwd", (4, 64, s, s, s, 1, p)), ("riqn_layernorm_bwd", (4, 128, s, s, None, 1, p)),
           ("riqn_colsum_add", (0, 4, s, p)), ("riqn_colsum_add", (4, 0, s, p)), ("riqn_colsum_add", (4, 4, None, p)),
           ("riqn_colsum_add", (4, 4, s, None)), ("riqn_ema_f32", (16, s, p, 0.0)),
           ("riqn_ema_f32", (16, s, p, 1.5)), ("riqn_ema_f32", (16, s, p, float("inf"))), ("riqn_ema_f32", (0, s, p, 0.1)),
           ("riqn_ema_f32", (16, None, p, 0.1)), ("riqn_add_f32", (0, s, s, p)), ("riqn_add_f32", (16, s, None, p)),
           ("riqn_linear_wgrad", (0, 4, 4, s, s, p, p)), ("riqn_linear_wgrad", (4, 0, 4, s, s, p, p)),
           ("riqn_linear_wgrad", (4, 4, 4, s, s, None, p))]
    for name, a in bad:
        with pytest.raises(RiqnError):
            call(name, *a)
    torch.cuda.synchronize()
    assert bool(torch.isnan(big.t[:big.n]).all()) and big.canaries_ok()


# ------------------------------------------------------------------------------------------------ validation
def test_oracle_statements():
    """The oracle's InfoNCE equals the float64 statement, and its EMA is the float32 one (the CPU half of the checks)."""
    rs = np.random.RandomState(3)
    za, zk, w = _inputs(9, "small", 3)
    rows, L = oc.infonce(torch.from_numpy(za).double(), torch.from_numpy(zk).double(), torch.from_numpy(w).double())
    r = _infonce64(za, zk, w, 1.0)
    assert np.allclose(rows.numpy(), r["rows"], rtol=1e-12, atol=1e-12) and np.allclose(L.numpy(), r["L"], rtol=1e-12)
    x = rs.standard_normal((5, 512)).astype(np.float32)
    assert np.allclose(oc.layer_norm(torch.from_numpy(x).double()).numpy(), _ln(x), atol=1e-12)
    t, xi = np.float32([1.0, 2.0]), np.float32([0.5, -3.0])
    assert np.array_equal(oc.ema(t, xi, 0.25), np.float32([0.625, -1.75]))


# ------------------------------------------------------------------------------------------------ learner (GPU)
CONFIGS = {"iqn": {}, "cvar": dict(risk_measure="cvar", risk_eta=0.25), "cql": dict(cql=1), "dqfd": dict(dqfd=1),
           "iqn_vr": dict(value_rescaling=1), "miqn": dict(munchausen=1), "fqf": dict(fqf=1), "qr": dict(qr_dqn=1),
           "mmd": dict(qr_dqn=1, mmd=1), "c51": dict(rainbow_only=1), "hl_gauss": dict(rainbow_only=1, hl_gauss=1)}


def _args(dev, B, fields, curl=True, **more):
    a = make_args(dev, B, cases.iqn_cfg(64, 64, 32), rainbow_only=bool(fields.get("rainbow_only")))
    for k, v in dict(fields, random_shift=4, **more).items():
        setattr(a, k, v)
    if curl:
        a.curl = 1
    return a


def _learner(dev, B, fields, curl=True, seed=0, **more):
    from rainbow_iqn_apex_b200 import Learner
    torch.manual_seed(seed)
    lr = Learner(_args(dev, B, fields, curl, **more), 18, None)
    lr.train()
    return lr


def _dev_batch(dev, B, seed):
    b = cases.make_batch(seed, B)
    return b, tuple(torch.from_numpy(b[k]).to(dev) for k in
                    ("states", "actions", "returns", "next_states", "nonterminals", "weights"))


class _TrunkSpy:
    """Wraps a DQN's backward_trunk: records the kept operands and the loss core's dfeat (before any addend)."""

    def __init__(self, net_):
        self.net, self.orig, self.calls = net_, net_.backward_trunk, []

        def spy(keep, dfeat):
            self.calls.append((keep, dfeat.clone()))
            return self.orig(keep, dfeat)
        net_.backward_trunk = spy


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_curl_learner_equals_plain_learner_past_the_trunk(cuda_dev, cfg):
    B = 32
    b, batch = _dev_batch(cuda_dev, B, 70)
    demo = torch.from_numpy((np.arange(B) % 3 == 0).astype(np.uint8)).to(cuda_dev) if cfg == "dqfd" else None
    runs = {}
    for on in (False, True):
        lr = _learner(cuda_dev, B, CONFIGS[cfg], curl=on, seed=21)
        spy = _TrunkSpy(lr.online_net)
        dbgs, ls = [], []
        for _ in range(2):              # two eager steps: the second draws its shifts from the advanced counters
            dbgs.append({})
            ls.append(lr.compute_gradients(*batch, debug=dbgs[-1], demo=demo).clone())
        torch.cuda.synchronize()
        runs[on] = (lr, spy, dbgs, ls, lr.online_net._flat_grad.clone())
    (pl, pspy, pdbgs, plosses, pgrad), (cl, cspy, cdbgs, closses, cgrad) = runs[False], runs[True]
    for pd, cd, pls, cls in zip(pdbgs, cdbgs, plosses, closses):
        assert torch.equal(pls, cls) and bool(torch.isfinite(cls).all())
        for s0, s1 in zip(pd["shifts"], cd["shifts"]):
            assert torch.equal(s0, s1)
    assert not torch.equal(cdbgs[0]["shifts"][0], cdbgs[1]["shifts"][0])
    cdbg = cdbgs[-1]
    n = cl.online_net._offsets[id(cl.online_net.conv3.bias)] + cl.online_net.conv3.bias.numel()
    assert torch.equal(pgrad[n:], cgrad[n:])
    assert not torch.equal(pgrad[:n], cgrad[:n])
    assert len(pspy.calls) == len(cspy.calls) == 2
    (_, dfeat_p), (keep, dfeat_rl) = pspy.calls[-1], cspy.calls[-1]
    assert torch.equal(dfeat_p, dfeat_rl)                          # the loss core's feature gradient is unchanged
    total = torch.from_numpy(dfeat_rl.cpu().numpy() + cdbg["dfeat_curl"].cpu().numpy()).to(cuda_dev)
    on = cl.online_net
    on.zero_grad()
    cspy.orig(keep, total)                                         # the standalone trunk backward, nothing armed
    torch.cuda.synchronize()
    assert torch.equal(on._flat_grad[:n], cgrad[:n])
    assert float(cl.curl_net._flat_grad.abs().sum()) > 0
    # the positive view: an independent shift under a key of its own; drawn from the shifts' stream before them (mutant)
    # the s_t / s_{t+n} shifts would move
    from rainbow_iqn_apex_b200 import augment
    assert on._shift_calls == pl.online_net._shift_calls == 2
    probe = _learner(cuda_dev, B, CONFIGS[cfg], curl=False, seed=21).online_net
    augment.draw_shifts(probe, B, 4)
    mut = augment.draw_shifts(probe, 2 * B, 4)
    assert not torch.equal(mut[B:], cdbgs[0]["shifts"][0])
    assert not torch.equal(cdbg["curl_shifts"], cdbg["shifts"][0])
    assert not torch.equal(cdbgs[0]["curl_shifts"], cdbgs[1]["curl_shifts"])


def _oracle_state(lr):
    p = {k: getattr(lr.curl_net, k).detach().cpu().clone().requires_grad_(True) for k in oc.NAMES}
    mc = {k: v.detach().cpu().clone() for k, v in lr.online_net.state_dict().items() if k in oc.CONV}
    mom = lr.momentum_net.state_dict()
    assert all(torch.equal(mom[k].cpu(), mc[k]) for k in oc.CONV)            # xi = theta at construction
    views = lr.curl_net.views(lr.momentum_projection)
    mp = {k: v.detach().cpu().clone() for k, v in zip(oc.PROJ, views)}
    return p, mc, mp


def _cos(a, b):
    a, b = a.double().ravel(), b.double().ravel()
    return float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["iqn", "c51"])
def test_learner_steps_vs_torch_oracle(cuda_dev, kind):
    from test_gpu_augment import shift_np
    B, steps, seed = 32, 3, 9900
    rainbow = kind == "c51"
    cfg = cases.iqn_cfg(64, 64, 32)
    params = net.make_params(seed, rainbow_only=rainbow)
    lr = _learner(cuda_dev, B, dict(rainbow_only=1) if rainbow else {}, seed=seed)
    load_params(lr.online_net, params)
    lr.update_target_net()
    from rainbow_iqn_apex_b200 import curl as dcurl
    n = dcurl.trunk_numel(lr.online_net)
    lr.momentum_net._flat[:n].copy_(lr.online_net._flat[:n])                 # xi = theta for the loaded weights
    lr.momentum_net._params_changed()
    coef, tau_m = lr.curl
    p_on, p_tg = net.to_torch(params, requires_grad=True), net.to_torch(params)
    cp, mc, mp = _oracle_state(lr)
    lrate, eps = (6.25e-5, 1.5e-4) if rainbow else (5e-5, 3.125e-4)
    adam = losses.Adam([k for k in p_on if net.is_trainable(k)], lr=lrate, eps=eps)
    cadam = losses.Adam(list(oc.NAMES), lr=lrate, eps=eps)
    ocfg = dict(atoms=51, v_min=-10.0, v_max=10.0, discount=0.99, n_step=3) if rainbow else cfg
    mom_tail = lr.momentum_net._flat[n:].cpu().numpy().copy()
    for step in range(steps):
        b, batch = _dev_batch(cuda_dev, B, 300 + step)
        rs = np.random.RandomState(seed + step)
        s_st, s_nx, s_k = (rs.randint(-4, 5, (B, 2)).astype(np.int32) for _ in range(3))
        noises = cases.make_noises(seed + 10 * step, rainbow_only=rainbow)
        taus = None if rainbow else tuple(torch.from_numpy(t) for t in cases.make_taus(seed + step, B, cfg))
        lr._inject = dict(noises=noises, taus=taus, shifts=(s_st, s_nx), curl_shifts=s_k)
        dbg = {}
        loss = lr.compute_gradients(*batch, debug=dbg)
        torch.cuda.synchronize()
        g_on = {k: p.grad.detach().cpu().clone() for k, p in lr.online_net.named_parameters()}
        g_cu = {k: getattr(lr.curl_net, k).grad.detach().cpu().clone() for k in oc.NAMES}
        pn = lr.curl_net.proj_numel
        xi0, xp0, c0 = (t.detach().cpu().numpy().copy() for t in (lr.momentum_net._flat[:n], lr.momentum_projection,
                                                                   lr.curl_net._flat))
        lr.apply_gradients()
        torch.cuda.synchronize()
        # the momentum update, after Adam, over the trunk prefix and the projection: bit for bit its float32 statement on
        # this step's device values (tau and 1 - tau swapped, before Adam, or over another range all fail here)
        theta, ctheta = lr.online_net._flat[:n].cpu().numpy(), lr.curl_net._flat.cpu().numpy()
        assert not np.array_equal(ctheta, c0)                                          # the CURL arena was stepped
        assert_bits("momentum trunk", f32_bits(lr.momentum_net._flat[:n].cpu().numpy()), f32_bits(oc.ema(theta, xi0, tau_m)))
        assert_bits("momentum projection", f32_bits(lr.momentum_projection.cpu().numpy()),
                    f32_bits(oc.ema(ctheta[:pn], xp0, tau_m)))
        assert not np.array_equal(lr.momentum_net._flat[:n].cpu().numpy(), xi0)
        assert np.array_equal(lr.momentum_net._flat[n:].cpu().numpy(), mom_tail)       # nothing past the trunk moves
        bs = dict(b, states=shift_np(b["states"], s_st), next_states=shift_np(b["next_states"], s_nx))
        x_k = torch.from_numpy(shift_np(b["states"], s_k)).float().div_(255)
        if step == 0:
            # mutant: the CURL term weighted by the IS weights (the bilinear's gradient on the pre-step parameters)
            with torch.no_grad():
                z_a = oc.project(cp, net.conv_trunk(p_on, cases.batch_to_torch(bs)[0]))
                z_k = oc.project(mp, net.conv_trunk(mc, x_k))
            wm = cp["bilinear"].detach().clone().requires_grad_(True)
            r_m, _ = oc.infonce(z_a, z_k, wm)
            (coef * (torch.from_numpy(b["weights"]) * r_m).mean()).backward()
            assert _cos(g_cu["bilinear"], wm.grad) < 0.9999
        okeep = {}
        o_loss, o_g, o_cg, o_dbg = oc.learn_step(p_on, p_tg, adam, cases.batch_to_torch(bs), torch.from_numpy(b["weights"]),
                                                 noises, taus, ocfg, cp, cadam, mc, mp, x_k, coef, tau_m,
                                                 rainbow_only=rainbow, keep=okeep)
        # the existing step tests' rule: 4e-4 relative on every row but the near-ties of a* (IQN: the two best mean
        # quantile values within 1e-4; C51, whose projection moves with a flipped a*: at most two rows)
        rel = np.abs(loss.cpu().numpy() - o_loss.numpy()) / np.abs(o_loss.numpy())
        if rainbow:
            tie = rel >= 4e-4
            assert tie.sum() <= 2, (step, int(tie.sum()), float(rel.max()))
        else:
            top2 = np.sort(okeep["q_sel"].detach().reshape(32, B, -1).mean(0).numpy(), axis=1)[:, -2:]
            tie = (top2[:, 1] - top2[:, 0]) < 1e-4
        assert np.max(rel[~tie]) < 4e-4, (step, float(np.max(rel[~tie])))
        rows = dbg["curl_loss"].cpu().numpy()
        assert np.max(np.abs(rows - o_dbg["rows"].numpy()) / (np.abs(o_dbg["rows"].numpy()) + 1e-3)) < 4e-3, step
        worst = min(_cos(g_cu[k], o_cg[k]) for k in oc.NAMES)
        assert worst >= 0.9999, (step, worst)
        # the existing step tests' bounds: 0.999, 0.98 for the convolutions (bf16 backward, ReLU kinks), after the first
        # step, where the two parameter sets have moved apart by Adam's rounding, 0.99 and 0.95
        for k in o_g:
            c = _cos(g_on[k], o_g[k])
            assert c >= (0.98 if k.startswith("conv") else 0.999) - (0 if step == 0 else 0.03), (step, k, c)
    # arenas, momentum and Adam moments after the steps
    for k in oc.NAMES:
        d = (getattr(lr.curl_net, k).detach().cpu() - cp[k].detach()).abs()
        # Adam moves a weight by about lr a step whatever its gradient: the arena must follow the oracle far closer than
        # that on all but a few elements (gradients near adam_eps, where lr * g / (|g| + eps) amplifies their rounding)
        assert float(d.max()) <= steps * lrate and int((d > 0.02 * lrate).sum()) <= max(8, d.numel() // 1000), k
    mom = lr.momentum_net.state_dict()
    for k in oc.CONV:
        assert float((mom[k].cpu() - mc[k]).abs().max()) <= steps * lrate
    for v, k in zip(lr.curl_net.views(lr.momentum_projection), oc.PROJ):
        assert float((v.cpu() - mp[k]).abs().max()) <= steps * lrate
    ca = lr.curl_optimiser
    for k in oc.NAMES:
        m, _ = ca._views(getattr(lr.curl_net, k))
        assert _cos(m.cpu(), cadam.m[k]) >= 0.9999, k
    named = dict(lr.online_net.named_parameters())
    for k in oc.CONV:
        m, _ = lr.optimiser._views(named[k])
        assert _cos(m.cpu(), adam.m[k]) >= 0.99, k


def _momentum_images(lr):
    """Copies of the key trunk's bf16 operand images (strip-ordered and im2col-ordered), as int16 bit patterns."""
    m = lr.momentum_net
    ims = [t for name in ("conv1", "conv2", "conv3") for t in (*m._strip_ops[name], *m._conv_ops[name])]
    return [t.view(torch.int16).clone() for t in ims if t is not None]


def _mirror_steps(dev, kind, k=3):
    """k steps of a CURL learner replayed from the captured graph of ``kind`` ("replay", "batch", "learn") and the same
    steps run eagerly by a twin through the same device step state.  Returns the two learners and their losses."""
    from rainbow_iqn_apex_b200 import Learner, ReplayMemory
    from rainbow_iqn_apex_b200.dynstate import DynState
    B = 32
    out = []
    for graph in (True, False):
        torch.manual_seed(3)
        args = _args(dev, B, {}, nb_actor=1, actor_capacity=512)
        lr = Learner(args, 18, None)
        lr.train()
        mem = ReplayMemory(args, None)
        rs = np.random.RandomState(1)
        nn_ = 512
        mem.transitions.append_arrays(0, 0, np.arange(nn_) % 97, rs.randint(0, 256, (nn_, 84, 84)).astype(np.uint8),
                                      rs.randint(0, 18, nn_), rs.randint(-1, 2, nn_).astype(np.float32),
                                      rs.uniform(size=nn_) < 0.03, (rs.uniform(0.1, 1, nn_) ** 0.2).astype(np.float32))
        for obj, sd in ((lr.online_net, 11), (lr.target_net, 12), (mem.transitions, 13)):
            obj._rng_seed = sd
        lr.momentum_net._refresh_tc_operands(force=True, h_done=True)
        lr._images0 = _momentum_images(lr)
        out.append((lr, mem))
    (a, mem_a), (b, mem_b) = out
    batches = [tuple(x.contiguous() for x in _dev_batch(dev, B, 40 + s)[1]) for s in range(k)]
    warm = {"replay": 3, "batch": 2, "learn": 2}[kind]
    if kind == "replay":
        a.enable_cuda_graph(mem_a)
    elif kind == "batch":
        a.enable_cuda_graph(mem_a)
        ex = tuple(t.contiguous() for t in mem_a.sample(B))
        a.enable_batch_graph(mem_a, ex)
    else:
        a.enable_learn_graph(batches[0])
    b._dyn = DynState(dev, slots=len(b._optimisers()))
    la, lb = [], []
    with b._attached(None if kind == "learn" else mem_b):
        if kind == "batch":          # the replay graph's capture first: its warm-up steps and its pre-capture write
            for _ in range(3):
                b._write_dyn(mem_b)
                b._step_post(mem_b, *b._step_pre(mem_b))
            b._write_dyn(mem_b)
        for _ in range(warm):
            if kind == "replay":
                b._write_dyn(mem_b)
                b._step_post(mem_b, *b._step_pre(mem_b))
            elif kind == "batch":
                b._write_dyn(mem_b)
                b._reset_step_streams()
                b._step_post(mem_b, ex[0], b.compute_gradients(*ex[1:]))
            else:
                b._write_dyn(None)
                b._reset_step_streams()
                b._step_post(None, None, b.compute_gradients(*batches[0]))
        b._dyn.epoch += 1
        for s in range(k):
            for lr in (a, b):           # the key trunk weights this step's refresh of the operand images reads
                m = lr.momentum_net
                lr._xi_before_last = m._flat[:m._offsets[id(m.conv3.bias)] + m.conv3.bias.numel()].clone()
            if kind == "replay":
                _, l1 = a.learn_and_update(mem_a)
                b._write_dyn(mem_b)
                idx, l2 = b._step_pre(mem_b)
                b._step_post(mem_b, idx, l2)
            elif kind == "batch":
                h = ex
                l1 = a._replay(a._graphs["batch"], h)
                b._write_dyn(mem_b)
                b._reset_step_streams()
                l2 = b.compute_gradients(*h[1:])
                b._step_post(mem_b, h[0], l2)
            else:
                l1 = a.learn_on_graph(batches[s])
                b._write_dyn(None)
                b._reset_step_streams()
                l2 = b.compute_gradients(*batches[s])
                b._step_post(None, None, l2)
            torch.cuda.synchronize()
            la.append(l1.clone())
            lb.append(l2.clone())
    return a, b, la, lb


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["replay", "batch", "learn"])
def test_graph_replays_equal_eager_steps(cuda_dev, kind):
    a, b, la, lb = _mirror_steps(cuda_dev, kind)
    for x, y in zip(la, lb):
        assert torch.equal(x, y) and bool(torch.isfinite(x).all())
    assert not torch.equal(la[0], la[1])
    for x, y in ((a.online_net._flat, b.online_net._flat), (a.curl_net._flat, b.curl_net._flat),
                 (a.momentum_net._flat, b.momentum_net._flat), (a.momentum_projection, b.momentum_projection),
                 (a.curl_optimiser._exp_avg, b.curl_optimiser._exp_avg)):
        assert torch.equal(x, y)
    for name in ("conv1", "conv2", "conv3"):      # the key trunk's operand images follow its weights in every replay
        for x, y in zip(a.momentum_net._strip_ops[name], b.momentum_net._strip_ops[name]):
            assert torch.equal(x.view(torch.int16), y.view(torch.int16))
    n = a.momentum_net._offsets[id(a.momentum_net.conv3.bias)] + a.momentum_net.conv3.bias.numel()
    assert not torch.equal(a.momentum_net._flat[:n], a.online_net._flat[:n])    # xi lags theta
    # the images the last replay used are those of the momentum weights it read (a rebuild from the current weights,
    # which the EMA has moved since the last replay's refresh, differs only through that last update: undo it first)
    for lr in (a, b):
        used = _momentum_images(lr)
        assert any(not torch.equal(x, y) for x, y in zip(used, lr._images0))      # the images followed the weights
        m = lr.momentum_net
        cur = m._flat[:n].clone()
        m._flat[:n].copy_(lr._xi_before_last)
        m._refresh_tc_operands(force=True, h_done=True)
        for x, y in zip(_momentum_images(lr), used):
            assert torch.equal(x, y)
        m._flat[:n].copy_(cur)


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal_and_checkpoints_round_trip(cuda_dev, tmp_path):
    from rainbow_iqn_apex_b200 import Agent
    B = 32
    res = []
    for _ in range(2):
        lr = _learner(cuda_dev, B, {}, seed=8)
        ls = [lr.learn_on_batch(*_dev_batch(cuda_dev, B, 50 + s)[1]).clone() for s in range(2)]
        torch.cuda.synchronize()
        res.append((lr, ls))
    (l1, a1), (l2, a2) = res
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    for x, y in ((l1.online_net._flat, l2.online_net._flat), (l1.curl_net._flat, l2.curl_net._flat),
                 (l1.momentum_net._flat, l2.momentum_net._flat), (l1.momentum_projection, l2.momentum_projection)):
        assert torch.equal(x, y)
    l1.save(str(tmp_path), 0, 2, "curl.pth")
    path = os.path.join(tmp_path, "curl.pth")
    ck = torch.load(path, map_location="cpu")
    assert {"curl_state_dict", "curl_optimiser_state_dict", "curl_momentum_state_dict"} <= set(ck)
    assert set(ck["model_state_dict"]) == set(net.layer_shapes(18))
    back = Agent(_args(cuda_dev, B, {}, model=path), 18, None)
    assert torch.equal(back.curl_net._flat, l1.curl_net._flat)
    assert back.curl_optimiser._step == l1.curl_optimiser._step == 2
    assert torch.equal(back.curl_optimiser._exp_avg, l1.curl_optimiser._exp_avg)
    assert torch.equal(back.curl_optimiser._exp_avg_sq, l1.curl_optimiser._exp_avg_sq)
    n = back.momentum_net._offsets[id(back.momentum_net.conv3.bias)] + back.momentum_net.conv3.bias.numel()
    assert torch.equal(back.momentum_net._flat[:n], l1.momentum_net._flat[:n])
    assert torch.equal(back.momentum_projection, l1.momentum_projection)
    # a plain checkpoint into a CURL agent: a fresh projection with xi = theta
    plain = _learner(cuda_dev, B, {}, curl=False, seed=8)
    plain.save(str(tmp_path), 0, 0, "plain.pth")
    c = Agent(_args(cuda_dev, B, {}, model=os.path.join(tmp_path, "plain.pth")), 18, None)
    assert torch.equal(c.online_net._flat, plain.online_net._flat)
    assert torch.equal(c.momentum_net._flat[:n], c.online_net._flat[:n])
    assert torch.equal(c.momentum_projection, c.curl_net._flat[:c.curl_net.proj_numel])
    # and a CURL checkpoint into a plain agent
    p2 = Agent(_args(cuda_dev, B, {}, curl=False, model=path), 18, None)
    assert torch.equal(p2.online_net._flat, l1.online_net._flat) and p2.curl_net is None


@pytest.mark.gpu
def test_construction(cuda_dev):
    from rainbow_iqn_apex_b200 import Learner
    torch.manual_seed(4)
    plain = Learner(_args(cuda_dev, 32, {}, curl=False), 18, None)
    torch.manual_seed(4)
    lr = Learner(_args(cuda_dev, 32, {}, curl_coef=0.5, curl_momentum=0.01), 18, None)
    assert lr.curl == (0.5, np.float32(0.01)) and plain.curl is None and plain.curl_net is None
    assert torch.equal(lr.online_net._flat, plain.online_net._flat) and lr.online_net._rng_seed == plain.online_net._rng_seed
    assert lr.curl_optimiser.param_groups[0]["lr"] == 5e-5 and lr.curl_optimiser.param_groups[0]["eps"] == 3.125e-4
    for bad in (dict(random_shift=0), dict(batch_size=1), dict(curl=2), dict(curl_coef=0.0), dict(curl_momentum=2.0)):
        a = _args(cuda_dev, 32, {})
        for k, v in bad.items():
            setattr(a, k, v)
        with pytest.raises(ValueError):
            Learner(a, 18, None)
    assert lr._dyn is None
    b = _dev_batch(cuda_dev, 32, 1)[1]
    from rainbow_iqn_apex_b200 import _lib
    lr.learn_on_batch(*b)
    plain.learn_on_batch(*b)
    c0 = _lib.launch_count()
    lr.learn_on_batch(*b)
    c1 = _lib.launch_count()
    plain.learn_on_batch(*b)
    c2 = _lib.launch_count()
    print(f"eager step launches: CURL {c1 - c0}, plain {c2 - c1}, extra {(c1 - c0) - (c2 - c1)}")
    assert (c1 - c0) > (c2 - c1)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_data_parallel_replica_runs_the_curl_step(cuda_dev):
    """A learner in a one-rank process group takes the data-parallel path (every arena all-reduced, CURL's included) and
    computes the same bits as the plain CURL learner."""
    import torch.distributed as dist
    from rainbow_iqn_apex_b200 import parallel
    B = 32
    batch = _dev_batch(cuda_dev, B, 12)[1]
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        out = []
        for dp in (False, True):
            lr = _learner(cuda_dev, B, {}, seed=1)
            if dp:
                lr.process_group = dist.group.WORLD
                assert lr.curl_net in lr._trained_nets() and lr.curl_optimiser in lr._optimisers()
            ls = [lr.learn_on_batch(*batch).clone() for _ in range(2)]
            torch.cuda.synchronize()
            out.append((ls, lr.online_net._flat.clone(), lr.curl_net._flat.clone(), lr.momentum_projection.clone()))
        for l1, l2 in zip(out[0][0], out[1][0]):
            assert torch.equal(l1, l2)
        for x, y in zip(out[0][1:], out[1][1:]):
            assert torch.equal(x, y)
        # parallel.make_data_parallel's CURL branch, run as for two ranks on this one-rank group: the projection, the
        # momentum encoder and its projection are broadcast from rank 0 (here: unchanged) and every optimiser averages
        lr = _learner(cuda_dev, B, {}, seed=1)
        lr.learn_on_batch(*batch)
        before = [t.clone() for t in (lr.curl_net._flat, lr.momentum_net._flat, lr.momentum_projection)]
        real = parallel.dist.get_world_size
        parallel.dist.get_world_size = lambda group=None: 2
        try:
            assert parallel.make_data_parallel(lr) is lr
        finally:
            parallel.dist.get_world_size = real
        assert lr.process_group is not None
        assert lr.optimiser.grad_scale == lr.curl_optimiser.grad_scale == 0.5
        for x, y in zip(before, (lr.curl_net._flat, lr.momentum_net._flat, lr.momentum_projection)):
            assert torch.equal(x, y)
    finally:
        dist.destroy_process_group()
