"""The EMA target and AdamW fields (target_ema, target_ema_tau, adamw, adamw_weight_decay) through config.read, the
float64 statement of AdamW (oracle/bbf.py) against torch.optim.AdamW, and the arena optimiser's state_dict between Adam
and AdamW.  Host-only."""
import ctypes
import math
import types

import numpy as np
import pytest
import torch
from torch import nn

from oracle import bbf
from rainbow_iqn_apex_b200 import config
from rainbow_iqn_apex_b200.arena import ArenaModule
from rainbow_iqn_apex_b200.optim import Adam

F32 = lambda x: ctypes.c_float(x).value
HEADS = [dict(), dict(rainbow_only=1), dict(qr_dqn=1)]
LOSSES = [dict(), dict(munchausen=1), dict(fqf=1), dict(qr_dqn=1, mmd=1), dict(rainbow_only=1, hl_gauss=1), dict(cql=1),
          dict(qr_dqn=1, cql=1), dict(dqfd=1), dict(qr_dqn=1, dqfd=1), dict(value_rescaling=1),
          dict(rainbow_only=1, value_rescaling=1), dict(random_shift=4), dict(curl=1, random_shift=4), dict(spr=1),
          dict(spr=1, random_shift=4, rainbow_only=1), dict(spr=1, qr_dqn=1, reset=1),
          dict(risk_measure="cvar", risk_eta=0.25)]


def _ns(**kw):
    a = types.SimpleNamespace(rainbow_only=0, num_tau_samples=64, batch_size=32, history_length=4, lr=6.25e-5)
    a.__dict__.update(kw)
    return a


def test_defaults_and_values():
    v = config.read(_ns(), 18)
    assert v["target_ema"] is None and v["adamw"] is None
    off = config.read(_ns(target_ema=0, target_ema_tau=-3, adamw=0, adamw_weight_decay="x"), 18)   # off: not read
    assert off == v
    on = config.read(_ns(target_ema=1, adamw=1), 18)
    assert on["target_ema"] == F32(0.005) and on["adamw"] == F32(0.1)         # BBF's, as the float32 the kernels take
    assert type(on["target_ema"]) is float and type(on["adamw"]) is float
    on = config.read(_ns(target_ema=True, target_ema_tau=1, adamw=True, adamw_weight_decay=0), 18)
    assert (on["target_ema"], on["adamw"]) == (1.0, 0.0)
    assert config.read(_ns(target_ema=1, target_ema_tau=1e-30), 18)["target_ema"] == F32(1e-30)
    assert config.read(_ns(adamw=1, adamw_weight_decay=1e6, lr=1e-7), 18)["adamw"] == 1e6


@pytest.mark.parametrize("bad", [dict(target_ema=2), dict(target_ema=0.5), dict(target_ema="1"), dict(target_ema=None),
                                 dict(target_ema_tau=0), dict(target_ema_tau=-0.1), dict(target_ema_tau=1.0000001),
                                 dict(target_ema_tau=1e-46), dict(target_ema_tau=math.nan),
                                 dict(target_ema_tau=math.inf), dict(target_ema_tau="0.005"),
                                 dict(target_ema_tau=True)])
def test_target_ema_refusals_name_the_field(bad):
    with pytest.raises(ValueError) as e:
        config.read(_ns(**dict(dict(target_ema=1), **bad)), 18)
    assert list(bad)[0] in str(e.value)


@pytest.mark.parametrize("bad", [dict(adamw=2), dict(adamw=-1), dict(adamw="1"), dict(adamw_weight_decay=-1e-9),
                                 dict(adamw_weight_decay=math.nan), dict(adamw_weight_decay=math.inf),
                                 dict(adamw_weight_decay=1e39), dict(adamw_weight_decay=None),
                                 dict(adamw_weight_decay=False)])
def test_adamw_refusals_name_the_field(bad):
    with pytest.raises(ValueError) as e:
        config.read(_ns(**dict(dict(adamw=1), **bad)), 18)
    assert list(bad)[0] in str(e.value)


@pytest.mark.parametrize("lr,wd,fqf_lr,ok", [(0.5, 1.99, None, True), (0.5, 2.0, None, False), (1.0, 1.0, None, False),
                                             (1e-4, 9999.0, None, True), (1e-4, 1.0001e4, None, False),
                                             (1e-4, 0.1, 2.5e-9, True), (1e-4, 0.1, 10.0, False),
                                             (1e-4, 1e4 * 0.9, 1.2e-4, False), (-1e-4, 0.1, None, False)])
def test_lr_times_decay_below_one(lr, wd, fqf_lr, ok):
    kw = dict(adamw=1, adamw_weight_decay=wd, lr=lr)
    if fqf_lr is not None:
        kw.update(fqf=1, fqf_fraction_lr=fqf_lr)
    if ok:
        d = config.read(_ns(**kw), 18)
        assert 0.0 < F32(1.0 - F32(lr) * d["adamw"]) <= 1.0
    else:
        with pytest.raises(ValueError) as e:
            config.read(_ns(**kw), 18)
        assert "adamw_weight_decay" in str(e.value)
        assert ("fqf_fraction_lr" if fqf_lr is not None and F32(lr) * F32(wd) < 1 else "lr") in str(e.value)
    # with the decay at 0, any lr is accepted
    config.read(_ns(**dict(kw, adamw_weight_decay=0.0)), 18)


@pytest.mark.parametrize("head", HEADS, ids=["iqn", "c51", "qr"])
@pytest.mark.parametrize("loss", LOSSES, ids=lambda v: "-".join(f"{k}={v[k]}" for k in v) or "plain")
def test_both_switches_combine_with_every_head_and_loss(head, loss):
    kw = dict(head, **loss)
    try:
        plain = config.read(_ns(**kw), 18)
    except ValueError:
        pytest.skip("not a combination of heads and losses")
    for extra in (dict(target_ema=1, target_ema_tau=0.01), dict(adamw=1, adamw_weight_decay=0.05),
                  dict(target_ema=1, adamw=1)):
        on = config.read(_ns(**dict(kw, **extra)), 18)
        switched = {k for k in ("target_ema", "adamw") if k in extra}
        assert all(on[k] is not None for k in switched)
        assert {k: v for k, v in on.items() if k not in switched} == {k: v for k, v in plain.items() if k not in switched}


def test_namespace_without_the_fields_reads_as_zero():
    for variant in HEADS + LOSSES[1:]:
        try:
            a = config.read(_ns(**variant), 18)
        except ValueError:
            continue
        b = config.read(_ns(target_ema=0, adamw=0, **variant), 18)
        assert a == b


# ------------------------------------------------------------------------------------------------ the statement
@pytest.mark.parametrize("wd", [0.0, 0.1, 3.0])
def test_oracle_adamw_equals_torch_adamw_in_float64(wd):
    rs = np.random.RandomState(int(wd * 10))
    n, lr, eps = 1000, 1e-3, 1.5e-4
    theta = rs.standard_normal(n)
    p = torch.tensor(theta, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.AdamW([p], lr=lr, eps=eps, weight_decay=wd, foreach=False)
    m = v = np.zeros(n)
    for t in range(1, 6):
        g = rs.standard_normal(n) * (10.0 ** rs.uniform(-4, 1, n))
        p.grad = torch.tensor(g)
        opt.step()
        theta, m, v = bbf.adamw_step_np(theta, g, m, v, t, lr, wd, eps=eps)
        st = opt.state[p]
        np.testing.assert_allclose(p.detach().numpy(), theta, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(st["exp_avg"].numpy(), m, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(st["exp_avg_sq"].numpy(), v, rtol=1e-12, atol=1e-30)


def test_decay_statement_is_torch_adamws_first_operation():
    """torch.optim.AdamW's param.mul_(1 - lr * wd) on a float32 tensor multiplies by the float32 of the double factor:
    bbf.decayed_f32's fl32(theta * d), for the float32 lr and wd riqn_adamw_step receives."""
    rs = np.random.RandomState(3)
    theta = (rs.standard_normal(100000) * 10.0 ** rs.uniform(-5, 3, 100000)).astype(np.float32)
    for lr, wd in ((F32(1e-4), F32(0.1)), (F32(6.25e-5), F32(3.0)), (F32(0.25), F32(2.5))):
        t = torch.from_numpy(theta.copy())
        t.mul_(1.0 - lr * wd)
        assert np.array_equal(t.numpy().view(np.uint32), bbf.decayed_f32(theta, lr, wd).view(np.uint32))
    # the EMA statement is xi + tau (theta - xi), not its mirror
    assert bbf.ema_f32(np.float32([1.0]), np.float32([0.0]), 0.25)[0] == np.float32(0.25)


# ------------------------------------------------------------------------------------------------ state_dict
class _Tiny(ArenaModule):
    NAMES = ("a", "b")

    def __init__(self):
        super().__init__()
        self.a, self.b = nn.Parameter(torch.randn(3, 5)), nn.Parameter(torch.randn(7))
        self._flatten(torch.device("cpu"))


def _adam(**kw):
    m = _Tiny()
    opt = Adam(m.parameters(), **kw)
    opt.module = m               # the parameters' owner is a weak reference
    return opt


def _stepped(opt, seed):
    g = torch.Generator().manual_seed(seed)
    opt._exp_avg.copy_(torch.randn(opt._exp_avg.shape, generator=g))
    opt._exp_avg_sq.copy_(torch.rand(opt._exp_avg.shape, generator=g))
    opt._step = 4 + seed
    return opt


@pytest.mark.parametrize("src_wd,dst_wd", [(0.0, 0.1), (0.1, 0.0), (0.1, 0.2)])
def test_state_dict_round_trips_between_adam_and_adamw(src_wd, dst_wd):
    src = _stepped(_adam(lr=1e-4, eps=1e-6, weight_decay=src_wd), 1)
    sd = src.state_dict()
    assert sd["param_groups"][0]["weight_decay"] == src_wd
    assert set(sd["param_groups"][0]) >= {"lr", "betas", "eps", "weight_decay", "params"}
    assert set(sd["state"][0]) == {"step", "exp_avg", "exp_avg_sq"} and len(sd["state"]) == 2
    dst = _adam(lr=2e-4, eps=1e-6, weight_decay=dst_wd)
    dst.load_state_dict(sd)
    assert dst._step == src._step
    for ps, pd in zip(src._params, dst._params):                        # the moments of every parameter
        assert all(torch.equal(x, y) for x, y in zip(src._views(ps), dst._views(pd)))
    assert dst.param_groups[0]["weight_decay"] == dst_wd             # the update rule stays the constructor's
    assert (dst.decay() is None) == (dst_wd == 0.0)
    if dst_wd:
        assert dst.decay() == F32(1.0 - F32(dst.param_groups[0]["lr"]) * F32(dst_wd))
    # a state saved before weight_decay was a param-group key loads too
    del sd["param_groups"][0]["weight_decay"]
    _adam(weight_decay=dst_wd).load_state_dict(sd)
