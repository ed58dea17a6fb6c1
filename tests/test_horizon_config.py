"""Update-horizon and discount annealing (BBF) on the host: the fields horizon_anneal, horizon_anneal_n,
horizon_anneal_gamma and horizon_anneal_steps through config.read (defaults, domains, refusals, every head and variant),
the schedule of rainbow_iqn_apex_b200/horizon.py against the float64 statement below (horizon_schedule, which
tests/test_gpu_horizon.py also checks the learner against), its restart at a reset, and the layout of
riqn_horizon_state in include/riqn_b200.h against the packing dynstate.HorizonState writes."""
import ctypes
import math
import os
import re
import struct
import types

import numpy as np
import pytest

from rainbow_iqn_apex_b200 import config, dynstate, horizon

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = [dict(), dict(rainbow_only=1), dict(qr_dqn=1), dict(munchausen=1), dict(fqf=1), dict(qr_dqn=1, mmd=1),
            dict(rainbow_only=1, hl_gauss=1), dict(cql=1), dict(qr_dqn=1, cql=1), dict(dqfd=1), dict(qr_dqn=1, dqfd=1),
            dict(value_rescaling=1), dict(rainbow_only=1, value_rescaling=1), dict(random_shift=4),
            dict(curl=1, random_shift=4), dict(spr=1), dict(reset=1), dict(target_ema=1, adamw=1)]


def horizon_schedule(n0, gamma0, steps, n1, gamma1, u):
    """The statement: BBF's update-horizon and discount annealing as this project reads it, in float64 numpy.
    f = clamp((P - u) / P, 0, 1); n = floor(exp(f ln n0 + (1 - f) ln n1) + 0.5) and gamma = 1 - exp(f ln(1 - gamma0) +
    (1 - f) ln(1 - gamma1)), with the end values themselves at f = 1 and f = 0."""
    f = np.clip((np.float64(steps) - np.float64(u)) / np.float64(steps), 0.0, 1.0)
    if f == 0.0:
        return n1, gamma1
    if f == 1.0:
        return n0, gamma0
    n = np.floor(np.exp(f * np.log(np.float64(n0)) + (1.0 - f) * np.log(np.float64(n1))) + 0.5)
    gamma = 1.0 - np.exp(f * np.log(1.0 - np.float64(gamma0)) + (1.0 - f) * np.log(1.0 - np.float64(gamma1)))
    return int(n), float(gamma)


def _ns(**kw):
    a = types.SimpleNamespace(rainbow_only=0, num_tau_samples=64, batch_size=32, history_length=4, multi_step=3,
                              discount=0.997, lr=1e-4)
    a.__dict__.update(kw)
    return a


def test_defaults_and_values():
    assert config.read(_ns(), 18)["horizon_anneal"] is None
    assert config.read(_ns(horizon_anneal=0, horizon_anneal_n=99, discount=1.0), 18)["horizon_anneal"] is None
    v = config.read(_ns(horizon_anneal=1), 18)["horizon_anneal"]
    assert v == (10, 0.97, 10000) and type(v[0]) is int and type(v[1]) is float and type(v[2]) is int
    v = config.read(_ns(horizon_anneal=True, horizon_anneal_n=1, horizon_anneal_gamma=0.5, horizon_anneal_steps=1), 18)
    assert v["horizon_anneal"] == (1, 0.5, 1)
    assert config.read(_ns(horizon_anneal=1, horizon_anneal_gamma=0.99), 18)["horizon_anneal"][1] == 0.99   # a double
    # the window limit: max(n0, multi_step) + history <= 16
    assert config.read(_ns(horizon_anneal=1, horizon_anneal_n=12), 18)["horizon_anneal"][0] == 12
    assert config.read(_ns(horizon_anneal=1, horizon_anneal_n=2, multi_step=12), 18)["horizon_anneal"][0] == 2
    assert config.read(_ns(horizon_anneal=1, horizon_anneal_n=14, history_length=2), 18)["horizon_anneal"][0] == 14


@pytest.mark.parametrize("bad, names", [
    (dict(horizon_anneal=2), ["horizon_anneal"]), (dict(horizon_anneal="1"), ["horizon_anneal"]),
    (dict(horizon_anneal_n=0), ["horizon_anneal_n"]), (dict(horizon_anneal_n=2.0), ["horizon_anneal_n"]),
    (dict(horizon_anneal_n=True), ["horizon_anneal_n"]), (dict(horizon_anneal_n=16), ["horizon_anneal_n"]),
    (dict(horizon_anneal_gamma=0.0), ["horizon_anneal_gamma"]), (dict(horizon_anneal_gamma=1.0), ["horizon_anneal_gamma"]),
    (dict(horizon_anneal_gamma=-0.5), ["horizon_anneal_gamma"]), (dict(horizon_anneal_gamma=math.nan), ["horizon_anneal_gamma"]),
    (dict(horizon_anneal_gamma="0.97"), ["horizon_anneal_gamma"]),
    (dict(horizon_anneal_steps=0), ["horizon_anneal_steps"]), (dict(horizon_anneal_steps=1.5), ["horizon_anneal_steps"]),
    (dict(discount=1.0), ["discount"]), (dict(discount=0.0), ["discount"]), (dict(discount=1.5), ["discount"]),
    (dict(discount=math.nan), ["discount"]), (dict(multi_step=0), ["multi_step"]),
    (dict(horizon_anneal_n=13), ["horizon_anneal_n", "multi_step", "history_length"]),
    (dict(multi_step=13, horizon_anneal_n=3), ["horizon_anneal_n", "multi_step", "history_length"]),
    (dict(history_length=7), ["horizon_anneal_n", "multi_step", "history_length"])])
def test_refusals_name_the_fields(bad, names):
    with pytest.raises(ValueError) as e:
        config.read(_ns(**dict(dict(horizon_anneal=1), **bad)), 18)
    for name in names:
        assert name in str(e.value)


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in v) or "iqn")
def test_anneal_combines_with_every_variant(variant):
    plain = config.read(_ns(**variant), 18)
    on = config.read(_ns(horizon_anneal=1, horizon_anneal_steps=8, **variant), 18)
    assert on["horizon_anneal"] == (10, 0.97, 8)
    assert {k: v for k, v in on.items() if k != "horizon_anneal"} == \
        {k: v for k, v in plain.items() if k != "horizon_anneal"}


CASES = [(10, 0.97, 10000, 3, 0.997), (10, 0.97, 8, 3, 0.997), (3, 0.9, 100, 10, 0.99), (12, 0.5, 7, 1, 0.999),
         (5, 0.99, 3, 5, 0.99), (1, 0.97, 1, 1, 0.997)]


@pytest.mark.parametrize("n0, gamma0, steps, n1, gamma1", CASES)
def test_schedule_against_the_oracle(n0, gamma0, steps, n1, gamma1):
    anneal = (n0, gamma0, steps)
    assert horizon.schedule(anneal, n1, gamma1, 0) == (n0, gamma0)
    for u in (steps, steps + 1, 10 * steps + 3):
        n, g = horizon.schedule(anneal, n1, gamma1, u)
        assert (n, g) == (n1, gamma1) and type(n) is int           # exactly the fixed configuration
    us = sorted(set(np.linspace(0, steps + 2, 200).astype(int).tolist()))
    ns, gs = [], []
    for u in us:
        n, g = horizon.schedule(anneal, n1, gamma1, u)
        want_n, want_g = horizon_schedule(n0, gamma0, steps, n1, gamma1, u)
        assert n == want_n, u
        assert abs(g - want_g) <= 4 * np.spacing(want_g), u
        # the rounding rule: the nearest integer to the log-linear n, halves up
        f = min(max((steps - u) / steps, 0.0), 1.0)
        x = math.exp(f * math.log(n0) + (1 - f) * math.log(n1))
        assert n == math.floor(x + 0.5) and abs(n - x) <= 0.5 + 1e-12
        assert min(n0, n1) <= n <= max(n0, n1) and min(gamma0, gamma1) - 1e-15 <= g <= max(gamma0, gamma1) + 1e-15
        ns.append(n)
        gs.append(g)
    step = 1 if n1 >= n0 else -1                                        # n is monotone from n0 to n1
    assert all((b - a) * step >= 0 for a, b in zip(ns, ns[1:]))
    gstep = 1 if gamma1 >= gamma0 else -1
    assert all((b - a) * gstep >= -1e-15 for a, b in zip(gs, gs[1:]))


def test_bbf_schedule_midpoint():
    """Halfway through BBF's schedule: n = round(sqrt(10 * 3)) = 5, 1 - gamma = sqrt(0.03 * 0.003)."""
    n, g = horizon.schedule((10, 0.97, 10000), 3, 0.997, 5000)
    assert n == 5 and abs((1 - g) - math.sqrt(0.03 * 0.003)) < 1e-15


def test_schedule_restarts_at_a_reset(monkeypatch):
    """Learner's bookkeeping without a device: the schedule runs over the updates since the last reset, scheduled or
    called, and _horizon_at counts a capture's warm-up steps ahead of the updates."""
    from rainbow_iqn_apex_b200 import learner, reset
    monkeypatch.setattr(reset, "reset", lambda agent, index: None)
    lr = object.__new__(learner.Learner)
    lr.__dict__.update(n=3, discount=0.997, horizon_anneal=(10, 0.97, 8), updates=0, resets=0, reset=(5, 0.5),
                       _horizon=object(), _horizon_base=0)
    sched = lambda u: horizon_schedule(10, 0.97, 8, 3, 0.997, u)
    assert lr.horizon() == (10, 0.97)
    lr._count_updates(3)
    assert lr.horizon() == sched(3) and lr._horizon_at(2) == sched(5)
    lr._count_updates(1)
    lr._count_updates(1)                          # the 5th update resets: the schedule starts again
    assert lr.resets == 1 and lr.horizon() == (10, 0.97)
    lr._count_updates(4)
    assert lr.horizon() == sched(4)
    lr.reset_networks()                           # called by hand
    assert lr.resets == 2 and lr.horizon() == (10, 0.97)
    lr._count_updates(20)                         # several intervals in one call: one reset, at its end
    assert lr.updates == 29 and lr.resets == 3 and lr.horizon() == (10, 0.97)
    lr.reset = None
    lr._count_updates(7)
    assert lr.horizon() == sched(7) and lr.horizon() != (3, 0.997)
    lr._count_updates(1)                          # the schedule's end is the fixed configuration
    assert lr.horizon() == (3, 0.997)
    lr._count_updates(100)
    assert lr.horizon() == (3, 0.997)


def test_fixed_learner_horizon_is_the_config():
    from rainbow_iqn_apex_b200 import learner
    lr = object.__new__(learner.Learner)
    lr.__dict__.update(n=3, discount=0.99, horizon_anneal=None, updates=17, _horizon=None, _discounts_fed=False)
    assert lr.horizon() == (3, 0.99) and lr.gamma_n() == float(0.99 ** 3)
    lr.__dict__.update(horizon_anneal=(10, 0.97, 8), _horizon=object(), _horizon_base=13)
    n, g = lr.horizon()
    assert (n, g) == horizon_schedule(10, 0.97, 8, 3, 0.99, 4) and lr.gamma_n() == float(g ** n)
    lr._discounts_fed = True
    assert lr.gamma_n() == 1.0


def _header_struct():
    text = open(os.path.join(ROOT, "include", "riqn_b200.h")).read()
    max_h = int(re.search(r"#define\s+RIQN_MAX_HORIZON\s+(\d+)", text).group(1))
    body = re.search(r"typedef struct riqn_horizon_state \{(.*?)\} riqn_horizon_state;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    ctypes_of = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double}
    fields = []
    for typ, name, count in re.findall(r"(\w+)\s+(\w+)\s*(?:\[(\w+)\])?\s*;", body):
        t = ctypes_of[typ]
        if count:
            t = t * (max_h if count == "RIQN_MAX_HORIZON" else int(count))
        fields.append((name, t))
    return max_h, type("riqn_horizon_state", (ctypes.Structure,), {"_fields_": fields})


def test_header_struct_matches_the_host_packing():
    max_h, S = _header_struct()
    assert max_h == dynstate.MAX_HORIZON
    assert [f[0] for f in S._fields_] == ["n_step", "gamma_n", "gamma_pow"]
    assert ctypes.sizeof(S) == struct.calcsize(dynstate.HORIZON_FMT) == 136
    # the offsets struct.pack_into writes each field at ("<": no padding) are the C layout's
    sizes = [struct.calcsize("<" + c) for c in ("i", "f")]
    assert S.n_step.offset == 0 and S.gamma_n.offset == sizes[0] and S.gamma_pow.offset == sum(sizes)
    assert S.gamma_pow.size == 8 * dynstate.MAX_HORIZON
    raw = bytearray(ctypes.sizeof(S))
    struct.pack_into(dynstate.HORIZON_FMT, raw, 0, 7, ctypes.c_float(0.9 ** 7).value, *[0.9 ** k for k in range(16)])
    s = S.from_buffer(raw)
    assert s.n_step == 7 and s.gamma_n == ctypes.c_float(0.9 ** 7).value and list(s.gamma_pow) == [0.9 ** k for k in range(16)]
