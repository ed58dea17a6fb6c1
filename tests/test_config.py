"""The agent's optional args fields (rainbow_iqn_apex_b200/config.py): every field's default and domain through
config.read and config.read_demo, the exact values and Python types the agent stores, and the whole switch matrix of
heads, loss variants, value rescaling, random shift, CURL and a risk measure against the combination table."""
import itertools
import math
import types

import numpy as np
import pytest

from rainbow_iqn_apex_b200 import config

F32 = np.float32
BW_DEFAULT = tuple(float(h) for h in range(1, 11))
BW_WIDE = tuple(float(x) for x in np.logspace(-3, 3, 16).astype(np.float32))
CVAR = dict(risk_measure="cvar", risk_eta=0.25)


def _ns(**kw):
    a = types.SimpleNamespace(rainbow_only=0, num_tau_samples=64, batch_size=32)
    a.__dict__.update(kw)
    return a


def _read(name, action_space=18, **kw):
    return config.read(_ns(**kw), action_space)[name]


def _same(got, want):
    """Equal, and of the same Python types (tuples element by element)."""
    assert got == want and type(got) is type(want), (got, want)
    if isinstance(want, tuple):
        for g, w in zip(got, want):
            _same(g, w)


def _rejects(base, bad, action_space=18):
    for kw in bad:
        with pytest.raises(ValueError):
            config.read(_ns(**dict(base, **kw)), action_space)


def test_munchausen():
    assert _read("munchausen") is None and _read("munchausen", munchausen=False) is None
    assert _read("munchausen", munchausen=0, munchausen_alpha=-1.0, munchausen_tau=0.0, munchausen_l0=1.0) is None
    _same(_read("munchausen", munchausen=1), (0.9, 0.03, -1.0))
    _same(_read("munchausen", munchausen=True, munchausen_alpha=F32(0.5), munchausen_tau=1, munchausen_l0=0),
          (0.5, 1.0, 0.0))
    _same(_read("munchausen", munchausen=np.int64(1), munchausen_alpha=0.0, munchausen_tau=1e-6, munchausen_l0=-0.0),
          (0.0, 1e-6, -0.0))
    bad = [dict(munchausen=2), dict(munchausen=0.5), dict(munchausen="1"), dict(munchausen=None)]
    bad += [dict(munchausen_alpha=v) for v in (-0.1, math.nan, math.inf, 1e39, True, "0.9")]
    bad += [dict(munchausen_tau=v) for v in (0.0, -0.03, 1e-50, math.nan, math.inf)]
    bad += [dict(munchausen_l0=v) for v in (0.1, math.nan, -math.inf, None)]
    bad += [dict(rainbow_only=1), CVAR]
    _rejects(dict(munchausen=1), bad)


def test_value_rescaling():
    assert _read("value_rescaling") is None and _read("value_rescaling", value_rescaling=False) is None
    assert _read("value_rescaling", value_rescaling=0, value_rescaling_eps=-1.0, munchausen=1) is None
    _same(_read("value_rescaling", value_rescaling=1), 1e-3)
    _same(_read("value_rescaling", value_rescaling=True, value_rescaling_eps=0), 0.0)
    _same(_read("value_rescaling", value_rescaling=np.int64(1), value_rescaling_eps=F32(0.01)), float(F32(0.01)))
    bad = [dict(value_rescaling=v) for v in (2, 0.5, "1", None)]
    bad += [dict(value_rescaling_eps=v) for v in (-1e-3, math.nan, math.inf, -math.inf, 1e39, True, "0.001", None)]
    bad += [dict(munchausen=1)]
    _rejects(dict(value_rescaling=1), bad)


def test_qr_dqn():
    assert _read("qr_dqn") is None and _read("qr_dqn", qr_dqn=False) is None
    assert _read("qr_dqn", 99, qr_dqn=0, num_tau_samples=1, rainbow_only=1) is None
    _same(_read("qr_dqn", 18, qr_dqn=1, num_tau_samples=64), 64)
    _same(_read("qr_dqn", 32, qr_dqn=np.int64(1), num_tau_samples=np.int32(2)), 2)
    _same(_read("qr_dqn", 1, qr_dqn=True, num_tau_samples=256), 256)
    assert config.read_head(_ns(qr_dqn=1, num_tau_samples=200), 18) == ("qr", 200)
    assert config.read_head(_ns(rainbow_only=1, num_tau_samples=1), 99) == ("c51", None)
    assert config.read_head(_ns(), 99) == ("iqn", None)
    bad = [dict(qr_dqn=v) for v in (2, 0.5, 1.0, "1", None)]
    bad += [dict(num_tau_samples=v) for v in (1, 257, 64.0, True, None)]
    bad += [dict(rainbow_only=1), dict(munchausen=1), dict(fqf=1), CVAR]
    _rejects(dict(qr_dqn=1), bad)
    for A in (33, 0):
        _rejects(dict(qr_dqn=1), [{}], action_space=A)
        with pytest.raises(ValueError):
            config.read_head(_ns(qr_dqn=1), A)


def test_fqf():
    assert _read("fqf") is None and _read("fqf", fqf=False) is None
    assert _read("fqf", fqf=0, fqf_fraction_lr=-1.0, fqf_entropy_coef=-1.0, rainbow_only=1) is None
    _same(_read("fqf", fqf=1), (2.5e-9, 0.0))
    _same(_read("fqf", fqf=np.int64(1), fqf_fraction_lr=F32(1e-4), fqf_entropy_coef=1, num_tau_samples=256),
          (float(F32(1e-4)), 1.0))
    bad = [dict(fqf=v) for v in (2, 0.5, "1", None)]
    bad += [dict(fqf_fraction_lr=v) for v in (0.0, -1e-9, 1e-50, math.nan, math.inf, 1e39, True, "1e-9")]
    bad += [dict(fqf_entropy_coef=v) for v in (-0.1, math.nan, math.inf, None)]
    bad += [dict(rainbow_only=1), dict(munchausen=1), CVAR]
    bad += [dict(num_tau_samples=v) for v in (1, 257, 8.0)]
    _rejects(dict(fqf=1), bad)


def test_mmd():
    assert config.FIELDS["mmd_bandwidths"][0] == BW_DEFAULT
    assert _read("mmd") is None and _read("mmd", mmd=False) is None
    assert _read("mmd", mmd=0, mmd_bandwidths="x", rainbow_only=1) is None
    _same(_read("mmd", mmd=1, qr_dqn=1), BW_DEFAULT)
    _same(_read("mmd", mmd=True, mmd_bandwidths=[2, 0.5], qr_dqn=1, num_tau_samples=8), (2.0, 0.5))
    _same(_read("mmd", mmd=np.int64(1), mmd_bandwidths=F32([3]), qr_dqn=1, num_tau_samples=2), (3.0,))
    _same(_read("mmd", mmd=1, mmd_bandwidths=BW_WIDE, qr_dqn=1, num_tau_samples=200), BW_WIDE)
    _same(_read("mmd", mmd=1, mmd_bandwidths=(1.0,) * 16, qr_dqn=1, num_tau_samples=2), (1.0,) * 16)
    bad = [dict(mmd=v) for v in (2, -1, 0.5, 1.0, "1", None)]
    bad += [dict(mmd_bandwidths=v) for v in ("1,2", b"12", 3.0, None, (1.0, True), (False,), (1.0, float("nan")),
                                             (float("inf"),), (-float("inf"),), (0.0,), (1.0, -2.0), (1e-50,), (1e-39,),
                                             (1e39,), ("1",), (1.0,) * 17, (), [])]
    bad += [dict(qr_dqn=0), dict(rainbow_only=1), dict(munchausen=1), dict(fqf=1), CVAR]
    _rejects(dict(mmd=1, mmd_bandwidths=BW_DEFAULT, qr_dqn=1), bad)


def test_hl_gauss():
    assert config.FIELDS["hl_gauss_sigma"][0] == 0.75
    assert _read("hl_gauss") is None and _read("hl_gauss", hl_gauss=False) is None
    assert _read("hl_gauss", hl_gauss=0, hl_gauss_sigma="x") is None
    _same(_read("hl_gauss", hl_gauss=1, rainbow_only=1), 0.75)
    _same(_read("hl_gauss", hl_gauss=True, hl_gauss_sigma=2, rainbow_only=True), 2.0)
    _same(_read("hl_gauss", hl_gauss=np.int64(1), hl_gauss_sigma=F32(0.1), rainbow_only=1), float(F32(0.1)))
    _same(_read("hl_gauss", hl_gauss=1, hl_gauss_sigma=0.1, rainbow_only=1), float(F32(0.1)))
    _same(_read("hl_gauss", hl_gauss=1, hl_gauss_sigma=1000, rainbow_only=1), 1000.0)
    assert _read("hl_gauss", hl_gauss=1, hl_gauss_sigma=1e-40, rainbow_only=1) > 0
    _same(_read("hl_gauss", hl_gauss=1, hl_gauss_sigma=1000.00001, rainbow_only=1), 1000.0)     # 1000 as a float32
    bad = [dict(hl_gauss=v) for v in (2, -1, 0.5, 1.0, "1", None)]
    bad += [dict(hl_gauss_sigma=v) for v in (0.0, -0.75, math.nan, math.inf, -math.inf, 1000.001, 1e39, 1e-50, True,
                                             "0.75", None, (0.75,))]
    bad += [dict(rainbow_only=0), dict(rainbow_only=False)]
    _rejects(dict(hl_gauss=1, hl_gauss_sigma=0.75, rainbow_only=1), bad)
    with pytest.raises(ValueError, match="rainbow_only"):
        config.read(_ns(hl_gauss=1, hl_gauss_sigma=0.75), 18)


def test_cql():
    assert config.FIELDS["cql_alpha"][0] == 1.0
    assert _read("cql") is None and _read("cql", cql=False) is None
    assert _read("cql", cql=0, cql_alpha="x", rainbow_only=1) is None
    _same(_read("cql", cql=1), 1.0)
    _same(_read("cql", cql=True, cql_alpha=4), 4.0)
    _same(_read("cql", cql=np.int64(1), cql_alpha=F32(0.1)), float(F32(0.1)))
    _same(_read("cql", cql=1, cql_alpha=0.1), float(F32(0.1)))
    assert _read("cql", cql=1, cql_alpha=1e-40) > 0
    _same(_read("cql", cql=1, cql_alpha=3e38), float(F32(3e38)))
    bad = [dict(cql=v) for v in (2, -1, 0.5, 1.0, "1", None)]
    bad += [dict(cql_alpha=v) for v in (0.0, -1.0, math.nan, math.inf, -math.inf, 1e39, 1e-50, True, "1", None, (1.0,))]
    bad += [dict(rainbow_only=1), dict(rainbow_only=True), dict(munchausen=1), dict(fqf=1), dict(mmd=1, qr_dqn=1)]
    _rejects(dict(cql=1, cql_alpha=1.0), bad)


def test_dqfd():
    assert {f: config.FIELDS[f][0] for f in ("dqfd_margin", "dqfd_lambda")} == {"dqfd_margin": 0.8, "dqfd_lambda": 1.0}
    assert _read("dqfd") is None and _read("dqfd", dqfd=False) is None
    assert _read("dqfd", dqfd=0, dqfd_margin="x", dqfd_lambda=None, rainbow_only=1) is None
    _same(_read("dqfd", dqfd=1), (float(F32(0.8)), 1.0))
    _same(_read("dqfd", dqfd=True, dqfd_margin=2, dqfd_lambda=4), (2.0, 4.0))
    _same(_read("dqfd", dqfd=np.int64(1), dqfd_margin=F32(0.1), dqfd_lambda=1e-40)[0], float(F32(0.1)))
    _same(_read("dqfd", dqfd=1, dqfd_margin=3e38, dqfd_lambda=3e38), (float(F32(3e38)),) * 2)
    bad = [dict(dqfd=v) for v in (2, -1, 0.5, 1.0, "1", None)]
    for name in ("dqfd_margin", "dqfd_lambda"):
        bad += [{name: v} for v in (0.0, -1.0, math.nan, math.inf, -math.inf, 1e39, 1e-50, True, "1", None, (1.0,))]
    bad += [dict(rainbow_only=1), dict(rainbow_only=True), dict(munchausen=1), dict(fqf=1), dict(mmd=1, qr_dqn=1),
            dict(cql=1)]
    _rejects(dict(dqfd=1, dqfd_margin=0.8, dqfd_lambda=1.0), bad)


def test_demo_replay():
    assert {f: config.FIELDS[f][0] for f in ("demo_segments", "demo_priority_bonus")} == \
        {"demo_segments": 0, "demo_priority_bonus": 0.0}

    def demo(nb, **kw):
        return config.read_demo(types.SimpleNamespace(nb_actor=nb, **kw))

    for nb in (1, 2, 7):
        _same(demo(nb), (0, 0.0))
        for d in range(nb + 1):
            _same(demo(nb, demo_segments=d, demo_priority_bonus=0.0), (d, 0.0))
            _same(demo(nb, demo_segments=np.int64(d), demo_priority_bonus=F32(1e-3)), (d, float(F32(1e-3))))
        for d in (-1, nb + 1, 1.0, 0.5, True, "1", None):
            with pytest.raises(ValueError):
                demo(nb, demo_segments=d, demo_priority_bonus=0.0)
    _same(demo(1, demo_segments=1, demo_priority_bonus=3e38)[1], float(F32(3e38)))
    _same(demo(1, demo_segments=1, demo_priority_bonus=1e-50)[1], 0.0)
    for v in (-1e-3, -1.0, math.nan, math.inf, -math.inf, 1e39, True, "1", None, (1.0,)):
        with pytest.raises(ValueError):
            demo(2, demo_segments=1, demo_priority_bonus=v)


def test_curl():
    assert {f: config.FIELDS[f][0] for f in ("curl_coef", "curl_momentum")} == {"curl_coef": 1.0, "curl_momentum": 0.001}
    assert _read("curl") is None and _read("curl", curl=False) is None
    _same(_read("curl", curl=1, random_shift=4, batch_size=32), (1.0, float(F32(0.001))))
    _same(_read("curl", curl=True, curl_coef=0.5, curl_momentum=1, random_shift=1, batch_size=2), (0.5, 1.0))
    bad = [dict(curl=v) for v in (2, 1.0, -1, "1")]
    bad += [dict(curl_coef=v) for v in (0.0, -1.0, float("nan"), float("inf"), 1e39, True, 1e-46)]
    bad += [dict(curl_momentum=v) for v in (0.0, 1.5, float("nan"), -0.1, False)]
    bad += [dict(random_shift=0), dict(batch_size=1), dict(batch_size=0), dict(batch_size=4097), dict(batch_size=2.0)]
    _rejects(dict(curl=1, curl_coef=1.0, curl_momentum=0.001, random_shift=4, batch_size=32), bad)


def test_random_shift():
    assert _read("random_shift") is None and _read("random_shift", random_shift=0) is None
    _same(_read("random_shift", random_shift=4), 4)
    _same(_read("random_shift", random_shift=np.int64(83)), 83)
    _same(_read("random_shift", random_shift=np.int32(1)), 1)
    _rejects({}, [dict(random_shift=v) for v in (True, False, 1.5, 4.0, -1, 84, float("nan"), "4", None)])


def test_risk():
    assert _read("risk") is None and _read("risk", risk_measure="neutral", risk_eta=None) is None
    assert _read("risk", **CVAR) == ("cvar", 0.25) and _read("risk", risk_measure="CPW", risk_eta=0.71) == ("cpw", 0.71)
    assert config.read_risk("qr", None, "neutral") is None and config.read_risk("iqn", "cql", "wang", -0.75) == ("wang", -0.75)
    for head, loss in (("c51", None), ("c51", "hl_gauss"), ("qr", None), ("qr", "cql"), ("iqn", "munchausen"),
                       ("iqn", "fqf")):
        with pytest.raises(ValueError):
            config.read_risk(head, loss, "wang", -0.75)
    _rejects({}, [dict(risk_measure="cvar", risk_eta=1.5), dict(risk_measure="mean-variance", risk_eta=0.5)])


# The combination table, written out: at most one loss variant, each on the heads that take it; a non-neutral risk
# measure on the IQN head with no loss variant, CQL or DQfD; value rescaling with every loss but Munchausen; CURL with
# random shift
TABLE = {"iqn": (None, "munchausen", "fqf", "cql", "dqfd"), "qr": (None, "cql", "dqfd", "mmd"), "c51": (None, "hl_gauss")}
RISK = (None, "cql", "dqfd")
LOSSES = ("munchausen", "fqf", "mmd", "hl_gauss", "cql", "dqfd")
SWITCHES = ("rainbow_only", "qr_dqn") + LOSSES + ("value_rescaling", "random_shift", "curl", "risk")


def _allowed(s):
    if s["rainbow_only"] and s["qr_dqn"]:
        return False
    head = "c51" if s["rainbow_only"] else "qr" if s["qr_dqn"] else "iqn"
    on = [name for name in LOSSES if s[name]]
    if len(on) > 1:
        return False
    loss = on[0] if on else None
    return (loss in TABLE[head] and not (s["risk"] and (head != "iqn" or loss not in RISK))
            and not (s["value_rescaling"] and loss == "munchausen") and not (s["curl"] and not s["random_shift"]))


def test_switch_matrix():
    """All 2^12 settings of the twelve switches (risk as CVaR(0.25), random_shift = 4, N = 64, 18 actions, batch 32):
    read accepts exactly the 81 the table allows."""
    accepted = 0
    for bits in itertools.product((0, 1), repeat=len(SWITCHES)):
        s = dict(zip(SWITCHES, bits))
        kw = {k: v for k, v in s.items() if k not in ("random_shift", "risk")}
        kw["random_shift"] = 4 * s["random_shift"]
        if s["risk"]:
            kw.update(CVAR)
        try:
            v = config.read(_ns(**kw), 18)
        except ValueError:
            assert not _allowed(s), s
            continue
        assert _allowed(s), s
        accepted += 1
        assert v["head"] == ("c51" if s["rainbow_only"] else "qr" if s["qr_dqn"] else "iqn")
        assert v["loss"] == next((name for name in LOSSES if s[name]), None)
        for name in LOSSES + ("value_rescaling", "curl"):
            assert (v[name] is not None) == bool(s[name]), (s, name)
        assert v["qr_dqn"] == (64 if s["qr_dqn"] else None) and v["random_shift"] == (4 if s["random_shift"] else None)
        assert v["risk"] == (("cvar", 0.25) if s["risk"] else None)
    assert accepted == 81
