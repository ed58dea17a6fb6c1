"""SPR's args fields through config.read (rainbow_iqn_apex_b200/config.py): defaults, domains, refusals, and every
setting of the other switches with spr on and off.  Host-only."""
import itertools
import math
import types

import pytest

from rainbow_iqn_apex_b200 import config

SWITCHES = ("qr_dqn", "rainbow_only", "munchausen", "fqf", "mmd", "hl_gauss", "cql", "dqfd", "value_rescaling", "curl")


def _ns(**kw):
    a = types.SimpleNamespace(rainbow_only=0, num_tau_samples=64, batch_size=32, history_length=4)
    a.__dict__.update(kw)
    return a


def test_defaults_and_values():
    assert config.read(_ns(), 18)["spr"] is None and config.read(_ns(spr=0, spr_steps=99), 18)["spr"] is None
    v = config.read(_ns(spr=1), 18)["spr"]
    assert v == (5, 2.0) and type(v[0]) is int and type(v[1]) is float
    assert config.read(_ns(spr=True, spr_steps=12, spr_coef=0.5), 64)["spr"] == (12, 0.5)
    assert config.read(_ns(spr=1, spr_steps=1, batch_size=4096), 1)["spr"] == (1, 2.0)


@pytest.mark.parametrize("bad", [dict(spr=2), dict(spr=0.5), dict(spr_steps=0), dict(spr_steps=13), dict(spr_steps=2.0),
                                 dict(spr_steps=True), dict(spr_coef=0.0), dict(spr_coef=-1.0), dict(spr_coef=math.nan),
                                 dict(spr_coef=math.inf), dict(spr_coef="2"), dict(curl=1, random_shift=4),
                                 dict(batch_size=4097), dict(batch_size=0), dict(history_length=5, spr_steps=12)])
def test_refusals_name_the_fields(bad):
    with pytest.raises(ValueError) as e:
        config.read(_ns(**dict(dict(spr=1), **bad)), 18)
    assert any(k in str(e.value) for k in list(bad) + ["spr"])


def test_more_than_64_actions_refused():
    config.read(_ns(spr=1), 64)
    with pytest.raises(ValueError, match="spr"):
        config.read(_ns(spr=1), 65)
    config.read(_ns(), 65)                      # without spr the action count is not SPR's concern


def test_spr_combines_with_every_setting_but_curl():
    """Over every setting of the ten switches, a risk measure and random_shift: with spr = 1, read accepts exactly the
    settings it accepts with spr = 0 that leave curl off."""
    n_plain = n_spr = 0
    for bits in itertools.product((0, 1), repeat=len(SWITCHES) + 2):
        kw = dict(zip(SWITCHES, bits[:len(SWITCHES)]))
        kw["random_shift"] = 4 * bits[-2]
        if bits[-1]:
            kw.update(risk_measure="cvar", risk_eta=0.25)
        try:
            config.read(_ns(**kw), 18)
            plain = True
        except ValueError:
            plain = False
        try:
            got = config.read(_ns(spr=1, **kw), 18)
            with_spr = True
        except ValueError:
            with_spr = False
        assert with_spr == (plain and not kw["curl"]), kw
        if with_spr:
            assert got["spr"] == (5, 2.0)
        n_plain += plain
        n_spr += with_spr
    assert n_spr > 0 and n_spr < n_plain
