"""The periodic-reset fields reset, reset_interval and reset_shrink through config.read (rainbow_iqn_apex_b200/config.py):
defaults, refusals, and reset = 1 with every head and every loss and auxiliary variant.  Host-only."""
import math
import types

import pytest

from rainbow_iqn_apex_b200 import config

VARIANTS = [dict(), dict(rainbow_only=1), dict(qr_dqn=1), dict(munchausen=1), dict(fqf=1), dict(qr_dqn=1, mmd=1),
            dict(rainbow_only=1, hl_gauss=1), dict(cql=1), dict(qr_dqn=1, cql=1), dict(dqfd=1), dict(qr_dqn=1, dqfd=1),
            dict(value_rescaling=1), dict(rainbow_only=1, value_rescaling=1), dict(random_shift=4),
            dict(curl=1, random_shift=4), dict(spr=1), dict(spr=1, random_shift=4, rainbow_only=1),
            dict(risk_measure="cvar", risk_eta=0.25)]


def _ns(**kw):
    a = types.SimpleNamespace(rainbow_only=0, num_tau_samples=64, batch_size=32, history_length=4)
    a.__dict__.update(kw)
    return a


def test_defaults_and_values():
    assert config.read(_ns(), 18)["reset"] is None
    assert config.read(_ns(reset=0, reset_interval=0, reset_shrink=7), 18)["reset"] is None   # off: not read
    v = config.read(_ns(reset=1), 18)["reset"]
    assert v == (40000, 0.5) and type(v[0]) is int and type(v[1]) is float
    assert config.read(_ns(reset=True, reset_interval=1, reset_shrink=0), 18)["reset"] == (1, 0.0)
    assert config.read(_ns(reset=1, reset_interval=10 ** 12, reset_shrink=1), 18)["reset"] == (10 ** 12, 1.0)
    v = config.read(_ns(reset=1, reset_shrink=0.8), 18)["reset"][1]
    assert v == 0.800000011920929                # the float32 the kernel receives


@pytest.mark.parametrize("bad", [dict(reset=2), dict(reset=0.5), dict(reset="1"), dict(reset=None),
                                 dict(reset_interval=0), dict(reset_interval=-1), dict(reset_interval=1.5),
                                 dict(reset_interval=True), dict(reset_shrink=-0.1), dict(reset_shrink=1.5),
                                 dict(reset_shrink=math.nan), dict(reset_shrink=math.inf), dict(reset_shrink="0.5")])
def test_refusals_name_the_field(bad):
    with pytest.raises(ValueError) as e:
        config.read(_ns(**dict(dict(reset=1), **bad)), 18)
    assert list(bad)[0] in str(e.value)


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "-".join(f"{k}={v[k]}" for k in v) or "iqn")
def test_reset_combines_with_every_variant(variant):
    plain = config.read(_ns(**variant), 18)
    on = config.read(_ns(reset=1, reset_interval=3, reset_shrink=0.25, **variant), 18)
    assert on["reset"] == (3, 0.25)
    assert {k: v for k, v in on.items() if k != "reset"} == {k: v for k, v in plain.items() if k != "reset"}
