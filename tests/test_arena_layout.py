"""CPU: the arena layouts (arena.layout, arena.ArenaModule) of the DQN's parameter and epsilon arenas and of the side
networks' arenas, as seeded constructions on the CPU lay them out.  Checkpointed Adam moments, the reset segment tables
and the device kernels index these arenas by offset, so neither an offset nor a length may move: every value below was
recorded from the layout code each module had before they shared one."""
import hashlib

import pytest
import torch

from helpers import make_args

# per module: arena lengths, (name, _riqn_offset, numel) of every parameter in named_parameters() order, the epsilon
# buffers' offsets in the DQN's epsilon arena, and the sha256 of the parameter arena's bytes after torch.manual_seed(0)
LAYOUTS = {
    "iqn": dict(
        flat=6726016, eps=3222099, sha256="529f13770f75a0275c4f9faaad1ef8efe3d020add3954328e7efeaa1b16d3ce6",
        params=[
            ("conv1.weight", 0, 8192), ("conv1.bias", 8192, 32), ("conv2.weight", 8256, 32768),
            ("conv2.bias", 41024, 64), ("conv3.weight", 41088, 36864), ("conv3.bias", 77952, 64),
            ("iqn_fc.weight", 78016, 200704), ("iqn_fc.bias", 278720, 3136), ("fcnoisy_h_v.weight_mu", 281856, 1605632),
            ("fcnoisy_h_v.weight_sigma", 3493120, 1605632), ("fcnoisy_h_v.bias_mu", 6704384, 512),
            ("fcnoisy_h_v.bias_sigma", 6705408, 512), ("fcnoisy_h_a.weight_mu", 1887488, 1605632),
            ("fcnoisy_h_a.weight_sigma", 5098752, 1605632), ("fcnoisy_h_a.bias_mu", 6704896, 512),
            ("fcnoisy_h_a.bias_sigma", 6705920, 512), ("fcnoisy_z_v.weight_mu", 6706432, 512),
            ("fcnoisy_z_v.weight_sigma", 6716160, 512), ("fcnoisy_z_v.bias_mu", 6725888, 1),
            ("fcnoisy_z_v.bias_sigma", 6725952, 1), ("fcnoisy_z_a.weight_mu", 6706944, 9216),
            ("fcnoisy_z_a.weight_sigma", 6716672, 9216), ("fcnoisy_z_a.bias_mu", 6725889, 18),
            ("fcnoisy_z_a.bias_sigma", 6725953, 18),
        ],
        eps_offsets=[
            ("fcnoisy_h_v.weight_epsilon", 0), ("fcnoisy_h_v.bias_epsilon", 3211264),
            ("fcnoisy_h_a.weight_epsilon", 1605632), ("fcnoisy_h_a.bias_epsilon", 3211776),
            ("fcnoisy_z_v.weight_epsilon", 3212288), ("fcnoisy_z_v.bias_epsilon", 3222016),
            ("fcnoisy_z_a.weight_epsilon", 3212800), ("fcnoisy_z_a.bias_epsilon", 3222017),
        ],
    ),
    "c51": dict(
        flat=7496896, eps=3709449, sha256="f101e878aea1c197d305eb280503a5f3cef491ff04b600c81a563920001580f5",
        params=[
            ("conv1.weight", 0, 8192), ("conv1.bias", 8192, 32), ("conv2.weight", 8256, 32768),
            ("conv2.bias", 41024, 64), ("conv3.weight", 41088, 36864), ("conv3.bias", 77952, 64),
            ("fcnoisy_h_v.weight_mu", 78016, 1605632), ("fcnoisy_h_v.weight_sigma", 3289280, 1605632),
            ("fcnoisy_h_v.bias_mu", 6500544, 512), ("fcnoisy_h_v.bias_sigma", 6501568, 512),
            ("fcnoisy_h_a.weight_mu", 1683648, 1605632), ("fcnoisy_h_a.weight_sigma", 4894912, 1605632),
            ("fcnoisy_h_a.bias_mu", 6501056, 512), ("fcnoisy_h_a.bias_sigma", 6502080, 512),
            ("fcnoisy_z_v.weight_mu", 6502592, 26112), ("fcnoisy_z_v.weight_sigma", 6998720, 26112),
            ("fcnoisy_z_v.bias_mu", 7494848, 51), ("fcnoisy_z_v.bias_sigma", 7495872, 51),
            ("fcnoisy_z_a.weight_mu", 6528704, 470016), ("fcnoisy_z_a.weight_sigma", 7024832, 470016),
            ("fcnoisy_z_a.bias_mu", 7494899, 918), ("fcnoisy_z_a.bias_sigma", 7495923, 918),
        ],
        eps_offsets=[
            ("fcnoisy_h_v.weight_epsilon", 0), ("fcnoisy_h_v.bias_epsilon", 3211264),
            ("fcnoisy_h_a.weight_epsilon", 1605632), ("fcnoisy_h_a.bias_epsilon", 3211776),
            ("fcnoisy_z_v.weight_epsilon", 3212288), ("fcnoisy_z_v.bias_epsilon", 3708416),
            ("fcnoisy_z_a.weight_epsilon", 3238400), ("fcnoisy_z_a.bias_epsilon", 3708467),
        ],
    ),
    "qr": dict(
        flat=7750208, eps=3836160, sha256="ffeb0afe7ca77c4c61c24b67355fd55364a947951ed1544825ed3d7f44a812a8",
        params=[
            ("conv1.weight", 0, 8192), ("conv1.bias", 8192, 32), ("conv2.weight", 8256, 32768),
            ("conv2.bias", 41024, 64), ("conv3.weight", 41088, 36864), ("conv3.bias", 77952, 64),
            ("fcnoisy_h_v.weight_mu", 78016, 1605632), ("fcnoisy_h_v.weight_sigma", 3289280, 1605632),
            ("fcnoisy_h_v.bias_mu", 6500544, 512), ("fcnoisy_h_v.bias_sigma", 6501568, 512),
            ("fcnoisy_h_a.weight_mu", 1683648, 1605632), ("fcnoisy_h_a.weight_sigma", 4894912, 1605632),
            ("fcnoisy_h_a.bias_mu", 6501056, 512), ("fcnoisy_h_a.bias_sigma", 6502080, 512),
            ("fcnoisy_z_v.weight_mu", 6502592, 32768), ("fcnoisy_z_v.weight_sigma", 7125184, 32768),
            ("fcnoisy_z_v.bias_mu", 7747776, 64), ("fcnoisy_z_v.bias_sigma", 7748992, 64),
            ("fcnoisy_z_a.weight_mu", 6535360, 589824), ("fcnoisy_z_a.weight_sigma", 7157952, 589824),
            ("fcnoisy_z_a.bias_mu", 7747840, 1152), ("fcnoisy_z_a.bias_sigma", 7749056, 1152),
        ],
        eps_offsets=[
            ("fcnoisy_h_v.weight_epsilon", 0), ("fcnoisy_h_v.bias_epsilon", 3211264),
            ("fcnoisy_h_a.weight_epsilon", 1605632), ("fcnoisy_h_a.bias_epsilon", 3211776),
            ("fcnoisy_z_v.weight_epsilon", 3212288), ("fcnoisy_z_v.bias_epsilon", 3834880),
            ("fcnoisy_z_a.weight_epsilon", 3245056), ("fcnoisy_z_a.bias_epsilon", 3834944),
        ],
    ),
    "fqf": dict(
        flat=200768, sha256="c377aeab3706428bfe20ed80b1929d4f47f7e064b30e594838533b2b093c0416",
        params=[
            ("weight", 0, 200704), ("bias", 200704, 64),
        ],
    ),
    "curl": dict(
        flat=1688192, proj_numel=1671808, sha256="c4d5282ded3b3c4624c5114dfae1e6a3bddd0e39f4ab2a8809a00e635b88cb5a",
        params=[
            ("weight_h", 0, 1605632), ("bias_h", 1605632, 512), ("weight_c", 1606144, 65536), ("bias_c", 1671680, 128),
            ("bilinear", 1671808, 16384),
        ],
    ),
    "spr": dict(
        flat=1772544, proj_numel=1671808, sha256="645c9beacc2c8cb8203bdf3452719bd1e6d8d42ac1fb045ed39db2eb0cf64ef6",
        params=[
            ("weight_h", 0, 1605632), ("bias_h", 1605632, 512), ("weight_c", 1606144, 65536), ("bias_c", 1671680, 128),
            ("weight_q", 1756032, 16384), ("bias_q", 1772416, 128), ("conv1.weight", 1671808, 47232),
            ("conv1.bias", 1719040, 64), ("conv2.weight", 1719104, 36864), ("conv2.bias", 1755968, 64),
        ],
    ),
}


def _build(kind):
    from rainbow_iqn_apex_b200.curl import CurlProjection
    from rainbow_iqn_apex_b200.fqf import FractionProposal
    from rainbow_iqn_apex_b200.model import DQN
    from rainbow_iqn_apex_b200.spr import SprNet
    torch.manual_seed(0)
    if kind == "fqf":
        return FractionProposal(64, "cpu")
    if kind == "curl":
        return CurlProjection("cpu")
    if kind == "spr":
        return SprNet(18, "cpu")
    args = make_args(torch.device("cpu"), rainbow_only=kind == "c51")
    if kind == "qr":
        args.qr_dqn = 1
    return DQN(args, 18)


@pytest.mark.parametrize("kind", list(LAYOUTS))
def test_arena_layout_is_pinned(kind):
    want, m = LAYOUTS[kind], _build(kind)
    assert m._flat.numel() == m._flat_grad.numel() == want["flat"]
    assert [(n, p._riqn_offset, p.numel()) for n, p in m.named_parameters()] == want["params"]
    for p in m.parameters():                # every parameter and its gradient are views of the arenas at that offset
        assert p.data_ptr() == m._flat.data_ptr() + 4 * p._riqn_offset
        assert p.grad.data_ptr() == m._flat_grad.data_ptr() + 4 * p._riqn_offset
    assert hashlib.sha256(m._flat.numpy().tobytes()).hexdigest() == want["sha256"]
    if "eps" in want:
        assert m._eps_flat.numel() == want["eps"]
        got = [(n, (b.data_ptr() - m._eps_flat.data_ptr()) // 4) for n, b in m.named_buffers() if "epsilon" in n]
        assert got == want["eps_offsets"]
    if "proj_numel" in want:
        assert m.proj_numel == want["proj_numel"]
