"""rainbow_iqn_apex_b200 -- H100-native (sm_90a) learner hot path of Rainbow-IQN Ape-X.

Same class surface as the reference package ``rainbowiqn`` for this path (SURVEY.md section 8b):
``Agent`` / ``Learner`` / ``Actor``, ``DQN`` / ``NoisyLinear``, ``ReplayMemory`` (= ReplayRedisMemory).
All arithmetic runs in hand-written CUDA kernels behind the C-ABI of include/riqn_b200.h; importing this
package never falls back to PyTorch or the CPU -- without the built library or an H100 it raises.
"""
from . import _lib  # noqa: F401
from .model import DQN, NoisyLinear  # noqa: F401
from .optim import Adam  # noqa: F401
from .agent import Agent  # noqa: F401
from .learner import Learner  # noqa: F401
from .actor import Actor  # noqa: F401
from .replay_memory import ReplayMemory, ReplayRedisMemory, SegmentTree, RedisSegmentTree  # noqa: F401

__all__ = ["DQN", "NoisyLinear", "Adam", "Agent", "Learner", "Actor", "ReplayMemory", "ReplayRedisMemory",
           "SegmentTree", "RedisSegmentTree"]
