"""H100-native DQN learner: same public surface as baselines/deepq/__init__.py:1-4."""
from .replay_buffer import ReplayBuffer, PrioritizedReplayBuffer  # noqa: F401
from .build_graph import build_train, build_act  # noqa: F401
from .deepq import learn, load_act, ActWrapper  # noqa: F401


def wrap_atari_dqn(env):
    raise NotImplementedError("atari wrappers are host-side env code (out of scope, SURVEY.md 2 #17)")
