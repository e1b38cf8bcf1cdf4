"""DDPG (baselines/ddpg) on the sm_90a kernels: `from baselines_b200.ddpg import ddpg; ddpg.learn(...)`."""
from . import ddpg  # noqa: F401
from .ddpg import learn  # noqa: F401
