from .c51 import C51
from .cql import CQL
from .d4pg import D4PG
from .discrete_sac import DiscreteSAC
from .dqn import DQN
from .edac import EDAC
from .group import LearnerGroup
from .iql import IQL
from .redq import REDQ
from .iqn import IQN
from .ppo import PPO
from .qrdqn import QRDQN
from .sac import SAC
from .td3 import DDPG, TD3
from .tqc import TQC
from .trpo import TRPO
from .vpg import VPG

__all__ = ["VPG", "TRPO", "PPO", "DDPG", "D4PG", "TD3", "SAC", "TQC", "CQL", "IQL", "REDQ", "EDAC", "DiscreteSAC", "DQN", "C51", "QRDQN", "IQN", "LearnerGroup"]
