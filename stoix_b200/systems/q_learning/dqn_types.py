"""Transition of the Q-learning systems -- same fields and order as stoix/systems/q_learning/dqn_types.py:9-15."""
from stoix_b200.systems.sac.sac_types import Transition

__all__ = ["Transition"]
