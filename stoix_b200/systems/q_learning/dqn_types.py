"""Transitions of the Q-learning systems -- same fields and order as stoix/systems/q_learning/dqn_types.py."""
from typing import Any, Dict, NamedTuple

import torch

from stoix_b200.systems.sac.sac_types import Transition


class RNNTransition(NamedTuple):
    """dqn_types.py RNNTransition (rec_r2d2): time-major (T, E, ...) rows; hstate is the carry entering the step."""
    obs: torch.Tensor
    action: torch.Tensor
    reward: torch.Tensor
    reset_hidden_state: torch.Tensor
    done: torch.Tensor
    truncated: torch.Tensor
    info: Dict[str, Any]
    hstate: torch.Tensor


__all__ = ["Transition", "RNNTransition"]
