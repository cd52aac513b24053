"""stoix/systems/impala/impala_types.py: the transition the IMPALA actors deliver (no value: the actors sample from the actor alone)."""
from __future__ import annotations

from typing import NamedTuple

import torch


class ImpalaTransition(NamedTuple):
    done: torch.Tensor
    truncated: torch.Tensor
    action: torch.Tensor
    reward: torch.Tensor
    log_prob: torch.Tensor
    obs: torch.Tensor
