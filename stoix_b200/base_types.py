"""State / transition / output contracts of the Anakin learner.

Same names and field order as stoix/base_types.py (:78-115, :172-197) so code written against the
reference keeps working; leaves are CUDA torch tensors instead of jax arrays.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, Generic, NamedTuple, Optional, TypeVar

import torch

Action = torch.Tensor
Value = torch.Tensor
Done = torch.Tensor
Truncated = torch.Tensor
Observation = torch.Tensor
Parameters = Any
OptStates = Any
State = Any
StoixState = TypeVar("StoixState")


class ActorCriticParams(NamedTuple):
    """stoix/base_types.py:78-82."""

    actor_params: Any
    critic_params: Any


class ActorCriticOptStates(NamedTuple):
    """stoix/base_types.py:85-89."""

    actor_opt_state: Any
    critic_opt_state: Any


class OnPolicyLearnerState(NamedTuple):
    """stoix/base_types.py:108-115."""

    params: Parameters
    opt_states: OptStates
    key: Any
    env_state: Any
    timestep: Any


class RNNOffPolicyLearnerState(NamedTuple):
    """stoix.base_types.RNNOffPolicyLearnerState (rec_r2d2): per update-batch shard lists of buffers, env states, timesteps, the
    done / truncated flags of the last step and the carried hidden states."""
    params: Any
    opt_states: Any
    buffer_state: Any
    key: Any
    env_state: Any
    timestep: Any
    done: Any
    truncated: Any
    hstates: Any


class AnakinExperimentOutput(NamedTuple, Generic[StoixState]):
    """stoix/base_types.py:172-177."""

    learner_state: StoixState
    episode_metrics: Dict[str, torch.Tensor]
    train_metrics: Dict[str, torch.Tensor]


class EvaluationOutput(NamedTuple, Generic[StoixState]):
    learner_state: StoixState
    episode_metrics: Dict[str, torch.Tensor]


LearnerFn = Callable[[StoixState], AnakinExperimentOutput[StoixState]]
ActorApply = Callable[..., Any]
CriticApply = Callable[[Any, Observation], Value]
