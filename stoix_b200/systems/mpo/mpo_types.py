"""MPO and V-MPO state and parameter containers -- same fields and order as stoix/systems/mpo/mpo_types.py:13-73; OnlineAndTarget as
stoix/base_types.py."""
from typing import Any, Dict, NamedTuple

import torch

from stoix_b200.systems.sac.sac_types import OnlineAndTarget  # noqa: F401  (re-exported: VMPOParams.actor_params)


class SequenceStep(NamedTuple):
    obs: torch.Tensor
    action: torch.Tensor
    reward: torch.Tensor
    done: torch.Tensor
    truncated: torch.Tensor
    log_prob: torch.Tensor
    info: Dict


class DualParams(NamedTuple):
    log_temperature: torch.Tensor
    log_alpha_mean: torch.Tensor
    log_alpha_stddev: torch.Tensor


class CategoricalDualParams(NamedTuple):
    log_temperature: torch.Tensor
    log_alpha: torch.Tensor


class VMPOParams(NamedTuple):
    actor_params: OnlineAndTarget
    critic_params: Any
    dual_params: Any


class VMPOOptStates(NamedTuple):
    actor_opt_state: Any
    critic_opt_state: Any
    dual_opt_state: Any


class VMPOLearnerState(NamedTuple):
    params: VMPOParams
    opt_states: VMPOOptStates
    key: Any
    env_state: Any
    timestep: Any
    learner_step_count: torch.Tensor   # int32 (1) on the device: the actor segment's Adam count


class MPOParams(NamedTuple):
    actor_params: OnlineAndTarget
    q_params: OnlineAndTarget
    dual_params: Any


class MPOOptStates(NamedTuple):
    actor_opt_state: Any
    q_opt_state: Any
    dual_opt_state: Any


class MPOLearnerState(NamedTuple):
    params: MPOParams
    opt_states: MPOOptStates
    buffer_state: Any   # one SequenceBuffer per update-batch shard
    key: Any
    env_state: Any
    timestep: Any
