"""Anakin V-MPO with a tanh-Normal actor on H100 -- drop-in for stoix/systems/mpo/ff_vmpo_continuous.py.  The learner is ff_vmpo's;
what differs is the action head (NormalAffineTanhDistributionHead on the env's bounds) and the duals: log_temperature,
log_alpha_mean and log_alpha_stddev, the two KL constraints taken per action dimension with per_dim_constraining
(ff_vmpo_continuous.py:112-215, 437-460)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.mpo.ff_vmpo import build_learner, get_learner_fn  # noqa: F401  (get_learner_fn: the reference's entry point)


def _continuous_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    action_space = env.action_space()   # ff_vmpo_continuous.py:392-395
    config.system.action_dim = int(action_space.shape[-1])
    config.system.action_minimum = float(action_space.minimum)
    config.system.action_maximum = float(action_space.maximum)
    return {"action_dim": config.system.action_dim, "minimum": config.system.action_minimum, "maximum": config.system.action_maximum}


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, networks, optimisers, environment and states (ff_vmpo_continuous.py:384-531)."""
    return build_learner(env, keys, config, _continuous_head_kwargs)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_vmpo_continuous.py:534-677) on the online actor."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2, policy=lambda s: s.params.actor_params.online)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_vmpo_continuous."""
    return anakin.entry_point(cfg, overrides, "default_ff_vmpo_continuous", run_experiment, "V-MPO")


if __name__ == "__main__":
    hydra_entry_point()
