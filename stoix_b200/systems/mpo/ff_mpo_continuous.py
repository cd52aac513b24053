"""Anakin MPO with a tanh-Normal actor on H100 -- drop-in for stoix/systems/mpo/ff_mpo_continuous.py.  The learner is ff_mpo's; what
differs is the action head (NormalAffineTanhDistributionHead on the env's bounds), the num_samples target-policy draws of the actor loss,
the decoupled loss (continuous_loss.py) and the duals: log_temperature, log_alpha_mean and log_alpha_stddev, per action dimension with
per_dim_constraining."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.mpo.ff_mpo import build_learner, get_learner_fn, get_warmup_fn  # noqa: F401  (the reference's entry points)


def _continuous_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    action_space = env.action_space()
    config.system.action_dim = int(action_space.shape[-1])
    config.system.action_minimum = float(action_space.minimum)
    config.system.action_maximum = float(action_space.maximum)
    return {"action_dim": config.system.action_dim, "minimum": config.system.action_minimum, "maximum": config.system.action_maximum}


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, networks, optimisers, buffer, environment and states (ff_mpo_continuous.py)."""
    return build_learner(env, keys, config, _continuous_head_kwargs)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment on the online actor."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2, policy=lambda s: s.params.actor_params.online)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_mpo_continuous."""
    return anakin.entry_point(cfg, overrides, "default_ff_mpo_continuous", run_experiment, "MPO")


if __name__ == "__main__":
    hydra_entry_point()
