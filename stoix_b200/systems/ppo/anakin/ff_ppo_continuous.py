"""Anakin feed-forward PPO with continuous actions on H100 -- drop-in for stoix/systems/ppo/anakin/ff_ppo_continuous.py.

The reference copies ff_ppo.py and changes the action head; here the learner of ff_ppo serves both heads: a
NormalAffineTanhDistributionHead actor gets a (T, E, A) float action buffer, the tanh-Normal sampler followed by
stx_tanh_normal_log_prob in the rollout, stx_ppo_continuous_minibatch_grads in the update (log_prob of the stored action, the
clipped surrogate and the seeded entropy estimate, ff_ppo_continuous.py:191-213), and a device-resident entropy RNG counter.
This module holds what differs: the action space read in learner_setup (ff_ppo_continuous.py:417-432), the uniform actions of
the observation-normalisation warm-up (:374-380) and the entry config.  fp32 only (arch.precision=bf16 raises)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import torch

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.anakin import ff_ppo as _ppo
from stoix_b200.systems.ppo.anakin.ff_ppo import get_learner_fn  # noqa: F401  (the shared learner, ff_ppo_continuous.py:49-370)


def _action_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    """Get the action dimension and bounds (ff_ppo_continuous.py:417-420) for the head (:426-431)."""
    space = env.action_space()
    config.system.action_dim = int(space.shape[-1])
    config.system.action_minimum = float(space.minimum)
    config.system.action_maximum = float(space.maximum)
    return {"action_dim": config.system.action_dim, "minimum": config.system.action_minimum, "maximum": config.system.action_maximum}


def _uniform_actions(config: DictConfig, E: int, gen: torch.Generator, dev) -> torch.Tensor:
    """Warm-up actions uniform in [action_minimum, action_maximum] (ff_ppo_continuous.py:374-380)."""
    lo, hi = float(config.system.action_minimum), float(config.system.action_maximum)
    return lo + (hi - lo) * torch.rand(E, int(config.system.action_dim), device=dev, generator=gen)


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, network, optimiser, environment and states (ff_ppo_continuous.py:413-545)."""
    return _ppo.build_learner(env, keys, config, _action_head_kwargs, _uniform_actions)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_ppo_continuous.py:548-700)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_ppo_continuous:
    `python -m stoix_b200.systems.ppo.anakin.ff_ppo_continuous arch.total_num_envs=1024 system.rollout_length=32 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_ppo_continuous", run_experiment, "PPO")


if __name__ == "__main__":
    hydra_entry_point()
