"""Anakin feed-forward KL-penalty PPO with continuous actions on H100 -- drop-in for
stoix/systems/ppo/anakin/ff_ppo_penalty_continuous.py.

ff_ppo_penalty's actor loss (ppo_penalty_loss, ff_ppo_penalty_continuous.py:137,150-179) on the tanh-Normal head of
ff_ppo_continuous: the KL of two tanh-Normals sharing the affine-tanh bijector is the KL of their base Normals, and the entropy is
the seeded one-sample estimate with ff_ppo_continuous's noise stream.  The learner of ff_ppo runs with loss="kl_penalty"; the
rollout keeps every step's loc | scale pre-activation as the behaviour policy.  Config default_ff_ppo_continuous; fp32 only."""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.anakin import ff_ppo as _ppo
from stoix_b200.systems.ppo.anakin import ff_ppo_continuous as _cont

LOSS = "kl_penalty"
get_learner_fn = partial(_ppo.get_learner_fn, loss=LOSS)  # ff_ppo_penalty_continuous.py:43-325


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, network, optimiser, environment and states (ff_ppo_penalty_continuous.py:328-442)."""
    return _ppo.build_learner(env, keys, config, _cont._action_head_kwargs, _cont._uniform_actions, loss=LOSS)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_ppo_penalty_continuous.py:445-592)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_ppo_continuous:
    `python -m stoix_b200.systems.ppo.anakin.ff_ppo_penalty_continuous arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_ppo_continuous", run_experiment, "PPO")


if __name__ == "__main__":
    hydra_entry_point()
