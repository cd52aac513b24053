"""Anakin feed-forward DPO (Discovered Policy Optimisation) with continuous actions on H100 -- drop-in for
stoix/systems/ppo/anakin/ff_dpo_continuous.py.

ff_ppo_continuous with the actor loss dpo_loss (stoix/utils/loss.py:50-65; ff_dpo_continuous.py:160-170): -mean(ratio A - drift),
drift = relu(x1 - alpha tanh(x1 / alpha)) where A >= 0 and relu(x2 - beta tanh(x2 / beta)) where A < 0, x1 = (ratio - 1) A,
x2 = log(ratio) A; no ratio clipping, the raw reward (no reward_scale, :123).  The learner of ff_ppo runs with loss="dpo".
Config default_ff_dpo_continuous (system ppo/ff_dpo: alpha, beta); fp32 only (arch.precision=bf16 raises)."""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.anakin import ff_ppo as _ppo
from stoix_b200.systems.ppo.anakin import ff_ppo_continuous as _cont

LOSS = "dpo"
get_learner_fn = partial(_ppo.get_learner_fn, loss=LOSS)  # ff_dpo_continuous.py:43-316


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, network, optimiser, environment and states (ff_dpo_continuous.py:319-433)."""
    return _ppo.build_learner(env, keys, config, _cont._action_head_kwargs, _cont._uniform_actions, loss=LOSS)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_dpo_continuous.py:436-583)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_dpo_continuous:
    `python -m stoix_b200.systems.ppo.anakin.ff_dpo_continuous arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_dpo_continuous", run_experiment, "PPO")


if __name__ == "__main__":
    hydra_entry_point()
