"""Anakin DQN-Reg on H100 -- drop-in for stoix/systems/q_learning/ff_dqn_reg.py: the learner body of ff_dqn with the q_learning_reg loss
(q_learning + regularizer_coeff mean(q_tm1[a]), ff_dqn_reg.py:165-176).  Default config: default_ff_dqn_reg."""
from __future__ import annotations

from typing import List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.systems import anakin
from stoix_b200.systems.q_learning import ff_dqn as _dqn
from stoix_b200.systems.q_learning.ff_dqn import get_warmup_fn  # noqa: F401  (same warm-up as ff_dqn)

LOSS = "q_learning_reg"


def get_learner_fn(env, q_apply_fn, q_update_fn, buffer_fns, config: DictConfig):
    return _dqn.get_learner_fn(env, q_apply_fn, q_update_fn, buffer_fns, config, loss=LOSS)


def learner_setup(env, keys: Tuple[int, int], config: DictConfig):
    return _dqn.learner_setup(env, keys, config, loss=LOSS)


def run_experiment(_config: DictConfig) -> float:
    return anakin.run_experiment(_config, learner_setup, net_keys=1, policy=_dqn.online_params)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    return anakin.entry_point(cfg, overrides, "default_ff_dqn_reg", run_experiment, "DQN-Reg")


if __name__ == "__main__":
    hydra_entry_point()
