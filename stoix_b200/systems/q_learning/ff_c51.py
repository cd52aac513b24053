"""Anakin C51 on H100 -- drop-in for stoix/systems/q_learning/ff_c51.py: the learner body of ff_dqn with the categorical_double_q_learning loss
(stoix/utils/loss.py; ff_c51.py:159-188) and the DistributionalDiscreteQNetwork head.  Default config: default_ff_c51."""
from __future__ import annotations

from typing import List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.systems import anakin
from stoix_b200.systems.q_learning import ff_dqn as _dqn
from stoix_b200.systems.q_learning.ff_dqn import get_warmup_fn  # noqa: F401  (same warm-up as ff_dqn)

LOSS = "categorical_double_q_learning"


class EvalActorWrapper:
    """The evaluation network (ff_c51.py:271-275): `apply` returns the head's EpsilonGreedy, element [0] of its tuple."""

    def __init__(self, actor: Actor):
        self.actor = actor

    def apply(self, params, x):
        return self.actor.apply(params, x)[0]


def get_learner_fn(env, q_apply_fn, q_update_fn, buffer_fns, config: DictConfig):
    return _dqn.get_learner_fn(env, q_apply_fn, q_update_fn, buffer_fns, config, loss=LOSS)


def learner_setup(env, keys: Tuple[int, int], config: DictConfig):
    learn, eval_q_network, state = _dqn.learner_setup(env, keys, config, loss=LOSS)
    return learn, EvalActorWrapper(eval_q_network), state


def run_experiment(_config: DictConfig) -> float:
    return anakin.run_experiment(_config, learner_setup, net_keys=1, policy=_dqn.online_params)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    return anakin.entry_point(cfg, overrides, "default_ff_c51", run_experiment, "C51")


if __name__ == "__main__":
    hydra_entry_point()
