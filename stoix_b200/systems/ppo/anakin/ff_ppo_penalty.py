"""Anakin feed-forward KL-penalty PPO on H100 -- drop-in for stoix/systems/ppo/anakin/ff_ppo_penalty.py.

The reference copies ff_ppo.py and changes the actor loss to ppo_penalty_loss (stoix/utils/loss.py:35-47; ff_ppo_penalty.py:137,
150-178): -mean(ratio A) + kl_penalty_coef * mean KL(behaviour || current), no ratio clipping, the behaviour policy being the actor
at the start of the update.  Here the learner of ff_ppo runs with loss="kl_penalty": the rollout keeps every step's logits as the
behaviour policy and the update runs stx_ppo_penalty_minibatch_grads.  Config default_ff_ppo (system.kl_penalty_coef); fp32 only
(arch.precision=bf16 raises)."""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Tuple

from stoix_b200.config import DictConfig
from stoix_b200.envs.base import Environment
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.anakin import ff_ppo as _ppo

LOSS = "kl_penalty"
get_learner_fn = partial(_ppo.get_learner_fn, loss=LOSS)  # ff_ppo_penalty.py:43-320


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, network, optimiser, environment and states (ff_ppo_penalty.py:323-432)."""
    return _ppo.build_learner(env, keys, config, _ppo._discrete_action_head_kwargs, _ppo._uniform_discrete_actions, loss=LOSS)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_ppo_penalty.py:435-582)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_ppo:
    `python -m stoix_b200.systems.ppo.anakin.ff_ppo_penalty arch.total_num_envs=1024 system.kl_penalty_coef=3.0 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_ppo", run_experiment, "PPO")


if __name__ == "__main__":
    hydra_entry_point()
