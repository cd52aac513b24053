"""Evaluator -- the cold-path counterpart of stoix/evaluator.py (get_distribution_act_fn :48,
get_ff_evaluator_fn :87, evaluator_setup :347): roll `num_eval_episodes` episodes in parallel with the
current actor parameters and report per-episode return / length.  Eager host loop over the same CUDA
kernels as training (it runs once per evaluation period, outside the accelerated path)."""
from __future__ import annotations

from typing import Callable, Dict, Tuple

import torch

from . import random as srandom


def get_distribution_act_fn(config, actor_apply: Callable) -> Callable:
    """stoix/evaluator.py:48-72: greedy -> mode of the distribution, else a sample."""

    def act_fn(params, observation, key):
        pi = actor_apply(params, observation)
        return pi.mode() if config.arch.evaluation_greedy else pi.sample(seed=key)

    return act_fn


def get_ff_evaluator_fn(env, act_fn: Callable, config, eval_multiplier: int = 1) -> Callable:
    n_episodes = int(config.arch.num_eval_episodes) * eval_multiplier
    max_steps = int(config.arch.get("max_eval_steps", 2000))

    def evaluator(params, key, running_statistics=None) -> Dict[str, torch.Tensor]:
        """running_statistics: normalise the observations like the learner does (stoix/evaluator.py:114-129)."""
        from .utils.running_statistics import normalize

        keys = srandom.split(key, n_episodes + 1)
        state, ts = env.reset(keys[:n_episodes])
        dev = ts.observation.device
        alive = torch.ones(n_episodes, dtype=torch.bool, device=dev)
        ret = torch.zeros(n_episodes, device=dev)
        length = torch.zeros(n_episodes, dtype=torch.int32, device=dev)
        for step in range(max_steps):
            observation = ts.observation if running_statistics is None else normalize(ts.observation, running_statistics)
            action = act_fn(params, observation, keys[-1] + step)
            state, ts = env.step(state, action)
            ret += ts.reward * alive
            length += alive.to(torch.int32)
            alive &= ~ts.last()
            if step % 50 == 49 and not bool(alive.any().item()):
                break
        return {"episode_return": ret, "episode_length": length}

    return evaluator


def evaluator_setup(eval_env, key_e, eval_act_fn: Callable, config) -> Tuple[Callable, Callable]:
    """stoix/evaluator.py:347-416: the periodic evaluator and the 10x 'absolute metric' evaluator."""
    del key_e
    return get_ff_evaluator_fn(eval_env, eval_act_fn, config), get_ff_evaluator_fn(eval_env, eval_act_fn, config, 10)


def get_rnn_evaluator_fn(env, actor_network, config, eval_multiplier: int = 1) -> Callable:
    """stoix/evaluator.py get_rnn_evaluator_fn: episodes in parallel with the hidden state carried and reset at episode starts."""
    n_episodes = int(config.arch.num_eval_episodes) * eval_multiplier
    max_steps = int(config.arch.get("max_eval_steps", 2000))

    def evaluator(params, key) -> Dict[str, torch.Tensor]:
        keys = srandom.split(key, n_episodes + 1)
        state, ts = env.reset(keys[:n_episodes])
        dev = ts.observation.device
        h = actor_network.rnn.initialize_carry(n_episodes, dev)
        reset = torch.zeros(n_episodes, dtype=torch.bool, device=dev)
        alive = torch.ones(n_episodes, dtype=torch.bool, device=dev)
        ret, length = torch.zeros(n_episodes, device=dev), torch.zeros(n_episodes, dtype=torch.int32, device=dev)
        for step in range(max_steps):
            h, pi = actor_network.apply(params, h, (ts.observation.float()[None], reset[None]))
            action = (pi.mode() if config.arch.evaluation_greedy else pi.sample(seed=keys[-1] + step))[0]
            state, ts = env.step(state, action)
            reset = ts.last()
            ret += ts.reward * alive
            length += alive.to(torch.int32)
            alive &= ~ts.last()
            if step % 50 == 49 and not bool(alive.any().item()):
                break
        return {"episode_return": ret, "episode_length": length}

    return evaluator
