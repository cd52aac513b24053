"""Environment factory -- the `environments.make(config) -> (env, eval_env)` face of
stoix/utils/make_env.py:436-466.  The JAX environment suites of the reference are not installable
here; the two environments the BASELINE configs name are provided natively on the GPU behind the same
interface (stoix_b200/envs/base.py)."""
from __future__ import annotations

from typing import Tuple

import torch

from ..envs.base import Environment


def make(config) -> Tuple[Environment, Environment]:
    name = config.env.env_name
    device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
    if device is None:
        raise RuntimeError("stoix_b200 environments live on the GPU; no CUDA device is visible")
    seed = int(config.arch.seed)
    rank = int(config.get("rank", 0))
    if name == "synthetic":
        from ..envs.synthetic import SyntheticBoxEnv

        kw = dict(config.env.kwargs)
        obs_dtype = torch.bfloat16 if str(config.arch.get("precision", "f32")) == "bf16" else torch.float32
        env = SyntheticBoxEnv(seed=seed + 7919 * rank, device=device, obs_dtype=obs_dtype, **kw)
        eval_env = SyntheticBoxEnv(seed=seed + 104729 + 7919 * rank, device=device, obs_dtype=obs_dtype, **kw)
        return env, eval_env
    if name == "synthetic_continuous":
        from ..envs.synthetic_continuous import SyntheticContinuousEnv

        kw = dict(config.env.kwargs)
        return (SyntheticContinuousEnv(seed=seed + 7919 * rank, device=device, **kw),
                SyntheticContinuousEnv(seed=seed + 104729 + 7919 * rank, device=device, **kw))
    if name == "gymnax":
        scenario = config.env.scenario.name
        if scenario != "CartPole-v1":
            raise NotImplementedError(f"gymnax scenario '{scenario}' is not built (only CartPole-v1)")
        from ..envs.cartpole import CartPoleEnv

        return CartPoleEnv(device=device, seed=seed + 7919 * rank), CartPoleEnv(device=device, seed=seed + 1 + 7919 * rank)
    raise NotImplementedError(f"environment suite '{name}' is outside the hot path of this build")
