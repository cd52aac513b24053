"""Sebulba feed-forward IMPALA on H100 -- drop-in for stoix/systems/impala/sebulba/ff_impala.py (MLP torso).

Same entry points (get_act_fn :107, get_rollout_fn :128, get_actor_thread :318, get_learner_step_fn :358, learner_setup :718,
run_experiment :809, hydra_entry_point :1039) and the same threads as Sebulba PPO, whose actor side, learner loop, evaluator and wiring this module runs
(stoix_b200/systems/ppo/sebulba/ff_ppo.py).  What is IMPALA's:

  reference (JAX)                                     here (H100)
  --------------------------------------------------  -------------------------------------------------------------
  act_fn: actor only, sample + log_prob               the inference server with ImpalaTransition storage: no critic launch
  hstack shards, reward mean / std over (T, E)        column blocks of one (T+1, E) buffer; stx_reward_stats, once per update
  minibatches = contiguous env-column blocks, in      per block: actor forward on T*Em rows and critic forward on (T+1)*Em rows
  order, one epoch; jax.grad of the summed V-trace    through int32 row tables built once, stx_vtrace_loss_grads (V-trace, both
  critic loss and the summed policy-gradient +        losses, head gradients, metrics: one launch), both backwards, one
  entropy actor loss                                  clip + RMSProp launch over [actor | critic]
  chain(clip_by_global_norm(40), rmsprop(lr))         stx_clip_rmsprop_step (the RMSProp rule of the fused clip + Adam kernel)

Quirk kept from the reference: d_t = gamma (1 - done) with done = timestep.last(), so truncation ends the V-trace like termination.
fp32 only (arch.precision=bf16 raises) and ONE learner device, as Sebulba PPO.
"""
from __future__ import annotations

import time
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import ActorApply, ActorCriticParams, CriticApply
from stoix_b200.config import DictConfig, compose
from stoix_b200.envs import cpu as cpu_envs
from stoix_b200.systems.impala.impala_types import ImpalaTransition
from stoix_b200.systems.ppo.sebulba import ff_ppo as seb
from stoix_b200.systems.ppo.sebulba.ff_ppo import CoreLearnerState, SebulbaExperimentOutput
from stoix_b200.utils.training import make_learning_rate

_METRIC_NAMES = ops.VTRACE_METRICS  # actor_loss, entropy, value_loss, q_estimate, pg_advantage


def check_config(config: DictConfig) -> None:
    """IMPALA's refusal: the bf16 tensor-core kernels implement the PPO losses only."""
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for IMPALA: the bf16 tensor-core kernels implement the PPO clipped surrogate "
                         "only, not the V-trace losses; use arch.precision=f32")


def minibatch_row_index(T: int, E: int, num_minibatches: int) -> np.ndarray:
    """int32 (num_minibatches, (T + 1) * Em): minibatch i is the env-column block [i Em, (i + 1) Em) with all T + 1 time rows
    (ff_impala.py:524-561), time-major: entry t Em + j is row t E + i Em + j of the flattened (T + 1, E) batch.  The actor reads the
    first T Em entries, the critic all of them."""
    Em = E // num_minibatches
    t = np.arange(T + 1)[:, None] * E
    return np.stack([(t + i * Em + np.arange(Em)[None, :]).reshape(-1) for i in range(num_minibatches)]).astype(np.int32)


def get_act_fn(apply_fns: Tuple[ActorApply, CriticApply]) -> Callable:
    """Action function for actor threads (ff_impala.py:107-125): (params, observation, rng_key) -> (action, log_prob, rng_key), the
    actor alone.  The actor threads themselves run the inference server with ImpalaTransition storage (same kernels)."""
    actor_apply_fn, _ = apply_fns

    def actor_fn(params: ActorCriticParams, observation: torch.Tensor, rng_key: int):
        rng_key, policy_key = srandom.split(rng_key, 2)
        pi = actor_apply_fn(params.actor_params, observation)
        action = pi.sample(seed=policy_key)
        return action, pi.log_prob(action), rng_key

    return actor_fn


def get_rollout_fn(*args, **kwargs) -> Callable[[int], None]:
    """Sebulba PPO's rollout function (ff_impala.py:128-315) delivering ImpalaTransition shards, without critic evaluation."""
    return seb.get_rollout_fn(*args, transition=ImpalaTransition, **kwargs)


def get_actor_thread(*args, **kwargs):
    """Sebulba PPO's actor thread (ff_impala.py:318-355) running get_rollout_fn above."""
    return seb.get_actor_thread(*args, transition=ImpalaTransition, **kwargs)


def get_learner_step_fn(apply_fns: Tuple[ActorApply, CriticApply], update_fns: Tuple[Callable, Callable], config: DictConfig) -> Callable:
    """Create the V-trace learner update (ff_impala.py:358-566) over the actors' shards."""
    check_config(config)
    actor_opt, critic_opt = update_fns[0].__self__, update_fns[1].__self__
    sysc = config.system
    T, nmb = int(sysc.rollout_length), int(sysc.num_minibatches)
    E = seb.learner_envs(config)
    if E % nmb:
        raise ValueError(f"num_minibatches={nmb} must divide the {E} environments of the learner batch (ff_impala.py:531)")
    Em = E // nmb
    norm = bool(sysc.normalize_rewards)
    hyper = dict(gamma=float(sysc.gamma), lambda_=float(sysc.vtrace_lambda), clip_rho=float(sysc.clip_rho_threshold),
                 clip_pg_rho=float(sysc.clip_pg_rho_threshold), ent_coef=float(sysc.ent_coef), vf_coef=float(sysc.vf_coef),
                 reward_scale=float(sysc.reward_scale), reward_eps=float(sysc.reward_eps))
    built: Dict[str, Any] = {}

    def _build(state: CoreLearnerState) -> None:
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        sa, sc, dev = a_tree.spec, c_tree.spec, a_tree.flat.device
        _, coff, total = ops.arena_offsets(sa, sc)
        D, A = sa.sizes[0], sa.sizes[-1]
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        built.update(sa=sa, sc=sc, coff=coff, D=D, arena=a_tree.arena,
                     plan=optax.adam_plan([(0, sa.param_count, actor_opt), (coff, sc.param_count, critic_opt)], dev, a_tree.arena_counts),
                     row_idx=torch.as_tensor(minibatch_row_index(T, E, nmb), device=dev),
                     obs=z(T + 1, E, D), action=z(T + 1, E, dt=torch.int32), log_prob=z(T + 1, E), reward=z(T + 1, E),
                     done=z(T + 1, E, dt=torch.uint8), truncated=z(T + 1, E, dt=torch.uint8),
                     logits=z(T * Em, A), values=z((T + 1) * Em), d_logits=z(T * Em, A), d_value=z((T + 1) * Em), grads=z(total),
                     metrics=z(nmb, len(_METRIC_NAMES)), reward_stats=z(2),
                     ws_a=ops.mlp_train_workspace(sa, T * Em, dev), ws_c=ops.mlp_train_workspace(sc, (T + 1) * Em, dev))

    def minibatch(i: int, a_tree) -> None:
        """_update_minibatch (ff_impala.py:397-522) on column block i: gradients of both losses, then one clip + RMSProp step."""
        b = built
        sa, sc, coff, arena, grads = b["sa"], b["sc"], b["coff"], b["arena"], b["grads"]
        idx = b["row_idx"][i]
        idx_a = idx[: T * Em]
        x = b["obs"].view((T + 1) * E, b["D"])
        cols = slice(i * Em, (i + 1) * Em)
        ops.mlp_forward_train(sa, arena, x, b["ws_a"], out=b["logits"], row_idx=idx_a)
        ops.mlp_forward_train(sc, arena[coff:], x, b["ws_c"], out=b["values"].view(-1, 1), row_idx=idx)
        ops.vtrace_loss_grads(b["logits"], b["values"], b["action"][:T, cols], b["log_prob"][:T, cols], b["reward"][:T, cols],
                              b["done"][:T, cols], b["d_logits"], b["d_value"], b["metrics"][i], reward_stats=b["reward_stats"] if norm else None,
                              **hyper)
        ops.mlp_backward(sa, arena, x, b["d_logits"], b["ws_a"], net_grad=grads, row_idx=idx_a)
        ops.mlp_backward(sc, arena[coff:], x, b["d_value"].view(-1, 1), b["ws_c"], net_grad=grads[coff:], row_idx=idx)
        ops.clip_adam_step(b["plan"], arena, grads, a_tree.arena_mu, a_tree.arena_nu)

    def _update_step(learner_state: CoreLearnerState, sharded_traj_batchs: List[ImpalaTransition]) -> Tuple[CoreLearnerState, Dict[str, torch.Tensor]]:
        if not built:
            _build(learner_state)
        b = built
        # Combine data from all actors: jnp.hstack along the env axis (:375) = column blocks of the learner's buffers
        off = 0
        for shard in sharded_traj_batchs:
            n = shard.action.shape[1]
            for name in ImpalaTransition._fields:
                b[name][:, off:off + n].copy_(getattr(shard, name), non_blocking=True)
            off += n
        assert off == E, f"the actors delivered {off} environments, the learner expects {E}"
        ops.reward_stats(b["reward"][:T], out=b["reward_stats"])  # the metrics, and the normalisation when it is on (:389-400)
        for i in range(nmb):  # jax.lax.scan over the minibatches, in order (:561)
            minibatch(i, learner_state.params.actor_params)
        loss_info = {name: b["metrics"][:, j].clone() for j, name in enumerate(_METRIC_NAMES)}
        loss_info.update(reward_mean=b["reward_stats"][0].clone(), reward_std=b["reward_stats"][1].clone())
        return learner_state, loss_info

    def learner_step_fn(learner_state: CoreLearnerState, traj_batch: List[ImpalaTransition]) -> SebulbaExperimentOutput:
        learner_state, loss_info = _update_step(learner_state, traj_batch)
        return SebulbaExperimentOutput(learner_state=learner_state, train_metrics=loss_info)

    learner_step_fn.built = built
    learner_step_fn.minibatch = minibatch
    return learner_step_fn


def learner_setup(env_factory: cpu_envs.EnvFactory, keys: Tuple[int, int, int], learner_devices: Sequence[torch.device],
                  config: DictConfig) -> Tuple[Callable, Tuple[ActorApply, CriticApply], CoreLearnerState]:
    """Setup learner networks and initial state (ff_impala.py:718-806): Sebulba PPO's networks and arena with
    chain(clip_by_global_norm(max_grad_norm), rmsprop(lr)) per network, the learning rate decaying over 1 epoch x num_minibatches
    optimiser steps per update."""
    check_config(config)
    sysc = config.system
    optim = lambda lr: optax.chain(optax.clip_by_global_norm(sysc.max_grad_norm),
                                   optax.rmsprop(make_learning_rate(lr, config, 1, sysc.num_minibatches)))
    return seb.learner_setup(env_factory, keys, learner_devices, config, optimisers=(optim(sysc.actor_lr), optim(sysc.critic_lr)),
                             step_fn_factory=get_learner_step_fn)


def run_experiment(_config: DictConfig) -> float:
    """Run IMPALA experiment (ff_impala.py:809-1036): Sebulba PPO's threads with IMPALA's actors and learner."""
    check_config(_config)
    return seb.run_experiment(_config, setup=learner_setup, transition=ImpalaTransition)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point (ff_impala.py:1039): `python -m stoix_b200.systems.impala.sebulba.ff_impala k=v ...`"""
    import sys

    if cfg is None:
        cfg = compose("default_ff_impala", overrides if overrides is not None else sys.argv[1:], config_dir="default/sebulba")
    t0 = time.perf_counter()
    perf = run_experiment(cfg)
    print(f"IMPALA experiment completed in {time.perf_counter() - t0:.2f}s with a final episode return of {perf}.")
    return perf


if __name__ == "__main__":
    hydra_entry_point()
