"""SyntheticBoxEnv -- the benchmark environment named by BASELINE.json configs[1]: Box observations
of dimension D drawn N(0,1), N(0,1) rewards, Bernoulli termination / truncation, with the reference's
auto-reset + episode-metrics wrapper semantics implemented in the step kernel
(stoix_b200/csrc/stx_env.cu).  Dynamics ignore the action: the env exists to fix shapes and memory
traffic of the training step, exactly like the reference's debug envs (stoix/utils/debug_env.py)
exist to exercise the learner."""
from __future__ import annotations

from typing import Any, Dict, Tuple

import torch

from .. import ops
from .base import ArraySpace, DiscreteSpace, Environment, StepOut, StepType, TimeStep, timestep_from_out


class SyntheticBoxEnv(Environment):
    def __init__(self, obs_dim: int = 64, num_actions: int = 8, p_term: float = 1.0 / 200, p_trunc: float = 1.0 / 500,
                 seed: int = 42, device="cuda", obs_dtype=torch.float32):
        self.obs_dim, self.num_actions = int(obs_dim), int(num_actions)
        self.p_term, self.p_trunc, self.seed = float(p_term), float(p_trunc), int(seed)
        self.device = torch.device(device)
        self.obs_dtype = obs_dtype

    def observation_space(self) -> ArraySpace:
        return ArraySpace((self.obs_dim,), torch.float32, self.device)

    def action_space(self) -> DiscreteSpace:
        return DiscreteSpace(self.num_actions)

    # -- functional face ---------------------------------------------------------------------------
    def reset(self, keys) -> Tuple[Dict[str, Any], TimeStep]:
        E = len(keys)
        dev = self.device
        state = {
            "seed": int(self.seed),  # per-shard stream: learner_setup sets env.seed before each reset
            "counter": torch.zeros(1, dtype=torch.int64, device=dev),  # global step index (uint64)
            "run_return": torch.zeros(E, dtype=torch.float32, device=dev),
            "run_length": torch.zeros(E, dtype=torch.int32, device=dev),
            "host_step": 0,
        }
        out = self._alloc(E)
        dummy = torch.zeros(E, dtype=torch.int32, device=dev)
        scratch_rr, scratch_rl = torch.zeros_like(state["run_return"]), torch.zeros_like(state["run_length"])
        # The first observation is the "reset" draw of step 2^62 (never reached by training).
        ops.synth_env_step(E, self.obs_dim, self.seed, 1 << 62, 2.0, 0.0, dummy, out.obs, out.next_obs, out.reward,
                           out.done, out.truncated, scratch_rr, scratch_rl, out.episode_return, out.episode_length,
                           out.is_terminal_step)
        ts = TimeStep(
            torch.full((E,), StepType.FIRST, dtype=torch.int8, device=dev),
            torch.zeros(E, device=dev), torch.ones(E, device=dev), out.obs,
            {"next_obs": out.obs,
             "episode_metrics": {"episode_return": torch.zeros(E, device=dev),
                                 "episode_length": torch.zeros(E, dtype=torch.int32, device=dev),
                                 "is_terminal_step": torch.zeros(E, dtype=torch.bool, device=dev)}},
        )
        return state, ts

    def _alloc(self, E: int) -> StepOut:
        dev, D = self.device, self.obs_dim
        return StepOut(
            torch.empty(E, D, dtype=self.obs_dtype, device=dev), torch.empty(E, D, dtype=self.obs_dtype, device=dev),
            torch.empty(E, device=dev), torch.empty(E, dtype=torch.uint8, device=dev),
            torch.empty(E, dtype=torch.uint8, device=dev), torch.empty(E, device=dev),
            torch.empty(E, dtype=torch.int32, device=dev), torch.empty(E, dtype=torch.uint8, device=dev),
        )

    def step(self, state, action) -> Tuple[Dict[str, Any], TimeStep]:
        E = state["run_return"].shape[0]
        out = self._alloc(E)
        self.step_into(state, action, out, state["host_step"])
        new_state = dict(state)
        new_state["host_step"] = state["host_step"] + 1
        return new_state, timestep_from_out(out)

    # -- zero-copy face used by the learner ---------------------------------------------------------
    def step_into(self, state, action: torch.Tensor, out: StepOut, t: int) -> None:
        """Step `t` (offset added to the device-resident counter) writing into `out`."""
        E = state["run_return"].shape[0]
        ops.synth_env_step(E, self.obs_dim, state["seed"], int(t), self.p_term, self.p_trunc, action, out.obs, out.next_obs,
                           out.reward, out.done, out.truncated, state["run_return"], state["run_length"],
                           out.episode_return, out.episode_length, out.is_terminal_step, dev_counter=state["counter"])

    # -- whole-rollout face (bf16 tensor-core path) ---------------------------------------------------
    fused_rollout_supported = True

    def fused_trajectory(self, state, shard, T: int) -> None:
        """Steps [0, T) of every env of the shard in one launch over the whole GPU (stx_synth_env_trajectory).  Valid because
        this env's dynamics ignore the action: obs[1..T], next_obs and the per-step scalars are bit-identical to T calls of
        step_into (the RNG counters are (env, absolute step)), and the policy then only reads the observations."""
        E = state["run_return"].shape[0]
        ops.synth_env_trajectory(E, self.obs_dim, T, state["seed"], 0, self.p_term, self.p_trunc, shard.obs[:T + 1], shard.next_obs[:T],
                                 shard.reward[:T], shard.terminated[:T], shard.truncated[:T], shard.episode_return[:T], shard.episode_length[:T],
                                 shard.is_terminal_step[:T], state["run_return"], state["run_length"], dev_counter=state["counter"])

    def fused_rollout(self, state, actor_spec, actor_params, actor_params_bf16, shard, T: int, cat_seed: int, cat_counter) -> None:
        """All T steps of env + policy: fused_trajectory, then the policy over its observations (stx_tc_rollout_policy)."""
        self.fused_trajectory(state, shard, T)
        ops.tc_rollout_policy(actor_spec, actor_params, actor_params_bf16, shard.obs[:T], shard.action[:T], shard.log_prob[:T], cat_seed, 0,
                              cat_counter)

    def advance(self, state, steps: int) -> None:
        """Move the device-resident step counter (end of a rollout; graph-capturable)."""
        ops.counter_add(state["counter"], steps)
