"""Sebulba feed-forward PPO on H100 -- drop-in for stoix/systems/ppo/sebulba/ff_ppo.py (MLP torso).

Same entry points (get_act_fn :123, get_rollout_fn :145, get_actor_thread :336, get_learner_step_fn :378,
get_learner_rollout_fn :568, get_learner_thread :661, learner_setup :703, run_experiment :801, hydra_entry_point :1026)
and the same thread topology: N actor threads per actor GPU stepping CPU environments, one learner thread, one evaluator
thread, joined by ParameterServer / OnPolicyPipeline queues (stoix_b200/utils/sebulba_utils.py).

  reference (JAX)                                     here (H100)
  --------------------------------------------------  -------------------------------------------------------------
  act_fn = jit(actor+critic apply, sample) per step    batched INFERENCE SERVER per actor thread: the thread's env batch
  obs -> device by an implicit transfer, action back   goes pinned-host -> cudaMemcpyAsync on the thread's own stream ->
  through np.asarray                                   actor + critic forward kernels (the Anakin K1 kernels) + sampling
                                                       kernel -> action back into a pinned buffer; ONE event wait per step
  trajectory = list of per-step pytrees, stacked and   preallocated (T+1, E, ...) device storage written in place; reward /
  device_put_sharded to the learners every rollout     done flags staged in pinned memory and uploaded once per rollout;
                                                       peer copies (NVLink) of the env-axis shards to the learner GPUs
  learner: hstack shards, GAE via values=, shuffled    shards land in column blocks of one (T+1, E_total) buffer; K2 GAE
  epochs x minibatches under pmap                      with v_t = values[1:]; the Anakin K3 / K4 kernels per minibatch
  params -> actors: device_put of the tree per device  one peer copy of the flat arena (+ bf16 shadow) per actor device

Scope of this build: one process; any number of actor devices / threads; ONE learner device (the reference's
`pmap(axis_name="learner_devices")` over several learner GPUs maps onto one process per GPU + the Anakin gradient
all-reduce and is not wired up here); MLP torso (BASELINE config 3 names a CNN/ResNet torso on Breakout: the conv
stack is outside the hot-path build, see DESIGN.md).
"""
from __future__ import annotations

import copy
import queue
import random
import threading
import time
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import ActorApply, ActorCriticOptStates, ActorCriticParams, CriticApply
from stoix_b200.config import DictConfig, compose, instantiate, to_container
from stoix_b200.envs import cpu as cpu_envs
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import FeedForwardCritic as Critic
from stoix_b200.utils.logger import LogEvent, StoixLogger
from stoix_b200.utils.sebulba_utils import (
    AsyncEvaluatorBase,
    OnPolicyPipeline,
    ParameterServer,
    ParamSnapshot,
    ThreadLifetime,
    TimingTracker,
)
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.training import make_learning_rate

_METRIC_NAMES = ("actor_loss", "entropy", "value_loss", "advantages", "pred_value", "target_value")


class PPOTransition(NamedTuple):
    """Transition tuple for Sebulba PPO: the Anakin one without bootstrap_value / info (sebulba/ff_ppo.py:68-77)."""

    done: torch.Tensor
    truncated: torch.Tensor
    action: torch.Tensor
    value: torch.Tensor
    reward: torch.Tensor
    log_prob: torch.Tensor
    obs: torch.Tensor


class CoreLearnerState(NamedTuple):
    """stoix/base_types.py CoreLearnerState: params, opt_states, key."""

    params: Any
    opt_states: Any
    key: Any


class SebulbaExperimentOutput(NamedTuple):
    learner_state: Any
    train_metrics: Dict[str, torch.Tensor]


def _precision(config) -> int:
    return ops.STX_PREC_BF16 if str(config.arch.get("precision", "f32")) == "bf16" else ops.STX_PREC_F32


# ---------------------------------------------------------------------------------------------------------------
# actor side
# ---------------------------------------------------------------------------------------------------------------


class InferenceServer:
    """The batched policy / value evaluation of ONE actor thread (sebulba/ff_ppo.py:123-143 `get_act_fn`, jitted onto the
    actor device at :160-161).  Owns a CUDA stream, pinned host buffers and the thread's (T+1)-step device storage.

    `transition` is the NamedTuple the storage is delivered as; one without a `value` field (IMPALA's actors sample from the actor
    alone) skips the critic forward."""

    def __init__(self, specs: Tuple[ops.MlpSpec, ops.MlpSpec], device: torch.device, num_envs: int, rollout_length: int,
                 precision: int, seed: int, thread_id: int, transition: type = PPOTransition):
        self.transition = transition
        self.critic = "value" in self.transition._fields
        self.sa, self.sc = specs
        self.device, self.E, self.T, self.precision, self.seed, self.tid = device, int(num_envs), int(rollout_length), precision, int(seed), thread_id
        _, self.coff, _ = ops.arena_offsets(self.sa, self.sc)
        D, A = self.sa.sizes[0], self.sa.sizes[-1]
        obs_dt = torch.bfloat16 if precision == ops.STX_PREC_BF16 else torch.float32
        with torch.cuda.device(device):
            self.stream = torch.cuda.Stream(device=device)
            z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
            n = self.T + 1
            self.obs = z(n, self.E, D, dt=obs_dt)
            self.action, self.value, self.log_prob = z(n, self.E, dt=torch.int32), z(n, self.E), z(n, self.E)
            self.reward, self.done, self.truncated = z(n, self.E), z(n, self.E, dt=torch.uint8), z(n, self.E, dt=torch.uint8)
            self.obs_f32 = z(self.E, D)
            self.logits = z(self.E, A)
            self.step_event = torch.cuda.Event()
        pin = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt).pin_memory()
        self.h_obs, self.h_action = pin(self.E, D), pin(self.E, dt=torch.int32)
        self.h_reward, self.h_done, self.h_trunc = pin(n, self.E), pin(n, self.E, dt=torch.uint8), pin(n, self.E, dt=torch.uint8)
        self.calls = 0
        self.h2d_bytes = self.d2h_bytes = 0

    def act(self, params: ParamSnapshot, observation: np.ndarray, slot: int) -> np.ndarray:
        """obs (host) -> action (host); value / log_prob / obs of the step stay on the device in storage row `slot`."""
        self.h_obs.numpy()[...] = observation.reshape(self.E, -1)
        a_flat, c_flat = params.arena[: self.coff], params.arena[self.coff:]
        a16 = params.arena_bf16[: self.coff] if params.arena_bf16 is not None else None
        c16 = params.arena_bf16[self.coff:] if params.arena_bf16 is not None else None
        key = f"sebulba-actor-{self.tid}"
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            if self.precision == ops.STX_PREC_BF16:
                self.obs_f32.copy_(self.h_obs, non_blocking=True)          # pinned cudaMemcpyAsync on the side stream
                ops.cast_bf16(self.obs_f32, out=self.obs[slot])
            else:
                self.obs[slot].copy_(self.h_obs, non_blocking=True)
            ops.mlp_forward(self.sa, a_flat, self.obs[slot], precision=self.precision, params_bf16=a16, out=self.logits, ws_key=key)
            ops.categorical(self.logits, None, self.seed, self.calls, out=(self.action[slot], self.log_prob[slot]))
            if self.critic:
                ops.mlp_forward(self.sc, c_flat, self.obs[slot], precision=self.precision, params_bf16=c16,
                                out=self.value[slot].view(self.E, 1), ws_key=key)
            self.h_action.copy_(self.action[slot], non_blocking=True)
            self.step_event.record(self.stream)
        self.step_event.synchronize()                                      # the host needs the actions to step the envs
        self.calls += 1
        self.h2d_bytes += self.h_obs.numel() * 4
        self.d2h_bytes += self.h_action.numel() * 4
        return self.h_action.numpy()

    def record(self, slot: int, timestep: cpu_envs.TimeStep) -> None:
        """reward / done / truncated of the step just taken (sebulba/ff_ppo.py:236-253), staged in pinned memory."""
        done = timestep.last()
        self.h_reward.numpy()[slot] = timestep.reward
        self.h_done.numpy()[slot] = done
        self.h_trunc.numpy()[slot] = np.logical_and(done, timestep.discount == 1)

    def flush(self, lo: int) -> None:
        """Upload the staged rows [lo, T] once per rollout."""
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            self.reward[lo:].copy_(self.h_reward[lo:], non_blocking=True)
            self.done[lo:].copy_(self.h_done[lo:], non_blocking=True)
            self.truncated[lo:].copy_(self.h_trunc[lo:], non_blocking=True)
        self.h2d_bytes += (self.T + 1 - lo) * self.E * 6

    def storage(self):
        return self.transition(*[getattr(self, name) for name in self.transition._fields])

    def carry_last(self) -> None:
        """Keep the last transition as row 0 of the next rollout (sebulba/ff_ppo.py:279)."""
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            for t in self.storage():
                t[0].copy_(t[self.T])
        for h in (self.h_reward, self.h_done, self.h_trunc):
            h[0].copy_(h[self.T])


def get_act_fn(apply_fns: Tuple[ActorApply, CriticApply]) -> Callable:
    """Action function for actor threads (sebulba/ff_ppo.py:123-143): (params, observation, rng_key) -> (action, value,
    log_prob, rng_key) on device tensors, through the public network faces.  The actor threads themselves use the
    InferenceServer (same kernels, preallocated buffers, pinned transfers)."""
    actor_apply_fn, critic_apply_fn = apply_fns

    def actor_fn(params: ActorCriticParams, observation: torch.Tensor, rng_key: int):
        rng_key, policy_key = srandom.split(rng_key, 2)
        pi = actor_apply_fn(params.actor_params, observation)
        value = critic_apply_fn(params.critic_params, observation)
        action = pi.sample(seed=policy_key)
        return action, value, pi.log_prob(action), rng_key

    return actor_fn


def get_rollout_fn(env_factory: cpu_envs.EnvFactory, actor_device: torch.device, parameter_server: ParameterServer,
                   rollout_pipeline: OnPolicyPipeline, apply_fns: Tuple[ActorApply, CriticApply], config: DictConfig,
                   logger: StoixLogger, learner_devices: Sequence[torch.device], seeds: List[int],
                   thread_lifetime: ThreadLifetime, transition: type = PPOTransition) -> Callable[[int], None]:
    """Create rollout function for actor threads (sebulba/ff_ppo.py:145-333).  `transition`: the type of the delivered shards (see
    InferenceServer)."""
    num_envs_per_actor = int(config.arch.actor.num_envs_per_actor)
    rollout_length = int(config.system.rollout_length)
    num_actor_threads = int(config.arch.actor.actor_per_device)
    len_actor_device_ids = len(config.arch.actor.device_ids)
    world_size = int(config.arch.world_size)
    actor_log_frequency = int(config.arch.actor.log_frequency)
    num_updates = int(config.arch.num_updates)
    synchronous = bool(config.arch.synchronous)
    n_learn = len(learner_devices)
    assert num_envs_per_actor % n_learn == 0, "num_envs_per_actor must divide across the learner devices"
    actor_net, critic_net = apply_fns[0].__self__, apply_fns[1].__self__
    obs_dim = int(np.prod(config.system.observation_shape))
    specs = (actor_net.spec_for(obs_dim), critic_net.spec_for(obs_dim))
    envs = env_factory(num_envs_per_actor)

    def rollout_fn(rng_key: int) -> None:
        thread_start_time = time.perf_counter()
        local_step_count, actor_policy_version, num_rollouts = 0, -1, 0
        timer = TimingTracker(maxlen=10)
        server = InferenceServer(specs, actor_device, num_envs_per_actor, rollout_length, _precision(config), int(rng_key) & ((1 << 62) - 1),
                                 thread_lifetime.id, transition)
        rollout_fn.server = server  # exposed for tests / bench
        episode_metrics_storage: List[Dict[str, np.ndarray]] = []
        timestep = envs.reset(seed=seeds)
        params: Optional[ParamSnapshot] = None
        have_rows = 0  # rows of the storage already valid at the start of the rollout (0, then 1)
        torch.cuda.set_device(actor_device)
        while not thread_lifetime.should_stop():
            num_steps_with_bootstrap = rollout_length + int(have_rows == 0)
            with timer.time("get_params_time"):
                # first rollout: initial policy; second rollout: do not wait (the first update is still running);
                # afterwards block for the updated policy -- sebulba/ff_ppo.py:204-213
                if not num_rollouts == 1 or synchronous:
                    with torch.cuda.stream(server.stream):
                        params = parameter_server.get_params(thread_lifetime.id)
                    actor_policy_version += 1
            if params is None:  # shutdown signal
                break
            with timer.time("single_actor_rollout_time"):
                for i in range(num_steps_with_bootstrap):
                    slot = have_rows + i
                    with timer.time("inference_time"):
                        cpu_action = server.act(params, timestep.observation, slot)
                    with timer.time("env_step_time"):
                        timestep = envs.step(cpu_action)
                    with timer.time("storage_time"):
                        server.record(slot, timestep)
                        episode_metrics_storage.append(timestep.extras["metrics"])
                    local_step_count += num_envs_per_actor
                num_rollouts += 1
            with timer.time("prepare_data_time"):
                server.flush(have_rows)
                # shard along the env axis onto the learner devices (sebulba/ff_ppo.py:164-169, 260-266): peer copies,
                # ordered behind this thread's stream
                per = num_envs_per_actor // n_learn
                ready = torch.cuda.Event()
                with torch.cuda.stream(server.stream):
                    shards = []
                    for li, ld in enumerate(learner_devices):
                        sl = slice(li * per, (li + 1) * per)
                        shards.append(transition(*[t[:, sl].to(ld, non_blocking=True) if ld != actor_device or n_learn > 1 else t.clone()
                                                   for t in server.storage()]))
                    ready.record(server.stream)
                payload = (local_step_count, actor_policy_version, (shards, ready))
            with timer.time("rollout_queue_put_time"):
                if not rollout_pipeline.send_rollout(thread_lifetime.id, payload):
                    print(f"Warning: Failed to send rollout from actor {thread_lifetime.id}")
            server.carry_last()
            have_rows = 1
            if num_rollouts % actor_log_frequency == 0 and thread_lifetime.id == 0:
                approximate_global_step = local_step_count * num_actor_threads * len_actor_device_ids * world_size
                elapsed = time.perf_counter() - thread_start_time
                logger.log({**timer.get_all_means(), "actor_policy_version": actor_policy_version,
                            "local_SPS": int(local_step_count / elapsed), "global_SPS": int(approximate_global_step / elapsed),
                            "num_rollouts": num_rollouts}, approximate_global_step, actor_policy_version, LogEvent.MISC)
                term = np.concatenate([m["is_terminal_step"] for m in episode_metrics_storage])
                if term.sum() > 1:
                    rets = np.concatenate([m["episode_return"] for m in episode_metrics_storage])[term]
                    lens = np.concatenate([m["episode_length"] for m in episode_metrics_storage])[term]
                    logger.log({"episode_return": torch.as_tensor(rets), "episode_length": torch.as_tensor(lens),
                                "num_completed_episodes_in_rollout_batch": len(rets)}, approximate_global_step, actor_policy_version,
                               LogEvent.ACT)
                    episode_metrics_storage.clear()
            if num_rollouts > num_updates:
                break
        rollout_fn.stats = {**timer.get_all_means(), "local_step_count": local_step_count, "num_rollouts": num_rollouts,
                            "elapsed_s": time.perf_counter() - thread_start_time, "h2d_bytes": server.h2d_bytes, "d2h_bytes": server.d2h_bytes}
        envs.close()

    return rollout_fn


def get_actor_thread(env_factory, actor_device, parameter_server, rollout_pipeline, apply_fns, rng_key, config, seeds, logger,
                     learner_devices, thread_lifetime, transition: type = PPOTransition) -> threading.Thread:
    """Create actor thread for environment data collection (sebulba/ff_ppo.py:336-375)."""
    rollout_fn = get_rollout_fn(env_factory=env_factory, actor_device=actor_device, parameter_server=parameter_server,
                                rollout_pipeline=rollout_pipeline, apply_fns=apply_fns, config=config, logger=logger,
                                learner_devices=learner_devices, seeds=seeds, thread_lifetime=thread_lifetime, transition=transition)
    th = threading.Thread(target=rollout_fn, args=(rng_key,), name=thread_lifetime.name)
    th.rollout_fn = rollout_fn
    return th


# ---------------------------------------------------------------------------------------------------------------
# learner side
# ---------------------------------------------------------------------------------------------------------------


def learner_envs(config: DictConfig) -> int:
    """Environments per learner batch (total_num_envs over the learner devices); refuses more than one learner device."""
    n_learn = len(config.arch.learner.device_ids)
    assert n_learn == 1, "this build drives ONE learner device per process (see the module docstring)"
    return int(config.arch.total_num_envs) // n_learn


def get_learner_step_fn(apply_fns: Tuple[ActorApply, CriticApply], update_fns: Tuple[Callable, Callable],
                        config: DictConfig) -> Callable:
    """Create learner update function (sebulba/ff_ppo.py:378-565): hstack the actors' shards, GAE through the `values=`
    interface (v_tm1 = values[:-1], v_t = values[1:], discount = (1 - done) * gamma, no truncation -- :399-411), then
    epochs x minibatches of the fused PPO gradient + clip/Adam kernels on obs[:-1] etc. (:516-519)."""
    actor_net, critic_net = apply_fns[0].__self__, apply_fns[1].__self__
    actor_opt, critic_opt = update_fns[0].__self__, update_fns[1].__self__
    sysc, arch = config.system, config.arch
    T, epochs, nmb = int(sysc.rollout_length), int(sysc.epochs), int(sysc.num_minibatches)
    E = learner_envs(config)   # envs_per_batch (:522)
    B = T * E
    assert B % nmb == 0, "rollout_length * envs_per_batch must be divisible by num_minibatches"
    mb = B // nmb
    precision = _precision(config)
    built: Dict[str, Any] = {}

    def _build(state: CoreLearnerState) -> None:
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        sa, sc, dev = a_tree.spec, c_tree.spec, a_tree.flat.device
        _, coff, total = ops.arena_offsets(sa, sc)
        D = sa.sizes[0]
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        obs_dt = torch.bfloat16 if precision == ops.STX_PREC_BF16 else torch.float32
        plan = optax.adam_plan([(0, sa.param_count, actor_opt), (coff, sc.param_count, critic_opt)], dev, a_tree.arena_counts)
        built.update(sa=sa, sc=sc, dev=dev, D=D, total=total, plan=plan, arena=a_tree.arena, arena_bf16=getattr(a_tree, "arena_bf16", None),
                     obs=z(T + 1, E, D, dt=obs_dt), action=z(T + 1, E, dt=torch.int32), value=z(T + 1, E), log_prob=z(T + 1, E),
                     reward=z(T + 1, E), done=z(T + 1, E, dt=torch.uint8), truncated=z(T + 1, E, dt=torch.uint8),
                     no_trunc=z(T, E, dt=torch.uint8), advantages=z(T, E), targets=z(T, E), perms=z(epochs, B, dt=torch.int32),
                     grads=z(total), metrics=z(epochs, nmb, 8), ws=ops.ppo_workspace(sa, sc, mb, precision, dev),
                     perm_ctr=torch.zeros(1, dtype=torch.int64, device=dev))

    def _update_step(learner_state: CoreLearnerState, sharded_traj_batchs: List[PPOTransition]) -> Tuple[CoreLearnerState, Dict[str, torch.Tensor]]:
        if not built:
            _build(learner_state)
        b = built
        a_tree = learner_state.params.actor_params
        # Combine data from all actors: jnp.hstack along the env axis (:394) = column blocks of the learner's buffers
        off = 0
        for shard in sharded_traj_batchs:
            n = shard.action.shape[1]
            for name in PPOTransition._fields:
                b[name][:, off:off + n].copy_(getattr(shard, name), non_blocking=True)
            off += n
        assert off == E, f"the actors delivered {off} environments, the learner expects {E}"
        # CALCULATE ADVANTAGE (:396-411): r_t = reward[:-1], d_t = (1 - done[:-1]) * gamma, values = value (all T+1 rows)
        _, _, adv_stats = ops.gae_ppo(b["reward"][:T], b["value"][:T], b["value"][1:], b["done"][:T], b["no_trunc"], float(sysc.gamma),
                                      float(sysc.gae_lambda), 1.0, 1 if sysc.standardize_advantages else 0,
                                      out=(b["advantages"], b["targets"]))
        D, sa, sc = b["D"], b["sa"], b["sc"]
        b["metrics"].zero_()
        for ep in range(epochs):  # _update_epoch (:413-541): one permutation per epoch, shared by every leaf (:526)
            ops.make_permutation(B, learner_state.key, ep, dev_counter=b["perm_ctr"], out=b["perms"][ep])
            batch = ops.PpoBatch(b["obs"][:T].view(B, D), b["action"][:T].view(B), b["log_prob"][:T].view(B), b["value"][:T].view(B),
                                 b["advantages"].view(B), b["targets"].view(B), adv_stats, b["perms"][ep])
            prenorm = precision == ops.STX_PREC_BF16
            for i in range(nmb):  # _update_minibatch (:416-511)
                ops.ppo_minibatch_grads(sa, sc, b["arena"], batch, i * mb, mb, float(sysc.clip_eps), float(sysc.ent_coef),
                                        float(sysc.vf_coef), bool(sysc.standardize_advantages), b["grads"], b["metrics"][ep, i], b["ws"],
                                        precision, 1.0, b["arena_bf16"], overwrite=True, adam_scratch=b["plan"].scratch if prenorm else None)
                ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu, params_bf16=b["arena_bf16"],
                                   prenorm=prenorm)
        ops.counter_add(b["perm_ctr"], epochs)
        loss_info = {name: b["metrics"][..., j].clone() for j, name in enumerate(_METRIC_NAMES)}
        return learner_state, loss_info

    def learner_step_fn(learner_state: CoreLearnerState, traj_batch: List[PPOTransition]) -> SebulbaExperimentOutput:
        learner_state, loss_info = _update_step(learner_state, traj_batch)
        return SebulbaExperimentOutput(learner_state=learner_state, train_metrics=loss_info)

    learner_step_fn.built = built
    return learner_step_fn


def get_learner_rollout_fn(config: DictConfig, parameter_server: ParameterServer, rollout_pipeline: OnPolicyPipeline,
                           learner_step_fn: Callable, logger: StoixLogger, async_evaluator: Optional[AsyncEvaluatorBase]) -> Callable:
    """Create learner rollout function for network updates (sebulba/ff_ppo.py:568-658)."""
    learner_log_frequency = int(config.arch.learner.log_frequency)
    num_evaluation = int(config.arch.num_evaluation)
    num_updates_per_eval = int(config.arch.num_updates_per_eval)
    learner_device = torch.device("cuda", int(config.arch.learner.device_ids[0]))

    def learner_rollout(learner_state: CoreLearnerState, rng_key: int) -> None:
        torch.cuda.set_device(learner_device)
        # own stream: the legacy default stream would serialise the learner with every actor stream of this device
        with torch.cuda.stream(torch.cuda.Stream(device=learner_device)):
            _learner_loop(learner_state, rng_key)

    def _learner_loop(learner_state: CoreLearnerState, rng_key: int) -> None:
        thread_start_time = time.perf_counter()
        learner_policy_version = 0
        timer = TimingTracker(maxlen=10)
        global_step_count = 0
        for eval_step in range(num_evaluation if num_evaluation > 0 else 1):
            for _ in range(num_updates_per_eval):
                with timer.time("rollout_queue_get_time"):
                    rollout_data = rollout_pipeline.collect_rollouts()
                sharded_storages, global_step_count = [], 0
                for local_step_count, _version, (shards, ready) in rollout_data:
                    global_step_count += local_step_count
                    torch.cuda.current_stream().wait_event(ready)   # the peer copies of this actor's shard
                    sharded_storages.append(shards[0])
                with timer.time("learn_step_time"):
                    learner_state, loss_info = learner_step_fn(learner_state, sharded_storages)
                learner_policy_version += 1
                with timer.time("params_queue_put_time"):
                    parameter_server.distribute_params(learner_state.params)
                if learner_policy_version % learner_log_frequency == 0:
                    logger.log({**timer.get_all_means(), "update_no": learner_policy_version, "timestep": global_step_count,
                                "learner_policy_version": learner_policy_version,
                                "learner_steps_per_seconds": int(learner_policy_version / (time.perf_counter() - thread_start_time))},
                               global_step_count, learner_policy_version, LogEvent.MISC)
                    logger.log(dict(loss_info), global_step_count, learner_policy_version, LogEvent.TRAIN)
            if num_evaluation > 0 and async_evaluator is not None:
                rng_key, eval_key = srandom.split(rng_key, 2)
                torch.cuda.current_stream().synchronize()
                async_evaluator.submit_evaluation(learner_state, eval_key, eval_step, global_step_count)
        torch.cuda.current_stream().synchronize()
        learner_rollout.stats = {**timer.get_all_means(), "updates": learner_policy_version, "elapsed_s": time.perf_counter() - thread_start_time,
                                 "global_step_count": global_step_count}
        learner_rollout.final_state = learner_state

    return learner_rollout


def get_learner_thread(config, learn_step, learner_state, parameter_server, rollout_pipeline, logger, async_evaluator, rng_key) -> threading.Thread:
    """Create learner thread for network updates (sebulba/ff_ppo.py:661-683)."""
    fn = get_learner_rollout_fn(config, parameter_server, rollout_pipeline, learn_step, logger, async_evaluator)
    th = threading.Thread(target=fn, args=(learner_state, rng_key), name="Learner")
    th.learner_rollout = fn
    return th


def stop_all_actor_threads(actor_thread_lifetimes, parameter_server, rollout_pipeline, actor_threads) -> None:
    """sebulba/ff_ppo.py:686-700."""
    for lt in actor_thread_lifetimes:
        lt.stop()
    parameter_server.clear_all_queues()
    rollout_pipeline.clear_all_queues()
    parameter_server.shutdown_actors()
    for th in actor_threads:
        th.join()


class AsyncEvaluator(AsyncEvaluatorBase):
    """PPO-specific asynchronous evaluator (sebulba/ff_ppo.py:80-120)."""

    def run(self) -> None:
        while not self.lifetime.should_stop():
            try:
                item = self.eval_queue.get(timeout=1.0)
            except queue.Empty:
                continue
            if item is None:
                break
            learner_state, eval_key, eval_step, global_step_count = item
            assert eval_step == self.eval_step, f"Expected eval_step {self.eval_step}, but got {eval_step}."
            actor_params = learner_state.params.actor_params
            eval_metrics = self.evaluator(actor_params, eval_key)
            self.logger.log(eval_metrics, global_step_count, eval_step, LogEvent.EVAL)
            episode_return = float(eval_metrics["episode_return"].float().mean().item())
            if self.save_checkpoint:
                self.checkpointer.save(timestep=global_step_count, unreplicated_learner_state=learner_state, episode_return=episode_return)
            self._update_best_params(episode_return, actor_params)
            self.add_eval_metrics(eval_metrics)
            self._update_evaluation_progress()

    def get_best_params(self) -> Any:
        return self.best_params


def get_sebulba_eval_fn(env_factory: cpu_envs.EnvFactory, act_fn: Callable, config: DictConfig, np_rng: np.random.Generator,
                        device: torch.device, eval_multiplier: int = 1) -> Tuple[Callable, Any]:
    """stoix/evaluator.py get_sebulba_eval_fn: roll num_eval_episodes episodes on CPU envs with the policy on `device`."""
    n_episodes = int(config.arch.num_eval_episodes) * eval_multiplier
    envs = env_factory(n_episodes)
    max_steps = int(config.arch.get("max_eval_steps", 2000))

    def evaluator(params, key) -> Dict[str, torch.Tensor]:
        seeds = np_rng.integers(np.iinfo(np.int32).max, size=n_episodes).tolist()
        ts = envs.reset(seed=seeds)
        alive = np.ones(n_episodes, bool)
        ret, length = np.zeros(n_episodes), np.zeros(n_episodes, np.int64)
        with torch.cuda.device(device):
            for step in range(max_steps):
                obs = torch.as_tensor(ts.observation, device=device)
                action = act_fn(params, obs, srandom.split(key, 1)[0] + step)
                ts = envs.step(action.cpu().numpy())
                ret += ts.reward * alive
                length += alive
                alive &= ~ts.last()
                if not alive.any():
                    break
        return {"episode_return": torch.as_tensor(ret, dtype=torch.float32), "episode_length": torch.as_tensor(length)}

    return evaluator, envs


def learner_setup(env_factory: cpu_envs.EnvFactory, keys: Tuple[int, int, int], learner_devices: Sequence[torch.device],
                  config: DictConfig, optimisers: Optional[Tuple[Any, Any]] = None,
                  step_fn_factory: Optional[Callable] = None) -> Tuple[Callable, Tuple[ActorApply, CriticApply], CoreLearnerState]:
    """Setup learner networks and initial state (sebulba/ff_ppo.py:703-798).  Another actor-critic Sebulba system passes its
    (actor, critic) optimisers and its get_learner_step_fn; the defaults are PPO's."""
    env = env_factory(num_envs=1)
    num_actions = int(env.action_space().num_values)
    obs_shape = tuple(env.observation_space().shape)
    config.system.action_dim = num_actions
    config.system.observation_shape = list(obs_shape)
    env.close()
    key, actor_net_key, critic_net_key = keys
    device = torch.device(learner_devices[0])

    actor_torso = instantiate(config.network.actor_network.pre_torso)
    actor_action_head = instantiate(config.network.actor_network.action_head, action_dim=num_actions)
    critic_torso = instantiate(config.network.critic_network.pre_torso)
    critic_head = instantiate(config.network.critic_network.critic_head)
    actor_network = Actor(torso=actor_torso, action_head=actor_action_head)
    critic_network = Critic(torso=critic_torso, critic_head=critic_head)
    precision = _precision(config)
    actor_network.precision = critic_network.precision = precision

    if optimisers is None:
        actor_lr = make_learning_rate(config.system.actor_lr, config, config.system.epochs, config.system.num_minibatches)
        critic_lr = make_learning_rate(config.system.critic_lr, config, config.system.epochs, config.system.num_minibatches)
        optimisers = (optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(actor_lr, eps=1e-5)),
                      optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(critic_lr, eps=1e-5)))
    actor_optim, critic_optim = optimisers

    obs_dim = int(np.prod(obs_shape))
    with torch.cuda.device(device):
        init_x = torch.zeros(1, obs_dim, device=device)
        sa, sc = actor_network.spec_for(obs_dim), critic_network.spec_for(obs_dim)
        _, coff, total = ops.arena_offsets(sa, sc)
        arena = torch.zeros(total, dtype=torch.float32, device=device)
        actor_params = actor_network.init(actor_net_key, init_x, flat=arena[:coff])
        critic_params = critic_network.init(critic_net_key, init_x, flat=arena[coff:])
        arena_bf16 = None
        if precision == ops.STX_PREC_BF16:
            arena_bf16 = ops.cast_bf16(arena)
            actor_params.flat_bf16, critic_params.flat_bf16 = arena_bf16[:coff], arena_bf16[coff:]
        actor_params.arena_bf16 = arena_bf16
        opt_states = ActorCriticOptStates(*optax.arena_state(actor_params, arena, [(0, sa.param_count), (coff, sc.param_count)]))
    params = ActorCriticParams(actor_params, critic_params)
    apply_fns = (actor_network.apply, critic_network.apply)
    update_fns = (actor_optim.update, critic_optim.update)
    learn_step = (step_fn_factory or get_learner_step_fn)(apply_fns, update_fns, config)
    if warm_start(config, arena) and arena_bf16 is not None:
        ops.cast_bf16(arena, out=arena_bf16)
    learner_state = CoreLearnerState(params, opt_states, int(key) & ((1 << 62) - 1))
    return learn_step, apply_fns, learner_state


def run_experiment(_config: DictConfig, setup: Optional[Callable] = None, transition: type = PPOTransition) -> float:
    """Run PPO experiment (sebulba/ff_ppo.py:801-1023).  Another Sebulba system runs through the same threads by passing its own
    `setup` (the signature of learner_setup) and the transition type its actors deliver."""
    from stoix_b200.evaluator import get_distribution_act_fn

    config = copy.deepcopy(_config)
    n_gpu = torch.cuda.device_count()
    if max(list(config.arch.actor.device_ids) + list(config.arch.learner.device_ids) + [int(config.arch.evaluator_device_id)]) >= n_gpu:
        raise ValueError(f"the config names device ids beyond the {n_gpu} visible GPUs")
    actor_devices = [torch.device("cuda", int(i)) for i in config.arch.actor.device_ids]
    learner_devices = [torch.device("cuda", int(i)) for i in config.arch.learner.device_ids]
    evaluator_device = torch.device("cuda", int(config.arch.evaluator_device_id))
    config.num_learner_devices, config.num_actor_devices = len(learner_devices), len(actor_devices)
    config.arch.world_size = 1
    config.arch.total_num_actor_threads = len(actor_devices) * int(config.arch.actor.actor_per_device)
    config = check_total_timesteps(config)

    env_factory = cpu_envs.make_factory(config)
    key, key_e, actor_net_key, critic_net_key = srandom.split(srandom.PRNGKey(config.arch.seed), 4)
    np_rng = np.random.default_rng(int(config.arch.seed))
    torch.cuda.set_device(learner_devices[0])
    learn_step, apply_fns, learner_state = (setup or learner_setup)(env_factory, (key, actor_net_key, critic_net_key), learner_devices, config)

    eval_act_fn = get_distribution_act_fn(config, apply_fns[0])
    evaluator, evaluator_envs = get_sebulba_eval_fn(env_factory, eval_act_fn, config, np_rng, evaluator_device)
    logger = StoixLogger(config)
    logger.log_config(to_container(config, resolve=True))
    save_checkpoint = bool(config.logger.checkpointing.save_model)
    checkpointer = None
    if save_checkpoint:
        from stoix_b200.utils.checkpointing import Checkpointer

        checkpointer = Checkpointer(metadata=to_container(config), model_name=config.system.system_name,
                                    **to_container(config.logger.checkpointing.save_args))
    random.seed(int(config.arch.seed))
    np.random.seed(int(config.arch.seed))

    parameter_server = ParameterServer(total_num_actors=config.arch.total_num_actor_threads, actor_devices=actor_devices,
                                       actors_per_device=int(config.arch.actor.actor_per_device), queue_maxsize=1)
    rollout_pipeline = OnPolicyPipeline(total_num_actors=config.arch.total_num_actor_threads, queue_maxsize=1)
    parameter_server.distribute_params(learner_state.params)

    actor_threads, lifetimes = [], []
    thread_keys = srandom.split(key, config.arch.total_num_actor_threads + 1)
    for d_idx, dev in enumerate(actor_devices):
        for thread_id in range(int(config.arch.actor.actor_per_device)):
            idx = d_idx * int(config.arch.actor.actor_per_device) + thread_id
            seeds = np_rng.integers(np.iinfo(np.int32).max, size=int(config.arch.actor.num_envs_per_actor)).tolist()
            lt = ThreadLifetime(thread_name=f"Actor-{dev.index}-{thread_id}-idx-{idx}", thread_id=idx)
            th = get_actor_thread(env_factory, dev, parameter_server, rollout_pipeline, apply_fns, thread_keys[idx], config, seeds, logger,
                                  learner_devices, lt, transition)
            th.start()
            actor_threads.append(th)
            lifetimes.append(lt)

    eval_lifetime = ThreadLifetime("AsyncEvaluator", 0)
    async_evaluator = AsyncEvaluator(evaluator=evaluator, logger=logger, config=config, checkpointer=checkpointer,
                                     save_checkpoint=save_checkpoint, lifetime=eval_lifetime)
    async_evaluator.start()
    learner_thread = get_learner_thread(config, learn_step, learner_state, parameter_server, rollout_pipeline, logger, async_evaluator, key_e)
    start = time.perf_counter()
    learner_thread.start()
    learner_thread.join()
    print(f"Learner took {time.perf_counter() - start:.2f}s.")
    stop_all_actor_threads(lifetimes, parameter_server, rollout_pipeline, actor_threads)
    async_evaluator.wait_for_all_evaluations(timeout=600)
    async_evaluator.shutdown()
    async_evaluator.join()
    if config.arch.absolute_metric and async_evaluator.get_best_params() is not None:
        from stoix_b200.networks.base import build_param_tree

        final = learner_thread.learner_rollout.final_state.params.actor_params
        best = build_param_tree(final.spec, async_evaluator.get_best_params(), "action_head")
        if final.flat_bf16 is not None:
            best.flat_bf16 = ops.cast_bf16(best.flat)
        abs_eval, abs_envs = get_sebulba_eval_fn(env_factory, eval_act_fn, config, np_rng, evaluator_device, eval_multiplier=10)
        metrics = abs_eval(best, srandom.split(key_e, 2)[1])
        logger.log(metrics, int(config.arch.total_timesteps), int(config.arch.num_evaluation) - 1, LogEvent.ABSOLUTE)
        abs_envs.close()
        perf = float(metrics[config.env.eval_metric].float().mean().item())
    else:
        perf = float(async_evaluator.get_final_episode_return())
    evaluator_envs.close()
    logger.stop()
    return perf


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point (sebulba/ff_ppo.py:1026-1045): `python -m stoix_b200.systems.ppo.sebulba.ff_ppo k=v ...`"""
    import sys

    if cfg is None:
        cfg = compose("default_ff_ppo", overrides if overrides is not None else sys.argv[1:], config_dir="default/sebulba")
    t0 = time.perf_counter()
    perf = run_experiment(cfg)
    print(f"PPO experiment completed in {time.perf_counter() - t0:.2f}s with a final episode return of {perf}.")
    return perf


if __name__ == "__main__":
    hydra_entry_point()
