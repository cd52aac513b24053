"""The host driver every Anakin system shares: ranks, shard seeding, the CUDA-graph policy of the update step, the experiment loop
and the entry point.  None of it is algorithm code; a system module hands in its learner_setup and what really differs between
systems (how many network keys it splits, which parameter tree is the policy, how it evaluates).

  reference (JAX)                                   here
  ------------------------------------------------  ----------------------------------------------------------------------
  pmap over devices                                  one process per GPU (torchrun); world() = (rank, world size)
  one XLA program per learn() call                   update_once: the first update eager, the second captured into a CUDA
                                                     graph, every later one a replay
  run_experiment (learn, log, evaluate, checkpoint)  run_experiment below, once for all Anakin systems
"""
from __future__ import annotations

import copy
import gc
import os
import sys
import time
from types import SimpleNamespace
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import random as srandom
from stoix_b200.config import DictConfig, compose, to_container
from stoix_b200.envs.base import Environment, StepOut, TimeStep
from stoix_b200.evaluator import evaluator_setup, get_distribution_act_fn
from stoix_b200.networks.base import build_param_tree
from stoix_b200.systems.sac.sac_types import Transition
from stoix_b200.utils import make_env as environments
from stoix_b200.utils.checkpointing import Checkpointer
from stoix_b200.utils.logger import LogEvent, StoixLogger
from stoix_b200.utils.total_timestep_checker import check_total_timesteps

_M62 = (1 << 62) - 1


def world() -> Tuple[int, int]:
    """(rank, world size) of this process; (0, 1) without a process group."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def owner(fn: Callable, kind: type, what: str) -> Any:
    """The object `fn` is bound to, which must be a `kind`.  The arithmetic of apply / update runs in the CUDA kernels; what a learner
    needs from these callables is the description they are bound to (layer sizes, optimiser hyper-parameters)."""
    obj = getattr(fn, "__self__", None)
    if not isinstance(obj, kind):
        raise TypeError(f"{what} must be a bound method of a stoix_b200 {kind.__name__} (got {fn!r}); arbitrary callables cannot be "
                        "lowered onto the CUDA kernels")
    return obj


def reset_shards(env: Environment, shard_keys: Sequence[int], config: DictConfig, rank: int) -> Tuple[List[Any], List[TimeStep]]:
    """Reset the arch.update_batch_size env shards of this rank: shard u from split(shard_keys[u], num_envs), and an env with a
    `seed` gets one per (rank, shard) so that no two shards draw the same stream."""
    E = int(config.arch.num_envs)
    env_states: List[Any] = []
    timesteps: List[TimeStep] = []
    for u in range(int(config.arch.update_batch_size)):
        if hasattr(env, "seed"):
            env.seed = (int(config.arch.seed) + 7919 * rank + 15485863 * u) & ((1 << 63) - 1)
        st, ts = env.reset(srandom.split(shard_keys[u], E))
        env_states.append(st)
        timesteps.append(ts)
    return env_states, timesteps


def rank_seeds(key: int, n: int, rank: int, world_size: int) -> Tuple[int, ...]:
    """This rank's n step seeds: split `key` into n per rank, masked to 62 bits (the kernels add shard and call offsets to them)."""
    step_key = srandom.split(key, n * world_size)
    return tuple(step_key[n * rank + i] & _M62 for i in range(n))


def step_env(env: Environment, env_states: List[Any], u: int, action: torch.Tensor, out: StepOut, t: int) -> None:
    """Step shard u with `action` and write the transition into `out`: in place through env.step_into when the env has it,
    otherwise env.step and a copy of its TimeStep (done = terminated, truncated = last and not terminated)."""
    if hasattr(env, "step_into"):
        env.step_into(env_states[u], action, out, t)
        return
    env_states[u], ts = env.step(env_states[u], action)
    out.obs.copy_(ts.observation)
    out.next_obs.copy_(ts.extras["next_obs"])
    out.reward.copy_(ts.reward)
    torch.eq(ts.discount, 0.0, out=out.done)
    torch.gt(ts.last(), out.done, out=out.truncated)   # last and not terminated
    em = ts.extras["episode_metrics"]
    out.episode_return.copy_(em["episode_return"])
    out.episode_length.copy_(em["episode_length"])
    out.is_terminal_step.copy_(em["is_terminal_step"])


class Trajectory:
    """What the environment writes in one (device, update-batch) shard's T-step rollout, time-major.  Row t of obs is the
    observation step t acts on; row T is the carry, the first observation of the next rollout.  terminated / truncated are the
    env's flags (StepOut.done / .truncated).  With raw_obs the environment writes fp32 observations into obs_raw / next_obs_raw
    and obs / next_obs (obs_dtype) hold the normalised copies the networks read."""

    perms: Optional[torch.Tensor] = None   # (epochs, T*E) int32 minibatch shuffles of the update, allocated by shuffle()

    def __init__(self, T: int, E: int, D: int, device, obs_dtype=torch.float32, raw_obs: bool = False):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.T = T
        self.obs, self.next_obs = z(T + 1, E, D, dt=obs_dtype), z(T, E, D, dt=obs_dtype)
        self.obs_raw, self.next_obs_raw = (z(T + 1, E, D), z(T, E, D)) if raw_obs else (None, None)
        self.reward = z(T, E)
        self.terminated, self.truncated = z(T, E, dt=torch.uint8), z(T, E, dt=torch.uint8)
        self.episode_return, self.episode_length = z(T, E), z(T, E, dt=torch.int32)
        self.is_terminal_step = z(T, E, dt=torch.uint8)

    @property
    def env_obs(self) -> torch.Tensor:
        """(T+1, E, D) observations as the environment produced them (raw when normalising)."""
        return self.obs if self.obs_raw is None else self.obs_raw

    def step_out(self, t: int) -> StepOut:
        nxt = self.next_obs if self.next_obs_raw is None else self.next_obs_raw
        return StepOut(self.env_obs[t + 1], nxt[t], self.reward[t], self.terminated[t], self.truncated[t], self.episode_return[t],
                       self.episode_length[t], self.is_terminal_step[t])

    def carry_in(self) -> None:
        """The latest observation (row T of the previous rollout) is the first of this rollout; the finished trajectory stays
        readable until then."""
        self.env_obs[0].copy_(self.env_obs[self.T])

    def advance(self, env: Environment, env_state: Any) -> None:
        """Move the env's device-resident step counter past this rollout (graph replays then step fresh numbers)."""
        if hasattr(env, "advance"):
            env.advance(env_state, self.T)


def shuffle(shards: Sequence[Trajectory], epochs: int, seed: int, counter: torch.Tensor) -> None:
    """SHUFFLE MINIBATCHES for all epochs of an update: one keyed permutation of the T*E flat rows per (shard, epoch), at stream
    position `counter`, into shard.perms."""
    for u, sh in enumerate(shards):
        n = sh.reward.numel()
        if sh.perms is None:
            sh.perms = torch.zeros(epochs, n, dtype=torch.int32, device=counter.device)
        for ep in range(epochs):
            ops.make_permutation(n, seed + u, ep, dev_counter=counter, out=sh.perms[ep])


def shuffle_beside(built: Dict[str, Any], epochs: int, seed: int, rollout: Callable[[], None]) -> None:
    """shuffle() on built["side_stream"] while `rollout()` runs on the current stream: forked before it, joined after it.  The
    permutations depend on the seed and built["perm_ctr"] only, not on the rollout, which leaves most SMs idle."""
    main, side = torch.cuda.current_stream(), built["side_stream"]
    side.wait_stream(main)  # fork (a graph branch when captured)
    with torch.cuda.stream(side):
        shuffle(built["shards"], epochs, seed, built["perm_ctr"])
    rollout()
    main.wait_stream(side)  # join


def ensure_built(built: Dict[str, Any], build: Callable[[Any], None], state: Any) -> None:
    """Build a learner once, from its first learner state: build(state) fills `built` (with its "shards"), and each shard's carry
    row T starts from state.timestep[u].observation."""
    if not built:
        build(state)
        for sh, ts in zip(built["shards"], state.timestep):
            sh.env_obs[-1].copy_(ts.observation)


_EPISODE_FIELDS = ("episode_return", "episode_length", "is_terminal_step")


def learn(built: Dict[str, Any], build: Callable[[Any], None], step: Callable[[Any], None], state: Any, config: DictConfig,
          extra_fields: Sequence[str] = (), buffers: Sequence[Any] = ()) -> Tuple[List[TimeStep], Dict[str, torch.Tensor], torch.Tensor]:
    """The body of every Anakin learner_fn around its update step: ensure_built, then arch.num_updates_per_eval update_once calls
    (buffers: the replay buffers each step adds its T*E transitions to).  Returns the timesteps the next learn() starts from,
    the episode metrics (plus each shard's `extra_fields`) as (n_upd, U, T, E) tensors, and built["metrics"] after every update,
    stacked as (n_upd, *metrics.shape)."""
    ensure_built(built, build, state)
    shards, metrics = built["shards"], built["metrics"]
    n_upd = int(config.arch.num_updates_per_eval)
    fields = _EPISODE_FIELDS + tuple(extra_fields)
    dtype = lambda name: torch.bool if name == "is_terminal_step" else getattr(shards[0], name).dtype
    ep_out = {name: torch.empty(n_upd, len(shards), *getattr(shards[0], name).shape, dtype=dtype(name), device=metrics.device)
              for name in fields}
    train_out = torch.empty(n_upd, *metrics.shape, dtype=metrics.dtype, device=metrics.device)
    items = shards[0].reward.numel()
    for k in range(n_upd):
        update_once(built, bool(config.arch.get("cuda_graph", True)), step, state, buffers, items)
        for u, sh in enumerate(shards):
            for name in fields:
                ep_out[name][k, u].copy_(getattr(sh, name))
        train_out[k].copy_(metrics)
    timestep = [ts._replace(observation=sh.env_obs[-1]) for ts, sh in zip(state.timestep, shards)]
    return timestep, ep_out, train_out


def replay_buffers(config: DictConfig, key: int, rank: int, n_devices: int, make: Callable[[int, int, int], Any]) -> List[Any]:
    """This rank's replay buffers, one per update-batch shard: system.total_buffer_size / total_batch_size are split evenly over
    (device, shard) into config.system.buffer_size / batch_size, and buffer u = make(buffer_size, batch_size, seed) with
    seed = split(key, n_devices * U)[rank * U + u]."""
    U = int(config.arch.update_batch_size)
    assert int(config.system.total_buffer_size) % n_devices == 0, "The total buffer size should be divisible by the number of devices!"
    assert int(config.system.total_batch_size) % n_devices == 0, "The total batch size should be divisible by the number of devices!"
    config.system.buffer_size = int(config.system.total_buffer_size) // (n_devices * U)
    config.system.batch_size = int(config.system.total_batch_size) // (n_devices * U)
    seeds = srandom.split(key, n_devices * U)
    return [make(config.system.buffer_size, config.system.batch_size, seeds[rank * U + u]) for u in range(U)]


def warmup_fn(env: Environment, draw: Callable[[torch.Tensor, int, int], torch.Tensor], buffer_add_fn: Callable,
              config: DictConfig) -> Callable:
    """The warm-up of an off-policy system: system.warmup_steps environment steps of one shard, acting with
    draw(obs, key, t), added to the buffer as one Transition (done = timestep.last())."""
    W = int(config.system.warmup_steps)

    def warmup(env_state, timestep: TimeStep, buffer_state, key: int):
        obs_l, act_l, rew_l, done_l, nobs_l = [], [], [], [], []
        for t in range(W):
            obs = timestep.observation.float().clone()
            action = draw(obs, key, t)
            env_state, timestep = env.step(env_state, action)
            obs_l.append(obs), act_l.append(action), rew_l.append(timestep.reward.float())
            done_l.append(timestep.last().to(torch.uint8)), nobs_l.append(timestep.extras["next_obs"].float())
        if W > 0:
            st = lambda xs: torch.stack(xs).contiguous()
            buffer_add_fn(buffer_state, Transition(st(obs_l), st(act_l), st(rew_l), st(done_l), st(nobs_l), {}))
        return env_state, timestep, key, buffer_state

    return warmup


def update_once(built: Dict[str, Any], use_graph: bool, step: Callable, state: Any, buffers: Sequence[Any] = (),
                items_per_step: int = 0) -> None:
    """Run one update step `step(state)`.  The first call runs eagerly (module loading, NCCL warm-up) and sets built["eager_done"];
    with use_graph the next one captures the step into built["graph"], and every call from then on replays it.

    buffers: replay buffers whose host mirror `added` counts the items the step adds.  Capturing launches nothing, so the mirrors
    are restored around it, and each replay adds items_per_step to them."""
    if use_graph and built["eager_done"] and built["graph"] is None:
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        # No cyclic GC while the stream is capturing: collecting an older learner (its CUDAGraph is destroyed in the collector)
        # is "not permitted when stream is capturing" and would invalidate this capture.
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        added = [buf.added for buf in buffers]
        try:
            with torch.cuda.graph(g):
                step(state)
        finally:
            if gc_was_enabled:
                gc.enable()
        for buf, n in zip(buffers, added):
            buf.added = n
        built["graph"] = g
    if built["graph"] is not None:
        built["graph"].replay()
        for buf in buffers:
            buf.added += items_per_step
    else:
        step(state)
        built["eager_done"] = True


def get_final_step_metrics(metrics: Dict[str, torch.Tensor]) -> Tuple[Dict[str, torch.Tensor], bool]:
    """stoa.get_final_step_metrics: keep the entries of finished episodes, and say whether there were any."""
    mask = metrics["is_terminal_step"]
    has_final = bool(mask.any().item())
    out = {k: (v[mask] if has_final else v.reshape(-1)[:0]) for k, v in metrics.items() if k != "is_terminal_step"}
    return out, has_final


def _ff_evaluators(eval_env: Environment, key_e: int, network: Any, config: DictConfig) -> Tuple[Callable, Callable]:
    return evaluator_setup(eval_env=eval_env, key_e=key_e, eval_act_fn=get_distribution_act_fn(config, network.apply), config=config)


def _ff_best_tree(network: Any, tree: Any, flat: torch.Tensor) -> Any:
    best = build_param_tree(tree.spec, flat, "action_head")
    if tree.flat_bf16 is not None:
        best.flat_bf16 = ops.cast_bf16(flat)
    return best


def _timed_eval(evaluator: Callable, params: Any, key: int, learner_state: Any) -> Tuple[Dict[str, torch.Tensor], float]:
    # the evaluator normalises observations like the learner when the learner state carries running statistics
    rs = getattr(learner_state, "running_statistics", None)
    start_time = time.time()
    out = evaluator(params, key) if rs is None else evaluator(params, key, running_statistics=rs)
    torch.cuda.synchronize()
    elapsed_time = time.time() - start_time
    out["steps_per_second"] = torch.tensor(int(out["episode_length"].sum().item()) / max(elapsed_time, 1e-9))
    return out, float(out["episode_return"].mean().item())


def run_experiment(_config: DictConfig, setup: Callable, *, net_keys: int, policy: Callable[[Any], Any] = lambda s: s.params.actor_params,
                   make_evaluators: Callable = _ff_evaluators, best_tree: Callable = _ff_best_tree) -> float:
    """Run an Anakin experiment (ff_ppo.py:554-706): arch.num_evaluation rounds of learn, log, evaluate and checkpoint, then the
    absolute metric of the best parameters.  Returns the mean env.eval_metric of the last evaluation.

    setup: the system's learner_setup(env, (key, *network_keys), config) -> (learn, network, learner_state), with net_keys network keys.
    policy(learner_state): the parameter tree that is evaluated, tracked as the best and checkpointed (as params.actor_params).
    make_evaluators(eval_env, key_e, network, config) -> (evaluator, absolute_metric_evaluator).
    best_tree(network, tree, flat): the evaluable tree of `tree`'s layout over the best flat parameters."""
    config = copy.deepcopy(_config)
    rank, n_devices = world()
    config.num_devices = n_devices
    config.rank = rank
    config = check_total_timesteps(config, quiet=rank != 0)
    assert config.arch.num_updates >= config.arch.num_evaluation, \
        "Number of updates per evaluation must be less than total number of updates."

    env, eval_env = environments.make(config=config)
    key, key_e, *net = srandom.split(srandom.PRNGKey(config.arch.seed), num=2 + net_keys)
    learn, network, learner_state = setup(env, (key, *net), config)
    evaluator, absolute_metric_evaluator = make_evaluators(eval_env, key_e, network, config)

    steps_per_rollout = (n_devices * config.arch.num_updates_per_eval * config.system.rollout_length
                         * config.arch.update_batch_size * config.arch.num_envs)
    opt_steps_per_eval = config.arch.num_updates_per_eval * config.system.epochs * config.system.get("num_minibatches", 1)

    logger = StoixLogger(config)
    logger.log_config(to_container(config, resolve=True))
    save_checkpoint = config.logger.checkpointing.save_model
    if save_checkpoint:
        checkpointer = Checkpointer(metadata=to_container(config), model_name=config.system.system_name,
                                    **to_container(config.logger.checkpointing.save_args))

    max_episode_return = -float("inf")
    best_params = policy(learner_state).flat.clone()
    evaluator_output = None
    eval_step = 0
    for eval_step in range(config.arch.num_evaluation):
        start_time = time.time()
        learner_output = learn(learner_state)
        torch.cuda.synchronize()  # jax.block_until_ready (ff_ppo.py:619)
        elapsed_time = time.time() - start_time
        t = int(steps_per_rollout * (eval_step + 1))
        episode_metrics, ep_completed = get_final_step_metrics(learner_output.episode_metrics)
        episode_metrics["steps_per_second"] = torch.tensor(steps_per_rollout / elapsed_time)

        logger.log({"timestep": t}, t, eval_step, LogEvent.MISC)
        if ep_completed:
            logger.log(episode_metrics, t, eval_step, LogEvent.ACT)
        train_metrics = dict(learner_output.train_metrics)
        train_metrics["steps_per_second"] = torch.tensor(opt_steps_per_eval / elapsed_time)
        logger.log(train_metrics, t, eval_step, LogEvent.TRAIN)

        learner_state = learner_output.learner_state
        trained_params = policy(learner_state)
        evaluator_output, episode_return = _timed_eval(evaluator, trained_params, srandom.split(key_e, eval_step + 2)[-1], learner_state)
        logger.log(evaluator_output, t, eval_step, LogEvent.EVAL)

        if save_checkpoint and rank == 0:
            view = SimpleNamespace(params=SimpleNamespace(actor_params=trained_params))  # what Checkpointer.save reads
            checkpointer.save(timestep=t, unreplicated_learner_state=view, episode_return=episode_return)

        if config.arch.absolute_metric and max_episode_return <= episode_return:
            best_params = trained_params.flat.clone()
            max_episode_return = episode_return

    if config.arch.absolute_metric:
        t = int(steps_per_rollout * (eval_step + 1))
        best = best_tree(network, policy(learner_state), best_params)
        evaluator_output, _ = _timed_eval(absolute_metric_evaluator, best, srandom.split(key_e, 1)[0], learner_state)
        logger.log(evaluator_output, t, eval_step, LogEvent.ABSOLUTE)

    logger.stop()
    return float(evaluator_output[config.env.eval_metric].float().mean().item())


def entry_point(cfg: Optional[DictConfig], overrides: Optional[List[str]], config_name: str, run: Callable[[DictConfig], float],
                label: str) -> float:
    """The body of every Anakin hydra_entry_point (ff_ppo.py:709-727).  Without hydra-core the composition happens here, from
    `overrides` or the command line; under torchrun each process joins the NCCL group on its local GPU."""
    if cfg is None:
        cfg = compose(config_name, overrides if overrides is not None else sys.argv[1:], config_dir="default/anakin")
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    t0 = time.time()
    eval_performance = run(cfg)
    if world()[0] == 0:
        print(f"{label} experiment completed in {time.time() - t0:.2f} seconds.")
    return eval_performance
