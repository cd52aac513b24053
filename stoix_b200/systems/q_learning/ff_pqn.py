"""Anakin PQN (parallel Q-networks) on H100 -- drop-in for stoix/systems/q_learning/ff_pqn.py.

Same entry points and signatures (get_learner_fn :44-220, learner_setup :223-330, run_experiment, hydra_entry_point) on the
machinery of ff_ppo: one process per GPU, a T-step rollout of (Q forward, epsilon-greedy sampler, env step) launches, the
targets from one scan launch, keyed permutations instead of shuffled copies, and the whole update step captured into a CUDA
graph after the first eager update.  What is new:

  reference (JAX)                                     here (H100)
  --------------------------------------------------  -----------------------------------------------------------------
  epsilon_schedule(count // (epochs * nmb)) per step  evaluated on the device from the optimiser count word, inside the
  + EpsilonGreedy(q, eps).sample                      sampler (stx_epsilon_greedy): graph replays follow the schedule
  Q(concat(obs, next_obs[T-1]))[1:] over (T+1) E rows the rollout keeps q[t] = Q(obs[t]) (it needed it to act) and one
                                                      E-row forward adds q[T] = Q(obs[T]); targets read rows 1..T
  batch_q_lambda (max over A, reverse lax.scan)       one launch of K2's scan with the max fused into its load
  jax.grad(_q_loss_fn)                                stx_mlp_forward_train on rows gathered through the permutation,
                                                      stx_q_loss_grads, stx_mlp_backward
  chain(clip_by_global_norm, radam)                   one stx_clip_radam_step launch over the parameter arena

Reusing q[t+1] = Q(obs[t+1]) in place of Q(next_obs[t]) is exact in value: the two observations differ only where step t ended
an episode (auto-reset), and there d_t = gamma (1 - done_t) = 0 removes both v_t and G_{t+1} from G_t.  The same holds for the
last row, where the reference reads next_obs[T-1].

Learning-rate schedule, as the reference builds it: ff_pqn.py:263 passes only `epochs` to make_learning_rate, so the schedule's
steps per update are `epochs` (not epochs * num_minibatches) and lr(k) = q_lr (1 - (k // epochs) / num_updates).  With
system.decay_learning_rates=True (default False) the rate therefore reaches zero after num_updates / num_minibatches updates
and turns negative after that; this module keeps that arithmetic.

fp32 only: arch.precision=bf16 raises (the tensor-core kernels implement relu / 2 x 256 / Categorical only).
"""
from __future__ import annotations

import copy
import gc
import sys
import time
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput, LearnerFn, OnPolicyLearnerState
from stoix_b200.config import DictConfig, compose, instantiate, to_container
from stoix_b200.envs.base import Environment, StepOut, TimeStep
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.heads import DiscreteQNetworkHead
from stoix_b200.utils import make_env as environments
from stoix_b200.utils.logger import LogEvent, StoixLogger
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
from stoix_b200.utils.training import make_learning_rate


def _world() -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _refuse_bf16(config: DictConfig) -> None:
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for ff_pqn: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not a Q network with its activation, LayerNorm and Q loss; use arch.precision=f32")


class _Shard:
    """Trajectory buffers of one (device, update-batch) shard, time-major: the Transition fields (dqn_types.py:9-15) plus the Q rows."""

    def __init__(self, T: int, E: int, D: int, A: int, device):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs = z(T + 1, E, D)                     # row t = last_timestep.observation of step t; row T = the next rollout's first
        self.next_obs = z(T, E, D)                    # timestep.extras["next_obs"]
        self.q = z(T + 1, E, A)                       # q[t] = Q(obs[t]) with the rollout's parameters
        self.action = z(T, E, dt=torch.int32)
        self.reward = z(T, E)
        self.done = z(T, E, dt=torch.uint8)           # terminated; the targets use done | truncated = timestep.last() (ff_pqn.py:84)
        self.truncated = z(T, E, dt=torch.uint8)
        self.episode_return = z(T, E)
        self.episode_length = z(T, E, dt=torch.int32)
        self.is_terminal_step = z(T, E, dt=torch.uint8)
        self.epsilon = z(T, E)                        # info["epsilon"], info["update_no"] (ff_pqn.py:85-86)
        self.update_no = z(T, E, dt=torch.int32)
        self.targets = z(T, E)
        self.perms = None

    def step_out(self, t: int) -> StepOut:
        return StepOut(self.obs[t + 1], self.next_obs[t], self.reward[t], self.done[t], self.truncated[t], self.episode_return[t],
                       self.episode_length[t], self.is_terminal_step[t])


def minibatch_grads(spec: ops.MlpSpec, params: torch.Tensor, rows: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]],
                    delta: float, grads: torch.Tensor, metric: torch.Tensor, ws: torch.Tensor, q_mb: torch.Tensor, dq_mb: torch.Tensor) -> None:
    """jax.grad(_q_loss_fn) + pmean over "batch" of one minibatch (ff_pqn.py:127-170).  rows: per shard (obs (B, D), minibatch row
    indices (mb), action (B), targets (B)).  Each shard runs the train-mode forward on its gathered rows, the Q-loss kernel and the
    backward; `grads` receives the mean over the U shards (the first overwrites, weight 1/U each) and metric[0] += mean q_loss."""
    U = len(rows)
    for u, (x, idx, action, targets) in enumerate(rows):
        ops.mlp_forward_train(spec, params, x, ws, out=q_mb, row_idx=idx)
        ops.q_loss_grads(q_mb, idx, action, targets, delta, dq_mb, metric, weight=1.0 / U)
        ops.mlp_backward(spec, params, x, dq_mb, ws, net_grad=grads, grad_weight=1.0 / U, overwrite=(u == 0), row_idx=idx)


def get_learner_fn(
    env: Environment,
    q_apply_fn: Callable,
    q_update_fn: Callable,
    epsilon_schedule: Callable,
    config: DictConfig,
) -> LearnerFn[OnPolicyLearnerState]:
    """Get the learner function (ff_pqn.py:44-220).

    q_apply_fn: the bound `apply` of the Q network (a FeedForwardActor with a DiscreteQNetworkHead); q_update_fn: the bound `update`
    of chain(clip_by_global_norm, radam); epsilon_schedule: linear_schedule / constant_schedule of this module (their constants are
    evaluated on the device).  The arithmetic runs in the kernels; these carry the shapes and hyper-parameters."""
    q_net = getattr(q_apply_fn, "__self__", None)
    if not isinstance(q_net, Actor) or not isinstance(q_net.action_head, DiscreteQNetworkHead):
        raise TypeError("get_learner_fn: q_apply_fn must be the bound `apply` of a FeedForwardActor with a DiscreteQNetworkHead")
    opt = getattr(q_update_fn, "__self__", None)
    if not isinstance(opt, optax.GradientTransformation) or opt.rule != "radam":
        raise TypeError("get_learner_fn: q_update_fn must be the bound `update` of chain(clip_by_global_norm(..), radam(..))")
    if not hasattr(epsilon_schedule, "device_schedule"):
        raise TypeError("get_learner_fn: epsilon_schedule must come from ff_pqn.linear_schedule / constant_schedule")
    _refuse_bf16(config)
    rank, world = _world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, nmb = int(sysc.epochs), int(sysc.num_minibatches)
    B = T * E
    assert B % nmb == 0, "rollout_length * num_envs must be divisible by num_minibatches"
    mb = B // nmb
    use_graph = bool(arch.get("cuda_graph", True))
    has_step_into = hasattr(env, "step_into")
    gamma, q_lambda, delta = float(sysc.gamma), float(sysc.q_lambda), float(sysc.huber_loss_parameter)
    sched = epsilon_schedule.device_schedule(epochs * nmb)
    built: Dict[str, Any] = {}

    def _build(state: OnPolicyLearnerState) -> None:
        tree = state.params
        spec = tree.spec
        dev = tree.flat.device
        D, A = spec.sizes[0], spec.sizes[-1]
        lr_sched = opt.schedule
        plan = ops.AdamPlan([(0, spec.param_count, opt.init_lr, opt.max_grad_norm)], dev, b1=opt.adam.b1, b2=opt.adam.b2, eps=opt.adam.eps,
                            decay=lr_sched is not None, steps_per_update=getattr(lr_sched, "steps_per_update", 1),
                            num_updates=getattr(lr_sched, "num_updates", 1), **opt.plan_kwargs())
        plan.counts = tree.arena_counts  # the optimiser counters live in the learner state (so a checkpoint carries them)
        built.update(
            spec=spec, dev=dev, plan=plan, shards=[_Shard(T, E, D, A, dev) for _ in range(U)],
            grads=torch.zeros(tree.arena.numel(), dtype=torch.float32, device=dev),
            metrics=torch.zeros(epochs, nmb, dtype=torch.float32, device=dev),
            ws=ops.mlp_train_workspace(spec, mb, dev),
            q_mb=torch.zeros(mb, A, dtype=torch.float32, device=dev), dq_mb=torch.zeros(mb, A, dtype=torch.float32, device=dev),
            roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # epsilon-greedy call index
            perm_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # shuffle stream index
            side_stream=torch.cuda.Stream(device=dev), graph=None, eager_done=False,
        )

    def _rollout_phase(state: OnPolicyLearnerState) -> None:
        """STEP ENVIRONMENT FOR ROLLOUT LENGTH (ff_pqn.py:54-95), then q[T] = Q(obs[T]) for the targets."""
        b = built
        tree = state.params
        count = b["plan"].counts[0:1]  # optax.tree_get(opt_states, "count") (ff_pqn.py:69)
        for u in range(U):
            sh: _Shard = b["shards"][u]
            for t in range(T):
                ops.mlp_forward(b["spec"], tree.flat, sh.obs[t], out=sh.q[t], ws_key="pqn")
                ops.epsilon_greedy(sh.q[t], sched, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], count=count, out=sh.action[t],
                                   epsilon_out=sh.epsilon[t], update_no_out=sh.update_no[t])
                if has_step_into:
                    env.step_into(state.env_state[u], sh.action[t], sh.step_out(t), t)
                else:
                    new_state, ts = env.step(state.env_state[u], sh.action[t])
                    state.env_state[u] = new_state
                    out = sh.step_out(t)
                    out.obs.copy_(ts.observation)
                    out.next_obs.copy_(ts.extras["next_obs"])
                    out.reward.copy_(ts.reward)
                    out.done.copy_(ts.discount == 0.0)
                    out.truncated.copy_(ts.last() & (ts.discount != 0.0))
                    em = ts.extras["episode_metrics"]
                    out.episode_return.copy_(em["episode_return"])
                    out.episode_length.copy_(em["episode_length"])
                    out.is_terminal_step.copy_(em["is_terminal_step"])
            ops.mlp_forward(b["spec"], tree.flat, sh.obs[T], out=sh.q[T], ws_key="pqn")

    def _targets_phase(state: OnPolicyLearnerState) -> None:
        """CALCULATE Q LAMBDA TARGETS (ff_pqn.py:97-120) with the rollout's parameters."""
        for u in range(U):
            sh: _Shard = built["shards"][u]
            ops.q_lambda(sh.q[1:], sh.reward, sh.done, sh.truncated, gamma, q_lambda, out=sh.targets)

    def _shuffle_phase(state: OnPolicyLearnerState) -> None:
        """SHUFFLE MINIBATCHES (ff_pqn.py:184-197): one keyed permutation per (shard, epoch), independent of the rollout."""
        b = built
        for u in range(U):
            sh = b["shards"][u]
            if sh.perms is None:
                sh.perms = torch.zeros(epochs, B, dtype=torch.int32, device=b["dev"])
            for ep in range(epochs):
                ops.make_permutation(B, state.key[1] + u, ep, dev_counter=b["perm_ctr"], out=sh.perms[ep])

    def _update_phase(state: OnPolicyLearnerState, shuffled: bool = False) -> None:
        """UPDATE EPOCHS (ff_pqn.py:122-207)."""
        b = built
        if not shuffled:
            _shuffle_phase(state)
        spec, tree = b["spec"], state.params
        D = spec.sizes[0]
        metrics, grads, ws, q_mb, dq_mb = b["metrics"], b["grads"], b["ws"], b["q_mb"], b["dq_mb"]
        opt_state = state.opt_states
        metrics.zero_()
        for ep in range(epochs):
            for i in range(nmb):  # _update_minibatch (ff_pqn.py:127-180)
                rows = [(sh.obs[:T].view(B, D), sh.perms[ep, i * mb:(i + 1) * mb], sh.action.view(B), sh.targets.view(B)) for sh in b["shards"]]
                minibatch_grads(spec, tree.flat, rows, delta, grads, metrics[ep, i:i + 1], ws, q_mb, dq_mb)
                if world > 1:  # pmean over "device": summed by NCCL here, scaled in the optimiser step
                    dist.all_reduce(grads, op=dist.ReduceOp.SUM)
                ops.clip_adam_step(b["plan"], tree.arena, grads, opt_state.mu, opt_state.nu, grad_scale=1.0 / world)
        if world > 1:
            dist.all_reduce(metrics, op=dist.ReduceOp.SUM)
            metrics.mul_(1.0 / world)

    def _carry_in_phase(state: OnPolicyLearnerState) -> None:
        for u in range(U):
            sh = built["shards"][u]
            sh.obs[0].copy_(sh.obs[T])

    def _advance_phase(state: OnPolicyLearnerState) -> None:
        b = built
        for u in range(U):
            if hasattr(env, "advance"):
                env.advance(state.env_state[u], T)
        ops.counter_add(b["roll_ctr"], T)
        ops.counter_add(b["perm_ctr"], epochs)

    def _update_step(state: OnPolicyLearnerState) -> None:
        """A single update (ff_pqn.py:50-210), in place on the learner state; the shuffles run on a side stream under the rollout."""
        _carry_in_phase(state)
        main = torch.cuda.current_stream()
        side = built["side_stream"]
        side.wait_stream(main)
        with torch.cuda.stream(side):
            _shuffle_phase(state)
        _rollout_phase(state)
        _targets_phase(state)
        main.wait_stream(side)
        _update_phase(state, shuffled=True)
        _advance_phase(state)

    def learner_fn(learner_state: OnPolicyLearnerState) -> AnakinExperimentOutput[OnPolicyLearnerState]:
        """Run arch.num_updates_per_eval update steps (ff_pqn.py:212-226)."""
        learner_fn.ensure_built(learner_state)
        b = built
        n_upd = int(arch.num_updates_per_eval)
        dev = b["dev"]
        ep_out = {
            "episode_return": torch.empty(n_upd, U, T, E, device=dev),
            "episode_length": torch.empty(n_upd, U, T, E, dtype=torch.int32, device=dev),
            "is_terminal_step": torch.empty(n_upd, U, T, E, dtype=torch.bool, device=dev),
            "epsilon": torch.empty(n_upd, U, T, E, device=dev),
            "update_no": torch.empty(n_upd, U, T, E, dtype=torch.int32, device=dev),
        }
        train_out = torch.empty(n_upd, epochs, nmb, device=dev)
        for k in range(n_upd):
            if use_graph and b["eager_done"] and b["graph"] is None:
                g = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                gc.collect()  # no cyclic GC while capturing (see ff_ppo)
                gc_was_enabled = gc.isenabled()
                gc.disable()
                try:
                    with torch.cuda.graph(g):
                        _update_step(learner_state)
                finally:
                    if gc_was_enabled:
                        gc.enable()
                b["graph"] = g
            if b["graph"] is not None:
                b["graph"].replay()
            else:
                _update_step(learner_state)  # the first update runs eagerly (module loading, NCCL warm-up)
                b["eager_done"] = True
            for u in range(U):
                sh = b["shards"][u]
                for name in ("episode_return", "episode_length", "is_terminal_step", "epsilon", "update_no"):
                    ep_out[name][k, u].copy_(getattr(sh, name))
            train_out[k].copy_(b["metrics"])
        new_ts = [learner_state.timestep[u]._replace(observation=b["shards"][u].obs[T]) for u in range(U)]
        learner_state = learner_state._replace(timestep=new_ts)
        return AnakinExperimentOutput(learner_state=learner_state, episode_metrics=ep_out, train_metrics={"q_loss": train_out})

    learner_fn.built = built
    learner_fn.update_step = _update_step
    learner_fn.phases = {"rollout": _rollout_phase, "targets": _targets_phase, "shuffle": _shuffle_phase, "update": _update_phase}

    def _ensure_built(st: OnPolicyLearnerState) -> None:
        if not built:
            _build(st)
            for u in range(U):
                built["shards"][u].obs[T].copy_(st.timestep[u].observation)

    learner_fn.ensure_built = _ensure_built
    return learner_fn


def linear_schedule(init_value: float, end_value: float, transition_steps: float) -> Callable:
    """optax.linear_schedule (transition_begin 0), evaluated in fp32 like the sampler kernel; `device_schedule(steps_per_update)` gives
    the constants stx_epsilon_greedy evaluates on the device."""
    import numpy as np

    f = np.float32

    def schedule(count):
        if not transition_steps > 0:
            return f(init_value)
        c = min(max(f(count), f(0)), f(transition_steps))
        frac = f(1) - f(c) / f(transition_steps)
        return (f(init_value) - f(end_value)) * f(frac) + f(end_value)

    schedule.device_schedule = lambda spu: ops.epsilon_schedule_struct(init_value, end_value, transition_steps, spu, decay=True)
    return schedule


def constant_schedule(value: float) -> Callable:
    """optax.constant_schedule."""
    import numpy as np

    schedule = lambda count: np.float32(value)
    schedule.device_schedule = lambda spu: ops.epsilon_schedule_struct(value, value, 0.0, spu, decay=False)
    return schedule


def learner_setup(env: Environment, keys: Tuple[int, int], config: DictConfig) -> Tuple[LearnerFn[OnPolicyLearnerState], Actor, OnPolicyLearnerState]:
    """Initialise learner_fn, network, optimiser, environment and states (ff_pqn.py:223-330).  Returns the EVAL network (epsilon =
    system.evaluation_epsilon) as the second element, which is what the reference hands to the evaluator."""
    _refuse_bf16(config)
    rank, world = _world()
    device = torch.device("cuda", torch.cuda.current_device())
    action_dim = int(env.action_space().num_values)
    config.system.action_dim = action_dim
    key, q_net_key = keys

    torso = instantiate(config.network.actor_network.pre_torso)
    head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.training_epsilon)
    q_network = Actor(torso=torso, action_head=head)
    eval_head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.evaluation_epsilon)
    eval_q_network = Actor(torso=torso, action_head=eval_head)

    q_lr = make_learning_rate(config.system.q_lr, config, config.system.epochs)  # epochs only, as ff_pqn.py:263 (module docstring)
    q_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.radam(q_lr))

    init_x = env.observation_space().generate_value()[None, ...].to(device)
    spec = q_network.spec_for(init_x.shape[-1])
    arena = torch.zeros((spec.param_count + 7) // 8 * 8, dtype=torch.float32, device=device)
    params = q_network.init(q_net_key, init_x, flat=arena)
    params.arena = arena
    mu, nu = torch.zeros_like(arena), torch.zeros_like(arena)
    counts = torch.zeros(2, dtype=torch.int32, device=device)   # {radam count, schedule count}, stepped in place by the learner
    opt_states = optax.OptState(counts[0:1], mu, nu, counts[1:2])
    params.arena_mu, params.arena_nu, params.arena_counts = mu, nu, counts
    if config.system.decay_epsilon:
        epsilon_schedule = linear_schedule(1.0, float(config.system.training_epsilon),
                                           float(config.arch.num_updates) * float(config.system.exploration_fraction))
    else:
        epsilon_schedule = constant_schedule(float(config.system.training_epsilon))

    learn = get_learner_fn(env, q_network.apply, q_optim.update, epsilon_schedule, config)

    U, E = int(config.arch.update_batch_size), int(config.arch.num_envs)
    env_states: List[Any] = []
    timesteps: List[TimeStep] = []
    shard_keys = srandom.split(key, U + 1)
    for u in range(U):
        if hasattr(env, "seed"):
            env.seed = (int(config.arch.seed) + 7919 * rank + 15485863 * u) & ((1 << 63) - 1)
        st, ts = env.reset(srandom.split(shard_keys[u], E))
        env_states.append(st)
        timesteps.append(ts)

    if config.logger.checkpointing.load_model:
        from stoix_b200.utils.checkpointing import Checkpointer

        loaded = Checkpointer(model_name=config.system.system_name, **to_container(config.logger.checkpointing.load_args))
        loaded.restore_params(arena)

    step_key = srandom.split(shard_keys[U], 2 * world)
    rollout_seed = step_key[2 * rank] & ((1 << 62) - 1)
    shuffle_seed = step_key[2 * rank + 1] & ((1 << 62) - 1)
    init_learner_state = OnPolicyLearnerState(params=params, opt_states=opt_states, key=(rollout_seed, shuffle_seed), env_state=env_states,
                                              timestep=timesteps)
    return learn, eval_q_network, init_learner_state


class _QParams(NamedTuple):
    actor_params: Any  # the Checkpointer stores the arenas of params.actor_params


class _CheckpointView(NamedTuple):
    params: _QParams


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_pqn.py:333-485)."""
    from stoix_b200.evaluator import evaluator_setup, get_distribution_act_fn
    from stoix_b200.systems.ppo.anakin.ff_ppo import get_final_step_metrics

    config = copy.deepcopy(_config)
    rank, world = _world()
    config.num_devices, config.rank = world, rank
    config = check_total_timesteps(config, quiet=rank != 0)
    assert config.arch.num_updates >= config.arch.num_evaluation, "Number of updates per evaluation must be less than total number of updates."
    env, eval_env = environments.make(config=config)
    key, key_e, q_net_key = srandom.split(srandom.PRNGKey(config.arch.seed), num=3)
    learn, eval_q_network, learner_state = learner_setup(env, (key, q_net_key), config)
    evaluator, absolute_metric_evaluator = evaluator_setup(eval_env=eval_env, key_e=key_e,
                                                           eval_act_fn=get_distribution_act_fn(config, eval_q_network.apply), config=config)
    steps_per_rollout = world * config.arch.num_updates_per_eval * config.system.rollout_length * config.arch.update_batch_size * config.arch.num_envs
    logger = StoixLogger(config)
    logger.log_config(to_container(config, resolve=True))
    save_checkpoint = config.logger.checkpointing.save_model
    if save_checkpoint:
        from stoix_b200.utils.checkpointing import Checkpointer

        checkpointer = Checkpointer(metadata=to_container(config), model_name=config.system.system_name,
                                    **to_container(config.logger.checkpointing.save_args))
    max_episode_return = -float("inf")
    best_params = learner_state.params.flat.clone()
    evaluator_output = None
    eval_step = 0
    for eval_step in range(config.arch.num_evaluation):
        start_time = time.time()
        learner_output = learn(learner_state)
        torch.cuda.synchronize()
        elapsed_time = time.time() - start_time
        t = int(steps_per_rollout * (eval_step + 1))
        episode_metrics, ep_completed = get_final_step_metrics(learner_output.episode_metrics)
        episode_metrics["steps_per_second"] = torch.tensor(steps_per_rollout / elapsed_time)
        logger.log({"timestep": t}, t, eval_step, LogEvent.MISC)
        if ep_completed:
            logger.log(episode_metrics, t, eval_step, LogEvent.ACT)
        train_metrics = dict(learner_output.train_metrics)
        opt_steps_per_eval = config.arch.num_updates_per_eval * config.system.epochs * config.system.num_minibatches
        train_metrics["steps_per_second"] = torch.tensor(opt_steps_per_eval / elapsed_time)
        logger.log(train_metrics, t, eval_step, LogEvent.TRAIN)
        start_time = time.time()
        trained_params = learner_output.learner_state.params
        evaluator_output = evaluator(trained_params, srandom.split(key_e, eval_step + 2)[-1])
        torch.cuda.synchronize()
        elapsed_time = time.time() - start_time
        episode_return = float(evaluator_output["episode_return"].mean().item())
        evaluator_output["steps_per_second"] = torch.tensor(int(evaluator_output["episode_length"].sum().item()) / max(elapsed_time, 1e-9))
        logger.log(evaluator_output, t, eval_step, LogEvent.EVAL)
        if save_checkpoint and rank == 0:
            checkpointer.save(timestep=t, unreplicated_learner_state=_CheckpointView(_QParams(trained_params)), episode_return=episode_return)
        if config.arch.absolute_metric and max_episode_return <= episode_return:
            best_params = trained_params.flat.clone()
            max_episode_return = episode_return
        learner_state = learner_output.learner_state
    if config.arch.absolute_metric:
        from stoix_b200.networks.base import build_param_tree

        start_time = time.time()
        t = int(steps_per_rollout * (eval_step + 1))
        best_tree = build_param_tree(learner_state.params.spec, best_params, "action_head")
        evaluator_output = absolute_metric_evaluator(best_tree, srandom.split(key_e, 1)[0])
        torch.cuda.synchronize()
        elapsed_time = time.time() - start_time
        evaluator_output["steps_per_second"] = torch.tensor(int(evaluator_output["episode_length"].sum().item()) / max(elapsed_time, 1e-9))
        logger.log(evaluator_output, t, eval_step, LogEvent.ABSOLUTE)
    logger.stop()
    return float(evaluator_output[config.env.eval_metric].float().mean().item())


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_pqn: `python -m stoix_b200.systems.q_learning.ff_pqn arch.total_num_envs=1024 ...`"""
    import os

    if cfg is None:
        cfg = compose("default_ff_pqn", overrides if overrides is not None else sys.argv[1:], config_dir="default/anakin")
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    t0 = time.time()
    eval_performance = run_experiment(cfg)
    if _world()[0] == 0:
        print(f"PQN experiment completed in {time.time() - t0:.2f} seconds.")
    return eval_performance


if __name__ == "__main__":
    hydra_entry_point()
