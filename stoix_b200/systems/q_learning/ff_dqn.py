"""Anakin DQN on H100 -- drop-in for stoix/systems/q_learning/ff_dqn.py, and the one learner body of ff_ddqn, ff_mdqn and ff_dqn_reg.

Same entry points and signatures (get_warmup_fn :37-89, get_learner_fn :92-258, learner_setup :261-414, run_experiment :417-556,
hydra_entry_point).  The four reference systems differ only in `_q_loss_fn`; here each is a `loss` rule of one per-row kernel
(stx_q_td_loss_grads), chosen by the thin modules ff_ddqn.py, ff_mdqn.py and ff_dqn_reg.py:

  rule                     reference loss                                          extra forward per shard and epoch
  -----------------------  ------------------------------------------------------  ---------------------------------------
  q_learning               utils/loss.py:106-124                                   -
  double_q_learning        utils/loss.py:127-146, selector Q(online, next_obs)     online on next_obs (ff_ddqn.py:154-155)
  munchausen_q_learning    utils/loss.py:190-223, Q(target, obs) for log pi        target on obs: ONE target forward over the
                                                                                   stacked (obs | next_obs) rows (ff_mdqn.py:154)
  q_learning_reg           q_learning + regularizer_coeff mean(q_tm1[a])           - (ff_dqn_reg.py:165-176)

  reference (JAX)                                      here (H100)
  ---------------------------------------------------  ------------------------------------------------------------------
  flashbax item buffer, int action (dqn_types.py)      discrete device ring (stx_replay_add_discrete / _sample_discrete):
                                                       one launch writes obs and next_obs as one (2M, D) block
  EpsilonGreedy(q, training_epsilon).sample            stx_mlp_forward + stx_epsilon_greedy (constant schedule) per step
  jax.grad(_q_loss_fn)                                 stx_mlp_forward_train (online, obs), stx_mlp_forward (target), the
                                                       loss kernel, stx_mlp_backward
  chain(clip_by_global_norm, adam(eps=1e-5))           one stx_clip_adam_step launch over the online arena
  optax.incremental_update after every step            one stx_polyak_update launch after every optimiser step
  one XLA program per learn() call                     one CUDA graph per update step (rollout + add + epochs), replayed

Every random stream position (epsilon-greedy calls, ring samples) is a device counter, so graph replays draw fresh numbers.
done = timestep.last() (ff_dqn.py:121): truncation cuts the bootstrap too, as in the reference.
fp32 only: arch.precision=bf16 raises.
"""
from __future__ import annotations

import copy
import gc
import os
import sys
import time
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput
from stoix_b200.config import DictConfig, compose, instantiate, to_container
from stoix_b200.envs.base import Environment, StepOut, TimeStep
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import build_param_tree
from stoix_b200.networks.heads import DiscreteQNetworkHead
from stoix_b200.systems.q_learning.dqn_types import Transition
from stoix_b200.systems.sac.sac_types import OffPolicyLearnerState, OnlineAndTarget
from stoix_b200.utils import make_env as environments
from stoix_b200.utils.logger import LogEvent, StoixLogger
from stoix_b200.utils.replay import DiscreteTransitionBuffer
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
from stoix_b200.utils.training import make_learning_rate

LOSSES = tuple(ops.Q_RULES)
_NAMES = {"q_learning": "DQN", "double_q_learning": "DDQN", "munchausen_q_learning": "MDQN", "q_learning_reg": "DQN-Reg"}


def _world() -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _refuse_unsupported(config: DictConfig) -> None:
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for the DQN family: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not a Q network with its activation, LayerNorm and Q loss; use arch.precision=f32")
    target = str(config.network.actor_network.action_head.get("_target_", ""))
    if not target.endswith("DiscreteQNetworkHead"):
        raise ValueError(f"the DQN family here runs the plain Q head (network=mlp_dqn); action head {target!r} (dueling, noisy, "
                         "distributional) is not implemented")


def loss_hyper(loss: str, config: DictConfig):
    """The StxQTdHyper of `loss` from config.system (the keys of system/q_learning/ff_{dqn,mdqn,dqn_reg}.yaml)."""
    s = config.system
    kw = dict(gamma=float(s.gamma), max_abs_reward=float(s.max_abs_reward), huber_delta=float(s.huber_loss_parameter))
    if loss == "munchausen_q_learning":
        kw.update(entropy_temperature=float(s.entropy_temperature), munchausen_coefficient=float(s.munchausen_coefficient),
                  clip_value_min=float(s.clip_value_min))
    if loss == "q_learning_reg":
        kw.update(regularizer_coeff=float(s.regularizer_coeff))
    return ops.q_td_hyper(**kw)


class _Rollout:
    """Trajectory buffers of one (device, update-batch) shard, time-major: the Transition fields (dqn_types.py) plus the Q rows."""

    def __init__(self, T: int, E: int, D: int, A: int, device):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs = z(T + 1, E, D)               # row t = last_timestep.observation of step t; row T = the next rollout's first
        self.next_obs = z(T, E, D)              # timestep.extras["next_obs"]
        self.q = z(T, E, A)                     # Q(online, obs[t]), the rows the sampler acted on
        self.action = z(T, E, dt=torch.int32)
        self.reward = z(T, E)
        self.terminated = z(T, E, dt=torch.uint8)
        self.truncated = z(T, E, dt=torch.uint8)
        self.done = z(T, E, dt=torch.uint8)     # timestep.last() = terminated | truncated (ff_dqn.py:121)
        self.episode_return = z(T, E)
        self.episode_length = z(T, E, dt=torch.int32)
        self.is_terminal_step = z(T, E, dt=torch.uint8)
        self.T = T

    def step_out(self, t: int) -> StepOut:
        return StepOut(self.obs[t + 1], self.next_obs[t], self.reward[t], self.terminated[t], self.truncated[t], self.episode_return[t],
                       self.episode_length[t], self.is_terminal_step[t])

    def transition(self) -> Transition:
        return Transition(self.obs[: self.T], self.action, self.reward, self.done, self.next_obs,
                          {"episode_return": self.episode_return, "episode_length": self.episode_length, "is_terminal_step": self.is_terminal_step})


class Batch(NamedTuple):
    """One sampled batch of M transitions: xs (2M, D) = obs rows then next_obs rows; action, reward, done (M)."""
    xs: torch.Tensor
    action: torch.Tensor
    reward: torch.Tensor
    done: torch.Tensor


class Work(NamedTuple):
    """Workspaces of batch_grads for M rows: ws (train-mode forward), q_tm1 (M, A), q_tgt (2M, A), q_sel (M, A), dq (M, A)."""
    ws: torch.Tensor
    q_tm1: torch.Tensor
    q_tgt: torch.Tensor
    q_sel: torch.Tensor
    dq: torch.Tensor


def make_work(spec: ops.MlpSpec, M: int, device) -> Work:
    A = spec.sizes[-1]
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
    return Work(ops.mlp_train_workspace(spec, M, device), z(M, A), z(2 * M, A), z(M, A), z(M, A))


def make_batch(M: int, D: int, device) -> Batch:
    return Batch(torch.zeros(2 * M, D, device=device), torch.zeros(M, dtype=torch.int32, device=device), torch.zeros(M, device=device),
                 torch.zeros(M, dtype=torch.uint8, device=device))


def batch_grads(loss: str, spec: ops.MlpSpec, online: torch.Tensor, target: torch.Tensor, batches: Sequence[Batch], hyper, grads: torch.Tensor,
                metric: torch.Tensor, work: Work) -> None:
    """jax.grad(_q_loss_fn) + pmean over "batch" of one epoch (ff_dqn.py:147-200): per shard the online train-mode forward on obs,
    the target forward on next_obs (MDQN: on obs and next_obs in one launch; DDQN adds the online forward on next_obs), the loss
    kernel and the backward.  `grads` receives the mean over the U shards (the first overwrites, weight 1/U each) and
    metric[0] += mean q_loss."""
    U = len(batches)
    q_tm1, q_tgt, q_sel, dq = work.q_tm1, work.q_tgt, work.q_sel, work.dq
    for u, b in enumerate(batches):
        M = int(b.action.numel())
        obs, nxt = b.xs[:M], b.xs[M:]
        ops.mlp_forward_train(spec, online, obs, work.ws, out=q_tm1)
        q_aux = None
        if loss == "munchausen_q_learning":
            ops.mlp_forward(spec, target, b.xs, out=q_tgt, ws_key="dqn_target")
            q_aux = q_tgt[:M]
        else:
            ops.mlp_forward(spec, target, nxt, out=q_tgt[M:], ws_key="dqn_target")
            if loss == "double_q_learning":
                q_aux = ops.mlp_forward(spec, online, nxt, out=q_sel, ws_key="dqn_selector")
        ops.q_td_loss_grads(loss, q_tm1, q_tgt[M:], b.action, b.reward, hyper, dq, metric, done=b.done, q_aux=q_aux, weight=1.0 / U)
        ops.mlp_backward(spec, online, obs, dq, work.ws, net_grad=grads, grad_weight=1.0 / U, overwrite=(u == 0))


def _owner(fn, kind, what):
    obj = getattr(fn, "__self__", None)
    if not isinstance(obj, kind):
        raise TypeError(f"{what} must be a bound method of a stoix_b200 {kind.__name__} (got {fn!r}); arbitrary callables cannot be "
                        "lowered onto the CUDA kernels")
    return obj


def get_warmup_fn(env: Environment, q_params: OnlineAndTarget, q_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """ff_dqn.py:37-89: `warmup_steps` environment steps with the initial online parameters and the training epsilon, added to
    the buffer (one shard per call)."""
    W = int(config.system.warmup_steps)

    def warmup(env_state, timestep: TimeStep, buffer_state, key: int):
        obs_l, act_l, rew_l, done_l, nobs_l = [], [], [], [], []
        for t in range(W):
            obs = timestep.observation.float().clone()
            action = q_apply_fn(q_params.online, obs).sample(seed=key, offset=t)
            env_state, timestep = env.step(env_state, action)
            obs_l.append(obs), act_l.append(action.to(torch.int32)), rew_l.append(timestep.reward.float())
            done_l.append(timestep.last().to(torch.uint8)), nobs_l.append(timestep.extras["next_obs"].float())
        if W > 0:
            st = lambda xs: torch.stack(xs).contiguous()
            buffer_add_fn(buffer_state, Transition(st(obs_l), st(act_l), st(rew_l), st(done_l), st(nobs_l), {}))
        return env_state, timestep, key, buffer_state

    return warmup


def get_learner_fn(env: Environment, q_apply_fn: Callable, q_update_fn: Callable, buffer_fns: Tuple[Callable, Callable], config: DictConfig,
                   loss: str = "q_learning"):
    """ff_dqn.py:92-258.  q_apply_fn: the bound `apply` of the Q network (a FeedForwardActor with a DiscreteQNetworkHead); q_update_fn:
    the bound `update` of chain(clip_by_global_norm, adam); buffer_fns = (DiscreteTransitionBuffer.add, .sample_into) unbound, applied
    to learner_state.buffer_state[u]; loss: one of LOSSES."""
    q_net = _owner(q_apply_fn, Actor, "q_apply_fn")
    if not isinstance(q_net.action_head, DiscreteQNetworkHead):
        raise TypeError("get_learner_fn: q_apply_fn must be the bound `apply` of a FeedForwardActor with a DiscreteQNetworkHead")
    opt = _owner(q_update_fn, optax.GradientTransformation, "q_update_fn")
    if loss not in LOSSES:
        raise ValueError(f"get_learner_fn: loss {loss!r} is not one of {LOSSES}")
    _refuse_unsupported(config)
    buffer_add_fn, buffer_sample_fn = buffer_fns
    rank, world = _world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, M = int(sysc.epochs), int(sysc.batch_size)
    tau = float(sysc.tau)
    hyper = loss_hyper(loss, config)
    sched = ops.epsilon_schedule_struct(float(sysc.training_epsilon), float(sysc.training_epsilon), 0.0, 1, decay=False)
    use_graph = bool(arch.get("cuda_graph", True))
    has_step_into = hasattr(env, "step_into")
    built: Dict[str, Any] = {}

    def _build(state: OffPolicyLearnerState) -> None:
        tree = state.params.online
        spec = tree.spec
        dev = tree.flat.device
        D, A = spec.sizes[0], spec.sizes[-1]
        lr_sched = opt.schedule
        plan = ops.AdamPlan([(0, spec.param_count, opt.init_lr, opt.max_grad_norm)], dev, b1=opt.adam.b1, b2=opt.adam.b2, eps=opt.adam.eps,
                            decay=lr_sched is not None, steps_per_update=getattr(lr_sched, "steps_per_update", 1),
                            num_updates=getattr(lr_sched, "num_updates", 1), **opt.plan_kwargs())
        plan.counts = tree.arena_counts   # the optimiser counters live in the learner state (so a checkpoint carries them)
        built.update(spec=spec, dev=dev, plan=plan, rollouts=[_Rollout(T, E, D, A, dev) for _ in range(U)],
                     batches=[make_batch(M, D, dev) for _ in range(U)], work=make_work(spec, M, dev),
                     grads=torch.zeros(tree.arena.numel(), dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, dtype=torch.float32, device=dev),
                     roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # epsilon-greedy call index
                     graph=None, eager_done=False)

    def _rollout_phase(state: OffPolicyLearnerState) -> None:
        """_env_step x rollout_length (ff_dqn.py:106-137) + buffer add (:142), per shard."""
        b = built
        online = state.params.online.flat
        for u in range(U):
            ro: _Rollout = b["rollouts"][u]
            for t in range(T):
                ops.mlp_forward(b["spec"], online, ro.obs[t], out=ro.q[t], ws_key="dqn_rollout")
                ops.epsilon_greedy(ro.q[t], sched, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], out=ro.action[t])
                if has_step_into:
                    env.step_into(state.env_state[u], ro.action[t], ro.step_out(t), t)
                else:
                    new_state, ts = env.step(state.env_state[u], ro.action[t])
                    state.env_state[u] = new_state
                    out = ro.step_out(t)
                    out.obs.copy_(ts.observation)
                    out.next_obs.copy_(ts.extras["next_obs"])
                    out.reward.copy_(ts.reward)
                    out.done.copy_(ts.discount == 0.0)
                    out.truncated.copy_(ts.last() & (ts.discount != 0.0))
                    em = ts.extras["episode_metrics"]
                    out.episode_return.copy_(em["episode_return"])
                    out.episode_length.copy_(em["episode_length"])
                    out.is_terminal_step.copy_(em["is_terminal_step"])
            torch.bitwise_or(ro.terminated, ro.truncated, out=ro.done)
            buffer_add_fn(state.buffer_state[u], ro.transition())

    def _update_epoch(state: OffPolicyLearnerState, ep: int, sample: bool = True, idx_in: Optional[torch.Tensor] = None) -> None:
        """One `_update_epoch` (ff_dqn.py:144-220): sample, gradients of every shard, mean over shards and devices, clip + Adam, Polyak."""
        b = built
        online, target = state.params.online, state.params.target
        if sample:   # SAMPLE TRANSITIONS (:182-186)
            for u in range(U):
                bt = b["batches"][u]
                buffer_sample_fn(state.buffer_state[u], bt.xs[:M], bt.xs[M:], bt.action, bt.reward, bt.done, idx_in=idx_in)
        metric = b["metrics"][ep: ep + 1]
        batch_grads(loss, b["spec"], online.flat, target.flat, b["batches"], hyper, b["grads"], metric, b["work"])
        if world > 1:   # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        ops.clip_adam_step(b["plan"], online.arena, b["grads"], state.opt_states.mu, state.opt_states.nu, grad_scale=1.0 / world)
        ops.polyak_update(target.arena, online.arena, tau)   # optax.incremental_update (:207-209)

    def _carry_in_phase(state: OffPolicyLearnerState) -> None:
        for ro in built["rollouts"]:
            ro.obs[0].copy_(ro.obs[T])

    def _advance_phase(state: OffPolicyLearnerState) -> None:
        for u in range(U):
            if hasattr(env, "advance"):
                env.advance(state.env_state[u], T)
        ops.counter_add(built["roll_ctr"], T)

    def _update_step(state: OffPolicyLearnerState) -> None:
        """A single update (ff_dqn.py:103-234), in place on the learner state."""
        _carry_in_phase(state)
        _rollout_phase(state)
        built["metrics"].zero_()
        for ep in range(epochs):
            _update_epoch(state, ep)
        if world > 1:
            dist.all_reduce(built["metrics"], op=dist.ReduceOp.SUM)
            built["metrics"].mul_(1.0 / world)
        _advance_phase(state)

    def learner_fn(learner_state: OffPolicyLearnerState) -> AnakinExperimentOutput:
        """arch.num_updates_per_eval update steps (ff_dqn.py:236-256)."""
        learner_fn.ensure_built(learner_state)
        b = built
        n_upd, dev = int(arch.num_updates_per_eval), b["dev"]
        ep_out = {"episode_return": torch.empty(n_upd, U, T, E, device=dev),
                  "episode_length": torch.empty(n_upd, U, T, E, dtype=torch.int32, device=dev),
                  "is_terminal_step": torch.empty(n_upd, U, T, E, dtype=torch.bool, device=dev)}
        train_out = torch.empty(n_upd, epochs, device=dev)
        for k in range(n_upd):
            if use_graph and b["eager_done"] and b["graph"] is None:
                g = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                gc.collect()   # no cyclic GC (which may destroy an older CUDAGraph) while the stream is capturing
                gc_was_enabled = gc.isenabled()
                gc.disable()
                added = [buf.added for buf in learner_state.buffer_state]   # capturing launches nothing: keep the host mirrors
                try:
                    with torch.cuda.graph(g):
                        _update_step(learner_state)
                finally:
                    if gc_was_enabled:
                        gc.enable()
                for buf, n in zip(learner_state.buffer_state, added):
                    buf.added = n
                b["graph"] = g
            if b["graph"] is not None:
                b["graph"].replay()
                for buf in learner_state.buffer_state:
                    buf.added += T * E   # host mirror of the item count under replay
            else:
                _update_step(learner_state)   # the first update runs eagerly (module loading, NCCL warm-up)
                b["eager_done"] = True
            for u in range(U):
                ro = b["rollouts"][u]
                ep_out["episode_return"][k, u].copy_(ro.episode_return)
                ep_out["episode_length"][k, u].copy_(ro.episode_length)
                ep_out["is_terminal_step"][k, u].copy_(ro.is_terminal_step)
            train_out[k].copy_(b["metrics"])
        new_ts = [learner_state.timestep[u]._replace(observation=b["rollouts"][u].obs[T]) for u in range(U)]
        learner_state = learner_state._replace(timestep=new_ts)
        return AnakinExperimentOutput(learner_state=learner_state, episode_metrics=ep_out, train_metrics={"q_loss": train_out})

    def _ensure_built(st: OffPolicyLearnerState) -> None:
        if not built:
            _build(st)
            for u in range(U):
                built["rollouts"][u].obs[T].copy_(st.timestep[u].observation)

    learner_fn.built = built
    learner_fn.ensure_built = _ensure_built
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.rollout_phase = _rollout_phase
    learner_fn.loss = loss
    return learner_fn


def learner_setup(env: Environment, keys: Tuple[int, int], config: DictConfig, loss: str = "q_learning"):
    """Initialise learner_fn, network, optimiser, buffer, environment and states (ff_dqn.py:261-414).  Returns the EVAL network
    (epsilon = system.evaluation_epsilon) as the second element, which is what the reference hands to the evaluator."""
    _refuse_unsupported(config)
    rank, world = _world()
    n_devices = world
    device = torch.device("cuda", torch.cuda.current_device())
    action_dim = int(env.action_space().num_values)
    config.system.action_dim = action_dim
    key, q_net_key = keys

    torso = instantiate(config.network.actor_network.pre_torso)
    head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.training_epsilon)
    q_network = Actor(torso=torso, action_head=head)
    eval_head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.evaluation_epsilon)
    eval_q_network = Actor(torso=torso, action_head=eval_head)

    q_lr = make_learning_rate(config.system.q_lr, config, config.system.epochs)
    q_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(q_lr, eps=1e-5))

    # Online parameters in one arena; the target arena starts as a copy of it (:303-307).
    init_x = env.observation_space().generate_value()[None, ...].to(device).float()
    spec = q_network.spec_for(init_x.shape[-1])
    arena = torch.zeros((spec.param_count + 7) // 8 * 8, dtype=torch.float32, device=device)
    online = q_network.init(q_net_key, init_x, flat=arena)
    online.arena = arena
    mu, nu = torch.zeros_like(arena), torch.zeros_like(arena)
    counts = torch.zeros(2, dtype=torch.int32, device=device)   # {adam count, schedule count}, stepped in place by the learner
    opt_states = optax.OptState(counts[0:1], mu, nu, counts[1:2])
    online.arena_mu, online.arena_nu, online.arena_counts = mu, nu, counts

    if config.logger.checkpointing.load_model:   # params only, as in the reference (:372-380)
        from stoix_b200.utils.checkpointing import Checkpointer

        loaded = Checkpointer(model_name=config.system.system_name, **to_container(config.logger.checkpointing.load_args))
        loaded.restore_params(arena)
    target_arena = arena.clone()
    target = build_param_tree(spec, target_arena, "action_head")
    target.arena = target_arena
    params = OnlineAndTarget(online, target)

    # Replay buffer (:316-347): one ring per (device, update-batch shard)
    U, E = int(config.arch.update_batch_size), int(config.arch.num_envs)
    assert int(config.system.total_buffer_size) % n_devices == 0, "The total buffer size should be divisible by the number of devices!"
    assert int(config.system.total_batch_size) % n_devices == 0, "The total batch size should be divisible by the number of devices!"
    config.system.buffer_size = int(config.system.total_buffer_size) // (n_devices * U)
    config.system.batch_size = int(config.system.total_batch_size) // (n_devices * U)
    shard_keys = srandom.split(key, U + 2)
    buffer_states = [DiscreteTransitionBuffer(config.system.buffer_size, config.system.batch_size, config.system.batch_size, init_x.shape[-1],
                                              device, seed=srandom.split(shard_keys[U], n_devices * U)[rank * U + u]) for u in range(U)]
    buffer_fns = (DiscreteTransitionBuffer.add, DiscreteTransitionBuffer.sample_into)

    learn = get_learner_fn(env, q_network.apply, q_optim.update, buffer_fns, config, loss=loss)
    warmup = get_warmup_fn(env, params, q_network.apply, DiscreteTransitionBuffer.add, config)

    env_states: List[Any] = []
    timesteps: List[TimeStep] = []
    for u in range(U):
        if hasattr(env, "seed"):
            env.seed = (int(config.arch.seed) + 7919 * rank + 15485863 * u) & ((1 << 63) - 1)
        st, ts = env.reset(srandom.split(shard_keys[u], E))
        env_states.append(st)
        timesteps.append(ts)

    # per-rank streams: rollout epsilon-greedy draws; warm-up draws on their own key (:383-409)
    step_key = srandom.split(shard_keys[U + 1], 2 * n_devices)
    m62 = (1 << 62) - 1
    act_seed, warm_seed = step_key[2 * rank] & m62, step_key[2 * rank + 1] & m62
    for u in range(U):
        env_states[u], timesteps[u], _, _ = warmup(env_states[u], timesteps[u], buffer_states[u], warm_seed + 0xA5A5 * u)

    # key = (rollout seed, warm-up seed): the rollout draws from key[0]; key[1] records where the warm-up drew from
    init_learner_state = OffPolicyLearnerState(params, opt_states, buffer_states, (act_seed, warm_seed), env_states, timesteps)
    return learn, eval_q_network, init_learner_state


class _QParams(NamedTuple):
    actor_params: Any   # the Checkpointer stores the arenas of params.actor_params: the online network


class _CheckpointView(NamedTuple):
    params: _QParams


def run_experiment(_config: DictConfig, loss: str = "q_learning") -> float:
    """Runs experiment (ff_dqn.py:417-556)."""
    from stoix_b200.evaluator import evaluator_setup, get_distribution_act_fn
    from stoix_b200.systems.sac.ff_sac import get_final_step_metrics

    config = copy.deepcopy(_config)
    rank, world = _world()
    config.num_devices, config.rank = world, rank
    config = check_total_timesteps(config, quiet=rank != 0)
    assert config.arch.num_updates >= config.arch.num_evaluation, "Number of updates per evaluation must be less than total number of updates."
    env, eval_env = environments.make(config=config)
    key, key_e, q_net_key = srandom.split(srandom.PRNGKey(config.arch.seed), num=3)
    learn, eval_q_network, learner_state = learner_setup(env, (key, q_net_key), config, loss=loss)
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
    best_params = learner_state.params.online.flat.clone()
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
        opt_steps_per_eval = config.arch.num_updates_per_eval * config.system.epochs   # (:495)
        train_metrics["steps_per_second"] = torch.tensor(opt_steps_per_eval / elapsed_time)
        logger.log(train_metrics, t, eval_step, LogEvent.TRAIN)
        start_time = time.time()
        trained_params = learner_output.learner_state.params.online
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
        start_time = time.time()
        t = int(steps_per_rollout * (eval_step + 1))
        best_tree = build_param_tree(learner_state.params.online.spec, best_params, "action_head")
        evaluator_output = absolute_metric_evaluator(best_tree, srandom.split(key_e, 1)[0])
        torch.cuda.synchronize()
        elapsed_time = time.time() - start_time
        evaluator_output["steps_per_second"] = torch.tensor(int(evaluator_output["episode_length"].sum().item()) / max(elapsed_time, 1e-9))
        logger.log(evaluator_output, t, eval_step, LogEvent.ABSOLUTE)
    logger.stop()
    return float(evaluator_output[config.env.eval_metric].float().mean().item())


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None, loss: str = "q_learning",
                      config_name: str = "default_ff_dqn") -> float:
    """Experiment entry point: `python -m stoix_b200.systems.q_learning.ff_dqn arch.total_num_envs=1024 ...`"""
    if cfg is None:
        cfg = compose(config_name, overrides if overrides is not None else sys.argv[1:], config_dir="default/anakin")
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    t0 = time.time()
    eval_performance = run_experiment(cfg, loss=loss)
    if _world()[0] == 0:
        print(f"{_NAMES[loss]} experiment completed in {time.time() - t0:.2f} seconds.")
    return eval_performance


if __name__ == "__main__":
    hydra_entry_point()
