"""Anakin R2D2 on H100 -- drop-in for stoix/systems/q_learning/rec_r2d2.py, fp32.

Same entry points (get_warmup_fn :39-155, get_learner_fn :158-478, learner_setup :481-760, run_experiment, hydra_entry_point) and
state contracts (RNNTransition, RNNOffPolicyLearnerState).  Behaviour restated from the reference: every rollout step runs the
recurrent network over one step from the carried hidden state, reset where the previous step was done or truncated, samples
epsilon-greedy and stores the carry that ENTERED the step; the loss re-runs both networks from the carry of each sequence's first
row, burns in over burn_in_length rows without gradient and learns on the rest.

  reference (JAX)                                        here (H100)
  -----------------------------------------------------  --------------------------------------------------------------------
  make_prioritised_trajectory_buffer(period, S)          the prioritised sequence ring (utils/replay.py PrioritisedSequenceBuffer):
                                                         Rainbow's sum tree over items every `period` rows, carries at item starts
  stop_gradient(burn-in forwards)                        pre-torso + GRU/LSTM sequence forward of the burn-in rows only (the
                                                         target runs burn-in and learn window as one forward of S rows)
  transformed_n_step_q_learning, IS weights, priorities  stx_r2d2_loss_grads: one launch (selector, h / h^-1 n-step targets, td,
                                                         weights, d Q, priorities, metrics)
  jax.grad through the learn window                      dueling backward, post MLP backward, GRU/LSTM BPTT, pre MLP backward
  pmean(batch); pmean(device); clip + adam; polyak       mean over shards; NCCL all-reduce; one clip + Adam launch; Polyak
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput, RNNOffPolicyLearnerState
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.evaluator import get_rnn_evaluator_fn
from stoix_b200.networks.recurrent import RecLayout, RecurrentActor, ScannedRNN
from stoix_b200.systems import anakin
from stoix_b200.systems.q_learning.dqn_types import RNNTransition
from stoix_b200.systems.sac.sac_types import OnlineAndTarget
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.replay import PrioritisedSequenceBuffer
from stoix_b200.utils.training import make_learning_rate

_pad8 = lambda n: (int(n) + 7) // 8 * 8
_HEADS = ("DuelingQNetwork", "DiscreteQNetworkHead")


def refuse_unsupported(config: DictConfig, n_devices: int = 1) -> None:
    """The reference's asserts (rec_r2d2.py:618-634) and what this port does not build, each with the reason."""
    sysc, net = config.system, config.network.actor_network
    if int(sysc.total_buffer_size) % n_devices != 0:
        raise ValueError("The total buffer size should be divisible by the number of devices!")
    if int(sysc.total_batch_size) % n_devices != 0:
        raise ValueError("The total batch size should be divisible by the number of devices!")
    if int(sysc.burn_in_length) >= int(sysc.sample_sequence_length):
        raise ValueError("The burn-in length must be less than the sample sequence length!")
    if int(sysc.period) > int(sysc.rollout_length):
        raise ValueError("The period must be less than or equal to the rollout length!")
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for rec_r2d2: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not the recurrent Q network; use arch.precision=f32")
    cell = str(net.rnn_layer.get("cell_type", "gru"))
    if {"optimised_lstm": "lstm"}.get(cell, cell) not in ("gru", "lstm"):
        raise ValueError(f"rec_r2d2 runs the gru and lstm cells (the CUDA sequence kernels); cell_type {cell!r} is not built")
    head = str(net.action_head.get("_target_", "")).rsplit(".", 1)[-1]
    if head not in _HEADS:
        raise ValueError(f"rec_r2d2 runs a DuelingQNetwork or DiscreteQNetworkHead action head; {head!r} is not implemented for it")
    if head == "DuelingQNetwork":
        post = net.post_torso
        if not bool(net.action_head.get("use_layer_norm", False)):
            raise ValueError("rec_r2d2's DuelingQNetwork needs use_layer_norm=True: that form's value branch ends in a LayerNorm over one "
                             "element, whose output is its bias; the branch without LayerNorm is not built")
        if not bool(post.get("use_layer_norm", False)) or str(post.get("activation", "relu")) != str(net.action_head.get("activation", "relu")):
            raise ValueError("rec_r2d2 runs the post-torso and the dueling advantage branch as one MLP: the post-torso needs use_layer_norm=True "
                             "and the activation of the head")
    U = int(config.arch.update_batch_size)
    E = int(config.arch.get("num_envs", None) or int(config.arch.total_num_envs) // (n_devices * U))
    L = int(sysc.total_buffer_size) // (n_devices * U) // E
    if L < int(sysc.sample_sequence_length):
        raise ValueError(f"rec_r2d2: the replay ring holds {L} time rows per env (total_buffer_size / (devices x update_batch_size x num_envs)), "
                         f"fewer than one sequence of sample_sequence_length={int(sysc.sample_sequence_length)}")


class _Shard(anakin.Trajectory):
    """Rollout rows of one (device, update-batch) shard, time-major: the RNNTransition fields, the carried hidden state and flags."""

    def __init__(self, T: int, E: int, D: int, Cd: int, A: int, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.action, self.reset = z(T, E, dt=torch.int32), z(T, E, dt=torch.uint8)
        self.hstate = z(T, E, Cd)                   # the carry entering step t
        self.h_cur = z(E, Cd)                       # the carried hidden state
        self.done_prev, self.trunc_prev = z(E, dt=torch.uint8), z(E, dt=torch.uint8)   # flags of the step before row 0
        self.q = z(E, A)

    def transition(self) -> RNNTransition:
        return RNNTransition(self.obs[: self.T], self.action, self.reward, self.reset, self.terminated, self.truncated,
                             {"episode_return": self.episode_return, "episode_length": self.episode_length,
                              "is_terminal_step": self.is_terminal_step}, self.hstate)


def rollout(net: RecurrentActor, tree, env: Environment, env_states: List[Any], u: int, sh: _Shard, sched, seed: int, counter: Optional[torch.Tensor]) -> None:
    """_env_step x T (rec_r2d2.py:199-263) of shard u in place: reset where the previous step ended, one recurrent step, epsilon-greedy
    at call offset t + *counter of `seed`, env step; the carry entering each step goes to sh.hstate."""
    for t in range(sh.T):
        prev_d, prev_t = (sh.done_prev, sh.trunc_prev) if t == 0 else (sh.terminated[t - 1], sh.truncated[t - 1])
        torch.bitwise_or(prev_d, prev_t, out=sh.reset[t])
        sh.hstate[t].copy_(sh.h_cur)
        h_new, q = net._forward(tree, sh.h_cur, (sh.obs[t][None], sh.reset[t][None]))
        sh.q.copy_(q[0])
        ops.epsilon_greedy(sh.q, sched, seed=seed, offset=t, dev_counter=counter, out=sh.action[t])
        anakin.step_env(env, env_states, u, sh.action[t], sh.step_out(t), t)
        sh.h_cur.copy_(h_new)
    sh.done_prev.copy_(sh.terminated[sh.T - 1]), sh.trunc_prev.copy_(sh.truncated[sh.T - 1])


class Batch:
    """One sampled batch of B sequences of S rows, time-major, with the carry of row 0, the items and p_i."""

    def __init__(self, S: int, B: int, D: int, Cd: int, device):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs, self.action, self.reward = z(S, B, D), z(S, B, dt=torch.int32), z(S, B)
        self.done, self.reset = z(S, B, dt=torch.uint8), z(S, B, dt=torch.uint8)
        self.carry0, self.idx, self.prob = z(B, Cd), z(B, dt=torch.int32), z(B)


class Work:
    """Workspaces of one sequence batch: burn-in, target and learn-window forwards, the learn window's backward, the loss rows."""

    def __init__(self, lay: RecLayout, S: int, burn_in: int, B: int, A: int, device):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        H, G, Tl = lay.H, lay.G, S - burn_in
        self.Tl = Tl
        self.gi_all, self.h_all, self.ws_all = z(S, B, G * H), z(S, B, H), lay.sequence_workspace(S, B, device)   # target, S rows
        self.gi_burn, self.h_burn = z(max(burn_in, 1), B, G * H), z(max(burn_in, 1), B, H)
        self.ws_burn = lay.sequence_workspace(max(burn_in, 1), B, device)
        self.carry_on, self.carry_tg = z(B, lay.S), z(B, lay.S)                                              # burned-in carries
        self.ws_pre, self.ws_post = ops.mlp_train_workspace(lay.spec_pre, Tl * B, device), ops.mlp_train_workspace(lay.spec_post, Tl * B, device)
        self.gi, self.d_gi, self.h_seq, self.d_h, self.ws_seq = z(Tl, B, G * H), z(Tl, B, G * H), z(Tl, B, H), z(Tl, B, H), lay.sequence_workspace(Tl, B, device)
        self.out, self.d_out = z(Tl * B, A), z(Tl * B, A)
        self.q, self.q_tg, self.d_q = z(Tl, B, A), z(Tl, B, A), z(Tl, B, A)
        self.priorities = z(B)


def _sequence(lay: RecLayout, p_flat: torch.Tensor, obs: torch.Tensor, reset: torch.Tensor, carry0: torch.Tensor, gi: torch.Tensor, h_seq: torch.Tensor,
              ws: torch.Tensor, carry_last: Optional[torch.Tensor], key: str) -> None:
    """Pre-torso + input projections of every row (inference) and the recurrence from carry0; carry_last (nullable) gets the last carry."""
    T, B, D = obs.shape
    ops.mlp_forward(lay.spec_pre, lay.blocks(p_flat)[0], obs.reshape(T * B, D), out=gi.view(T * B, -1), ws_key=key)
    lay.sequence_forward(p_flat, gi, reset, carry0, ws, out=h_seq, carry_last=carry_last)


def _head(lay: RecLayout, p_flat: torch.Tensor, out: torch.Tensor, q: torch.Tensor) -> None:
    if lay.dueling:
        ops.dueling_q(out, lay.value_bias(p_flat), out=q.view(out.shape))
    else:
        q.view(out.shape).copy_(out)


def batch_grads(lay: RecLayout, online: torch.Tensor, target: torch.Tensor, bt: Batch, work: Work, burn_in: int, hyper: Dict[str, float],
                count: Optional[torch.Tensor], grads: torch.Tensor, metric: torch.Tensor, weight: float, overwrite: bool) -> None:
    """jax.grad(_q_loss_fn) of one sampled batch (rec_r2d2.py:290-411): burn-in and learn-window forwards of both networks, the fused
    loss, and the backward through the learn window into `grads` (weight g, overwritten or added); the new priorities land in
    work.priorities and metric[0..6) += weight * the reference's metrics."""
    S, B, D = bt.obs.shape
    Tl, w = work.Tl, work
    # target: burn-in and learn window as one forward of S rows; only the learn rows reach the head
    _sequence(lay, target, bt.obs, bt.reset, bt.carry0, w.gi_all, w.h_all, w.ws_all, None, "r2d2_tg_pre")
    post_t = lay.blocks(target)[3]
    ops.mlp_forward(lay.spec_post, post_t, w.h_all[burn_in:].reshape(Tl * B, lay.H), out=w.out, ws_key="r2d2_tg_post")
    _head(lay, target, w.out, w.q_tg)
    # online: burn-in without gradient, then the learn window in train mode from the burned-in carry
    carry = bt.carry0
    if burn_in > 0:
        _sequence(lay, online, bt.obs[:burn_in], bt.reset[:burn_in], bt.carry0, w.gi_burn, w.h_burn, w.ws_burn, w.carry_on, "r2d2_burn_pre")
        carry = w.carry_on
    pre, _, _, post = lay.blocks(online)
    g_pre, _, _, g_post = lay.blocks(grads)
    obs_l, reset_l = bt.obs[burn_in:].reshape(Tl * B, D), bt.reset[burn_in:]
    ops.mlp_forward_train(lay.spec_pre, pre, obs_l, w.ws_pre, out=w.gi.view(Tl * B, -1))
    lay.sequence_forward(online, w.gi, reset_l, carry, w.ws_seq, out=w.h_seq)
    ops.mlp_forward_train(lay.spec_post, post, w.h_seq.view(Tl * B, lay.H), w.ws_post, out=w.out)
    _head(lay, online, w.out, w.q)
    ops.r2d2_loss_grads(w.q, w.q_tg, bt.action[burn_in:], bt.reward[burn_in:], bt.done[burn_in:], bt.prob, w.d_q, w.priorities, metric,
                        count=count, weight=weight, **hyper)
    if lay.dueling:
        ops.dueling_q_backward(w.d_q.view(Tl * B, -1), w.d_out, lay.value_bias(grads), weight=weight, overwrite=overwrite)
    else:
        w.d_out.copy_(w.d_q.view(Tl * B, -1))
    ops.mlp_backward(lay.spec_post, post, w.h_seq.view(Tl * B, lay.H), w.d_out, w.ws_post, net_grad=g_post, grad_weight=weight, overwrite=overwrite,
                     d_input=w.d_h.view(Tl * B, lay.H))
    lay.sequence_backward(online, grads, w.d_h, reset_l, w.ws_seq, w.d_gi, weight, overwrite)
    ops.mlp_backward(lay.spec_pre, pre, obs_l, w.d_gi.view(Tl * B, -1), w.ws_pre, net_grad=g_pre, grad_weight=weight, overwrite=overwrite)


def get_warmup_fn(env: Environment, q_params: OnlineAndTarget, q_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """rec_r2d2.py:39-155: system.warmup_steps environment steps of one shard with the initial online parameters, added to the
    buffer as one RNNTransition.  warmup(env_state, timestep, buffer_state, key, hstate, done, truncated) -> the carried values."""
    net = anakin.owner(q_apply_fn, RecurrentActor, "q_apply_fn")
    W = int(config.system.warmup_steps)
    sched = ops.epsilon_schedule_struct(float(config.system.training_epsilon), float(config.system.training_epsilon), 0.0, 1, decay=False)

    def warmup(env_state, timestep, buffer_state, key: int, hstate: torch.Tensor, done: torch.Tensor, truncated: torch.Tensor):
        if W <= 0:
            return env_state, timestep, key, buffer_state, hstate, done, truncated
        E, D = timestep.observation.shape[0], timestep.observation.shape[-1]
        sh = _Shard(W, E, D, hstate.shape[-1], net.head.out_dim, hstate.device)
        sh.obs[0].copy_(timestep.observation)
        sh.h_cur.copy_(hstate), sh.done_prev.copy_(done), sh.trunc_prev.copy_(truncated)
        states = [env_state]
        rollout(net, q_params.online, env, states, 0, sh, sched, key, None)
        sh.advance(env, states[0])
        buffer_add_fn(buffer_state, sh.transition())
        return (states[0], timestep._replace(observation=sh.obs[W].clone()), key, buffer_state, sh.h_cur.clone(), sh.done_prev.bool(),
                sh.trunc_prev.bool())

    return warmup


def get_learner_fn(env: Environment, q_apply_fn: Callable, q_update_fn: Callable, buffer_fns: Tuple[Callable, Callable, Callable],
                   importance_weight_scheduler_fn: Tuple[float, float], config: DictConfig):
    """rec_r2d2.py:158-478.  q_apply_fn: the bound `apply` of a RecurrentActor; q_update_fn: the bound `update` of chain(clip_by_global_norm,
    adam); buffer_fns = (PrioritisedSequenceBuffer.add, .sample_into, .set_priorities); the importance sampling schedule as
    (init_value, transition_steps) of optax.linear_schedule(init_value, 1.0, transition_steps).  The value transform is rlax's
    SIGNED_HYPERBOLIC_PAIR, inside stx_r2d2_loss_grads."""
    net = anakin.owner(q_apply_fn, RecurrentActor, "q_apply_fn")
    opt = anakin.owner(q_update_fn, optax.GradientTransformation, "q_update_fn")
    rank, world = anakin.world()
    refuse_unsupported(config, world)
    buffer_add_fn, buffer_sample_fn, buffer_set_fn = buffer_fns
    beta0, beta_steps = importance_weight_scheduler_fn
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, S, burn_in = int(sysc.epochs), int(sysc.sample_sequence_length), int(sysc.burn_in_length)
    A = net.head.out_dim
    hyper = dict(n=int(sysc.n_step), gamma=float(sysc.gamma), max_abs_reward=float(sysc.max_abs_reward), eta=float(sysc.priority_eta),
                 beta0=float(beta0), beta_steps=float(beta_steps))
    sched = ops.epsilon_schedule_struct(float(sysc.training_epsilon), float(sysc.training_epsilon), 0.0, 1, decay=False)
    built: Dict[str, Any] = {}

    def _build(state: RNNOffPolicyLearnerState) -> None:
        tree = state.params.online
        lay: RecLayout = tree.layout
        dev = tree.flat.device
        D, B = lay.spec_pre.sizes[0], int(sysc.batch_size)
        shards = [_Shard(T, E, D, lay.S, A, dev) for _ in range(U)]
        for sh, h, d, tr in zip(shards, state.hstates, state.done, state.truncated):
            sh.h_cur.copy_(h), sh.done_prev.copy_(d), sh.trunc_prev.copy_(tr)
        built.update(layout=lay, dev=dev, plan=optax.adam_plan([(0, lay.param_count, opt)], dev, tree.arena_counts), shards=shards,
                     batches=[Batch(S, B, D, lay.S, dev) for _ in range(U)], work=Work(lay, S, burn_in, B, A, dev),
                     grads=torch.zeros(tree.arena.numel(), dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, ops._lib.STX_R2D2_METRICS, dtype=torch.float32, device=dev),
                     roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev), graph=None, eager_done=False)

    def _rollout_phase(state: RNNOffPolicyLearnerState) -> None:
        """_env_step x rollout_length (rec_r2d2.py:266-268) + buffer add (:285), per shard."""
        b = built
        for u in range(U):
            sh: _Shard = b["shards"][u]
            rollout(net, state.params.online, env, state.env_state, u, sh, sched, state.key[0] + u, b["roll_ctr"])
            buffer_add_fn(state.buffer_state[u], sh.transition())

    def _update_epoch(state: RNNOffPolicyLearnerState, ep: int, sample: bool = True) -> None:
        """One `_update_epoch` (rec_r2d2.py:287-439): sample, gradients and priorities of every shard, mean over shards and devices,
        clip + Adam, Polyak."""
        b = built
        online, target = state.params.online, state.params.target
        count = online.arena_counts[0:1]
        for u in range(U):
            bt: Batch = b["batches"][u]
            if sample:
                buffer_sample_fn(state.buffer_state[u], bt.obs, bt.action, bt.reward, bt.done, bt.reset, bt.carry0, bt.idx, bt.prob)
            batch_grads(b["layout"], online.flat, target.flat, bt, b["work"], burn_in, hyper, count, b["grads"], b["metrics"][ep], 1.0 / U, u == 0)
            buffer_set_fn(state.buffer_state[u], bt.idx, b["work"].priorities)
        if world > 1:   # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        ops.clip_adam_step(b["plan"], online.arena, b["grads"], online.arena_mu, online.arena_nu, grad_scale=1.0 / world)
        ops.polyak_update(target.arena, online.arena, float(sysc.tau))   # optax.incremental_update (:430-432)

    def _update_step(state: RNNOffPolicyLearnerState) -> None:
        """A single update (rec_r2d2.py:196-455), in place on the learner state."""
        for sh in built["shards"]:
            sh.carry_in()
        _rollout_phase(state)
        built["metrics"].zero_()
        for ep in range(epochs):
            _update_epoch(state, ep)
        if world > 1:
            dist.all_reduce(built["metrics"], op=dist.ReduceOp.SUM)
            built["metrics"].mul_(1.0 / world)
        for sh, env_state in zip(built["shards"], state.env_state):
            sh.advance(env, env_state)
        ops.counter_add(built["roll_ctr"], T)

    def learner_fn(learner_state: RNNOffPolicyLearnerState) -> AnakinExperimentOutput:
        """arch.num_updates_per_eval update steps (rec_r2d2.py:457-476)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, buffers=learner_state.buffer_state)
        shards = built["shards"]
        learner_state = learner_state._replace(timestep=timestep, done=[sh.done_prev.bool() for sh in shards],
                                               truncated=[sh.trunc_prev.bool() for sh in shards], hstates=[sh.h_cur for sh in shards])
        train_metrics = {name: train_out[..., j] for j, name in enumerate(ops.R2D2_METRICS)}
        return AnakinExperimentOutput(learner_state=learner_state, episode_metrics=episode_metrics, train_metrics=train_metrics)

    learner_fn.built = built
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.rollout_phase = _rollout_phase
    return learner_fn


def learner_setup(env: Environment, keys: Tuple[int, int], config: DictConfig):
    """Initialise learner_fn, networks, optimiser, buffers, environment and states (rec_r2d2.py:481-760)."""
    rank, n_devices = anakin.world()
    refuse_unsupported(config, n_devices)
    device = torch.device("cuda", torch.cuda.current_device())
    action_dim = int(env.action_space().num_values)
    config.system.action_dim = action_dim
    key, q_net_key = keys

    net = config.network.actor_network
    pre_torso, post_torso = instantiate(net.pre_torso), instantiate(net.post_torso)
    hidden, cell = int(net.rnn_layer.hidden_state_dim), str(net.rnn_layer.cell_type)
    make = lambda eps: RecurrentActor(pre_torso=pre_torso, hidden_state_dim=hidden, cell_type=cell, post_torso=post_torso,
                                      action_head=instantiate(net.action_head, action_dim=action_dim, epsilon=eps))
    q_network, eval_q_network = make(config.system.training_epsilon), make(config.system.evaluation_epsilon)
    actor_rnn = ScannedRNN(hidden, cell)

    q_lr = make_learning_rate(config.system.q_lr, config, config.system.epochs)
    q_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(q_lr, eps=1e-5))
    # optax.linear_schedule(importance_sampling_exponent, 1.0, num_updates * epochs) (:569-574), evaluated on the device
    beta_schedule = (float(config.system.importance_sampling_exponent), float(int(config.arch.num_updates) * int(config.system.epochs)))

    U, E = int(config.arch.update_batch_size), int(config.arch.num_envs)
    init_obs = env.observation_space().generate_value().to(device).float()[None, None].repeat(1, E, 1)
    init_x = (init_obs, torch.zeros(1, E, dtype=torch.bool, device=device))
    init_hstates = actor_rnn.initialize_carry(E, device)
    lay = q_network.layout_for(init_obs.shape[-1])
    arena = torch.zeros(_pad8(lay.param_count), dtype=torch.float32, device=device)
    online = q_network.init(q_net_key, init_hstates, init_x, flat=arena)
    (opt_states,) = optax.arena_state(online, arena, [(0, lay.param_count)])
    warm_start(config, arena)
    target_arena = arena.clone()
    target = q_network.build_tree(lay, target_arena)
    target.arena = target_arena
    params = OnlineAndTarget(online, target)

    # prioritised sequence replay (:605-655): one ring per (device, update-batch shard)
    shard_keys = srandom.split(key, U + 2)
    sysc = config.system
    buffer_states = anakin.replay_buffers(config, shard_keys[U], rank, n_devices, lambda size, batch, seed: PrioritisedSequenceBuffer(
        size, batch, int(sysc.sample_sequence_length), E, int(sysc.period), float(sysc.priority_exponent), init_obs.shape[-1], lay.S, device, seed=seed))
    buffer_fns = (PrioritisedSequenceBuffer.add, PrioritisedSequenceBuffer.sample_into, PrioritisedSequenceBuffer.set_priorities)

    learn = get_learner_fn(env, q_network.apply, q_optim.update, buffer_fns, beta_schedule, config)
    warmup = get_warmup_fn(env, params, q_network.apply, PrioritisedSequenceBuffer.add, config)

    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)
    act_seed, warm_seed = anakin.rank_seeds(shard_keys[U + 1], 2, rank, n_devices)
    dones = [torch.zeros(E, dtype=torch.bool, device=device) for _ in range(U)]
    truncs = [torch.zeros(E, dtype=torch.bool, device=device) for _ in range(U)]
    hstates = [init_hstates.clone() for _ in range(U)]
    for u in range(U):
        env_states[u], timesteps[u], _, _, hstates[u], dones[u], truncs[u] = warmup(env_states[u], timesteps[u], buffer_states[u],
                                                                                   warm_seed + 0xA5A5 * u, hstates[u], dones[u], truncs[u])
    init_learner_state = RNNOffPolicyLearnerState(params, opt_states, buffer_states, (act_seed, warm_seed), env_states, timesteps, dones, truncs, hstates)
    return learn, eval_q_network, init_learner_state


def _online(state: RNNOffPolicyLearnerState):
    return state.params.online


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (rec_r2d2.py:763-890), evaluating with the hidden state carried (get_rnn_evaluator_fn) at evaluation_epsilon."""
    return anakin.run_experiment(
        _config, learner_setup, net_keys=1, policy=_online,
        make_evaluators=lambda eval_env, key_e, net, config: (get_rnn_evaluator_fn(eval_env, net, config),
                                                              get_rnn_evaluator_fn(eval_env, net, config, 10)),
        best_tree=lambda net, tree, flat: net.build_tree(tree.layout, flat))


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point: `python -m stoix_b200.systems.q_learning.rec_r2d2 arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_rec_r2d2", run_experiment, "R2D2")


if __name__ == "__main__":
    hydra_entry_point()
