"""Anakin Rainbow on H100 -- drop-in for stoix/systems/q_learning/ff_rainbow.py.

Same entry points (get_warmup_fn :50-102, get_learner_fn :105-320, learner_setup :339-510, run_experiment, hydra_entry_point).  The
learner body is ff_dqn's (shards, rollout, clip + Adam, Polyak, graph-captured update step); what Rainbow changes:

  reference (JAX)                                        here (H100)
  -----------------------------------------------------  --------------------------------------------------------------------
  NoisyDistributionalDuelingQNetwork apply, fresh noise  stx_noisy_weights (noise + mu + sigma o eps into a dense arena), the
  per call (rngs={"noise": key})                         fp32 MLP forward on it, stx_dueling_combine (networks/dueling.py)
  jax.grad through the noisy layers                      stx_mlp_backward on the effective arena, stx_dueling_backward before
                                                         it, stx_noisy_fold (d mu, d sigma) after it
  make_prioritised_trajectory_buffer + n-step target     the prioritised n-step ring (utils/replay.py PrioritisedTrajectoryBuffer)
  (:222-246)                                             one launch per sample: draws, n-step rows, p_i, importance weights
  categorical_double_q_learning, mean(w loss) (:196-204) stx_categorical_q_loss_grads_weighted; loss_rows -> set_priorities
  importance_sampling_exponent linear schedule           evaluated on the device from the Adam count word before the step

Noise streams: each shard has one seed; rollout step t draws call t, epoch ep draws calls T + 3 ep (online on obs, differentiated),
T + 3 ep + 1 (target on next_obs) and T + 3 ep + 2 (online on next_obs, the selector), offset by a device counter that advances by
T + 3 epochs per update, so graph replays draw fresh noise.  The evaluator uses one fixed draw from the setup's noise key
(ff_rainbow.py:531-541).  The loss bootstraps with gamma, not gamma^n (:185-186).  fp32 only.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.dueling import NoisyDistributionalDuelingQNetwork, NoisyFeedForwardActor
from stoix_b200.systems import anakin
from stoix_b200.systems.q_learning.ff_dqn import _Shard, online_params
from stoix_b200.systems.sac.sac_types import OffPolicyLearnerState, OnlineAndTarget
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.replay import PrioritisedTrajectoryBuffer
from stoix_b200.utils.training import make_learning_rate


def _refuse_unsupported(config: DictConfig) -> None:
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for ff_rainbow: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not the noisy dueling C51 network; use arch.precision=f32")
    net = config.network.actor_network
    torso, head = str(net.pre_torso.get("_target_", "")), str(net.action_head.get("_target_", ""))
    if torso.rsplit(".", 1)[-1] != "NoisyMLPTorso" or head.rsplit(".", 1)[-1] != "NoisyDistributionalDuelingQNetwork":
        raise ValueError(f"ff_rainbow runs the NoisyMLPTorso + NoisyDistributionalDuelingQNetwork pair (network=mlp_noisy_dueling_c51); torso "
                         f"{torso!r} with head {head!r} is not implemented for it")
    if bool(net.pre_torso.get("use_layer_norm", False)) or bool(net.action_head.get("use_layer_norm", False)):
        raise ValueError("use_layer_norm=True is not available for ff_rainbow: the noisy layers are materialised into the fp32 MLP without "
                         "LayerNorm; use use_layer_norm=False")
    if str(net.pre_torso.get("activation", "relu")) != str(net.action_head.get("activation", "relu")):
        raise ValueError("ff_rainbow runs the torso and the dueling branches as one MLP: their activations must be the same")


class Batch(NamedTuple):
    """One sampled batch of M n-step transitions: xs (2M, D) = obs then next_obs rows; action, reward, done; the items, p_i and w_i."""
    xs: torch.Tensor
    action: torch.Tensor
    reward: torch.Tensor
    done: torch.Tensor
    idx: torch.Tensor
    prob: torch.Tensor
    weight: torch.Tensor


def make_batch(M: int, D: int, device) -> Batch:
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
    return Batch(z(2 * M, D), z(M, dt=torch.int32), z(M), z(M, dt=torch.uint8), z(M, dt=torch.int32), z(M), z(M))


class Work:
    """Workspaces of one shard-epoch: three effective arenas and noise buffers (online on obs, target on next_obs, online on
    next_obs), the train-mode forward workspace, head rows, logits, the selector's expected Q, gradients and per-row losses."""

    def __init__(self, layout, M: int, A: int, N: int, device):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        self.eff = [layout.scratch(device) for _ in range(3)]
        self.eff_grad = z(layout.eff_count)
        self.ws = ops.mlp_train_workspace(layout.spec, M, device)
        self.head = [z(M, N + A * N) for _ in range(3)]
        self.logits = [z(M, A * N) for _ in range(3)]
        self.q_sel, self.d_logits, self.d_head, self.loss_rows = z(M, A), z(M, A * N), z(M, N + A * N), z(M)


def batch_grads(layout, online: torch.Tensor, target: torch.Tensor, batches: Sequence[Batch], buffers: Sequence[PrioritisedTrajectoryBuffer],
                head: NoisyDistributionalDuelingQNetwork, hyper, seeds: Sequence[int], call: int, counter: torch.Tensor, grads: torch.Tensor,
                metric: torch.Tensor, work: Work, set_priorities: Callable = PrioritisedTrajectoryBuffer.set_priorities) -> None:
    """jax.grad(_q_loss_fn) + set_priorities + pmean over "batch" of one epoch (ff_rainbow.py:159-275) for the U shards: the three
    noisy forwards (calls `call`, +1, +2 of each shard's noise stream), the weighted C51 loss, the new priorities (the shard's own
    unweighted losses), the backward and the fold; `grads` receives the mean over the shards, metric[0] += mean_u mean(w loss)."""
    U = len(batches)
    A, N, atoms = head.action_dim, head.num_atoms, head.atoms(grads.device)
    spec = layout.spec
    for u, b in enumerate(batches):
        M = int(b.action.numel())
        obs, nxt = b.xs[:M], b.xs[M:]
        for k, (params, x) in enumerate(((online, obs), (target, nxt), (online, nxt))):
            eff, noise = work.eff[k]
            layout.weights(params, eff, noise, seeds[u], call + k, counter)
            if k == 0:
                ops.mlp_forward_train(spec, eff, x, work.ws, out=work.head[0])
            else:
                ops.mlp_forward(spec, eff, x, out=work.head[k], ws_key=f"rainbow_fwd{k}")
            ops.dueling_combine(work.head[k], A, N, out=work.logits[k])
        ops.dist_q_values("categorical", work.logits[2], A, N, atoms, out=work.q_sel)
        ops.categorical_q_loss_grads(work.logits[0], work.logits[1], work.q_sel, atoms, atoms, b.action, b.reward, hyper, work.d_logits, metric,
                                     done=b.done, loss_rows=work.loss_rows, weight=1.0 / U, scratch_key="rainbow_loss", row_weight=b.weight)
        set_priorities(buffers[u], b.idx, work.loss_rows)
        ops.dueling_backward(work.d_logits, A, N, out=work.d_head)
        ops.mlp_backward(spec, work.eff[0][0], obs, work.d_head, work.ws, net_grad=work.eff_grad, grad_weight=1.0 / U, overwrite=True)
        layout.fold(work.eff_grad, work.eff[0][1], grads, overwrite=(u == 0))


def get_warmup_fn(env: Environment, q_params: OnlineAndTarget, q_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """ff_rainbow.py:50-102: `warmup_steps` environment steps with the initial online parameters, fresh noise every step."""
    def draw(obs, key, t):
        pi, _, _ = q_apply_fn(q_params.online, obs, seed=key, offset=t)
        return pi.sample(seed=key, offset=t).to(torch.int32)

    return anakin.warmup_fn(env, draw, buffer_add_fn, config)


def get_learner_fn(env: Environment, q_apply_fn: Callable, q_update_fn: Callable, buffer_fns: Tuple[Callable, Callable, Callable],
                   importance_weight_scheduler_fn: Tuple[float, float], config: DictConfig):
    """ff_rainbow.py:105-320.  q_apply_fn: the bound `apply` of a NoisyFeedForwardActor; q_update_fn: the bound `update` of chain(
    clip_by_global_norm, adam); buffer_fns = (PrioritisedTrajectoryBuffer.add, .sample_into, .set_priorities); the importance
    sampling schedule as (init_value, transition_steps) of optax.linear_schedule(init_value, 1.0, transition_steps)."""
    q_net = anakin.owner(q_apply_fn, NoisyFeedForwardActor, "q_apply_fn")
    opt = anakin.owner(q_update_fn, optax.GradientTransformation, "q_update_fn")
    _refuse_unsupported(config)
    buffer_add_fn, buffer_sample_fn, buffer_set_fn = buffer_fns
    beta0, beta_steps = importance_weight_scheduler_fn
    head = q_net.action_head
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, M, gamma = int(sysc.epochs), int(sysc.batch_size), float(sysc.gamma)
    tau = float(sysc.tau)
    A, N = head.action_dim, head.num_atoms
    sched = ops.epsilon_schedule_struct(float(sysc.training_epsilon), float(sysc.training_epsilon), 0.0, 1, decay=False)
    built: Dict[str, Any] = {}

    def _build(state: OffPolicyLearnerState) -> None:
        tree = state.params.online
        lay = tree.layout
        dev = tree.flat.device
        D = lay.spec.sizes[0]
        shards = [_Shard(T, E, D, A, dev) for _ in range(U)]
        built.update(layout=lay, head=head, dev=dev, plan=optax.adam_plan([(0, lay.param_count, opt)], dev, tree.arena_counts), shards=shards,
                     hyper=ops.dist_q_hyper(gamma=gamma, max_abs_reward=float(sysc.max_abs_reward)),
                     roll_eff=lay.scratch(dev), head_out=torch.zeros(E, N + A * N, device=dev), logits=torch.zeros(E, A * N, device=dev),
                     batches=[make_batch(M, D, dev) for _ in range(U)], work=Work(lay, M, A, N, dev),
                     grads=torch.zeros(tree.arena.numel(), dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, dtype=torch.float32, device=dev),
                     roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),    # epsilon-greedy call index
                     noise_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # noise call index of every shard's stream
                     graph=None, eager_done=False)

    def _seeds(state: OffPolicyLearnerState) -> List[int]:
        return [(state.key[2] + u) & ((1 << 62) - 1) for u in range(U)]

    def _rollout_phase(state: OffPolicyLearnerState) -> None:
        """_env_step x rollout_length (ff_rainbow.py:117-150) + buffer add (:157), per shard."""
        b = built
        lay, online = b["layout"], state.params.online.flat
        eff, noise = b["roll_eff"]
        atoms = head.atoms(b["dev"])
        for u, seed in enumerate(_seeds(state)):
            ro: _Shard = b["shards"][u]
            for t in range(T):
                lay.weights(online, eff, noise, seed, t, b["noise_ctr"])
                ops.mlp_forward(lay.spec, eff, ro.obs[t], out=b["head_out"], ws_key="rainbow_rollout")
                ops.dueling_combine(b["head_out"], A, N, out=b["logits"])
                ops.dist_q_values("categorical", b["logits"], A, N, atoms, out=ro.q[t])
                ops.epsilon_greedy(ro.q[t], sched, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], out=ro.action[t])
                anakin.step_env(env, state.env_state, u, ro.action[t], ro.step_out(t), t)
            torch.bitwise_or(ro.terminated, ro.truncated, out=ro.done)
            buffer_add_fn(state.buffer_state[u], ro.transition())

    def _update_epoch(state: OffPolicyLearnerState, ep: int, sample: bool = True) -> None:
        """One `_update_epoch` (ff_rainbow.py:152-292): sample, gradients and priorities of every shard, mean over shards and
        devices, clip + Adam, Polyak."""
        b = built
        online, target = state.params.online, state.params.target
        count = online.arena_counts[0:1]
        if sample:
            for u in range(U):
                bt = b["batches"][u]
                buffer_sample_fn(state.buffer_state[u], bt.xs[:M], bt.xs[M:], bt.action, bt.reward, bt.done, bt.idx, bt.prob, bt.weight, gamma,
                                 beta0, beta_steps, count=count)
        metric = b["metrics"][ep: ep + 1]
        batch_grads(b["layout"], online.flat, target.flat, b["batches"], state.buffer_state, head, b["hyper"], _seeds(state), T + 3 * ep,
                    b["noise_ctr"], b["grads"], metric, b["work"], buffer_set_fn)
        if world > 1:   # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        ops.clip_adam_step(b["plan"], online.arena, b["grads"], online.arena_mu, online.arena_nu, grad_scale=1.0 / world)
        ops.polyak_update(target.arena, online.arena, tau)   # optax.incremental_update (:265-267)

    def _update_step(state: OffPolicyLearnerState) -> None:
        """A single update (ff_rainbow.py:112-300), in place on the learner state."""
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
        ops.counter_add(built["noise_ctr"], T + 3 * epochs)

    def learner_fn(learner_state: OffPolicyLearnerState) -> AnakinExperimentOutput:
        """arch.num_updates_per_eval update steps (ff_rainbow.py:302-320)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, buffers=learner_state.buffer_state)
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics={"q_loss": train_out})

    learner_fn.built = built
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.rollout_phase = _rollout_phase
    return learner_fn


class EvalActorWrapper:
    """The evaluation network (ff_rainbow.py:323-329 with get_distribution_act_fn's fixed rngs, :531-541): every forward uses the
    same noise draw, call 0 of the setup's noise key; `apply` returns the head's EpsilonGreedy."""

    def __init__(self, actor: NoisyFeedForwardActor, noise_seed: int):
        self.actor, self.noise_seed = actor, int(noise_seed)

    def apply(self, params, x):
        return self.actor.apply(params, x, seed=self.noise_seed, offset=0)[0]


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, network, optimiser, buffer, environment and states (ff_rainbow.py:339-510)."""
    _refuse_unsupported(config)
    rank, n_devices = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())
    action_dim = int(env.action_space().num_values)
    config.system.action_dim = action_dim
    key, q_net_key, noise_key = keys

    torso = instantiate(config.network.actor_network.pre_torso)
    head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.training_epsilon)
    q_network = NoisyFeedForwardActor(action_head=head, torso=torso)
    eval_head = instantiate(config.network.actor_network.action_head, action_dim=action_dim, epsilon=config.system.evaluation_epsilon)
    eval_q_network = EvalActorWrapper(NoisyFeedForwardActor(action_head=eval_head, torso=torso), noise_key & ((1 << 62) - 1))

    q_lr = make_learning_rate(config.system.q_lr, config, config.system.epochs)
    q_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(q_lr, eps=1e-5))
    # optax.linear_schedule(importance_sampling_exponent, 1.0, num_updates * epochs) (:386-391), evaluated on the device
    beta_schedule = (float(config.system.importance_sampling_exponent), float(int(config.arch.num_updates) * int(config.system.epochs)))

    init_x = env.observation_space().generate_value()[None, ...].to(device).float()
    lay = q_network.layout(init_x.shape[-1])
    arena = torch.zeros((lay.param_count + 7) // 8 * 8, dtype=torch.float32, device=device)
    online = q_network.init(q_net_key, init_x, flat=arena)
    (opt_states,) = optax.arena_state(online, arena, [(0, lay.param_count)])
    warm_start(config, arena)
    target_arena = arena.clone()
    target = lay.tree(target_arena)
    target.arena = target_arena
    params = OnlineAndTarget(online, target)

    # Prioritised replay (:433-442): one ring per (device, update-batch shard)
    U, E = int(config.arch.update_batch_size), int(config.arch.num_envs)
    shard_keys = srandom.split(key, U + 2)
    n_step, alpha, D = int(config.system.n_step), float(config.system.priority_exponent), init_x.shape[-1]
    buffer_states = anakin.replay_buffers(config, shard_keys[U], rank, n_devices,
                                          lambda size, batch, seed: PrioritisedTrajectoryBuffer(size, n_step, batch, E, alpha, D, device, seed=seed))
    buffer_fns = (PrioritisedTrajectoryBuffer.add, PrioritisedTrajectoryBuffer.sample_into, PrioritisedTrajectoryBuffer.set_priorities)

    learn = get_learner_fn(env, q_network.apply, q_optim.update, buffer_fns, beta_schedule, config)
    warmup = get_warmup_fn(env, params, q_network.apply, PrioritisedTrajectoryBuffer.add, config)

    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    # per-rank streams: rollout epsilon-greedy draws, warm-up draws, the training noise of every shard
    act_seed, warm_seed, noise_seed = anakin.rank_seeds(shard_keys[U + 1], 3, rank, n_devices)
    for u in range(U):
        env_states[u], timesteps[u], _, _ = warmup(env_states[u], timesteps[u], buffer_states[u], warm_seed + 0xA5A5 * u)

    init_learner_state = OffPolicyLearnerState(params, opt_states, buffer_states, (act_seed, warm_seed, noise_seed), env_states, timesteps)
    return learn, eval_q_network, init_learner_state


def _best_tree(network: EvalActorWrapper, tree, flat: torch.Tensor):
    return tree.layout.tree(flat)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_rainbow.py:513-640)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2, policy=online_params, best_tree=_best_tree)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point: `python -m stoix_b200.systems.q_learning.ff_rainbow arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_rainbow", run_experiment, "Rainbow")


if __name__ == "__main__":
    hydra_entry_point()
