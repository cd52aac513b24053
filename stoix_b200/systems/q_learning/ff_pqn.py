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

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput, LearnerFn, OnPolicyLearnerState
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.heads import DiscreteQNetworkHead
from stoix_b200.systems import anakin
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.training import make_learning_rate


def _refuse_bf16(config: DictConfig) -> None:
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for ff_pqn: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not a Q network with its activation, LayerNorm and Q loss; use arch.precision=f32")


class _Shard(anakin.Trajectory):
    """Trajectory buffers of one (device, update-batch) shard, time-major: the Transition fields (dqn_types.py:9-15) plus the Q rows."""

    def __init__(self, T: int, E: int, D: int, A: int, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.done = self.terminated                   # the targets use done | truncated = timestep.last() (ff_pqn.py:84)
        self.q = z(T + 1, E, A)                       # q[t] = Q(obs[t]) with the rollout's parameters
        self.action = z(T, E, dt=torch.int32)
        self.epsilon = z(T, E)                        # info["epsilon"], info["update_no"] (ff_pqn.py:85-86)
        self.update_no = z(T, E, dt=torch.int32)
        self.targets = z(T, E)


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
    q_net = anakin.owner(q_apply_fn, Actor, "q_apply_fn")
    if not isinstance(q_net.action_head, DiscreteQNetworkHead):
        raise TypeError("get_learner_fn: q_apply_fn must be the bound `apply` of a FeedForwardActor with a DiscreteQNetworkHead")
    opt = anakin.owner(q_update_fn, optax.GradientTransformation, "q_update_fn")
    if opt.rule != "radam":
        raise TypeError("get_learner_fn: q_update_fn must be the bound `update` of chain(clip_by_global_norm(..), radam(..))")
    if not hasattr(epsilon_schedule, "device_schedule"):
        raise TypeError("get_learner_fn: epsilon_schedule must come from ff_pqn.linear_schedule / constant_schedule")
    _refuse_bf16(config)
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, nmb = int(sysc.epochs), int(sysc.num_minibatches)
    B = T * E
    assert B % nmb == 0, "rollout_length * num_envs must be divisible by num_minibatches"
    mb = B // nmb
    gamma, q_lambda, delta = float(sysc.gamma), float(sysc.q_lambda), float(sysc.huber_loss_parameter)
    sched = epsilon_schedule.device_schedule(epochs * nmb)
    built: Dict[str, Any] = {}

    def _build(state: OnPolicyLearnerState) -> None:
        tree = state.params
        spec = tree.spec
        dev = tree.flat.device
        D, A = spec.sizes[0], spec.sizes[-1]
        built.update(
            spec=spec, dev=dev, plan=optax.adam_plan([(0, spec.param_count, opt)], dev, tree.arena_counts), shards=[_Shard(T, E, D, A, dev) for _ in range(U)],
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
                anakin.step_env(env, state.env_state, u, sh.action[t], sh.step_out(t), t)
            ops.mlp_forward(b["spec"], tree.flat, sh.obs[T], out=sh.q[T], ws_key="pqn")

    def _targets_phase(state: OnPolicyLearnerState) -> None:
        """CALCULATE Q LAMBDA TARGETS (ff_pqn.py:97-120) with the rollout's parameters."""
        for u in range(U):
            sh: _Shard = built["shards"][u]
            ops.q_lambda(sh.q[1:], sh.reward, sh.done, sh.truncated, gamma, q_lambda, out=sh.targets)

    def _shuffle_phase(state: OnPolicyLearnerState) -> None:
        """SHUFFLE MINIBATCHES (ff_pqn.py:184-197): one keyed permutation per (shard, epoch), independent of the rollout."""
        anakin.shuffle(built["shards"], epochs, state.key[1], built["perm_ctr"])

    def _update_phase(state: OnPolicyLearnerState, shuffled: bool = False) -> None:
        """UPDATE EPOCHS (ff_pqn.py:122-207)."""
        b = built
        if not shuffled:
            _shuffle_phase(state)
        spec, tree = b["spec"], state.params
        D = spec.sizes[0]
        metrics, grads, ws, q_mb, dq_mb = b["metrics"], b["grads"], b["ws"], b["q_mb"], b["dq_mb"]
        metrics.zero_()
        for ep in range(epochs):
            for i in range(nmb):  # _update_minibatch (ff_pqn.py:127-180)
                rows = [(sh.obs[:T].view(B, D), sh.perms[ep, i * mb:(i + 1) * mb], sh.action.view(B), sh.targets.view(B)) for sh in b["shards"]]
                minibatch_grads(spec, tree.flat, rows, delta, grads, metrics[ep, i:i + 1], ws, q_mb, dq_mb)
                if world > 1:  # pmean over "device": summed by NCCL here, scaled in the optimiser step
                    dist.all_reduce(grads, op=dist.ReduceOp.SUM)
                ops.clip_adam_step(b["plan"], tree.arena, grads, tree.arena_mu, tree.arena_nu, grad_scale=1.0 / world)
        if world > 1:
            dist.all_reduce(metrics, op=dist.ReduceOp.SUM)
            metrics.mul_(1.0 / world)

    def _rollout_targets(state: OnPolicyLearnerState) -> None:
        _rollout_phase(state)
        _targets_phase(state)

    def _update_step(state: OnPolicyLearnerState) -> None:
        """A single update (ff_pqn.py:50-210), in place on the learner state; the shuffles run on a side stream under the rollout."""
        b = built
        for sh in b["shards"]:
            sh.carry_in()
        anakin.shuffle_beside(b, epochs, state.key[1], lambda: _rollout_targets(state))
        _update_phase(state, shuffled=True)
        for sh, env_state in zip(b["shards"], state.env_state):
            sh.advance(env, env_state)
        ops.counter_add(b["roll_ctr"], T)
        ops.counter_add(b["perm_ctr"], epochs)

    def learner_fn(learner_state: OnPolicyLearnerState) -> AnakinExperimentOutput[OnPolicyLearnerState]:
        """Run arch.num_updates_per_eval update steps (ff_pqn.py:212-226)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, extra_fields=("epsilon", "update_no"))
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics={"q_loss": train_out})

    learner_fn.built = built
    learner_fn.update_step = _update_step
    learner_fn.phases = {"rollout": _rollout_phase, "targets": _targets_phase, "shuffle": _shuffle_phase, "update": _update_phase}
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
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
    rank, world = anakin.world()
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
    (opt_states,) = optax.arena_state(params, arena, [(0, spec.param_count)])
    if config.system.decay_epsilon:
        epsilon_schedule = linear_schedule(1.0, float(config.system.training_epsilon),
                                           float(config.arch.num_updates) * float(config.system.exploration_fraction))
    else:
        epsilon_schedule = constant_schedule(float(config.system.training_epsilon))

    learn = get_learner_fn(env, q_network.apply, q_optim.update, epsilon_schedule, config)

    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 1)
    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    warm_start(config, arena)

    rollout_seed, shuffle_seed = anakin.rank_seeds(shard_keys[U], 2, rank, world)
    init_learner_state = OnPolicyLearnerState(params=params, opt_states=opt_states, key=(rollout_seed, shuffle_seed), env_state=env_states,
                                              timestep=timesteps)
    return learn, eval_q_network, init_learner_state


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_pqn.py:333-485): the Q network's parameters are evaluated, tracked and checkpointed."""
    return anakin.run_experiment(_config, learner_setup, net_keys=1, policy=lambda s: s.params)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_pqn: `python -m stoix_b200.systems.q_learning.ff_pqn arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_pqn", run_experiment, "PQN")


if __name__ == "__main__":
    hydra_entry_point()
