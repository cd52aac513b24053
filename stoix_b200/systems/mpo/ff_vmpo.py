"""Anakin V-MPO on H100 -- drop-in for stoix/systems/mpo/ff_vmpo.py (Categorical actor); ff_vmpo_continuous.py runs the same learner
with a tanh-Normal actor.

Same entry points and signatures (get_learner_fn :55-324, learner_setup :327-456, run_experiment :459-602, hydra_entry_point) and
the same learner-state shape (mpo_types.py: OnlineAndTarget actor, critic, duals, three optimiser states, learner_step_count):

  reference (JAX)                                     here (H100)
  --------------------------------------------------  -----------------------------------------------------------------
  lax.scan over T env steps with the TARGET actor     T x (target actor forward, sampler, env step) launches
  epochs x full-batch update, no minibatches          per epoch and shard: critic forward on all T E rows, GAE (K2) or
                                                      n-step returns on v[0:T-1] / v[1:T], the exact top-k selection
                                                      (stx_vmpo_topk), target + online actor forwards on the (T-1) E rows,
                                                      one fused V-MPO loss (stx_vmpo_loss_grads: head, dual and value
                                                      gradients), the two backwards
  3 x chain(clip_by_global_norm, adam) + clip at -18  one clip + Adam launch over [actor | critic | duals], then
  + periodic_update(target, actor_target_period)      stx_vmpo_after_step (clamp, and copy online -> target when the actor
                                                      segment's Adam count, = learner_step_count, is a multiple of the period)
  pmean(batch); pmean(device)                         mean over update-batch shards; one NCCL all-reduce of the gradient arena
  one XLA program per learn() call                    one CUDA graph per update step, replayed

The top-k selection and the softmax weights stay per (device, shard), as in the reference.  The truncation flag is recorded but not
used by the targets (ff_vmpo.py:184-208): after a truncation the bootstrap is the next row's value, the reset observation.

fp32 only: arch.precision=bf16 raises.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput, LearnerFn
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import FeedForwardCritic as Critic
from stoix_b200.networks.base import build_param_tree
from stoix_b200.networks.heads import CategoricalHead, NormalAffineTanhDistributionHead
from stoix_b200.systems import anakin
from stoix_b200.systems.mpo.mpo_types import (
    CategoricalDualParams,
    DualParams,
    OnlineAndTarget,
    VMPOLearnerState,
    VMPOOptStates,
    VMPOParams,
)
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.training import make_learning_rate

_pad8 = lambda n: (int(n) + 7) // 8 * 8


def vmpo_arena_layout(actor: ops.MlpSpec, critic: ops.MlpSpec, n_dual: int) -> Dict[str, int]:
    """[actor | critic | duals], every block padded to 8 floats (each optimiser segment starts on a float4 boundary); the dual
    segment holds exactly the n_dual dual scalars."""
    off_c = _pad8(actor.param_count)
    off_d = off_c + _pad8(critic.param_count)
    return {"actor": 0, "critic": off_c, "duals": off_d, "n_dual": int(n_dual), "total": off_d + _pad8(n_dual)}


def dual_count(tanh_head: Optional[NormalAffineTanhDistributionHead], per_dim: bool) -> int:
    """log_temperature plus one log_alpha (Categorical) or log_alpha_mean and log_alpha_stddev of D' scalars each (D' = action_dim
    with per_dim_constraining, else 1) -- ff_vmpo.py:377-383, ff_vmpo_continuous.py:437-460."""
    if tanh_head is None:
        return 2
    return 1 + 2 * (tanh_head.action_dim if per_dim else 1)


def _actor_head(actor_net: Actor) -> Optional[NormalAffineTanhDistributionHead]:
    head = actor_net.action_head
    if isinstance(head, NormalAffineTanhDistributionHead):
        return head
    if isinstance(head, CategoricalHead):
        return None
    raise ValueError(f"V-MPO implements the Categorical (CategoricalHead) and tanh-Normal (NormalAffineTanhDistributionHead) actors; got "
                     f"{type(head).__name__}")


def check_config(config: DictConfig) -> None:
    """The refusals of both V-MPO systems: bf16, and rollouts too short to have a row after the last step is dropped."""
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for V-MPO: the bf16 tensor-core kernels implement the PPO clipped "
                         "surrogate only, not the top-k selection, the temperature and the KL-constrained loss; use arch.precision=f32")
    if int(config.system.rollout_length) < 2:
        raise ValueError(f"system.rollout_length={config.system.rollout_length}: V-MPO drops the last step of the rollout (ff_vmpo.py:123, "
                         "167), so it needs rollout_length >= 2")


class _Shard(anakin.Trajectory):
    """One (device, update-batch) shard: the SequenceStep fields (time-major) and the full-batch epoch buffers."""

    def __init__(self, T: int, E: int, D: int, W: int, act_dim: int, epochs: int, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        N = (T - 1) * E
        self.done = self.terminated                     # done = (discount == 0): terminated only (ff_vmpo.py:85)
        self.action = z(T, E, act_dim) if act_dim > 0 else z(T, E, dt=torch.int32)
        self.log_prob = z(T, E)
        self.head = z(E, W)                             # the rollout's target-actor head output of one step
        self.r, self.d = z(T, E), z(T, E)               # clip(reward), (1 - done) gamma: fixed over the epochs
        self.value, self.d_value = z(T, E), z(T, E)     # current critic on all T rows; d l2 loss / d v (zero on row T-1)
        self.head_o, self.head_t, self.d_head = z(N, W), z(N, W), z(N, W)
        self.mask = z(epochs, N, dt=torch.uint8)        # the selection of every epoch
        self.tau, self.count = z(1), z(1, dt=torch.int32)
        self.adv: Optional[torch.Tensor] = None
        self.targets: Optional[torch.Tensor] = None



def get_learner_fn(
    env: Environment,
    apply_fns: Tuple[Callable, Callable],
    update_fns: Tuple[Callable, Callable, Callable],
    config: DictConfig,
) -> LearnerFn[VMPOLearnerState]:
    """Get the learner function (ff_vmpo.py:55-324; ff_vmpo_continuous.py for a tanh-Normal actor).

    apply_fns: (actor_network.apply, critic_network.apply); update_fns: the actor, critic and dual optimisers' `.update`.  They are
    read for the shapes and hyper-parameters they are bound to; the arithmetic runs in the kernels named in the module header."""
    actor_apply_fn, critic_apply_fn = apply_fns
    actor_net = anakin.owner(actor_apply_fn, Actor, "apply_fns[0]")
    anakin.owner(critic_apply_fn, Critic, "apply_fns[1]")
    actor_opt, critic_opt, dual_opt = (anakin.owner(f, optax.GradientTransformation, f"update_fns[{i}]") for i, f in enumerate(update_fns))
    check_config(config)
    tanh_head = _actor_head(actor_net)
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, N = int(sysc.epochs), (T - 1) * E
    gamma, max_abs_reward = float(sysc.gamma), float(sysc.max_abs_reward)
    period = int(sysc.actor_target_period)
    per_dim = bool(sysc.get("per_dim_constraining", True))
    n_step = int(sysc.n_step_for_sequence_bootstrap) if bool(sysc.use_n_step_bootstrap) else 0
    kind = "tanh_normal" if tanh_head is not None else "categorical"
    eps_alpha = float(sysc.epsilon_mean) if tanh_head is not None else float(sysc.epsilon_policy)
    eps_stddev = float(sysc.epsilon_stddev) if tanh_head is not None else 0.0
    built: Dict[str, Any] = {}

    def _build(state: VMPOLearnerState) -> None:
        a_tree = state.params.actor_params.online
        sa, sc = a_tree.spec, state.params.critic_params.spec
        dev = a_tree.flat.device
        lay = vmpo_arena_layout(sa, sc, dual_count(tanh_head, per_dim))
        D, W = sa.sizes[0], sa.sizes[-1]
        segs = [(lay["actor"], sa.param_count, actor_opt), (lay["critic"], sc.param_count, critic_opt), (lay["duals"], lay["n_dual"], dual_opt)]
        built.update(
            sa=sa, sc=sc, dev=dev, lay=lay, D=D, arena=a_tree.arena, target=state.params.actor_params.target.flat,
            plan=optax.adam_plan(segs, dev, a_tree.arena_counts),
            shards=[_Shard(T, E, D, W, tanh_head.action_dim if tanh_head is not None else 0, epochs, dev) for _ in range(U)],
            grads=torch.zeros(lay["total"], dtype=torch.float32, device=dev),
            metrics=torch.zeros(epochs, len(ops.VMPO_METRICS), dtype=torch.float32, device=dev),
            ws_a=ops.mlp_train_workspace(sa, N, dev), ws_c=ops.mlp_train_workspace(sc, T * E, dev),
            roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # sampler call index
            graph=None, eager_done=False,
        )

    def _rollout_phase(state: VMPOLearnerState) -> None:
        """STEP ENVIRONMENT FOR ROLLOUT LENGTH (ff_vmpo.py:68-101), acting with the target actor; then r and d of the update."""
        b = built
        target = state.params.actor_params.target
        for u in range(U):
            sh: _Shard = b["shards"][u]
            for t in range(T):
                ops.mlp_forward(b["sa"], target.flat, sh.obs[t], out=sh.head, ws_key="vmpo")
                if tanh_head is None:
                    ops.categorical(sh.head, None, state.key[0] + u, t, b["roll_ctr"], out=(sh.action[t], sh.log_prob[t]))
                else:
                    lo, hi, ms = tanh_head.minimum, tanh_head.maximum, tanh_head.min_scale
                    ops.tanh_normal_sample(sh.head, lo, hi, ms, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], action_out=sh.action[t],
                                           want_eps=False)
                    ops.tanh_normal_log_prob(sh.head, sh.action[t], lo, hi, ms, out=sh.log_prob[t])
                anakin.step_env(env, state.env_state, u, sh.action[t], sh.step_out(t), t)
            torch.clamp(sh.reward, -max_abs_reward, max_abs_reward, out=sh.r)            # ff_vmpo.py:184-189
            torch.mul(1.0 - sh.done.float(), gamma, out=sh.d)

    def _targets(u: int, state: VMPOLearnerState) -> None:
        """Current critic on all T rows, then advantages and targets on the first T-1 (ff_vmpo.py:190-208)."""
        b, sh = built, built["shards"][u]
        sc, D = b["sc"], b["D"]
        ops.mlp_forward_train(sc, b["arena"][b["lay"]["critic"]:], sh.obs[:T].view(T * E, D), b["ws_c"], out=sh.value.view(T * E, 1))
        if n_step:
            sh.targets, sh.adv = ops.n_step_returns(sh.r[:-1], sh.d[:-1], sh.value[1:], n_step, v_tm1=sh.value[:-1], out=sh.targets,
                                                    adv_out=sh.adv)
        else:
            sh.adv, sh.targets, _ = ops.gae_generic(sh.r[:-1], sh.d[:-1], float(sysc.gae_lambda), sh.value[:-1], sh.value[1:])

    def _shard_grads(u: int, ep: int, state: VMPOLearnerState) -> None:
        """jax.grad of _actor_loss_fn (actor + duals) and _critic_loss_fn on shard u (ff_vmpo.py:114-226), weight 1/U."""
        b, sh = built, built["shards"][u]
        sa, sc, lay, D = b["sa"], b["sc"], b["lay"], b["D"]
        arena, grads, first = b["arena"], b["grads"], u == 0
        x_a = sh.obs[: T - 1].view(N, D)
        ops.vmpo_topk(sh.adv.view(N), tau=sh.tau, mask=sh.mask[ep], count=sh.count)
        ops.mlp_forward_train(sa, b["target"], x_a, b["ws_a"], out=sh.head_t)
        ops.mlp_forward_train(sa, arena, x_a, b["ws_a"], out=sh.head_o)
        lo, hi, ms = (tanh_head.minimum, tanh_head.maximum, tanh_head.min_scale) if tanh_head is not None else (-1.0, 1.0, 1e-3)
        ops.vmpo_loss_grads(kind, sh.head_o, sh.head_t, sh.action[: T - 1].reshape(N, -1) if tanh_head is not None else sh.action[: T - 1].reshape(N),
                            sh.adv.view(N), sh.mask[ep], sh.count, sh.value.view(T * E), sh.targets.view(N), arena[lay["duals"]: lay["duals"] + lay["n_dual"]],
                            sh.d_head, grads[lay["duals"]: lay["duals"] + lay["n_dual"]], b["metrics"][ep], float(sysc.epsilon), eps_alpha, eps_stddev,
                            per_dim=per_dim, d_value=sh.d_value.view(T * E), minimum=lo, maximum=hi, min_scale=ms, weight=1.0 / U, overwrite=first)
        ops.mlp_backward(sa, arena, x_a, sh.d_head, b["ws_a"], net_grad=grads[lay["actor"]:], grad_weight=1.0 / U, overwrite=first)
        ops.mlp_backward(sc, arena[lay["critic"]:], sh.obs[:T].view(T * E, D), sh.d_value.view(T * E, 1), b["ws_c"], net_grad=grads[lay["critic"]:],
                         grad_weight=1.0 / U, overwrite=first)

    def _update_epoch(state: VMPOLearnerState, ep: int) -> None:
        """One _update_epoch (ff_vmpo.py:111-289): targets and gradients of every shard, pmean, the three optimiser steps in one
        launch, the dual clamp and the periodic target update."""
        b = built
        for u in range(U):
            _targets(u, state)
            _shard_grads(u, ep, state)
        if world > 1:  # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        a_tree, lay = state.params.actor_params.online, b["lay"]
        ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu, grad_scale=1.0 / world)
        ops.vmpo_after_step(b["arena"][lay["duals"]: lay["duals"] + lay["n_dual"]], b["arena"][: b["sa"].param_count], b["target"],
                            b["plan"].counts[0:1], period)

    def _update_phase(state: VMPOLearnerState) -> None:
        """UPDATE EPOCHS (ff_vmpo.py:291-296)."""
        b = built
        b["metrics"].zero_()
        for ep in range(epochs):
            _update_epoch(state, ep)
        if world > 1:
            dist.all_reduce(b["metrics"], op=dist.ReduceOp.SUM)
            b["metrics"].mul_(1.0 / world)

    def _update_step(state: VMPOLearnerState) -> None:
        """A single update (ff_vmpo.py:67-303), in place on the learner state."""
        b = built
        for sh in b["shards"]:
            sh.carry_in()
        _rollout_phase(state)
        _update_phase(state)
        for sh, env_state in zip(b["shards"], state.env_state):
            sh.advance(env, env_state)
        ops.counter_add(b["roll_ctr"], T)

    def learner_fn(learner_state: VMPOLearnerState) -> AnakinExperimentOutput[VMPOLearnerState]:
        """Run arch.num_updates_per_eval update steps (ff_vmpo.py:305-322)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config)
        names = ops.VMPO_METRICS if tanh_head is not None else tuple(n for n in ops.VMPO_METRICS if n != "alpha_stddev")
        train_metrics = {("alpha_mean" if tanh_head is not None and n == "alpha" else n): train_out[..., ops.VMPO_METRICS.index(n)] for n in names}
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics=train_metrics)

    learner_fn.built = built
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    # "targets": one epoch's critic evaluation and targets of every shard (the update phase runs it `epochs` times)
    learner_fn.phases = {"rollout": _rollout_phase, "targets": lambda st: [_targets(u, st) for u in range(U)], "update": _update_phase}
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    return learner_fn


def _discrete_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    action_dim = int(env.action_space().num_values)   # ff_vmpo.py:335-336
    config.system.action_dim = action_dim
    return {"action_dim": action_dim}


def build_learner(env: Environment, keys: Tuple[int, int, int], config: DictConfig,
                  head_kwargs: Callable[[Environment, DictConfig], Dict[str, Any]]) -> Tuple[LearnerFn[VMPOLearnerState], Actor, VMPOLearnerState]:
    """The body of both systems' learner_setup (ff_vmpo.py:327-456, ff_vmpo_continuous.py:384-531).  head_kwargs(env, config) reads
    the action space, records it in config.system and returns the action head's constructor arguments."""
    check_config(config)
    rank, world = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())
    kwargs = head_kwargs(env, config)
    key, actor_net_key, critic_net_key = keys

    actor_network = Actor(torso=instantiate(config.network.actor_network.pre_torso),
                          action_head=instantiate(config.network.actor_network.action_head, **kwargs))
    critic_network = Critic(torso=instantiate(config.network.critic_network.pre_torso), critic_head=instantiate(config.network.critic_network.critic_head))
    tanh_head = _actor_head(actor_network)
    per_dim = bool(config.system.get("per_dim_constraining", True))

    lrs = [make_learning_rate(config.system[name], config, config.system.epochs) for name in ("actor_lr", "critic_lr", "dual_lr")]
    actor_optim, critic_optim, dual_optim = (optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(lr, eps=1e-5)) for lr in lrs)

    init_x = env.observation_space().generate_value()[None, ...].to(device).float()
    sa, sc = actor_network.spec_for(init_x.shape[-1]), critic_network.spec_for(init_x.shape[-1])
    lay = vmpo_arena_layout(sa, sc, dual_count(tanh_head, per_dim))
    arena = torch.zeros(lay["total"], dtype=torch.float32, device=device)
    actor_params = actor_network.init(actor_net_key, init_x, flat=arena[lay["actor"]:])
    critic_params = critic_network.init(critic_net_key, init_x, flat=arena[lay["critic"]:])

    # Dual parameters (ff_vmpo.py:377-383; ff_vmpo_continuous.py:437-460) in the arena's dual segment.
    duals = arena[lay["duals"]: lay["duals"] + lay["n_dual"]]
    duals[0] = float(config.system.init_log_temperature)
    if tanh_head is None:
        duals[1] = float(config.system.init_log_alpha)
        dual_params = CategoricalDualParams(duals[0:1], duals[1:2])
    else:
        d = (lay["n_dual"] - 1) // 2
        duals[1: 1 + d] = float(config.system.init_log_alpha_mean)
        duals[1 + d:] = float(config.system.init_log_alpha_stddev)
        dual_params = DualParams(duals[0:1], duals[1: 1 + d], duals[1 + d:])

    opt_states = VMPOOptStates(*optax.arena_state(actor_params, arena, [(lay["actor"], sa.param_count), (lay["critic"], sc.param_count),
                                                                         (lay["duals"], lay["n_dual"])]))
    learn = get_learner_fn(env, (actor_network.apply, critic_network.apply), (actor_optim.update, critic_optim.update, dual_optim.update), config)

    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 1)
    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    warm_start(config, arena)   # parameters only (ff_vmpo.py:422-431); the target starts as a copy of the online actor
    target_arena = arena[: sa.param_count].clone()
    target_params = build_param_tree(sa, target_arena, "action_head")
    params = VMPOParams(OnlineAndTarget(actor_params, target_params), critic_params, dual_params)

    rollout_seed, _ = anakin.rank_seeds(shard_keys[U], 2, rank, world)
    learner_step_count = actor_params.arena_counts[0:1]   # the actor segment's Adam count (ff_vmpo.py:438, 266)
    init_learner_state = VMPOLearnerState(params, opt_states, (rollout_seed,), env_states, timesteps, learner_step_count)
    return learn, actor_network, init_learner_state


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig) -> Tuple[LearnerFn[VMPOLearnerState], Actor, VMPOLearnerState]:
    """Initialise learner_fn, networks, optimisers, environment and states (ff_vmpo.py:327-456)."""
    return build_learner(env, keys, config, _discrete_head_kwargs)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_vmpo.py:459-602): the ONLINE actor is evaluated, tracked and checkpointed (:488-489, :519)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2, policy=lambda s: s.params.actor_params.online)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_vmpo: `python -m stoix_b200.systems.mpo.ff_vmpo arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_vmpo", run_experiment, "V-MPO")


if __name__ == "__main__":
    hydra_entry_point()
