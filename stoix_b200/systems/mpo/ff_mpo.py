"""Anakin MPO on H100 -- drop-in for stoix/systems/mpo/ff_mpo.py (Categorical actor); ff_mpo_continuous.py runs the same learner
with a tanh-Normal actor and the decoupled loss.

Same entry points and signatures (get_warmup_fn :57-112, get_learner_fn :115-426, learner_setup :429-607, run_experiment :610-753,
hydra_entry_point) and the same learner-state shape (mpo_types.py: OnlineAndTarget actor and Q, duals, three optimiser states and
the replay buffer state):

  reference (JAX)                                     here (H100)
  --------------------------------------------------  -----------------------------------------------------------------
  flashbax trajectory buffer (add / sample)           device sequence ring (stx_replay_add_sequence / _sample_sequence): one
                                                      launch writes the B sampled sequences time-major into the epoch buffers
  target Q on all A one-hot actions / num_samples     stx_mpo_sample_actions writes every target-Q input row of the epoch in one
  target-policy draws (actor loss) and on N sampled   launch: the actor-loss rows, N bootstrap draws, the stored action; one fp32
  actions (bootstrap), per state                      stx_mlp_forward of the target Q runs over all of them
  categorical_mpo_loss / mpo_loss + jax.grad          stx_mpo_loss_grads: head gradient, dual gradients, metrics and the
                                                      bootstrap value v_t = mean_N Q in one launch
  Retrace / n-step / GAE targets, l2 loss             stx_retrace_f32 / stx_n_step_returns_f32 / K2 stx_gae_generic_f32 on
                                                      time-major views of v_t, then stx_mpo_q_grad
  3 x chain(clip_by_global_norm, adam), clip at -18,  one clip + Adam launch over [actor | Q | duals], the -18 clamp of
  incremental_update of both targets                  stx_vmpo_after_step, one stx_polyak_update over the [actor | Q] target arena
  pmean(batch); pmean(device)                         mean over update-batch shards; one NCCL all-reduce of the gradient arena
  one XLA program per learn() call                    one CUDA graph per update step, replayed

Reference quirks kept: the truncation flag is stored but not read by the targets; the bootstrap draws N actions from the
Categorical policy although it could enumerate its A actions (the actor loss does enumerate them); the continuous _q_loss_fn reads the
stored actions through the enclosing `sequence` (ff_mpo_continuous.py:232), the same values as its own argument.

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
from stoix_b200.networks.base import FeedForwardQ, build_param_tree
from stoix_b200.networks.heads import CategoricalHead, NormalAffineTanhDistributionHead
from stoix_b200.systems import anakin
from stoix_b200.systems.mpo.ff_vmpo import dual_count
from stoix_b200.systems.mpo.mpo_types import CategoricalDualParams, DualParams, MPOLearnerState, MPOOptStates, MPOParams, OnlineAndTarget, SequenceStep
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.replay import SequenceBuffer
from stoix_b200.utils.training import make_learning_rate

_pad8 = lambda n: (int(n) + 7) // 8 * 8
_NO_COPY_PERIOD = 2**31 - 1   # stx_vmpo_after_step copies only when the Adam count is a multiple of this, which it never reaches


def mpo_arena_layout(actor: ops.MlpSpec, q: ops.MlpSpec, n_dual: int = 2) -> Dict[str, int]:
    """[actor | Q | duals], every block padded to 8 floats; the duals are [log_temperature, log_alpha] (Categorical) or
    [log_temperature, log_alpha_mean (C), log_alpha_stddev (C)] (tanh-Normal).  The target arena mirrors [actor | Q] = arena[0:duals]."""
    off_q = _pad8(actor.param_count)
    off_d = off_q + _pad8(q.param_count)
    return {"actor": 0, "q": off_q, "duals": off_d, "n_dual": int(n_dual), "total": off_d + _pad8(n_dual)}


def check_config(config: DictConfig) -> None:
    """The refusals of both MPO systems: bf16, period != 1, sequences too short to have a target, and a first sample before one
    sequence has been written."""
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for MPO: the bf16 tensor-core kernels implement the PPO clipped surrogate only, "
                         "not the sampled-action E-step and the KL-constrained loss; use arch.precision=f32")
    if int(config.system.get("period", 1)) != 1:
        raise ValueError(f"system.period={config.system.period}: only period 1 is implemented (both reference MPO configs use 1)")
    if int(config.system.sample_sequence_length) < 2:
        raise ValueError(f"system.sample_sequence_length={config.system.sample_sequence_length}: the Q targets of a sequence need a next "
                         "row (ff_mpo.py:277-303), so it must be >= 2")
    if int(config.system.warmup_steps) + int(config.system.rollout_length) < int(config.system.sample_sequence_length):
        raise ValueError(f"system.warmup_steps={config.system.warmup_steps} + rollout_length={config.system.rollout_length} time rows are written "
                         f"before the first sample, fewer than one sequence of sample_sequence_length={config.system.sample_sequence_length}")


def _actor_head(actor_net: Actor) -> Optional[NormalAffineTanhDistributionHead]:
    """The tanh-Normal head, None for the Categorical head; any other head is refused."""
    head = actor_net.action_head
    if isinstance(head, NormalAffineTanhDistributionHead):
        return head
    if isinstance(head, CategoricalHead):
        return None
    raise ValueError(f"MPO implements the Categorical (CategoricalHead) and tanh-Normal (NormalAffineTanhDistributionHead) actors; got "
                     f"{type(head).__name__}")


class _Shard(anakin.Trajectory):
    """One (device, update-batch) shard: the rollout's SequenceStep fields (time-major), its replay buffer and the epoch buffers of
    one sampled batch of B sequences of S rows (M = S B states, time-major)."""

    def __init__(self, T: int, E: int, S: int, B: int, D: int, A: int, NL: int, N: int, tanh: bool, sa: ops.MlpSpec, sq: ops.MlpSpec,
                 buffer: SequenceBuffer, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        M, W = S * B, sa.sizes[-1]
        self.done = self.terminated                     # done = (discount == 0): terminated only (ff_mpo.py:146)
        self.action = z(T, E, A) if tanh else z(T, E, dt=torch.int32)
        self.log_prob, self.head = z(T, E), z(E, W)
        self.buffer = buffer
        self.s_obs, self.s_reward = z(S, B, D), z(S, B)
        self.s_action = z(S, B, A) if tanh else z(S, B, dt=torch.int32)
        self.s_done, self.s_log_prob = z(S, B, dt=torch.uint8), z(S, B)
        self.head_o, self.head_t, self.d_head = z(M, W), z(M, W), z(M, W)
        self.act_cont = z(NL, M, A) if tanh else None   # the unclipped actor-loss draws of the target policy
        self.xq = z((NL + N + 1) * M, D + A)            # target-Q input rows: NL actor-loss rows, N bootstrap draws, the stored action
        self.q_t = z((NL + N + 1) * M, 1)               # target Q of those rows
        self.q_on, self.dq = z(S, B), z(S, B)           # online Q on the stored actions and d q_loss / d q
        self.log_rho, self.r, self.d, self.v = z(S, B), z(S, B), z(S, B), z(S, B)
        self.targets = z(S - 1, B)
        self.ws_a, self.ws_q = ops.mlp_train_workspace(sa, M, device), ops.mlp_train_workspace(sq, M, device)

    def sequence_step(self) -> SequenceStep:
        return SequenceStep(self.obs[: self.T], self.action, self.reward, self.done, self.truncated, self.log_prob,
                            {"episode_return": self.episode_return, "episode_length": self.episode_length, "is_terminal_step": self.is_terminal_step})


def get_warmup_fn(env: Environment, params: MPOParams, actor_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """ff_mpo.py:57-112: `warmup_steps` environment steps of one shard with the online actor, added to its buffer as SequenceSteps
    (with the behaviour log_prob, which Retrace reads)."""
    W = int(config.system.warmup_steps)

    def warmup(env_state, timestep, buffer_state, key: int):
        obs_l, act_l, rew_l, done_l, trunc_l, lp_l = [], [], [], [], [], []
        for t in range(W):
            obs = timestep.observation.float().clone()
            pi = actor_apply_fn(params.actor_params.online, obs)
            action = pi.sample(seed=key, offset=t, dev_counter=None)
            log_prob = pi.log_prob(action)
            env_state, timestep = env.step(env_state, action)
            done = timestep.discount == 0.0
            obs_l.append(obs), act_l.append(action if action.is_floating_point() else action.to(torch.int32)), rew_l.append(timestep.reward.float()), lp_l.append(log_prob.float())
            done_l.append(done.to(torch.uint8)), trunc_l.append((timestep.last() & ~done).to(torch.uint8))
        if W > 0:
            st = lambda xs: torch.stack(xs).contiguous()
            buffer_add_fn(buffer_state, SequenceStep(st(obs_l), st(act_l), st(rew_l), st(done_l), st(trunc_l), st(lp_l), {}))
        return env_state, timestep, key, buffer_state

    return warmup


def get_learner_fn(env: Environment, apply_fns: Tuple[Callable, Callable], update_fns: Tuple[Callable, Callable, Callable],
                   buffer_fns: Tuple[Callable, Callable], config: DictConfig) -> LearnerFn[MPOLearnerState]:
    """Get the learner function (ff_mpo.py:115-426).  apply_fns = (actor_network.apply, q_network.apply), update_fns = the actor, Q
    and dual optimisers' `.update`: read for the shapes and hyper-parameters they are bound to.  buffer_fns = (SequenceBuffer.add,
    SequenceBuffer.sample_into) unbound, applied to learner_state.buffer_state[u]."""
    actor_apply_fn, q_apply_fn = apply_fns
    actor_net = anakin.owner(actor_apply_fn, Actor, "apply_fns[0]")
    anakin.owner(q_apply_fn, FeedForwardQ, "apply_fns[1]")
    actor_opt, q_opt, dual_opt = (anakin.owner(f, optax.GradientTransformation, f"update_fns[{i}]") for i, f in enumerate(update_fns))
    buffer_add_fn, buffer_sample_fn = buffer_fns
    check_config(config)
    tanh_head = _actor_head(actor_net)
    kind = "tanh_normal" if tanh_head is not None else "categorical"
    per_dim = bool(config.system.get("per_dim_constraining", True))
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, B, S = int(sysc.epochs), int(sysc.batch_size), int(sysc.sample_sequence_length)
    M = S * B
    stochastic = bool(sysc.stochastic_policy_eval)
    N = int(sysc.num_samples) if stochastic else 1
    gamma, tau, max_abs_reward = float(sysc.gamma), float(sysc.tau), float(sysc.max_abs_reward)
    use_retrace, n_step = bool(sysc.use_retrace), (int(sysc.n_step_for_sequence_bootstrap) if bool(sysc.use_n_step_bootstrap) else 0)
    online_bootstrap = bool(sysc.use_online_policy_to_bootstrap)
    eps_policy = float(sysc.epsilon_mean) if tanh_head is not None else float(sysc.epsilon_policy)
    eps_stddev = float(sysc.epsilon_stddev) if tanh_head is not None else 0.0
    lo, hi, ms = (tanh_head.minimum, tanh_head.maximum, tanh_head.min_scale) if tanh_head is not None else (-1.0, 1.0, 1e-3)
    metric_names = ops.MPO_CONTINUOUS_METRICS if tanh_head is not None else ops.MPO_METRICS
    built: Dict[str, Any] = {}

    def _build(state: MPOLearnerState) -> None:
        a_tree = state.params.actor_params.online
        sa, sq = a_tree.spec, state.params.q_params.online.spec
        dev = a_tree.flat.device
        lay = mpo_arena_layout(sa, sq, dual_count(tanh_head, per_dim))
        D = sa.sizes[0]
        A = tanh_head.action_dim if tanh_head is not None else sa.sizes[-1]
        NL = int(sysc.num_samples) if tanh_head is not None else A
        segs = [(lay["actor"], sa.param_count, actor_opt), (lay["q"], sq.param_count, q_opt), (lay["duals"], lay["n_dual"], dual_opt)]
        built.update(
            sa=sa, sq=sq, dev=dev, lay=lay, D=D, A=A, NL=NL, arena=a_tree.arena, target=a_tree.target_arena,
            plan=optax.adam_plan(segs, dev, a_tree.arena_counts),
            shards=[_Shard(T, E, S, B, D, A, NL, N, tanh_head is not None, sa, sq, state.buffer_state[u], dev) for u in range(U)],
            grads=torch.zeros(lay["total"], dtype=torch.float32, device=dev),
            metrics=torch.zeros(epochs, len(metric_names), dtype=torch.float32, device=dev),
            no_copy=torch.zeros(2, dtype=torch.float32, device=dev),   # the after-step kernel's (unused) target-copy pair
            roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),    # rollout sampler call index
            act_ctr=torch.zeros(1, dtype=torch.int64, device=dev),     # bootstrap-draw call index
            graph=None, eager_done=False,
        )

    def _rollout_phase(state: MPOLearnerState) -> None:
        """STEP ENVIRONMENT FOR ROLLOUT LENGTH with the online actor, then add the trajectory to the buffer (ff_mpo.py:130-169)."""
        b = built
        for u in range(U):
            sh: _Shard = b["shards"][u]
            for t in range(T):
                ops.mlp_forward(b["sa"], b["arena"], sh.obs[t], out=sh.head, ws_key="mpo_rollout")
                if tanh_head is None:
                    ops.categorical(sh.head, None, state.key[0] + u, t, b["roll_ctr"], out=(sh.action[t], sh.log_prob[t]))
                else:
                    ops.tanh_normal_sample(sh.head, lo, hi, ms, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], action_out=sh.action[t],
                                           want_eps=False)
                    ops.tanh_normal_log_prob(sh.head, sh.action[t], lo, hi, ms, out=sh.log_prob[t])
                anakin.step_env(env, state.env_state, u, sh.action[t], sh.step_out(t), t)
            buffer_add_fn(sh.buffer, sh.sequence_step())

    def _shard_grads(u: int, ep: int, state: MPOLearnerState, sample: bool = True, idx_in: Optional[torch.Tensor] = None,
                     act_in: Optional[torch.Tensor] = None, eps_in: Optional[torch.Tensor] = None) -> None:
        """Sample B sequences, then jax.grad of _actor_loss_fn (actor + duals) and of _q_loss_fn on shard u (ff_mpo.py:174-339), weight
        1/U.  idx_in / act_in / eps_in: injected sequence indices, Categorical bootstrap actions, tanh-Normal noise (tests)."""
        b, sh = built, built["shards"][u]
        sa, sq, lay, D, A, NL = b["sa"], b["sq"], b["lay"], b["D"], b["A"], b["NL"]
        arena, target, grads, first, w = b["arena"], b["target"], b["grads"], u == 0, 1.0 / U
        nd = lay["n_dual"]
        duals, d_grads = arena[lay["duals"]: lay["duals"] + nd], grads[lay["duals"]: lay["duals"] + nd]
        if sample:
            buffer_sample_fn(sh.buffer, sh.s_obs, sh.s_action, sh.s_reward, sh.s_done, sh.s_log_prob, idx_in=idx_in)
        x = sh.s_obs.view(M, D)
        ops.mlp_forward(sa, target, x, out=sh.head_t, ws_key="mpo_target_actor")
        ops.mlp_forward_train(sa, arena, x, sh.ws_a, out=sh.head_o)
        ops.mpo_sample_actions(x, sh.head_t, sh.head_o if online_bootstrap else sh.head_t, sh.s_action.view(M, -1) if tanh_head is not None
                               else sh.s_action.view(M), sh.s_log_prob.view(M), sh.s_reward.view(M), sh.s_done.view(M), N, sh.xq, sh.log_rho.view(M),
                               sh.r.view(M), sh.d.view(M), gamma, max_abs_reward, stochastic=stochastic, seed=state.key[1] + 0x9E37 * u,
                               dev_counter=b["act_ctr"], act_in=act_in, kind=kind, NL=NL, act_cont_out=sh.act_cont, eps_in=eps_in, minimum=lo,
                               maximum=hi, min_scale=ms)
        rows = (NL + N + (1 if use_retrace else 0)) * M
        ops.mlp_forward(sq, target[lay["q"]:], sh.xq[:rows], out=sh.q_t[:rows], ws_key="mpo_target_q")
        x_on = sh.xq[(NL + N) * M:]
        ops.mlp_forward_train(sq, arena[lay["q"]:], x_on, sh.ws_q, out=sh.q_on.view(M, 1))
        ops.mpo_loss_grads(sh.head_o, sh.head_t, sh.q_t[: NL * M], duals, sh.d_head, d_grads, b["metrics"][ep], float(sysc.epsilon), eps_policy,
                           q_boot=sh.q_t[NL * M: (NL + N) * M], v=sh.v.view(M), weight=w, overwrite=first, kind=kind, actions=sh.act_cont,
                           epsilon_stddev=eps_stddev, per_dim=per_dim, minimum=lo, maximum=hi, min_scale=ms)
        if use_retrace:   # batch_retrace_continuous(online_q_t[:, :-1], target_q_t[:, 1:-1], v_t[:, 1:], r_t[:, :-1], d_t[:, :-1], log_rhos[:, 1:-1])
            q_stored = sh.q_t[(NL + N) * M:].view(S, B)
            ops.retrace(q_stored[1: S - 1], sh.v[1:], sh.r[:-1], sh.d[:-1], sh.log_rho[1: S - 1], float(sysc.retrace_lambda), out=sh.targets)
        elif n_step:
            ops.n_step_returns(sh.r[:-1], sh.d[:-1], sh.v[1:], n_step, out=sh.targets)
        else:
            _, tgt, _ = ops.gae_generic(sh.r[:-1], sh.d[:-1], float(sysc.gae_lambda), sh.v[:-1], sh.v[1:])
            sh.targets.copy_(tgt)
        ops.mpo_q_grad(sh.q_on, sh.targets, sh.dq, metric=b["metrics"][ep, len(metric_names) - 1:], weight=w)
        ops.mlp_backward(sa, arena, x, sh.d_head, sh.ws_a, net_grad=grads[lay["actor"]:], grad_weight=w, overwrite=first)
        ops.mlp_backward(sq, arena[lay["q"]:], x_on, sh.dq.view(M, 1), sh.ws_q, net_grad=grads[lay["q"]:], grad_weight=w, overwrite=first)

    def _update_epoch(state: MPOLearnerState, ep: int, sample: bool = True, idx_in=None, act_in=None, eps_in=None) -> None:
        """One _update_epoch (ff_mpo.py:171-391): gradients of every shard, pmean, the three optimiser steps in one launch, the dual
        clamp and the Polyak update of both targets."""
        b = built
        for u in range(U):
            _shard_grads(u, ep, state, sample=sample, idx_in=idx_in, act_in=act_in, eps_in=eps_in)
        ops.counter_add(b["act_ctr"], 1)
        if world > 1:   # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        a_tree, lay = state.params.actor_params.online, b["lay"]
        ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu, grad_scale=1.0 / world)
        ops.vmpo_after_step(b["arena"][lay["duals"]: lay["duals"] + lay["n_dual"]], b["no_copy"][0:1], b["no_copy"][1:2], b["plan"].counts[4:5],
                            _NO_COPY_PERIOD)
        ops.polyak_update(b["target"], b["arena"][: lay["duals"]], tau)

    def _update_phase(state: MPOLearnerState) -> None:
        """UPDATE EPOCHS (ff_mpo.py:393-398)."""
        b = built
        b["metrics"].zero_()
        for ep in range(epochs):
            _update_epoch(state, ep)
        if world > 1:
            dist.all_reduce(b["metrics"], op=dist.ReduceOp.SUM)
            b["metrics"].mul_(1.0 / world)

    def _update_step(state: MPOLearnerState) -> None:
        """A single update (ff_mpo.py:129-405), in place on the learner state."""
        b = built
        for sh in b["shards"]:
            sh.carry_in()
        _rollout_phase(state)
        _update_phase(state)
        for sh, env_state in zip(b["shards"], state.env_state):
            sh.advance(env, env_state)
        ops.counter_add(b["roll_ctr"], T)

    def learner_fn(learner_state: MPOLearnerState) -> AnakinExperimentOutput[MPOLearnerState]:
        """Run arch.num_updates_per_eval update steps (ff_mpo.py:407-424)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, buffers=learner_state.buffer_state)
        train_metrics = {n: train_out[..., j] for j, n in enumerate(metric_names)}
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics=train_metrics)

    learner_fn.built = built
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.shard_grads = _shard_grads
    learner_fn.rollout_phase = _rollout_phase
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    return learner_fn


def _discrete_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    action_dim = int(env.action_space().num_values)   # ff_mpo.py:437-438
    config.system.action_dim = action_dim
    return {"action_dim": action_dim}


def build_learner(env: Environment, keys: Tuple[int, int, int], config: DictConfig,
                  head_kwargs: Callable[[Environment, DictConfig], Dict[str, Any]]) -> Tuple[LearnerFn[MPOLearnerState], Actor, MPOLearnerState]:
    """The body of both systems' learner_setup (ff_mpo.py:429-607, ff_mpo_continuous.py).  head_kwargs(env, config) reads the action
    space, records it in config.system and returns the action head's constructor arguments."""
    check_config(config)
    rank, n_devices = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())
    kwargs = head_kwargs(env, config)
    key, actor_net_key, q_net_key = keys

    actor_network = Actor(torso=instantiate(config.network.actor_network.pre_torso),
                          action_head=instantiate(config.network.actor_network.action_head, **kwargs))
    tanh_head = _actor_head(actor_network)
    per_dim = bool(config.system.get("per_dim_constraining", True))
    act_in_dim = tanh_head.action_dim if tanh_head is not None else int(kwargs["action_dim"])   # one-hot width or action dims
    q_network = FeedForwardQ(critic_head=instantiate(config.network.q_network.critic_head), torso=instantiate(config.network.q_network.pre_torso),
                             input_layer=instantiate(config.network.q_network.input_layer))

    lrs = [make_learning_rate(config.system[name], config, config.system.epochs) for name in ("actor_lr", "q_lr", "dual_lr")]
    actor_optim, q_optim, dual_optim = (optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(lr, eps=1e-5)) for lr in lrs)

    init_x = env.observation_space().generate_value()[None, ...].to(device).float()
    init_xa = torch.cat([init_x, torch.zeros(1, act_in_dim, device=device)], dim=-1)   # [obs | one_hot(a)] or [obs | a]
    sa, sq = actor_network.spec_for(init_x.shape[-1]), q_network.spec_for(init_xa.shape[-1])
    lay = mpo_arena_layout(sa, sq, dual_count(tanh_head, per_dim))
    arena = torch.zeros(lay["total"], dtype=torch.float32, device=device)
    actor_params = actor_network.init(actor_net_key, init_x, flat=arena[lay["actor"]:])
    q_params = q_network.init(q_net_key, init_xa, flat=arena[lay["q"]:])

    nd = lay["n_dual"]
    duals = arena[lay["duals"]: lay["duals"] + nd]   # ff_mpo.py:484-491, ff_mpo_continuous.py:500-522
    duals[0] = float(config.system.init_log_temperature)
    if tanh_head is None:
        duals[1] = float(config.system.init_log_alpha)
        dual_params = CategoricalDualParams(duals[0:1], duals[1:2])
    else:
        c = (nd - 1) // 2
        duals[1: 1 + c] = float(config.system.init_log_alpha_mean)
        duals[1 + c:] = float(config.system.init_log_alpha_stddev)
        dual_params = DualParams(duals[0:1], duals[1: 1 + c], duals[1 + c:])
    opt_states = MPOOptStates(*optax.arena_state(actor_params, arena, [(lay["actor"], sa.param_count), (lay["q"], sq.param_count), (lay["duals"], nd)]))

    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 2)
    E = int(config.arch.num_envs)
    buffer_states = anakin.replay_buffers(
        config, shard_keys[U], rank, n_devices,
        lambda size, batch, seed: SequenceBuffer(size, batch, int(config.system.sample_sequence_length), E, init_x.shape[-1], device,
                                                 period=int(config.system.period), seed=seed,
                                                 act_dim=tanh_head.action_dim if tanh_head is not None else 0))
    learn = get_learner_fn(env, (actor_network.apply, q_network.apply), (actor_optim.update, q_optim.update, dual_optim.update),
                           (SequenceBuffer.add, SequenceBuffer.sample_into), config)

    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)
    warm_start(config, arena)   # parameters only (ff_mpo.py:569-578); the targets start as copies of the online networks
    target_arena = arena[: lay["duals"]].clone()
    actor_params.target_arena = target_arena
    params = MPOParams(OnlineAndTarget(actor_params, build_param_tree(sa, target_arena, "action_head")),
                       OnlineAndTarget(q_params, build_param_tree(sq, target_arena[lay["q"]:], "critic_head")), dual_params)

    rollout_seed, act_seed, warm_seed = anakin.rank_seeds(shard_keys[U + 1], 3, rank, n_devices)
    warmup = get_warmup_fn(env, params, actor_network.apply, SequenceBuffer.add, config)
    for u in range(U):   # ff_mpo.py:599-602
        env_states[u], timesteps[u], _, _ = warmup(env_states[u], timesteps[u], buffer_states[u], warm_seed + 0xA5A5 * u)
    init_learner_state = MPOLearnerState(params, opt_states, buffer_states, (rollout_seed, act_seed), env_states, timesteps)
    return learn, actor_network, init_learner_state


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig) -> Tuple[LearnerFn[MPOLearnerState], Actor, MPOLearnerState]:
    """Initialise learner_fn, networks, optimisers, buffer, environment and states (ff_mpo.py:429-607)."""
    return build_learner(env, keys, config, _discrete_head_kwargs)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_mpo.py:610-753): the ONLINE actor is evaluated, tracked and checkpointed (:639-640, :698-699)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2, policy=lambda s: s.params.actor_params.online)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point with config default_ff_mpo: `python -m stoix_b200.systems.mpo.ff_mpo arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_mpo", run_experiment, "MPO")


if __name__ == "__main__":
    hydra_entry_point()
