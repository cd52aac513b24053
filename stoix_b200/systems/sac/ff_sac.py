"""Anakin feed-forward SAC on H100 -- drop-in for stoix/systems/sac/ff_sac.py (SURVEY.md 8f row 4, fp32).

Same entry points and signatures (get_warmup_fn :40-92, get_learner_fn :95-344, learner_setup :347-513, run_experiment :516,
hydra_entry_point) and the same state / output contracts (sac_types.py), on a different machine:

  reference (JAX)                                      here (H100)
  ---------------------------------------------------  ------------------------------------------------------------------
  flashbax item buffer (add / sample, host-traced)      device ring buffer, write position in HBM (stx_replay_add / _sample):
                                                        ONE launch lays the sampled batch out as the three network inputs
  3 x jax.grad (actor, twin-Q, alpha) per epoch         train-mode MLP kernels (stx_mlp_forward_train / _backward: silu,
                                                        LayerNorm), tanh-Normal head kernels with reparameterised backward,
                                                        three small loss kernels; the actor loss reaches the policy through
                                                        d Q / d action of the twin-Q backward (no parameter gradients there)
  3 x optax.chain(clip, adam) + incremental_update      one fused clip+Adam launch over [actor | q1 q2 | log_alpha], one Polyak
  pmean(batch); pmean(device)                           mean over update-batch shards; one NCCL all-reduce of the gradient arena
  one XLA program per learn() call                      one CUDA graph per update step (rollout + add + epochs), replayed

Every random stream position (policy noise, replay indices) is a device counter, so graph replays draw fresh numbers.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import FeedForwardQ, MultiNetwork, build_param_tree
from stoix_b200.systems import anakin
from stoix_b200.systems.sac.sac_types import OffPolicyLearnerState, OnlineAndTarget, SACOptStates, SACParams, Transition
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.replay import TransitionBuffer
from stoix_b200.utils.training import make_learning_rate

_METRIC_NAMES = ("actor_loss", "entropy", "q_loss", "q_error", "q1_pred", "q2_pred", "alpha_loss", "alpha")
_pad8 = lambda n: (int(n) + 7) // 8 * 8


def sac_arena_layout(actor: ops.MlpSpec, q: ops.MlpSpec) -> Dict[str, int]:
    """[actor | q1 | q2 | log_alpha], every block padded to 8 floats; the Q optimiser segment is q1..q2 (both networks: ONE global
    norm, like optax over the MultiNetwork tree); the target arena mirrors the [q1 | q2] block."""
    off_q1 = _pad8(actor.param_count)
    off_q2 = off_q1 + _pad8(q.param_count)
    off_alpha = off_q2 + _pad8(q.param_count)
    return {"actor": 0, "q1": off_q1, "q2": off_q2, "alpha": off_alpha, "total": off_alpha + 8, "q_block": off_alpha - off_q1}


class _Shard(anakin.Trajectory):
    """Per (device, update-batch) shard: rollout trajectory (Transition fields, time-major), replay buffer, epoch workspaces."""

    def __init__(self, T: int, E: int, B: int, D: int, A: int, sa: ops.MlpSpec, sq: ops.MlpSpec, buffer: TransitionBuffer, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.action = z(T, E, A)
        self.done = z(T, E, dt=torch.uint8)         # timestep.last() = terminated | truncated
        self.buffer = buffer
        # one sampled batch as the three network inputs (obs | action), leading dimension D + A
        self.xq_old, self.xq_new, self.xq_next = z(B, D + A), z(B, D + A), z(B, D + A)
        self.b_reward, self.b_done, self.b_idx = z(B), z(B, dt=torch.uint8), z(B, dt=torch.int32)
        self.ws_actor, self.ws_actor_next = ops.mlp_train_workspace(sa, B, device), ops.mlp_train_workspace(sa, B, device)
        self.ws_q = [ops.mlp_train_workspace(sq, B, device) for _ in range(2)]
        self.ws_qt = [ops.mlp_train_workspace(sq, B, device) for _ in range(2)]
        self.head, self.head_next, self.d_head = z(B, 2 * A), z(B, 2 * A), z(B, 2 * A)
        self.q = [z(B, 1) for _ in range(2)]        # Q_k(obs, .) -- first on the fresh action, then on the stored one
        self.nq = [z(B, 1) for _ in range(2)]       # target Q_k(next_obs, next action)
        self.dq = [z(B, 1) for _ in range(2)]
        self.d_in = [z(B, D + A) for _ in range(2)]

    def transition(self) -> Transition:
        return Transition(self.obs[: self.T], self.action, self.reward, self.done, self.next_obs,
                          {"episode_return": self.episode_return, "episode_length": self.episode_length, "is_terminal_step": self.is_terminal_step})


def get_warmup_fn(env: Environment, params: SACParams, actor_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """ff_sac.py:40-92: `warmup_steps` environment steps with the initial policy, added to the buffer (one shard per call)."""
    draw = lambda obs, key, t: actor_apply_fn(params.actor_params, obs).sample(seed=key, offset=t, dev_counter=None)
    return anakin.warmup_fn(env, draw, buffer_add_fn, config)


def get_learner_fn(env: Environment, apply_fns: Tuple[Callable, Callable], update_fns: Tuple[Callable, Callable, Callable],
                   buffer_fns: Tuple[Callable, Callable], config: DictConfig):
    """ff_sac.py:95-344.  apply_fns = (actor_network.apply, double_q_network.apply), update_fns = the three optimisers' `.update`;
    they are read for the shapes / hyper-parameters they are bound to, the arithmetic runs in the kernels named in the header.
    buffer_fns = (TransitionBuffer.add, TransitionBuffer.sample_into) unbound, applied to learner_state.buffer_state[u]."""
    actor_apply_fn, q_apply_fn = apply_fns
    actor_net = anakin.owner(actor_apply_fn, Actor, "apply_fns[0]")
    anakin.owner(q_apply_fn, MultiNetwork, "apply_fns[1]")
    actor_opt, q_opt, alpha_opt = (anakin.owner(f, optax.GradientTransformation, f"update_fns[{i}]") for i, f in enumerate(update_fns))
    buffer_add_fn, buffer_sample_fn = buffer_fns
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, B = int(sysc.epochs), int(sysc.batch_size)
    gamma, tau, autotune = float(sysc.gamma), float(sysc.tau), bool(sysc.autotune)
    target_entropy = float(sysc.target_entropy)
    lo, hi = float(sysc.action_minimum), float(sysc.action_maximum)
    min_scale = float(actor_net.action_head.min_scale)
    built: Dict[str, Any] = {}

    def _build(state: OffPolicyLearnerState) -> None:
        a_tree = state.params.actor_params
        sa, sq = a_tree.spec, state.params.q_params.online[0].spec
        dev = a_tree.flat.device
        lay = sac_arena_layout(sa, sq)
        D, A = sa.sizes[0], sa.sizes[-1] // 2
        segs = [(lay["actor"], sa.param_count, actor_opt), (lay["q1"], lay["q_block"], q_opt)] + ([(lay["alpha"], 1, alpha_opt)] if autotune else [])
        plan = optax.adam_plan(segs, dev, a_tree.arena_counts[: 2 * len(segs)])
        shards = [_Shard(T, E, B, D, A, sa, sq, state.buffer_state[u], dev) for u in range(U)]
        built.update(sa=sa, sq=sq, dev=dev, lay=lay, D=D, A=A, plan=plan, shards=shards, arena=a_tree.arena, target=a_tree.target_arena,
                     grads=torch.zeros(lay["total"], dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, 8, dtype=torch.float32, device=dev),
                     act_ctr=torch.zeros(1, dtype=torch.int64, device=dev),     # policy-noise stream position (rollout)
                     eps_ctr=torch.zeros(1, dtype=torch.int64, device=dev),     # policy-noise stream position (losses)
                     graph=None, eager_done=False)

    def _rollout_phase(state: OffPolicyLearnerState) -> None:
        """_env_step x rollout_length (ff_sac.py:114-146) + buffer add (:149-150), per shard."""
        b = built
        act_seed = state.key[0]
        for u in range(U):
            sh = b["shards"][u]
            for t in range(T):   # SELECT ACTION (the policy's sample, written in place) + STEP ENVIRONMENT (:121-140)
                pi = actor_apply_fn(state.params.actor_params, sh.obs[t])
                ops.tanh_normal_sample(pi.head_out, pi.minimum, pi.maximum, pi.min_scale, seed=act_seed + 0x9E37 * u, offset=t,
                                       dev_counter=b["act_ctr"], action_out=sh.action[t], want_eps=False)
                anakin.step_env(env, state.env_state, u, sh.action[t], sh.step_out(t), t)
            torch.bitwise_or(sh.terminated, sh.truncated, out=sh.done)
            buffer_add_fn(sh.buffer, sh.transition())
        ops.counter_add(b["act_ctr"], T)

    def _epoch_grads(state: OffPolicyLearnerState, u: int, metrics: torch.Tensor, noise: Optional[Dict[str, torch.Tensor]] = None,
                     sample: bool = True, idx_in: Optional[torch.Tensor] = None) -> None:
        """The three losses of one `_update_epoch` on shard u's batch and their gradients, accumulated (weight 1/U) into the
        gradient arena (ff_sac.py:157-226, 229-283).  noise = {"actor", "q", "alpha"}: injected standard normals (tests)."""
        b, sh = built, built["shards"][u]
        sa, sq, lay, D, A = b["sa"], b["sq"], b["lay"], b["D"], b["A"]
        arena, target, grads = b["arena"], b["target"], b["grads"]
        p_actor = arena[lay["actor"]:]
        p_q = [arena[lay["q1"]:], arena[lay["q2"]:]]
        p_qt = [target[0:], target[lay["q2"] - lay["q1"]:]]
        log_alpha = arena[lay["alpha"]: lay["alpha"] + 1]
        w, first = 1.0 / U, u == 0
        eps_seed = state.key[1] + 0x51ED * u
        nz = noise or {}
        if sample:   # SAMPLE TRANSITIONS (:226-227): one launch writes (obs | action), (obs | .), (next_obs | .), reward, done
            buffer_sample_fn(sh.buffer, sh.xq_old, sh.b_reward, sh.b_done, xq_new=sh.xq_new, xq_next=sh.xq_next, idx_in=idx_in, idx_out=sh.b_idx)
        # ---- actor loss (:207-226): mean(alpha * log_prob(a) - min_k Q_k(obs, a)), a = reparameterised sample ----
        ops.mlp_forward_train(sa, p_actor, sh.xq_new, sh.ws_actor, out=sh.head)
        _, logp_new, eps1 = ops.tanh_normal_sample(sh.head, lo, hi, min_scale, eps=nz.get("actor"), seed=eps_seed, offset=0, dev_counter=b["eps_ctr"],
                                                   action_out=sh.xq_new[:, D:])
        for k in range(2):
            ops.mlp_forward_train(sq, p_q[k], sh.xq_new, sh.ws_q[k], out=sh.q[k])
        ops.sac_actor_seed(sh.q[0], sh.q[1], logp_new, log_alpha, sh.dq[0], sh.dq[1], metrics=metrics, weight=w)
        for k in range(2):   # input gradients only: the Q parameters are constants of the actor loss
            ops.mlp_backward(sq, p_q[k], sh.xq_new, sh.dq[k], sh.ws_q[k], net_grad=None, d_input=sh.d_in[k])
        sh.d_in[0].add_(sh.d_in[1])
        ops.tanh_normal_backward(sh.head, eps1, lo, hi, log_alpha, 1.0 / B, sh.d_in[0][:, D:], min_scale, out=sh.d_head)
        ops.mlp_backward(sa, p_actor, sh.xq_new, sh.d_head, sh.ws_actor, net_grad=grads[lay["actor"]:], grad_weight=w, overwrite=first)
        # ---- Q loss (:177-205): 0.5 mean((Q_k(obs, action) - target)^2), target from the TARGET networks on a fresh next action ----
        for k in range(2):
            ops.mlp_forward_train(sq, p_q[k], sh.xq_old, sh.ws_q[k], out=sh.q[k])
        ops.mlp_forward_train(sa, p_actor, sh.xq_next, sh.ws_actor_next, out=sh.head_next)
        _, logp_next, _ = ops.tanh_normal_sample(sh.head_next, lo, hi, min_scale, eps=nz.get("q"), seed=eps_seed, offset=1, dev_counter=b["eps_ctr"],
                                                 action_out=sh.xq_next[:, D:], want_eps=False)
        for k in range(2):
            ops.mlp_forward_train(sq, p_qt[k], sh.xq_next, sh.ws_qt[k], out=sh.nq[k])
        ops.sac_q_loss(sh.q[0], sh.q[1], sh.nq[0], sh.nq[1], logp_next, sh.b_reward, sh.b_done, log_alpha, gamma, sh.dq[0], sh.dq[1],
                       metrics=metrics, weight=w)
        for k, name in enumerate(("q1", "q2")):
            ops.mlp_backward(sq, p_q[k], sh.xq_old, sh.dq[k], sh.ws_q[k], net_grad=grads[lay[name]:], grad_weight=w, overwrite=first)
        # ---- alpha loss (:157-175): mean(alpha * (-log_prob(a') - target_entropy)), a' a second sample of pi(. | obs) ----
        _, logp_alpha, _ = ops.tanh_normal_sample(sh.head, lo, hi, min_scale, eps=nz.get("alpha"), seed=eps_seed, offset=2, dev_counter=b["eps_ctr"],
                                                  want_eps=False)
        ops.sac_alpha_grad(logp_alpha, log_alpha, target_entropy, autotune, grads[lay["alpha"]: lay["alpha"] + 1], grad_weight=w, overwrite=first,
                           metrics=metrics, weight=w)

    def _update_epoch(state: OffPolicyLearnerState, ep: int, noise=None, sample: bool = True, idx_in=None) -> None:
        """One `_update_epoch` (ff_sac.py:219-321): gradients of every shard, mean over shards and devices, the three optimisers in
        one launch (alpha first in the reference: its update uses the OLD alpha in all three losses, as here), Polyak."""
        b = built
        metrics = b["metrics"][ep]
        metrics.zero_()
        for u in range(U):
            _epoch_grads(state, u, metrics, noise=noise, sample=sample, idx_in=idx_in)
        ops.counter_add(b["eps_ctr"], 3)
        if world > 1:
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
            dist.all_reduce(metrics, op=dist.ReduceOp.SUM)
            metrics.mul_(1.0 / world)
        a_tree = state.params.actor_params
        ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu, grad_scale=1.0 / world)
        lay = b["lay"]
        ops.polyak_update(b["target"], b["arena"][lay["q1"]: lay["alpha"]], tau)   # optax.incremental_update (:296-299)

    def _update_step(state: OffPolicyLearnerState) -> None:
        for sh in built["shards"]:
            sh.carry_in()
        _rollout_phase(state)
        for ep in range(epochs):
            _update_epoch(state, ep)
        for sh, env_state in zip(built["shards"], state.env_state):
            sh.advance(env, env_state)

    def learner_fn(learner_state: OffPolicyLearnerState) -> AnakinExperimentOutput:
        """arch.num_updates_per_eval update steps (ff_sac.py:330-344)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, buffers=learner_state.buffer_state)
        train_metrics = {name: train_out[..., j] for j, name in enumerate(_METRIC_NAMES)}
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics=train_metrics)

    learner_fn.built = built
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.rollout_phase = _rollout_phase
    return learner_fn


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, networks, optimisers, buffer, environment and states (ff_sac.py:347-513)."""
    rank, n_devices = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())

    action_space = env.action_space()
    action_dim = int(action_space.shape[-1])
    config.system.action_dim = action_dim
    config.system.action_minimum = float(action_space.minimum)
    config.system.action_maximum = float(action_space.maximum)

    key, actor_net_key, q_net_key = keys

    # Define actor_network, q_network and optimisers (:360-393).
    actor_torso = instantiate(config.network.actor_network.pre_torso)
    actor_action_head = instantiate(config.network.actor_network.action_head, action_dim=action_dim,
                                    minimum=config.system.action_minimum, maximum=config.system.action_maximum)
    actor_network = Actor(torso=actor_torso, action_head=actor_action_head)

    def create_q_network(cfg: DictConfig) -> FeedForwardQ:
        return FeedForwardQ(critic_head=instantiate(cfg.network.q_network.critic_head), torso=instantiate(cfg.network.q_network.pre_torso),
                            input_layer=instantiate(cfg.network.q_network.input_layer))

    double_q_network = MultiNetwork([create_q_network(config), create_q_network(config)])

    actor_lr = make_learning_rate(config.system.actor_lr, config, config.system.epochs)
    q_lr = make_learning_rate(config.system.q_lr, config, config.system.epochs)
    alpha_lr = make_learning_rate(config.system.alpha_lr, config, config.system.epochs)
    actor_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(actor_lr, eps=1e-5))
    q_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(q_lr, eps=1e-5))
    alpha_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(alpha_lr, eps=1e-5))

    init_x = env.observation_space().generate_value()[None, ...].to(device).float()
    init_a = torch.zeros(1, action_dim, device=device)
    init_xa = torch.cat([init_x, init_a], dim=-1)

    # One flat arena [actor | q1 | q2 | log_alpha]; the target Q networks mirror the [q1 | q2] block (:398-426).
    sa = actor_network.spec_for(init_x.shape[-1])
    sq = double_q_network.networks[0].spec_for(init_xa.shape[-1])
    lay = sac_arena_layout(sa, sq)
    arena = torch.zeros(lay["total"], dtype=torch.float32, device=device)
    actor_params = actor_network.init(actor_net_key, init_x, flat=arena[lay["actor"]:])
    online_q_params = double_q_network.init(q_net_key, init_xa, flats=[arena[lay["q1"]:], arena[lay["q2"]:]])
    target_arena = arena[lay["q1"]: lay["alpha"]].clone()
    target_q_params = [build_param_tree(sq, target_arena[off:], "critic_head") for off in (0, lay["q2"] - lay["q1"])]

    # Automatic entropy tuning (:405-412)
    target_entropy = -float(config.system.target_entropy_scale) * action_dim
    log_alpha = arena[lay["alpha"]: lay["alpha"] + 1]
    if not config.system.autotune:
        import math

        log_alpha.fill_(math.log(float(config.system.init_alpha)))
    config.system.target_entropy = target_entropy

    # three optimiser states, the alpha one stepped only with autotune
    opt_states = SACOptStates(*optax.arena_state(actor_params, arena, [(lay["actor"], sa.param_count), (lay["q1"], lay["q_block"]), (lay["alpha"], 1)]))
    actor_params.target_arena = target_arena
    params = SACParams(actor_params, OnlineAndTarget(online_q_params, target_q_params), log_alpha)

    apply_fns = (actor_network.apply, double_q_network.apply)
    update_fns = (actor_optim.update, q_optim.update, alpha_optim.update)

    # Replay buffer (:429-456): one ring per (device, update-batch shard)
    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 2)
    buffer_states = anakin.replay_buffers(config, shard_keys[U], rank, n_devices,
                                          lambda size, batch, seed: TransitionBuffer(size, batch, batch, init_x.shape[-1], action_dim, device, seed=seed))
    buffer_fns = (TransitionBuffer.add, TransitionBuffer.sample_into)

    learn = get_learner_fn(env, apply_fns, update_fns, buffer_fns, config)
    warmup = get_warmup_fn(env, params, actor_network.apply, TransitionBuffer.add, config)

    # Initialise environment states and timesteps across update-batch shards (:463-474).
    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    if warm_start(config, arena):   # (:477-486)
        target_arena.copy_(arena[lay["q1"]: lay["alpha"]])

    # per-rank streams: (rollout policy noise, loss noise); warm-up noise on its own key (:489-496)
    act_seed, eps_seed, warm_seed = anakin.rank_seeds(shard_keys[U + 1], 3, rank, n_devices)

    # Warm up the buffer (:507-509).
    for u in range(U):
        env_states[u], timesteps[u], _, _ = warmup(env_states[u], timesteps[u], buffer_states[u], warm_seed + 0xA5A5 * u)

    init_learner_state = OffPolicyLearnerState(params, opt_states, buffer_states, (act_seed, eps_seed), env_states, timesteps)
    return learn, actor_network, init_learner_state


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_sac.py:516-675)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point: `python -m stoix_b200.systems.sac.ff_sac arch.total_num_envs=1024 system.total_batch_size=256 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_sac", run_experiment, "SAC")


if __name__ == "__main__":
    hydra_entry_point()
