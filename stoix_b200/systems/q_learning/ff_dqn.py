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

The distributional systems ff_c51 and ff_qr_dqn run the same body with a head of A N outputs per row (column a N + i = action
a, atom / quantile i) and a loss kernel of their own; the rollout and the warm-up put stx_dist_q_values (the expected Q) between
the forward and epsilon-greedy, so the shard's q (T, E, A) holds expected values:

  loss                            kernel                          extra forward per shard and epoch
  ------------------------------  ------------------------------  -------------------------------------------------------------
  categorical_double_q_learning   stx_categorical_q_loss_grads    online on next_obs + stx_dist_q_values (ff_c51.py:165-168)
  quantile_q_learning             stx_quantile_q_loss_grads       - (the selector is the target distribution, ff_qr_dqn.py:193-194)

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

from functools import partial
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import AnakinExperimentOutput
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import build_param_tree
from stoix_b200.networks.heads import DiscreteQNetworkHead, DistributionalDiscreteQNetwork, QuantileDiscreteQNetwork
from stoix_b200.systems import anakin
from stoix_b200.systems.q_learning.dqn_types import Transition
from stoix_b200.systems.sac.sac_types import OffPolicyLearnerState, OnlineAndTarget
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.replay import DiscreteTransitionBuffer
from stoix_b200.utils.training import make_learning_rate

# the distributional losses: loss -> (head class, stx_dist_q_values kind, system, network config)
DIST_LOSSES = {"categorical_double_q_learning": (DistributionalDiscreteQNetwork, "categorical", "ff_c51", "mlp_c51"),
               "quantile_q_learning": (QuantileDiscreteQNetwork, "quantile", "ff_qr_dqn", "mlp_qr_dqn")}
LOSSES = tuple(ops.Q_RULES) + tuple(DIST_LOSSES)
_NAMES = {"q_learning": "DQN", "double_q_learning": "DDQN", "munchausen_q_learning": "MDQN", "q_learning_reg": "DQN-Reg",
          "categorical_double_q_learning": "C51", "quantile_q_learning": "QR-DQN"}


def _refuse_unsupported(config: DictConfig, loss: str = "q_learning") -> None:
    if str(config.arch.get("precision", "f32")) == "bf16":
        raise ValueError("arch.precision=bf16 is not available for the DQN family: the bf16 tensor-core kernels implement the relu 2 x 256 "
                         "Categorical actor-critic only, not a Q network with its activation, LayerNorm and Q loss; use arch.precision=f32")
    target = str(config.network.actor_network.action_head.get("_target_", ""))
    name = target.rsplit(".", 1)[-1]
    dist = {v[0].__name__: (k, v[2], v[3]) for k, v in DIST_LOSSES.items()}
    if loss in DIST_LOSSES:
        _, _, system, network = DIST_LOSSES[loss]
        if name != DIST_LOSSES[loss][0].__name__:
            raise ValueError(f"{system} runs the {DIST_LOSSES[loss][0].__name__} head (network={network}); action head {target!r} is not "
                             "implemented for it")
    elif name in dist:
        raise ValueError(f"action head {target!r} is a distributional head: it runs with {dist[name][1]} (network={dist[name][2]}), not "
                         f"with the {loss} loss")
    elif not target.endswith("DiscreteQNetworkHead"):
        raise ValueError(f"the DQN family here runs the plain Q head (network=mlp_dqn); action head {target!r} (dueling, noisy, "
                         "distributional) is not implemented")


class DistLoss(NamedTuple):
    """The hyper-parameters of a distributional loss: the kernel's StxDistQHyper, the action count A, the atom / quantile count N
    and the support row (N) every sample shares: the C51 atoms, or QR-DQN's quantile midpoints tau_i = (i + 0.5) / N."""
    hyper: Any
    A: int
    N: int
    support: torch.Tensor


def loss_hyper(loss: str, config: DictConfig, head: Any = None, device=None):
    """The StxQTdHyper of `loss` from config.system (the keys of system/q_learning/ff_{dqn,mdqn,dqn_reg}.yaml); for a distributional
    loss the DistLoss of `head` on `device`."""
    s = config.system
    if loss in DIST_LOSSES:
        huber = float(s.huber_loss_parameter) if loss == "quantile_q_learning" else 0.0
        hyper = ops.dist_q_hyper(gamma=float(s.gamma), max_abs_reward=float(s.max_abs_reward), huber_delta=huber)
        if loss == "categorical_double_q_learning":
            return DistLoss(hyper, head.action_dim, head.num_atoms, head.atoms(device))
        N = head.num_quantiles
        tau = (torch.arange(N, dtype=torch.float32) + 0.5) / N   # ff_qr_dqn.py:180-182, in float32
        return DistLoss(hyper, head.action_dim, N, tau.to(device))
    kw = dict(gamma=float(s.gamma), max_abs_reward=float(s.max_abs_reward), huber_delta=float(s.huber_loss_parameter))
    if loss == "munchausen_q_learning":
        kw.update(entropy_temperature=float(s.entropy_temperature), munchausen_coefficient=float(s.munchausen_coefficient),
                  clip_value_min=float(s.clip_value_min))
    if loss == "q_learning_reg":
        kw.update(regularizer_coeff=float(s.regularizer_coeff))
    return ops.q_td_hyper(**kw)


class _Shard(anakin.Trajectory):
    """Trajectory buffers of one (device, update-batch) shard, time-major: the Transition fields (dqn_types.py) plus the Q rows."""

    def __init__(self, T: int, E: int, D: int, A: int, device):
        super().__init__(T, E, D, device)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.q = z(T, E, A)                     # Q(online, obs[t]), the rows the sampler acted on
        self.action = z(T, E, dt=torch.int32)
        self.done = z(T, E, dt=torch.uint8)     # timestep.last() = terminated | truncated (ff_dqn.py:121)

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
    """Workspaces of batch_grads for M rows of head width A: ws (train-mode forward), q_tm1 (M, A), q_tgt (2M, A), q_sel (M, A),
    dq (M, A); for C51 q_val (M, n_actions), the selector's expected Q."""
    ws: torch.Tensor
    q_tm1: torch.Tensor
    q_tgt: torch.Tensor
    q_sel: torch.Tensor
    dq: torch.Tensor
    q_val: Optional[torch.Tensor] = None


def make_work(spec: ops.MlpSpec, M: int, device, n_actions: Optional[int] = None) -> Work:
    A = spec.sizes[-1]
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
    return Work(ops.mlp_train_workspace(spec, M, device), z(M, A), z(2 * M, A), z(M, A), z(M, A), None if n_actions is None else z(M, n_actions))


def make_batch(M: int, D: int, device) -> Batch:
    return Batch(torch.zeros(2 * M, D, device=device), torch.zeros(M, dtype=torch.int32, device=device), torch.zeros(M, device=device),
                 torch.zeros(M, dtype=torch.uint8, device=device))


def batch_grads(loss: str, spec: ops.MlpSpec, online: torch.Tensor, target: torch.Tensor, batches: Sequence[Batch], hyper, grads: torch.Tensor,
                metric: torch.Tensor, work: Work) -> None:
    """jax.grad(_q_loss_fn) + pmean over "batch" of one epoch (ff_dqn.py:147-200): per shard the online train-mode forward on obs,
    the target forward on next_obs (MDQN: on obs and next_obs in one launch; DDQN adds the online forward on next_obs), the loss
    kernel and the backward.  `grads` receives the mean over the U shards (the first overwrites, weight 1/U each) and
    metric[0] += mean q_loss.  The distributional losses take a DistLoss as `hyper`: C51 adds the online forward on next_obs and
    its expected Q as the selector (ff_c51.py:165-168); QR-DQN selects on the target distribution inside its kernel."""
    U = len(batches)
    q_tm1, q_tgt, q_sel, dq = work.q_tm1, work.q_tgt, work.q_sel, work.dq
    for u, b in enumerate(batches):
        M = int(b.action.numel())
        obs, nxt = b.xs[:M], b.xs[M:]
        ops.mlp_forward_train(spec, online, obs, work.ws, out=q_tm1)
        q_aux = None
        if loss in DIST_LOSSES:
            ops.mlp_forward(spec, target, nxt, out=q_tgt[M:], ws_key="dqn_target")
            if loss == "categorical_double_q_learning":
                ops.mlp_forward(spec, online, nxt, out=q_sel, ws_key="dqn_selector")
                ops.dist_q_values("categorical", q_sel, hyper.A, hyper.N, hyper.support, out=work.q_val)
                ops.categorical_q_loss_grads(q_tm1, q_tgt[M:], work.q_val, hyper.support, hyper.support, b.action, b.reward, hyper.hyper, dq,
                                             metric, done=b.done, weight=1.0 / U)
            else:
                ops.quantile_q_loss_grads(q_tm1, q_tgt[M:], hyper.support, b.action, b.reward, hyper.hyper, dq, metric, hyper.A, done=b.done,
                                          weight=1.0 / U)
        elif loss == "munchausen_q_learning":
            ops.mlp_forward(spec, target, b.xs, out=q_tgt, ws_key="dqn_target")
            q_aux = q_tgt[:M]
        else:
            ops.mlp_forward(spec, target, nxt, out=q_tgt[M:], ws_key="dqn_target")
            if loss == "double_q_learning":
                q_aux = ops.mlp_forward(spec, online, nxt, out=q_sel, ws_key="dqn_selector")
        if loss not in DIST_LOSSES:
            ops.q_td_loss_grads(loss, q_tm1, q_tgt[M:], b.action, b.reward, hyper, dq, metric, done=b.done, q_aux=q_aux, weight=1.0 / U)
        ops.mlp_backward(spec, online, obs, dq, work.ws, net_grad=grads, grad_weight=1.0 / U, overwrite=(u == 0))


def get_warmup_fn(env: Environment, q_params: OnlineAndTarget, q_apply_fn: Callable, buffer_add_fn: Callable, config: DictConfig) -> Callable:
    """ff_dqn.py:37-89: `warmup_steps` environment steps with the initial online parameters and the training epsilon, added to
    the buffer (one shard per call)."""
    def draw(obs, key, t):
        pi = q_apply_fn(q_params.online, obs)
        pi = pi[0] if isinstance(pi, tuple) else pi   # the distributional heads return (EpsilonGreedy(expected q), ...)
        return pi.sample(seed=key, offset=t).to(torch.int32)

    return anakin.warmup_fn(env, draw, buffer_add_fn, config)


def get_learner_fn(env: Environment, q_apply_fn: Callable, q_update_fn: Callable, buffer_fns: Tuple[Callable, Callable], config: DictConfig,
                   loss: str = "q_learning"):
    """ff_dqn.py:92-258.  q_apply_fn: the bound `apply` of the Q network (a FeedForwardActor with a DiscreteQNetworkHead); q_update_fn:
    the bound `update` of chain(clip_by_global_norm, adam); buffer_fns = (DiscreteTransitionBuffer.add, .sample_into) unbound, applied
    to learner_state.buffer_state[u]; loss: one of LOSSES (a distributional loss needs its head, DIST_LOSSES)."""
    q_net = anakin.owner(q_apply_fn, Actor, "q_apply_fn")
    if loss not in LOSSES:
        raise ValueError(f"get_learner_fn: loss {loss!r} is not one of {LOSSES}")
    head_cls = DIST_LOSSES[loss][0] if loss in DIST_LOSSES else DiscreteQNetworkHead
    if not isinstance(q_net.action_head, head_cls):
        raise TypeError(f"get_learner_fn: q_apply_fn must be the bound `apply` of a FeedForwardActor with a {head_cls.__name__}")
    opt = anakin.owner(q_update_fn, optax.GradientTransformation, "q_update_fn")
    _refuse_unsupported(config, loss)
    dist_kind = DIST_LOSSES[loss][1] if loss in DIST_LOSSES else None
    buffer_add_fn, buffer_sample_fn = buffer_fns
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, M = int(sysc.epochs), int(sysc.batch_size)
    tau = float(sysc.tau)
    sched = ops.epsilon_schedule_struct(float(sysc.training_epsilon), float(sysc.training_epsilon), 0.0, 1, decay=False)
    built: Dict[str, Any] = {}

    def _build(state: OffPolicyLearnerState) -> None:
        tree = state.params.online
        spec = tree.spec
        dev = tree.flat.device
        D, A = spec.sizes[0], (q_net.action_head.action_dim if dist_kind else spec.sizes[-1])
        shards = [_Shard(T, E, D, A, dev) for _ in range(U)]
        # "rollouts": the name this list had before it was "shards" like every other learner's; callers that read it keep working
        built.update(spec=spec, dev=dev, plan=optax.adam_plan([(0, spec.param_count, opt)], dev, tree.arena_counts),
                     shards=shards, rollouts=shards, hyper=loss_hyper(loss, config, q_net.action_head, dev),
                     head_out=torch.zeros(E, spec.sizes[-1], device=dev) if dist_kind else None,   # the rollout's A N head row
                     batches=[make_batch(M, D, dev) for _ in range(U)],
                     work=make_work(spec, M, dev, A if loss == "categorical_double_q_learning" else None),
                     grads=torch.zeros(tree.arena.numel(), dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, dtype=torch.float32, device=dev),
                     roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # epsilon-greedy call index
                     graph=None, eager_done=False)

    def _rollout_phase(state: OffPolicyLearnerState) -> None:
        """_env_step x rollout_length (ff_dqn.py:106-137) + buffer add (:142), per shard."""
        b = built
        online = state.params.online.flat
        for u in range(U):
            ro: _Shard = b["shards"][u]
            for t in range(T):
                if dist_kind:
                    ops.mlp_forward(b["spec"], online, ro.obs[t], out=b["head_out"], ws_key="dqn_rollout")
                    h = b["hyper"]
                    ops.dist_q_values(dist_kind, b["head_out"], h.A, h.N, h.support, out=ro.q[t])
                else:
                    ops.mlp_forward(b["spec"], online, ro.obs[t], out=ro.q[t], ws_key="dqn_rollout")
                ops.epsilon_greedy(ro.q[t], sched, seed=state.key[0] + u, offset=t, dev_counter=b["roll_ctr"], out=ro.action[t])
                anakin.step_env(env, state.env_state, u, ro.action[t], ro.step_out(t), t)
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
        batch_grads(loss, b["spec"], online.flat, target.flat, b["batches"], b["hyper"], b["grads"], metric, b["work"])
        if world > 1:   # pmean over "device": summed by NCCL here, scaled in the optimiser step
            dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
        ops.clip_adam_step(b["plan"], online.arena, b["grads"], online.arena_mu, online.arena_nu, grad_scale=1.0 / world)
        ops.polyak_update(target.arena, online.arena, tau)   # optax.incremental_update (:207-209)

    def _update_step(state: OffPolicyLearnerState) -> None:
        """A single update (ff_dqn.py:103-234), in place on the learner state."""
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

    def learner_fn(learner_state: OffPolicyLearnerState) -> AnakinExperimentOutput:
        """arch.num_updates_per_eval update steps (ff_dqn.py:236-256)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config, buffers=learner_state.buffer_state)
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics={"q_loss": train_out})

    learner_fn.built = built
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    learner_fn.update_step = _update_step
    learner_fn.update_epoch = _update_epoch
    learner_fn.rollout_phase = _rollout_phase
    learner_fn.loss = loss
    return learner_fn


def learner_setup(env: Environment, keys: Tuple[int, int], config: DictConfig, loss: str = "q_learning"):
    """Initialise learner_fn, network, optimiser, buffer, environment and states (ff_dqn.py:261-414).  Returns the EVAL network
    (epsilon = system.evaluation_epsilon) as the second element, which is what the reference hands to the evaluator."""
    _refuse_unsupported(config, loss)
    rank, n_devices = anakin.world()
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
    (opt_states,) = optax.arena_state(online, arena, [(0, spec.param_count)])
    warm_start(config, arena)   # (:372-380)
    target_arena = arena.clone()
    target = build_param_tree(spec, target_arena, "action_head")
    target.arena = target_arena
    params = OnlineAndTarget(online, target)

    # Replay buffer (:316-347): one ring per (device, update-batch shard)
    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 2)
    buffer_states = anakin.replay_buffers(config, shard_keys[U], rank, n_devices,
                                          lambda size, batch, seed: DiscreteTransitionBuffer(size, batch, batch, init_x.shape[-1], device, seed=seed))
    buffer_fns = (DiscreteTransitionBuffer.add, DiscreteTransitionBuffer.sample_into)

    learn = get_learner_fn(env, q_network.apply, q_optim.update, buffer_fns, config, loss=loss)
    warmup = get_warmup_fn(env, params, q_network.apply, DiscreteTransitionBuffer.add, config)

    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    # per-rank streams: rollout epsilon-greedy draws; warm-up draws on their own key (:383-409)
    act_seed, warm_seed = anakin.rank_seeds(shard_keys[U + 1], 2, rank, n_devices)
    for u in range(U):
        env_states[u], timesteps[u], _, _ = warmup(env_states[u], timesteps[u], buffer_states[u], warm_seed + 0xA5A5 * u)

    # key = (rollout seed, warm-up seed): the rollout draws from key[0]; key[1] records where the warm-up drew from
    init_learner_state = OffPolicyLearnerState(params, opt_states, buffer_states, (act_seed, warm_seed), env_states, timesteps)
    return learn, eval_q_network, init_learner_state


def online_params(learner_state: OffPolicyLearnerState):
    """The policy of the DQN family: the online network, which is evaluated, tracked and checkpointed."""
    return learner_state.params.online


def run_experiment(_config: DictConfig, loss: str = "q_learning") -> float:
    """Runs experiment (ff_dqn.py:417-556)."""
    return anakin.run_experiment(_config, partial(learner_setup, loss=loss), net_keys=1, policy=online_params)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None, loss: str = "q_learning",
                      config_name: str = "default_ff_dqn") -> float:
    """Experiment entry point: `python -m stoix_b200.systems.q_learning.ff_dqn arch.total_num_envs=1024 ...`"""
    return anakin.entry_point(cfg, overrides, config_name, partial(run_experiment, loss=loss), _NAMES[loss])


if __name__ == "__main__":
    hydra_entry_point()
