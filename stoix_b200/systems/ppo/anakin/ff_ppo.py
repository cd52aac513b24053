"""Anakin feed-forward PPO on H100 -- drop-in for stoix/systems/ppo/anakin/ff_ppo.py.

Same entry points and signatures (get_learner_fn :49-54, learner_setup :424-426, run_experiment :554,
hydra_entry_point :709-727) and the same state / output contracts (stoix_b200/base_types.py), but a
different machine underneath:

  reference (JAX)                                 here (H100)
  ----------------------------------------------  -------------------------------------------------
  pmap over devices                               one process per GPU (torchrun), rank = device index
  lax.scan over T env steps, 3 MLP applies/step   T x (actor MLP kernel + sample kernel + env kernel);
                                                  the two critic evaluations are batched over the
                                                  whole (T*E) rollout afterwards (same params, same
                                                  rows => same values, 2 launches instead of 2T)
  lax.scan reverse over T for GAE                 one chunked parallel-scan launch (K2)
  permutation + take (shuffled copy per epoch)    keyed bijection -> index vector; kernels gather
  jax.grad of two loss fns                        fused forward/loss/backward launches (K3)
  pmean(batch) ; pmean(device)                    mean over local shards ; NCCL all-reduce of one flat
                                                  gradient arena
  2 x optax.chain(clip, adam) over 12 leaves      one fused clip+Adam launch over the arena (K4)
  one XLA program per learn() call                one CUDA graph per update step, replayed

The per-update work is captured into a CUDA graph after the first (eager) update; every RNG stream
position lives in device memory so replays draw fresh numbers.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import (
    ActorApply,
    ActorCriticOptStates,
    ActorCriticParams,
    AnakinExperimentOutput,
    CriticApply,
    LearnerFn,
    OnPolicyLearnerState,
)
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment
from stoix_b200.networks.base import FeedForwardActor as Actor
from stoix_b200.networks.base import FeedForwardCritic as Critic
from stoix_b200.networks.heads import NormalAffineTanhDistributionHead
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.ppo_types import PPOTransition
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.training import make_learning_rate

# The bf16 fused rollout's SM split: persistent policy CTAs; the critic's forward runs beside them on the other SMs.
POLICY_CTAS = 82
_METRIC_NAMES = ("actor_loss", "entropy", "value_loss", "advantages", "pred_value", "target_value")
# The actor loss of the update: ppo_clip_loss (ff_ppo*), ppo_penalty_loss (ff_ppo_penalty*) or dpo_loss (ff_dpo_continuous).  The
# variants report the reference's loss_info keys (ff_ppo_penalty.py:172-176,195-197; ff_dpo_continuous.py:166-169,187-189) as
# (name, metrics slot) pairs; slot 6 is the KL divergence the penalty kernels accumulate.
LOSS_VARIANTS = ("clip", "kl_penalty", "dpo")
_VARIANT_METRICS = {
    "clip": tuple((name, j) for j, name in enumerate(_METRIC_NAMES)),
    "kl_penalty": (("actor_loss", 0), ("entropy", 1), ("kl_divergence", ops.METRIC_SLOT_KL), ("value_loss", 2)),
    "dpo": (("actor_loss", 0), ("entropy", 1), ("value_loss", 2)),
}


class _Shard(anakin.Trajectory):
    """Trajectory buffers of one (device, update-batch) shard: PPOTransition fields, time-major.  With normalize_observations the
    environment writes raw fp32 observations (they feed the running statistics, ff_ppo.py:145-162) and obs / next_obs hold the
    normalised copies every network kernel reads (:90-94,113-115)."""

    def __init__(self, T: int, E: int, D: int, A: int, obs_dtype, device, normalize: bool = False, act_dim: int = 0,
                 behaviour: bool = False):
        super().__init__(T, E, D, device, obs_dtype=obs_dtype, raw_obs=normalize)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.done = self.terminated   # the transition's done: terminated only, truncation bootstraps
        # Categorical: (T, E) int32 action indices; tanh-Normal (act_dim > 0): (T, E, act_dim) float32 actions
        self.action = z(T, E, act_dim) if act_dim > 0 else z(T, E, dt=torch.int32)
        self.log_prob = z(T, E)
        self.value = z(T, E)
        self.bootstrap_value = z(T, E)
        self.advantages = z(T, E)
        self.targets = z(T, E)
        self.logits = z(E, A)                        # actor head output of one step: logits, or loc | scale pre-activation
        # KL penalty: the head output of every rollout step is kept as the behaviour policy of the update (the rollout actor is
        # the actor at the start of the update, ff_ppo_penalty.py:137, evaluated on the same rows the minibatches read)
        self.behaviour = z(T, E, A) if behaviour else None
        self.adv_stats: Optional[torch.Tensor] = None

    def transition(self, T: int) -> PPOTransition:
        info = {"episode_return": self.episode_return, "episode_length": self.episode_length,
                "is_terminal_step": self.is_terminal_step.bool()}
        return PPOTransition(self.done.bool(), self.truncated.bool(), self.action, self.value, self.reward,
                             self.bootstrap_value, self.log_prob, self.obs[:T], info)


def get_learner_fn(
    env: Environment,
    apply_fns: Tuple[ActorApply, CriticApply],
    update_fns: Tuple[Callable, Callable],
    config: DictConfig,
    loss: str = "clip",
) -> LearnerFn[OnPolicyLearnerState]:
    """Get the learner function (ff_ppo.py:49-372).

    apply_fns: (actor_network.apply, critic_network.apply) bound methods; update_fns:
    (actor_optim.update, critic_optim.update) handles from stoix_b200.optim -- both are used for the
    network shapes / optimiser hyper-parameters they carry; the arithmetic runs in the fused kernels.
    loss: the actor loss, one of LOSS_VARIANTS -- "clip" (ff_ppo, ff_ppo_continuous), "kl_penalty" (ff_ppo_penalty,
    ff_ppo_penalty_continuous) or "dpo" (ff_dpo_continuous, tanh-Normal actor only).
    """
    actor_apply_fn, critic_apply_fn = apply_fns
    actor_net, critic_net = anakin.owner(actor_apply_fn, Actor, "apply_fns[0]"), anakin.owner(critic_apply_fn, Critic, "apply_fns[1]")
    actor_opt = anakin.owner(update_fns[0], optax.GradientTransformation, "update_fns[0]")
    critic_opt = anakin.owner(update_fns[1], optax.GradientTransformation, "update_fns[1]")
    rank, world = anakin.world()

    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, nmb = int(sysc.epochs), int(sysc.num_minibatches)
    B = T * E
    assert B % nmb == 0, "rollout_length * num_envs must be divisible by num_minibatches"
    mb = B // nmb
    precision = ops.STX_PREC_BF16 if str(arch.get("precision", "f32")) == "bf16" else ops.STX_PREC_F32
    # The actor head decides the action buffer, the rollout sampler, the gradient entry and the entropy RNG; everything else
    # (GAE, shuffles, shards, all-reduce, observation normalisation, graph capture) is shared.
    tanh_head = actor_net.action_head if isinstance(actor_net.action_head, NormalAffineTanhDistributionHead) else None
    if tanh_head is not None and precision == ops.STX_PREC_BF16:
        raise ValueError("arch.precision=bf16 is not available with a tanh-Normal actor (NormalAffineTanhDistributionHead): the bf16 "
                         "tensor-core PPO kernels implement the Categorical head only; use arch.precision=f32")
    if loss not in LOSS_VARIANTS:
        raise ValueError(f"get_learner_fn: loss={loss!r}; expected one of {LOSS_VARIANTS}")
    if loss != "clip" and precision == ops.STX_PREC_BF16:
        raise ValueError(f"arch.precision=bf16 is not available with the {loss} actor loss: the bf16 tensor-core PPO kernels implement the "
                         "clipped surrogate only; use arch.precision=f32")
    if loss == "dpo" and tanh_head is None:
        raise ValueError("the dpo actor loss needs a tanh-Normal actor (NormalAffineTanhDistributionHead); the reference has no discrete DPO")
    kl_coef = float(sysc.kl_penalty_coef) if loss == "kl_penalty" else 0.0
    dpo_alpha, dpo_beta = (float(sysc.alpha), float(sysc.beta)) if loss == "dpo" else (0.0, 0.0)
    # ff_dpo_continuous.py:123 uses the raw reward; the clip and penalty systems scale it (ff_ppo_penalty.py:123)
    reward_scale = 1.0 if loss == "dpo" else float(sysc.reward_scale)

    built: Dict[str, Any] = {}

    def _build(state: OnPolicyLearnerState) -> None:
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        sa, sc = a_tree.spec, c_tree.spec
        dev = a_tree.flat.device
        arena = state.params.actor_params.arena
        _, coff, total = ops.arena_offsets(sa, sc)
        D, A = sa.sizes[0], sa.sizes[-1]
        obs_dtype = torch.bfloat16 if precision == ops.STX_PREC_BF16 else torch.float32
        rs = getattr(state, "running_statistics", None)
        act_dim = tanh_head.action_dim if tanh_head is not None else 0
        shards = [_Shard(T, E, D, A, obs_dtype, dev, normalize=rs is not None, act_dim=act_dim, behaviour=loss == "kl_penalty")
                  for _ in range(U)]
        plan = optax.adam_plan([(0, sa.param_count, actor_opt), (coff, sc.param_count, critic_opt)], dev, a_tree.arena_counts)
        peers = None
        if world > 1 and bool(arch.get("fused_allreduce", True)) and (epochs * nmb) % 2 == 0 and world <= 8:
            try:  # gradient arenas in NVLink peer memory: the all-reduce is fused into the optimiser kernel
                peers = ops.PeerGradBuffers(total, dev)
            except Exception as e:  # symmetric memory unavailable (no P2P): NCCL all-reduce + K4
                if rank == 0:
                    print(f"[stoix_b200] fused all-reduce unavailable ({type(e).__name__}: {e}); using NCCL all-reduce")
                peers = None
        built.update(
            sa=sa, sc=sc, dev=dev, arena=arena, coff=coff, total=total, shards=shards, plan=plan,
            grads=torch.zeros(total, dtype=torch.float32, device=dev),
            metrics=torch.zeros(epochs, nmb, 8, dtype=torch.float32, device=dev),
            ws=ops.ppo_workspace(sa, sc, mb, precision, dev),
            arena_bf16=getattr(state.params.actor_params, "arena_bf16", None),
            peers_obj=peers,
            peers=None,
            roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # categorical call index
            perm_ctr=torch.zeros(1, dtype=torch.int64, device=dev),   # shuffle stream index
            ent_ctr=torch.zeros(1, dtype=torch.int64, device=dev),    # tanh-Normal entropy noise: minibatch call index
            side_stream=torch.cuda.Stream(device=dev),                # the shuffles run here, underneath the rollout
            critic_stream=torch.cuda.Stream(device=dev),              # critic evaluation beside the fused rollout's policy
            rs=rs, rs_sums=torch.zeros(2 * D + 1, dtype=torch.float64, device=dev) if rs is not None else None,
            graph=None, eager_done=False,
        )

    def _env_step(state: OnPolicyLearnerState, u: int, t: int, seeds: Tuple[int, int]) -> None:
        """One vectorised env step of shard u (ff_ppo.py:81-135) writing the transition in place."""
        b = built
        sh: _Shard = b["shards"][u]
        a_tree = state.params.actor_params
        if b["rs"] is not None:  # normalise the observation with the PRE-update statistics (ff_ppo.py:90-94)
            ops.obs_normalize(sh.obs_raw[t], b["rs"].mean, b["rs"].std, out=sh.obs[t])
        # SELECT ACTION (ff_ppo.py:97-101): logits -> sample -> log_prob; the KL penalty keeps the head output as behaviour[t]
        head = sh.logits if sh.behaviour is None else sh.behaviour[t]
        ops.mlp_forward(b["sa"], a_tree.flat, sh.obs[t], precision=precision, params_bf16=a_tree.flat_bf16, out=head, ws_key="learner")
        if tanh_head is None:
            ops.categorical(head, None, seeds[0] + u, t, b["roll_ctr"], out=(sh.action[t], sh.log_prob[t]))
        else:  # sample, then score the stored action by the inverse path the loss uses (ff_ppo_continuous.py:98-101)
            lo, hi, ms = tanh_head.minimum, tanh_head.maximum, tanh_head.min_scale
            ops.tanh_normal_sample(head, lo, hi, ms, seed=seeds[0] + u, offset=t, dev_counter=b["roll_ctr"], action_out=sh.action[t],
                                   want_eps=False)
            ops.tanh_normal_log_prob(head, sh.action[t], lo, hi, ms, out=sh.log_prob[t])
        # STEP ENVIRONMENT (ff_ppo.py:104-116)
        anakin.step_env(env, state.env_state, u, sh.action[t], sh.step_out(t), t)

    def _rollout_phase(state: OnPolicyLearnerState) -> None:
        """STEP ENVIRONMENT FOR ROLLOUT LENGTH (ff_ppo.py:138-140) + the batched critic evaluations."""
        b = built
        sa, sc = b["sa"], b["sc"]
        c_tree = state.params.critic_params
        D = sa.sizes[0]
        a_tree = state.params.actor_params
        fused = (precision == ops.STX_PREC_BF16 and bool(arch.get("fused_rollout", True)) and E % 128 == 0
                 and getattr(env, "fused_rollout_supported", False) and b["rs"] is None)
        # The two critic evaluations of _env_step (value = critic(obs_t), bootstrap_value = critic(next_obs_t), ff_ppo.py:99,
        # 113-116) depend only on the observations, so they are batched over (steps x envs) rows.
        main = torch.cuda.current_stream()

        def critic_rows(sh: _Shard, t_lo: int, t_hi: int) -> None:
            n = (t_hi - t_lo) * E
            ops.mlp_forward(sc, c_tree.flat, sh.obs[t_lo:t_hi].view(n, D), precision=precision, params_bf16=c_tree.flat_bf16,
                            out=sh.value[t_lo:t_hi].view(n, 1), ws_key="learner-critic")
            ops.mlp_forward(sc, c_tree.flat, sh.next_obs[t_lo:t_hi].view(n, D), precision=precision, params_bf16=c_tree.flat_bf16,
                            out=sh.bootstrap_value[t_lo:t_hi].view(n, 1), ws_key="learner-critic")

        for u in range(U):
            sh: _Shard = b["shards"][u]
            if fused:
                # Envs whose dynamics ignore the action: the whole trajectory first, in one launch over the whole GPU.  The
                # policy of step t then needs only obs[t], so the actor and the critic (once per observation) are both
                # batched over all T x E rows: persistent launches over the SMs, POLICY_CTAS of them for the actor and the
                # rest for the critic on a second stream beside it (both are bound by their tensor-core chains, so the split
                # only balances their lengths).  arch.rollout_chunks is accepted and no longer read.
                env.fused_trajectory(state.env_state[u], sh, T)
                side = b["critic_stream"]
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    ops.set_forward_cta_budget(ops.NUM_SMS - POLICY_CTAS)
                    ops.tc_rollout_values(sc, c_tree.flat, c_tree.flat_bf16, sh.obs, sh.next_obs, sh.is_terminal_step, sh.value,
                                          sh.bootstrap_value, ws_key="learner-rollout-values")
                    ops.set_forward_cta_budget(0)
                ops.tc_rollout_policy(sa, a_tree.flat, a_tree.flat_bf16, sh.obs[:T], sh.action, sh.log_prob, state.key[0] + u, 0,
                                      b["roll_ctr"], max_ctas=POLICY_CTAS)
                main.wait_stream(side)
            else:
                for t in range(T):
                    _env_step(state, u, t, state.key)
                if b["rs"] is not None:  # bootstrap observations, same pre-update statistics (ff_ppo.py:113-115), one launch
                    ops.obs_normalize(sh.next_obs_raw, b["rs"].mean, b["rs"].std, out=sh.next_obs)
                critic_rows(sh, 0, T)

    def _stats_phase(state: OnPolicyLearnerState) -> None:
        """UPDATE RUNNING STATISTICS (ff_ppo.py:145-162) with the raw trajectory observations of every shard ("batch")
        and rank ("device"), std limits 5e-4 / 5e4.  Runs after the rollout: everything in this update that is
        normalised (rollout inputs, the minibatch observations of the epochs) used the statistics from before it."""
        b = built
        if b["rs"] is None:
            return
        from stoix_b200.utils import running_statistics as rstat

        rstat.update_statistics_(b["rs"], [sh.obs_raw[:T] for sh in b["shards"]], std_min_value=5e-4, std_max_value=5e4,
                                 pmap_axes=["device", "batch"], validate_shapes=False, sums=b["rs_sums"])

    def _gae_phase(state: OnPolicyLearnerState) -> None:
        """CALCULATE ADVANTAGE (ff_ppo.py:164-179)."""
        for u in range(U):
            sh: _Shard = built["shards"][u]
            _, _, sh.adv_stats = ops.gae_ppo(
                sh.reward, sh.value, sh.bootstrap_value, sh.done, sh.truncated, float(sysc.gamma),
                float(sysc.gae_lambda), reward_scale, 1 if sysc.standardize_advantages else 0,
                out=(sh.advantages, sh.targets),
            )

    def _update_phase(state: OnPolicyLearnerState, shuffled: bool = False) -> None:
        """UPDATE EPOCHS (ff_ppo.py:181-338), after SHUFFLE MINIBATCHES (:294-307) unless the update step ran it under the rollout."""
        b = built
        if not shuffled:
            anakin.shuffle(b["shards"], epochs, state.key[1], b["perm_ctr"])
        sa, sc = b["sa"], b["sc"]
        a_tree = state.params.actor_params
        seeds = state.key
        D = sa.sizes[0]
        metrics = b["metrics"]
        metrics.zero_()
        grads = b["grads"]
        for ep in range(epochs):  # _update_epoch (ff_ppo.py:286-322)
            batches = []
            for u in range(U):
                sh = b["shards"][u]
                batches.append(ops.PpoBatch(sh.obs[:T].view(B, D), sh.action.view(B, -1) if tanh_head is not None else sh.action.view(B),
                                            sh.log_prob.view(B), sh.value.view(B),
                                            sh.advantages.view(B), sh.targets.view(B), sh.adv_stats, sh.perms[ep]))
            # single shard on a single device: the gradient reduction can hand sum(g^2) straight to the fused
            # optimiser (no separate norm pass / grid barrier); otherwise the all-reduce sits in between.
            prenorm = precision == ops.STX_PREC_BF16 and U == 1 and world == 1
            peers = b["peers_obj"]
            for i in range(nmb):  # _update_minibatch (ff_ppo.py:184-284)
                which = (ep * nmb + i) & 1
                if peers is not None:
                    grads = peers.bufs[which]  # ping-pong arenas in peer-mapped memory
                for u in range(U):  # vmap over "batch" + pmean("batch") (ff_ppo.py:253-256); first shard overwrites
                    sh = b["shards"][u]
                    behaviour = sh.behaviour.view(B, -1) if sh.behaviour is not None else None
                    if loss != "clip" and tanh_head is not None:
                        # ff_ppo_penalty_continuous.py:149-179 / ff_dpo_continuous.py:148-170, entropy noise as below
                        kind = ops.STX_PPO_KL_PENALTY if loss == "kl_penalty" else ops.STX_PPO_DPO
                        ops.ppo_variant_continuous_minibatch_grads(
                            sa, sc, b["arena"], batches[u], i * mb, mb, kind, float(sysc.clip_eps), float(sysc.ent_coef), float(sysc.vf_coef),
                            bool(sysc.standardize_advantages), grads, metrics[ep, i], b["ws"], tanh_head.minimum, tanh_head.maximum,
                            tanh_head.min_scale, behaviour=behaviour, kl_coef=kl_coef, dpo_alpha=dpo_alpha, dpo_beta=dpo_beta,
                            seed=seeds[0] + u, offset=ep * nmb + i, dev_counter=b["ent_ctr"], grad_weight=1.0 / U, overwrite=(u == 0))
                        continue
                    if loss == "kl_penalty":  # ff_ppo_penalty.py:149-210
                        ops.ppo_penalty_minibatch_grads(sa, sc, b["arena"], batches[u], i * mb, mb, behaviour, kl_coef, float(sysc.clip_eps),
                                                        float(sysc.ent_coef), float(sysc.vf_coef), bool(sysc.standardize_advantages), grads,
                                                        metrics[ep, i], b["ws"], grad_weight=1.0 / U, overwrite=(u == 0))
                        continue
                    if tanh_head is not None:
                        # entropy noise of this minibatch: (shard seed, row, call = ep * nmb + i + *ent_ctr)
                        ops.ppo_continuous_minibatch_grads(sa, sc, b["arena"], batches[u], i * mb, mb, float(sysc.clip_eps), float(sysc.ent_coef),
                                                           float(sysc.vf_coef), bool(sysc.standardize_advantages), grads, metrics[ep, i], b["ws"],
                                                           tanh_head.minimum, tanh_head.maximum, tanh_head.min_scale, seed=seeds[0] + u,
                                                           offset=ep * nmb + i, dev_counter=b["ent_ctr"], grad_weight=1.0 / U,
                                                           overwrite=(u == 0))
                        continue
                    ops.ppo_minibatch_grads(sa, sc, b["arena"], batches[u], i * mb, mb, float(sysc.clip_eps),
                                            float(sysc.ent_coef), float(sysc.vf_coef), bool(sysc.standardize_advantages),
                                            grads, metrics[ep, i], b["ws"], precision, 1.0 / U, b["arena_bf16"],
                                            overwrite=(u == 0), adam_scratch=b["plan"].scratch if prenorm else None)
                if peers is not None:
                    # pmean over "device" (ff_ppo.py:258-261) + both optimiser updates (:264-273) in ONE launch:
                    # one-shot all-reduce by direct NVLink peer loads fused into clip+Adam
                    ops.allreduce_clip_adam_step(b["plan"], peers, which, b["arena"], a_tree.arena_mu, a_tree.arena_nu,
                                                 params_bf16=b["arena_bf16"])
                    continue
                if world > 1:  # pmean over "device": summed by NCCL here, scaled in K4
                    dist.all_reduce(grads, op=dist.ReduceOp.SUM)
                # UPDATE ACTOR AND CRITIC PARAMS AND OPTIMISER STATE (ff_ppo.py:264-273), one launch
                ops.clip_adam_step(b["plan"], b["arena"], grads, a_tree.arena_mu, a_tree.arena_nu,
                                   grad_scale=1.0 / world, params_bf16=b["arena_bf16"], prenorm=prenorm)
        if world > 1:
            dist.all_reduce(metrics, op=dist.ReduceOp.SUM)
            metrics.mul_(1.0 / world)

    def _rollout_stats_gae(state: OnPolicyLearnerState) -> None:
        _rollout_phase(state)
        _stats_phase(state)
        _gae_phase(state)

    def _update_step(state: OnPolicyLearnerState) -> None:
        """A single update of the network (ff_ppo.py:61-341), in place on the learner state."""
        b = built
        for sh in b["shards"]:   # learner_state.timestep of ff_ppo.py:131-134
            sh.carry_in()
        # the shuffles run underneath the rollout, which occupies E/64 of the 132 SMs
        anakin.shuffle_beside(b, epochs, state.key[1], lambda: _rollout_stats_gae(state))
        _update_phase(state, shuffled=True)
        # advance the device-resident RNG stream positions (graph replays then draw fresh numbers)
        for sh, env_state in zip(b["shards"], state.env_state):
            sh.advance(env, env_state)
        ops.counter_add(b["roll_ctr"], T)
        ops.counter_add(b["perm_ctr"], epochs)
        if tanh_head is not None:
            ops.counter_add(b["ent_ctr"], epochs * nmb)

    def learner_fn(learner_state: OnPolicyLearnerState) -> AnakinExperimentOutput[OnPolicyLearnerState]:
        """Run arch.num_updates_per_eval update steps (ff_ppo.py:343-370)."""
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config)
        train_metrics = {name: train_out[..., j] for name, j in _VARIANT_METRICS[loss]}
        return AnakinExperimentOutput(learner_state=learner_state._replace(timestep=timestep), episode_metrics=episode_metrics,
                                      train_metrics=train_metrics)

    learner_fn.built = built  # exposed for tests / bench (trajectory buffers, graph handle)
    learner_fn.update_step = _update_step
    learner_fn.phases = {"rollout": _rollout_phase, "stats": _stats_phase, "gae": _gae_phase, "update": _update_phase}
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    return learner_fn


def _discrete_action_head_kwargs(env: Environment, config: DictConfig) -> Dict[str, Any]:
    """Get number/dimension of actions (ff_ppo.py:432-433)."""
    num_actions = int(env.action_space().num_values)
    config.system.action_dim = num_actions
    return {"action_dim": num_actions}


def _uniform_discrete_actions(config: DictConfig, E: int, gen: torch.Generator, dev) -> torch.Tensor:
    return torch.randint(0, int(config.system.action_dim), (E,), device=dev, generator=gen, dtype=torch.int32)


def learner_setup(
    env: Environment, keys: Tuple[int, int, int], config: DictConfig
) -> Tuple[LearnerFn[OnPolicyLearnerState], Actor, OnPolicyLearnerState]:
    """Initialise learner_fn, network, optimiser, environment and states (ff_ppo.py:424-551)."""
    return build_learner(env, keys, config, _discrete_action_head_kwargs, _uniform_discrete_actions)


def build_learner(
    env: Environment, keys: Tuple[int, int, int], config: DictConfig,
    action_head_kwargs: Callable[[Environment, DictConfig], Dict[str, Any]],
    random_actions: Callable[[DictConfig, int, torch.Generator, Any], torch.Tensor],
    loss: str = "clip",
) -> Tuple[LearnerFn[OnPolicyLearnerState], Actor, OnPolicyLearnerState]:
    """The body of learner_setup shared by the PPO variants.  `action_head_kwargs(env, config)` reads the action space, records
    it in config.system and returns the action head's constructor arguments; `random_actions(config, E, gen, device)` draws the
    uniform actions of the observation-normalisation warm-up; `loss` is get_learner_fn's actor-loss variant."""
    rank, world = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())

    head_kwargs = action_head_kwargs(env, config)

    key, actor_net_key, critic_net_key = keys

    # Define network and optimiser (ff_ppo.py:439-463).
    actor_torso = instantiate(config.network.actor_network.pre_torso)
    actor_action_head = instantiate(config.network.actor_network.action_head, **head_kwargs)
    critic_torso = instantiate(config.network.critic_network.pre_torso)
    critic_head = instantiate(config.network.critic_network.critic_head)

    actor_network = Actor(torso=actor_torso, action_head=actor_action_head)
    critic_network = Critic(torso=critic_torso, critic_head=critic_head)
    precision = ops.STX_PREC_BF16 if str(config.arch.get("precision", "f32")) == "bf16" else ops.STX_PREC_F32
    actor_network.precision = critic_network.precision = precision

    actor_lr = make_learning_rate(config.system.actor_lr, config, config.system.epochs, config.system.num_minibatches)
    critic_lr = make_learning_rate(config.system.critic_lr, config, config.system.epochs, config.system.num_minibatches)
    actor_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(actor_lr, eps=1e-5))
    critic_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(critic_lr, eps=1e-5))

    # Initialise observation (ff_ppo.py:466-467).
    init_x = env.observation_space().generate_value()[None, ...].to(device)

    # One flat arena [actor | pad | critic | pad] holds both networks (SURVEY.md 2a: K4, C1).
    sa, sc = actor_network.spec_for(init_x.shape[-1]), critic_network.spec_for(init_x.shape[-1])
    _, coff, total = ops.arena_offsets(sa, sc)
    arena = torch.zeros(total, dtype=torch.float32, device=device)
    actor_params = actor_network.init(actor_net_key, init_x, flat=arena[:coff])
    critic_params = critic_network.init(critic_net_key, init_x, flat=arena[coff:])
    arena_bf16 = None
    if precision == ops.STX_PREC_BF16:
        arena_bf16 = ops.cast_bf16(arena)
        actor_params.flat_bf16, critic_params.flat_bf16 = arena_bf16[:coff], arena_bf16[coff:]
    actor_params.arena_bf16 = arena_bf16

    # Optimiser state (ScaleByAdamState, ScaleByScheduleState per network); the flat arenas ride along on the actor tree.
    params = ActorCriticParams(actor_params, critic_params)
    opt_states = ActorCriticOptStates(*optax.arena_state(actor_params, arena, [(0, sa.param_count), (coff, sc.param_count)]))

    apply_fns = (actor_network.apply, critic_network.apply)
    update_fns = (actor_optim.update, critic_optim.update)
    learn = get_learner_fn(env, apply_fns, update_fns, config, loss=loss)

    # Initialise environment states and timesteps across update-batch shards (ff_ppo.py:492-501).
    U = int(config.arch.update_batch_size)
    shard_keys = srandom.split(key, U + 1)
    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)

    # Load model from checkpoint if specified (ff_ppo.py:504-512) -- params only, as in the reference.
    if warm_start(config, arena) and arena_bf16 is not None:
        ops.cast_bf16(arena, out=arena_bf16)

    # step keys: (sampling seed, shuffle seed) -- per-rank streams like the per-device keys at :515-518
    rollout_seed, shuffle_seed = anakin.rank_seeds(shard_keys[U], 2, rank, world)

    init_learner_state = OnPolicyLearnerState(
        params=params, opt_states=opt_states, key=(rollout_seed, shuffle_seed), env_state=env_states, timestep=timesteps,
    )
    # If normalizing observations, initialize running statistics from warm-up rollouts (ff_ppo.py:539-549); this adds a
    # `running_statistics` field to the learner state.
    if config.system.get("normalize_observations", False):  # ff_dpo.yaml has no such key
        from stoix_b200.utils import running_statistics as rstat

        warmup_observations = _collect_obs_norm_rollouts(env, key, config, random_actions)
        running_statistics = rstat.initialize_statistics_from_data(init_x[0], warmup_observations)
        init_learner_state = rstat.create_with_running_statistics(init_learner_state, running_statistics)
    return learn, actor_network, init_learner_state


def _collect_obs_norm_rollouts(env: Environment, key: int, config: DictConfig, random_actions=_uniform_discrete_actions) -> torch.Tensor:
    """Collect observations for observation normalisation by taking uniformly random actions for
    system.obs_norm_warmup_steps steps (ff_ppo.py:375-421); not counted in the timestep budget.
    Returns (warmup_steps + 1, num_envs, *obs_shape) raw observations of this rank's env shard."""
    steps, E = int(config.system.obs_norm_warmup_steps), int(config.arch.num_envs)
    rank = anakin.world()[0]
    if rank == 0:
        print(f"Initializing observation normalization with {steps * int(config.arch.total_num_envs)} observations... "
              "Be aware, we do not count this in the timestep budget.")
    keys = srandom.split(key, E + 1)
    if hasattr(env, "seed"):
        env.seed = (int(config.arch.seed) + 104729 * (rank + 1)) & ((1 << 63) - 1)
    env_state, ts = env.reset(keys[:E])
    dev = ts.observation.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(int(keys[E]) & ((1 << 62) - 1))
    obs = [ts.observation.float().clone()]
    for _ in range(steps):
        action = random_actions(config, E, gen, dev)
        env_state, ts = env.step(env_state, action)
        obs.append(ts.observation.float().clone())
    return torch.stack(obs, 0)


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (ff_ppo.py:554-706)."""
    return anakin.run_experiment(_config, learner_setup, net_keys=2)


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """Experiment entry point (ff_ppo.py:709-727).  Without hydra-core the composition happens here:
    `python -m stoix_b200.systems.ppo.anakin.ff_ppo env=synthetic/box arch.total_num_envs=4096 ...`"""
    return anakin.entry_point(cfg, overrides, "default_ff_ppo", run_experiment, "PPO")


if __name__ == "__main__":
    hydra_entry_point()
