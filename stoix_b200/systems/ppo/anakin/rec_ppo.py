"""Anakin recurrent PPO on H100 -- drop-in for stoix/systems/ppo/anakin/rec_ppo.py (SURVEY.md 8f row 3), fp32.

Same entry points (get_learner_fn :38, learner_setup :431, run_experiment :593, hydra_entry_point) and state contracts
(RNNLearnerState, RNNPPOTransition, ActorCriticHiddenStates).  Behaviour restated from the reference, including its details:
the hidden state is reset where the PREVIOUS transition ended (done | truncated); the transition stores the hidden states AFTER
its step and the losses re-run the networks from `hstates[0]` of the chunk; GAE goes through the `values=` interface with
discount_t = (1 - last_done_t) * gamma; minibatches are column subsets of the batch reshaped to (chunk, num_envs * num_chunks).

  reference (JAX)                                   here (H100)
  ------------------------------------------------  -----------------------------------------------------------------------
  nn.scan of GRUCell over T inside jax.grad         pre-torso + input projections of ALL steps as one MLP launch chain,
                                                    RecLayout.sequence_forward / _backward for the recurrence (BPTT with the saved
                                                    gates, d W_h as one GEMM over the stored sequences), post-torso + head as
                                                    one MLP chain; the losses' output gradients from stx_ppo_head_grads
  permutation + take of the whole batch per epoch   keyed bijection over the columns; kernels gather rows through an index
  2 x optax.chain(clip, adam)                       one fused clip+Adam launch over [actor | critic]
  pmean(batch); pmean(device)                       mean over shards; NCCL all-reduce of the flat gradient arena
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from stoix_b200 import ops
from stoix_b200 import optim as optax
from stoix_b200 import random as srandom
from stoix_b200.base_types import ActorCriticOptStates, ActorCriticParams, AnakinExperimentOutput
from stoix_b200.config import DictConfig, instantiate
from stoix_b200.envs.base import Environment, StepOut
from stoix_b200.evaluator import get_rnn_evaluator_fn
from stoix_b200.networks.recurrent import RecLayout, RecurrentActor, RecurrentCritic, ScannedRNN
from stoix_b200.systems import anakin
from stoix_b200.systems.ppo.ppo_types import ActorCriticHiddenStates, RNNLearnerState, RNNPPOTransition
from stoix_b200.utils.checkpointing import warm_start
from stoix_b200.utils.training import make_learning_rate

_METRIC_NAMES = ("actor_loss", "entropy", "value_loss", "advantages", "pred_value", "target_value")
_pad8 = lambda n: (int(n) + 7) // 8 * 8


class _Shard:
    """Trajectory of one (device, update-batch) shard, time-major (RNNPPOTransition fields + the carried row T)."""

    def __init__(self, T: int, E: int, D: int, H: int, device):   # H = carry width (2 x hidden for lstm)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs = z(T + 1, E, D)                       # row t = last_timestep.observation of step t, row T = the carry
        self.env_obs = self.obs                         # the rows anakin.learn seeds and carries
        self.done, self.trunc = z(T + 1, E, dt=torch.uint8), z(T + 1, E, dt=torch.uint8)   # flags BEFORE step t
        self.reset = z(T + 1, E, dt=torch.uint8)        # done | truncated
        self.action = z(T, E, dt=torch.int32)
        self.value, self.reward, self.log_prob = z(T + 1, E), z(T, E), z(T, E)             # value row T = masked bootstrap value
        self.h_actor, self.h_critic = z(T, E, H), z(T, E, H)                               # hidden states AFTER step t
        self.h_a_cur, self.h_c_cur = z(E, H), z(E, H)                                     # carried hidden states
        self.discount = z(T, E)
        self.advantages, self.targets, self.adv_stats = z(T, E), z(T, E), z(2)
        self.episode_return, self.episode_length = z(T, E), z(T, E, dt=torch.int32)
        self.is_terminal_step = z(T, E, dt=torch.bool)
        self.next_obs_scratch = z(E, D)                 # extras["next_obs"] is not used by rec_ppo

    def transition(self, T: int) -> RNNPPOTransition:
        return RNNPPOTransition(self.done[:T], self.trunc[:T], self.action, self.value[:T], self.reward, self.log_prob, self.obs[:T],
                                ActorCriticHiddenStates(self.h_actor, self.h_critic),
                                {"episode_return": self.episode_return, "episode_length": self.episode_length, "is_terminal_step": self.is_terminal_step})


class _NetWs:
    """Train-mode workspaces of one recurrent network for a minibatch of `chunk` x `C` rows."""

    def __init__(self, lay: RecLayout, chunk: int, C: int, out_dim: int, device):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        M, H = chunk * C, lay.H
        self.ws_pre, self.ws_post = ops.mlp_train_workspace(lay.spec_pre, M, device), ops.mlp_train_workspace(lay.spec_post, M, device)
        self.ws_seq = lay.sequence_workspace(chunk, C, device)
        self.gi, self.d_gi = z(chunk, C, lay.G * H), z(chunk, C, lay.G * H)
        self.h_seq, self.d_h = z(chunk, C, H), z(chunk, C, H)
        self.h0 = z(C, lay.S)
        self.out, self.d_out = z(M, out_dim), z(M, out_dim)


def get_learner_fn(env: Environment, apply_fns: Tuple[Callable, Callable], update_fns: Tuple[Callable, Callable], config: DictConfig):
    """Get the learner function (rec_ppo.py:38-428)."""
    actor_apply_fn, critic_apply_fn = apply_fns
    actor_net, critic_net = anakin.owner(actor_apply_fn, RecurrentActor, "apply_fns[0]"), anakin.owner(critic_apply_fn, RecurrentCritic, "apply_fns[1]")
    actor_opt, critic_opt = (anakin.owner(f, optax.GradientTransformation, f"update_fns[{i}]") for i, f in enumerate(update_fns))
    rank, world = anakin.world()
    sysc, arch = config.system, config.arch
    T, E, U = int(sysc.rollout_length), int(arch.num_envs), int(arch.update_batch_size)
    epochs, nmb = int(sysc.epochs), int(sysc.num_minibatches)
    chunk = int(sysc.recurrent_chunk_size) if sysc.get("recurrent_chunk_size", None) else T
    assert T % chunk == 0, "rollout_length must be divisible by recurrent_chunk_size"
    nc = T // chunk
    cols_total = E * nc
    assert cols_total % nmb == 0, "num_envs * num_recurrent_chunks must be divisible by num_minibatches"
    C = cols_total // nmb
    gamma, lam = float(sysc.gamma), float(sysc.gae_lambda)
    has_step_into = hasattr(env, "step_into")
    built: Dict[str, Any] = {}

    def _build(state: RNNLearnerState) -> None:
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        la, lc = a_tree.layout, c_tree.layout
        dev = a_tree.flat.device
        D, A, H = la.spec_pre.sizes[0], la.spec_post.sizes[-1], la.S   # H: carry width
        coff = _pad8(la.param_count)
        total = coff + _pad8(lc.param_count)
        plan = optax.adam_plan([(0, la.param_count, actor_opt), (coff, lc.param_count, critic_opt)], dev, a_tree.arena_counts)
        built.update(la=la, lc=lc, dev=dev, D=D, A=A, H=H, coff=coff, total=total, plan=plan, arena=a_tree.arena,
                     shards=[_Shard(T, E, D, H, dev) for _ in range(U)],
                     ws_a=_NetWs(la, chunk, C, A, dev), ws_c=_NetWs(lc, chunk, C, 1, dev),
                     grads=torch.zeros(total, dtype=torch.float32, device=dev),
                     metrics=torch.zeros(epochs, nmb, 8, dtype=torch.float32, device=dev),
                     logits=torch.zeros(E, A, device=dev), reset_mb=torch.zeros(chunk, C, dtype=torch.uint8, device=dev),
                     roll_ctr=torch.zeros(1, dtype=torch.int64, device=dev), perm_ctr=torch.zeros(1, dtype=torch.int64, device=dev),
                     side_stream=torch.cuda.Stream(device=dev), metrics_c=torch.zeros(8, dtype=torch.float32, device=dev),
                     graph=None, eager_done=False,
                     t_rows=(torch.arange(chunk, device=dev, dtype=torch.int64) * cols_total)[:, None])
        for sh, done, trunc, h in zip(built["shards"], state.done, state.truncated, state.hstates):   # the carried flags and hidden states
            sh.done[T].copy_(done), sh.trunc[T].copy_(trunc)
            sh.h_a_cur.copy_(h.policy_hidden_state), sh.h_c_cur.copy_(h.critic_hidden_state)

    def _net_step(net, tree, h_cur: torch.Tensor, obs_t: torch.Tensor, reset_t: torch.Tensor):
        """One step of a recurrent network (rec_ppo.py:90-101): T = 1 sequence."""
        h_new, out = net._forward(tree, h_cur, (obs_t[None], reset_t[None]))
        return h_new, out[0]

    def _rollout_phase(state: RNNLearnerState) -> None:
        """_env_step x rollout_length (rec_ppo.py:69-143) + the bootstrap value (:146-163), per shard, in place."""
        b = built
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        for u in range(U):
            sh: _Shard = b["shards"][u]
            for t in range(T):
                torch.bitwise_or(sh.done[t], sh.trunc[t], out=sh.reset[t])           # reset_hidden_state (:86)
                main, side = torch.cuda.current_stream(), b["side_stream"]
                side.wait_stream(main)
                with torch.cuda.stream(side):      # the critic's step beside the actor's step, sampling and env step
                    h_c, value = _net_step(critic_net, c_tree, sh.h_c_cur, sh.obs[t], sh.reset[t])
                    sh.value[t].copy_(value.reshape(-1))
                    sh.h_critic[t].copy_(h_c), sh.h_c_cur.copy_(h_c)
                    h_c.record_stream(side), value.record_stream(side)
                h_a, logits = _net_step(actor_net, a_tree, sh.h_a_cur, sh.obs[t], sh.reset[t])
                ops.categorical(logits.contiguous(), None, state.key[0] + u, t, b["roll_ctr"], out=(sh.action[t], sh.log_prob[t]))
                sh.h_actor[t].copy_(h_a), sh.h_a_cur.copy_(h_a)
                # the env writes the transition rows in place; flags land in row t + 1, the ones BEFORE that step (:105-106)
                anakin.step_env(env, state.env_state, u, sh.action[t],
                                StepOut(sh.obs[t + 1], sh.next_obs_scratch, sh.reward[t], sh.done[t + 1], sh.trunc[t + 1], sh.episode_return[t],
                                        sh.episode_length[t], sh.is_terminal_step[t].view(torch.uint8)), t)
                main.wait_stream(side)             # next step (and the bootstrap value) read h_c_cur / obs written on both streams
            torch.bitwise_or(sh.done[T], sh.trunc[T], out=sh.reset[T])
            _, last_val = _net_step(critic_net, c_tree, sh.h_c_cur, sh.obs[T], sh.reset[T])
            sh.value[T].copy_(torch.where(sh.done[T].bool(), torch.zeros_like(last_val.reshape(-1)), last_val.reshape(-1)))   # :160-163
            if has_step_into and hasattr(env, "advance"):
                env.advance(state.env_state[u], T)
        ops.counter_add(b["roll_ctr"], T)

    def _gae_phase(state: RNNLearnerState) -> None:
        """rec_ppo.py:165-179: discount from the flags stored WITH the transition (the ones before the step), values = [value, last_val]."""
        for u in range(U):
            sh: _Shard = built["shards"][u]
            torch.mul(1.0 - sh.done[:T].float(), gamma, out=sh.discount)
            adv, tgt, stats = ops.gae_generic(sh.reward, sh.discount, lam, sh.value[:T], sh.value[1:], None, 1 if sysc.standardize_advantages else 0)
            sh.advantages.copy_(adv), sh.targets.copy_(tgt)
            if stats is not None:
                sh.adv_stats.copy_(stats)

    def _net_grads(lay: RecLayout, p_flat: torch.Tensor, g_flat: torch.Tensor, w: _NetWs, sh: _Shard, h_store: torch.Tensor, idx: torch.Tensor,
                   is_actor: bool, metrics: torch.Tensor, weight: float, overwrite: bool) -> None:
        """Forward over the chunk, loss head, backward through time for one network on the rows `idx` (rec_ppo.py:207-262)."""
        b = built
        D, H = b["D"], lay.H
        pre, _, _, post = lay.blocks(p_flat)
        g_pre, _, _, g_post = lay.blocks(g_flat)
        obs_flat = sh.obs[:T].reshape(T * E, D)
        ops.mlp_forward_train(lay.spec_pre, pre, obs_flat, w.ws_pre, out=w.gi.view(chunk * C, lay.G * H), row_idx=idx)
        ops.gather_rows(h_store.reshape(T * E, lay.S), idx[:C], w.h0)                    # hstates[0] of the chunk (:216-218)
        lay.sequence_forward(p_flat, w.gi, b["reset_mb"], w.h0, w.ws_seq, out=w.h_seq)
        ops.mlp_forward_train(lay.spec_post, post, w.h_seq.view(chunk * C, H), w.ws_post, out=w.out)
        stats = sh.adv_stats if sysc.standardize_advantages else None
        ops.ppo_head_grads(w.out if is_actor else None, None if is_actor else w.out, idx, sh.action.reshape(-1), sh.log_prob.reshape(-1),
                           sh.value[:T].reshape(-1), sh.advantages.reshape(-1), sh.targets.reshape(-1), stats, float(sysc.clip_eps), float(sysc.ent_coef),
                           float(sysc.vf_coef), w.d_out if is_actor else None, None if is_actor else w.d_out, metrics, weight=weight,
                           scratch_key="ppo_head_actor" if is_actor else "ppo_head_critic")
        ops.mlp_backward(lay.spec_post, post, w.h_seq.view(chunk * C, H), w.d_out, w.ws_post, net_grad=g_post, grad_weight=weight, overwrite=overwrite,
                         d_input=w.d_h.view(chunk * C, H))
        lay.sequence_backward(p_flat, g_flat, w.d_h, b["reset_mb"], w.ws_seq, w.d_gi, weight, overwrite)
        ops.mlp_backward(lay.spec_pre, pre, obs_flat, w.d_gi.view(chunk * C, lay.G * H), w.ws_pre, net_grad=g_pre, grad_weight=weight, overwrite=overwrite,
                         row_idx=idx)

    def _minibatch_grads(state: RNNLearnerState, u: int, cols: torch.Tensor, metrics: torch.Tensor, overwrite: bool) -> None:
        b, sh = built, built["shards"][u]
        idx = (b["t_rows"] + cols.to(torch.int64)[None, :]).reshape(-1).to(torch.int32)  # row of (t', column j) in the flat (T * E) arrays
        ops.gather_rows(sh.reset[:T].reshape(-1), idx, b["reset_mb"].view(-1))           # done | truncated of the rows (:211, :240)
        a_tree, c_tree = state.params.actor_params, state.params.critic_params
        # the two networks are independent until the optimiser: the critic's chain of small launches runs on a second stream beside
        # the actor's (each kernel of the recurrence fills a fraction of the GPU); own metric slots, summed after the join
        main, side = torch.cuda.current_stream(), b["side_stream"]
        b["metrics_c"].zero_()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            _net_grads(b["lc"], c_tree.flat, b["grads"][b["coff"]:], b["ws_c"], sh, sh.h_critic, idx, False, b["metrics_c"], 1.0 / U, overwrite)
        _net_grads(b["la"], a_tree.flat, b["grads"], b["ws_a"], sh, sh.h_actor, idx, True, metrics, 1.0 / U, overwrite)
        main.wait_stream(side)
        metrics.add_(b["metrics_c"])

    def _update_phase(state: RNNLearnerState, cols_override: Optional[torch.Tensor] = None) -> None:
        """UPDATE EPOCHS (rec_ppo.py:181-384)."""
        b = built
        metrics = b["metrics"]
        metrics.zero_()
        a_tree = state.params.actor_params
        for ep in range(epochs):
            perms = [cols_override[ep] if cols_override is not None else
                     ops.make_permutation(cols_total, state.key[1] + u, ep, dev_counter=b["perm_ctr"], device=b["dev"]) for u in range(U)]
            for i in range(nmb):
                for u in range(U):
                    _minibatch_grads(state, u, perms[u][i * C:(i + 1) * C], metrics[ep, i], overwrite=(u == 0))
                if world > 1:
                    dist.all_reduce(b["grads"], op=dist.ReduceOp.SUM)
                ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu, grad_scale=1.0 / world)
        ops.counter_add(b["perm_ctr"], epochs)
        if world > 1:
            dist.all_reduce(metrics, op=dist.ReduceOp.SUM)
            metrics.mul_(1.0 / world)

    def _update_step(state: RNNLearnerState) -> None:
        for u in range(U):   # the last observation / flags of the previous rollout (row T) start this one; the finished
            sh = built["shards"][u]                                                  # trajectory stays readable until then
            sh.obs[0].copy_(sh.obs[T]), sh.done[0].copy_(sh.done[T]), sh.trunc[0].copy_(sh.trunc[T])
        _rollout_phase(state)
        _gae_phase(state)
        _update_phase(state)

    def learner_fn(learner_state: RNNLearnerState) -> AnakinExperimentOutput:
        # one CUDA graph per update step: ~10k launches replayed
        timestep, episode_metrics, train_out = anakin.learn(built, _build, _update_step, learner_state, config)
        shards = built["shards"]
        learner_state = learner_state._replace(
            timestep=timestep, done=[sh.done[T].bool() for sh in shards], truncated=[sh.trunc[T].bool() for sh in shards],
            hstates=[ActorCriticHiddenStates(sh.h_a_cur, sh.h_c_cur) for sh in shards])
        train_metrics = {name: train_out[..., j] for j, name in enumerate(_METRIC_NAMES)}
        return AnakinExperimentOutput(learner_state=learner_state, episode_metrics=episode_metrics, train_metrics=train_metrics)

    learner_fn.built = built
    learner_fn.ensure_built = lambda st: anakin.ensure_built(built, _build, st)
    learner_fn.phases = {"rollout": _rollout_phase, "gae": _gae_phase, "update": _update_phase}
    learner_fn.update_step = _update_step
    learner_fn.geometry = {"chunk": chunk, "num_chunks": nc, "cols_per_minibatch": C}
    return learner_fn


def learner_setup(env: Environment, keys: Tuple[int, int, int], config: DictConfig):
    """Initialise learner_fn, networks, optimisers, environment and states (rec_ppo.py:431-590)."""
    rank, world = anakin.world()
    device = torch.device("cuda", torch.cuda.current_device())
    num_actions = int(env.action_space().num_values)
    config.system.action_dim = num_actions
    key, actor_net_key, critic_net_key = keys

    net_a, net_c = config.network.actor_network, config.network.critic_network
    actor_network = RecurrentActor(pre_torso=instantiate(net_a.pre_torso), hidden_state_dim=int(net_c.rnn_layer.hidden_state_dim),
                                   cell_type=str(net_c.rnn_layer.cell_type), post_torso=instantiate(net_a.post_torso),
                                   action_head=instantiate(net_a.action_head, action_dim=num_actions))   # (sic) the reference reads the critic's rnn_layer for both (:456-469)
    critic_network = RecurrentCritic(pre_torso=instantiate(net_c.pre_torso), hidden_state_dim=int(net_c.rnn_layer.hidden_state_dim),
                                     cell_type=str(net_c.rnn_layer.cell_type), post_torso=instantiate(net_c.post_torso),
                                     critic_head=instantiate(net_c.critic_head))
    actor_rnn = ScannedRNN(int(net_a.rnn_layer.hidden_state_dim), str(net_a.rnn_layer.cell_type))
    critic_rnn = ScannedRNN(int(net_c.rnn_layer.hidden_state_dim), str(net_c.rnn_layer.cell_type))

    actor_lr = make_learning_rate(config.system.actor_lr, config, config.system.epochs, config.system.num_minibatches)
    critic_lr = make_learning_rate(config.system.critic_lr, config, config.system.epochs, config.system.num_minibatches)
    actor_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(actor_lr, eps=1e-5))
    critic_optim = optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm), optax.adam(critic_lr, eps=1e-5))

    U, E = int(config.arch.update_batch_size), int(config.arch.num_envs)
    init_obs = env.observation_space().generate_value().to(device).float()[None, None].repeat(1, E, 1)
    init_x = (init_obs, torch.zeros(1, E, dtype=torch.bool, device=device))
    init_policy_hstate = actor_rnn.initialize_carry(E, device)
    init_critic_hstate = critic_rnn.initialize_carry(E, device)

    la, lc = actor_network.layout_for(init_obs.shape[-1]), critic_network.layout_for(init_obs.shape[-1])
    coff = _pad8(la.param_count)
    arena = torch.zeros(coff + _pad8(lc.param_count), dtype=torch.float32, device=device)
    actor_params = actor_network.init(actor_net_key, init_policy_hstate, init_x, flat=arena[:coff])
    critic_params = critic_network.init(critic_net_key, init_critic_hstate, init_x, flat=arena[coff:])
    opt_states = ActorCriticOptStates(*optax.arena_state(actor_params, arena, [(0, la.param_count), (coff, lc.param_count)]))

    apply_fns = (actor_network.apply, critic_network.apply)
    update_fns = (actor_optim.update, critic_optim.update)
    learn = get_learner_fn(env, apply_fns, update_fns, config)

    params = ActorCriticParams(actor_params, critic_params)
    warm_start(config, arena)

    shard_keys = srandom.split(key, U + 1)
    env_states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)
    dones = [torch.zeros(E, dtype=torch.bool, device=device) for _ in range(U)]
    truncs = [torch.zeros(E, dtype=torch.bool, device=device) for _ in range(U)]
    hstates = [ActorCriticHiddenStates(init_policy_hstate.clone(), init_critic_hstate.clone()) for _ in range(U)]
    init_learner_state = RNNLearnerState(params, opt_states, anakin.rank_seeds(shard_keys[U], 2, rank, world),
                                         env_states, timesteps, dones, truncs, hstates)
    return learn, actor_network, init_learner_state


def run_experiment(_config: DictConfig) -> float:
    """Runs experiment (rec_ppo.py:593-750), evaluating with the hidden state carried (get_rnn_evaluator_fn)."""
    return anakin.run_experiment(
        _config, learner_setup, net_keys=2,
        make_evaluators=lambda eval_env, key_e, net, config: (get_rnn_evaluator_fn(eval_env, net, config),
                                                              get_rnn_evaluator_fn(eval_env, net, config, 10)),
        best_tree=lambda net, tree, flat: net.build_tree(tree.layout, flat))


def hydra_entry_point(cfg: Optional[DictConfig] = None, overrides: Optional[List[str]] = None) -> float:
    """`python -m stoix_b200.systems.ppo.anakin.rec_ppo env=gymnax/cartpole arch.total_num_envs=256 ...`"""
    return anakin.entry_point(cfg, overrides, "default_rec_ppo", run_experiment, "Recurrent PPO")


if __name__ == "__main__":
    hydra_entry_point()
