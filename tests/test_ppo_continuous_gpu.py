"""Continuous-action PPO on the GPU against the fp64 oracle (tests/ppo_continuous_oracle.py): the tanh-Normal log-prob of given
actions, the PPO head gradients with injected entropy noise, the entropy noise stream, the distribution faces, teacher-forced
minibatch gradients, whole update steps (eager and CUDA graph), U = 2 shards, the refusals, observation normalisation, and
learning on the synthetic continuous-control bandit."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import ppo_continuous_oracle as PC

pytestmark = pytest.mark.gpu

LO, HI = -1.0, 1.0


def _np(t):
    return t.detach().float().cpu().numpy().astype(np.float64)


def _dev(x, dt=torch.float32):
    return torch.tensor(np.asarray(x), dtype=dt, device="cuda")


def _head_and_actions(rng, M, A, scale):
    head = rng.normal(0.0, scale, (M, 2 * A)).astype(np.float32)
    action = np.tanh(rng.normal(0.0, 1.5, (M, A))).astype(np.float32)
    return head, _at_the_bounds(action)


def _at_the_bounds(action):
    lo_t, hi_t = np.float32(LO + 1e-3), np.float32(HI - 1e-3)
    action[0:4, 0] = lo_t                       # at the clip thresholds
    action[4:8, 1] = hi_t
    action[8:12, 2] = np.float32(LO)            # beyond them
    action[12:16, 0] = np.float32(HI)
    action[16:20, 1] = np.float32(-0.9995)
    return action


def _sampled(rng, head, minimum=LO, maximum=HI):
    """Actions drawn from the policy the head describes, as the rollout stores them.  The surrogate's ratio exp(logp_new -
    logp_old) turns the fp32 ABSOLUTE error of a log-prob into a RELATIVE error of the gradient, so rows scored far outside
    their policy (|log_prob| in the thousands: a narrow Normal and an unrelated action) would lose digits in any fp32
    implementation; the loss only ever sees actions sampled from (a recent version of) the policy."""
    A = head.shape[1] // 2
    sigma = np.logaddexp(head[:, A:].astype(np.float64), 0.0) + 1e-3
    u = head[:, :A] + sigma * rng.normal(size=(head.shape[0], A))
    return (0.5 * (minimum + maximum) + 0.5 * (maximum - minimum) * np.tanh(u)).astype(np.float32)


@pytest.mark.parametrize("scale", [1.0, 4.0])
def test_log_prob_of_given_actions_matches_oracle(scale):
    from stoix_b200 import ops

    rng = np.random.default_rng(11)
    head, action = _head_and_actions(rng, 512, 6, scale)
    wide = torch.zeros(512, 20, device="cuda")
    wide[:, 5:11] = _dev(action)
    lp = ops.tanh_normal_log_prob(_dev(head), wide[:, 5:11], LO, HI)
    ref, _ = PC.log_prob_given(head.astype(np.float64), action.astype(np.float64), LO, HI)
    np.testing.assert_allclose(_np(lp), ref, rtol=2e-4, atol=2e-4)


def test_head_grads_match_oracle_with_injected_noise():
    from stoix_b200 import ops

    rng = np.random.default_rng(5)
    B, mb, A = 700, 300, 6
    head = rng.normal(0.0, 0.7, (mb, 2 * A)).astype(np.float32)
    idx = rng.permutation(B)[:mb].astype(np.int32)
    action = np.tanh(rng.normal(size=(B, A))).astype(np.float32)
    action[idx] = _at_the_bounds(_sampled(rng, head))
    eps = rng.normal(size=(mb, A)).astype(np.float32)
    adv = rng.normal(size=B).astype(np.float32)
    lp_new, _ = PC.log_prob_given(head.astype(np.float64), action[idx].astype(np.float64), LO, HI)
    logp_old = np.zeros(B, np.float32)
    logp_old[idx] = (lp_new + rng.normal(0.0, 0.3, mb)).astype(np.float32)
    stats = np.array([adv.mean(), 1.0 / adv.std()], np.float32)
    d, metrics = ops.ppo_tanh_normal_head_grads(_dev(head), _dev(idx, torch.int32), _dev(action), _dev(logp_old), _dev(adv), _dev(stats), 0.2, 0.01,
                                                LO, HI, eps_in=_dev(eps))
    adv_m = (adv[idx].astype(np.float64) - stats[0]) * np.float64(stats[1])
    _, dref, info = PC.actor_loss_and_dhead(head.astype(np.float64), action[idx].astype(np.float64), logp_old[idx].astype(np.float64), adv_m,
                                            0.2, 0.01, eps.astype(np.float64), LO, HI)
    np.testing.assert_allclose(_np(d), dref, rtol=2e-3, atol=2e-6)
    m = _np(metrics)
    np.testing.assert_allclose(m[[0, 1, 3]], [info["actor_loss"], info["entropy"], info["advantages"]], rtol=2e-4, atol=1e-6)
    assert m[2] == 0 and m[4] == 0 and m[5] == 0


def test_entropy_noise_stream():
    from stoix_b200 import ops

    M, A = 4096, 6
    head = torch.zeros(M, 2 * A, device="cuda")
    ctr = torch.tensor([5], dtype=torch.int64, device="cuda")
    _, e1 = ops.tanh_normal_entropy(head, LO, HI, seed=1234, offset=2, dev_counter=ctr, want_eps=True)
    _, e2 = ops.tanh_normal_entropy(head, LO, HI, seed=1234, offset=7, want_eps=True)   # same call index 7
    _, e3 = ops.tanh_normal_entropy(head, LO, HI, seed=1234, offset=3, dev_counter=ctr, want_eps=True)
    assert torch.equal(e1, e2)
    assert not torch.equal(e1, e3)
    x = _np(e1)
    assert abs(x.mean()) < 0.05 and abs(x.std() - 1.0) < 0.05
    np.testing.assert_allclose(x, PC.entropy_noise(1234, M, A, 7), rtol=0, atol=1e-6)
    # the minibatch loss draws the same words for minibatch row m
    _, action = _head_and_actions(np.random.default_rng(0), M, A, 1.0)
    eo = torch.empty(M, A, device="cuda")
    zeros = torch.zeros(M, device="cuda")
    ops.ppo_tanh_normal_head_grads(head, None, _dev(action), zeros, zeros, None, 0.2, 0.01, LO, HI, seed=1234, offset=7, eps_out=eo)
    assert torch.equal(eo, e1)


def test_distribution_faces():
    from stoix_b200.networks.heads import NormalAffineTanhDistributionHead

    rng = np.random.default_rng(2)
    head, action = _head_and_actions(rng, 256, 6, 2.0)
    pi = NormalAffineTanhDistributionHead(6, LO, HI).distribution(_dev(head))
    np.testing.assert_allclose(_np(pi.log_prob(_dev(action))), PC.log_prob_given(head.astype(np.float64), action.astype(np.float64), LO, HI)[0],
                               rtol=2e-4, atol=2e-4)
    ent = pi.entropy(seed=99)
    ref, _ = PC.entropy_estimate(head.astype(np.float64), PC.entropy_noise(99, 256, 6, 0).astype(np.float64), LO, HI)
    np.testing.assert_allclose(_np(ent), ref, rtol=2e-4, atol=2e-4)
    a = pi.sample(seed=3)
    assert pi.log_prob(a) is pi._last[1]          # the sampled action keeps the sampler's value (SAC relies on it)
    np.testing.assert_allclose(_np(pi.log_prob(a.clone())), _np(pi._last[1]), rtol=2e-4, atol=2e-4)


def _nets(D, A, layers, act, seed):
    from stoix_b200 import ops

    sa = ops.MlpSpec(tuple([D, *layers, 2 * A]), activation=act)
    sc = ops.MlpSpec(tuple([D, *layers, 1]), activation=act)
    _, coff, total = ops.arena_offsets(sa, sc)
    rng = np.random.default_rng(seed)
    arena = np.zeros(total, np.float32)
    for spec, off in ((sa, 0), (sc, coff)):  # LeCun-normal kernels, small biases
        for i, (w, b) in enumerate(spec.layer_slices()):
            arena[off + w.start: off + w.stop] = rng.normal(0.0, 1.0 / np.sqrt(spec.sizes[i]), w.stop - w.start)
            arena[off + b.start: off + b.stop] = rng.normal(0.0, 0.1, b.stop - b.start)
    return sa, sc, coff, total, arena


@pytest.mark.parametrize("D,A,layers,act,B,mb", [(12, 3, [32, 32], "tanh", 512, 128), (17, 6, [256, 256, 256, 256], "silu", 4096, 1024)])
def test_minibatch_grads_teacher_forced(D, A, layers, act, B, mb):
    from stoix_b200 import ops

    sa, sc, coff, total, arena = _nets(D, A, layers, act, 1)
    rng = np.random.default_rng(4)
    obs = rng.normal(size=(B, D)).astype(np.float32)
    adv = rng.normal(size=B).astype(np.float32)
    tgt = rng.normal(size=B).astype(np.float32)
    v_old = (tgt + rng.normal(0.0, 0.3, B)).astype(np.float32)
    perm = rng.permutation(B).astype(np.int32)
    mb_off = mb  # the second minibatch
    a_or = O.MLPParams.from_flat(arena[: sa.param_count].astype(np.float64), list(sa.sizes), act)
    c_or = O.MLPParams.from_flat(arena[coff: coff + sc.param_count].astype(np.float64), list(sc.sizes), act)
    head_all, _ = O.mlp_forward(a_or, obs.astype(np.float64))
    # Samples of the policy only: a threshold value forced onto a row whose policy sits far from it scores |z| ~ 30 in a tail,
    # where the Mills-ratio terms dominate the gradient norm with fp32 relative errors near 1e-4 (those rows are covered per
    # element by the head tests above); a sample reaches a tail only with a moderate z.
    action = _sampled(rng, head_all)
    lp_all, _ = PC.log_prob_given(head_all, action.astype(np.float64), LO, HI)
    logp_old = (lp_all + rng.normal(0.0, 0.2, B)).astype(np.float32)
    stats = np.array([adv.mean(), 1.0 / adv.std()], np.float32)
    batch = ops.PpoBatch(_dev(obs), _dev(action), _dev(logp_old), _dev(v_old), _dev(adv), _dev(tgt), _dev(stats), _dev(perm, torch.int32))
    ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_F32, "cuda")
    params = _dev(arena)
    grads = []
    for _ in range(2):
        g = torch.zeros(total, device="cuda")
        metrics = torch.zeros(6, device="cuda")
        eps_out = torch.empty(mb, A, device="cuda")
        ops.ppo_continuous_minibatch_grads(sa, sc, params, batch, mb_off, mb, 0.2, 0.01, 0.5, True, g, metrics, ws, LO, HI, seed=77, offset=3,
                                           eps_out=eps_out, overwrite=True)
        grads.append(g)
    torch.cuda.synchronize()
    assert torch.equal(grads[0], grads[1])           # deterministic: fixed reduction orders
    idx = perm[mb_off: mb_off + mb]
    np.testing.assert_allclose(_np(eps_out), PC.entropy_noise(77, mb, A, 3), atol=1e-6, rtol=0)
    adv_m = (adv[idx].astype(np.float64) - stats[0]) * np.float64(stats[1])
    head, a_acts = O.mlp_forward(a_or, obs[idx].astype(np.float64))
    _, dhead, a_info = PC.actor_loss_and_dhead(head, action[idx].astype(np.float64), logp_old[idx].astype(np.float64), adv_m, 0.2, 0.01,
                                               _np(eps_out), LO, HI)
    a_g = O.mlp_backward(a_or, a_acts, dhead).flat()
    v, c_acts = O.mlp_forward(c_or, obs[idx].astype(np.float64))
    _, dv, c_info = O.critic_loss_and_dvalue(v[:, 0], v_old[idx].astype(np.float64), tgt[idx].astype(np.float64), 0.2, 0.5)
    c_g = O.mlp_backward(c_or, c_acts, dv[:, None]).flat()
    g = _np(grads[0])
    for got, ref in ((g[: sa.param_count], a_g), (g[coff: coff + sc.param_count], c_g)):
        assert np.linalg.norm(got - ref) <= 1e-5 * np.linalg.norm(ref)
    m = _np(metrics)
    np.testing.assert_allclose(m[[0, 1, 2, 3]], [a_info["actor_loss"], a_info["entropy"], c_info["value_loss"], a_info["advantages"]],
                               rtol=2e-4, atol=1e-6)


def _cfg(overrides):
    from stoix_b200.config import compose

    base = ["arch.num_evaluation=1", "arch.absolute_metric=False", "arch.num_eval_episodes=8", "logger.use_console=False"]
    cfg = compose("default_ff_ppo_continuous", base + overrides, config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    return cfg


def _setup(cfg):
    from stoix_b200 import random as srandom
    from stoix_b200.systems.ppo.anakin import ff_ppo_continuous
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = check_total_timesteps(cfg, quiet=True)
    env, eval_env = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 4)
    learn, actor_net, state = ff_ppo_continuous.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    return cfg, env, eval_env, learn, actor_net, state


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("E,T,nmb,layers,obs_dim,A", [(8, 16, 4, [32, 32], 12, 3), (16, 8, 2, [256, 256, 256, 256], 17, 6)])
def test_update_step_matches_oracle(E, T, nmb, layers, obs_dim, A, graph):
    from stoix_b200 import ops

    n_updates, epochs = 3, 4
    cfg = _cfg([f"arch.total_num_envs={E}", f"system.rollout_length={T}", f"system.num_minibatches={nmb}", f"arch.total_timesteps={E * T * n_updates}",
                f"arch.cuda_graph={graph}", f"network.actor_network.pre_torso.layer_sizes={layers}",
                f"network.critic_network.pre_torso.layer_sizes={layers}", f"env.kwargs.obs_dim={obs_dim}", f"env.kwargs.act_dim={A}",
                "env.kwargs.p_term=0.05", "env.kwargs.p_trunc=0.05"])
    cfg, env, _, learn, _, state = _setup(cfg)
    assert cfg.arch.num_updates == n_updates
    with torch.no_grad():  # non-trivial heads and biases so that every gradient path is exercised
        arena = state.params.actor_params.arena
        arena.add_(torch.randn(arena.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 0.05)
    sa, sc = state.params.actor_params.spec, state.params.critic_params.spec
    actor = O.MLPParams.from_flat(_np(state.params.actor_params.flat), list(sa.sizes), sa.activation)
    critic = O.MLPParams.from_flat(_np(state.params.critic_params.flat), list(sc.sizes), sc.activation)
    a_st = O.AdamState(np.zeros(actor.flat().size), np.zeros(actor.flat().size))
    c_st = O.AdamState(np.zeros(critic.flat().size), np.zeros(critic.flat().size))
    h = O.PPOHyper(epochs=epochs, num_minibatches=nmb, num_updates=n_updates)
    mb = T * E // nmb
    for upd in range(n_updates):
        cfg.arch.num_updates_per_eval = 1
        out = learn(state)
        state = out.learner_state
        torch.cuda.synchronize()
        sh = learn.built["shards"][0]
        traj = O.Trajectory(obs=_np(sh.obs[:T]), action=_np(sh.action), reward=_np(sh.reward), done=sh.done.cpu().numpy().astype(bool),
                            truncated=sh.truncated.cpu().numpy().astype(bool), next_obs=_np(sh.next_obs))
        assert sh.action.shape == (T, E, A) and sh.action.dtype == torch.float32
        PC.evaluate_rollout(actor, critic, traj, LO, HI)
        np.testing.assert_allclose(_np(sh.log_prob), traj.log_prob, rtol=2e-4, atol=2e-4)
        np.testing.assert_allclose(_np(sh.value), traj.value, rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(_np(sh.bootstrap_value), traj.bootstrap_value, rtol=1e-4, atol=2e-6)
        traj.log_prob = _np(sh.log_prob)  # the behaviour log-prob the learner stored (checked above)
        perms = np.stack([ops.make_permutation(T * E, state.key[1], ep + epochs * upd, device="cuda").cpu().numpy() for ep in range(epochs)])
        eps = np.stack([np.stack([PC.entropy_noise(state.key[0], mb, A, ep * nmb + i + upd * epochs * nmb) for i in range(nmb)])
                        for ep in range(epochs)]).astype(np.float64)
        actor, critic, metrics, adv, tgt = PC.ppo_update(actor, critic, a_st, c_st, traj, perms, h, eps, LO, HI)
        for name in ("actor_loss", "entropy", "value_loss"):
            np.testing.assert_allclose(_np(out.train_metrics[name][0]), metrics[name], rtol=2e-4, atol=2e-6)
        np.testing.assert_allclose(_np(state.params.actor_params.flat), actor.flat(), rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(_np(state.params.critic_params.flat), critic.flat(), rtol=1e-4, atol=2e-6)
    assert state.params.actor_params.arena_counts.cpu().tolist() == [n_updates * epochs * nmb] * 4
    assert int(learn.built["ent_ctr"].item()) == n_updates * epochs * nmb


def test_update_batch_size_two():
    cfg = _cfg(["arch.total_num_envs=32", "arch.update_batch_size=2", "system.rollout_length=8", "system.num_minibatches=2",
                "arch.total_timesteps=1024", "network.actor_network.pre_torso.layer_sizes=[32,32]",
                "network.critic_network.pre_torso.layer_sizes=[32,32]"])
    cfg, _, _, learn, _, state = _setup(cfg)
    p0 = state.params.actor_params.arena.clone()
    out = learn(state)
    torch.cuda.synchronize()
    assert out.episode_metrics["episode_return"].shape == (int(cfg.arch.num_updates_per_eval), 2, 8, 16)
    assert torch.isfinite(out.learner_state.params.actor_params.arena).all()
    assert not torch.equal(p0, out.learner_state.params.actor_params.arena)
    s0, s1 = learn.built["shards"]
    assert not torch.equal(s0.obs, s1.obs) and not torch.equal(s0.action, s1.action) and not torch.equal(s0.perms, s1.perms)


def test_bf16_refused_and_observation_normalisation_runs():
    with pytest.raises(ValueError, match="tanh-Normal"):
        _setup(_cfg(["arch.total_num_envs=16", "system.rollout_length=8", "arch.total_timesteps=256", "arch.precision=bf16"]))
    cfg = _cfg(["arch.total_num_envs=16", "system.rollout_length=8", "system.num_minibatches=2", "arch.total_timesteps=512",
                "system.normalize_observations=True", "system.obs_norm_warmup_steps=4", "network.actor_network.pre_torso.layer_sizes=[32,32]",
                "network.critic_network.pre_torso.layer_sizes=[32,32]"])
    cfg, _, _, learn, _, state = _setup(cfg)
    out = learn(state)
    torch.cuda.synchronize()
    rs = out.learner_state.running_statistics
    assert torch.isfinite(rs.mean).all() and torch.isfinite(rs.std).all() and (rs.std > 0).all()
    assert torch.isfinite(out.learner_state.params.actor_params.arena).all()


def test_greedy_policy_learns_the_bandit():
    """Untrained greedy policy: tanh(loc ~ 0) ~ 0 scores E[tanh(Z)^2] ~ -0.394 per step; PPO must push it above -0.2."""
    from stoix_b200.evaluator import get_distribution_act_fn, get_ff_evaluator_fn

    cfg = _cfg(["arch.total_num_envs=1024", "system.rollout_length=16", "arch.total_timesteps=4000000", "arch.num_evaluation=1",
                "arch.evaluation_greedy=True", "arch.num_eval_episodes=64"])
    cfg, _, eval_env, learn, actor_net, state = _setup(cfg)
    evaluate = get_ff_evaluator_fn(eval_env, get_distribution_act_fn(cfg, actor_net.apply), cfg)

    def per_step_reward(st):
        o = evaluate(st.params.actor_params, 5)
        return float((o["episode_return"] / o["episode_length"].float()).mean().item())

    before = per_step_reward(state)
    out = learn(state)
    torch.cuda.synchronize()
    after = per_step_reward(out.learner_state)
    assert before < -0.3, before
    assert after > -0.2, (before, after)
