"""CPU checks of the IMPALA oracle (tests/impala_oracle.py) and of IMPALA's host logic: the closed-form head gradients against torch
autograd of the reference losses as written, the V-trace special cases, RMSProp, the column-block row tables and the configs."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import impala_oracle as I


def _batch(rng, T, Em, A, shift=0.0):
    logits = rng.standard_normal((T, Em, A))
    values = rng.standard_normal((T + 1, Em))
    action = rng.integers(0, A, (T, Em))
    lp_b = O.categorical_log_prob(logits, action) + shift + 0.5 * rng.standard_normal((T, Em))
    reward = rng.standard_normal((T, Em))
    done = rng.random((T, Em)) < 0.2
    done[0, 0] = done[-1, -1] = True
    return logits, values, action, lp_b, reward, done


def _torch_losses(logits, values, action, lp_b, reward, done, h: I.VtraceHyper):
    """ff_impala.py:397-522 in torch fp64 exactly as written: rho from the actor (no gradient into the critic loss), the V-trace scan,
    stop_gradient on vs and on pg_advantage, summed losses."""
    z = torch.tensor(logits, requires_grad=True)
    v = torch.tensor(values, requires_grad=True)
    a = torch.tensor(action)
    lp = torch.log_softmax(z, -1)
    logp = lp.gather(-1, a[..., None])[..., 0]
    rho = torch.exp(logp.detach() - torch.tensor(lp_b))
    d = h.gamma * (1.0 - torch.tensor(done, dtype=torch.float64))
    r = torch.tensor(reward)
    v_tm1, v_t = v[:-1], v[1:]
    c = h.lambda_ * torch.clamp(rho, max=1.0)
    delta = torch.clamp(rho, max=h.clip_rho) * (r + d * v_t - v_tm1)
    accs, acc = [], torch.zeros_like(r[0])
    for t in range(r.shape[0] - 1, -1, -1):
        acc = delta[t] + d[t] * c[t] * acc
        accs.append(acc)
    errors = (torch.stack(accs[::-1]) + v_tm1).detach() - v_tm1
    vs = errors + v_tm1
    q = r + d * torch.cat([h.lambda_ * vs[1:] + (1 - h.lambda_) * v_tm1[1:], v_t[-1:]], 0)
    pg = (torch.clamp(rho, max=h.clip_pg_rho) * (q - v_tm1)).detach()
    value_loss = 0.5 * (errors ** 2).sum()
    ent = -(lp.exp() * lp).sum()
    actor_loss = -(pg * logp).sum()
    (h.vf_coef * value_loss + actor_loss - h.ent_coef * ent).backward()
    return z.grad.numpy(), v.grad.numpy(), {"actor_loss": actor_loss.item(), "entropy": ent.item(), "value_loss": value_loss.item(),
                                            "q_estimate": q.mean().item(), "pg_advantage": pg.mean().item()}


@pytest.mark.parametrize("lam,clip_rho,clip_pg,shift", [(1.0, 1.0, 1.0, 0.0), (0.9, 2.0, 0.5, 0.0), (0.9, 1.0, 1.0, 4.0), (1.0, 1.0, 1.0, -4.0)])
def test_head_grads_match_autograd_of_the_reference_losses(lam, clip_rho, clip_pg, shift):
    rng = np.random.default_rng(1)
    batch = _batch(rng, 9, 5, 6, shift)
    h = I.VtraceHyper(gamma=0.97, lambda_=lam, clip_rho=clip_rho, clip_pg_rho=clip_pg, ent_coef=0.03, vf_coef=0.7)
    dz, dv, m = I.loss_and_head_grads(*batch, h)
    tz, tv, tm = _torch_losses(*batch, h)
    np.testing.assert_allclose(dz, tz, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dv, tv, rtol=1e-12, atol=1e-12)
    assert np.all(dv[-1] == 0.0)
    for k in m:
        np.testing.assert_allclose(m[k], tm[k], rtol=1e-12, atol=1e-12)


def test_vtrace_on_policy_lambda_one_is_gae():
    """rho = 1, lambda = 1: vs - v_tm1 is GAE(lambda = 1) of the PPO oracle, and pg_adv = q - v_tm1 is the same advantage."""
    rng = np.random.default_rng(2)
    T, E = 12, 4
    v = rng.standard_normal((T + 1, E))
    r = rng.standard_normal((T, E))
    d = 0.99 * (rng.random((T, E)) > 0.2)
    err, pg, q = I.vtrace(v[:-1], v[1:], r, d, np.ones((T, E)), 1.0)
    adv, _ = O.gae(r, d, 1.0, v_tm1=v[:-1], v_t=v[1:], time_major=True)
    np.testing.assert_allclose(err, adv, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(pg, adv, rtol=1e-12, atol=1e-12)


def test_vtrace_lambda_zero_is_the_one_step_target_with_clipped_rho():
    rng = np.random.default_rng(3)
    T, E = 7, 3
    v = rng.standard_normal((T + 1, E))
    r = rng.standard_normal((T, E))
    d = 0.9 * (rng.random((T, E)) > 0.3)
    rho = np.exp(2 * rng.standard_normal((T, E)))
    err, pg, q = I.vtrace(v[:-1], v[1:], r, d, rho, 0.0, clip_rho=1.5, clip_pg_rho=0.8)
    np.testing.assert_allclose(err, np.minimum(1.5, rho) * (r + d * v[1:] - v[:-1]), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(q, r + d * v[1:], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(pg, np.minimum(0.8, rho) * (r + d * v[1:] - v[:-1]), rtol=1e-12, atol=1e-12)


def test_reward_normalisation_uses_the_population_std():
    r = np.array([[1.0, 2.0], [3.0, 6.0]])
    got = I.normalize_rewards(r, scale=2.0, eps=0.0)
    np.testing.assert_allclose(got, 2.0 * (r - 3.0) / np.sqrt(((r - 3.0) ** 2).mean()))


def test_rmsprop_matches_torch_rmsprop():
    """optax.rmsprop's defaults = torch.optim.RMSprop(alpha=decay, eps inside the root is optax's; torch adds eps outside) -- so compare with
    eps = 0 where the two agree, over several steps with clipping off."""
    rng = np.random.default_rng(4)
    n = 11
    p0 = rng.standard_normal(n)
    st = I.RmspropState(np.zeros(n))
    p = p0.copy()
    w = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.RMSprop([w], lr=1e-2, alpha=0.9, eps=0.0)
    for _ in range(4):
        g = rng.standard_normal(n)
        p = I.clip_rmsprop_step(p, g, st, 1e-2, 1e30, decay=0.9, eps=0.0)
        w.grad = torch.tensor(g)
        opt.step()
    np.testing.assert_allclose(p, w.detach().numpy(), rtol=1e-12, atol=1e-14)
    assert st.count == st.sched_count == 4


def test_rmsprop_clips_by_the_global_norm():
    g = np.array([3.0, 4.0])
    st = I.RmspropState(np.zeros(2))
    p = I.clip_rmsprop_step(np.zeros(2), g, st, 1.0, 1.0, decay=0.5, eps=0.0)
    np.testing.assert_allclose(st.nu, 0.5 * (g / 5.0) ** 2)
    np.testing.assert_allclose(p, -(g / 5.0) / np.sqrt(st.nu))


def test_whole_update_walks_the_column_blocks_in_order():
    """Two minibatches: the second block's gradient is taken at the parameters the first block's step left."""
    rng = np.random.default_rng(5)
    T, E, D, A = 4, 6, 3, 3
    actor, critic = O.init_mlp(rng, [D, 8, A], 0.5), O.init_mlp(rng, [D, 8, 1], 1.0)
    obs = rng.standard_normal((T + 1, E, D))
    act = rng.integers(0, A, (T + 1, E))
    lp = rng.standard_normal((T + 1, E)) - 1.0
    rew, done = rng.standard_normal((T + 1, E)), rng.random((T + 1, E)) < 0.2
    h = I.ImpalaHyper(num_minibatches=2, actor_lr=1e-2, critic_lr=1e-2, num_updates=3, normalize_rewards=True)
    n_a, n_c = actor.flat().size, critic.flat().size
    a2, c2, ms, stats = I.update(actor, critic, I.RmspropState(np.zeros(n_a)), I.RmspropState(np.zeros(n_c)), obs, act, lp, rew, done, h)
    assert len(ms) == 2 and stats == (pytest.approx(rew[:T].mean()), pytest.approx(rew[:T].std()))
    # the first block alone, by hand
    r = I.normalize_rewards(rew[:T], 1.0, 1e-8)
    x = obs[:, :3]
    logits, ca = O.mlp_forward(actor, x[:T].reshape(-1, D))
    v, cc = O.mlp_forward(critic, x.reshape(-1, D))
    dz, dv, m0 = I.loss_and_head_grads(logits.reshape(T, 3, A), v.reshape(T + 1, 3), act[:T, :3], lp[:T, :3], r[:, :3], done[:T, :3], h)
    assert m0 == ms[0]
    st = I.RmspropState(np.zeros(n_a))
    a1 = I.clip_rmsprop_step(actor.flat(), O.mlp_backward(actor, ca, dz.reshape(-1, A)).flat(), st, 1e-2, 40.0)
    assert not np.allclose(a1, a2.flat())  # the second block moved it again


def test_row_tables_and_configs():
    from stoix_b200.config import compose
    from stoix_b200.systems.impala.sebulba import ff_impala

    T, E, nmb = 3, 8, 4
    rows = ff_impala.minibatch_row_index(T, E, nmb)
    assert rows.dtype == np.int32 and rows.shape == (nmb, (T + 1) * 2)
    grid = np.arange((T + 1) * E).reshape(T + 1, E)
    for i in range(nmb):
        np.testing.assert_array_equal(rows[i], grid[:, 2 * i: 2 * i + 2].reshape(-1))
    assert np.array_equal(np.sort(rows.reshape(-1)), np.arange((T + 1) * E))

    cfg = compose("default_ff_impala", ["system.vtrace_lambda=0.9"], config_dir="default/sebulba")
    s = cfg.system
    assert s.system_name == "ff_impala" and s.vtrace_lambda == 0.9
    assert (s.actor_lr, s.critic_lr, s.rollout_length, s.gamma, s.clip_rho_threshold, s.clip_pg_rho_threshold) == (6e-4, 6e-4, 128, 0.99, 1.0, 1.0)
    assert (s.ent_coef, s.vf_coef, s.max_grad_norm, s.normalize_rewards, s.reward_scale, s.reward_eps) == (0.01, 0.5, 40.0, False, 1.0, 1e-8)
    assert s.num_minibatches == 4 and s.decay_learning_rates is True
    assert cfg.arch.architecture_name == "sebulba" and cfg.env.env_name == "synthetic"
    cp = compose("default_ff_impala", ["env=gymnax/cartpole"], config_dir="default/sebulba")
    assert cp.env.scenario.name == "CartPole-v1"


def test_rmsprop_facade_and_refusals():
    from stoix_b200 import optim

    opt = optim.chain(optim.clip_by_global_norm(40.0), optim.rmsprop(6e-4))
    assert opt.rule == "rmsprop" and opt.max_grad_norm == 40.0 and opt.init_lr == 6e-4
    assert (opt.adam.decay, opt.adam.eps) == (0.9, 1e-8)
    for bad in (dict(centered=True), dict(momentum=0.9), dict(nesterov=True), dict(bias_correction=True)):
        with pytest.raises(NotImplementedError):
            optim.rmsprop(1e-3, **bad)


def test_bf16_refused_on_the_host():
    from stoix_b200.config import compose
    from stoix_b200.systems.impala.sebulba import ff_impala

    cfg = compose("default_ff_impala", ["arch.precision=bf16"], config_dir="default/sebulba")
    with pytest.raises(ValueError, match="bf16"):
        ff_impala.check_config(cfg)
    with pytest.raises(ValueError, match="bf16"):
        ff_impala.run_experiment(cfg)


def test_launch_file_is_the_implementation_module():
    import importlib

    from stoix_b200.systems.impala.sebulba import ff_impala

    mod = importlib.import_module("stoix.systems.impala.sebulba.ff_impala")
    assert mod is ff_impala
    for name in ("get_act_fn", "get_rollout_fn", "get_actor_thread", "get_learner_step_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
        assert callable(getattr(mod, name))
