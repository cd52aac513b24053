"""CPU checks of ff_mpo: tests/mpo_oracle.py against torch autograd of a transcription of the reference loss, Retrace and n-step
against transcriptions of the reference, the sequence-buffer rules, configs, launch file, arena layout and refusals."""
import os

import numpy as np
import pytest
import torch

from tests import mpo_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _reference_categorical_loss(zo, zt, q, duals, epsilon, epsilon_policy):
    """discrete_loss.py:49-106 transcribed into torch, stop_gradient as detach; returns the scalar loss jax.grad differentiates."""
    q = q.t()                                                                 # [D, B] -> [B, D]
    temperature = torch.nn.functional.softplus(duals[0]) + 1e-8
    alpha = torch.nn.functional.softplus(duals[1]) + 1e-8
    tempered = q.detach() / temperature
    unnormalized = tempered + torch.log_softmax(zt, -1)
    logits_e_step = torch.log_softmax(unnormalized, -1)
    log_normalizer = unnormalized[:, 0] - logits_e_step[:, 0]
    loss_temperature = temperature * (epsilon + log_normalizer.mean())
    p_e = torch.exp(logits_e_step)
    loss_policy = (-(p_e * torch.log_softmax(zo, -1)).sum(-1)).mean()       # Categorical.cross_entropy
    lpt, lpo = torch.log_softmax(zt, -1), torch.log_softmax(zo, -1)
    kl = (torch.exp(lpt) * (lpt - lpo)).sum(-1)
    mean_kl = kl.mean(0)
    loss_kl = alpha.detach() * mean_kl
    loss_alpha = alpha * (epsilon_policy - mean_kl.detach())
    return (loss_policy + loss_kl + loss_alpha + loss_temperature).mean()


@pytest.mark.parametrize("M,A,seed", [(1, 2, 0), (7, 2, 1), (64, 5, 2), (33, 32, 3)])
def test_categorical_oracle_against_autograd(M, A, seed):
    g = torch.Generator().manual_seed(seed)
    zo = torch.randn(M, A, generator=g, dtype=torch.float64, requires_grad=True)
    zt = torch.randn(M, A, generator=g, dtype=torch.float64)
    q = torch.randn(A, M, generator=g, dtype=torch.float64) * 4
    duals = torch.tensor([0.7, -2.0], dtype=torch.float64, requires_grad=True)
    loss = _reference_categorical_loss(zo, zt, q, duals, 0.01, 1e-3)
    loss.backward()
    dh, dg, _ = orc.categorical_loss(zo.detach().numpy(), zt.numpy(), q.numpy(), duals.detach().numpy(), 0.01, 1e-3)
    np.testing.assert_allclose(dh, zo.grad.numpy(), rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(dg, duals.grad.numpy(), rtol=1e-10, atol=1e-13)


def test_categorical_oracle_metrics():
    g = torch.Generator().manual_seed(5)
    zo, zt, q = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((9, 3), (9, 3), (3, 9)))
    _, _, mt = orc.categorical_loss(zo.numpy(), zt.numpy(), q.numpy(), np.array([0.1, 0.2]), 0.01, 1e-3)
    lpo, lpt = torch.log_softmax(zo, -1), torch.log_softmax(zt, -1)
    assert mt["entropy_online"] == pytest.approx(float(-(lpo.exp() * lpo).sum(-1).mean()))
    assert mt["q_min"] == pytest.approx(float(q.t().min(0).values.mean()))
    assert mt["kl_mean_rel"] == pytest.approx(float((lpt.exp() * (lpt - lpo)).sum(-1).mean()) / 1e-3)
    assert mt["loss_alpha"] + mt["loss_kl"] == pytest.approx(mt["alpha"] * 1e-3)


def _reference_general_returns(q_t, v_t, r_t, discount_t, c_t):
    """multistep.py:250-267 transcribed (batch-major inputs, reverse scan)."""
    q_t, v_t, r_t, discount_t, c_t = (x.T for x in (q_t, v_t, r_t, discount_t, c_t))
    g = r_t[-1] + discount_t[-1] * v_t[-1]
    out = [g]
    acc = g
    for reward, discount, c, v, q in reversed(list(zip(r_t[:-1], discount_t[:-1], c_t, v_t[:-1], q_t))):
        acc = reward + discount * (v - c * q + c * acc)
        out.insert(0, acc)
    return np.stack(out).T


@pytest.mark.parametrize("B,S,lam", [(3, 2, 0.95), (4, 8, 0.95), (2, 16, 1.0)])
def test_retrace_oracle_against_reference(B, S, lam):
    """ff_mpo.py:276-284: batch_retrace_continuous(online_q_t[:, :-1], target_q_t[:, 1:-1], v_t[:, 1:], r_t[:, :-1], d_t[:, :-1],
    log_rhos[:, 1:-1]) against the oracle on the time-major views the learner passes."""
    rng = np.random.default_rng(B * S)
    tq, v, r, lr = (rng.normal(size=(B, S)) for _ in range(4))
    d = 0.99 * (rng.random((B, S)) > 0.2)
    c = np.minimum(1.0, np.exp(lr[:, 1:-1])) * lam
    want = _reference_general_returns(tq[:, 1:-1], v[:, 1:], r[:, :-1], d[:, :-1], c)
    got = orc.retrace(tq.T[1: S - 1], v.T[1:], r.T[:-1], d.T[:-1], lr.T[1: S - 1], lam).T
    np.testing.assert_allclose(got, want, rtol=1e-12)


def _reference_n_step(r_t, discount_t, v_t, n):
    """multistep.py:178-207 transcribed, lambda 1."""
    r_t, discount_t, v_t = r_t.T, discount_t.T, v_t.T
    T, Bn = r_t.shape
    lam = np.ones_like(discount_t)
    pad = min(n - 1, T)
    targets = np.concatenate([v_t[n - 1:], np.array([v_t[-1]] * pad).reshape(pad, Bn)], axis=0)
    r_t = np.concatenate([r_t, np.zeros((n - 1, Bn))])
    discount_t = np.concatenate([discount_t, np.ones((n - 1, Bn))])
    lam = np.concatenate([lam, np.ones((n - 1, Bn))])
    v_t = np.concatenate([v_t, np.array([v_t[-1]] * (n - 1)).reshape(n - 1, Bn)])
    for i in reversed(range(n)):
        targets = r_t[i: i + T] + discount_t[i: i + T] * ((1.0 - lam[i: i + T]) * v_t[i: i + T] + lam[i: i + T] * targets)
    return targets.T


@pytest.mark.parametrize("T,n", [(7, 5), (3, 5), (8, 1)])
def test_n_step_oracle_against_reference(T, n):
    rng = np.random.default_rng(T + n)
    r, v = rng.normal(size=(4, T)), rng.normal(size=(4, T))
    d = 0.99 * (rng.random((4, T)) > 0.3)
    np.testing.assert_allclose(orc.n_step_targets(r.T, d.T, v.T, n).T, _reference_n_step(r, d, v, n), rtol=1e-12)


def test_gae_oracle_against_definition():
    rng = np.random.default_rng(0)
    r, d, v = rng.normal(size=(5, 3)), 0.9 * np.ones((5, 3)), rng.normal(size=(6, 3))
    tgt = orc.gae_targets(r, d, 1.0, v)
    # lambda = 1: the discounted return bootstrapped from v[K]
    want = np.zeros_like(r)
    g = v[5]
    for k in range(4, -1, -1):
        g = r[k] + d[k] * g
        want[k] = g
    np.testing.assert_allclose(tgt, want, rtol=1e-12)


def test_sequence_ring_rules():
    """The valid starts never straddle the write head, before and after the ring wraps."""
    ring = orc.SequenceRing(L=6, E=1, D=1)
    z = lambda T: (np.zeros((T, 1, 1)), np.zeros((T, 1), np.int32), np.arange(T, dtype=np.float32)[:, None], np.zeros((T, 1), np.uint8),
                   np.zeros((T, 1), np.float32))
    ring.add(*z(3))
    assert ring.valid_starts(2) == [0, 1]
    ring.add(*z(5))          # wraps: w = 2, every row written
    assert (ring.w, ring.c) == (2, 6)
    assert ring.valid_starts(3) == [2, 3, 4, 5]
    _, _, rew, _, _, where = ring.sample(3, [(0, 0), (0, 3)])
    assert where == [(0, 2), (0, 5)]
    np.testing.assert_array_equal(rew.T, [[2, 0, 1], [2, 3, 4]])   # ring rows hold rewards [3, 4, 2, 0, 1, 2]


def _cfg(over=()):
    from stoix_b200.config import compose
    return compose("default_ff_mpo", list(over), config_dir="default/anakin")


def test_configs_carry_reference_values():
    cfg = _cfg()
    s = cfg.system
    assert (s.system_name, s.rollout_length, s.epochs, s.warmup_steps, s.total_buffer_size, s.total_batch_size) == ("ff_mpo", 8, 16, 16, 50000, 32)
    assert (s.sample_sequence_length, s.period, s.num_samples, s.tau, s.max_grad_norm) == (8, 1, 20, 0.005, 40.0)
    assert (s.epsilon, s.epsilon_policy, s.init_log_temperature, s.init_log_alpha, s.retrace_lambda, s.gae_lambda) == (0.01, 1e-3, 3.0, 3.0, 0.95, 0.95)
    assert (s.use_retrace, s.use_n_step_bootstrap, s.stochastic_policy_eval, s.use_online_policy_to_bootstrap) == (False, False, True, False)
    n = cfg.network
    assert list(n.actor_network.pre_torso.layer_sizes) == [256, 256] and n.actor_network.pre_torso.activation == "silu"
    assert n.q_network.input_layer._target_ == "stoix.networks.inputs.EmbeddingActionInput"
    assert cfg.env.scenario.name.lower().startswith("cartpole") or "cartpole" in str(cfg.env).lower()


def test_launch_file_is_the_implementation():
    import importlib

    from stoix_b200.systems.mpo import ff_mpo
    assert importlib.import_module("stoix.systems.mpo.ff_mpo") is ff_mpo
    assert os.path.exists(os.path.join(ROOT, "stoix", "systems", "mpo", "ff_mpo.py"))


def test_arena_layout():
    from stoix_b200 import ops
    from stoix_b200.systems.mpo.ff_mpo import mpo_arena_layout
    sa, sq = ops.MlpSpec((4, 256, 256, 2), "silu"), ops.MlpSpec((6, 256, 256, 1), "silu")
    lay = mpo_arena_layout(sa, sq)
    assert lay["actor"] == 0 and lay["q"] % 8 == 0 and lay["duals"] % 8 == 0 and lay["total"] % 8 == 0
    assert lay["q"] >= sa.param_count and lay["duals"] - lay["q"] >= sq.param_count and lay["total"] - lay["duals"] >= 2


def test_learner_state_fields_follow_reference():
    from stoix_b200.systems.mpo.mpo_types import MPOLearnerState, MPOOptStates, MPOParams
    assert MPOParams._fields == ("actor_params", "q_params", "dual_params")
    assert MPOOptStates._fields == ("actor_opt_state", "q_opt_state", "dual_opt_state")
    assert MPOLearnerState._fields == ("params", "opt_states", "buffer_state", "key", "env_state", "timestep")


@pytest.mark.parametrize("over,match", [(("arch.precision=bf16",), "bf16"), (("system.period=2",), "period"),
                                        (("system.sample_sequence_length=1",), "sample_sequence_length")])
def test_refusals(over, match):
    from stoix_b200.systems.mpo.ff_mpo import check_config
    with pytest.raises(ValueError, match=match):
        check_config(_cfg(over))
    check_config(_cfg())


def test_buffer_refusals():
    from stoix_b200.utils.replay import SequenceBuffer
    with pytest.raises(ValueError, match="period"):
        SequenceBuffer(1000, 4, 8, 10, 3, "cpu", period=2)
    with pytest.raises(ValueError, match="fewer than one sequence"):
        SequenceBuffer(70, 4, 8, 10, 3, "cpu")


def test_head_refusal():
    from stoix_b200.networks.base import FeedForwardActor
    from stoix_b200.networks.heads import DiscreteQNetworkHead
    from stoix_b200.networks.torso import MLPTorso
    from stoix_b200.systems.mpo.ff_mpo import _actor_head
    with pytest.raises(ValueError, match="Categorical"):
        _actor_head(FeedForwardActor(DiscreteQNetworkHead(action_dim=2), MLPTorso([8])))


def test_warmup_shorter_than_a_sequence_is_refused():
    from stoix_b200.systems.mpo.ff_mpo import check_config
    with pytest.raises(ValueError, match="before the first sample"):
        check_config(_cfg(("system.warmup_steps=0", "system.rollout_length=4")))


def test_continuous_configs_carry_reference_values():
    from stoix_b200.config import compose
    cfg = compose("default_ff_mpo_continuous", [], config_dir="default/anakin")
    s = cfg.system
    assert (s.epochs, s.total_buffer_size, s.total_batch_size, s.sample_sequence_length, s.num_samples, s.max_grad_norm) == (72, 200000, 256, 16, 128, 0.5)
    assert (s.epsilon, s.epsilon_mean, s.epsilon_stddev, s.init_log_temperature, s.init_log_alpha_mean, s.init_log_alpha_stddev) == \
        (0.05, 0.05, 0.0005, 10.0, 10.0, 500.0)
    assert s.per_dim_constraining is True and s.dual_lr == 1e-3
    assert list(cfg.network.q_network.pre_torso.layer_sizes) == [256] * 4
    import importlib

    from stoix_b200.systems.mpo import ff_mpo_continuous
    assert importlib.import_module("stoix.systems.mpo.ff_mpo_continuous") is ff_mpo_continuous
