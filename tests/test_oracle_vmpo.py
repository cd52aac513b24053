"""CPU checks of V-MPO: the fp64 oracle's analytic gradients against torch.autograd of the restated rlax.vmpo_loss, the n-step
returns against a direct transcription of multistep.py:148-210, the configs, launch files, arena layout and refusals."""
import math

import numpy as np
import pytest
import torch

from tests import vmpo_oracle as V


def _autograd_loss(kind, head, head_t, action, adv, duals, eps, eps_a, eps_s, per_dim, lo=-1.0, hi=1.0, min_scale=1e-3):
    """rlax.vmpo_loss restated in torch (module docstring of tests/vmpo_oracle.py); the actions lie inside the tanh clip band."""
    head = torch.tensor(head, requires_grad=True)
    duals = torch.tensor(duals, requires_grad=True)
    head_t = torch.tensor(head_t)
    adv = torch.tensor(adv)
    N = adv.numel()
    k = int(0.5 * N)
    tau = torch.sort(adv, descending=True).values[k - 1]
    mask = adv >= tau
    K = mask.sum()
    eta = torch.nn.functional.softplus(duals[0]) + 1e-8
    x = adv / eta
    lse = torch.logsumexp(x[mask], 0)
    w = torch.where(mask, torch.exp(x - lse), torch.zeros_like(x)).detach()
    if kind == "categorical":
        lp = torch.log_softmax(head, -1)
        lq = torch.log_softmax(head_t, -1)
        logp = lp[torch.arange(N), torch.tensor(action, dtype=torch.long)]
        kls = [((lq.exp() * (lq - lp)).sum(-1), duals[1:2], eps_a)]
    else:
        A = head.shape[1] // 2
        mu, sig = head[:, :A], torch.nn.functional.softplus(head[:, A:]) + min_scale
        mu_t, sig_t = head_t[:, :A], torch.nn.functional.softplus(head_t[:, A:]) + min_scale
        s, sh = (hi - lo) / 2, (hi + lo) / 2
        u = torch.atanh((torch.tensor(action) - sh) / s)
        z = (u - mu) / sig
        fldj = 2.0 * (math.log(2.0) - u - torch.nn.functional.softplus(-2.0 * u))
        logp = (-0.5 * z * z - torch.log(sig) - 0.5 * math.log(2 * math.pi) - fldj - math.log(s)).sum(-1)
        km = (mu - mu_t) ** 2 / (2 * sig_t ** 2)
        ks = torch.log(sig / sig_t) + sig_t ** 2 / (2 * sig ** 2) - 0.5
        if per_dim:
            kls = [(km, duals[1:1 + A], eps_a), (ks, duals[1 + A:], eps_s)]
        else:
            kls = [(km.sum(-1), duals[1:2], eps_a), (ks.sum(-1), duals[2:3], eps_s)]
    loss = -(w * logp).sum() + eta * (eps + lse - torch.log(K.double()))
    for kl, la, e in kls:
        alpha = torch.nn.functional.softplus(la) + 1e-8
        mean_kl = kl.mean(0)
        loss = loss + (alpha.detach() * mean_kl).sum() + (alpha * (e - mean_kl.detach())).sum()
    loss.backward()
    return float(loss.detach()), head.grad.numpy(), duals.grad.numpy()


@pytest.mark.parametrize("kind,per_dim", [("categorical", True), ("tanh_normal", True), ("tanh_normal", False)])
def test_oracle_gradients_match_autograd(kind, per_dim):
    rng = np.random.default_rng(7)
    N, A = 37, 3
    W = A if kind == "categorical" else 2 * A
    head = rng.normal(size=(N, W))
    head_t = head + 0.3 * rng.normal(size=(N, W))
    action = rng.integers(0, A, N) if kind == "categorical" else rng.uniform(-0.9, 0.9, (N, A))
    adv = rng.normal(size=N) * 3
    adv[:5] = np.sort(adv)[::-1][N // 2 - 1]   # ties at tau
    n_dual = 2 if kind == "categorical" else 1 + 2 * (A if per_dim else 1)
    duals = rng.normal(size=n_dual)
    out = V.vmpo_loss(kind, head, head_t, action, adv, duals, 0.1, 0.01, 0.005, per_dim)
    loss, g_head, g_duals = _autograd_loss(kind, head, head_t, action, adv, duals, 0.1, 0.01, 0.005, per_dim)
    assert out["K"] > N // 2
    np.testing.assert_allclose(out["loss"], loss, rtol=1e-12)
    np.testing.assert_allclose(out["d_head"], g_head, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(out["d_duals"], g_duals, rtol=1e-9, atol=1e-12)


def test_topk_float_tie_rule():
    adv = np.array([3.0, -0.0, 0.0, 0.0, -1.0, -2.0], np.float32)
    tau, mask, K = V.topk_select(adv)   # k = 3: the third largest is a zero; both signed zeros tie
    assert tau == 0.0 and K == 4 and mask.tolist() == [True, True, True, True, False, False]


def _n_step_transcription(r_t, discount_t, v_t, n, lambda_t=1.0):
    """multistep.py:148-210 line by line in NumPy."""
    r_t, discount_t, v_t = (np.swapaxes(x, 0, 1) for x in (r_t, discount_t, v_t))
    seq_len, batch_size = r_t.shape
    lambda_t = np.ones_like(discount_t) * lambda_t
    pad_size = min(n - 1, seq_len)
    targets = np.concatenate([v_t[n - 1:], np.array([v_t[-1]] * pad_size).reshape(pad_size, batch_size)], axis=0)
    r_t = np.concatenate([r_t, np.zeros((n - 1, batch_size))], axis=0)
    discount_t = np.concatenate([discount_t, np.ones((n - 1, batch_size))], axis=0)
    lambda_t = np.concatenate([lambda_t, np.ones((n - 1, batch_size))], axis=0)
    v_t = np.concatenate([v_t, np.array([v_t[-1]] * (n - 1)).reshape(n - 1, batch_size)], axis=0)
    for i in reversed(range(n)):
        r_ = r_t[i:i + seq_len]
        discount_ = discount_t[i:i + seq_len]
        lambda_ = lambda_t[i:i + seq_len]
        v_ = v_t[i:i + seq_len]
        targets = r_ + discount_ * ((1.0 - lambda_) * v_ + lambda_ * targets)
    return np.swapaxes(targets, 0, 1)


@pytest.mark.parametrize("n_of_T", ["1", "3", "T", "T+2"])
@pytest.mark.parametrize("lam", [1.0, 0.7])
def test_n_step_returns_match_transcription(n_of_T, lam):
    rng = np.random.default_rng(3)
    B, T = 5, 9
    n = {"1": 1, "3": 3, "T": T, "T+2": T + 2}[n_of_T]
    r = rng.normal(size=(B, T))
    d = 0.99 * (rng.random((B, T)) > 0.2)
    v = rng.normal(size=(B, T))
    np.testing.assert_allclose(V.n_step_returns(r, d, v, n, lam), _n_step_transcription(r, d, v, n, lam), rtol=1e-13, atol=1e-13)


# the reference's stoix/configs/system/mpo/ff_vmpo.yaml and ff_vmpo_continuous.yaml
_REF_DISCRETE = dict(system_name="ff_vmpo", rollout_length=32, epochs=16, actor_lr=3e-4, critic_lr=3e-4, dual_lr=1e-2, actor_target_period=50,
                     gamma=0.99, max_grad_norm=1.0, decay_learning_rates=False, max_abs_reward=20000, epsilon=0.5, epsilon_policy=0.001,
                     init_log_temperature=3.0, init_log_alpha=3.0, use_n_step_bootstrap=False, n_step_for_sequence_bootstrap=5, gae_lambda=0.95)
_REF_CONTINUOUS = dict(system_name="ff_vmpo", rollout_length=32, epochs=16, actor_lr=3e-4, critic_lr=3e-4, dual_lr=1e-2, actor_target_period=50,
                       gamma=0.99, max_grad_norm=0.5, decay_learning_rates=False, max_abs_reward=20000, epsilon=0.05, epsilon_mean=0.05,
                       epsilon_stddev=0.0005, init_log_temperature=10.0, init_log_alpha_mean=10, init_log_alpha_stddev=500, per_dim_constraining=True,
                       use_n_step_bootstrap=False, n_step_for_sequence_bootstrap=10, gae_lambda=0.95)


@pytest.mark.parametrize("name,ref,head,env", [("default_ff_vmpo", _REF_DISCRETE, "CategoricalHead", "gymnax"),
                                               ("default_ff_vmpo_continuous", _REF_CONTINUOUS, "NormalAffineTanhDistributionHead", "synthetic_continuous")])
def test_config_composition(name, ref, head, env):
    from stoix_b200.config import compose

    cfg = compose(name, [], config_dir="default/anakin")
    for k, v in ref.items():
        assert cfg.system[k] == v, k
    assert cfg.network.actor_network.action_head._target_.endswith(head)
    assert cfg.env.env_name == env


def test_launch_files_alias_the_implementation():
    import stoix.systems.mpo.ff_vmpo as a
    import stoix.systems.mpo.ff_vmpo_continuous as b
    from stoix_b200.systems.mpo import ff_vmpo, ff_vmpo_continuous

    assert a is ff_vmpo and b is ff_vmpo_continuous
    for m in (a, b):
        for fn in ("get_learner_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
            assert callable(getattr(m, fn))


@pytest.mark.parametrize("action_dim,per_dim,n_dual", [(None, True, 2), (6, True, 13), (6, False, 3)])
def test_arena_layout(action_dim, per_dim, n_dual):
    from stoix_b200 import ops
    from stoix_b200.networks.heads import NormalAffineTanhDistributionHead
    from stoix_b200.systems.mpo.ff_vmpo import dual_count, vmpo_arena_layout

    head = None if action_dim is None else NormalAffineTanhDistributionHead(action_dim, -1.0, 1.0)
    assert dual_count(head, per_dim) == n_dual
    sa, sc = ops.MlpSpec((5, 256, 256, 2 * (action_dim or 1))), ops.MlpSpec((5, 256, 256, 1))
    lay = vmpo_arena_layout(sa, sc, n_dual)
    assert lay["actor"] == 0 and lay["critic"] % 4 == 0 and lay["duals"] % 4 == 0
    assert lay["critic"] >= sa.param_count and lay["duals"] >= lay["critic"] + sc.param_count
    assert lay["n_dual"] == n_dual and lay["total"] >= lay["duals"] + n_dual and lay["total"] % 8 == 0


def test_refusals():
    from stoix_b200.config import compose
    from stoix_b200.systems.mpo.ff_vmpo import _actor_head, check_config
    from stoix_b200.utils.multistep import batch_n_step_bootstrapped_returns

    cfg = compose("default_ff_vmpo", ["arch.precision=bf16"], config_dir="default/anakin")
    with pytest.raises(ValueError, match="bf16"):
        check_config(cfg)
    cfg = compose("default_ff_vmpo", ["system.rollout_length=1"], config_dir="default/anakin")
    with pytest.raises(ValueError, match="rollout_length"):
        check_config(cfg)

    class _Net:
        action_head = object()

    with pytest.raises(ValueError, match="Categorical"):
        _actor_head(_Net())
    with pytest.raises(ValueError, match="scalar lambda_t"):
        batch_n_step_bootstrapped_returns(torch.zeros(2, 3), torch.zeros(2, 3), torch.zeros(2, 3), 2, lambda_t=torch.ones(2, 3))
