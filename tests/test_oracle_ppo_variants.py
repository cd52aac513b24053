"""CPU checks of the PPO variants (KL penalty, DPO): the oracle's hand-derived actor-loss gradients against torch.autograd of the
literal reference formulas in float64 (KL = 0 rows, rows in both clipped tails, DPO rows in all four branches), the entry
configs, the `stoix.*` aliases and the layout of the new C struct."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import ppo_continuous_oracle as PC
from tests import ppo_variants_oracle as PV

LO, HI = -1.0, 1.0
F = torch.nn.functional


def _t(x, grad=False):
    return torch.tensor(np.asarray(x, np.float64), requires_grad=grad)


def _torch_tanh_normal(head, action, eps, minimum, maximum, min_scale=1e-3, epsilon=1e-3):
    """log_prob of given actions (distributions.py:56-80, clipped tails) and the seeded entropy estimate (:85-88), per row."""
    A = head.shape[-1] // 2
    loc, sigma = head[:, :A], F.softplus(head[:, A:]) + min_scale
    s, sh = (maximum - minimum) / 2.0, (minimum + maximum) / 2.0
    lo, hi = minimum + epsilon, maximum - epsilon
    u_lo, u_hi = np.arctanh((lo - sh) / s), np.arctanh((hi - sh) / s)
    ev = action.clamp(lo, hi)
    u = torch.atanh(((ev - sh) / s).clamp(-1 + 1e-15, 1 - 1e-15))
    fldj = lambda x: 2.0 * (np.log(2.0) - x - F.softplus(-2.0 * x))
    inner = torch.distributions.Normal(loc, sigma).log_prob(u) - fldj(u) - np.log(s)
    left = torch.special.log_ndtr((u_lo - loc) / sigma) - np.log(epsilon)
    right = torch.special.log_ndtr(-(u_hi - loc) / sigma) - np.log(epsilon)
    lp = torch.where(ev <= lo, left, torch.where(ev >= hi, right, inner)).sum(-1)
    H = (torch.distributions.Normal(loc, sigma).entropy() + np.log(s) + fldj(loc + sigma * eps)).sum(-1)
    return lp, H


def _torch_dpo(lp, lp_old, gae, alpha, beta):
    """stoix/utils/loss.py:50-65 verbatim."""
    log_diff = lp - lp_old
    ratio = torch.exp(log_diff)
    is_pos = (gae >= 0.0).double()
    r1 = ratio - 1.0
    drift1 = torch.relu(r1 * gae - alpha * torch.tanh(r1 * gae / alpha))
    drift2 = torch.relu(log_diff * gae - beta * torch.tanh(log_diff * gae / beta))
    drift = drift1 * is_pos + drift2 * (1 - is_pos)
    return -(ratio * gae - drift).mean()


def test_categorical_penalty_gradient_matches_autograd():
    rng = np.random.default_rng(1)
    M, A, beta, ent = 96, 7, 3.0, 0.01
    logits = rng.normal(0.0, 1.5, (M, A))
    b_logits = logits + rng.normal(0.0, 0.4, (M, A))
    b_logits[:8] = logits[:8]               # KL = 0 rows
    b_logits[8:12] = logits[8:12] + 2.5     # a shifted copy: the same distribution, KL = 0
    action = rng.integers(0, A, M)
    adv = rng.normal(size=M)
    logp_old = O.categorical_log_prob(logits, action) + rng.normal(0.0, 0.3, M)
    total, dlogits, info = PV.penalty_actor_loss_and_dlogits(logits, b_logits, action, logp_old, adv, beta, ent)

    z = _t(logits, True)
    lp = F.log_softmax(z, -1)
    lpb = F.log_softmax(_t(b_logits), -1)      # behaviour_policy: no gradient
    ratio = torch.exp(lp[torch.arange(M), torch.as_tensor(action)] - _t(logp_old))
    kl_rows = (lpb.exp() * (lpb - lp)).sum(-1)   # b_pi.kl_divergence(pi)
    kl = kl_rows.mean()
    loss_actor = -(ratio * _t(adv) - beta * kl).mean()
    H = -(lp.exp() * lp).sum(-1).mean()
    (loss_actor - ent * H).backward()
    np.testing.assert_allclose(total, (loss_actor - ent * H).item(), rtol=1e-12)
    np.testing.assert_allclose([info["actor_loss"], info["entropy"], info["kl_divergence"]], [loss_actor.item(), H.item(), kl.item()], rtol=1e-12)
    np.testing.assert_allclose(dlogits, z.grad.numpy(), rtol=1e-9, atol=1e-13)
    np.testing.assert_allclose(PV.categorical_kl(b_logits, logits)[:12], 0.0, atol=1e-14)
    assert (PV.categorical_kl(b_logits, logits)[12:] > 0).all()


@pytest.mark.parametrize("kind", [PV.KL_PENALTY, PV.DPO])
def test_tanh_normal_variant_gradient_matches_autograd(kind):
    rng = np.random.default_rng(7)
    M, A, beta, ent, alpha, dbeta = 64, 6, 3.0, 0.001, 2.0, 0.6
    head = rng.normal(0.0, 1.0, (M, 2 * A))
    b_head = head + rng.normal(0.0, 0.3, (M, 2 * A))
    b_head[:8] = head[:8]                 # KL = 0 rows
    action = np.tanh(rng.normal(0.0, 1.5, (M, A)))
    action[:4, 0] = LO + 1e-3 - 1e-4      # beyond the left clip threshold
    action[4:8, 1] = HI - 1e-3 + 1e-4     # beyond the right one
    action[8:10, 2] = LO                  # at the bounds
    action[10:12, 3] = HI
    eps = rng.normal(size=(M, A))
    adv = rng.normal(size=M)
    lp_ref, _ = PC.log_prob_given(head, action, LO, HI)
    logp_old = lp_ref + rng.normal(0.0, 0.3, M)
    total, dhead, info = PV.tanh_variant_actor_loss_and_dhead(kind, head, action, logp_old, adv, ent, eps, LO, HI, b_head, beta, alpha, dbeta)

    th = _t(head, True)
    lp, H = _torch_tanh_normal(th, _t(action), _t(eps), LO, HI)
    if kind == PV.KL_PENALTY:
        A_ = A
        sb = F.softplus(_t(b_head[:, A_:])) + 1e-3
        s = F.softplus(th[:, A_:]) + 1e-3
        # torch's Normal-Normal KL of the base distributions, summed over the Independent dimension
        kl_rows = torch.distributions.kl_divergence(torch.distributions.Normal(_t(b_head[:, :A_]), sb), torch.distributions.Normal(th[:, :A_], s)).sum(-1)
        kl = kl_rows.mean()
        loss_actor = -(torch.exp(lp - _t(logp_old)) * _t(adv) - beta * kl).mean()
        np.testing.assert_allclose(info["kl_divergence"], kl.item(), rtol=1e-12)
        np.testing.assert_allclose(kl_rows.detach().numpy()[:8], 0.0, atol=1e-14)
    else:
        loss_actor = _torch_dpo(lp, _t(logp_old), _t(adv), alpha, dbeta)
    t_total = loss_actor - ent * H.mean()
    t_total.backward()
    np.testing.assert_allclose(total, t_total.item(), rtol=1e-10)
    np.testing.assert_allclose(info["actor_loss"], loss_actor.item(), rtol=1e-10)
    np.testing.assert_allclose(dhead, th.grad.numpy(), rtol=1e-8, atol=1e-12)


def test_dpo_rows_in_all_four_branches():
    rng = np.random.default_rng(3)
    n = 64
    ld = np.concatenate([rng.uniform(0.01, 0.8, n), rng.uniform(-0.8, -0.01, n), rng.uniform(-0.8, -0.01, n), rng.uniform(0.01, 0.8, n)])
    adv = np.concatenate([rng.uniform(0.1, 3.0, n), rng.uniform(0.1, 3.0, n), -rng.uniform(0.1, 3.0, n), -rng.uniform(0.1, 3.0, n)])
    ld[:2], adv[:2] = 0.0, 1.0       # y = 0 exactly: relu'(0) = 0
    adv[n:n + 2] = 0.0               # A = 0 counts as A >= 0
    ratio = np.exp(ld)
    y1 = (ratio - 1) * adv - 2.0 * np.tanh((ratio - 1) * adv / 2.0)
    y2 = ld * adv - 0.6 * np.tanh(ld * adv / 0.6)
    pos = adv >= 0
    assert (pos & (y1 > 0)).any() and (pos & (y1 <= 0)).any() and (~pos & (y2 > 0)).any() and (~pos & (y2 <= 0)).any()
    rows, d = PV.dpo_rows(ld, adv, 2.0, 0.6)
    t_ld = _t(ld, True)
    loss = _torch_dpo(t_ld, _t(np.zeros_like(ld)), _t(adv), 2.0, 0.6)
    loss.backward()
    np.testing.assert_allclose(rows.mean(), loss.item(), rtol=1e-12)
    np.testing.assert_allclose(d / ld.size, t_ld.grad.numpy(), rtol=1e-10, atol=1e-15)


def test_tanh_normal_kl_is_the_base_normal_kl():
    """KL is invariant under the shared affine-tanh bijection: a Monte-Carlo estimate in ACTION space (log-densities of the
    squashed distributions, no clipping) agrees with the closed form."""
    rng = np.random.default_rng(5)
    hp, hq = np.array([[0.3, -0.2, 0.1, 0.4]]), np.array([[0.1, 0.2, -0.3, 0.2]])
    kl, _ = PV.tanh_normal_kl(hp, hq)
    A = 2
    mp, sp = hp[0, :A], np.logaddexp(hp[0, A:], 0) + 1e-3
    mq, sq = hq[0, :A], np.logaddexp(hq[0, A:], 0) + 1e-3
    u = mp + sp * rng.normal(size=(400000, A))
    a = np.tanh(u)

    def log_density(a, m, s):
        x = np.arctanh(a)
        return (-0.5 * ((x - m) / s) ** 2 - np.log(s) - 0.5 * np.log(2 * np.pi) - np.log1p(-a * a)).sum(-1)

    mc = (log_density(a, mp, sp) - log_density(a, mq, sq)).mean()
    assert abs(mc - kl[0]) < 5e-3, (mc, kl[0])


def test_configs_compose_and_aliases_resolve():
    import importlib

    from stoix_b200.config import compose
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_dpo_continuous", ["arch.total_num_envs=1024"], config_dir="default/anakin")
    assert cfg.env.env_name == "synthetic_continuous"
    s = cfg.system
    assert (s.system_name, s.alpha, s.beta, s.ent_coef, s.vf_coef, s.rollout_length, s.decay_learning_rates) == ("ff_dpo", 2.0, 0.6, 0.001, 1.0, 16,
                                                                                                                 False)
    for key in ("reward_scale", "kl_penalty_coef", "normalize_observations"):
        assert s.get(key, None) is None
    cfg.num_devices, cfg.rank = 1, 0
    check_total_timesteps(cfg, quiet=True)
    assert compose("default_ff_ppo", [], config_dir="default/anakin").system.kl_penalty_coef == 3.0
    assert compose("default_ff_ppo_continuous", [], config_dir="default/anakin").system.kl_penalty_coef == 3.0
    for name in ("ff_ppo_penalty", "ff_ppo_penalty_continuous", "ff_dpo_continuous"):
        impl = importlib.import_module(f"stoix_b200.systems.ppo.anakin.{name}")
        assert importlib.import_module(f"stoix.systems.ppo.anakin.{name}") is impl
        for fn in ("get_learner_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
            assert callable(getattr(impl, fn))
    from stoix.utils import loss

    assert callable(loss.ppo_penalty_loss) and callable(loss.dpo_loss)


def test_ppo_variant_struct_layout():
    from stoix_b200 import _lib

    S = _lib.StxPpoVariant
    assert ctypes.sizeof(S) == 8 + 4 * 4
    assert [getattr(S, f).offset for f in ("behaviour", "kind", "kl_coef", "dpo_alpha", "dpo_beta")] == [0, 8, 12, 16, 20]
    assert (_lib.STX_PPO_KL_PENALTY, _lib.STX_PPO_DPO) == (1, 2)
