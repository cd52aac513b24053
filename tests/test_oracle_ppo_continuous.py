"""CPU checks of continuous-action PPO: the oracle's hand-derived actor-loss gradient against torch.autograd (a direct float64
restatement with torch.special.log_ndtr, rows in both clipped tails included), the entry config and its shape derivation,
and the layout of the new C struct."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import ppo_continuous_oracle as PC

LO, HI = -1.0, 1.0


def _torch_actor_loss(head, action, logp_old, adv, eps, clip_eps, ent_coef, minimum, maximum, min_scale=1e-3, epsilon=1e-3):
    A = head.shape[-1] // 2
    loc, raw = head[:, :A], head[:, A:]
    sigma = torch.nn.functional.softplus(raw) + min_scale
    s, sh = (maximum - minimum) / 2.0, (minimum + maximum) / 2.0
    lo, hi = minimum + epsilon, maximum - epsilon
    u_lo, u_hi = np.arctanh((lo - sh) / s), np.arctanh((hi - sh) / s)
    ev = action.clamp(lo, hi)
    u = torch.atanh(((ev - sh) / s).clamp(-1 + 1e-15, 1 - 1e-15))
    fldj = lambda x: 2.0 * (np.log(2.0) - x - torch.nn.functional.softplus(-2.0 * x))
    inner = torch.distributions.Normal(loc, sigma).log_prob(u) - fldj(u) - np.log(s)
    left = torch.special.log_ndtr((u_lo - loc) / sigma) - np.log(epsilon)
    right = torch.special.log_ndtr(-(u_hi - loc) / sigma) - np.log(epsilon)
    lp = torch.where(ev <= lo, left, torch.where(ev >= hi, right, inner)).sum(-1)
    ratio = torch.exp(lp - logp_old)
    loss_actor = -torch.minimum(ratio * adv, ratio.clamp(1 - clip_eps, 1 + clip_eps) * adv).mean()
    us = loc + sigma * eps
    H = (torch.distributions.Normal(loc, sigma).entropy() + np.log(s) + fldj(us)).sum(-1)
    return loss_actor - ent_coef * H.mean(), lp, H


@pytest.mark.parametrize("scale", [1.0, 4.0])
def test_actor_gradient_matches_autograd(scale):
    rng = np.random.default_rng(7 + int(scale))
    M, A = 64, 6
    head = rng.normal(0.0, scale, (M, 2 * A))
    action = np.tanh(rng.normal(0.0, 1.5, (M, A)))
    action[:4, 0] = LO + 1e-3 - 1e-4   # beyond the left clip threshold
    action[4:8, 1] = HI - 1e-3 + 1e-4  # beyond the right one
    action[8:10, 2] = LO                # at the bounds
    action[10:12, 3] = HI
    eps = rng.normal(size=(M, A))
    adv = rng.normal(size=M)
    lp_ref, _ = PC.log_prob_given(head, action, LO, HI)
    logp_old = lp_ref + rng.normal(0.0, 0.3, M)
    total, dhead, info = PC.actor_loss_and_dhead(head, action, logp_old, adv, 0.2, 0.01, eps, LO, HI)

    th = torch.tensor(head, requires_grad=True)
    t_total, t_lp, t_H = _torch_actor_loss(th, torch.tensor(action), torch.tensor(logp_old), torch.tensor(adv), torch.tensor(eps), 0.2, 0.01, LO, HI)
    t_total.backward()
    np.testing.assert_allclose(lp_ref, t_lp.detach().numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(info["entropy"], t_H.detach().numpy().mean(), rtol=1e-10)
    np.testing.assert_allclose(total, t_total.item(), rtol=1e-10)
    np.testing.assert_allclose(dhead, th.grad.numpy(), rtol=1e-8, atol=1e-12)
    # both tails and the band are exercised, and the surrogate is clipped on some rows
    _, t_lp_tails = PC.log_prob_given(head[:12], action[:12], LO, HI)
    assert np.isfinite(t_lp_tails).all()
    ratio = np.exp(lp_ref - logp_old)
    assert ((ratio < 0.8) | (ratio > 1.2)).any() and ((ratio > 0.8) & (ratio < 1.2)).any()


def test_log_prob_of_a_sample_matches_the_sac_oracle():
    from oracle import sac_oracle as S

    rng = np.random.default_rng(3)
    head = rng.normal(0.0, 2.0, (128, 8))
    t = S.head_sample(head, rng.normal(size=(128, 4)), LO, HI)
    lp, _ = PC.log_prob_given(head, t.action, LO, HI)
    np.testing.assert_allclose(lp, t.log_prob, rtol=1e-9, atol=1e-9)


def test_entry_config_composes_and_derives_shapes():
    from stoix_b200.config import compose, instantiate
    from stoix_b200.networks.heads import NormalAffineTanhDistributionHead, ScalarCriticHead
    from stoix_b200.networks.torso import MLPTorso
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_ppo_continuous", ["arch.total_num_envs=1024", "system.rollout_length=32"], config_dir="default/anakin")
    assert cfg.env.env_name == "synthetic_continuous"
    net = cfg.network
    head = instantiate(net.actor_network.action_head, action_dim=6, minimum=-1.0, maximum=1.0)
    assert isinstance(head, NormalAffineTanhDistributionHead) and head.out_dim == 12
    assert isinstance(instantiate(net.critic_network.critic_head), ScalarCriticHead)
    for torso in (net.actor_network.pre_torso, net.critic_network.pre_torso):
        t = instantiate(torso)
        assert isinstance(t, MLPTorso) and list(t.layer_sizes) == [256, 256, 256, 256] and t.activation == "silu"
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    ne, nu, nue = O.derive_shapes(1024, 1, int(cfg.arch.update_batch_size), int(cfg.arch.total_timesteps), 32, int(cfg.arch.num_evaluation))
    assert (int(cfg.arch.num_envs), int(cfg.arch.num_updates), int(cfg.arch.num_updates_per_eval)) == (ne, nu, nue)


def test_tanh_normal_ppo_struct_layout():
    from stoix_b200 import _lib

    S = _lib.StxTanhNormalPpo
    assert ctypes.sizeof(S) == 4 * 8 + 2 * 8 + 4 * 4
    assert [getattr(S, f).offset for f in ("action", "eps_in", "eps_out", "dev_counter", "seed", "offset", "minimum", "maximum", "min_scale")] == \
        [0, 8, 16, 24, 32, 40, 48, 52, 56]
