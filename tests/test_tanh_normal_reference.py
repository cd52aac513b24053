"""tests/tanh_normal_reference.py on the CPU: its values against the existing fp64 oracles (oracle/sac_oracle.py,
tests/ppo_continuous_oracle.py, tests/ppo_variants_oracle.py) at ordinary inputs, its two forms of the Mills ratio against each
other, and its error bound against an fp32 emulation of the Mills ratio in the far tail."""
import numpy as np
import pytest
from scipy.special import erfcx, log_ndtr

from oracle import sac_oracle as S
from tests import ppo_continuous_oracle as PC
from tests import ppo_variants_oracle as PV
from tests import tanh_normal_reference as R

# The reference runs at the kernels' fp32 constants (lo = min + 1e-3f, min_scale = 1e-3f); the oracles use 1e-3 in fp64.  Near
# the clip band u_lo = atanh(lo) moves by about 1e-8 / (1 - lo^2), so ordinary inputs agree to a few 1e-6 relative.
RTOL = 1e-4


def _inputs(seed, M=200, A=5, lo=-1.0, hi=1.0, raw_mean=0.0):
    rng = np.random.default_rng(seed)
    head = rng.normal(0.0, 1.0, (M, 2 * A))
    head[:, A:] += raw_mean
    head = head.astype(np.float32).astype(np.float64)
    eps = rng.normal(size=(M, A)).astype(np.float32).astype(np.float64)
    s, sh = 0.5 * (hi - lo), 0.5 * (hi + lo)
    action = (sh + s * np.tanh(rng.normal(0.0, 1.5, (M, A)))).astype(np.float32)
    action[:10, 0], action[10:20, 1] = np.float32(lo), np.float32(hi)   # in the tails
    return head, eps, action


def test_mills_forms_agree():
    z = np.linspace(-30.0, 30.0, 6001)
    exp_form = np.exp(-0.5 * z * z - R.LOG_SQRT_2PI - log_ndtr(z))
    m = R.mills(R.Err(z)).v
    np.testing.assert_allclose(m, np.sqrt(2.0 / np.pi) / erfcx(-z / np.sqrt(2.0)), rtol=0, atol=0)
    np.testing.assert_allclose(m, exp_form, rtol=1e-12)


@pytest.mark.parametrize("lo,hi", [(-1.0, 1.0), (-2.0, 0.5)])
def test_sample_and_backward_match_sac_oracle(lo, hi):
    head, eps, _ = _inputs(1, lo=lo, hi=hi)
    A = head.shape[1] // 2
    g = R.geometry(lo, hi)
    a, lp, br = R.sample_dim(head[:, :A], head[:, A:], eps, g)
    t = S.head_sample(head, eps, lo, hi)
    np.testing.assert_allclose(a.v, t.action, rtol=1e-7)
    np.testing.assert_array_equal(br, t.branch)
    np.testing.assert_allclose(lp.sum(-1).v, t.log_prob, rtol=RTOL)
    rng = np.random.default_rng(2)
    ga = rng.normal(size=eps.shape)
    d_loc, d_raw = R.backward_dim(head[:, :A], head[:, A:], eps, ga, R.Err(0.25), br, g)
    want = S.head_log_prob_grad(t, np.full(head.shape[0], 0.25), ga, lo, hi)
    np.testing.assert_allclose(np.concatenate([d_loc.v, d_raw.v], -1), want, rtol=RTOL, atol=1e-9)


def test_log_prob_given_entropy_and_kl_match_oracles():
    head, eps, action = _inputs(3)
    A = head.shape[1] // 2
    g = R.geometry(-1.0, 1.0)
    lp, d_loc, d_sig, br, sigma = R.log_prob_given_dim(head[:, :A], head[:, A:], action, g)
    assert (br != 0).any() and (br == 0).any()
    want_lp, want_d = PC.log_prob_given(head, action.astype(np.float64), -1.0, 1.0)
    np.testing.assert_allclose(lp.sum(-1).v, want_lp, rtol=RTOL)
    np.testing.assert_allclose(np.concatenate([d_loc.v, d_sig.v * S.sigmoid(head[:, A:])], -1), want_d, rtol=RTOL, atol=1e-9)
    h, _, _ = R.entropy_dim(head[:, :A], head[:, A:], eps, g)
    np.testing.assert_allclose(h.sum(-1).v, PC.entropy_estimate(head, eps, -1.0, 1.0)[0], rtol=1e-6, atol=1e-8)
    b = head + np.random.default_rng(4).normal(0.0, 0.3, head.shape)
    kl, d_mu, d_sigma = R.normal_kl_dim(b[:, :A], b[:, A:], head[:, :A], head[:, A:])
    want_kl, want_g = PV.tanh_normal_kl(b, head)
    np.testing.assert_allclose(kl.sum(-1).v, want_kl, rtol=1e-7, atol=1e-12)
    np.testing.assert_allclose(np.concatenate([d_mu.v, d_sigma.v * S.sigmoid(head[:, A:])], -1), want_g, rtol=1e-7, atol=1e-12)


@pytest.mark.parametrize("kind", ["clip", "kl", "dpo"])
def test_ppo_heads_match_oracles(kind):
    # The lo / hi difference moves a tail row's log-prob by up to m(z) 1e-5 / sigma, which the ratio carries into every element of
    # the row: sigma near 1.3 keeps that near 1e-4.
    head, eps, action = _inputs(5, raw_mean=1.0)
    M, A = head.shape[0], head.shape[1] // 2
    rng = np.random.default_rng(6)
    lp, _ = PC.log_prob_given(head, action.astype(np.float64), -1.0, 1.0)
    logp_old = lp + rng.normal(0.0, 0.3, M)
    adv = rng.normal(size=M)
    b = head + rng.normal(0.0, 0.2, head.shape)
    d, loss, ent, kl = R.ppo_head(kind, head, action, logp_old, adv, eps, -1.0, 1.0, 0.2, 0.01, b_head=b, kl_coef=0.5)
    if kind == "clip":
        _, want, info = PC.actor_loss_and_dhead(head, action.astype(np.float64), logp_old, adv, 0.2, 0.01, eps, -1.0, 1.0)
    else:
        _, want, info = PV.tanh_variant_actor_loss_and_dhead(PV.KL_PENALTY if kind == "kl" else PV.DPO, head, action.astype(np.float64),
                                                             logp_old, adv, 0.01, eps, -1.0, 1.0, b_head=b, kl_coef=0.5)
    np.testing.assert_allclose(d.v, want, rtol=10 * RTOL, atol=1e-5)
    np.testing.assert_allclose(loss.v.mean(), info["actor_loss"], rtol=RTOL)
    np.testing.assert_allclose(ent.v.mean(), info["entropy"], rtol=1e-7)


def test_philox_normals_is_the_entropy_stream():
    np.testing.assert_array_equal(R.philox_normals(1234, 37, 6, 7, R.TAG_PPO_ENTROPY), PC.entropy_noise(1234, 37, 6, 7))


def _fp32_mills(z32, old):
    """An fp32 emulation of the two forms of mills(z) in log_ndtrf's erfcx branch (t >= 3), with scipy's erfcx rounded to fp32
    standing in for erfcxf."""
    f = np.float32
    t = f(-z32 * f(0.70710678118654752))
    ex = f(erfcx(np.float64(t)))
    if old:
        lnd = f(f(np.log(f(f(0.5) * ex))) - f(t * t))
        return np.float64(f(np.exp(f(f(f(f(-0.5) * z32) * z32) - f(0.9189385332046727)) - lnd)))
    return np.float64(f(f(0.7978845608028654) / ex))


@pytest.mark.parametrize("z", [-100.0, -200.0, -545.0, -1500.0])
def test_mills_bound_separates_the_two_fp32_forms(z):
    """Beyond t = 64 (z < -90.5), at an exact fp32 z, sqrt(2/pi)/erfcx(t) lies inside the reference's bound and the
    exp(-z^2/2 - ... - log Phi) form does not: its error grows as z^2 2^-24."""
    m = R.mills(R.Err(z))
    assert abs(_fp32_mills(np.float32(z), old=False) - m.v) <= m.e
    assert abs(_fp32_mills(np.float32(z), old=True) - m.v) > 4 * m.e


def test_exact_sum_guard():
    R.assert_exact_sums(np.full(1000, 0.125), 2.0 ** -3)
    with pytest.raises(AssertionError):
        R.assert_exact_sums(np.full(3, 0.1), 2.0 ** -3)
    with pytest.raises(AssertionError):
        R.assert_exact_sums(np.full(1 << 22, 7.0), 1.0)
