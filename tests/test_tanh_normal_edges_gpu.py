"""The tanh-Normal head kernels and the SAC loss heads on the GPU at their branch edges and far tails, against the fp64 reference of
tests/tanh_normal_reference.py.

Tolerance: every element must lie within twice the reference's error bound (`Err.e`), which is derived from the fp32 operations
of the kernel's path (each + - * / adds 2^-24 of its result, each CUDA math function its documented ulp, and inputs' bounds pass
through the derivative; see the reference's docstring).  On well-conditioned elements that is a few 1e-7 relative; it widens only
where the operation itself is ill-conditioned in fp32: by z^2 2^-24 in the Normal density, 1/(1 - x^2) in atanh next to the clip
band, 1/sigma where sigma = min_scale, and log_prob's absolute error in the PPO ratio.  The factor 2 covers the second-order
terms of the first-order bound.  A Mills ratio computed as exp(-z^2/2 - log sqrt(2 pi) - log Phi(z)) beyond z = -90.5 misses
this bound (its relative error is near z^2 2^-24: 5e-4 at z = -200, 6e-2 at z = -1500).

Branches are discrete, so they are never given a tolerance: a given action's branch is the fp32 comparison the reference makes;
a sampled action's branch is that of the kernel's fp32 action, which is first checked against the reference's action.

The SAC loss heads (`stx_sac_actor_seed`, `stx_sac_q_loss`, `stx_sac_alpha_grad`) run on dyadic data whose sums are exact in any
order, so dq1, dq2, the alpha gradient and all eight metrics slots must equal the reference bit for bit."""
import numpy as np
import pytest
import torch

from tests import ppo_continuous_oracle as PC
from tests import tanh_normal_reference as R

pytestmark = pytest.mark.gpu

BOUNDS = [(-1.0, 1.0), (-2.0, 0.5)]
A_LIST = [1, 3, 4, 5, 8, 17]
RAWS = [-80.0, -20.0, 0.0, 20.0, 80.0]
# z of the clipped tails: far left (the erfcx branch of log Phi, t = -z / sqrt 2 >= 3), both sides of t = 3 and of the Mills
# ratio's switch to sqrt(2/pi) / erfcx(t) at t = 64 (z = -90.5), and far right
Z_TAIL = [-3000.0, -1500.0, -545.0, -200.0, -100.0, -91.0, -90.0, -50.0, -10.0, -4.3, -4.2426, -4.2, -1.0, 0.0, 3.0, 10.0, 40.0]
Z_MODERATE = [-10.0, -4.3, -4.2426, -4.2, -1.0, 0.0, 3.0, 10.0]


def _dev(x, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), device="cuda").to(dt)


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _within(got, ref: R.Err, what: str, factor: float = 2.0):
    got = np.asarray(got, np.float64)
    tol = factor * ref.e + 2.0 ** -40 * np.abs(ref.v)
    diff = np.abs(got - ref.v)
    bad = ~(diff <= tol)
    if bad.any():
        k = np.argsort(-np.nan_to_num(diff / np.maximum(tol, 1e-300), nan=np.inf).ravel())[:5]
        rows = [(np.unravel_index(i, got.shape), got.ravel()[i], ref.v.ravel()[i], diff.ravel()[i] / max(abs(ref.v.ravel()[i]), 1e-300),
                 tol.ravel()[i]) for i in k]
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} outside the bound; worst (index, got, ref, rel err, tol): {rows}")


def _sigma(raw):
    return np.logaddexp(np.asarray(raw, np.float64), 0.0) + float(np.float32(1e-3))


def _ulp_step(x, n):
    x = np.float32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, np.float32(np.inf if n > 0 else -np.inf))
    return x


def _given_grid(M, A, lo_b, hi_b, seed, z_list=Z_TAIL, raws=RAWS):
    """(head (M, 2A), action (M, A)) fp32: every element one case of the grid, cycled over the (row, dim) slots.
    Cases: the thresholds lo / hi exactly, one and two ulp either side, min and max exactly; the clipped tails at each z of
    z_list for each raw of RAWS (so sigma = min_scale exactly and the sigmoid is 0 or 1); and interior actions."""
    g = R.geometry(lo_b, hi_b)
    rng = np.random.default_rng(seed)
    cases = []
    for a in (g.lo, g.hi):
        for n in (-2, -1, 0, 1, 2):
            cases.append(("edge", _ulp_step(a, n), None))
    cases += [("edge", np.float32(lo_b), None), ("edge", np.float32(hi_b), None)]
    for z in z_list:
        for raw in [r for r in raws if abs(r) < 50] if abs(z) > 600 else raws:
            cases.append(("left", z, raw))
            cases.append(("right", z, raw))
    cases += [("interior", None, None)] * 8
    n = M * A
    order = np.arange(n) % len(cases)
    rng.shuffle(order)
    loc, raw, act = np.zeros(n), np.zeros(n), np.zeros(n, np.float32)
    for k, c in enumerate(order):
        kind, p, r = cases[c]
        if kind == "edge":
            loc[k], raw[k], act[k] = rng.normal(0.0, 2.0), rng.normal(0.0, 2.0), p
        elif kind == "interior":
            loc[k], raw[k] = rng.normal(0.0, 2.0), rng.normal(0.0, 2.0)
            act[k] = np.float32(0.5 * (lo_b + hi_b) + 0.5 * (hi_b - lo_b) * np.tanh(rng.normal(0.0, 1.5)))
        elif kind == "left":   # z = (u_lo - loc) / sigma, the event clipped below lo
            raw[k], loc[k] = r, g.u_lo.v - p * _sigma(r)
            act[k] = np.float32(lo_b) if rng.random() < 0.5 else g.lo
        else:                  # z = -(u_hi - loc) / sigma, the event clipped above hi
            raw[k], loc[k] = r, g.u_hi.v + p * _sigma(r)
            act[k] = np.float32(hi_b) if rng.random() < 0.5 else g.hi
    head = np.concatenate([loc.reshape(M, A), raw.reshape(M, A)], 1).astype(np.float32)
    return head, act.reshape(M, A)


def _sample_grid(M, A, lo_b, hi_b, seed):
    """(head, eps) fp32 for the sampling kernels: eps chosen so that the pre-tanh sample lands at the thresholds (u_lo, u_hi,
    and a few ulp of the action either side), deep in the tails, or saturates tanh (|loc + sigma eps| > 9); the rest N(0, 1)."""
    g = R.geometry(lo_b, hi_b)
    head, _ = _given_grid(M, A, lo_b, hi_b, seed, z_list=Z_MODERATE)
    rng = np.random.default_rng(seed + 1)
    loc, raw = head[:, :A].astype(np.float64), head[:, A:].astype(np.float64)
    sig = _sigma(raw)
    s, sh = 0.5 * (hi_b - lo_b), 0.5 * (hi_b + lo_b)
    targets = [np.arctanh((float(_ulp_step(t, n)) - sh) / s) for t in (g.lo, g.hi) for n in (-1, 0, 1)]
    targets += [g.u_lo.v - 1.0, g.u_hi.v + 1.0, -9.5, 9.5, -12.0, 12.0]
    pick = rng.integers(0, len(targets) + 4, size=loc.shape)
    u_t = np.array(targets + [np.nan] * 4)[pick]
    eps = np.where(np.isnan(u_t), rng.normal(size=loc.shape), (u_t - loc) / sig)
    return head, eps.astype(np.float32)


# ------------------------------------------------------------------------------------------------------ log-prob of given actions


@pytest.mark.parametrize("lo_b,hi_b", BOUNDS)
@pytest.mark.parametrize("A", A_LIST)
def test_log_prob_given_at_edges_and_tails(A, lo_b, hi_b):
    """stx_tanh_normal_log_prob per row; the action is a column block of a wider matrix (ld_action > A)."""
    from stoix_b200 import ops

    for M in (1, 389):
        head, act = _given_grid(M, A, lo_b, hi_b, seed=A * 7 + M)
        wide = torch.zeros(M, A + 5, device="cuda")
        wide[:, 3:3 + A] = _dev(act)
        lp = ops.tanh_normal_log_prob(_dev(head), wide[:, 3:3 + A], lo_b, hi_b)
        ref, _, _, br, _ = R.log_prob_given_dim(head[:, :A].astype(np.float64), head[:, A:].astype(np.float64), act, R.geometry(lo_b, hi_b))
        assert (br < 0).any() and (br > 0).any() or M == 1
        _within(_np(lp), ref.sum(-1), f"log_prob M={M} A={A}")


# ------------------------------------------------------------------------------------------------------ sample and backward


@pytest.mark.parametrize("lo_b,hi_b", BOUNDS)
@pytest.mark.parametrize("A", A_LIST)
def test_sample_and_backward_at_edges_and_tails(A, lo_b, hi_b):
    """stx_tanh_normal_sample with injected noise (action, per-row log_prob) and stx_tanh_normal_backward (d loc, d raw), whose
    clipped-tail gradients are the Mills ratio at z = (u_lo - loc) / sigma: the noise sends rows into the tails far from their
    loc, so z reaches -3000 (sigma = min_scale, loc - u_lo = 3)."""
    from stoix_b200 import ops

    g = R.geometry(lo_b, hi_b)
    for M in (1, 389):
        head, eps = _sample_grid(M, A, lo_b, hi_b, seed=A * 11 + M)
        loc, raw = head[:, :A].astype(np.float64), head[:, A:].astype(np.float64)
        wide = torch.zeros(M, A + 9, device="cuda")
        act, lp, _ = ops.tanh_normal_sample(_dev(head), lo_b, hi_b, eps=_dev(eps), action_out=wide[:, 9:])
        a32 = act.cpu().numpy()
        a_ref, lp_ref, br = R.sample_dim(loc, raw, eps.astype(np.float64), g, action32=a32)
        _within(a32, a_ref, f"action M={M} A={A}")
        assert float(wide[:, :9].abs().max()) == 0.0
        _within(_np(lp), lp_ref.sum(-1), f"sample log_prob M={M} A={A}")
        rng = np.random.default_rng(A + M)
        ga = rng.normal(size=(M, A)).astype(np.float32)
        gwide = torch.zeros(M, A + 2, device="cuda")
        gwide[:, 2:] = _dev(ga)
        log_alpha, scale = np.float32(0.3), np.float32(1.0 / max(M, 1))
        d = ops.tanh_normal_backward(_dev(head), _dev(eps), lo_b, hi_b, _dev([log_alpha]), float(scale), gwide[:, 2:])
        gl = float(scale) * R.expf(R.Err(float(log_alpha)))
        d_loc, d_raw = R.backward_dim(loc, raw, eps.astype(np.float64), ga.astype(np.float64), gl, br, g)
        dd = _np(d)
        _within(dd[:, :A], d_loc, f"backward d_loc M={M} A={A}")
        _within(dd[:, A:], d_raw, f"backward d_raw M={M} A={A}")


def test_far_tail_backward_covers_the_mills_range():
    """One dimension per z of Z_TAIL in the left and the right tail, sigma = min_scale and sigma = softplus(0) + min_scale, through
    stx_tanh_normal_backward with only the log-prob term (g_action = 0): d loc = -gl m(z) / sigma."""
    from stoix_b200 import ops

    lo_b, hi_b = -1.0, 1.0
    g = R.geometry(lo_b, hi_b)
    rows = [(side, z, raw) for side in (-1, 1) for z in Z_TAIL for raw in (-80.0, 0.0)]
    M = len(rows)
    loc, raw, eps = np.zeros((M, 1)), np.zeros((M, 1)), np.zeros((M, 1))
    for i, (side, z, r) in enumerate(rows):
        sg = _sigma(r)
        raw[i], loc[i] = r, (g.u_lo.v - z * sg) if side < 0 else (g.u_hi.v + z * sg)
        eps[i] = (((g.u_lo.v - 1.0) if side < 0 else (g.u_hi.v + 1.0)) - float(np.float32(loc[i, 0]))) / sg
    head = np.concatenate([loc, raw], 1).astype(np.float32)
    eps = eps.astype(np.float32)
    act, _, _ = ops.tanh_normal_sample(_dev(head), lo_b, hi_b, eps=_dev(eps))
    a32 = act.cpu().numpy()
    _, _, br = R.sample_dim(head[:, :1].astype(np.float64), head[:, 1:].astype(np.float64), eps.astype(np.float64), g, action32=a32)
    assert np.array_equal(br[:, 0], np.array([s for s, _, _ in rows]))
    d = _np(ops.tanh_normal_backward(_dev(head), _dev(eps), lo_b, hi_b, None, 1.0, None))
    d_loc, d_raw = R.backward_dim(head[:, :1].astype(np.float64), head[:, 1:].astype(np.float64), eps.astype(np.float64), 0.0, R.Err(1.0), br, g)
    _within(d[:, :1], d_loc, "far-tail d_loc")
    _within(d[:, 1:], d_raw, "far-tail d_raw")


@pytest.mark.parametrize("A", [3, 5, 17])
def test_philox_noise_of_sample_and_entropy(A):
    """Philox draws of the sampler (tag "SAC1") and of the entropy estimate (tag "PPOE") against their stream functions; eps_out
    is the noise the kernel used: feeding it back as eps_in gives the same bits."""
    from stoix_b200 import ops

    lo_b, hi_b = -2.0, 0.5
    M = 389
    head, _ = _given_grid(M, A, lo_b, hi_b, seed=A, z_list=Z_MODERATE)
    ctr = torch.tensor([3], dtype=torch.int64, device="cuda")
    act, lp, e = ops.tanh_normal_sample(_dev(head), lo_b, hi_b, seed=2024, offset=4, dev_counter=ctr)
    np.testing.assert_allclose(_np(e), R.philox_normals(2024, M, A, 7, R.TAG_SAC), rtol=0, atol=1e-6)
    act2, lp2, _ = ops.tanh_normal_sample(_dev(head), lo_b, hi_b, eps=e.clone())
    assert torch.equal(act, act2) and torch.equal(lp, lp2)
    a_ref, lp_ref, _ = R.sample_dim(head[:, :A].astype(np.float64), head[:, A:].astype(np.float64), _np(e), R.geometry(lo_b, hi_b),
                                    action32=act.cpu().numpy())
    _within(act.cpu().numpy(), a_ref, "Philox action")
    _within(_np(lp), lp_ref.sum(-1), "Philox log_prob")
    ent, ee = ops.tanh_normal_entropy(_dev(head), lo_b, hi_b, seed=2024, offset=4, dev_counter=ctr, want_eps=True)
    np.testing.assert_allclose(_np(ee), PC.entropy_noise(2024, M, A, 7), rtol=0, atol=1e-6)
    ent2, _ = ops.tanh_normal_entropy(_dev(head), lo_b, hi_b, eps=ee.clone())
    assert torch.equal(ent, ent2)


# ------------------------------------------------------------------------------------------------------ entropy and KL


@pytest.mark.parametrize("lo_b,hi_b", BOUNDS)
@pytest.mark.parametrize("A", A_LIST)
def test_entropy_estimate_with_saturated_tanh(A, lo_b, hi_b):
    """stx_tanh_normal_entropy with injected noise, including |loc + sigma eps| > 9 (tanh saturated in fp32)."""
    from stoix_b200 import ops

    for M in (1, 389):
        head, eps = _sample_grid(M, A, lo_b, hi_b, seed=A * 13 + M)
        ent, _ = ops.tanh_normal_entropy(_dev(head), lo_b, hi_b, eps=_dev(eps))
        h, _, _ = R.entropy_dim(head[:, :A].astype(np.float64), head[:, A:].astype(np.float64), eps.astype(np.float64), R.geometry(lo_b, hi_b))
        _within(_np(ent), h.sum(-1), f"entropy M={M} A={A}")


@pytest.mark.parametrize("A", A_LIST)
def test_normal_kl_over_scale_ratios(A):
    """stx_tanh_normal_kl with sigma_b / sigma from 1e-3 to 1e3 (raw pairs around min_scale and far above it); identical heads give
    KL exactly 0."""
    from stoix_b200 import ops

    rng = np.random.default_rng(A)
    M = 389
    ratios = 10.0 ** rng.uniform(-3.0, 3.0, (M, A))
    sq = 10.0 ** rng.uniform(-2.0, 1.0, (M, A))
    sb = sq * ratios
    ms = float(np.float32(1e-3))
    raw_of = lambda s: np.where(s - ms > 20.0, s - ms, np.log(np.expm1(np.clip(s - ms, 1e-30, 20.0))))
    rq, rb = raw_of(sq), raw_of(sb)
    rq[:, 0], rb[:, 0] = -80.0, np.where(np.arange(M) % 2 == 0, -80.0, 20.0)   # sigma = min_scale on one or both sides
    hq = np.concatenate([rng.normal(0.0, 1.0, (M, A)), rq], 1).astype(np.float32)
    hb = np.concatenate([rng.normal(0.0, 1.0, (M, A)), rb], 1).astype(np.float32)
    kl = _np(ops.tanh_normal_kl(_dev(hb), _dev(hq)))
    ref, _, _ = R.normal_kl_dim(hb[:, :A].astype(np.float64), hb[:, A:].astype(np.float64), hq[:, :A].astype(np.float64),
                                hq[:, A:].astype(np.float64))
    _within(kl, ref.sum(-1), f"KL A={A}")
    assert float(ops.tanh_normal_kl(_dev(hq), _dev(hq)).abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------ PPO head gradients


def _ppo_case(kind, A, lo_b, hi_b, mb, seed):
    rng = np.random.default_rng(seed)
    B = mb + 37
    # sigma >= softplus(0) in the tails: at sigma = min_scale the fp32 rounding of u_lo alone moves z by 1e-3 and log_prob by
    # m(z) 1e-3, which the ratio spreads over the whole row (those tails are covered by the tests above and the far-tail test below)
    head, act_mb = _given_grid(mb, A, lo_b, hi_b, seed, z_list=Z_MODERATE, raws=[0.0, 20.0, 80.0])
    head[:, A:] = np.maximum(head[:, A:], np.float32(0.0))
    idx = rng.permutation(B)[:mb].astype(np.int32)
    action = np.tanh(rng.normal(size=(B, A))).astype(np.float32)
    action[idx] = act_mb
    g = R.geometry(lo_b, hi_b)
    lp, _, _, _, _ = R.log_prob_given_dim(head[:, :A].astype(np.float64), head[:, A:].astype(np.float64), act_mb, g)
    logp_old = np.zeros(B, np.float32)
    logp_old[idx] = (lp.sum(-1).v + rng.normal(0.0, 0.3, mb)).astype(np.float32)
    adv = rng.normal(size=B).astype(np.float32)
    adv[idx[: mb // 4]] = 0.0
    eps = rng.normal(size=(mb, A)).astype(np.float32)
    eps[:, 0] = np.where(rng.random(mb) < 0.3, np.float32(40.0), eps[:, 0])   # saturated tanh in the entropy term
    behaviour = (np.concatenate([head[:, :A], head[:, A:]], 1) + rng.normal(0.0, 0.5, head.shape)).astype(np.float32)
    b_rows = np.zeros((B, 2 * A), np.float32)
    b_rows[idx] = behaviour
    return head, idx, action, logp_old, adv, eps, b_rows


@pytest.mark.parametrize("kind", ["clip", "kl", "dpo"])
@pytest.mark.parametrize("lo_b,hi_b", BOUNDS)
@pytest.mark.parametrize("A", A_LIST)
def test_ppo_head_grads_at_edges(kind, A, lo_b, hi_b):
    """stx_ppo_tanh_normal_head_grads (clip) and stx_ppo_variant_tanh_normal_head_grads (KL penalty, DPO) with injected entropy
    noise, rows through a permutation, mb = 1 and mb = 389 (not a multiple of the 256-thread grid); tails here reach |z| = 10, where
    the ratio exp(log_prob - logp_old) is still well conditioned.  Metrics (actor loss, entropy, advantage or KL means) to the
    sum of the rows' bounds."""
    from stoix_b200 import ops

    for mb in (1, 389):
        head, idx, action, logp_old, adv, eps, b_rows = _ppo_case(kind, A, lo_b, hi_b, mb, seed=A * 17 + mb)
        ent_coef, kl_coef = 0.01, 0.7
        if kind == "clip":
            d, met = ops.ppo_tanh_normal_head_grads(_dev(head), _dev(idx, torch.int32), _dev(action), _dev(logp_old), _dev(adv), None, 0.2,
                                                    ent_coef, lo_b, hi_b, eps_in=_dev(eps))
        else:
            k = ops.STX_PPO_KL_PENALTY if kind == "kl" else ops.STX_PPO_DPO
            d, met = ops.ppo_variant_tanh_normal_head_grads(_dev(head), _dev(idx, torch.int32), k, _dev(action), _dev(logp_old), _dev(adv), None,
                                                            ent_coef, lo_b, hi_b, behaviour=_dev(b_rows), kl_coef=kl_coef, eps_in=_dev(eps))
        dref, loss, ent, kl = R.ppo_head(kind, head, action[idx], logp_old[idx], adv[idx], eps.astype(np.float64), lo_b, hi_b, 0.2, ent_coef,
                                         b_head=b_rows[idx], kl_coef=kl_coef)
        _within(_np(d), dref, f"{kind} d_head mb={mb} A={A}")
        m = _np(met)
        mean = lambda x: R.Err(x.v.mean(), x.e.mean() + 2 * R.U * np.abs(x.v).mean())
        _within(m[0], mean(loss), f"{kind} actor_loss")
        _within(m[1], mean(ent), f"{kind} entropy")
        if kind == "clip":
            _within(m[3], mean(R.Err(adv[idx].astype(np.float64))), "advantages")
        if kind == "kl":
            _within(m[6], mean(kl), "kl_divergence")


def test_ppo_head_grads_far_tail_mills():
    """The given-action Mills derivatives of TanhNormalRow over z in Z_TAIL, one row per launch (mb = 1, A = 1, ent_coef = 0).
    At z = -3000 log_prob is near -4.5e6 and its fp32 rounding alone moves the ratio by tens of percent, so the row's ratio is
    taken from the kernel: with a clip range that contains every ratio and A = 1, metrics slot 0 is -ratio exactly."""
    from stoix_b200 import ops

    lo_b, hi_b = -1.0, 1.0
    g = R.geometry(lo_b, hi_b)
    for side in (-1, 1):
        for z in Z_TAIL:
            for r in (-80.0, 0.0):
                sg = _sigma(r)
                loc = (g.u_lo.v - z * sg) if side < 0 else (g.u_hi.v + z * sg)
                head = np.array([[loc, r]], np.float32)
                act = np.array([[lo_b if side < 0 else hi_b]], np.float32)
                lp, _, _, _, _ = R.log_prob_given_dim(head[:, :1].astype(np.float64), head[:, 1:].astype(np.float64), act, g)
                logp_old = np.array([lp.v[0, 0]], np.float32)
                adv = np.ones(1, np.float32)
                d, met = ops.ppo_tanh_normal_head_grads(_dev(head), None, _dev(act), _dev(logp_old), _dev(adv), None, 3e38, 0.0, lo_b, hi_b,
                                                        eps_in=torch.zeros(1, 1, device="cuda"))
                ratio = -_np(met)[0]
                dref, _, _, _ = R.ppo_head("clip", head, act, logp_old, adv, np.zeros((1, 1)), lo_b, hi_b, 3e38, 0.0, ratio=np.array([ratio]))
                _within(_np(d), dref, f"PPO far tail side={side} z={z} raw={r}")


def test_identical_behaviour_gives_zero_kl():
    """KL penalty with the behaviour head equal to the current head: kl_divergence exactly 0 and d loc free of any KL term."""
    from stoix_b200 import ops

    A, mb = 5, 389
    head, idx, action, logp_old, adv, eps, b_rows = _ppo_case("kl", A, -1.0, 1.0, mb, seed=3)
    b_rows[idx] = head
    d1, met = ops.ppo_variant_tanh_normal_head_grads(_dev(head), _dev(idx, torch.int32), ops.STX_PPO_KL_PENALTY, _dev(action), _dev(logp_old),
                                                     _dev(adv), None, 0.01, -1.0, 1.0, behaviour=_dev(b_rows), kl_coef=0.7, eps_in=_dev(eps))
    assert float(met[6]) == 0.0
    d0, _ = ops.ppo_variant_tanh_normal_head_grads(_dev(head), _dev(idx, torch.int32), ops.STX_PPO_KL_PENALTY, _dev(action), _dev(logp_old),
                                                   _dev(adv), None, 0.01, -1.0, 1.0, behaviour=_dev(b_rows), kl_coef=0.0, eps_in=_dev(eps))
    assert torch.equal(d1[:, :A], d0[:, :A])


# ------------------------------------------------------------------------------------------------------ SAC loss heads, exact


def _dyadic(rng, n, lo, hi, unit=0.125):
    return (rng.integers(int(lo / unit), int(hi / unit) + 1, n) * unit).astype(np.float64)


@pytest.mark.parametrize("M", [1, 1023, 1024, 1025, 5000])
@pytest.mark.parametrize("log_alpha", [0.0, -np.inf])
@pytest.mark.parametrize("flags", [(1.0, True, True), (0.5, False, False), (0.25, True, False)])
def test_sac_loss_heads_exact(M, log_alpha, flags):
    """stx_sac_actor_seed, stx_sac_q_loss and stx_sac_alpha_grad into one metrics buffer, as the learner runs them: q1 == q2 ties on a
    quarter of the rows (the gradient goes to q1), done rows, weight / overwrite / autotune on and off.  alpha = exp(log_alpha) is 1
    or 0, both exact.  The metrics start from dyadic values when M is a power of two (1/M is exact, so every accumulation is), from
    zero otherwise."""
    from stoix_b200 import ops

    weight, overwrite, autotune = flags
    rng = np.random.default_rng(M)
    alpha = float(np.exp(log_alpha))
    q1, q2 = _dyadic(rng, M, -1, 1), _dyadic(rng, M, -1, 1)
    tie = rng.random(M) < 0.25
    q2[tie] = q1[tie]
    lp = _dyadic(rng, M, -4, 4)
    nq1, nq2, nlp = _dyadic(rng, M, -1, 1), _dyadic(rng, M, -1, 1), _dyadic(rng, M, -1, 1)
    reward = _dyadic(rng, M, -1, 1)
    done = rng.random(M) < 0.3
    gamma = 0.5 if M > 1025 else 0.75
    pow2 = (M & (M - 1)) == 0
    m0 = np.array([0.5, -0.25, 1.0, 0.125, -2.0, 4.0, 0.75, -1.5]) if pow2 else np.zeros(8)
    metrics = _dev(m0)
    la = _dev([log_alpha])
    dq1, dq2 = torch.full((M,), 7.0, device="cuda"), torch.full((M,), 7.0, device="cuda")
    ops.sac_actor_seed(_dev(q1), _dev(q2), _dev(lp), la, dq1, dq2, metrics, weight)
    ra1, ra2, mref = R.sac_actor_seed(q1, q2, lp, alpha, m0, weight)
    assert np.array_equal(_np(dq1), ra1) and np.array_equal(_np(dq2), ra2)
    assert (ra1[tie] != 0).all() and (ra2[tie] == 0).all()
    ops.sac_q_loss(_dev(q1), _dev(q2), _dev(nq1), _dev(nq2), _dev(nlp), _dev(reward), _dev(done, torch.uint8), la, gamma, dq1, dq2, metrics, weight)
    rq1, rq2, mref = R.sac_q_loss(q1, q2, nq1, nq2, nlp, reward, done, alpha, gamma, mref, weight)
    assert np.array_equal(_np(dq1), rq1) and np.array_equal(_np(dq2), rq2)
    grad0 = 0.375
    grad = _dev([grad0])
    ops.sac_alpha_grad(_dev(lp), la, -1.5, autotune, grad, grad_weight=0.5, overwrite=overwrite, metrics=metrics, weight=weight)
    gref, mref = R.sac_alpha_grad(lp, alpha, -1.5, autotune, grad0, 0.5, overwrite, mref, weight)
    assert float(grad[0]) == gref
    got = _np(metrics)
    assert np.array_equal(got, mref), (got, mref)
