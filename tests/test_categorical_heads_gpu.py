"""The categorical samplers and heads on the GPU against tests/categorical_reference.py.

* stx_categorical's Gumbel-max draws, action for action, from the restated Philox stream: A from 1 to 1024, seeds with a high word,
  calls crossing 2^32; the same for the fused bf16 rollout, whose logits are recomputed with the per-step bf16 forward.
* MPO's inverse-CDF bootstrap draws, draw for draw, including a launch whose draws fall in the fp32 remainder of the running sum.
* Log-prob, entropy, KL and the fp32 PPO head gradients against fp64 on the edge families (saturated rows, improbable taken actions,
  exact ties, offsets up to 1e5).

Error bounds.  An action must equal the fp64 argmax wherever the two best fp64 scores differ by more than 2^-20 max(1, |z|, |noise|)
of those two (the fp32 noise -logf(-logf(u)) and the sum z + noise carry a few ulp at that magnitude); inside that band it must be
one of the near-tied actions, and such rows stay below 1e-3 of the launch.  An MPO draw must equal the fp64 inverse CDF unless u lies
within 2^-21 of a cumulative boundary (the fp32 running sum of up to 32 expf terms).  Log-prob and entropy are held to
2 ulp32(max_j |z_j|) + max(2^-21, (A + 4) 2^-24) max(1, |ref|).  The second term is the rounding of an fp32 sum over A terms.  The
first is the absorption of the low bits of logf(sum) in lse = zmax + logf(sum) at large offsets (ulp(1e5) = 2^-7), which shifts every log-probability of the row by up to half an ulp of zmax; the kernels keep that
form so that the sampler, the fused rollout, K3a and the loss rows agree bit for bit.  The same shift enters the gradients and the KL
through p_j and log p_j, and their bounds carry it explicitly."""
import numpy as np
import pytest
import torch

from tests import categorical_reference as R

pytestmark = pytest.mark.gpu

SEED_HI = 0x9E3779B97F4A7C15     # a seed whose high word is not zero
CALL_WRAP = (1 << 32) - 2


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device="cuda:0")


def _np(t):
    return t.detach().cpu().numpy()


def _ops():
    from stoix_b200 import ops
    return ops


def _sum_rel(A):
    """Relative rounding of an fp32 sum over A terms (A - 1 additions, expf / logf and a product): 2^-21 up to A = 4."""
    return max(2.0 ** -21, (A + 4) * 2.0 ** -24)


def _logp_tol(z32, ref):
    return 2.0 * R.ulp32(np.abs(z32).max(axis=1)) + _sum_rel(z32.shape[1]) * np.maximum(1.0, np.abs(ref))


def _assert_within(got, ref, tol, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = np.flatnonzero(~(err <= tol))
    assert bad.size == 0, (f"{what}: {bad.size} rows outside the bound, rows {bad[:6].tolist()}: got {np.asarray(got)[bad[:6]].tolist()} "
                           f"ref {ref[bad[:6]].tolist()} bound {tol[bad[:6]].tolist()}")
    return float((err / tol).max()) if err.size else 0.0


def _sample_logits(E, A, rng):
    z = (rng.standard_normal((E, A)) * 2.0).astype(np.float32)
    z[::3] = 0.0                       # every third row all equal: the draw is the noise alone
    return z


# E * ceil(A / 4) stays below ~0.6M counters per call
@pytest.mark.parametrize("A,E", [(1, 70000), (2, 257), (3, 255), (4, 1), (5, 70000), (8, 257), (9, 70000), (16, 255), (17, 257),
                                 (32, 70000), (33, 255), (255, 257), (255, 1), (1024, 255), (1024, 257)])
def test_gumbel_draws_match_philox_restatement(A, E):
    ops = _ops()
    rng = np.random.default_rng(A * 100003 + E)
    z = _sample_logits(E, A, rng)
    zt = _t(z)
    near = 0
    draws = [(SEED_HI, 0, None), (7, 5, None)] + [(SEED_HI, CALL_WRAP, k) for k in range(4)]
    for seed, offset, k in draws:
        ctr = None if k is None else torch.tensor([k], dtype=torch.int64, device="cuda:0")
        a, lp, ent = ops.categorical(zt, seed=seed, offset=offset, dev_counter=ctr, want_entropy=True)
        call = offset + (k or 0)
        ref = R.gumbel_actions(z, seed, call)
        got = _np(a)
        near += R.check_gumbel_actions(got, ref, f"A={A} E={E} seed={seed:#x} call={call:#x}")
        z64 = z.astype(np.float64)
        _assert_within(_np(lp), R.categorical_log_prob(z64, got), _logp_tol(z, R.categorical_log_prob(z64, got)), "sampled log_prob")
        _assert_within(_np(ent), R.categorical_entropy(z64), _logp_tol(z, R.categorical_entropy(z64)), "entropy")
        if k is not None:  # offset + counter is the call: the same draws as offset + k with no counter
            a2, lp2, _ = ops.categorical(zt, seed=seed, offset=offset + k)
            assert torch.equal(a, a2) and torch.equal(lp, lp2)
    print(f"A={A} E={E}: {len(draws) * E} draws, {near} near ties")
    if A >= 255:  # wide rows: the top groups of actions are drawn too (the noise does not wrap below 1024 actions)
        a, _, _ = ops.categorical(_t(np.zeros((4096, A), np.float32)), seed=SEED_HI, offset=3)
        got = _np(a)
        R.check_gumbel_actions(got, R.gumbel_actions(np.zeros((4096, A), np.float32), SEED_HI, 3), f"A={A} equal logits")
        assert got.max() >= A - 8


def test_categorical_refuses_more_than_1024_actions():
    """Past 1024 actions the 8-bit group field of the counter would repeat the noise of actions 0..3 (tests/test_categorical_reference.py):
    stx_categorical refuses the shape instead of drawing from a biased distribution."""
    ops = _ops()
    z = torch.zeros(4, 1025, device="cuda:0")
    with pytest.raises(ops.StxError, match="A=1025"):
        ops.categorical(z, seed=1)
    with pytest.raises(ops.StxError, match="A=1025"):
        ops.categorical(z, action=torch.zeros(4, dtype=torch.int32, device="cuda:0"))
    a, _, _ = ops.categorical(torch.zeros(4, 1024, device="cuda:0"), seed=1)
    assert 0 <= int(a.min()) and int(a.max()) < 1024


@pytest.mark.parametrize("A", [1, 2, 3, 8, 32])
def test_log_prob_and_entropy_on_edge_rows(A):
    """Score mode (the taken action given: the most and the least probable of each row) and sample mode, against fp64."""
    ops = _ops()
    z, act = R.edge_rows(A, np.random.default_rng(A))
    z64 = z.astype(np.float64)
    _, lp, ent = ops.categorical(_t(z), action=_t(act, torch.int32), want_entropy=True)
    ref_lp, ref_h = R.categorical_log_prob(z64, act), R.categorical_entropy(z64)
    r1 = _assert_within(_np(lp), ref_lp, _logp_tol(z, ref_lp), f"A={A} log_prob (score)")
    r2 = _assert_within(_np(ent), ref_h, _logp_tol(z, ref_h), f"A={A} entropy")
    a, lps, ents = ops.categorical(_t(z), seed=SEED_HI, offset=CALL_WRAP + 1, want_entropy=True)
    got = _np(a)
    assert got.min() >= 0 and got.max() < A
    ref_lps = R.categorical_log_prob(z64, got)
    # Gumbel noise lies in [-log(-log 2^-24), -log(-log(1 - 2^-24))] = [-2.8, 16.6]: no draw is further below the best logit
    assert (ref_lps > -(19.5 + np.log(A))).all(), "the sampler drew an action its noise cannot reach"
    r3 = _assert_within(_np(lps), ref_lps, _logp_tol(z, ref_lps), f"A={A} log_prob (sample)")
    assert torch.equal(ents, ent)
    print(f"A={A}: {len(z)} rows, worst error / bound: log_prob {r1:.3f}, entropy {r2:.3f}, sampled log_prob {r3:.3f}")


def _actor(rng, D, A):
    from oracle import ppo_oracle as O

    p = O.init_mlp(rng, [D, 256, 256, A], 1.0)
    for i in range(3):
        p.b[i] = rng.standard_normal(p.b[i].shape) * 0.1
    p.W[-1] = rng.standard_normal(p.W[-1].shape) * 0.3
    if A > 1:  # saturated rows: the other actions sit 30, 90 and 110 below action 0; column 1 swings widely, so some rows are open
        p.b[-1] = -np.array([0.0] + [30.0, 90.0, 110.0] * 5)[:A]
        p.W[-1][:, 1] *= 30.0
    return p


@pytest.mark.parametrize("E", [64, 8704])
@pytest.mark.parametrize("A", [1, 2, 5, 16])
def test_fused_rollout_draws_match_philox_restatement(A, E):
    """stx_tc_rollout_synth's actions and log-probs against the reference on the logits of each step, recomputed from the
    trajectory's bf16 observations with the per-step bf16 forward (bit-identical to the fused chain); calls cross 2^32."""
    ops = _ops()
    D, T, cat_seed, cat_offset = 16, 4, SEED_HI, (1 << 32) - 3
    rng = np.random.default_rng(A * 7 + E)
    spec = ops.MlpSpec((D, 256, 256, A))
    params = _t(_actor(rng, D, A).flat())
    shadow = ops.cast_bf16(params)
    dev = "cuda:0"
    obs = torch.zeros(T + 1, E, D, dtype=torch.bfloat16, device=dev)
    obs[0] = _t(rng.standard_normal((E, D))).to(torch.bfloat16)
    z = lambda dt: torch.zeros(T, E, dtype=dt, device=dev)
    next_obs = torch.zeros(T, E, D, dtype=torch.bfloat16, device=dev)
    action, log_prob, reward = z(torch.int32), z(torch.float32), z(torch.float32)
    done, trunc, term = z(torch.uint8), z(torch.uint8), z(torch.uint8)
    ep_ret, ep_len = z(torch.float32), z(torch.int32)
    run_ret, run_len = torch.zeros(E, device=dev), torch.zeros(E, dtype=torch.int32, device=dev)
    env_ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    cat_ctr = torch.ones(1, dtype=torch.int64, device=dev)
    ops.tc_rollout_synth(spec, params, shadow, obs, next_obs, action, log_prob, reward, done, trunc, ep_ret, ep_len, term, run_ret, run_len,
                         11, 0, env_ctr, 0.05, 0.05, cat_seed, cat_offset, cat_ctr)
    torch.cuda.synchronize()
    near = 0
    for t in range(T):
        logits = ops.mlp_forward(spec, params, obs[t].contiguous(), precision=ops.STX_PREC_BF16, params_bf16=shadow)
        zl = _np(logits)
        call = cat_offset + t + 1
        got = _np(action[t])
        near += R.check_gumbel_actions(got, R.gumbel_actions(zl, cat_seed, call), f"A={A} E={E} step {t} call={call:#x}")
        z64 = zl.astype(np.float64)
        ref = R.categorical_log_prob(z64, got)
        _assert_within(_np(log_prob[t]), ref, _logp_tol(zl, ref), f"A={A} E={E} step {t} log_prob")
        # the per-step head on the same logits: the same draw and the same bits
        a2, lp2, _ = ops.categorical(logits, seed=cat_seed, offset=call)
        assert torch.equal(a2, action[t]) and torch.equal(lp2, log_prob[t])
    if A > 1:
        gaps = np.sort(zl, axis=1)[:, -1] - np.sort(zl, axis=1)[:, -2]
        print(f"A={A} E={E}: {near} near ties; top-two logit gap {gaps.min():.2f} .. {gaps.max():.2f}")
        assert (gaps > 25).any(), "the actor should give saturated rows"


def _mpo_call(ops, logits_b, N, seed, call, stochastic=True, D=1):
    M, A = logits_b.shape
    dev = "cuda:0"
    lb = _t(logits_b)
    obs = torch.zeros(M, D, device=dev)
    act_out = torch.full((N, M), -1, dtype=torch.int32, device=dev)
    xq = torch.empty(((A + N + 1) * M, D + A), device=dev)
    log_rho, r, d = (torch.empty(M, device=dev) for _ in range(3))
    ops.mpo_sample_actions(obs, lb, lb, torch.zeros(M, dtype=torch.int32, device=dev), torch.zeros(M, device=dev), torch.zeros(M, device=dev),
                           torch.zeros(M, dtype=torch.uint8, device=dev), N, xq, log_rho, r, d, 0.99, 1.0, stochastic=stochastic, seed=seed,
                           dev_counter=torch.tensor([call], dtype=torch.int64, device=dev), act_out=act_out)
    torch.cuda.synchronize()
    got = _np(act_out).astype(np.int64)
    del xq
    return got


def _check_mpo_draws(got, ref, what):
    A = ref.prob.shape[1]
    assert got.min() >= 0 and got.max() < A, f"{what}: action out of range"
    p_got = np.take_along_axis(ref.prob, got.T, axis=1).T
    zero = np.argwhere(p_got < 1e-30)
    assert len(zero) == 0, (f"{what}: {len(zero)} draws took an action of fp64 probability below 1e-30: (n, i) {zero[:6].tolist()}, "
                            f"actions {got[tuple(zero[:6].T)].tolist()}, u {ref.u[tuple(zero[:6].T)].tolist()}")
    far = ref.distance > 2.0 ** -21
    bad = np.argwhere(far & (got != ref.action))
    assert len(bad) == 0, (f"{what}: {len(bad)} draws differ from the fp64 inverse CDF away from a boundary: (n, i) {bad[:6].tolist()}, "
                           f"kernel {got[tuple(bad[:6].T)].tolist()} reference {ref.action[tuple(bad[:6].T)].tolist()}")
    return int((~far).sum())


@pytest.mark.parametrize("A", [2, 3, 7, 32])
def test_mpo_draws_match_inverse_cdf(A):
    """Bootstrap draws of ff_mpo (stochastic) draw for draw, on rows whose last action has logit -200 (fp32 probability 0) and on
    open rows; the mode (stochastic=False) is the first maximum on rows with exact ties."""
    ops = _ops()
    rng = np.random.default_rng(A)
    M, N, call, seed = 1024, 256, (1 << 32) + 3, SEED_HI
    zb = (rng.standard_normal((M, A)) * 2.0).astype(np.float32)
    zb[::2, -1] = -200.0
    got = _mpo_call(ops, zb, N, seed, call)
    ref = R.mpo_draws(zb, seed, call, N, M)
    n_edge = _check_mpo_draws(got, ref, f"A={A}")
    print(f"A={A}: {N * M} draws, {n_edge} within 2^-21 of a boundary")
    # the mode: ties at the maximum (signed zeros included) resolve to the first
    zm = zb.copy()
    if A >= 2:
        zm[1::4, 0], zm[1::4, A - 1] = 5.0, 5.0
        zm[2::4, :] = 0.0
        zm[3::4, 0], zm[3::4, 1] = -0.0, 0.0
        zm[3::4, 2:] = -1.0
    mode = _mpo_call(ops, zm, 1, seed, call, stochastic=False)
    np.testing.assert_array_equal(mode[0], np.argmax(zm.astype(np.float64), axis=1))


def test_mpo_remainder_never_draws_an_impossible_action():
    """4.2M draws of a seed whose u01 values reach past the fp32 running sum of their rows: those draws fall in the remainder of the
    inverse CDF.  The last action of every row has logit -200; a remainder draw must go to the last action the policy can take."""
    ops = _ops()
    case = R.mpo_remainder_case()
    ref = R.mpo_draws(case.logits, case.seed, case.call, case.N, case.M)
    hit = np.argwhere(ref.u >= np.float32(R.U_HIGH))
    assert len(hit) >= 2, "the remainder case needs draws past the fp32 sum"
    got = _mpo_call(ops, case.logits, case.N, case.seed, case.call)
    print(f"remainder draws (n, i) {hit.tolist()}: kernel actions {got[tuple(hit.T)].tolist()}, u {ref.u[tuple(hit.T)].tolist()}, "
          f"fp32 sums {ref.sum32[hit[:, 1]].tolist()}")
    _check_mpo_draws(got, ref, "remainder case")
    np.testing.assert_array_equal(got[tuple(hit.T)], ref.action32[tuple(hit.T)])


RATIOS = (0.5, 1.0, 1.1, 1.5)   # below, inside (twice) and above the clip band [0.8, 1.2]
ADVS = (1.5, -2.5, 0.7, -0.3, 2.0)


def _head_inputs(A, rng):
    z, act = R.edge_rows(A, rng)
    z64 = z.astype(np.float64)
    n = len(z)
    ratio = np.array([RATIOS[i % 4] for i in range(n)])
    adv = np.array([ADVS[i % 5] for i in range(n)])
    logp_old = (R.categorical_log_prob(z64, act) - np.log(ratio)).astype(np.float32)
    return z, act, logp_old, adv.astype(np.float32)


def _dlogits_bound(z, dlogp, ce, extra=0.0):
    """rtol 1e-5, atol 2^-20 max|adv| / mb (the fp32 roundings of p near 1), plus the lse shift delta = 2 ulp32(max|z|) of the row
    and the rounding of its sum of exponentials, carried through p_j (relative delta), log p_j (absolute delta) and the ratio
    (relative delta)."""
    z64 = z.astype(np.float64)
    lp = R.log_softmax(z64)
    p = np.exp(lp)
    H = -(p * lp).sum(1, keepdims=True)
    delta = 2.0 * R.ulp32(np.abs(z64).max(1, keepdims=True)) + _sum_rel(z.shape[1])
    return delta * (np.abs(dlogp)[:, None] * (1.0 + 2.0 * p) + ce * p * (np.abs(lp + H) + 3.0)) + extra


@pytest.mark.parametrize("A", [1, 2, 3, 8, 31, 32])
def test_ppo_head_grads_on_edge_rows(A):
    """CategoricalRow of the fp32 minibatch kernels (ops.ppo_head_grads, ClipLoss) and the KL-penalty head against fp64: ratios
    below, inside and above the clip band, taken actions down to log-probability -1e4, saturated and tied rows, offsets to 1e5."""
    ops = _ops()
    rng = np.random.default_rng(100 + A)
    z, act, logp_old, adv = _head_inputs(A, rng)
    mb = len(z)
    z64 = z.astype(np.float64)
    atol = 2.0 ** -20 * np.abs(adv).max() / mb
    zeros = _t(np.zeros(mb, np.float32))
    d = torch.zeros(mb, A, device="cuda:0")
    metrics = torch.zeros(8, device="cuda:0")
    ops.ppo_head_grads(_t(z), None, None, _t(act, torch.int32), _t(logp_old), zeros, _t(adv), zeros, None, 0.2, 0.01, 0.5, d, None, metrics)
    _, ref, _ = R.ppo_clip_head(z64, act, logp_old.astype(np.float64), adv.astype(np.float64), 0.2, 0.01)
    ratio = np.exp(R.categorical_log_prob(z64, act) - logp_old.astype(np.float64))
    l1, l2 = ratio * adv, np.clip(ratio, 0.8, 1.2) * adv
    dlogp = np.where((l1 < l2) | ((ratio >= 0.8) & (ratio <= 1.2)), -adv * ratio, 0.0) / mb
    assert (dlogp == 0).any() and (dlogp != 0).any(), "both the clipped and the unclipped branch"
    tol = 1e-5 * np.abs(ref) + atol + _dlogits_bound(z, dlogp, 0.01 / mb)
    err = np.abs(_np(d).astype(np.float64) - ref)
    bad = np.argwhere(~(err <= tol))
    assert bad.size == 0, f"A={A} clip head: {len(bad)} entries out of bound, (row, j) {bad[:6].tolist()}, err {err[tuple(bad[:6].T)].tolist()}"
    print(f"A={A} clip head: {mb} rows, worst error / bound {float((err / tol).max()):.3f}")

    # KL penalty: behaviour logits from other edge rows, so KL(behaviour || pi) reaches 1e4
    beh = z[rng.permutation(mb)]
    d2, _ = ops.ppo_penalty_head_grads(_t(z), None, _t(beh), _t(act, torch.int32), _t(logp_old), _t(adv), None, 0.7, 0.01)
    _, ref2, _ = R.ppo_penalty_head(z64, beh.astype(np.float64), act, logp_old.astype(np.float64), adv.astype(np.float64), 0.7, 0.01)
    pb = np.exp(R.log_softmax(beh.astype(np.float64)))
    p = np.exp(R.log_softmax(z64))
    ck = 0.7 / mb
    extra = ck * (2.0 * R.ulp32(np.abs(beh).max(1, keepdims=True)) * pb + 2.0 * R.ulp32(np.abs(z).max(1, keepdims=True)) * p)
    tol2 = 1e-5 * np.abs(ref2) + atol + _dlogits_bound(z, -adv * ratio / mb, 0.01 / mb, extra)
    err2 = np.abs(_np(d2).astype(np.float64) - ref2)
    bad = np.argwhere(~(err2 <= tol2))
    assert bad.size == 0, f"A={A} penalty head: {len(bad)} entries out of bound, (row, j) {bad[:6].tolist()}, err {err2[tuple(bad[:6].T)].tolist()}"
    print(f"A={A} penalty head: worst error / bound {float((err2 / tol2).max()):.3f}")


@pytest.mark.parametrize("A", [1, 2, 3, 8, 31, 32])
def test_categorical_kl_on_edge_rows(A):
    """KL(p || q) of identical rows is exactly 0; otherwise it matches fp64 within the lse shifts of both rows and is never below
    -(2^-22 max(1, max|log p|) + those shifts)."""
    ops = _ops()
    rng = np.random.default_rng(200 + A)
    z, _ = R.edge_rows(A, rng)
    zt = _t(z)
    assert (_np(ops.categorical_kl(zt, zt)) == 0).all()
    near = (z + rng.standard_normal(z.shape).astype(np.float32) * np.float32(0.01)).astype(np.float32)
    for q in (z[rng.permutation(len(z))], near, z[::-1].copy()):
        kl = _np(ops.categorical_kl(zt, _t(q))).astype(np.float64)
        ref = R.categorical_kl(z.astype(np.float64), q.astype(np.float64))
        shift = 2.0 * (R.ulp32(np.abs(z).max(1)) + R.ulp32(np.abs(q).max(1)))
        lp = R.log_softmax(z.astype(np.float64))
        floor = 2.0 ** -22 * np.maximum(1.0, np.abs(np.where(np.exp(lp) > 0, lp, 0.0)).max(1)) + shift
        assert (kl >= -floor).all(), f"A={A}: KL below its floor at rows {np.flatnonzero(kl < -floor)[:6].tolist()}"
        p = np.exp(lp)
        mass = np.maximum(1.0, (p * np.abs(lp - R.log_softmax(q.astype(np.float64)))).sum(1))
        _assert_within(kl, ref, shift * (1.0 + np.abs(ref)) + _sum_rel(A) * mass, f"A={A} KL")
