"""The grid-capped kernels past one wave of their grid (shapes from tests/grid_waves.py), where every block runs its grid-stride
loop more than once and its last trip is ragged: V-MPO's stats, gradient and after-step kernels, the categorical and tanh-Normal MPO
losses, the PPO value faces, the observation statistics and normalisation, and the Polyak update, each against its fp64 oracle at
the tolerances of its in-wave tests, each launched twice for the same bits.  The loss and statistics kernels also run small, large
and small again on one cached scratch: the third run gives the bits of the first."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from oracle import running_statistics as RO
from tests import grid_waves as W
from tests import mpo_oracle as MO
from tests import ppo_variants_oracle as PV
from tests import vmpo_oracle as V

pytestmark = pytest.mark.gpu


def _close(got, want, rtol=1e-5, atol_rel=1e-6, what=""):
    """test_vmpo_gpu's rule: rtol with atol = atol_rel times the largest magnitude of the compared array."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol_rel * max(1.0, float(np.abs(want).max(initial=0.0))), err_msg=what)


def _t(x, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(x))
    return (x if dtype is None else x.to(dtype)).cuda()


def _same_bits(a, b, what):
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), f"{what}: {k} differs between launches"


# ------------------------------------------------------------------------------------------------------------ V-MPO loss ----
VMPO_N = W.VMPO_STATS.shapes
EXTRA_VALUE_ROWS = 9   # d_value rows past N: zero, and past a wave of vmpo_grads_kernel at the largest N


def _vmpo_inputs(kind, per_dim, A, N, seed):
    """Advantages over eta = softplus(0) + 1e-8 so that A / eta over the selected rows spans about 90 (exp: 1e39), with a trend
    along the rows so that block maxima differ by tens; the single largest advantage in row N - 1, in the last block's ragged trip."""
    rng = np.random.default_rng(seed)
    Wd = A if kind == "categorical" else 2 * A
    head = rng.normal(size=(N, Wd)).astype(np.float32)
    head_t = (head + 0.2 * rng.normal(size=(N, Wd))).astype(np.float32)
    if kind == "categorical":
        action = rng.integers(0, A, N).astype(np.int32)
    else:
        action = rng.uniform(-0.95, 0.95, (N, A)).astype(np.float32)
    eta = float(V.dual_value(0.0))
    x = 120.0 * rng.random(N) + 60.0 * np.arange(N) / N
    x[N - 1] = x.max() + 1.0
    adv = (x * eta).astype(np.float32)
    n_dual = 2 if kind == "categorical" else 1 + 2 * (A if per_dim else 1)
    duals = rng.normal(size=n_dual).astype(np.float32)
    duals[0] = 0.0
    value = rng.normal(size=N + EXTRA_VALUE_ROWS).astype(np.float32)
    targets = rng.normal(size=N).astype(np.float32)
    return head, head_t, action, adv, duals, value, targets


def _vmpo_run(kind, per_dim, inputs):
    from stoix_b200 import ops

    head, head_t, action, adv, duals, value, targets = (_t(x) for x in inputs)
    _, mask, count = ops.vmpo_topk(adv)
    d_head, d_value = torch.empty_like(head), torch.full_like(value, 7.0)
    dual_grad, metrics = torch.zeros_like(duals), torch.zeros(9, device="cuda")
    ops.vmpo_loss_grads(kind, head, head_t, action, adv, mask, count, value, targets, duals, d_head, dual_grad, metrics, 0.1, 0.01, 0.005,
                        per_dim=per_dim, d_value=d_value, minimum=-1.0, maximum=1.0, weight=0.5)
    torch.cuda.synchronize()
    return {"d_head": d_head.cpu().numpy(), "d_value": d_value.cpu().numpy(), "dual_grad": dual_grad.cpu().numpy(), "metrics": metrics.cpu().numpy(),
            "mask": mask.cpu().numpy().astype(bool), "K": int(count.item())}


_VMPO_KINDS = [("categorical", True, 7), ("tanh_normal", True, 3), ("tanh_normal", False, 3)]


@pytest.mark.parametrize("kind,per_dim,A", _VMPO_KINDS)
@pytest.mark.parametrize("shape", list(VMPO_N))
def test_vmpo_loss_past_the_grid(kind, per_dim, A, shape):
    N = VMPO_N[shape]
    inputs = _vmpo_inputs(kind, per_dim, A, N, seed=N + A + per_dim)
    head, head_t, action, adv, duals, value, targets = inputs
    got = _vmpo_run(kind, per_dim, inputs)
    tau, mask, K = V.topk_select(adv)
    assert np.array_equal(got["mask"], mask) and got["K"] == K and mask[N - 1]
    want = V.vmpo_loss(kind, head, head_t, action, adv, duals, 0.1, 0.01, 0.005, per_dim, mask=mask)
    x = adv[mask].astype(np.float64) / V.dual_value(0.0)
    assert x.max() - x.min() > np.log(1e30)     # exp(A / eta - m) over the selection spans more than 1e30
    _close(got["d_head"], want["d_head"], what="d_head")
    _close(got["dual_grad"], 0.5 * want["d_duals"], what="dual_grad")
    vl, dv = V.value_loss(value[:N], targets)
    m = want["metrics"].copy()
    m[8] = vl
    _close(got["metrics"], 0.5 * m, what="metrics")
    _close(got["d_value"][:N], dv, what="d_value")
    assert np.all(got["d_value"][N:] == 0.0)
    _same_bits(got, _vmpo_run(kind, per_dim, inputs), "vmpo_loss_grads")


def test_vmpo_after_step_past_the_grid():
    from stoix_b200 import ops

    P = W.VMPO_AFTER_STEP.shapes["P"]
    online = torch.randn(P, device="cuda")
    duals0 = torch.tensor([-30.0, -18.0, -17.5, 4.0, float("nan"), -18.5], device="cuda")
    for c, copies in ((3, False), (10, True)):
        runs = []
        for _ in range(2):
            duals, target = duals0.clone(), torch.full((P,), -3.0, device="cuda")
            ops.vmpo_after_step(duals, online, target, torch.tensor([c], dtype=torch.int32, device="cuda"), 5)
            torch.cuda.synchronize()
            runs.append((duals.cpu().numpy(), target.cpu().numpy()))
        d, tg = runs[0]
        assert d[:4].tolist() == [-18.0, -18.0, -17.5, 4.0] and np.isnan(d[4]) and d[5] == -18.0
        if copies:
            assert np.array_equal(tg.view(np.uint32), online.cpu().numpy().view(np.uint32))
        else:
            assert np.all(tg == -3.0)
        assert np.array_equal(runs[1][0].view(np.uint32), d.view(np.uint32)) and np.array_equal(runs[1][1], tg)


# -------------------------------------------------------------------------------------------------------------- MPO loss ----
MPO_M = W.MPO_CATEGORICAL.shapes["M"]


def _mpo_extremes(rng, q, M):
    """For every action j: its minimum and maximum of q in rows of the last (ragged) trip of blocks 0 and 1."""
    grid, per_block = W.trips(W.MPO_CATEGORICAL, M)
    last = (max(per_block) - 1) * grid * 256
    rows = rng.choice(np.arange(last, M), size=2 * q.shape[0], replace=False)
    for j in range(q.shape[0]):
        q[j, rows[2 * j]] = q[j].min() - 3.0 - j
        q[j, rows[2 * j + 1]] = q[j].max() + 3.0 + j
    return rows


def _mpo_categorical_inputs(M, A, N, seed):
    rng = np.random.default_rng(seed)
    zo, zt = rng.normal(size=(M, A)).astype(np.float32), rng.normal(size=(M, A)).astype(np.float32)
    q = (rng.normal(size=(A, M)) * 5).astype(np.float32)
    rows = _mpo_extremes(rng, q, M)
    qb = rng.normal(size=(N, M)).astype(np.float32)
    return zo, zt, q, np.array([0.3, -1.2], np.float32), qb, rows


def _mpo_categorical_run(zo, zt, q, duals, qb):
    from stoix_b200 import ops

    M, A = zo.shape
    d_head, dual_grad, metrics, v = torch.zeros(M, A, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(14, device="cuda"), torch.zeros(M, device="cuda")
    ops.mpo_loss_grads(_t(zo), _t(zt), _t(q), _t(duals), d_head, dual_grad, metrics, 0.01, 1e-3, q_boot=_t(qb), v=v, weight=0.5)
    torch.cuda.synchronize()
    return {"d_head": d_head.cpu().numpy(), "dual_grad": dual_grad.cpu().numpy(), "metrics": metrics.cpu().numpy(), "v": v.cpu().numpy()}


def test_mpo_categorical_loss_past_the_grid():
    A, N = 5, 4
    zo, zt, q, duals, qb, _ = _mpo_categorical_inputs(MPO_M, A, N, seed=11)
    got = _mpo_categorical_run(zo, zt, q, duals, qb)
    dh, dg, mt = MO.categorical_loss(zo, zt, q, duals, 0.01, 1e-3)
    np.testing.assert_allclose(got["d_head"], dh, rtol=1e-5, atol=2e-6 / MPO_M)
    np.testing.assert_allclose(got["dual_grad"], 0.5 * dg, rtol=1e-5, atol=1e-7)
    want = 0.5 * np.array([mt[k] for k in MO.METRICS])
    gm = got["metrics"][:13].astype(np.float64)
    atol = np.full(13, 1e-6)
    atol[MO.METRICS.index("kl_mean_rel")], atol[MO.METRICS.index("kl_q_rel")] = 1e-6 / 1e-3, 1e-6 / 0.01
    assert np.all(np.abs(gm[:11] - want[:11]) <= atol[:11] + 1e-5 * np.abs(want[:11])), (gm, want)
    assert MO.METRICS[11:] == ("q_min", "q_max")
    np.testing.assert_allclose(gm[11:], want[11:], rtol=1e-6, atol=0)      # exact per-action extremes, from the ragged trip
    np.testing.assert_allclose(got["v"], qb.astype(np.float64).mean(0), rtol=1e-6, atol=1e-6)
    _same_bits(got, _mpo_categorical_run(zo, zt, q, duals, qb), "mpo categorical")


def _mpo_tanh_inputs(M, A, NL, per_dim, seed):
    """test_mpo_gpu's draws, with the heads clipped to [-0.75, 0.75]: at this M the unclipped tails reach target scales whose KL
    gradient terms (about 100) cancel to within the fp32 rounding of a term, which the in-wave tolerance of 1e-6 / M never meets."""
    rng = np.random.default_rng(seed)
    h, ht = (np.clip(rng.normal(size=(M, 2 * A)) * 0.5, -0.75, 0.75).astype(np.float32) for _ in range(2))
    q = (rng.normal(size=(NL, M)) * 3).astype(np.float32)
    _mpo_extremes(rng, q, M)
    acts = (np.tanh(rng.normal(size=(NL, M, A))) * 0.95).astype(np.float32)   # inside the clip band
    C = A if per_dim else 1
    return h, ht, q, acts, rng.normal(size=1 + 2 * C).astype(np.float32)


def _mpo_tanh_run(h, ht, q, acts, duals, per_dim):
    from stoix_b200 import ops

    M, Wd = h.shape
    d_head, dual_grad, metrics = torch.zeros(M, Wd, device="cuda"), torch.zeros(duals.size, device="cuda"), torch.zeros(14, device="cuda")
    ops.mpo_loss_grads(_t(h), _t(ht), _t(q), _t(duals), d_head, dual_grad, metrics, 0.05, 0.05, kind="tanh_normal", actions=_t(acts),
                       epsilon_stddev=5e-4, per_dim=per_dim, weight=0.5)
    torch.cuda.synchronize()
    return {"d_head": d_head.cpu().numpy(), "dual_grad": dual_grad.cpu().numpy(), "metrics": metrics.cpu().numpy()}


@pytest.mark.parametrize("per_dim", [True, False])
def test_mpo_tanh_loss_past_the_grid(per_dim):
    A, NL = 3, 4
    h, ht, q, acts, duals = _mpo_tanh_inputs(MPO_M, A, NL, per_dim, seed=12 + per_dim)
    got = _mpo_tanh_run(h, ht, q, acts, duals, per_dim)
    dh, dg, mt = MO.continuous_loss(h, ht, q, acts, duals, 0.05, 0.05, 5e-4, per_dim, -1.0, 1.0)
    np.testing.assert_allclose(got["d_head"], dh, rtol=1e-4, atol=1e-6 / MPO_M)
    np.testing.assert_allclose(got["dual_grad"], 0.5 * dg, rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(got["metrics"][:13], 0.5 * np.array([mt[k] for k in MO.CONTINUOUS_METRICS]), rtol=1e-4, atol=1e-6)
    _same_bits(got, _mpo_tanh_run(h, ht, q, acts, duals, per_dim), "mpo tanh-Normal")


# ------------------------------------------------------------------------------------------------------ PPO value faces ----
def test_ppo_value_faces_past_the_grid():
    """n crosses both caps: 264 blocks for the clip and value faces (one partial per block), 132 for the penalty and DPO faces (two)."""
    from stoix_b200.networks.heads import NormalAffineTanhDistributionHead
    from stoix_b200.utils import loss

    n = W.FACE_ONE_PART.shapes["n"]
    assert n == W.FACE_TWO_PARTS.shapes["n"]
    rng = np.random.default_rng(21)
    a, b, c = (rng.standard_normal(n).astype(np.float32) * 0.4 for _ in range(3))
    c[-1] = 30.0                                               # an outlier in the ragged last trip
    f64 = lambda x: x.astype(np.float64)

    def faces():
        out = {"clip": loss.ppo_clip_loss(_t(a), _t(b), _t(c), 0.2).item(), "value": loss.clipped_value_loss(_t(a), _t(b), _t(c), 0.2).item()}
        pl, pk = loss.ppo_penalty_loss(_t(a), _t(b), _t(c), 3.0, pi, b_pi)
        out.update(penalty=pl.item(), penalty_kl=pk.item(), dpo=loss.dpo_loss(_t(a), _t(b), _t(c), 2.0, 0.6).item())
        return {k: np.float32(v) for k, v in out.items()}

    A = 3
    head = NormalAffineTanhDistributionHead(A, -1.0, 1.0)
    hb, hp = rng.normal(0, 1, (n, 2 * A)).astype(np.float32), rng.normal(0, 1, (n, 2 * A)).astype(np.float32)
    b_pi, pi = head.distribution(_t(hb)), head.distribution(_t(hp))
    got = faces()
    np.testing.assert_allclose(got["clip"], O.ppo_clip_loss(f64(a), f64(b), f64(c), 0.2), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got["value"], O.clipped_value_loss(f64(a), f64(b), f64(c), 0.2), rtol=1e-5, atol=1e-7)
    kl_rows = PV.tanh_normal_kl(b_pi.head_out.double().cpu().numpy(), pi.head_out.double().cpu().numpy())[0]
    ratio = np.exp(f64(a) - b)
    np.testing.assert_allclose([got["penalty"], got["penalty_kl"]], [-(ratio * c).mean() + 3.0 * kl_rows.mean(), kl_rows.mean()], rtol=1e-4)
    rows, _ = PV.dpo_rows(f64(a) - b, f64(c), 2.0, 0.6)
    np.testing.assert_allclose(got["dpo"], rows.mean(), rtol=1e-4, atol=1e-7)
    _same_bits(got, faces(), "loss faces")


# ------------------------------------------------------------------------------------------------- observation statistics ----
_STATS = {"D17": (17, W.OBS_ACC_D17, False), "D256": (256, W.OBS_ACC_D256, False), "D64_misaligned": (64, W.OBS_ACC_D64_MISALIGNED, True)}


def _stats_batch(D, rows, seed):
    rng = np.random.default_rng(seed)
    scale, shift = rng.uniform(0.1, 5.0, D), rng.uniform(-3, 3, D)
    x = (rng.standard_normal((rows, D)) * scale + shift).astype(np.float32)
    x[-1] = (shift + 50.0 * scale).astype(np.float32)           # an outlier row in the ragged last trip
    return x, (rng.standard_normal((40, D)) * scale + shift).astype(np.float32)


def _device_rows(x, misaligned):
    """x on the device; misaligned: a view one float into a larger buffer (not 16-byte aligned: the scalar form even when D % 4 == 0)."""
    if not misaligned:
        return _t(x)
    buf = torch.empty(x.size + 1, dtype=torch.float32, device="cuda")
    v = buf[1:].view(x.shape)
    v.copy_(torch.from_numpy(x))
    assert v.data_ptr() % 16 != 0
    return v


def _stats_update(x_dev, D, first, w=None):
    """initialise, absorb `first`, then absorb x_dev (with weights w): the state tensors after each step."""
    from stoix_b200 import ops

    count, mean = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(D, device="cuda")
    sv, std = torch.zeros(D, device="cuda"), torch.ones(D, device="cuda")
    for xx, ww in ((_t(first), None), (x_dev, w)):
        sums = ops.running_stats_accumulate(xx, mean, ww)
        ops.running_stats_finalize(sums, count, mean, sv, std, 5e-4, 5e4)
    torch.cuda.synchronize()
    return {"count": count.cpu().numpy(), "mean": mean.cpu().numpy(), "sv": sv.cpu().numpy(), "std": std.cpu().numpy(), "sums": sums.cpu().numpy()}


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("case", list(_STATS))
def test_running_statistics_past_the_grid(case, weighted):
    D, loop, misaligned = _STATS[case]
    rows = loop.shapes["rows"]
    x, first = _stats_batch(D, rows, seed=D + weighted)
    w = None
    if weighted:
        w = np.random.default_rng(D).integers(0, 3, rows).astype(np.float32)   # integer weights: weight k == the row repeated k times
        w[-1] = 2.0
        assert (w == 0).any()
    x_dev = _device_rows(x, misaligned)
    w_dev = None if w is None else _t(w)
    got = _stats_update(x_dev, D, first, w_dev)
    ref = RO.update(RO.initialize((D,)), [first.astype(np.float64)], std_min_value=5e-4, std_max_value=5e4)
    rep = x if w is None else np.repeat(x, w.astype(np.int64), axis=0)
    ref = RO.update(ref, [rep.astype(np.float64)], std_min_value=5e-4, std_max_value=5e4)
    assert int(got["count"][0]) == int(ref.count)
    np.testing.assert_allclose(got["mean"], ref.mean, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got["sv"], ref.summed_variance, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(got["std"], ref.std, rtol=1e-5, atol=1e-7)
    _same_bits(got, _stats_update(x_dev, D, first, w_dev), "running statistics")


_NORM = {"D17": (17, 70_001), "D64": (64, 40_000)}


@pytest.mark.parametrize("max_abs", [None, 0.5])
@pytest.mark.parametrize("case", list(_NORM))
def test_obs_normalize_past_the_grid(case, max_abs):
    """fp32 and bf16 outputs, and a bf16 output one element off its 8-byte alignment (the scalar form at D = 64)."""
    from stoix_b200 import ops

    D, rows = _NORM[case]
    assert rows * D in set(W.OBS_NORM_SCALAR.shapes.values()) | {4 * v for v in W.OBS_NORM_VEC.shapes.values()}
    rng = np.random.default_rng(D)
    x = (rng.standard_normal((rows, D)) * rng.uniform(0.1, 5.0, D) + rng.uniform(-3, 3, D)).astype(np.float32)
    x[-1] = 1e4
    mean, std = rng.uniform(-3, 3, D).astype(np.float32), rng.uniform(0.1, 5.0, D).astype(np.float32)
    want = RO.normalize(x.astype(np.float64), RO.RunningStatistics(1.0, mean.astype(np.float64), np.zeros(D), std.astype(np.float64)), max_abs)
    xd, md, sd = _t(x), _t(mean), _t(std)

    def run():
        f32 = ops.obs_normalize(xd, md, sd, max_abs_value=max_abs)
        b16 = ops.obs_normalize(xd, md, sd, out_dtype=torch.bfloat16, max_abs_value=max_abs)
        off = torch.empty(x.size + 1, dtype=torch.bfloat16, device="cuda")[1:].view(rows, D)
        ops.obs_normalize(xd, md, sd, out=off, max_abs_value=max_abs)
        torch.cuda.synchronize()
        return {"f32": f32.cpu().numpy(), "bf16": b16.float().cpu().numpy(), "bf16_off": off.float().cpu().numpy()}

    got = run()
    np.testing.assert_allclose(got["f32"], want, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(got["bf16"], want, rtol=2 ** -8, atol=1e-6)
    np.testing.assert_array_equal(got["bf16_off"], got["bf16"])
    _same_bits(got, run(), "obs_normalize")


# ------------------------------------------------------------------------------------------------------------------ Polyak ----
def test_polyak_past_the_grid():
    """target = tau online + (1 - tau) target within 2 fp32 ulps of fp64 (the compiler may contract it into an FMA).  online and
    target share a sign per element, so no cancellation leaves the two products' roundings large against the result."""
    from stoix_b200 import ops

    n, tau = W.POLYAK.shapes["n"], 0.005
    rng = np.random.default_rng(3)
    sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    online = (sign * rng.uniform(0.5, 4.0, n)).astype(np.float32)
    target = (sign * rng.uniform(0.5, 4.0, n)).astype(np.float32)
    tau32 = np.float32(tau)
    want = np.float64(tau32) * online + np.float64(np.float32(1.0) - tau32) * target
    runs = []
    for _ in range(2):
        t = _t(target)
        ops.polyak_update(t, _t(online), tau)
        torch.cuda.synchronize()
        runs.append(t.cpu().numpy())
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(runs[0].astype(np.float64) - want) / ulp
    assert err.max() <= 2.0, (int(err.argmax()), float(err.max()))
    assert np.array_equal(runs[0].view(np.uint32), runs[1].view(np.uint32))


# --------------------------------------------------------------------------------------------------------- scratch reuse ----
def test_vmpo_loss_scratch_reuse_across_grid_sizes():
    small = _vmpo_inputs("tanh_normal", True, 3, 1000, seed=1)
    first = _vmpo_run("tanh_normal", True, small)
    _vmpo_run("tanh_normal", True, _vmpo_inputs("tanh_normal", True, 3, VMPO_N["three_waves"], seed=2))
    _same_bits(first, _vmpo_run("tanh_normal", True, small), "vmpo small / large / small")


def test_mpo_loss_scratch_reuse_across_grid_sizes():
    zo, zt, q, duals, qb, _ = _mpo_categorical_inputs(1000, 5, 4, seed=3)
    first = _mpo_categorical_run(zo, zt, q, duals, qb)
    _mpo_categorical_run(*_mpo_categorical_inputs(MPO_M, 5, 4, seed=4)[:5])
    _same_bits(first, _mpo_categorical_run(zo, zt, q, duals, qb), "mpo small / large / small")


@pytest.mark.parametrize("case", list(_STATS))
def test_running_statistics_scratch_reuse_across_grid_sizes(case):
    D, loop, misaligned = _STATS[case]
    x_small, first = _stats_batch(D, 1000, seed=5)
    small = _device_rows(x_small, misaligned)
    a = _stats_update(small, D, first)
    _stats_update(_device_rows(_stats_batch(D, loop.shapes["rows"], seed=6)[0], misaligned), D, first)
    _same_bits(a, _stats_update(small, D, first), "running statistics small / large / small")
