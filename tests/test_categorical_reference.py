"""The categorical sampler restatements and edge families of tests/categorical_reference.py, on the CPU: counter layouts, u01,
the fp64 inverse CDF, and the seeds the GPU tests rely on."""
import numpy as np
import pytest

from oracle.synth_env import philox4x32, u01
from tests import categorical_reference as R

# the calls of tests/test_categorical_heads_gpu.py: small offsets, offset 2^32 - 2 with device counters 0..3, the rollout's
# cat_offset 2^32 - 3 + t + counter, and the seed-and-call pair of the remainder case
GPU_CALLS = sorted({0, 1, 5, 7, *[(1 << 32) - 3 + k for k in range(8)], (1 << 32) + 7})
GPU_ROWS = [0, 1, 3, 255, 256, 8703, 69999, (1 << 32) - 1, 1 << 32, (1 << 32) + 1]


def test_philox_known_answers():
    """Philox4x32-10 known-answer vectors (Salmon et al., Random123)."""
    got = philox4x32(0, 0, 0, 0, 0, 0)
    assert [int(w) for w in got] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    got = philox4x32(*[0xFFFFFFFF] * 4, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(w) for w in got] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    got = philox4x32(0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0)
    assert [int(w) for w in got] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_u01_restatement():
    """u01(x) = ((x >> 9) + 1/2) 2^-23 exactly in fp32: 2^23 distinct values strictly inside (0, 1), from 2^-24 to 1 - 2^-24."""
    x = np.concatenate([np.array([0, 1, 511, 512, 0x7FFFFFFF, 0x80000000, 0xFFFFFDFF, 0xFFFFFE00, 0xFFFFFFFF], np.uint64),
                        np.random.default_rng(0).integers(0, 1 << 32, 100000, dtype=np.uint64)])
    u = u01(x)
    assert u.dtype == np.float32
    exact = ((x >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    np.testing.assert_array_equal(u.astype(np.float64), exact)
    assert u[0] == 2.0 ** -24 and u[8] == 1.0 - 2.0 ** -24
    assert (u > 0).all() and (u < 1).all()
    # the two u01 values at or above 1 - 2^-22, the ones the remainder case needs
    assert (u01(np.arange(0xFFFFF800, 0xFFFFFFFF + 1, 512, dtype=np.uint64)) >= R.U_HIGH).sum() == 2


def test_gumbel_counters_distinct_below_1024_actions():
    """(row, call, group) counters of the draws the GPU tests make are pairwise distinct for groups < 256; group 256 is group 0's
    counter, so actions 1024..1027 would get the noise of actions 0..3: why stx_categorical refuses A > 1024."""
    c = np.stack([np.stack([w.ravel() for w in R.gumbel_counters(GPU_ROWS, call, np.arange(256))], 1) for call in GPU_CALLS])
    c = c.reshape(-1, 4)
    assert len(np.unique(c, axis=0)) == len(c) == len(GPU_CALLS) * len(GPU_ROWS) * 256
    for call in GPU_CALLS:
        for w256, w0 in zip(R.gumbel_counters(GPU_ROWS, call, [256]), R.gumbel_counters(GPU_ROWS, call, [0])):
            np.testing.assert_array_equal(w256, w0)
    u = R.gumbel_uniforms(3, 5, np.arange(4), 1028)
    np.testing.assert_array_equal(u[:, 1024:], u[:, :4])
    assert len(np.unique(u[:, :1024])) == 4 * 1024


def test_gumbel_restatement_ties_and_wide_rows():
    """First index on exact score ties; with equal logits every action of a 1024-wide row is drawn, the highest ones included."""
    z = np.zeros((4, 3), np.float32)
    d = R.gumbel_actions(z, 1, 2)
    assert d.action.tolist() == np.argmax(d.score, 1).tolist() and (d.margin > 0).all()
    d = R.gumbel_actions(np.zeros((4096, 1024), np.float32), 11, 0)
    assert d.action.max() >= 1020 and len(np.unique(d.action)) > 900
    d = R.gumbel_actions(np.zeros((7, 1), np.float32), 11, 0)
    assert (d.action == 0).all() and np.isinf(d.margin).all()
    # frequencies of the restatement follow the softmax (16384 rows: within 2.5e-2)
    zz = np.tile(np.array([[0.0, 1.0, -1.0, 2.0, 0.5]], np.float32), (16384, 1))
    f = np.bincount(R.gumbel_actions(zz, 5, 9).action, minlength=5) / 16384
    assert np.abs(f - np.exp(R.log_softmax(zz[0].astype(np.float64)))).max() < 2.5e-2


def test_inverse_cdf_hand_cases():
    assert [R.inverse_cdf([0.5, 0.25, 0.25], u) for u in (0.0, 0.49, 0.5, 0.74, 0.75, 0.999)] == [0, 0, 1, 1, 2, 2]
    assert R.inverse_cdf([0.0, 1.0], 1e-9) == 1
    assert R.inverse_cdf([0.2, 0.8, 0.0], 0.99999) == 1
    assert R.inverse_cdf([0.2, 0.8, 0.0], 1.0) == 2       # at or above the whole sum: the last index, as np.searchsorted + clip
    rng = np.random.default_rng(1)
    z = (rng.standard_normal((50, 6)) * 3).astype(np.float32)
    d = R.mpo_draws(z, 9, (1 << 32) + 3, 20, 50)
    for n in range(20):
        for i in range(50):
            assert d.action[n, i] == R.inverse_cdf(d.prob[i], float(d.u[n, i]))
    far = d.distance > 2.0 ** -21
    np.testing.assert_array_equal(d.action32[far], d.action[far])


def test_mpo_uniform_counter_layout():
    """u of draw (n, i) is u01 of word 0 at counter (n M + i lo, hi, call lo, "MPOA" ^ call hi), keyed by (seed lo, seed hi)."""
    seed, call, N, M = 0x0123456789ABCDEF, (5 << 32) + 17, 3, 7
    u = R.mpo_uniforms(seed, call, N, M)
    for n, i in ((0, 0), (1, 3), (2, 6)):
        ctr = n * M + i
        w = philox4x32(ctr & R.M32, ctr >> 32, call & R.M32, R.TAG_MPOA ^ (call >> 32), seed & R.M32, seed >> 32)
        assert u[n, i] == u01(w[0])


def test_mpo_remainder_case_is_not_vacuous():
    """The remainder case's rows all end their fp32 sum at or below 1 - 2^-21 and its seed draws u >= 1 - 2^-22 at least twice:
    each such draw exceeds the whole fp32 sum.  The emulated fixed kernel gives it to the last action of positive fp32 probability
    (31 of 32: the last logit is -200), and the fp64 inverse CDF agrees but for draws within 2^-21 of a boundary."""
    case = R.mpo_remainder_case()
    assert case.logits.shape == (case.M, 32)
    d = R.mpo_draws(case.logits, case.seed, case.call, case.N, case.M)
    assert (d.sum32 <= np.float32(R.SUM_LOW)).all()
    hit = d.u >= np.float32(R.U_HIGH)
    assert hit.sum() >= 2, hit.sum()
    assert (d.u[hit] >= d.sum32[np.nonzero(hit)[1]]).all()
    assert (d.action32[hit] == 30).all()
    assert (d.prob[:, 31] < 1e-30).all()
    assert (d.action32 != 31).all()
    far = d.distance > 2.0 ** -21
    np.testing.assert_array_equal(d.action32[far], d.action[far])
    assert (d.distance[hit] <= 2.0 ** -21).all()


@pytest.mark.parametrize("A", [1, 2, 3, 8, 31, 32])
def test_edge_rows_and_fp64_heads(A):
    """The edge families reach the regimes they are for, and the fp64 references stay finite on them."""
    z, act = R.edge_rows(A, np.random.default_rng(A))
    assert z.dtype == np.float32 and act.dtype == np.int32 and len(z) == len(act)
    z64 = z.astype(np.float64)
    lp = R.categorical_log_prob(z64, act)
    h = R.categorical_entropy(z64)
    assert np.isfinite(lp).all() and (lp <= 0).all() and np.isfinite(h).all() and (h >= -1e-12).all() and (h <= np.log(A) + 1e-9).all()
    assert np.abs(z64).max() >= 1e5
    if A > 1:
        spread = z64.max(1) - z64.min(1)
        assert spread.max() >= 1e4 and lp.min() < -745.0          # fp64 probabilities underflow to 0 too
        assert ((spread > 104) & (spread < 120)).any()            # fp32 expf underflows (gap > ~104)
        assert (np.signbit(z) & (z == 0)).any()                   # signed zeros at tied maxima
        pos = np.isin(np.arange(len(z)) % 2, [1])                 # odd rows take the least probable action
        assert (lp[pos] <= lp[~pos] + 1e-12).all()
    kl = R.categorical_kl(z64, z64[::-1].copy())
    assert np.isfinite(kl).all() and (kl >= -1e-9).all()
    _, dl, _ = R.ppo_clip_head(z64, act, lp - 0.1, np.ones(len(z)), 0.2, 0.01)
    assert np.isfinite(dl).all()
