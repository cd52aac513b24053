"""CPU checks of tests/prio_reference.py: the fp64 inverse CDF against a brute-force search, the fixed fp32 descent within δ on random
trees at every fp32 cumulative boundary, and the earlier fall-through rule breaking δ on a committed tree."""
import numpy as np
import pytest

from tests import prio_reference as P
from tests import r2d2_oracle as orc
from tests import rainbow_oracle as R


def _leaves(rng, n, kind):
    if kind == "uniform":
        x = rng.random(n)
    elif kind == "loguniform":
        x = 10.0 ** rng.uniform(-6, 6, n)
    elif kind == "heavy":
        x = rng.random(n)
        x = x * (1e-6 / x.sum())
        x[rng.integers(n)] = 1.0 - 1e-6
    else:
        x = np.ones(n)
    x = x.astype(np.float32)
    if n > 2:
        x[rng.random(n) < 0.1] = 0   # zero leaves, as invalid items leave them
        x[-(n // 3):] = 0            # a tail of zeros past the last positive leaf
        x[0] = max(x[0], np.float32(1e-3))
    return x


def test_tree_levels_are_in_order_fp32_sums():
    rng = np.random.default_rng(0)
    x = (10.0 ** rng.uniform(-6, 6, 1057)).astype(np.float32)
    lv = P.tree_levels(x)
    assert [len(a) for a in lv] == [1057, 34, 2, 1] and P.height(1057) == 4 and P.height(1) == 1 and P.height(32) == 2
    for child, parent in zip(lv, lv[1:]):
        want = [orc._fsum(child[i:i + 32]) for i in range(0, len(child), 32)]
        np.testing.assert_array_equal(parent, np.array(want, np.float32))
    flat = np.concatenate(lv)
    assert len(flat) == R.tree_floats(1057)
    for a, b in zip(P.split_levels(flat, 1057), lv):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("n", [1, 2, 31, 33, 700])
def test_reference_draw_is_the_brute_force_inverse_cdf(n):
    rng = np.random.default_rng(n)
    leaves = _leaves(rng, n, "loguniform") if n > 1 else np.array([0.5], np.float32)
    M = 64
    r = np.arange(M)
    u = rng.random(M).astype(np.float32)
    u[:3] = [0.0, P.U_MAX, 0.5]
    u[-1] = P.U_MAX
    ref = P.Reference(leaves)
    got = ref.draws(r, u, M)
    lv = [float(x) for x in leaves]
    for m in range(M):
        v = (r[m] + float(u[m])) * ref.sigma / M
        acc, want = 0.0, None
        for i, p in enumerate(lv):
            acc += p
            if acc > v and p > 0:
                want = i
                break
        if want is None:
            want = max(i for i, p in enumerate(lv) if p > 0)
        assert got[m] == want, m
    assert P.Reference(np.zeros(5, np.float32)).draws(r, u, M).tolist() == [0] * M


def test_boundary_uniforms_put_v_on_the_boundaries():
    rng = np.random.default_rng(3)
    lv = P.tree_levels(_leaves(rng, 5000, "uniform"))
    for level in range(len(lv) - 1):
        r, u, hit = P.boundary_uniforms(lv, level, 512)
        v = P.device_v(r, u, lv[-1][0], 512)
        b = np.unique(np.cumsum(lv[level], dtype=np.float32))
        b = b[b > 0]
        assert ((u >= 0) & (u < 1)).all()
        np.testing.assert_array_equal(v[hit], b[hit])
        assert hit.mean() > 0.5 and (v >= b).all()
    r, u, _ = P.boundary_uniforms(lv, len(lv) - 2, 512)   # the last boundary of the root's children is the total: v = total
    assert r[-1] == 511 and P.device_v(r[-1:], u[-1:], lv[-1][0], 512)[0] == lv[-1][0]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1024, 1025, 5000, 32769])
@pytest.mark.parametrize("kind", ["uniform", "loguniform", "heavy", "equal"])
def test_fixed_descent_stays_within_delta(n, kind):
    """Philox-like uniforms, u = 0 and U_MAX in every stratum, and every level's fp32 cumulative boundaries: every draw lies within δ
    of v64, lands on a positive leaf, and equals the reference draw wherever v64 is more than δ from every boundary."""
    rng = np.random.default_rng(n * 7 + len(kind))
    leaves = _leaves(rng, n, kind)
    lv, ref = P.tree_levels(leaves), P.Reference(leaves)
    M = 512
    pairs = [(np.arange(M), rng.random(M).astype(np.float32)), (np.arange(M), np.zeros(M, np.float32)), (np.arange(M), np.full(M, P.U_MAX))]
    for level in range(len(lv) - 1):
        r, u, _ = P.boundary_uniforms(lv, level, M)
        pairs.append((r, u))
    worst, falls = 0.0, 0
    for r, u in pairs:
        v = P.device_v(r, u, lv[-1][0], M)
        k = P.descend(lv, v)
        j = ref.judge(r, u, M, k)
        assert (leaves[k] > 0).all()
        assert (j.ratio <= 1.0).all(), (n, kind, j.ratio.max())
        np.testing.assert_array_equal(k[j.far], j.ref[j.far])
        worst = max(worst, float(j.ratio.max()))
        falls += int((P.descend(lv, v, fixed=False) != k).sum())
    print(f"[prio reference] n={n} {kind}: worst distance / delta {worst:.3g}, draws the earlier rule misplaces {falls}")


def test_boundaries_expose_the_earlier_rule_on_random_trees():
    """Over random trees the boundary uniforms make the descent fall through, and the earlier rule then misses δ by orders of
    magnitude: the boundary cases are not vacuous."""
    rng = np.random.default_rng(11)
    worst, falls = 0.0, 0
    for _ in range(40):
        n = int(rng.integers(1100, 40000))
        leaves = _leaves(rng, n, "uniform" if rng.random() < 0.5 else "loguniform")
        lv = P.tree_levels(leaves)
        for level in range(len(lv) - 1):
            r, u, _ = P.boundary_uniforms(lv, level, 512)
            v = P.device_v(r, u, lv[-1][0], 512)
            old, new = P.descend(lv, v, fixed=False), P.descend(lv, v)
            falls += int((old != new).sum())
            worst = max(worst, float(P.Reference(leaves).judge(r, u, 512, old).ratio.max()))
    print(f"[prio reference] earlier rule on 40 random trees: {falls} misplaced draws, worst distance / delta {worst:.3g}")
    assert falls > 0 and worst > 100


def test_earlier_rule_breaks_delta_on_the_two_halves_tree():
    leaves = P.two_halves_tree()
    lv = P.tree_levels(leaves)
    assert lv[2].tolist() == [np.float32(1 + 3 * 2.0 ** -23), 1.0] and lv[3][0] == np.float32(2 + 4 * 2.0 ** -23)
    M = 512
    r, u = np.array([M - 1]), np.array([P.U_MAX])
    v = P.device_v(r, u, lv[-1][0], M)
    assert v[0] == lv[-1][0]   # v = total
    old, new = P.descend(lv, v, fixed=False), P.descend(lv, v)
    assert old.tolist() == [1024] and new.tolist() == [2047]
    ref = P.Reference(leaves)
    bad, good = ref.judge(r, u, M, old), ref.judge(r, u, M, new)
    assert good.ratio[0] == 0 and good.ref[0] == 2047
    assert bad.ratio[0] > 1e4   # half the mass, against δ = 2^-16 Σ


def test_oracle_samplers_take_the_last_positive_leaf_at_the_total():
    """rainbow_oracle.PrioRing.sample (fp64 searchsorted) and r2d2_oracle.Ring.sample_items (the fp32 descent) at v = total and at the
    two-halves tree's fall-through."""
    ring = R.PrioRing(4, 1, 1, 1, 1.0)
    ring.prio = np.array([1.0, 2.0, 0.0, 0.0])
    assert ring.sample(np.array([0.0, P.U_MAX])).tolist() == [0, 1]
    ring.prio = np.array([0.1, 0.2, 0.3, 0.0])   # v exactly at the cumulative sum's end: the last positive item, not len(prio)
    assert ring.sample(np.array([0.5, 1.0])).tolist() == [1, 2]
    ring.prio = np.zeros(4)
    assert ring.sample(np.array([0.5, 0.5])).tolist() == [0, 0]
    r2 = orc.Ring(2048, 1, 1, 1, 1.0)
    r2.leaves = P.two_halves_tree().astype(np.float64)
    u = np.full(512, 0.5, np.float32)
    u[-1] = P.U_MAX
    lv = P.tree_levels(P.two_halves_tree())
    want = P.descend(lv, P.device_v(np.arange(512), u, lv[-1][0], 512))
    assert want[-1] == 2047
    np.testing.assert_array_equal(r2.sample_items(u), want)


@pytest.mark.parametrize("beta0", [0.4, 0.6])
@pytest.mark.parametrize("steps", [0.0, 1000.0, 300.0])
def test_beta32_is_the_fp64_schedule_within_rounding(beta0, steps):
    for count in (None, 0, 1, 299, 300, 999, 1000, 10000, -3):
        want = R.beta_at(0 if count is None else count, float(np.float32(beta0)), steps)
        assert abs(float(P.beta32(count, beta0, steps)) - want) <= 3 * P.EPS32 * want
    assert P.beta32(5, beta0, 0.0) == np.float32(beta0) and P.beta32(1000, beta0, 1000.0) == 1.0
