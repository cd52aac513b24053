"""The prioritised replay sampler on the GPU against the fp64 inverse CDF of tests/prio_reference.py: Rainbow's ring
(ops.PrioritisedRing) and R2D2's (ops.R2d2Ring) on sum trees of 1 to 5 levels, up to Rainbow's shipped 1024 x 976 items, with the
Philox stream at M = 512, u = 0 and the largest u01 in every stratum, and uniforms that put v on every level's fp32 cumulative
boundaries, where fp32 rounding makes the descent fall through.  Every draw lands on a positive leaf within δ of v64 (and on the
reference leaf where v64 is more than δ from every boundary); p is fp32(leaf / root); the importance weights match fp64 on the
device's own probabilities; set_priorities keeps every parent the in-order fp32 sum of its children; two launches give the same bits."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from stoix_b200 import ops
from tests import prio_reference as P
from tests import rainbow_oracle as R

pytestmark = pytest.mark.gpu

M = 512
BETA0, STEPS = 0.4, 1000.0
t_ = lambda x: torch.tensor(x, device="cuda")

# items: (envs, rows) of Rainbow's ring; heights 1 .. 5, every level's last parent ragged where the count allows
RAINBOW = {1: (1, 1), 31: (1, 31), 32: (1, 32), 33: (3, 11), 1024: (4, 256), 1025: (5, 205), 32769: (3, 10923), 999424: (1024, 976)}
# R2D2's ring: (envs, rows, seq_len, period); 2048 items is the shipped shape (100 000 // 1024 rows, period 40)
R2D2 = {1: (1, 1, 1, 1), 33: (3, 11, 2, 1), 1025: (5, 205, 2, 1), 2048: (1024, 97, 80, 40), 256000: (1000, 256, 2, 1)}
KINDS = ["uniform", "loguniform", "heavy", "equal", "partial"]


def _priorities(rng, n, kind):
    """Priorities of the n valid items: uniform; log-uniform on [1e-6, 1e6] with both extremes present (a 1e12 probability ratio,
    the 1e-6 on the first valid item, which u = 0 in stratum 0 draws); one item with 1 - 1e-6 of the mass; all equal."""
    if kind in ("uniform", "partial"):
        return (1.0 - rng.random(n)).astype(np.float32)
    if kind == "loguniform":
        x = 10.0 ** rng.uniform(-6, 6, n)
        x[0] = 1e-6
        x[n // 2] = 1e6
        return x.astype(np.float32)
    if kind == "heavy":
        x = np.full(n, 1e-6 / max(n - 1, 1))
        x[n // 3] = 1.0 - 1e-6
        return x.astype(np.float32)
    return np.ones(n, np.float32)


def _check_tree(tree: torch.Tensor, items: int) -> np.ndarray:
    """Every internal node is the in-order fp32 sum of its children, bit for bit; returns the leaves."""
    got = P.split_levels(tree.cpu().numpy(), items)
    for lv, (a, b) in enumerate(zip(got[1:], P.tree_levels(got[0])[1:])):
        np.testing.assert_array_equal(a, b, err_msg=f"level {lv + 1} of {items} items")
    return got[0]


def _rainbow_ring(items, kind, alpha):
    E, L = RAINBOW[items]
    n = min(2, L)   # the item starting at the write head's last row is invalid: zero leaves throughout the tree
    T = L if kind != "partial" else max(n, L // 3)
    ring = ops.PrioritisedRing(L, E, 1, n, alpha, "cuda")
    obs = torch.zeros(T, E, 1, device="cuda")
    ops.replay_add_prioritised(ring, obs, torch.zeros(T, E, dtype=torch.int32, device="cuda"), torch.zeros(T, E, device="cuda"),
                               torch.zeros(T, E, dtype=torch.uint8, device="cuda"), obs)
    return ring


def _r2d2_ring(items, kind, alpha):
    E, L, S, p = R2D2[items]
    T = L if kind != "partial" else max(S, L // 3)
    if items == 2048:
        T = 80   # the shipped ring after 80 rows: item 0 of every env valid, item 1 (rows 40 ..) not yet
    ring = ops.R2d2Ring(L, E, 1, 1, S, p, alpha, "cuda")
    z = lambda dt=torch.float32: torch.zeros(T, E, dtype=dt, device="cuda")
    ops.r2d2_ring_add(ring, z().unsqueeze(-1), z(torch.int32), z(), z(torch.uint8), z(torch.uint8), z(torch.uint8), z().unsqueeze(-1))
    return ring


def _set_all(ring, set_fn, kind, alpha, rng):
    """Priorities on every valid item (the leaves the add left positive), read back with the rebuilt tree."""
    valid = np.flatnonzero(ring.priorities.cpu().numpy() > 0).astype(np.int32)
    assert len(valid) > 0
    pr = _priorities(rng, len(valid), kind)
    set_fn(ring, t_(valid), t_(pr))
    leaves = _check_tree(ring.tree, len(ring.priorities))
    np.testing.assert_allclose(leaves[valid], pr.astype(np.float64) ** alpha, rtol=1e-6)   # powf: within an ulp or two
    assert np.count_nonzero(leaves) == len(valid)
    return leaves


def _uniform_sets(leaves, rng):
    """(name, u (M) or None for the Philox stream) of one case: three Philox calls, u = 0 and the largest u01 in every stratum, and
    for every level the uniforms that put v on its fp32 cumulative boundaries (at most 2048 per level, 8 calls)."""
    sets = [("philox", None)] * 3 + [("u=0", np.zeros(M, np.float32)), ("u=max", np.full(M, P.U_MAX, np.float32))]
    lv = P.tree_levels(leaves)
    for level in range(len(lv) - 1):
        r, u, _ = P.boundary_uniforms(lv, level, M, limit=2048, rng=rng)
        sets += [(f"boundaries of level {level}", c) for c in P.uniform_calls(r, u, M, max_calls=8)]
    return sets


class _Sampler:
    """One ring's sampler with its outputs; run() launches twice and checks the two give the same bits."""

    def __init__(self, ring, rainbow: bool):
        self.ring, self.rainbow = ring, rainbow
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
        if rainbow:
            self.out = dict(obs=z(M, 1), next_obs=z(M, 1), action=z(M, dt=torch.int32), reward=z(M), done=z(M, dt=torch.uint8),
                            idx=z(M, dt=torch.int32), prob=z(M), weight=z(M))
        else:
            S = ring.seq_len
            self.out = dict(obs=z(S, M, 1), action=z(S, M, dt=torch.int32), reward=z(S, M), done=z(S, M, dt=torch.uint8),
                            reset=z(S, M, dt=torch.uint8), carry0=z(M, 1), idx=z(M, dt=torch.int32), prob=z(M))
        self.ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.seed = 20261018

    def _launch(self, u, count, beta0, steps):
        o = self.out
        kw = dict(u_in=t_(u)) if u is not None else dict(offset=3, dev_counter=self.ctr)
        if self.rainbow:
            ops.replay_sample_prioritised(self.ring, M, self.seed, o["obs"], o["next_obs"], o["action"], o["reward"], o["done"], o["idx"],
                                          o["prob"], o["weight"], 0.99, beta0, steps, count=count, **kw)
        else:
            ops.r2d2_ring_sample(self.ring, self.seed, o["obs"], o["action"], o["reward"], o["done"], o["reset"], o["carry0"], o["idx"], o["prob"],
                                 **kw)
        return {k: v.clone() for k, v in o.items()}

    def run(self, u, count=None, beta0=BETA0, steps=STEPS):
        """(u used, idx, prob, weight or None); the Philox stream's u restated by rainbow_oracle.prio_uniforms."""
        a, b = self._launch(u, count, beta0, steps), self._launch(u, count, beta0, steps)
        for k in a:
            assert torch.equal(a[k], b[k]), f"two launches differ in {k}"
        if u is None:
            u = R.prio_uniforms(self.seed, 3 + int(self.ctr.item()), M)
            ops.counter_add(self.ctr, 1)
        w = a["weight"].double().cpu().numpy() if self.rainbow else None
        return u, a["idx"].cpu().numpy().astype(np.int64), a["prob"].cpu().numpy(), w


def _check_draws(ref: P.Reference, leaves, root, u, idx, prob, what):
    r = np.arange(M)
    j = ref.judge(r, u, M, idx)
    if ref.sigma > 0:
        assert (leaves[idx] > 0).all(), f"{what}: a draw on a zero leaf"
    bad = np.flatnonzero(j.ratio > 1.0)
    assert not len(bad), (f"{what}: draw {bad[0]} (u={u[bad[0]]!r}) on leaf {idx[bad[0]]}, reference {j.ref[bad[0]]}: "
                          f"{j.ratio[bad[0]]:.3g} delta from v64 (delta = {j.delta:.3g}, total {ref.sigma:.6g})")
    np.testing.assert_array_equal(idx[j.far], j.ref[j.far], err_msg=f"{what}: far from every boundary, off the reference")
    if root > 0:
        np.testing.assert_array_equal(prob, (leaves[idx] / np.float32(root)).astype(np.float32), err_msg=what)
        want = leaves[idx].astype(np.float64) / ref.sigma
        assert (np.abs(prob - want) <= (31 * ref.h + 2) * P.EPS32 * want).all(), what
    else:
        assert (prob == 0).all() and (idx == 0).all(), what
    return float(j.ratio.max())


def _check_weights(w, prob, count, beta0, steps, what):
    want = R.importance_weights(prob, P.beta32(count, beta0, steps))
    np.testing.assert_allclose(w, want, rtol=2e-6, atol=0, err_msg=what)


def _run_case(ring, rainbow, leaves, rng, label):
    """Every uniform set of one tree; prints the worst distance over δ."""
    ref = P.Reference(leaves)
    root = float(ring.tree[-1].item())
    sampler = _Sampler(ring, rainbow)
    worst = 0.0
    for name, u in _uniform_sets(leaves, rng):
        u, idx, prob, w = sampler.run(u)
        worst = max(worst, _check_draws(ref, leaves, root, u, idx, prob, f"{label}, {name}"))
        if w is not None:
            _check_weights(w, prob, None, BETA0, STEPS, f"{label}, {name}")
    print(f"[prio tree] {label}: height {ref.h}, worst draw distance / delta {worst:.3g}")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("items", list(RAINBOW))
def test_rainbow_draws_against_the_fp64_inverse_cdf(items, kind):
    rng = np.random.default_rng(items * 10 + KINDS.index(kind))
    ring = _rainbow_ring(items, kind, 1.0)
    leaves = _set_all(ring, ops.replay_set_priorities, kind, 1.0, rng)
    _run_case(ring, True, leaves, rng, f"rainbow {items} items, {kind}")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("items", list(R2D2))
def test_r2d2_draws_against_the_fp64_inverse_cdf(items, kind):
    rng = np.random.default_rng(items * 10 + KINDS.index(kind) + 1)
    ring = _r2d2_ring(items, kind, 1.0)
    leaves = _set_all(ring, ops.r2d2_ring_set_priorities, kind, 1.0, rng)
    _run_case(ring, False, leaves, rng, f"r2d2 {items} items, {kind}")


@pytest.mark.parametrize("rainbow", [True, False])
def test_priority_exponent_one_half(rainbow):
    """alpha = 0.5 (Rainbow's shipped exponent): the leaves come from powf, and the draws are judged on them."""
    rng = np.random.default_rng(5)
    items = 32769 if rainbow else 256000
    ring = (_rainbow_ring if rainbow else _r2d2_ring)(items, "loguniform", 0.5)
    leaves = _set_all(ring, ops.replay_set_priorities if rainbow else ops.r2d2_ring_set_priorities, "loguniform", 0.5, rng)
    _run_case(ring, rainbow, leaves, rng, f"{'rainbow' if rainbow else 'r2d2'} {items} items, log-uniform, alpha 0.5")


@pytest.mark.parametrize("rainbow", [True, False])
def test_fall_through_at_the_root_of_the_two_halves_tree(rainbow):
    """prio_reference.two_halves_tree: v = total (the largest u01 in the last stratum) falls through at the root; the draw is the last
    leaf, where the earlier rule took leaf 1024, half the mass away."""
    leaves = P.two_halves_tree()
    if rainbow:
        ring = ops.PrioritisedRing(1024, 2, 1, 1, 1.0, "cuda")
        obs = torch.zeros(1024, 2, 1, device="cuda")
        ops.replay_add_prioritised(ring, obs, torch.zeros(1024, 2, dtype=torch.int32, device="cuda"), torch.zeros(1024, 2, device="cuda"),
                                   torch.zeros(1024, 2, dtype=torch.uint8, device="cuda"), obs)
        ops.replay_set_priorities(ring, t_(np.arange(2048, dtype=np.int32)), t_(leaves))
    else:
        ring = ops.R2d2Ring(1024, 2, 1, 1, 1, 1, 1.0, "cuda")
        z = lambda dt=torch.float32: torch.zeros(1024, 2, dtype=dt, device="cuda")
        ops.r2d2_ring_add(ring, z().unsqueeze(-1), z(torch.int32), z(), z(torch.uint8), z(torch.uint8), z(torch.uint8), z().unsqueeze(-1))
        ops.r2d2_ring_set_priorities(ring, t_(np.arange(2048, dtype=np.int32)), t_(leaves))
    np.testing.assert_array_equal(_check_tree(ring.tree, 2048), leaves)   # powf(x, 1) = x: the constructed tree
    u = np.full(M, 0.5, np.float32)
    u[-1] = P.U_MAX
    u, idx, prob, w = _Sampler(ring, rainbow).run(u)
    ref = P.Reference(leaves)
    print(f"[prio tree] two halves ({'rainbow' if rainbow else 'r2d2'}): last draw on leaf {idx[-1]}")
    assert idx[-1] == 2047
    _check_draws(ref, leaves, float(ring.tree[-1].item()), u, idx, prob, "two halves")


def test_importance_weights_against_fp64():
    """Rainbow's weights at a 1e12 probability ratio across the beta schedule (count 0, 1, steps - 1, steps, 10 steps, none, steps 0),
    and R2D2's (1 / (p + 1e-6))^beta weights out of r2d2_loss_grads at the same points; both on the device's own probabilities."""
    rng = np.random.default_rng(9)
    ring = _rainbow_ring(32769, "loguniform", 1.0)
    leaves = _set_all(ring, ops.replay_set_priorities, "loguniform", 1.0, rng)
    sampler = _Sampler(ring, True)
    steps = 1000.0
    points = [(c, steps) for c in (0, 1, 999, 1000, 10000)] + [(None, steps), (7, 0.0)]
    ratio = 0.0
    for count, st in points:
        for u in (np.zeros(M, np.float32), None):
            cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
            _, idx, prob, w = sampler.run(u, count=cnt, steps=st)
            assert (prob > 0).all()
            ratio = max(ratio, float(prob.max() / prob.min()))
            _check_weights(w, prob, count, BETA0, st, f"rainbow count {count} steps {st}")
    print(f"[prio tree] rainbow weights: largest probability ratio in a batch {ratio:.3g}")
    assert ratio > 1e11

    r2 = _r2d2_ring(2048, "loguniform", 1.0)
    _set_all(r2, ops.r2d2_ring_set_priorities, "loguniform", 1.0, rng)
    s2 = _Sampler(r2, False)
    B, A = M, 2
    # T = 2, n = 1, done: the target is h(0) = 0, and q = -1 at the taken action makes every TD error exactly 1, so with B a power of
    # two d_q = -w_b / B exactly
    q = torch.zeros(2, B, A, device="cuda")
    q[0, :, 0] = -1.0
    action, reward, done = torch.zeros(2, B, dtype=torch.int32, device="cuda"), torch.zeros(2, B, device="cuda"), torch.ones(2, B, dtype=torch.uint8, device="cuda")
    for count, st in points:
        _, _, prob, _ = s2.run(np.zeros(M, np.float32) if count == 0 else None)
        cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
        d_q, pr, metrics, td = torch.zeros_like(q), torch.zeros(B, device="cuda"), torch.zeros(6, device="cuda"), torch.zeros(1, B, device="cuda")
        ops.r2d2_loss_grads(q, torch.zeros_like(q), action, reward, done, t_(prob), d_q, pr, metrics, n=1, gamma=0.99, max_abs_reward=1000.0, eta=0.9,
                            beta0=0.6, beta_steps=st, count=cnt, td=td)
        assert (td == 1).all()
        w = -d_q[0, :, 0].double().cpu().numpy() * B
        np.testing.assert_allclose(w, R.importance_weights(prob.astype(np.float64) + 1e-6, P.beta32(count, 0.6, st)), rtol=2e-6, atol=0,
                                   err_msg=f"r2d2 count {count} steps {st}")


@pytest.mark.parametrize("rainbow", [True, False])
def test_set_priorities_at_depth(rainbow):
    """512 indices with duplicates on Rainbow's 999 424-leaf tree (R2D2: 256 000): every parent stays the in-order fp32 sum of its
    children, untouched leaves keep their bits, the last duplicate wins, max_priority rises to the largest new value; the add and the
    set, each run twice from the same state, give the same bits."""
    rng = np.random.default_rng(17)
    items = 999424 if rainbow else 256000
    make, set_fn = (_rainbow_ring, ops.replay_set_priorities) if rainbow else (_r2d2_ring, ops.r2d2_ring_set_priorities)
    ring, ring2 = make(items, "uniform", 0.5), make(items, "uniform", 0.5)   # the add twice
    assert torch.equal(ring.tree, ring2.tree) and torch.equal(ring.state, ring2.state)
    del ring2
    _set_all(ring, set_fn, "uniform", 0.5, rng)
    valid = np.flatnonzero(ring.priorities.cpu().numpy() > 0)
    idx = rng.choice(valid, 512).astype(np.int32)
    idx[100:110] = idx[0]   # the last occurrence (row 109) wins
    idx[300] = idx[5]
    pr = (rng.random(512) * 4).astype(np.float32)
    before, maxp = ring.priorities.cpu().numpy().copy(), float(ring.max_priority.item())
    tree0, max0 = ring.tree.clone(), ring.max_priority.clone()
    set_fn(ring, t_(idx), t_(pr))
    first = ring.tree.clone(), ring.max_priority.clone()
    ring.tree.copy_(tree0), ring.max_priority.copy_(max0)
    set_fn(ring, t_(idx), t_(pr))
    assert torch.equal(ring.tree, first[0]) and torch.equal(ring.max_priority, first[1])
    leaves = _check_tree(ring.tree, items)
    last = {int(i): m for m, i in enumerate(idx)}
    touched = np.array(sorted(last))
    untouched = np.setdiff1d(np.arange(items), touched)
    np.testing.assert_array_equal(leaves[untouched], before[untouched])
    np.testing.assert_allclose(leaves[touched], pr[[last[i] for i in touched]].astype(np.float64) ** 0.5, rtol=1e-6)
    assert leaves[idx[0]] == pytest.approx(float(pr[109]) ** 0.5, rel=1e-6)
    assert ring.max_priority.item() == pytest.approx(max(maxp, float((pr.astype(np.float64) ** 0.5).max())), rel=1e-6)


def test_rainbow_ring_without_a_valid_item():
    """No item has its n rows yet: every draw is item 0 with p 0 and weight 1 (not the NaN of 0 / 0), at every beta."""
    ring = ops.PrioritisedRing(8, 2, 1, 3, 0.5, "cuda")
    obs = torch.zeros(1, 2, 1, device="cuda")
    ops.replay_add_prioritised(ring, obs, torch.zeros(1, 2, dtype=torch.int32, device="cuda"), torch.zeros(1, 2, device="cuda"),
                               torch.zeros(1, 2, dtype=torch.uint8, device="cuda"), obs)
    assert not ring.tree.any()
    sampler = _Sampler(ring, True)
    for u, count, st in ((None, None, 1000.0), (np.full(M, 0.5, np.float32), 10, 20.0), (None, None, 0.0)):
        cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
        _, idx, prob, w = sampler.run(u, count=cnt, steps=st)
        assert (idx == 0).all() and (prob == 0).all() and (w == 1).all()
