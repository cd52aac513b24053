"""fp64 reference of the prioritised replay sampler (stoix_b200/csrc/stx_prio_tree.cuh, the sum tree of Rainbow's and R2D2's rings)
  --  TEST INFRASTRUCTURE, NumPy only.

The sampler promises stratified, proportional sampling (include/stx.h): draw r of M, with uniform u, takes the position
v = (r + u) total / M in the priority mass and returns the leaf whose cumulative interval holds it.  The device walks a fan-out-32 tree
of fp32 sums; this module states the same draw in fp64 and bounds how far fp32 rounding may move it.

  * `Reference`: Σ = the fp64 sum of the device's fp32 leaves, C_i their fp64 cumulative sums, v64 = (r + u) Σ / M.  The draw is
    the first leaf with C_i > v64 (its priority is then positive); if v64 >= Σ, the last positive leaf.  `Reference.judge` measures
    a batch of draws against the bound δ.
  * `delta`: δ = 64 h 2^-24 Σ (h the tree height), the bound on the distance between v64 and the interval [C_{k-1}, C_k] of the leaf
    k an fp32 descent returns; its derivation is in its docstring.
  * `tree_levels` / `descend`: the device's tree (every parent the in-order fp32 sum of its children) and its fp32 descent, restated
    vectorised; `descend(..., fixed=False)` keeps the earlier rule, which after a fall-through enters the first positive child at every
    level below and so lands at the start of the subtree instead of its end.
  * `boundary_uniforms`: (r, u) pairs whose fp32 v lands on a level's fp32 cumulative boundaries, where rounding leaves v at or past
    a node's in-order sum and the descent falls through; `uniform_calls` packs them into M-draw sampler calls.
  * `beta32`: the fp32 importance-sampling schedule of the Rainbow sampler and the R2D2 loss, restated.
  * `two_halves_tree`: a committed 2048-leaf tree on which v = total falls through at the root and the earlier rule misplaces the draw
    by half the mass.
"""
from __future__ import annotations

from typing import List, NamedTuple

import numpy as np

FANOUT = 32
EPS32 = 2.0 ** -24          # unit roundoff of fp32
U_MAX = np.float32(1.0 - 2.0 ** -24)   # the largest u01


def height(items: int) -> int:
    """Levels of the tree over `items` leaves, leaves and root included (prio::tree_height)."""
    n, c = 1, int(items)
    while c > 1:
        c, n = (c + FANOUT - 1) // FANOUT, n + 1
    return n


def _fp32_group_sums(ch: np.ndarray) -> np.ndarray:
    """In-order fp32 sums of consecutive groups of FANOUT: the level padded with zeros, its FANOUT columns added left to right."""
    pad = (-len(ch)) % FANOUT
    g = np.concatenate([ch.astype(np.float32), np.zeros(pad, np.float32)]).reshape(-1, FANOUT)
    s = np.zeros(len(g), np.float32)
    for c in range(FANOUT):
        s = (s + g[:, c]).astype(np.float32)
    return s


def tree_levels(leaves: np.ndarray) -> List[np.ndarray]:
    """The device's tree over fp32 leaves: levels leaves first, root last, each parent the in-order fp32 sum of its children."""
    levels = [np.asarray(leaves, np.float32)]
    while len(levels[-1]) > 1:
        levels.append(_fp32_group_sums(levels[-1]))
    return levels


def split_levels(tree: np.ndarray, items: int) -> List[np.ndarray]:
    """The flat device tree (stx_prio_tree_floats floats) as its levels, leaves first."""
    out, off, c = [], 0, int(items)
    while True:
        out.append(np.asarray(tree[off:off + c], np.float32))
        if c <= 1:
            return out
        off, c = off + c, (c + FANOUT - 1) // FANOUT


def device_v(r, u, root: float, M: int) -> np.ndarray:
    """v = ((r + u) root) / M with every operation rounded to fp32, as tree_descend forms it."""
    x = (np.asarray(r).astype(np.float32) + np.asarray(u, np.float32)).astype(np.float32)
    return ((x * np.float32(root)).astype(np.float32) / np.float32(M)).astype(np.float32)


def descend(levels: List[np.ndarray], v: np.ndarray, fixed: bool = True) -> np.ndarray:
    """tree_descend for every v (fp32) at once: at each node the children in order, entering the first with v < s, else v -= s (fp32).
    If none takes v (a fall-through), the last child with s > 0; with `fixed`, v becomes +inf, so every level below also takes its last
    positive child and the draw ends on the last positive leaf of the subtree.  Without `fixed` (the earlier rule) v keeps the
    remainder, about 0, and the levels below enter their first positive child."""
    v = np.array(v, np.float32, copy=True)
    node = np.zeros(len(v), np.int64)
    cols = np.arange(FANOUT)
    for lv in range(len(levels) - 1, 0, -1):
        ch = levels[lv - 1]
        c0 = node * FANOUT
        idx = c0[:, None] + cols[None, :]
        s = np.where(idx < len(ch), ch[np.minimum(idx, len(ch) - 1)], np.float32(0)).astype(np.float32)
        pick = np.full(len(v), -1, np.int64)
        last_pos = np.zeros(len(v), np.int64)
        for c in range(FANOUT):   # children past the level's end are 0: neither entered nor positive, and v -= 0 keeps v
            sc = s[:, c]
            last_pos = np.where(sc > 0, c, last_pos)
            open_ = pick < 0
            take = open_ & (v < sc)
            pick = np.where(take, c, pick)
            with np.errstate(invalid="ignore"):
                v = np.where(open_ & ~take, (v - sc).astype(np.float32), v)
        fell = pick < 0
        if fixed:
            v = np.where(fell, np.float32(np.inf), v)
        node = c0 + np.where(fell, last_pos, pick)
    return node


def delta(sigma: float, h: int) -> float:
    """δ = 64 h 2^-24 Σ: how far an fp32 descent's leaf interval may lie from v64.  First order in u = 2^-24, for a draw k that
    ends on leaf k, with f = (r + u) / M in [0, 1] and S(N) the exact mass below node N:

      * node sums: a parent is the in-order fp32 sum of at most 32 nonnegative children, so its own rounding ρ(N) is at most 31 u S(N).
        The root is R = Σ + Σ_N ρ(N); the descent compares v with the fp32 sums of the subtrees it skips, whose error is the ρ of the
        nodes inside them.  The position error these leave is f (R - Σ) - Σ_skipped ρ = f Σ_other ρ - (1 - f) Σ_skipped ρ.  The nodes of
        one height partition the leaves and both coefficients are at most 1, so each level above the leaves adds at most 31 u Σ:
        31 (h - 1) u Σ in all.  (The fp32 root alone is within the same 31 (h - 1) u Σ of Σ.)
      * forming v = fl(fl(fl(r + u) R) / M): r + u rounds to within ulp(M) / 2, a relative u, and the product and the quotient
        round once each: 3 u Σ.
      * subtractions: a level decides after at most 31 of its children are subtracted (a 32nd remainder only follows a fall-through,
        and the fixed rule no longer reads it), each result at most v <= Σ: 31 (h - 1) u Σ.

    So v64 lies in [C_{k-1} - E, C_k + E] with E = (62 (h - 1) + 3) u Σ <= 64 h u Σ, the 2 h + 59 u Σ left over covering the
    second-order terms.  A fall-through at node N ends on the last positive leaf k of N, C_k = the end of N's mass: falling through
    means v is at or past that end up to E, and N's parent entered N because v was below it, so the same bound holds."""
    return 64.0 * h * EPS32 * sigma


class Judgement(NamedTuple):
    ratio: np.ndarray        # distance of v64 from [C_{k-1}, C_k] over δ, per draw
    far: np.ndarray          # v64 is more than δ from every boundary C_i (and from 0): the draw must equal the reference
    ref: np.ndarray          # the reference draws
    delta: float


class Reference:
    """The fp64 inverse CDF over fp32 leaves (module docstring): Σ = the fp64 sum of the leaves, C_i their fp64 cumulative sums."""

    def __init__(self, leaves: np.ndarray):
        self.leaves = np.asarray(leaves, np.float32)
        self.C = np.cumsum(self.leaves.astype(np.float64))
        self.sigma = float(self.C[-1])
        self.h = height(len(self.leaves))
        self.delta = delta(self.sigma, self.h)
        self.bounds = np.concatenate([[0.0], self.C])
        pos = np.flatnonzero(self.leaves > 0)
        self.last_pos = int(pos[-1]) if len(pos) else -1

    def v64(self, r, u, M: int) -> np.ndarray:
        return (np.asarray(r, np.float64) + np.asarray(u, np.float32).astype(np.float64)) * self.sigma / M

    def draws(self, r, u, M: int) -> np.ndarray:
        """The first leaf with C_i > v64 (its priority is then positive); if v64 >= Σ, the last positive leaf.  With every leaf 0
        there is no positive leaf: leaf 0, where a descent through an all-zero tree ends."""
        v = self.v64(r, u, M)
        if self.last_pos < 0:
            return np.zeros(len(v), np.int64)
        # searchsorted(right) is the first C_i > v64; past the last positive leaf C stays at Σ, so v64 >= Σ clips to it
        return np.minimum(np.searchsorted(self.C, v, side="right"), self.last_pos).astype(np.int64)

    def judge(self, r, u, M: int, got: np.ndarray) -> Judgement:
        """Each draw's distance from v64 over δ, and where it must equal the reference draw."""
        v = self.v64(r, u, M)
        k = np.asarray(got, np.int64)
        lo = np.where(k > 0, self.C[np.maximum(k - 1, 0)], 0.0)
        dist = np.maximum(np.maximum(lo - v, v - self.C[k]), 0.0)
        B = self.bounds
        j = np.searchsorted(B, v)
        near = np.minimum(np.abs(v - B[np.clip(j - 1, 0, len(B) - 1)]), np.abs(B[np.clip(j, 0, len(B) - 1)] - v))
        ratio = dist / self.delta if self.delta > 0 else np.where(dist > 0, np.inf, 0.0)
        return Judgement(ratio, near > self.delta, self.draws(r, u, M), self.delta)


def boundary_uniforms(levels: List[np.ndarray], level: int, M: int, limit: int = 0, rng=None):
    """(r, u) pairs whose fp32 v = device_v(r, u, root, M) lands on the fp32 in-order cumulative sums of level `level`'s nodes (0 =
    the leaves), where the descent's remainders reach a node's sum and fall through.  Zero and repeated boundaries are dropped;
    `limit` keeps that many (the first and last among them).  Where no fp32 u hits a boundary exactly, the nearest v at or above
    it.  Returns (r, u, hit) with hit marking the exact ones."""
    root = np.float32(levels[-1][0])
    b = np.unique(np.cumsum(levels[level], dtype=np.float32))
    b = b[b > 0]
    if limit and len(b) > limit:
        rng = rng or np.random.default_rng(0)
        keep = np.concatenate([[0, len(b) - 1], rng.choice(np.arange(1, len(b) - 1), limit - 2, replace=False)])
        b = b[np.sort(keep)]
    t = b.astype(np.float64)
    x = t * M / float(root)
    r = np.clip(np.floor(x), 0, M - 1).astype(np.int64)
    best_u = np.full(len(t), U_MAX, np.float32)
    best_err = np.full(len(t), np.inf)
    hit = np.zeros(len(t), bool)
    x32 = x.astype(np.float32)
    cands = [x32]
    lo = hi = x32
    for _ in range(6):
        lo, hi = np.nextafter(lo, np.float32(-1)), np.nextafter(hi, np.float32(2 * M))
        cands += [lo, hi]
    for xc in cands:
        uc = (xc - r.astype(np.float32)).astype(np.float32)   # exact: r <= xc <= 2 r, or r = 0
        uc = np.where(uc >= 1, U_MAX, uc).astype(np.float32)
        ok = (uc >= 0) & (uc < 1)
        v = device_v(r, uc, root, M).astype(np.float64)
        err = np.where(v >= t, v - t, np.inf)   # at or above the boundary
        exact = ok & (v == t)
        better = ok & ~hit & (exact | (err < best_err))
        best_u = np.where(better, uc, best_u)
        best_err = np.where(better, err, best_err)
        hit |= exact
    return r, best_u, hit


def uniform_calls(r: np.ndarray, u: np.ndarray, M: int, max_calls: int, fill: float = 0.5) -> List[np.ndarray]:
    """Pack (r, u) pairs into sampler calls of M uniforms: the j-th pair of stratum r goes to call j, strata without a pair take
    `fill`; at most max_calls calls (later pairs of a crowded stratum are dropped)."""
    order = np.argsort(r, kind="stable")
    r, u = r[order], u[order]
    first = np.searchsorted(r, r, side="left")
    slot = np.arange(len(r)) - first
    calls = []
    for j in range(min(max_calls, int(slot.max()) + 1 if len(r) else 0)):
        c = np.full(M, np.float32(fill), np.float32)
        c[r[slot == j]] = u[slot == j]
        calls.append(c)
    return calls


def beta32(count, beta0: float, steps: float) -> np.float32:
    """beta of the importance weights as the Rainbow sampler and the R2D2 loss evaluate it in fp32: c = clip(count, 0, steps),
    beta = (beta0 - 1)(1 - c / steps) + 1, each operation rounded; beta0 when steps <= 0; count None is 0.  Its rounding (a few
    2^-24 relative) moves a weight (p_min / p)^beta by that much times |log w|: 3e-6 at a 1e12 probability ratio, so the weights are
    checked against fp64 at this beta, and this beta against the fp64 schedule."""
    f = np.float32
    b0 = f(beta0)
    if not steps > 0:
        return b0
    c = f(min(max(float(count or 0), 0.0), float(f(steps))))
    return f(f(f(b0 - f(1)) * f(f(1) - f(c / f(steps)))) + f(1))


def two_halves_tree() -> np.ndarray:
    """2048 leaves, two root children: every leaf 2^-10 except leaf 0, 2^-10 + 3 2^-23.  Every sum below the root is exact, so the
    children are 1 + 3 2^-23 and 1, and the root rounds up to 2 + 4 2^-23.  v = total (the last stratum at u = U_MAX) leaves the
    remainder 1 + 2^-23 >= 1 after the first child: the descent falls through at the root, and the earlier rule then lands on leaf
    1024, the start of the second half, half the mass from v64."""
    x = np.full(2048, 2.0 ** -10, np.float32)
    x[0] = np.float32(2.0 ** -10 + 3 * 2.0 ** -23)
    return x
