"""Restatements of the categorical action samplers and fp64 references of the categorical heads  --  TEST INFRASTRUCTURE.

Samplers, from their Philox4x32-10 streams (oracle/synth_env.philox4x32 and u01, the counter layouts of include/stx.h):
  * `gumbel_actions`: stx_categorical's Gumbel-max draw (and the fused bf16 rollout's, which uses the same counters).  Action j
    takes word j & 3 of Philox(seed lo, seed hi; row lo, call lo, (call >> 32) ^ ((row >> 32) << 16) ^ ((j / 4) << 24), "CATG").
    The scores z_j - log(-log u_j) are evaluated in fp64 from the exact fp32 u_j; the argmax is the first index on exact ties (the
    kernel's strict `>`), and the fp64 margin between the two best scores says where an fp32 evaluation may pick the other one.
  * `mpo_draws`: the inverse-CDF draw of mpo_rows_kernel, u = u01(word 0 of Philox(seed lo, seed hi; ctr lo, ctr hi, call lo,
    "MPOA" ^ call hi)), ctr = n M + i, against the fp64 softmax; with each draw's distance from the nearest cumulative boundary and
    an fp32 emulation of the kernel's running sum (exp rounded to fp32 from fp64, so the emulation is the same on every CPU),
    which shows where the fp32 sum ends below the largest u01 and leaves a remainder.

Heads: the fp64 log-softmax, entropy, KL and PPO head gradients are those of oracle/ppo_oracle.py and tests/ppo_variants_oracle.py.

`edge_rows` builds the logit rows where categorical heads go wrong: gaps between the best logit and the others from 0 to 1e4 (past
the fp32 underflow of exp at ~88 / ~104 and of every fp64 probability at ~745), common offsets up to +-1e5 (where lse = zmax +
log(sum) absorbs the low bits of log(sum)), all-equal rows, exact ties at the maximum with -0.0 / +0.0, and taken actions that are
the most and the least probable."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from oracle import ppo_oracle as O
from oracle.synth_env import philox4x32, u01
from tests import ppo_variants_oracle as PV

TAG_CATG = 0x43415447
TAG_MPOA = 0x4D504F41
MAX_GUMBEL_ACTIONS = 1024   # 256 groups of 4 in the 8-bit group field of the counter
M32 = 0xFFFFFFFF

log_softmax = O.log_softmax
categorical_log_prob = O.categorical_log_prob
categorical_entropy = O.categorical_entropy
categorical_kl = PV.categorical_kl
ppo_clip_head = O.actor_loss_and_dlogits
ppo_penalty_head = PV.penalty_actor_loss_and_dlogits

GAPS = (0.0, 1e-3, 1.0, 10.0, 30.0, 88.0, 90.0, 104.0, 110.0, 1e4)
OFFSETS = (0.0, 1e3, -1e3, 1e5, -1e5)


def ulp32(x) -> np.ndarray:
    """The spacing of fp32 at |x| (fp64)."""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def split_seed(seed: int):
    seed = int(seed) & ((1 << 64) - 1)
    return seed & M32, seed >> 32


# ------------------------------------------------------------------------------------------------ Gumbel-max (stx_categorical)


def gumbel_counters(rows, call: int, groups):
    """The Philox counter words (c0, c1, c2, c3) of (row, group) for one call, broadcast to (rows, groups)."""
    rows = np.asarray(rows, np.uint64).reshape(-1, 1)
    groups = np.asarray(groups, np.uint64).reshape(1, -1)
    call = int(call) & ((1 << 64) - 1)
    c0 = rows & np.uint64(M32)
    c1 = np.uint64(call & M32)
    c2 = (np.uint64(call >> 32) ^ (((rows >> np.uint64(32)) << np.uint64(16)) & np.uint64(M32))
          ^ ((groups << np.uint64(24)) & np.uint64(M32)))
    c3 = np.uint64(TAG_CATG)
    return np.broadcast_arrays(c0, c1, c2, c3)


def gumbel_uniforms(seed: int, call: int, rows, A: int) -> np.ndarray:
    """u (len(rows), A) fp32: the uniform of action j is u01 of word j & 3 of group j / 4."""
    k0, k1 = split_seed(seed)
    G = (A + 3) // 4
    w = philox4x32(*gumbel_counters(rows, call, np.arange(G)), k0, k1)   # 4 x (rows, G)
    words = np.stack(w, axis=-1).reshape(len(np.atleast_1d(rows)), 4 * G)[:, :A]
    return u01(words)


class GumbelDraw(NamedTuple):
    action: np.ndarray   # (E,) int64: fp64 argmax, first index on exact ties
    margin: np.ndarray   # (E,) fp64: best score - second best (inf for A = 1)
    scale: np.ndarray    # (E,) fp64: max(1, |z|, |noise|) over the two best actions, the magnitude their fp32 scores are rounded at
    score: np.ndarray    # (E, A) fp64 scores


def gumbel_actions(logits32: np.ndarray, seed: int, call: int, rows=None) -> GumbelDraw:
    """stx_categorical's draw for logits (E, A) fp32 of rows `rows` (default 0..E-1) at call = offset + *dev_counter."""
    z = np.asarray(logits32, np.float32).astype(np.float64)
    E, A = z.shape
    rows = np.arange(E) if rows is None else np.asarray(rows)
    u = gumbel_uniforms(seed, call, rows, A).astype(np.float64)
    noise = -np.log(-np.log(u))
    s = z + noise
    a = np.argmax(s, axis=1)
    r = np.arange(E)
    if A == 1:
        margin = np.full(E, np.inf)
        scale = np.maximum(1.0, np.maximum(np.abs(z[:, 0]), np.abs(noise[:, 0])))
    else:
        top2 = np.argsort(-s, axis=1, kind="stable")[:, :2]
        margin = s[r, top2[:, 0]] - s[r, top2[:, 1]]
        mags = np.maximum(np.abs(np.take_along_axis(z, top2, 1)), np.abs(np.take_along_axis(noise, top2, 1)))
        scale = np.maximum(1.0, mags.max(axis=1))
    return GumbelDraw(a, margin, scale, s)


def check_gumbel_actions(got: np.ndarray, ref: GumbelDraw, what: str, max_near_tie_frac: float = 1e-3) -> int:
    """The kernel's action equals the fp64 argmax wherever the top-two margin exceeds 2^-20 scale; where it does not, the kernel's
    action must itself score within that band of the best.  Returns the number of such near ties (bounded by max_near_tie_frac)."""
    got = np.asarray(got, np.int64)
    E, A = ref.score.shape
    assert got.shape == (E,) and got.min() >= 0 and got.max() < A, f"{what}: action out of range"
    tol = 2.0 ** -20 * ref.scale
    clear = ref.margin > tol
    bad = np.flatnonzero(clear & (got != ref.action))
    assert bad.size == 0, (f"{what}: {bad.size} draws differ from the Philox restatement, rows {bad[:8].tolist()}: "
                           f"kernel {got[bad[:8]].tolist()} reference {ref.action[bad[:8]].tolist()} margins {ref.margin[bad[:8]].tolist()}")
    near = np.flatnonzero(~clear)
    if near.size:
        best = ref.score[near, ref.action[near]]
        picked = ref.score[near, got[near]]
        off = near[best - picked > tol[near]]
        assert off.size == 0, f"{what}: near-tie rows {off[:8].tolist()} drew an action outside the tie"
    assert near.size <= max_near_tie_frac * E, f"{what}: {near.size} near ties in {E} rows"
    return int(near.size)


# ------------------------------------------------------------------------------------------------ MPO inverse CDF


class MpoDraws(NamedTuple):
    u: np.ndarray          # (N, M) fp32 uniforms
    action: np.ndarray     # (N, M) fp64 inverse CDF: the first j with u < C_j
    distance: np.ndarray   # (N, M) fp64 distance of u from the nearest cumulative boundary C_0 .. C_{A-1}
    prob: np.ndarray       # (M, A) fp64 softmax
    sum32: np.ndarray      # (M,) fp32 emulation of the kernel's running sum after the last action
    action32: np.ndarray   # (N, M) the draw of that emulation, the remainder to the last action of positive fp32 probability


def mpo_uniforms(seed: int, call: int, N: int, M: int) -> np.ndarray:
    k0, k1 = split_seed(seed)
    call = int(call) & ((1 << 64) - 1)
    ctr = np.arange(N * M, dtype=np.uint64)
    w0, _, _, _ = philox4x32(ctr & np.uint64(M32), ctr >> np.uint64(32), np.uint64(call & M32), np.uint64(TAG_MPOA ^ (call >> 32)), k0, k1)
    return u01(w0).reshape(N, M)


def softmax_fp32_emulation(logits32: np.ndarray) -> np.ndarray:
    """(M, A) fp32 probabilities as the kernel forms them: zmax, se = sum expf(z - zmax), lse = zmax + logf(se), p = expf(z - lse),
    every operation rounded to fp32 (exp and log from fp64)."""
    z = np.asarray(logits32, np.float32)
    zmax = z.max(axis=1, keepdims=True)
    e = np.exp((z - zmax).astype(np.float64)).astype(np.float32)
    se = np.zeros((z.shape[0], 1), np.float32)
    for j in range(z.shape[1]):
        se = (se + e[:, j:j + 1]).astype(np.float32)
    lse = (zmax + np.log(se.astype(np.float64)).astype(np.float32)).astype(np.float32)
    return np.exp((z - lse).astype(np.float64)).astype(np.float32)


def mpo_draws(logits32: np.ndarray, seed: int, call: int, N: int, M: int) -> MpoDraws:
    z = np.asarray(logits32, np.float32)
    assert z.shape[0] == M
    A = z.shape[1]
    u = mpo_uniforms(seed, call, N, M)
    u64 = u.astype(np.float64)
    p = np.exp(log_softmax(z.astype(np.float64)))
    C = np.cumsum(p, axis=1)
    act = np.zeros((N, M), np.int64)
    dist = np.full((N, M), np.inf)
    for j in range(A):
        act += (C[None, :, j] <= u64)
        dist = np.minimum(dist, np.abs(u64 - C[None, :, j]))
    act = np.minimum(act, A - 1)
    p32 = softmax_fp32_emulation(z)
    cum = np.zeros(M, np.float32)
    act32 = np.full((N, M), -1, np.int64)
    last = np.zeros(M, np.int64)
    for j in range(A):
        cum = (cum + p32[:, j]).astype(np.float32)
        last = np.where(p32[:, j] > 0, j, last)
        act32 = np.where((act32 < 0) & (u < cum[None, :]), j, act32)
    act32 = np.where(act32 < 0, last[None, :], act32)
    return MpoDraws(u, act, dist, p, cum, act32)


class RemainderCase(NamedTuple):
    logits: np.ndarray   # (M, A) fp32, the last logit -200 (fp32 probability 0)
    seed: int
    call: int
    N: int
    M: int


U_HIGH = 1.0 - 2.0 ** -22       # a u01 at or above this ...
SUM_LOW = 1.0 - 2.0 ** -21      # ... on a row whose fp32 sum is at or below this falls in the remainder, with 2^-22 to spare


def mpo_remainder_case() -> RemainderCase:
    """Bootstrap rows whose fp32 running sum ends at or below 1 - 2^-21 (about 0.3 % of random rows of 32 logits), and a seed
    whose 4.2M draws include u01 values at or above 1 - 2^-22: those draws fall in the remainder of the inverse CDF."""
    A, M, N = 32, 256, 16384
    z = np.random.default_rng(2024).standard_normal((200000, A)).astype(np.float32)
    z[:, -1] = -200.0
    p32 = softmax_fp32_emulation(z)
    cum = np.zeros(len(z), np.float32)
    for j in range(A):
        cum = (cum + p32[:, j]).astype(np.float32)
    rows = np.flatnonzero(cum <= np.float32(SUM_LOW))[:M]
    assert rows.size == M
    return RemainderCase(z[rows], 14, (1 << 32) + 7, N, M)


def inverse_cdf(p: np.ndarray, u: float) -> int:
    """The first j with u < p_0 + ... + p_j (fp64), the last index if u is at or above the whole sum."""
    return int(min(np.searchsorted(np.cumsum(np.asarray(p, np.float64)), u, side="right"), len(p) - 1))


# ------------------------------------------------------------------------------------------------ edge families of logit rows


def edge_rows(A: int, rng: np.random.Generator):
    """Logit rows (R, A) fp32 and a taken action per row (R,) int32 over the edge families; every row appears with its most
    probable action and (A > 1) with its least probable one."""
    rows, acts = [], []

    def add(z):
        z = np.asarray(z, np.float32)
        z64 = z.astype(np.float64)
        rows.extend([z, z])
        acts.extend([int(np.argmax(z64)), int(np.argmin(z64))])

    for off in OFFSETS:
        add(np.full(A, off))                                        # all equal
        for gap in GAPS:
            k = int(rng.integers(A))
            z = np.full(A, off, np.float64)
            z[k] = off + gap                                        # one dominant logit
            add(z)
            add(off - gap * rng.permutation(np.linspace(0.0, 1.0, A)))   # spread over [off - gap, off]
            add(off + gap * rng.standard_normal(A) / 3.0)           # random at scale gap
    if A >= 2:                                                       # exact ties at the maximum, signed zeros
        for lead in ((-0.0, 0.0), (0.0, -0.0), (0.0, 0.0), (-0.0, -0.0)):
            for low in (-1.0, -30.0, -110.0):
                z = np.full(A, low, np.float32)
                z[0], z[A - 1] = lead
                add(z)
                z = np.full(A, low, np.float32)
                z[A // 2], z[0] = lead
                add(z)
    return np.stack(rows).astype(np.float32), np.asarray(acts, np.int32)
