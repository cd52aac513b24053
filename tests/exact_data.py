"""Exactly representable data for the bf16 tensor-core kernels -- TEST INFRASTRUCTURE (like golden_runner.py).

Why exact data.  The tensor-core kernels round every GEMM operand to bf16 and accumulate in fp32 in an order of their
own (wgmma K steps, split-K CTAs, a fixed-order reduce).  On random data that order shows in the last bits, so the
gradient checks of tests/test_tc_gpu.py are norm-wise (5e-3 per tensor), and a kernel that drops or re-reads one row
of a 32768-row minibatch still passes them.  Here every operand and every intermediate is exactly representable:

* weights in {-1, 0, +1} (sparse, with bounded nonzeros per row and column), small integer biases, observations in
  {-1, 0, +1}: every forward value is an integer, and |h1|, |h2| <= 256 are exact in bf16 (8 significant bits);
* critic targets = value + a nonzero integer in +-[1, 7], a huge clip_eps (or v_old = value), vf_coef 0.5 and a
  power-of-two minibatch: dz = dv * 0.5 / mb is an integer multiple of the grid 0.5 / mb, and so are dh2, dh1 and
  every weight gradient;
* every fp32 accumulation (a GEMM's K loop, a whole-minibatch split-K sum on one CTA, the bias and metric sums) stays
  below 2^20 grid units, whatever the order: fp32 holds 2^24 units exactly, the rest is margin for the truncating
  alignment inside the tensor-core accumulator.

Then the kernels' results are exact, the fp64 oracle agrees bit for bit, and so does every reduction order: one
misplaced row is a hard failure at any shape.  `check_forward` / `check_ppo` assert all of the above on the data they
are given and are run on the CPU (tests/test_exact_data.py) at every shape the GPU tests use.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import ppo_oracle as O

H = 256
ACC_LIMIT = 2 ** 20          # grid units any fp32 accumulation may reach
VF_COEF = 0.5
BIG_CLIP = 1e6               # dv = v - target exactly, whatever v_old
_TERNARY = np.array([-1, 0, 0, 1], np.int8)   # P(0) = 1/2: sparse activations keep the minibatch sums small
_DV = np.arange(1, 8)                          # |value - target|, P(k) ~ 2^-k: mean 2, so that dW2 = h2^T dz over
_DV_P = 0.5 ** _DV / (0.5 ** _DV).sum()        # 65536 rows stays below ACC_LIMIT

# ---- the shapes the GPU tests run (tests/test_tc_exact_gpu.py); tests/test_exact_data.py self-checks every one ----
# K1 forward: (M, D, A).  M: one row, partial tiles, 2 x 132 tiles (one per warpgroup of a full grid) and one row more,
# and 8193 tiles; D not a multiple of 16 and heads of 9 - 15 columns (zero-filled K and N).
FORWARD_CASES = [(1, 64, 8), (63, 8, 1), (65, 24, 3), (64 * 264, 40, 9), (64 * 264 + 1, 56, 15), (524288 + 37, 64, 16),
                 (524288 + 37, 24, 9)]
# K3 critic: (B, mb_off, mb, D, A_actor, use_perm).  B = 524352 > 2^19: permutation indices >= 2^19.
CRITIC_CASES = [(384, 128, 128, 24, 16, True), (1024, 512, 256, 8, 3, False), (16384, 4096, 8192, 64, 8, True),
                (524352, 5 * 32768, 32768, 64, 8, True), (524352, 458752, 65536, 24, 9, True),
                (524352, 524352 - 65536 - 64, 65536, 8, 16, False), (131072, 0, 32768, 24, 1, False)]
# K3 actor, hot rows: (B, mb_off, mb, D, A)
HOT_CASES = [(16384, 4096, 8192, 64, 8), (524352, 3 * 32768, 32768, 24, 16)]
# K3 on a workspace sized for mb = 32768, then mb = 128 on the same workspace: (B, D, A, windows)
STALE_CASE = (65536, 24, 8, [(0, 32768), (32768, 128)])


def ternary(rng: np.random.Generator, shape) -> np.ndarray:
    return _TERNARY[rng.integers(0, 4, size=shape)]


def exact_mlp(rng: np.random.Generator, D: int, A: int, head_density: float) -> O.MLPParams:
    """MLP [D, 256, 256, A] with weights in {-1, 0, +1}: <= 4 nonzeros per column of W0, <= 8 per row and column of W1
    (a sum of 8 signed permutations, collisions left out), head entries nonzero with probability `head_density`;
    integer biases b0 in [-1, 1], b1 in [-3, -1], b2 in [-3, 3]."""
    W0 = np.zeros((D, H))
    for j in range(H):
        rows = rng.choice(D, size=min(4, D), replace=False)
        W0[rows, j] = rng.choice([-1.0, 1.0], size=rows.size)
    W1 = np.zeros((H, H))
    for _ in range(8):
        cols = rng.permutation(H)
        free = W1[np.arange(H), cols] == 0
        W1[np.arange(H)[free], cols[free]] = rng.choice([-1.0, 1.0], size=int(free.sum()))
    W2 = rng.choice([-1.0, 0.0, 1.0], size=(H, A), p=[head_density / 2, 1 - head_density, head_density / 2])
    b = [rng.integers(-1, 2, H).astype(np.float64), rng.integers(-3, 0, H).astype(np.float64), rng.integers(-3, 4, A).astype(np.float64)]
    return O.MLPParams([W0, W1, W2], b)


def forward_problem(M: int, D: int, A: int) -> Tuple[O.MLPParams, np.ndarray]:
    """(network, int8 observations (M, D)) of FORWARD_CASES entry (M, D, A)."""
    rng = np.random.default_rng(M + 100 * D + A)
    return exact_mlp(rng, D, A, 1.0 / 8), ternary(rng, (M, D))


def forward(p: O.MLPParams, x: np.ndarray, chunk: int = 65536) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(out, h1, h2) as float32 from the unrounded fp64 oracle (equal to the bf16-operand oracle on this data:
    check_forward), in row chunks to bound host memory."""
    M = x.shape[0]
    out, h1, h2 = np.empty((M, p.W[2].shape[1]), np.float32), np.empty((M, H), np.float32), np.empty((M, H), np.float32)
    for r in range(0, M, chunk):
        o, acts = O.mlp_forward(p, x[r:r + chunk].astype(np.float64))
        out[r:r + chunk], h1[r:r + chunk], h2[r:r + chunk] = o, acts[1], acts[2]
    return out, h1, h2


def _exact_in(x: np.ndarray, dtype) -> bool:
    x = np.asarray(x, np.float64)
    return bool(np.array_equal(x.astype(dtype).astype(np.float64), x))


def _bf16_exact(x: np.ndarray) -> bool:
    x = np.asarray(x, np.float64)
    return _exact_in(x, np.float32) and bool(np.array_equal(O._bf16_round(x.astype(np.float32)).astype(np.float64), x))


def _on_grid(x: np.ndarray, unit: float) -> bool:
    q = np.asarray(x, np.float64) / unit
    return bool(np.array_equal(q, np.round(q)))


def check_forward(p: O.MLPParams, x_sample: np.ndarray) -> Dict[str, float]:
    """Asserts that the forward pass of `p` is exact in bf16 for EVERY input row in {-1, 0, +1}^D (a bound per hidden
    unit from the weights alone: |h1| <= |W0|^T 1 + |b0| etc.), and that on `x_sample` the bf16-operand oracle equals
    the unrounded fp64 oracle bit for bit and some pre-activations sit exactly at the ReLU kink.  Returns the bounds."""
    W0, W1, W2 = (np.abs(w) for w in p.W)
    assert all(np.isin(w, (-1.0, 0.0, 1.0)).all() for w in p.W) and all(_on_grid(b, 1.0) for b in p.b)
    h1max = W0.sum(0) + np.abs(p.b[0])
    h2max = h1max @ W1 + np.abs(p.b[1])
    outmax = h2max @ W2 + np.abs(p.b[2])
    assert h1max.max() <= 256 and h2max.max() <= 256, "hidden activations must be integers of <= 8 significant bits"
    assert outmax.max() < ACC_LIMIT
    x = x_sample.astype(np.float64)
    assert np.isin(x, (-1.0, 0.0, 1.0)).all()
    ref, ra = O.mlp_forward(p, x)
    got, ga = O.mlp_forward(p, x, bf16_operands=True)
    assert np.array_equal(got, ref) and all(np.array_equal(ga[i], ra[i]) for i in range(3))
    assert _exact_in(ref, np.float32)
    kinks = [int((ra.pre[i] == 0).sum()) for i in range(2)]
    assert min(kinks) > 0, "want pre-activations exactly at the ReLU kink"
    return {"h1max": float(h1max.max()), "h2max": float(h2max.max()), "outmax": float(outmax.max()), "kinks": float(min(kinks))}


# ------------------------------------------------------------------------------------------------------------------
# K3: one PPO minibatch
# ------------------------------------------------------------------------------------------------------------------


@dataclass
class PpoProblem:
    actor: O.MLPParams
    critic: O.MLPParams
    obs: np.ndarray        # int8 (B, D) in {-1, 0, +1}
    action: np.ndarray     # int32 (B,)
    logp_old: np.ndarray   # float32 (B,)
    v_old: np.ndarray
    adv: np.ndarray        # raw advantages; the kernels are called with standardize=False
    tgt: np.ndarray
    perm: Optional[np.ndarray]
    clip_eps: float
    ent_coef: float = 0.0
    vf_coef: float = VF_COEF

    def rows(self, mb_off: int, mb: int) -> np.ndarray:
        return self.perm[mb_off:mb_off + mb].astype(np.int64) if self.perm is not None else np.arange(mb_off, mb_off + mb)


def ppo_problem(B: int, D: int, A: int, windows: Sequence[Tuple[int, int]], seed: int, use_perm: bool = True,
                hot: Optional[Dict[int, float]] = None) -> PpoProblem:
    """Exact PPO data on B rows; loss inputs are filled for the rows of the minibatches `windows` [(mb_off, mb), ...].

    hot=None (critic mode): advantages 0 and ent_coef 0, so the actor gradient is exactly zero; clip_eps 1e6, v_old =
    value + an integer in [-3, 3], target = value - an integer in +-[1, 7] (dv never 0, small |dv| likelier).
    hot={minibatch position: advantage} (actor mode): those rows of the FIRST window carry the given advantage, every
    other row 0; clip_eps 0.2 with logp_old = the oracle's log-prob (ratio ~ 1, inside the band) and v_old = value, so the
    critic stays exact."""
    rng = np.random.default_rng(seed)
    actor, critic = exact_mlp(rng, D, A, 1.0 / 16), exact_mlp(rng, D, 1, 1.0 / 8)
    obs = ternary(rng, (B, D))
    action = rng.integers(0, A, B).astype(np.int32)
    perm = rng.permutation(B).astype(np.int32) if use_perm else None
    z = lambda: np.zeros(B, np.float32)
    pb = PpoProblem(actor, critic, obs, action, z(), z(), z(), z(), perm, BIG_CLIP if hot is None else 0.2)
    for w, (mb_off, mb) in enumerate(windows):
        idx = pb.rows(mb_off, mb)
        x = obs[idx].astype(np.float64)
        v = O.mlp_forward(critic, x)[0][:, 0]
        k = rng.choice(_DV, size=mb, p=_DV_P) * rng.choice([-1, 1], mb)
        pb.tgt[idx] = v - k
        if hot is None:
            pb.v_old[idx] = v + rng.integers(-3, 4, mb)
        else:
            pb.v_old[idx] = v
            lg = O.mlp_forward(actor, x)[0]
            pb.logp_old[idx] = O.categorical_log_prob(lg, action[idx])
            if w == 0:
                for pos, a in hot.items():
                    pb.adv[idx[pos]] = a
    return pb


def critic_problem(B: int, mb_off: int, mb: int, D: int, A: int, use_perm: bool) -> PpoProblem:
    """The problem of CRITIC_CASES entry (B, mb_off, mb, D, A, use_perm)."""
    return ppo_problem(B, D, A, [(mb_off, mb)], seed=B + mb + D, use_perm=use_perm)


def hot_problem(B: int, mb_off: int, mb: int, D: int, A: int) -> PpoProblem:
    """The problem of HOT_CASES entry (B, mb_off, mb, D, A): advantages +-1, +-2 at hot_positions(mb)."""
    hot = {pos: (-1.0) ** k * (1 + k % 2) for k, pos in enumerate(hot_positions(mb))}
    return ppo_problem(B, D, A, [(mb_off, mb)], seed=B + mb + A, hot=hot)


def arena_layout(D: int, A: int) -> Tuple[int, int, int, int]:
    """(actor param count, critic offset, critic param count, arena size): the padded layout of ops.arena_offsets."""
    count = lambda n_out: D * H + H + H * H + H + H * n_out + n_out
    na, nc = count(A), count(1)
    coff = (na + 7) // 8 * 8
    return na, coff, nc, coff + (nc + 7) // 8 * 8


def ppo_oracle(pb: PpoProblem, mb_off: int, mb: int, bf16: bool = True, rows: Optional[np.ndarray] = None,
               obs_rows: Optional[np.ndarray] = None):
    """The minibatch gradient (flat arena, float64) and the six metrics [actor_loss, entropy, value_loss, adv mean, value
    mean, target mean] of ff_ppo's losses; `rows` / `obs_rows` override which rows are summed / whose observations are
    read (fault models of tests/test_exact_data.py).  1/mb scaling as in the kernels: the loss is a mean over mb rows."""
    idx = pb.rows(mb_off, mb) if rows is None else rows
    x = pb.obs[idx if obs_rows is None else obs_rows].astype(np.float64)
    m_scale = len(idx) / mb   # oracle means are over len(idx) rows; the kernels divide by mb
    D, A = pb.obs.shape[1], pb.actor.W[2].shape[1]
    na, coff, nc, total = arena_layout(D, A)
    g = np.zeros(total)
    lg, aa = O.mlp_forward(pb.actor, x, bf16)
    _, dlg, ai = O.actor_loss_and_dlogits(lg, pb.action[idx], pb.logp_old[idx].astype(np.float64), pb.adv[idx].astype(np.float64),
                                          pb.clip_eps, pb.ent_coef)
    g[:na] = O.mlp_backward(pb.actor, aa, dlg * m_scale, bf16).flat()
    v, ca = O.mlp_forward(pb.critic, x, bf16)
    _, dv, ci = O.critic_loss_and_dvalue(v[:, 0], pb.v_old[idx].astype(np.float64), pb.tgt[idx].astype(np.float64), pb.clip_eps, pb.vf_coef)
    g[coff:coff + nc] = O.mlp_backward(pb.critic, ca, dv[:, None] * m_scale, bf16).flat()
    metrics = np.array([ai["actor_loss"], ai["entropy"], ci["value_loss"], pb.adv[idx].mean(), v[:, 0].mean(),
                        pb.tgt[idx].astype(np.float64).mean()]) * m_scale
    return g, metrics


def check_ppo(pb: PpoProblem, mb_off: int, mb: int) -> Dict[str, float]:
    """Asserts, for the critic of minibatch [mb_off, mb_off + mb): the bf16-operand oracle equals the unrounded fp64
    oracle bit for bit (gradient and value_loss / value mean / target mean) and is fp32-representable; dz, dh2, dh1 are
    bf16-exact multiples of the grid 0.5 / mb; every accumulation the kernels make (dh GEMMs, the three weight-gradient
    GEMMs over the whole minibatch, the bias column sums, the metric sums) stays below ACC_LIMIT grid units.  Returns
    the largest accumulation per quantity, in grid units."""
    assert mb & (mb - 1) == 0, "1/mb must be exact"
    idx = pb.rows(mb_off, mb)
    x = pb.obs[idx].astype(np.float64)
    D, A = pb.obs.shape[1], pb.actor.W[2].shape[1]
    _, coff, nc, _ = arena_layout(D, A)
    g16, m16 = ppo_oracle(pb, mb_off, mb, bf16=True)
    g64, m64 = ppo_oracle(pb, mb_off, mb, bf16=False)
    assert np.array_equal(g16[coff:coff + nc], g64[coff:coff + nc]) and np.array_equal(m16[2:], m64[2:])
    assert _exact_in(g64[coff:coff + nc], np.float32) and _exact_in(m64[2:], np.float32)
    # the critic's intermediates as the kernels form them
    c = pb.critic
    v, acts = O.mlp_forward(c, x)
    h1, h2 = acts[1], acts[2]
    dv = v[:, 0] - pb.tgt[idx]
    assert _on_grid(dv, 1.0) and (dv != 0).all() and np.abs(dv).max() <= 7
    unit = pb.vf_coef / mb
    dz = pb.vf_coef * dv[:, None] / mb
    dh2 = (dz @ c.W[2].T) * (h2 > 0)
    dh1 = (dh2 @ c.W[1].T) * (h1 > 0)
    for name, t in (("dz", dz), ("dh2", dh2), ("dh1", dh1)):
        assert _on_grid(t, unit) and _bf16_exact(t), f"{name} is not a bf16-exact multiple of 0.5/mb"
    ab = np.abs
    acc = {
        "dh2": (ab(dz) @ ab(c.W[2]).T).max() / unit, "dh1": (ab(dh2) @ ab(c.W[1]).T).max() / unit,
        "dW0": (ab(x).T @ ab(dh1)).max() / unit, "dW1": (ab(h1).T @ ab(dh2)).max() / unit, "dW2": (ab(h2).T @ ab(dz)).max() / unit,
        "db": max(ab(dh1).sum(0).max(), ab(dh2).sum(0).max(), ab(dz).sum()) / unit,
        "value sum": ab(v).sum(), "target sum": ab(pb.tgt[idx].astype(np.float64)).sum(), "loss sum": (dv * dv).sum(),
    }
    worst = max(acc, key=acc.get)
    assert acc[worst] < ACC_LIMIT, f"{worst} accumulates {acc[worst]:.0f} grid units (limit {ACC_LIMIT})"
    return acc


def last_chunk_row(mb: int, n_cta: int, cta: int) -> int:
    """First minibatch position of the LAST 64-row chunk that split-K CTA `cta` of a K3b job with `n_cta` CTAs reads
    (the producer walks chunk num_chunks - 1 - (cta + it * n_cta), it = 0 .. my_chunks - 1: stx_tc_ppo.cu tc_dw_kernel)."""
    chunks = mb // 64
    mine = (chunks - cta + n_cta - 1) // n_cta
    return 64 * (chunks - 1 - (cta + (mine - 1) * n_cta))


def hot_positions(mb: int) -> List[int]:
    """Minibatch positions carrying an advantage in the hot-row test: tile edges 0, 63, 64, 127, the last row, and rows in
    the last chunk of a dW1 CTA (default split 19 CTAs per half) and of a dW0 CTA (15) after their 4-stage rings wrapped."""
    return sorted({0, 63, 64, 127, mb - 1, last_chunk_row(mb, 19, 5) + 37, last_chunk_row(mb, 15, 2) + 5})
