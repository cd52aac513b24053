"""Exactly representable data for the GRU sequence kernels (stx_rnn.cu) -- TEST INFRASTRUCTURE (like simt_exact_data.py).

The GRU entry points run one of four launch forms (the 2-CTA cluster kernels, the persistent kernels with R = 4 rows and
KS = 2 reduction groups or R = 8 rows and KS = 1, and a per-step form of one SIMT GEMM and one gate kernel per step), each
with its own summation order: KS partials of h W_h, rank-0-first sums of the two cluster halves, NB column blocks of
d(gh) W_h^T, the weight-gradient GEMM split over the T E rows.  On random data those orders show in the last bits.  Here
every order gives the same bits:

* the gates are exact because each pre-activation is one of three codes: sigmoid(128) = 1 (expf(-128) underflows),
  sigmoid(-128) = 0 (expf(128) = inf), sigmoid(0) = 1/2, tanh(+-128) = +-1, tanh(0) = 0, so r, z in {0, 1/2, 1}, n in
  {-1, 0, 1}, and r (1 - r), z (1 - z), 1 - n^2 are 0, 1/4 or 1.  The generator runs the recurrence in fp64 and sets
  gi_r = code_r - gh_r, gi_z = code_z - gh_z, gi_n = code_n - r (gh_n + b_hn);
* h0, W_h (entries +-1, about three per column), b_hn, d_h_seq, the overwrite=False starting gradients and grad_weight
  are small integers times powers of two; z = 1/2 is only drawn where it keeps h on a 1/4 grid;
* `check_exact` proves, per output element with that element's own finest grid, that every product the kernels form (h W_h
  per step, d(gh) W_h^T plus the direct term per step, every split of the d(W_h) GEMM and the sum over the splits, the
  d(b_hn) column sums, the overwrite=False accumulation) has a sum of |terms| below 2^24 grid units, and that every
  element-wise intermediate of the gate forward and backward is an fp32 value.  Then any summation order and any FMA
  contraction gives the fp64 result: the kernels and the oracle must agree bit for bit.

`launch_form` mirrors the host selection of stx_gru_sequence_* / stx_lstm_sequence_* (gru_cluster_ok, gru_persistent_ok,
lstm_cluster_ok, thread counts, dynamic shared memory).  It is a coverage aid, not an oracle: tests/test_rnn_exact_data.py
asserts that CASES reach every form on both sides of every limit.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np

from oracle import rec_oracle as R

S = 128.0                    # saturating pre-activation code
UNIT_LIMIT = 2 ** 24         # fp32 holds every integer number of grid units below this exactly
GRAD_WEIGHT = 0.5
DH_GRID = 0.25
GRAD0_GRID = 2.0 ** -10
SMEM_LIMIT = 227 * 1024      # kGruSmemLimit and the cluster opt-in
PERSISTENT_MIN_T = 4         # kPersistentMinT
GRU_ITEMS = 3                # kGruItems
CL_R, CL_KS = 4, 2           # kLstmR, kLstmKS (also the GRU cluster kernels)
NO_GRID = 10 ** 6            # log2 grid of an exact zero: larger than any real one


# ---------------------------------------------------------------------------------------------------------------------
# host-logic mirror (stx_rnn.cu)
# ---------------------------------------------------------------------------------------------------------------------


def _c32(x: int) -> int:
    return (x + 31) // 32 * 32


def _c4(x: int) -> int:
    return (x + 3) // 4 * 4


def gru_seq_smem(R_: int, KS: int, H: int) -> Tuple[int, int]:
    """GruSmem<R, KS>::fwd_bytes / bwd_bytes."""
    w = _c4(H * (3 * H + 1))
    return (w + H * R_ + KS * R_ * 3 * H) * 4, (w + 3 * H * R_ + 3 * KS * R_ * H + R_ * H) * 4


def gru_cl_smem(H: int) -> Tuple[int, int]:
    """GruClSmem::fwd_bytes / bwd_bytes."""
    Hq = H // 2
    w = _c4(H * (3 * Hq + 1))
    return (w + 2 * H * CL_R + CL_KS * CL_R * 3 * Hq) * 4, (w + 3 * Hq * CL_R + 3 * CL_R * H + 3 * CL_R * Hq) * 4


def lstm_cl_smem(H: int) -> Tuple[int, int]:
    """LstmSmem::fwd_bytes / bwd_bytes."""
    Hq = H // 2
    w = _c4(H * (2 * H + 1))
    return ((w + 2 * H * CL_R + Hq * CL_R + CL_KS * CL_R * 2 * H) * 4,
            (w + 2 * H * CL_R + 2 * CL_KS * CL_R * H + 2 * CL_R * Hq + 2 * CL_R * Hq) * 4)


@dataclass(frozen=True)
class Form:
    cell: str        # gru | lstm
    name: str        # cluster | seq<4,2> | seq<8,1> | per-step
    threads: int     # of the sequence kernel (per-step: the gate kernels' 256)
    smem_fwd: int    # dynamic shared memory of the sequence kernels (0 for per-step)
    smem_bwd: int

    def fwd_launches(self, T: int) -> int:
        """stx_launch_count() delta of one forward: the sequence kernel, or the init kernel + one gate kernel per step (the
        SIMT GEMMs are not counted)."""
        return 1 + T if self.name == "per-step" else 1

    def bwd_launches(self, T: int, d_h0: bool, d_w: bool) -> int:
        """... of one backward: the sequence kernel or T gate kernels (+ the d(h0) / d(carry0) kernel), then the d(W_h)
        reductions (GRU: d(W_h) and d(b_hn); LSTM: d(W_h))."""
        red = (2 if self.cell == "gru" else 1) if d_w else 0
        return (T + int(d_h0) if self.name == "per-step" else 1) + red


def _off(env: Dict[str, str], key: str) -> bool:
    return env.get(key, "")[:1] == "0"


def launch_form(cell: str, T: int, E: int, H: int, env: Optional[Dict[str, str]] = None) -> Form:
    env = env or {}
    if cell == "gru":
        if not _off(env, "STX_GRU_CLUSTER") and E < 1024 and T >= PERSISTENT_MIN_T and H >= 2 and H % 2 == 0:
            th = _c32(CL_KS * 3 * (H // 2))
            f, b = gru_cl_smem(H)
            if th <= 1024 and (H // 2) * CL_R <= th and 3 * H <= th and f <= SMEM_LIMIT and b <= SMEM_LIMIT:
                return Form(cell, "cluster", th, f, b)
        sizes = gru_seq_smem(8, 1, H) + gru_seq_smem(4, 2, H)
        if not _off(env, "STX_GRU_PERSISTENT") and H >= 2 and _c32(6 * H) <= 1024 and max(sizes) <= SMEM_LIMIT and T >= PERSISTENT_MIN_T:
            R_, KS = (8, 1) if E >= 1024 else (4, 2)
            th = _c32(KS * 3 * H)
            assert H * R_ <= GRU_ITEMS * th and 3 * KS * H <= th, "kGruItems / column-block thread check"
            return Form(cell, f"seq<{R_},{KS}>", th, *gru_seq_smem(R_, KS, H))
        return Form(cell, "per-step", 256, 0, 0)
    assert cell == "lstm"
    th = _c32(CL_KS * 2 * H)
    f, b = lstm_cl_smem(H)
    if (not _off(env, "STX_LSTM_CLUSTER") and H >= 2 and H % 2 == 0 and th <= 1024 and (H // 2) * CL_R <= th and 2 * CL_KS * H <= th
            and f <= SMEM_LIMIT and b <= SMEM_LIMIT and T >= PERSISTENT_MIN_T):
        return Form(cell, "cluster", th, f, b)
    return Form(cell, "per-step", 256, 0, 0)


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class Case:
    name: str
    T: int
    E: int
    H: int
    env: Tuple[Tuple[str, str], ...] = ()
    zero: float = 0.15         # fraction of zero-point (non-saturating) gate codes
    reset: float = 0.4         # reset rate of the random rows

    @property
    def env_dict(self) -> Dict[str, str]:
        return dict(self.env)

    @property
    def form(self) -> Form:
        return launch_form("gru", self.T, self.E, self.H, self.env_dict)


NO_CLUSTER = (("STX_GRU_CLUSTER", "0"),)
PER_STEP = (("STX_GRU_CLUSTER", "0"), ("STX_GRU_PERSISTENT", "0"))

# tests/test_rnn_exact_gpu.py runs every case; the comment names the form the default selection (or `env`) gives and why
# the case is there (tests/test_rnn_exact_data.py asserts the coverage with launch_form).
CASES = [
    Case("cl_20", 4, 33, 20),                               # cluster, ragged last tile (33 = 8 x 4 + 1)
    Case("cl_t8", 8, 33, 20),                               # cluster, longer chain
    Case("cl_e1", 4, 1, 20),                                # cluster, one row
    Case("cl_e1023", 4, 1023, 20),        # cluster at the last E below 1024, 3-row last tile
    Case("cl_h188", 4, 5, 188),                             # cluster at its shared-memory limit (bwd 230,864 B)
    Case("seq42_h3", 4, 5, 3),                              # H odd: no cluster -> <4,2>
    Case("seq42_h129", 4, 5, 129),                          # <4,2> at H = 129 (odd)
    Case("seq81_e1024", 4, 1024, 20),     # E = 1024 -> <8,1>
    Case("seq81_h129", 4, 1024, 129),     # <8,1>, H = 129
    Case("seq81_h130", 4, 1025, 130),     # <8,1> at its limit (bwd 232,448 B), 1-row last tile
    Case("ps_h131", 4, 5, 131),                             # one above the persistent limit: per-step
    Case("ps_h131_e1025", 4, 1025, 131),  # per-step with E >= 1024
    Case("ps_h187", 4, 3, 187),                             # odd, above 130: per-step
    Case("ps_h189", 4, 3, 189),                             # odd, above the cluster limit
    Case("ps_h190", 4, 3, 190),                             # even, one step above the cluster limit: per-step
    Case("ps_t3", 3, 33, 20),                               # T = 3 < kPersistentMinT: per-step
    Case("ps_t1_rollout", 1, 2048, 128),                    # the rollout step of scripts/bench_rec.py
    Case("ps_t1_e3", 1, 3, 20),                             # T = 1, E = 3
    Case("nc_seq42_h130", 4, 5, 130, NO_CLUSTER),           # <4,2> at H = 130 (bwd 224,128 B)
    Case("nc_seq42_e1023", 4, 1023, 20, NO_CLUSTER),   # <4,2>, 3-row last tile
    Case("nc_seq42_t8", 8, 33, 20, NO_CLUSTER),             # <4,2>, longer chain
    Case("nc_seq81_e1025", 4, 1025, 20, NO_CLUSTER),   # <8,1>, 1-row last tile
    Case("ps_forced", 6, 33, 20, PER_STEP),                 # STX_GRU_PERSISTENT=0: per-step at T >= 4
    Case("ps_forced_e1024", 4, 1024, 20, PER_STEP),
]
CASE_BY_NAME = {c.name: c for c in CASES}
ENV_GROUPS = sorted({c.env for c in CASES})

# (T, E, H) of the LSTM cases of the bound arm of tests/test_rnn_exact_gpu.py (LSTM gates cannot be exact: tanh(c) of a
# dyadic c is not): both forms, both sides of the cluster limit, odd H, T = 3, and the two shapes of scripts/bench_rec.py
LSTM_CASES = [(6, 40, 12), (4, 5, 161), (4, 5, 162), (4, 5, 163), (4, 5, 164), (3, 33, 12), (1, 2048, 128), (256, 128, 128)]


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------


@dataclass
class Problem:
    case: Case
    gi: np.ndarray       # (T, E, 3H) float32
    reset: np.ndarray    # (T, E) bool
    h0: np.ndarray       # (E, H) float32
    Wh: np.ndarray       # (H, 3H) float32
    bhn: np.ndarray      # (H,) float32
    d_h: np.ndarray      # (T, E, H) float32
    dW0: np.ndarray      # (H, 3H) float32: starting d(W_h) of the overwrite=False call
    db0: np.ndarray      # (H,) float32


def _codes(rng, shape, zero, allow_zero=None):
    c = np.where(rng.random(shape) < 0.5, -S, S)
    z = rng.random(shape) < zero
    if allow_zero is not None:
        z &= allow_zero
    return np.where(z, 0.0, c)


def _sig(x):
    with np.errstate(over="ignore"):
        return np.where(x < -88.0, 0.0, 1.0 / (1.0 + np.exp(-x)))   # expf overflows to inf below -88.7: 1 / inf = 0


def make_problem(case: Case) -> Problem:
    rng = np.random.default_rng(zlib.crc32(case.name.encode()))
    T, E, H = case.T, case.E, case.H
    Wh = np.zeros((H, 3 * H))
    for c in range(3 * H):
        rows = rng.choice(H, size=min(3, H), replace=False)
        Wh[rows, c] = rng.choice([-1.0, 1.0], size=rows.size)
    bhn = rng.integers(-1, 2, H) / 2
    h0 = rng.integers(-2, 3, (E, H)) / 2
    reset = rng.random((T, E)) < case.reset
    if E >= 3:
        reset[:, 0], reset[:, 1] = True, False     # a row that resets every step, a row that never does
    d_h = rng.integers(-1, 2, (T, E, H)) * DH_GRID
    dW0 = rng.integers(-3, 4, (H, 3 * H)) * GRAD0_GRID
    db0 = rng.integers(-3, 4, H) * GRAD0_GRID
    gi = np.zeros((T, E, 3 * H))
    h = h0
    for t in range(T):
        hp = np.where(reset[t][:, None], 0.0, h)
        gh = hp @ Wh
        cr = _codes(rng, (E, H), case.zero)
        cz = _codes(rng, (E, H), case.zero, allow_zero=(hp * 2 == np.round(hp * 2)))   # z = 1/2 keeps h on a 1/4 grid
        cn = _codes(rng, (E, H), case.zero)
        r, z, n = _sig(cr), _sig(cz), np.tanh(cn)
        ghn = gh[:, 2 * H:] + bhn
        gi[t] = np.concatenate([cr - gh[:, :H], cz - gh[:, H:2 * H], cn - r * ghn], 1)
        h = (1.0 - z) * n + z * hp
    f32 = lambda a: np.asarray(a, np.float32)
    return Problem(case, f32(gi), reset, f32(h0), f32(Wh), f32(bhn), f32(d_h), f32(dW0), f32(db0))


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference, with the kernel faults of tests/test_rnn_exact_data.py as variants
# ---------------------------------------------------------------------------------------------------------------------


@dataclass
class Chain:
    hp: np.ndarray       # (T, E, H) state entering each step (after its reset)
    gh: np.ndarray       # (T, E, 3H) hp W_h
    r: np.ndarray
    z: np.ndarray
    n: np.ndarray
    ghn: np.ndarray      # (T, E, H) gh_n + b_hn
    h_seq: np.ndarray
    dh: np.ndarray       # (T, E, H) d(h_t): d_h_seq + what arrives from step t + 1
    dgh: np.ndarray      # (T, E, 3H)
    d_gi: np.ndarray
    direct: np.ndarray   # (T, E, H) dh z
    dWh: np.ndarray      # sum_t hp_t^T dgh_t (grad_weight 1)
    dbhn: np.ndarray
    dh0: np.ndarray


FAULTS = ("ks_partial_dropped", "stale_peer_h", "stale_peer_inbox", "reset_early", "ragged_row_dropped_from_dh0",
          "dbhn_from_z_part", "direct_term_dropped")


def chain(pb: Problem, fault: Optional[str] = None, at: Tuple[int, int] = (0, 0)) -> Chain:
    """The GRU forward and backward in fp64.  `fault` (one of FAULTS) makes it compute what a kernel with that fault would,
    at step / first row `at` = (t, e0) where it applies to one step of one tile."""
    T, E, H = pb.case.T, pb.case.E, pb.case.H
    Hq, kper = H // 2, (H + 1) // 2
    f64 = lambda a: np.asarray(a, np.float64)
    gi, h0, Wh, bhn, d_h = f64(pb.gi), f64(pb.h0), f64(pb.Wh), f64(pb.bhn), f64(pb.d_h)
    reset = pb.reset.copy()
    ft, fe = at
    if fault == "reset_early":   # the reset of (ft, fe) cuts the state entering step ft - 1 instead
        assert reset[ft, fe] and not reset[ft - 1, fe]
        reset[ft, fe], reset[ft - 1, fe] = False, True
    tile = slice(fe, fe + CL_R)
    hp_all, gh_all, rs, zs, ns, ghns, hs = (np.zeros((T, E, k)) for k in (H, 3 * H, H, H, H, H, H))
    h = h0
    for t in range(T):
        hp = np.where(reset[t][:, None], 0.0, h)
        gh = hp @ Wh
        if fault == "ks_partial_dropped" and t == ft:          # reduction group 1 (k >= kper) lost for one tile
            gh[tile] = hp[tile, :kper] @ Wh[:kper]
        if fault == "stale_peer_h" and t == ft:                # CTA 0 of one cluster reads the peer's half of h_{t-1}
            mix = hp[tile].copy()
            mix[:, Hq:] = hp_all[t - 1, tile, Hq:]
            cols = np.concatenate([np.arange(Hq) + g * H for g in range(3)])
            gh[tile, :] = np.where(np.isin(np.arange(3 * H), cols), mix @ Wh, gh[tile])
        ghn = gh[:, 2 * H:] + bhn
        r = _sig(gi[t][:, :H] + gh[:, :H])
        z = _sig(gi[t][:, H:2 * H] + gh[:, H:2 * H])
        n = np.tanh(gi[t][:, 2 * H:] + r * ghn)
        h = (1.0 - z) * n + z * hp
        hp_all[t], gh_all[t], rs[t], zs[t], ns[t], ghns[t], hs[t] = hp, gh, r, z, n, ghn, h
    dh_all, dgh_all, dgi_all, direct_all = np.zeros((T, E, H)), np.zeros((T, E, 3 * H)), np.zeros((T, E, 3 * H)), np.zeros((T, E, H))
    dh_rec = np.zeros((E, H))
    prev_dgh = np.zeros((E, 3 * H))
    for t in range(T - 1, -1, -1):
        hp, r, z, n, ghn = hp_all[t], rs[t], zs[t], ns[t], ghns[t]
        dh = d_h[t] + dh_rec
        dn, dz = dh * (1.0 - z), dh * (hp - n)
        dpn = dn * (1.0 - n * n)
        dpr, dpz = dpn * ghn * r * (1.0 - r), dz * z * (1.0 - z)
        dgh = np.concatenate([dpr, dpz, dpn * r], 1)
        direct = dh * z
        dhp = dgh @ Wh.T
        if fault == "stale_peer_inbox" and t == ft:            # CTA 0 adds the peer's partial of step t + 1 (the other inbox)
            peer = np.concatenate([np.arange(Hq, H) + g * H for g in range(3)])
            dhp[tile, :Hq] += (prev_dgh[tile][:, peer] - dgh[tile][:, peer]) @ Wh[:Hq, peer].T
        if fault != "direct_term_dropped":
            dhp = dhp + direct
        dh_rec = np.where(reset[t][:, None], 0.0, dhp)
        dh_all[t], dgh_all[t], direct_all[t] = dh, dgh, direct
        dgi_all[t] = np.concatenate([dpr, dpz, dpn], 1)
        prev_dgh = dgh
    dWh = np.einsum("tek,tec->kc", hp_all, dgh_all)
    dbhn = dgh_all[:, :, (H if fault == "dbhn_from_z_part" else 2 * H):][:, :, :H].sum((0, 1))
    dh0 = dh_rec.copy()
    if fault == "ragged_row_dropped_from_dh0":
        dh0[E - 1] = 0.0
    return Chain(hp_all, gh_all, rs, zs, ns, ghns, hs, dh_all, dgh_all, dgi_all, direct_all, dWh, dbhn, dh0)


@dataclass
class Reference:
    h_seq: np.ndarray     # float32
    d_gi: np.ndarray
    d_wh: np.ndarray      # overwrite=True, grad_weight 1
    d_bhn: np.ndarray
    d_wh_acc: np.ndarray  # overwrite=False, grad_weight GRAD_WEIGHT, from dW0
    d_bhn_acc: np.ndarray
    d_h0: np.ndarray


def reference(pb: Problem, fault: Optional[str] = None, at: Tuple[int, int] = (0, 0)) -> Reference:
    ch = chain(pb, fault, at)
    f32 = lambda a: np.asarray(a, np.float64).astype(np.float32)
    return Reference(f32(ch.h_seq), f32(ch.d_gi), f32(ch.dWh), f32(ch.dbhn), f32(pb.dW0.astype(np.float64) + GRAD_WEIGHT * ch.dWh),
                     f32(pb.db0.astype(np.float64) + GRAD_WEIGHT * ch.dbhn), f32(ch.dh0))


# ---------------------------------------------------------------------------------------------------------------------
# the exactness invariant
# ---------------------------------------------------------------------------------------------------------------------


def lgrid(a) -> np.ndarray:
    """Per element: log2 of the largest power of two that divides it (NO_GRID for 0)."""
    a = np.asarray(a, np.float64)
    m, e = np.frexp(a)
    im = np.abs(m * 2.0 ** 53).astype(np.int64)
    low = im & -im
    return np.where(a == 0, NO_GRID, e - 53 + np.log2(np.maximum(low, 1)).astype(np.int64))


def grid_matmul(la: np.ndarray, lb: np.ndarray) -> np.ndarray:
    """Per element of A @ B: log2 of the finest grid among its nonzero terms A[i, k] B[k, j] (NO_GRID if none), from the
    per-element grids la = lgrid(A), lb = lgrid(B).  One indicator product per pair of grid levels."""
    out = np.full((la.shape[0], lb.shape[1]), NO_GRID, np.int64)
    lv_a = np.unique(la[la < NO_GRID])
    lv_b = np.unique(lb[lb < NO_GRID])
    ib = {v: (lb == v).astype(np.float32) for v in lv_b}
    for va in lv_a:
        ia = (la == va).astype(np.float32)
        for vb in lv_b:
            hit = (ia @ ib[vb]) > 0
            out = np.where(hit & (va + vb < out), va + vb, out)
    return out


def _exact_f32(a) -> bool:
    a = np.asarray(a, np.float64)
    return bool(np.array_equal(a.astype(np.float32).astype(np.float64), a))


def _units(abs_sum: np.ndarray, lg: np.ndarray) -> float:
    """Largest sum of |terms| in units of each element's own grid."""
    live = lg < NO_GRID
    return float((abs_sum[live] * np.exp2(-lg[live].astype(np.float64))).max()) if live.any() else 0.0


def check_exact(pb: Problem) -> Dict[str, float]:
    """Asserts that every sum and element-wise step of every GRU form on `pb` is exact in fp32 whatever its order, and that
    the reference equals oracle/rec_oracle.py's.  Returns the largest sum per quantity as a fraction of 2^24."""
    c = pb.case
    T, E, H = c.T, c.E, c.H
    ch = chain(pb)
    ab = np.abs
    worst: Dict[str, float] = {}

    def need(name, units):
        worst[name] = max(worst.get(name, 0.0), units / UNIT_LIMIT)
        assert units < UNIT_LIMIT, f"{c.name}: {name} sums {units:.0f} grid units (limit 2^24)"

    def exact(name, *arrays):
        for a in arrays:
            assert _exact_f32(a), f"{c.name}: {name} is not an fp32 value"

    Wh, bhn = pb.Wh.astype(np.float64), pb.bhn.astype(np.float64)
    lw, lw_t = lgrid(Wh), lgrid(Wh.T)
    lb = np.concatenate([np.full(2 * H, NO_GRID), lgrid(bhn)])
    bias = np.concatenate([np.zeros(2 * H), ab(bhn)])
    for t in range(T):
        # forward: gh = hp W_h (KS partials, cluster halves) + b_hn on the n part; then the pre-activations hit their codes
        hp, gh = ch.hp[t], ch.gh[t]
        need("h W_h (+ b_hn)", _units(ab(hp) @ ab(Wh) + bias, np.minimum(grid_matmul(lgrid(hp), lw), lb)))
        r, z, n, ghn = ch.r[t], ch.z[t], ch.n[t], ch.ghn[t]
        assert set(np.unique(r)) <= {0.0, 0.5, 1.0} and set(np.unique(z)) <= {0.0, 0.5, 1.0} and set(np.unique(n)) <= {-1.0, 0.0, 1.0}
        gi = pb.gi[t].astype(np.float64)
        assert np.array_equal(np.concatenate([gi[:, :H] + gh[:, :H], gi[:, H:2 * H] + gh[:, H:2 * H], gi[:, 2 * H:] + r * ghn], 1) % S, np.zeros_like(gi))
        exact("forward gate", gh, ghn, r * ghn, gi[:, 2 * H:] + r * ghn, 1.0 - z, (1.0 - z) * n, z * hp, ch.h_seq[t])
        # backward: dh_t = d_h_t + [dh_{t+1} z_{t+1} + d(gh_{t+1}) W_h^T] (NB column blocks, the two cluster halves, the
        # SIMT DX GEMM + the direct term), cut by reset_{t+1}
        if t + 1 < T:
            keep = ~pb.reset[t + 1][:, None]
            dgh1, dir1 = ch.dgh[t + 1] * keep, ch.direct[t + 1] * keep
            lg = np.minimum(np.minimum(grid_matmul(lgrid(dgh1), lw_t), lgrid(dir1)), lgrid(pb.d_h[t]))
            need("d(h_t)", _units(ab(dgh1) @ ab(Wh).T + ab(dir1) + ab(pb.d_h[t].astype(np.float64)), lg))
        dh = ch.dh[t]
        dn, dz = dh * (1.0 - z), dh * (hp - n)
        dpn = dn * (1.0 - n * n)
        exact("backward gate", dh, hp - n, dn, dz, dpn, dpn * ghn, dpn * ghn * r, dz * z, ch.dgh[t], ch.d_gi[t], ch.direct[t])
    # d(W_h) = sum over the T E rows of hp^T d(gh), any split of the rows; d(b_hn) = column sums of the n part
    hp2, dgh2 = ch.hp.reshape(T * E, H), ch.dgh.reshape(T * E, 3 * H)
    lg_w = grid_matmul(lgrid(hp2.T), lgrid(dgh2))
    s_w = ab(hp2).T @ ab(dgh2)
    need("d(W_h)", _units(s_w, lg_w))
    dn_part = dgh2[:, 2 * H:]
    lg_b = lgrid(dn_part).min(0)
    s_b = ab(dn_part).sum(0)
    need("d(b_hn)", _units(s_b, lg_b))
    # overwrite=False: start + grad_weight * sum (a power of two: exact)
    assert GRAD_WEIGHT == 2.0 ** round(np.log2(GRAD_WEIGHT))
    lgw = int(round(np.log2(GRAD_WEIGHT)))
    for name, start, s, lg in (("d(W_h) accumulation", pb.dW0, s_w, lg_w), ("d(b_hn) accumulation", pb.db0, s_b, lg_b)):
        lga = np.minimum(lgrid(start), np.where(lg < NO_GRID, lg + lgw, NO_GRID))
        need(name, _units(ab(start.astype(np.float64)) + GRAD_WEIGHT * s, lga))
    ref = reference(pb)
    exact("results", ch.dWh, ch.dbhn, ch.dh0, pb.dW0.astype(np.float64) + GRAD_WEIGHT * ch.dWh, pb.db0.astype(np.float64) + GRAD_WEIGHT * ch.dbhn)
    # the project's oracle gives the same fp32 results (its sigmoid(-128) is 2.6e-56 instead of 0, which rounds away)
    f64 = lambda a: a.astype(np.float64)
    hs_o, cache = R.gru_forward(f64(pb.gi), pb.reset, f64(pb.h0), f64(pb.Wh), f64(pb.bhn))
    dgi_o, dWh_o, dbhn_o, dh0_o = R.gru_backward(cache, pb.reset, f64(pb.d_h), f64(pb.Wh))
    for got, want in ((ref.h_seq, hs_o), (ref.d_gi, dgi_o), (ref.d_wh, dWh_o), (ref.d_bhn, dbhn_o), (ref.d_h0, dh0_o)):
        np.testing.assert_array_equal(got, want.astype(np.float32))
    worst["zero-point gates"] = float(np.mean(ch.r == 0.5) + np.mean(ch.z == 0.5) + np.mean(ch.n == 0.0)) / 3
    worst["live d(h0)"] = float(np.mean(ch.dh0 != 0))
    return worst
