"""Exactly representable data for the fp32 CUDA-core MLP path -- TEST INFRASTRUCTURE (like exact_data.py).

The fp32 path (stx_simt_gemm.cuh driven by simt_forward / simt_backward in stx_mlp.cu) accumulates in an order of its
own: 64x64 tiles walking K in steps of 16, 32x32 panels walking it in 256-wide chunks split over even and odd k, weight
gradients summed per split of the batch and then over the splits in a fixed order.  On random data that order shows in
the last bits, so tolerance-based tests cannot see a fault confined to a small part of the gradient arena.  Here every
value is a small integer times a power of two:

* observations in {-3..3}, weights in {-2..2}/4 (sparse), biases in {-2..2}/4, d(out) in {-3..3}/2^6, an overwrite=0
  starting gradient in {-3..3}/2^12 and grad_weight = 1/2; relu and identity networks only (every other activation is
  inexact and is tested element-wise in tests/test_simt_mlp_gpu.py);
* every operand of every GEMM lies on a power-of-two grid, so every product lies on the product of the two grids, and
  `check_exact` asserts that for every GEMM the kernels run (each forward layer, each d(hidden) and d(input) GEMM, each
  weight-gradient split, the sum over the splits, the bias sums and the overwrite=0 accumulation) the sum of the
  absolute values of its terms is below 2^24 grid units.  Then every partial sum, in any order, is an integer number of
  grid units below 2^24: exact in fp32.  The kernels and the fp64 oracle must agree bit for bit.

Pre-activations exactly 0 occur on purpose: the kernel's relu'(z) = (z > 0) and the oracle's agree there.

`launch_plan` mirrors the host logic of launch_gemm (tile choice) and pick_splits (stx_mlp.cu).  It is a coverage aid,
not an oracle: tests/test_simt_exact_data.py asserts that CASES reach every tiling and split path.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle import ppo_oracle as O

UNIT_LIMIT = 2 ** 24          # fp32 holds every integer number of grid units below this exactly
NUM_SMS = 132                 # H100 SXM: launch_gemm's kPanelBelowCtas
GRAD_WEIGHT = 0.5
DOUT_GRID = 2.0 ** -6
GRAD0_GRID = 2.0 ** -12
POISON = 1.0e4 + 0.5          # padding columns of a strided x: reading one breaks exactness everywhere


@dataclass(frozen=True)
class Case:
    """One network and batch.  B > 0: x has B rows of pitch ldx and the batch is gathered through row_idx (M entries)."""
    name: str
    sizes: Tuple[int, ...]
    activation: str
    M: int
    B: int = 0
    ldx: int = 0
    density: float = 0.0      # fraction of nonzero weights; 0: about 6 nonzeros per column

    @property
    def gathered(self) -> bool:
        return self.B > 0


# The cases tests/test_simt_mlp_gpu.py runs; the comment says which paths each one is there for (test_simt_exact_data.py
# asserts the coverage with launch_plan).
CASES = [
    Case("m1", (5, 24, 3), "relu", 1),                                # one row; K, N not multiples of 16
    Case("m5", (13, 40, 17, 1), "identity", 5, B=9, ldx=16),          # five rows gathered from a strided x
    Case("k300", (300, 264, 5), "relu", 300),                         # panel K > 256 (FWD, d(input)); one split of 300 rows
    Case("cta131", (20, 64, 64, 1), "relu", 8384),                    # N = 64 at 131 CTAs: panel; DW splits of 262 rows
    Case("cta132", (20, 64, 64, 1), "relu", 8385, B=9000, ldx=24),    # 132 CTAs: 64x64, N = 1 head too; ragged last split
    Case("bench", (64, 256, 256, 8), "relu", 32768),                  # 64x64 everywhere, 66 splits
    Case("split128", (16, 128, 1), "identity", 32768, B=40000, ldx=20),  # 128 splits of 256 rows, 64x64 DW of layer 0
    Case("thin128", (16, 64, 1), "relu", 32768),                      # 128 splits on the panel DW
    Case("ragged", (48, 200, 3), "relu", 37000, B=37001, ldx=53),     # ragged tiles and splits, N = 200
]
CASE_BY_NAME = {c.name: c for c in CASES}


# ---------------------------------------------------------------------------------------------------------------------
# host-logic mirror (stx_simt_gemm.cuh launch_gemm, stx_mlp.cu pick_splits / simt_backward)
# ---------------------------------------------------------------------------------------------------------------------


def pick_splits(sizes, mb: int) -> int:
    s = min(max(mb // 512, 1), 32)
    min_tiles = min(((sizes[i] + 63) // 64) * ((sizes[i + 1] + 63) // 64) for i in range(len(sizes) - 1))
    want = min((2 * NUM_SMS + min_tiles - 1) // min_tiles, mb // 256, 128)
    return max(s, want)


def tiling(mode: str, M: int, N: int, K: int, splits: int = 1) -> str:
    """'64' or 'panel': the kernel launch_gemm<mode> picks."""
    out_rows = K if mode == "DW" else M
    z = splits if mode == "DW" else 1
    ctas64 = -(-out_rows // 64) * -(-N // 64) * z
    return "64" if ctas64 >= NUM_SMS else "panel"


@dataclass(frozen=True)
class Launch:
    mode: str       # FWD | DX | DW
    layer: int
    M: int
    N: int
    K: int          # reduction length (DW: output rows = in dim)
    splits: int
    rows_per_split: int
    tile: str

    @property
    def chunks(self) -> int:
        """256-wide chunks the panel kernel walks (FWD/DX: K; DW: rows per split)."""
        red = self.rows_per_split if self.mode == "DW" else self.K
        return -(-red // 256)


def launch_plan(sizes, M: int, d_input: bool = True) -> List[Launch]:
    """GEMM launches of stx_mlp_forward_train + stx_mlp_backward (net_grad and, if asked, d_input) in order."""
    n = len(sizes) - 1
    out = []
    mk = lambda mode, layer, MM, N, K, s=1, rps=0: Launch(mode, layer, MM, N, K, s, rps, tiling(mode, MM, N, K, s))
    for i in range(n):
        out.append(mk("FWD", i, M, sizes[i + 1], sizes[i]))
    splits = pick_splits(sizes, M)
    rps = -(-M // splits)
    for i in range(n - 1, -1, -1):
        out.append(mk("DW", i, M, sizes[i + 1], sizes[i], splits, rps))
        if i == 0 and d_input:
            out.append(mk("DX", 0, M, sizes[0], sizes[1]))
        if i > 0:
            out.append(mk("DX", i, M, sizes[i], sizes[i + 1]))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------


@dataclass
class Problem:
    case: Case
    net: O.MLPParams
    xbuf: np.ndarray                # (B or M, ldx) float32; columns >= in dim hold POISON
    row_idx: Optional[np.ndarray]   # int32 (M,) or None
    d_out: np.ndarray               # (M, out) float32
    grad0: np.ndarray               # flat arena float32: the starting gradient of the overwrite=0 call

    @property
    def x(self) -> np.ndarray:
        """The batch as the first layer reads it: (M, in) float64."""
        rows = self.xbuf if self.row_idx is None else self.xbuf[self.row_idx]
        return rows[:, :self.case.sizes[0]].astype(np.float64)


def _sparse_ints(rng, shape, lo, hi, density):
    v = rng.integers(lo, hi + 1, size=shape)
    return np.where(rng.random(shape) < density, v, 0).astype(np.float64)


def make_problem(case: Case) -> Problem:
    rng = np.random.default_rng(sum(case.sizes) * 7919 + case.M + 13 * case.B)
    s = case.sizes
    W, b = [], []
    for i in range(len(s) - 1):
        dens = case.density or min(0.5, 6.0 / s[i])
        w = _sparse_ints(rng, (s[i], s[i + 1]), -2, 2, dens) / 4
        w[rng.integers(0, s[i], s[i + 1]), np.arange(s[i + 1])] = rng.choice([-0.5, -0.25, 0.25, 0.5], s[i + 1])  # no dead column
        W.append(w)
        b.append(rng.integers(-2, 3, s[i + 1]) / 4)
    net = O.MLPParams(W, b, case.activation)
    rows = case.B if case.gathered else case.M
    ldx = case.ldx or s[0]
    xbuf = np.full((rows, ldx), POISON, np.float32)
    xbuf[:, :s[0]] = _sparse_ints(rng, (rows, s[0]), -3, 3, 0.5)
    row_idx = rng.choice(case.B, size=case.M, replace=case.M > case.B).astype(np.int32) if case.gathered else None
    d_out = (_sparse_ints(rng, (case.M, s[-1]), -3, 3, 0.5) * DOUT_GRID).astype(np.float32)
    grad0 = (_sparse_ints(rng, net.flat().size, -3, 3, 0.75) * GRAD0_GRID).astype(np.float32)
    return Problem(case, net, xbuf, row_idx, d_out, grad0)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------------


@dataclass
class Chain:
    """The fp64 forward / backward of one problem: layer inputs, pre-activations and d(Dense output) per layer."""
    out: np.ndarray
    inputs: List[np.ndarray]   # inputs[i]: what layer i multiplies (M, sizes[i])
    pre: List[np.ndarray]      # pre[i]: Dense output of layer i
    d: List[np.ndarray]        # d[i]: d(loss)/d(pre[i])
    d_input: np.ndarray        # d[0] @ W0^T


def chain(net: O.MLPParams, x: np.ndarray, d_out: np.ndarray) -> Chain:
    out, acts = O.mlp_forward(net, x)
    _, fp = O.ACTIVATIONS[net.activation]
    n = len(net.W)
    d = [None] * n
    d[n - 1] = d_out.astype(np.float64)
    for i in range(n - 1, 0, -1):
        d[i - 1] = (d[i] @ net.W[i].T) * fp(acts.pre[i - 1])
    return Chain(out, list(acts), list(acts.pre), d, d[0] @ net.W[0].T)


def layer_grads(net: O.MLPParams, ch: Chain, rows: Optional[Dict[int, np.ndarray]] = None,
                bias_rows: Optional[Dict[int, np.ndarray]] = None) -> np.ndarray:
    """Flat gradient arena (fp64, grad_weight 1): dW_i = inputs[i][r]^T d[i][r], db_i = sum d[i][r'], with r = rows[i] and
    r' = bias_rows[i] (default all rows).  The row subsets model kernel faults for tests/test_simt_exact_data.py."""
    rows, bias_rows = rows or {}, bias_rows or {}
    gW, gb = [], []
    for i in range(len(net.W)):
        r = rows.get(i, slice(None))
        gW.append(ch.inputs[i][r].T @ ch.d[i][r])
        gb.append(ch.d[i][bias_rows.get(i, slice(None))].sum(0))
    return O.MLPParams(gW, gb, net.activation).flat()


@dataclass
class Reference:
    out: np.ndarray           # float32
    grad: np.ndarray          # flat, overwrite=1: GRAD_WEIGHT * dL/dparams
    grad_acc: np.ndarray      # flat, overwrite=0: grad0 + GRAD_WEIGHT * dL/dparams
    d_input: np.ndarray


def reference(pb: Problem) -> Reference:
    """Oracle results as float32 (exact on this data: check_exact); the parameter gradient comes from O.mlp_backward."""
    x = pb.x
    ch = chain(pb.net, x, pb.d_out)
    _, acts = O.mlp_forward(pb.net, x)
    g = O.mlp_backward(pb.net, acts, pb.d_out.astype(np.float64)).flat()
    f32 = lambda a: np.asarray(a, np.float64).astype(np.float32)
    return Reference(f32(ch.out), f32(GRAD_WEIGHT * g), f32(pb.grad0.astype(np.float64) + GRAD_WEIGHT * g), f32(ch.d_input))


# ---------------------------------------------------------------------------------------------------------------------
# the exactness invariant
# ---------------------------------------------------------------------------------------------------------------------


def grid(a: np.ndarray) -> float:
    """The coarsest power of two 2^e (e <= 0) that every entry of `a` is an integer multiple of; inf for all zeros."""
    a = np.asarray(a, np.float64)
    if not a.any():
        return np.inf
    for e in range(0, -60, -1):
        q = a * 2.0 ** -e
        if np.array_equal(q, np.round(q)):
            return 2.0 ** e
    raise AssertionError("not on any power-of-two grid above 2^-60")


def _exact_f32(a) -> bool:
    a = np.asarray(a, np.float64)
    return bool(np.array_equal(a.astype(np.float32).astype(np.float64), a))


def _units(terms_abs: np.ndarray, unit: float) -> float:
    """Largest entry of a sum of |terms|, in grid units."""
    return float(terms_abs.max() / unit) if terms_abs.size and np.isfinite(unit) else 0.0


def check_exact(pb: Problem) -> Dict[str, float]:
    """Asserts that every GEMM, split, reduction and accumulation the fp32 path performs on `pb` is exact in any order:
    operands are fp32 values on power-of-two grids and each sum of |terms| stays below 2^24 units of the product grid.
    Returns the largest such sum per quantity as a fraction of 2^24, and the number of pre-activations exactly at 0."""
    c, net = pb.case, pb.net
    assert c.activation in ("relu", "identity")
    x = pb.x
    ch = chain(net, x, pb.d_out)
    ab = np.abs
    n = len(net.W)
    worst: Dict[str, float] = {}

    def need(name: str, units: float):
        worst[name] = units / UNIT_LIMIT
        assert units < UNIT_LIMIT, f"{c.name}: {name} sums {units:.0f} grid units (limit 2^24)"

    for t in [x, pb.d_out, pb.grad0, *net.W, *net.b]:
        assert _exact_f32(t) and np.isfinite(grid(t)) or not np.asarray(t).any()
    assert GRAD_WEIGHT == 2.0 ** round(np.log2(GRAD_WEIGHT)), "grad_weight must be a power of two"
    # forward: U_i = H_i W_i + b_i; relu / identity of an exact U is exact
    for i in range(n):
        unit = grid(ch.inputs[i]) * grid(net.W[i])
        if np.isfinite(unit):
            assert np.all(np.round(net.b[i] / unit) == net.b[i] / unit), f"b{i} off the product grid"
        need(f"FWD{i}", _units(ab(ch.inputs[i]) @ ab(net.W[i]) + ab(net.b[i]), unit))
        assert _exact_f32(ch.pre[i])
    # backward: d(hidden) and d(input) GEMMs (the relu mask multiplies by exactly 0 or 1)
    for i in range(n - 1, -1, -1):
        need(f"DX{i}", _units(ab(ch.d[i]) @ ab(net.W[i]).T, grid(ch.d[i]) * grid(net.W[i])))
    assert _exact_f32(ch.d_input)
    # weight gradients: each split of rows_per_split rows, the fixed-order sum over the splits, the bias sums, then
    # grad_weight * s (a power of two: exact) and, for overwrite=0, grad0 + grad_weight * s
    splits = pick_splits(c.sizes, c.M)
    rps = -(-c.M // splits)
    g_total = O.MLPParams([ab(ch.inputs[i]).T @ ab(ch.d[i]) for i in range(n)], [ab(ch.d[i]).sum(0) for i in range(n)]).flat()
    units_flat = np.empty_like(g_total)
    o = 0
    for i in range(n):
        A, D = ch.inputs[i], ch.d[i]
        unit, ubias = grid(A) * grid(D), grid(D)
        per_split = max(_units(ab(A[z:z + rps]).T @ ab(D[z:z + rps]), unit) for z in range(0, c.M, rps))
        need(f"DW{i} per split", per_split)
        need(f"DW{i} over splits", _units(g_total[o:o + A.shape[1] * D.shape[1]], unit))
        need(f"db{i}", _units(ab(D).sum(0), ubias))
        nw = A.shape[1] * D.shape[1]
        units_flat[o:o + nw], units_flat[o + nw:o + nw + D.shape[1]] = unit, ubias
        o += nw + D.shape[1]
    acc_unit = np.minimum(GRAD_WEIGHT * units_flat, grid(pb.grad0))
    assert np.all(np.round(pb.grad0 / acc_unit) == pb.grad0 / acc_unit)
    need("overwrite=0 accumulation", float(((ab(pb.grad0) + GRAD_WEIGHT * g_total) / acc_unit).max()))
    ref = reference(pb)
    assert _exact_f32(pb.grad0.astype(np.float64) + GRAD_WEIGHT * layer_grads(net, ch))
    np.testing.assert_array_equal(ref.grad, (GRAD_WEIGHT * layer_grads(net, ch)).astype(np.float32))  # chain == oracle
    worst["zeros"] = float(sum(int((p == 0).sum()) for p in ch.pre[:-1]))
    if c.activation == "relu":
        assert worst["zeros"] > 0, f"{c.name}: want pre-activations exactly at the relu kink"
    return worst
