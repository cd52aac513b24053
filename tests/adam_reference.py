"""One optimiser step of the clip + Adam kernel (K4, stoix_b200/csrc/stx_adam.cu) in float64, with a per-element error
bound derived from the kernel's fp32 arithmetic.

`step(p, mu, nu, counts, g, segs, hyper)` takes the state BEFORE the step (what the kernel read) and returns what the step
must produce and how far the kernel may be from it.  Nothing is chained: every GPU test feeds it the kernel's own pre-step
state, so the bounds only have to cover one step's roundings, and they are derived, not tuned (see `_segment`).

The kernel's arithmetic per segment (s_* are per-segment scalars, everything fp32 unless marked):
    g_norm = (float) sqrt(ss)                        ss: double, see NORM_* below
    clip   = g_norm < max_norm ? 1 : max_norm / g_norm
    gs     = grad_scale * clip
    lr     = init_lr * (1 - (float) k / (float) num_updates),  k = sched_count / steps_per_update   (decay; else init_lr)
    bc1    = 1 - powf(b1, count + 1),  bc2 = 1 - powf(b2, count + 1)
  per element:
    ge = g * gs;  m' = b1 * m + (1 - b1) * ge;  v' = b2 * v + (1 - b2) * ge * ge
    p' = p - lr * ((m' / bc1) / (sqrtf(v' / bc2) + eps));  shadow = bf16_rn(p')
  counts[2s] += 1, counts[2s + 1] += 1.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

U32 = 2.0 ** -24          # unit roundoff of fp32 round-to-nearest: |fl(x) - x| <= U32 |x| for normal x
U64 = 2.0 ** -53
TINY = 2.0 ** -149        # >= the absolute rounding error of one fp32 operation in the subnormal range (gradual underflow)
POWF_ULP = 4              # CUDA Math API / CUDA C++ Programming Guide, "Mathematical Functions", single-precision table:
#                           powf(x, y) has a maximum error of 4 ulp over the full range (no -use_fast_math in this build)
KERNEL_THREADS = 132 * 256   # clip_adam_kernel: one block of 256 threads per SM, always 132 blocks
NORM_LOCAL = "local"      # fp32 sum of squares per thread, then double (local and one-shot forms)
NORM_DOUBLE = "double"    # squares of the fp32 gradient summed in double (prenorm form: tc_reduce_kernel)

f32 = np.float32


@dataclass
class Hyper:
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-5
    grad_scale: float = 1.0
    decay: bool = True
    steps_per_update: int = 1
    num_updates: int = 1


Seg = Tuple[int, int, float, float]   # (offset, count, init_lr, max_grad_norm), as ops.AdamPlan takes it


@dataclass
class Step:
    """Expected outputs (float64 / int) and per-element absolute bounds of one step over the whole arena."""
    p: np.ndarray
    mu: np.ndarray
    nu: np.ndarray
    counts: np.ndarray
    gnorm: np.ndarray
    shadow: np.ndarray            # bf16 round-to-nearest-even of the expected p, as float64
    p_bound: np.ndarray
    mu_bound: np.ndarray
    nu_bound: np.ndarray
    gnorm_bound: np.ndarray
    shadow_bound: np.ndarray
    clipped: np.ndarray           # per segment: did the clip trigger
    inside: np.ndarray            # bool mask of the arena: element belongs to a segment


def _gam(k: int, e: float = U32) -> float:
    """Relative bound of k compounded roundings: (1 + e)^k - 1."""
    return (1.0 + e) ** k - 1.0


def bf16_rne(x: np.ndarray) -> np.ndarray:
    """bf16 round-to-nearest-even of fp32 values, returned as float64 (what __float2bfloat16_rn stores)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    nan = np.isnan(np.asarray(x, dtype=np.float32))
    r = np.where(nan, b, r).astype(np.uint32)
    return r.view(np.float32).astype(np.float64)


def norm_items(count: int, threads: int = KERNEL_THREADS) -> int:
    """float4 items one thread squares and sums in fp32 in the local form's grid-stride loop over a segment."""
    return max(1, -(-(count // 4) // threads))


def _segment(p, m, v, g, count_adam, count_sched, seg: Seg, h: Hyper, norm: str):
    """Expected values and bounds of one segment.  All inputs are the fp32 values the kernel read, as float64."""
    off, cnt, init_lr, max_norm = seg
    b1, b2, eps, gsc = (float(f32(x)) for x in (h.b1, h.b2, h.eps, h.grad_scale))
    ob1, ob2 = 1.0 - b1, 1.0 - b2          # exact in fp32 too (Sterbenz: b in [1/2, 1])
    init_lr, max_norm = float(f32(init_lr)), float(f32(max_norm))

    # ---- global norm of the scaled gradient ----
    x = g * gsc                             # exact: 24 x 24 significant bits fit a double
    ss = float(np.dot(x, x))                # relative error <= cnt * U64 (any summation order of non-negative terms)
    gn = math.sqrt(ss)
    if norm == NORM_LOCAL:
        # A thread squares and sums in fp32: ge = g * gs (1 rounding, squared: 2), ge * ge (1), the 3 adds inside a float4
        # item, then one add per item into its accumulator (norm_items float4 items + the scalar tail) -- at most items + 7
        # roundings on any term.  All terms are >= 0, so the per-thread sums, and hence ss, carry at most
        # (1 + U32)^(items + 7) - 1 relatively.  The block / partial sums in double add <= cnt * U64, sqrt in double 1 U64,
        # the cast to float 1 U32.
        m_r = norm_items(cnt) + 7
        eps_n = math.sqrt(1.0 + _gam(m_r)) * (1.0 + (cnt + 2) * U64) * (1.0 + U32) - 1.0
    elif norm == NORM_DOUBLE:
        # (double) o * o is exact, the sums and the two multiplications by grad_scale round in double: (cnt + 4) U64,
        # then sqrt in double and the cast to float (1 U32).
        eps_n = (1.0 + (cnt + 5) * U64) * (1.0 + U32) - 1.0
    else:
        raise ValueError(norm)
    gn_bound = eps_n * gn + TINY
    # the kernel compares its own fp32 norm with max_norm: the case must not sit inside the norm's error band
    if (gn - gn_bound) < max_norm <= (gn + gn_bound):
        raise ValueError(f"segment at {off}: norm {gn:.9g} is within its error bound {gn_bound:.2g} of max_grad_norm {max_norm:.9g}; "
                         "the clip decision is ambiguous -- choose other data")
    clipped = gn >= max_norm
    if clipped:
        gs = gsc * (max_norm / gn)
        # clip = fl(max_norm / g_norm) with g_norm = gn (1 + d), |d| <= eps_n: relative (1 + U32) / (1 - eps_n) - 1; gs = fl(gsc * clip)
        # one more U32
        eps_gs = (1.0 + U32) ** 2 / (1.0 - eps_n) - 1.0
    else:
        gs, eps_gs = gsc, 0.0               # gsc * 1.0f is exact
    GE = g * gs
    eps_g = (1.0 + eps_gs) * (1.0 + U32) - 1.0   # ge = fl(g * gs)

    # ---- moments ----
    # m' = b1 m + ob1 ge: each product rounds at most once (FMA contraction only removes a rounding), the sum once.
    M = b1 * m + ob1 * GE
    E_m = np.abs(b1 * m) * _gam(2) + np.abs(ob1 * GE) * ((1.0 + eps_g) * (1.0 + U32) ** 2 - 1.0) + 3 * TINY
    # v' = b2 v + (ob2 ge) ge: ge enters twice, two products and the sum round.
    V = b2 * v + ob2 * GE * GE
    E_v = np.abs(b2 * v) * _gam(2) + (ob2 * GE * GE) * ((1.0 + eps_g) ** 2 * (1.0 + U32) ** 3 - 1.0) + 4 * TINY

    # ---- per-segment scalars ----
    c = int(count_adam) + 1

    def bias(b):
        pw = b ** c
        BC = 1.0 - pw
        # powf within POWF_ULP ulp of b^c, and ulp(y) <= 2^-23 |y|: |powf - pw| <= 4 * 2^-23 * pw.  1 - powf rounds once.
        # Relative to BC that is 4 * 2^-23 * b^c / (1 - b^c) (large for b2 = 0.999 at small counts), times (1 + U32).
        return BC, (1.0 + POWF_ULP * 2.0 ** -23 * pw / BC) * (1.0 + U32) - 1.0

    BC1, eps_bc1 = bias(b1)
    BC2, eps_bc2 = bias(b2)
    if h.decay:
        k = int(count_sched) // int(h.steps_per_update)          # read before the increment
        q = k / int(h.num_updates)
        LR = init_lr * (1.0 - q)
        # fl(k / N) is off by <= U32 q; 1 - that loses it relative to (1 - q): U32 q / (1 - q) (= U32 (N - 1) on the last
        # update: the cancellation), the subtraction and the product with init_lr round once each.
        eps_lr = 0.0 if q == 1.0 else (1.0 + U32 * q / abs(1.0 - q)) * (1.0 + U32) ** 2 - 1.0
    else:
        LR, eps_lr = init_lr, 0.0

    # ---- update u = (m' / bc1) / (sqrt(v' / bc2) + eps), absolute error propagated through each operation ----
    Q1 = M / BC1
    E_q1 = ((np.abs(M) + E_m) * ((1.0 + U32) / (1.0 - eps_bc1) - 1.0) + E_m) / BC1 + TINY
    R = V / BC2                                                    # >= 0
    E_r = ((V + E_v) * ((1.0 + U32) / (1.0 - eps_bc2) - 1.0) + E_v) / BC2 + TINY
    S = np.sqrt(R)
    with np.errstate(divide="ignore", invalid="ignore"):
        E_s0 = np.minimum(np.where(R > 0, E_r / np.sqrt(np.where(R > 0, R, 1.0)), np.inf), np.sqrt(E_r))   # |sqrt a - sqrt b|
    E_s = E_s0 + U32 * (S + E_s0) + TINY                                                               # sqrtf rounds once
    Dn = S + eps
    E_d = E_s + U32 * (Dn + E_s)                                                                       # + eps rounds once
    Uv = Q1 / Dn
    E_u0 = (E_q1 + np.abs(Uv) * E_d) / (Dn - E_d)
    E_u = E_u0 + U32 * (np.abs(Uv) + E_u0) + TINY                                                      # the division
    # p' = p - lr u: lr carries eps_lr, the product rounds once (unless fused), the difference once (<= 1/2 ulp(p')).
    Pn = p - LR * Uv
    E_lu = LR * E_u * (1.0 + eps_lr) + LR * np.abs(Uv) * eps_lr
    E_prod = E_lu + U32 * (LR * np.abs(Uv) + E_lu)
    E_p = E_prod + U32 * (np.abs(Pn) + E_prod) + TINY
    return dict(p=Pn, mu=M, nu=V, gnorm=gn, p_b=E_p, mu_b=E_m, nu_b=E_v, gn_b=gn_bound, clipped=clipped)


def step(p, mu, nu, counts, g, segs: Sequence[Seg], hyper: Hyper, norm: str = NORM_LOCAL) -> Step:
    """Expected result of one clip + Adam step from the pre-step state (fp32 arrays of the whole arena, int counts[2 nseg])."""
    p, mu, nu, g = (np.asarray(a, dtype=np.float32).astype(np.float64) for a in (p, mu, nu, g))
    counts = np.asarray(counts, dtype=np.int64)
    out = {k: a.copy() for k, a in (("p", p), ("mu", mu), ("nu", nu))}
    bnd = {k: np.zeros_like(p) for k in ("p", "mu", "nu")}
    inside = np.zeros(p.shape, bool)
    gnorm, gn_b, clipped = [], [], []
    for s, seg in enumerate(segs):
        off, cnt = int(seg[0]), int(seg[1])
        sl = slice(off, off + cnt)
        r = _segment(p[sl], mu[sl], nu[sl], g[sl], counts[2 * s], counts[2 * s + 1], seg, hyper, norm)
        for k in ("p", "mu", "nu"):
            out[k][sl], bnd[k][sl] = r[k], r[k + "_b"]
        inside[sl] = True
        gnorm.append(r["gnorm"]), gn_b.append(r["gn_b"]), clipped.append(r["clipped"])
    new_counts = counts.copy()
    new_counts[: 2 * len(segs)] += 1
    shadow = bf16_rne(out["p"].astype(np.float32))
    # shadow of the expected p: within the p bound plus half a bf16 ulp (2^-9 relative) of the value
    sh_b = bnd["p"] + 2.0 ** -8 * (np.abs(out["p"]) + bnd["p"])
    return Step(out["p"], out["mu"], out["nu"], new_counts, np.array(gnorm), shadow, bnd["p"], bnd["mu"], bnd["nu"],
                np.array(gn_b), sh_b, np.array(clipped), inside)


def check(got: dict, want: Step, pre: dict, label: str = "") -> None:
    """Compare one step's outputs with the reference.  got / pre: dict of numpy arrays p, mu, nu, counts, gnorm (got only), and
    optionally shadow (bf16 as float64 / any float) and g (the gradient arena, pre = before the step, got = after).
    Exact: counts; shadow == bf16_rne(got p); every float outside the segments unchanged in p, mu, nu, shadow; the gradient
    arena unchanged.  Within the bounds: p, mu, nu, gnorm."""
    tag = f"{label}: " if label else ""
    np.testing.assert_array_equal(np.asarray(got["counts"]), want.counts, err_msg=f"{tag}counts")
    for k, bound in (("p", want.p_bound), ("mu", want.mu_bound), ("nu", want.nu_bound)):
        a = np.asarray(got[k], dtype=np.float32).astype(np.float64)
        exp = getattr(want, k)
        err = np.abs(a - exp)
        bad = ~(err <= bound)
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            ratio = float(np.max(np.where(want.inside, err / np.maximum(bound, 1e-300), 0.0)))
            raise AssertionError(f"{tag}{k}: {int(bad.sum())} elements outside the bound (first at {i}: got {a[i]!r}, want {exp[i]!r}, "
                                 f"bound {bound[i]:.3g}, inside a segment: {bool(want.inside[i])}); worst err/bound {ratio:.3g}")
        out = ~want.inside
        if out.any() and not np.array_equal(a[out].view(np.uint64), np.asarray(pre[k], np.float32).astype(np.float64)[out].view(np.uint64)):
            raise AssertionError(f"{tag}{k}: a float outside the segments changed")
    gn = np.asarray(got["gnorm"], dtype=np.float32).astype(np.float64)[: len(want.gnorm)]
    bad = ~(np.abs(gn - want.gnorm) <= want.gnorm_bound)
    if bad.any():
        raise AssertionError(f"{tag}gnorm: got {gn.tolist()}, want {want.gnorm.tolist()}, bound {want.gnorm_bound.tolist()}")
    if "shadow" in got and got["shadow"] is not None:
        sh = np.asarray(got["shadow"], dtype=np.float64)
        p32 = np.asarray(got["p"], dtype=np.float32)
        rne = bf16_rne(p32)
        inside = want.inside
        if not np.array_equal(sh[inside], rne[inside]):
            i = int(np.flatnonzero(sh[inside] != rne[inside])[0])
            raise AssertionError(f"{tag}shadow != bf16_rn(new params) at {int(np.flatnonzero(inside)[i])}")
        if not np.array_equal(sh[~inside], np.asarray(pre["shadow"], np.float64)[~inside]):
            raise AssertionError(f"{tag}shadow: a value outside the segments changed")
    if "g" in got and got["g"] is not None:
        if not np.array_equal(np.asarray(got["g"], np.float32).view(np.uint32), np.asarray(pre["g"], np.float32).view(np.uint32)):
            raise AssertionError(f"{tag}the gradient arena changed")


def worst_relative_bounds(want: Step) -> dict:
    """Largest bound / |value| over the segment elements whose value is not tiny: what the derivations allow, for the record."""
    res = {}
    for k in ("p", "mu", "nu"):
        v, b = np.abs(getattr(want, k))[want.inside], getattr(want, k + "_bound")[want.inside]
        big = v > 1e-6 * max(float(v.max()) if v.size else 0.0, 1e-30)
        res[k] = float((b[big] / v[big]).max()) if big.any() else 0.0
    res["gnorm"] = float(max((want.gnorm_bound / np.maximum(want.gnorm, 1e-300)).tolist() or [0.0]))
    return res


# ---------------------------------------------------------------------------------------------------------------------------
# Segment layouts and pre-step states shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------------


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


# The 8-segment layout: scalar tail only (1, 2, 3), float4 body + tail (5, 131), one float4 short of / one past a full grid
# stride of 132 x 256 threads (135168 floats), several grid-stride passes (3 x 135168 + 7); 8 = the segment limit.
STRIDE = 4 * KERNEL_THREADS
EIGHT_COUNTS = (1, 2, 3, 5, 131, STRIDE - 1, STRIDE + 1, 3 * STRIDE + 7)


def layout(name: str) -> Tuple[List[Seg], int]:
    """(segments, arena length) of a named layout."""
    from stoix_b200 import ops

    if name == "bench":   # ff_ppo's actor / critic arena: MLP [256, 256], obs dim 64, 8 actions (bench.py's workload)
        sa, sc = ops.MlpSpec((64, 256, 256, 8)), ops.MlpSpec((64, 256, 256, 1))
        _, coff, total = ops.arena_offsets(sa, sc)
        return [(0, sa.param_count, 3e-4, 0.5), (coff, sc.param_count, 3e-4, 0.5)], total
    if name == "sac":     # ff_sac: actor, the [q1 | q2] block as ONE optimiser, the 1-element log_alpha segment
        from stoix_b200.systems.sac.ff_sac import sac_arena_layout

        sa = ops.MlpSpec((17, 256, 256, 256, 256, 12), activation="silu")
        sq = ops.MlpSpec((23, 256, 256, 256, 256, 1), activation="silu", use_layer_norm=True)
        lay = sac_arena_layout(sa, sq)
        return [(lay["actor"], sa.param_count, 3e-4, 0.5), (lay["q1"], lay["q_block"], 3e-4, 0.5), (lay["alpha"], 1, 3e-4, 0.5)], lay["total"]
    if name == "eight":
        segs, off = [], 0
        for i, cnt in enumerate(EIGHT_COUNTS):
            segs.append((off, cnt, 1e-3 * (1 + i % 3), 0.5))
            off = _pad8(off + cnt) + 8          # at least 8 floats of padding between segments
        return segs, off
    raise KeyError(name)


LAYOUTS = ("bench", "sac", "eight")


def make_state(segs: Sequence[Seg], total: int, rng: np.random.Generator, *, counts=None):
    """A pre-step state with sentinel values in the padding (so that writes outside the segments show), nu >= 0."""
    p = np.full(total, 7.25, np.float32)
    mu = np.full(total, -3.5, np.float32)
    nu = np.full(total, 11.0, np.float32)
    for off, cnt, _, _ in segs:
        p[off:off + cnt] = rng.standard_normal(cnt) * 0.3
        mu[off:off + cnt] = rng.standard_normal(cnt) * 1e-3
        nu[off:off + cnt] = np.abs(rng.standard_normal(cnt)) * 1e-5
    c = np.zeros(2 * len(segs), np.int32) if counts is None else np.asarray(counts, np.int32)
    return p, mu, nu, c


def make_grad(segs: Sequence[Seg], total: int, rng: np.random.Generator, grad_scale: float, step: int, pad_value: float = 1e3):
    """Gradient arena for one step: segment 0 has an all-zero gradient on odd steps, the rest alternate between a norm far
    above max_grad_norm (clip active) and far below it (inactive); the padding holds `pad_value` (the local kernel must not
    read it)."""
    g = np.full(total, pad_value, np.float32)
    for s, (off, cnt, _, mgn) in enumerate(segs):
        if s == 0 and step % 2 == 1:
            g[off:off + cnt] = 0.0
            continue
        active = (s + step) % 2 == 0
        target = mgn * (4.0 if active else 0.25) / grad_scale    # norm of grad_scale * g, far from the clip threshold
        x = rng.standard_normal(cnt)
        g[off:off + cnt] = (x * (target / max(np.linalg.norm(x), 1e-30))).astype(np.float32)
    return g
