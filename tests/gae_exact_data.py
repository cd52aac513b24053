"""Exactly representable data for the K2 scan (stx_gae.cu) -- TEST INFRASTRUCTURE (like rnn_exact_data.py).

K2 evaluates the reverse recurrence acc_t = d_t + c_t acc_{t+1} as a composition of affine maps: each thread scans kL steps,
32 chunk maps are composed by a warp shuffle scan, segments of 32 kL steps are walked from the end with a carry, and the
TMA kernel does the same on (kGE x kGT) tiles.  Each launch form associates the maps differently, so on random data they
differ in the last bits.  Here they cannot:

* every coefficient c_t is 0 or 1: gamma = lambda = 1 and the flags set c to 0 (PPO form), the discount / lambda /
  truncation arrays are in {0, 1} (generic and lambda forms), lambda in {0, 1} or a {0, 1} array (lambda forms);
* rewards, values, bootstrap values and Q rows are small integers, reward_scale is a power of two.

Then every d_t, every product of c's and every fma of the scan is an integer below 2^24 (asserted per case from the sum of
|d| along each env), so any association gives the fp64 result.  The advantage statistics are exact too: each thread sums
its advantages and their squares in fp32 (asserted below 2^24 for the form with the most elements per thread), the block
and grid sums are fp64 sums of integers, and `stats` below repeats the kernel's finishing operations in fp64.

`launch_form` mirrors the host selection of launch_gae (tuning code, E, alignment, input form).  It is a coverage aid and
gives the per-thread element counts of the bound, not an oracle: tests/test_gae_exact_data.py asserts that the cases reach
every instantiation of gae_scan_kernel for each input form, every gae_tma_kernel shape and the TMA fallback.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from fractions import Fraction
from functools import lru_cache
from typing import Dict, Optional, Tuple

import numpy as np

from oracle import ppo_oracle as O
from tests import pqn_oracle as P

UNIT_LIMIT = 2 ** 24     # fp32 holds every integer below this exactly
NUM_SMS = 132            # kNumSMs
CHUNKS = 32              # kChunks

# every code stx_gae_set_tuning accepts: 0 = the default selection; 2, 4, 8 = gae_scan_kernel<In, 4, quads>; 416 = two resident
# 512-thread blocks per SM; 500 / 501 = the TMA kernel's 32x128 / 64x64 tiles (PPO form only)
CODES = (0, 2, 4, 8, 416, 500, 501)

# input form of each face: which In struct of stx_gae.cu the call runs
FACES = {
    "gae_ppo": "PpoIn",                        # ops.gae_ppo: gamma = lambda = 1, done / truncated flags, reward_scale 2 or 1/2
    "gae_generic": "GenericIn",                # ops.gae_generic, scalar lambda = 1, no truncation
    "gae_generic_trunc": "GenericIn",          # ... scalar lambda = 1, {0, 1} truncation array
    "gae_generic_lam_t": "GenericIn",          # ... {0, 1} lambda array, no truncation
    "gae_generic_lam_t_trunc": "GenericIn",    # ... {0, 1} lambda array and truncation array
    "q_lambda": "LambdaIn",                    # ops.q_lambda: gamma = lambda = 1, done / truncated flags, A columns
    "lambda_returns": "LambdaIn",              # ops.lambda_returns: {0, 1} discounts, scalar lambda = 1, v_t (T, E) (A = 1)
    "lambda_returns_lam_t": "LambdaIn",        # ... {0, 1} lambda array, v_t (T, E, A)
}
STANDARDIZING_FACES = ("gae_ppo", "gae_generic_lam_t_trunc")

# (T, E): one step, one segment minus one, exactly one, one plus one, two, a ragged last one, several; E a multiple of every
# block's envs (128 k), 128 k +- 4, E % 4 != 0 (the VEC = 1 kernel), E % 16 == 0 with E % kGE != 0 for every TMA tile width
# (48, 96 = 32 . 3, 16912 = 128 . 132 + 16) and T % kGT != 0; 16912 also gives every TMA shape more tiles than blocks
SHAPES = ((1, 132), (4, 37), (4, 512), (127, 124), (128, 128), (129, 48), (129, 16912), (256, 260), (300, 96), (300, 1020),
          (513, 40), (513, 37))

# the large shapes at which launch_gae's default selection picks its other paths (tests/test_gae_exact_gpu.py)
DEFAULT_PATH_SHAPES = {
    "gae_ppo": ((4, 32772), (4, 262148), (129, 32768), (4, 65536)),   # TMA declines (E % 16) -> <4,8>; -> 4xx; TMA 32x128; 64x64
    "gae_generic_lam_t_trunc": ((4, 262144),),                        # the 4xx default (E / 4 >= 65536)
    "q_lambda": ((4, 262144),),
    "lambda_returns_lam_t": ((3, 262144),),
}


# ---------------------------------------------------------------------------------------------------------------------
# host-logic mirror (launch_gae in stx_gae.cu)
# ---------------------------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class Form:
    kind: str            # "scan" (gae_scan_kernel<In, VEC, QUADS, kL, MINB>) or "tma" (gae_tma_kernel<kGE, kGT>)
    a: int               # scan: VEC;   tma: kGE
    b: int               # scan: QUADS; tma: kGT
    kL: int = 4
    minb: int = 1

    @property
    def name(self) -> str:
        return f"scan<{self.a},{self.b},{self.kL},{self.minb}>" if self.kind == "scan" else f"tma<{self.a},{self.b}>"

    def elements_per_thread(self, T: int, E: int) -> int:
        """Most advantages one thread adds into its fp32 lsum / lsq."""
        if self.kind == "scan":
            return self.kL * self.a * -(-T // (self.kL * CHUNKS))
        kGE, kGT = self.a, self.b
        tiles = -(-E // kGE)
        per_block = -(-tiles // min(tiles, NUM_SMS))
        return (kGT // CHUNKS) * 4 * -(-T // kGT) * per_block


def launch_form(face: str, code: int, E: int, vec4: Optional[bool] = None, tma_aligned: bool = True) -> Form:
    """The kernel launch_gae runs.  vec4: E % 4 == 0 and the pointers the entry point checks are 16-byte aligned (default:
    E % 4 == 0); tma_aligned: done / truncated 16-byte aligned (the PPO form's TMA condition besides E % 16)."""
    vec4 = (E % 4 == 0) if vec4 is None else vec4
    if vec4 and FACES[face] == "PpoIn" and (code in (500, 501) or (code == 0 and E >= 32768)) and E % 16 == 0 and tma_aligned:
        wide = code == 501 or (code != 500 and E >= 65536)
        return Form("tma", 64, 64) if wide else Form("tma", 32, 128)
    forced = code in (2, 4, 8)
    if vec4 and (code == 416 or (not forced and E // 4 >= 65536)):
        return Form("scan", 4, 16, 4, 2)
    if vec4:
        qt = E // 4
        return Form("scan", 4, code if forced else (8 if qt >= 8 * NUM_SMS * 2 else (4 if qt >= 4 * NUM_SMS else 2)))
    return Form("scan", 1, 16)


# the 5 gae_scan_kernel instantiations launch_gae has per input form, and the 2 gae_tma_kernel shapes
SCAN_FORMS = tuple(Form("scan", *f) for f in ((4, 16, 4, 2), (4, 8, 4, 1), (4, 4, 4, 1), (4, 2, 4, 1), (1, 16, 4, 1)))
TMA_FORMS = (Form("tma", 32, 128), Form("tma", 64, 64))


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------


@dataclass
class Case:
    face: str
    T: int
    E: int
    inputs: Dict[str, np.ndarray]          # the arrays the face takes, float32 / bool, every value exact
    scalars: Dict[str, float]              # gamma, lambda, reward_scale as the face takes them
    d: np.ndarray                          # (T, E) int64: the affine map of each step, acc_t = d_t + c_t acc_{t+1}
    c: np.ndarray                          # (T, E) int64 in {0, 1}
    v: np.ndarray                          # (T, E) int64: what the targets add to acc (v_tm1; 0 for the lambda forms)
    adv: np.ndarray                        # (T, E) float32 oracle result (the lambda forms: None)
    targets: np.ndarray                    # (T, E) float32 oracle result


def _flags(rng, shape, p):
    return rng.random(shape) < p


def _resets(rng, T, E, p=0.04):
    """{0, 1} coefficient pattern: c = 0 with probability p; env 0 never resets (one chain through every segment), env 1
    resets every step, env 2 resets exactly at the segment starts of the 2- and 4-step forms (t % 64 == 0)."""
    zero = _flags(rng, (T, E), p)
    if E >= 3:
        zero[:, 0], zero[:, 1] = False, True
        zero[:, 2] = (np.arange(T) % 64) == 0
    return zero


def _ints(rng, shape, lo=-2, hi=2):
    return rng.integers(lo, hi + 1, size=shape)


@lru_cache(maxsize=None)
def make_case(face: str, T: int, E: int) -> Case:
    """The exact case of `face` at (T, E), with its fp64 oracle results (cached: every tuning code reuses it)."""
    assert face in FACES
    rng = np.random.default_rng(zlib.crc32(f"{face}/{T}/{E}".encode()))
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    zero = _resets(rng, T, E)
    if face == "gae_ppo":
        rs = 0.5 if (T + E) % 2 else 2.0
        reward = _ints(rng, (T, E), -1, 1) * (2 if rs == 0.5 else 1)
        value, boot = _ints(rng, (T, E)), _ints(rng, (T, E))
        # a reset is a done (bootstrap dropped) or a truncation (bootstrap kept, chain cut)
        done = zero & _flags(rng, (T, E), 0.5)
        trunc = zero & ~done
        done |= trunc & _flags(rng, (T, E), 0.2)          # done and truncated together: done wins the discount
        disc = 1 - done.astype(np.int64)
        d = (reward * 2 if rs == 2.0 else reward // 2) + disc * boot - value
        c = disc * (1 - trunc.astype(np.int64))
        inputs = dict(reward=f32(reward), value=f32(value), bootstrap_value=f32(boot), done=done, truncated=trunc)
        scalars = dict(gamma=1.0, gae_lambda=1.0, reward_scale=rs)
        r_t, d_t, tr = O.ppo_gae_inputs(reward, done, trunc, 1.0, rs)
        adv, tgt = O.gae(r_t, d_t, 1.0, v_tm1=value.astype(np.float64), v_t=boot.astype(np.float64), truncation_t=tr, time_major=True)
        return _finish(Case(face, T, E, inputs, scalars, d, c, value, f32(adv), f32(tgt)))
    if face.startswith("gae_generic"):
        r, v_tm1, v_t = _ints(rng, (T, E)), _ints(rng, (T, E)), _ints(rng, (T, E))
        # split the zero coefficients between the discount, lambda and truncation arrays the face has
        use_lam, use_tr = "lam_t" in face, "trunc" in face
        which = rng.integers(0, 1 + use_lam + use_tr, size=(T, E))
        disc = 1 - (zero & (which == 0)).astype(np.int64)
        lam = 1 - (zero & (which == 1)).astype(np.int64) if use_lam else np.ones((T, E), np.int64)
        tr = (zero & (which == (1 + use_lam))).astype(np.int64) if use_tr else np.zeros((T, E), np.int64)
        if use_tr:   # a truncated step whose discount is also 0, and a 1 in lambda there: c stays 0
            tr |= (disc == 0) & _flags(rng, (T, E), 0.3)
        d = r + disc * v_t - v_tm1
        c = disc * lam * (1 - tr)
        inputs = dict(r_t=f32(r), discount_t=f32(disc), v_tm1=f32(v_tm1), v_t=f32(v_t))
        inputs["lambda_"] = f32(lam) if use_lam else None
        inputs["truncation_t"] = f32(tr) if use_tr else None
        scalars = dict(lambda_=1.0)
        adv, tgt = O.gae(r, disc, lam if use_lam else 1.0, v_tm1=v_tm1, v_t=v_t, truncation_t=tr if use_tr else None, time_major=True)
        return _finish(Case(face, T, E, inputs, scalars, d, c, v_tm1, f32(adv), f32(tgt)))
    # lambda returns: G_t = r_t + disc_t [(1 - lam_t) v_t + lam_t G_{t+1}], G_T = v_{T-1}; v_t = max over A columns of q
    A = 1 if face == "lambda_returns" else (1, 3, 18)[(T + E) % 3]
    q = _ints(rng, (T, E, A), -2, 2)                       # 5 levels: ties across actions are common
    if A > 1 and E >= 1:
        q[:, 0, :] = 1                                     # env 0: every action tied
    vmax = q.max(axis=-1)
    r = _ints(rng, (T, E))
    if face == "q_lambda":
        done = zero & _flags(rng, (T, E), 0.5)
        trunc = (zero & ~done) | (done & _flags(rng, (T, E), 0.2))
        disc = 1 - (done | trunc).astype(np.int64)
        lam = np.ones((T, E), np.int64)
        inputs = dict(q_t=f32(q), reward=f32(r), done=done, truncated=trunc)
        scalars = dict(gamma=1.0, q_lambda_=1.0)
        want = P.batch_q_lambda(r, disc, q, 1.0)
    else:
        use_lam = face == "lambda_returns_lam_t"
        which = rng.integers(0, 1 + use_lam, size=(T, E))
        disc = 1 - (zero & (which == 0)).astype(np.int64)
        lam = 1 - (zero & (which == 1)).astype(np.int64) if use_lam else np.ones((T, E), np.int64)
        inputs = dict(r_t=f32(r), discount_t=f32(disc), v_t=f32(q if use_lam else q[..., 0]))
        inputs["lambda_"] = f32(lam) if use_lam else None
        scalars = dict(lambda_=1.0)
        want = P.batch_q_lambda(r, disc, q, lam) if use_lam else P.batch_lambda_returns(r, disc, q[..., 0], 1.0)
    last = np.zeros((T, E), bool)
    last[T - 1] = True
    d = r + disc * np.where(last, 1, 1 - lam) * vmax
    c = np.where(last, 0, disc * lam)
    return _finish(Case(face, T, E, inputs, scalars, d, c, np.zeros((T, E), np.int64), None, f32(want)))


def _finish(case: Case) -> Case:
    check_exact(case)
    return case


# ---------------------------------------------------------------------------------------------------------------------
# the exactness invariant and the statistics
# ---------------------------------------------------------------------------------------------------------------------


def column_bound(case: Case) -> int:
    """Largest |value| any affine-map composition, partial scan or target of one env can reach: the sum of |d| along the
    env plus the largest |v| (every c is 0 or 1, so each composed map is x -> B + {0, 1} x with |B| <= sum |d|)."""
    return int(np.abs(case.d).sum(axis=0).max() + np.abs(case.v).max())


def forms_of(case: Case):
    return {launch_form(case.face, code, case.E) for code in CODES}


def stats_bound(case: Case) -> Tuple[int, int]:
    """(largest fp32 lsq any thread of any form of this case accumulates, the same bound for lsum), from the element count
    per thread and the largest |adv|."""
    n = max(f.elements_per_thread(case.T, case.E) for f in forms_of(case))
    m = int(np.abs(case.adv.astype(np.float64)).max())
    return n * m * m, n * m


def check_exact(case: Case) -> None:
    assert np.isin(case.c, (0, 1)).all(), f"{case.face} {case.T}x{case.E}: a coefficient is not 0 or 1"
    assert column_bound(case) < UNIT_LIMIT, f"{case.face} {case.T}x{case.E}: partial sums reach {column_bound(case)} (limit 2^24)"
    for name, a in case.inputs.items():
        if a is not None and a.dtype == np.float32:
            assert np.array_equal(a, np.round(a)) and np.abs(a).max() < 2 ** 12, f"{case.face}: {name} is not a small integer"
    if case.face in STANDARDIZING_FACES:
        sq, s = stats_bound(case)
        assert sq < UNIT_LIMIT and s < UNIT_LIMIT, f"{case.face} {case.T}x{case.E}: per-thread sum of squares bound {sq} (limit 2^24)"


def stats(adv: np.ndarray) -> np.ndarray:
    """The kernel's [(float)(S / n), (float)(1 / sqrt(var + 1e-5))] in fp64 with its operation order: S and Q are exact
    integers here; var = fma(-mean, mean, Q / n) (nvcc contracts Q / n - mean * mean into one DFMA)."""
    a = np.asarray(adv, np.float64)
    assert np.array_equal(a, np.round(a))
    n = float(a.size)
    S, Q = float(a.sum()), float((a * a).sum())
    assert abs(S) < 2 ** 53 and Q < 2 ** 53
    mean = S / n
    var = float(Fraction(Q / n) - Fraction(mean) * Fraction(mean))   # one rounding, as the fused multiply-add
    rstd = 1.0 / np.sqrt(var + 1e-5)
    return np.array([mean, rstd], np.float32)


def standardized(adv: np.ndarray, st: np.ndarray) -> np.ndarray:
    """standardize_inplace_kernel: (adv - mean) * rstd, each operation rounded to fp32."""
    a = np.asarray(adv, np.float32)
    return ((a - np.float32(st[0])).astype(np.float32) * np.float32(st[1])).astype(np.float32)


def sequential_scan(case: Case) -> Tuple[Optional[np.ndarray], np.ndarray]:
    """The recurrence in int64, one step at a time from the end, from the case's (d, c, v): (advantages or None, targets)."""
    acc = np.zeros(case.E, np.int64)
    out = np.zeros((case.T, case.E), np.int64)
    for t in range(case.T - 1, -1, -1):
        acc = case.d[t] + case.c[t] * acc
        out[t] = acc
    if FACES[case.face] == "LambdaIn":
        return None, out
    return out, out + case.v
