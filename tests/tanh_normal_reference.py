"""fp64 reference of the tanh-Normal policy head and the SAC loss heads, with a per-element error bound  --  TEST INFRASTRUCTURE.

Each function evaluates, in float64, the operation of one kernel at that kernel's fp32 inputs and fp32 constants:
  * head geometry (`Geometry`): s, shift, lo = min + 1e-3f and hi = max - 1e-3f are the kernel's fp32 values, and the branch
    of a dimension is decided by comparing the fp32 action with them, as the kernel does;
  * sample / log-prob of a sample (`sample_dim`), log-prob of a given action and its derivatives (`log_prob_given_dim`), the
    reparameterised backward (`backward_dim`), the entropy estimate (`entropy_dim`), the Normal KL and its derivatives
    (`normal_kl_dim`), and the PPO clip / KL-penalty / DPO head gradients with the entropy term (`ppo_head`);
  * log Phi from scipy.special.log_ndtr and the Mills ratio phi/Phi as sqrt(2/pi) / erfcx(-z/sqrt 2), which has no cancellation
    in either tail.

Every value is an `Err`: the fp64 value and a first-order bound on the error of an fp32 evaluation of the same expression.
Each fp32 operation adds its own rounding, 2^-24 |result| for + - * / (plus 2^-149 for gradual underflow) and k * 2^-23 |result|
for a CUDA math function of k ulp (expf 2, logf 1, log1pf 1, expm1f 1, tanhf 2, atanhf 3, coshf 2, erfcf 4, erfcxf 4), and passes
its inputs' bounds on through |df/dx|.  So the bound of a path is derived from the fp32 operations of that path, and grows only
where the computation is ill-conditioned (z^2 in the Normal density, 1/(1 - x^2) in atanh near the clip band, the difference
of two logs in the KL).  log Phi and the Mills ratio are bounded as the well-conditioned computations they should be: the
error of the input z times the derivative, plus a few ulp; the Mills ratio, below t = -z / sqrt 2 = 64 where the kernels take
it as exp(-z^2/2 - log sqrt(2 pi) - log Phi(z)), also gets that exponent's roundings (2^-24 z^2 and more).  Beyond t = 64 the
exp form is NOT inside the bound: its relative error keeps growing as z^2 2^-24 (5e-4 at z = -200, 6e-2 at z = -1500).

The SAC loss-head references (`sac_actor_seed`, `sac_q_loss`, `sac_alpha_grad`) are exact: on dyadic data whose sums are exact
in any order (`assert_exact_sums`), the only roundings left are the kernels' fp32 constant 1/M, one product with it, and the
division by M of the alpha loss; the reference applies the same roundings, so the kernels must match it bit for bit."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
from scipy.special import erfcx, log_ndtr

from oracle.synth_env import normal2, philox4x32

U = 2.0 ** -24           # unit roundoff of fp32
ULP = 2.0 ** -23         # one ulp, relative, at worst
TINY = 2.0 ** -149       # the smallest fp32 subnormal: absolute rounding of a result in the subnormal range
SQRT_2_OVER_PI = np.sqrt(2.0 / np.pi)
LOG_SQRT_2PI = 0.5 * np.log(2.0 * np.pi)
EPSILON32 = float(np.float32(1e-3))   # the clip band of the kernels (kTanhNormalEpsilon), as the fp32 constant they use
MILLS_ERFCX_FROM = 64.0              # t = -z / sqrt 2 from which the kernels take the Mills ratio as sqrt(2/pi) / erfcx(t)
TAG_SAC = 0x53414331
TAG_PPO_ENTROPY = 0x50504F45
# fp32 constants of the kernels, with their rounding as the bound
C_LOG_SQRT_2PI_ERR = U * LOG_SQRT_2PI
C_LN2_ERR = U * np.log(2.0)


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


class Err:
    """An fp64 value and a bound on the error of its fp32 evaluation (elementwise arrays)."""

    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()

    @staticmethod
    def of(x) -> "Err":
        return x if isinstance(x, Err) else Err(x, 0.0)

    @staticmethod
    def _rnd(v, k=0.5):
        return k * ULP * np.abs(v) + TINY

    def __add__(self, o):
        o = Err.of(o)
        v = self.v + o.v
        return Err(v, self.e + o.e + Err._rnd(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = Err.of(o)
        v = self.v - o.v
        return Err(v, self.e + o.e + Err._rnd(v))

    def __rsub__(self, o):
        return Err.of(o) - self

    def __neg__(self):
        return Err(-self.v, self.e)

    def __mul__(self, o):
        o = Err.of(o)
        v = self.v * o.v
        return Err(v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + Err._rnd(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Err.of(o)
        v = self.v / o.v
        return Err(v, (self.e + np.abs(v) * o.e) / np.abs(o.v) + Err._rnd(v))

    def __rtruediv__(self, o):
        return Err.of(o) / self

    def fn(self, v, dv, ulps):
        """A CUDA math function of `ulps` ulp with value v and derivative dv at self."""
        with np.errstate(invalid="ignore"):
            return Err(v, np.nan_to_num(np.abs(dv) * self.e, nan=0.0, posinf=np.inf) + Err._rnd(v, ulps))

    def where(self, mask, other: "Err") -> "Err":
        return Err(np.where(mask, self.v, other.v), np.where(mask, self.e, other.e))

    def sum(self, axis=-1) -> "Err":
        """A left-to-right fp32 sum: each partial sum adds its rounding; bounded by (n - 1) * U * sum |x_i| + sum e_i."""
        n = self.v.shape[axis]
        v = self.v.sum(axis)
        return Err(v, self.e.sum(axis) + (n - 1) * U * np.abs(self.v).sum(axis) + n * TINY)


def expf(x: Err) -> Err:
    v = np.exp(x.v)
    return x.fn(v, v, 2)


def logf(x: Err) -> Err:
    return x.fn(np.log(x.v), 1.0 / x.v, 1)


def expm1f(x: Err) -> Err:
    return x.fn(np.expm1(x.v), np.exp(x.v), 1)


def tanhf(x: Err) -> Err:
    v = np.tanh(x.v)
    return x.fn(v, 1.0 - v * v, 2)


def atanhf(x: Err) -> Err:
    with np.errstate(divide="ignore", invalid="ignore"):
        return x.fn(np.arctanh(x.v), 1.0 / (1.0 - x.v * x.v), 3)


def coshf(x: Err) -> Err:
    return x.fn(np.cosh(x.v), np.sinh(x.v), 2)


def softplusf(x: Err) -> Err:
    """max(x, 0) + log1p(exp(-|x|)): expf 2 ulp, log1pf 1 ulp, one add."""
    y = np.exp(-np.abs(x.v))
    l1 = np.log1p(y)
    v = np.maximum(x.v, 0.0) + l1
    sig = 0.5 * (1.0 + np.tanh(0.5 * x.v))
    return Err(v, sig * x.e + 2 * ULP * y / (1.0 + y) + Err._rnd(l1, 1) + Err._rnd(v))


def sigmoidf(x: Err) -> Err:
    """1 / (1 + exp(-x)): expf 2 ulp, one add, one divide."""
    with np.errstate(over="ignore"):
        y = np.exp(-x.v)
        v = 1.0 / (1.0 + y)
    return Err(v, v * (1.0 - v) * x.e + v * (2 * ULP * y / (1.0 + y) + 2 * U) + TINY)


def mills(z: Err) -> Err:
    """phi(z) / Phi(z) = sqrt(2/pi) / erfcx(-z / sqrt 2) in fp64.  Bound: the error of z (and of t = -z * 0.7071f, 2^-23 relative)
    through dm/dz = -m (z + m), plus 6 ulp for t >= MILLS_ERFCX_FROM (erfcxf, the divide, the constant) or, below it, the
    roundings of the exponent -z^2/2 - log sqrt(2 pi) - log Phi(z) (2^-24 z^2 and more) and of expf."""
    t = -z.v / np.sqrt(2.0)
    with np.errstate(over="ignore"):
        m = SQRT_2_OVER_PI / erfcx(t)
    dm = np.abs(m * (z.v + m))
    lp = log_ndtr(z.v)
    arg = -0.5 * z.v * z.v - LOG_SQRT_2PI - lp
    alg_exp = m * (2 * ULP + U * (2.0 * z.v * z.v + 2.0 + np.abs(arg)) + ULP * (5.0 + 2.0 * np.abs(lp)))
    alg = np.where(t >= MILLS_ERFCX_FROM, 6 * ULP * m, alg_exp)
    return Err(m, dm * (z.e + 2 * U * np.abs(z.v)) + alg + TINY)


def log_ndtr_f(z: Err) -> Err:
    """log Phi(z) (scipy).  Bound: m(z) times the error of z and of t, plus erfcf / erfcxf (4 ulp) through logf, logf's own ulp,
    and in the erfcx tail the roundings of t * t and of the difference."""
    t = -z.v / np.sqrt(2.0)
    v = log_ndtr(z.v)
    with np.errstate(over="ignore"):
        m = SQRT_2_OVER_PI / erfcx(t)
    ln_half_erfcx = np.log(0.5 * erfcx(np.maximum(t, 3.0)))
    alg = np.where(t >= 3.0, ULP * (5.0 + np.abs(ln_half_erfcx)) + U * (t * t + np.abs(v)), ULP * (5.0 + 2.0 * np.abs(v)))
    return Err(v, m * (z.e + 2 * U * np.abs(z.v)) + alg + TINY)


def _lsp() -> Err:
    return Err(LOG_SQRT_2PI, C_LOG_SQRT_2PI_ERR)


def fldj(x: Err) -> Err:
    """forward log-det-Jacobian of tanh, 2 (log 2 - x - softplus(-2x)), in the kernels' order of operations."""
    return 2.0 * ((Err(np.log(2.0), C_LN2_ERR) - x) - softplusf(-2.0 * x))


# ---------------------------------------------------------------------------------------------------------- head geometry


@dataclass
class Geometry:
    """HeadGeom of the kernels: fp32 s, shift, lo, hi (exact, as the kernel has them), u_lo / u_hi / log s / log eps as Err."""

    s: float
    sh: float
    lo: np.float32
    hi: np.float32
    u_lo: Err
    u_hi: Err
    log_s: Err
    log_eps: Err


def geometry(minimum: float, maximum: float) -> Geometry:
    mn, mx, ep = np.float32(minimum), np.float32(maximum), np.float32(1e-3)
    s, sh = np.float32(0.5) * (mx - mn), np.float32(0.5) * (mn + mx)
    lo, hi = mn + ep, mx - ep
    us = [atanhf((Err(float(b)) - float(sh)) / float(s)) for b in (lo, hi)]
    return Geometry(float(s), float(sh), lo, hi, us[0], us[1], logf(Err(float(s))), logf(Err(EPSILON32)))


def sigma_of(raw: Err, min_scale: float) -> Err:
    return softplusf(raw) + float(np.float32(min_scale))


def branch_of(action32: np.ndarray, g: Geometry) -> np.ndarray:
    """-1 left tail, +1 right tail, 0 inside the clip band: the kernels' fp32 comparisons of the (clipped) fp32 action."""
    a = np.asarray(action32, np.float32)
    ev = np.minimum(np.maximum(a, g.lo), g.hi)
    return np.where(ev <= g.lo, -1, np.where(ev >= g.hi, 1, 0))


def _tails(loc: Err, sigma: Err, g: Geometry):
    """(z, log_prob, mills) of the left and right tails."""
    zl = (g.u_lo - loc) / sigma
    zr = -((g.u_hi - loc) / sigma)
    return [(z, log_ndtr_f(z) - g.log_eps, mills(z)) for z in (zl, zr)]


def _pick(branch, left: Err, right: Err, band: Err) -> Err:
    return left.where(branch < 0, right.where(branch > 0, band))


def log_prob_given_dim(loc, raw, action32, g: Geometry, min_scale: float = 1e-3):
    """tanh_normal_log_prob_given: (lp, d lp / d loc, d lp / d sigma, branch, sigma) of each (row, dim) of a GIVEN fp32 action."""
    loc, raw = Err.of(loc), Err.of(raw)
    sigma = sigma_of(raw, min_scale)
    br = branch_of(action32, g)
    ev = np.minimum(np.maximum(np.asarray(action32, np.float32), g.lo), g.hi).astype(np.float64)
    (zl, lpl, ml), (zr, lpr, mr) = _tails(loc, sigma, g)
    u = atanhf((Err(ev) - g.sh) / g.s)
    z = (u - loc) / sigma
    lp_band = -0.5 * z * z - logf(sigma) - _lsp() - fldj(u) - g.log_s
    lp = _pick(br, lpl, lpr, lp_band)
    d_loc = _pick(br, -ml / sigma, mr / sigma, z / sigma)
    d_sigma = _pick(br, -(ml * zl) / sigma, -(mr * zr) / sigma, (z * z - 1.0) / sigma)
    return lp, d_loc, d_sigma, br, sigma


def sample_dim(loc, raw, eps, g: Geometry, min_scale: float = 1e-3, action32: Optional[np.ndarray] = None):
    """tanh_normal_sample per (row, dim): (action, lp, branch).  The branch is that of `action32` (the kernel's fp32 action, which
    the caller has checked against `action`), or of the fp64 action rounded to fp32 when it is not given."""
    loc, raw, eps = Err.of(loc), Err.of(raw), Err.of(eps)
    sigma = sigma_of(raw, min_scale)
    u = loc + sigma * eps
    a = g.sh + g.s * tanhf(u)
    br = branch_of(np.float32(a.v) if action32 is None else action32, g)
    (_, lpl, _), (_, lpr, _) = _tails(loc, sigma, g)
    lp_band = -0.5 * eps * eps - logf(sigma) - _lsp() - fldj(u) - g.log_s
    return a, _pick(br, lpl, lpr, lp_band), br


def backward_dim(loc, raw, eps, g_action, gl: Err, branch, g: Geometry, min_scale: float = 1e-3):
    """tanh_normal_backward per (row, dim): (d loc, d raw) of gl * log_prob + g_action * action with eps held fixed."""
    loc, raw, eps = Err.of(loc), Err.of(raw), Err.of(eps)
    sigma = sigma_of(raw, min_scale)
    u = loc + sigma * eps
    th = tanhf(u)
    du = Err.of(g_action) * g.s * (1.0 - th * th)
    (zl, _, ml), (zr, _, mr) = _tails(loc, sigma, g)
    d_loc = du + _pick(branch, gl * ml * (-1.0 / sigma), gl * mr * (1.0 / sigma), gl * 2.0 * th)
    d_sigma = du * eps + _pick(branch, gl * ml * (-zl / sigma), gl * mr * (-zr / sigma), gl * (2.0 * th * eps - 1.0 / sigma))
    return d_loc, d_sigma * sigmoidf(raw)


def entropy_dim(loc, raw, eps, g: Geometry, min_scale: float = 1e-3):
    """tanh_normal_entropy_dim and its derivatives: (H, dH/dloc = -2 tanh u', dH/dsigma = 1/sigma - 2 tanh(u') eps', sigma, th)."""
    loc, raw, eps = Err.of(loc), Err.of(raw), Err.of(eps)
    sigma = sigma_of(raw, min_scale)
    u = loc + sigma * eps
    h = (0.5 + _lsp()) + logf(sigma) + g.log_s + fldj(u)
    return h, sigma, tanhf(u)


def normal_kl_dim(mu_b, raw_b, mu, raw, min_scale: float = 1e-3):
    """normal_kl: KL(N(mu_b, sigma_b) || N(mu, sigma)) = 0.5 (dm/sigma)^2 + 0.5 expm1(2 d) - d, d = log sigma_b - log sigma, and its
    derivatives with respect to mu and sigma, in the kernel's arrangement."""
    mu_b, mu = Err.of(mu_b), Err.of(mu)
    sb, s = sigma_of(Err.of(raw_b), min_scale), sigma_of(Err.of(raw), min_scale)
    dm = mu_b - mu
    q = sb * sb + dm * dm
    inv = 1.0 / s
    dls = logf(sb) - logf(s)
    z = dm * inv
    kl = 0.5 * z * z + 0.5 * expm1f(2.0 * dls) - dls
    return kl, -dm * inv * inv, inv - q * inv * inv * inv


# ---------------------------------------------------------------------------------------------------------- PPO heads


def _ambiguous(x: Err, at: float) -> np.ndarray:
    return np.abs(x.v - at) <= x.e


def ppo_head(kind: str, head, action32, logp_old, adv, eps, minimum, maximum, clip_eps=0.2, ent_coef=0.01, b_head=None, kl_coef=0.0,
             dpo_alpha=2.0, dpo_beta=0.6, min_scale=1e-3, ratio: Optional[np.ndarray] = None):
    """The per-row kernel of stx_ppo_tanh_normal_head_grads (kind "clip") and stx_ppo_variant_tanh_normal_head_grads ("kl", "dpo")
    on rows m = 0..mb-1 with action / logp_old / adv / eps already gathered per row.  Returns (d head (mb, 2A), loss rows,
    entropy rows, kl rows) as Err.  `ratio` (optional, fp32 per row) replaces exp(logp - logp_old) by the kernel's own ratio.
    Where a branch condition (the clip band, DPO's y > 0) is within its error bound of the switch point, both sides are
    accepted: the bound of the derivative grows by the difference between the two branches."""
    head = np.asarray(head, np.float64)
    mb, A = head.shape[0], head.shape[1] // 2
    g = geometry(minimum, maximum)
    loc, raw = Err(head[:, :A]), Err(head[:, A:])
    lp, d_loc_lp, d_sig_lp, _, sigma = log_prob_given_dim(loc, raw, action32, g, min_scale)
    h, _, th = entropy_dim(loc, raw, eps, g, min_scale)
    logp, ent = lp.sum(-1), h.sum(-1)
    adv = np.asarray(adv, np.float64)
    inv_m = float(np.float32(1.0) / np.float32(mb))
    ld = logp - np.asarray(logp_old, np.float64)
    r = expf(ld) if ratio is None else Err(np.asarray(ratio, np.float64))
    kl = Err(np.zeros(mb))
    if kind == "clip":
        l1 = r * adv
        rc = np.clip(r.v, 1.0 - clip_eps, 1.0 + clip_eps)
        active = (l1.v < rc * adv) | ((r.v >= 1.0 - clip_eps) & (r.v <= 1.0 + clip_eps))
        loss = -Err(np.minimum(l1.v, rc * adv), l1.e)
        dl = -Err(adv) * r * inv_m
        amb = _ambiguous(r, 1.0 - clip_eps) | _ambiguous(r, 1.0 + clip_eps)
        dlogp = Err(np.where(active, dl.v, 0.0), np.where(active, dl.e, 0.0) + np.where(amb, np.abs(dl.v), 0.0))
    elif kind == "kl":
        kl_d, kl_mu, kl_sig = normal_kl_dim(np.asarray(b_head)[:, :A], np.asarray(b_head)[:, A:], loc, raw, min_scale)
        kl = kl_d.sum(-1)
        loss = -(r * adv) + kl_coef * kl
        dlogp = -Err(adv) * r * inv_m
    else:
        x1, x2 = (r - 1.0) * adv, ld * adv
        t1, t2 = tanhf(x1 / dpo_alpha), tanhf(x2 / dpo_beta)
        y1, y2 = x1 - dpo_alpha * t1, x2 - dpo_beta * t2
        pos = adv >= 0.0
        drift = Err(np.where(pos, np.maximum(y1.v, 0.0), np.maximum(y2.v, 0.0)), np.where(pos, y1.e, y2.e))
        loss = -(r * adv - drift)
        sh1 = 1.0 / coshf(x1 / dpo_alpha)
        plain, full_pos, full_neg = -r * adv, -r * adv * sh1 * sh1, (t2 * t2 - r) * adv
        d = full_pos.where(y1.v > 0, plain).where(pos, full_neg.where(y2.v > 0, plain))
        alt = np.where(pos, np.where(y1.v > 0, plain.v, full_pos.v), np.where(y2.v > 0, plain.v, full_neg.v))
        amb = np.where(pos, _ambiguous(y1, 0.0), _ambiguous(y2, 0.0))
        d = Err(d.v, d.e + np.where(amb, np.abs(d.v - alt), 0.0))
        dlogp = d * inv_m
    ck, ce = float(np.float32(kl_coef) * np.float32(inv_m)), float(np.float32(ent_coef) * np.float32(inv_m))
    dlogp2 = Err(np.broadcast_to(dlogp.v[:, None], d_loc_lp.v.shape), np.broadcast_to(dlogp.e[:, None], d_loc_lp.v.shape))
    eps = Err.of(eps)
    d_loc = dlogp2 * d_loc_lp + ce * 2.0 * th
    d_sig = dlogp2 * d_sig_lp - ce * (1.0 / sigma - 2.0 * th * eps)
    if kind == "kl":
        d_loc = d_loc + ck * kl_mu
        d_sig = d_sig + ck * kl_sig
    d_raw = d_sig * sigmoidf(raw)
    dhead = Err(np.concatenate([d_loc.v, d_raw.v], -1), np.concatenate([d_loc.e, d_raw.e], -1))
    return dhead, loss, ent, kl


# ---------------------------------------------------------------------------------------------------------- noise streams


def philox_normals(seed: int, rows: int, A: int, call: int, tag: int) -> np.ndarray:
    """(rows, A) fp32 standard normals of the head kernels' Philox layout: counter (row, call, (call >> 32) ^ (group << 20) ^
    ((row >> 32) << 8), tag) under key (seed lo, seed hi), four normals per group of four dims.  tag TAG_SAC: stx_tanh_normal_sample;
    TAG_PPO_ENTROPY: the entropy estimate (tests/ppo_continuous_oracle.entropy_noise)."""
    groups = (A + 3) // 4
    m = np.arange(rows, dtype=np.uint64)[:, None]
    gr = np.arange(groups, dtype=np.uint64)[None, :]
    c2 = (np.uint64(call >> 32) ^ (gr << np.uint64(20)) ^ ((m >> np.uint64(32)) << np.uint64(8))) & np.uint64(0xFFFFFFFF)
    r = philox4x32(m, np.uint64(call & 0xFFFFFFFF), c2, np.uint64(tag), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    a0, a1 = normal2(r[0], r[1])
    b0, b1 = normal2(r[2], r[3])
    return np.stack([a0, a1, b0, b1], axis=-1).reshape(rows, groups * 4)[:, :A]


# ---------------------------------------------------------------------------------------------------------- SAC loss heads (exact)


def assert_exact_sums(terms: np.ndarray, unit: float) -> None:
    """Every term is a multiple of `unit` and sum |term| < 2^24 unit: then every partial sum, in any order, is an fp32 number."""
    t = np.asarray(terms, np.float64)
    k = t / unit
    assert np.array_equal(k, np.round(k)), "terms are not multiples of the unit"
    assert np.abs(k).sum() < 2.0 ** 24, "the sum needs more than 24 bits"
    assert np.array_equal(f32(t), t), "a term is not an fp32 number"


def _inv32(M: int) -> float:
    return float(np.float32(1.0) / np.float32(M))


def sac_actor_seed(q1, q2, log_prob, alpha: float, metrics, weight: float):
    """sac_actor_seed_kernel: dq_k = -1/M (fp32 constant) on the first minimum (ties to q1); metrics[0] += weight * sum(alpha lp -
    min q) * (1/M), metrics[1] += weight * sum(-lp) * (1/M)."""
    M = len(q1)
    inv = _inv32(M)
    first = q1 <= q2
    dq1, dq2 = np.where(first, -inv, 0.0), np.where(first, 0.0, -inv)
    terms = alpha * log_prob - np.minimum(q1, q2)
    assert_exact_sums(terms, 2.0 ** -8)
    assert_exact_sums(-log_prob, 2.0 ** -8)
    m = metrics.copy()
    m[0] = f32(m[0] + f32(weight * terms.sum() * inv))
    m[1] = f32(m[1] + f32(weight * (-log_prob).sum() * inv))
    return f32(dq1), f32(dq2), m


def sac_q_loss(q1, q2, nq1, nq2, nlp, reward, done, alpha: float, gamma: float, metrics, weight: float):
    """sac_q_loss_kernel: target = r + (1 - d) gamma (min nq - alpha nlp), e_k = q_k - target, dq_k = (0.5 e_k) * (1/M);
    metrics[2..5] += weight * {0.5 sum(e1^2 + e2^2) 0.5, sum |e1| + |e2| 0.5, sum nq1, sum nq2} * (1/M)."""
    M = len(q1)
    inv = _inv32(M)
    target = reward + np.where(done, 0.0, 1.0) * gamma * (np.minimum(nq1, nq2) - alpha * nlp)
    assert np.array_equal(f32(target), target)
    e1, e2 = q1 - target, q2 - target
    sq, ab = e1 * e1 + e2 * e2, np.abs(e1) + np.abs(e2)
    for t in (sq, ab, nq1, nq2):
        assert_exact_sums(t, 2.0 ** -10 if gamma == 0.75 else 2.0 ** -8)
    m = metrics.copy()
    m[2] = f32(m[2] + f32(weight * 0.5 * sq.sum() * 0.5 * inv))
    m[3] = f32(m[3] + f32(weight * ab.sum() * 0.5 * inv))
    m[4] = f32(m[4] + f32(weight * nq1.sum() * inv))
    m[5] = f32(m[5] + f32(weight * nq2.sum() * inv))
    return f32(0.5 * e1 * inv), f32(0.5 * e2 * inv), m


def sac_alpha_grad(log_prob, alpha: float, target_entropy: float, autotune: bool, grad0: float, grad_weight: float, overwrite: bool,
                   metrics, weight: float):
    """sac_alpha_grad_kernel: loss = alpha * sum(-lp - target_entropy) / M (one fp32 division; fp64 then fp32 rounds the same, since
    53 >= 2 * 24 + 2); grad = (overwrite ? 0 : grad) + autotune * grad_weight * loss; metrics[6] += weight * autotune * loss,
    metrics[7] += weight * alpha."""
    M = len(log_prob)
    terms = -log_prob - target_entropy
    assert_exact_sums(terms, 2.0 ** -8)
    loss = f32(alpha * terms.sum() / M)
    g = f32((0.0 if overwrite else grad0) + (grad_weight * loss if autotune else 0.0))
    m = metrics.copy()
    m[6] = f32(m[6] + weight * (loss if autotune else 0.0))
    m[7] = f32(m[7] + weight * alpha)
    return g, m
