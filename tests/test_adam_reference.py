"""CPU checks of the one-step clip + Adam reference (tests/adam_reference.py) that tests/test_adam_exact_gpu.py rests on.

A NumPy float32 emulation of clip_adam_kernel (stoix_b200/csrc/stx_adam.cu) -- the same operations in the same order, every
FMA contraction the compiler may choose built from exact float64 products -- must pass the reference's bounds on every
layout the GPU tests run, with both norm forms.  The same emulation with one defect each must fail them, and so must any
output off by 1e-3 relative: the bounds are derived, and tight enough to matter."""
import numpy as np
import pytest

from tests import adam_reference as R

f32 = np.float32
NONE, FIRST, SECOND = "none", "fma_first", "fma_second"   # which product of `a * b + c * d` the compiler fuses


def _fma(a, b, c):
    """fma in fp32 from the exact float64 product (24 x 24 bits) and one rounding of the sum to fp32."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _local_norm(x: np.ndarray, fma: str, drop_partial: bool) -> f32:
    """phase 1 of clip_adam_kernel<false, 0>: per thread an fp32 sum over its float4 items (grid stride 132 x 256) and the
    scalar tail, then per-block partials in double, summed in double."""
    T = R.KERNEL_THREADS
    n4 = x.size // 4
    body = x[: 4 * n4].reshape(n4, 4)
    if fma == NONE:
        q = ((body[:, 0] * body[:, 0] + body[:, 1] * body[:, 1]) + body[:, 2] * body[:, 2]) + body[:, 3] * body[:, 3]
    else:
        q = _fma(body[:, 3], body[:, 3], _fma(body[:, 2], body[:, 2], _fma(body[:, 1], body[:, 1], body[:, 0] * body[:, 0])))
    rounds = -(-n4 // T)
    qq = np.zeros(rounds * T, f32)
    qq[:n4] = q
    acc = np.zeros(T, f32)
    for r in range(rounds):
        acc = acc + qq[r * T:(r + 1) * T]
    tail = x[4 * n4:]
    nt = tail.size
    acc[:nt] = acc[:nt] + tail * tail if fma == NONE else _fma(tail, tail, acc[:nt])
    partials = acc.astype(np.float64).reshape(132, 256).sum(axis=1)
    if drop_partial:
        partials[0] = 0.0
    return f32(np.sqrt(partials.sum()))


def emulate(p, mu, nu, counts, g, shadow, segs, h: R.Hyper, norm=R.NORM_LOCAL, fma=NONE, defect=None):
    """clip_adam_kernel in NumPy float32.  defect: None or one of DEFECTS."""
    p, mu, nu, g = (np.array(a, f32) for a in (p, mu, nu, g))
    shadow = np.array(shadow, np.float64)
    p0 = p.copy()
    counts = np.array(counts, np.int64)
    b1, b2, eps, gsc = f32(h.b1), f32(h.b2), f32(h.eps), f32(h.grad_scale)
    ob1, ob2 = f32(1) - b1, f32(1) - b2
    gnorm = np.zeros(len(segs), f32)
    for s, (off, cnt, init_lr, mgn) in enumerate(segs):
        sl = slice(off, off + cnt)
        gs_in = g[sl]
        if norm == R.NORM_LOCAL:
            gn = _local_norm(gs_in * gsc, fma, defect == "partial_dropped")
        else:
            part = np.sum(gs_in.astype(np.float64) ** 2)
            gn = f32(np.sqrt(part * float(gsc) * float(gsc)))
        mgn = f32(mgn)
        trig = gn < mgn
        if defect == "clip_inverted":
            trig = not trig
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            clip = f32(1) if trig else mgn / gn
        c = counts[2 * s] + (0 if defect == "bias_count" else 1)
        lr = f32(init_lr)
        if h.decay:
            k = (counts[2 * s + 1] + (1 if defect == "schedule_after_increment" else 0)) // h.steps_per_update
            lr = f32(init_lr) * (f32(1) - f32(k) / f32(h.num_updates))
        gs = gsc * clip
        bc1 = f32(1) - np.power(b1, f32(c))
        bc2 = f32(1) - np.power(b2, f32(c))
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            ge = g[sl] * gs
            m, v, pp = mu[sl], nu[sl], p[sl]
            if fma == NONE:
                me = b1 * m + ob1 * ge
                ve = b2 * v + (ob2 * ge) * ge
            elif fma == FIRST:
                me = _fma(b1, m, ob1 * ge)
                ve = _fma(b2, v, (ob2 * ge) * ge)
            else:
                me = _fma(ob1, ge, b1 * m)
                ve = _fma(ob2 * ge, ge, b2 * v)
            u = (me / bc1) / (np.sqrt(ve / bc2) + eps)
            pn = pp - lr * u if fma == NONE else _fma(-lr, u, pp)
        keep = np.zeros(cnt, bool)
        if defect == "tail_shifted" and cnt % 4:
            keep[4 * (cnt // 4)] = True          # the loop starts one element late: the first tail element is never written
        mu[sl] = np.where(keep, m, me)
        nu[sl] = np.where(keep, v, ve)
        p[sl] = np.where(keep, pp, pn)
        src = p0[sl] if defect == "shadow_pre_step" else p[sl]
        shadow[sl] = np.where(keep, shadow[sl], R.bf16_rne(src))
        gnorm[s] = gn
    counts[: 2 * len(segs)] += 1
    return dict(p=p, mu=mu, nu=nu, counts=counts, gnorm=gnorm, shadow=shadow, g=g)


DEFECTS = ("clip_inverted", "schedule_after_increment", "partial_dropped", "tail_shifted", "shadow_pre_step", "bias_count")

_cache = {}


def _setup(name):
    if name not in _cache:
        _cache[name] = R.layout(name)
    return _cache[name]


def _run(name, norm, fma, defect=None, steps=2, first_count=10, perturb=None):
    """Emulated steps from a fresh state; each checked against the reference from its own pre-step state.  spu 3 and 4 updates:
    the steps read schedule counts 10, 11 (the last update; 11 is its last step)."""
    segs, total = _setup(name)
    rng = np.random.default_rng(len(segs) * 7 + first_count)
    p, mu, nu, counts = R.make_state(segs, total, rng, counts=[first_count] * (2 * len(segs)))
    shadow = R.bf16_rne(p)
    for st in range(steps):
        h = R.Hyper(grad_scale=(1.0, 0.25)[st % 2], decay=True, steps_per_update=3, num_updates=4)
        g = R.make_grad(segs, total, rng, h.grad_scale, st)
        pre = dict(p=p, mu=mu, nu=nu, counts=counts, shadow=shadow, g=g)
        want = R.step(p, mu, nu, counts, g, segs, h, norm=norm)
        got = emulate(p, mu, nu, counts, g, shadow, segs, h, norm=norm, fma=fma, defect=defect)
        if perturb is not None:
            perturb(got, pre)
        R.check(got, want, pre, label=f"{name} step {st}")
        p, mu, nu, counts, shadow = got["p"], got["mu"], got["nu"], got["counts"], got["shadow"]
    return want


@pytest.mark.parametrize("norm", [R.NORM_LOCAL, R.NORM_DOUBLE])
@pytest.mark.parametrize("fma", [NONE, FIRST, SECOND])
@pytest.mark.parametrize("name", R.LAYOUTS)
def test_emulated_kernel_passes_reference(name, fma, norm):
    want = _run(name, norm, fma)
    assert want.clipped.any() and not want.clipped.all(), "each step wants one segment clipped and one not"


@pytest.mark.parametrize("defect", DEFECTS)
def test_emulated_defect_fails_reference(defect):
    with pytest.raises(AssertionError):
        _run("eight", R.NORM_LOCAL, FIRST, defect=defect)


def _scale_step(key, rel):
    def f(got, pre):
        if key == "p":   # the parameter step, not the parameter
            got["p"] = (pre["p"].astype(np.float64) + (got["p"].astype(np.float64) - pre["p"]) * (1 + rel)).astype(f32)
            got["shadow"] = R.bf16_rne(got["p"])   # a consistent shadow: only the step is wrong
        else:
            got[key] = (np.asarray(got[key], np.float64) * (1 + rel)).astype(f32)
    return f


@pytest.mark.parametrize("key", ["p", "mu", "nu", "gnorm"])
def test_relative_error_of_1e3_fails_reference(key):
    """mu, nu, the reported norm or the parameter step off by 1e-3 relative: outside the bounds, at the first step (count 1,
    where the powf term of the bias correction bound is largest)."""
    _run("bench", R.NORM_LOCAL, NONE, steps=1, first_count=0)                     # passes as is
    with pytest.raises(AssertionError):
        _run("bench", R.NORM_LOCAL, NONE, steps=1, first_count=0, perturb=_scale_step(key, 1e-3))


@pytest.mark.parametrize("name", R.LAYOUTS)
def test_bounds_stay_near_fp32_rounding(name):
    """Norm-wise size of the derived bounds relative to the values: mu, nu, p and the norm a few fp32 ulps (< 1e-5); the bound on
    the parameter STEP lr * u is printed: at count 1 the documented powf error of b2^c = 0.999 (4 ulp) over 1 - 0.999 dominates."""
    segs, total = _setup(name)
    rng = np.random.default_rng(1)
    for first in (0, 10):
        p, mu, nu, counts = R.make_state(segs, total, rng, counts=[first] * (2 * len(segs)))
        h = R.Hyper(decay=True, steps_per_update=3, num_updates=4)
        g = R.make_grad(segs, total, rng, 1.0, 0)
        w = R.step(p, mu, nu, counts, g, segs, h)
        ins = w.inside
        rel = {k: float(np.linalg.norm(getattr(w, k + "_bound")[ins]) / np.linalg.norm(getattr(w, k)[ins])) for k in ("p", "mu", "nu")}
        rel["gnorm"] = float(np.max(w.gnorm_bound / np.maximum(w.gnorm, 1e-30)))
        dp = np.abs(w.p - p.astype(np.float64))[ins]
        step_rel = float(np.linalg.norm(w.p_bound[ins]) / np.linalg.norm(dp))
        print(f"{name} count {first}: norm-wise bound / value " + ", ".join(f"{k} {v:.2e}" for k, v in rel.items())
              + f"; bound / parameter step {step_rel:.2e}")
        for k, v in rel.items():
            assert v < 1e-5, f"{name} count {first}: {k} bound {v:.2e} relative"
        # the step bound includes the final rounding of p (1/2 ulp of |p| ~ 0.3), which the step itself cannot beat
        assert step_rel < 1e-2, step_rel
