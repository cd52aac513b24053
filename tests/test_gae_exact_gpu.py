"""K2 (stx_gae.cu) across every launch form and input form, against fp64 references.

A. Exact data (tests/gae_exact_data.py): every tuning code x every face x SHAPES must give the oracle's advantages and
   targets bit for bit; the 5xx codes on the generic and lambda forms (and on a PPO shape with E % 16 != 0) fall back to
   the default selection, which must be exact too.
B. Statistics: standardize 1 and 2 on the PPO and generic forms, every code: `stats` and the standardised advantages equal
   the fp64 reproduction of the kernel's finish bit for bit, call after call on one cached scratch with E changing between.
C. Real-valued data (gamma 0.99, lambda 0.95, random flags, a random lambda array) at the multi-segment and ragged shapes:
   rtol / atol 1e-5 (BASELINE.md section 4); NaN and -inf entries in q_t follow jnp.max; two identical calls are equal.
D. The default selection at the sizes where it picks its other paths, unaligned views, and the tuning-code -> kernel mapping
   seen by the profiler, codes outside the accepted set refused.
"""
import ctypes
import re

import numpy as np
import pytest
import torch

from stoix_b200 import _lib, ops
from tests import gae_exact_data as X
from tests import pqn_oracle as P
from oracle import ppo_oracle as O

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-5, 1e-5


@pytest.fixture
def tuning():
    """stx_gae_set_tuning is process-global: set it per call, restore the default selection whatever happens."""
    lib = _lib.load()
    lib.stx_gae_set_tuning.argtypes = [ctypes.c_int]
    try:
        yield lambda code: lib.stx_gae_set_tuning(int(code))
    finally:
        lib.stx_gae_set_tuning(0)


_DEV = {}


def _dev(case):
    """Device copies of a case's inputs and oracle results (cached: every code reuses them)."""
    key = (case.face, case.T, case.E)
    if key not in _DEV:
        t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")
        _DEV[key] = ({k: t(v) for k, v in case.inputs.items()}, t(case.adv), t(case.targets))
    return _DEV[key]


def _call(face, x, standardize=0, scalars=None, out=None):
    """One call of the face's op on the device inputs x; returns (advantages or None, targets, stats or None)."""
    s = scalars or {}
    if face == "gae_ppo":
        return ops.gae_ppo(x["reward"], x["value"], x["bootstrap_value"], x["done"], x["truncated"], s.get("gamma", 1.0),
                           s.get("gae_lambda", 1.0), s.get("reward_scale", 1.0), standardize)
    if face.startswith("gae_generic"):
        lam = x["lambda_"] if x.get("lambda_") is not None else s.get("lambda_", 1.0)
        return ops.gae_generic(x["r_t"], x["discount_t"], lam, x["v_tm1"], x["v_t"], x.get("truncation_t"), standardize)
    if face == "q_lambda":
        return None, ops.q_lambda(x["q_t"], x["reward"], x["done"], x["truncated"], s.get("gamma", 1.0), s.get("q_lambda_", 1.0), out=out), None
    lam = x["lambda_"] if x.get("lambda_") is not None else s.get("lambda_", 1.0)
    return None, ops.lambda_returns(x["r_t"], x["discount_t"], x["v_t"], lam), None


def _run(case, standardize=0, x=None, out=None):
    return _call(case.face, x if x is not None else _dev(case)[0], standardize, case.scalars, out)


def _assert_equal(got, want, what):
    if isinstance(got, torch.Tensor) and isinstance(want, torch.Tensor) and torch.equal(got, want):
        return
    g = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = want.cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want)
    assert g.shape == w.shape, f"{what}: shape {g.shape} vs {w.shape}"
    bad = np.argwhere(g != w)
    assert bad.size == 0, (f"{what}: {len(bad)} of {w.size} entries differ from the oracle; first at (t, e) = {bad[0].tolist()}: "
                           f"kernel {g[tuple(bad[0])]!r} oracle {w[tuple(bad[0])]!r}")


def _form(case, code):
    return X.launch_form(case.face, code, case.E).name


# ---------------------------------------------------------------------------------------------------------------------
# A. every form x every face, exact
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("code", X.CODES)
@pytest.mark.parametrize("face", list(X.FACES))
def test_every_form_bit_exact(face, code, tuning):
    for T, E in X.SHAPES:
        case = X.make_case(face, T, E)
        _, adv_o, tgt_o = _dev(case)
        tuning(code)
        adv, tgt, _ = _run(case)
        tuning(0)
        what = f"{face} code {code} ({_form(case, code)}) T={T} E={E}"
        _assert_equal(tgt, tgt_o, what + " targets")
        if adv_o is not None:
            _assert_equal(adv, adv_o, what + " advantages")
    print(f"{face} code {code}: {len(X.SHAPES)} shapes bit-exact")


# ---------------------------------------------------------------------------------------------------------------------
# B. statistics, exact
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("code", X.CODES)
@pytest.mark.parametrize("face", X.STANDARDIZING_FACES)
def test_statistics_bit_exact(face, code, tuning):
    """The largest E first (it sizes the scratch), then the other shapes, then the first again: every call reuses the same
    scratch, so a last-block ticket that does not reset its counter, or a partial from an earlier grid, shows."""
    shapes = sorted(X.SHAPES, key=lambda s: -s[1])
    shapes = shapes + shapes[:1]
    ptr = None
    for T, E in shapes:
        case = X.make_case(face, T, E)
        _, adv_o, tgt_o = _dev(case)
        st_o = X.stats(case.adv)
        z_o = X.standardized(case.adv, st_o)
        what = f"{face} code {code} ({_form(case, code)}) T={T} E={E}"
        for standardize in (1, 2):
            tuning(code)
            adv, tgt, st = _run(case, standardize)
            tuning(0)
            scratch = ops._scratch[("gae", str(adv.device))].data_ptr()
            assert ptr is None or scratch == ptr, "the scratch was reallocated: the calls did not share it"
            ptr = scratch
            _assert_equal(st, st_o, f"{what} standardize={standardize} stats [mean, rstd]")
            _assert_equal(tgt, tgt_o, f"{what} standardize={standardize} targets")
            _assert_equal(adv, adv_o if standardize == 1 else z_o, f"{what} standardize={standardize} advantages")


# ---------------------------------------------------------------------------------------------------------------------
# C. real-valued data against fp64
# ---------------------------------------------------------------------------------------------------------------------

REAL_FACES = ("gae_ppo", "gae_generic_lam_t_trunc", "q_lambda", "lambda_returns_lam_t")
REAL_SHAPES = ((129, 48), (256, 260), (300, 96), (300, 1020), (513, 37))


def _real_case(face, T, E):
    """Inputs and the fp64 oracle on random values; the lambda forms get NaN and -inf entries in q_t at envs 3..5."""
    rng = np.random.default_rng(T * 7919 + E)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    gamma, lam = 0.99, 0.95
    done = rng.random((T, E)) < 0.03
    trunc = (rng.random((T, E)) < 0.02) & ~done
    if face == "gae_ppo":
        reward, value, boot = (f32(rng.standard_normal((T, E))) for _ in range(3))
        r_t, d_t, tr = O.ppo_gae_inputs(reward, done, trunc, gamma, 0.5)
        adv, tgt = O.gae(r_t, d_t, lam, v_tm1=value.astype(np.float64), v_t=boot.astype(np.float64), truncation_t=tr, time_major=True)
        x = dict(reward=reward, value=value, bootstrap_value=boot, done=done, truncated=trunc)
        return x, dict(gamma=gamma, gae_lambda=lam, reward_scale=0.5), adv, tgt
    if face == "gae_generic_lam_t_trunc":
        r, v_tm1, v_t = (f32(rng.standard_normal((T, E))) for _ in range(3))
        disc = f32(gamma * (1.0 - done))
        lam_t = f32(rng.random((T, E)))
        tr = f32(trunc)
        adv, tgt = O.gae(r, disc, lam_t, v_tm1=v_tm1, v_t=v_t, truncation_t=tr, time_major=True)
        return dict(r_t=r, discount_t=disc, lambda_=lam_t, v_tm1=v_tm1, v_t=v_t, truncation_t=tr), {}, adv, tgt
    A = 5
    q = rng.standard_normal((T, E, A))
    if E >= 6:
        nan = rng.random((T, A)) < 0.02
        q[:, 3][nan] = np.nan                                 # env 3: a NaN in any column poisons the row's max
        q[:, 4][rng.random((T, A)) < 0.1] = -np.inf           # env 4: single -inf entries leave the max finite
        q[rng.random(T) < 0.05, 5, :] = -np.inf               # env 5: whole rows of -inf
        q[T - 1, 5, :] = -np.inf                              # ... including the last step
    q = f32(q)
    r = f32(rng.standard_normal((T, E)))
    if face == "q_lambda":
        want = P.batch_q_lambda(r, gamma * (1.0 - (done | trunc)), q, lam)
        return dict(q_t=q, reward=r, done=done, truncated=trunc), dict(gamma=gamma, q_lambda_=lam), None, want
    disc = f32(gamma * (1.0 - (done | trunc)))
    lam_t = f32(rng.uniform(0.05, 0.95, (T, E)))
    want = P.batch_q_lambda(r, disc, q, lam_t)
    return dict(r_t=r, discount_t=disc, v_t=q, lambda_=lam_t), {}, None, want


def _assert_close(got, want, what):
    g = got.double().cpu().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(want)), f"{what}: NaN positions differ from the oracle"
    assert np.array_equal(np.isneginf(g), np.isneginf(want)) and np.array_equal(np.isposinf(g), np.isposinf(want)), f"{what}: inf positions differ"
    np.testing.assert_allclose(g, want, rtol=RTOL, atol=ATOL, err_msg=what)


@pytest.mark.parametrize("code", X.CODES)
@pytest.mark.parametrize("face", REAL_FACES)
def test_real_values_against_fp64(face, code, tuning):
    for T, E in REAL_SHAPES:
        x, scalars, adv_o, tgt_o = _real_case(face, T, E)
        xd = {k: torch.as_tensor(v, device="cuda:0") for k, v in x.items()}
        what = f"{face} code {code} ({X.launch_form(face, code, E).name}) T={T} E={E}"
        tuning(code)
        first = _call(face, xd, 1 if adv_o is not None else 0, scalars)
        second = _call(face, xd, 1 if adv_o is not None else 0, scalars)
        tuning(0)
        for a, b in zip(first, second):   # determinism: the same call gives the same bits (NaNs included), statistics too
            assert (a is None and b is None) or torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{what}: two identical calls differ"
        adv, tgt, _ = first
        _assert_close(tgt, tgt_o, what + " targets")
        if adv_o is not None:
            _assert_close(adv, adv_o, what + " advantages")
        if face in ("q_lambda", "lambda_returns_lam_t") and E >= 6:
            g = tgt.cpu().numpy()
            assert np.isnan(g[:, 3]).any() and np.isfinite(g[:, 6:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# D. default selection at large E, unaligned views, the code -> kernel mapping
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("face,T,E", [(f, T, E) for f, s in X.DEFAULT_PATH_SHAPES.items() for T, E in s], ids=str)
def test_default_selection_at_large_E(face, T, E):
    """The default selection (code 0) where it picks the 4xx form, declines TMA (E % 16), or runs TMA with a segment carry;
    the standardising faces also run standardize=2 after the kernel (after TMA at E = 32768 and 65536)."""
    case = X.make_case(face, T, E)
    _, adv_o, tgt_o = _dev(case)
    what = f"{face} default ({X.launch_form(face, 0, E).name}) T={T} E={E}"
    std = 2 if face in X.STANDARDIZING_FACES else 0
    adv, tgt, st = _run(case, std)
    _assert_equal(tgt, tgt_o, what + " targets")
    if std:
        st_o = X.stats(case.adv)
        _assert_equal(st, st_o, what + " stats")
        _assert_equal(adv, X.standardized(case.adv, st_o), what + " standardised advantages")


def _offset_view(t):
    """The same values at a 1-element offset: data_ptr is not 16-byte aligned."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("face", [f for f in X.FACES if f != "gae_ppo"])
@pytest.mark.parametrize("T,E", [(129, 48), (300, 1020), (513, 37)])
def test_unaligned_views(face, T, E):
    """Inputs at a 1-element offset.  The generic and lambda forms load their inputs one element at a time, so they keep the
    vec4 kernels (only the outputs' alignment selects VEC = 1); an unaligned q_lambda `out` selects the VEC = 1 kernel."""
    case = X.make_case(face, T, E)
    x, adv_o, tgt_o = _dev(case)
    xv = {k: None if v is None else _offset_view(v) for k, v in x.items()}
    out = _offset_view(torch.zeros(T, E, device="cuda:0")) if face == "q_lambda" else None
    adv, tgt, _ = _run(case, x=xv, out=out)
    _assert_equal(tgt, tgt_o, f"{face} unaligned T={T} E={E} targets")
    if adv_o is not None:
        _assert_equal(adv, adv_o, f"{face} unaligned T={T} E={E} advantages")


_SCAN_RE = (re.compile(r"gae_scan_kernel<[^<>]*?(PpoIn|GenericIn|LambdaIn), (\d+), (\d+), (\d+), (\d+)>"),
            re.compile(r"gae_scan_kernelINS0_\d+(PpoIn|GenericIn|LambdaIn)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E"))
_TMA_RE = (re.compile(r"gae_tma_kernel<(\d+), (\d+)>"), re.compile(r"gae_tma_kernelILi(\d+)ELi(\d+)E"))


def _kernel_form(name):
    for rx in _SCAN_RE:
        m = rx.search(name)
        if m:
            return m.group(1), X.Form("scan", *(int(g) for g in m.groups()[1:])).name
    for rx in _TMA_RE:
        m = rx.search(name)
        if m:
            return "PpoIn", X.Form("tma", int(m.group(1)), int(m.group(2))).name
    return None


STX_E_ARG = -1              # include/stx.h
REJECTED = (16, 308, 502)   # codes of launch forms K2 does not have: 16 quads, 2 steps per thread, 128 x 32 TMA tiles


@pytest.mark.parametrize("face", ["gae_ppo", "gae_generic", "q_lambda", "lambda_returns"])
def test_codes_launch_the_mirrored_kernels(face, tuning):
    """The kernel each tuning code launches, as the profiler names it, is the one launch_form (the mapping the tests above
    rely on) says: every code at E = 48 (TMA-eligible for the PPO form), code 0 at E = 37 (VEC = 1).  A code outside
    X.CODES is refused with STX_E_ARG and leaves the default selection in place for the next call."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    runs = [(code, 4, 48) for code in X.CODES + REJECTED] + [(0, 4, 37)]
    cases = [(code, X.make_case(face, T, E)) for code, T, E in runs]
    for _, case in cases:
        _dev(case)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for code, case in cases:
            assert tuning(code) == (0 if code in X.CODES else STX_E_ARG), f"stx_gae_set_tuning({code})"
            _run(case)
            tuning(0)
            torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and ("gae_scan_kernel" in e.name or "gae_tma_kernel" in e.name)),
                     key=lambda e: e.time_range.start)
    got = [_kernel_form(e.name) for e in kernels]
    assert None not in got, f"unrecognised kernel names: {[e.name for e in kernels]}"
    want = [(X.FACES[face], X.launch_form(face, code if code in X.CODES else 0, case.E).name) for code, case in cases]
    assert got == want, "\n".join(f"code {c} E={cs.E}: launched {g}, mirror {w}" for (c, cs), g, w in zip(cases, got, want) if g != w)
