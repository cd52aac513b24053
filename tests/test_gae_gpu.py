"""K2 parity: the CUDA GAE kernel vs (i) the reference's golden vectors, (ii) the fp64 oracle on
random inputs incl. ragged shapes, (iii) size-independent properties at the benchmark's full size.
Tolerance (fp32 kernel vs fp64 oracle, T<=300): rtol 1e-5, atol 1e-5 (BASELINE.md section 4)."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests.golden_runner import load_cases, run_case

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-5, 1e-5


def _dev():
    return torch.device("cuda:0")


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device=_dev())


@pytest.mark.parametrize("case", load_cases(), ids=lambda c: c["name"])
def test_golden_vectors_through_public_api(case):
    from stoix_b200.utils.multistep import batch_truncated_generalized_advantage_estimation as gae

    def fn(r_t, discount_t, lambda_, **kw):
        lam = _t(lambda_) if isinstance(lambda_, np.ndarray) else lambda_
        tm = kw.pop("time_major", False)
        a, t = gae(_t(r_t), _t(discount_t), lam, time_major=tm, **{k: _t(v) for k, v in kw.items()})
        return a.cpu().numpy(), t.cpu().numpy()

    run_case(case, fn)


def _random_ppo_inputs(T, E, seed, p_done=0.02, p_trunc=0.01):
    rng = np.random.default_rng(seed)
    reward = rng.standard_normal((T, E)).astype(np.float32)
    value = rng.standard_normal((T, E)).astype(np.float32)
    boot = rng.standard_normal((T, E)).astype(np.float32)
    done = rng.random((T, E)) < p_done
    trunc = (~done) & (rng.random((T, E)) < p_trunc)
    return reward, value, boot, done, trunc


@pytest.mark.parametrize("T,E", [(128, 4096), (16, 4), (1, 8), (5, 3), (129, 36), (300, 20), (128, 6), (7, 1), (260, 1024)])
@pytest.mark.parametrize("standardize", [0, 1, 2])
def test_ppo_form_vs_oracle(T, E, standardize):
    from stoix_b200 import ops

    reward, value, boot, done, trunc = _random_ppo_inputs(T, E, seed=T * 1000 + E)
    gamma, lam, rs = 0.99, 0.95, 0.5
    r_t, d_t, tr = O.ppo_gae_inputs(reward, done, trunc, gamma, rs)
    adv_o, tgt_o = O.gae(r_t, d_t, lam, v_tm1=value.astype(np.float64), v_t=boot.astype(np.float64), truncation_t=tr, time_major=True)
    adv, tgt, stats = ops.gae_ppo(_t(reward), _t(value), _t(boot), _t(done, torch.bool), _t(trunc, torch.bool), gamma, lam, rs, standardize)
    np.testing.assert_allclose(tgt.cpu().numpy(), tgt_o, rtol=RTOL, atol=ATOL)
    if standardize:
        mean = adv_o.mean()
        rstd = 1.0 / np.sqrt((adv_o * adv_o).mean() - mean * mean + 1e-5)
        np.testing.assert_allclose(stats.cpu().numpy(), [mean, rstd], rtol=1e-5, atol=1e-6)
    if standardize == 2:
        np.testing.assert_allclose(adv.cpu().numpy(), O.standardize(adv_o), rtol=1e-4, atol=2e-5)
    else:
        np.testing.assert_allclose(adv.cpu().numpy(), adv_o, rtol=RTOL, atol=ATOL)


def test_unaligned_views_take_scalar_path():
    """Row pitch not a multiple of 4 / misaligned base pointers must still be exact (VEC=1 kernel)."""
    from stoix_b200 import ops

    T, E = 33, 10
    reward, value, boot, done, trunc = _random_ppo_inputs(T, E, seed=7)
    r_t, d_t, tr = O.ppo_gae_inputs(reward, done, trunc, 0.9, 1.0)
    adv_o, tgt_o = O.gae(r_t, d_t, 0.8, v_tm1=value.astype(np.float64), v_t=boot.astype(np.float64), truncation_t=tr, time_major=True)

    def off(x, dtype=torch.float32):  # allocate with a 1-element offset so data_ptr is not 16B aligned
        buf = torch.empty(T * E + 1, dtype=dtype, device=_dev())
        v = buf[1:].view(T, E)
        v.copy_(torch.as_tensor(x, dtype=dtype))
        return v

    adv, tgt, _ = ops.gae_ppo(off(reward), off(value), off(boot), off(done, torch.bool), off(trunc, torch.bool), 0.9, 0.8, 1.0, 0)
    np.testing.assert_allclose(adv.cpu().numpy(), adv_o, rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(tgt.cpu().numpy(), tgt_o, rtol=RTOL, atol=ATOL)


def test_generic_form_array_lambda_and_truncation():
    from stoix_b200 import ops

    rng = np.random.default_rng(11)
    T, E = 40, 12
    r = rng.standard_normal((T, E)).astype(np.float32)
    disc = (rng.random((T, E)) * 0.99).astype(np.float32)
    lam = rng.random((T, E)).astype(np.float32)
    vt1 = rng.standard_normal((T, E)).astype(np.float32)
    vt = rng.standard_normal((T, E)).astype(np.float32)
    tr = (rng.random((T, E)) < 0.1).astype(np.float32)
    adv_o, tgt_o = O.gae(r, disc, lam, v_tm1=vt1, v_t=vt, truncation_t=tr, time_major=True)
    adv, tgt, _ = ops.gae_generic(_t(r), _t(disc), _t(lam), _t(vt1), _t(vt), _t(tr))
    np.testing.assert_allclose(adv.cpu().numpy(), adv_o, rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(tgt.cpu().numpy(), tgt_o, rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("quads", [2, 4, 8, 416, 500, 501])
def test_every_block_shape_agrees(quads):
    import ctypes

    from stoix_b200 import _lib, ops

    lib = _lib.load()
    lib.stx_gae_set_tuning.argtypes = [ctypes.c_int]
    reward, value, boot, done, trunc = _random_ppo_inputs(128, 1024, seed=3)
    args = (_t(reward), _t(value), _t(boot), _t(done, torch.bool), _t(trunc, torch.bool), 0.99, 0.95, 1.0, 1)
    lib.stx_gae_set_tuning(0)
    a0, t0, s0 = ops.gae_ppo(*args)
    assert lib.stx_gae_set_tuning(quads) == 0
    try:
        a1, t1, s1 = ops.gae_ppo(*args)
    finally:
        lib.stx_gae_set_tuning(0)
    if quads != 501:  # same 4-step chunking (500 = the TMA-pipelined kernel, 32 x 128 tiles) -> bit-identical
        assert torch.equal(a0, a1) and torch.equal(t0, t1)
    else:             # 2-step chunking (501 = TMA kernel with 64 x 64 tiles) re-associates the composition: equal to fp32 rounding
        np.testing.assert_allclose(a0.cpu().numpy(), a1.cpu().numpy(), rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(t0.cpu().numpy(), t1.cpu().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(s0.cpu().numpy(), s1.cpu().numpy(), rtol=1e-5)


@pytest.mark.parametrize("T,E", [(128, 1024), (100, 48), (300, 1040), (1, 16), (129, 4112)])
@pytest.mark.parametrize("standardize", [0, 1])
@pytest.mark.parametrize("code", [500, 501])
def test_tma_form_vs_oracle(T, E, standardize, code):
    """The TMA-pipelined persistent kernel (the default from E = 262144 up), forced at small shapes: ragged last segment
    (T % 128), ragged last env tile (E % 32), several segments per tile (carry across segments), one block walking many tiles."""
    import ctypes

    from stoix_b200 import _lib, ops

    lib = _lib.load()
    lib.stx_gae_set_tuning.argtypes = [ctypes.c_int]
    reward, value, boot, done, trunc = _random_ppo_inputs(T, E, seed=11, p_done=0.05, p_trunc=0.05)
    assert lib.stx_gae_set_tuning(code) == 0   # 500: 32 envs x 128 steps per tile, 501: 64 x 64
    try:
        adv, tgt, stats = ops.gae_ppo(_t(reward), _t(value), _t(boot), _t(done, torch.bool), _t(trunc, torch.bool), 0.99, 0.95, 1.0, standardize)
    finally:
        lib.stx_gae_set_tuning(0)
    r_t, d_t, tr = O.ppo_gae_inputs(reward, done, trunc, 0.99, 1.0)
    adv_o, tgt_o = O.gae(r_t, d_t, 0.95, v_tm1=value.astype(np.float64), v_t=boot.astype(np.float64), truncation_t=tr, time_major=True)
    np.testing.assert_allclose(adv.cpu().numpy(), adv_o, rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(tgt.cpu().numpy(), tgt_o, rtol=RTOL, atol=ATOL)
    if standardize:
        np.testing.assert_allclose(stats.cpu().numpy()[0], adv_o.mean(), rtol=1e-4, atol=1e-5)


def test_full_size_properties():
    """At (T=128, E=65536) the fp64 oracle loop is still cheap for a slice; the rest is checked by
    properties: (a) targets - advantages == v_tm1, (b) columns are independent (a slice equals the
    kernel run on that slice alone), (c) termination blocks credit: adv[t] == delta[t] where done[t],
    (d) linearity in (reward, values) for fixed flags, (e) determinism."""
    from stoix_b200 import ops

    T, E = 128, 65536
    reward, value, boot, done, trunc = _random_ppo_inputs(T, E, seed=5, p_done=0.005, p_trunc=0.002)
    g = lambda: ops.gae_ppo(_t(reward), _t(value), _t(boot), _t(done, torch.bool), _t(trunc, torch.bool), 0.99, 0.95, 1.0, 1)
    adv, tgt, stats = g()
    adv2, tgt2, stats2 = g()
    assert torch.equal(adv, adv2) and torch.equal(tgt, tgt2) and torch.equal(stats, stats2)  # (e)
    a = adv.cpu().numpy()
    np.testing.assert_allclose(tgt.cpu().numpy() - a, value, rtol=0, atol=2e-5)  # (a)
    sl = slice(1000, 1064)
    r_t, d_t, tr = O.ppo_gae_inputs(reward[:, sl], done[:, sl], trunc[:, sl], 0.99, 1.0)
    adv_o, _ = O.gae(r_t, d_t, 0.95, v_tm1=value[:, sl].astype(np.float64), v_t=boot[:, sl].astype(np.float64), truncation_t=tr, time_major=True)
    np.testing.assert_allclose(a[:, sl], adv_o, rtol=RTOL, atol=ATOL)  # (b) vs oracle on a slice
    delta = reward + (1.0 - done) * 0.99 * boot - value
    np.testing.assert_allclose(a[done], delta[done], rtol=1e-6, atol=1e-6)  # (c)
    np.testing.assert_allclose(a[trunc], delta[trunc], rtol=1e-6, atol=1e-6)
    adv_s, _, _ = ops.gae_ppo(_t(2 * reward), _t(2 * value), _t(2 * boot), _t(done, torch.bool), _t(trunc, torch.bool), 0.99, 0.95, 1.0, 0)
    np.testing.assert_allclose(adv_s.cpu().numpy(), 2 * a, rtol=1e-6, atol=1e-6)  # (d) exact scaling by 2
    m = a.astype(np.float64).mean()
    np.testing.assert_allclose(stats.cpu().numpy()[0], m, rtol=1e-4, atol=1e-6)


def test_cpu_tensor_is_rejected():
    from stoix_b200 import ops
    from stoix_b200._lib import StxError

    x = torch.zeros(4, 4)
    with pytest.raises(StxError):
        ops.gae_ppo(x, x, x, x.bool(), x.bool(), 0.99, 0.95)
