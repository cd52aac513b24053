"""bf16 tensor-core kernels (K1 forward, K3a / K3b / reduce) on exactly representable data (tests/exact_data.py).

Every operand and intermediate is exact in bf16 and every accumulation stays below 2^20 grid units, so the kernels'
results do not depend on summation order: they must equal the fp64 oracle BIT FOR BIT (torch.equal / array_equal), at
any shape, under every split-K partition and launch switch.  One misplaced, dropped or re-read row fails these tests;
the norm-wise 5e-3 bounds of tests/test_tc_gpu.py cannot see it at the benchmark shape (tests/test_exact_data.py).

That wgmma's fp32 accumulation is exact for such data is an assumption about the hardware, not the code; the K1 cases
at M = 1 and 63 (one tile, one warpgroup) and the K3 case at mb = 128 (one tile per network, default split) test it
before any multi-tile indexing is involved.  Measured on an H100 80GB HBM3 (400 W power limit): every case below, the
largest accumulating 5.6e5 grid units (dW2 at mb = 65536), equals the oracle bit for bit; the hot-row actor gradients
stay within 0.1 of their tolerance.  No kernel bug was found.  The whole file runs in about 2 minutes there.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import exact_data as X

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), device="cuda:0").to(dtype)


def _assert_equal(got: np.ndarray, ref: np.ndarray, what: str):
    ref = np.asarray(ref, np.float32)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (f"{what}: {len(bad)} of {ref.size} entries differ from the oracle; first at {bad[0].tolist()}: "
                           f"kernel {got[tuple(bad[0])]} oracle {ref[tuple(bad[0])]}")


# ---------------------------------------------------------------------------------------------------------------------
# K1: fused MLP forward
# ---------------------------------------------------------------------------------------------------------------------


def _k1_inputs(M, D, A):
    from stoix_b200 import ops

    net, x = X.forward_problem(M, D, A)
    spec = ops.MlpSpec((D, 256, 256, A))
    params = _t(net.flat())
    return net, x, spec, params, ops.cast_bf16(params), _t(x, torch.bfloat16)


def _check_forward(net, x, out, h1, h2, what):
    ref_out, ref_h1, ref_h2 = X.forward(net, x)
    _assert_equal(out.cpu().numpy(), ref_out, f"{what} out")
    _assert_equal(h1.cpu().numpy(), ref_h1, f"{what} h1")
    _assert_equal(h2.cpu().numpy(), ref_h2, f"{what} h2")


@pytest.mark.parametrize("M,D,A", X.FORWARD_CASES)
def test_k1_forward_is_exact(M, D, A):
    """out, h1, h2 of the debug entry point and out of the public one equal the oracle exactly."""
    from stoix_b200 import ops

    net, x, spec, params, shadow, xb = _k1_inputs(M, D, A)
    out, h1, h2 = ops.tc_debug_forward(spec, params, shadow, xb)
    out2 = ops.mlp_forward(spec, params, xb, precision=ops.STX_PREC_BF16, params_bf16=shadow)
    torch.cuda.synchronize()
    _check_forward(net, x, out, h1, h2, f"M={M} D={D} A={A}")
    assert torch.equal(out, out2)


def test_k1_forward_cta_budget_is_bit_identical():
    """Grids capped at 1 and 7 CTAs: each warpgroup walks thousands of tiles (8193 tiles over 2 or 14 warpgroups) through
    its 2-stage TMA ring; the results equal the uncapped run (and the oracle)."""
    from stoix_b200 import ops

    M, D, A = 524288 + 37, 24, 9
    net, x, spec, params, shadow, xb = _k1_inputs(M, D, A)
    ref = ops.tc_debug_forward(spec, params, shadow, xb)
    for budget in (1, 7):
        try:
            ops.set_forward_cta_budget(budget)
            got = ops.tc_debug_forward(spec, params, shadow, xb)
            out2 = ops.mlp_forward(spec, params, xb, precision=ops.STX_PREC_BF16, params_bf16=shadow)
            torch.cuda.synchronize()
        finally:
            ops.set_forward_cta_budget(0)
        for name, a, b in zip(("out", "h1", "h2"), got, ref):
            assert torch.equal(a, b), f"budget {budget}: {name} differs from the uncapped run"
        assert torch.equal(out2, ref[0])
    _check_forward(net, x, *ref, f"M={M} D={D} A={A}")


def test_k1_forward_strided_rows():
    """Input rows with a pitch of 72 elements for D = 64 (ldx > D, through the C ABI): the 8 padding columns, filled with
    values that would change every output, must not be read."""
    from stoix_b200 import _lib, ops

    M, D, A = 64 * 264 + 1, 64, 16
    net, x, spec, params, shadow, xb = _k1_inputs(M, D, A)
    buf = torch.full((M, 72), 3.0, dtype=torch.bfloat16, device="cuda:0")
    buf[:, :D] = xb
    out, h1, h2 = (torch.empty(M, n, device="cuda:0") for n in (A, 256, 256))
    m = spec.c_struct(params, shadow)
    p = lambda t: C.c_void_p(t.data_ptr())
    _lib.check(_lib.load().stx_tc_debug_forward(C.byref(m), p(buf), 72, M, p(out), p(h1), p(h2),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)), "stx_tc_debug_forward")
    torch.cuda.synchronize()
    _check_forward(net, x, out, h1, h2, "ldx=72")


# ---------------------------------------------------------------------------------------------------------------------
# K3: PPO minibatch gradients
# ---------------------------------------------------------------------------------------------------------------------


def _k3_setup(pb: X.PpoProblem):
    from stoix_b200 import ops

    D, A = pb.obs.shape[1], pb.actor.W[2].shape[1]
    na, coff, nc, total = X.arena_layout(D, A)
    sa, sc = ops.MlpSpec((D, 256, 256, A)), ops.MlpSpec((D, 256, 256, 1))
    assert ops.arena_offsets(sa, sc) == (0, coff, total)
    flat = np.zeros(total, np.float32)
    flat[:na], flat[coff:coff + nc] = pb.actor.flat(), pb.critic.flat()
    arena = _t(flat)
    batch = ops.PpoBatch(_t(pb.obs, torch.bfloat16), _t(pb.action, torch.int32), _t(pb.logp_old), _t(pb.v_old), _t(pb.adv),
                         _t(pb.tgt), adv_stats=None, perm=_t(pb.perm, torch.int32) if pb.perm is not None else None)
    return sa, sc, arena, ops.cast_bf16(arena), batch, total


def _k3_run(pb: X.PpoProblem, windows, ws_mb=None):
    """Gradient arena and metrics of ops.ppo_minibatch_grads (bf16, no standardisation) for each (mb_off, mb) of `windows`,
    one fresh arena per call, all on ONE workspace sized for ws_mb (default: the largest minibatch)."""
    from stoix_b200 import ops

    sa, sc, arena, shadow, batch, total = _k3_setup(pb)
    ws = ops.ppo_workspace(sa, sc, ws_mb or max(mb for _, mb in windows), ops.STX_PREC_BF16, "cuda:0")
    res = []
    for mb_off, mb in windows:
        grads, metrics = torch.zeros(total, device="cuda:0"), torch.zeros(8, device="cuda:0")
        ops.ppo_minibatch_grads(sa, sc, arena, batch, mb_off, mb, pb.clip_eps, pb.ent_coef, pb.vf_coef, False, grads, metrics, ws,
                                precision=ops.STX_PREC_BF16, param_arena_bf16=shadow)
        res.append((grads, metrics))
    torch.cuda.synchronize()
    return [(g.cpu().numpy(), m.cpu().numpy()) for g, m in res]


def _check_critic_exact(pb, mb_off, mb, g, mt, what):
    """Critic tensors, value_loss, value mean and target mean equal the oracle; with advantages 0 and ent_coef 0 the actor
    gradient, the actor loss and the advantage mean are exactly 0 (idle CTAs leave no garbage)."""
    D, A = pb.obs.shape[1], pb.actor.W[2].shape[1]
    na, coff, nc, total = X.arena_layout(D, A)
    ref, rm = X.ppo_oracle(pb, mb_off, mb)
    _assert_equal(g[coff:coff + nc], ref[coff:coff + nc], f"{what}: critic gradient")
    assert not g[:na].any(), f"{what}: actor gradient must be exactly zero, {np.count_nonzero(g[:na])} entries are not"
    assert not g[na:coff].any() and not g[coff + nc:].any(), f"{what}: arena padding written"
    _assert_equal(mt[[2, 4, 5]], rm[[2, 4, 5]], f"{what}: value_loss / value mean / target mean")
    assert mt[0] == 0 and mt[3] == 0, f"{what}: actor loss {mt[0]} and advantage mean {mt[3]} must be 0"


@pytest.mark.parametrize("B,mb_off,mb,D,A,use_perm", X.CRITIC_CASES)
def test_k3_critic_is_exact(B, mb_off, mb, D, A, use_perm):
    pb = X.critic_problem(B, mb_off, mb, D, A, use_perm)
    (g, mt), = _k3_run(pb, [(mb_off, mb)])
    _check_critic_exact(pb, mb_off, mb, g, mt, f"B={B} mb={mb} D={D}")


def test_k3_stale_partials_do_not_leak():
    """mb = 32768, then mb = 128 on the same workspace: the second gradient equals its oracle (no partial of the first call,
    whose K3b CTAs each wrote many chunks, survives into the second, where most CTAs are idle)."""
    B, D, A, windows = X.STALE_CASE
    pb = X.ppo_problem(B, D, A, windows, seed=B + D)
    for (mb_off, mb), (g, mt) in zip(windows, _k3_run(pb, windows)):
        _check_critic_exact(pb, mb_off, mb, g, mt, f"mb={mb} on a workspace for {windows[0][1]}")


def _actor_tolerance(pb: X.PpoProblem, rows: np.ndarray, dlogits: np.ndarray) -> np.ndarray:
    """Per-entry bound on |kernel - oracle| of the actor gradient (flat, actor part), from the rows that carry a nonzero dz.

    The softmax is not exact: the kernel's dz (fast exp / log, fp32) and the oracle's (fp64) round to bf16 on either side
    of a rounding boundary at most, i.e. differ by <= 1 bf16 ulp <= 2^-7 |dz|.  dh2 = (dz W2^T) masked inherits that and
    rounds once more, dh1 once more: <= 3 ulps relative to the magnitude bounds P2 = (|dz| |W2|^T) masked, P1 =
    (P2 |W1|^T) masked, and every weight / bias gradient sums such terms.  Tolerance: 4 ulps (2^-5) of the magnitude
    bound of each entry; the forward values are exact."""
    p = pb.actor
    x = pb.obs[rows].astype(np.float64)
    _, acts = X.O.mlp_forward(p, x)
    h1, h2 = acts[1], acts[2]
    dz = np.abs(dlogits)
    p2 = (dz @ np.abs(p.W[2]).T) * (h2 > 0)
    p1 = (p2 @ np.abs(p.W[1]).T) * (h1 > 0)
    mag = X.O.MLPParams([np.abs(x).T @ p1, h1.T @ p2, h2.T @ dz], [p1.sum(0), p2.sum(0), dz.sum(0)]).flat()
    return 2.0 ** -5 * mag


def _hot_reference(pb: X.PpoProblem, mb_off: int, mb: int, positions):
    """Oracle actor gradient and tolerance from the hot rows alone (every other row has advantage 0 and ent_coef is 0, so
    its dz is exactly 0)."""
    idx = pb.rows(mb_off, mb)
    rows = idx[np.asarray(positions)]
    g, _ = X.ppo_oracle(pb, mb_off, mb, rows=rows)
    x = pb.obs[rows].astype(np.float64)
    lg = X.O.mlp_forward(pb.actor, x)[0]
    _, dlg, _ = X.O.actor_loss_and_dlogits(lg, pb.action[rows], pb.logp_old[rows].astype(np.float64), pb.adv[rows].astype(np.float64),
                                           pb.clip_eps, pb.ent_coef)
    na = X.arena_layout(pb.obs.shape[1], pb.actor.W[2].shape[1])[0]
    return g[:na], _actor_tolerance(pb, rows, dlg * len(rows) / mb)


@pytest.mark.parametrize("B,mb_off,mb,D,A", X.HOT_CASES)
def test_k3_actor_hot_rows(B, mb_off, mb, D, A):
    """ent_coef = 0 and a nonzero advantage on a few rows only: minibatch positions 0, 63, 64, 127, mb - 1 and rows in the
    last chunk of a dW1 and a dW0 split-K CTA.  The actor gradient matches the bf16-rounding oracle entry by entry within
    the tolerance of _actor_tolerance; the same check against the oracle with one hot row moved by one position fails
    (negative control).  The critic stays exact (v_old = value)."""
    pb = X.hot_problem(B, mb_off, mb, D, A)
    positions = X.hot_positions(mb)
    (g, mt), = _k3_run(pb, [(mb_off, mb)])
    na, coff, nc, _ = X.arena_layout(D, A)
    ref, rm = X.ppo_oracle(pb, mb_off, mb)
    _assert_equal(g[coff:coff + nc], ref[coff:coff + nc], "critic gradient")
    ref_a, tol = _hot_reference(pb, mb_off, mb, positions)
    np.testing.assert_allclose(ref_a, ref[:na], rtol=1e-12, atol=1e-15)   # the hot rows are the whole actor gradient
    got = g[:na].astype(np.float64)
    err = np.abs(got - ref_a)
    print(f"mb={mb}: hot rows {positions}; max |err| / tolerance = {(err / np.maximum(tol, 1e-30)).max():.3f}, "
          f"{np.count_nonzero(ref_a)} nonzero entries")
    assert (err <= tol).all(), f"{np.count_nonzero(err > tol)} actor gradient entries outside the tolerance"
    idx = pb.rows(mb_off, mb)
    for pos, to in ((0, 1), (64, 65), (mb - 1, mb - 2)):   # negative controls: the hot row one position off
        moved = X.PpoProblem(**{**pb.__dict__, "adv": pb.adv.copy()})
        moved.adv[idx[to]], moved.adv[idx[pos]] = pb.adv[idx[pos]], 0.0
        ref_m, tol_m = _hot_reference(moved, mb_off, mb, [to if q == pos else q for q in positions])
        assert not (np.abs(got - ref_m) <= tol_m).all(), f"hot row {pos} -> {to}: the tolerance cannot tell the rows apart"


# ---- dispatch invariance: switches read once per process, so every setting runs in a child process ----
_DISPATCH = [{}, {"STX_PDL": "0"}]
# mb = 128 (most K3b CTAs idle) and the benchmark minibatch (every K3b ring wraps); tests/test_k3_layout.py checks both facts
_DISPATCH_CASES = [X.CRITIC_CASES[0], X.CRITIC_CASES[3]]


def _dispatch_child(path: str) -> None:
    out = {}
    for i, case in enumerate(_DISPATCH_CASES):
        (g, mt), = _k3_run(X.critic_problem(*case), [case[1:3]])
        out[f"g{i}"], out[f"m{i}"] = g, mt
    np.savez(path, **out)


@pytest.mark.parametrize("env", _DISPATCH, ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()) or "default")
def test_k3_dispatch_invariance(env, tmp_path):
    """Chained (programmatic dependent launch) and serialised launches (STX_PDL=0), at mb = 128, where most K3b CTAs have
    no chunk, and at the benchmark minibatch, where every K3b CTA wraps its ring: the gradient arena equals the oracle bit
    for bit under each, hence they are bit-identical to each other."""
    path = str(tmp_path / "k3.npz")
    code = (f"import os; os.environ.update({env!r}); import sys; sys.path.insert(0, os.getcwd());"
            f"import tests.test_tc_exact_gpu as m; m._dispatch_child({path!r}); print('child-ok')")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert "child-ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    res = np.load(path)
    for i, case in enumerate(_DISPATCH_CASES):
        _check_critic_exact(X.critic_problem(*case), case[1], case[2], res[f"g{i}"], res[f"m{i}"], f"{env} mb={case[2]}")
