"""The fp32 train-mode MLP (stx_mlp_forward_train / stx_mlp_backward / stx_mlp_forward, stx_simt_gemm.cuh) against fp64
references, in three tiers.

A. Exact data (tests/simt_exact_data.py): every GEMM, split and reduction is exact in any order, so forward output,
   parameter gradients (overwrite 1 and 0), d(input), the d(input)-only call, gathered strided input and the inference
   entry must equal the oracle bit for bit, on every tiling and split path.
B. Element-wise epilogues: "identity sandwich" networks [N, N, N] with W0 = W1 = I and b1 = 0.  Each GEMM then adds
   exact zeros to one product, so the output IS the kernel's f(U) or f(LN(U)), d(input) IS its activation / LayerNorm
   backward of d(out), and the gradient arena holds the column sums (db0, or LayerNorm dgamma / dbeta).  Each element is
   held to c * 2^-24 * scale, scale a first-order bound from the magnitudes of the formula's terms (_tier_b_case); deliberately
   wrong references (a neighbouring activation's derivative, LayerNorm eps 1e-5, the uh * mean(dhat * uh) term dropped)
   must fail the same bound.
C. Composition at the shipped shapes against the fp64 oracle: per-element running error bounds where the forward is
   exact (relu at M = 32768), per-tensor norm-wise bounds for LayerNorm + silu and silu networks.
"""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import simt_exact_data as S

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
ACTS = ["relu", "tanh", "silu", "elu", "gelu", "sigmoid", "softplus", "identity"]


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), device="cuda:0").to(dtype)


def _np(t):
    return t.detach().cpu().numpy()


def _assert_equal(got, ref, what):
    ref = np.asarray(ref, np.float32)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (f"{what}: {len(bad)} of {ref.size} entries differ from the oracle; first at {bad[0].tolist()}: "
                           f"kernel {got[tuple(bad[0])]} oracle {ref[tuple(bad[0])]}")


# ---------------------------------------------------------------------------------------------------------------------
# Tier A: exact data
# ---------------------------------------------------------------------------------------------------------------------


def _run_exact(pb: S.Problem):
    """Every entry point on one problem; net_grad / d_input start filled with 7.0 so that a skipped write shows."""
    from stoix_b200 import ops

    c = pb.case
    spec = ops.MlpSpec(c.sizes, c.activation)
    params, xbuf, d_out = _t(pb.net.flat()), _t(pb.xbuf), _t(pb.d_out)
    ridx = _t(pb.row_idx, torch.int32) if c.gathered else None
    ws = ops.mlp_train_workspace(spec, c.M, "cuda:0")
    out = ops.mlp_forward_train(spec, params, xbuf, ws, row_idx=ridx)
    grad = torch.full((spec.param_count,), 7.0, device="cuda:0")
    d_in = torch.full((c.M, c.sizes[0]), 7.0, device="cuda:0")
    ops.mlp_backward(spec, params, xbuf, d_out, ws, net_grad=grad, grad_weight=S.GRAD_WEIGHT, overwrite=True, d_input=d_in, row_idx=ridx)
    grad_acc = _t(pb.grad0)
    ops.mlp_backward(spec, params, xbuf, d_out, ws, net_grad=grad_acc, grad_weight=S.GRAD_WEIGHT, overwrite=False, row_idx=ridx)
    grad_before = grad.clone()
    d_in_only = torch.full((c.M, c.sizes[0]), 7.0, device="cuda:0")
    ops.mlp_backward(spec, params, xbuf, d_out, ws, d_input=d_in_only, row_idx=ridx)
    out_inf = ops.mlp_forward(spec, params, xbuf[:, :c.sizes[0]].contiguous(), row_idx=ridx)
    torch.cuda.synchronize()
    assert torch.equal(grad, grad_before), "the d_input-only call changed a parameter gradient"
    return {k: _np(v) for k, v in dict(out=out, out_inf=out_inf, grad=grad, grad_acc=grad_acc, d_input=d_in, d_input_only=d_in_only).items()}


def _check_exact(got, ref: S.Reference, what):
    for k, r in (("out", ref.out), ("out_inf", ref.out), ("grad", ref.grad), ("grad_acc", ref.grad_acc), ("d_input", ref.d_input),
                 ("d_input_only", ref.d_input)):
        _assert_equal(got[k], r, f"{what}: {k}")


@pytest.mark.parametrize("name", [c.name for c in S.CASES])
def test_exact_case(name):
    """Forward (train and inference), gradients with overwrite 1 and 0, d(input), the d(input)-only call: equal to the
    oracle bit for bit; a second run equals the first."""
    c = S.CASE_BY_NAME[name]
    plan = S.launch_plan(c.sizes, c.M)
    print(f"{name} {c.sizes} M={c.M}: splits {next(l for l in plan if l.mode == 'DW').splits}, "
          + " ".join(f"{l.mode}{l.layer}:{l.tile}" for l in plan))
    pb = S.make_problem(c)
    ref = S.reference(pb)
    got = _run_exact(pb)
    _check_exact(got, ref, name)
    again = _run_exact(pb)
    for k in got:
        assert np.array_equal(got[k], again[k]), f"{name}: {k} differs between two identical calls"


def test_layernorm_wider_than_1024_is_refused():
    from stoix_b200 import ops

    spec = ops.MlpSpec((8, 1056, 1), "silu", use_layer_norm=True)
    params, x = torch.zeros(spec.param_count, device="cuda:0"), torch.zeros(4, 8, device="cuda:0")
    with pytest.raises(ops.StxError, match=r"rc=-2"):
        ops.mlp_forward_train(spec, params, x, ops.mlp_train_workspace(spec, 4, "cuda:0"))


# ---------------------------------------------------------------------------------------------------------------------
# Tier B: element-wise epilogues on identity sandwiches
# ---------------------------------------------------------------------------------------------------------------------

C_ELEM = 8.0      # ulps of one fp32 formula (the kernel's expf / tanhf / expm1f / log1pf are within 2 ulps each)
C_TOL = 2.0       # safety factor on the whole first-order bound
_H = 1e-4


def _mag_f(act, z):
    """Sum of |terms| of the kernel's act_fwd(z), with the sensitivity of tanh's argument for gelu (units of |f|)."""
    t = np.tanh(0.7978845608028654 * (z + 0.044715 * z ** 3))
    f, _ = O.ACTIVATIONS[act]
    if act in ("relu", "identity"):
        return np.zeros_like(z)
    if act == "gelu":
        return 0.5 * np.abs(z) * (1 + np.abs(t) + (1 - t * t) * np.abs(0.7978845608028654 * (z + 0.044715 * z ** 3)))
    return np.abs(f(z))


def _mag_g(act, z):
    """Sum of |terms| of the kernel's act_grad(z) (1 - s or 1 - t^2 cancel to an absolute error of the order of 1 ulp of 1)."""
    s = 1.0 / (1.0 + np.exp(-z))
    t = np.tanh(0.7978845608028654 * (z + 0.044715 * z ** 3))
    arg = np.abs(0.7978845608028654 * (z + 0.044715 * z ** 3))
    return {"relu": 0 * z, "identity": 0 * z, "tanh": 1 + 0 * z, "silu": s * (1 + 2 * np.abs(z)) + 1e-30, "elu": np.where(z > 0, 0, np.exp(z)),
            "gelu": 0.5 * (1 + np.abs(t)) + (1 - t * t) * arg
                    + 0.5 * np.abs(z) * 0.7978845608028654 * (1 + 0.134145 * z * z) * (1 + 2 * np.abs(t) * (np.abs(t) + (1 - t * t) * arg)),
            "sigmoid": s, "softplus": s}[act]


def _fpp(act, z):
    _, fp = O.ACTIVATIONS[act]
    return np.abs(fp(z + _H) - fp(z - _H)) / (2 * _H) if act not in ("relu", "identity") else 0 * z


def _ln_forward(u, gamma, beta, act, eps=O.LN_EPS):
    mean = u.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((u - mean) ** 2).mean(-1, keepdims=True) + eps)
    uh = (u - mean) * rstd
    z = uh * gamma + beta
    return O.ACTIVATIONS[act][0](z), z, uh, rstd


def _ln_backward(d, z, uh, rstd, gamma, act, drop_s2=False):
    dz = d * O.ACTIVATIONS[act][1](z)
    dhat = dz * gamma
    s2 = 0.0 if drop_s2 else (dhat * uh).mean(-1, keepdims=True)
    return rstd * (dhat - dhat.mean(-1, keepdims=True) - uh * s2), (dz * uh).sum(0), dz.sum(0)


def _sandwich(rng, N, act, ln):
    """[N, N, N] with W0 = W1 = I, head bias 0; no LayerNorm: b0 = 0 (U = x exactly); LayerNorm: random scale / bias."""
    I = np.eye(N)
    if ln:
        return O.MLPParams([I, I], [1.0 + 0.3 * rng.standard_normal(N), np.zeros(N)], act, [0.2 * rng.standard_normal(N), None])
    return O.MLPParams([I, I], [np.zeros(N), np.zeros(N)], act)


def _run_sandwich(net, N, ln, x, d):
    from stoix_b200 import ops

    spec = ops.MlpSpec((N, N, N), net.activation, use_layer_norm=ln)
    params = _t(net.flat().astype(np.float32))
    M = x.shape[0]
    ws = ops.mlp_train_workspace(spec, M, "cuda:0")
    xt = _t(x)
    out = ops.mlp_forward_train(spec, params, xt, ws)
    grad, d_in = torch.zeros(spec.param_count, device="cuda:0"), torch.empty(M, N, device="cuda:0")
    ops.mlp_backward(spec, params, xt, _t(d), ws, net_grad=grad, d_input=d_in)
    torch.cuda.synchronize()
    sl = spec.layer_slices()[0][1]
    g = _np(grad)
    cols = (g[sl], g[spec.ln_bias_slices()[0]]) if ln else (g[sl],)
    return _np(out), _np(d_in), cols


def _tier_b_case(act, ln, N, Ms=(1, 7, 300, 37000), controls_at=300):
    from stoix_b200 import ops

    rng = np.random.default_rng(1000 * ACTS.index(act) + 2 * N + int(ln))
    net = _sandwich(rng, N, act, ln)
    spec = ops.MlpSpec((N, N, N), act, use_layer_norm=ln)
    assert spec.param_count == net.flat().size
    L = -(-N // 32) + 7                          # serial adds per lane + 5 shuffle levels + 2: mean / variance / row sums
    worst = {}
    for M in Ms:
        if ln:   # small row variance: LayerNorm's eps matters at the 1 % level (negative control below)
            x = (0.05 + 0.02 * rng.standard_normal((M, N))).astype(np.float32)
        else:
            x = (2.5 * rng.standard_normal((M, N))).astype(np.float32)
        d = rng.standard_normal((M, N)).astype(np.float32)
        out, d_in, cols = _run_sandwich(net, N, ln, x, d)
        u, d64 = x.astype(np.float64), d.astype(np.float64)
        ref_out, acts = O.mlp_forward(net, u)
        gref = O.MLPParams.from_flat(O.mlp_backward(net, acts, d64).flat(), (N, N, N), act, ln)
        if ln:
            gamma, beta = net.b[0], net.ln_bias[0]
            h, z, uh, rstd = _ln_forward(u, gamma, beta, act)
            np.testing.assert_allclose(h, ref_out, rtol=1e-12, atol=1e-14)            # the local LayerNorm == the oracle
            r_din, dg, db = _ln_backward(d64, z, uh, rstd, gamma, act)
            np.testing.assert_allclose(dg, gref.b[0], rtol=1e-10, atol=1e-12)
            np.testing.assert_allclose(db, gref.ln_bias[0], rtol=1e-10, atol=1e-12)
            # first-order error bounds (units of 2^-24)
            mabs = np.abs(u).mean(-1, keepdims=True)
            e_uh = rstd * L * mabs + np.abs(uh) * (L / 2 + 6)
            e_z = np.abs(gamma) * e_uh + np.abs(z) + np.abs(beta)
            fp = O.ACTIVATIONS[act][1](z)
            tol_out = C_TOL * U * (np.abs(fp) * e_z + C_ELEM * _mag_f(act, z))
            dz = d64 * fp
            e_dz = np.abs(d64) * (_fpp(act, z) * e_z + C_ELEM * _mag_g(act, z)) + np.abs(dz)
            dhat = dz * gamma
            e_dhat = np.abs(gamma) * e_dz + np.abs(dhat)
            s2 = (dhat * uh).mean(-1, keepdims=True)
            e_s1 = e_dhat.mean(-1, keepdims=True) + L * np.abs(dhat).mean(-1, keepdims=True)
            e_s2 = (e_dhat * np.abs(uh) + np.abs(dhat) * e_uh).mean(-1, keepdims=True) + L * np.abs(dhat * uh).mean(-1, keepdims=True)
            e_din = rstd * (e_dhat + e_s1 + e_uh * np.abs(s2) + np.abs(uh) * e_s2
                            + 3 * (np.abs(dhat) + np.abs(dhat).mean(-1, keepdims=True) + np.abs(uh * s2))) + np.abs(r_din) * (L / 2 + 3)
            tol_din = C_TOL * U * e_din
            ln_rows = min(-(-(-(-M // 296)) // 8) * 8, 128)   # stx_mlp.cu carve(): rows per ln_backward block
            chain = ln_rows // 8 + 8 + -(-M // ln_rows) + 2    # rows per warp, warps, blocks: summed in that order
            tol_cols = [C_TOL * U * ((e_dz * np.abs(uh) + np.abs(dz) * e_uh).sum(0) + chain * np.abs(dz * uh).sum(0)),
                        C_TOL * U * (e_dz.sum(0) + chain * np.abs(dz).sum(0))]
            ref_cols = [dg, db]
        else:
            r_din = d64 * O.ACTIVATIONS[act][1](u)
            tol_out = C_TOL * U * C_ELEM * _mag_f(act, u)
            e_din = np.abs(d64) * C_ELEM * _mag_g(act, u) + np.abs(r_din)
            tol_din = C_TOL * U * np.where(_mag_g(act, u) > 0, e_din, 0)
            splits = S.pick_splits((N, N, N), M)
            chain = -(-M // splits) + splits + 2
            tol_cols = [C_TOL * U * (e_din.sum(0) + chain * np.abs(r_din).sum(0))]
            ref_cols = [gref.b[0]]
        checks = [("out", out, ref_out, tol_out), ("d_input", d_in, r_din, tol_din)] + [
            (nm, g, r, tl) for nm, g, r, tl in zip(("dgamma", "dbeta") if ln else ("db0",), cols, ref_cols, tol_cols)]
        for nm, got, ref, tol in checks:
            err = np.abs(got.astype(np.float64) - ref)
            ratio = float((err / np.maximum(tol, 1e-300)).max()) if (tol > 0).any() else 0.0
            key = f"M={M} {nm}"
            worst[key] = ratio
            bad = err > tol
            assert not bad.any(), f"{act} ln={ln} N={N} {key}: {bad.sum()} of {bad.size} outside c 2^-24 scale; worst ratio {ratio:.2f}"
        if M == controls_at:   # negative controls: deliberately wrong references must fail the same bounds
            wrong_act = ACTS[(ACTS.index(act) + 1) % len(ACTS)]
            if ln:
                h5, _, _, _ = _ln_forward(u, gamma, beta, act, eps=1e-5)
                assert (np.abs(out - h5) > tol_out).any(), "LayerNorm eps 1e-5: the bound cannot tell"
                nos2, _, _ = _ln_backward(d64, z, uh, rstd, gamma, act, drop_s2=True)
                assert (np.abs(d_in - nos2) > tol_din).any(), "uh * mean(dhat * uh) dropped: the bound cannot tell"
                wz, _, _ = _ln_backward(d64, z, uh, rstd, gamma, wrong_act)
                assert (np.abs(d_in - wz) > tol_din).any(), f"{wrong_act}' in place of {act}': the bound cannot tell"
            else:
                wrong = d64 * O.ACTIVATIONS[wrong_act][1](u)
                assert (np.abs(d_in - wrong) > tol_din).any(), f"{wrong_act}' in place of {act}': the bound cannot tell"
    print(f"{act} ln={ln} N={N}: worst |err| / tolerance " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("N", [200, 256])
@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("act", ACTS)
def test_epilogue_elementwise(act, ln, N):
    """M = 37000 (ln_backward's 128-row cap, a ragged last block) at N = 256 only: it dominates the file's run time."""
    _tier_b_case(act, ln, N, Ms=(1, 7, 300, 37000) if N == 256 else (1, 7, 300))


@pytest.mark.parametrize("N", [32, 48, 768, 769, 1024])
def test_layernorm_silu_widths(N):
    """Up to the widest LayerNorm check_mlp accepts: above 768 the backward needs more than 48 KiB of shared memory.
    (M = 37000, the ln_backward row cap, runs at N = 256 above.)"""
    _tier_b_case("silu", True, N, Ms=(1, 7, 300))


# ---------------------------------------------------------------------------------------------------------------------
# Tier C: composition at the shipped shapes
# ---------------------------------------------------------------------------------------------------------------------


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-300))


def _run_train(spec, net, x, d):
    from stoix_b200 import ops

    params, xt = _t(net.flat().astype(np.float32)), _t(x)
    M = x.shape[0]
    ws = ops.mlp_train_workspace(spec, M, "cuda:0")
    out = ops.mlp_forward_train(spec, params, xt, ws)
    grad, d_in = torch.zeros(spec.param_count, device="cuda:0"), torch.empty(M, spec.sizes[0], device="cuda:0")
    ops.mlp_backward(spec, params, xt, _t(d), ws, net_grad=grad, d_input=d_in)
    torch.cuda.synchronize()
    return _np(out), _np(grad), _np(d_in)


def _d_input_silu(net, sizes, ln, x, d):
    """d(input) of a silu network in fp64 autograd on the CPU (flax Dense / LayerNorm(eps 1e-6) / silu)."""
    import torch.nn.functional as F

    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    h, n = xt, len(net.W)
    for i in range(n):
        W, b = torch.tensor(net.W[i]), torch.tensor(net.b[i])
        if ln and i < n - 1:
            z = F.layer_norm(h @ W, (sizes[i + 1],), b, torch.tensor(net.ln_bias[i]), eps=O.LN_EPS)
        else:
            z = h @ W + b
        h = F.silu(z) if i < n - 1 else z
    h.backward(torch.tensor(d, dtype=torch.float64))
    return xt.grad.numpy()


@pytest.mark.parametrize("sizes,act,ln,M", [
    ((23, 256, 256, 256, 256, 1), "silu", True, 256),     # SAC Q network (mlp_sac.yaml) at the shipped batch
    ((23, 256, 256, 256, 256, 1), "silu", True, 4096),
    ((17, 256, 256, 256, 256, 12), "silu", False, 256),   # continuous actor, A = 6
    ((17, 256, 256, 256, 256, 12), "silu", False, 4096),
])
def test_shipped_networks_normwise(sizes, act, ln, M):
    """Random data, fp64 oracle, per tensor: forward 1e-5, every parameter gradient tensor and d(input) 1e-4 norm-wise
    (the fp32 minibatch tests allow 5e-3 over the whole network)."""
    from stoix_b200 import ops

    rng = np.random.default_rng(M + sizes[-1] + int(ln))
    n = len(sizes) - 1
    p = O.init_mlp(rng, sizes, 1.0)
    b = [0.1 * rng.standard_normal(sizes[i + 1]) + (1.0 if ln and i < n - 1 else 0.0) for i in range(n)]
    lnb = [0.1 * rng.standard_normal(sizes[i + 1]) if i < n - 1 else None for i in range(n)] if ln else None
    net = O.MLPParams(p.W, b, act, lnb)
    spec = ops.MlpSpec(tuple(sizes), act, use_layer_norm=ln)
    x = rng.standard_normal((M, sizes[0])).astype(np.float32)
    d = (rng.standard_normal((M, sizes[-1])) / M).astype(np.float32)
    out, grad, d_in = _run_train(spec, net, x, d)
    ref_out, acts = O.mlp_forward(net, x.astype(np.float64))
    g = O.mlp_backward(net, acts, d.astype(np.float64))
    d0 = _d_input_silu(net, sizes, ln, x, d)
    errs = {"out": _rel(out, ref_out)}
    gk = O.MLPParams.from_flat(grad.astype(np.float64), sizes, act, ln)
    for i in range(n):
        errs[f"dW{i}"], errs[f"b{i}"] = _rel(gk.W[i], g.W[i]), _rel(gk.b[i], g.b[i])
        if ln and i < n - 1:
            errs[f"lnb{i}"] = _rel(gk.ln_bias[i], g.ln_bias[i])
    errs["d_input"] = _rel(d_in, d0)
    print(f"{sizes} {act} ln={ln} M={M}: norm-wise " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert errs.pop("out") < 1e-5
    bad = {k: v for k, v in errs.items() if v >= 1e-4}
    assert not bad, bad


def test_bench_shape_relu_per_element():
    """[64, 256, 256, 8] relu at M = 32768 (66 weight-gradient splits): the exact-data forward (so no pre-activation can
    land on the other side of the kink) with a random d(out).  Every gradient entry and d(input) within the running
    error bound of its fp32 sums: (reduction length + 2) * 2^-24 * sum |terms|, propagated through the layers."""
    from stoix_b200 import ops

    pb = S.make_problem(S.CASE_BY_NAME["bench"])
    c = pb.case
    rng = np.random.default_rng(5)
    d = rng.standard_normal((c.M, c.sizes[-1])).astype(np.float32)
    x = pb.x
    out, grad, d_in = _run_train(ops.MlpSpec(c.sizes, c.activation), pb.net, x.astype(np.float32), d)
    ch = S.chain(pb.net, x, d)
    _assert_equal(out, ch.out, "bench forward (exact)")
    n = len(pb.net.W)
    splits = S.pick_splits(c.sizes, c.M)
    red = -(-c.M // splits) + splits + 2
    err_d = [None] * n
    err_d[n - 1] = np.zeros_like(ch.d[n - 1])
    for i in range(n - 1, 0, -1):
        mask = (ch.pre[i - 1] > 0)
        err_d[i - 1] = ((err_d[i] + (c.sizes[i + 1] + 2) * U * np.abs(ch.d[i])) @ np.abs(pb.net.W[i]).T) * mask
    tol_din = (err_d[0] + (c.sizes[1] + 2) * U * np.abs(ch.d[0])) @ np.abs(pb.net.W[0]).T
    tol = O.MLPParams([np.abs(ch.inputs[i]).T @ (err_d[i] + red * U * np.abs(ch.d[i])) for i in range(n)],
                      [(err_d[i] + red * U * np.abs(ch.d[i])).sum(0) for i in range(n)]).flat()
    ref = S.layer_grads(pb.net, ch)
    for nm, got, r, tl in (("grad", grad, ref, tol), ("d_input", d_in, ch.d_input, tol_din)):
        err = np.abs(got.astype(np.float64) - r)
        print(f"bench relu M={c.M}: {nm} worst |err| / bound {float((err / np.maximum(tl, 1e-300)).max()):.3f}")
        assert (err <= tl).all(), f"{nm}: {(err > tl).sum()} entries outside the running error bound"
