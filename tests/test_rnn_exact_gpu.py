"""The GRU and LSTM sequence kernels (stx_rnn.cu) against fp64 references, across their launch forms.

A. Precondition: the device's sigmoid and tanh give exactly 1, 0, 1/2 and +-1, 0 at the pre-activations +-128 and 0.
B. Exact GRU data (tests/rnn_exact_data.py): every form is exact in any summation order, so h_seq, d(gi), d(W_h), d(b_hn)
   and d(h0) must equal the oracle bit for bit, with overwrite True / False, without d(h0) and without d(W_h) / d(b_hn).
   The cases that need STX_GRU_CLUSTER / STX_GRU_PERSISTENT (read once per process) run in one child per setting.  The
   stx_launch_count() delta tells the per-step form (1 + T forward launches) from the single-kernel forms (1); the host
   mirror launch_form names which single-kernel form that is.
C. Bounds (LSTM, whose tanh(c) cannot be exact, and GRU at long T): each element is held to a first-order error bound in
   units of 2^-24 propagated through the steps (|J| e plus each operation's rounding: gamma_n sum|terms| per product,
   the documented 2-ulp bounds of expf / tanhf); deliberately wrong references must fail the same bound.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import rnn_exact_data as X

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), device="cuda:0").to(dtype)


def _np(t):
    return t.detach().cpu().numpy()


def _launches():
    from stoix_b200 import _lib

    torch.cuda.synchronize()
    return int(_lib.load().stx_launch_count())


def _assert_equal(got, ref, what):
    ref = np.asarray(ref, np.float32)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (f"{what}: {len(bad)} of {ref.size} entries differ from the oracle; first at {bad[0].tolist()}: "
                           f"kernel {got[tuple(bad[0])]!r} oracle {ref[tuple(bad[0])]!r}")


# ---------------------------------------------------------------------------------------------------------------------
# A. precondition
# ---------------------------------------------------------------------------------------------------------------------


def test_gate_functions_are_exact_at_the_codes():
    """T = 1, W_h = 0, b_hn = 0, h0 = 1: h = (1 - z) n + z, so h = z where n = tanh(0) = 0 and h = n where z = sigmoid(-128)
    = 0.  Units 0-2 read sigmoid(128), sigmoid(-128), sigmoid(0); units 3-5 read tanh(128), tanh(-128), tanh(0)."""
    from stoix_b200 import ops

    S = X.S
    H, E = 6, 1
    code_z = np.array([S, -S, 0.0, -S, -S, -S])
    code_n = np.array([0.0, 0.0, 0.0, S, -S, 0.0])
    gi = np.concatenate([np.zeros(H), code_z, code_n])[None, None].astype(np.float32)
    ws = ops.gru_workspace(1, E, H, "cuda:0")
    h = _np(ops.gru_sequence_forward(_t(gi), _t(np.zeros((1, E)), torch.uint8), _t(np.ones((E, H))), _t(np.zeros((H, 3 * H))), _t(np.zeros(H)), ws))[0, 0]
    names = ["sigmoid(128)", "sigmoid(-128)", "sigmoid(0)", "tanh(128)", "tanh(-128)", "tanh(0)"]
    want = np.array([1.0, 0.0, 0.5, 1.0, -1.0, 0.0], np.float32)
    print("device: " + ", ".join(f"{n} = {v!r}" for n, v in zip(names, h.tolist())))
    bad = [f"{n} = {v!r} (want {w})" for n, v, w in zip(names, h.tolist(), want.tolist()) if v != w]
    assert not bad, "the exact GRU data rests on these gate values; the device gave " + ", ".join(bad)


# ---------------------------------------------------------------------------------------------------------------------
# B. exact GRU data
# ---------------------------------------------------------------------------------------------------------------------


def _run_exact(pb: X.Problem):
    """Forward, then three backward calls: (a) overwrite=False, grad_weight 1/2 onto dW0 / db0, with d(h0); (b) overwrite=True,
    grad_weight 1, no d(h0); (c) no d(W_h) / d(b_hn).  Outputs start at 7.0 so that a skipped write shows."""
    from stoix_b200 import ops

    c = pb.case
    T, E, H = c.T, c.E, c.H
    reset = _t(pb.reset, torch.uint8)
    Wh = _t(pb.Wh)
    ws = ops.gru_workspace(T, E, H, "cuda:0")
    out, n = {}, {}
    l0 = _launches()
    out["h_seq"] = ops.gru_sequence_forward(_t(pb.gi), reset, _t(pb.h0), Wh, _t(pb.bhn), ws)
    l1 = _launches()
    n["fwd"] = l1 - l0
    d_gi_a, d_h0_a = torch.full((T, E, 3 * H), 7.0, device="cuda:0"), torch.full((E, H), 7.0, device="cuda:0")
    d_wh_acc, d_bhn_acc = _t(pb.dW0), _t(pb.db0)
    ops.gru_sequence_backward(_t(pb.d_h), reset, Wh, ws, d_gi_a, d_w_h=d_wh_acc, d_b_hn=d_bhn_acc, grad_weight=X.GRAD_WEIGHT, overwrite=False, d_h0=d_h0_a)
    l2 = _launches()
    d_gi_b, d_wh, d_bhn = torch.full((T, E, 3 * H), 7.0, device="cuda:0"), torch.full((H, 3 * H), 7.0, device="cuda:0"), torch.full((H,), 7.0, device="cuda:0")
    ops.gru_sequence_backward(_t(pb.d_h), reset, Wh, ws, d_gi_b, d_w_h=d_wh, d_b_hn=d_bhn)
    l3 = _launches()
    d_gi_c, d_h0_c = torch.full((T, E, 3 * H), 7.0, device="cuda:0"), torch.full((E, H), 7.0, device="cuda:0")
    ops.gru_sequence_backward(_t(pb.d_h), reset, Wh, ws, d_gi_c, d_h0=d_h0_c)
    l4 = _launches()
    n["bwd_acc_dh0"], n["bwd_no_dh0"], n["bwd_no_dw"] = l2 - l1, l3 - l2, l4 - l3
    out.update(d_gi_a=d_gi_a, d_h0_a=d_h0_a, d_wh_acc=d_wh_acc, d_bhn_acc=d_bhn_acc, d_gi_b=d_gi_b, d_wh=d_wh, d_bhn=d_bhn, d_gi_c=d_gi_c, d_h0_c=d_h0_c)
    return {k: _np(v) for k, v in out.items()}, n


def _check_exact(name, got, launches):
    c = X.CASE_BY_NAME[name]
    fm = c.form
    ref = X.reference(X.make_problem(c))
    want = {"fwd": fm.fwd_launches(c.T), "bwd_acc_dh0": fm.bwd_launches(c.T, True, True), "bwd_no_dh0": fm.bwd_launches(c.T, False, True),
            "bwd_no_dw": fm.bwd_launches(c.T, True, False)}
    print(f"{name:16s} T={c.T} E={c.E} H={c.H} {fm.name:9s} smem bwd {fm.smem_bwd:6d}: launches {launches}")
    assert launches == want, f"{name}: launches {launches}, the {fm.name} form gives {want}"
    for k, r in (("h_seq", ref.h_seq), ("d_gi_a", ref.d_gi), ("d_gi_b", ref.d_gi), ("d_gi_c", ref.d_gi), ("d_h0_a", ref.d_h0), ("d_h0_c", ref.d_h0),
                 ("d_wh_acc", ref.d_wh_acc), ("d_bhn_acc", ref.d_bhn_acc), ("d_wh", ref.d_wh), ("d_bhn", ref.d_bhn)):
        _assert_equal(got[k], r, f"{name} ({fm.name}): {k}")


def _group_child(env_key: str, path: str) -> None:
    res, counts = {}, {}
    for c in X.CASES:
        if json.dumps(c.env) == env_key:
            got, n = _run_exact(X.make_problem(c))
            res.update({f"{c.name}.{k}": v for k, v in got.items()})
            counts[c.name] = n
    np.savez(path, **res)
    with open(path + ".json", "w") as f:
        json.dump(counts, f)


@pytest.mark.parametrize("env", X.ENV_GROUPS, ids=lambda e: "+".join(f"{k}={v}" for k, v in e) or "default")
def test_exact_gru_cases(env, tmp_path):
    names = [c.name for c in X.CASES if c.env == env]
    if not env:
        for name in names:
            got, n = _run_exact(X.make_problem(X.CASE_BY_NAME[name]))
            _check_exact(name, got, n)
        return
    path = str(tmp_path / "res.npz")
    sets = "; ".join(f"os.environ[{k!r}] = {v!r}" for k, v in env)
    code = (f"import os; {sets}; import sys; sys.path.insert(0, os.getcwd());"
            f"import tests.test_rnn_exact_gpu as m; m._group_child({json.dumps(env)!r}, {path!r}); print('child-ok')")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "child-ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    res = np.load(path)
    with open(path + ".json") as f:
        counts = json.load(f)
    for name in names:
        _check_exact(name, {k.split(".", 1)[1]: res[k] for k in res.files if k.startswith(name + ".")}, counts[name])


# ---------------------------------------------------------------------------------------------------------------------
# C. first-order error bounds
# ---------------------------------------------------------------------------------------------------------------------


def _gamma(n):
    return n * U / (1 - n * U)


class B:
    """A value computed in fp64 and a first-order bound on the distance of the kernel's fp32 value from it."""

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else e

    def __add__(self, o):
        v = self.v + o.v
        return B(v, self.e + o.e + U * np.abs(v))

    def __mul__(self, o):
        v = self.v * o.v
        return B(v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + U * np.abs(v))

    def one_minus(self):
        v = 1.0 - self.v
        return B(v, self.e + U * np.abs(v))

    def sigmoid(self):   # 1 / (1 + expf(-x)): expf within 2 ulp, then two correctly rounded operations: < 6u relative
        v = 1.0 / (1.0 + np.exp(-self.v))
        return B(v, v * (1 - v) * self.e + 8 * U * v)

    def tanh(self):      # tanhf within 2 ulp
        v = np.tanh(self.v)
        return B(v, (1 - v * v) * self.e + 4 * U * np.abs(v))

    def cols(self, a, b):
        return B(self.v[..., a:b], self.e[..., a:b])

    def where(self, cut):
        return B(np.where(cut, 0.0, self.v), np.where(cut, 0.0, self.e))


def _matmul(x: B, W: np.ndarray, extra: B = None) -> B:
    """x W (+ extra) summed in any order: |x.e| |W| + gamma_n sum|terms|."""
    aw = np.abs(W)
    k = W.shape[0] + (extra is not None)
    v = x.v @ W + (0 if extra is None else extra.v)
    s = np.abs(x.v) @ aw + (0 if extra is None else np.abs(extra.v))
    return B(v, x.e @ aw + (0 if extra is None else extra.e) + _gamma(k) * s)


def _row_sum(a: B, b: B) -> B:
    """a^T b over all rows (the d(W_h) GEMM and its splits, any order)."""
    v = a.v.T @ b.v
    return B(v, np.abs(a.v).T @ b.e + a.e.T @ np.abs(b.v) + _gamma(a.v.shape[0]) * (np.abs(a.v).T @ np.abs(b.v)))


def lstm_bound(gi, reset, carry0, Wh, d_h, wrong=None):
    """lstm_forward / lstm_backward of oracle/rec_oracle.py in the kernels' operation order, with bounds.  `wrong` names a
    deliberately wrong reference."""
    T, E, H4 = gi.shape
    H = H4 // 4
    if wrong == "i_f_swapped":
        perm = np.r_[H:2 * H, 0:H, 2 * H:4 * H]
        out = lstm_bound(gi[..., perm], reset, carry0, Wh[:, perm], d_h)
        inv = np.argsort(perm)
        out["d_gi"] = B(out["d_gi"].v[..., inv], out["d_gi"].e[..., inv])
        out["d_wh"] = B(out["d_wh"].v[:, inv], out["d_wh"].e[:, inv])
        return out
    c0 = carry0[:, H:] if wrong == "carry0_swapped" else carry0[:, :H]
    h0 = carry0[:, :H] if wrong == "carry0_swapped" else carry0[:, H:]
    c, h = B(c0), B(h0)
    cache, hs = [], []
    for t in range(T):
        cut = reset[t][:, None]
        cp = c if wrong == "c_not_reset" else c.where(cut)
        hp = h.where(cut)
        z = _matmul(hp, Wh, B(gi[t]))
        i, f, g, o = z.cols(0, H).sigmoid(), z.cols(H, 2 * H).sigmoid(), z.cols(2 * H, 3 * H).tanh(), z.cols(3 * H, 4 * H).sigmoid()
        c = f * cp + i * g
        tc = c.tanh()
        h = o * tc
        hs.append(h)
        cache.append((cp, hp, i, f, g, o, tc))
    last = (h, c) if wrong == "carry_last_swapped" else (c, h)
    dh_rec, dc_rec = B(np.zeros((E, H))), B(np.zeros((E, H)))
    d_gi = [None] * T
    for t in range(T - 1, -1, -1):
        cp, hp, i, f, g, o, tc = cache[t]
        dh = B(d_h[t]) + dh_rec
        dc = dc_rec + dh * o * (tc * tc).one_minus()
        dz = [dc * g * i * i.one_minus(), dc * cp * f * f.one_minus(), dc * i * (g * g).one_minus(), dh * tc * o * o.one_minus()]
        d_gi[t] = B(np.concatenate([d.v for d in dz], 1), np.concatenate([d.e for d in dz], 1))
        cut = reset[t][:, None]
        dh_rec = _matmul(d_gi[t], Wh.T).where(cut)
        dcp = dc * f
        dc_rec = dcp if wrong == "dc_not_cut" else dcp.where(cut)
    dcarry = (dh_rec, dc_rec) if wrong == "d_carry0_swapped" else (dc_rec, dh_rec)
    cat = lambda xs, ax: B(np.concatenate([x.v for x in xs], ax), np.concatenate([x.e for x in xs], ax))
    hp_all = cat([cache[t][1] for t in range(T)], 0)
    dgi_all = cat(d_gi, 0)
    stack = lambda xs: B(np.stack([x.v for x in xs]), np.stack([x.e for x in xs]))
    return {"h_seq": stack(hs), "carry_last": cat(last, 1), "d_gi": stack(d_gi), "d_wh": _row_sum(hp_all, dgi_all), "d_carry0": cat(dcarry, 1)}


def gru_bound(gi, reset, h0, Wh, bhn, d_h, wrong=None):
    T, E, H3 = gi.shape
    H = H3 // 3
    h = B(h0)
    cache, hs = [], []
    for t in range(T):
        hp = h.where(reset[t][:, None])
        gh = _matmul(hp, Wh)
        g = B(gi[t])
        if wrong == "bhn_outside_r":
            ghn = gh.cols(2 * H, 3 * H)
            r = (g.cols(0, H) + gh.cols(0, H)).sigmoid()
            n = (g.cols(2 * H, 3 * H) + r * ghn + B(bhn)).tanh()
        else:
            ghn = gh.cols(2 * H, 3 * H) + B(bhn)
            r = (g.cols(0, H) + gh.cols(0, H)).sigmoid()
            n = (g.cols(2 * H, 3 * H) + r * ghn).tanh()
        z = (g.cols(H, 2 * H) + gh.cols(H, 2 * H)).sigmoid()
        h = z.one_minus() * n + z * hp
        hs.append(h)
        cache.append((hp, r, z, n, ghn))
    dh_rec = B(np.zeros((E, H)))
    d_gi, dgh_all = [None] * T, [None] * T
    for t in range(T - 1, -1, -1):
        hp, r, z, n, ghn = cache[t]
        dh = B(d_h[t]) + dh_rec
        dn = dh * z.one_minus()
        dz = dh * (hp + B(-n.v, n.e))
        dpn = dn * (n * n).one_minus()
        dpr = dpn * ghn * r * r.one_minus()
        dpz = dz * z * z.one_minus()
        dgn = dpn * r
        cat = lambda xs: B(np.concatenate([x.v for x in xs], 1), np.concatenate([x.e for x in xs], 1))
        dgh_all[t], d_gi[t] = cat([dpr, dpz, dgn]), cat([dpr, dpz, dpn])
        dh_rec = _matmul(dgh_all[t], Wh.T, dh * z).where(reset[t][:, None])
    stack = lambda xs: B(np.stack([x.v for x in xs]), np.stack([x.e for x in xs]))
    flat = lambda xs: B(np.concatenate([x.v for x in xs], 0), np.concatenate([x.e for x in xs], 0))
    hp_all, dgh = flat([c_[0] for c_ in cache]), flat(dgh_all)
    dbhn = B(dgh.v[:, 2 * H:].sum(0), dgh.e[:, 2 * H:].sum(0) + _gamma(dgh.v.shape[0]) * np.abs(dgh.v[:, 2 * H:]).sum(0))
    return {"h_seq": stack(hs), "d_gi": stack(d_gi), "d_wh": _row_sum(hp_all, dgh), "d_bhn": dbhn, "d_h0": dh_rec}


def _excess(got, ref: B):
    """Largest |kernel - reference| / (2 x bound); <= 1 passes.  The factor 2 covers the dropped second-order terms."""
    err = np.abs(got.astype(np.float64) - ref.v)
    return float((err / (2 * ref.e + 1e-37)).max())


def _bound_data(cell, T, E, H, seed):
    rng = np.random.default_rng(seed)
    G = 4 if cell == "lstm" else 3
    f32 = lambda a: np.asarray(a, np.float32)
    gi = f32(rng.standard_normal((T, E, G * H)))
    Wh = f32(rng.standard_normal((H, G * H)) * (0.25 / np.sqrt(H)))   # |J| < 1 per step: the bound stays finite over 256 steps
    carry = f32(rng.standard_normal((E, 2 * H if cell == "lstm" else H)))
    bhn = f32(rng.standard_normal(H) * 0.1)
    reset = rng.random((T, E)) < 0.2
    d_h = f32(rng.standard_normal((T, E, H)))
    acc0 = f32(rng.standard_normal((H, G * H)))
    return gi, Wh, carry, bhn, reset, d_h, acc0


LSTM_WRONG = ("c_not_reset", "dc_not_cut", "carry0_swapped", "carry_last_swapped", "d_carry0_swapped", "i_f_swapped")


@pytest.mark.parametrize("T,E,H", X.LSTM_CASES)
def test_lstm_within_error_bound(T, E, H):
    """Forward with carry_last, backward with overwrite=False onto a starting d(W_h) and d_carry0, then overwrite=True
    without d_carry0: every element within the propagated bound; each wrong reference fails it."""
    from stoix_b200 import ops

    fm = X.launch_form("lstm", T, E, H)
    gi, Wh, carry0, _, reset, d_h, acc0 = _bound_data("lstm", T, E, H, T * 1000 + E + H)
    f64 = lambda a: a.astype(np.float64)
    ws = ops.lstm_workspace(T, E, H, "cuda:0")
    last = torch.full((E, 2 * H), 7.0, device="cuda:0")
    l0 = _launches()
    h_seq = ops.lstm_sequence_forward(_t(gi), _t(reset, torch.uint8), _t(carry0), _t(Wh), ws, carry_last=last)
    l1 = _launches()
    d_gi, d_wh_acc, d_c0 = torch.full((T, E, 4 * H), 7.0, device="cuda:0"), _t(acc0), torch.full((E, 2 * H), 7.0, device="cuda:0")
    ops.lstm_sequence_backward(_t(d_h), _t(reset, torch.uint8), _t(Wh), ws, d_gi, d_w_h=d_wh_acc, grad_weight=0.25, overwrite=False, d_carry0=d_c0)
    l2 = _launches()
    d_gi2, d_wh = torch.full((T, E, 4 * H), 7.0, device="cuda:0"), torch.full((H, 4 * H), 7.0, device="cuda:0")
    ops.lstm_sequence_backward(_t(d_h), _t(reset, torch.uint8), _t(Wh), ws, d_gi2, d_w_h=d_wh)
    l3 = _launches()
    assert (l1 - l0, l2 - l1, l3 - l2) == (fm.fwd_launches(T), fm.bwd_launches(T, True, True), fm.bwd_launches(T, False, True)), fm.name
    got = {"h_seq": _np(h_seq), "carry_last": _np(last), "d_gi": _np(d_gi), "d_carry0": _np(d_c0), "d_wh": _np(d_wh), "d_gi2": _np(d_gi2),
           "d_wh_acc": _np(d_wh_acc)}
    ref = lstm_bound(f64(gi), reset, f64(carry0), f64(Wh), f64(d_h))
    acc = ref["d_wh"]
    acc_v = f64(acc0) + 0.25 * acc.v
    ref["d_wh_acc"] = B(acc_v, 0.25 * acc.e + U * np.abs(acc_v))
    ref["d_gi2"] = ref["d_gi"]
    ex = {k: _excess(got[k], ref[k]) for k in got}
    print(f"lstm T={T} E={E} H={H} {fm.name}: |err| / (2 bound) " + ", ".join(f"{k} {v:.2g}" for k, v in ex.items())
          + f"; median bound on h_seq {np.median(ref['h_seq'].e) / U:.3g} units of 2^-24")
    bad = {k: v for k, v in ex.items() if not v <= 1}
    assert not bad, f"lstm {fm.name} T={T} E={E} H={H}: outside the bound {bad}"
    for w in LSTM_WRONG:
        if w in ("c_not_reset", "dc_not_cut") and not reset[1:].any():
            continue
        wr = lstm_bound(f64(gi), reset, f64(carry0), f64(Wh), f64(d_h), wrong=w)
        worst = max(_excess(got[k], wr[k]) for k in ("h_seq", "carry_last", "d_gi", "d_carry0", "d_wh"))
        assert worst > 1, f"wrong reference {w} passes the bound ({worst:.3g})"


GRU_BOUND_CASES = [(1, 2048, 128), (256, 128, 128), (12, 40, 20)]


@pytest.mark.parametrize("T,E,H", GRU_BOUND_CASES)
def test_gru_within_error_bound(T, E, H):
    """The rollout step and the training chunk of scripts/bench_rec.py on random data; b_hn added outside r (...) must fail."""
    from stoix_b200 import ops

    fm = X.launch_form("gru", T, E, H)
    gi, Wh, h0, bhn, reset, d_h, acc0 = _bound_data("gru", T, E, H, T * 1000 + E + H)
    f64 = lambda a: a.astype(np.float64)
    ws = ops.gru_workspace(T, E, H, "cuda:0")
    l0 = _launches()
    h_seq = ops.gru_sequence_forward(_t(gi), _t(reset, torch.uint8), _t(h0), _t(Wh), _t(bhn), ws)
    l1 = _launches()
    d_gi, d_wh, d_bhn, d_h0 = (torch.full(s, 7.0, device="cuda:0") for s in ((T, E, 3 * H), (H, 3 * H), (H,), (E, H)))
    ops.gru_sequence_backward(_t(d_h), _t(reset, torch.uint8), _t(Wh), ws, d_gi, d_w_h=d_wh, d_b_hn=d_bhn, d_h0=d_h0)
    l2 = _launches()
    assert (l1 - l0, l2 - l1) == (fm.fwd_launches(T), fm.bwd_launches(T, True, True)), fm.name
    got = {"h_seq": _np(h_seq), "d_gi": _np(d_gi), "d_wh": _np(d_wh), "d_bhn": _np(d_bhn), "d_h0": _np(d_h0)}
    ref = gru_bound(f64(gi), reset, f64(h0), f64(Wh), f64(bhn), f64(d_h))
    ex = {k: _excess(got[k], ref[k]) for k in got}
    print(f"gru T={T} E={E} H={H} {fm.name}: |err| / (2 bound) " + ", ".join(f"{k} {v:.2g}" for k, v in ex.items()))
    bad = {k: v for k, v in ex.items() if not v <= 1}
    assert not bad, f"gru {fm.name} T={T} E={E} H={H}: outside the bound {bad}"
    wr = gru_bound(f64(gi), reset, f64(h0), f64(Wh), f64(bhn), f64(d_h), wrong="bhn_outside_r")
    worst = max(_excess(got[k], wr[k]) for k in got)
    assert worst > 1, f"wrong reference bhn_outside_r passes the bound ({worst:.3g})"
