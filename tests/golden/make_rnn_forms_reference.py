"""Bit-level reference of the GRU and LSTM sequence kernels (stx_rnn.cu) in every launch form.

Seeded random inputs (not the exactly representable data of tests/rnn_exact_data.py, which hides summation order and FMA
contraction by design) run through each form: the 2-CTA cluster kernels, the persistent GRU kernels seq<4,2> and seq<8,1>,
and the per-step form of one SIMT GEMM and one gate kernel per step.  Each case runs one forward and two backward calls:
(acc) overwrite=False onto a random starting gradient with grad_weight 1/2 and with d(h0) / d(carry0), and (ovw)
overwrite=True without it.  Rows are ragged against the row tiles and resets are random.  Recorded per case: the form
tests/rnn_exact_data.launch_form names (which proves what the case reaches), the stx_launch_count() delta of each call,
and the SHA-256 of every output with a seeded sample of its values for diagnosing a mismatch.

The kernels are deterministic (fixed-order partial sums), so the hashes pin every float expression and summation order.
Cases that need STX_GRU_CLUSTER / STX_GRU_PERSISTENT / STX_LSTM_CLUSTER (read once per process) run in one child process per
setting.  Generate on an H100 with the build the reference should describe:

    python tests/golden/make_rnn_forms_reference.py tests/golden/rnn_forms_reference.json
"""
from __future__ import annotations

import hashlib
import json
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
N_SAMPLE = 32

NO_GRU_CLUSTER = (("STX_GRU_CLUSTER", "0"),)
NO_LSTM_CLUSTER = (("STX_LSTM_CLUSTER", "0"),)

# (name, cell, T, E, H, env); the comment is the form launch_form gives
CASES = [
    ("gru_cluster", "gru", 8, 301, 128, ()),                       # cluster, ragged last tile
    ("gru_cluster_h20", "gru", 5, 33, 20, ()),                     # cluster, small H
    ("gru_seq42_h63", "gru", 6, 37, 63, ()),                       # odd H: seq<4,2>
    ("gru_seq42_nocluster", "gru", 8, 301, 128, NO_GRU_CLUSTER),   # seq<4,2> at the cluster's shape
    ("gru_seq81", "gru", 5, 1027, 128, ()),                        # E >= 1024: seq<8,1>
    ("gru_step_t3", "gru", 3, 301, 128, ()),                       # T < 4: per-step
    ("gru_step_h256", "gru", 8, 67, 256, ()),                      # H = 256 (R2D2's default): per-step
    ("lstm_cluster", "lstm", 8, 301, 128, ()),                     # cluster
    ("lstm_cluster_h20", "lstm", 5, 33, 20, ()),                   # cluster, small H
    ("lstm_step_t3", "lstm", 3, 301, 128, ()),                     # T < 4: per-step
    ("lstm_step_nocluster", "lstm", 8, 301, 128, NO_LSTM_CLUSTER),  # per-step at the cluster's shape
    ("lstm_step_h63", "lstm", 6, 37, 63, ()),                      # odd H: per-step
]


def _digest(t) -> dict:
    a = t.detach().cpu().contiguous().numpy()
    flat = a.reshape(-1).view(np.uint32)
    pick = np.random.default_rng(flat.size).choice(flat.size, min(N_SAMPLE, flat.size), replace=False)
    return {"sha256": hashlib.sha256(a.tobytes()).hexdigest(), "sample_index": pick.tolist(), "sample_f32_hex": flat[pick].tobytes().hex()}


def run_case(name, cell, T, E, H, env) -> dict:
    import torch

    from stoix_b200 import _lib, ops
    from tests import rnn_exact_data as X

    dev = torch.device("cuda:0")
    lib = _lib.load()
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    G = 3 if cell == "gru" else 4
    nc = 1 if cell == "gru" else 2
    f = lambda *shape, s=1.0: torch.tensor(rng.standard_normal(shape).astype(np.float32) * np.float32(s), device=dev)
    gi, w_h = f(T, E, G * H), f(H, G * H, s=1.0 / np.sqrt(H))
    carry0, b_hn = f(E, nc * H, s=0.5), f(H, s=0.3)
    reset = torch.tensor(rng.random((T, E)) < 0.2, device=dev)
    d_h = f(T, E, H)
    dw0, db0 = f(H, G * H, s=0.1), f(H, s=0.1)
    ws = (ops.gru_workspace if cell == "gru" else ops.lstm_workspace)(T, E, H, dev)

    def count(fn):
        torch.cuda.synchronize()
        l0 = lib.stx_launch_count()
        fn()
        torch.cuda.synchronize()
        return int(lib.stx_launch_count() - l0)

    out, launches = {}, {}
    if cell == "gru":
        launches["fwd"] = count(lambda: out.update(h_seq=ops.gru_sequence_forward(gi, reset, carry0, w_h, b_hn, ws)))
        d_gi, d_h0, d_w, d_b = torch.zeros(T, E, G * H, device=dev), torch.zeros(E, H, device=dev), dw0.clone(), db0.clone()
        launches["bwd_acc"] = count(lambda: ops.gru_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=d_w, d_b_hn=d_b, grad_weight=0.5,
                                                                       overwrite=False, d_h0=d_h0))
        out.update(d_gi_acc=d_gi, d_w_h_acc=d_w, d_b_hn_acc=d_b, d_h0_acc=d_h0)
        d_gi, d_w, d_b = torch.zeros(T, E, G * H, device=dev), torch.zeros(H, G * H, device=dev), torch.zeros(H, device=dev)
        launches["bwd_ovw"] = count(lambda: ops.gru_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=d_w, d_b_hn=d_b))
        out.update(d_gi_ovw=d_gi, d_w_h_ovw=d_w, d_b_hn_ovw=d_b)
    else:
        carry_last = torch.zeros(E, 2 * H, device=dev)
        launches["fwd"] = count(lambda: out.update(h_seq=ops.lstm_sequence_forward(gi, reset, carry0, w_h, ws, carry_last=carry_last)))
        out["carry_last"] = carry_last
        d_gi, d_c0, d_w = torch.zeros(T, E, G * H, device=dev), torch.zeros(E, 2 * H, device=dev), dw0.clone()
        launches["bwd_acc"] = count(lambda: ops.lstm_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=d_w, grad_weight=0.5, overwrite=False,
                                                                        d_carry0=d_c0))
        out.update(d_gi_acc=d_gi, d_w_h_acc=d_w, d_carry0_acc=d_c0)
        d_gi, d_w = torch.zeros(T, E, G * H, device=dev), torch.zeros(H, G * H, device=dev)
        launches["bwd_ovw"] = count(lambda: ops.lstm_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=d_w))
        out.update(d_gi_ovw=d_gi, d_w_h_ovw=d_w)
    form = X.launch_form(cell, T, E, H, dict(env)).name
    return {"name": name, "cell": cell, "shape": [T, E, H], "env": dict(env), "form": form, "launches": launches,
            "outputs": {k: _digest(v) for k, v in out.items()}}


def run_group(env) -> list:
    """The cases of one environment setting, in this process (which must have been started with `env` set)."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    return [run_case(*c) for c in CASES if c[5] == env]


def run_all() -> dict:
    """Runs every case on cuda:0 with the library in this tree: the default setting here, the others in child processes."""
    by_name = {}
    for env in sorted({c[5] for c in CASES}):
        if not env:
            recs = run_group(env)
        else:
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "group.json")
                code = (f"import json, sys; sys.path.insert(0, {HERE!r}); import make_rnn_forms_reference as m;"
                        f"json.dump(m.run_group({env!r}), open({path!r}, 'w')); print('child-ok')")
                r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=ROOT,
                                   env={**os.environ, **dict(env)})
                assert "child-ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
                with open(path) as fh:
                    recs = json.load(fh)
        by_name.update({r["name"]: r for r in recs})
    return {"cases": [by_name[c[0]] for c in CASES]}


if __name__ == "__main__":
    rec = run_all()
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=0)
    print(json.dumps([{"name": c["name"], "form": c["form"], "launches": c["launches"]} for c in rec["cases"]]))
