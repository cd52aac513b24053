"""Bit-level reference of the bf16 PPO minibatch gradient step (K3a + K3b + reduce) at the benchmark shape.

Seeded NumPy inputs (B = 524288 rows, D = 64, actor head A = 8, a random permutation, weights x 0.05); two mb = 32768 windows and
one mb = 128 window, each computed from a zeroed gradient arena with overwrite=True.  Recorded per window: the SHA-256 of the
gradient-arena bytes and of the six metric floats, plus a seeded sample of 4096 gradient entries for diagnosing a mismatch.

The hashes pin the rounding of every gradient entry, so a change to the order in which the kernels sum rows shows up here even
where the order-insensitive exact-data tests (tests/test_tc_exact_gpu.py) cannot see it.  Generate on an H100 with the build
the reference should describe:

    python tests/golden/make_k3_reference.py tests/golden/k3_bf16_reference.json
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, D, A, H = 524288, 64, 8, 256
WINDOWS = ((0, 32768), (11 * 32768, 32768), (1000 * 128, 128))  # (mb_off, mb)
N_SAMPLE = 4096


def make_inputs(total: int) -> dict:
    rng = np.random.default_rng(20261015)
    adv = rng.standard_normal(B).astype(np.float32)
    return {
        "arena": (rng.standard_normal(total) * 0.05).astype(np.float32),
        "obs": rng.standard_normal((B, D)).astype(np.float32),
        "action": rng.integers(0, A, B).astype(np.int32),
        "log_prob": (-rng.random(B) * 2.0 - 0.5).astype(np.float32),
        "value": rng.standard_normal(B).astype(np.float32),
        "adv": adv,
        "tgt": rng.standard_normal(B).astype(np.float32),
        "adv_stats": np.array([adv.astype(np.float64).mean(), 1.0 / adv.astype(np.float64).std()], dtype=np.float32),
        "perm": rng.permutation(B).astype(np.int32),
    }


def sample_index(total: int) -> np.ndarray:
    """Gradient-arena entries whose values the reference keeps (float32 little-endian, hex) beside the hashes."""
    return np.random.default_rng(7).choice(total, N_SAMPLE, replace=False)


def run_windows() -> dict:
    """Runs the windows on cuda:0 with the library in this tree; returns the record make_k3_reference writes."""
    import torch

    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from stoix_b200 import ops

    dev = torch.device("cuda:0")
    sa, sc = ops.MlpSpec((D, H, H, A)), ops.MlpSpec((D, H, H, 1))
    _, _, total = ops.arena_offsets(sa, sc)
    x = make_inputs(total)
    t = lambda k: torch.from_numpy(x[k]).to(dev)
    arena = t("arena")
    shadow = ops.cast_bf16(arena)
    batch = ops.PpoBatch(t("obs").to(torch.bfloat16), t("action"), t("log_prob"), t("value"), t("adv"), t("tgt"), t("adv_stats"),
                         t("perm"))
    sample = sample_index(total)
    out = []
    for mb_off, mb in WINDOWS:
        ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_BF16, dev)
        grads, metrics = torch.zeros(total, device=dev), torch.zeros(8, device=dev)
        ops.ppo_minibatch_grads(sa, sc, arena, batch, mb_off, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws, ops.STX_PREC_BF16, 1.0,
                                shadow, overwrite=True)
        g, m = grads.cpu().numpy(), metrics[:6].cpu().numpy()
        out.append({"mb_off": mb_off, "mb": mb, "grad_sha256": hashlib.sha256(g.tobytes()).hexdigest(),
                    "metrics_sha256": hashlib.sha256(m.tobytes()).hexdigest(), "metrics": [float(v) for v in m],
                    "sample_f32_hex": g[sample].tobytes().hex()})
    return {"shape": {"B": B, "D": D, "A": A, "H": H}, "n_params": int(total), "windows": out}


if __name__ == "__main__":
    rec = run_windows()
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f)
    print(json.dumps([{k: w[k] for k in ("mb_off", "mb", "grad_sha256", "metrics_sha256")} for w in rec["windows"]], indent=1))
