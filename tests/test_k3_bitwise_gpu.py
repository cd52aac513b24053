"""The bf16 PPO minibatch gradient step (K3a + K3b + reduce) reproduces a recorded reference bit for bit.

The reference (tests/golden/k3_bf16_reference.json, written by tests/golden/make_k3_reference.py) holds SHA-256 hashes of the
whole gradient arena and the metrics at the benchmark shape.  The exact-data tests accept any summation order; this one pins the
rounding, so a kernel change that reorders the sums over rows or partials fails here."""
import importlib.util
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _reference_module():
    spec = importlib.util.spec_from_file_location("make_k3_reference", os.path.join(HERE, "golden", "make_k3_reference.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_k3_gradients_match_the_reference_bit_for_bit():
    mod = _reference_module()
    with open(os.path.join(HERE, "golden", "k3_bf16_reference.json")) as f:
        ref = json.load(f)
    got = mod.run_windows()
    assert got["n_params"] == ref["n_params"]
    for g, r in zip(got["windows"], ref["windows"]):
        what = f"window mb_off={r['mb_off']} mb={r['mb']}"
        gs = np.frombuffer(bytes.fromhex(g["sample_f32_hex"]), dtype=np.float32)
        rs = np.frombuffer(bytes.fromhex(r["sample_f32_hex"]), dtype=np.float32)
        diff = np.flatnonzero(gs.view(np.uint32) != rs.view(np.uint32))
        detail = f"{diff.size} of {rs.size} sampled entries differ, max |diff| {np.abs(gs - rs).max():.3e}"
        assert g["grad_sha256"] == r["grad_sha256"], f"{what}: gradient arena differs from the reference ({detail})"
        assert g["metrics_sha256"] == r["metrics_sha256"], f"{what}: metrics {g['metrics']} != {r['metrics']}"
