"""The GRU and LSTM sequence kernels reproduce a recorded reference bit for bit in every launch form, with the same launches.

The reference (tests/golden/rnn_forms_reference.json, written by tests/golden/make_rnn_forms_reference.py) holds SHA-256 hashes
of every output of the forward and backward of each form (cluster, seq<4,2>, seq<8,1>, per-step) on seeded random inputs.
tests/test_rnn_exact_gpu.py accepts any summation order and FMA contraction by design; this one pins them."""
import importlib.util
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _reference_module():
    spec = importlib.util.spec_from_file_location("make_rnn_forms_reference", os.path.join(HERE, "golden", "make_rnn_forms_reference.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_rnn_forms_match_the_reference_bit_for_bit():
    with open(os.path.join(HERE, "golden", "rnn_forms_reference.json")) as f:
        ref = json.load(f)
    got = _reference_module().run_all()
    assert [c["name"] for c in got["cases"]] == [c["name"] for c in ref["cases"]]
    failures = []
    for g, r in zip(got["cases"], ref["cases"]):
        if g["form"] != r["form"]:
            failures.append(f"{r['name']}: reaches {g['form']}, reference {r['form']}")
        if g["launches"] != r["launches"]:
            failures.append(f"{r['name']}: launches {g['launches']}, reference {r['launches']}")
        assert g["outputs"].keys() == r["outputs"].keys(), r["name"]
        for k, ro in r["outputs"].items():
            go = g["outputs"][k]
            if go["sha256"] == ro["sha256"]:
                continue
            gs = np.frombuffer(bytes.fromhex(go["sample_f32_hex"]), dtype=np.float32)
            rs = np.frombuffer(bytes.fromhex(ro["sample_f32_hex"]), dtype=np.float32)
            diff = np.flatnonzero(gs.view(np.uint32) != rs.view(np.uint32))
            failures.append(f"{r['name']} ({r['form']}) {k}: differs from the reference; {diff.size} of {rs.size} sampled values differ"
                            + (f", max |diff| {np.abs(gs[diff] - rs[diff]).max():.3e}" if diff.size else ""))
    assert not failures, "\n".join(failures)
