"""CPU checks of the GRU exact-data generator (tests/rnn_exact_data.py) that tests/test_rnn_exact_gpu.py rests on.

1. Every case the GPU file runs is exact: each sum and element-wise step of every launch form stays below 2^24 grid units
   or is an fp32 value, so any summation order gives the oracle's bits.
2. The cases reach every launch form on both sides of every limit of the host selection (mirrored by launch_form), the E
   and T switches, ragged last tiles and the reset patterns that the kernels treat specially.
3. On that data an exact comparison sees small kernel faults; whether the tolerances of tests/test_rec_gpu.py would have
   accepted each one is printed next to it."""
import numpy as np
import pytest

from tests import rnn_exact_data as X


@pytest.mark.parametrize("case", X.CASES, ids=lambda c: c.name)
def test_case_data_is_exact(case):
    worst = X.check_exact(X.make_problem(case))
    print(f"{case.name} T={case.T} E={case.E} H={case.H}: " + ", ".join(f"{k} {v:.2g}" for k, v in worst.items()))


def test_host_mirror_at_the_shared_memory_limits():
    """The opt-in maximum is 232,448 B; one step above each limit the form changes."""
    assert X.gru_seq_smem(8, 1, 130)[1] == 232448 == X.SMEM_LIMIT and X.gru_seq_smem(8, 1, 131)[1] > X.SMEM_LIMIT
    assert X.gru_cl_smem(188)[1] == 230864 and X.gru_cl_smem(190)[1] > X.SMEM_LIMIT
    assert X.lstm_cl_smem(162)[1] == 231344 and X.lstm_cl_smem(164)[1] > X.SMEM_LIMIT
    f = lambda *a, **k: X.launch_form(*a, **k).name
    assert [f("gru", 4, 5, h) for h in (128, 129, 130, 131)] == ["cluster", "seq<4,2>", "cluster", "per-step"]
    assert [f("gru", 4, 1024, h) for h in (129, 130, 131)] == ["seq<8,1>", "seq<8,1>", "per-step"]
    assert [f("gru", 4, 5, h) for h in (187, 188, 189, 190)] == ["per-step", "cluster", "per-step", "per-step"]
    assert [f("gru", 4, e, 20) for e in (1023, 1024)] == ["cluster", "seq<8,1>"]
    assert [f("gru", t, 5, 20) for t in (3, 4)] == ["per-step", "cluster"]
    assert f("gru", 4, 5, 130, {"STX_GRU_CLUSTER": "0"}) == "seq<4,2>"
    assert f("gru", 4, 5, 20, {"STX_GRU_CLUSTER": "0", "STX_GRU_PERSISTENT": "0"}) == "per-step"
    assert [f("lstm", 4, 5, h) for h in (161, 162, 163, 164)] == ["per-step", "cluster", "per-step", "per-step"]
    assert [f("lstm", t, 5, 20) for t in (3, 4)] == ["per-step", "cluster"]
    assert f("lstm", 4, 5, 20, {"STX_LSTM_CLUSTER": "0"}) == "per-step"


def test_cases_cover_every_form_and_switch():
    rows = []
    for c in X.CASES:
        fm = c.form
        rows.append((c, fm))
        env = " ".join(f"{k}={v}" for k, v in c.env) or "-"
        print(f"{c.name:16s} T={c.T:2d} E={c.E:5d} H={c.H:3d} {env:40s} {fm.name:9s} threads {fm.threads:4d} "
              f"smem fwd {fm.smem_fwd:6d} bwd {fm.smem_bwd:6d} launches fwd {fm.fwd_launches(c.T)}")
    forms = {fm.name for _, fm in rows}
    assert forms == {"cluster", "seq<4,2>", "seq<8,1>", "per-step"}, forms
    hs = lambda name: {c.H for c, fm in rows if fm.name == name}
    assert {188} <= hs("cluster") and {189, 190} <= hs("per-step"), "both sides of the cluster limit"
    assert {129, 130} <= hs("seq<8,1>") and {129, 130} <= hs("seq<4,2>") and 131 in hs("per-step"), "both sides of the persistent limit"
    assert 3 in hs("seq<4,2>") and 187 in hs("per-step")
    big = {name: max(fm.smem_bwd for _, fm in rows if fm.name == name) for name in ("cluster", "seq<4,2>", "seq<8,1>")}
    print("largest dynamic shared memory per form (bwd):", big)
    assert big == {"cluster": 230864, "seq<4,2>": 224128, "seq<8,1>": 232448}
    assert {1, 3, 5, 1023, 1024, 1025} <= {c.E for c in X.CASES}
    assert {1, 3, 4} <= {c.T for c in X.CASES}
    es = lambda name: {c.E for c, fm in rows if fm.name == name}
    assert 1023 in es("cluster") and 1023 in es("seq<4,2>") and {1024, 1025} <= es("seq<8,1>") and {1024, 1025, 2048} <= es("per-step")
    assert any(c.E % 4 for c, fm in rows if fm.name in ("cluster", "seq<4,2>")) and any(c.E % 8 for c, fm in rows if fm.name == "seq<8,1>")
    assert any(c.T >= 4 for c, fm in rows if fm.name == "per-step"), "the per-step form of a sequence the persistent forms would take"
    # reset patterns
    pat = {k: False for k in ("reset at t = 0", "back-to-back resets", "reset on the last step", "row resetting every step", "row never resetting")}
    for c in X.CASES:
        r = X.make_problem(c).reset
        pat["reset at t = 0"] |= bool(r[0].any())
        pat["back-to-back resets"] |= bool((r[1:] & r[:-1]).any())
        pat["reset on the last step"] |= c.T > 1 and bool(r[-1].any())
        pat["row resetting every step"] |= c.T > 1 and bool(r.all(0).any())
        pat["row never resetting"] |= c.T > 1 and bool((~r).all(0).any())
    assert all(pat.values()), pat
    for c in X.LSTM_CASES:
        print(f"lstm {c}: {X.launch_form('lstm', *c).name}")
    lstm = {(c[2], X.launch_form("lstm", *c).name) for c in X.LSTM_CASES}
    assert {(162, "cluster"), (164, "per-step")} <= lstm and any(h % 2 and f == "per-step" for h, f in lstm)


def _tolerance_verdict(bad: X.Reference, ref: X.Reference) -> str:
    """Whether tests/test_rec_gpu.py::_gru_case's tolerances accept `bad` as a kernel result for `ref`."""
    rel = lambda a, b: float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b.astype(np.float64)), 1e-30))
    ok = (np.allclose(bad.h_seq, ref.h_seq, rtol=2e-5, atol=2e-6) and np.allclose(bad.d_gi, ref.d_gi, rtol=1e-4, atol=1e-5)
          and np.allclose(bad.d_h0, ref.d_h0, rtol=1e-4, atol=1e-5) and rel(bad.d_wh, ref.d_wh) < 1e-5 and rel(bad.d_bhn, ref.d_bhn) < 1e-5)
    return "accepted" if ok else "rejected"


def test_exact_comparison_sees_small_faults():
    """Each fault below, applied to the fp64 oracle, changes at least one compared element, so the exact comparison of the
    GPU tests fails on it.  The tile faults hit rows 8..11 (one R = 4 tile, one cluster) at step 2 of an 8-step case."""
    pb = X.make_problem(X.CASE_BY_NAME["cl_t8"])
    ref = X.reference(pb)
    t_e = [(t, e) for t in range(2, pb.case.T) for e in range(2, pb.case.E) if pb.reset[t, e] and not pb.reset[t - 1, e]]
    # the last row of a ragged tile: the first case whose last row has a live d(h0)
    rag = next(X.make_problem(c) for c in X.CASES if c.E % 4 and c.E > 1 and X.chain(X.make_problem(c)).dh0[-1].any())
    at = {"ks_partial_dropped": (2, 8), "stale_peer_h": (2, 8), "stale_peer_inbox": (2, 8), "reset_early": t_e[0]}
    for fault in X.FAULTS:
        p = rag if fault == "ragged_row_dropped_from_dh0" else pb
        good = ref if p is pb else X.reference(p)
        bad = X.reference(p, fault, at.get(fault, (0, 0)))
        diff = {k: int((getattr(bad, k) != getattr(good, k)).sum()) for k in ("h_seq", "d_gi", "d_wh", "d_bhn", "d_h0")}
        print(f"{fault:30s} ({p.case.name}) elements that differ: " + ", ".join(f"{k} {v}" for k, v in diff.items())
              + f"; test_rec_gpu tolerances: {_tolerance_verdict(bad, good)}")
        assert sum(diff.values()) > 0, f"{fault}: the exact comparison must see the fault"
