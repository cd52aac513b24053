"""CPU checks of the fp32 exact-data generator (tests/simt_exact_data.py) that tests/test_simt_mlp_gpu.py rests on.

1. Every case the GPU file runs is exact: each GEMM, split, reduction and accumulation of the fp32 path stays below 2^24
   grid units, so any summation order gives the oracle's bits.
2. The cases reach every tiling and weight-gradient split path of launch_gemm / pick_splits (mirrored on the host).
3. On that data an exact comparison sees faults confined to a small part of the gradient arena; the tolerance of the
   existing fp32 minibatch test (_assert_grads_close) is reported next to each, for comparison."""
import numpy as np
import pytest

from tests import simt_exact_data as S


@pytest.mark.parametrize("case", S.CASES, ids=lambda c: c.name)
def test_case_data_is_exact(case):
    worst = S.check_exact(S.make_problem(case))
    print(f"{case.name} {case.sizes} M={case.M}: " + ", ".join(f"{k} {v:.2g}" for k, v in worst.items()))


def _plans():
    return {c.name: S.launch_plan(c.sizes, c.M) for c in S.CASES}


def test_cases_cover_every_tiling_and_split_path():
    plans = _plans()
    every = [(name, l) for name, p in plans.items() for l in p]
    for name, p in plans.items():
        dw = next(l for l in p if l.mode == "DW")
        print(f"{name:9s} splits {dw.splits:3d} x {dw.rows_per_split:4d} rows: "
              + " ".join(f"{l.mode}{l.layer}:{l.tile}" for l in p))
    for mode in ("FWD", "DX", "DW"):
        tiles = {l.tile for _, l in every if l.mode == mode}
        assert {"panel", "64"} <= tiles, f"{mode}: tilings reached {tiles}"
    assert any(l.tile == "panel" and l.mode != "DW" and l.K > 256 for _, l in every), "panel FWD/DX with K > 256"
    assert any(l.tile == "panel" and l.mode == "DW" and l.rows_per_split > 256 for _, l in every), "panel DW, > 256 rows per split"
    fwd64 = {(l.M, l.tile) for _, l in every if l.mode == "FWD" and l.N == 64}
    assert (8384, "panel") in fwd64 and (8385, "64") in fwd64, "the 131 / 132 CTA switch at N = 64"
    assert any(l.mode == "FWD" and l.N == 1 and l.tile == "64" for _, l in every), "an N = 1 head on the 64x64 kernel"
    splits = {l.splits for _, l in every if l.mode == "DW"}
    assert 1 in splits and 128 in splits, splits
    assert any(l.mode == "DW" and l.tile == "64" and l.splits == 128 for _, l in every)
    assert any(l.mode == "DW" and l.tile == "panel" and l.splits == 128 for _, l in every)
    assert any(l.mode == "DW" and l.splits > 1 and l.M % l.rows_per_split for _, l in every), "a ragged last split"
    for mode in ("FWD", "DX", "DW"):
        for tile in ("panel", "64"):
            ls = [l for _, l in every if l.mode == mode and l.tile == tile]
            assert any(l.K % 16 for l in ls) and any(l.N % 16 for l in ls), f"{mode} {tile}: K and N not multiples of 16"
    assert {1, 5} <= {c.M for c in S.CASES}
    assert any(c.gathered and c.ldx > c.sizes[0] for c in S.CASES)


def test_host_mirror_matches_known_splits():
    """pick_splits at the shapes its comment in stx_mlp.cu names."""
    assert S.pick_splits((64, 256, 256, 8), 32768) == 66
    assert S.pick_splits((32, 128, 384), 32768) == 128
    assert S.pick_splits((64, 256, 256, 8), 300) == 1
    assert S.pick_splits((64, 256, 256, 8), 4096) == 16


def _first_active_row(ch, layer, start):
    act = (np.abs(ch.inputs[layer]).sum(1) > 0) & (np.abs(ch.d[layer]).sum(1) > 0)
    return start + int(np.argmax(act[start:]))


def test_exact_comparison_sees_small_faults():
    """Each fault below changes at least one gradient or output element, so the exact comparison of the GPU tests fails
    on it.  Whether the tolerance of tests/test_kernels_gpu.py::_assert_grads_close would have accepted the same fault is
    printed, not asserted (that is a property of the older test, not of the kernels)."""
    from tests.test_kernels_gpu import _assert_grads_close

    pb = S.make_problem(S.CASE_BY_NAME["bench"])
    M = pb.case.M
    ch = S.chain(pb.net, pb.x, pb.d_out)
    ref = S.layer_grads(pb.net, ch)
    splits = S.pick_splits(pb.case.sizes, M)
    rps = -(-M // splits)
    all_rows = np.arange(M)
    r = _first_active_row(ch, 1, 777)
    z0 = 5 * rps + 16 * 3                                   # one BK = 16 step of the 64x64 DW kernel inside split 5
    faults = {
        "one row dropped (dW1, db1)": dict(rows={1: np.delete(all_rows, r)}, bias_rows={1: np.delete(all_rows, r)}),
        "one 16-row K chunk dropped (dW1)": dict(rows={1: np.r_[all_rows[:z0], all_rows[z0 + 16:]]}),
        "one DW split dropped (dW2, db2)": dict(rows={2: np.r_[all_rows[:7 * rps], all_rows[8 * rps:]]},
                                                bias_rows={2: np.r_[all_rows[:7 * rps], all_rows[8 * rps:]]}),
        "one bias term lost (db1)": dict(bias_rows={1: np.delete(all_rows, r)}),
    }
    results = {}
    for label, kw in faults.items():
        results[label] = S.GRAD_WEIGHT * S.layer_grads(pb.net, ch, **kw), S.GRAD_WEIGHT * ref
    # gather index off by one for one batch row (a gathered case: x read through row_idx)
    pg = S.make_problem(S.CASE_BY_NAME["ragged"])
    chg = S.chain(pg.net, pg.x, pg.d_out)
    m = _first_active_row(chg, 0, 100)
    bad = S.Problem(pg.case, pg.net, pg.xbuf, pg.row_idx.copy(), pg.d_out, pg.grad0)
    bad.row_idx[m] = (bad.row_idx[m] + 1) % pg.case.B
    chb = S.chain(bad.net, bad.x, bad.d_out)
    assert not np.array_equal(chb.out.astype(np.float32), chg.out.astype(np.float32)), "off-by-one gather: output unchanged"
    results["gather index off by one"] = S.GRAD_WEIGHT * S.layer_grads(bad.net, chb), S.GRAD_WEIGHT * S.layer_grads(pg.net, chg)
    for label, (g, gref) in results.items():
        g32, r32 = g.astype(np.float32), gref.astype(np.float32)
        n_diff = int((g32 != r32).sum())
        mb = pg.case.M if label.startswith("gather") else M
        try:
            _assert_grads_close(g, gref, mb)
            verdict = "accepted"
        except AssertionError:
            verdict = "rejected"
        rel = np.linalg.norm(g - gref) / np.linalg.norm(gref)
        print(f"{label:34s} entries that differ {n_diff:6d}, norm-wise {rel:.1e}; _assert_grads_close: {verdict}")
        assert n_diff > 0, f"{label}: the exact comparison must see the fault"
