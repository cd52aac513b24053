"""CPU checks of the K2 exact-data generator (tests/gae_exact_data.py) that tests/test_gae_exact_gpu.py rests on.

1. Every case is exact: coefficients in {0, 1}, small-integer inputs, partial sums and the per-thread fp32 statistics sums of
   every launch form below 2^24.
2. The fp64 oracles (oracle.ppo_oracle.gae, tests/pqn_oracle) give integer results on these cases, and an int64 sequential
   scan written from the affine maps alone agrees with them.
3. The shapes reach every gae_scan_kernel instantiation for each input form, every gae_tma_kernel shape and the TMA
   fallback, through the tuning codes and the default selection (host mirror launch_form)."""
import numpy as np
import pytest

from tests import gae_exact_data as X

ALL_CASES = [(f, T, E) for f in X.FACES for (T, E) in X.SHAPES] + \
            [(f, T, E) for f, shapes in X.DEFAULT_PATH_SHAPES.items() for (T, E) in shapes]


@pytest.mark.parametrize("face,T,E", ALL_CASES, ids=lambda v: str(v))
def test_case_is_exact_and_the_oracles_agree(face, T, E):
    case = X.make_case(face, T, E)   # asserts the exactness invariant
    adv, tgt = X.sequential_scan(case)
    for name, got in (("targets", case.targets), ("advantages", case.adv)):
        if got is None:
            continue
        assert np.array_equal(got, np.round(got)), f"{name}: the oracle gave a non-integer"
        want = tgt if name == "targets" else adv
        np.testing.assert_array_equal(got, want.astype(np.float32), err_msg=f"{face} {T}x{E} {name}: oracle vs int64 scan")
    # the cases are not trivial: env 0 is one chain through every segment (the lambda forms' last step has c = 0), env 1
    # is cut at every step
    assert case.c[:T - 1, 0].all() and not case.c[:, 1].any()
    if X.FACES[face] != "LambdaIn":
        assert case.c[:, 0].all()


@pytest.mark.parametrize("face", X.STANDARDIZING_FACES)
def test_statistics_bound_and_reproduction(face):
    """The per-thread fp32 sums stay exact for every form; `stats` is the fp64 arithmetic of the kernel's finish."""
    worst = 0.0
    for T, E in X.SHAPES:
        case = X.make_case(face, T, E)
        sq, _ = X.stats_bound(case)
        worst = max(worst, sq / X.UNIT_LIMIT)
        st = X.stats(case.adv)
        a = case.adv.astype(np.float64)
        mean = a.mean()
        np.testing.assert_allclose(st, [mean, 1.0 / np.sqrt((a * a).mean() - mean * mean + 1e-5)], rtol=1e-6)
        z = X.standardized(case.adv, st)
        assert z.dtype == np.float32
        np.testing.assert_allclose(z, (a - mean) * st[1], rtol=1e-5, atol=1e-5)
    print(f"{face}: largest per-thread sum of squares {worst:.3f} of 2^24")
    assert worst < 1.0


def test_host_mirror_matches_launch_gae():
    f = lambda face, code, E, **k: X.launch_form(face, code, E, **k).name
    # default selection by E
    assert [f("gae_ppo", 0, E) for E in (8, 2112, 2116, 8448, 32768, 32772, 65536, 262144, 262148)] == [
        "scan<4,2,4,1>", "scan<4,4,4,1>", "scan<4,4,4,1>", "scan<4,8,4,1>", "tma<32,128>", "scan<4,8,4,1>", "tma<64,64>",
        "tma<64,64>", "scan<4,16,4,2>"]
    assert [f("gae_generic", 0, E) for E in (32768, 262140, 262144)] == ["scan<4,8,4,1>", "scan<4,8,4,1>", "scan<4,16,4,2>"]
    assert f("gae_ppo", 0, 37) == f("gae_ppo", 416, 48, vec4=False) == f("q_lambda", 500, 64, vec4=False) == "scan<1,16,4,1>"
    # forced codes; the 5xx codes fall back to the default selection where TMA declines
    assert [f("gae_ppo", c, 1024) for c in (2, 4, 8, 416, 500, 501)] == [
        "scan<4,2,4,1>", "scan<4,4,4,1>", "scan<4,8,4,1>", "scan<4,16,4,2>", "tma<32,128>", "tma<64,64>"]
    assert [f("gae_ppo", c, 1028) for c in (500, 501)] == ["scan<4,2,4,1>"] * 2
    assert f("gae_ppo", 500, 1024, tma_aligned=False) == "scan<4,2,4,1>"
    assert [f(face, 501, 1024) for face in ("gae_generic", "q_lambda", "lambda_returns")] == ["scan<4,2,4,1>"] * 3
    assert f("gae_ppo", 500, 262148) == f("gae_generic", 501, 262144) == "scan<4,16,4,2>"
    assert [f("gae_generic", c, 262144) for c in (2, 4, 8)] == ["scan<4,2,4,1>", "scan<4,4,4,1>", "scan<4,8,4,1>"]


def test_cases_reach_every_form():
    """Through the tuning codes at SHAPES (and the default selection at DEFAULT_PATH_SHAPES), every input form runs every
    gae_scan_kernel instantiation at more than one segment and at a ragged E, the PPO form every TMA shape, and the TMA
    fallback at E % 16 != 0."""
    reached = {}
    for face in X.FACES:
        for T, E in X.SHAPES:
            for code in X.CODES:
                form = X.launch_form(face, code, E)
                reached.setdefault((X.FACES[face], form), []).append((code, T, E))
        for T, E in X.DEFAULT_PATH_SHAPES.get(face, ()):
            reached.setdefault((X.FACES[face], X.launch_form(face, 0, E)), []).append((0, T, E))
    envs = lambda fm: fm.a * fm.b
    for In in ("PpoIn", "GenericIn", "LambdaIn"):
        for fm in X.SCAN_FORMS:
            runs = reached.get((In, fm), [])
            assert runs, f"{In} never runs {fm.name}"
            assert any(T > 32 * fm.kL for _, T, _ in runs), f"{In} {fm.name}: never more than one segment"
            assert any(T % (32 * fm.kL) for _, T, _ in runs), f"{In} {fm.name}: never a ragged last segment"
            assert any(E % envs(fm) for _, _, E in runs), f"{In} {fm.name}: never a ragged last block"
            assert any(E % envs(fm) == 0 for _, _, E in runs) or fm.a == 1, f"{In} {fm.name}: never a full last block"
    for fm in X.TMA_FORMS:
        runs = reached.get(("PpoIn", fm), [])
        assert any(E % fm.a and T > fm.b and T % fm.b for _, T, E in runs), f"{fm.name}: never ragged in both E and T"
        assert any(-(-E // fm.a) > X.NUM_SMS for _, _, E in runs), f"{fm.name}: never several tiles per block"
    # the fallback: a 5xx code (or the default at E >= 32768) whose TMA declines because E % 16 != 0
    assert any(X.launch_form("gae_ppo", c, E).kind == "scan" and E % 4 == 0 and E % 16 for c in (500, 501)
               for _, E in X.SHAPES)
    assert X.launch_form("gae_ppo", 0, 32772).name == "scan<4,8,4,1>" and X.launch_form("gae_ppo", 0, 262148).name == "scan<4,16,4,2>"
