"""The grid caps of tests/grid_waves.py against the kernel sources, and its shapes against those caps: if a cap line changes, or a
cap is raised until a shape fits in one wave, the failing case names the kernel and the shape that no longer loops.  No GPU."""
import pytest

from tests import grid_waves as W

_SOURCES = {}


def _source(name):
    if name not in _SOURCES:
        _SOURCES[name] = (W.CSRC / name).read_text()
    return _SOURCES[name]


def test_sm_count_is_the_one_the_table_assumes():
    assert W.SMS_LINE[1] in _source(W.SMS_LINE[0])


@pytest.mark.parametrize("loop", W.LOOPS, ids=lambda l: l.kernel)
def test_cap_lines_are_in_the_sources(loop):
    assert loop.kernel.split("<")[0].split(" ")[0] in _source(loop.source)
    for name, line in loop.cap_lines:
        assert line in _source(name), f"{loop.kernel}: {name} no longer contains {line!r}"


_CASES = [(loop, name, n) for loop in W.LOOPS for name, n in loop.shapes.items()]


@pytest.mark.parametrize("loop,name,n", _CASES, ids=[f"{l.kernel}-{s}" for l, s, _ in _CASES])
def test_every_shape_loops_with_a_ragged_last_trip(loop, name, n):
    grid, per_block = W.trips(loop, n)
    assert grid == loop.cap, f"{loop.kernel} at {name} = {n} {loop.unit}: grid {grid} below the cap {loop.cap}"
    assert max(per_block) >= 2, f"{loop.kernel} at {name} = {n} {loop.unit} fits in one wave of {loop.wave}"
    assert W.ragged(loop, n), f"{loop.kernel} at {name} = {n} {loop.unit}: a whole number of waves, no ragged last trip"


def test_trips_helper():
    loop = W.Loop("k", "x.cu", (), cap=4, block_rows=8, unit="rows")
    assert W.trips(loop, 1) == (1, [1])
    assert W.trips(loop, 32) == (4, [1, 1, 1, 1])
    assert W.trips(loop, 33) == (4, [2, 1, 1, 1])
    assert W.trips(loop, 72) == (4, [3, 2, 2, 2])
    assert not W.ragged(loop, 64) and W.ragged(loop, 65)
    unrolled = W.Loop("k", "x.cu", (), cap=2, block_rows=3, unit="rows", unroll=8)   # a trip: rows b*3 + (8k + u)*6 + r, u < 8
    assert W.trips(unrolled, 48) == (2, [1, 1]) and W.trips(unrolled, 49) == (2, [2, 1]) and W.trips(unrolled, 52) == (2, [2, 2])
    assert W.VMPO_STATS.wave == 67_584 and W.VMPO_GRADS.wave == 270_336 and W.OBS_ACC_D17.wave == 63_360 and W.OBS_ACC_D256.wave == 16_896
