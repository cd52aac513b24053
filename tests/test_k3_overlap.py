"""K3a and K3b keep an MMA group in flight while they do other work (CPU: compile stx_tc_ppo.cu and read the SASS).

K3a issues both halves of its first GEMM before it waits for the first (`WARPGROUP.DEPBAR.LE gsb0, 0x1`) and gathers the next
tile's rows with cp.async (`LDGSTS`) meanwhile.  K3b's consumers wait for chunk k - 1 only, with chunk k in flight.  Both
must do so without local memory beyond K3a's one parked profiling clock."""
import re
import subprocess

import pytest

from stoix_b200 import build
from tests.test_wgmma_pipeline import _sass, _tool

K3A, K3B = "tc_ppo_fwd_bwd_kernel", "tc_dw_kernel"


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    if _tool("cuobjdump") is None:
        pytest.skip("cuobjdump not found")
    obj = tmp_path_factory.mktemp("k3_overlap") / "stx_tc_ppo.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", str(build.CSRC / "stx_tc_ppo.cu"), "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stderr, obj


@pytest.mark.parametrize("kernel", [K3A, K3B])
def test_waits_with_one_group_in_flight(compiled, kernel):
    sass = _sass(compiled[1], kernel)
    assert any(re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x1\b", ln) for ln in sass), f"{kernel}: every wgmma wait drains all groups"


def test_k3a_gathers_with_cp_async(compiled):
    sass = _sass(compiled[1], K3A)
    assert any(re.search(r"\bLDGSTS\b", ln) for ln in sass), "K3a: no cp.async (LDGSTS) in the tile gather"


def test_k3a_local_memory_is_the_parked_clock_only(compiled):
    sass = _sass(compiled[1], K3A)
    local = [ln.strip() for ln in sass if re.search(r"\b(LDL|STL)\b", ln)]
    assert len(local) <= 2, f"K3a: {len(local)} local-memory accesses:\n" + "\n".join(local[:8])


def test_k3b_does_not_spill(compiled):
    log = compiled[0].splitlines()
    props = [i for i, ln in enumerate(log) if "Function properties for" in ln and K3B in ln]
    assert len(props) == 1, f"{K3B}: {len(props)} entries in the ptxas report"
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log[props[0] + 1])
    assert m and m.groups() == ("0", "0"), f"{K3B}: {log[props[0] + 1].strip()}"
