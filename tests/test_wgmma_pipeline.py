"""The wgmma kernels keep their MMAs asynchronous: no calls and no local-memory arrays (CPU: compile and read the SASS).

A call anywhere in a kernel (printf, the library slow path of a division or sqrtf) makes ptxas serialise every wgmma in it
(warning C7510): each MMA then waits for the previous one to finish instead of queueing behind it.  A dynamically indexed
register array lands in local memory.  This test compiles the tensor-core sources with the library's flags and checks, per
kernel, that neither has crept back."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from stoix_b200 import build

KERNELS = {  # source -> kernels that run wgmma
    "stx_tc_ppo.cu": ["tc_ppo_fwd_bwd_kernel", "tc_dw_kernel"],
    "stx_tc_mlp.cu": ["tc_mlp_fwd_kernel"],
    "stx_tc_rollout.cu": ["tc_rollout_kernel"],
}


def _tool(name):
    nvcc = Path(build._nvcc())
    path = nvcc.parent / name
    return str(path) if path.exists() else shutil.which(name)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    if _tool("cuobjdump") is None:
        pytest.skip("cuobjdump not found")
    out = tmp_path_factory.mktemp("wgmma")
    res = {}
    for src in KERNELS:
        obj = out / (Path(src).stem + ".o")
        r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", str(build.CSRC / src), "-o", str(obj)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        res[src] = (r.stderr, obj)
    return res


def _sass(obj, kernel):
    listing = subprocess.run([_tool("cuobjdump"), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", listing)
    mine = [f for f in funcs[1:] if re.match(rf"\S*{kernel}\S*\n", f)]
    assert len(mine) == 1, f"{kernel}: {len(mine)} functions in the SASS listing"
    return [ln for ln in mine[0].splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", ln)]


@pytest.mark.parametrize("src", sorted(KERNELS))
def test_no_serialised_wgmma(compiled, src):
    log, _ = compiled[src]
    assert "C7510" not in log, f"{src}: ptxas serialises wgmma:\n" + "\n".join(ln for ln in log.splitlines() if "C7510" in ln)


@pytest.mark.parametrize("src,kernel", [(s, k) for s, ks in sorted(KERNELS.items()) for k in ks])
def test_kernel_has_no_call_and_pipelines_its_mma(compiled, src, kernel):
    sass = _sass(compiled[src][1], kernel)
    calls = [ln for ln in sass if re.search(r"\bCALL\b", ln)]
    assert not calls, f"{kernel}: {len(calls)} calls, e.g. {calls[0].strip()}"
    n_mma = sum("HGMMA" in ln for ln in sass)
    n_wait = sum("WARPGROUP.DEPBAR" in ln for ln in sass)
    assert n_mma > 0 and n_wait < n_mma, f"{kernel}: {n_wait} warpgroup waits for {n_mma} HGMMA (one wait per MMA: serialised)"


def test_k3a_keeps_its_bias_gradient_butterfly_in_registers(compiled):
    # K3a runs at the full register file (255 registers) without local memory.  The colsum_half butterfly in local memory was
    # ~250 accesses per thread and tile; one L2 policy kept live across the tile loop spills too (hence one per store site).
    sass = _sass(compiled["stx_tc_ppo.cu"][1], "tc_ppo_fwd_bwd_kernel")
    local = [ln.strip() for ln in sass if re.search(r"\b(LDL|STL)\b", ln)]
    assert not local, f"K3a: {len(local)} local-memory accesses:\n" + "\n".join(local[:8])
