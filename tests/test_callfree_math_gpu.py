"""The call-free reciprocal and square root of stx_common.cuh return exactly the IEEE bits on every input of their ranges.

They replace 1.0f / x in K3a's softmax and sqrtf in the Box-Muller draw shared by the environment, the fused rollout and the
CPU oracle (oracle/synth_env.py), so a single differing bit would change trajectories and gradients.  The reference is
1.0f / x and sqrtf(x) computed on the same device."""
import struct

import pytest


def _bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fn,lo,hi", [
    (0, 1.0, 16.0),              # reciprocal: the softmax denominator of at most 16 logits, one of them e^0 (2^25 + 1 values)
    (1, 2.0 ** -101, 64.0),      # square root: its stated range up to 64 (normal2 uses (1.1e-7, 33.3])
])
def test_callfree_math_is_bit_exact(fn, lo, hi):
    import torch

    from stoix_b200 import _lib

    lib = _lib.load()
    out = torch.tensor([0, -1], dtype=torch.int64, device="cuda")  # [mismatches, first mismatching pattern]
    _lib.check(lib.stx_debug_callfree_math(fn, _bits(lo), _bits(hi), out.data_ptr(), None), "stx_debug_callfree_math")
    bad, first = out.cpu().tolist()
    assert bad == 0, f"{bad} inputs differ from the IEEE result, the first at bits 0x{first & 0xFFFFFFFF:08x}"
