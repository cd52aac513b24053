"""The grid-capped kernels whose blocks loop: each kernel's grid cap, as its launch code writes it, and the shapes that drive every
such kernel past one wave of its grid.

Each of these kernels caps its grid at a small multiple of the SM count; past the cap every block runs a grid-stride loop and
carries its state (running maxima, min / max columns, per-warp KL accumulators, fp64 partials) from one trip to the next.  A
`Loop` names a kernel, the source lines of its cap, and the rows one block covers per trip; `trips` gives the grid and every
block's trip count at a shape.  tests/test_grid_waves.py checks on any machine that the cap lines are still in the sources and that
every shape below loops with a ragged last trip; tests/test_grid_stride_gpu.py runs the kernels at these shapes against the fp64
oracles.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Tuple

CSRC = Path(__file__).resolve().parents[1] / "stoix_b200" / "csrc"
NUM_SMS = 132   # kNumSMs of stx_common.cuh: the SMs of an H100 SXM
SMS_LINE = ("stx_common.cuh", "constexpr int kNumSMs = 132;")


@dataclass(frozen=True)
class Loop:
    """kernel: the __global__ function; source: its file under stoix_b200/csrc; cap_lines: (file, text) pairs that must appear
    verbatim, the cap and whatever sizes a block's trip; cap: the grid cap in blocks; block_rows: loop items (rows, elements or
    float4 groups, see `unit`) that size the grid, one block's share of a wave; unroll: items per block row per trip (the obs-norm
    accumulate loads 8 rows per thread per trip); shapes: name -> loop items, each past the cap."""

    kernel: str
    source: str
    cap_lines: Tuple[Tuple[str, str], ...]
    cap: int
    block_rows: int
    unit: str
    shapes: Dict[str, int] = field(default_factory=dict)
    unroll: int = 1

    @property
    def wave(self) -> int:
        """Items one trip of the capped grid covers."""
        return self.cap * self.block_rows * self.unroll


def trips(loop: Loop, n: int) -> Tuple[int, List[int]]:
    """(grid, trips of each block) of `loop` over n items, as the launch code sizes the grid and the kernel strides."""
    grid = max(1, min(-(-n // loop.block_rows), loop.cap))
    per_trip = grid * loop.block_rows * loop.unroll
    return grid, [-(-(n - b * loop.block_rows) // per_trip) for b in range(grid)]


def ragged(loop: Loop, n: int) -> bool:
    """The last trip covers less than a full wave of the grid."""
    grid, _ = trips(loop, n)
    return n % (grid * loop.block_rows * loop.unroll) != 0


def obsnorm_rpp(D: int, vec: bool) -> int:
    """Rows per block pass of stats_accumulate_kernel (stx_running_stats_accumulate): 256 threads over D / V lanes per row."""
    L = D // 4 if vec else D
    return max(256 // L, 1)


_VMPO, _MPO, _PPO, _OBS, _SAC = "stx_vmpo.cu", "stx_mpo.cu", "stx_ppo_fp32.cu", "stx_obsnorm.cu", "stx_sac.cu"
_VMPO_STATS_WAVE = 2 * NUM_SMS * 256       # 67,584 rows
_VMPO_ROWS_WAVE = 8 * NUM_SMS * 256        # 270,336 rows
_OBS_ACC = ((_OBS, "if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;"), (_OBS, "constexpr int kUnroll = 8;"),
            (_OBS, "const int rpp = 256 / L > 0 ? 256 / L : 1;"))
_OBS_NORM = ((_OBS, "if (blocks > 16 * kNumSMs) blocks = 16 * kNumSMs;"),)
_FACE = ((_PPO, "const int64_t cap = 2 / Face::kParts * kNumSMs, need = (n + 255) / 256;"),)

VMPO_STATS = Loop("vmpo_stats_kernel", _VMPO,
                  ((_VMPO, "constexpr unsigned kLossGrid = 2 * kNumSMs;"),
                   (_VMPO, "const unsigned grid = (unsigned)std::min<int64_t>((a.N + kThreads - 1) / kThreads, kLossGrid);")),
                  2 * NUM_SMS, 256, "rows",
                  {"bench": 8192 * 32, "three_waves": 3 * _VMPO_STATS_WAVE + 1001, "two_row_waves": 2 * _VMPO_ROWS_WAVE + 77})
VMPO_GRADS = Loop("vmpo_grads_kernel", _VMPO,
                  ((_VMPO, "const unsigned grid_rows = (unsigned)std::min<int64_t>((rows + kThreads - 1) / kThreads, 8 * kNumSMs);"),),
                  8 * NUM_SMS, 256, "rows (max(N, value_rows))", {"two_row_waves": 2 * _VMPO_ROWS_WAVE + 77 + 9})
VMPO_AFTER_STEP = Loop("vmpo_after_step_kernel", _VMPO,
                       ((_VMPO, "const unsigned grid = (unsigned)std::min<int64_t>((n + kThreads - 1) / kThreads, 8 * kNumSMs);"),),
                       8 * NUM_SMS, 256, "params", {"P": 600_001})
MPO_CATEGORICAL = Loop("mpo_categorical_kernel", _MPO,
                       ((_MPO, "constexpr unsigned kLossGrid = 2 * kNumSMs;"),
                        (_MPO, "const unsigned grid = (unsigned)std::min<int64_t>((a.M + kThreads - 1) / kThreads, kLossGrid);")),
                       2 * NUM_SMS, 256, "states", {"M": 2 * _VMPO_STATS_WAVE + 333})
MPO_TANH = Loop("mpo_tanh_kernel", _MPO, MPO_CATEGORICAL.cap_lines, 2 * NUM_SMS, 256, "states", {"M": 2 * _VMPO_STATS_WAVE + 333})
_FACE_N = {"n": 2 * _VMPO_STATS_WAVE + 5}
FACE_ONE_PART = Loop("loss_face_kernel<SurrogateFace<ClipLoss>>, <ValueFace>", _PPO,
                     _FACE + (("stx_ppo_loss.cuh", "static constexpr int kExtraSlot = 3, kFaceParts = 1;"),
                              ("stx_ppo_loss.cuh", "static constexpr int kParts = 1;")),
                     2 * NUM_SMS, 256, "elements", _FACE_N)
FACE_TWO_PARTS = Loop("loss_face_kernel<SurrogateFace<KlPenaltyLoss>>, <SurrogateFace<DpoLoss>>", _PPO,
                      _FACE + (("stx_ppo_loss.cuh", "static constexpr int kExtraSlot = kSlotKl, kFaceParts = 2;"),
                               ("stx_ppo_loss.cuh", "static constexpr int kExtraSlot = -1, kFaceParts = 2;")),
                      NUM_SMS, 256, "elements", _FACE_N)
OBS_ACC_D17 = Loop("stats_accumulate_kernel<1> (D = 17)", _OBS, _OBS_ACC, 4 * NUM_SMS, obsnorm_rpp(17, False), "rows",
                   {"rows": 2 * 4 * NUM_SMS * obsnorm_rpp(17, False) * 8 + 123}, unroll=8)
OBS_ACC_D256 = Loop("stats_accumulate_kernel<4> (D = 256)", _OBS, _OBS_ACC, 4 * NUM_SMS, obsnorm_rpp(256, True), "rows",
                    {"rows": 3 * 4 * NUM_SMS * obsnorm_rpp(256, True) * 8 + 5}, unroll=8)
OBS_ACC_D64_MISALIGNED = Loop("stats_accumulate_kernel<1> (D = 64, x not 16-byte aligned)", _OBS,
                              _OBS_ACC + ((_OBS, "const bool vec = D % 4 == 0 && aligned16(x);"),), 4 * NUM_SMS, obsnorm_rpp(64, False), "rows",
                              {"rows": 2 * 4 * NUM_SMS * obsnorm_rpp(64, False) * 8 + 77}, unroll=8)
OBS_NORM_SCALAR = Loop("obs_normalize_scalar_kernel", _OBS, _OBS_NORM, 16 * NUM_SMS, 256, "elements",
                       {"D17": 70_001 * 17, "D64_misaligned_bf16": 40_000 * 64})
OBS_NORM_VEC = Loop("obs_normalize_kernel", _OBS, _OBS_NORM, 16 * NUM_SMS, 256, "float4 groups", {"D64": 40_000 * 64 // 4})
POLYAK = Loop("polyak_kernel", _SAC, ((_SAC, "if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;"),), 8 * NUM_SMS, 256, "elements",
              {"n": 600_001})

LOOPS = (VMPO_STATS, VMPO_GRADS, VMPO_AFTER_STEP, MPO_CATEGORICAL, MPO_TANH, FACE_ONE_PART, FACE_TWO_PARTS, OBS_ACC_D17, OBS_ACC_D256,
         OBS_ACC_D64_MISALIGNED, OBS_NORM_SCALAR, OBS_NORM_VEC, POLYAK)
