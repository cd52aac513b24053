// K1 (bf16 path): fused 3-layer MLP forward on Hopper tensor cores (wgmma).
//
// Reference semantics: FeedForwardActor / FeedForwardCritic.apply with an MLPTorso[256,256] and a Dense
// head (stoix/networks/base.py:18-59, torso.py:24-33, heads.py:36,134):  out = (relu(relu(x W0 + b0) W1 +
// b1)) W2 + b2.  The reference runs three XLA GEMMs + fusions per apply; here ONE persistent kernel keeps
// all weights of the network resident in shared memory (W0 32 KB + W1 128 KB + W2 8 KB, bf16) and chains
// the three GEMMs of a 64-row tile through registers:
//
//   TMA(X tile, 128B swizzle) -> smem --wgmma SS--> acc (fp32 regs) --+b0, relu, bf16--> A1 (regs)
//   --wgmma RS (A from registers)--> acc --epilogue--> A2 --RS--> head --> +b2 -> HBM
//
// so hidden activations never leave the SM (SURVEY.md 7 "Keeping activations out of HBM").
// Two warpgroups per CTA, each running its own sequence of 64-row tiles (one TMA X ring of 2 stages per warpgroup), so
// the epilogue math of one warpgroup overlaps the MMAs of the other.  256-wide layers run as two N=128 halves to keep
// the accumulator at 64 registers per thread.  Weight images: stx_tc_ptx.cuh.
// Shapes: hidden = [256,256] exactly, input dim D <= 64 (multiple of 8; zero-filled by TMA), head <= 16.
#include <cuda.h>

#include "stx_common.cuh"
#include "stx_tc_ptx.cuh"

namespace stx {
namespace tc {

constexpr int kTileM = 64;
constexpr int kH = 256;
constexpr int kWG = 2;
constexpr int kThreads = 128 * kWG;

// shared-memory map (bytes from a 1024-aligned base): weight images, then per warpgroup 2 X stages of 8 KB
constexpr uint32_t kOffX = kImgWBytes;
constexpr uint32_t kOffBias = kOffX + kWG * 2 * 8192;  // b0[256] b1[256] b2[16]
constexpr uint32_t kOffBar = kOffBias + (256 + 256 + 16) * 4;
constexpr uint32_t kSmemBytes = kOffBar + 64 + 1024;  // + alignment slack

struct FwdParams {
  const __nv_bfloat16* w2;  // [256 x A] row-major (bf16 shadow arena)
  const float *b0, *b1, *b2;
  float* out;               // [M x A]
  float* dbg_h1;            // optional [M x 256] post-activation of layer 0 (bring-up / tests)
  float* dbg_h2;            // optional [M x 256]
  int64_t M;
  int A;
  int num_tiles;
  const int32_t* dev_rows;  // optional: the row count is read from the device (M is then the capacity of x)
};

__device__ __forceinline__ void store_dbg(float* dbg, const uint32_t (&a)[64], int64_t row, int64_t M, int lane) {
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int64_t rr = row + 8 * (i & 1);
    if (rr < M) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&a[i]);
      *reinterpret_cast<float2*>(dbg + rr * kH + 8 * (i >> 1) + 2 * (lane & 3)) = make_float2(__bfloat162float(v.x), __bfloat162float(v.y));
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1)
    tc_mlp_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW0,
                      const __grid_constant__ CUtensorMap tmW1, const FwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  // align by OFFSET (not through an integer cast) so that the compiler keeps the shared address space (LDS/STS)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  float* s_b0 = reinterpret_cast<float*>(smem + kOffBias);
  float* s_b1 = s_b0 + 256;
  float* s_b2 = s_b1 + 256;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* w_full = bars;
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, warp = t >> 5, lane = threadIdx.x & 31;
  uint64_t* x_full = bars + 1 + 2 * wg;  // [2] per warpgroup

  int64_t M = p.M;
  int num_tiles = p.num_tiles;
  if (p.dev_rows != nullptr) {  // a row count known only on the device: CTAs without a tile leave before loading weights
    M = *p.dev_rows;
    num_tiles = (int)((M + kTileM - 1) / kTileM);
    if ((int)blockIdx.x * kWG >= num_tiles) return;
  }

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    for (int i = 0; i < 2 * kWG; ++i) mbar_init(&bars[1 + i], 1);
    fence_barrier_init();
    tma_prefetch_desc(&tmX);
    mbar_arrive_expect_tx(w_full, 32768 + 131072);
    for (int j = 0; j < 4; ++j) tma_load_2d(smem + kImgW0 + j * 8192, &tmW0, w_full, j * 64, 0);
    for (int j = 0; j < 4; ++j) tma_load_2d(smem + kImgW1 + j * 32768, &tmW1, w_full, j * 64, 0);
  }
  stage_w2_bias(smem, p.w2, p.b0, p.b1, p.b2, p.A, s_b0, s_b1, s_b2);
  fence_async_proxy();  // generic-proxy smem writes -> visible to the tensor-core (async) proxy
  __syncthreads();

  const int n_wg = (int)gridDim.x * kWG, g = (int)blockIdx.x * kWG + wg;
  const int my_tiles = g < num_tiles ? (num_tiles - g + n_wg - 1) / n_wg : 0;
  uint8_t* xs = smem + kOffX + wg * 16384;
  if (t == 0 && my_tiles > 0) {
    mbar_arrive_expect_tx(&x_full[0], 8192);
    tma_load_2d(xs, &tmX, &x_full[0], 0, g * kTileM);
  }
  mbar_wait(w_full, 0, 1);
  for (int it = 0; it < my_tiles; ++it) {
    const int s = it & 1, tile = g + it * n_wg;
    wg_sync(1 + wg);  // every warp of this warpgroup is done with stage s ^ 1 (tile it - 1)
    if (t == 0 && it + 1 < my_tiles) {
      mbar_arrive_expect_tx(&x_full[s ^ 1], 8192);
      tma_load_2d(xs + (s ^ 1) * 8192, &tmX, &x_full[s ^ 1], 0, (tile + n_wg) * kTileM);
    }
    mbar_wait(&x_full[s], (it >> 1) & 1, 2);
    const int64_t row = (int64_t)tile * kTileM + warp * 16 + (lane >> 2);
    float acc[64];
    uint32_t a1[64], a2[64];
    wg_zero(acc);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_x_w0(acc, smem_u32(xs + s * 8192), sbase, h);
      epi_bias_relu(acc, s_b0, h, a1, lane);
    }
    if (p.dbg_h1 != nullptr) store_dbg(p.dbg_h1, a1, row, M, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_a_w1(acc, a1, sbase, h);
      epi_bias_relu(acc, s_b1, h, a2, lane);
    }
    if (p.dbg_h2 != nullptr) store_dbg(p.dbg_h2, a2, row, M, lane);
    float z[8];
    wg_zero(z);
    gemm_a_w2(z, a2, sbase);
#pragma unroll
    for (int i = 0; i < 8; ++i) {  // z[i]: row + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane % 4) + (i & 1)
      const int64_t rr = row + 8 * ((i >> 1) & 1);
      const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      if (rr < M && col < p.A) p.out[rr * p.A + col] = z[i] + s_b2[col];
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}

// 2D bf16 tensor map: `rows` x `cols` with row pitch `pitch_elems`; box = box_rows x box_cols
static int make_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows,
                       uint32_t box_cols, CUtensorMapSwizzle sw) {
  EncodeTiledFn enc = get_encode();
  STX_REQUIRE(enc != nullptr, STX_E_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  STX_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (pitch_elems * 2) % 16 == 0, STX_E_ALIGN,
              "TMA source must be 16-byte aligned with a 16-byte multiple row pitch (base %p pitch %llu elems)", base,
              (unsigned long long)pitch_elems);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  STX_REQUIRE(r == CUDA_SUCCESS, STX_E_ARG, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return STX_OK;
}

int make_map_2d_pub(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows,
                    uint32_t box_cols) {
  return make_map_2d(m, base, rows, cols, pitch_elems, box_rows, box_cols, CU_TENSOR_MAP_SWIZZLE_128B);
}

// Tiled activation matrix [tiles*128 rows x 8*colgroups] (layout of stx_tc_ppo.cu::tiled_ptr) seen as a 2D
// array of 8-byte words: inner = the 2 KB (128 rows x 16 B) block of one (tile, column group), outer =
// tile*colgroups + group.  Box = 64 rows (128 words) x box_cg column groups, no swizzle.
int make_map_tiled(CUtensorMap* m, const void* base, uint64_t tiles, uint32_t colgroups, uint32_t box_cg) {
  EncodeTiledFn enc = get_encode();
  STX_REQUIRE(enc != nullptr, STX_E_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  STX_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, STX_E_ALIGN, "TMA source must be 16-byte aligned");
  cuuint64_t dims[2] = {256, tiles * colgroups};
  cuuint64_t strides[1] = {2048};
  cuuint32_t box[2] = {128, box_cg};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  STX_REQUIRE(r == CUDA_SUCCESS, STX_E_ARG, "cuTensorMapEncodeTiled (tiled activations) failed with CUresult %d", (int)r);
  return STX_OK;
}

static int g_forward_ctas = 0;  // stx_tc_set_forward_ctas: grid cap of the persistent forward kernel (0 = all SMs)

static bool tc_shape_ok(const StxMlp* m) {
  return m->n_layers == 3 && m->sizes[1] == kH && m->sizes[2] == kH && m->sizes[0] <= 64 && m->sizes[0] % 8 == 0 &&
         m->sizes[3] >= 1 && m->sizes[3] <= 16 && m->activation == STX_ACT_RELU && !m->use_layer_norm;
}

int tc_forward_impl(const StxMlp* m, const void* x, int64_t ldx, int64_t M, float* out, float* dbg_h1, float* dbg_h2,
                    cudaStream_t st, const int32_t* dev_rows = nullptr, int max_ctas = 0) {
  STX_REQUIRE(tc_shape_ok(m), STX_E_SHAPE,
              "STX_PREC_BF16 MLP kernels need a relu torso without LayerNorm and sizes [D<=64 (mult of 8), 256, 256, head<=16]; got %d layers [%d,%d,%d,%d]",
              m->n_layers, m->sizes[0], m->sizes[1], m->sizes[2], m->sizes[3]);
  STX_REQUIRE(m->params_bf16 != nullptr, STX_E_ARG, "STX_PREC_BF16 needs StxMlp.params_bf16 (bf16 shadow of the arena)");
  const int D = m->sizes[0], A = m->sizes[3];
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(m->params_bf16);
  const int64_t off_w1 = (int64_t)D * kH + kH, off_w2 = off_w1 + (int64_t)kH * kH + kH;
  CUtensorMap tmX, tmW0, tmW1;
  if (int rc = make_map_2d(&tmX, x, (uint64_t)M, (uint64_t)D, (uint64_t)ldx, kTileM, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return rc;
  if (int rc = make_map_2d(&tmW0, w, (uint64_t)D, kH, kH, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return rc;
  if (int rc = make_map_2d(&tmW1, w + off_w1, kH, kH, kH, 256, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return rc;
  FwdParams p{};
  p.w2 = w + off_w2;
  p.b0 = m->params + (int64_t)D * kH;
  p.b1 = m->params + off_w1 + (int64_t)kH * kH;
  p.b2 = m->params + off_w2 + (int64_t)kH * A;
  p.out = out, p.dbg_h1 = dbg_h1, p.dbg_h2 = dbg_h2, p.M = M, p.A = A;
  p.num_tiles = (int)((M + kTileM - 1) / kTileM);
  p.dev_rows = dev_rows;
  STX_CUDA_OK(opt_in_smem<tc_mlp_fwd_kernel>(kSmemBytes));
  if (int rc = use_trap_record(st)) return rc;
  int cap = (g_forward_ctas > 0 && g_forward_ctas < kNumSMs) ? g_forward_ctas : kNumSMs;
  if (max_ctas > 0 && max_ctas < cap) cap = max_ctas;
  const int want = (p.num_tiles + kWG - 1) / kWG;
  const int grid = want < cap ? want : cap;
  tc_mlp_fwd_kernel<<<grid, kThreads, kSmemBytes, st>>>(tmX, tmW0, tmW1, p);
  STX_LAUNCH_OK();
  return STX_OK;
}

// ---- the rollout's critic values, one forward per observation -----------------------------------------------------
// value[t] = critic(obs[t]) and bootstrap_value[t] = critic(next_obs[t]) (ff_ppo.py:99, 113-116).  next_obs[t] equals
// obs[t + 1] wherever the episode did not end at step t, so one forward over obs[0..T] serves both, and only the rows
// where an episode ended (is_terminal: obs[t + 1] is then the reset observation) are evaluated again on next_obs.  The
// forward is row-independent (each output row depends on its own input row and the weights only, summed in a fixed
// order), so every value has the bits of the two full passes.

// Rows with is_terminal set: slot[r] = their position in the compacted list, their next_obs rows copied to xe[slot].
// The slot order depends on the block schedule; the values do not.
__global__ void ended_rows_kernel(const uint8_t* __restrict__ is_terminal, const uint4* __restrict__ next_obs, int64_t n, int row_chunks,
                                  int32_t* __restrict__ slot, uint4* __restrict__ xe, int32_t* __restrict__ count) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const bool ended = r < n && is_terminal[r] != 0;
  const uint32_t ballot = __ballot_sync(0xffffffffu, ended);
  if (ballot == 0u) return;
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0) base = atomicAdd(count, __popc(ballot));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (!ended) return;
  const int k = base + __popc(ballot & ((1u << lane) - 1u));
  slot[r] = k;
  for (int c = 0; c < row_chunks; ++c) xe[(int64_t)k * row_chunks + c] = next_obs[r * row_chunks + c];
}

__global__ void rollout_values_kernel(const float* __restrict__ vals, const uint8_t* __restrict__ is_terminal, const int32_t* __restrict__ slot,
                                      const float* __restrict__ ended_vals, int64_t n, int64_t E, float* __restrict__ value,
                                      float* __restrict__ bootstrap) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= n) return;
  value[r] = vals[r];
  bootstrap[r] = is_terminal[r] != 0 ? ended_vals[slot[r]] : vals[r + E];
}

}  // namespace tc

size_t tc_mlp_forward_workspace_bytes(const StxMlp*, int64_t) { return 256; }

int tc_mlp_forward(const StxMlp* mlp, const void* x, int64_t ldx, const int32_t* row_idx, int64_t M, float* out, void*, size_t,
                   cudaStream_t st) {
  STX_REQUIRE(row_idx == nullptr, STX_E_UNSUPPORTED, "STX_PREC_BF16 stx_mlp_forward does not take a row gather");
  return tc::tc_forward_impl(mlp, x, ldx, M, out, nullptr, nullptr, st);
}

}  // namespace stx

extern "C" void stx_tc_set_forward_ctas(int n) { stx::tc::g_forward_ctas = n; }

// Bring-up / test hook: forward that also returns the bf16-rounded hidden activations.
extern "C" int stx_tc_debug_forward(const StxMlp* mlp, const void* x, int64_t ldx, int64_t M, float* out, float* h1, float* h2,
                                    void* stream) {
  return stx::tc::tc_forward_impl(mlp, x, ldx, M, out, h1, h2, (cudaStream_t)stream);
}

// Workspace of stx_tc_rollout_values: vals ((T+1) E f32), ended values (T E f32), slots (T E i32), the count, then the
// compacted next_obs rows (T E x D bf16), each part 256-byte aligned.
static size_t rv_align(size_t b) { return (b + 255) & ~(size_t)255; }
extern "C" size_t stx_tc_rollout_values_workspace_bytes(int T, int64_t E, int D) {
  const size_t n = (size_t)T * (size_t)E;
  return rv_align((n + E) * 4) + rv_align(n * 4) + rv_align(n * 4) + 256 + rv_align(n * (size_t)D * 2);
}

extern "C" int stx_tc_rollout_values(const StxMlp* critic, const void* obs, const void* next_obs, const uint8_t* is_terminal, int T,
                                     int64_t E, float* value, float* bootstrap_value, void* ws, size_t ws_bytes, void* stream) {
  using namespace stx;
  STX_REQUIRE(critic && obs && next_obs && is_terminal && value && bootstrap_value && ws, STX_E_ARG, "stx_tc_rollout_values: null pointer");
  STX_REQUIRE(T > 0 && E > 0 && (int64_t)(T + 1) * E < (1ll << 31), STX_E_SHAPE, "stx_tc_rollout_values: T=%d E=%lld", T, (long long)E);
  STX_REQUIRE(critic->sizes[critic->n_layers] == 1, STX_E_SHAPE, "stx_tc_rollout_values: the critic must have one output");
  const int D = critic->sizes[0];
  STX_REQUIRE(D % 8 == 0, STX_E_SHAPE, "stx_tc_rollout_values: D=%d must be a multiple of 8", D);
  STX_REQUIRE(ws_bytes >= stx_tc_rollout_values_workspace_bytes(T, E, D), STX_E_ARG, "stx_tc_rollout_values: workspace too small");
  const cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = (int64_t)T * E;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  float* vals = reinterpret_cast<float*>(w);
  w += rv_align((size_t)(n + E) * 4);
  float* ended_vals = reinterpret_cast<float*>(w);
  w += rv_align((size_t)n * 4);
  int32_t* slot = reinterpret_cast<int32_t*>(w);
  w += rv_align((size_t)n * 4);
  int32_t* count = reinterpret_cast<int32_t*>(w);
  w += 256;
  void* xe = w;
  STX_CUDA_OK(cudaMemsetAsync(count, 0, sizeof(int32_t), st));
  const unsigned grid = (unsigned)((n + 255) / 256);
  tc::ended_rows_kernel<<<grid, 256, 0, st>>>(is_terminal, reinterpret_cast<const uint4*>(next_obs), n, D / 8, slot,
                                              reinterpret_cast<uint4*>(xe), count);
  STX_LAUNCH_OK();
  if (int rc = tc::tc_forward_impl(critic, obs, D, n + E, vals, nullptr, nullptr, st)) return rc;
  // ~0.7 % of the rows at the benchmark's termination rates: a few dozen tiles, one per warpgroup
  if (int rc = tc::tc_forward_impl(critic, xe, D, n, ended_vals, nullptr, nullptr, st, count, 48)) return rc;
  tc::rollout_values_kernel<<<grid, 256, 0, st>>>(vals, is_terminal, slot, ended_vals, n, E, value, bootstrap_value);
  STX_LAUNCH_OK();
  return STX_OK;
}
