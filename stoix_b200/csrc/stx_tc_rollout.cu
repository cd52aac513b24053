// Fused persistent rollout for the synthetic Box environment (bf16 / wgmma path).
//
// Reference semantics: the T-step lax.scan of _env_step (stoix/systems/ppo/anakin/ff_ppo.py:81-140) for
// the actor side: logits = actor(obs_t) -> action ~ Categorical -> log_prob -> env.step.  (value /
// bootstrap_value are evaluated beside it by stx_tc_rollout_values, see ff_ppo.py in this repo.)
//
// SyntheticBoxEnv's dynamics do not depend on the action (stx_env.cu), so its whole trajectory is produced BEFORE the
// policy runs, by synth_env_trajectory_kernel over the whole GPU (same Philox streams as stx_synth_env_step =>
// bit-identical trajectory).  The policy of step t then depends only on obs[t] and the actor, not on step t - 1: the
// T x E rows are independent work.  A persistent CTA (actor weights loaded into shared memory once) walks the 64-row tiles
// w = blockIdx.x, blockIdx.x + gridDim.x, ... of the flat (T E, D) observation matrix; tile w is step t = 64 w / E, envs
// 64 w mod E .. + 63, so the grid can span every SM instead of one CTA per 64 envs.
// Warp roles:
//   warps 0..3   one warpgroup: the layer chain of stx_tc_mlp.cu on wgmma (activations in registers), then
//                Gumbel-max sampling + log-prob of the logits (same Philox counters as stx_categorical =>
//                identical actions for identical logits).
//   warp 4       loader: one TMA box per tile (64 rows of obs) into a ring of 128B-swizzled stages, kStages tiles
//                ahead of the MMA warpgroup.
//   warps 5..6   Gumbel noise: one thread per row draws the A uniforms of its (env, step) (the Philox counters of
//                stx_categorical) and writes -log(-log u) into a shared-memory ring, up to kStages tiles ahead, so the
//                MMA warpgroup's sampling only adds and compares.
// Environments whose dynamics depend on the action use the unfused per-step path.
#include <cuda.h>

#include "stx_common.cuh"
#include "stx_tc_ptx.cuh"

namespace stx {
namespace tc {

int make_map_2d_pub(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows,
                    uint32_t box_cols);

namespace ro {

constexpr int kTileM = 64;
constexpr int kStages = 4;              // observation tiles in flight
constexpr int kThreads = 128 + 32 + 64;  // the MMA warpgroup, the loader warp, two Gumbel warps

constexpr uint32_t kOffX = kImgWBytes;  // kStages x 8 KB
constexpr uint32_t kOffG = kOffX + kStages * 8192;  // kStages x 64 rows x 16 floats of Gumbel noise
constexpr uint32_t kOffBias = kOffG + kStages * kTileM * 16 * 4;
constexpr uint32_t kOffBar = kOffBias + 528 * 4;
constexpr uint32_t kSmemBytes = kOffBar + 256 + 1024;
static_assert(kSmemBytes <= 232448, "rollout kernel: shared memory over the per-block limit");

constexpr uint32_t kTagCat = 0x43415447u;

struct Params {
  const __nv_bfloat16* w2;
  const float *b0, *b1, *b2;
  int A, T;
  int64_t E;
  int num_tiles;    // T E / 64
  int32_t* action;  // (T, E)
  float* log_prob;
  // policy RNG
  uint64_t cat_seed, cat_offset;
  const uint64_t* cat_counter;
};

__global__ void __launch_bounds__(kThreads, 1)
    tc_rollout_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW0,
                      const __grid_constant__ CUtensorMap tmW1, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  // align by OFFSET (not through an integer cast) so that the compiler keeps the shared address space (LDS/STS)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  float* s_b0 = reinterpret_cast<float*>(smem + kOffBias);
  float* s_b1 = s_b0 + 256;
  float* s_b2 = s_b1 + 256;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* x_full = bars;              // [kStages] loader -> MMA: observation tile of the step in the stage
  uint64_t* x_empty = bars + kStages;   // [kStages] MMA -> loader: layer 0 has read the stage
  uint64_t* w_full = bars + 2 * kStages;
  uint64_t* g_full = bars + 2 * kStages + 1;   // [kStages] Gumbel warps -> MMA: the step's noise is in the stage
  uint64_t* g_empty = bars + 3 * kStages + 1;  // [kStages] MMA -> Gumbel warps: the sampling has read the stage
  float* s_g = reinterpret_cast<float*>(smem + kOffG);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&x_full[s], 1);
      mbar_init(&x_empty[s], 4);  // one arrival per MMA warp
      mbar_init(&g_full[s], 2);   // one arrival per Gumbel warp
      mbar_init(&g_empty[s], 4);
    }
    mbar_init(w_full, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(w_full, 32768 + 131072);
    for (int j = 0; j < 4; ++j) tma_load_2d(smem + kImgW0 + j * 8192, &tmW0, w_full, j * 64, 0);
    for (int j = 0; j < 4; ++j) tma_load_2d(smem + kImgW1 + j * 32768, &tmW1, w_full, j * 64, 0);
  }
  stage_w2_bias(smem, p.w2, p.b0, p.b1, p.b2, p.A, s_b0, s_b1, s_b2);
  fence_async_proxy();
  __syncthreads();

  if (warp >= 5) {
    // ===================== Gumbel noise of row r, call = offset + t + *counter (stx_categorical's counters) =====================
    const int r = threadIdx.x - 160;
    const uint64_t call0 = p.cat_offset + (p.cat_counter ? *p.cat_counter : 0ull);
    const uint2 ckey = make_uint2((uint32_t)p.cat_seed, (uint32_t)(p.cat_seed >> 32));
    const int A = p.A;
    for (int i = 0, w = blockIdx.x; w < p.num_tiles; ++i, w += gridDim.x) {
      const int s = i % kStages;
      if (i >= kStages) mbar_wait(&g_empty[s], ((i / kStages) - 1) & 1, 33);  // the sampling of tile i - kStages has read it
      const uint32_t row = (uint32_t)w * kTileM + r, n_env = (uint32_t)p.E;  // T E < 2^31: 32-bit division (no call)
      const uint32_t t = row / n_env;
      const int64_t e = row - t * n_env;
      const uint64_t call = call0 + (uint64_t)t;
      const uint32_t c2 = (uint32_t)(call >> 32) ^ ((uint32_t)((uint64_t)e >> 32) << 16);
      float* g = s_g + (s * kTileM + r) * 16;
#pragma unroll
      for (int j0 = 0; j0 < 16; j0 += 4) {
        if (j0 < A) {
          const uint4 rr = Philox::rand4(make_uint4((uint32_t)e, (uint32_t)call, c2 ^ ((uint32_t)(j0 >> 2) << 24), kTagCat), ckey);
          const uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (j0 + k < A) g[j0 + k] = -logf(-logf(u01(w[k])));
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&g_full[s]);
    }
  } else if (warp == 4) {
    // ===================== loader: flat observation rows [64 w, 64 w + 64) -> stage i % kStages =====================
    if (lane == 0) {
      tma_prefetch_desc(&tmX);
      for (int i = 0, w = blockIdx.x; w < p.num_tiles; ++i, w += gridDim.x) {
        const int s = i % kStages;
        if (i >= kStages) mbar_wait(&x_empty[s], ((i / kStages) - 1) & 1, 30);  // layer 0 of tile i - kStages has read it
        mbar_arrive_expect_tx(&x_full[s], 8192);
        tma_load_2d(smem + kOffX + s * 8192, &tmX, &x_full[s], 0, w * kTileM);
      }
    }
  } else {
    // ===================== the MMA warpgroup =====================
    const int q4 = lane & 3;
    const int row = warp * 16 + (lane >> 2);  // rows row and row + 8 of the tile; lanes q4 = 0 / 1 sample them
    const int lrow = row + 8 * (q4 & 1);
    mbar_wait(w_full, 0, 31);
    for (int i = 0, w = blockIdx.x; w < p.num_tiles; ++i, w += gridDim.x) {
      const int s = i % kStages;
      mbar_wait(&x_full[s], (i / kStages) & 1, 32);
      float acc[64];
      uint32_t a1[64], a2[64];
      wg_zero(acc);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        gemm_x_w0(acc, sbase + kOffX + s * 8192, sbase, h);
        if (h == 1 && lane == 0) mbar_arrive(&x_empty[s]);  // both halves of layer 0 have read the stage
        epi_bias_relu(acc, s_b0, h, a1, lane);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        gemm_a_w1(acc, a1, sbase, h);
        epi_bias_relu(acc, s_b1, h, a2, lane);
      }
      float zr[8];
      wg_zero(zr);
      gemm_a_w2(zr, a2, sbase);
      // the 16 logits of row (q4 = 0) / row + 8 (q4 = 1), gathered from the 4 lanes of the quad
      float z[16];
#pragma unroll
      for (int src = 0; src < 4; ++src) {
        const int sl = (lane & ~3) | src;
#pragma unroll
        for (int i = 0; i < 8; ++i) {  // zr[i]: row + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 src + (i & 1)
          const float v = __shfl_sync(0xffffffffu, zr[i], sl);
          if (((i >> 1) & 1) == (q4 & 1)) z[8 * (i >> 2) + 2 * src + (i & 1)] = v;
        }
      }
      if (q4 < 2) {
        const int A = p.A;
        float zmax = -INFINITY;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          z[j] += s_b2[j];
          if (j < A) zmax = fmaxf(zmax, z[j]);
        }
        float se = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < A) se += expf(z[j] - zmax);
        const float lse = zmax + logf(se);
        // Gumbel-max with the noise the Gumbel warps drew for this row and step
        mbar_wait(&g_full[s], (i / kStages) & 1, 34);
        const float* g = s_g + (s * kTileM + lrow) * 16;
        float best = -INFINITY, za = 0.f;
        int a = 0;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < A) {
            const float sc = z[j] + g[j];
            if (sc > best) best = sc, a = j, za = z[j];
          }
        const int64_t o = (int64_t)w * kTileM + lrow;  // (t, e) of the time-major (T, E) arrays
        p.action[o] = a;
        p.log_prob[o] = za - lse;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&g_empty[s]);
    }
  }
}

}  // namespace ro
}  // namespace tc
}  // namespace stx

using namespace stx;

extern "C" int stx_synth_env_trajectory(int64_t E, int D, int T, uint64_t seed, uint64_t step, const uint64_t* dev_counter, float p_term,
                                        float p_trunc, void* obs, void* next_obs, float* reward, uint8_t* done, uint8_t* truncated,
                                        float* ep_return, int32_t* ep_length, uint8_t* is_terminal, float* run_return,
                                        int32_t* run_length, void* stream);

extern "C" int stx_tc_rollout_policy(const StxMlp* actor, const void* obs, int32_t* action, float* log_prob, int T, int64_t E,
                                     uint64_t cat_seed, uint64_t cat_offset, const uint64_t* cat_counter, int max_ctas, void* stream) {
  using namespace stx::tc;
  STX_REQUIRE(actor && obs && action && log_prob, STX_E_ARG, "stx_tc_rollout_policy: null pointer");
  STX_REQUIRE(actor->n_layers == 3 && actor->sizes[1] == 256 && actor->sizes[2] == 256 && actor->sizes[0] <= 64 &&
                  actor->sizes[0] % 8 == 0 && actor->sizes[3] >= 1 && actor->sizes[3] <= 16 && actor->activation == STX_ACT_RELU &&
                  !actor->use_layer_norm,
              STX_E_SHAPE, "stx_tc_rollout_policy: actor must be MLP [D<=64 (mult of 8), 256, 256, A<=16]");
  STX_REQUIRE(E > 0 && E % 64 == 0 && T > 0, STX_E_SHAPE, "stx_tc_rollout_policy: num_envs (%lld) must be a multiple of 64", (long long)E);
  STX_REQUIRE((int64_t)T * E < (1ll << 31), STX_E_SHAPE, "stx_tc_rollout_policy: T * E must stay below 2^31 rows");
  STX_REQUIRE(actor->params_bf16 != nullptr, STX_E_ARG, "stx_tc_rollout_policy needs the bf16 shadow arena");
  const int D = actor->sizes[0], A = actor->sizes[3];
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(actor->params_bf16);
  const int64_t off_w1 = (int64_t)D * 256 + 256, off_w2 = off_w1 + 65536 + 256;
  CUtensorMap tmX, tmW0, tmW1;
  if (int rc = make_map_2d_pub(&tmX, obs, (uint64_t)T * (uint64_t)E, (uint64_t)D, (uint64_t)D, 64, 64)) return rc;
  if (int rc = make_map_2d_pub(&tmW0, w, (uint64_t)D, 256, 256, 64, 64)) return rc;
  if (int rc = make_map_2d_pub(&tmW1, w + off_w1, 256, 256, 256, 256, 64)) return rc;
  ro::Params p{};
  p.w2 = w + off_w2;
  p.b0 = actor->params + (int64_t)D * 256, p.b1 = actor->params + off_w1 + 65536, p.b2 = actor->params + off_w2 + (int64_t)256 * A;
  p.A = A, p.T = T, p.E = E;
  p.num_tiles = (int)((int64_t)T * E / ro::kTileM);
  p.action = action, p.log_prob = log_prob;
  p.cat_seed = cat_seed, p.cat_offset = cat_offset, p.cat_counter = cat_counter;
  STX_CUDA_OK(stx::opt_in_smem<ro::tc_rollout_kernel>(ro::kSmemBytes));
  if (int rc = use_trap_record((cudaStream_t)stream)) return rc;
  const int cap = (max_ctas > 0 && max_ctas < kNumSMs) ? max_ctas : kNumSMs;
  const int grid = p.num_tiles < cap ? p.num_tiles : cap;
  ro::tc_rollout_kernel<<<(unsigned)grid, ro::kThreads, ro::kSmemBytes, (cudaStream_t)stream>>>(tmX, tmW0, tmW1, p);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_tc_rollout_synth(const StxMlp* actor, void* obs, void* next_obs, int32_t* action, float* log_prob, float* reward,
                                    uint8_t* done, uint8_t* truncated, float* ep_return, int32_t* ep_length, uint8_t* is_terminal,
                                    float* run_return, int32_t* run_length, int T, int64_t E, uint64_t env_seed, uint64_t env_step,
                                    const uint64_t* env_counter, float p_term, float p_trunc, uint64_t cat_seed, uint64_t cat_offset,
                                    const uint64_t* cat_counter, void* stream) {
  STX_REQUIRE(actor && obs && next_obs && action && log_prob && reward && done && truncated && ep_return && ep_length &&
                  is_terminal && run_return && run_length,
              STX_E_ARG, "stx_tc_rollout_synth: null pointer");
  STX_REQUIRE(E > 0 && E % 64 == 0 && T > 0, STX_E_SHAPE, "stx_tc_rollout_synth: num_envs (%lld) must be a multiple of 64", (long long)E);
  if (int rc = stx_synth_env_trajectory(E, actor->sizes[0], T, env_seed, env_step, env_counter, p_term, p_trunc, obs, next_obs, reward,
                                        done, truncated, ep_return, ep_length, is_terminal, run_return, run_length, stream))
    return rc;
  return stx_tc_rollout_policy(actor, obs, action, log_prob, T, E, cat_seed, cat_offset, cat_counter, 0, stream);
}
