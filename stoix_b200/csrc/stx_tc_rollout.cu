// Fused persistent rollout for the synthetic Box environment (bf16 / wgmma path).
//
// Reference semantics: the T-step lax.scan of _env_step (stoix/systems/ppo/anakin/ff_ppo.py:81-140) for
// the actor side: logits = actor(obs_t) -> action ~ Categorical -> log_prob -> env.step.  (value /
// bootstrap_value are evaluated afterwards in two batched critic launches, see ff_ppo.py in this repo.)
//
// One CTA owns 64 environments for the WHOLE rollout (grid = E/64), so the actor's weights are loaded into
// shared memory once per rollout instead of once per step, and the T sequential steps cost one launch.
// Warp roles:
//   warps 0..3   one warpgroup: the layer chain of stx_tc_mlp.cu on wgmma (activations in registers), then
//                Gumbel-max sampling + log-prob of the logits (same Philox counters as stx_categorical =>
//                identical actions for identical logits).
//   warps 4..7   environment producers (two threads per env row, each drawing half of its features: the Philox draws
//                and normal transforms of a step cost more issue slots than the MMA chain of the step when one warp per
//                32 rows has to produce them all): SyntheticBoxEnv's dynamics do not depend on
//                the action (stx_env.cu), so the producers run one step AHEAD of the policy: while the
//                tensor cores evaluate step t they draw step t's outcome and observation t+1 (same Philox
//                streams as stx_synth_env_step => bit-identical trajectory), write the trajectory rows and
//                drop the next observation tile straight into 128B-swizzled shared memory.
// Environments whose dynamics depend on the action use the unfused per-step path.
#include <cuda.h>

#include "stx_common.cuh"
#include "stx_tc_ptx.cuh"

namespace stx {
namespace tc {

int make_map_2d_pub(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows,
                    uint32_t box_cols);

namespace ro {

constexpr int kTileM = 64, kH = 256;
constexpr int kProdWarps = 4;
constexpr int kThreads = 128 + 32 * kProdWarps;  // 256

constexpr uint32_t kOffX = kImgWBytes;  // 2 stages x 8 KB
constexpr uint32_t kOffBias = kOffX + 2 * 8192;
constexpr uint32_t kOffBar = kOffBias + 528 * 4;
constexpr uint32_t kSmemBytes = kOffBar + 64 + 1024;

constexpr uint32_t kTagObs = 0x4f425331u, kTagReset = 0x52535431u, kTagStep = 0x53545031u, kTagCat = 0x43415447u;

struct Params {
  const __nv_bfloat16* w2;
  const float *b0, *b1, *b2;
  int A, D, T;
  int64_t E;
  // trajectory (time-major)
  __nv_bfloat16* obs;       // (T+1, E, D): row 0 is the input observation, rows 1..T are written
  __nv_bfloat16* next_obs;  // (T, E, D)
  int32_t* action;          // (T, E)
  float* log_prob;
  float* reward;
  uint8_t *done, *truncated, *is_terminal;
  float* ep_return;
  int32_t* ep_length;
  float* run_return;        // (E) carried episode bookkeeping
  int32_t* run_length;
  // env RNG
  uint64_t env_seed, env_step;
  const uint64_t* env_counter;
  float p_term, p_trunc;
  // policy RNG
  uint64_t cat_seed, cat_offset;
  const uint64_t* cat_counter;
};

__global__ void __launch_bounds__(kThreads, 1)
    tc_rollout_kernel(const __grid_constant__ CUtensorMap tmW0, const __grid_constant__ CUtensorMap tmW1, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  // align by OFFSET (not through an integer cast) so that the compiler keeps the shared address space (LDS/STS)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  float* s_b0 = reinterpret_cast<float*>(smem + kOffBias);
  float* s_b1 = s_b0 + 256;
  float* s_b2 = s_b1 + 256;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* x_full = bars;       // [2] producers -> MMA: observation tile of the step in the stage
  uint64_t* x_empty = bars + 2;  // [2] MMA -> producers: layer 0 has read the stage
  uint64_t* w_full = bars + 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tile_row0 = (int64_t)blockIdx.x * kTileM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&x_full[s], kProdWarps);
      mbar_init(&x_empty[s], 4);  // one arrival per MMA warp
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

  if (warp >= 4) {
    // ===================== environment producers: two threads per env row =====================
    const int r = (threadIdx.x - 128) & 63, hf = (threadIdx.x - 128) >> 6;  // row, half of its 16-byte chunks: c = 4 hf + cc
    const int64_t e = tile_row0 + r;
    const int dchunks = p.D >> 3;
    const uint64_t step0 = p.env_step + (p.env_counter ? *p.env_counter : 0ull);
    const uint2 key = make_uint2((uint32_t)p.env_seed, (uint32_t)(p.env_seed >> 32));
    float run_ret = p.run_return[e];
    int run_len = p.run_length[e];
    // stage 0 <- obs[0] (the carried observation)
    {
      uint8_t* xs = smem + kOffX + r * 128;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = 4 * hf + cc;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (c < dchunks) v = *reinterpret_cast<const uint4*>(p.obs + e * p.D + c * 8);
        *reinterpret_cast<uint4*>(xs + ((c ^ (r & 7)) << 4)) = v;
      }
      fence_async_proxy();
      __syncwarp();
      if (lane == 0) mbar_arrive(&x_full[0]);
    }
    for (int t = 0; t < p.T; ++t) {
      const uint64_t step = step0 + (uint64_t)t;
      const uint32_t e_lo = (uint32_t)e, st_lo = (uint32_t)step;
      const uint32_t hi = ((uint32_t)((uint64_t)e >> 32) << 16) ^ (uint32_t)(step >> 32);
      const uint4 rs = Philox::rand4(make_uint4(e_lo, st_lo, hi, kTagStep), key);
      const bool term = u01(rs.z) < p.p_term;
      const bool trunc = !term && (u01(rs.w) < p.p_trunc);
      const bool last = term || trunc;
      __nv_bfloat16* nrow = p.next_obs + ((int64_t)t * p.E + e) * p.D;
      __nv_bfloat16* orow = p.obs + ((int64_t)(t + 1) * p.E + e) * p.D;
      const int s = (t + 1) & 1;
      const bool fill = t + 1 < p.T;  // next observation tile -> smem stage (t+1)&1 (consumed by the forward of step t+1)
      if (fill && t >= 1) mbar_wait(&x_empty[s], (((t - 1) >> 1) & 1), 30);  // layer 0 of step t-1 has read this stage
      uint8_t* xs = smem + kOffX + s * 8192 + r * 128;
#pragma unroll 1
      for (int cc = 0; cc < 4; ++cc) {
        const int c = 4 * hf + cc;
        uint4 nx = make_uint4(0u, 0u, 0u, 0u), ob;
        if (c < dchunks) {
          uint32_t w[4];
#pragma unroll
          for (int g2 = 0; g2 < 2; ++g2) {
            const uint32_t grp = (uint32_t)(2 * c + g2);
            const uint4 ro_ = Philox::rand4(make_uint4(e_lo, st_lo, hi ^ (grp << 8), kTagObs), key);
            const float2 a = normal2(ro_.x, ro_.y), b = normal2(ro_.z, ro_.w);
            w[2 * g2] = pack_bf16(a.x, a.y);
            w[2 * g2 + 1] = pack_bf16(b.x, b.y);
          }
          nx = make_uint4(w[0], w[1], w[2], w[3]);
        }
        ob = nx;
        if (last && c < dchunks) {
          uint32_t w[4];
#pragma unroll
          for (int g2 = 0; g2 < 2; ++g2) {
            const uint32_t grp = (uint32_t)(2 * c + g2);
            const uint4 rr = Philox::rand4(make_uint4(e_lo, st_lo, hi ^ (grp << 8), kTagReset), key);
            const float2 a = normal2(rr.x, rr.y), b = normal2(rr.z, rr.w);
            w[2 * g2] = pack_bf16(a.x, a.y);
            w[2 * g2 + 1] = pack_bf16(b.x, b.y);
          }
          ob = make_uint4(w[0], w[1], w[2], w[3]);
        }
        if (c < dchunks) {  // trajectory rows (global)
          *reinterpret_cast<uint4*>(nrow + c * 8) = nx;
          *reinterpret_cast<uint4*>(orow + c * 8) = ob;
        }
        if (fill) *reinterpret_cast<uint4*>(xs + ((c ^ (r & 7)) << 4)) = ob;
      }
      if (hf == 0) {
        const float rwd = normal2(rs.x, rs.y).x;
        const int64_t o = (int64_t)t * p.E + e;
        const float ret = run_ret + rwd;
        const int len = run_len + 1;
        p.reward[o] = rwd;
        p.done[o] = term ? 1 : 0;
        p.truncated[o] = trunc ? 1 : 0;
        p.ep_return[o] = ret;
        p.ep_length[o] = len;
        p.is_terminal[o] = last ? 1 : 0;
        run_ret = last ? 0.f : ret;
        run_len = last ? 0 : len;
      }
      if (fill) {
        fence_async_proxy();
        __syncwarp();
        if (lane == 0) mbar_arrive(&x_full[s]);
      }
    }
    if (hf == 0) p.run_return[e] = run_ret, p.run_length[e] = run_len;
  } else {
    // ===================== the MMA warpgroup =====================
    const int q4 = lane & 3;
    const int row = warp * 16 + (lane >> 2);  // rows row and row + 8 of the tile; lanes q4 = 0 / 1 sample them
    const int64_t e = tile_row0 + row + 8 * (q4 & 1);
    const uint64_t call0 = p.cat_offset + (p.cat_counter ? *p.cat_counter : 0ull);
    const uint2 ckey = make_uint2((uint32_t)p.cat_seed, (uint32_t)(p.cat_seed >> 32));
    mbar_wait(w_full, 0, 31);
    for (int t = 0; t < p.T; ++t) {
      const int s = t & 1;
      mbar_wait(&x_full[s], (t >> 1) & 1, 32);
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
        // Gumbel-max with the counters of stx_categorical: (row, call = offset + t + *counter)
        const uint64_t call = call0 + (uint64_t)t;
        const uint32_t c2 = (uint32_t)(call >> 32) ^ ((uint32_t)((uint64_t)e >> 32) << 16);
        float best = -INFINITY, za = 0.f;
        int a = 0;
#pragma unroll
        for (int j0 = 0; j0 < 16; j0 += 4) {
          if (j0 < A) {
            const uint4 rr = Philox::rand4(make_uint4((uint32_t)e, (uint32_t)call, c2 ^ ((uint32_t)(j0 >> 2) << 24), kTagCat), ckey);
            const uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (j0 + k < A) {
                const float sc = z[j0 + k] + (-logf(-logf(u01(w[k]))));
                if (sc > best) best = sc, a = j0 + k, za = z[j0 + k];
              }
          }
        }
        const int64_t o = (int64_t)t * p.E + e;
        p.action[o] = a;
        p.log_prob[o] = za - lse;
      }
    }
  }
}

}  // namespace ro
}  // namespace tc
}  // namespace stx

using namespace stx;

extern "C" int stx_tc_rollout_synth(const StxMlp* actor, void* obs, void* next_obs, int32_t* action, float* log_prob, float* reward,
                                    uint8_t* done, uint8_t* truncated, float* ep_return, int32_t* ep_length, uint8_t* is_terminal,
                                    float* run_return, int32_t* run_length, int T, int64_t E, uint64_t env_seed, uint64_t env_step,
                                    const uint64_t* env_counter, float p_term, float p_trunc, uint64_t cat_seed, uint64_t cat_offset,
                                    const uint64_t* cat_counter, void* stream) {
  using namespace stx::tc;
  STX_REQUIRE(actor && obs && next_obs && action && log_prob && reward && done && truncated && ep_return && ep_length &&
                  is_terminal && run_return && run_length,
              STX_E_ARG, "stx_tc_rollout_synth: null pointer");
  STX_REQUIRE(actor->n_layers == 3 && actor->sizes[1] == 256 && actor->sizes[2] == 256 && actor->sizes[0] <= 64 &&
                  actor->sizes[0] % 8 == 0 && actor->sizes[3] >= 1 && actor->sizes[3] <= 16 && actor->activation == STX_ACT_RELU &&
                  !actor->use_layer_norm,
              STX_E_SHAPE, "stx_tc_rollout_synth: actor must be MLP [D<=64 (mult of 8), 256, 256, A<=16]");
  STX_REQUIRE(E > 0 && E % 64 == 0 && T > 0, STX_E_SHAPE, "stx_tc_rollout_synth: num_envs (%lld) must be a multiple of 64", (long long)E);
  STX_REQUIRE(actor->params_bf16 != nullptr, STX_E_ARG, "stx_tc_rollout_synth needs the bf16 shadow arena");
  const int D = actor->sizes[0], A = actor->sizes[3];
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(actor->params_bf16);
  const int64_t off_w1 = (int64_t)D * 256 + 256, off_w2 = off_w1 + 65536 + 256;
  CUtensorMap tmW0, tmW1;
  if (int rc = make_map_2d_pub(&tmW0, w, (uint64_t)D, 256, 256, 64, 64)) return rc;
  if (int rc = make_map_2d_pub(&tmW1, w + off_w1, 256, 256, 256, 256, 64)) return rc;
  ro::Params p{};
  p.w2 = w + off_w2;
  p.b0 = actor->params + (int64_t)D * 256, p.b1 = actor->params + off_w1 + 65536, p.b2 = actor->params + off_w2 + (int64_t)256 * A;
  p.A = A, p.D = D, p.T = T, p.E = E;
  p.obs = reinterpret_cast<__nv_bfloat16*>(obs), p.next_obs = reinterpret_cast<__nv_bfloat16*>(next_obs);
  p.action = action, p.log_prob = log_prob, p.reward = reward, p.done = done, p.truncated = truncated, p.is_terminal = is_terminal;
  p.ep_return = ep_return, p.ep_length = ep_length, p.run_return = run_return, p.run_length = run_length;
  p.env_seed = env_seed, p.env_step = env_step, p.env_counter = env_counter, p.p_term = p_term, p.p_trunc = p_trunc;
  p.cat_seed = cat_seed, p.cat_offset = cat_offset, p.cat_counter = cat_counter;
  static bool attr_set = false;
  if (!attr_set) {
    STX_CUDA_OK(cudaFuncSetAttribute(ro::tc_rollout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ro::kSmemBytes));
    attr_set = true;
  }
  if (int rc = use_trap_record((cudaStream_t)stream)) return rc;
  ro::tc_rollout_kernel<<<(unsigned)(E / ro::kTileM), ro::kThreads, ro::kSmemBytes, (cudaStream_t)stream>>>(tmW0, tmW1, p);
  STX_LAUNCH_OK();
  return STX_OK;
}
