// K2 -- generalized advantage estimation as a chunked parallel reverse scan over (T, E).
//
// Reference: batch_truncated_generalized_advantage_estimation, stoix/utils/multistep.py:14-145, as
// called at stoix/systems/ppo/anakin/ff_ppo.py:164-179 (time-major, truncation flags, standardise).
// The reference runs a T-iteration lax.scan of (E,)-wide fusions (multistep.py:119-130).  Here the
// first-order linear recurrence  acc_t = delta_t + c_t * acc_{t+1},  c_t = disc_t*lambda_t*(1-trunc_t)
// is evaluated as a composition of affine maps:
//   * a thread owns L=4 consecutive timesteps of VEC (=4, float4) adjacent envs: one pass of coalesced
//     128-bit streaming loads, a local scan in registers yielding its chunk map x -> B + A*x;
//   * the 32 chunk maps of one env (one 128-step segment) are suffix-composed with a 5-step warp
//     shuffle scan; longer rollouts walk segments from the end carrying one value per env;
//   * every element is read once and written once: 22 B/element in PPO form (SURVEY.md 8d).
// Advantage standardisation statistics (jax.nn.standardize, multistep.py:138-139) are reduced in
// double precision with a deterministic two-level reduction finished by the last block to arrive.
#include "stx_common.cuh"
#include "stx_tc_ptx.cuh"

#include <type_traits>

namespace stx {
namespace {

constexpr int kChunks = 32;  // chunk lanes per block == warp width (suffix scan by shuffles)

// An input form's load yields, per element, the affine map acc_t = d + c * acc_{t+1} and the value v the targets add to acc.
// kTargetsOnly: the form's result is acc itself, stored as the targets (no advantages, no statistics).
struct PpoIn {  // exactly what ff_ppo.py:164-169 feeds
  static constexpr bool kTargetsOnly = false;
  const float *reward, *v_tm1, *v_t;
  const uint8_t *done, *trunc;
  float gamma, lambda, reward_scale;
  // one element's map from its inputs; done / trunc are the flag bytes (nonzero: set)
  __device__ __forceinline__ void map(float r, float vt, float vtm1, uint32_t done_b, uint32_t trunc_b, float& d, float& c) const {
    const float disc = (1.0f - (done_b ? 1.f : 0.f)) * gamma;      // ff_ppo.py:167-168
    d = r * reward_scale + disc * vt - vtm1;                       // multistep.py:116
    c = disc * lambda * (1.0f - (trunc_b ? 1.f : 0.f));            // multistep.py:123
  }
  // four adjacent envs: one flag byte per env in fd / ft
  __device__ __forceinline__ void map4(float4 r, float4 vtm1, float4 vt, uint32_t fd, uint32_t ft, float* d, float* c, float* v) const {
    const float r4[4] = {r.x, r.y, r.z, r.w}, e4[4] = {vt.x, vt.y, vt.z, vt.w};
    v[0] = vtm1.x, v[1] = vtm1.y, v[2] = vtm1.z, v[3] = vtm1.w;
#pragma unroll
    for (int k = 0; k < 4; ++k) map(r4[k], e4[k], v[k], (fd >> (8 * k)) & 0xffu, (ft >> (8 * k)) & 0xffu, d[k], c[k]);
  }
  template <int VEC>
  __device__ __forceinline__ void load(int64_t off, float* d, float* c, float* v) const {
    if constexpr (VEC == 4) {
      map4(ldg_stream4(reward + off), ldg_stream4(v_tm1 + off), ldg_stream4(v_t + off), ldg_stream_u32(done + off),
           ldg_stream_u32(trunc + off), d, c, v);
    } else {
      v[0] = __ldg(v_tm1 + off);
      map(__ldg(reward + off), __ldg(v_t + off), v[0], __ldg(done + off), __ldg(trunc + off), d[0], c[0]);
    }
  }
};

struct GenericIn {  // float discount / lambda / truncation arrays (multistep.py:97-105)
  static constexpr bool kTargetsOnly = false;
  const float *r, *disc, *lam_t, *v_tm1, *v_t, *trunc;
  float lambda;
  template <int VEC>
  __device__ __forceinline__ void load(int64_t off, float* d, float* c, float* v) const {
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      const float dk = __ldg(disc + off + k);
      const float lk = lam_t ? __ldg(lam_t + off + k) : lambda;
      const float tk = trunc ? __ldg(trunc + off + k) : 0.f;
      v[k] = __ldg(v_tm1 + off + k);
      d[k] = __ldg(r + off + k) + dk * __ldg(v_t + off + k) - v[k];
      c[k] = dk * lk * (1.0f - tk);
    }
  }
};

// Lambda returns (batch_lambda_returns, multistep.py:384-408) with v_t = max over the A columns of q (batch_q_lambda,
// :559-569; A = 1: v_t itself):  G_t = r_t + d_t [(1 - lambda) v_t + lambda G_{t+1}], the scan starting from G_T = v_t[T-1], i.e.
// the affine map a_t = r_t + d_t (1 - lambda) v_t, c_t = d_t lambda, and on the last step a = r + d v, c = 0.  The discount is
// either a float array or gamma (1 - (done | truncated)) from the rollout's flags (ff_pqn.py:107-109, done = timestep.last()).
struct LambdaIn {
  static constexpr bool kTargetsOnly = true;
  const float *q, *r, *disc, *lam_t;  // q: (T, E, A); disc / lam_t nullable
  const uint8_t *done, *trunc;         // used when disc is NULL
  int A;
  float gamma, lambda;
  int64_t last;                        // flat offset of the first element of step T-1
  template <int VEC>
  __device__ __forceinline__ void load(int64_t off, float* d, float* c, float* v) const {
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      const int64_t i = off + k;
      const float* row = q + i * A;
      float vmax = __ldg(row);
      for (int j = 1; j < A; ++j) {  // NaN-propagating max, as jnp.max (fmaxf would drop a NaN)
        const float x = __ldg(row + j);
        vmax = (x > vmax || x != x) ? x : vmax;
      }
      const float dk = disc ? __ldg(disc + i) : ((__ldg(done + i) | __ldg(trunc + i)) ? 0.f : gamma);
      const float lk = lam_t ? __ldg(lam_t + i) : lambda;
      const bool is_last = i >= last;
      d[k] = __ldg(r + i) + dk * ((is_last ? 1.0f : 1.0f - lk) * vmax);
      c[k] = is_last ? 0.f : dk * lk;
      v[k] = 0.f;
    }
  }
};

// ---- the scan steps both kernels run -----------------------------------------------------------------------------------
// A block covers W - 1 envs x 32 chunks of kL timesteps; the thread of chunk `chunk` owns VEC envs from column `col`.  sA / sB
// are padded to W = envs + 1 columns.

// Local reverse scan of the thread's kL x VEC maps: step j's acc is b[j] + a[j] * (acc entering the chunk); the chunk's whole
// map (a[0], b[0]) goes to sA / sB.
template <int kL, int VEC, int W>
__device__ __forceinline__ void scan_chunk(const float (&d)[kL][VEC], const float (&c)[kL][VEC], float (&a)[kL][VEC], float (&b)[kL][VEC],
                                           float (&sA)[kChunks][W], float (&sB)[kChunks][W], int chunk, int col) {
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    float rb = 0.f, ra = 1.f;
#pragma unroll
    for (int j = kL - 1; j >= 0; --j) {
      rb = fmaf(c[j][k], rb, d[j][k]);
      ra = c[j][k] * ra;
      b[j][k] = rb;
      a[j][k] = ra;
    }
    sA[chunk][col + k] = ra;
    sB[chunk][col + k] = rb;
  }
}

// Suffix composition over the 32 chunks of each env: warp w owns envs w*VEC .. w*VEC+VEC-1, lane = chunk index.  Leaves the acc
// entering each chunk in sA and the acc entering the previous (earlier) segment in sCarry.
template <int VEC, int W>
__device__ __forceinline__ void compose_chunks(float (&sA)[kChunks][W], const float (&sB)[kChunks][W], float* sCarry, int lane, int warp) {
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const int env = warp * VEC + k;
    float A = sA[lane][env], B = sB[lane][env];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const float A2 = __shfl_down_sync(0xffffffffu, A, off);
      const float B2 = __shfl_down_sync(0xffffffffu, B, off);
      if (lane + off < 32) {
        B = fmaf(A, B2, B);
        A = A * A2;
      }
    }
    const float carry = sCarry[env];
    const float Ae = __shfl_down_sync(0xffffffffu, A, 1), Be = __shfl_down_sync(0xffffffffu, B, 1);
    sA[lane][env] = (lane == 31) ? carry : fmaf(Ae, carry, Be);  // acc entering this chunk
    __syncwarp();
    if (lane == 0) sCarry[env] = fmaf(A, carry, B);  // acc entering the previous (earlier) segment
  }
}

template <int VEC>
__device__ __forceinline__ void store_row(float* p, const float* x) {
  if constexpr (VEC == 4)
    stg_stream4(p, make_float4(x[0], x[1], x[2], x[3]));
  else
    p[0] = x[0];
}

// The chunk's results from the acc entering it (sA): the advantages, the targets and their statistics' per-thread sums, or the
// targets alone (kTargetsOnly).
template <bool kTargetsOnly, int kL, int VEC, int W>
__device__ __forceinline__ void store_chunk(const float (&a)[kL][VEC], const float (&b)[kL][VEC], const float (&v)[kL][VEC],
                                            const float (&sA)[kChunks][W], int chunk, int col, int tbase, int T, int E, int e0,
                                            bool env_ok, float* __restrict__ adv, float* __restrict__ tgt, float& lsum, float& lsq) {
#pragma unroll
  for (int j = 0; j < kL; ++j) {
    const int t = tbase + j;
    float av[VEC], tv[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      av[k] = fmaf(a[j][k], sA[chunk][col + k], b[j][k]);
      tv[k] = v[j][k] + av[k];  // multistep.py:132: targets use the un-standardised advantage
    }
    if (env_ok && t < T) {
      const int64_t off = (int64_t)t * E + e0;
      if constexpr (kTargetsOnly) {
        store_row<VEC>(tgt + off, av);
      } else {
        store_row<VEC>(adv + off, av);
        store_row<VEC>(tgt + off, tv);
#pragma unroll
        for (int k = 0; k < VEC; ++k) lsum += av[k], lsq = fmaf(av[k], av[k], lsq);
      }
    }
  }
}

// Advantage statistics: each block's fp64 sums to partials; the last block to arrive adds them up in block order and writes
// stats = [mean, rstd].
__device__ __forceinline__ void finish_stats(float lsum, float lsq, double* sRed, double2* __restrict__ partials, unsigned int* counter,
                                             float* __restrict__ stats, int T, int E) {
  const double bs = block_sum<double>((double)lsum, sRed);
  const double bq = block_sum<double>((double)lsq, sRed);
  if (threadIdx.x == 0) partials[blockIdx.x] = make_double2(bs, bq);
  if (last_block_ticket(counter, gridDim.x)) {
    double s = 0.0, q2 = 0.0;
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) {
      const double2 p = partials[i];
      s += p.x, q2 += p.y;
    }
    s = block_sum<double>(s, sRed);
    q2 = block_sum<double>(q2, sRed);
    if (threadIdx.x == 0) {
      const double n = (double)T * (double)E;
      const double mean = s / n;
      const double var = q2 / n - mean * mean;  // jax.nn.standardize: E[x^2] - E[x]^2
      stats[0] = (float)mean;
      stats[1] = (float)(1.0 / sqrt(var + 1e-5));
    }
  }
}

// MINB: resident blocks per SM the register allocation must allow.  A block runs load -> barrier -> scan -> barrier ->
// store with nothing overlapped inside it, so HBM only stays busy if ANOTHER block of the same SM is in its load phase
// meanwhile: the saturating shapes use 2 x 512 threads (<= 64 registers) instead of 1 x 1024.
template <class In, int VEC, int QUADS, int kL = 4, int MINB = 1>
__global__ void __launch_bounds__(QUADS* kChunks, MINB)
    gae_scan_kernel(In in, int T, int E, float* __restrict__ adv, float* __restrict__ tgt,
                    int want_stats, double2* __restrict__ partials, unsigned int* counter,
                    float* __restrict__ stats) {
  constexpr int ENVS = QUADS * VEC;  // envs per block
  constexpr int kSeg = kL * kChunks;  // timesteps covered per pass over the block
  const int q = threadIdx.x % QUADS, chunk = threadIdx.x / QUADS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int e0 = (blockIdx.x * QUADS + q) * VEC;
  const bool env_ok = e0 < E;

  __shared__ float sA[kChunks][ENVS + 1], sB[kChunks][ENVS + 1];  // sA is reused for acc_in
  __shared__ float sCarry[ENVS];
  __shared__ double sRed[32];
  if (threadIdx.x < ENVS) sCarry[threadIdx.x] = 0.f;  // multistep.py:127: acc starts at zero

  float lsum = 0.f, lsq = 0.f;
  const int nseg = (T + kSeg - 1) / kSeg;
  for (int s = nseg - 1; s >= 0; --s) {
    const int tbase = s * kSeg + chunk * kL;
    float d[kL][VEC], c[kL][VEC], v[kL][VEC];
#pragma unroll
    for (int j = 0; j < kL; ++j) {
      const int t = tbase + j;
      if (env_ok && t < T) {
        in.template load<VEC>((int64_t)t * E + e0, d[j], c[j], v[j]);
      } else {
#pragma unroll
        for (int k = 0; k < VEC; ++k) d[j][k] = 0.f, c[j][k] = 1.f, v[j][k] = 0.f;  // identity map
      }
    }
    float a[kL][VEC], b[kL][VEC];
    scan_chunk(d, c, a, b, sA, sB, chunk, q * VEC);
    __syncthreads();
    compose_chunks<VEC>(sA, sB, sCarry, lane, warp);
    __syncthreads();
    store_chunk<In::kTargetsOnly>(a, b, v, sA, chunk, q * VEC, tbase, T, E, e0, env_ok, adv, tgt, lsum, lsq);
  }
  if (want_stats) finish_stats(lsum, lsq, sRed, partials, counter, stats, T, E);
}

__global__ void standardize_inplace_kernel(float* __restrict__ adv, int64_t n,
                                           const float* __restrict__ stats) {
  const float mean = stats[0], rstd = stats[1];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
    adv[i] = (adv[i] - mean) * rstd;
}

// ---- TMA-pipelined form for the saturating shapes (PPO inputs) -------------------------------------------------------
// gae_scan_kernel runs load -> barrier -> scan -> barrier -> store per block with nothing overlapped inside it; two resident
// blocks per SM hide part of that (0.69 of the copy peak).  Here ONE persistent block per SM walks its env tiles
// (kGE envs x kGT timesteps, 5 arrays = 56 KB) through a 3-stage shared-memory ring filled by TMA (one 2-D box per array and
// stage, one mbarrier per stage): the loads of the next two tiles are in flight while the current one is scanned and stored,
// so the HBM read stream never stops.  The arithmetic is the scan steps above, reading the inputs from shared memory.
// Tile shapes: 32 envs x 128 timesteps (4 timesteps per thread, the association order of gae_scan_kernel) or 64 x 64 (2 per
// thread, two segments per 128-step rollout): half as many distinct rows -- hence 2 MB pages -- in flight per tile, which is what
// matters once the row pitch E * 4 B exceeds the page size .
constexpr int kGStages = 3;
template <int kGE, int kGT>
struct GaeStageT {
  float r[kGT][kGE], v[kGT][kGE], vt[kGT][kGE];
  uint8_t dn[kGT][kGE], tr[kGT][kGE];
};
constexpr uint32_t kGaeSmemBytes = kGStages * (3 * 128 * 32 * 4 + 2 * 128 * 32) + 1024;  // both shapes: 4096 elements per stage

template <int kGE, int kGT>
__global__ void __launch_bounds__(kGE / 4 * kChunks, 1)
    gae_tma_kernel(const __grid_constant__ CUtensorMap m_r, const __grid_constant__ CUtensorMap m_v, const __grid_constant__ CUtensorMap m_vt,
                   const __grid_constant__ CUtensorMap m_dn, const __grid_constant__ CUtensorMap m_tr, PpoIn in, int T, int E,
                   float* __restrict__ adv, float* __restrict__ tgt, int want_stats, double2* __restrict__ partials, unsigned int* counter,
                   float* __restrict__ stats) {
  using namespace tc;
  using GaeStage = GaeStageT<kGE, kGT>;
  static_assert(sizeof(GaeStage) * kGStages + 1024 == kGaeSmemBytes, "stage layout");
  constexpr int VEC = 4, QUADS = kGE / VEC, kL = kGT / kChunks;  // QUADS quads x 32 chunks of kL timesteps
  extern __shared__ uint8_t gsm_raw[];
  GaeStage* stages = reinterpret_cast<GaeStage*>((reinterpret_cast<uintptr_t>(gsm_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full[kGStages];
  __shared__ float sA[kChunks][kGE + 1], sB[kChunks][kGE + 1];
  __shared__ float sCarry[kGE];
  __shared__ double sRed[32];
  const int q = threadIdx.x % QUADS, chunk = threadIdx.x / QUADS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_tiles = (E + kGE - 1) / kGE, nseg = (T + kGT - 1) / kGT;
  const int my_tiles = ((int)blockIdx.x < n_tiles) ? (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  const int64_t my_items = (int64_t)my_tiles * nseg;  // item k: tile blockIdx + (k / nseg) * grid, segment nseg-1 - k % nseg (last first)

  auto issue = [&](int64_t k) {  // one thread
    GaeStage& st = stages[k % kGStages];
    uint64_t* bar = &full[k % kGStages];
    const int e0 = ((int)blockIdx.x + (int)(k / nseg) * (int)gridDim.x) * kGE;
    const int t0 = (nseg - 1 - (int)(k % nseg)) * kGT;
    mbar_arrive_expect_tx(bar, (uint32_t)sizeof(GaeStage));  // out-of-range rows / envs are zero-filled and counted
    tma_load_2d(&st.r[0][0], &m_r, bar, e0, t0);
    tma_load_2d(&st.v[0][0], &m_v, bar, e0, t0);
    tma_load_2d(&st.vt[0][0], &m_vt, bar, e0, t0);
    tma_load_2d(&st.dn[0][0], &m_dn, bar, e0, t0);
    tma_load_2d(&st.tr[0][0], &m_tr, bar, e0, t0);
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < kGStages; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
    for (int64_t k = 0; k < kGStages && k < my_items; ++k) issue(k);
  }
  __syncthreads();

  float lsum = 0.f, lsq = 0.f;
  for (int64_t k = 0; k < my_items; ++k) {
    const int seg = nseg - 1 - (int)(k % nseg);
    const int e0 = ((int)blockIdx.x + (int)(k / nseg) * (int)gridDim.x) * kGE + q * VEC;
    const bool env_ok = e0 < E;
    const int tbase = seg * kGT + chunk * kL, rbase = chunk * kL, col = q * VEC;
    if (seg == nseg - 1 && threadIdx.x < kGE) sCarry[threadIdx.x] = 0.f;  // multistep.py:127: acc starts at zero (read after the barrier below)
    const GaeStage& st = stages[k % kGStages];
    mbar_wait(&full[k % kGStages], (uint32_t)((k / kGStages) & 1), 900);
    float d[kL][VEC], c[kL][VEC], v[kL][VEC];
#pragma unroll
    for (int j = 0; j < kL; ++j) {
      const int row = rbase + j;
      in.map4(*reinterpret_cast<const float4*>(&st.r[row][col]), *reinterpret_cast<const float4*>(&st.v[row][col]),
              *reinterpret_cast<const float4*>(&st.vt[row][col]), *reinterpret_cast<const uint32_t*>(&st.dn[row][col]),
              *reinterpret_cast<const uint32_t*>(&st.tr[row][col]), d[j], c[j], v[j]);
      if (!env_ok || tbase + j >= T) {
#pragma unroll
        for (int kk = 0; kk < VEC; ++kk) d[j][kk] = 0.f, c[j][kk] = 1.f;  // identity map outside the array
      }
    }
    float a[kL][VEC], b[kL][VEC];
    scan_chunk(d, c, a, b, sA, sB, chunk, col);
    __syncthreads();  // every thread has consumed this stage: refill it with the tile three items ahead
    if (threadIdx.x == 0 && k + kGStages < my_items) issue(k + kGStages);
    compose_chunks<VEC>(sA, sB, sCarry, lane, warp);
    __syncthreads();
    store_chunk<false>(a, b, v, sA, chunk, col, tbase, T, E, e0, env_ok, adv, tgt, lsum, lsq);
  }
  if (want_stats) finish_stats(lsum, lsq, sRed, partials, counter, stats, T, E);
}

int g_tuning = 0;  // stx_gae_set_tuning's code

typedef CUresult (*GaeEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
GaeEncodeFn gae_encode_fn() {
  static GaeEncodeFn fn = nullptr;
  if (fn == nullptr) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<GaeEncodeFn>(sym);
  }
  return fn;
}
// (T x E) row-major array of 4-byte or 1-byte elements, box = box_t rows x box_e columns
bool gae_make_map(CUtensorMap* m, const void* base, int T, int E, bool f32, int box_e, int box_t) {
  GaeEncodeFn enc = gae_encode_fn();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)E, (cuuint64_t)T};
  cuuint64_t strides[1] = {(cuuint64_t)E * (f32 ? 4u : 1u)};
  cuuint32_t box[2] = {(cuuint32_t)box_e, (cuuint32_t)box_t};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// returns STX_OK if launched, 1 if the TMA form cannot take these arguments (the caller falls back), < 0 on errors
template <int kGE, int kGT>
int launch_gae_tma_shape(const PpoIn& in, int T, int E, int want, float* adv, float* tgt, float* stats, double2* partials, unsigned int* counter,
                         cudaStream_t st) {
  // the five tensor maps depend on (pointers, T, E) only: keep the last few sets (encoding them costs ~10 us of host time per map,
  // during which an eager caller leaves the GPU idle; a captured graph bakes them in anyway)
  struct MapSet {
    const void* key[5];
    int T, E;
    CUtensorMap m[5];
    bool valid;
  };
  static thread_local MapSet cache[4] = {};
  static thread_local int next_slot = 0;
  const void* key[5] = {in.reward, in.v_tm1, in.v_t, in.done, in.trunc};
  MapSet* ms = nullptr;
  for (auto& c : cache)
    if (c.valid && c.T == T && c.E == E && c.key[0] == key[0] && c.key[1] == key[1] && c.key[2] == key[2] && c.key[3] == key[3] && c.key[4] == key[4])
      ms = &c;
  if (!ms) {
    MapSet fresh{};
    for (int i = 0; i < 5; ++i) {
      fresh.key[i] = key[i];
      if (!gae_make_map(&fresh.m[i], key[i], T, E, i < 3, kGE, kGT)) return 1;
    }
    fresh.T = T, fresh.E = E, fresh.valid = true;
    ms = &cache[next_slot];
    next_slot = (next_slot + 1) % 4;
    *ms = fresh;
  }
  const CUtensorMap &mr = ms->m[0], &mv = ms->m[1], &mvt = ms->m[2], &mdn = ms->m[3], &mtr = ms->m[4];
  STX_CUDA_OK(opt_in_smem<gae_tma_kernel<kGE, kGT>>(kGaeSmemBytes));
  if (int rc = tc::use_trap_record(st)) return rc;
  const int n_tiles = (E + kGE - 1) / kGE;
  const int grid = n_tiles < kNumSMs ? n_tiles : kNumSMs;
  gae_tma_kernel<kGE, kGT><<<grid, kGE / 4 * kChunks, kGaeSmemBytes, st>>>(mr, mv, mvt, mdn, mtr, in, T, E, adv, tgt, want, partials, counter,
                                                                           stats);
  STX_LAUNCH_OK();
  return STX_OK;
}
int launch_gae_tma(const PpoIn& in, int T, int E, int want, float* adv, float* tgt, float* stats, double2* partials, unsigned int* counter,
                   cudaStream_t st) {
  if (E % 16 != 0 || !aligned16(in.done) || !aligned16(in.trunc)) return 1;  // TMA: 16-byte aligned rows of the byte arrays
  // 32 x 128 tiles up to E = 32768, 64 x 64 from E = 65536: once the row pitch exceeds the page size, 64 x 64 tiles halve the
  // rows (pages) in flight per tile
  const bool wide = g_tuning == 501 || (g_tuning != 500 && E >= 65536);
  return wide ? launch_gae_tma_shape<64, 64>(in, T, E, want, adv, tgt, stats, partials, counter, st)
              : launch_gae_tma_shape<32, 128>(in, T, E, want, adv, tgt, stats, partials, counter, st);
}

template <class In>
int launch_gae(const In& in, int T, int E, bool vec4, int standardize, float* adv, float* tgt,
               float* stats, void* scratch, cudaStream_t st) {
  // (the statistics' scratch; the lambda-return forms take none)
  unsigned int* counter = reinterpret_cast<unsigned int*>(scratch);
  double2* partials = scratch ? reinterpret_cast<double2*>(reinterpret_cast<char*>(scratch) + 16) : nullptr;
  const int want = standardize != 0;
  int rc = 1;  // STX_OK once the TMA kernel has run; 1 while it has not
  // large PPO shapes: the TMA-pipelined persistent kernel (codes 500 / 501 force its 32x128 / 64x64 tiles, any other non-zero
  // code disables it; where it declines, the 5xx codes take the default selection below)
  if constexpr (std::is_same_v<In, PpoIn>) {
    if (vec4 && (g_tuning == 500 || g_tuning == 501 || (g_tuning == 0 && E >= 32768)))
      rc = launch_gae_tma(in, T, E, want, adv, tgt, stats, partials, counter, st);
  }
  if (rc < 0) return rc;
  const bool forced_quads = g_tuning == 2 || g_tuning == 4 || g_tuning == 8;
  if (rc == STX_OK) {
  } else if (vec4 && (g_tuning == 416 || (!forced_quads && E / 4 >= 65536))) {
    // saturating shapes: two resident 512-thread blocks per SM (code 416)
    const int grid = (E / 4 + 15) / 16;
    gae_scan_kernel<In, 4, 16, 4, 2><<<grid, 16 * kChunks, 0, st>>>(in, T, E, adv, tgt, want, partials, counter, stats);
  } else if (vec4) {
    // Small E is latency-bound: more, smaller blocks; wider rows per block once the grid is large.  Codes 2, 4, 8 force the quads.
    const int quads_total = E / 4;
    const int quads = forced_quads ? g_tuning : (quads_total >= 8 * kNumSMs * 2 ? 8 : (quads_total >= 4 * kNumSMs ? 4 : 2));
    const int grid = (quads_total + quads - 1) / quads;
    if (quads == 8)
      gae_scan_kernel<In, 4, 8><<<grid, 8 * kChunks, 0, st>>>(in, T, E, adv, tgt, want, partials, counter, stats);
    else if (quads == 4)
      gae_scan_kernel<In, 4, 4><<<grid, 4 * kChunks, 0, st>>>(in, T, E, adv, tgt, want, partials, counter, stats);
    else
      gae_scan_kernel<In, 4, 2><<<grid, 2 * kChunks, 0, st>>>(in, T, E, adv, tgt, want, partials, counter, stats);
  } else {
    const int grid = (E + 15) / 16;
    gae_scan_kernel<In, 1, 16><<<grid, 16 * kChunks, 0, st>>>(in, T, E, adv, tgt, want, partials, counter, stats);
  }
  STX_LAUNCH_OK();
  if (standardize == 2) {
    const int64_t n = (int64_t)T * E;
    const int grid = (int)((n + 1023) / 1024 < 4 * kNumSMs ? (n + 1023) / 1024 : 4 * kNumSMs);
    standardize_inplace_kernel<<<grid > 0 ? grid : 1, 256, 0, st>>>(adv, n, stats);
    STX_LAUNCH_OK();
  }
  return STX_OK;
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" size_t stx_gae_scratch_bytes(int T, int E) {
  (void)T;
  const size_t blocks = (size_t)(E > 0 ? E : 1) / 8 + 2;  // smallest block covers 8 envs
  return 16 + blocks * sizeof(double2);
}

extern "C" int stx_gae_set_tuning(int code) {
  STX_REQUIRE(code == 0 || code == 2 || code == 4 || code == 8 || code == 416 || code == 500 || code == 501, STX_E_ARG,
              "stx_gae_set_tuning: unknown code %d", code);
  g_tuning = code;
  return STX_OK;
}

static int check_common(int T, int E, int standardize, const void* adv, const void* tgt,
                        const void* stats, const void* scratch) {
  STX_REQUIRE(T > 0 && E > 0, STX_E_ARG, "stx_gae: T=%d E=%d must be positive", T, E);
  STX_REQUIRE(adv && tgt, STX_E_ARG, "stx_gae: null output");
  STX_REQUIRE(standardize >= 0 && standardize <= 2, STX_E_ARG, "stx_gae: standardize=%d", standardize);
  STX_REQUIRE(standardize == 0 || (stats && scratch), STX_E_ARG, "stx_gae: stats/scratch required when standardising");
  return STX_OK;
}

extern "C" int stx_gae_ppo_f32(const float* reward, const float* v_tm1, const float* v_t,
                               const uint8_t* done, const uint8_t* truncated, int T, int E,
                               float gamma, float lambda_, float reward_scale, int standardize,
                               float* adv, float* targets, float* stats, void* scratch,
                               void* stream) {
  if (int rc = check_common(T, E, standardize, adv, targets, stats, scratch)) return rc;
  STX_REQUIRE(reward && v_tm1 && v_t && done && truncated, STX_E_ARG, "stx_gae_ppo_f32: null input");
  const bool vec4 = (E % 4 == 0) && aligned16(reward) && aligned16(v_tm1) && aligned16(v_t) &&
                    aligned16(adv) && aligned16(targets) &&
                    (reinterpret_cast<uintptr_t>(done) % 4 == 0) &&
                    (reinterpret_cast<uintptr_t>(truncated) % 4 == 0);
  PpoIn in{reward, v_tm1, v_t, done, truncated, gamma, lambda_, reward_scale};
  return launch_gae(in, T, E, vec4, standardize, adv, targets, stats, scratch, (cudaStream_t)stream);
}

extern "C" int stx_gae_generic_f32(const float* r_t, const float* discount_t, const float* lambda_t,
                                   float lambda_, const float* v_tm1, const float* v_t,
                                   const float* truncation_t, int T, int E, int standardize,
                                   float* adv, float* targets, float* stats, void* scratch,
                                   void* stream) {
  if (int rc = check_common(T, E, standardize, adv, targets, stats, scratch)) return rc;
  STX_REQUIRE(r_t && discount_t && v_tm1 && v_t, STX_E_ARG, "stx_gae_generic_f32: null input");
  const bool vec4 = (E % 4 == 0) && aligned16(adv) && aligned16(targets);
  GenericIn in{r_t, discount_t, lambda_t, v_tm1, v_t, truncation_t, lambda_};
  return launch_gae(in, T, E, vec4, standardize, adv, targets, stats, scratch, (cudaStream_t)stream);
}

extern "C" int stx_q_lambda_f32(const float* q_t, int A, const float* r_t, const uint8_t* done, const uint8_t* truncated, int T, int E,
                                float gamma, float lambda_, float* targets, void* stream) {
  STX_REQUIRE(q_t && r_t && done && truncated && targets, STX_E_ARG, "stx_q_lambda_f32: null pointer");
  STX_REQUIRE(T > 0 && E > 0 && A > 0, STX_E_ARG, "stx_q_lambda_f32: T=%d E=%d A=%d must be positive", T, E, A);
  LambdaIn in{q_t, r_t, nullptr, nullptr, done, truncated, A, gamma, lambda_, (int64_t)(T - 1) * E};
  const bool vec4 = (E % 4 == 0) && aligned16(targets);
  return launch_gae(in, T, E, vec4, 0, nullptr, targets, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int stx_lambda_returns_f32(const float* r_t, const float* discount_t, const float* v_t, int A, const float* lambda_t, float lambda_,
                                      int T, int E, float* targets, void* stream) {
  STX_REQUIRE(r_t && discount_t && v_t && targets, STX_E_ARG, "stx_lambda_returns_f32: null pointer");
  STX_REQUIRE(T > 0 && E > 0 && A > 0, STX_E_ARG, "stx_lambda_returns_f32: T=%d E=%d A=%d must be positive", T, E, A);
  LambdaIn in{v_t, r_t, discount_t, lambda_t, nullptr, nullptr, A, 0.f, lambda_, (int64_t)(T - 1) * E};
  const bool vec4 = (E % 4 == 0) && aligned16(targets);
  return launch_gae(in, T, E, vec4, 0, nullptr, targets, nullptr, nullptr, (cudaStream_t)stream);
}
