// fp32 CUDA-core GEMM family for the parity path (STX_PREC_F32).
//
// The reference is fp32 everywhere (SURVEY.md "facts"), so this path keeps every product and
// accumulation in fp32 and is what the tight-tolerance parity tests run.  The bf16 wgmma path
// (stx_tc_*.cu) is the throughput path.  Three flavours of one 64x64x16 register-tiled kernel:
//   FWD : U[m,n]  = sum_k H_prev[row(m),k] * W[k,n] (+ b[n])                nn.Dense, torso.py:26
//   DX  : dU_prev[m,k] = (sum_n dY[m,n] * W[k,n]) * f'(U_prev[m,k])         backward through the activation (no-LayerNorm torso)
//   DW  : dWp[z][k,n] = sum_{m in slice z} H_prev[row(m),k] * dY[m,n],  dbp[z][n] = sum dY[m,n]
// Hidden layers keep BOTH the pre-activation U (the Dense output: f' and the LayerNorm backward are evaluated from it) and the
// layer output H the next GEMMs multiply, computed ONCE per element:
//   H = f(U)                               MLPTorso(activation=f): FWD epilogue               torso.py:31-32, networks/utils.py:9-24
//   H = f(LN(U) * scale + bias)            MLPTorso(use_layer_norm=True): ln_apply_kernel (Dense without bias, eps 1e-6) torso.py:26-30
// (rebuilding H on every operand load cost 8 redundant exp per element and made the small GEMMs transcendental-bound).
// All shapes are bounds-checked (D=4, A=2 of CartPole work).  Split-M partials of DW are reduced in
// a fixed order by reduce_partials_kernel -> run-to-run deterministic gradients.
#pragma once
#include "stx_common.cuh"

namespace stx {
namespace simt {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
constexpr int kThreads = (BM / TM) * (BN / TN);  // 256

enum Mode { FWD = 0, DX = 1, DW = 2 };

// Activation table of stoix/networks/utils.py:9-24 (flax.linen names): value and derivative from the pre-activation.
__device__ __forceinline__ float act_fwd(int kind, float z) {
  switch (kind) {
    case STX_ACT_RELU: return fmaxf(z, 0.f);
    case STX_ACT_TANH: return tanhf(z);
    case STX_ACT_SILU: return z / (1.f + expf(-z));
    case STX_ACT_ELU: return z > 0.f ? z : expm1f(z);
    case STX_ACT_GELU: {  // nn.gelu default approximate=True
      const float t = tanhf(0.7978845608028654f * (z + 0.044715f * z * z * z));
      return 0.5f * z * (1.f + t);
    }
    case STX_ACT_SIGMOID: return 1.f / (1.f + expf(-z));
    case STX_ACT_SOFTPLUS: return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z)));
    default: return z;  // identity / none
  }
}
__device__ __forceinline__ float act_grad(int kind, float z) {
  switch (kind) {
    case STX_ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case STX_ACT_TANH: {
      const float t = tanhf(z);
      return 1.f - t * t;
    }
    case STX_ACT_SILU: {
      const float s = 1.f / (1.f + expf(-z));
      return s * (1.f + z * (1.f - s));
    }
    case STX_ACT_ELU: return z > 0.f ? 1.f : expf(z);
    case STX_ACT_GELU: {
      const float c = 0.7978845608028654f, inner = c * (z + 0.044715f * z * z * z), t = tanhf(inner);
      return 0.5f * (1.f + t) + 0.5f * z * (1.f - t * t) * c * (1.f + 3.f * 0.044715f * z * z);
    }
    case STX_ACT_SIGMOID: {
      const float s = 1.f / (1.f + expf(-z));
      return s * (1.f - s);
    }
    case STX_ACT_SOFTPLUS: return 1.f / (1.f + expf(-z));
    default: return 1.f;
  }
}

struct GemmArgs {
  // FWD: A=H_prev (M x K, lda, optional row gather), B=W (K x N), C=U (M x N, nullable), C_act=f(U) (nullable)
  // DX : A=dY (M x Nr, lda=Nr), B=W (Kout x Nr) used transposed, C=dX (M x Kout), mask=U (M x Kout)
  // DW : A=H_prev (rows x Kout, gathered), B=dY (rows x N), C=partials [z][Kout x N]
  const float* A;
  const float* B;
  float* C;
  float* C_act;          // FWD: post-activation copy f(U) for the next layer's GEMMs (no-LayerNorm torsos); nullable
  int c_act;             // FWD: the activation of C_act
  const float* bias;     // FWD
  const float* mask;     // DX: pre-activation tensor of the producing layer (ld = N)
  const int32_t* rowidx; // FWD/DW: gather index for A rows (nullable)
  float* dbias;          // DW: partial db [z][N]
  int64_t M;             // FWD/DX: output rows.  DW: total sample rows (reduction length)
  int N;                 // output columns
  int K;                 // FWD: reduction (in dim).  DX: reduction (= layer out dim).  DW: output rows (in dim)
  int64_t lda;
  int mask_act;          // DX epilogue: activation whose derivative (from `mask` = U) multiplies the result; < 0: none
  int64_t rows_per_split;  // DW
  int64_t part_stride;   // DW: floats between split partials of this layer
  int64_t dbias_stride;  // DW
};

// Epilogue shared by both tilings: one output element.
template <int MODE>
__device__ __forceinline__ void store_out(const GemmArgs& g, int64_t m, int n, float acc) {
  if (MODE == FWD) {
    const float u = acc + (g.bias ? __ldg(g.bias + n) : 0.f);
    if (g.C) g.C[m * g.N + n] = u;                                   // pre-activation (backward: f' and LayerNorm need it)
    if (g.C_act) g.C_act[m * g.N + n] = act_fwd(g.c_act, u);         // what the next GEMM multiplies
  } else {
    const float d = (g.mask && g.mask_act >= 0) ? act_grad(g.mask_act, __ldg(g.mask + m * g.N + n)) : 1.f;
    g.C[m * g.N + n] = acc * d;
  }
}

// Register-tiled GEMM, one shared-memory stage + register prefetch: the global loads of step k+1 are issued before the products
// of step k and land in registers while the FMAs run.  64x64 output tiles, 16 values of the reduction per step, 4x4 outputs
// per thread.  (128x128 tiles with 8x8 outputs per thread measured slower.)
template <int MODE>
__global__ void __launch_bounds__(kThreads) gemm_kernel(GemmArgs g) {
  constexpr int LA = BM * BK / kThreads, LB = BN * BK / kThreads;
  static_assert(BM * BK % kThreads == 0 && BN * BK % kThreads == 0 && TN % 2 == 0 && TM % 4 == 0 && TN % 4 == 0, "tile shape");
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int64_t m0 = (int64_t)blockIdx.y * BM;  // output row tile
  const int n0 = blockIdx.x * BN;               // output col tile
  float2 acc[TM][TN / 2];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN / 2; ++j) acc[i][j] = make_float2(0.f, 0.f);
  float dbacc[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) dbacc[j] = 0.f;

  // reduction range
  int64_t r_begin = 0, r_end;
  if (MODE == DW) {
    r_begin = (int64_t)blockIdx.z * g.rows_per_split;
    r_end = r_begin + g.rows_per_split;
    if (r_end > g.M) r_end = g.M;
  } else {
    r_end = g.K;
  }
  const int out_rows = (MODE == DW) ? g.K : 0;  // DW: output rows = in-dim

  float va[LA], vb[LB];
  auto load_tiles = [&](int64_t r0) {   // all loads into registers (read-only path): nothing between them depends on shared memory
    if (MODE == FWD || MODE == DX) {    // A[row(m)][r0 + kk]: kk fastest in memory -> As[kk][m]
#pragma unroll
      for (int u = 0; u < LA; ++u) {
        const int i = tid + u * kThreads, kk = i % BK, mm = i / BK;
        const int64_t m = m0 + mm, k = r0 + kk;
        const bool ok = m < g.M && k < r_end;
        const int64_t row = ok ? ((MODE == FWD && g.rowidx) ? (int64_t)__ldg(g.rowidx + m) : m) : 0;
        va[u] = ok ? __ldg(g.A + row * g.lda + k) : 0.f;
      }
    } else {                            // DW: A(f, r) = H[row(r)][f]; f (feature) fastest in memory. As[kk = r][mm = f]
#pragma unroll
      for (int u = 0; u < LA; ++u) {
        const int i = tid + u * kThreads, mm = i % BM, kk = i / BM;
        const int64_t r = r0 + kk, f = m0 + mm;
        const bool ok = r < r_end && f < out_rows;
        const int64_t row = ok ? (g.rowidx ? (int64_t)__ldg(g.rowidx + r) : r) : 0;
        va[u] = ok ? __ldg(g.A + row * g.lda + f) : 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < LB; ++u) {
      const int i = tid + u * kThreads;
      if (MODE == DX) {                 // B(kk, j) = W[j][r0 + kk], W (Kout x Nr) row-major; reduction fastest in memory
        const int kk = i % BK, nn = i / BK;
        const int64_t k = r0 + kk;
        const int j = n0 + nn;
        vb[u] = (k < r_end && j < g.N) ? __ldg(g.B + (int64_t)j * g.K + k) : 0.f;
      } else {                          // FWD: W[k][n]; DW: dY[r][n]
        const int nn = i % BN, kk = i / BN;
        const int64_t k = r0 + kk;
        const int n = n0 + nn;
        vb[u] = (k < r_end && n < g.N) ? __ldg(g.B + k * g.N + n) : 0.f;
      }
    }
  };
  if (r_begin < r_end) load_tiles(r_begin);
  for (int64_t r0 = r_begin; r0 < r_end; r0 += BK) {
#pragma unroll
    for (int u = 0; u < LA; ++u) {
      const int i = tid + u * kThreads;
      if (MODE == DW) As[i / BM][i % BM] = va[u];
      else As[i % BK][i / BK] = va[u];
    }
#pragma unroll
    for (int u = 0; u < LB; ++u) {
      const int i = tid + u * kThreads;
      if (MODE == DX) Bs[i % BK][i / BK] = vb[u];
      else Bs[i / BN][i % BN] = vb[u];
    }
    __syncthreads();
    if (r0 + BK < r_end) load_tiles(r0 + BK);   // in flight under the products below
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
        a[i] = v.x, a[i + 1] = v.y, a[i + 2] = v.z, a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN + j]);
        b[j] = v.x, b[j + 1] = v.y, b[j + 2] = v.z, b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN / 2; ++j) fma2(acc[i][j], a[i], make_float2(b[2 * j], b[2 * j + 1]));
      if (MODE == DW) {
#pragma unroll
        for (int j = 0; j < TN; ++j) dbacc[j] += b[j];
      }
    }
    __syncthreads();
  }

  // ---- epilogue ----
  if (MODE != DW) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int64_t m = m0 + ty * TM + i;
      if (m >= g.M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        if (n < g.N) store_out<MODE>(g, m, n, (j & 1) ? acc[i][j / 2].y : acc[i][j / 2].x);
      }
    }
  } else {
    float* Cp = g.C + (int64_t)blockIdx.z * g.part_stride;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int64_t f = m0 + ty * TM + i;
      if (f >= out_rows) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        if (n < g.N) Cp[f * g.N + n] = (j & 1) ? acc[i][j / 2].y : acc[i][j / 2].x;
      }
    }
    if (blockIdx.y == 0 && ty == 0 && g.dbias) {
      float* dbp = g.dbias + (int64_t)blockIdx.z * g.dbias_stride;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        if (n < g.N) dbp[n] = dbacc[j];
      }
    }
  }
}

// ---- small-grid variant ------------------------------------------------------------------------------------------------
// When the 64x64 tiling above gives fewer CTAs than the GPU has SMs (batch-256 SAC epochs, 1024-env rollouts, heads), each CTA
// is a serial chain of K/16 load -> sync -> fma -> sync steps and the GEMM costs tens of microseconds of pure latency.  This
// variant uses 32x32 output tiles (4x the CTAs) and stages the WHOLE reduction panel (<= 256 at a time) in shared memory: every
// global load of both panels is in flight before the first shared store (ONE exposed memory latency), then the two halves of
// the CTA (128 threads each, 2x4 outputs per thread) take the even / odd k of the panel and their partial sums are added in a
// fixed order (even + odd) through shared memory => deterministic.
constexpr int PM = 32, PN = 32, PK = 256, PTM = 2, PTN = 4;
constexpr int kPanelHalf = (PM / PTM) * (PN / PTN);  // 128 threads cover the tile once
constexpr int kPanelThreads = 2 * kPanelHalf;        // 256
constexpr int kPanelWarps = kPanelThreads / 32;
constexpr int kAsLd = PM + 2, kBsLd = PN + 4;        // float2 / float4 aligned rows
constexpr uint32_t kPanelSmemBytes = PK * (kAsLd + kBsLd) * 4;
constexpr int kPanelLoads = PM * PK / kPanelThreads; // 32 per thread and panel

// Panel element owned by (thread, u) in the two global layouts:
//   reduction index fastest in memory (FWD-A, DX-A, DX-B): warp w takes tile rows w, w + 8, ..; lanes walk k  -> coalesced
//   tile column fastest in memory    (FWD-B, DW-A, DW-B): warp w takes panel rows w, w + 8, ..; lane = column -> coalesced
__device__ __forceinline__ void panel_coord_red(int u, int& mm, int& kk) {
  mm = (threadIdx.x >> 5) + kPanelWarps * (u / (PK / 32));
  kk = (threadIdx.x & 31) + 32 * (u % (PK / 32));
}
__device__ __forceinline__ void panel_coord_col(int u, int& mm, int& kk) {
  mm = threadIdx.x & 31;
  kk = (threadIdx.x >> 5) + kPanelWarps * u;
}

template <int MODE>
__global__ void __launch_bounds__(kPanelThreads) gemm_panel_kernel(GemmArgs g) {
  extern __shared__ __align__(16) float psm[];
  float* As = psm;               // [PK][kAsLd]: As[kk][m]
  float* Bs = psm + PK * kAsLd;  // [PK][kBsLd]: Bs[kk][n]
  const int tid = threadIdx.x;
  const int half = tid / kPanelHalf, t = tid % kPanelHalf;
  const int tx = t % (PN / PTN), ty = t / (PN / PTN);
  const int64_t m0 = (int64_t)blockIdx.y * PM;
  const int n0 = blockIdx.x * PN;
  float acc[PTM][PTN];
#pragma unroll
  for (int i = 0; i < PTM; ++i)
#pragma unroll
    for (int j = 0; j < PTN; ++j) acc[i][j] = 0.f;
  float dbacc[PTN] = {0.f, 0.f, 0.f, 0.f};

  int64_t r_begin = 0, r_end;
  if (MODE == DW) {
    r_begin = (int64_t)blockIdx.z * g.rows_per_split;
    r_end = r_begin + g.rows_per_split;
    if (r_end > g.M) r_end = g.M;
  } else {
    r_end = g.K;
  }
  const int out_rows = (MODE == DW) ? g.K : 0;

  for (int64_t r0 = r_begin; r0 < r_end; r0 += PK) {
    const int kc = (int)((r_end - r0) < PK ? (r_end - r0) : PK);
    float va[kPanelLoads], vb[kPanelLoads];
    // ---- A panel ----
#pragma unroll
    for (int u = 0; u < kPanelLoads; ++u) {
      int mm, kk;
      if (MODE == DW) {  // A(f, r) = H[row(r)][f]
        panel_coord_col(u, mm, kk);
        const int64_t f = m0 + mm;
        const bool ok = kk < kc && f < out_rows;
        const int64_t row = ok ? (g.rowidx ? (int64_t)__ldg(g.rowidx + r0 + kk) : r0 + kk) : 0;
        va[u] = ok ? __ldg(g.A + row * g.lda + f) : 0.f;
      } else {           // A[row(m)][r0 + kk]
        panel_coord_red(u, mm, kk);
        const int64_t m = m0 + mm;
        const bool ok = kk < kc && m < g.M;
        const int64_t row = ok ? ((MODE == FWD && g.rowidx) ? (int64_t)__ldg(g.rowidx + m) : m) : 0;
        va[u] = ok ? __ldg(g.A + row * g.lda + r0 + kk) : 0.f;
      }
    }
    // ---- B panel ----
#pragma unroll
    for (int u = 0; u < kPanelLoads; ++u) {
      int nn, kk;
      if (MODE == DX) {  // B(kk, j) = W[j][r0 + kk]
        panel_coord_red(u, nn, kk);
        const int j = n0 + nn;
        vb[u] = (kk < kc && j < g.N) ? __ldg(g.B + (int64_t)j * g.K + r0 + kk) : 0.f;
      } else {           // FWD: W[k][n]; DW: dY[r][n]
        panel_coord_col(u, nn, kk);
        const int n = n0 + nn;
        vb[u] = (kk < kc && n < g.N) ? __ldg(g.B + (r0 + kk) * g.N + n) : 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < kPanelLoads; ++u) {
      int mm, kk;
      if (MODE == DW) panel_coord_col(u, mm, kk);
      else panel_coord_red(u, mm, kk);
      if (kk < kc) As[kk * kAsLd + mm] = va[u];
    }
#pragma unroll
    for (int u = 0; u < kPanelLoads; ++u) {
      int nn, kk;
      if (MODE == DX) panel_coord_red(u, nn, kk);
      else panel_coord_col(u, nn, kk);
      if (kk < kc) Bs[kk * kBsLd + nn] = vb[u];
    }
    __syncthreads();
    float2 acc2[PTM][PTN / 2];
#pragma unroll
    for (int i = 0; i < PTM; ++i) acc2[i][0] = make_float2(acc[i][0], acc[i][1]), acc2[i][1] = make_float2(acc[i][2], acc[i][3]);
#pragma unroll 8
    for (int kk = half; kk < kc; kk += 2) {
      const float2 a = *reinterpret_cast<const float2*>(As + kk * kAsLd + ty * PTM);
      const float4 b = *reinterpret_cast<const float4*>(Bs + kk * kBsLd + tx * PTN);
      fma2(acc2[0][0], a.x, make_float2(b.x, b.y)), fma2(acc2[0][1], a.x, make_float2(b.z, b.w));
      fma2(acc2[1][0], a.y, make_float2(b.x, b.y)), fma2(acc2[1][1], a.y, make_float2(b.z, b.w));
      if (MODE == DW) dbacc[0] += b.x, dbacc[1] += b.y, dbacc[2] += b.z, dbacc[3] += b.w;
    }
#pragma unroll
    for (int i = 0; i < PTM; ++i) acc[i][0] = acc2[i][0].x, acc[i][1] = acc2[i][0].y, acc[i][2] = acc2[i][1].x, acc[i][3] = acc2[i][1].y;
    __syncthreads();
  }

  // ---- even-k half + odd-k half (fixed order), then the epilogue on the first half ----
  float* red = psm;  // [kPanelHalf][12]
  if (half == 1) {
    float* r = red + t * 12;
#pragma unroll
    for (int i = 0; i < PTM; ++i)
#pragma unroll
      for (int j = 0; j < PTN; ++j) r[i * PTN + j] = acc[i][j];
#pragma unroll
    for (int j = 0; j < PTN; ++j) r[8 + j] = dbacc[j];
  }
  __syncthreads();
  if (half == 1) return;
  {
    const float* r = red + t * 12;
#pragma unroll
    for (int i = 0; i < PTM; ++i)
#pragma unroll
      for (int j = 0; j < PTN; ++j) acc[i][j] += r[i * PTN + j];
#pragma unroll
    for (int j = 0; j < PTN; ++j) dbacc[j] += r[8 + j];
  }
  if (MODE != DW) {
#pragma unroll
    for (int i = 0; i < PTM; ++i) {
      const int64_t m = m0 + ty * PTM + i;
      if (m >= g.M) continue;
#pragma unroll
      for (int j = 0; j < PTN; ++j) {
        const int n = n0 + tx * PTN + j;
        if (n < g.N) store_out<MODE>(g, m, n, acc[i][j]);
      }
    }
  } else {
    float* Cp = g.C + (int64_t)blockIdx.z * g.part_stride;
#pragma unroll
    for (int i = 0; i < PTM; ++i) {
      const int64_t f = m0 + ty * PTM + i;
      if (f >= out_rows) continue;
#pragma unroll
      for (int j = 0; j < PTN; ++j) {
        const int n = n0 + tx * PTN + j;
        if (n < g.N) Cp[f * g.N + n] = acc[i][j];
      }
    }
    if (blockIdx.y == 0 && ty == 0 && g.dbias) {
      float* dbp = g.dbias + (int64_t)blockIdx.z * g.dbias_stride;
#pragma unroll
      for (int j = 0; j < PTN; ++j) {
        const int n = n0 + tx * PTN + j;
        if (n < g.N) dbp[n] = dbacc[j];
      }
    }
  }
}

// One entry point for the three GEMM flavours: picks the tiling from the grid the 64x64 kernel would get.
constexpr int kPanelBelowCtas = kNumSMs;
template <int MODE>
inline cudaError_t launch_gemm(const GemmArgs& g, int splits, cudaStream_t st) {
  const int64_t out_rows = (MODE == DW) ? g.K : g.M;
  const int64_t ctas64 = ((out_rows + BM - 1) / BM) * ((g.N + BN - 1) / BN) * (MODE == DW ? splits : 1);
  if (ctas64 >= kPanelBelowCtas) {
    dim3 grid((g.N + BN - 1) / BN, (unsigned)((out_rows + BM - 1) / BM), MODE == DW ? splits : 1);
    gemm_kernel<MODE><<<grid, kThreads, 0, st>>>(g);
    return cudaGetLastError();
  }
  cudaError_t e = opt_in_smem<gemm_panel_kernel<MODE>>(kPanelSmemBytes);
  if (e != cudaSuccess) return e;
  dim3 grid((g.N + PN - 1) / PN, (unsigned)((out_rows + PM - 1) / PM), MODE == DW ? splits : 1);
  gemm_panel_kernel<MODE><<<grid, kPanelThreads, kPanelSmemBytes, st>>>(g);
  return cudaGetLastError();
}

// grad[i] += w * sum_z part[z*stride + i]   (fixed order over z -> deterministic)
static __global__ void reduce_partials_kernel(const float* __restrict__ part, int splits, int64_t stride,
                                       int64_t n, float w, float* __restrict__ grad, int overwrite) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += part[(int64_t)z * stride + i];
  grad[i] = overwrite ? w * s : grad[i] + w * s;
}

// ---- LayerNorm (flax nn.LayerNorm defaults: epsilon 1e-6, scale + bias, over the feature axis) ---------------------
// per-row statistics of U (M x N): stats[m] = (mean, 1/sqrt(var + eps)) (nullable) and the layer output
// H[m] = f((U[m] - mean) * rstd * gamma + beta) that the next GEMM multiplies (H may alias U).  One warp per row.
static __global__ void ln_apply_kernel(const float* U, int64_t M, int N, const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                float* __restrict__ stats, float* H) {
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* u = U + row * N;
  float s = 0.f;
  for (int k = lane; k < N; k += 32) s += u[k];
  const float mean = warp_sum(s) / (float)N;
  float q = 0.f;
  for (int k = lane; k < N; k += 32) {
    const float d = u[k] - mean;
    q = fmaf(d, d, q);
  }
  const float var = warp_sum(q) / (float)N;
  const float rstd = rsqrtf(var + 1e-6f);
  if (lane == 0 && stats) stats[2 * row] = mean, stats[2 * row + 1] = rstd;
  float* h = H + row * N;
  for (int k = lane; k < N; k += 32) h[k] = act_fwd(act, (u[k] - mean) * rstd * __ldg(gamma + k) + __ldg(beta + k));
}

// Backward through h = f(z), z = uhat * gamma + beta, uhat = (u - mean) * rstd for the rows of one layer:
//   dz = dh * f'(z);  dgamma += sum_rows dz * uhat;  dbeta += sum_rows dz;  dhat = dz * gamma;
//   du = rstd * (dhat - mean_k(dhat) - uhat * mean_k(dhat * uhat))
// One warp per row; warp w of a block walks rows r0 + w, r0 + w + kLnWarps, ... in order and keeps its column sums of
// (dz * uhat | dz) in registers (lane l owns columns l, l + 32, ...); the warps' sums are merged through shared memory in
// warp order -> part[block][2N], reduced over blocks in a fixed order by reduce_partials_kernel: deterministic.
// D (M x N) holds dh on entry and du on exit.  N <= 32 * kLnMaxCols.
constexpr int kLnWarps = 8, kLnMaxCols = 32;
static __global__ void __launch_bounds__(32 * kLnWarps) ln_backward_kernel(float* __restrict__ D, const float* __restrict__ U,
                                                                  const float* __restrict__ stats, const float* __restrict__ gamma,
                                                                  const float* __restrict__ beta, int act, int64_t M, int N,
                                                                  int rows_per_block, float* __restrict__ part) {
  extern __shared__ float swarp[];  // [kLnWarps][2N]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float ag[kLnMaxCols], ab[kLnMaxCols];
#pragma unroll
  for (int j = 0; j < kLnMaxCols; ++j) ag[j] = 0.f, ab[j] = 0.f;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  for (int64_t row = r0 + warp; row < r0 + rows_per_block && row < M; row += kLnWarps) {
    const float mean = stats[2 * row], rstd = stats[2 * row + 1];
    float* d = D + row * N;
    const float* u = U + row * N;
    float s1 = 0.f, s2 = 0.f;
    for (int k = lane; k < N; k += 32) {
      const float uh = (u[k] - mean) * rstd;
      const float dhat = d[k] * act_grad(act, uh * gamma[k] + beta[k]) * gamma[k];
      s1 += dhat;
      s2 = fmaf(dhat, uh, s2);
    }
    s1 = warp_sum(s1) / (float)N;
    s2 = warp_sum(s2) / (float)N;
#pragma unroll
    for (int j = 0; j < kLnMaxCols; ++j) {
      const int k = lane + 32 * j;
      if (k < N) {
        const float uh = (u[k] - mean) * rstd;
        const float dz = d[k] * act_grad(act, uh * gamma[k] + beta[k]);
        d[k] = rstd * (dz * gamma[k] - s1 - uh * s2);
        ag[j] = fmaf(dz, uh, ag[j]);
        ab[j] += dz;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kLnMaxCols; ++j) {
    const int k = lane + 32 * j;
    if (k < N) swarp[(warp * 2 + 0) * N + k] = ag[j], swarp[(warp * 2 + 1) * N + k] = ab[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * N; i += blockDim.x) {
    const int which = i / N, k = i % N;
    float acc = 0.f;
    for (int w = 0; w < kLnWarps; ++w) acc += swarp[(w * 2 + which) * N + k];
    part[(int64_t)blockIdx.x * 2 * N + i] = acc;
  }
}

// ln_backward_kernel takes kLnWarps * 2N floats of dynamic shared memory: 64 KiB at the widest width check_mlp accepts
// (N = 32 * kLnMaxCols), more than the 48 KiB a launch may use without opting in (every width above 768).  The opt-in is made
// once per device for the largest size.
constexpr uint32_t kLnMaxSmemBytes = sizeof(float) * kLnWarps * 2 * 32 * kLnMaxCols;
static inline cudaError_t launch_ln_backward(float* D, const float* U, const float* stats, const float* gamma, const float* beta, int act, int64_t M,
                                      int N, int rows_per_block, int blocks, float* part, cudaStream_t st) {
  cudaError_t e = opt_in_smem<ln_backward_kernel>(kLnMaxSmemBytes);
  if (e != cudaSuccess) return e;
  ln_backward_kernel<<<blocks, 32 * kLnWarps, sizeof(float) * kLnWarps * 2 * N, st>>>(D, U, stats, gamma, beta, act, M, N, rows_per_block, part);
  return cudaGetLastError();
}

}  // namespace simt
}  // namespace stx
