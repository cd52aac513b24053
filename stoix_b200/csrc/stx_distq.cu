// Distributional Q-learning (C51, QR-DQN): the expected-Q reduction of the two heads and the two fused loss + gradient kernels.
//
// Reference: DistributionalDiscreteQNetwork / QuantileDiscreteQNetwork (stoix/networks/heads.py:236-292), categorical_double_q_learning
// (stoix/utils/loss.py:81-103) with rlax.categorical_l2_project, and quantile_q_learning + quantile_regression_loss (:226-314), each
// under jax.grad as ff_c51.py:159-188 / ff_qr_dqn.py:159-202 call them.  Semantics and tie conventions: include/stx.h.
//
// Launch form of both losses: one row of the sampled batch is spread over TPR threads of a 256-thread CTA (TPR = 32, 64, 128, 256
// for N <= 32, <= 64, <= 128, larger; 256 / TPR rows per CTA).  Thread `lane` of a row owns columns lane, lane + TPR, ...; each
// owned column loops over the row's N partner columns (staged in shared memory) in index order, and every row-wide sum or max
// is a warp butterfly followed by the row's warp totals in warp order.  Nothing depends on scheduling, so two launches on the
// same inputs give the same bits.  A CTA's rows past M read row M - 1 and write nothing.
#include "stx_common.cuh"
#include "stx_loss_rows.cuh"

namespace stx {
namespace {

constexpr int kDistThreads = 256;

// Sum (MAX = false) or max over the TPR threads of this thread's row; every thread of the row gets the same bits (a + b = b + a
// in IEEE arithmetic, so the butterfly leaves one value in all lanes).  Synchronises the CTA: every thread must call it.
template <int TPR, bool MAX>
__device__ __forceinline__ float row_reduce(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, u) : v + u;
  }
  __syncthreads();  // the previous call's readers are done with `red`
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  constexpr int kW = TPR / 32;
  const int w0 = (threadIdx.x / TPR) * kW;
  float r = red[w0];
#pragma unroll
  for (int k = 1; k < kW; ++k) r = MAX ? fmaxf(r, red[w0 + k]) : r + red[w0 + k];
  return r;
}

// sum_i softmax(z)_i atoms_i in max-subtracted form, i in order.
__device__ __forceinline__ float categorical_expectation(const float* __restrict__ z, const float* __restrict__ atoms, int N) {
  float mx = z[0];
  for (int i = 1; i < N; ++i) mx = fmaxf(mx, z[i]);
  float s = 0.f;
  for (int i = 0; i < N; ++i) s += expf(z[i] - mx);
  float q = 0.f;
  for (int i = 0; i < N; ++i) q += (expf(z[i] - mx) / s) * atoms[i];
  return q;
}

// jnp.mean over the quantiles: (sum_i q_i) / N, i in order.  The QR loss's greedy selector uses the same expression.
__device__ __forceinline__ float quantile_mean(const float* __restrict__ q, int N) {
  float s = 0.f;
  for (int i = 0; i < N; ++i) s += q[i];
  return s / (float)N;
}

__global__ void __launch_bounds__(256) dist_q_values_kernel(int kind, const float* __restrict__ head, int64_t MA, int N,
                                                            const float* __restrict__ atoms, float* __restrict__ q) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;  // k = m A + a: its N columns start at k N
  if (k >= MA) return;
  q[k] = kind == STX_DIST_CATEGORICAL ? categorical_expectation(head + k * N, atoms, N) : quantile_mean(head + k * N, N);
}

struct DistRow {  // the row this thread works on, its reward and discount
  int64_t m, mm;  // row index; the row read (m clamped to M - 1)
  bool live;
  float r, d;
};

__device__ __forceinline__ DistRow dist_row(int TPR, int64_t M, const float* reward, const uint8_t* done, const float* discount,
                                            const StxDistQHyper& h) {
  DistRow w;
  w.m = (int64_t)blockIdx.x * (kDistThreads / TPR) + threadIdx.x / TPR;
  w.live = w.m < M;
  w.mm = w.live ? w.m : M - 1;
  w.r = fminf(fmaxf(reward[w.mm], -h.max_abs_reward), h.max_abs_reward);  // jnp.clip(reward, -max, max)
  w.d = discount ? discount[w.mm] : (1.f - (float)done[w.mm]) * h.gamma;  // (1 - done) gamma
  return w;
}

// Zero the row's A N gradient columns outside action a (the columns of a are written by their owners).
__device__ __forceinline__ void zero_other_actions(float* __restrict__ row, int a, int A, int N, int lane, int TPR) {
  const int64_t W = (int64_t)A * N, lo = (int64_t)a * N, hi = lo + N;
  for (int64_t k = lane; k < W; k += TPR)
    if (k < lo || k >= hi) row[k] = 0.f;
}

// ---- C51: categorical_double_q_learning.  Shared memory per row: clipped target atoms zp (N), target probabilities p (N), the
// projected target t (N, each entry touched by its owner only).  WEIGHTED (Rainbow): row m's gradient is scaled by w[m] and its
// metric term is w[m] loss; the unweighted instantiation is the kernel ff_c51 runs.
template <int TPR, bool WEIGHTED>
__global__ void __launch_bounds__(kDistThreads) categorical_q_loss_kernel(
    LossRows rows, const float* __restrict__ logits_tm1, const float* __restrict__ logits_t, const float* __restrict__ q_sel,
    const float* __restrict__ atoms_tm1, int64_t ld_tm1, const float* __restrict__ atoms_t, int64_t ld_t, const int32_t* __restrict__ action,
    const float* __restrict__ reward, const uint8_t* __restrict__ done, const float* __restrict__ discount, const float* __restrict__ row_w, int A,
    int N, StxDistQHyper h, float* __restrict__ d_logits, float* __restrict__ loss_rows) {
  extern __shared__ float smem[];
  __shared__ float red[kDistThreads / 32];
  const int lane = threadIdx.x % TPR;
  const DistRow w = dist_row(TPR, rows.mb, reward, done, discount, h);
  float* zp = smem + (threadIdx.x / TPR) * 3 * N;
  float* p = zp + N;
  float* t = p + N;
  const int64_t W = (int64_t)A * N;
  const float* zq = atoms_tm1 + w.mm * ld_tm1;
  const float* zt = atoms_t + w.mm * ld_t;
  const float vmin = zq[0], vmax = zq[N - 1];

  int best = 0;  // q_t_selector.argmax(-1): the first maximal index
  {
    const float* s = q_sel + w.mm * A;
    float bv = s[0];
    for (int j = 1; j < A; ++j)
      if (s[j] > bv) bv = s[j], best = j;
  }
  // p = softmax(logits_t[a*]) (jax.nn.softmax: exp(x - max) / sum), zp = clip(r + d atoms_t, vmin, vmax)
  const float* lt = logits_t + w.mm * W + (int64_t)best * N;
  float mx = -INFINITY;
  for (int k = lane; k < N; k += TPR) mx = fmaxf(mx, lt[k]);
  mx = row_reduce<TPR, true>(mx, red);
  float se = 0.f;
  for (int k = lane; k < N; k += TPR) {
    const float e = expf(lt[k] - mx);
    p[k] = e;
    se += e;
  }
  se = row_reduce<TPR, false>(se, red);
  for (int k = lane; k < N; k += TPR) {
    p[k] = p[k] / se;
    zp[k] = fminf(fmaxf(w.r + w.d * zt[k], vmin), vmax);
  }
  __syncthreads();

  // rlax.categorical_l2_project, gathered: t_i = sum_j clip(1 - delta_hat_ji, 0, 1) p_j, delta_ji = zp_j - zq_i,
  // delta_hat = delta d_pos_i (delta >= 0) or -delta d_neg_i (delta < 0); d_pos / d_neg are the inverse spacings to the next /
  // previous atom, 0 where that spacing is not positive (the wrapped neighbours at both ends, identical atoms).
  for (int i = lane; i < N; i += TPR) {
    const float z = zq[i];
    const float sp = (i + 1 < N ? zq[i + 1] : vmin) - z, sn = z - (i > 0 ? zq[i - 1] : vmax);
    const float dpos = sp > 0.f ? 1.f / sp : 0.f, dneg = sn > 0.f ? 1.f / sn : 0.f;
    float acc = 0.f;
    for (int j = 0; j < N; ++j) {
      const float delta = zp[j] - z;
      const float dh = delta >= 0.f ? delta * dpos : -(delta * dneg);
      acc += fminf(fmaxf(1.f - dh, 0.f), 1.f) * p[j];
    }
    t[i] = acc;
  }

  // cross-entropy against log_softmax(logits_tm1[a]) and its gradient
  const int a = action[w.mm];
  const float* la = logits_tm1 + w.mm * W + (int64_t)a * N;
  float lm = -INFINITY;
  for (int k = lane; k < N; k += TPR) lm = fmaxf(lm, la[k]);
  lm = row_reduce<TPR, true>(lm, red);
  float sa = 0.f, st = 0.f;
  for (int k = lane; k < N; k += TPR) {
    sa += expf(la[k] - lm);
    st += t[k];
  }
  sa = row_reduce<TPR, false>(sa, red);
  st = row_reduce<TPR, false>(st, red);
  const float lse = logf(sa);
  const float inv_m = 1.0f / (float)rows.mb;
  float ce = 0.f;
  for (int k = lane; k < N; k += TPR) {
    const float sh = la[k] - lm;
    ce += t[k] * (sh - lse);
    if (w.live) {
      const float g = ((expf(sh) / sa) * st - t[k]) * inv_m;
      d_logits[w.m * W + (int64_t)a * N + k] = WEIGHTED ? __fmul_rn(g, row_w[w.mm]) : g;
    }
  }
  const float loss = -row_reduce<TPR, false>(ce, red);
  if (w.live) {
    zero_other_actions(d_logits + w.m * W, a, A, N, lane, TPR);
    if (loss_rows && lane == 0) loss_rows[w.m] = loss;
  }
  const float term = WEIGHTED ? __fmul_rn(row_w[w.mm], loss) : loss;
  reduce_metrics<1>({(w.live && lane == 0) ? (double)term : 0.0}, {0}, rows);
}

// ---- QR-DQN: quantile_q_learning.  Shared memory per row: the target quantiles (N) and the selector means (A).
template <int TPR>
__global__ void __launch_bounds__(kDistThreads) quantile_q_loss_kernel(
    LossRows rows, const float* __restrict__ q_tm1, const float* __restrict__ q_t, const float* __restrict__ q_sel, const float* __restrict__ tau,
    int64_t ld_tau, const int32_t* __restrict__ action, const float* __restrict__ reward, const uint8_t* __restrict__ done,
    const float* __restrict__ discount, int A, int N, StxDistQHyper h, float* __restrict__ d_q, float* __restrict__ loss_rows) {
  extern __shared__ float smem[];
  __shared__ float red[kDistThreads / 32];
  const int lane = threadIdx.x % TPR;
  const DistRow w = dist_row(TPR, rows.mb, reward, done, discount, h);
  float* tgt = smem + (threadIdx.x / TPR) * (N + A);
  float* sel = tgt + N;
  const int64_t W = (int64_t)A * N;

  for (int b = lane; b < A; b += TPR) sel[b] = quantile_mean(q_sel + w.mm * W + (int64_t)b * N, N);
  __syncthreads();
  int best = 0;  // jnp.argmax(mean over quantiles): the first maximal index
  for (int b = 1; b < A; ++b)
    if (sel[b] > sel[best]) best = b;
  const float* qt = q_t + w.mm * W + (int64_t)best * N;
  for (int j = lane; j < N; j += TPR) tgt[j] = w.r + w.d * qt[j];
  __syncthreads();

  const int a = action[w.mm];
  const float* src = q_tm1 + w.mm * W + (int64_t)a * N;
  const float* tau_row = tau + w.mm * ld_tau;
  const float kappa = h.huber_delta, inv_n = 1.0f / (float)N, inv_m = 1.0f / (float)rows.mb;
  float part = 0.f;  // this thread's share of sum_i mean_j
  for (int i = lane; i < N; i += TPR) {
    const float s = src[i], ti = tau_row[i];
    float al = 0.f, ag = 0.f;
    for (int j = 0; j < N; ++j) {
      const float delta = tgt[j] - s;
      const float wt = fabsf(ti - (delta < 0.f ? 1.f : 0.f));  // delta_neg = (delta < 0): delta = 0 weighs tau_i
      float l, g;
      if (kappa > 0.f) {
        td_loss(delta, kappa, l, g);  // rlax.huber_loss and its derivative clip(delta, -kappa, kappa)
      } else {
        l = fabsf(delta);
        g = delta >= 0.f ? 1.f : -1.f;  // lax.abs's JVP: select(x >= 0, g, -g)
      }
      al += wt * l;
      ag += wt * g;
    }
    part += al / (float)N;
    if (w.live) d_q[w.m * W + (int64_t)a * N + i] = -(ag * inv_n) * inv_m;
  }
  const float loss = row_reduce<TPR, false>(part, red);
  if (w.live) {
    zero_other_actions(d_q + w.m * W, a, A, N, lane, TPR);
    if (loss_rows && lane == 0) loss_rows[w.m] = loss;
  }
  reduce_metrics<1>({(w.live && lane == 0) ? (double)loss : 0.0}, {0}, rows);
}

// Threads per row by N (see the file comment); the same switch points for both losses.
int dist_tpr(int N) { return N <= 32 ? 32 : N <= 64 ? 64 : N <= 128 ? 128 : 256; }

LossRows dist_rows(int64_t M, float* metrics, float weight, void* scratch) {
  return {nullptr, 0, M, reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256), reinterpret_cast<unsigned int*>(scratch), metrics,
          weight};
}

int check_loss_args(const void* a, const void* b, const void* aux, const int32_t* action, const float* reward, const uint8_t* done,
                    const float* discount, int64_t M, int A, int N, const StxDistQHyper* hyper, const float* grad, const float* metrics,
                    const void* scratch, size_t smem, const char* who) {
  STX_REQUIRE(a && b && aux && action && reward && (done || discount) && hyper && grad && metrics && scratch, STX_E_ARG, "%s: null pointer", who);
  STX_REQUIRE(M > 0 && A > 0 && N > 0, STX_E_SHAPE, "%s: M=%lld A=%d N=%d", who, (long long)M, A, N);
  STX_REQUIRE(N <= STX_DIST_MAX_N && smem <= 48 * 1024, STX_E_SHAPE, "%s: N=%d A=%d need %zu bytes of shared memory per CTA (N <= %d)", who, N, A,
              smem, STX_DIST_MAX_N);
  return STX_OK;
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" size_t stx_dist_q_scratch_bytes(int64_t M) { return 256 + (size_t)(M > 0 ? M : 1) * 6 * sizeof(double); }

extern "C" int stx_dist_q_values(int kind, const float* head, int64_t M, int A, int N, const float* atoms, float* q, void* stream) {
  STX_REQUIRE(head && q && (kind != STX_DIST_CATEGORICAL || atoms), STX_E_ARG, "stx_dist_q_values: null pointer");
  STX_REQUIRE(kind == STX_DIST_CATEGORICAL || kind == STX_DIST_QUANTILE, STX_E_UNSUPPORTED, "stx_dist_q_values: kind %d", kind);
  STX_REQUIRE(M > 0 && A > 0 && N > 0, STX_E_SHAPE, "stx_dist_q_values: M=%lld A=%d N=%d", (long long)M, A, N);
  const int64_t MA = M * A;
  dist_q_values_kernel<<<(unsigned)((MA + 255) / 256), 256, 0, (cudaStream_t)stream>>>(kind, head, MA, N, atoms, q);
  STX_LAUNCH_OK();
  return STX_OK;
}

namespace stx {
namespace {
int categorical_loss(const float* logits_tm1, const float* logits_t, const float* q_sel, const float* atoms_tm1, int64_t ld_atoms_tm1,
                     const float* atoms_t, int64_t ld_atoms_t, const int32_t* action, const float* reward, const uint8_t* done, const float* discount,
                     const float* row_w, int64_t M, int A, int N, const StxDistQHyper* hyper, float* d_logits, float* loss_rows, float* metrics,
                     float weight, void* scratch, void* stream, const char* who) {
  const int tpr = dist_tpr(N);
  const size_t smem = (size_t)(kDistThreads / tpr) * 3 * (size_t)N * sizeof(float);
  if (int rc = check_loss_args(logits_tm1, logits_t, q_sel, action, reward, done, discount, M, A, N, hyper, d_logits, metrics, scratch, smem, who))
    return rc;
  STX_REQUIRE(atoms_tm1 && atoms_t && ld_atoms_tm1 >= 0 && ld_atoms_t >= 0, STX_E_ARG, "%s: null atoms or negative row stride", who);
  const LossRows r = dist_rows(M, metrics, weight, scratch);
  const unsigned grid = (unsigned)((M + kDistThreads / tpr - 1) / (kDistThreads / tpr));
  cudaStream_t st = (cudaStream_t)stream;
  const StxDistQHyper h = *hyper;
#define STX_C51(T, WT)                                                                                                                       \
  categorical_q_loss_kernel<T, WT><<<grid, kDistThreads, smem, st>>>(r, logits_tm1, logits_t, q_sel, atoms_tm1, ld_atoms_tm1, atoms_t, ld_atoms_t, \
                                                                     action, reward, done, discount, row_w, A, N, h, d_logits, loss_rows)
#define STX_C51_TPR(WT)            \
  switch (tpr) {                   \
    case 32: STX_C51(32, WT); break;   \
    case 64: STX_C51(64, WT); break;   \
    case 128: STX_C51(128, WT); break; \
    default: STX_C51(256, WT); break;  \
  }
  if (row_w) {
    STX_C51_TPR(true)
  } else {
    STX_C51_TPR(false)
  }
#undef STX_C51_TPR
#undef STX_C51
  STX_LAUNCH_OK();
  return STX_OK;
}
}  // namespace
}  // namespace stx

extern "C" int stx_categorical_q_loss_grads(const float* logits_tm1, const float* logits_t, const float* q_sel, const float* atoms_tm1,
                                            int64_t ld_atoms_tm1, const float* atoms_t, int64_t ld_atoms_t, const int32_t* action,
                                            const float* reward, const uint8_t* done, const float* discount, int64_t M, int A, int N,
                                            const StxDistQHyper* hyper, float* d_logits, float* loss_rows, float* metrics, float weight,
                                            void* scratch, void* stream) {
  return categorical_loss(logits_tm1, logits_t, q_sel, atoms_tm1, ld_atoms_tm1, atoms_t, ld_atoms_t, action, reward, done, discount, nullptr, M, A, N,
                          hyper, d_logits, loss_rows, metrics, weight, scratch, stream, "stx_categorical_q_loss_grads");
}

extern "C" int stx_categorical_q_loss_grads_weighted(const float* logits_tm1, const float* logits_t, const float* q_sel, const float* atoms_tm1,
                                                     int64_t ld_atoms_tm1, const float* atoms_t, int64_t ld_atoms_t, const int32_t* action,
                                                     const float* reward, const uint8_t* done, const float* discount, const float* w, int64_t M, int A,
                                                     int N, const StxDistQHyper* hyper, float* d_logits, float* loss_rows, float* metrics, float weight,
                                                     void* scratch, void* stream) {
  return categorical_loss(logits_tm1, logits_t, q_sel, atoms_tm1, ld_atoms_tm1, atoms_t, ld_atoms_t, action, reward, done, discount, w, M, A, N, hyper,
                          d_logits, loss_rows, metrics, weight, scratch, stream, "stx_categorical_q_loss_grads_weighted");
}

extern "C" int stx_quantile_q_loss_grads(const float* q_tm1, const float* q_t, const float* q_sel, const float* tau, int64_t ld_tau,
                                         const int32_t* action, const float* reward, const uint8_t* done, const float* discount, int64_t M, int A,
                                         int N, const StxDistQHyper* hyper, float* d_q, float* loss_rows, float* metrics, float weight,
                                         void* scratch, void* stream) {
  const char* who = "stx_quantile_q_loss_grads";
  const int tpr = dist_tpr(N);
  const size_t smem = (size_t)(kDistThreads / tpr) * ((size_t)N + (size_t)A) * sizeof(float);
  if (int rc = check_loss_args(q_tm1, q_t, tau, action, reward, done, discount, M, A, N, hyper, d_q, metrics, scratch, smem, who)) return rc;
  STX_REQUIRE(ld_tau >= 0, STX_E_ARG, "%s: negative tau row stride", who);
  const LossRows r = dist_rows(M, metrics, weight, scratch);
  const unsigned grid = (unsigned)((M + kDistThreads / tpr - 1) / (kDistThreads / tpr));
  cudaStream_t st = (cudaStream_t)stream;
  const StxDistQHyper h = *hyper;
  const float* sel = q_sel ? q_sel : q_t;
#define STX_QR(T)                                                                                                                      \
  quantile_q_loss_kernel<T><<<grid, kDistThreads, smem, st>>>(r, q_tm1, q_t, sel, tau, ld_tau, action, reward, done, discount, A, N, h, d_q, \
                                                              loss_rows)
  switch (tpr) {
    case 32: STX_QR(32); break;
    case 64: STX_QR(64); break;
    case 128: STX_QR(128); break;
    default: STX_QR(256); break;
  }
#undef STX_QR
  STX_LAUNCH_OK();
  return STX_OK;
}
