// MPO (stoix/systems/mpo/ff_mpo.py, ff_mpo_continuous.py) on sm_90a: the time-major sequence replay ring, the per-state rows of the
// sampled-action target-Q evaluation, the fused categorical and decoupled tanh-Normal MPO losses with their head and dual gradients,
// Retrace targets and the Q loss gradient.
// Semantics: include/stx.h; the reference rules are restated in tests/mpo_oracle.py.  fp32 data; whole-batch sums are fp64 and
// reduced in a fixed order, so two launches on the same inputs give the same bits.
#include <algorithm>

#include "stx_common.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr unsigned kLossGrid = 2 * kNumSMs;
constexpr int kSums = 8;  // lse, sum w q, sum w (q - qbar) logpi_o, cross-entropy, KL, KL non-parametric, entropy online / target
constexpr int kPartStride = kSums + 2 * STX_MPO_MAX_A;  // + per-action min and max of q over the block's rows
constexpr uint32_t kSeqTag = 0x53455153u;  // "SEQS"
constexpr uint32_t kActTag = 0x4D504F41u;  // "MPOA"
constexpr float kMpoFloatEpsilon = 1e-8f;  // _MPO_FLOAT_EPSILON (discrete_loss.py:12)

__device__ __forceinline__ float mpo_dual(float x) { return softplusf(x) + kMpoFloatEpsilon; }

__device__ __forceinline__ float row_lse(const float* z, int A) {
  float mx = -INFINITY;
  for (int j = 0; j < A; ++j) mx = fmaxf(mx, z[j]);
  float s = 0.f;
  for (int j = 0; j < A; ++j) s += expf(z[j] - mx);
  return mx + logf(s);
}

// uniform integer in [0, n) from one random word
__device__ __forceinline__ int64_t uniform_int(uint32_t x, int64_t n) { return (int64_t)(((uint64_t)x * (uint64_t)n) >> 32); }

// ---------------------------------------------------------------------------------------------------------- the ring ----
// Row (t, e) of the (T, E) batch into ring row (w + t) mod L; one warp per row.  Only the newest L time rows of a longer batch.
__global__ void seq_write_kernel(StxSeqRing rb, const float* __restrict__ obs, const uint32_t* __restrict__ action, const float* __restrict__ reward,
                                 const uint8_t* __restrict__ done, const uint8_t* __restrict__ truncated, const float* __restrict__ log_prob, int T,
                                 int skip) {
  const int64_t E = rb.envs, r = skip * E + blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= (int64_t)T * E) return;
  const int lane = threadIdx.x & 31;
  const int64_t t = r / E, e = r % E;
  const int64_t slot = ((rb.state[0] + t) % rb.length) * E + e;
  const int D = rb.obs_dim;
  const int W = rb.act_words;
  for (int c = lane; c < D; c += 32) rb.obs[slot * D + c] = obs[r * D + c];
  for (int c = lane; c < W; c += 32) static_cast<uint32_t*>(rb.action)[slot * W + c] = action[r * W + c];
  if (lane == 0) {
    rb.reward[slot] = reward[r];
    rb.done[slot] = done[r];
    rb.truncated[slot] = truncated[r];
    rb.log_prob[slot] = log_prob[r];
  }
}

__global__ void seq_advance_kernel(StxSeqRing rb, int T) {
  rb.state[0] = (rb.state[0] + T) % rb.length;
  rb.state[1] = min(rb.state[1] + (int64_t)T, rb.length);
}

// Sequence b: env e uniform in [0, E), start k uniform among the c - S + 1 valid starts counted from the oldest row w - c; rows
// t = 0 .. S-1 into the time-major (S, B) outputs.  One warp per (t, b).
__global__ void __launch_bounds__(256) seq_sample_kernel(StxSeqRing rb, int B, int S, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ counter,
                                                         const int32_t* __restrict__ idx_in, int32_t* __restrict__ idx_out, float* __restrict__ obs,
                                                         uint32_t* __restrict__ action, float* __restrict__ reward, uint8_t* __restrict__ done,
                                                         float* __restrict__ log_prob) {
  const int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= (int64_t)S * B) return;
  const int lane = threadIdx.x & 31;
  const int t = (int)(r / B), b = (int)(r % B);
  const int64_t L = rb.length, w = rb.state[0], c = rb.state[1];
  const int64_t n_valid = max(c - S + 1, (int64_t)1);
  int64_t e, k;
  if (idx_in) {
    e = idx_in[2 * b], k = idx_in[2 * b + 1];
  } else {
    const uint64_t call = offset + (counter ? *counter : 0ull);
    const uint4 wd = Philox::rand4(make_uint4((uint32_t)b, (uint32_t)call, (uint32_t)(call >> 32), kSeqTag),
                                   make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    e = uniform_int(wd.x, rb.envs), k = uniform_int(wd.y, n_valid);
  }
  const int64_t start = ((w - c + k) % L + L) % L;
  const int64_t slot = ((start + t) % L) * rb.envs + e;
  const int D = rb.obs_dim;
  const int W = rb.act_words;
  for (int cc = lane; cc < D; cc += 32) obs[r * D + cc] = rb.obs[slot * D + cc];
  for (int cc = lane; cc < W; cc += 32) action[r * W + cc] = static_cast<const uint32_t*>(rb.action)[slot * W + cc];
  if (lane == 0) {
    reward[r] = rb.reward[slot];
    done[r] = rb.done[slot];
    log_prob[r] = rb.log_prob[slot];
    if (idx_out && t == 0) idx_out[2 * b] = (int32_t)e, idx_out[2 * b + 1] = (int32_t)start;
  }
}

bool ring_ok(const StxSeqRing* rb) {
  return rb && rb->obs && rb->action && rb->reward && rb->done && rb->truncated && rb->log_prob && rb->state && rb->length > 0 && rb->envs > 0 &&
         rb->obs_dim > 0 && rb->act_words >= 1 && (int64_t)rb->envs * rb->length <= INT32_MAX;
}

// ------------------------------------------------------------------------------------------------ target-Q input rows ----
// One warp per row of xq ((A + N + 1) M, D + A): block j < A is [obs_i | one_hot(j)], block A + n is [obs_i | one_hot(a_ni)] with
// a_ni drawn from Categorical(logits_b[i]) (or its mode), block A + N is [obs_i | one_hot(action_i)].  The stored block's warp
// also writes log_rho, r and d of state i.
__global__ void __launch_bounds__(256) mpo_rows_kernel(StxMpoRows a, uint64_t call0, const uint64_t* __restrict__ counter) {
  const int64_t M = a.M, r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int A = a.A, N = a.N, D = a.D, W = D + A, NL = a.NL;
  if (r >= (int64_t)(NL + N + 1) * M) return;
  const int lane = threadIdx.x & 31;
  const int blk = (int)(r / M);
  const int64_t i = r % M;
  int act;
  if (blk < NL) {
    act = blk;
  } else if (blk < NL + N) {
    const int n = blk - NL;
    const float* z = a.logits_b + i * A;
    if (a.act_in) {
      act = a.act_in[(int64_t)n * M + i];
    } else if (!a.stochastic) {
      act = 0;  // the mode: the first maximum
      for (int j = 1; j < A; ++j)
        if (z[j] > z[act]) act = j;
    } else {
      const uint64_t call = call0 + (counter ? *counter : 0ull);
      const uint64_t ctr = (uint64_t)n * (uint64_t)M + (uint64_t)i;
      const uint4 wd = Philox::rand4(make_uint4((uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)call, kActTag ^ (uint32_t)(call >> 32)),
                                     make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
      const float u = u01(wd.x);
      const float lse = row_lse(z, A);
      // inverse CDF.  The fp32 sum can end below u (u01 reaches 1 - 2^-24): that remainder goes to the last action with positive
      // fp32 probability, never to an action whose probability has underflowed to 0
      float cum = 0.f;
      int last = 0;
      act = -1;
      for (int j = 0; j < A; ++j) {
        const float p = expf(z[j] - lse);
        if (p > 0.f) last = j;
        cum += p;
        if (u < cum) {
          act = j;
          break;
        }
      }
      if (act < 0) act = last;
    }
    if (lane == 0 && a.act_out) a.act_out[(int64_t)n * M + i] = act;
  } else {
    act = static_cast<const int32_t*>(a.action)[i];
    if (lane == 0) {
      const float* zt = a.logits_t + i * A;
      a.log_rho[i] = (zt[act] - row_lse(zt, A)) - a.log_prob[i];
      a.r[i] = fminf(fmaxf(a.reward[i], -a.max_abs_reward), a.max_abs_reward);
      a.d[i] = (1.f - (float)a.done[i]) * a.gamma;
    }
  }
  float* row = a.xq + r * W;
  const float* o = a.obs + i * D;
  for (int c = lane; c < W; c += 32) row[c] = c < D ? o[c] : (c - D == act ? 1.f : 0.f);
}


// tanh-Normal: one warp per row, lane c >= D writes action dimension j = c - D.  Block n < NL: a draw of the target policy (the
// unclipped value also to act_cont_out), block NL + n: a draw of the bootstrap policy or its mode, block NL + N: the stored action.
__global__ void __launch_bounds__(256) mpo_rows_tanh_kernel(StxMpoRows a, uint64_t call0, const uint64_t* __restrict__ counter) {
  const int64_t M = a.M, r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int A = a.A, N = a.N, D = a.D, W = D + A, NL = a.NL;
  if (r >= (int64_t)(NL + N + 1) * M) return;
  const int lane = threadIdx.x & 31;
  const int blk = (int)(r / M);
  const int64_t i = r % M;
  const HeadGeom geo = head_geom(a.minimum, a.maximum, kTanhNormalEpsilon);
  const uint64_t call = call0 + (counter ? *counter : 0ull);
  float* row = a.xq + r * W;
  const float* o = a.obs + i * D;
  for (int c = lane; c < W; c += 32) {
    if (c < D) {
      row[c] = o[c];
      continue;
    }
    const int j = c - D;
    float act;
    if (blk < NL + N) {
      const float* h = (blk < NL ? a.logits_t : a.logits_b) + i * 2 * A;
      const float loc = h[j], sigma = softplusf(h[A + j]) + a.min_scale;
      float u = loc;
      if (blk < NL || a.stochastic) {
        float e;
        if (a.eps_in) {
          e = a.eps_in[r * A + j];
        } else {
          const uint4 wd = Philox::rand4(make_uint4((uint32_t)r, (uint32_t)(r >> 32), (uint32_t)j, kActTag ^ (uint32_t)call),
                                         make_uint2((uint32_t)a.seed ^ (uint32_t)(call >> 32), (uint32_t)(a.seed >> 32)));
          e = normal2(wd.x, wd.y).x;
        }
        u = loc + sigma * e;
      }
      act = geo.sh + geo.s * tanhf(u);
      if (blk < NL) a.act_cont_out[r * A + j] = act;
    } else {
      act = static_cast<const float*>(a.action)[i * A + j];
    }
    row[c] = fminf(fmaxf(act, a.minimum), a.maximum);
  }
  if (blk == NL + N && lane == 0) {
    const float* ht = a.logits_t + i * 2 * A;
    const float* act = static_cast<const float*>(a.action) + i * A;
    float lp = 0.f;
    for (int j = 0; j < A; ++j) lp += tanh_normal_log_prob_given(ht[j], softplusf(ht[A + j]) + a.min_scale, act[j], geo).lp;
    a.log_rho[i] = lp - a.log_prob[i];
    a.r[i] = fminf(fmaxf(a.reward[i], -a.max_abs_reward), a.max_abs_reward);
    a.d[i] = (1.f - (float)a.done[i]) * a.gamma;
  }
}

// ------------------------------------------------------------------------------------------------- categorical loss ----
struct LossScratch {
  double part[kLossGrid * kPartStride];
  unsigned int ticket;
};

// One thread per state: its head gradient and the batch partial sums; the last block combines the blocks in block order and
// writes the dual gradients and the metrics.
__global__ void __launch_bounds__(kThreads) mpo_categorical_kernel(StxMpoLoss a, LossScratch* sc) {
  const int A = a.A, N = a.N;
  const int64_t M = a.M, stride = (int64_t)gridDim.x * blockDim.x;
  const float eta = mpo_dual(a.duals[0]), alpha = mpo_dual(a.duals[1]);
  const float inv_eta = 1.f / eta, invM = 1.f / (float)M;
  __shared__ double sm[32];
  __shared__ float qext[kWarps][2 * STX_MPO_MAX_A];
  double acc[kSums] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int c = threadIdx.x; c < kWarps * 2 * STX_MPO_MAX_A; c += blockDim.x) (&qext[0][0])[c] = (c % (2 * STX_MPO_MAX_A)) < STX_MPO_MAX_A ? INFINITY : -INFINITY;
  __syncthreads();
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < M; base += stride) {  // trip count uniform over the block
    const int64_t i = base + threadIdx.x;
    const bool ok = i < M;
    const int64_t ii = ok ? i : 0;
    const float* zo = a.head + ii * A;
    const float* zt = a.head_target + ii * A;
    const float lse_o = row_lse(zo, A), lse_t = row_lse(zt, A);
    float mu = -INFINITY;
    for (int j = 0; j < A; ++j) mu = fmaxf(mu, a.q[j * M + ii] * inv_eta + (zt[j] - lse_t));
    float su = 0.f;
    for (int j = 0; j < A; ++j) su += expf(a.q[j * M + ii] * inv_eta + (zt[j] - lse_t) - mu);
    const float lse_u = mu + logf(su);
    float wq = 0.f, ce = 0.f, kl = 0.f, klnp = 0.f, ent_o = 0.f, ent_t = 0.f;
    float* dz = a.d_head + ii * A;
    for (int j = 0; j < A; ++j) {
      const float q = a.q[j * M + ii], lpo = zo[j] - lse_o, lpt = zt[j] - lse_t;
      const float u = q * inv_eta + lpt, w = expf(u - lse_u), po = expf(lpo), pt = expf(lpt);
      wq += w * q, ce -= w * lpo, kl += pt * (lpt - lpo), klnp += w * (u - lse_u - lpt), ent_o -= po * lpo, ent_t -= pt * lpt;
      if (ok) dz[j] = invM * ((po - w) + alpha * (po - pt));
    }
    float wdq = 0.f;
    for (int j = 0; j < A; ++j) {
      const float q = a.q[j * M + ii], lpt = zt[j] - lse_t;
      wdq += expf(q * inv_eta + lpt - lse_u) * (q - wq) * (zo[j] - lse_o);
    }
    if (ok) {
      const float vals[kSums] = {lse_u, wq, wdq, ce, kl, klnp, ent_o, ent_t};
#pragma unroll
      for (int s = 0; s < kSums; ++s) acc[s] += (double)vals[s];
      if (a.q_boot && a.v) {
        float s = 0.f;
        for (int n = 0; n < N; ++n) s += a.q_boot[(int64_t)n * M + i];
        a.v[i] = __fdiv_rn(s, (float)N);
      }
    }
    // per-action min / max over the rows: warp reduce, one writer per (warp, column)
    for (int j = 0; j < A; ++j) {
      float lo = ok ? a.q[j * M + i] : INFINITY, hi = ok ? a.q[j * M + i] : -INFINITY;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)), hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      if ((threadIdx.x & 31) == 0) {
        float* qe = qext[threadIdx.x >> 5];
        qe[j] = fminf(qe[j], lo), qe[STX_MPO_MAX_A + j] = fmaxf(qe[STX_MPO_MAX_A + j], hi);
      }
    }
  }
  double* part = sc->part + (size_t)blockIdx.x * kPartStride;
#pragma unroll
  for (int s = 0; s < kSums; ++s) {
    const double v = block_sum<double>(acc[s], sm);
    if (threadIdx.x == 0) part[s] = v;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < A; j += blockDim.x) {
    float lo = INFINITY, hi = -INFINITY;
    for (int w = 0; w < kWarps; ++w) lo = fminf(lo, qext[w][j]), hi = fmaxf(hi, qext[w][STX_MPO_MAX_A + j]);
    part[kSums + j] = lo, part[kSums + STX_MPO_MAX_A + j] = hi;
  }
  if (!last_block_ticket(&sc->ticket, gridDim.x)) return;

  // ---- last block: combine the blocks in block order ----
  __shared__ double tot[kPartStride];
  const unsigned G = gridDim.x;
  for (int c = threadIdx.x; c < kSums + 2 * A; c += blockDim.x) {
    const int col = c < kSums ? c : (c < kSums + A ? c : c - A + STX_MPO_MAX_A);
    double s = c < kSums ? 0.0 : (c < kSums + A ? INFINITY : -INFINITY);
    for (unsigned b = 0; b < G; ++b) {
      const double p = sc->part[(size_t)b * kPartStride + col];
      s = c < kSums ? s + p : (c < kSums + A ? fmin(s, p) : fmax(s, p));
    }
    tot[col] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double invMd = 1.0 / (double)M, e = (double)eta, al = (double)alpha;
  const double m_lse = tot[0] * invMd, m_wq = tot[1] * invMd, m_wdq = tot[2] * invMd, m_ce = tot[3] * invMd, mean_kl = tot[4] * invMd;
  const double m_klnp = tot[5] * invMd, m_ento = tot[6] * invMd, m_entt = tot[7] * invMd;
  // d/d eta of eta (eps + mean lse) and of the cross-entropy through the E-step weights (discrete_loss.py:135-145, 74)
  const double g_eta = (double)a.epsilon + m_lse - m_wq / e + m_wdq / (e * e);
  const double g_alpha = (double)a.epsilon_policy - mean_kl;
  const double gs[2] = {g_eta * (double)sigmoidf_(a.duals[0]), g_alpha * (double)sigmoidf_(a.duals[1])};
  for (int d = 0; d < 2; ++d) {
    const float v = a.weight * (float)gs[d];
    a.dual_grad[d] = a.overwrite ? v : a.dual_grad[d] + v;
  }
  double qmin = 0.0, qmax = 0.0;
  for (int j = 0; j < A; ++j) qmin += tot[kSums + j], qmax += tot[kSums + STX_MPO_MAX_A + j];
  const double vals[STX_MPO_METRICS - 1] = {e, al, e * ((double)a.epsilon + m_lse), al * ((double)a.epsilon_policy - mean_kl), m_ce, al * mean_kl, m_klnp,
                                            m_ento, m_entt, mean_kl / (double)a.epsilon_policy, m_klnp / (double)a.epsilon, qmin / A, qmax / A};
  for (int k = 0; k < STX_MPO_METRICS - 1; ++k) a.metrics[k] += a.weight * (float)vals[k];
}


// Warp sum of a KL column into this warp's slot: one writer per slot, fixed order.
__device__ __forceinline__ void kl_col_add(double (*acc)[2 * STX_MPO_MAX_A], int c, float v) {
  const double s = warp_sum<double>((double)v);
  if ((threadIdx.x & 31) == 0) acc[threadIdx.x >> 5][c] += s;
}

// The decoupled MPO loss (continuous_loss.py:152-303): one thread per state; the last block combines the blocks in block order.
__global__ void __launch_bounds__(kThreads) mpo_tanh_kernel(StxMpoLoss a, LossScratch* sc) {
  const int A = a.A, N = a.N, NL = a.NL;
  const int half = a.per_dim ? A : 1, ncol = 2 * half;
  const int64_t M = a.M, stride = (int64_t)gridDim.x * blockDim.x;
  const float eta = mpo_dual(a.duals[0]), inv_eta = 1.f / eta, invM = 1.f / (float)M;
  const HeadGeom geo = head_geom(a.minimum, a.maximum, kTanhNormalEpsilon);
  __shared__ double sm[32];
  __shared__ double acc[kWarps][2 * STX_MPO_MAX_A];
  for (int c = threadIdx.x; c < kWarps * 2 * STX_MPO_MAX_A; c += blockDim.x) (&acc[0][0])[c] = 0.0;
  __syncthreads();
  double sums[5] = {0, 0, 0, 0, 0};  // lse, sum w q, KL non-parametric, cross-entropy (fixed stddev), cross-entropy (fixed mean)
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < M; base += stride) {  // trip count uniform over the block
    const int64_t i = base + threadIdx.x;
    const bool ok = i < M;
    const int64_t ii = ok ? i : 0;
    const float* q = a.q + ii;
    float mq = -INFINITY;
    for (int n = 0; n < NL; ++n) mq = fmaxf(mq, q[(int64_t)n * M] * inv_eta);
    float su = 0.f;
    for (int n = 0; n < NL; ++n) su += expf(q[(int64_t)n * M] * inv_eta - mq);
    const float lse = mq + logf(su);
    float wq = 0.f, klnp = 0.f;
    for (int n = 0; n < NL; ++n) {
      const float qn = q[(int64_t)n * M], w = expf(qn * inv_eta - lse);
      wq += w * qn, klnp += w * logf((float)NL * w + 1e-8f);
    }
    const float* h = a.head + ii * 2 * A;
    const float* ht = a.head_target + ii * 2 * A;
    float* dh = a.d_head + ii * 2 * A;
    float ce_m = 0.f, ce_s = 0.f, km_sum = 0.f, ks_sum = 0.f;
    for (int j = 0; j < A; ++j) {
      const float loc = h[j], raw = h[A + j], sigma = softplusf(raw) + a.min_scale;
      const float loc_t = ht[j], sigma_t = softplusf(ht[A + j]) + a.min_scale;
      float cm = 0.f, cs = 0.f, dl = 0.f, ds = 0.f;
      // the two cross-entropies in two passes: one log-probability per iteration keeps the loop within the registers
      for (int n = 0; n < NL; ++n) {
        const float w = expf(q[(int64_t)n * M] * inv_eta - lse);
        const TanhNormalDim pm = tanh_normal_log_prob_given(loc, sigma_t, a.actions[((int64_t)n * M + ii) * A + j], geo);
        cm -= w * pm.lp, dl -= w * pm.d_loc;
      }
      for (int n = 0; n < NL; ++n) {
        const float w = expf(q[(int64_t)n * M] * inv_eta - lse);
        const TanhNormalDim ps = tanh_normal_log_prob_given(loc_t, sigma, a.actions[((int64_t)n * M + ii) * A + j], geo);
        cs -= w * ps.lp, ds -= w * ps.d_sigma;
      }
      const NormalKl km = normal_kl(loc_t, sigma_t, loc, sigma_t), ks = normal_kl(loc_t, sigma_t, loc_t, sigma);
      const int c_m = a.per_dim ? j : 0, c_s = half + c_m;
      if (ok) {
        dh[j] = invM * (dl + mpo_dual(a.duals[1 + c_m]) * km.d_mu);
        dh[A + j] = invM * (ds + mpo_dual(a.duals[1 + c_s]) * ks.d_sigma) * sigmoidf_(raw);
      }
      ce_m += cm, ce_s += cs;
      if (a.per_dim) {
        kl_col_add(acc, c_m, ok ? km.kl : 0.f);
        kl_col_add(acc, c_s, ok ? ks.kl : 0.f);
      } else {
        km_sum += km.kl, ks_sum += ks.kl;
      }
    }
    if (!a.per_dim) {
      kl_col_add(acc, 0, ok ? km_sum : 0.f);
      kl_col_add(acc, 1, ok ? ks_sum : 0.f);
    }
    if (ok) {
      const float vals[5] = {lse, wq, klnp, ce_m, ce_s};
#pragma unroll
      for (int k = 0; k < 5; ++k) sums[k] += (double)vals[k];
      if (a.q_boot && a.v) {
        float s = 0.f;
        for (int n = 0; n < N; ++n) s += a.q_boot[(int64_t)n * M + i];
        a.v[i] = __fdiv_rn(s, (float)N);
      }
    }
  }
  double* part = sc->part + (size_t)blockIdx.x * kPartStride;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const double v = block_sum<double>(sums[k], sm);
    if (threadIdx.x == 0) part[k] = v;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < ncol; c += blockDim.x) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += acc[w][c];
    part[kSums + c] = t;
  }
  if (!last_block_ticket(&sc->ticket, gridDim.x)) return;

  __shared__ double tot[kPartStride];
  const unsigned G = gridDim.x;
  for (int c = threadIdx.x; c < kSums + ncol; c += blockDim.x) {
    if (c >= 5 && c < kSums) continue;
    double t = 0.0;
    for (unsigned b = 0; b < G; ++b) t += sc->part[(size_t)b * kPartStride + c];
    tot[c] = t;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double invMd = 1.0 / (double)M, e = (double)eta;
  const double m_lse = tot[0] * invMd, m_wq = tot[1] * invMd, m_klnp = tot[2] * invMd, m_cem = tot[3] * invMd, m_ces = tot[4] * invMd;
  const double log_nl = log((double)NL);
  const double g_eta = (double)a.epsilon + m_lse - log_nl - m_wq / e;
  const float w = a.weight;
  auto put = [&](int d, double g) {
    const float v = w * (float)g;
    a.dual_grad[d] = a.overwrite ? v : a.dual_grad[d] + v;
  };
  put(0, g_eta * (double)sigmoidf_(a.duals[0]));
  double al_m = 0, al_s = 0, la_m = 0, la_s = 0, lk_m = 0, lk_s = 0, kl_m = 0, kl_s = 0;
  for (int c = 0; c < ncol; ++c) {
    const double al = (double)mpo_dual(a.duals[1 + c]), kl = tot[kSums + c] * invMd;
    const double eps = c < half ? (double)a.epsilon_policy : (double)a.epsilon_stddev;
    put(1 + c, (eps - kl) * (double)sigmoidf_(a.duals[1 + c]));
    if (c < half) al_m += al / half, la_m += al * (eps - kl), lk_m += al * kl, kl_m += kl / half;
    else al_s += al / half, la_s += al * (eps - kl), lk_s += al * kl, kl_s += kl / half;
  }
  const double vals[STX_MPO_METRICS - 1] = {e, al_m, al_s, e * ((double)a.epsilon + m_lse - log_nl), la_m, la_s, m_cem, m_ces, lk_m, lk_s, kl_m, kl_s, m_klnp};
#pragma unroll
  for (int k = 0; k < STX_MPO_METRICS - 1; ++k) a.metrics[k] += w * (float)vals[k];
}

// -------------------------------------------------------------------------------------------------------- Retrace ----
// batch_general_off_policy_returns_from_q_and_v (multistep.py:210-267), time-major: g_{K-1} = r + d v, then for k = K-2 .. 0
// g_k = r_k + d_k ((v_k - c_k q_k) + c_k g_{k+1}) with c = lambda min(1, exp(log_rho)) (batch_retrace_continuous, :302).
__global__ void retrace_kernel(const float* __restrict__ q_t, const float* __restrict__ v_t, const float* __restrict__ r_t, const float* __restrict__ d_t,
                               const float* __restrict__ log_rho, const float* __restrict__ c_t, float lam, int K, int E, float* __restrict__ targets) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  auto at = [&](int k) { return (int64_t)k * E + e; };
  float g = __fadd_rn(r_t[at(K - 1)], __fmul_rn(d_t[at(K - 1)], v_t[at(K - 1)]));
  targets[at(K - 1)] = g;
  for (int k = K - 2; k >= 0; --k) {
    const float c = c_t ? c_t[at(k)] : __fmul_rn(fminf(1.f, expf(log_rho[at(k)])), lam);
    const float inner = __fadd_rn(__fsub_rn(v_t[at(k)], __fmul_rn(c, q_t[at(k)])), __fmul_rn(c, g));
    g = __fadd_rn(r_t[at(k)], __fmul_rn(d_t[at(k)], inner));
    targets[at(k)] = g;
  }
}

// ------------------------------------------------------------------------------------------------- Q loss gradient ----
// dq = (q - target) / (B (S-1)) on rows 0 .. S-2, 0 on row S-1; metric += weight * mean 0.5 (q - target)^2.  One block.
__global__ void __launch_bounds__(1024) q_grad_kernel(const float* __restrict__ q, const float* __restrict__ targets, int S, int B, float* __restrict__ dq,
                                                      float* __restrict__ metric, float weight) {
  __shared__ double sm[32];
  const int64_t n = (int64_t)(S - 1) * B, total = (int64_t)S * B;
  const float inv = 1.f / (float)n;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < total; i += blockDim.x) {
    if (i < n) {
      const float td = q[i] - targets[i];
      dq[i] = td * inv;
      s += 0.5 * (double)td * (double)td;
    } else {
      dq[i] = 0.f;
    }
  }
  s = block_sum<double>(s, sm);
  if (threadIdx.x == 0 && metric) *metric += weight * (float)(s / (double)n);
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int stx_replay_add_sequence(const StxSeqRing* rb, const float* obs, const void* action, const float* reward, const uint8_t* done,
                                       const uint8_t* truncated, const float* log_prob, int T, void* stream) {
  STX_REQUIRE(ring_ok(rb) && obs && action && reward && done && truncated && log_prob && T > 0, STX_E_ARG, "stx_replay_add_sequence: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int skip = T > rb->length ? T - (int)rb->length : 0;
  const int64_t rows = (int64_t)(T - skip) * rb->envs;
  seq_write_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(*rb, obs, (const uint32_t*)action, reward, done, truncated, log_prob, T, skip);
  STX_LAUNCH_OK();
  seq_advance_kernel<<<1, 1, 0, st>>>(*rb, T);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_replay_sample_sequence(const StxSeqRing* rb, int B, int S, int period, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                                          const int32_t* idx_in, int32_t* idx_out, float* obs, void* action, float* reward, uint8_t* done, float* log_prob,
                                          void* stream) {
  STX_REQUIRE(ring_ok(rb) && obs && action && reward && done && log_prob, STX_E_ARG, "stx_replay_sample_sequence: bad arguments");
  STX_REQUIRE(period == 1, STX_E_UNSUPPORTED, "stx_replay_sample_sequence: period=%d (only period 1 is implemented)", period);
  STX_REQUIRE(B > 0 && S > 0 && S <= rb->length, STX_E_SHAPE, "stx_replay_sample_sequence: B=%d S=%d with %lld time rows", B, S, (long long)rb->length);
  const int64_t rows = (int64_t)S * B;
  seq_sample_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(*rb, B, S, seed, offset, dev_counter, idx_in, idx_out, obs, (uint32_t*)action,
                                                                                 reward, done, log_prob);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_mpo_sample_actions(const StxMpoRows* rows, uint64_t offset, const uint64_t* dev_counter, void* stream) {
  STX_REQUIRE(rows, STX_E_ARG, "stx_mpo_sample_actions: null pointer");
  const StxMpoRows a = *rows;
  const bool tanh = a.kind == STX_MPO_TANH_NORMAL;
  STX_REQUIRE(a.kind == STX_MPO_CATEGORICAL || tanh, STX_E_UNSUPPORTED, "stx_mpo_sample_actions: kind %d", a.kind);
  STX_REQUIRE(a.M >= 1 && a.D >= 1 && a.A >= 1 && a.A <= STX_MPO_MAX_A && a.N >= 1 && a.NL >= 1 && (tanh || a.NL == a.A), STX_E_SHAPE,
              "stx_mpo_sample_actions: M=%lld D=%d A=%d N=%d NL=%d", (long long)a.M, a.D, a.A, a.N, a.NL);
  STX_REQUIRE(a.obs && a.logits_t && a.logits_b && a.action && a.log_prob && a.reward && a.done && a.xq && a.log_rho && a.r && a.d &&
                  (!tanh || a.act_cont_out),
              STX_E_ARG, "stx_mpo_sample_actions: null pointer");
  const int64_t n = (int64_t)(a.NL + a.N + 1) * a.M;
  if (tanh) mpo_rows_tanh_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a, offset, dev_counter);
  else mpo_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a, offset, dev_counter);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" size_t stx_mpo_loss_scratch_bytes(void) { return sizeof(LossScratch); }

extern "C" int stx_mpo_loss_grads(const StxMpoLoss* loss, void* scratch, void* stream) {
  STX_REQUIRE(loss && scratch, STX_E_ARG, "stx_mpo_loss_grads: null pointer");
  const StxMpoLoss a = *loss;
  const bool tanh = a.kind == STX_MPO_TANH_NORMAL;
  STX_REQUIRE(a.kind == STX_MPO_CATEGORICAL || tanh, STX_E_UNSUPPORTED, "stx_mpo_loss_grads: kind %d", a.kind);
  STX_REQUIRE(a.M >= 1 && a.A >= 1 && a.A <= STX_MPO_MAX_A && a.NL >= 1 && (tanh || a.NL == a.A), STX_E_SHAPE, "stx_mpo_loss_grads: M=%lld A=%d (1..%d) NL=%d",
              (long long)a.M, a.A, STX_MPO_MAX_A, a.NL);
  STX_REQUIRE(a.head && a.head_target && a.q && a.duals && a.d_head && a.dual_grad && a.metrics && (!tanh || a.actions), STX_E_ARG,
              "stx_mpo_loss_grads: null pointer");
  STX_REQUIRE(!a.q_boot || (a.v && a.N >= 1), STX_E_ARG, "stx_mpo_loss_grads: q_boot needs v and N >= 1");
  const unsigned grid = (unsigned)std::min<int64_t>((a.M + kThreads - 1) / kThreads, kLossGrid);
  if (tanh) mpo_tanh_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a, (LossScratch*)scratch);
  else mpo_categorical_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a, (LossScratch*)scratch);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_retrace_f32(const float* q_t, const float* v_t, const float* r_t, const float* discount_t, const float* log_rho, const float* c_t,
                               float lambda_, int K, int E, float* targets, void* stream) {
  STX_REQUIRE(v_t && r_t && discount_t && targets && (K < 2 || (q_t && (log_rho || c_t))), STX_E_ARG, "stx_retrace_f32: null pointer");
  STX_REQUIRE(K >= 1 && E >= 1, STX_E_SHAPE, "stx_retrace_f32: K=%d E=%d", K, E);
  retrace_kernel<<<(unsigned)((E + 127) / 128), 128, 0, (cudaStream_t)stream>>>(q_t, v_t, r_t, discount_t, log_rho, c_t, lambda_, K, E,
                                                                                                     targets);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_mpo_q_grad(const float* q, const float* targets, int S, int B, float* dq, float* metric, float weight, void* stream) {
  STX_REQUIRE(q && targets && dq, STX_E_ARG, "stx_mpo_q_grad: null pointer");
  STX_REQUIRE(S >= 2 && B >= 1, STX_E_SHAPE, "stx_mpo_q_grad: S=%d B=%d (S >= 2)", S, B);
  q_grad_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(q, targets, S, B, dq, metric, weight);
  STX_LAUNCH_OK();
  return STX_OK;
}
