// V-MPO (stoix/systems/mpo/ff_vmpo.py, ff_vmpo_continuous.py) on sm_90a: the exact top-half selection of the advantages, the fused
// rlax.vmpo_loss with its head and dual gradients (Categorical and tanh-Normal heads) and the critic's l2 value loss, the after-step
// dual clamp + periodic target copy, and batch_n_step_bootstrapped_returns.  The rlax rules are restated in tests/vmpo_oracle.py
// and include/stx.h.  fp32 data; every whole-shard sum is fp64 and reduced in a fixed order, so two launches give the same bits.
#include <algorithm>

#include "stx_common.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxKlCols = 2 * STX_VMPO_MAX_A;
constexpr int kPartStride = 6 + kMaxKlCols;  // per block: max, Z, sum e A, sum e logp, sum A, sum td^2 / 2, KL columns
constexpr unsigned kLossGrid = 2 * kNumSMs;
constexpr unsigned kTopkGrid = 4 * kNumSMs;
constexpr float kMpoFloatEpsilon = 1e-8f;  // _MPO_FLOAT_EPSILON (continuous_loss.py:19)
constexpr float kMinLogDual = -18.f;       // _MIN_LOG_TEMPERATURE = _MIN_LOG_ALPHA (continuous_loss.py:20-21)

// ---------------------------------------------------------------------------------------------------- exact top-k ----
// Order-preserving keys: a > b as floats (neither NaN) iff key(a) > key(b), except that key(+0) > key(-0).
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k); }

struct TopkScratch {
  uint32_t hist[2048];  // zero between passes: the last block of a pass clears it
  uint32_t ticket;
  uint32_t prefix;      // key bits found so far
  uint32_t k_rem;       // rank of the wanted key among the keys that share the prefix
  uint32_t pad;
};

// Radix pass p of 3 (key bits 31..21, 20..10, 9..0): histogram of the next bits of every key that shares the prefix, then the last
// block walks the bins from the top down to the one holding the k_rem-th largest key.  Integer counts: the result does not depend
// on the order of the atomics.
__global__ void __launch_bounds__(kThreads) topk_pass_kernel(const float* __restrict__ adv, int64_t n, uint32_t k, int pass, TopkScratch* st,
                                                             float* __restrict__ tau, int32_t* __restrict__ count) {
  const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
  const int bits = pass == 2 ? 10 : 11;
  const uint32_t nb = 1u << bits;
  const uint32_t pmask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + bits));
  const uint32_t prefix = pass == 0 ? 0u : st->prefix;
  __shared__ uint32_t h[2048];
  for (uint32_t b = threadIdx.x; b < nb; b += blockDim.x) h[b] = 0u;
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t key = order_key(adv[i]);
    if ((key & pmask) == prefix) atomicAdd(&h[(key >> shift) & (nb - 1u)], 1u);
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < nb; b += blockDim.x)
    if (h[b]) atomicAdd(&st->hist[b], h[b]);
  if (!last_block_ticket(&st->ticket, gridDim.x)) return;
  const uint32_t k_rem = pass == 0 ? k : st->k_rem;
  const uint32_t per = nb / kThreads;  // thread t owns bins nb-1-t*per down to nb-(t+1)*per
  uint32_t cnt[8], s = 0u;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    cnt[j] = 0u;
    if ((uint32_t)j < per) {
      const uint32_t b = nb - 1u - threadIdx.x * per - j;
      cnt[j] = st->hist[b];
      st->hist[b] = 0u;
      s += cnt[j];
    }
  }
  __shared__ uint32_t scan[kThreads];
  scan[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < kThreads; o <<= 1) {
    const uint32_t v = threadIdx.x >= (unsigned)o ? scan[threadIdx.x - o] : 0u;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  const uint32_t incl = scan[threadIdx.x], excl = incl - s;
  if (excl < k_rem && k_rem <= incl) {  // exactly one thread
    uint32_t c = excl;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if ((uint32_t)j >= per) break;
      if (c + cnt[j] >= k_rem) {
        const uint32_t p = prefix | ((nb - 1u - threadIdx.x * per - j) << shift);
        st->prefix = p;
        st->k_rem = k_rem - c;
        if (pass == 2) {
          *tau = key_float(p);
          *count = 0;
        }
        break;
      }
      c += cnt[j];
    }
  }
}

// mask = (adv >= tau) as floats (so -0 and +0 tie) and K = |mask|
__global__ void __launch_bounds__(kThreads) topk_mask_kernel(const float* __restrict__ adv, int64_t n, const float* __restrict__ tau,
                                                             uint8_t* __restrict__ mask, int32_t* __restrict__ count) {
  const float t = *tau;
  int c = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool sel = adv[i] >= t;
    mask[i] = sel ? 1 : 0;
    c += sel ? 1 : 0;
  }
  __shared__ int sm[32];
  c = block_sum<int>(c, sm);
  if (threadIdx.x == 0 && c) atomicAdd(count, c);
}

// ------------------------------------------------------------------------------------------------ the fused loss ----
struct LossScratch {
  double part[kLossGrid * kPartStride];
  double stats[4];  // m, Z for the weights
  unsigned int ticket;
};

__device__ __forceinline__ float dual_value(float x) { return softplusf(x) + kMpoFloatEpsilon; }

// Categorical row: log softmax normaliser of a row of A logits.
__device__ __forceinline__ float row_lse(const float* z, int A) {
  float mx = -INFINITY;
  for (int j = 0; j < A; ++j) mx = fmaxf(mx, z[j]);
  float s = 0.f;
  for (int j = 0; j < A; ++j) s += expf(z[j] - mx);
  return mx + logf(s);
}

__device__ __forceinline__ double block_max(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  double r = -INFINITY;
  for (int i = 0; i < kWarps; ++i) r = fmax(r, sm[i]);
  return r;
}

// Warp sum of a KL column into this warp's slot: one writer per slot, fixed order.
__device__ __forceinline__ void kl_col_add(double (*acc)[kMaxKlCols], int c, float v) {
  const double s = warp_sum<double>((double)v);
  if ((threadIdx.x & 31) == 0) acc[threadIdx.x >> 5][c] += s;
}

__device__ __forceinline__ void put_dual_grad(const StxVmpoLoss& a, int d, double g) {
  const float v = a.weight * (float)g;
  a.dual_grad[d] = a.overwrite ? v : a.dual_grad[d] + v;
}

// Pass over the shard: temperature statistics of the selected rows (per-block max, then sums rescaled to it), KL columns, the
// advantage and value-loss sums.  The last block combines the blocks in order and writes the dual gradients, the metrics and (m, Z).
template <bool kTanh>
__global__ void __launch_bounds__(kThreads) vmpo_stats_kernel(StxVmpoLoss a, LossScratch* sc) {
  const int A = a.A;
  const int ncol = kTanh ? (a.per_dim ? 2 * A : 2) : 1;
  const double eta = (double)dual_value(a.duals[0]), inv_eta = 1.0 / eta;
  __shared__ double acc[kWarps][kMaxKlCols];
  __shared__ double sm[32];
  for (int c = threadIdx.x; c < kWarps * kMaxKlCols; c += blockDim.x) (&acc[0][0])[c] = 0.0;
  const int64_t N = a.N, stride = (int64_t)gridDim.x * blockDim.x;
  double mb = -INFINITY;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride)
    if (a.mask[i]) mb = fmax(mb, (double)a.adv[i] * inv_eta);
  mb = block_max(mb, sm);
  const HeadGeom geo = head_geom(a.minimum, a.maximum, kTanhNormalEpsilon);
  double z = 0.0, ea = 0.0, elp = 0.0, sa = 0.0, td2 = 0.0;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < N; base += stride) {  // trip count uniform over the block
    const int64_t i = base + threadIdx.x;
    const bool ok = i < N;
    float logp = 0.f;
    if constexpr (kTanh) {
      const float* h = a.head + (ok ? i : 0) * 2 * A;
      const float* ht = a.head_target + (ok ? i : 0) * 2 * A;
      const float* act = a.action_cont + (ok ? i : 0) * A;
      float km_sum = 0.f, ks_sum = 0.f;
      for (int j = 0; j < A; ++j) {
        float km = 0.f, ks = 0.f;
        if (ok) {
          const float loc = h[j], sigma = softplusf(h[A + j]) + a.min_scale;
          const float loc_t = ht[j], sigma_t = softplusf(ht[A + j]) + a.min_scale;
          logp += tanh_normal_log_prob_given(loc, sigma, act[j], geo).lp;
          km = normal_kl(loc_t, sigma_t, loc, sigma_t).kl;
          ks = normal_kl(loc_t, sigma_t, loc_t, sigma).kl;
        }
        if (a.per_dim) {
          kl_col_add(acc, j, km);
          kl_col_add(acc, A + j, ks);
        } else {
          km_sum += km, ks_sum += ks;
        }
      }
      if (!a.per_dim) {
        kl_col_add(acc, 0, km_sum);
        kl_col_add(acc, 1, ks_sum);
      }
    } else {
      float kl = 0.f;
      if (ok) {
        const float* zo = a.head + i * A;
        const float* zt = a.head_target + i * A;
        const float lse = row_lse(zo, A), lse_t = row_lse(zt, A);
        logp = zo[a.action[i]] - lse;
        for (int j = 0; j < A; ++j) {
          const float lq = zt[j] - lse_t;
          kl += expf(lq) * (lq - (zo[j] - lse));
        }
      }
      kl_col_add(acc, 0, kl);
    }
    if (ok) {
      const float adv = a.adv[i], td = a.targets[i] - a.value[i];
      sa += (double)adv;
      td2 += 0.5 * (double)td * (double)td;
      if (a.mask[i]) {
        const double e = exp((double)adv * inv_eta - mb);
        z += e, ea += e * (double)adv, elp += e * (double)logp;
      }
    }
  }
  double* part = sc->part + (size_t)blockIdx.x * kPartStride;
  const double sums[5] = {z, ea, elp, sa, td2};
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    const double s = block_sum<double>(sums[q], sm);
    if (threadIdx.x == 0) part[1 + q] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) part[0] = mb;
  for (int c = threadIdx.x; c < ncol; c += blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += acc[w][c];
    part[6 + c] = s;
  }
  if (!last_block_ticket(&sc->ticket, gridDim.x)) return;

  // ---- last block: combine the blocks in block order ----
  const unsigned G = gridDim.x;
  double m = -INFINITY;
  for (unsigned b = 0; b < G; ++b) m = fmax(m, sc->part[(size_t)b * kPartStride]);
  __shared__ double tot[6 + kMaxKlCols];
  const int t = threadIdx.x;
  if (t < 5 + ncol) {
    double s = 0.0;
    for (unsigned b = 0; b < G; ++b) {
      const double* p = sc->part + (size_t)b * kPartStride;
      if (t < 3) {
        if (p[1] > 0.0) s += p[1 + t] * exp(p[0] - m);  // the temperature sums, rescaled from the block's max to m
      } else {
        s += p[1 + t];
      }
    }
    tot[1 + t] = s;
  }
  __syncthreads();
  if (t != 0) return;
  const double Z = tot[1], EA = tot[2], ELP = tot[3], SA = tot[4], TD2 = tot[5];
  const double invN = 1.0 / (double)N, K = (double)*a.count;
  sc->stats[0] = m, sc->stats[1] = Z;
  const float lt = a.duals[0];
  const double lse = log(Z) + m;
  const double loss_temperature = eta * ((double)a.epsilon + lse - log(K));
  const double g_eta = (double)a.epsilon + lse - log(K) - EA / Z / eta;
  const float w = a.weight;
  put_dual_grad(a, 0, g_eta * (double)sigmoidf_(lt));
  double loss_kl = 0.0, loss_alpha = 0.0, alpha_m = 0.0, alpha_s = 0.0;
  const int half = kTanh ? ncol / 2 : 1;  // columns [0, half) constrain the mean (or the Categorical KL), [half, ncol) the stddev
  for (int c = 0; c < ncol; ++c) {
    const float la = a.duals[1 + c];
    const double alpha = (double)dual_value(la), mean_kl = tot[6 + c] * invN;
    const double eps = c < half ? (double)a.epsilon_alpha : (double)a.epsilon_stddev;
    loss_kl += alpha * mean_kl;
    loss_alpha += alpha * (eps - mean_kl);
    put_dual_grad(a, 1 + c, (eps - mean_kl) * (double)sigmoidf_(la));
    if (c < half) alpha_m += alpha / (double)half;
    else alpha_s += alpha / (double)half;
  }
  float* mt = a.metrics;
  mt[0] += w * (float)(-ELP / Z), mt[1] += w * (float)loss_kl, mt[2] += w * (float)loss_alpha;
  mt[3] += w * (float)loss_temperature, mt[4] += w * (float)eta, mt[5] += w * (float)alpha_m, mt[6] += w * (float)alpha_s;
  mt[7] += w * (float)(SA * invN), mt[8] += w * (float)(TD2 * invN);
}

// Per row: w = exp(A / eta - m) / Z on the selected rows, d head of L_pi + L_kl, and d value of the l2 value loss.
template <bool kTanh>
__global__ void __launch_bounds__(kThreads) vmpo_grads_kernel(StxVmpoLoss a, const LossScratch* sc) {
  const int A = a.A;
  const double m = sc->stats[0], Z = sc->stats[1];
  const double inv_eta = 1.0 / (double)dual_value(a.duals[0]);
  const int64_t N = a.N, rows = a.value_rows > N ? a.value_rows : N;
  const float invN = 1.f / (float)N;
  const HeadGeom geo = head_geom(a.minimum, a.maximum, kTanhNormalEpsilon);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += stride) {
    if (a.d_value && i < a.value_rows) a.d_value[i] = i < N ? -(a.targets[i] - a.value[i]) * invN : 0.f;
    if (i >= N) continue;
    const float wi = a.mask[i] ? (float)(exp((double)a.adv[i] * inv_eta - m) / Z) : 0.f;
    if constexpr (kTanh) {
      const float* h = a.head + i * 2 * A;
      const float* ht = a.head_target + i * 2 * A;
      const float* act = a.action_cont + i * A;
      float* dh = a.d_head + i * 2 * A;
      for (int j = 0; j < A; ++j) {
        const int cm = a.per_dim ? j : 0, cs = a.per_dim ? A + j : 1;
        const float am = dual_value(a.duals[1 + cm]) * invN, as = dual_value(a.duals[1 + cs]) * invN;
        const float loc = h[j], raw = h[A + j], sigma = softplusf(raw) + a.min_scale;
        const float loc_t = ht[j], sigma_t = softplusf(ht[A + j]) + a.min_scale;
        const TanhNormalDim lp = tanh_normal_log_prob_given(loc, sigma, act[j], geo);
        const NormalKl km = normal_kl(loc_t, sigma_t, loc, sigma_t), ks = normal_kl(loc_t, sigma_t, loc_t, sigma);
        dh[j] = -wi * lp.d_loc + am * km.d_mu;
        dh[A + j] = (-wi * lp.d_sigma + as * ks.d_sigma) * sigmoidf_(raw);
      }
    } else {
      const float* zo = a.head + i * A;
      const float* zt = a.head_target + i * A;
      float* dz = a.d_head + i * A;
      const float lse = row_lse(zo, A), lse_t = row_lse(zt, A), an = dual_value(a.duals[1]) * invN;
      const int act = a.action[i];
      for (int j = 0; j < A; ++j) {
        const float p = expf(zo[j] - lse), q = expf(zt[j] - lse_t);
        dz[j] = -wi * ((j == act ? 1.f : 0.f) - p) + an * (p - q);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------- after step ----
__global__ void __launch_bounds__(kThreads) vmpo_after_step_kernel(float* __restrict__ duals, int n_dual, const float* __restrict__ online,
                                                                   float* __restrict__ target, int64_t P, const int32_t* __restrict__ count, int period) {
  const bool copy = (*count % period) == 0;
  const int64_t n = P > n_dual ? P : (int64_t)n_dual, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i < n_dual) {
      const float x = duals[i];
      duals[i] = x < kMinLogDual ? kMinLogDual : x;  // jnp.maximum(-18, x): a NaN stays NaN
    }
    if (copy && i < P) target[i] = online[i];
  }
}

// ------------------------------------------------------------------------------------------------- n-step returns ----
__global__ void __launch_bounds__(kThreads) n_step_returns_kernel(const float* __restrict__ r, const float* __restrict__ d, const float* __restrict__ v,
                                                                  const float* __restrict__ v_tm1, int T, int E, int n, float lam,
                                                                  float* __restrict__ targets, float* __restrict__ adv) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)T * E) return;
  const int t = (int)(idx / E), e = (int)(idx % E);
  const float v_last = v[(int64_t)(T - 1) * E + e];
  const int64_t t0 = (int64_t)t + n - 1;
  float g = t0 < T ? v[t0 * E + e] : v_last;  // v_t shifted by n, padded with its last value
  for (int i = n - 1; i >= 0; --i) {            // multistep.py:204-209, padded steps read r = 0, discount = 1, lambda = 1
    const int64_t s = (int64_t)t + i;
    const bool in = s < T;
    const float rr = in ? r[s * E + e] : 0.f, dd = in ? d[s * E + e] : 1.f, ll = in ? lam : 1.f, vv = in ? v[s * E + e] : v_last;
    g = __fadd_rn(rr, __fmul_rn(dd, __fadd_rn(__fmul_rn(__fsub_rn(1.f, ll), vv), __fmul_rn(ll, g))));
  }
  targets[idx] = g;
  if (adv) adv[idx] = __fsub_rn(g, v_tm1[idx]);
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" size_t stx_vmpo_topk_scratch_bytes(void) { return sizeof(TopkScratch); }

extern "C" int stx_vmpo_topk(const float* adv, int64_t N, int64_t k, float* tau, uint8_t* mask, int32_t* count, void* scratch, void* stream) {
  STX_REQUIRE(adv && tau && count && scratch, STX_E_ARG, "stx_vmpo_topk: null pointer");
  STX_REQUIRE(N >= 2 && N <= 0x7FFFFFFF, STX_E_SHAPE, "stx_vmpo_topk: N=%lld rows (2 .. 2^31-1; V-MPO needs rollout_length >= 2 and envs)",
              (long long)N);
  STX_REQUIRE(k >= 1 && k <= N, STX_E_ARG, "stx_vmpo_topk: k=%lld outside 1..N=%lld", (long long)k, (long long)N);
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)std::min<int64_t>((N + 8 * kThreads - 1) / (8 * kThreads), kTopkGrid);
  for (int pass = 0; pass < 3; ++pass) {
    topk_pass_kernel<<<grid, kThreads, 0, st>>>(adv, N, (uint32_t)k, pass, (TopkScratch*)scratch, tau, count);
    STX_LAUNCH_OK();
  }
  if (mask) {
    topk_mask_kernel<<<grid, kThreads, 0, st>>>(adv, N, tau, mask, count);
    STX_LAUNCH_OK();
  }
  return STX_OK;
}

extern "C" size_t stx_vmpo_loss_scratch_bytes(void) { return sizeof(LossScratch); }

extern "C" int stx_vmpo_loss_grads(const StxVmpoLoss* loss, void* scratch, void* stream) {
  STX_REQUIRE(loss && scratch, STX_E_ARG, "stx_vmpo_loss_grads: null pointer");
  const StxVmpoLoss a = *loss;
  const bool tanh = a.kind == STX_VMPO_TANH_NORMAL;
  STX_REQUIRE(a.kind == STX_VMPO_CATEGORICAL || tanh, STX_E_UNSUPPORTED, "stx_vmpo_loss_grads: kind %d", a.kind);
  STX_REQUIRE(a.N >= 2, STX_E_SHAPE, "stx_vmpo_loss_grads: N=%lld rows (at least 2)", (long long)a.N);
  STX_REQUIRE(a.A >= 1 && a.A <= STX_VMPO_MAX_A, STX_E_SHAPE, "stx_vmpo_loss_grads: A=%d (1..%d)", a.A, STX_VMPO_MAX_A);
  STX_REQUIRE(a.head && a.head_target && a.adv && a.mask && a.count && a.value && a.targets && a.duals && a.d_head && a.dual_grad && a.metrics,
              STX_E_ARG, "stx_vmpo_loss_grads: null pointer");
  STX_REQUIRE(tanh ? a.action_cont != nullptr : a.action != nullptr, STX_E_ARG, "stx_vmpo_loss_grads: null action");
  STX_REQUIRE(a.value_rows >= 0 && (a.value_rows == 0 || a.d_value), STX_E_ARG, "stx_vmpo_loss_grads: value_rows=%lld without d_value",
              (long long)a.value_rows);
  cudaStream_t st = (cudaStream_t)stream;
  LossScratch* sc = (LossScratch*)scratch;
  const unsigned grid = (unsigned)std::min<int64_t>((a.N + kThreads - 1) / kThreads, kLossGrid);
  const int64_t rows = std::max<int64_t>(a.N, a.value_rows);
  const unsigned grid_rows = (unsigned)std::min<int64_t>((rows + kThreads - 1) / kThreads, 8 * kNumSMs);
  if (tanh) {
    vmpo_stats_kernel<true><<<grid, kThreads, 0, st>>>(a, sc);
    STX_LAUNCH_OK();
    vmpo_grads_kernel<true><<<grid_rows, kThreads, 0, st>>>(a, sc);
  } else {
    vmpo_stats_kernel<false><<<grid, kThreads, 0, st>>>(a, sc);
    STX_LAUNCH_OK();
    vmpo_grads_kernel<false><<<grid_rows, kThreads, 0, st>>>(a, sc);
  }
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_vmpo_after_step(float* duals, int n_dual, const float* online, float* target, int64_t P, const int32_t* count, int period,
                                   void* stream) {
  STX_REQUIRE(duals && online && target && count, STX_E_ARG, "stx_vmpo_after_step: null pointer");
  STX_REQUIRE(n_dual >= 1 && P >= 1, STX_E_SHAPE, "stx_vmpo_after_step: n_dual=%d P=%lld", n_dual, (long long)P);
  STX_REQUIRE(period >= 1, STX_E_ARG, "stx_vmpo_after_step: actor_target_period=%d (at least 1)", period);
  const int64_t n = std::max<int64_t>(P, n_dual);
  const unsigned grid = (unsigned)std::min<int64_t>((n + kThreads - 1) / kThreads, 8 * kNumSMs);
  vmpo_after_step_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(duals, n_dual, online, target, P, count, period);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_n_step_returns_f32(const float* r_t, const float* discount_t, const float* v_t, const float* v_tm1, int T, int E, int n,
                                      float lambda_, float* targets, float* adv, void* stream) {
  STX_REQUIRE(r_t && discount_t && v_t && targets && (!adv || v_tm1), STX_E_ARG, "stx_n_step_returns_f32: null pointer");
  STX_REQUIRE(T >= 1 && E >= 1, STX_E_SHAPE, "stx_n_step_returns_f32: T=%d E=%d", T, E);
  STX_REQUIRE(n >= 1, STX_E_ARG, "stx_n_step_returns_f32: n=%d (at least 1)", n);
  const int64_t total = (int64_t)T * E;
  n_step_returns_kernel<<<(unsigned)((total + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(r_t, discount_t, v_t, v_tm1, T, E, n,
                                                                                                                lambda_, targets, adv);
  STX_LAUNCH_OK();
  return STX_OK;
}
