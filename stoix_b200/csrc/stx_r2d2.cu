// R2D2 (stoix/systems/q_learning/rec_r2d2.py) on sm_90a: the prioritised sequence ring with a period, the dueling Q combine of
// DuelingQNetwork with its final LayerNorm, and the fused transformed n-step double-Q loss.
// Semantics: include/stx.h; the reference rules are restated in tests/r2d2_oracle.py.  The whole-batch sums are fp64 and reduced in a
// fixed order, so two launches on the same inputs give the same bits.
#include "stx_common.cuh"
#include "stx_prio_tree.cuh"

namespace stx {
namespace {


constexpr int kThreads = 256;
constexpr int kAddThreads = 512;   // the one CTA of an add or a set_priorities

// ---------------------------------------------------------------------------------------------------------- the ring ----
__host__ __device__ inline int64_t ring_items(const StxR2d2Ring& rb) { return (int64_t)rb.envs * (rb.length / rb.period); }

// Row (t, e) of the (T, E) batch into ring row (w + t) mod L; one warp per row, only the newest L time rows of a longer batch.  A
// row that starts an item also stores the carry entering the step.
__global__ void r2d2_write_kernel(StxR2d2Ring rb, const float* __restrict__ obs, const int32_t* __restrict__ action, const float* __restrict__ reward,
                                  const uint8_t* __restrict__ done, const uint8_t* __restrict__ truncated, const uint8_t* __restrict__ reset,
                                  const float* __restrict__ carry, int T, int skip) {
  const int64_t E = rb.envs, r = skip * E + blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= (int64_t)T * E) return;
  const int lane = threadIdx.x & 31;
  const int64_t t = r / E, e = r % E;
  const int64_t row = (rb.state[0] + t) % rb.length, slot = row * E + e;
  const int D = rb.obs_dim, Cd = rb.carry_dim;
  for (int c = lane; c < D; c += 32) rb.obs[slot * D + c] = obs[r * D + c];
  const int64_t K = rb.length / rb.period;
  if (row % rb.period == 0 && row / rb.period < K) {
    const int64_t cs = (row / rb.period) * E + e;
    for (int c = lane; c < Cd; c += 32) rb.carry[cs * Cd + c] = carry[r * Cd + c];
  }
  if (lane == 0) {
    rb.action[slot] = action[r];
    rb.reward[slot] = reward[r];
    rb.done[slot] = done[r];
    rb.truncated[slot] = truncated[r];
    rb.reset[slot] = reset[r];
  }
}

// The items whose rows the add touched (start rows w0 - S + 1 .. w0 + T - 1 mod L) get max_priority if valid, else 0; then every
// parent is rebuilt from its children, and the write index and fill count advance.  One CTA.
__global__ void __launch_bounds__(kAddThreads) r2d2_add_kernel(StxR2d2Ring rb, int T) {
  const int64_t L = rb.length, S = rb.seq_len, p = rb.period, K = L / p, items = ring_items(rb);
  const int64_t w0 = rb.state[0], w1 = (w0 + T) % L, c1 = min(rb.state[1] + (int64_t)T, L);
  const int64_t win = min((int64_t)T + S - 1, L), first = ((w0 - (S - 1)) % L + L) % L;
  const float maxp = *rb.max_priority;
  for (int64_t j = threadIdx.x; j < items; j += blockDim.x) {
    const int64_t start = (j % K) * p;
    if ((start - first + L) % L >= win) continue;
    const int64_t age = ((w1 - 1 - start) % L + L) % L;
    rb.tree[j] = (age >= S - 1 && age < c1) ? maxp : 0.f;
  }
  const int n = prio::tree_height(items);
  for (int l = 1; l < n; ++l) {
    __syncthreads();
    const int64_t cnt_ch = prio::level_count(items, l - 1), off_ch = prio::level_offset(items, l - 1);
    const int64_t cnt = prio::level_count(items, l), off = off_ch + cnt_ch;
    const float* ch = rb.tree + off_ch;
    for (int64_t node = threadIdx.x; node < cnt; node += blockDim.x) {
      const int64_t c0 = node * STX_PRIO_FANOUT, c1n = min(c0 + STX_PRIO_FANOUT, cnt_ch);
      float s = 0.f;
      for (int64_t c = c0; c < c1n; ++c) s = __fadd_rn(s, ch[c]);
      rb.tree[off + node] = s;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    rb.state[0] = w1;
    rb.state[1] = c1;
  }
}

struct R2d2Out {
  float *obs, *reward, *carry0, *prob;
  int32_t *action, *idx;
  uint8_t *done, *reset;
};

// One CTA per sequence b: warp 0 draws the stratum's item (one descent), then the warps copy its S rows, warp w rows w, w + 8, ...;
// the CTA also writes the item's carry, its index and p_i = leaf / total.
__global__ void __launch_bounds__(kThreads) r2d2_sample_kernel(StxR2d2Ring rb, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ counter,
                                                               const float* __restrict__ u_in, R2d2Out o) {
  __shared__ int64_t item;
  const int64_t b = blockIdx.x, B = gridDim.x, S = rb.seq_len, items = ring_items(rb);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0) {
    const uint64_t call = offset + (counter ? *counter : 0ull);
    const int64_t i = prio::tree_descend(rb.tree, items, b, prio::stratum_uniform(b, seed, call, u_in), B);
    if (lane == 0) {
      item = i;
      const float total = rb.tree[prio::root_offset(items)];
      o.idx[b] = (int32_t)i;
      o.prob[b] = total > 0.f ? __fdiv_rn(rb.tree[i], total) : 0.f;   // no valid item: every draw is item 0 with p 0
    }
  }
  __syncthreads();
  const int64_t L = rb.length, E = rb.envs, K = L / rb.period, e = item / K, k = item % K;
  const int D = rb.obs_dim, Cd = rb.carry_dim;
  for (int c = threadIdx.x; c < Cd; c += blockDim.x) o.carry0[b * Cd + c] = rb.carry[(k * E + e) * Cd + c];
  for (int64_t t = warp; t < S; t += blockDim.x >> 5) {
    const int64_t slot = ((k * rb.period + t) % L) * E + e, r = t * B + b;
    for (int c = lane; c < D; c += 32) o.obs[r * D + c] = rb.obs[slot * D + c];
    if (lane == 0) {
      o.action[r] = rb.action[slot];
      o.reward[r] = rb.reward[slot];
      o.done[r] = rb.done[slot];
      o.reset[r] = rb.reset[slot];
    }
  }
}

__global__ void __launch_bounds__(kAddThreads) r2d2_set_kernel(StxR2d2Ring rb, const int32_t* __restrict__ idx, const float* __restrict__ pr, int64_t M) {
  prio::set_priorities(rb.tree, rb.owner, rb.max_priority, rb.priority_exponent, ring_items(rb), idx, pr, M);
}

bool ring_ok(const StxR2d2Ring* rb) {
  return rb && rb->obs && rb->action && rb->reward && rb->done && rb->truncated && rb->reset && rb->carry && rb->tree && rb->state && rb->max_priority &&
         rb->owner && rb->length > 0 && rb->envs > 0 && rb->obs_dim > 0 && rb->carry_dim > 0 && rb->period > 0 && rb->period <= rb->length &&
         rb->seq_len > 0 && rb->seq_len <= rb->length && (int64_t)rb->envs * rb->length <= INT32_MAX;
}

// ------------------------------------------------------------------------------------------------ value transform ----
// rlax.SIGNED_HYPERBOLIC_PAIR, evaluated without cancellation near 0:
//   h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x             with sqrt(|x| + 1) - 1 = |x| / (sqrt(|x| + 1) + 1)
//   h^-1(x) = sign(x) (z^2 - 1), z = (sqrt(1 + 4 eps (eps + 1 + |x|)) - 1) / (2 eps), written as z = 1 + delta with
//   delta = 2 |x| (1 - 2 eps / (1 + 2 eps + s)) / (s + 1), s = sqrt(1 + 4 eps (eps + 1 + |x|)), and z^2 - 1 = delta (2 + delta).
__device__ __forceinline__ float tx_h(float x, float eps) {
  const float ax = fabsf(x);
  const float m = __fdiv_rn(ax, __fadd_rn(sqrtf(__fadd_rn(ax, 1.f)), 1.f));
  return __fadd_rn(copysignf(m, x), __fmul_rn(eps, x));
}

__device__ __forceinline__ float tx_h_inv(float x, float eps) {
  const float ax = fabsf(x);
  const float s = sqrtf(__fadd_rn(1.f, __fmul_rn(4.f * eps, __fadd_rn(eps + 1.f, ax))));
  const float f = __fsub_rn(1.f, __fdiv_rn(2.f * eps, __fadd_rn(1.f + 2.f * eps, s)));
  const float delta = __fdiv_rn(__fmul_rn(2.f * ax, f), __fadd_rn(s, 1.f));
  return copysignf(__fmul_rn(delta, __fadd_rn(2.f, delta)), x);
}

__global__ void tx_kernel(const float* __restrict__ x, int64_t n, int inverse, float eps, float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = inverse ? tx_h_inv(x[i], eps) : tx_h(x[i], eps);
}

// ------------------------------------------------------------------------------------------------------- the loss ----
constexpr int kPart = 5;  // per sequence: w_b loss_b, sum of online Q, priority, max_t |td|, mean_t |td|

// One CTA per sequence b.  Dynamic shared memory: v (T - 1) and td (T - 1) floats.
__global__ void __launch_bounds__(kThreads) r2d2_loss_kernel(StxR2d2Loss a, double* __restrict__ part, unsigned int* __restrict__ ticket) {
  extern __shared__ float sm[];
  __shared__ double red[kThreads];
  __shared__ float sh_w;
  const int b = blockIdx.x, T = a.T, B = a.B, A = a.A, n = a.n, seq = T - 1;
  float* v = sm;
  float* td = sm + seq;
  double qsum = 0.0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const float* q = a.q + ((int64_t)t * B + b) * A;
    int best = 0;
    for (int j = 0; j < A; ++j) {
      qsum += (double)q[j];
      if (q[j] > q[best]) best = j;  // jnp.argmax: the first maximum
    }
    if (t >= 1) v[t - 1] = a.q_target[((int64_t)t * B + b) * A + best];
  }
  red[threadIdx.x] = qsum;
  __syncthreads();
  for (int t = threadIdx.x; t < seq; t += blockDim.x) {
    // rlax.transformed_n_step_returns: targets start from v shifted by n - 1 (padded with its last value); then for i = n-1 .. 0,
    // targets = h(r_{t+i} + d_{t+i} h^-1(targets)), with r padded by zeros and d by ones past the window.
    float g = v[min(t + n - 1, seq - 1)];
    for (int i = n - 1; i >= 0; --i) {
      const int k = t + i;
      float r = 0.f, d = 1.f;
      if (k < seq) {
        const int64_t rk = (int64_t)k * B + b;
        r = fminf(fmaxf(a.reward[rk], -a.max_abs_reward), a.max_abs_reward);
        d = __fmul_rn(1.f - (float)a.done[rk], a.gamma);
      }
      g = tx_h(__fadd_rn(r, __fmul_rn(d, tx_h_inv(g, a.tx_eps))), a.tx_eps);
    }
    const int64_t rt = (int64_t)t * B + b;
    td[t] = __fsub_rn(g, a.q[rt * A + a.action[rt]]);
    if (a.td) a.td[rt] = td[t];
  }
  // beta = optax.linear_schedule(beta0 -> 1 over beta_steps) at the Adam count; w_b = (1 / (p_b + 1e-6))^beta / max over the batch
  float beta = a.beta0;
  if (a.beta_steps > 0.f) {
    const float c = fminf(fmaxf((float)(a.count ? *a.count : 0), 0.f), a.beta_steps);
    beta = __fadd_rn(__fmul_rn(a.beta0 - 1.f, 1.f - __fdiv_rn(c, a.beta_steps)), 1.f);
  }
  float mx = 0.f;
  for (int j = threadIdx.x; j < B; j += blockDim.x) mx = fmaxf(mx, powf(__fdiv_rn(1.f, __fadd_rn(a.prob[j], 1e-6f)), beta));
  for (int k = 16; k > 0; k >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, k));
  __shared__ float wmax[kThreads / 32];
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = wmax[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, wmax[k]);
    const float w = __fdiv_rn(powf(__fdiv_rn(1.f, __fadd_rn(a.prob[b], 1e-6f)), beta), m);
    double sq = 0.0, sabs = 0.0, qs = 0.0;
    float mabs = 0.f;
    for (int t = 0; t < seq; ++t) {
      sq += (double)td[t] * (double)td[t];
      sabs += (double)fabsf(td[t]);
      mabs = fmaxf(mabs, fabsf(td[t]));
    }
    for (int k = 0; k < (int)blockDim.x; ++k) qs += red[k];
    const double mean_abs = sabs / seq;
    const float pr = (float)((double)a.eta * mabs + (1.0 - (double)a.eta) * mean_abs);
    a.priorities[b] = pr;
    double* pb = part + (int64_t)b * kPart;
    pb[0] = (double)w * 0.5 * sq, pb[1] = qs, pb[2] = pr, pb[3] = mabs, pb[4] = mean_abs;
    sh_w = w;
  }
  __syncthreads();
  const float scale = __fdiv_rn(sh_w, (float)B);
  for (int k = threadIdx.x; k < T * A; k += blockDim.x) {
    const int t = k / A, j = k % A;
    const int64_t rt = (int64_t)t * B + b;
    a.d_q[rt * A + j] = (t < seq && j == a.action[rt]) ? -__fmul_rn(scale, td[t]) : 0.f;
  }
  if (!last_block_ticket(ticket, gridDim.x)) return;
  if (threadIdx.x < STX_R2D2_METRICS) {   // metric c: one fixed-order fp64 pass over the sequences' partials
    const int c = threadIdx.x, col = c <= 2 ? c : c - 1;   // partial columns: w loss, sum q, priority (max, then mean), max |td|, mean |td|
    double s = c == 2 ? -INFINITY : 0.0;
    for (int j = 0; j < B; ++j) {
      const double v = part[(int64_t)j * kPart + col];
      s = c == 2 ? fmax(s, v) : s + v;
    }
    const double m = c == 1 ? s / ((double)T * B * A) : (c == 2 ? s : s / B);
    a.metrics[c] += a.weight * (float)m;
  }
}

// ---------------------------------------------------------------------------------------------------------- dueling ----
__global__ void dueling_q_kernel(const float* __restrict__ adv, const float* __restrict__ value, int64_t M, int A, float* __restrict__ q) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* x = adv + m * A;
  float s = 0.f;
  for (int j = 0; j < A; ++j) s = __fadd_rn(s, x[j]);
  const float mean = __fdiv_rn(s, (float)A), v = *value;
  for (int j = 0; j < A; ++j) q[m * A + j] = __fadd_rn(v, __fsub_rn(x[j], mean));
}

// Block 0 reduces d value = sum over rows and actions of dq (each thread its rows in order, then the threads in order); the other
// blocks write d adv = dq - mean_a dq, one thread per row.
__global__ void __launch_bounds__(kThreads) dueling_q_backward_kernel(const float* __restrict__ dq, int64_t M, int A, float* __restrict__ d_adv,
                                                                      float* __restrict__ d_value, float weight, int overwrite) {
  if (blockIdx.x == 0) {
    __shared__ float red[kThreads];
    float s = 0.f;
    for (int64_t m = threadIdx.x; m < M; m += blockDim.x)
      for (int j = 0; j < A; ++j) s = __fadd_rn(s, dq[m * A + j]);
    red[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int k = 0; k < (int)blockDim.x; ++k) tot = __fadd_rn(tot, red[k]);
      *d_value = overwrite ? __fmul_rn(weight, tot) : __fadd_rn(*d_value, __fmul_rn(weight, tot));
    }
    return;
  }
  const int64_t m = (blockIdx.x - 1) * (int64_t)blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* g = dq + m * A;
  float s = 0.f;
  for (int j = 0; j < A; ++j) s = __fadd_rn(s, g[j]);
  const float mean = __fdiv_rn(s, (float)A);
  for (int j = 0; j < A; ++j) d_adv[m * A + j] = __fsub_rn(g[j], mean);
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int64_t stx_r2d2_tree_floats(const StxR2d2Ring* rb) {
  if (!rb || rb->period <= 0) return 0;
  return stx_prio_tree_floats(ring_items(*rb));
}

extern "C" int stx_r2d2_ring_add(const StxR2d2Ring* rb, const float* obs, const int32_t* action, const float* reward, const uint8_t* done,
                                 const uint8_t* truncated, const uint8_t* reset, const float* carry, int T, void* stream) {
  STX_REQUIRE(ring_ok(rb) && obs && action && reward && done && truncated && reset && carry && T > 0, STX_E_ARG, "stx_r2d2_ring_add: bad arguments");
  STX_REQUIRE(rb->length / rb->period >= 1, STX_E_SHAPE, "stx_r2d2_ring_add: no item fits L=%lld with period %d", (long long)rb->length, rb->period);
  cudaStream_t st = (cudaStream_t)stream;
  const int skip = T > rb->length ? T - (int)rb->length : 0;  // more rows than the ring holds: only the newest L survive
  const int64_t rows = (int64_t)(T - skip) * rb->envs;
  r2d2_write_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(*rb, obs, action, reward, done, truncated, reset, carry, T, skip);
  STX_LAUNCH_OK();
  r2d2_add_kernel<<<1, kAddThreads, 0, st>>>(*rb, T);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_r2d2_ring_sample(const StxR2d2Ring* rb, int B, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const float* u_in,
                                    float* obs, int32_t* action, float* reward, uint8_t* done, uint8_t* reset, float* carry0, int32_t* idx_out,
                                    float* prob_out, void* stream) {
  STX_REQUIRE(ring_ok(rb) && obs && action && reward && done && reset && carry0 && idx_out && prob_out && B > 0, STX_E_ARG,
              "stx_r2d2_ring_sample: bad arguments");
  const R2d2Out o{obs, reward, carry0, prob_out, action, idx_out, done, reset};
  r2d2_sample_kernel<<<(unsigned)B, kThreads, 0, (cudaStream_t)stream>>>(*rb, seed, offset, dev_counter, u_in, o);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_r2d2_ring_set_priorities(const StxR2d2Ring* rb, const int32_t* idx, const float* priorities, int64_t M, void* stream) {
  STX_REQUIRE(ring_ok(rb) && idx && priorities && M > 0 && M <= INT32_MAX, STX_E_ARG, "stx_r2d2_ring_set_priorities: bad arguments");
  r2d2_set_kernel<<<1, kAddThreads, 0, (cudaStream_t)stream>>>(*rb, idx, priorities, M);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_r2d2_value_transform(const float* x, int64_t n, int inverse, float eps, float* out, void* stream) {
  STX_REQUIRE(x && out && n > 0, STX_E_ARG, "stx_r2d2_value_transform: bad arguments");
  tx_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, n, inverse, eps, out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" size_t stx_r2d2_loss_scratch_bytes(int B) { return B > 0 ? 256 + sizeof(double) * kPart * (size_t)B : 0; }

extern "C" int stx_r2d2_loss_grads(const StxR2d2Loss* a, void* scratch, void* stream) {
  STX_REQUIRE(a && scratch && a->q && a->q_target && a->action && a->reward && a->done && a->prob && a->d_q && a->priorities && a->metrics, STX_E_ARG,
              "stx_r2d2_loss_grads: null pointer");
  STX_REQUIRE(a->T >= 2 && a->B > 0 && a->A > 0 && a->n >= 1 && a->tx_eps > 0.f, STX_E_SHAPE, "stx_r2d2_loss_grads: T=%d B=%d A=%d n=%d", a->T, a->B,
              a->A, a->n);
  const size_t smem = sizeof(float) * 2 * (size_t)(a->T - 1);
  STX_REQUIRE(smem <= 48 * 1024, STX_E_SHAPE, "stx_r2d2_loss_grads: learn window T=%d too long", a->T);
  char* s = reinterpret_cast<char*>(scratch);
  r2d2_loss_kernel<<<(unsigned)a->B, kThreads, smem, (cudaStream_t)stream>>>(*a, reinterpret_cast<double*>(s + 256),
                                                                              reinterpret_cast<unsigned int*>(s));
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_dueling_q(const float* adv, const float* value, int64_t M, int A, float* q, void* stream) {
  STX_REQUIRE(adv && value && q && M > 0 && A > 0, STX_E_ARG, "stx_dueling_q: bad arguments");
  dueling_q_kernel<<<(unsigned)((M + 255) / 256), 256, 0, (cudaStream_t)stream>>>(adv, value, M, A, q);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_dueling_q_backward(const float* d_q, int64_t M, int A, float* d_adv, float* d_value, float weight, int overwrite, void* stream) {
  STX_REQUIRE(d_q && d_adv && d_value && M > 0 && A > 0, STX_E_ARG, "stx_dueling_q_backward: bad arguments");
  dueling_q_backward_kernel<<<(unsigned)(1 + (M + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(d_q, M, A, d_adv, d_value, weight,
                                                                                                                   overwrite);
  STX_LAUNCH_OK();
  return STX_OK;
}
