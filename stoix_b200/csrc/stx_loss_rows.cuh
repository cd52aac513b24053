// What every fused loss kernel shares: the rows it reads (LossRows), its deterministic metric reduction (reduce_metrics), and
// the TD-error element of the Q losses (td_loss).  Used by the PPO / PQN / DQN losses (stx_ppo_loss.cuh, stx_ppo_fp32.cu) and
// the distributional Q losses (stx_distq.cu).
#pragma once
#include "stx_common.cuh"

namespace stx {

// The minibatch rows of a loss kernel and where it accumulates its metrics.
struct LossRows {
  const int32_t* idx;     // perm + mb_off (nullable -> row0 + m)
  int64_t row0, mb;
  double* partials;       // [grid][6] per-block metric partials
  unsigned int* counter;  // last-block ticket, zero between calls
  float* metrics;         // accumulated with weight
  float weight;
  __device__ __forceinline__ int64_t src(int64_t m) const { return idx ? (int64_t)idx[m] : row0 + m; }
};

// Deterministic metric reduction of the loss kernels: per-block partials, then the last block sums them in block order.
// Partial column k (of the 6 per block) feeds metrics[slot[k]].
template <int N>
__device__ __forceinline__ void reduce_metrics(const double (&v)[N], const int (&slot)[N], const LossRows& r) {
  __shared__ double sm[32];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const double s = block_sum<double>(v[k], sm);
    if (threadIdx.x == 0) r.partials[(int64_t)blockIdx.x * 6 + k] = s;
  }
  if (last_block_ticket(r.counter, gridDim.x)) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      double s = 0.0;
      for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) s += r.partials[(int64_t)i * 6 + k];
      s = block_sum<double>(s, sm);
      if (threadIdx.x == 0) r.metrics[slot[k]] += r.weight * (float)(s / (double)r.mb);
    }
  }
}

// ---- rlax.l2_loss / rlax.huber_loss of a TD error and d loss / d td, the element of every Q loss here (and of the quantile
// Huber loss, stx_distq.cu):
//   l2:    loss = td^2 / 2,                                       g = td
//   Huber: loss = q^2 / 2 + delta (|td| - q), q = min(|td|, delta),  g = clip(td, -delta, delta)   (delta > 0)
// so d loss / d q[a] = -g.  At |td| = delta both Huber branches give the same value (delta^2 / 2) and the same derivative
// (td = clip(td)), so the tie needs no rule.
__device__ __forceinline__ void td_loss(float td, float delta, float& loss, float& g) {
  if (delta > 0.f) {  // rlax.huber_loss
    const float ax = fabsf(td), quad = fminf(ax, delta), lin = ax - quad;
    loss = 0.5f * quad * quad + delta * lin;
    g = fminf(fmaxf(td, -delta), delta);
  } else {  // rlax.l2_loss
    loss = 0.5f * td * td;
    g = td;
  }
}

}  // namespace stx
