// IMPALA (stoix/systems/impala/sebulba/ff_impala.py) on sm_90a: the reward statistics of one learner batch and the fused V-trace
// loss of one minibatch (rlax.vtrace_td_error_and_advantage per env column, the summed critic and actor losses, their head
// gradients and metrics).  The rlax rules are restated in include/stx.h and tests/impala_oracle.py.  fp32 data; the metric sums are
// fp64 and reduced in a fixed order, so two launches on the same inputs give the same bits.
#include <algorithm>

#include "stx_common.cuh"

namespace stx {
namespace {

constexpr int kThreads = 128;                 // = rows of one time tile: thread i owns row t0 + i of its column
constexpr int kTile = kThreads;
constexpr unsigned kGrid = 2 * kNumSMs;       // column blocks beyond this loop over the columns
constexpr int kMetrics = STX_VTRACE_METRICS;  // actor_loss, entropy, value_loss, sum q_estimate, sum pg_advantage
constexpr int kStatsThreads = 1024;

struct VtraceScratch {
  double part[kGrid * kMetrics];
  unsigned int ticket;
};

// One launch over (T, E) rewards: mean and population std (two passes, fp64, one block: a fixed summation order).
__global__ void __launch_bounds__(kStatsThreads) reward_stats_kernel(const float* __restrict__ r, int T, int E, int64_t ld,
                                                                     float* __restrict__ stats) {
  __shared__ double sm[32];
  __shared__ double s_mean;
  const int64_t n = (int64_t)T * E;
  double s = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) s += (double)r[(k / E) * ld + k % E];
  s = block_sum<double>(s, sm);
  if (threadIdx.x == 0) s_mean = s / (double)n;
  __syncthreads();
  const double mean = s_mean;
  double q = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
    const double d = (double)r[(k / E) * ld + k % E] - mean;
    q += d * d;
  }
  q = block_sum<double>(q, sm);
  if (threadIdx.x == 0) {
    stats[0] = (float)mean;
    stats[1] = (float)sqrt(q / (double)n);
  }
}

// Block b walks the columns j = b, b + grid, ...; per column the time tiles from the last to the first.  Per tile: every thread
// takes one row (log-softmax, rho, entropy, reward, discount, values) into shared memory, thread 0 runs the reverse V-trace scan
// over the tile (carrying acc, vs_{t+1} and v_tm1_{t+1} from the tile after it), then every thread writes its row's head gradients.
__global__ void __launch_bounds__(kThreads) vtrace_loss_kernel(StxVtraceLoss a, VtraceScratch* sc) {
  __shared__ float s_rho[kTile], s_r[kTile], s_d[kTile], s_v[kTile], s_vn[kTile], s_err[kTile], s_pg[kTile], s_q[kTile];
  __shared__ double sm[32];
  const int A = a.A, Em = a.Em, T = a.T, i = threadIdx.x;
  const int64_t ld = a.ld;
  const bool norm = a.reward_stats != nullptr;
  const float r_mean = norm ? a.reward_stats[0] : 0.f, r_den = norm ? a.reward_stats[1] + a.reward_eps : 1.f;
  double m_actor = 0.0, m_ent = 0.0, m_vl = 0.0, m_q = 0.0, m_pg = 0.0;
  const int ntiles = (T + kTile - 1) / kTile;
  for (int j = blockIdx.x; j < Em; j += gridDim.x) {
    float acc = 0.f, vs_next = 0.f, v_next = 0.f;  // thread 0: the scan's carries across tiles
    for (int tile = ntiles - 1; tile >= 0; --tile) {
      const int t0 = tile * kTile, n = min(kTile, T - t0), t = t0 + i;
      const bool ok = i < n;
      const float* z = a.logits + ((int64_t)t * Em + j) * A;
      float lse = 0.f, ent = 0.f, lpa = 0.f;
      int act = 0;
      if (ok) {
        float mx = -INFINITY;
        for (int k = 0; k < A; ++k) mx = fmaxf(mx, z[k]);
        float s = 0.f;
        for (int k = 0; k < A; ++k) s += expf(z[k] - mx);
        lse = mx + logf(s);
        for (int k = 0; k < A; ++k) {
          const float lp = z[k] - lse;
          ent -= expf(lp) * lp;
        }
        const int64_t o = (int64_t)t * ld + j;
        act = a.action[o];
        lpa = z[act] - lse;
        float r = a.reward[o];
        if (norm) r = a.reward_scale * (r - r_mean) / r_den;
        s_rho[i] = expf(lpa - a.log_prob_b[o]);
        s_r[i] = r;
        s_d[i] = a.done[o] ? 0.f : a.gamma;
        s_v[i] = a.values[(int64_t)t * Em + j];
        s_vn[i] = a.values[(int64_t)(t + 1) * Em + j];
      }
      __syncthreads();
      if (i == 0) {
        for (int k = n - 1; k >= 0; --k) {
          const float rho = s_rho[k], r = s_r[k], d = s_d[k], v = s_v[k], vt = s_vn[k];
          const float c = fminf(1.f, rho) * a.lambda_;
          const float td = fminf(a.clip_rho, rho) * (r + d * vt - v);
          acc = td + d * c * acc;
          const float vs = acc + v;
          const float q = (t0 + k == T - 1) ? r + d * vt : r + d * (a.lambda_ * vs_next + (1.f - a.lambda_) * v_next);
          s_err[k] = vs - v;
          s_q[k] = q;
          s_pg[k] = fminf(a.clip_pg_rho, rho) * (q - v);
          vs_next = vs, v_next = v;
        }
      }
      __syncthreads();
      if (ok) {
        const float pg = s_pg[i], err = s_err[i];
        float* dz = a.d_logits + ((int64_t)t * Em + j) * A;
        for (int k = 0; k < A; ++k) {
          const float lp = z[k] - lse, p = expf(lp);
          dz[k] = -pg * ((k == act ? 1.f : 0.f) - p) + a.ent_coef * p * (lp + ent);
        }
        a.d_value[(int64_t)t * Em + j] = -a.vf_coef * err;
        m_actor -= (double)pg * (double)lpa;
        m_ent += (double)ent;
        m_vl += 0.5 * (double)err * (double)err;
        m_q += (double)s_q[i];
        m_pg += (double)pg;
      }
      __syncthreads();  // the next tile overwrites the shared rows
    }
    if (i == 0) a.d_value[(int64_t)T * Em + j] = 0.f;  // the bootstrap row gets no gradient
  }
  const double sums[kMetrics] = {m_actor, m_ent, m_vl, m_q, m_pg};
#pragma unroll
  for (int q = 0; q < kMetrics; ++q) {
    const double s = block_sum<double>(sums[q], sm);
    if (i == 0) sc->part[(size_t)blockIdx.x * kMetrics + q] = s;
  }
  if (!last_block_ticket(&sc->ticket, gridDim.x)) return;
  if (i < kMetrics) {
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += sc->part[(size_t)b * kMetrics + i];
    if (i >= 3) s /= (double)T * (double)Em;  // q_estimate and pg_advantage are reported as means
    a.metrics[i] = (float)s;
  }
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int stx_reward_stats(const float* reward, int T, int E, int64_t ld, float* stats, void* stream) {
  STX_REQUIRE(reward && stats, STX_E_ARG, "stx_reward_stats: null pointer");
  STX_REQUIRE(T >= 1 && E >= 1 && ld >= E, STX_E_SHAPE, "stx_reward_stats: T=%d E=%d ld=%lld", T, E, (long long)ld);
  reward_stats_kernel<<<1, kStatsThreads, 0, (cudaStream_t)stream>>>(reward, T, E, ld, stats);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" size_t stx_vtrace_loss_scratch_bytes(void) { return sizeof(VtraceScratch); }

extern "C" int stx_vtrace_loss_grads(const StxVtraceLoss* loss, void* scratch, void* stream) {
  STX_REQUIRE(loss && scratch, STX_E_ARG, "stx_vtrace_loss_grads: null pointer");
  const StxVtraceLoss a = *loss;
  STX_REQUIRE(a.logits && a.values && a.action && a.log_prob_b && a.reward && a.done && a.d_logits && a.d_value && a.metrics, STX_E_ARG,
              "stx_vtrace_loss_grads: null pointer");
  STX_REQUIRE(a.T >= 1 && a.Em >= 1 && a.A >= 1 && a.ld >= a.Em, STX_E_SHAPE, "stx_vtrace_loss_grads: T=%d Em=%d A=%d ld=%lld", a.T, a.Em,
              a.A, (long long)a.ld);
  const unsigned grid = (unsigned)std::min<int64_t>(a.Em, kGrid);
  vtrace_loss_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a, (VtraceScratch*)scratch);
  STX_LAUNCH_OK();
  return STX_OK;
}
