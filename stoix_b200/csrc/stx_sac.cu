// ff_sac building blocks (fp32): tanh-Normal policy head, the three SAC loss heads, Polyak update, replay-buffer gather.
//
// Reference: stoix/systems/sac/ff_sac.py:149-321 (one `_update_epoch`), stoix/networks/heads.py:44-65
// (NormalAffineTanhDistributionHead: loc = Dense, scale = softplus(Dense) + min_scale), stoix/networks/distributions.py:19-79
// (AffineTanhTransformedDistribution: Normal -> tanh -> scale/shift onto [minimum, maximum]; log_prob clips the event to
// [minimum + eps, maximum - eps] and replaces the density in the two tails by log cdf / log survival minus log eps).
// tensorflow-probability (0.25.0) is not vendored in the reference; its pieces are restated from their published
// definitions: Normal.log_prob, log_cdf / log_survival_function, bijectors.Tanh.forward_log_det_jacobian(x) =
// 2 (log 2 - x - softplus(-2x)).  The networks themselves (silu MLPs, LayerNorm twin-Q) run on the generic train-mode MLP
// entry points of stx_mlp.cu; everything here is elementwise / row-wise and HBM- or latency-bound.
#include "stx_common.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {
namespace {

constexpr uint32_t kTagSac = 0x53414331u;

// One thread per row: action = shift + s tanh(loc + sigma eps) and log_prob (sum over the action dims).
// eps_in == nullptr: eps ~ N(0,1) from Philox keyed by (seed; row, call = offset + *counter, dim pair); eps_out keeps it.
__global__ void tanh_normal_sample_kernel(const float* __restrict__ head, int64_t M, int A, const float* __restrict__ eps_in,
                                          uint64_t seed, uint64_t offset, const uint64_t* __restrict__ counter, float minimum, float maximum,
                                          float min_scale, float epsilon, float* __restrict__ action, int64_t ld_action,
                                          float* __restrict__ log_prob, float* __restrict__ eps_out) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= M) return;
  const HeadGeom g = head_geom(minimum, maximum, epsilon);
  const uint64_t call = offset + (counter ? *counter : 0ull);
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  float lp = 0.f;
  for (int j0 = 0; j0 < A; j0 += 4) {
    float e[4];
    if (eps_in) {
      for (int k = 0; k < 4; ++k) e[k] = j0 + k < A ? eps_in[r * A + j0 + k] : 0.f;
    } else {
      const uint4 w = Philox::rand4(make_uint4((uint32_t)r, (uint32_t)call, (uint32_t)(call >> 32) ^ ((uint32_t)(j0 >> 2) << 20) ^
                                                                                  ((uint32_t)((uint64_t)r >> 32) << 8), kTagSac), key);
      const float2 n0 = normal2(w.x, w.y), n1 = normal2(w.z, w.w);
      e[0] = n0.x, e[1] = n0.y, e[2] = n1.x, e[3] = n1.y;
    }
    for (int k = 0; k < 4 && j0 + k < A; ++k) {
      const int j = j0 + k;
      const float loc = head[r * 2 * A + j], sigma = softplusf(head[r * 2 * A + A + j]) + min_scale;
      const float u = loc + sigma * e[k];
      const float a = g.sh + g.s * tanhf(u);
      float l;
      if (a <= g.lo) l = log_ndtrf((g.u_lo - loc) / sigma) - g.log_eps;
      else if (a >= g.hi) l = log_ndtrf(-(g.u_hi - loc) / sigma) - g.log_eps;
      else l = -0.5f * e[k] * e[k] - logf(sigma) - kLogSqrt2Pi - 2.f * (0.6931471805599453f - u - softplusf(-2.f * u)) - g.log_s;
      lp += l;
      action[r * ld_action + j] = a;
      if (eps_out) eps_out[r * A + j] = e[k];
    }
  }
  if (log_prob) log_prob[r] = lp;
}

// d(loss)/d(head output) for loss = g_logp * sum_rows log_prob + sum g_action . action, eps held fixed (reparameterisation).
__global__ void tanh_normal_backward_kernel(const float* __restrict__ head, const float* __restrict__ eps, int64_t M, int A, float minimum,
                                            float maximum, float min_scale, float epsilon, const float* __restrict__ log_alpha,
                                            float g_logp_scale, const float* __restrict__ g_action, int64_t ld_ga,
                                            float* __restrict__ d_head) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= M * A) return;
  const int64_t r = i / A;
  const int j = (int)(i % A);
  const HeadGeom g = head_geom(minimum, maximum, epsilon);
  const float gl = g_logp_scale * (log_alpha ? expf(*log_alpha) : 1.f);
  const float loc = head[r * 2 * A + j], raw = head[r * 2 * A + A + j], sigma = softplusf(raw) + min_scale, e = eps[r * A + j];
  const float u = loc + sigma * e, th = tanhf(u), a = g.sh + g.s * th;
  const float du = (g_action ? g_action[r * ld_ga + j] : 0.f) * g.s * (1.f - th * th);
  float d_loc = du, d_sigma = du * e;
  if (a <= g.lo) {
    const float z = (g.u_lo - loc) / sigma, m = mills(z);
    d_loc += gl * m * (-1.f / sigma), d_sigma += gl * m * (-z / sigma);
  } else if (a >= g.hi) {
    const float z = -(g.u_hi - loc) / sigma, m = mills(z);
    d_loc += gl * m * (1.f / sigma), d_sigma += gl * m * (-z / sigma);
  } else {
    d_loc += gl * 2.f * th, d_sigma += gl * (2.f * th * e - 1.f / sigma);
  }
  d_head[r * 2 * A + j] = d_loc;
  d_head[r * 2 * A + A + j] = d_sigma * sigmoidf_(raw);
}

// ---- loss heads: ONE block (SAC batches are a few hundred to a few thousand rows), deterministic block sums ----
// metrics layout (8 floats, accumulated with `weight`): actor_loss, entropy, q_loss, q_error, q1_pred, q2_pred, alpha_loss, alpha

// Actor loss (ff_sac.py:207-226): mean(alpha * log_prob - min_k q_k): seeds dq_k = -1/M on the arg-min network.
__global__ void __launch_bounds__(1024) sac_actor_seed_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                            const float* __restrict__ log_prob, const float* __restrict__ log_alpha, int64_t M,
                                                            float* __restrict__ dq1, float* __restrict__ dq2, float* __restrict__ metrics,
                                                            float weight) {
  __shared__ float sred[32];
  const float alpha = expf(*log_alpha), inv = 1.f / (float)M;
  float l = 0.f, h = 0.f;
  for (int64_t r = threadIdx.x; r < M; r += blockDim.x) {
    const bool first = q1[r] <= q2[r];  // jnp.min gradient goes to the first minimum; ties split in JAX -- measure zero here
    dq1[r] = first ? -inv : 0.f;
    dq2[r] = first ? 0.f : -inv;
    l += alpha * log_prob[r] - fminf(q1[r], q2[r]);
    h -= log_prob[r];
  }
  l = block_sum<float>(l, sred);
  h = block_sum<float>(h, sred);
  if (threadIdx.x == 0 && metrics) metrics[0] += weight * l * inv, metrics[1] += weight * h * inv;
}

// Q loss (ff_sac.py:177-205): target = r + (1 - done) gamma (min next_q - alpha next_log_prob); dq_k = (q_k - target) / (2M).
__global__ void __launch_bounds__(1024) sac_q_loss_kernel(const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ nq1,
                                                        const float* __restrict__ nq2, const float* __restrict__ next_log_prob,
                                                        const float* __restrict__ reward, const uint8_t* __restrict__ done,
                                                        const float* __restrict__ log_alpha, float gamma, int64_t M, float* __restrict__ dq1,
                                                        float* __restrict__ dq2, float* __restrict__ metrics, float weight) {
  __shared__ float sred[32];
  const float alpha = expf(*log_alpha), inv = 1.f / (float)M;
  float sl = 0.f, se = 0.f, s1 = 0.f, s2 = 0.f;
  for (int64_t r = threadIdx.x; r < M; r += blockDim.x) {
    const float next_v = fminf(nq1[r], nq2[r]) - alpha * next_log_prob[r];
    const float target = reward[r] + (done[r] ? 0.f : 1.f) * gamma * next_v;
    const float e1 = q1[r] - target, e2 = q2[r] - target;
    dq1[r] = 0.5f * e1 * inv, dq2[r] = 0.5f * e2 * inv;
    sl += e1 * e1 + e2 * e2, se += fabsf(e1) + fabsf(e2), s1 += nq1[r], s2 += nq2[r];
  }
  sl = block_sum<float>(sl, sred), se = block_sum<float>(se, sred), s1 = block_sum<float>(s1, sred), s2 = block_sum<float>(s2, sred);
  if (threadIdx.x == 0 && metrics) {
    metrics[2] += weight * 0.5f * sl * 0.5f * inv, metrics[3] += weight * se * 0.5f * inv;
    metrics[4] += weight * s1 * inv, metrics[5] += weight * s2 * inv;
  }
}

// Alpha loss (ff_sac.py:157-175): mean(alpha * stop_gradient(-log_prob - target_entropy)); d/d log_alpha = the loss.
__global__ void __launch_bounds__(1024) sac_alpha_grad_kernel(const float* __restrict__ log_prob, const float* __restrict__ log_alpha,
                                                            float target_entropy, int64_t M, int autotune, float* __restrict__ grad,
                                                            float grad_weight, int overwrite, float* __restrict__ metrics, float weight) {
  __shared__ float sred[32];
  const float alpha = expf(*log_alpha);
  float s = 0.f;
  for (int64_t r = threadIdx.x; r < M; r += blockDim.x) s += -log_prob[r] - target_entropy;
  s = block_sum<float>(s, sred);
  if (threadIdx.x == 0) {
    const float loss = alpha * s / (float)M;
    if (grad) grad[0] = (overwrite ? 0.f : grad[0]) + (autotune ? grad_weight * loss : 0.f);
    if (metrics) metrics[6] += weight * (autotune ? loss : 0.f), metrics[7] += weight * alpha;
  }
}

// optax.incremental_update(new, old, tau): target = tau * online + (1 - tau) * target
__global__ void polyak_kernel(float* __restrict__ target, const float* __restrict__ online, int64_t n, float tau) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) target[i] = tau * online[i] + (1.f - tau) * target[i];
}

// ---- replay buffer: uniform indices + row gather (flashbax item buffer sample: uniform with replacement over the filled part) ----
// Sample index r of a call: word r & 3 of Philox (seed; r / 4, call, tag), scaled to floor(u * n), u in [0, 1).  Every sampler
// (stx_uniform_indices and both rings) draws through this function, so they agree index for index.
__device__ __forceinline__ int64_t uniform_index(int64_t r, uint64_t seed, uint64_t call, uint64_t n) {
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const uint4 w = Philox::rand4(make_uint4((uint32_t)(r >> 2), (uint32_t)call, (uint32_t)(call >> 32), 0x52504c59u), key);
  const uint32_t v[4] = {w.x, w.y, w.z, w.w};
  return (int64_t)(((uint64_t)v[r & 3] * n) >> 32);
}

__global__ void uniform_index_kernel(int32_t* __restrict__ idx, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ counter,
                                     const int64_t* __restrict__ range) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i * 4 >= M) return;
  const uint64_t call = offset + (counter ? *counter : 0ull);
  const uint64_t n = (uint64_t)*range;
  for (int k = 0; k < 4 && i * 4 + k < M; ++k) idx[i * 4 + k] = (int32_t)uniform_index(i * 4 + k, seed, call, n);
}

// dst[r, 0:C] (leading dim ld_dst) = src[idx[r], 0:C]; one warp per row, coalesced
__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, int64_t M, int C, float* __restrict__ dst,
                                   int64_t ld_dst) {
  const int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= M) return;
  const float* s = src + (int64_t)idx[r] * C;
  for (int c = threadIdx.x & 31; c < C; c += 32) dst[r * ld_dst + c] = s[c];
}
__global__ void gather_bytes_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ idx, int64_t M, uint8_t* __restrict__ dst) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r < M) dst[r] = src[idx[r]];
}

// ---- transition ring buffers (obs, action, reward, done, next_obs): the flashbax item buffer of ff_sac.py:449-456 /
// ff_dqn.py:339-347 with its write position / fill count in DEVICE memory, so add + sample are stream-ordered and CUDA-graph
// replayable.  One template over the ring (StxReplay: float action rows of act_dim; StxReplayDiscrete: one int32 action per
// row); one warp per row.
__device__ __forceinline__ int action_cols(const StxReplay& rb) { return rb.act_dim; }
__device__ __forceinline__ int action_cols(const StxReplayDiscrete&) { return 1; }

template <class Ring, class Act>
__global__ void replay_add_kernel(Ring rb, const float* __restrict__ obs, const Act* __restrict__ action, const float* __restrict__ reward,
                                  const uint8_t* __restrict__ done, const float* __restrict__ next_obs, int64_t n, int64_t skip) {
  const int64_t r = skip + blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n) return;
  const int lane = threadIdx.x & 31;
  const int64_t slot = (rb.state[0] + r) % rb.capacity;
  const int D = rb.obs_dim, A = action_cols(rb);
  for (int c = lane; c < D; c += 32) {
    rb.obs[slot * D + c] = obs[r * D + c];
    rb.next_obs[slot * D + c] = next_obs[r * D + c];
  }
  for (int c = lane; c < A; c += 32) rb.action[slot * A + c] = action[r * A + c];
  if (lane == 0) {
    rb.reward[slot] = reward[r];
    rb.done[slot] = done[r];
  }
}
template <class Ring>
__global__ void replay_advance_kernel(Ring rb, int64_t n) {
  rb.state[0] = (rb.state[0] + n) % rb.capacity;
  rb.state[1] = min(rb.state[1] + n, rb.capacity);
}

// Where a sampled row goes.  SAC: the three network inputs of one epoch, xq_old = (obs | stored action), xq_new = (obs | .),
// xq_next = (next_obs | .); the action columns of xq_new / xq_next are filled later by the policy-head sampler.
struct SacInputs {
  float *xq_old, *xq_new, *xq_next;
  int64_t ld;
  __device__ __forceinline__ void row(const StxReplay& rb, int64_t j, int64_t r, int lane) const {
    const int D = rb.obs_dim, A = rb.act_dim;
    for (int c = lane; c < D; c += 32) {
      const float o = rb.obs[j * D + c];
      xq_old[r * ld + c] = o;
      if (xq_new) xq_new[r * ld + c] = o;
      if (xq_next) xq_next[r * ld + c] = rb.next_obs[j * D + c];
    }
    for (int c = lane; c < A; c += 32) xq_old[r * ld + D + c] = rb.action[j * A + c];
  }
};
// DQN: the Transition fields as they are, obs / next_obs (M, obs_dim) and action (M).
struct DiscreteBatch {
  float *obs, *next_obs;
  int32_t* action;
  __device__ __forceinline__ void row(const StxReplayDiscrete& rb, int64_t j, int64_t r, int lane) const {
    const int D = rb.obs_dim;
    for (int c = lane; c < D; c += 32) {
      obs[r * D + c] = rb.obs[j * D + c];
      next_obs[r * D + c] = rb.next_obs[j * D + c];
    }
    if (lane == 0) action[r] = rb.action[j];
  }
};

// Sample M items uniformly with replacement (the indices of uniform_index_kernel) or take idx_in.
template <class Ring, class Out>
__global__ void replay_sample_kernel(Ring rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ counter,
                                     const int32_t* __restrict__ idx_in, Out out, float* __restrict__ reward, uint8_t* __restrict__ done,
                                     int32_t* __restrict__ idx_out) {
  const int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= M) return;
  const int lane = threadIdx.x & 31;
  const int64_t j = idx_in ? (int64_t)idx_in[r] : uniform_index(r, seed, offset + (counter ? *counter : 0ull), (uint64_t)rb.state[1]);
  out.row(rb, j, r, lane);
  if (lane == 0) {
    reward[r] = rb.reward[j];
    done[r] = rb.done[j];
    if (idx_out) idx_out[r] = (int32_t)j;
  }
}

template <class Ring, class Act>
int replay_add(const Ring& rb, const float* obs, const Act* action, const float* reward, const uint8_t* done, const float* next_obs, int64_t n,
               cudaStream_t st) {
  const int64_t skip = n > rb.capacity ? n - rb.capacity : 0;   // more rows than slots: only the newest `capacity` survive
  replay_add_kernel<Ring, Act><<<(unsigned)((n - skip + 7) / 8), 256, 0, st>>>(rb, obs, action, reward, done, next_obs, n, skip);
  STX_LAUNCH_OK();
  replay_advance_kernel<Ring><<<1, 1, 0, st>>>(rb, n);
  STX_LAUNCH_OK();
  return STX_OK;
}

template <class Ring, class Out>
int replay_sample(const Ring& rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* counter, const int32_t* idx_in, const Out& out,
                  float* reward, uint8_t* done, int32_t* idx_out, cudaStream_t st) {
  replay_sample_kernel<Ring, Out><<<(unsigned)((M + 7) / 8), 256, 0, st>>>(rb, M, seed, offset, counter, idx_in, out, reward, done, idx_out);
  STX_LAUNCH_OK();
  return STX_OK;
}

}  // namespace
}  // namespace stx

using namespace stx;

static bool replay_ok(const StxReplay* rb) {
  return rb && rb->obs && rb->action && rb->reward && rb->done && rb->next_obs && rb->state && rb->capacity > 0 && rb->obs_dim > 0 && rb->act_dim > 0;
}

extern "C" int stx_replay_add(const StxReplay* rb, const float* obs, const float* action, const float* reward, const uint8_t* done,
                              const float* next_obs, int64_t n, void* stream) {
  STX_REQUIRE(replay_ok(rb) && obs && action && reward && done && next_obs && n > 0, STX_E_ARG, "stx_replay_add: bad arguments");
  return replay_add(*rb, obs, action, reward, done, next_obs, n, (cudaStream_t)stream);
}

extern "C" int stx_replay_sample(const StxReplay* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const int32_t* idx_in,
                                 float* xq_old, float* xq_new, float* xq_next, int64_t ld, float* reward, uint8_t* done, int32_t* idx_out,
                                 void* stream) {
  STX_REQUIRE(replay_ok(rb) && xq_old && reward && done && M > 0 && ld >= rb->obs_dim + rb->act_dim, STX_E_ARG, "stx_replay_sample: bad arguments");
  return replay_sample(*rb, M, seed, offset, dev_counter, idx_in, SacInputs{xq_old, xq_new, xq_next, ld}, reward, done, idx_out,
                       (cudaStream_t)stream);
}

static bool replay_ok(const StxReplayDiscrete* rb) {
  return rb && rb->obs && rb->action && rb->reward && rb->done && rb->next_obs && rb->state && rb->capacity > 0 && rb->obs_dim > 0;
}

extern "C" int stx_replay_add_discrete(const StxReplayDiscrete* rb, const float* obs, const int32_t* action, const float* reward,
                                       const uint8_t* done, const float* next_obs, int64_t n, void* stream) {
  STX_REQUIRE(replay_ok(rb) && obs && action && reward && done && next_obs && n > 0, STX_E_ARG, "stx_replay_add_discrete: bad arguments");
  return replay_add(*rb, obs, action, reward, done, next_obs, n, (cudaStream_t)stream);
}

extern "C" int stx_replay_sample_discrete(const StxReplayDiscrete* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                                          const int32_t* idx_in, float* obs, float* next_obs, int32_t* action, float* reward, uint8_t* done,
                                          int32_t* idx_out, void* stream) {
  STX_REQUIRE(replay_ok(rb) && obs && next_obs && action && reward && done && M > 0, STX_E_ARG, "stx_replay_sample_discrete: bad arguments");
  return replay_sample(*rb, M, seed, offset, dev_counter, idx_in, DiscreteBatch{obs, next_obs, action}, reward, done, idx_out,
                       (cudaStream_t)stream);
}

extern "C" int stx_tanh_normal_sample(const float* head_out, int64_t M, int A, const float* eps_in, uint64_t seed, uint64_t offset,
                                      const uint64_t* dev_counter, float minimum, float maximum, float min_scale, float* action, int64_t ld_action,
                                      float* log_prob, float* eps_out, void* stream) {
  STX_REQUIRE(head_out && action && M > 0 && A > 0 && ld_action >= A && maximum > minimum, STX_E_ARG, "stx_tanh_normal_sample: bad arguments");
  tanh_normal_sample_kernel<<<(unsigned)((M + 127) / 128), 128, 0, (cudaStream_t)stream>>>(head_out, M, A, eps_in, seed, offset, dev_counter, minimum,
                                                                                          maximum, min_scale, 1e-3f, action, ld_action, log_prob, eps_out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_tanh_normal_backward(const float* head_out, const float* eps, int64_t M, int A, float minimum, float maximum, float min_scale,
                                        const float* log_alpha, float g_logp_scale, const float* g_action, int64_t ld_g_action, float* d_head_out,
                                        void* stream) {
  STX_REQUIRE(head_out && eps && d_head_out && M > 0 && A > 0 && maximum > minimum, STX_E_ARG, "stx_tanh_normal_backward: bad arguments");
  STX_REQUIRE(!g_action || ld_g_action >= A, STX_E_SHAPE, "stx_tanh_normal_backward: ld_g_action < A");
  const int64_t n = M * A;
  tanh_normal_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(head_out, eps, M, A, minimum, maximum, min_scale, 1e-3f,
                                                                                            log_alpha, g_logp_scale, g_action, ld_g_action, d_head_out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_sac_actor_seed(const float* q1, const float* q2, const float* log_prob, const float* log_alpha, int64_t M, float* dq1,
                                  float* dq2, float* metrics, float weight, void* stream) {
  STX_REQUIRE(q1 && q2 && log_prob && log_alpha && dq1 && dq2 && M > 0, STX_E_ARG, "stx_sac_actor_seed: bad arguments");
  sac_actor_seed_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(q1, q2, log_prob, log_alpha, M, dq1, dq2, metrics, weight);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_sac_q_loss(const float* q1, const float* q2, const float* next_q1, const float* next_q2, const float* next_log_prob,
                              const float* reward, const uint8_t* done, const float* log_alpha, float gamma, int64_t M, float* dq1, float* dq2,
                              float* metrics, float weight, void* stream) {
  STX_REQUIRE(q1 && q2 && next_q1 && next_q2 && next_log_prob && reward && done && log_alpha && dq1 && dq2 && M > 0, STX_E_ARG,
              "stx_sac_q_loss: bad arguments");
  sac_q_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(q1, q2, next_q1, next_q2, next_log_prob, reward, done, log_alpha, gamma, M, dq1, dq2, metrics,
                                                         weight);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_sac_alpha_grad(const float* log_prob, const float* log_alpha, float target_entropy, int64_t M, int autotune, float* grad,
                                  float grad_weight, int overwrite, float* metrics, float weight, void* stream) {
  STX_REQUIRE(log_prob && log_alpha && M > 0, STX_E_ARG, "stx_sac_alpha_grad: bad arguments");
  sac_alpha_grad_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(log_prob, log_alpha, target_entropy, M, autotune, grad, grad_weight, overwrite, metrics,
                                                             weight);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_polyak_update(float* target, const float* online, int64_t n, float tau, void* stream) {
  STX_REQUIRE(target && online && n >= 0, STX_E_ARG, "stx_polyak_update: bad arguments");
  if (n == 0) return STX_OK;
  int64_t blocks = (n + 255) / 256;
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  polyak_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(target, online, n, tau);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_uniform_indices(int32_t* idx, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const int64_t* range,
                                   void* stream) {
  STX_REQUIRE(idx && range && M > 0, STX_E_ARG, "stx_uniform_indices: bad arguments");
  uniform_index_kernel<<<(unsigned)((M / 4 + 256) / 256), 256, 0, (cudaStream_t)stream>>>(idx, M, seed, offset, dev_counter, range);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_gather_rows_f32(const float* src, const int32_t* idx, int64_t M, int C, float* dst, int64_t ld_dst, void* stream) {
  STX_REQUIRE(src && idx && dst && M > 0 && C > 0 && ld_dst >= C, STX_E_ARG, "stx_gather_rows_f32: bad arguments");
  gather_rows_kernel<<<(unsigned)((M + 7) / 8), 256, 0, (cudaStream_t)stream>>>(src, idx, M, C, dst, ld_dst);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_gather_u8(const uint8_t* src, const int32_t* idx, int64_t M, uint8_t* dst, void* stream) {
  STX_REQUIRE(src && idx && dst && M > 0, STX_E_ARG, "stx_gather_u8: bad arguments");
  gather_bytes_kernel<<<(unsigned)((M + 255) / 256), 256, 0, (cudaStream_t)stream>>>(src, idx, M, dst);
  STX_LAUNCH_OK();
  return STX_OK;
}
