// Rainbow (ff_rainbow): noisy layers materialised into a dense MLP arena, the dueling distributional combine, and the prioritised
// n-step trajectory ring with its deterministic sum tree.  Semantics: include/stx.h.
//
// Reference: NoisyLinear (stoix/networks/layers.py:71-169), NoisyDistributionalDuelingQNetwork (stoix/networks/dueling.py:90-124), and
// fbx.make_prioritised_trajectory_buffer with the n-step target of stoix/systems/q_learning/ff_rainbow.py:222-246.
#include "stx_common.cuh"
#include "stx_prio_tree.cuh"

namespace stx {
namespace {

using prio::kTreeThreads;
using prio::tree_rebuild;

constexpr uint32_t kNoiseTag = 0x4E4F4953u;  // "NOIS"

// ---- noisy layers ----------------------------------------------------------------------------------------------------------------

// f(z) = sign(z) sqrt|z| of the normal drawn for noise element j of call `call`.
__device__ __forceinline__ float noise_draw(int64_t j, uint64_t seed, uint64_t call) {
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const uint4 w = Philox::rand4(make_uint4((uint32_t)j, (uint32_t)call, (uint32_t)(call >> 32), kNoiseTag), key);
  const float z = normal2(w.x, w.y).x;
  return z > 0.f ? sqrtf(z) : (z < 0.f ? -sqrtf(-z) : 0.f);
}

// Block b of a noisy-layer launch: rows 0 .. in-1 of layer l, then one block for the layer's bias (in + 1 blocks per layer).
__device__ __forceinline__ int noisy_block(const StxNoisyNet& net, int& row) {
  int b = blockIdx.x, l = 0;
  while (l < net.n_layers - 1 && b >= net.layers[l].in + 1) b -= net.layers[l].in + 1, ++l;
  row = b;
  return l;
}

__global__ void __launch_bounds__(256) noisy_weights_kernel(StxNoisyNet net, const float* __restrict__ params, float* __restrict__ eff,
                                                            float* __restrict__ noise, int draw, uint64_t seed, uint64_t offset,
                                                            const uint64_t* __restrict__ counter) {
  int r;
  const StxNoisyLayer L = net.layers[noisy_block(net, r)];
  const uint64_t call = offset + (counter ? *counter : 0ull);
  const int64_t nin = L.noise, nout = L.noise + L.in, W = (int64_t)L.in * L.out;
  const float* mu_w = params + L.param;
  const float* mu_b = mu_w + W;
  const float* sg_w = mu_b + L.out;
  const float* sg_b = sg_w + W;
  // with draw, every block draws the f values it needs itself (no block reads `noise`, the owners of each entry write it)
  auto f = [&](int64_t j) { return draw ? noise_draw(j, seed, call) : noise[j]; };
  if (r < L.in) {
    const float fin = f(nin + r);
    for (int c = threadIdx.x; c < L.out; c += blockDim.x) {
      const int64_t k = (int64_t)r * L.out + c;
      eff[L.eff_w + (int64_t)r * L.ld + c] = __fadd_rn(mu_w[k], __fmul_rn(sg_w[k], __fmul_rn(fin, f(nout + c))));
    }
    if (draw && threadIdx.x == 0) noise[nin + r] = fin;
  } else {
    for (int c = threadIdx.x; c < L.out; c += blockDim.x) {
      const float fo = f(nout + c);
      eff[L.eff_b + c] = __fadd_rn(mu_b[c], __fmul_rn(sg_b[c], fo));
      if (draw) noise[nout + c] = fo;
    }
  }
}

__global__ void __launch_bounds__(256) noisy_fold_kernel(StxNoisyNet net, const float* __restrict__ eff_grad, const float* __restrict__ noise,
                                                         float* __restrict__ grad, int overwrite) {
  int r;
  const StxNoisyLayer L = net.layers[noisy_block(net, r)];
  const int64_t nin = L.noise, nout = L.noise + L.in, W = (int64_t)L.in * L.out;
  float* g_mu_w = grad + L.param;
  float* g_mu_b = g_mu_w + W;
  float* g_sg_w = g_mu_b + L.out;
  float* g_sg_b = g_sg_w + W;
  if (r < L.in) {
    const float fin = noise[nin + r];
    for (int c = threadIdx.x; c < L.out; c += blockDim.x) {
      const int64_t k = (int64_t)r * L.out + c;
      const float g = eff_grad[L.eff_w + (int64_t)r * L.ld + c], gs = __fmul_rn(g, __fmul_rn(fin, noise[nout + c]));
      g_mu_w[k] = overwrite ? g : __fadd_rn(g_mu_w[k], g);
      g_sg_w[k] = overwrite ? gs : __fadd_rn(g_sg_w[k], gs);
    }
  } else {
    for (int c = threadIdx.x; c < L.out; c += blockDim.x) {
      const float g = eff_grad[L.eff_b + c], gs = __fmul_rn(g, noise[nout + c]);
      g_mu_b[c] = overwrite ? g : __fadd_rn(g_mu_b[c], g);
      g_sg_b[c] = overwrite ? gs : __fadd_rn(g_sg_b[c], gs);
    }
  }
}

// ---- dueling combine: one thread per (row, atom) ------------------------------------------------------------------------------------

__global__ void dueling_combine_kernel(const float* __restrict__ head, int64_t M, int A, int N, float* __restrict__ q) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= M * N) return;
  const int64_t m = k / N;
  const int i = (int)(k % N);
  const float* row = head + m * (int64_t)(N + A * N);
  const float* adv = row + N + i;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s = __fadd_rn(s, adv[(int64_t)a * N]);
  const float mean = __fdiv_rn(s, (float)A), v = row[i];
  float* out = q + m * (int64_t)A * N + i;
  for (int a = 0; a < A; ++a) out[(int64_t)a * N] = __fsub_rn(__fadd_rn(v, adv[(int64_t)a * N]), mean);
}

__global__ void dueling_backward_kernel(const float* __restrict__ dq, int64_t M, int A, int N, float* __restrict__ d_head) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= M * N) return;
  const int64_t m = k / N;
  const int i = (int)(k % N);
  const float* g = dq + m * (int64_t)A * N + i;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s = __fadd_rn(s, g[(int64_t)a * N]);
  const float mean = __fdiv_rn(s, (float)A);
  float* row = d_head + m * (int64_t)(N + A * N);
  row[i] = s;
  for (int a = 0; a < A; ++a) row[N + (int64_t)a * N + i] = __fsub_rn(g[(int64_t)a * N], mean);
}

// ---- prioritised ring: add --------------------------------------------------------------------------------------------------------

// Rows (t, e) of the (T, E) batch, t >= skip, into ring row (w + t) mod L; one warp per row.
__global__ void prio_write_kernel(StxReplayPrioritised rb, const float* __restrict__ obs, const int32_t* __restrict__ action,
                                  const float* __restrict__ reward, const uint8_t* __restrict__ done, const float* __restrict__ next_obs, int T,
                                  int skip) {
  const int64_t E = rb.envs, r = skip * E + blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= (int64_t)T * E) return;
  const int lane = threadIdx.x & 31;
  const int64_t t = r / E, e = r % E;
  const int64_t slot = ((rb.state[0] + t) % rb.length) * E + e;
  const int D = rb.obs_dim;
  for (int c = lane; c < D; c += 32) {
    rb.obs[slot * D + c] = obs[r * D + c];
    rb.next_obs[slot * D + c] = next_obs[r * D + c];
  }
  if (lane == 0) {
    rb.action[slot] = action[r];
    rb.reward[slot] = reward[r];
    rb.done[slot] = done[r];
  }
}

// Priorities of the items the add touched, their ancestors, then the write index.  One CTA.
__global__ void __launch_bounds__(kTreeThreads) prio_add_kernel(StxReplayPrioritised rb, int T) {
  const int64_t L = rb.length, E = rb.envs, n = rb.n_step;
  const int64_t w0 = rb.state[0], w1 = (w0 + T) % L, c1 = min(rb.state[1] + (int64_t)T, L);
  const int64_t W = min((int64_t)T + n - 1, L), start = ((w0 - (n - 1)) % L + L) % L;
  const float maxp = *rb.max_priority;
  auto leaf = [&](int64_t j) { return (j / W) * L + (start + j % W) % L; };  // dirty item j: env j / W, start row start + j % W
  for (int64_t j = threadIdx.x; j < E * W; j += blockDim.x) {
    const int64_t p = (start + j % W) % L, age = ((w1 - 1 - p) % L + L) % L;
    rb.tree[leaf(j)] = (age >= n - 1 && age < c1) ? maxp : 0.f;
  }
  tree_rebuild(rb.tree, E * L, E * W, leaf);
  __syncthreads();
  if (threadIdx.x == 0) {
    rb.state[0] = w1;
    rb.state[1] = c1;
  }
}

// ---- prioritised ring: sample -----------------------------------------------------------------------------------------------------

struct PrioOut {
  float *obs, *next_obs, *reward, *prob, *weight;
  int32_t *action, *idx;
  uint8_t* done;
};

__global__ void __launch_bounds__(256) prio_sample_kernel(StxReplayPrioritised rb, int64_t M, uint64_t seed, uint64_t offset,
                                                          const uint64_t* __restrict__ counter, const float* __restrict__ u_in,
                                                          const int32_t* __restrict__ count, float beta0, float beta_steps, float gamma, PrioOut o,
                                                          unsigned int* __restrict__ ticket) {
  const int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t items = (int64_t)rb.envs * rb.length;
  if (r < M) {
    const uint64_t call = offset + (counter ? *counter : 0ull);
    const float total = rb.tree[prio::root_offset(items)];
    const int64_t node = prio::tree_descend(rb.tree, items, r, prio::stratum_uniform(r, seed, call, u_in), M);
    const int64_t i = node, L = rb.length, E = rb.envs, e = i / L, p = i % L;
    const int n = rb.n_step, D = rb.obs_dim;
    const int64_t s0 = p * E + e, sn = ((p + n - 1) % L) * E + e;
    for (int c = lane; c < D; c += 32) {
      o.obs[r * D + c] = rb.obs[s0 * D + c];
      o.next_obs[r * D + c] = rb.next_obs[sn * D + c];
    }
    if (lane == 0) {
      float g = rb.reward[sn];
      uint8_t any = rb.done[sn];
      for (int k = n - 2; k >= 0; --k) {
        const int64_t sk = ((p + k) % L) * E + e;
        const float d = __fmul_rn(1.f - (float)rb.done[sk], gamma);
        g = __fadd_rn(rb.reward[sk], __fmul_rn(d, g));
        any |= rb.done[sk];
      }
      o.reward[r] = g;
      o.done[r] = any ? 1 : 0;
      o.action[r] = rb.action[s0];
      o.idx[r] = (int32_t)i;
      o.prob[r] = total > 0.f ? __fdiv_rn(rb.tree[i], total) : 0.f;   // no valid item: every draw is item 0 with p 0
    }
  }
  // the importance weights need the whole batch: the last block to finish computes them
  if (!last_block_ticket(ticket, gridDim.x)) return;
  if (!(rb.tree[prio::root_offset(items)] > 0.f)) {   // p 0 everywhere: weights of 1, not (1/0)^beta / max = inf / inf
    for (int64_t m = threadIdx.x; m < M; m += blockDim.x) o.weight[m] = 1.f;
    return;
  }
  float beta = beta0;
  if (beta_steps > 0.f) {
    const float c = fminf(fmaxf((float)(count ? *count : 0), 0.f), beta_steps);
    beta = __fadd_rn(__fmul_rn(beta0 - 1.f, 1.f - __fdiv_rn(c, beta_steps)), 1.f);
  }
  __shared__ float red[32];
  float mx = 0.f;
  for (int64_t m = threadIdx.x; m < M; m += blockDim.x) {
    const float iw = powf(__fdiv_rn(1.f, o.prob[m]), beta);
    o.weight[m] = iw;
    mx = fmaxf(mx, iw);
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, k));
  if (lane == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int k = 1; k < (int)(blockDim.x >> 5); ++k) mx = fmaxf(mx, red[k]);
  for (int64_t m = threadIdx.x; m < M; m += blockDim.x) o.weight[m] = __fdiv_rn(o.weight[m], mx);
}

// ---- prioritised ring: set_priorities ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kTreeThreads) prio_set_kernel(StxReplayPrioritised rb, const int32_t* __restrict__ idx, const float* __restrict__ pr,
                                                                int64_t M) {
  prio::set_priorities(rb.tree, rb.owner, rb.max_priority, rb.priority_exponent, (int64_t)rb.envs * rb.length, idx, pr, M);
}

bool noisy_ok(const StxNoisyNet* net, int64_t* blocks) {
  if (!net || net->n_layers < 1 || net->n_layers > STX_NOISY_MAX_LAYERS) return false;
  *blocks = 0;
  for (int l = 0; l < net->n_layers; ++l) {
    const StxNoisyLayer& L = net->layers[l];
    if (L.in <= 0 || L.out <= 0 || L.ld < L.out || L.param < 0 || L.eff_w < 0 || L.eff_b < 0 || L.noise < 0) return false;
    *blocks += L.in + 1;
  }
  return true;
}

bool prio_ok(const StxReplayPrioritised* rb) {
  return rb && rb->obs && rb->action && rb->reward && rb->done && rb->next_obs && rb->tree && rb->state && rb->max_priority && rb->owner && rb->length > 0 &&
         rb->envs > 0 && rb->obs_dim > 0 && rb->n_step > 0 && rb->n_step <= rb->length && (int64_t)rb->envs * rb->length <= INT32_MAX;
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int stx_noisy_weights(const StxNoisyNet* net, const float* params, float* eff, float* noise, int draw, uint64_t seed, uint64_t offset,
                                 const uint64_t* dev_counter, void* stream) {
  int64_t blocks = 0;
  STX_REQUIRE(noisy_ok(net, &blocks), STX_E_SHAPE, "stx_noisy_weights: bad layer table");
  STX_REQUIRE(params && eff && noise, STX_E_ARG, "stx_noisy_weights: null pointer");
  noisy_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(*net, params, eff, noise, draw, seed, offset, dev_counter);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_noisy_fold(const StxNoisyNet* net, const float* eff_grad, const float* noise, float* grad, int overwrite, void* stream) {
  int64_t blocks = 0;
  STX_REQUIRE(noisy_ok(net, &blocks), STX_E_SHAPE, "stx_noisy_fold: bad layer table");
  STX_REQUIRE(eff_grad && noise && grad, STX_E_ARG, "stx_noisy_fold: null pointer");
  noisy_fold_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(*net, eff_grad, noise, grad, overwrite);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_dueling_combine(const float* head, int64_t M, int A, int N, float* q_logits, void* stream) {
  STX_REQUIRE(head && q_logits && M > 0 && A > 0 && N > 0, STX_E_ARG, "stx_dueling_combine: bad arguments");
  dueling_combine_kernel<<<(unsigned)((M * N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(head, M, A, N, q_logits);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_dueling_backward(const float* d_q_logits, int64_t M, int A, int N, float* d_head, void* stream) {
  STX_REQUIRE(d_q_logits && d_head && M > 0 && A > 0 && N > 0, STX_E_ARG, "stx_dueling_backward: bad arguments");
  dueling_backward_kernel<<<(unsigned)((M * N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_q_logits, M, A, N, d_head);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int64_t stx_prio_tree_floats(int64_t items) {
  if (items <= 0) return 0;
  return prio::root_offset(items) + 1;
}

extern "C" size_t stx_prio_scratch_bytes(void) { return 256; }

extern "C" int stx_replay_add_prioritised(const StxReplayPrioritised* rb, const float* obs, const int32_t* action, const float* reward,
                                          const uint8_t* done, const float* next_obs, int T, void* stream) {
  STX_REQUIRE(prio_ok(rb) && obs && action && reward && done && next_obs && T > 0, STX_E_ARG, "stx_replay_add_prioritised: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int skip = T > rb->length ? T - (int)rb->length : 0;  // more rows than the ring holds: only the newest L survive
  const int64_t rows = (int64_t)(T - skip) * rb->envs;
  prio_write_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(*rb, obs, action, reward, done, next_obs, T, skip);
  STX_LAUNCH_OK();
  prio_add_kernel<<<1, kTreeThreads, 0, st>>>(*rb, T);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_replay_sample_prioritised(const StxReplayPrioritised* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                                             const float* u_in, const int32_t* count, float beta0, float beta_steps, float gamma, float* obs,
                                             float* next_obs, int32_t* action, float* reward, uint8_t* done, int32_t* idx_out, float* prob_out,
                                             float* weight_out, void* scratch, void* stream) {
  STX_REQUIRE(prio_ok(rb) && obs && next_obs && action && reward && done && idx_out && prob_out && weight_out && scratch && M > 0, STX_E_ARG,
              "stx_replay_sample_prioritised: bad arguments");
  const PrioOut o{obs, next_obs, reward, prob_out, weight_out, action, idx_out, done};
  prio_sample_kernel<<<(unsigned)((M + 7) / 8), 256, 0, (cudaStream_t)stream>>>(*rb, M, seed, offset, dev_counter, u_in, count, beta0, beta_steps, gamma,
                                                                               o, reinterpret_cast<unsigned int*>(scratch));
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_replay_set_priorities(const StxReplayPrioritised* rb, const int32_t* idx, const float* priorities, int64_t M, void* stream) {
  STX_REQUIRE(prio_ok(rb) && idx && priorities && M > 0, STX_E_ARG, "stx_replay_set_priorities: bad arguments");
  STX_REQUIRE(M <= INT32_MAX, STX_E_SHAPE, "stx_replay_set_priorities: M=%lld", (long long)M);
  prio_set_kernel<<<1, kTreeThreads, 0, (cudaStream_t)stream>>>(*rb, idx, priorities, M);
  STX_LAUNCH_OK();
  return STX_OK;
}
