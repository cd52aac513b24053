// Synthetic Box environment step (the named benchmark env, BASELINE.json configs[1] / SURVEY.md 8d)
// and the keyed-bijection minibatch shuffle.
//
// Environment contract restated from the reference's call sites (stoa is not vendored):
//   * AutoResetWrapper(next_obs_in_extras=True)  stoix/utils/make_env.py:56-60: on the last step of
//     an episode timestep.observation is the RESET observation and extras["next_obs"] the true
//     successor (ff_ppo.py:110-116);
//   * discount == 0 <=> termination; last() & discount != 0 <=> truncation (ff_ppo.py:107-108);
//   * RecordEpisodeMetrics: running return/length, published with is_terminal_step on the final step
//     (same logic spelled out in stoix/wrappers/envpool.py:94-133).
// One thread per (env, 4-observation-feature group): Philox4x32-10 keyed by seed, counter =
// (env, step, lane, stream-tag), so the trajectory is a pure function of (seed, step, env) and the
// CPU oracle in tests/ regenerates it exactly.  The draws and transforms live in stx_synth_env.cuh, shared by the
// per-step kernel and the whole-trajectory kernel.
#include "stx_synth_env.cuh"

namespace stx {
namespace {

template <bool BF16>
__device__ __forceinline__ void store4(void* base, int64_t off, int n_valid, const float* v) {
  if (BF16) {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base) + off;
    for (int k = 0; k < n_valid; ++k) p[k] = __float2bfloat16_rn(v[k]);
  } else {
    float* p = reinterpret_cast<float*>(base) + off;
    for (int k = 0; k < n_valid; ++k) p[k] = v[k];
  }
}

template <bool BF16>
__global__ void synth_env_step_kernel(int64_t E, int D, uint64_t seed, uint64_t step_base,
                                      const uint64_t* __restrict__ dev_counter, float p_term,
                                      float p_trunc, void* __restrict__ obs_out,
                                      void* __restrict__ next_obs, float* __restrict__ reward,
                                      uint8_t* __restrict__ done, uint8_t* __restrict__ truncated,
                                      float* __restrict__ run_return, int32_t* __restrict__ run_length,
                                      float* __restrict__ ep_return, int32_t* __restrict__ ep_length,
                                      uint8_t* __restrict__ is_terminal) {
  const int groups = (D + 3) / 4;
  const int64_t gid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (gid >= E * groups) return;
  const int64_t e = gid / groups;
  const int grp = (int)(gid % groups);
  const uint64_t step = step_base + (dev_counter ? *dev_counter : 0ull);
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const synth::Ctr c = synth::counter(e, step);

  // step outcome (recomputed by every feature-group thread of the env: 1 Philox call, no sync needed)
  const synth::Outcome oc = synth::outcome(c, key, p_term, p_trunc);
  const bool last = oc.term || oc.trunc;

  const float4 a = synth::features4(c, key, (uint32_t)grp, synth::kTagObs);
  const float nxt[4] = {a.x, a.y, a.z, a.w};
  const int nv = D - grp * 4 < 4 ? D - grp * 4 : 4;
  const int64_t off = e * D + grp * 4;
  store4<BF16>(next_obs, off, nv, nxt);
  if (last) {
    const float4 r = synth::features4(c, key, (uint32_t)grp, synth::kTagReset);
    const float rst[4] = {r.x, r.y, r.z, r.w};
    store4<BF16>(obs_out, off, nv, rst);
  } else {
    store4<BF16>(obs_out, off, nv, nxt);
  }
  if (grp == 0) {
    float ret = run_return[e];
    int32_t len = run_length[e];
    synth::record(oc, ret, len, e, reward, done, truncated, ep_return, ep_length, is_terminal);
    run_return[e] = ret;
    run_length[e] = len;
  }
}

__device__ __forceinline__ uint2 pack4_bf16(float4 v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  return make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
}

// Steps [0, T) of all E envs in one launch (bf16 observations).  The dynamics ignore the action, so the whole trajectory
// can be produced before the policy runs.  L lanes per env (the next power of two >= D / 4 feature groups, within one
// warp); lane j owns feature group j for every step.  The step outcomes are drawn L steps at a time, lane j drawing step
// t0 + j, and handed to the env's lanes by shuffles; lane 0 keeps the episode bookkeeping and writes the per-step scalars.
// Every value comes from the same stx_synth_env.cuh draws as synth_env_step_kernel: the trajectory is bit-identical to T
// calls of stx_synth_env_step.
__global__ void __launch_bounds__(256) synth_env_trajectory_kernel(
    int64_t E, int D, int T, int L, uint64_t seed, uint64_t step_base, const uint64_t* __restrict__ dev_counter, float p_term,
    float p_trunc, __nv_bfloat16* __restrict__ obs, __nv_bfloat16* __restrict__ next_obs, float* __restrict__ reward,
    uint8_t* __restrict__ done, uint8_t* __restrict__ truncated, float* __restrict__ ep_return, int32_t* __restrict__ ep_length,
    uint8_t* __restrict__ is_terminal, float* __restrict__ run_return, int32_t* __restrict__ run_length) {
  const int64_t gid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t e = gid / L;
  const int j = (int)(threadIdx.x & (L - 1));
  const bool live = e < E;  // lanes past the last env still take part in the shuffles
  const int groups = D >> 2;
  const uint64_t step0 = step_base + (dev_counter ? *dev_counter : 0ull);
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  float run_ret = 0.f;
  int32_t run_len = 0;
  if (live && j == 0) run_ret = run_return[e], run_len = run_length[e];
  for (int t0 = 0; t0 < T; t0 += L) {
    synth::Outcome mine{0.f, false, false};
    if (live && t0 + j < T) mine = synth::outcome(synth::counter(e, step0 + (uint64_t)(t0 + j)), key, p_term, p_trunc);
    const uint32_t mine_f = (mine.term ? 1u : 0u) | (mine.trunc ? 2u : 0u);
    const int n = T - t0 < L ? T - t0 : L;
    for (int k = 0; k < n; ++k) {
      const int t = t0 + k;
      const float r = __shfl_sync(0xffffffffu, mine.reward, k, L);
      const uint32_t f = __shfl_sync(0xffffffffu, mine_f, k, L);
      if (!live) continue;
      const synth::Outcome o{r, (f & 1u) != 0u, (f & 2u) != 0u};
      const int64_t i = (int64_t)t * E + e;
      if (j == 0) synth::record(o, run_ret, run_len, i, reward, done, truncated, ep_return, ep_length, is_terminal);
      if (j < groups) {
        const synth::Ctr c = synth::counter(e, step0 + (uint64_t)t);
        const uint2 nx = pack4_bf16(synth::features4(c, key, (uint32_t)j, synth::kTagObs));
        const uint2 ob = (f != 0u) ? pack4_bf16(synth::features4(c, key, (uint32_t)j, synth::kTagReset)) : nx;
        *reinterpret_cast<uint2*>(next_obs + i * D + 4 * j) = nx;
        *reinterpret_cast<uint2*>(obs + (i + E) * D + 4 * j) = ob;  // obs row t + 1
      }
    }
  }
  if (live && j == 0) run_return[e] = run_ret, run_length[e] = run_len;
}

// ---- keyed bijection on [0, n): cycle-walking 6-round Feistel over the next power of 4 ------
// Round function: a 32-bit avalanche mixer (two multiply / xor-shift stages) of (right half + round key); the six
// round keys come from one Philox draw per thread.  (A Philox block per round made this shuffle a 36 us compute-bound
// kernel; a shuffle needs a keyed bijection with good diffusion, not a cryptographic round function.)
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x21f0aaadu;
  x ^= x >> 15;
  x *= 0x735a2d97u;
  x ^= x >> 15;
  return x;
}
__device__ __forceinline__ uint32_t feistel(uint32_t x, int half_bits, const uint32_t (&rk)[6]) {
  const uint32_t mask = (1u << half_bits) - 1u;
  uint32_t l = x >> half_bits, r = x & mask;
#pragma unroll
  for (int round = 0; round < 6; ++round) {
    const uint32_t nl = r, nr = l ^ (mix32(r + rk[round]) & mask);
    l = nl, r = nr;
  }
  return (l << half_bits) | r;
}

__global__ void permutation_kernel(int32_t* __restrict__ perm, int64_t n, int half_bits, uint64_t seed,
                                   uint64_t stream_base, const uint64_t* __restrict__ dev_counter) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t sid = stream_base + (dev_counter ? *dev_counter : 0ull);
  const uint64_t k = seed ^ (sid * 0x9E3779B97F4A7C15ull + 0xD1B54A32D192ED03ull);
  const uint2 key = make_uint2((uint32_t)k, (uint32_t)(k >> 32));
  const uint4 k0 = Philox::rand4(make_uint4(0u, 0u, 0x5045524du, 0u), key), k1 = Philox::rand4(make_uint4(1u, 0u, 0x5045524du, 0u), key);
  const uint32_t rk[6] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y};
  uint32_t x = (uint32_t)i;
  do {
    x = feistel(x, half_bits, rk);  // a bijection on [0, 4^half_bits); walk the cycle back into [0, n)
  } while (x >= (uint64_t)n);
  perm[i] = (int32_t)x;
}

}  // namespace
}  // namespace stx

using namespace stx;

__global__ void counter_add_kernel(uint64_t* c, uint64_t inc) { *c += inc; }

extern "C" int stx_counter_add(uint64_t* counter, uint64_t inc, void* stream) {
  STX_REQUIRE(counter, STX_E_ARG, "stx_counter_add: null counter");
  counter_add_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counter, inc);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_synth_env_step(int64_t E, int D, uint64_t seed, uint64_t step,
                                  const uint64_t* dev_counter, float p_term,
                                  float p_trunc, const int32_t* action, void* obs_out,
                                  void* next_obs, int obs_bf16, float* reward, uint8_t* done,
                                  uint8_t* truncated, float* run_return, int32_t* run_length,
                                  float* ep_return, int32_t* ep_length, uint8_t* is_terminal,
                                  void* stream) {
  (void)action;  // the synthetic dynamics ignore the action (it only fixes shapes and bandwidth)
  STX_REQUIRE(E > 0 && D > 0, STX_E_SHAPE, "stx_synth_env_step: E=%lld D=%d", (long long)E, D);
  STX_REQUIRE(obs_out && next_obs && reward && done && truncated && run_return && run_length &&
                  ep_return && ep_length && is_terminal,
              STX_E_ARG, "stx_synth_env_step: null pointer");
  const int groups = (D + 3) / 4;
  const int64_t total = E * groups;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (obs_bf16)
    synth_env_step_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(E, D, seed, step, dev_counter, p_term, p_trunc, obs_out, next_obs, reward, done, truncated, run_return, run_length, ep_return, ep_length, is_terminal);
  else
    synth_env_step_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(E, D, seed, step, dev_counter, p_term, p_trunc, obs_out, next_obs, reward, done, truncated, run_return, run_length, ep_return, ep_length, is_terminal);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_synth_env_trajectory(int64_t E, int D, int T, uint64_t seed, uint64_t step, const uint64_t* dev_counter, float p_term,
                                        float p_trunc, void* obs, void* next_obs, float* reward, uint8_t* done, uint8_t* truncated,
                                        float* ep_return, int32_t* ep_length, uint8_t* is_terminal, float* run_return,
                                        int32_t* run_length, void* stream) {
  STX_REQUIRE(E > 0 && T > 0 && D > 0 && D % 4 == 0 && D <= 128, STX_E_SHAPE,
              "stx_synth_env_trajectory: E=%lld T=%d D=%d (D must be a multiple of 4, at most 128)", (long long)E, T, D);
  STX_REQUIRE(obs && next_obs && reward && done && truncated && ep_return && ep_length && is_terminal && run_return && run_length,
              STX_E_ARG, "stx_synth_env_trajectory: null pointer");
  int L = 1;
  while (L < D / 4) L <<= 1;
  const int64_t threads = E * L;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  synth_env_trajectory_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      E, D, T, L, seed, step, dev_counter, p_term, p_trunc, reinterpret_cast<__nv_bfloat16*>(obs), reinterpret_cast<__nv_bfloat16*>(next_obs),
      reward, done, truncated, ep_return, ep_length, is_terminal, run_return, run_length);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_make_permutation(int32_t* perm, int64_t n, uint64_t seed, uint64_t stream_id,
                                    const uint64_t* dev_counter, void* stream) {
  STX_REQUIRE(perm && n > 0 && n < (1ll << 31), STX_E_ARG, "stx_make_permutation: n=%lld", (long long)n);
  int half_bits = 1;
  while ((1ll << (2 * half_bits)) < n) ++half_bits;
  permutation_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(perm, n, half_bits, seed, stream_id, dev_counter);
  STX_LAUNCH_OK();
  return STX_OK;
}
