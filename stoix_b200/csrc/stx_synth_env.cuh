// SyntheticBoxEnv's per-step draws and transforms: the ONE implementation shared by every kernel that steps this env
// (synth_env_step_kernel and synth_env_trajectory_kernel in stx_env.cu), so that the per-step path and the whole-trajectory
// path cannot drift apart.  Philox4x32-10 keyed by the env seed; counter = (env low, step low, env high << 16 ^ step high),
// the observation feature group xor-ed into the third word (<< 8) and a stream tag in the fourth, so the trajectory is a
// pure function of (seed, step, env).
#pragma once

#include "stx_common.cuh"

namespace stx {
namespace synth {

constexpr uint32_t kTagObs = 0x4f425331u;    // successor observation
constexpr uint32_t kTagReset = 0x52535431u;  // reset observation
constexpr uint32_t kTagStep = 0x53545031u;   // reward / termination / truncation

struct Ctr {
  uint32_t e_lo, st_lo, hi;
};
__device__ __forceinline__ Ctr counter(int64_t e, uint64_t step) {
  return Ctr{(uint32_t)e, (uint32_t)step, ((uint32_t)((uint64_t)e >> 32) << 16) ^ (uint32_t)(step >> 32)};
}

struct Outcome {
  float reward;
  bool term, trunc;
};
// reward ~ N(0, 1), termination with probability p_term, truncation (only if not terminated) with probability p_trunc
__device__ __forceinline__ Outcome outcome(const Ctr& c, uint2 key, float p_term, float p_trunc) {
  const uint4 rs = Philox::rand4(make_uint4(c.e_lo, c.st_lo, c.hi, kTagStep), key);
  Outcome o;
  o.reward = normal2(rs.x, rs.y).x;
  o.term = u01(rs.z) < p_term;
  o.trunc = !o.term && (u01(rs.w) < p_trunc);
  return o;
}

// The four N(0, 1) features of group `grp` (features 4 grp .. 4 grp + 3) of the successor (kTagObs) or reset (kTagReset)
// observation.
__device__ __forceinline__ float4 features4(const Ctr& c, uint2 key, uint32_t grp, uint32_t tag) {
  const uint4 r = Philox::rand4(make_uint4(c.e_lo, c.st_lo, c.hi ^ (grp << 8), tag), key);
  const float2 a = normal2(r.x, r.y), b = normal2(r.z, r.w);
  return make_float4(a.x, a.y, b.x, b.y);
}

// The transition's scalars of one env and step at index i of the (T, E) arrays, and RecordEpisodeMetrics: running
// return / length, published with is_terminal on the episode's last step, then reset.
__device__ __forceinline__ void record(const Outcome& o, float& run_ret, int32_t& run_len, int64_t i, float* reward, uint8_t* done,
                                       uint8_t* truncated, float* ep_return, int32_t* ep_length, uint8_t* is_terminal) {
  const bool last = o.term || o.trunc;
  const float ret = run_ret + o.reward;
  const int32_t len = run_len + 1;
  reward[i] = o.reward;
  done[i] = o.term ? 1 : 0;
  truncated[i] = o.trunc ? 1 : 0;
  ep_return[i] = ret;  // running totals; the finished episode's totals when is_terminal
  ep_length[i] = len;
  is_terminal[i] = last ? 1 : 0;
  run_ret = last ? 0.f : ret;
  run_len = last ? 0 : len;
}

}  // namespace synth
}  // namespace stx
