// The deterministic sum tree of the prioritised replay rings (Rainbow's n-step ring in stx_rainbow.cu, R2D2's sequence ring in
// stx_r2d2.cu): fan-out STX_PRIO_FANOUT over the items, leaves first, every parent the sum of its children in index order, rebuilt
// from them after every change (no atomics).  Semantics: include/stx.h.
#pragma once
#include "stx_common.cuh"

namespace stx {
namespace prio {

constexpr uint32_t kPrioTag = 0x5052494Fu;  // "PRIO"
constexpr int kTreeThreads = 1024;          // the one CTA that rewrites leaves and rebuilds their ancestors

// Level l (leaves l = 0, the root last) holds level_count(items, l) nodes from float level_offset(items, l).  Computed by short loops
// rather than kept in a table: a dynamically indexed table lives in local memory.
__host__ __device__ inline int64_t level_count(int64_t items, int l) {
  int64_t c = items;
  for (int k = 0; k < l; ++k) c = (c + STX_PRIO_FANOUT - 1) / STX_PRIO_FANOUT;
  return c;
}

__host__ __device__ inline int64_t level_offset(int64_t items, int l) {
  int64_t o = 0, c = items;
  for (int k = 0; k < l; ++k) o += c, c = (c + STX_PRIO_FANOUT - 1) / STX_PRIO_FANOUT;
  return o;
}

__host__ __device__ inline int tree_height(int64_t items) {  // levels, leaves and root included
  int n = 1;
  for (int64_t c = items; c > 1; c = (c + STX_PRIO_FANOUT - 1) / STX_PRIO_FANOUT) ++n;
  return n;
}

__host__ __device__ inline int64_t root_offset(int64_t items) { return level_offset(items, tree_height(items) - 1); }

// Rebuild the ancestors of the dirty leaves leaf(0 .. nd-1), level by level, each parent as the sum of its children in index order.
// Several dirty leaves share a parent: each of their threads writes the same sum.  Whole CTA.
template <class Leaf>
__device__ void tree_rebuild(float* __restrict__ tree, int64_t items, int64_t nd, Leaf leaf) {
  const int n = tree_height(items);
  int64_t span = 1;
  for (int l = 1; l < n; ++l) {
    __syncthreads();
    span *= STX_PRIO_FANOUT;
    const int64_t cnt_ch = level_count(items, l - 1), off_ch = level_offset(items, l - 1), off = off_ch + cnt_ch;
    for (int64_t j = threadIdx.x; j < nd; j += blockDim.x) {
      const int64_t node = leaf(j) / span, c0 = node * STX_PRIO_FANOUT;
      const int64_t c1 = min(c0 + STX_PRIO_FANOUT, cnt_ch);
      const float* ch = tree + off_ch;
      float s = 0.f;
      for (int64_t c = c0; c < c1; ++c) s = __fadd_rn(s, ch[c]);
      tree[off + node] = s;
    }
  }
}

// The stratum's uniform of sample r: u_in[r], or u01 of word r & 3 of Philox(seed; r / 4, call, call >> 32, "PRIO").
__device__ __forceinline__ float stratum_uniform(int64_t r, uint64_t seed, uint64_t call, const float* __restrict__ u_in) {
  if (u_in) return u_in[r];
  const uint4 wd = Philox::rand4(make_uint4((uint32_t)(r >> 2), (uint32_t)call, (uint32_t)(call >> 32), kPrioTag),
                                 make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const int w = (int)(r & 3);
  return u01(w == 0 ? wd.x : w == 1 ? wd.y : w == 2 ? wd.z : wd.w);
}

// Stratified descent of one warp (every lane gets the leaf): v = ((r + u) total) / M from the root; at each node the children in
// order, entering the first with v < s, else v -= s.  If none takes v (fp32 rounding left v at or past the node's sum), the last child
// with s > 0, and at every level below the last positive child too (v = +inf): the draw ends on the subtree's last positive leaf,
// next to v, not on its first.
__device__ __forceinline__ int64_t tree_descend(const float* __restrict__ tree, int64_t items, int64_t r, float u, int64_t M) {
  const int lane = threadIdx.x & 31;
  const int n = tree_height(items);
  const float total = tree[level_offset(items, n - 1)];
  float v = __fdiv_rn(__fmul_rn(__fadd_rn((float)r, u), total), (float)M);
  int64_t node = 0;  // index within level l
  for (int l = n - 1; l > 0; --l) {
    const int64_t c0 = node * STX_PRIO_FANOUT, nc = min((int64_t)STX_PRIO_FANOUT, level_count(items, l - 1) - c0);
    const float s_lane = lane < nc ? tree[level_offset(items, l - 1) + c0 + lane] : 0.f;
    int pick = -1, last_pos = 0;
    for (int c = 0; c < nc; ++c) {  // every lane runs the same sequence on the same values
      const float s = __shfl_sync(0xffffffffu, s_lane, c);
      if (s > 0.f) last_pos = c;
      if (pick < 0) {
        if (v < s) pick = c;
        else v = __fsub_rn(v, s);
      }
    }
    if (pick < 0) v = INFINITY;
    node = c0 + (pick < 0 ? last_pos : pick);
  }
  return node;
}

// set_priorities over `items` leaves, one CTA of kTreeThreads.  Duplicates in O(M): every row claims its leaf with an integer
// atomicMax of its batch position in `owner` (-1 between calls), so the last occurrence in batch order owns the leaf whatever the
// scheduling; the owner writes the value and resets the claim after the rebuild.
__device__ __forceinline__ void set_priorities(float* __restrict__ tree, int32_t* __restrict__ owner, float* __restrict__ max_priority,
                                               float exponent, int64_t items, const int32_t* __restrict__ idx, const float* __restrict__ pr,
                                               int64_t M) {
  __shared__ float red[kTreeThreads / 32];
  for (int64_t m = threadIdx.x; m < M; m += blockDim.x) atomicMax(owner + idx[m], (int)m);
  __syncthreads();
  float mx = -INFINITY;
  for (int64_t m = threadIdx.x; m < M; m += blockDim.x) {
    const float v = powf(pr[m], exponent);
    mx = fmaxf(mx, v);
    if (owner[idx[m]] == (int)m) tree[idx[m]] = v;
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, k));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  tree_rebuild(tree, items, M, [&](int64_t j) { return (int64_t)idx[j]; });
  __syncthreads();  // every owner test above is done before the claims are cleared
  for (int64_t m = threadIdx.x; m < M; m += blockDim.x) owner[idx[m]] = -1;
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, red[k]);
    *max_priority = fmaxf(*max_priority, m);
  }
}

}  // namespace prio
}  // namespace stx
