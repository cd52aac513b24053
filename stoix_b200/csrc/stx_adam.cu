// K4 -- fused multi-segment global-norm clip + Adam + LR schedule + apply (+ bf16 weight shadow).
//
// Reference: optax.chain(optax.clip_by_global_norm(max_grad_norm), optax.adam(lr, eps=1e-5)) built at
// stoix/systems/ppo/anakin/ff_ppo.py:449-463 and applied at :264-273 (update + apply_updates), with
// the linear schedule of stoix/utils/training.py:24-26.  optax (0.2.7.dev0 @17411bc) is not vendored
// in the reference; the arithmetic below restates its published definitions (SURVEY.md A.5):
//   g_norm = sqrt(sum g^2) over the segment;  g <- g              if g_norm <  max_norm
//                                              g <- g/g_norm*max  otherwise
//   mu = b1*mu + (1-b1)*g ; nu = b2*nu + (1-b2)*g^2 ; c = count+1
//   u  = (mu/(1-b1^c)) / (sqrt(nu/(1-b2^c)) + eps)
//   lr = init_lr * (1 - (sched_count // steps_per_update) / num_updates)    [read before increment]
//   p  = p - lr*u
// The reference launches dozens of tiny XLA fusions per optimiser (12 leaves x 2 networks); here it
// is ONE launch over the flat arena for all segments (actor and critic are separate optimisers =
// separate segments, clipped separately).  Phase 1 writes per-block sum-of-squares partials, a
// software grid barrier (grid <= co-resident capacity) separates it from phase 2, which re-reduces
// the partials in a fixed order (deterministic) and applies the update with 128-bit accesses.
#include "stx_common.cuh"

namespace stx {
namespace {

constexpr int kAdamThreads = 256;

// ---- C1 fused into K4: one-shot all-reduce over NVLink peer memory ------------------------------------
// Every rank's gradient arena lives in symmetric (peer-mapped) memory.  Rank r announces "my gradients of
// call #gen are complete" by writing gen into slot r of every peer's signal pad (block 0), every block waits until
// all peers announced the same (polling the local pad), then each rank sums the W arenas in rank order straight from peer memory (ld.global
// over NVLink) -- identical association order everywhere => bit-identical parameters on all ranks.  The
// gradient arenas are ping-ponged by the caller, so this single handshake per call also guarantees that a
// buffer is not overwritten while a peer may still be reading it (see DESIGN.md section 5).
struct PeerSync {
  const float* peer_grads[8];   // this call's gradient arena on every rank (peer-mapped pointers)
  unsigned int* peer_pads[8];   // signal pads of every rank (slot [rank] is written by that rank)
  unsigned int* my_pad;
  unsigned int* local_gen;      // device counter: number of completed calls
  float* gsum;                  // local arena receiving the summed gradient
  int world, rank;
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void grid_barrier(unsigned long long* arrive) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned long long t = atomicAdd(arrive, 1ull);
    const unsigned long long target = (t / gridDim.x + 1ull) * gridDim.x;
    unsigned int spins = 0;
    unsigned long long t0 = 0ull;
    while (*reinterpret_cast<volatile unsigned long long*>(arrive) < target) spin_guard(spins, t0, "optimiser grid barrier");
    __threadfence();
  }
  __syncthreads();
}

// The update rule of phase 2, a compile-time choice: Adam (stx_clip_adam_step and the fused all-reduce), optax.scale_by_radam
// (stx_clip_radam_step) or optax.scale_by_rms at optax.rmsprop's defaults (stx_clip_rmsprop_step, which reads and writes nu only).  The rectifier of RAdam depends on the step count only; it is derived once per segment in double
// precision next to the bias corrections: rho_t = rho_inf - 2 t b2^t / (1 - b2^t) subtracts two numbers of nearly the same size
// (rho_inf = 1999 at b2 = 0.999), which in fp32 puts a relative error of 1.8e-3 on r_t at t = 6 (DESIGN.md section 2, tolerance scheme).
struct RadamArgs {
  float eps_root, threshold;
};
enum UpdateRule : int { kRuleAdam = 0, kRuleRadam = 1, kRuleRmsprop = 2 };

// PEER: 0 = local gradients; 1 = one-shot all-reduce (every rank loads all W arenas).
template <bool PRENORM, int PEER, int RULE = kRuleAdam>
__global__ void __launch_bounds__(kAdamThreads)
    clip_adam_kernel(float* __restrict__ P, const float* G, float* __restrict__ MU,
                     float* __restrict__ NU, int32_t* __restrict__ counts,
                     const StxAdamSeg* __restrict__ segs, int nseg, StxAdamHyper h,
                     __nv_bfloat16* __restrict__ P16, float* __restrict__ gnorm_out,
                     AdamScratch* scratch, const PeerSync ps, const RadamArgs rx) {
  double* partials = scratch->partials;
  __shared__ double sred[32];
  __shared__ StxAdamSeg s_seg[kAdamMaxSegs];
  __shared__ float s_gs[kAdamMaxSegs], s_bc1[kAdamMaxSegs], s_bc2[kAdamMaxSegs], s_lr[kAdamMaxSegs], s_gn[kAdamMaxSegs];
  __shared__ float s_rect[kAdamMaxSegs];  // kRuleRadam: r_t, or 0 on the un-rectified branch (rho_t < threshold)
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int gthreads = gridDim.x * blockDim.x;
  griddep_launch();
  griddep_wait();  // gradients (and, with PRENORM, their sum-of-squares partials) come from the previous kernel
  if ((int)threadIdx.x < nseg) s_seg[threadIdx.x] = segs[threadIdx.x];
  __syncthreads();

  if (PEER == 1) {
    // ---- phase 0: cross-rank handshake, then all-reduce by direct peer loads into ps.gsum ----
    const unsigned int gen = *reinterpret_cast<volatile unsigned int*>(ps.local_gen) + 1u;
    // block 0 announces; EVERY block polls the local signal pad itself (one hop instead of pad -> block 0 -> flag)
    if ((int)threadIdx.x < ps.world) {
      const int peer = threadIdx.x;
      if (blockIdx.x == 0) {
        __threadfence_system();
        st_release_sys(ps.peer_pads[peer] + ps.rank, gen);
      }
      unsigned int spins = 0;
      unsigned long long t0 = 0ull;
      while (ld_acquire_sys(ps.my_pad + peer) < gen) spin_guard(spins, t0, "peer gradient hand-shake");
    }
    __syncthreads();
    for (int s = 0; s < nseg; ++s) {
      const StxAdamSeg seg = s_seg[s];
      const int64_t n4 = seg.count / 4;
      float ss = 0.f;  // sum of squares of the scaled sum, accumulated in the order of phase 1 (which PEER then skips)
      for (int64_t i = gtid; i < n4; i += gthreads) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 v[8];
#pragma unroll
        for (int r = 0; r < 8; ++r)  // every peer load in flight before the first add
          if (r < ps.world) v[r] = __ldcg(reinterpret_cast<const float4*>(ps.peer_grads[r] + seg.offset) + i);
#pragma unroll
        for (int r = 0; r < 8; ++r)  // fixed rank order on every rank
          if (r < ps.world) acc.x += v[r].x, acc.y += v[r].y, acc.z += v[r].z, acc.w += v[r].w;
        reinterpret_cast<float4*>(ps.gsum + seg.offset)[i] = acc;
        float4 g = acc;
        g.x *= h.grad_scale, g.y *= h.grad_scale, g.z *= h.grad_scale, g.w *= h.grad_scale;
        ss += g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
      }
      for (int64_t i = n4 * 4 + gtid; i < seg.count; i += gthreads) {
        float acc = 0.f;
        for (int r = 0; r < ps.world; ++r) acc += __ldcg(ps.peer_grads[r] + seg.offset + i);
        ps.gsum[seg.offset + i] = acc;
        const float g = acc * h.grad_scale;
        ss += g * g;
      }
      const double bs = block_sum<double>((double)ss, sred);
      if (threadIdx.x == 0) partials[(int64_t)s * gridDim.x + blockIdx.x] = bs;
    }
    __syncthreads();  // this block re-reads only what it wrote (same index mapping in phase 2)
    G = ps.gsum;
  }

  // ---- phase 1: per-segment sum of squares of (grad * grad_scale) ----
  // (PRENORM: the producer of the gradients already left sum(g^2) partials of the unscaled gradients here)
  for (int s = 0; s < nseg && !PRENORM && !PEER; ++s) {
    const StxAdamSeg seg = s_seg[s];
    const float4* g4 = reinterpret_cast<const float4*>(G + seg.offset);
    const int64_t n4 = seg.count / 4;
    float acc = 0.f;
    for (int64_t i = gtid; i < n4; i += gthreads) {
      float4 g = g4[i];
      g.x *= h.grad_scale, g.y *= h.grad_scale, g.z *= h.grad_scale, g.w *= h.grad_scale;
      acc += g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
    }
    for (int64_t i = n4 * 4 + gtid; i < seg.count; i += gthreads) {
      const float g = G[seg.offset + i] * h.grad_scale;
      acc += g * g;
    }
    const double bs = block_sum<double>((double)acc, sred);
    if (threadIdx.x == 0) partials[(int64_t)s * gridDim.x + blockIdx.x] = bs;
  }
  if (!PRENORM) grid_barrier(&scratch->arrive);
  if (PEER == 1 && gtid == 0) *ps.local_gen = *ps.local_gen + 1u;  // every block read local_gen before this barrier

  // ---- phase 2 ----
  // PRENORM: the gradients are final at kernel entry, so the first item of the first two segments is requested
  // BEFORE the norm reduction: its loads overlap the (dependent) partials round trip.
  // parameters, moments, gradients and the bf16 shadow (the next K3a's weights) stay L2-resident under the activation
  // stream of the surrounding kernels: this kernel is a chain of dependent round trips
  const uint64_t pol_keep = l2_evict_last();
  constexpr int kPf = 2;
  float4 pf_g[kPf], pf_m[kPf], pf_v[kPf], pf_p[kPf];
  if (PRENORM) {
#pragma unroll
    for (int s = 0; s < kPf; ++s)
      if (s < nseg && gtid < s_seg[s].count / 4) {
        const int64_t o = s_seg[s].offset;
        pf_g[s] = ld_hint(reinterpret_cast<const float4*>(G + o) + gtid, pol_keep);
        pf_m[s] = ld_hint(reinterpret_cast<const float4*>(MU + o) + gtid, pol_keep);
        pf_v[s] = ld_hint(reinterpret_cast<const float4*>(NU + o) + gtid, pol_keep);
        pf_p[s] = ld_hint(reinterpret_cast<const float4*>(P + o) + gtid, pol_keep);
      }
  }
  // every block re-reduces the per-block partials in the same fixed order (warp s <-> segment s: lane-strided
  // loads, xor-butterfly) and lane 0 derives the segment's scalars once for the whole block
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < nseg) {
    const int s = warp;
    const unsigned int nparts = PRENORM ? (unsigned int)__ldcg(&scratch->n_partials) : gridDim.x;
    const double* vp = partials + (int64_t)s * nparts;
    int32_t cnt_adam = 0, cnt_sched = 0;  // requested together with the partials (one round trip, not two)
    if (lane == 0) cnt_adam = counts[2 * s], cnt_sched = counts[2 * s + 1];
    double part = 0.0;
    for (unsigned int b = lane; b < nparts; b += 32) part += __ldcg(vp + b);
    part = warp_sum(part);
    if (lane == 0) {
      const double ss = PRENORM ? part * (double)h.grad_scale * (double)h.grad_scale : part;
      const float g_norm = (float)sqrt(ss);
      // optax.clip_by_global_norm: trigger = g_norm < max_norm
      const float clip = (g_norm < s_seg[s].max_grad_norm) ? 1.0f : s_seg[s].max_grad_norm / g_norm;
      const int32_t c = cnt_adam + 1;
      float lr = s_seg[s].init_lr;
      if (h.decay) {
        const int32_t k = cnt_sched / h.steps_per_update;  // floor division, utils/training.py:25
        lr = s_seg[s].init_lr * (1.0f - (float)k / (float)h.num_updates);
      }
      s_gs[s] = h.grad_scale * clip;
      s_bc1[s] = 1.0f - powf(h.b1, (float)c);
      s_bc2[s] = 1.0f - powf(h.b2, (float)c);
      s_lr[s] = lr;
      s_gn[s] = g_norm;
      if constexpr (RULE == kRuleRadam) {  // optax.scale_by_radam, rectifier in double precision
        const double b2 = (double)h.b2, t = (double)c;
        const double rho_inf = 2.0 / (1.0 - b2) - 1.0;
        const double b2t = pow(b2, t);
        const double rho = rho_inf - 2.0 * t * b2t / (1.0 - b2t);
        s_rect[s] = rho >= (double)rx.threshold
                        ? (float)sqrt((rho - 4.0) * (rho - 2.0) * rho_inf / ((rho_inf - 4.0) * (rho_inf - 2.0) * rho))
                        : 0.f;
      }
    }
  }
  __syncthreads();
  const float ob1 = 1.0f - h.b1, ob2 = 1.0f - h.b2;
  for (int s = 0; s < nseg; ++s) {
    const StxAdamSeg seg = s_seg[s];
    const float gs = s_gs[s], bc1 = s_bc1[s], bc2 = s_bc2[s], lr = s_lr[s];
    const float rect = RULE == kRuleRadam ? s_rect[s] : 0.f;
    // the step direction of one element: Adam's, or RAdam's (r_t mhat / (sqrt(vhat + eps_root) + eps), else mhat)
    auto direction = [&](float me, float ve) -> float {
      if constexpr (RULE == kRuleRadam) {
        const float mh = me / bc1;
        return rect > 0.f ? rect * mh / (sqrtf(ve / bc2 + rx.eps_root) + h.eps) : mh;
      } else {
        return (me / bc1) / (sqrtf(ve / bc2) + h.eps);
      }
    };
    float* p = P + seg.offset;
    float* mu = MU + seg.offset;
    float* nu = NU + seg.offset;
    const float* g = G + seg.offset;
    const int64_t n4 = seg.count / 4;
    for (int64_t i = gtid; i < n4; i += gthreads) {
      float4 gv, m, v, pv;
      if (PRENORM && s < kPf && i == gtid) {
        gv = pf_g[s < kPf ? s : 0], m = pf_m[s < kPf ? s : 0], v = pf_v[s < kPf ? s : 0], pv = pf_p[s < kPf ? s : 0];
      } else {
        gv = ld_hint(reinterpret_cast<const float4*>(g) + i, pol_keep);
        if constexpr (RULE == kRuleRmsprop) m = make_float4(0.f, 0.f, 0.f, 0.f);
        else m = ld_hint(reinterpret_cast<const float4*>(mu) + i, pol_keep);
        v = ld_hint(reinterpret_cast<const float4*>(nu) + i, pol_keep);
        pv = ld_hint(reinterpret_cast<const float4*>(p) + i, pol_keep);
      }
      float ge[4] = {gv.x * gs, gv.y * gs, gv.z * gs, gv.w * gs};
      float me[4] = {m.x, m.y, m.z, m.w}, ve[4] = {v.x, v.y, v.z, v.w}, pe[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (RULE == kRuleRmsprop) {  // optax.scale_by_rms, eps inside the square root
          ve[k] = ob2 * ge[k] * ge[k] + h.b2 * ve[k];
          pe[k] = pe[k] - lr * (ge[k] / sqrtf(ve[k] + h.eps));
        } else {
          me[k] = h.b1 * me[k] + ob1 * ge[k];
          ve[k] = h.b2 * ve[k] + ob2 * ge[k] * ge[k];
          const float u = direction(me[k], ve[k]);
          pe[k] = pe[k] - lr * u;
        }
      }
      if constexpr (RULE != kRuleRmsprop) st_hint(reinterpret_cast<float4*>(mu) + i, make_float4(me[0], me[1], me[2], me[3]), pol_keep);
      st_hint(reinterpret_cast<float4*>(nu) + i, make_float4(ve[0], ve[1], ve[2], ve[3]), pol_keep);
      st_hint(reinterpret_cast<float4*>(p) + i, make_float4(pe[0], pe[1], pe[2], pe[3]), pol_keep);
      if (P16) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(pe[0], pe[1]), hi = __floats2bfloat162_rn(pe[2], pe[3]);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&lo);
        pk.y = *reinterpret_cast<uint32_t*>(&hi);
        st_hint(reinterpret_cast<uint2*>(P16 + seg.offset) + i, pk, pol_keep);
      }
    }
    for (int64_t i = n4 * 4 + gtid; i < seg.count; i += gthreads) {
      const float ge = g[i] * gs;
      float pn;
      if constexpr (RULE == kRuleRmsprop) {
        const float ve = ob2 * ge * ge + h.b2 * nu[i];
        pn = p[i] - lr * (ge / sqrtf(ve + h.eps));
        nu[i] = ve, p[i] = pn;
      } else {
        const float me = h.b1 * mu[i] + ob1 * ge;
        const float ve = h.b2 * nu[i] + ob2 * ge * ge;
        const float u = direction(me, ve);
        pn = p[i] - lr * u;
        mu[i] = me, nu[i] = ve, p[i] = pn;
      }
      if (P16) P16[seg.offset + i] = __float2bfloat16_rn(pn);
    }
  }
  // The step counters are read by every block (above) and advanced by whichever block finishes LAST: no block can
  // still need the old values then, with or without the grid barrier.
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned long long t = atomicAdd(&scratch->finish, 1ull);
    if (t % gridDim.x == gridDim.x - 1) {
      for (int s = 0; s < nseg; ++s) {
        counts[2 * s] += 1;
        counts[2 * s + 1] += 1;
        if (gnorm_out) gnorm_out[s] = s_gn[s];
      }
    }
  }
}

__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = __float2bfloat16_rn(src[i]);
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" size_t stx_adam_scratch_bytes(int nseg) {
  (void)nseg;
  return sizeof(AdamScratch);
}

// Host-side mirror of the segment table is needed to size the grid: callers pass the total span.
extern "C" int stx_clip_adam_step(float* param_arena, const float* grad_arena, float* mu, float* nu,
                                  int32_t* counts, const StxAdamSeg* segs, int nseg,
                                  const StxAdamHyper* hyper, void* params_bf16, float* gnorm_out,
                                  void* scratch, void* stream) {
  STX_REQUIRE(param_arena && grad_arena && mu && nu && counts && segs && hyper && scratch, STX_E_ARG,
              "stx_clip_adam_step: null pointer");
  STX_REQUIRE(nseg >= 1 && nseg <= kAdamMaxSegs, STX_E_SHAPE, "stx_clip_adam_step: nseg=%d (max %d)", nseg, kAdamMaxSegs);
  STX_REQUIRE(aligned16(param_arena) && aligned16(grad_arena) && aligned16(mu) && aligned16(nu), STX_E_ALIGN,
              "stx_clip_adam_step: arenas must be 16-byte aligned");
  STX_REQUIRE(hyper->steps_per_update > 0 && hyper->num_updates > 0, STX_E_ARG,
              "stx_clip_adam_step: steps_per_update/num_updates must be positive");
  // The grid is fixed (one wave) so the barrier ticket arithmetic is launch-invariant.
  const int grid = kNumSMs;
  const PeerSync none{};
  if (hyper->prenorm)
    STX_CUDA_OK(launch_pdl(clip_adam_kernel<true, 0>, dim3(grid), dim3(kAdamThreads), 0, (cudaStream_t)stream, param_arena, grad_arena,
                           mu, nu, counts, segs, nseg, *hyper, reinterpret_cast<__nv_bfloat16*>(params_bf16), gnorm_out,
                           reinterpret_cast<AdamScratch*>(scratch), none, RadamArgs{}));
  else
    STX_CUDA_OK(launch_pdl(clip_adam_kernel<false, 0>, dim3(grid), dim3(kAdamThreads), 0, (cudaStream_t)stream, param_arena, grad_arena,
                           mu, nu, counts, segs, nseg, *hyper, reinterpret_cast<__nv_bfloat16*>(params_bf16), gnorm_out,
                           reinterpret_cast<AdamScratch*>(scratch), none, RadamArgs{}));
  STX_LAUNCH_OK();
  return STX_OK;
}

// clip + RAdam: the same launch as stx_clip_adam_step with the RAdam rule (PQN, ff_pqn.py:263-267).
extern "C" int stx_clip_radam_step(float* param_arena, const float* grad_arena, float* mu, float* nu, int32_t* counts, const StxAdamSeg* segs,
                                   int nseg, const StxRadamHyper* hyper, void* params_bf16, float* gnorm_out, void* scratch, void* stream) {
  STX_REQUIRE(param_arena && grad_arena && mu && nu && counts && segs && hyper && scratch, STX_E_ARG, "stx_clip_radam_step: null pointer");
  STX_REQUIRE(nseg >= 1 && nseg <= kAdamMaxSegs, STX_E_SHAPE, "stx_clip_radam_step: nseg=%d (max %d)", nseg, kAdamMaxSegs);
  STX_REQUIRE(aligned16(param_arena) && aligned16(grad_arena) && aligned16(mu) && aligned16(nu), STX_E_ALIGN,
              "stx_clip_radam_step: arenas must be 16-byte aligned");
  STX_REQUIRE(hyper->adam.steps_per_update > 0 && hyper->adam.num_updates > 0, STX_E_ARG,
              "stx_clip_radam_step: steps_per_update/num_updates must be positive");
  STX_REQUIRE(!hyper->adam.prenorm, STX_E_ARG, "stx_clip_radam_step: prenorm is not available with RAdam");
  STX_REQUIRE(hyper->eps_root >= 0.f, STX_E_ARG, "stx_clip_radam_step: eps_root=%g must be >= 0", (double)hyper->eps_root);
  const PeerSync none{};
  STX_CUDA_OK(launch_pdl(clip_adam_kernel<false, 0, kRuleRadam>, dim3(kNumSMs), dim3(kAdamThreads), 0, (cudaStream_t)stream, param_arena, grad_arena,
                         mu, nu, counts, segs, nseg, hyper->adam, reinterpret_cast<__nv_bfloat16*>(params_bf16), gnorm_out,
                         reinterpret_cast<AdamScratch*>(scratch), none, RadamArgs{hyper->eps_root, hyper->threshold}));
  STX_LAUNCH_OK();
  return STX_OK;
}

// clip + RMSProp: the same launch with optax.rmsprop at its defaults (IMPALA, ff_impala.py:754-766); the mu arena is not touched.
extern "C" int stx_clip_rmsprop_step(float* param_arena, const float* grad_arena, float* nu, int32_t* counts, const StxAdamSeg* segs, int nseg,
                                     const StxAdamHyper* hyper, void* params_bf16, float* gnorm_out, void* scratch, void* stream) {
  STX_REQUIRE(param_arena && grad_arena && nu && counts && segs && hyper && scratch, STX_E_ARG, "stx_clip_rmsprop_step: null pointer");
  STX_REQUIRE(nseg >= 1 && nseg <= kAdamMaxSegs, STX_E_SHAPE, "stx_clip_rmsprop_step: nseg=%d (max %d)", nseg, kAdamMaxSegs);
  STX_REQUIRE(aligned16(param_arena) && aligned16(grad_arena) && aligned16(nu), STX_E_ALIGN, "stx_clip_rmsprop_step: arenas must be 16-byte aligned");
  STX_REQUIRE(hyper->steps_per_update > 0 && hyper->num_updates > 0, STX_E_ARG,
              "stx_clip_rmsprop_step: steps_per_update/num_updates must be positive");
  STX_REQUIRE(!hyper->prenorm, STX_E_ARG, "stx_clip_rmsprop_step: prenorm is not available with RMSProp");
  const PeerSync none{};
  STX_CUDA_OK(launch_pdl(clip_adam_kernel<false, 0, kRuleRmsprop>, dim3(kNumSMs), dim3(kAdamThreads), 0, (cudaStream_t)stream, param_arena,
                         grad_arena, static_cast<float*>(nullptr), nu, counts, segs, nseg, *hyper, reinterpret_cast<__nv_bfloat16*>(params_bf16),
                         gnorm_out, reinterpret_cast<AdamScratch*>(scratch), none, RadamArgs{}));
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
  STX_REQUIRE(src && dst && n >= 0, STX_E_ARG, "stx_cast_f32_to_bf16: bad args");
  if (n == 0) return STX_OK;
  int64_t blocks = (n + 255) / 256;
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  cast_bf16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  STX_LAUNCH_OK();
  return STX_OK;
}

// Fused gradient all-reduce + clip + Adam (one launch per optimiser step on every rank).
extern "C" int stx_allreduce_clip_adam_step(float* param_arena, const float* const* peer_grads, void* const* peer_signal_pads,
                                            int world, int rank, int pad_slot_offset, float* gsum, float* mu, float* nu,
                                            int32_t* counts, const StxAdamSeg* segs, int nseg, const StxAdamHyper* hyper,
                                            void* params_bf16, float* gnorm_out, void* scratch, void* stream) {
  STX_REQUIRE(param_arena && peer_grads && peer_signal_pads && gsum && mu && nu && counts && segs && hyper && scratch, STX_E_ARG,
              "stx_allreduce_clip_adam_step: null pointer");
  STX_REQUIRE(world >= 2 && world <= 8 && rank >= 0 && rank < world, STX_E_SHAPE, "stx_allreduce_clip_adam_step: world=%d rank=%d (2..8 ranks)", world, rank);
  STX_REQUIRE(nseg >= 1 && nseg <= kAdamMaxSegs, STX_E_SHAPE, "stx_allreduce_clip_adam_step: nseg=%d", nseg);
  STX_REQUIRE(!hyper->prenorm, STX_E_ARG, "stx_allreduce_clip_adam_step: prenorm is a single-device shortcut");
  PeerSync ps{};
  for (int r = 0; r < world; ++r) {
    STX_REQUIRE(peer_grads[r] && peer_signal_pads[r], STX_E_ARG, "stx_allreduce_clip_adam_step: null peer pointer %d", r);
    ps.peer_grads[r] = peer_grads[r];
    ps.peer_pads[r] = reinterpret_cast<unsigned int*>(peer_signal_pads[r]) + pad_slot_offset;
  }
  ps.my_pad = ps.peer_pads[rank];
  ps.local_gen = &reinterpret_cast<AdamScratch*>(scratch)->gen;
  ps.gsum = gsum, ps.world = world, ps.rank = rank;
  STX_CUDA_OK(launch_pdl(clip_adam_kernel<false, 1>, dim3(kNumSMs), dim3(kAdamThreads), 0, (cudaStream_t)stream, param_arena,
                         static_cast<const float*>(gsum), mu, nu, counts, segs, nseg, *hyper,
                         reinterpret_cast<__nv_bfloat16*>(params_bf16), gnorm_out, reinterpret_cast<AdamScratch*>(scratch), ps, RadamArgs{}));
  STX_LAUNCH_OK();
  return STX_OK;
}
