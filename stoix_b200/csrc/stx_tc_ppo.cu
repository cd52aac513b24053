// K3 (bf16 path): the PPO minibatch gradient step on Hopper tensor cores (wgmma).
//
// Reference semantics: _actor_loss_fn / _critic_loss_fn + jax.grad for one minibatch
// (stoix/systems/ppo/anakin/ff_ppo.py:184-247; losses stoix/utils/loss.py:17-32,68-78).  Three launches:
//
//  tc_ppo_fwd_bwd_kernel (K3a)  one persistent CTA per SM; CTAs [0, n_a) run the actor, the rest the critic.
//      Two warpgroups per CTA, each running its own sequence of 64-row tiles (rows gathered through the shuffle
//      permutation straight into 128B-swizzled smem):
//        G0 X*W0 -> E0 h1=relu(.+b0) -> G1 h1*W1 -> E1 h2 -> G2 h2*W2 -> E2 loss + d(logits|value) ->
//        G3 dz*W2^T -> E3 dh2 = .*(h2>0) -> G4 dh2*W1^T -> E4 dh1 = .*(h1>0)
//      All five GEMMs run on wgmma with the activations resident in registers (A operand from registers: the
//      accumulator of one GEMM packed to bf16 is the A operand of the next); W1's single smem image serves as
//      MN-major B (forward) and K-major B (backward).  256-wide GEMMs run as two N=128 halves (64 accumulator
//      registers).  The epilogues also emit h2, dh1, dz (bf16) and the h2 > 0 sign mask for the weight-gradient GEMMs,
//      reduce the bias gradients (quad butterfly + per-warp smem slices, fixed order) and accumulate the loss metrics.
//  tc_dw_kernel (K3b)  split-K GEMMs dW = A^T * B over the minibatch rows with both operands MN-major, on a fixed plan of
//      CTAs per job (kDwCtasW1 / W2 / W0), two consumer warpgroups with fp32 register accumulators and a third warpgroup that
//      feeds them:
//        dW2 = h2^T dz (N=16), dW0^T = dh1^T x (N=64): 4-stage TMA/mbarrier ring of A and B (one producer warp);
//        dW1 = h1^T dh2 in two jobs of 128 hidden units (N=256): the third warpgroup rebuilds h1[:, half] = relu(x W0 + b0)
//        and dh2 = (dz W2^T) * mask per 64-row chunk from x, dz and the mask (12 KB instead of 96 KB of stored h1 and dh2)
//        with K3a's own instruction sequences, into double-buffered smem images that the consumers multiply.
//      The activations travel K3a -> K3b in a tiled layout [tile of 128 rows][8-column group][row][8]:
//      one TMA box of K3b lands 64 rows of every column group as un-swizzled core matrices (8 rows x 16 B).
//  tc_reduce_kernel     fixed-order reduction of the per-CTA partials into the flat fp32 gradient arena
//      (deterministic; also the bias gradients and the six loss metrics); optionally leaves the sum(g^2)
//      partials of both networks for clip + Adam (PRENORM).
// The three kernels (and K4 behind them) are chained with programmatic dependent launch; activations carry
// evict_first, partials / gradients evict_last L2 policies (see stx_common.cuh).
#include <cuda.h>

#include "stx_common.cuh"
#include "stx_tc_ptx.cuh"

namespace stx {
namespace tc {

int make_map_2d_pub(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows,
                    uint32_t box_cols);  // stx_tc_mlp.cu (SWIZZLE_128B bf16)
int make_map_tiled(CUtensorMap* m, const void* base, uint64_t tiles, uint32_t colgroups, uint32_t box_cg);  // stx_tc_mlp.cu

// optional instrumentation hook of the C ABI (stx_tc_debug_set_prof_buffer): K3b's [gridDim][8] per-CTA profile record
__device__ long long* g_prof_buf = nullptr;

__device__ __forceinline__ long long globaltimer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

constexpr int kH = 256;
constexpr int kWTile = 64;               // rows per warpgroup tile
constexpr int kFbThreads = 256;          // two warpgroups

// ---- K3a shared-memory map ------------------------------------------------------------------------
// Each warpgroup has two stages of its tile inputs: the tile being computed and the next one, gathered with cp.async meanwhile.
constexpr uint32_t kOffX = kImgWBytes;               // [2 warpgroups][2 stages] X tile, 8 KB
constexpr uint32_t kOffLoss = kOffX + 4 * 8192;      // [2 warpgroups][2 stages][3][64] per-row loss inputs (see gather_tile)
constexpr uint32_t kLossStageBytes = 3 * 64 * 4;
constexpr uint32_t kOffBias = kOffLoss + 4 * kLossStageBytes;  // b0[256] b1[256] b2[16]
constexpr uint32_t kOffDb = kOffBias + 528 * 4;      // [8 warps][db0[256] db1[256] db2[16]] accumulators
constexpr uint32_t kOffBar = kOffDb + 8 * 528 * 4;
constexpr uint32_t kFbSmemBytes = kOffBar + 64 + 1024;
// + the kernel's static s_mw[8][6]; 227 KB is the most a block may use on sm_90
static_assert(kFbSmemBytes + 8 * 6 * 4 <= 227 * 1024, "K3a shared memory exceeds the per-block limit");

struct FbNet {
  const __nv_bfloat16* w2;   // [256 x A] bf16
  const float *b0, *b1, *b2;
  __nv_bfloat16 *h2, *dh1;            // [mb x 256], tiled layout (see tiled_ptr)
  __nv_bfloat16* dz;                   // [mb x 16] tiled (columns >= A are zero)
  uint4* mask;                         // [mb / 64][128]: h2 > 0 bits of each 64-row tile in fragment order (see mask_bit)
  float* db_part;                      // [n_cta_of_net][528]
  int A;
  int is_actor;
};

struct FbParams {
  FbNet net[2];
  int n_cta[2];             // CTAs per net (actor first)
  const __nv_bfloat16* obs; // [B x D]
  __nv_bfloat16* xg;        // [mb x 64] gathered input rows, tiled layout (written by the actor CTAs)
  const int32_t* idx;       // perm + mb_off, or nullptr (then rows are row0 + i)
  int64_t row0;
  const int32_t* action;
  const float *logp_old, *v_old, *adv, *tgt, *adv_stats;
  float* metric_part;       // [gridDim][8]
  int D;
  int mb;
  float inv_m;              // 1 / mb, computed on the host (a device division would be a library call in this kernel)
  float clip_eps, ent_coef, vf_coef;
};

// Tiled activation layout shared by K3a (writer) and K3b (reader): element (row, col) of a [mb x 8*CG]
// matrix lives at ((row/128 * CG + col/8) * 128 + row%128) * 8 + col%8.
__device__ __forceinline__ __nv_bfloat16* tiled_ptr(__nv_bfloat16* base, int64_t row, int col, int CG) {
  return base + (((row >> 7) * CG + (col >> 3)) * 128 + (row & 127)) * 8 + (col & 7);
}

// Sign mask of h2 in fragment order: thread t of the warpgroup that owns a 64-row tile keeps the bits of its register operand
// a2[64] (rows 16 (t / 32) + (t % 32) / 4 (+ 8), see stx_tc_ptx.cuh) in one uint4: element e of a2[32 h + i] is bit
// 2 (i % 16) + e of word 2 h + i / 16.  K3b's rebuild of dh2 runs the same MMA with the same thread <-> (row, column) mapping,
// so each thread reads back exactly its own 16 bytes.
__device__ __forceinline__ int mask_word(int h, int i) { return 2 * h + (i >> 4); }
__device__ __forceinline__ uint32_t mask_bit(int i, int e) { return (uint32_t)(2 * (i & 15) + e); }

// Stores half h of a packed 64 x 256 register operand (a: its 32 words of half h; rows row0, row0 + 8 of the thread, see
// stx_tc_ptx.cuh) to the tiled layout.  evict_first, like every activation store: K3b reads each activation once.  (The policy
// is created per store site: one policy kept live across the whole K3a tile loop costs it spills.)
__device__ __forceinline__ void store_act(__nv_bfloat16* base, const uint32_t* a, int h, int64_t row0, int lane) {
  const uint64_t pol = l2_evict_first();
#pragma unroll
  for (int i = 0; i < 32; ++i)
    st_hint(reinterpret_cast<uint32_t*>(tiled_ptr(base, row0 + 8 * (i & 1), 128 * h + 8 * (i >> 1) + 2 * (lane & 3), 32)), a[i], pol);
}

// cp.async global -> shared, L2 only (every gathered row is read once here); src_bytes = 0 zero-fills the 16 bytes
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// One reduce-scatter step of colsum_half at lane distance S, on entries k, k + 4, k + 8, ... of one class (v[j] = entry k + 4 j):
// of the 2 S entries still held, lane l keeps half (l & S) and adds its partner's copy of it.  S is a template parameter so
// that every index into v is a compile-time constant (a loop over S leaves the inner loop rolled and v in local memory).
template <int S>
__device__ __forceinline__ void colsum_step(float (&v)[8], int lane) {
  const bool hi = (lane & S) != 0;
#pragma unroll
  for (int j = 0; j < S / 4; ++j) {
    const float send = hi ? v[j] : v[j + S / 4];
    const float keep = hi ? v[j + S / 4] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, S);
  }
}

// Column sums over the 64 rows of a warpgroup tile, half h: x = accumulator-layout values of this thread.  The 8 lanes that
// share lane % 4 hold the same columns; a reduce-scatter butterfly over the 32 row-pair sums e (e = 2 j + b: x[4 j + b] +
// x[4 j + b + 2]) leaves lane l with the totals of its entries 4 (l/4) + k, k < 4.  The butterfly pairs e with e + 16, e + 8,
// e + 4, so the four classes e % 4 = k reduce independently: one class at a time keeps 8 partial sums live instead of 32.
// dst: this warp's slice (every column written by exactly one lane of the warp: fixed order, no atomics).
__device__ __forceinline__ void colsum_half(const float (&x)[64], float* dst, int h, int lane) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = k + 4 * j, i = 4 * (e >> 1) + (e & 1);
      v[j] = x[i] + x[i + 2];
    }
    colsum_step<16>(v, lane);
    colsum_step<8>(v, lane);
    colsum_step<4>(v, lane);
    const int m = 4 * (lane >> 2) + k;
    dst[128 * h + 8 * (m >> 1) + 2 * (lane & 3) + (m & 1)] += v[0];
  }
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Actor head of one row, spread over the 4 lanes of a quad (zz: this lane's 4 logits incl. bias, columns col[k]):
// softmax statistics with ONE exponential per logit (e_j = exp(z_j - zmax), p_j = e_j / sum(e), log p_j = (z_j - zmax) -
// log(sum(e))), the clipped-surrogate loss and d(loss)/d(logits) incl. the entropy bonus.  Fast intrinsics: this path
// carries bf16-level error anyway.  Loss and entropy come out identical in the 4 lanes.
__device__ __forceinline__ void actor_head_quad(float (&zz)[4], const int (&col)[4], int A, int a, float logp_old, float adv,
                                                float clip_eps, float ent_coef, float inv_m, float (&dz)[4], float& loss, float& ent_out) {
  float zmax = -INFINITY;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (col[k] < A) zmax = fmaxf(zmax, zz[k]);
  zmax = quad_max(zmax);
  float ex[4], se = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    zz[k] -= zmax;
    ex[k] = col[k] < A ? __expf(zz[k]) : 0.f;
    se += ex[k];
  }
  se = quad_sum(se);
  const float lse = __logf(se), inv_se = rcp_rn_callfree(se);  // se in [1, 16]
  float ent = 0.f, logp_a = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (col[k] < A) {
      const float lp = zz[k] - lse;
      ent -= ex[k] * inv_se * lp;
      if (col[k] == a) logp_a = lp;
    }
  ent = quad_sum(ent);
  logp_a = quad_sum(logp_a);
  const float ratio = __expf(logp_a - logp_old);
  const float l1 = ratio * adv;
  const float l2 = fminf(fmaxf(ratio, 1.0f - clip_eps), 1.0f + clip_eps) * adv;
  const bool in_band = (ratio >= 1.0f - clip_eps) && (ratio <= 1.0f + clip_eps);
  const float dlogp = ((l1 < l2) || in_band) ? -adv * ratio * inv_m : 0.f;
  const float ce = ent_coef * inv_m;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float lp = zz[k] - lse, pr = ex[k] * inv_se;
    dz[k] = col[k] < A ? dlogp * ((col[k] == a ? 1.f : 0.f) - pr) + ce * pr * (lp + ent) : 0.f;
  }
  loss = -fminf(l1, l2);
  ent_out = ent;
}

__global__ void __launch_bounds__(kFbThreads, 1)
    tc_ppo_fwd_bwd_kernel(const __grid_constant__ CUtensorMap tmW0a, const __grid_constant__ CUtensorMap tmW1a,
                          const __grid_constant__ CUtensorMap tmW0c, const __grid_constant__ CUtensorMap tmW1c,
                          const FbParams p) {
  extern __shared__ uint8_t smem_raw[];
  // align by OFFSET (not through an integer cast) so that the compiler keeps the shared address space: LDS/STS, not generic LD/ST
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  float* s_b0 = reinterpret_cast<float*>(smem + kOffBias);
  float* s_b1 = s_b0 + 256;
  float* s_b2 = s_b1 + 256;
  float* s_db = reinterpret_cast<float*>(smem + kOffDb);  // [8][528]: one slice per warp -> no atomics, fixed order
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + kOffBar);

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, warp = threadIdx.x >> 5, wq = warp & 3, lane = threadIdx.x & 31;
  const int q4 = lane & 3;
  const int which = (int)blockIdx.x < p.n_cta[0] ? 0 : 1;
  const FbNet& net = p.net[which];
  const int cta_in_net = which == 0 ? (int)blockIdx.x : (int)blockIdx.x - p.n_cta[0];
  const int n_wg = 2 * p.n_cta[which], g = 2 * cta_in_net + wg;
  const int num_tiles = p.mb / kWTile;
  const int my_tiles = g < num_tiles ? (num_tiles - g + n_wg - 1) / n_wg : 0;
  const CUtensorMap* tmW0 = which == 0 ? &tmW0a : &tmW0c;
  const CUtensorMap* tmW1 = which == 0 ? &tmW1a : &tmW1c;

  const uint32_t xs0 = sbase + kOffX + wg * 2 * 8192;  // this warpgroup's X stages
  float* li0 = reinterpret_cast<float*>(smem + kOffLoss + wg * 2 * kLossStageBytes);  // and its loss-input stages
  const int dchunks = p.D >> 3;  // 16-byte chunks per observation row
  // Starts the gather of a tile into stage s as one cp.async group: two threads per row, 4 chunks of 16 bytes each (zeros past
  // D), and the row's loss inputs, stage layout [3][64]: action | logp_old | adv (actor), - | v_old | tgt (critic).
  auto gather_tile = [&](int tile, int s) {
    const int r = t >> 1, hf = t & 1;
    const int64_t mrow = (int64_t)tile * kWTile + r;
    const int64_t src = p.idx ? (int64_t)p.idx[mrow] : p.row0 + mrow;
    const __nv_bfloat16* row = p.obs + src * p.D;
    const uint32_t xd = xs0 + s * 8192 + r * 128;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int c = hf * 4 + cc;
      cp_async16(xd + ((c ^ (r & 7)) << 4), c < dchunks ? row + c * 8 : row, c < dchunks ? 16u : 0u);  // Swizzle<3,4,3>
    }
    const uint32_t ld = smem_u32(li0 + s * 192 + r);
    if (net.is_actor) {
      if (hf == 0) cp_async4(ld, p.action + src), cp_async4(ld + 256, p.logp_old + src);
      else cp_async4(ld + 512, p.adv + src);
    } else {
      if (hf == 0) cp_async4(ld + 256, p.v_old + src);
      else cp_async4(ld + 512, p.tgt + src);
    }
    cp_async_commit();
  };

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    fence_barrier_init();
    tma_prefetch_desc(tmW0);
    tma_prefetch_desc(tmW1);
  }
  griddep_launch();  // K3b cannot co-reside with this CTA anyway; lets its launch be queued early
  for (int i = threadIdx.x; i < 8 * 528; i += kFbThreads) s_db[i] = 0.f;
  griddep_wait();  // everything above overlapped the previous optimiser kernel; the weights below are its output
  if (my_tiles > 0) gather_tile(g, 0);  // the permutation and the rollout data are written earlier in the chain too
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(w_full, 32768 + 131072);
    const uint64_t pol_keep = l2_evict_last();  // the bf16 weights (K4's output) stay L2-resident for all CTAs and the next step
    for (int j = 0; j < 4; ++j) tma_load_2d_hint(smem + kImgW0 + j * 8192, tmW0, w_full, j * 64, 0, pol_keep);
    for (int j = 0; j < 4; ++j) tma_load_2d_hint(smem + kImgW1 + j * 32768, tmW1, w_full, j * 64, 0, pol_keep);
  }
  stage_w2_bias(smem, net.w2, net.b0, net.b1, net.b2, net.A, s_b0, s_b1, s_b2);
  fence_async_proxy();
  __syncthreads();

  float m_acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // actor_loss, entropy, value_loss, adv, pred value, target
  float* dbw = s_db + warp * 528;
  const float inv_m = p.inv_m;
  float adv_mean = 0.f, adv_rstd = 1.f;
  if (p.adv_stats) adv_mean = p.adv_stats[0], adv_rstd = p.adv_stats[1];
  mbar_wait(w_full, 0, 2);

  for (int it = 0; it < my_tiles; ++it) {
    const int tile = g + it * n_wg, s = it & 1;
    const uint32_t xs = xs0 + s * 8192;
    const float* li = li0 + s * 192;
    cp_async_wait_all();
    fence_async_proxy();  // this thread's cp.async writes (generic proxy) -> the wgmma reads of X (async proxy)
    wg_sync(1 + wg);      // the whole tile has landed, and every warp is done with the previous tile and so with stage s ^ 1
    const int64_t row0 = (int64_t)tile * kWTile + wq * 16 + (lane >> 2);  // rows row0 and row0 + 8 of this thread
    float acc[64], acc1[64];
    uint32_t a1[64], a2[64];
    wg_zero(acc);
    wg_zero(acc1);
    // ---------------- G0 / E0, G1 / E1: hidden layers ----------------
    // G0 issues both halves before it waits for the first, so that half 1's MMAs run during half 0's epilogue and the gather
    // below.  (The later 256-wide GEMMs run one half at a time: a second accumulator does not fit next to h1 and h2 there.)
    gemm_x_w0_issue(acc, xs, sbase, 0);
    gemm_x_w0_issue(acc1, xs, sbase, 1);
    if (which == 0) {  // the gathered rows for K3b's dW0, copied from the X stage
      const int r = t >> 1, hf = t & 1;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = hf * 4 + cc;
        const uint4 v = *reinterpret_cast<const uint4*>(smem + (xs - sbase) + r * 128 + ((c ^ (r & 7)) << 4));
        st_hint(reinterpret_cast<uint4*>(tiled_ptr(p.xg, (int64_t)tile * kWTile + r, 8 * c, 8)), v, l2_evict_first());
      }
    }
    if (it + 1 < my_tiles) gather_tile(tile + n_wg, s ^ 1);
    wg_wait<1>();
    wg_fence_acc(acc);
    epi_bias_relu(acc, s_b0, 0, a1, lane);
    wg_wait_all(acc1);
    epi_bias_relu(acc1, s_b0, 1, a1, lane);
    // G1's MMAs read acc although its first k-step does not accumulate: zeroing it here, not before G1, would keep half 0's
    // values live next to acc1 and a1 through E0 (ptxas then serialises every wgmma of the kernel, C7512)
    wg_zero(acc);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_a_w1(acc, a1, sbase, h);
      epi_bias_relu(acc, s_b1, h, a2, lane);
      store_act(net.h2, &a2[32 * h], h, row0, lane);
    }
    // ---------------- G2 / E2: head + loss + d(head) ----------------
    float z[8];
    wg_zero(z);
    gemm_a_w2(z, a2, sbase);
    float dz[8];  // accumulator layout: dz[i] = row0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 q4 + (i & 1)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int ix[4] = {2 * rr, 2 * rr + 1, 4 + 2 * rr, 5 + 2 * rr};
      const int col[4] = {2 * q4, 2 * q4 + 1, 8 + 2 * q4, 9 + 2 * q4};
      const int rl = wq * 16 + (lane >> 2) + 8 * rr;  // the row's index in the tile's loss-input stage
      if (net.is_actor) {
        float zz[4], d4[4], loss, ent;
#pragma unroll
        for (int k = 0; k < 4; ++k) zz[k] = z[ix[k]] + s_b2[col[k]];
        const float adv = (li[128 + rl] - adv_mean) * adv_rstd;
        actor_head_quad(zz, col, net.A, __float_as_int(li[rl]), li[64 + rl], adv, p.clip_eps, p.ent_coef, inv_m, d4, loss, ent);
#pragma unroll
        for (int k = 0; k < 4; ++k) dz[ix[k]] = d4[k];
        if (q4 == 0) m_acc[0] += loss, m_acc[1] += ent, m_acc[3] += adv;
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) dz[ix[k]] = 0.f;
        if (q4 == 0) {  // the value is column 0
          const float v = z[2 * rr] + s_b2[0], vo = li[64 + rl], tg = li[128 + rl];
          const float diff = v - vo;
          const float vclip = vo + fminf(fmaxf(diff, -p.clip_eps), p.clip_eps);
          const float e1 = v - tg, e2 = vclip - tg, q1 = e1 * e1, q2 = e2 * e2;
          const float g2 = (fabsf(diff) < p.clip_eps) ? e2 : 0.f;
          const float dv = q1 > q2 ? e1 : (q1 < q2 ? g2 : 0.5f * (e1 + g2));
          dz[2 * rr] = p.vf_coef * dv * inv_m;
          m_acc[2] += 0.5f * fmaxf(q1, q2), m_acc[4] += v, m_acc[5] += tg;
        }
      }
    }
    uint32_t dzp[4];  // dz as the A operand of G3 (K = 16)
#pragma unroll
    for (int k = 0; k < 4; ++k) dzp[k] = pack_bf16(dz[2 * k], dz[2 * k + 1]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      st_hint(reinterpret_cast<uint32_t*>(tiled_ptr(net.dz, row0 + 8 * (k & 1), 8 * (k >> 1) + 2 * q4, 2)), dzp[k], l2_evict_first());
    {  // head bias gradient: column sums of dz over the tile rows of this warp
      float cs[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) cs[k] = dz[(k >> 1) * 4 + (k & 1)] + dz[(k >> 1) * 4 + 2 + (k & 1)];
#pragma unroll
      for (int s = 4; s <= 16; s <<= 1)
#pragma unroll
        for (int k = 0; k < 4; ++k) cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], s);
      if (lane < 4)
#pragma unroll
        for (int k = 0; k < 4; ++k) dbw[512 + 8 * (k >> 1) + 2 * lane + (k & 1)] += cs[k];
    }
    // ---------------- G3 / E3: dh2 = (dz W2^T) * (h2 > 0), replaces h2 as the A operand of G4 ----------------
    uint32_t mw[4] = {0u, 0u, 0u, 0u};  // h2 > 0 (fragment order): K3b rebuilds dh2 for dW1 from dz and this mask
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_dz_w2t(acc, dzp, sbase, h);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        // h is post-relu (>= 0): positive <=> bf16 bit pattern non-zero (and not -0)
        const uint32_t hm = a2[32 * h + i];
        const bool p0 = (hm & 0x7FFFu) != 0u, p1 = (hm & 0x7FFF0000u) != 0u;
        mw[mask_word(h, i)] |= ((uint32_t)p0 << mask_bit(i, 0)) | ((uint32_t)p1 << mask_bit(i, 1));
        acc[2 * i] = p0 ? acc[2 * i] : 0.f;
        acc[2 * i + 1] = p1 ? acc[2 * i + 1] : 0.f;
        a2[32 * h + i] = pack_bf16(acc[2 * i], acc[2 * i + 1]);
      }
      colsum_half(acc, dbw + 256, h, lane);  // db1
    }
    st_hint(net.mask + (int64_t)tile * 128 + t, make_uint4(mw[0], mw[1], mw[2], mw[3]), l2_evict_first());
    // ---------------- G4 / E4: dh1 = (dh2 W1^T) * (h1 > 0) ----------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_a_w1t(acc, a2, sbase, h);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const uint32_t hm = a1[32 * h + i];
        const uint32_t pk = pack_bf16((hm & 0x7FFFu) != 0u ? acc[2 * i] : 0.f, (hm & 0x7FFF0000u) != 0u ? acc[2 * i + 1] : 0.f);
        a1[32 * h + i] = pk;
        const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&pk);
        acc[2 * i] = __bfloat162float(v.x), acc[2 * i + 1] = __bfloat162float(v.y);  // db0 sums the bf16 dh1 that K3b's dW0 uses
      }
      store_act(net.dh1, &a1[32 * h], h, row0, lane);
      colsum_half(acc, dbw, h, lane);  // db0
    }
  }
  // ---- teardown: bias-gradient and metric partials of this CTA ----
  __syncthreads();
  const uint64_t pol_keep = l2_evict_last();  // read by the reduce kernel after K3b has streamed the activations through L2
  for (int i = threadIdx.x; i < 528; i += kFbThreads) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) acc += s_db[w * 528 + i];
    st_hint(&net.db_part[(int64_t)cta_in_net * 528 + i], acc, pol_keep);
  }
  {
    __shared__ float s_mw[kFbThreads / 32][6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float w = warp_sum(m_acc[k]);
      if (lane == 0) s_mw[warp][k] = w;
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      float acc = 0.f;
      if (threadIdx.x < 6)
        for (int w = 0; w < kFbThreads / 32; ++w) acc += s_mw[w][threadIdx.x];
      st_hint(&p.metric_part[(int64_t)blockIdx.x * 8 + threadIdx.x], acc, pol_keep);
    }
  }
}

// =============================== K3b: dW = A^T * B ===============================================
constexpr int kDwThreads = 384;  // warpgroups 0, 1: MMA consumers; warpgroup 2: TMA producer (warp 8) / dW1 operand rebuild
constexpr int kDwStages = 4;
constexpr uint32_t kDwStageBytes = 49152;  // A [64 x 256] 32 KB + B [64 x <=128] 16 KB
constexpr uint32_t kDwOffBar = kDwStages * kDwStageBytes;
constexpr uint32_t kDwSmemBytes = kDwOffBar + 128 + 1024;
constexpr int kMaxJobs = 8;

// dW1 role shared-memory map (inside the ring area of the other roles): a 4-stage ring of the chunk inputs (x 8 KB, dz 2 KB,
// mask 2 KB), two buffers of the rebuilt operands (h1 half [16 colgroups][64 rows][8] 16 KB, dh2 [32][64][8] 32 KB, the tiled
// core-matrix layout that K3b's MMAs read), the W0 column half (2 SW128 boxes), the W2 image, b0 of the half.
constexpr uint32_t kW1StageBytes = 12288;
constexpr uint32_t kW1OffImg = kDwStages * kW1StageBytes;
constexpr uint32_t kW1ImgBytes = 49152;
constexpr uint32_t kW1OffW0 = kW1OffImg + 2 * kW1ImgBytes;
constexpr uint32_t kW1OffW2 = kW1OffW0 + 16384;
constexpr uint32_t kW1OffB0 = kW1OffW2 + 8192;
static_assert(kW1OffB0 + 128 * 4 <= kDwOffBar, "dW1 role smem exceeds the ring area");

// One weight-gradient GEMM over the rows this CTA is given.
//   rebuild == 0: part = A^T * B[:, 8 b_cg0 .. 8 b_cg0 + N), A and B streamed from K3a's tiled activations.
//   rebuild == 1: rows [m0, m0 + 128) of dW1 = h1^T dh2 (N = 256): h1[:, m0 ..] = relu(x W0 + b0) and dh2 = (dz W2^T) * mask are
//                 rebuilt per 64-row chunk from x (map a), dz (map b) and the h2 sign mask with K3a's own instruction sequences,
//                 so the operands are bit-identical to what K3a computed.
struct DwJob {
  float* part;     // [n_cta][256 x N] fp32 partials; rebuild: the two [n_cta][256 x 128] arrays of output halves, back to back
  int N;           // 16, 64 or 128 (rebuild: 256)
  int map;         // index of the (A, B) tensor-map pair in DwMaps
  int b_cg;        // column groups of the whole B matrix
  int b_cg0;       // first column group of B taken by this job
  int cta_begin;   // first CTA of this job
  int n_cta;
  int num_chunks;  // mb / 64
  int rebuild;
  int m0;          // rebuild: first hidden unit (0 or 128)
  int net;         // rebuild: index of the network's W0 map in DwMaps
  int A;           // rebuild: head width
  const uint4* mask;         // rebuild: K3a's h2 sign mask
  const __nv_bfloat16* w2;   // rebuild: [256 x A] bf16
  const float* b0;           // rebuild: [256] fp32 (as K3a reads it)
};
struct DwParams {
  DwJob job[kMaxJobs];
  int n_jobs;
};
struct DwMaps {
  CUtensorMap a[kMaxJobs];  // tiled [mb x 256]: 2D u64 view {256 per (tile, colgroup), tiles*32}, box {128, 32}
  CUtensorMap b[kMaxJobs];  // tiled [mb x 8 b_cg]: box {128, N/8}
  CUtensorMap w0[2];        // per network: W0 bf16 [D x 256], SW128 boxes [64 x 64] (as K3a)
};

template <int N>
__device__ __forceinline__ void dw_consume(uint8_t* smem, uint64_t* full, uint64_t* empty, const DwJob& job, int cta, int my_chunks) {
  const uint32_t sbase = smem_u32(smem);
  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  float acc[2][N / 2];
  wg_zero(acc[0]);
  wg_zero(acc[1]);
  for (int k = 0; k < my_chunks; ++k) {
    const int s = k % kDwStages;
    mbar_wait(&full[s], (k / kDwStages) & 1, 21);
    const uint32_t a0 = sbase + s * kDwStageBytes, b0 = a0 + 32768;
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {  // 16 rows (K) per step = two core-matrix row groups of 128 B
      const uint64_t db = wg_desc(b0 + ks * 256, 128, 1024, WG_INTERLEAVE);
#pragma unroll
      for (int m = 0; m < 2; ++m) {  // M blocks of 64 hidden units = 8 column groups of A
        const uint64_t da = wg_desc(a0 + (2 * wg + m) * 8192 + ks * 256, 128, 1024, WG_INTERLEAVE);
        const uint32_t accum = (k > 0 || ks > 0) ? 1u : 0u;
        if constexpr (N == 64) wg_mma_ss_n64<1, 1>(acc[m], da, db, accum);
        else wg_mma_ss_n16<1, 1>(acc[m], da, db, accum);
      }
    }
    wg_commit();
    // chunk k stays in flight while this warp waits for chunk k + 1: only chunk k - 1's stage is known to be read
    wg_wait<1>();
    __syncwarp();
    if (k > 0 && lane == 0) mbar_arrive(&empty[(k - 1) % kDwStages]);
  }
  wg_wait<0>();
  wg_fence_acc(acc[0]);
  wg_fence_acc(acc[1]);
  // partial layout [N/4][256 rows][4]: element (m, c) at ((c/4) * 256 + m) * 4 + c % 4
  const uint64_t pol_keep = l2_evict_last();  // the reduce kernel reads these next: keep them in L2 under the activation stream
  float* out = job.part + (int64_t)cta * 256 * N;
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int r = (2 * wg + m) * 64 + wq * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int c = 8 * j + 2 * (lane & 3);
        float* dst = out + ((int64_t)(c >> 2) * 256 + r + 8 * rr) * 4 + (c & 3);
        st_hint(reinterpret_cast<uint2*>(dst), make_uint2(__float_as_uint(acc[m][4 * j + 2 * rr]), __float_as_uint(acc[m][4 * j + 2 * rr + 1])), pol_keep);
      }
  }
}

// dW1 consumers: warpgroup w owns hidden units m0 + 64 w .. + 63 and all 256 output columns (two N=128 accumulators).  Per chunk
// the products run in the order of the column-split kernel this replaces (16-row steps ks, then chunks), and the partials land
// in its layout ([output half][n_cta][N/4 = 32][256 rows][4]), so the reduce and its summation order are unchanged.
__device__ __forceinline__ void dw1_consume(uint8_t* smem, uint64_t* img_full, uint64_t* img_empty, const DwJob& job, int cta,
                                            int my_chunks) {
  const uint32_t sbase = smem_u32(smem);
  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  float acc[2][64];
  wg_zero(acc[0]);
  wg_zero(acc[1]);
  for (int k = 0; k < my_chunks; ++k) {
    const int b = k & 1;
    mbar_wait(&img_full[b], (k >> 1) & 1, 23);
    const uint32_t h1 = sbase + kW1OffImg + b * kW1ImgBytes, dh2 = h1 + 16384;
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t da = wg_desc(h1 + wg * 8192 + ks * 256, 128, 1024, WG_INTERLEAVE);
#pragma unroll
      for (int nh = 0; nh < 2; ++nh)
        wg_mma_ss_n128<1, 1>(acc[nh], da, wg_desc(dh2 + nh * 16384 + ks * 256, 128, 1024, WG_INTERLEAVE), (k > 0 || ks > 0) ? 1u : 0u);
    }
    wg_commit();
    // as dw_consume: release chunk k - 1's image once its MMAs are done, with chunk k still in flight.  The rebuild of chunk
    // k + 1 waits for exactly that release (the image it overwrites is chunk k - 1's).
    wg_wait<1>();
    __syncwarp();
    if (k > 0 && lane == 0) mbar_arrive(&img_empty[b ^ 1]);
  }
  wg_wait<0>();
  wg_fence_acc(acc[0]);
  wg_fence_acc(acc[1]);
  const uint64_t pol_keep = l2_evict_last();
  const int r = job.m0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int nh = 0; nh < 2; ++nh) {
    float* out = job.part + (int64_t)(nh * job.n_cta + cta) * 256 * 128;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int c = 8 * j + 2 * (lane & 3);
        float* dst = out + ((int64_t)(c >> 2) * 256 + r + 8 * rr) * 4 + (c & 3);
        st_hint(reinterpret_cast<uint2*>(dst), make_uint2(__float_as_uint(acc[nh][4 * j + 2 * rr]), __float_as_uint(acc[nh][4 * j + 2 * rr + 1])), pol_keep);
      }
  }
}

// dW1 operand rebuild (warpgroup 2): thread t plays K3a's thread t of the warpgroup that ran the chunk's 64-row tile.  Chunk k's
// operands go to image buffer k % 2 while the consumers multiply chunk k - 1 out of the other buffer.  Thread 0 also keeps the
// input ring full.  The MMAs of the rebuild and of the consumers share the SM's tensor cores in issue order: a rebuild GEMM issued
// after the consumers have queued chunk k's 16 MMAs waits for all of them.  So chunk k + 1's first GEMM (x W0, the largest) is
// issued before chunk k's image is signalled, and its epilogue runs while the consumers' MMAs do.
__device__ __forceinline__ void dw1_rebuild(uint8_t* smem, uint64_t* full, uint64_t* img_full, uint64_t* img_empty, uint64_t* w_full,
                                            const CUtensorMap* map_x, const CUtensorMap* map_dz, const DwJob& job, int cta,
                                            int my_chunks, uint64_t pol_stream) {
  const uint32_t sbase = smem_u32(smem);
  const int t = threadIdx.x & 127, wq = t >> 5, lane = t & 31, q4 = lane & 3;
  const float* s_b0 = reinterpret_cast<const float*>(smem + kW1OffB0);
  auto load_chunk = [&](int it) {
    // newest rows first, as the streamed jobs (K3a wrote the last tiles most recently)
    const int chunk = job.num_chunks - 1 - (cta + it * job.n_cta);
    const int tile = chunk >> 1, r0 = (chunk & 1) * 64, s = it % kDwStages;
    uint8_t* st = smem + s * kW1StageBytes;
    mbar_arrive_expect_tx(&full[s], kW1StageBytes);
    tma_load_2d_hint(st, map_x, &full[s], r0 * 2, tile * 8, pol_stream);
    tma_load_2d_hint(st + 8192, map_dz, &full[s], r0 * 2, tile * 2, pol_stream);
    bulk_load_hint(st + 10240, job.mask + (int64_t)chunk * 128, 2048, &full[s], pol_stream);
  };
  if (t == 0)
    for (int it = 0; it < kDwStages && it < my_chunks; ++it) load_chunk(it);
  mbar_wait(w_full, 0, 24);
  for (int it = 0; it < my_chunks; ++it) {
    const int s = it % kDwStages, b = it & 1;
    uint8_t* st = smem + s * kW1StageBytes;
    uint8_t* h1img = smem + kW1OffImg + b * kW1ImgBytes;
    uint8_t* dh2img = h1img + 16384;
    const int r = wq * 16 + (lane >> 2);  // rows r and r + 8 of the chunk
    float acc[64];
    uint32_t a[64];
    // h1[:, m0 ..] = relu(x W0[:, m0 ..] + b0[m0 ..]): K3a's G0 / E0 with x K-major from the tiled layout ([colgroup][row][8])
    mbar_wait(&full[s], (it / kDwStages) & 1, 25);
    wg_zero(acc);  // the first k-step does not accumulate, but the MMA still reads acc
    gemm_x_w0_at_issue(acc, wg_desc(smem_u32(st), 1024, 128, WG_INTERLEAVE), 2048, sbase + kW1OffW0, 0);
    if (it > 0) {  // chunk it - 1's image, signalled behind chunk it's first GEMM
      mbar_arrive(&img_full[b ^ 1]);
      wg_sync(3);  // every thread of this warpgroup is done with ring stage s - 1
      if (t == 0 && it - 1 + kDwStages < my_chunks) load_chunk(it - 1 + kDwStages);
    }
    wg_wait_all(acc);
    epi_bias_relu(acc, s_b0, 0, a, lane);
    if (it >= 2) mbar_wait(&img_empty[b], ((it >> 1) - 1) & 1, 26);
#pragma unroll
    for (int i = 0; i < 32; ++i)
      *reinterpret_cast<uint32_t*>(h1img + (i >> 1) * 1024 + (r + 8 * (i & 1)) * 16 + 4 * q4) = a[i];
    // dh2 = (dz W2^T) * (h2 > 0): K3a's G3 / E3 with dz in the A-fragment layout and the mask words this thread wrote there
    uint32_t dzp[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) dzp[k] = *reinterpret_cast<const uint32_t*>(st + 8192 + (k >> 1) * 1024 + (r + 8 * (k & 1)) * 16 + 4 * q4);
    const uint4 m4 = *reinterpret_cast<const uint4*>(st + 10240 + 16 * t);
    const uint32_t mw[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gemm_dz_w2t_at(acc, dzp, sbase + kW1OffW2, h);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const uint32_t w = mw[mask_word(h, i)];
        acc[2 * i] = (w >> mask_bit(i, 0)) & 1u ? acc[2 * i] : 0.f;
        acc[2 * i + 1] = (w >> mask_bit(i, 1)) & 1u ? acc[2 * i + 1] : 0.f;
        *reinterpret_cast<uint32_t*>(dh2img + (16 * h + (i >> 1)) * 1024 + (r + 8 * (i & 1)) * 16 + 4 * q4) = pack_bf16(acc[2 * i], acc[2 * i + 1]);
      }
    }
    fence_async_proxy();  // generic-proxy image stores -> visible to the consumers' wgmma
  }
  if (my_chunks > 0) mbar_arrive(&img_full[(my_chunks - 1) & 1]);
}

__global__ void __launch_bounds__(kDwThreads, 1) tc_dw_kernel(const __grid_constant__ DwMaps maps, const DwParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kDwOffBar);
  uint64_t* full = bars;                 // [kDwStages]
  uint64_t* empty = bars + kDwStages;    // [kDwStages]
  uint64_t* img_full = bars + 2 * kDwStages;   // [2] dW1 role
  uint64_t* img_empty = img_full + 2;          // [2]
  uint64_t* w_full = img_empty + 2;
  const int warp = threadIdx.x >> 5;
  const long long prof_t0 = clock64();

  int j = 0;
  while (j + 1 < p.n_jobs && (int)blockIdx.x >= p.job[j + 1].cta_begin) ++j;
  const DwJob& job = p.job[j];
  const int cta = (int)blockIdx.x - job.cta_begin;
  const int my_chunks = cta < job.num_chunks ? (job.num_chunks - cta + job.n_cta - 1) / job.n_cta : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kDwStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&img_full[b], 128);  // every rebuild thread, after its own proxy fence
      mbar_init(&img_empty[b], 8);
    }
    mbar_init(w_full, 1);
    fence_barrier_init();
    tma_prefetch_desc(&maps.a[job.map]);
    tma_prefetch_desc(&maps.b[job.map]);
  }
  griddep_launch();
  __syncthreads();
  griddep_wait();  // the activations are K3a's output; the partials written below were read by the previous reduce
  if (threadIdx.x == 0 && g_prof_buf != nullptr) {
    long long* prof = g_prof_buf + (int64_t)blockIdx.x * 8;
    prof[2] = clock64() - prof_t0, prof[3] = globaltimer_ns();
  }

  const uint64_t pol_stream = l2_evict_first();  // every activation tile is read exactly once
  if (job.rebuild) {
    // weights of the job's network (after griddep_wait: the previous optimiser step wrote them), as K3a stages them
    if (threadIdx.x == 256) {
      mbar_arrive_expect_tx(w_full, 16384);
      const uint64_t pol_keep = l2_evict_last();
      for (int jb = 0; jb < 2; ++jb) tma_load_2d_hint(smem + kW1OffW0 + jb * 8192, &maps.w0[job.net], w_full, job.m0 + 64 * jb, 0, pol_keep);
    }
    stage_w2(smem + kW1OffW2, job.w2, job.A);
    if (threadIdx.x < 128) reinterpret_cast<float*>(smem + kW1OffB0)[threadIdx.x] = job.b0[job.m0 + threadIdx.x];
    fence_async_proxy();
    __syncthreads();
  }
  // 384 threads x 168 registers: the consumers' 128 accumulators + addressing need more than 168, the producer / rebuild
  // warpgroup fewer (2 x 128 x 200 + 128 x 104 = 384 x 168)
  if (warp >= 8) {
    setmaxnreg_dec<104>();
    if (job.rebuild) {
      dw1_rebuild(smem, full, img_full, img_empty, w_full, &maps.a[job.map], &maps.b[job.map], job, cta, my_chunks, pol_stream);
    } else if (warp == 8 && elect_one()) {
      for (int it = 0; it < my_chunks; ++it) {
        // newest rows first (K3a wrote the last tiles most recently, so they are the likeliest L2 residents)
        const int chunk = job.num_chunks - 1 - (cta + it * job.n_cta);  // 64 rows: half of a 128-row tile
        const int tile = chunk >> 1, r0 = (chunk & 1) * 64;
        const int s = it % kDwStages;
        if (it >= kDwStages) mbar_wait(&empty[s], ((it / kDwStages) & 1) ^ 1, 20);
        uint8_t* st = smem + s * kDwStageBytes;
        mbar_arrive_expect_tx(&full[s], 32768 + (uint32_t)job.N * 128);
        // one box = rows r0..r0+63 of the column groups: smem image [colgroup][row][16 B]
        tma_load_2d_hint(st, &maps.a[job.map], &full[s], r0 * 2, tile * 32, pol_stream);
        tma_load_2d_hint(st + 32768, &maps.b[job.map], &full[s], r0 * 2, tile * job.b_cg + job.b_cg0, pol_stream);
      }
    }
  } else {
    setmaxnreg_inc<200>();
    if (job.rebuild) dw1_consume(smem, img_full, img_empty, job, cta, my_chunks);
    else if (job.N == 64) dw_consume<64>(smem, full, empty, job, cta, my_chunks);
    else dw_consume<16>(smem, full, empty, job, cta, my_chunks);
  }
  __syncthreads();
  if (g_prof_buf != nullptr && threadIdx.x == 0) {
    long long* prof = g_prof_buf + (int64_t)blockIdx.x * 8;
    prof[0] = 2 + j, prof[1] = clock64() - prof_t0, prof[4] = globaltimer_ns(), prof[5] = my_chunks;
  }
}

// =============================== reduce partials -> gradient arena ================================
struct RedSeg {
  const float* part;    // partial base (source view: rows x cols with leading dimension src_ld)
  int64_t part_stride;  // floats between the partials of consecutive CTAs
  int n_part;
  int rows, cols;       // elements to take from the source view
  int src_ld;
  int transpose;        // 0: dst[r*dst_ld + c]   1: dst[c*dst_ld + r]
  int dst_ld;
  int64_t dst_off;
  int net;              // optimiser segment (0 actor, 1 critic) for the sum-of-squares side output
  int cg4;              // 1: source is a K3b partial in [cols/4][256 rows][4] order (items enumerate it linearly)
  int items;            // rows*cols/4 (vec) or rows*cols
};
struct RedParams {
  RedSeg seg[14];
  int n_seg;
  int total_items;
  const float* metric_part;  // [n_cta_total][8]
  int n_cta_total;
  float* metrics;            // [6] accumulated
  float weight;
  float inv_mb;
  int overwrite;
  double* sumsq;             // nullable: [2][gridDim] block partials of sum((weight*g)^2) per optimiser segment
  unsigned long long* sumsq_count;  // where the number of block partials per segment (= gridDim) is published
};

constexpr int kRedThreads = 352;  // x 528 blocks >= the ~173k gradient entries of the benchmark networks: one element per thread
constexpr int kRedMaxBlocks = 4 * kNumSMs;
static_assert(2 * kRedMaxBlocks <= kAdamMaxSegs * kNumSMs, "AdamScratch::partials must hold 2 segments x kRedMaxBlocks block partials");

// Fixed-order reduction of the per-CTA partials into the gradient arena.  One launch, every segment
// concurrently; 4 independent accumulators per element for load-level parallelism; the association order
// is fixed => run-to-run deterministic gradients.  Optionally leaves the per-block sum of squares of the
// reduced gradient for clip + Adam (PRENORM: it then skips its own norm pass and grid barrier).
__global__ void __launch_bounds__(kRedThreads, 4) tc_reduce_kernel(const RedParams p, float* __restrict__ grad) {
  griddep_launch();
  griddep_wait();
  const uint64_t pol_keep = l2_evict_last();  // partials and gradients: small, reused every step, latency-critical
  double sq0 = 0.0, sq1 = 0.0;
  for (int gi = blockIdx.x * blockDim.x + threadIdx.x; gi < p.total_items; gi += gridDim.x * blockDim.x) {
    int s = 0, i = gi;
    while (i >= p.seg[s].items) i -= p.seg[s].items, ++s;
    const RedSeg& g = p.seg[s];
    {
      int r, c;
      const float* src;
      if (g.cg4) {  // linear walk over the partial: coalesced reads; (r, c) = (row, column) of the K3b output
        r = (i & 1023) >> 2, c = ((i >> 10) << 2) | (i & 3);
        if (c >= g.cols) continue;
        src = g.part + i;
      } else {
        r = i / g.cols, c = i % g.cols;
        src = g.part + (int64_t)r * g.src_ld + c;
      }
      // latency-bound (the partials were evicted by the activation traffic: every round trip goes to DRAM): 8 independent
      // loads in flight per thread and round trip, 4 accumulation chains in a fixed order.  (16 per round trip with
      // predicated tails measured 3x SLOWER: the batch no longer fits the scoreboard/registers the compiler allots.)
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      const int64_t S = g.part_stride;
      int k = 0;
      for (; k + 8 <= g.n_part; k += 8) {
        const float* q = src + (int64_t)k * S;
        const float v0 = ld_hint(q, pol_keep), v1 = ld_hint(q + S, pol_keep), v2 = ld_hint(q + 2 * S, pol_keep), v3 = ld_hint(q + 3 * S, pol_keep);
        const float v4 = ld_hint(q + 4 * S, pol_keep), v5 = ld_hint(q + 5 * S, pol_keep), v6 = ld_hint(q + 6 * S, pol_keep), v7 = ld_hint(q + 7 * S, pol_keep);
        a0 += v0, a1 += v1, a2 += v2, a3 += v3;
        a0 += v4, a1 += v5, a2 += v6, a3 += v7;
      }
      if (k < g.n_part) {  // up to 7 left: one more batch of independent (predicated) loads
        const float* q = src + (int64_t)k * S;
        const int n = g.n_part - k;
        const float v0 = ld_hint(q, pol_keep), v1 = n > 1 ? ld_hint(q + S, pol_keep) : 0.f, v2 = n > 2 ? ld_hint(q + 2 * S, pol_keep) : 0.f;
        const float v3 = n > 3 ? ld_hint(q + 3 * S, pol_keep) : 0.f, v4 = n > 4 ? ld_hint(q + 4 * S, pol_keep) : 0.f, v5 = n > 5 ? ld_hint(q + 5 * S, pol_keep) : 0.f;
        const float v6 = n > 6 ? ld_hint(q + 6 * S, pol_keep) : 0.f;
        a0 += v0, a1 += v1, a2 += v2, a3 += v3;
        a0 += v4, a1 += v5, a2 += v6;
      }
      float* dst = grad + g.dst_off + (g.transpose ? (int64_t)c * g.dst_ld + r : (int64_t)r * g.dst_ld + c);
      float o = p.weight * ((a0 + a1) + (a2 + a3));
      if (!p.overwrite) o += *dst;
      st_hint(dst, o, pol_keep);
      if (g.net) sq1 += (double)o * o;
      else sq0 += (double)o * o;
    }
  }
  if (p.sumsq != nullptr) {  // only meaningful with overwrite (then o is the whole gradient)
    __shared__ double sred[32];
#pragma unroll
    for (int n = 0; n < 2; ++n) {
      const double b = block_sum<double>(n == 0 ? sq0 : sq1, sred);
      if (threadIdx.x == 0) p.sumsq[(int64_t)n * gridDim.x + blockIdx.x] = b;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *p.sumsq_count = gridDim.x;
  }
  if (blockIdx.x == 0 && threadIdx.x < 6) {
    float acc = 0.f;
    for (int k = 0; k < p.n_cta_total; ++k) acc += p.metric_part[(int64_t)k * 8 + threadIdx.x];
    p.metrics[threadIdx.x] += p.weight * acc * p.inv_mb;
  }
}

// =============================== host side =======================================================
inline size_t al(size_t x) { return (x + 255) / 256 * 256; }

struct TcWs {
  __nv_bfloat16 *h2[2], *dh1[2], *dz[2], *xg;
  uint4* mask[2];
  float *part_w1[2][2], *part_w2[2], *part_w0[2], *db_part[2], *metric_part;
  size_t bytes;
};

constexpr int kCtaPerNet = kNumSMs / 2;              // 66
// Launch plan, per network (x 2 networks = 132 CTAs): K3a on 66 CTAs, then K3b with 19 + 19 / 13 / 15 split-K CTAs for
// the two row halves of dW1 / dW2 / dW0 (the fastest split of the sweeps in DESIGN.md).  Each dW1 CTA sums the same rows in
// the same order as the column-split jobs that first set this plan, so the plan keeps the gradients' rounding; the split
// decides which rows each partial holds.
constexpr int kDwCtasW1 = 19, kDwCtasW2 = 13, kDwCtasW0 = 15;
static_assert(2 * kDwCtasW1 + kDwCtasW2 + kDwCtasW0 == kCtaPerNet, "K3b's jobs of a network must take its 66 CTAs");

TcWs carve_tc(int64_t mb, char* base) {
  TcWs w{};
  size_t o = 0;
  auto take = [&](size_t bytes) {
    char* q = base ? base + o : nullptr;
    o += al(bytes);
    return q;
  };
  for (int n = 0; n < 2; ++n) {
    w.h2[n] = (__nv_bfloat16*)take((size_t)mb * 256 * 2);
    w.dh1[n] = (__nv_bfloat16*)take((size_t)mb * 256 * 2);
    w.dz[n] = (__nv_bfloat16*)take((size_t)mb * 16 * 2);
    w.mask[n] = (uint4*)take((size_t)mb * 256 / 8);
    // the dW1 half-jobs write both output halves: [1] must follow [0] directly (the size is a multiple of the alignment)
    for (int hh = 0; hh < 2; ++hh) w.part_w1[n][hh] = (float*)take((size_t)kDwCtasW1 * 256 * 128 * 4);
    w.part_w2[n] = (float*)take((size_t)kDwCtasW2 * 256 * 16 * 4);
    w.part_w0[n] = (float*)take((size_t)kDwCtasW0 * 256 * 64 * 4);
    w.db_part[n] = (float*)take((size_t)kCtaPerNet * 528 * 4);
  }
  w.xg = (__nv_bfloat16*)take((size_t)mb * 64 * 2);
  w.metric_part = (float*)take((size_t)kNumSMs * 8 * 4);
  w.bytes = o;
  return w;
}

bool tc_ppo_shape_ok(const StxMlp* m) {
  return m->n_layers == 3 && m->sizes[1] == kH && m->sizes[2] == kH && m->sizes[0] <= 64 && m->sizes[0] % 8 == 0 &&
         m->sizes[3] >= 1 && m->sizes[3] <= 16 && m->activation == STX_ACT_RELU && !m->use_layer_norm;
}

}  // namespace tc

size_t tc_ppo_workspace_bytes(const StxMlp* a, const StxMlp* c, int64_t mb) {
  (void)a, (void)c;
  return tc::carve_tc(mb, nullptr).bytes;
}

int tc_ppo_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, int64_t mb_off, int64_t mb,
                           const StxPpoHyper* h, float grad_weight, float* grad_arena, float* metrics, void* ws_raw, size_t,
                           cudaStream_t st) {
  using namespace tc;
  STX_REQUIRE(tc_ppo_shape_ok(actor) && tc_ppo_shape_ok(critic), STX_E_SHAPE,
              "STX_PREC_BF16 PPO kernels need a relu MLP without LayerNorm, sizes [D<=64 (mult of 8), 256, 256, head<=16]");
  STX_REQUIRE(mb % 128 == 0, STX_E_SHAPE, "STX_PREC_BF16 PPO kernels need a minibatch that is a multiple of 128 rows (got %lld)", (long long)mb);
  STX_REQUIRE(actor->params_bf16 && critic->params_bf16, STX_E_ARG, "STX_PREC_BF16 needs the bf16 shadow arenas");
  const int D = actor->sizes[0];
  const StxMlp* nets[2] = {actor, critic};
  TcWs ws = carve_tc(mb, reinterpret_cast<char*>(ws_raw));
  int64_t aoff, coff, total;
  stx_ppo_arena_offsets(actor, critic, &aoff, &coff, &total);
  const int64_t noff[2] = {aoff, coff};
  const int n_fb = kCtaPerNet;  // K3a CTAs per network

  // ---- K3a parameters ----
  FbParams fp{};
  CUtensorMap tmW0[2], tmW1[2];
  for (int n = 0; n < 2; ++n) {
    const StxMlp* m = nets[n];
    const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(m->params_bf16);
    const int A = m->sizes[3];
    const int64_t off_w1 = (int64_t)D * kH + kH, off_w2 = off_w1 + (int64_t)kH * kH + kH;
    if (int rc = make_map_2d_pub(&tmW0[n], w, (uint64_t)D, kH, kH, 64, 64)) return rc;
    if (int rc = make_map_2d_pub(&tmW1[n], w + off_w1, kH, kH, kH, 256, 64)) return rc;
    FbNet& fn = fp.net[n];
    fn.w2 = w + off_w2;
    fn.b0 = m->params + (int64_t)D * kH, fn.b1 = m->params + off_w1 + (int64_t)kH * kH, fn.b2 = m->params + off_w2 + (int64_t)kH * A;
    fn.h2 = ws.h2[n], fn.dh1 = ws.dh1[n], fn.dz = ws.dz[n], fn.mask = ws.mask[n];
    fn.db_part = ws.db_part[n], fn.A = A, fn.is_actor = (n == 0);
    fp.n_cta[n] = n_fb;
  }
  fp.obs = reinterpret_cast<const __nv_bfloat16*>(b->obs);
  fp.xg = ws.xg;
  fp.idx = b->perm ? b->perm + mb_off : nullptr;
  fp.row0 = mb_off;
  fp.action = b->action, fp.logp_old = b->log_prob, fp.v_old = b->value, fp.adv = b->advantages, fp.tgt = b->targets;
  fp.adv_stats = h->standardize_advantages ? b->adv_stats : nullptr;
  fp.metric_part = ws.metric_part;
  fp.D = D, fp.mb = (int)mb, fp.inv_m = 1.0f / (float)mb, fp.clip_eps = h->clip_eps, fp.ent_coef = h->ent_coef, fp.vf_coef = h->vf_coef;

  // ---- K3b parameters ----
  DwMaps maps;
  DwParams dp{};
  maps.w0[0] = tmW0[0], maps.w0[1] = tmW0[1];
  int cta = 0, jn = 0;
  const int chunks = (int)(mb / 64);
  const uint64_t tiles = (uint64_t)(mb / 128);
  for (int n = 0; n < 2; ++n) {
    auto add_job = [&](float* part, int N, const __nv_bfloat16* a, const __nv_bfloat16* bm, int b_cg, int b_cg0, int n_cta) -> int {
      DwJob& j = dp.job[jn];
      if (int rc = make_map_tiled(&maps.a[jn], a, tiles, 32, 32)) return rc;
      if (int rc = make_map_tiled(&maps.b[jn], bm, tiles, (uint32_t)b_cg, (uint32_t)(N / 8))) return rc;
      j.part = part, j.N = N, j.map = jn, j.b_cg = b_cg, j.b_cg0 = b_cg0, j.cta_begin = cta, j.n_cta = n_cta, j.num_chunks = chunks;
      cta += n_cta, ++jn;
      return STX_OK;
    };
    // dW1 = h1^T dh2 (two row halves, operands rebuilt from xg, dz and the mask), dW2 = h2^T dz, dW0^T = dh1^T xg
    for (int hh = 0; hh < 2; ++hh) {
      DwJob& j = dp.job[jn];
      if (int rc = make_map_tiled(&maps.a[jn], ws.xg, tiles, 8, 8)) return rc;
      if (int rc = make_map_tiled(&maps.b[jn], ws.dz[n], tiles, 2, 2)) return rc;
      j.part = ws.part_w1[n][0], j.N = 256, j.map = jn, j.cta_begin = cta, j.n_cta = kDwCtasW1, j.num_chunks = chunks;
      j.rebuild = 1, j.m0 = 128 * hh, j.net = n, j.A = fp.net[n].A, j.mask = ws.mask[n], j.w2 = fp.net[n].w2, j.b0 = fp.net[n].b0;
      cta += kDwCtasW1, ++jn;
    }
    if (int rc = add_job(ws.part_w2[n], 16, ws.h2[n], ws.dz[n], 2, 0, kDwCtasW2)) return rc;
    if (int rc = add_job(ws.part_w0[n], 64, ws.dh1[n], ws.xg, 8, 0, kDwCtasW0)) return rc;
  }
  dp.n_jobs = jn;

  // ---- launches ----
  STX_CUDA_OK(opt_in_smem<tc_ppo_fwd_bwd_kernel>(kFbSmemBytes));
  STX_CUDA_OK(opt_in_smem<tc_dw_kernel>(kDwSmemBytes));
  if (int rc = use_trap_record(st)) return rc;
  STX_CUDA_OK(launch_pdl(tc_ppo_fwd_bwd_kernel, dim3(2 * n_fb), dim3(kFbThreads), kFbSmemBytes, st, tmW0[0], tmW1[0], tmW0[1],
                         tmW1[1], fp));
  STX_LAUNCH_OK();
  STX_CUDA_OK(launch_pdl(tc_dw_kernel, dim3(cta), dim3(kDwThreads), kDwSmemBytes, st, maps, dp));
  STX_LAUNCH_OK();

  // ---- reduce ----
  RedParams rp{};
  int sidx = 0;
  auto add_seg = [&](const float* part, int64_t stride, int n_part, int rows, int cols, int src_ld, int transpose, int dst_ld,
                     int64_t dst_off, int net_id, int cg4) {
    RedSeg g{};
    g.part = part, g.part_stride = stride, g.n_part = n_part, g.rows = rows, g.cols = cols, g.src_ld = src_ld;
    g.transpose = transpose, g.dst_ld = dst_ld, g.dst_off = dst_off, g.net = net_id;
    g.cg4 = cg4;
    g.items = cg4 ? ((cols + 3) / 4) * 1024 : rows * cols;  // scalar items (4x the threads of a float4 version: measurably faster)
    rp.total_items += g.items;
    rp.seg[sidx++] = g;
  };
  for (int n = 0; n < 2; ++n) {
    const int A = nets[n]->sizes[3];
    const int64_t o_w0 = noff[n], o_b0 = o_w0 + (int64_t)D * kH, o_w1 = o_b0 + kH, o_b1 = o_w1 + (int64_t)kH * kH, o_w2 = o_b1 + kH,
                  o_b2 = o_w2 + (int64_t)kH * A;
    add_seg(ws.part_w1[n][0], 256 * 128, kDwCtasW1, kH, 128, 128, 0, kH, o_w1, n, 1);         // dW1[in][out], out 0..127
    add_seg(ws.part_w1[n][1], 256 * 128, kDwCtasW1, kH, 128, 128, 0, kH, o_w1 + 128, n, 1);   // out 128..255
    add_seg(ws.part_w0[n], 256 * 64, kDwCtasW0, kH, D, 64, 1, kH, o_w0, n, 1);      // part(j, d) -> W0[d][j]
    add_seg(ws.part_w2[n], 256 * 16, kDwCtasW2, kH, A, 16, 0, A, o_w2, n, 1);       // dW2[j][a]
    add_seg(ws.db_part[n], 528, n_fb, 1, kH, 528, 0, kH, o_b0, n, 0);
    add_seg(ws.db_part[n] + 256, 528, n_fb, 1, kH, 528, 0, kH, o_b1, n, 0);
    add_seg(ws.db_part[n] + 512, 528, n_fb, 1, A, 528, 0, A, o_b2, n, 0);
  }
  rp.n_seg = sidx;
  rp.metric_part = ws.metric_part, rp.n_cta_total = 2 * n_fb, rp.metrics = metrics;
  rp.weight = grad_weight, rp.inv_mb = 1.0f / (float)mb;
  rp.overwrite = h->overwrite_grads;
  // side output for clip + Adam (PRENORM): the block partials and their count in its scratch
  AdamScratch* adam_scratch = static_cast<AdamScratch*>(h->adam_scratch);
  if (rp.overwrite && adam_scratch) rp.sumsq = adam_scratch->partials, rp.sumsq_count = &adam_scratch->n_partials;
  int red_blocks = (rp.total_items + kRedThreads - 1) / kRedThreads;  // one item per thread, blocks spread over all SMs
  if (red_blocks > kRedMaxBlocks) red_blocks = kRedMaxBlocks;
  STX_CUDA_OK(launch_pdl(tc_reduce_kernel, dim3(red_blocks), dim3(kRedThreads), 0, st, rp, grad_arena));
  STX_LAUNCH_OK();
  return STX_OK;
}

}  // namespace stx

extern "C" int stx_tc_debug_set_prof_buffer(long long* buf) {
  cudaError_t e = cudaMemcpyToSymbol(stx::tc::g_prof_buf, &buf, sizeof(buf));
  return e == cudaSuccess ? 0 : (int)e;
}
