// Thin inline-PTX wrappers for the Hopper (sm_90a) tensor-core path: mbarrier, TMA (cp.async.bulk.tensor),
// warpgroup MMA (wgmma.mma_async) and its shared-memory matrix descriptors.  Bit layouts follow the PTX ISA
// "Asynchronous Warpgroup Level Matrix Multiply-Accumulate" chapter.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "stx_common.cuh"

namespace stx {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier --------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_async_proxy() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"  // %3: suspend-time hint -> the warp
      "selp.u32 %0, 1, 0, p;\n\t}"                                        // sleeps in hardware instead of
      : "=r"(ok)                                                           // burning issue slots in a spin loop
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
// Non-suspending probe of a phase (spin-wait building block: lowest wake-up latency, burns issue slots).
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// This translation unit's pointer to the process-wide TrapRecord (stx_common.cuh); set by use_trap_record().
static __device__ TrapRecord* g_trap_record = nullptr;

// Bounded wait: a protocol bug traps instead of hanging the GPU.  The first thread to time out records where in the host-
// mapped TrapRecord, which _lib.py reports with the error.  No printf: a call would serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) {
      volatile TrapRecord* r = g_trap_record;
      if (r != nullptr && atomicCAS_system(const_cast<uint32_t*>(&r->claimed), 0u, 1u) == 0u) {
        r->block = blockIdx.x, r->thread = threadIdx.x, r->tag = (uint32_t)tag, r->parity = parity;
        __threadfence_system();
      }
      __trap();
    }
  }
}

// Host: points g_trap_record of the calling translation unit at the process-wide record, once per device.  Skipped while
// `st` is being captured (a synchronous copy is not allowed then); the pointer is device state, so the next eager call
// also covers the kernels of graphs captured before it.
static inline int use_trap_record(cudaStream_t st) {
  static unsigned long long done = 0;  // bit d: set on device d
  int dev = 0;
  STX_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 64 && ((done >> dev) & 1ull)) return STX_OK;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  STX_CUDA_OK(cudaStreamIsCapturing(st, &cs));
  if (cs != cudaStreamCaptureStatusNone) return STX_OK;
  TrapRecord* host = trap_record();
  STX_REQUIRE(host != nullptr, STX_E_UNSUPPORTED, "could not allocate the host-mapped mbarrier timeout record");
  TrapRecord* dptr = nullptr;
  STX_CUDA_OK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dptr), host, 0));
  STX_CUDA_OK(cudaMemcpyToSymbol(g_trap_record, &dptr, sizeof(dptr)));
  if (dev < 64) done |= 1ull << dev;
  return STX_OK;
}

// ---- TMA -------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tile load: coordinates (c0 = innermost element index, c1 = row)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// same with an L2 cache-policy operand (createpolicy): evict_first for operands that are read exactly once
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// 1D bulk copy global -> shared (bytes: multiple of 16, both addresses 16-byte aligned) with an L2 cache-policy operand
__device__ __forceinline__ void bulk_load_hint(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// ---- wgmma ------------------------------------------------------------------------------------
// A warpgroup (4 consecutive warps, first warp index a multiple of 4) computes D[64 x N] (+)= A[64 x 16] * B[16 x N] per
// instruction.  D lives in registers: thread t = 32 w + l holds rows 16 w + l/4 and 16 w + l/4 + 8; for every 8-column
// block j it holds d[4j + {0,1}] = (row, 8j + 2(l%4) + {0,1}) and d[4j + {2,3}] = (row + 8, same columns).  An A operand
// in registers has the same shape per 16-wide K block, so packing consecutive accumulator pairs to bf16x2 turns the
// output of one GEMM into the A operand of the next without leaving the registers.
enum : uint32_t { WG_INTERLEAVE = 0, WG_SW128 = 1 };

// Shared-memory matrix descriptor (64-bit), LBO / SBO in bytes (multiples of 16), canonical layouts of the PTX ISA:
//   K-major, no swizzle:  SBO = stride of 8-row groups (M/N), LBO = stride of 8-element core matrices along K
//   K-major, 128B swizzle: SBO = stride of 8-row groups (1024 for packed rows), LBO unused
//   MN-major, no swizzle: SBO = stride of 8-element core matrices along M/N, LBO = stride of 8-row groups along K
//   MN-major, 128B swizzle: LBO = stride of 64-element blocks along M/N, SBO = stride of 8-row groups along K
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)(layout & 3u) << 62;
  return d;
}
__device__ __forceinline__ uint64_t wg_adv(uint64_t desc, uint32_t bytes) { return desc + (uint64_t)(bytes >> 4); }  // start field, no carry

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier of the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// SS form: A and B from shared memory (TA / TB: 1 = the operand is MN-major); RS form: A from registers (4 x bf16x2).
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_ss_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_ss_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_ss_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wg_mma_rs_n16(float (&d)[8], const uint32_t* a, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, %14;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wg_mma_rs_n128(float (&d)[64], const uint32_t* a, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits), .y = hi
  return *reinterpret_cast<uint32_t*>(&v);
}

// bf16x2( relu(acc0 + b.x), relu(acc1 + b.y) ): two adds + one convert with the ReLU folded in (cvt.rn.relu.bf16x2.f32:
// negative inputs give +0, the rest rounds to nearest even); the same bits as fmaxf(acc + b, 0) followed by the rounding.
__device__ __forceinline__ uint32_t bias_relu_pack_bf16(uint32_t acc0, uint32_t acc1, float2 b) {
  const float v0 = __fadd_rn(__uint_as_float(acc0), b.x), v1 = __fadd_rn(__uint_as_float(acc1), b.y);
  uint32_t d;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(v1), "f"(v0));  // first source -> upper half
  return d;
}

// per-warpgroup register budget (every thread of the warpgroup executes it): hand registers from a producer warpgroup to the others
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- MLP[D<=64, 256, 256, A<=16] building blocks (one warpgroup, one 64-row tile) ----------------------------------
// Shared-memory images of the weights (the same images serve the forward and the backward pass):
//   W1 (256 x 256, row-major (in, out)): 4 TMA boxes [256 rows x 64 columns] of 128B-swizzled rows at kImgW1 + 32768 j
//      (j = column block): MN-major B operand of the forward, K-major B operand of the backward (W1^T).
//   W0 (D x 256): 4 boxes [64 rows x 64 columns] at kImgW0 + 8192 j (rows >= D zero-filled by TMA).
//   W2 (256 x A): element (j, n) at kImgW2 + (j/8)*256 + (n/8)*128 + (j%8)*16 + (n%8)*2, zero for n >= A (no swizzle).
//   X  (64 rows x 64 columns, bf16): 128B-swizzled rows, 16-byte chunk c of row r at r*128 + ((c ^ (r%8)) << 4).
constexpr uint32_t kImgW1 = 0, kImgW0 = 131072, kImgW2 = 163840, kImgWBytes = 172032;

// W2 image (layout above, at img) staged by all threads of the block (generic proxy; the caller fences and synchronises)
__device__ __forceinline__ void stage_w2(uint8_t* img, const __nv_bfloat16* w2, int A) {
  for (int j = threadIdx.x; j < 256; j += blockDim.x) {  // one thread per W2 row: its (<=16) loads are in flight together
    uint32_t pk[8];
    unsigned short e[16];
#pragma unroll
    for (int n = 0; n < 16; ++n) e[n] = n < A ? reinterpret_cast<const unsigned short*>(w2)[j * A + n] : (unsigned short)0;
#pragma unroll
    for (int n = 0; n < 8; ++n) pk[n] = (uint32_t)e[2 * n] | ((uint32_t)e[2 * n + 1] << 16);
    uint8_t* dst = img + (j >> 3) * 256 + (j & 7) * 16;
    *reinterpret_cast<uint4*>(dst) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    *reinterpret_cast<uint4*>(dst + 128) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
  }
}
// W2 image and biases staged by all threads of the block (generic proxy; the caller fences and synchronises)
__device__ __forceinline__ void stage_w2_bias(uint8_t* smem, const __nv_bfloat16* w2, const float* b0, const float* b1, const float* b2,
                                              int A, float* s_b0, float* s_b1, float* s_b2) {
  stage_w2(smem + kImgW2, w2, A);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_b0[i] = b0[i], s_b1[i] = b1[i];
  if (threadIdx.x < 16) s_b2[threadIdx.x] = threadIdx.x < A ? b2[threadIdx.x] : 0.f;
}

template <int R>
__device__ __forceinline__ void wg_zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}

// waits for every committed MMA group of the warpgroup, the last of which writes acc
__device__ __forceinline__ void wg_wait_all(float (&acc)[64]) {
  wg_wait<0>();
  wg_fence_acc(acc);
}

// acc = X * W0[:, 128 h .. 128 h + 127]   (K = 64).  dx: K-major descriptor of the 64 x 64 X tile, advanced by x_kstep bytes
// per 16 columns; w0_img: W0 image (layout above).  The _issue forms commit the MMAs as one group and return without waiting
// for it (the caller waits, e.g. with wg_wait_all); the others wait.  Both run the same MMAs.
__device__ __forceinline__ void gemm_x_w0_at_issue(float (&acc)[64], uint64_t dx, uint32_t x_kstep, uint32_t w0_img, int h) {
  const uint64_t db = wg_desc(w0_img + h * 16384, 8192, 1024, WG_SW128);
  wg_fence_acc(acc);
  wg_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wg_mma_ss_n128<0, 1>(acc, wg_adv(dx, k * x_kstep), wg_adv(db, k * 2048), k > 0);
  wg_commit();
}
__device__ __forceinline__ void gemm_x_w0_at(float (&acc)[64], uint64_t dx, uint32_t x_kstep, uint32_t w0_img, int h) {
  gemm_x_w0_at_issue(acc, dx, x_kstep, w0_img, h);
  wg_wait_all(acc);
}
// X as the 128B-swizzled tile of the layout above
__device__ __forceinline__ void gemm_x_w0_issue(float (&acc)[64], uint32_t s_x, uint32_t sbase, int h) {
  gemm_x_w0_at_issue(acc, wg_desc(s_x, 16, 1024, WG_SW128), 32, sbase + kImgW0, h);
}
__device__ __forceinline__ void gemm_x_w0(float (&acc)[64], uint32_t s_x, uint32_t sbase, int h) {
  gemm_x_w0_issue(acc, s_x, sbase, h);
  wg_wait_all(acc);
}
// acc = A * W1[:, 128 h ..]   (A: 64 x 256 in registers, 16 K blocks of 4 bf16x2)
__device__ __forceinline__ void gemm_a_w1(float (&acc)[64], const uint32_t (&a)[64], uint32_t sbase, int h) {
  const uint64_t db = wg_desc(sbase + kImgW1 + h * 65536, 32768, 1024, WG_SW128);
  wg_fence_acc(acc);
  wg_fence();
#pragma unroll
  for (int kb = 0; kb < 16; ++kb) wg_mma_rs_n128<1>(acc, &a[4 * kb], wg_adv(db, kb * 2048), kb > 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
// acc = A * W1^T[:, 128 h ..]  (the W1 image read K-major: K = output unit, N = input unit)
__device__ __forceinline__ void gemm_a_w1t(float (&acc)[64], const uint32_t (&a)[64], uint32_t sbase, int h) {
  const uint64_t db = wg_desc(sbase + kImgW1 + h * 16384, 16, 1024, WG_SW128);
  wg_fence_acc(acc);
  wg_fence();
#pragma unroll
  for (int kb = 0; kb < 16; ++kb) wg_mma_rs_n128<0>(acc, &a[4 * kb], wg_adv(db, (kb >> 2) * 32768 + (kb & 3) * 32), kb > 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
// z = A * W2   (64 x 16; columns >= A are zero)
__device__ __forceinline__ void gemm_a_w2(float (&z)[8], const uint32_t (&a)[64], uint32_t sbase) {
  const uint64_t db = wg_desc(sbase + kImgW2, 256, 128, WG_INTERLEAVE);
  wg_fence_acc(z);
  wg_fence();
#pragma unroll
  for (int kb = 0; kb < 16; ++kb) wg_mma_rs_n16<1>(z, &a[4 * kb], wg_adv(db, kb * 512), kb > 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(z);
}
// acc = dZ * W2^T[:, 128 h ..]  (dZ: 64 x 16 in registers, the W2 image at w2_img read K-major)
__device__ __forceinline__ void gemm_dz_w2t_at(float (&acc)[64], const uint32_t (&dz)[4], uint32_t w2_img, int h) {
  wg_fence_acc(acc);
  wg_fence();
  wg_mma_rs_n128<0>(acc, dz, wg_desc(w2_img + h * 4096, 128, 256, WG_INTERLEAVE), 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
__device__ __forceinline__ void gemm_dz_w2t(float (&acc)[64], const uint32_t (&dz)[4], uint32_t sbase, int h) {
  gemm_dz_w2t_at(acc, dz, sbase + kImgW2, h);
}
// half h of a hidden layer's epilogue: a[32 h + i] = bf16x2(relu(acc[2i] + b), relu(acc[2i+1] + b)), the A operand of the next GEMM
__device__ __forceinline__ void epi_bias_relu(const float (&acc)[64], const float* bias, int h, uint32_t (&a)[64], int lane) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 128 * h + 8 * (i >> 1) + 2 * (lane & 3));
    a[32 * h + i] = bias_relu_pack_bf16(__float_as_uint(acc[2 * i]), __float_as_uint(acc[2 * i + 1]), b);
  }
}

}  // namespace tc
}  // namespace stx
