// Micro-benchmark: per-SM global store throughput (diagnostic only).
//   mode 0: st.global.v4, one warp instruction = 512 contiguous bytes (the K3a epilogue pattern)
//   mode 1: same bytes staged in shared memory and written with cp.async.bulk (shared -> global), 16 KB per bulk copy
//   mode 2: st.global.v4 with each thread writing 64 contiguous bytes (4 x v4) -> fewer, fuller sectors per instruction stream
// footprint per CTA is a parameter: small = L2-resident, large = streams to HBM.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int MODE>
__global__ void k(int iters, size_t cta_bytes, uint8_t* gbuf, long long* out) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  uint8_t* base = gbuf + (size_t)blockIdx.x * cta_bytes;
  const size_t mask = cta_bytes - 1;
  __syncthreads();
  const long long t0 = clock64();
  if (MODE == 0) {
    for (int i = 0; i < iters; ++i) {
      const size_t off = ((size_t)(i * nwarps + warp) * 2048) & mask;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<uint4*>(base + off + j * 512 + lane * 16) = make_uint4(i, j, lane, warp);
    }
  } else if (MODE == 2) {
    for (int i = 0; i < iters; ++i) {
      const size_t off = ((size_t)(i * nwarps + warp) * 2048) & mask;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<uint4*>(base + off + lane * 64 + j * 16) = make_uint4(i, j, lane, warp);
    }
  } else {
    // every warp fills its 2 KB slice of a 16 KB buffer (8 warps), then one thread issues the bulk store
    for (int i = 0; i < iters; ++i) {
      uint8_t* sb = sm + (i & 1) * 16384;
      if (i >= 2 && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(sb + warp * 2048 + j * 512 + lane * 16) = make_uint4(i, j, lane, warp);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      if (threadIdx.x == 0) {
        const size_t off = ((size_t)i * 16384) & mask;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(base + off), "r"(smem_u32(sb)), "r"(16384) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  __syncthreads();
  const long long t1 = clock64();
  if (threadIdx.x == 0) out[blockIdx.x] = t1 - t0;
}

int main() {
  long long* out;
  uint8_t* gbuf;
  const size_t big = (size_t)4 << 20;  // 4 MB per CTA -> 592 MB total
  cudaMalloc(&out, 132 * 8);
  cudaMalloc(&gbuf, 132 * big);
  cudaFuncSetAttribute(k<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
  const int iters = 4000;
  for (int grid : {132, 66, 32, 8})
  for (size_t cta_bytes : {(size_t)65536, big})
    for (int mode = 0; mode < 2; ++mode)
      for (int warps : {8}) {
        if (grid != 132 && mode == 1) continue;
        for (int rep = 0; rep < 2; ++rep) {
          if (mode == 0) k<0><<<grid, warps * 32>>>(iters, cta_bytes, gbuf, out);
          if (mode == 1) k<1><<<grid, warps * 32, 32768>>>(iters, cta_bytes, gbuf, out);
          cudaError_t e = cudaDeviceSynchronize();
          if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
        }
        long long h[132];
        cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
        long long mx = 0;
        for (int i = 0; i < grid; ++i) mx = h[i] > mx ? h[i] : mx;
        const double bytes = mode == 1 ? (double)iters * 16384.0 : (double)warps * iters * 2048.0;
        printf("grid %3d footprint/CTA %7zu KB mode %d warps %2d: %.1f B/clk/SM (CTA 0), %.1f (slowest CTA)\n", grid, cta_bytes >> 10, mode, warps, bytes / h[0], bytes / mx);
      }
  return 0;
}
