// Library-wide entry points: version, thread-local error string, the mbarrier timeout record, a check of the call-free math.
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include "stx_common.cuh"

namespace stx {
namespace {
thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};
std::atomic<TrapRecord*> g_trap{nullptr};  // trap_record() once it has been allocated

TrapRecord* alloc_trap_record() {
  void* p = nullptr;
  if (cudaHostAlloc(&p, sizeof(TrapRecord), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return nullptr;
  *static_cast<TrapRecord*>(p) = TrapRecord{};
  return static_cast<TrapRecord*>(p);
}

// Counts the inputs with bit patterns in [lo, hi] where the call-free helper differs in any bit from the IEEE operation
// (fn 0: rcp_rn_callfree vs 1.0f / x, fn 1: sqrt_rn_callfree vs sqrtf); out[1] takes the smallest such pattern.
__global__ void callfree_math_check_kernel(int fn, uint32_t lo, uint32_t hi, unsigned long long* out) {
  unsigned long long bad = 0, first = ~0ull;
  for (uint64_t b = (uint64_t)lo + blockIdx.x * blockDim.x + threadIdx.x; b <= hi; b += (uint64_t)gridDim.x * blockDim.x) {
    const float x = __uint_as_float((uint32_t)b);
    const float got = fn == 0 ? rcp_rn_callfree(x) : sqrt_rn_callfree(x);
    const float want = fn == 0 ? 1.0f / x : sqrtf(x);
    if (__float_as_uint(got) != __float_as_uint(want)) ++bad, first = first < b ? first : b;
  }
  if (bad) atomicAdd(&out[0], bad), atomicMin(&out[1], first);
}
}  // namespace

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool pdl_enabled() {
  static const bool on = !(getenv("STX_PDL") && atoi(getenv("STX_PDL")) == 0);
  return on;
}
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
TrapRecord* trap_record() {
  static TrapRecord* const rec = alloc_trap_record();
  g_trap.store(rec);
  return rec;
}
}  // namespace stx

extern "C" int stx_version(void) { return STX_VERSION; }
extern "C" const char* stx_last_error_string(void) { return stx::g_err; }
extern "C" unsigned long long stx_launch_count(void) { return stx::g_launches.load(); }

extern "C" const char* stx_tc_trap_message(void) {
  static char msg[160];
  const volatile stx::TrapRecord* r = stx::g_trap.load();
  if (r == nullptr || r->claimed == 0u) return "";
  snprintf(msg, sizeof(msg), "mbarrier wait timeout in a tensor-core kernel: block %u thread %u tag %u parity %u", r->block,
           r->thread, r->tag, r->parity);
  return msg;
}

extern "C" int stx_debug_callfree_math(int fn, uint32_t lo, uint32_t hi, unsigned long long* out, void* stream) {
  STX_REQUIRE(out != nullptr && (fn == 0 || fn == 1) && lo <= hi, STX_E_ARG, "stx_debug_callfree_math: bad arguments");
  stx::callfree_math_check_kernel<<<4 * stx::kNumSMs, 256, 0, (cudaStream_t)stream>>>(fn, lo, hi, out);
  STX_LAUNCH_OK();
  return STX_OK;
}
