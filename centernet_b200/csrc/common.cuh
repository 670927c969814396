// Shared device/host helpers for the centernet_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <atomic>
#include "../../include/centernet_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900 || !defined(__CUDA_ARCH_FEAT_SM90_ALL))
#error "centernet_b200 is written for sm_90a (H100) only"
#endif

namespace cnb {

// ------------------------------------------------------------------ host side
void set_error(const char *fmt, ...);
extern std::atomic<unsigned long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

#define CNB_REQUIRE(cond, code, ...)            \
  do {                                          \
    if (!(cond)) {                              \
      cnb::set_error(__VA_ARGS__);              \
      return (code);                            \
    }                                           \
  } while (0)

#define CNB_CHECK_LAUNCH(what)                                                   \
  do {                                                                           \
    cudaError_t e__ = cudaGetLastError();                                        \
    if (e__ != cudaSuccess) {                                                    \
      cnb::set_error("%s: CUDA error: %s", (what), cudaGetErrorString(e__));     \
      return CNB_ECUDA;                                                          \
    }                                                                            \
  } while (0)

// A failed runtime call also leaves its (non-sticky) error as the last error; CNB_CUDA clears it, or the next
// CNB_CHECK_LAUNCH would report it against an unrelated launch.
#define CNB_CUDA(call)                                                           \
  do {                                                                           \
    cudaError_t e__ = (call);                                                    \
    if (e__ != cudaSuccess) {                                                    \
      cnb::set_error("%s: CUDA error: %s", #call, cudaGetErrorString(e__));      \
      (void)cudaGetLastError();                                                  \
      return CNB_ECUDA;                                                          \
    }                                                                            \
  } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
inline int num_sms() {
  int dev = 0, n = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}
inline bool dtype_known(int dt) { return dt == CNB_DTYPE_F32 || dt == CNB_DTYPE_F16 || dt == CNB_DTYPE_BF16; }

// ---------------------------------------------------------------- device side
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Waits with a watchdog: a protocol bug must surface as a loud failure (trap -> the host sees a launch
// error on its next CUDA call), never as a kernel that spins forever.  ~2 s at 2 GHz.  No printf here:
// a device printf in the wait path costs the hot kernel registers and a stack frame.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (UBLKCP in SASS).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
// Exact widening of one map / head element to fp32 (every fp16 and bf16 value, subnormals and infinities included,
// is a float: the result equals torch's .float()).
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

#define CNB_NEG_INF (__int_as_float(0xff800000))

// 64-bit selection key: (fp32 bits of a strictly positive score) << 32 | ~flat_index.
// Larger key == better under (score desc, flat index asc).
__device__ __forceinline__ unsigned long long make_key(uint32_t score_bits, uint32_t flat_idx) {
  return ((unsigned long long)score_bits << 32) | (unsigned long long)(0xffffffffu - flat_idx);
}
__device__ __forceinline__ uint32_t key_idx(unsigned long long k) { return 0xffffffffu - (uint32_t)k; }
__device__ __forceinline__ uint32_t key_bits(unsigned long long k) { return (uint32_t)(k >> 32); }
#endif  // __CUDACC__

}  // namespace cnb
