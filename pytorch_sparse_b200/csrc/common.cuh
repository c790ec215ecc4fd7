// common.cuh — shared helpers for the libtsb200 kernels (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <limits>
#include <type_traits>

#include "../../include/tsb200.h"

#define TSB_CUDA_TRY(expr)                   \
  do {                                       \
    cudaError_t _e = (expr);                 \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

#define TSB_LAUNCH_CHECK()                   \
  do {                                       \
    cudaError_t _e = cudaGetLastError();     \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

namespace tsb {

constexpr int kDefaultSMs = 132;  // H100 SXM (used only if the attribute query fails)
constexpr int kMaxDevices = 64;

// SM count of the CURRENT device, queried once per device and cached (thread-safe: idempotent atomic stores).
static inline int num_sms() {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return kDefaultSMs;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v > 0) return v;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1) v = kDefaultSMs;
  cache[dev].store(v, std::memory_order_relaxed);
  return v;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- element type traits ---------------------------------------------------------------
// acc_t: the type sums are accumulated in (fp32 for 16/32-bit floats, the type itself otherwise).
template <typename T> struct Traits {
  using acc_t = T;
  static __host__ __device__ __forceinline__ acc_t to_acc(T v) { return v; }
  static __host__ __device__ __forceinline__ T from_acc(acc_t v) { return v; }
  static __host__ __device__ __forceinline__ T lowest() { return std::numeric_limits<T>::lowest(); }
  static __host__ __device__ __forceinline__ T highest() { return std::numeric_limits<T>::max(); }
};
template <> struct Traits<float> {
  using acc_t = float;
  static __host__ __device__ __forceinline__ float to_acc(float v) { return v; }
  static __host__ __device__ __forceinline__ float from_acc(float v) { return v; }
  static __host__ __device__ __forceinline__ float lowest() { return -3.402823466e+38f; }
  static __host__ __device__ __forceinline__ float highest() { return 3.402823466e+38f; }
};
template <> struct Traits<double> {
  using acc_t = double;
  static __host__ __device__ __forceinline__ double to_acc(double v) { return v; }
  static __host__ __device__ __forceinline__ double from_acc(double v) { return v; }
  static __host__ __device__ __forceinline__ double lowest() { return -1.7976931348623157e+308; }
  static __host__ __device__ __forceinline__ double highest() { return 1.7976931348623157e+308; }
};
template <> struct Traits<__half> {
  using acc_t = float;
  static __device__ __forceinline__ float to_acc(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_acc(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ __half lowest() { return __ushort_as_half(0xFBFF); }   // -65504
  static __device__ __forceinline__ __half highest() { return __ushort_as_half(0x7BFF); }  // 65504
};
template <> struct Traits<__nv_bfloat16> {
  using acc_t = float;
  static __device__ __forceinline__ float to_acc(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_acc(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ __nv_bfloat16 lowest() { return __ushort_as_bfloat16(0xFF7F); }
  static __device__ __forceinline__ __nv_bfloat16 highest() { return __ushort_as_bfloat16(0x7F7F); }
};

template <typename T> struct is_float16 : std::false_type {};
template <> struct is_float16<__half> : std::true_type {};
template <> struct is_float16<__nv_bfloat16> : std::true_type {};

static inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case TSB200_F32: return 4;
    case TSB200_F64: return 8;
    case TSB200_F16: return 2;
    case TSB200_BF16: return 2;
    case TSB200_I32: return 4;
    case TSB200_I64: return 8;
    case TSB200_I16: return 2;
    case TSB200_I8: return 1;
    case TSB200_U8: return 1;
    default: return 0;
  }
}

// Runtime dtype -> compile-time type. `fn` is a generic lambda taking a value of the type.
template <typename F> static inline int dispatch_dtype(int dtype, F&& fn) {
  switch (dtype) {
    case TSB200_F32: return fn(float{});
    case TSB200_F64: return fn(double{});
    case TSB200_F16: return fn(__half{});
    case TSB200_BF16: return fn(__nv_bfloat16{});
    case TSB200_I32: return fn(int32_t{});
    case TSB200_I64: return fn(int64_t{});
    case TSB200_I16: return fn(int16_t{});
    case TSB200_I8: return fn(int8_t{});
    case TSB200_U8: return fn(uint8_t{});
    default: return TSB200_ERR_INVALID_ARG;
  }
}
template <typename F> static inline int dispatch_float_dtype(int dtype, F&& fn) {
  switch (dtype) {
    case TSB200_F32: return fn(float{});
    case TSB200_F64: return fn(double{});
    case TSB200_F16: return fn(__half{});
    case TSB200_BF16: return fn(__nv_bfloat16{});
    default: return TSB200_ERR_UNSUPPORTED;
  }
}

// ---- PTX helpers -----------------------------------------------------------------------
// 128-bit read-only gather that prefers to stay in L2 (the dense operand is re-read E/N times).
__device__ __forceinline__ uint64_t make_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// Range policy over the dense operand: the first `primary_bytes` of [base, base + total_bytes) are kept with
// evict_last, the rest is streamed with evict_first. When the operand is larger than L2 a blanket evict_last protects
// nothing from itself (every line has the same priority); pinning a fixed slice that FITS turns that slice's
// gathers into guaranteed hits and lets the remainder stream past it.
__device__ __forceinline__ uint64_t make_policy_range(const void* base, uint32_t primary_bytes, uint32_t total_bytes) {
  uint64_t pol;
  asm volatile("createpolicy.range.global.L2::evict_last.L2::evict_first.b64 %0, [%1], %2, %3;"
               : "=l"(pol) : "l"(base), "r"(primary_bytes), "r"(total_bytes));
  return pol;
}
__device__ __forceinline__ uint64_t make_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint4 ldg128_hint(const void* p, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
// scalar read-only loads with an L2 eviction-priority hint (operands that are re-read while a large output
// streams through L2, e.g. B in SpSpMM)
__device__ __forceinline__ uint64_t ldg64_hint(const void* p, uint64_t pol) {
  uint64_t r;
  asm volatile("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint32_t ldg32_hint(const void* p, uint64_t pol) {
  uint32_t r;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ float ldg_hint(const float* p, uint64_t pol) { return __uint_as_float(ldg32_hint(p, pol)); }
__device__ __forceinline__ double ldg_hint(const double* p, uint64_t pol) {
  return __longlong_as_double((long long)ldg64_hint(p, pol));
}
// predicated form: loads only when `pred`, otherwise leaves `r` untouched (the address is not dereferenced)
__device__ __forceinline__ void ldg128_hint_pred(uint4& r, const void* p, uint64_t pol, bool pred) {
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t"
      "@q ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %6;\n\t}"
      : "+r"(r.x), "+r"(r.y), "+r"(r.z), "+r"(r.w)
      : "l"(p), "r"((int)pred), "l"(pol));
}
__device__ __forceinline__ uint4 ldg128(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// streaming 128-bit store (outputs are written once, never re-read by the kernel).
__device__ __forceinline__ void stg128_stream(void* p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
// cp.async (LDGSTS) with zero-fill: copies `src_bytes` (<= CP) bytes and zero-fills the rest.
template <int CP> __device__ __forceinline__ void cp_async_zfill(void* smem_dst, const void* gsrc,
                                                                   int src_bytes) {
  uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(d), "l"(gsrc), "n"(CP),
               "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

}  // namespace tsb
