// spmm_common.cuh — pieces shared by the SpMM forward (spmm_fw.cu) and the row-wise SDDMM (spmm_bw.cu):
// work-queue records, kernel parameters, the per-warp cp.async index ring and the 16-byte vector math.
#pragma once

#include "common.cuh"

namespace tsb {

enum : int { R_SUM = TSB200_SUM, R_MEAN = TSB200_MEAN, R_MIN = TSB200_MIN, R_MAX = TSB200_MAX };

constexpr int kWarpsPerCta = 8;
constexpr int kRing = 128;      // entries per warp ring (4 windows of 32)
constexpr int kRingAlloc = kRing + 32;  // + mirror of window slot 0, so 32 consecutive entries never wrap
constexpr int kPrefetch = 2;    // windows issued ahead of the one being consumed
constexpr int kLongT = 256;     // rows longer than this are split into segments
constexpr int kSeg = 256;       // nnz per segment
constexpr int kItemCap = 1024;  // nnz budget of one 32-row work item before rows are deferred

struct Segment {      // 32 B
  int64_t row_b;      // b * M + row
  int64_t start, end; // absolute nnz range
  int64_t slot;       // partial slot, or -1: single-segment row, finalise directly
};
struct LongRow {      // 24 B
  int64_t row_b;
  int64_t first_slot;
  int64_t nseg_count;  // (nseg << 40) | count   (count = row degree < 2^40)
};

struct SpmmParams {
  const int64_t* rowptr;
  const int64_t* col;
  const void* value;
  const void* mat;
  void* out;
  int64_t* arg_out;
  int64_t B, M, N, K, E;
  int item_shift;  // work item = (1 << item_shift) consecutive rows, <= 32
  int mean;  // SUM kernels: divide by max(count,1) at the end
  int k0;  // first column handled by this launch (column tiling for very wide K)
  // column-block pipelining (SUM only): the product is built from several launches over disjoint column blocks of
  // A that share an fp32 partial [B, M, K]:  1 = write the partial, 2 = add to it, 3 = add to it and write `out`
  float* partial;
  int acc_mode;
  // planned mode (tsb200_spmm_plan, B == 1): which rows go through the segment list is known up front — bit r of
  // plan_mask[r / 32] — the list itself (segs / longs above) lives in the plan, its sizes are host-known, and the
  // main kernel drains it itself once the row items are gone (no segment / combine launches)
  const uint32_t* plan_mask;
  const uint32_t* seg_lr;   // long-row index of every segment (for the last-finisher combine)
  uint32_t* long_done;      // per call, zeroed: finished segments per long row
  int64_t n_seg, n_long;
  // workspace
  unsigned int* counters;  // [0] item counter, [1] #segments, [2] #long rows, [3] #partial slots
  Segment* segs;
  LongRow* longs;
  void* part_val;      // acc_t [slots, K]
  int64_t* part_arg;   // int64 [slots, K] (min/max)
  int64_t seg_cap, long_cap, slot_cap;
};

// ---- per-warp streaming index ring ------------------------------------------------------------
template <typename T> struct IndexRing {
  bool has_val;
  int64_t* s_col;
  T* s_val;
  const int64_t* col;
  const T* val;
  int64_t base;   // absolute nnz index of ring-relative 0 (multiple of 32)
  int64_t limit;  // absolute end of the range being streamed (windows past it are not fetched)
  int issued_w;   // last window issued
  int ready_w;    // windows <= ready_w are complete and visible to the whole warp

  // start streaming a new nnz range [.., limit_): copies still in flight from the previous range
  // (its last prefetched windows) must land before their slots are reused.
  __device__ __forceinline__ void reset(int64_t base_, int64_t limit_) {
    cp_async_wait<0>();
    __syncwarp();
    base = base_;
    limit = limit_;
    issued_w = -0x40000000;
    ready_w = -0x40000000;
  }
  __device__ __forceinline__ void issue(int w, int lane) {
    const int64_t abs0 = base + (int64_t)w * 32;
    const int ws = (w & 3) << 5;
    const bool mirror = ws == 0;  // slots [0,32) are duplicated at [kRing, kRing+32)
    {
      const int64_t a = abs0 + lane;
      const bool ok = a < limit;
      const void* src = ok ? (const void*)(col + a) : (const void*)col;
      cp_async_zfill<8>(s_col + ws + lane, src, ok ? 8 : 0);
      if (mirror) cp_async_zfill<8>(s_col + kRing + lane, src, ok ? 8 : 0);
    }
    if (has_val) {
      if constexpr (sizeof(T) >= 4) {
        const int64_t a = abs0 + lane;
        const bool ok = a < limit;
        const void* src = ok ? (const void*)(val + a) : (const void*)val;
        cp_async_zfill<sizeof(T)>(s_val + ws + lane, src, ok ? (int)sizeof(T) : 0);
        if (mirror) cp_async_zfill<sizeof(T)>(s_val + kRing + lane, src, ok ? (int)sizeof(T) : 0);
      } else {
        constexpr int EPL = 4 / sizeof(T);  // entries per lane copy
        if (lane < 32 / EPL) {
          const int64_t a = abs0 + (int64_t)lane * EPL;
          const int64_t rem = limit - a;
          const int nb = rem <= 0 ? 0 : (rem >= EPL ? 4 : (int)rem * (int)sizeof(T));
          const void* src = nb ? (const void*)(val + a) : (const void*)val;
          cp_async_zfill<4>(s_val + ws + lane * EPL, src, nb);
          if (mirror) cp_async_zfill<4>(s_val + kRing + lane * EPL, src, nb);
        }
      }
    }
    cp_async_commit();
  }
  // make ring-relative entries [lo_rel, hi_rel) readable (hi_rel - lo_rel <= 32)
  __device__ __forceinline__ void ensure(int lo_rel, int hi_rel, int lane) {
    const int need_w = (hi_rel - 1) >> 5;
    if (need_w <= ready_w) return;
    const int low_w = lo_rel >> 5;
    if (issued_w < need_w + kPrefetch) {
      __syncwarp();  // every lane is done reading the windows about to be overwritten
      if (issued_w < low_w - 1) {  // skip-ahead (deferred rows): drain before slots are reused out of order
        cp_async_wait<0>();
        __syncwarp();
        issued_w = low_w - 1;
      }
      while (issued_w < need_w + kPrefetch) issue(++issued_w, lane);
    }
    cp_async_wait<kPrefetch>();
    __syncwarp();
    ready_w = issued_w - kPrefetch;
  }
};

// ---- accumulator helpers -----------------------------------------------------------------------
// Vec<T>: how one 16-byte gather of T is folded into fp32 accumulators.
//   * bf16 / f16: both halves of a packed pair are widened to fp32 (exact: a bf16 widens with a shift or a mask,
//     an f16 with one conversion) and folded with FFMA. The product of two 16-bit values is exact in fp32, so this
//     rounds once per term, exactly like a fused mixed-precision FMA would.
//   * the nnz value travels as the raw storage bits (`vraw`), 1.0 when has_value=false.
template <typename T> struct Vec;
template <> struct Vec<float> {
  static constexpr int VEC = 4;
  using vraw = float;
  static __device__ __forceinline__ vraw one() { return 1.f; }
  static __device__ __forceinline__ float vfloat(vraw v) { return v; }
  static __device__ __forceinline__ void fma(float* acc, vraw v, const uint4& d) {
    acc[0] = fmaf(v, __uint_as_float(d.x), acc[0]);
    acc[1] = fmaf(v, __uint_as_float(d.y), acc[1]);
    acc[2] = fmaf(v, __uint_as_float(d.z), acc[2]);
    acc[3] = fmaf(v, __uint_as_float(d.w), acc[3]);
  }
  static __device__ __forceinline__ void unpack(const uint4& d, float* f) {
    f[0] = __uint_as_float(d.x); f[1] = __uint_as_float(d.y);
    f[2] = __uint_as_float(d.z); f[3] = __uint_as_float(d.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                      __float_as_uint(f[3]));
  }
  static __device__ __forceinline__ float round_prod(float x) { return x; }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int VEC = 8;
  using vraw = unsigned short;
  static __device__ __forceinline__ vraw one() { return 0x3F80; }
  static __device__ __forceinline__ float vfloat(vraw v) { return __uint_as_float((uint32_t)v << 16); }
  static __device__ __forceinline__ void fma(float* acc, vraw v, const uint4& d) {
    const float vf = vfloat(v);
    float f[VEC];
    unpack(d, f);
#pragma unroll
    for (int i = 0; i < VEC; i++) acc[i] = fmaf(vf, f[i], acc[i]);
  }
  static __device__ __forceinline__ void unpack(const uint4& d, float* f) {
    const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  static __device__ __forceinline__ float round_prod(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
};
template <> struct Vec<__half> {
  static constexpr int VEC = 8;
  using vraw = unsigned short;
  static __device__ __forceinline__ vraw one() { return 0x3C00; }
  static __device__ __forceinline__ float vfloat(vraw v) { return __half2float(__ushort_as_half(v)); }
  static __device__ __forceinline__ void fma(float* acc, vraw v, const uint4& d) {
    const float vf = vfloat(v);
    float f[VEC];
    unpack(d, f);
#pragma unroll
    for (int i = 0; i < VEC; i++) acc[i] = fmaf(vf, f[i], acc[i]);
  }
  static __device__ __forceinline__ void unpack(const uint4& d, float* f) {
    const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  // min/max compare on the product rounded to the storage type, as the reference does
  // (csrc/cpu/spmm_cpu.cpp:81-83 forms `val * mat` in scalar_t).
  static __device__ __forceinline__ float round_prod(float x) { return __half2float(__float2half_rn(x)); }
};


// workspace layout of the row-split kernels (work counters, deferred segments, partials)
struct WsLayout {
  size_t counters, segs, longs, part_val, part_arg, total;
  int64_t seg_cap, long_cap, slot_cap;
};
static inline WsLayout ws_layout(int64_t B, int64_t K, int64_t E, bool arg, bool partials = true) {
  WsLayout L;
  const int64_t EB = E * (B > 0 ? B : 1);
  L.seg_cap = EB / 32 + EB / 128 + 64;
  L.long_cap = EB / kLongT + 64;
  L.slot_cap = EB / 128 + 64;
  size_t off = 0;
  L.counters = off; off += 256;
  L.segs = off; off += align_up((size_t)L.seg_cap * sizeof(Segment), 256);
  L.longs = off; off += align_up((size_t)L.long_cap * sizeof(LongRow), 256);
  L.part_val = off; off += partials ? align_up((size_t)L.slot_cap * (size_t)K * sizeof(float), 256) : 0;
  L.part_arg = off; off += (partials && arg) ? align_up((size_t)L.slot_cap * (size_t)K * sizeof(int64_t), 256) : 0;
  L.total = off;
  return L;
}

static inline int grid_for(const void* kernel, int threads) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  return per_sm * num_sms();
}

// Persistent-grid size of one kernel instantiation, cached PER DEVICE (the occupancy query costs microseconds per
// launch otherwise). Lock-free: racing threads compute the same value.
struct GridCache {
  std::atomic<int> v[kMaxDevices];
  int get(const void* kernel, int threads) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return grid_for(kernel, threads);
    int g = v[dev].load(std::memory_order_relaxed);
    if (g <= 0) {
      g = grid_for(kernel, threads);
      v[dev].store(g, std::memory_order_relaxed);
    }
    return g;
  }
};

}  // namespace tsb
