// spmm_common.cuh — pieces shared by the SpMM forward (spmm_fw.cu) and the row-wise SDDMM (spmm_bw.cu):
// work-queue records, kernel parameters, the row-deferral rule, the per-warp cp.async index ring, the 16-byte
// vector math, and on the host the workspace binding, the row-split limits and launch, and the dtype switch.
#pragma once

#include <cstdlib>
#include <initializer_list>

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
  // fp8 dense operand (tsb200_spmm_fw_fp8): the weight of entry e is fl32(value[e] * scale[col[e] * scale_stride]),
  // scale_stride 0 = one scale for the whole operand, 1 = one per dense row
  const float* scale;
  uint32_t scale_stride;
  // e4m3 result (tsb200_spmm_fw_fp8_quant): `out` is e4m3 [M, K], out_scale[m] = amax_k |y[m,k]| / 448 (1 if not > 0)
  float* out_scale;
  // residual (RES kernels; tsb200_spmm_fw_fp8_res, tsb200_spmm_fw_res): row m of the result is y[m] +
  // fl32(res_scale[m * res_stride] * res[m]), res [M, K] of the dense operand's element type (e4m3 or T), added after
  // the mean's division and before the e4m3 quantisation
  const void* res;
  const float* res_scale;
  uint32_t res_stride;
  // multi-head operands (tsb200_spmm_heads / tsb200_sddmm_heads, HEADS kernels only): K = heads * D, and the weight of
  // column k of entry e is value[e * heads + k / D]. It fills the struct's tail padding, so the parameter offsets of
  // every kernel that takes further arguments stay as they were.
  int heads;
};

// ---- the deferral rule of the row-split kernels -------------------------------------------------
// Whether this lane's row (deg nnz) of a work item goes to the segment list instead of being walked by the item's
// warp: it is longer than kLongT, or it lies past the item's kItemCap-nnz budget (a prefix sum over the lanes of the
// degrees of the rows that are not long). Called by all 32 lanes. The SpMM forward's main kernels, its plan kernel
// and the row-wise SDDMM all defer by this one rule, so planned and unplanned products walk the same rows.
__device__ __forceinline__ bool defer_row(int deg, int lane) {
  const bool is_long = deg > kLongT;
  int cum = is_long ? 0 : deg;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, cum, off);
    if (lane >= off) cum += t;
  }
  return (deg > 0) && (is_long || cum > kItemCap);
}

// Lane 0's ticket from the counter c (0 on the other lanes): the work items, and the planned drain's segments, of the
// row-split kernels are handed out this way.
__device__ __forceinline__ unsigned int take_ticket(unsigned int* c, int lane) {
  unsigned int t = 0;
  if (lane == 0) t = atomicAdd(c, 1u);
  return t;
}

// ---- per-warp streaming index ring ------------------------------------------------------------
template <typename T> struct Vec;
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

  // bind to this warp's shared arrays and to the index stream of p (entries [0, p.E)). VALUES: p.value streams next to
  // the column words, or, when there is none, the value half holds a constant 1 (filled here, once). Without VALUES
  // (the SDDMM, per-head weights) only the column words stream.
  template <bool VALUES>
  __device__ __forceinline__ void bind(const SpmmParams& p, int64_t* s_col_, T* s_val_, int lane) {
    s_col = s_col_;
    s_val = s_val_;
    has_val = VALUES && p.value != nullptr;
    if constexpr (VALUES) {
      if (!has_val) {
        using VR = typename Vec<T>::vraw;
        for (int i = lane; i < kRingAlloc; i += 32) reinterpret_cast<VR*>(s_val)[i] = Vec<T>::one();
        __syncwarp();
      }
    }
    col = p.col;
    val = VALUES ? (const T*)p.value : nullptr;
    limit = p.E;
  }
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
// e4m3 dense operand: a 16-byte gather is 16 elements, widened pairwise through f16x2 (cvt.rn.f16x2.e4m3x2, sm_89+)
// and then to fp32; both steps are exact (every e4m3 value, NaN included, is an f16 value). Only the unpack is used:
// values and outputs keep their own type (Vec<T> above).
template <> struct Vec<__nv_fp8_e4m3> {
  static constexpr int VEC = 16;
  static __device__ __forceinline__ void unpack(const uint4& d, float* f) {
    const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        uint32_t r;
        asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((unsigned short)(w[i] >> (16 * h))));
        const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&r));
        f[4 * i + 2 * h] = t.x;
        f[4 * i + 2 * h + 1] = t.y;
      }
    }
  }
};

// ---- e4m3 result with a per-row scale (tsb200_spmm_fw_fp8_quant) ---------------------------------------------------
// The definition is torch's quantize_fp8 on the CPU: s = amax|y| / 448 (IEEE division), 1 when amax is not > 0, then
// e4m3(y / s). The amax keeps NaN (torch's amax propagates it; fmaxf would drop it), so a row holding NaN gets s = 1.
__device__ __forceinline__ float amax_nan(float m, float a) { return (a > m || a != a) ? a : m; }
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f; }

// two floats as e4m3 (lo in the low byte), following torch's non-saturating float8_e4m3fn cast: round to nearest even,
// subnormals kept, -0 stays -0, and a magnitude past 464 (the midpoint above 448) or an inf becomes NaN.
// cvt.rn.satfinite clamps those to +-448, so they are patched afterwards.
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  unsigned short r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  uint32_t w = r;
  if (fabsf(lo) > 464.f) w = (w & 0xff00u) | 0x7fu;
  if (fabsf(hi) > 464.f) w = (w & 0x00ffu) | 0x7f00u;
  return w;
}
__device__ __forceinline__ uint8_t e4m3_quant(float y, float s) { return (uint8_t)e4m3x2(__fdiv_rn(y, s), 0.f); }

// 16 results of one lane, divided by the row scale, as one 16-byte vector of e4m3
__device__ __forceinline__ uint4 e4m3_pack16(const float* f, float s) {
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; j++)
    w[j] = e4m3x2(__fdiv_rn(f[4 * j], s), __fdiv_rn(f[4 * j + 1], s)) |
           (e4m3x2(__fdiv_rn(f[4 * j + 2], s), __fdiv_rn(f[4 * j + 3], s)) << 16);
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- residual (tsb200_spmm_fw_fp8_res, tsb200_spmm_fw_res) ---------------------------------------------------------
// z = fl(y + fl(rs * r)) in the accumulator type (fp32, fp64 for fp64): one IEEE product and one IEEE add, never
// contracted to an FMA. The residual R has the dense operand's element type: e4m3 (stored as bytes, with its own
// per-row scale) or the result type T. It is read once, so it is loaded with the streaming (evict-first) hint.
__device__ __forceinline__ float e4m3_to_f32(uint8_t b) {
  uint32_t r;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((unsigned short)b));
  return __half2float(__ushort_as_half((unsigned short)(r & 0xffffu)));
}
template <typename R> struct ResElem {  // storage and exact widening of one residual element
  using raw = R;
  static __device__ __forceinline__ typename Traits<R>::acc_t widen(R r) { return Traits<R>::to_acc(r); }
};
template <> struct ResElem<__nv_fp8_e4m3> {
  using raw = uint8_t;
  static __device__ __forceinline__ float widen(uint8_t r) { return e4m3_to_f32(r); }
};
template <typename A> __device__ __forceinline__ A res_add(A y, A rs, A r) {
  if constexpr (std::is_same<A, double>::value) return __dadd_rn(y, __dmul_rn(rs, r));
  else return __fadd_rn(y, __fmul_rn(rs, r));
}
// one lane's Vec<R>::VEC consecutive fp32 results plus their residual columns (one 16-byte load)
template <typename R> __device__ __forceinline__ void res_add_vec(float* f, const typename ResElem<R>::raw* r, float rs) {
  float q[Vec<R>::VEC];
  Vec<R>::unpack(__ldcs(reinterpret_cast<const uint4*>(r)), q);
#pragma unroll
  for (int i = 0; i < Vec<R>::VEC; i++) f[i] = res_add(f[i], rs, q[i]);
}
// the residual row at this launch's first column (the row stores); res_at: one element (the combines)
template <typename R> __device__ __forceinline__ const typename ResElem<R>::raw* res_row(const SpmmParams& p,
                                                                                        int64_t row) {
  return (const typename ResElem<R>::raw*)p.res + row * p.K + p.k0;
}
template <typename R> __device__ __forceinline__ const typename ResElem<R>::raw* res_at(const SpmmParams& p, int64_t row,
                                                                                       int64_t k) {
  return (const typename ResElem<R>::raw*)p.res + row * p.K + k;
}
__device__ __forceinline__ float res_scale(const SpmmParams& p, int64_t row) {
  return __ldg(p.res_scale + row * p.res_stride);
}


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
// binds an unplanned workspace (layout L at ws) to p: work counters, segment queue, long rows, partials; no plan
static inline void bind_ws(SpmmParams& p, char* ws, const WsLayout& L, bool arg) {
  p.plan_mask = nullptr; p.seg_lr = nullptr; p.long_done = nullptr; p.n_seg = 0; p.n_long = 0;
  p.counters = (unsigned int*)(ws + L.counters);
  p.segs = (Segment*)(ws + L.segs);
  p.longs = (LongRow*)(ws + L.longs);
  p.part_val = ws + L.part_val;
  p.part_arg = arg ? (int64_t*)(ws + L.part_arg) : nullptr;
  p.seg_cap = L.seg_cap; p.long_cap = L.long_cap; p.slot_cap = L.slot_cap;
}
// checks an unplanned workspace for p (layout ws_layout(p.B, p.K, p.E, ...)) and binds it: 0, TSB200_ERR_WORKSPACE
// when it is missing or short, else TSB200_ERR_INVALID_ARG when it is not 256-byte aligned
static inline int bind_unplanned(SpmmParams& p, void* workspace, size_t bytes, bool arg, bool partials = true) {
  const WsLayout L = ws_layout(p.B, p.K, p.E, arg, partials);
  if (!workspace || bytes < L.total) return TSB200_ERR_WORKSPACE;
  if ((uintptr_t)workspace & 255) return TSB200_ERR_INVALID_ARG;
  bind_ws(p, (char*)workspace, L, arg);
  return 0;
}

// Extents the row-split kernels index in 32-bit arithmetic: E entries (an index ring reads up to 64 past the last), N
// dense rows of row_bytes each, and M rows of a second dense operand where a kernel gathers those by row index.
static inline bool rowsplit_extents(int64_t E, int64_t N, int64_t row_bytes, int64_t M = 0) {
  return E < ((int64_t)1 << 31) - 64 && N < ((int64_t)1 << 32) && row_bytes < ((int64_t)1 << 31) &&
         M < ((int64_t)1 << 32);
}
// Pointer alignments of the row-split kernels: dense operands, dense results and arg_out 16 B (vector loads and
// stores), col 8 B (cp.async), values and scales 4 B. A NULL (absent) operand passes.
static inline bool rowsplit_aligned(std::initializer_list<const void*> rows, const void* col,
                                    std::initializer_list<const void*> words = {}) {
  for (const void* r : rows)
    if ((uintptr_t)r & 15) return false;
  for (const void* w : words)
    if ((uintptr_t)w & 3) return false;
  return !((uintptr_t)col & 7);
}

// Runtime dtype -> compile-time type for the vector kernels (F32, F16, BF16); TSB200_ERR_UNSUPPORTED for any other.
template <typename F> static inline int dispatch_vec_dtype(int dtype, F&& fn) {
  switch (dtype) {
    case TSB200_F32: return fn(float{});
    case TSB200_F16: return fn(__half{});
    case TSB200_BF16: return fn(__nv_bfloat16{});
    default: return TSB200_ERR_UNSUPPORTED;
  }
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

// Work item of the SpMM forward and SDDMM row kernels: 2^s consecutive rows, s <= 5. Small matrices shrink it, so that
// each of the grid_main * kWarpsPerCta resident warps gets at least two items of the `rows` rows (all batches).
// TSB200_SPMM_ITEM_SHIFT = 0..5, read on every call, fixes s instead: a test knob, so that small matrices can run
// every item size. Unset or out of range, it is ignored.
static inline int item_shift_for(int64_t rows, int grid_main) {
  const int64_t want = rows / ((int64_t)grid_main * kWarpsPerCta * 2);
  int s = 0;
  while (s < 5 && ((int64_t)2 << s) <= want) s++;
  const char* ev = getenv("TSB200_SPMM_ITEM_SHIFT");
  if (!ev) return s;
  char* end = nullptr;
  const long v = strtol(ev, &end, 10);
  return (end != ev && *end == '\0' && v >= 0 && v <= 5) ? (int)v : s;
}

// The unplanned row-split launch: the work counters cleared, the main kernel over the row items, then the segment
// kernel over the rows the main kernel deferred; `args` follow p in both kernels. The grid caches are the caller's,
// one pair per kernel instantiation: a cache shared by two kernels would give one of them the other's grid.
template <typename Kernel, typename... A>
static int launch_rowsplit(Kernel* kmain, Kernel* kseg, GridCache& gc_main, GridCache& gc_seg, SpmmParams& p,
                           cudaStream_t st, A... args) {
  const int grid_main = gc_main.get((const void*)kmain, kWarpsPerCta * 32);
  const int grid_seg = gc_seg.get((const void*)kseg, kWarpsPerCta * 32);
  p.item_shift = item_shift_for(p.M * p.B, grid_main);
  const int64_t n_items = ((p.M + (1 << p.item_shift) - 1) >> p.item_shift) * p.B;
  TSB_CUDA_TRY(cudaMemsetAsync(p.counters, 0, 64, st));
  const int gm = (int)min((int64_t)grid_main, (n_items + kWarpsPerCta - 1) / kWarpsPerCta);
  kmain<<<gm, kWarpsPerCta * 32, 0, st>>>(p, args...);
  TSB_LAUNCH_CHECK();
  kseg<<<grid_seg, kWarpsPerCta * 32, 0, st>>>(p, args...);
  TSB_LAUNCH_CHECK();
  return 0;
}

// CTAs of 256 threads for a generic kernel that gives each of n_warps rows (or entries) a warp: one warp each, at most
// cap_per_sm CTAs per SM
static inline int warp_grid(int64_t n_warps, int cap_per_sm) {
  return (int)min((n_warps + 7) / 8, (int64_t)num_sms() * cap_per_sm);
}

// ---- the row-split kernels' building blocks: value loads, the engine hooks, the segment queue, the work-item
// front, a lane's columns, the segment walk, and on the host the plan and planned-workspace layouts. The SpMM
// forward (spmm_fw.cu) and the softmax aggregation (spmm_softmax_aggr.cu) both build their kernels from these.
template <typename T> __device__ __forceinline__ typename Vec<T>::vraw load_vraw(const T* p);
template <> __device__ __forceinline__ float load_vraw<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ unsigned short load_vraw<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __ldg(reinterpret_cast<const unsigned short*>(p));
}
template <> __device__ __forceinline__ unsigned short load_vraw<__half>(const __half* p) {
  return __ldg(reinterpret_cast<const unsigned short*>(p));
}

template <typename Eng> __device__ __forceinline__ void set_scale(Eng& eng, const SpmmParams& p) {
  if constexpr (Eng::Q8) {
    eng.scale = p.scale;
    eng.sstride = p.scale_stride;
  }
}
// HEADS: the head of each of this lane's chunks (chunk ch starts at column k0 + (ch * LPR + li) * VEC), computed once
// per kernel by head_cols, and handed to every row's engine by set_heads
template <bool HEADS, int LPR, int VEC, int CH>
__device__ __forceinline__ void head_cols(int (&hcol)[HEADS ? CH : 1], const SpmmParams& p, int li) {
  if constexpr (HEADS) {
    const int D = (int)(p.K / p.heads);
#pragma unroll
    for (int ch = 0; ch < CH; ch++) hcol[ch] = (p.k0 + (ch * LPR + li) * VEC) / D;
  }
}
template <bool HEADS, typename Eng, int NH>
__device__ __forceinline__ void set_heads(Eng& eng, const SpmmParams& p, const int (&hcol)[NH]) {
  if constexpr (HEADS) {
    eng.hval = (decltype(eng.hval))p.value;
    eng.heads = p.heads;
#pragma unroll
    for (int i = 0; i < NH; i++) eng.hcol[i] = hcol[i];
  }
}

// queue a row deferred by defer_row (row r0 + lane of batch b, nnz [rp0, rp1), deg = rp1 - rp0) as segments of
// <= kSeg nnz; a row of several segments also gets a LongRow and one partial slot per segment, for the combine
__device__ __forceinline__ void push_row_segments(const SpmmParams& p, int64_t b, int64_t r0, int lane, int64_t rp0,
                                                  int64_t rp1, int deg) {
  const int nseg = (deg + kSeg - 1) / kSeg;
  const unsigned seg0 = atomicAdd(&p.counters[1], (unsigned)nseg);
  int64_t slot0 = -1;
  if (nseg > 1) {
    slot0 = atomicAdd(&p.counters[3], (unsigned)nseg);
    const unsigned lr = atomicAdd(&p.counters[2], 1u);
    if ((int64_t)lr < p.long_cap) {
      LongRow L;
      L.row_b = b * p.M + r0 + lane;
      L.first_slot = slot0;
      L.nseg_count = ((int64_t)nseg << 40) | (int64_t)deg;
      p.longs[lr] = L;
    }
  }
  for (int sgi = 0; sgi < nseg; sgi++) {
    if ((int64_t)seg0 + sgi < p.seg_cap) {
      Segment S;
      S.row_b = b * p.M + r0 + lane;
      S.start = rp0 + (int64_t)sgi * kSeg;
      S.end = min(rp1, S.start + kSeg);
      S.slot = slot0 < 0 ? -1 : slot0 + sgi;
      p.segs[seg0 + sgi] = S;
    }
  }
}

// ---- the front of a main kernel's work items ------------------------------------------------------
// A warp takes tickets from p.counters[0]; start() takes the next one as an item starts, so that the atomic's latency
// hides behind the item. Ticket t is row block t % nblk of batch b = t / nblk: rows [r0, r0 + nrows), 2^item_shift of
// them but fewer at the end. Lane l holds the nnz range [rp0, rp1) of row r0 + l (lanes >= nrows: the item's end).
//   for (WorkItem it(p, lane); it.start(p, lane); it.advance()) { ... }
struct WorkItem {
  int item_rows;
  int64_t nblk, n_items;
  unsigned int ticket, next_ticket;
  int64_t b, r0, rp0, rp1;
  int nrows;

  __device__ __forceinline__ WorkItem(const SpmmParams& p, int lane) {
    item_rows = 1 << p.item_shift;
    nblk = (p.M + item_rows - 1) >> p.item_shift;
    n_items = nblk * p.B;
    ticket = __shfl_sync(0xffffffffu, take_ticket(&p.counters[0], lane), 0);
  }
  __device__ __forceinline__ bool start(const SpmmParams& p, int lane) {
    if ((int64_t)ticket >= n_items) return false;
    next_ticket = take_ticket(&p.counters[0], lane);
    b = ticket / nblk;
    r0 = (ticket - b * nblk) << p.item_shift;
    nrows = (int)min((int64_t)item_rows, p.M - r0);
    rp0 = __ldg(p.rowptr + r0 + min(lane, nrows));
    rp1 = __ldg(p.rowptr + r0 + min(lane + 1, nrows));
    return true;
  }
  __device__ __forceinline__ void advance() { ticket = __shfl_sync(0xffffffffu, next_ticket, 0); }
  // planned kernels: the item's rows in the segment list, bit r of plan_mask[r / 32], clipped to nrows
  __device__ __forceinline__ unsigned plan_defer_mask(const SpmmParams& p) const {
    const uint32_t w = __ldg(p.plan_mask + (r0 >> 5));
    return (w >> (r0 & 31)) & (nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u));
  }
};

// ---- a lane's columns in the row-per-warp kernels ---------------------------------------------------
// Chunk ch of lane li starts at column k0 + (ch * LPR + li) * VEC; col_ok[ch]: it lies inside the row. row_bytes is
// one dense row, lane_off the byte offset of the lane's first column in it, hcol (HEADS) the head of each chunk.
template <typename X, int LPR, int VEC, int CH, bool HEADS>
__device__ __forceinline__ void lane_cols(const SpmmParams& p, int li, bool (&col_ok)[CH], int (&hcol)[HEADS ? CH : 1],
                                          uint32_t& row_bytes, int64_t& lane_off) {
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = p.k0 + (ch * LPR + li) * VEC < p.K;
  head_cols<HEADS, LPR, VEC, CH>(hcol, p, li);
  row_bytes = (uint32_t)(p.K * (int64_t)sizeof(X));
  lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(X);
}

// walk segment S (of batch b; B == 1 in the planned drain) with the row engine eng, which then holds the segment's
// result in every lane group. The segment kernel and the planned drain both walk segments here, which is what makes
// planned and unplanned products agree on the rows they defer. Each finishes a segment itself, in its own branch
// order (the order decides their machine code): the row store for a whole row, else the fp32 partial.
template <bool HEADS, typename Eng, typename T, int CH, int NH>
__device__ __forceinline__ void walk_segment(Eng& eng, const SpmmParams& p, const Segment& S, int64_t b,
                                             IndexRing<T>& ring, const bool (&col_ok)[CH], const int (&hcol)[NH],
                                             uint32_t row_bytes, int64_t lane_off, int lane, int g, uint64_t pol) {
  const int64_t base = S.start & ~(int64_t)31;
  ring.reset(base, S.end);
  const char* matb = (const char*)p.mat + b * p.N * (int64_t)row_bytes + lane_off;
  asm volatile("" : "+l"(matb));
  eng.init();
  set_scale(eng, p);
  set_heads<HEADS>(eng, p, hcol);
  eng.accumulate(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, pol);
  eng.reduce_groups();
}

struct PlanLayout {
  size_t header, mask, segs, seg_lr, longs, total;
  int64_t seg_cap, long_cap;
};
static inline PlanLayout plan_layout(int64_t M, int64_t E) {
  PlanLayout L;
  const WsLayout W = ws_layout(1, 1, E, false, false);
  L.seg_cap = W.seg_cap;
  L.long_cap = W.long_cap;
  size_t off = 0;
  L.header = off; off += 256;
  L.mask = off; off += align_up((size_t)((M + 31) / 32 + 1) * 4, 256);
  L.segs = off; off += align_up((size_t)L.seg_cap * sizeof(Segment), 256);
  L.seg_lr = off; off += align_up((size_t)L.seg_cap * 4, 256);
  L.longs = off; off += align_up((size_t)L.long_cap * sizeof(LongRow), 256);
  L.total = off;
  return L;
}
struct PlannedWs {
  size_t counters, long_done, part_val, part_arg, total;
};
static inline PlannedWs planned_ws(int64_t K, int64_t n_long, int64_t n_slot, bool arg) {
  PlannedWs L;
  size_t off = 0;
  L.counters = off; off += 256;
  L.long_done = off; off += align_up((size_t)(n_long > 0 ? n_long : 1) * 4, 256);
  L.part_val = off; off += align_up((size_t)(n_slot > 0 ? n_slot : 1) * (size_t)K * sizeof(float), 256);
  L.part_arg = off; off += arg ? align_up((size_t)(n_slot > 0 ? n_slot : 1) * (size_t)K * sizeof(int64_t), 256) : 0;
  L.total = off;
  return L;
}
// checks a plan of p.M rows and p.E nnz (tsb200_spmm_plan, with its counts) and its planned workspace, then binds
// both to p: 0 or the error code
static inline int bind_plan(SpmmParams& p, const void* plan, size_t plan_bytes, int64_t n_seg, int64_t n_long,
                     int64_t n_slot, void* workspace, size_t workspace_bytes, bool arg) {
  const PlanLayout PL = plan_layout(p.M, p.E);
  if (plan_bytes < PL.total) return TSB200_ERR_WORKSPACE;
  if (n_seg > PL.seg_cap || n_long > PL.long_cap || ((uintptr_t)plan & 255)) return TSB200_ERR_INVALID_ARG;
  const PlannedWs W = planned_ws(p.K, n_long, n_slot, arg);
  if (!workspace || workspace_bytes < W.total) return TSB200_ERR_WORKSPACE;
  if ((uintptr_t)workspace & 255) return TSB200_ERR_INVALID_ARG;
  char* ws = (char*)workspace;
  const char* pl = (const char*)plan;
  p.counters = (unsigned int*)(ws + W.counters);
  p.long_done = (uint32_t*)(ws + W.long_done);   // directly behind the counters: one memset clears both
  p.segs = (Segment*)(pl + PL.segs);
  p.longs = (LongRow*)(pl + PL.longs);
  p.seg_lr = (const uint32_t*)(pl + PL.seg_lr);
  p.plan_mask = (const uint32_t*)(pl + PL.mask);
  p.n_seg = n_seg; p.n_long = n_long;
  p.part_val = ws + W.part_val;
  p.part_arg = arg ? (int64_t*)(ws + W.part_arg) : nullptr;
  p.seg_cap = PL.seg_cap; p.long_cap = PL.long_cap; p.slot_cap = n_slot;
  return 0;
}
// a plan and its planned workspace, or else an unplanned workspace: 0 or the error code
static inline int bind_workspace(SpmmParams& p, const void* plan, size_t plan_bytes, int64_t n_seg, int64_t n_long,
                          int64_t n_slot, void* workspace, size_t workspace_bytes, bool arg) {
  return plan ? bind_plan(p, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, arg)
              : bind_unplanned(p, workspace, workspace_bytes, arg);
}

__device__ __forceinline__ void long_row_counts(const LongRow& L, int& nseg, int64_t& count) {
  nseg = (int)(L.nseg_count >> 40);
  count = L.nseg_count & (((int64_t)1 << 40) - 1);
}

}  // namespace tsb
