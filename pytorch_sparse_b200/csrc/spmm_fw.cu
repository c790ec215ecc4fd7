// spmm_fw.cu — CSR SpMM forward for sm_90a.
//
// Replaces spmm_fw -> spmm_cpu / spmm_cuda of the reference
// (csrc/spmm.cpp:22-35, csrc/cpu/spmm_cpu.cpp:8-101, csrc/cuda/spmm_cuda.cu:13-155).
//
// Design (row-split CSR, HBM/L2-gather bound; see DESIGN.md §SpMM):
//   * work item = 32 consecutive rows, pulled by a WARP from a global atomic counter
//     (persistent grid: every SM x resident CTAs);
//   * the item's rowptr slice lives in lane registers (one coalesced 264 B read);
//   * col/value of the item's contiguous nnz range stream through a per-warp shared-memory
//     ring filled by cp.async (LDGSTS) 32-entry windows, issued 2 windows ahead of use, so the
//     index stream is read exactly once, fully coalesced, and never stalls the gathers;
//   * the dense operand is gathered with 128-bit loads: LPR lanes x 16 B cover one row of
//     `mat` (CH chunks if a row is wider than 512 B); the 32/LPR lane groups of a warp work on
//     different nnz of the same row, U gathers in flight per lane; fp32 accumulation;
//   * groups are combined with __shfl_xor, consecutive lanes own consecutive 16 B column
//     vectors => fully coalesced 128-bit streaming stores;
//   * load balance for power-law rows: rows longer than LONG_T nnz and rows beyond an
//     item's nnz budget are deferred into a device-side segment queue (<= SEG nnz each); a
//     second kernel runs one warp per segment, a third combines multi-segment rows in
//     segment order (deterministic; min/max keep the smallest-e tie-break).
//   * the dense operand may be FP8 (e4m3, tsb200_spmm_fw_fp8): the same kernels with the dense type X split from the
//     value / output type T; 16 columns per 128-bit gather, each entry weighted by value * scale[col], fp32 min/max;
//   * anything the vector path cannot take (K*sizeof(T) % 16 != 0, integer / fp64 types,
//     unaligned pointers, E >= 2^31) goes to a generic lane-per-column kernel that walks the
//     nnz sequentially exactly like csrc/cpu/spmm_cpu.cpp:75-88 (bit-identical for fp32/fp64).
#include "spmm_common.cuh"

namespace tsb {

// arg_out of one column from an engine's arg slot (0x7fffffff: no entry won): the winner's nnz index, or the sentinel
// E. A row store passes E itself for an empty row (`count > 0 ? stored_arg(..) : E`); with that test in here the
// compiler lays the stores out differently.
__device__ __forceinline__ int64_t stored_arg(int a, int64_t E) { return a != 0x7fffffff ? (int64_t)a : E; }
// the VEC arg slots of one chunk of a row of degree count, as longlong2 pairs streamed to arg_row (every row store)
template <int VEC>
__device__ __forceinline__ void store_args(int64_t* __restrict__ arg_row, const int* arg, int64_t count, int64_t E) {
#pragma unroll
  for (int i = 0; i < VEC; i += 2) {
    longlong2 a2;
    a2.x = count > 0 ? stored_arg(arg[i], E) : E;
    a2.y = count > 0 ? stored_arg(arg[i + 1], E) : E;
    stg128_stream(arg_row + i, *reinterpret_cast<uint4*>(&a2));
  }
}

// T = value / output type, X = dense-operand type: T itself, or __nv_fp8_e4m3 (tsb200_spmm_fw_fp8), in which case
// every entry's weight is fl32(value * scale[col]) and a 16-byte gather carries 16 columns.
// HEADS (tsb200_spmm_heads, sum only): the value is [E, heads] and a 16-byte chunk lies inside one head, so the lane
// weighs chunk ch of entry e by hval[e * heads + hcol[ch]], loaded next to the column word instead of the ring's value.
template <typename T, int RED, int LPR, int CH, int U, typename X = T, bool HEADS = false> struct RowEngine {
  using V = Vec<T>;
  static constexpr bool Q8 = !std::is_same<X, T>::value;
  static constexpr int VEC = Vec<X>::VEC;
  static constexpr int G = 32 / LPR;
  static constexpr int NA = VEC * CH;
  static constexpr bool ARG = (RED == R_MIN || RED == R_MAX);

  float acc[NA];
  int arg[ARG ? NA : 1];
  const float* scale;  // Q8 only
  uint32_t sstride;
  const T* hval;       // HEADS only
  int heads;
  int hcol[HEADS ? CH : 1];

  __device__ __forceinline__ float acc_float(int i) const { return acc[i]; }

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < NA; i++) {
      if (RED == R_MIN) acc[i] = Traits<T>::to_acc(Traits<T>::highest());
      else if (RED == R_MAX) acc[i] = Traits<T>::to_acc(Traits<T>::lowest());
      else acc[i] = 0.f;
    }
    if (ARG) {
#pragma unroll
      for (int i = 0; i < NA; i++) arg[i] = 0x7fffffff;
    }
  }

  // one step of the min/max update (compare on the product rounded to the storage type); vf = the entry's weight
  __device__ __forceinline__ void minmax_step(float* a, int* ar, float vf, const uint4& d, int jabs) {
    float f[VEC];
    Vec<X>::unpack(d, f);
#pragma unroll
    for (int i = 0; i < VEC; i++) {
      const float p = V::round_prod(vf * f[i]);  // v == 1 when has_value=false => p == f
      const bool better = (RED == R_MIN) ? (p < a[i]) : (p > a[i]);
      if (better) {
        a[i] = p;
        ar[i] = jabs;
      }
    }
  }

  // scale of the dense row an entry gathers (fp8 operand); stride 0 reads one value for the whole operand
  __device__ __forceinline__ float row_scale(uint32_t c) const { return __ldg(scale + (size_t)c * sstride); }

  // one gathered vector of one entry: v = raw value, s = its dense row's scale (Q8), d = the 16 bytes
  __device__ __forceinline__ void step(int ch, typename V::vraw v, float s, const uint4& d, int jabs) {
    if constexpr (RED == R_SUM) {
      if constexpr (Q8) {
        const float w = V::vfloat(v) * s;
        float f[VEC];
        Vec<X>::unpack(d, f);
#pragma unroll
        for (int i = 0; i < VEC; i++) acc[ch * VEC + i] = fmaf(w, f[i], acc[ch * VEC + i]);
      } else {
        V::fma(&acc[ch * VEC], v, d);
      }
    } else {
      minmax_step(&acc[ch * VEC], &arg[ch * VEC], Q8 ? V::vfloat(v) * s : V::vfloat(v), d, jabs);
    }
  }

  // accumulate ring-relative nnz [s, e) of one row. `matb` points at this lane's first column of
  // batch b. The row is walked in chunks of up to U steps (a step = G nnz, one per lane group);
  // every step of a chunk issues its 128-bit gather before the first FMA of the chunk. Full chunks
  // take an unpredicated path; the (warp-uniform) step count of the last chunk is honoured exactly
  // with early exits — no padded work. Thanks to the ring mirror the <= 32 entries of a chunk are
  // contiguous in shared memory: one base pointer, immediate offsets.
  __device__ __forceinline__ void accumulate(IndexRing<T>& ring, int s, int e,
                                             const char* __restrict__ matb, uint32_t row_bytes,
                                             const bool (&col_ok)[CH], int lane, int g, uint64_t pol) {
    using VR = typename V::vraw;
    for (int j0 = s; j0 < e; j0 += U * G) {
      const int jend = min(e, j0 + U * G);
      ring.ensure(j0, jend, lane);
      const int slot0 = (j0 + g) & (kRing - 1);
      const uint32_t* pc = reinterpret_cast<const uint32_t*>(ring.s_col + slot0);  // low words (N < 2^32)
      const VR* pv = reinterpret_cast<const VR*>(ring.s_val) + slot0;
      const int jabs0 = (int)ring.base + j0 + g;  // absolute nnz index of step 0 (E < 2^31)
      uint4 d[U][CH];
      VR v[U];
      VR hv[HEADS ? U : 1][HEADS ? CH : 1];
      float sc[U];
      if (jend - j0 == U * G) {  // full chunk: every lane group has work in every step
#pragma unroll
        for (int u = 0; u < U; u++) {
          const uint32_t c = pc[2 * u * G];
          if constexpr (!HEADS) v[u] = pv[u * G];
          const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (col_ok[ch]) d[u][ch] = ldg128_hint(src + ch * (LPR * 16), pol);
            if constexpr (HEADS)
              if (col_ok[ch]) hv[u][ch] = load_vraw<T>(hval + (int64_t)(jabs0 + u * G) * heads + hcol[ch]);
          }
          if constexpr (Q8) sc[u] = row_scale(c);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (!col_ok[ch]) continue;
            if constexpr (HEADS) step(ch, hv[u][ch], 1.f, d[u][ch], jabs0 + u * G);
            else step(ch, v[u], Q8 ? sc[u] : 1.f, d[u][ch], jabs0 + u * G);
          }
        }
      } else {
        const int nst = (jend - j0 + G - 1) / G;  // steps in this chunk, 1..U (warp-uniform)
        const int jrel = jend - j0 - g;            // lane group g is active in step u iff u*G < jrel
        bool act[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (u >= nst) break;
          act[u] = u * G < jrel;
          const uint32_t c = pc[2 * u * G];
          if constexpr (!HEADS) v[u] = pv[u * G];
          const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (act[u] && col_ok[ch]) d[u][ch] = ldg128_hint(src + ch * (LPR * 16), pol);
            if constexpr (HEADS)
              if (act[u] && col_ok[ch]) hv[u][ch] = load_vraw<T>(hval + (int64_t)(jabs0 + u * G) * heads + hcol[ch]);
          }
          if constexpr (Q8) sc[u] = act[u] ? row_scale(c) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (u >= nst) break;
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (!(act[u] && col_ok[ch])) continue;
            if constexpr (HEADS) step(ch, hv[u][ch], 1.f, d[u][ch], jabs0 + u * G);
            else step(ch, v[u], Q8 ? sc[u] : 1.f, d[u][ch], jabs0 + u * G);
          }
        }
      }
    }
  }

  // combine the G lane groups; afterwards every group holds the row result.
  __device__ __forceinline__ void reduce_groups() {
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
#pragma unroll
      for (int i = 0; i < NA; i++) {
        const float ov = __shfl_xor_sync(0xffffffffu, acc[i], off);
        if (RED == R_SUM) {
          acc[i] += ov;
        } else {
          const int oa = __shfl_xor_sync(0xffffffffu, arg[i], off);
          const bool better = (RED == R_MIN) ? (ov < acc[i]) : (ov > acc[i]);
          if (better || (ov == acc[i] && oa < arg[i])) {
            acc[i] = ov;
            arg[i] = oa;
          }
        }
      }
    }
  }

  // final write of one row (group 0 lanes). count = row degree. RES: res_row is the row's residual (element type X)
  // at this launch's first column and rs its scale; the lane adds its VEC residual columns per chunk after the mean's
  // division.
  template <bool RES = false>
  __device__ __forceinline__ void store_row(T* __restrict__ out_row, int64_t* __restrict__ arg_row,
                                            int64_t count, int64_t E, const bool (&col_ok)[CH], int li,
                                            bool mean, float* __restrict__ part_row = nullptr, int acc_mode = 0,
                                            const typename ResElem<X>::raw* __restrict__ res_row = nullptr,
                                            float rs = 0.f) {
    static_assert(!RES || RED == R_SUM, "residual: sum / mean");
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      float f[VEC];
#pragma unroll
      for (int i = 0; i < VEC; i++) {
        float a = acc[ch * VEC + i];
        if (RED == R_SUM && mean) a = a / (float)(count > 0 ? count : 1);
        if (ARG && count == 0) a = 0.f;
        f[i] = a;
      }
      const int koff = (ch * LPR + li) * VEC;
      if constexpr (RES) res_add_vec<X>(f, res_row + koff, rs);
      if (RED == R_SUM && acc_mode) {  // column-block pipelining: fp32 partial shared by the launches of one product
        float4* pr = reinterpret_cast<float4*>(part_row + koff);
        if (acc_mode != 1) {
#pragma unroll
          for (int i = 0; i < VEC; i += 4) {
            const float4 q = pr[i >> 2];
            f[i] += q.x; f[i + 1] += q.y; f[i + 2] += q.z; f[i + 3] += q.w;
          }
        }
        if (acc_mode != 3) {
#pragma unroll
          for (int i = 0; i < VEC; i += 4) pr[i >> 2] = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
          continue;
        }
      }
#pragma unroll
      for (int i = 0; i < VEC; i += V::VEC) stg128_stream(out_row + koff + i, V::pack(f + i));  // 2-4 stores for Q8
      if (ARG) store_args<VEC>(arg_row + koff, &arg[ch * VEC], count, E);
    }
  }

  // final write of one row as e4m3 with its own scale (tsb200_spmm_fw_fp8_quant; T = float, one column tile). Called
  // by all LPR lanes that hold the row (group 0 of a row-per-warp kernel, a row's own group in the group-per-row
  // kernel): the row's amax is a shuffle over exactly those lanes, then every lane writes its 16 bytes per chunk.
  // RES: the residual is added (as in store_row) before the row amax.
  template <bool RES = false>
  __device__ __forceinline__ void store_row_q8(uint8_t* __restrict__ out_row, float* __restrict__ scale_out,
                                               int64_t* __restrict__ arg_row, int64_t count, int64_t E,
                                               const bool (&col_ok)[CH], int li, bool mean,
                                               const uint8_t* __restrict__ res_row = nullptr, float rs = 0.f) {
    static_assert(VEC == 16 && std::is_same<T, float>::value, "e4m3 result: fp8 operand, fp32 accumulation");
    static_assert(!RES || RED == R_SUM, "residual: sum / mean");
    float amax = 0.f;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
#pragma unroll
      for (int i = 0; i < VEC; i++) {
        float a = acc[ch * VEC + i];
        if (RED == R_SUM && mean) a = a / (float)(count > 0 ? count : 1);
        if (ARG && count == 0) a = 0.f;
        acc[ch * VEC + i] = a;
        if constexpr (!RES) amax = amax_nan(amax, fabsf(a));
      }
      if constexpr (RES) {
        res_add_vec<X>(&acc[ch * VEC], res_row + (ch * LPR + li) * VEC, rs);
#pragma unroll
        for (int i = 0; i < VEC; i++) amax = amax_nan(amax, fabsf(acc[ch * VEC + i]));
      }
    }
    const unsigned gmask = LPR == 32 ? 0xffffffffu : (((1u << LPR) - 1u) << ((threadIdx.x & 31) & ~(LPR - 1)));
#pragma unroll
    for (int off = 1; off < LPR; off <<= 1) amax = amax_nan(amax, __shfl_xor_sync(gmask, amax, off));
    const float s = e4m3_row_scale(amax);
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
      stg128_stream(out_row + koff, e4m3_pack16(&acc[ch * VEC], s));
      if (ARG) store_args<VEC>(arg_row + koff, &arg[ch * VEC], count, E);
    }
    if (li == 0) *scale_out = s;
  }
};

// ---- packed 16-bit min/max engine --------------------------------------------------------------
// For bf16 / f16 the reference compares products ROUNDED to the storage type, so the whole min/max
// recurrence can stay in packed 16-bit pairs: HMUL2 (round-to-nearest product of two pairs), HSETP2
// (two strict compares -> two predicates, false on NaN like the reference's `>`), and a per-half select of the
// new extreme — instead of unpack / fp32 multiply / re-round / compare / select. The extreme is selected by the
// strict compare, not formed with max.x2 / min.x2: those order -0 below +0, so a later -0 would replace a +0
// minimum (or +0 a -0 maximum) without moving arg_out. Values are bit-identical to the float path; ties still keep
// the smallest nnz index.
template <typename T> struct Pk;
template <> struct Pk<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t mul(uint32_t a, uint32_t b) {
    uint32_t r; asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
  }
  // per-half strict compare of product p against the running extreme a (false on NaN): 0xffff in each half that wins
  template <bool MAX> static __device__ __forceinline__ uint32_t better(uint32_t p, uint32_t a) {
    uint32_t m;
    if (MAX) asm("{\n\t.reg .pred q0, q1;\n\tsetp.gt.bf16x2 q0|q1, %1, %2;\n\tselp.b32 %0, 0x0000ffff, 0, q0;\n\t"
                 "@q1 or.b32 %0, %0, 0xffff0000;\n\t}" : "=r"(m) : "r"(p), "r"(a));
    else asm("{\n\t.reg .pred q0, q1;\n\tsetp.lt.bf16x2 q0|q1, %1, %2;\n\tselp.b32 %0, 0x0000ffff, 0, q0;\n\t"
             "@q1 or.b32 %0, %0, 0xffff0000;\n\t}" : "=r"(m) : "r"(p), "r"(a));
    return m;
  }
  // per-half masks: better (strict) and equal
  template <bool MAX> static __device__ __forceinline__ void cmp(uint32_t o, uint32_t m, bool& b0, bool& b1, bool& e0, bool& e1) {
    uint32_t x0, x1, y0, y1;
    if (MAX) asm("{\n\t.reg .pred q0, q1;\n\tsetp.gt.bf16x2 q0|q1, %4, %5;\n\tselp.u32 %0, 1, 0, q0;\n\tselp.u32 %1, 1, 0, q1;\n\t"
                 "setp.eq.bf16x2 q0|q1, %4, %5;\n\tselp.u32 %2, 1, 0, q0;\n\tselp.u32 %3, 1, 0, q1;\n\t}"
                 : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(o), "r"(m));
    else asm("{\n\t.reg .pred q0, q1;\n\tsetp.lt.bf16x2 q0|q1, %4, %5;\n\tselp.u32 %0, 1, 0, q0;\n\tselp.u32 %1, 1, 0, q1;\n\t"
             "setp.eq.bf16x2 q0|q1, %4, %5;\n\tselp.u32 %2, 1, 0, q0;\n\tselp.u32 %3, 1, 0, q1;\n\t}"
             : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(o), "r"(m));
    b0 = x0; b1 = x1; e0 = y0; e1 = y1;
  }
  static __device__ __forceinline__ uint32_t splat(unsigned short v) { return (uint32_t)v | ((uint32_t)v << 16); }
  static __device__ __forceinline__ float half_to_float(uint32_t w, int hi) {
    return __uint_as_float(hi ? (w & 0xffff0000u) : (w << 16));
  }
  static __device__ __forceinline__ uint32_t extreme(bool max_) { return max_ ? 0xFF7FFF7Fu : 0x7F7F7F7Fu; }  // lowest / highest
};
template <> struct Pk<__half> {
  static __device__ __forceinline__ uint32_t mul(uint32_t a, uint32_t b) {
    uint32_t r; asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
  }
  template <bool MAX> static __device__ __forceinline__ uint32_t better(uint32_t p, uint32_t a) {
    uint32_t m;
    if (MAX) asm("{\n\t.reg .pred q0, q1;\n\tsetp.gt.f16x2 q0|q1, %1, %2;\n\tselp.b32 %0, 0x0000ffff, 0, q0;\n\t"
                 "@q1 or.b32 %0, %0, 0xffff0000;\n\t}" : "=r"(m) : "r"(p), "r"(a));
    else asm("{\n\t.reg .pred q0, q1;\n\tsetp.lt.f16x2 q0|q1, %1, %2;\n\tselp.b32 %0, 0x0000ffff, 0, q0;\n\t"
             "@q1 or.b32 %0, %0, 0xffff0000;\n\t}" : "=r"(m) : "r"(p), "r"(a));
    return m;
  }
  template <bool MAX> static __device__ __forceinline__ void cmp(uint32_t o, uint32_t m, bool& b0, bool& b1, bool& e0, bool& e1) {
    uint32_t x0, x1, y0, y1;
    if (MAX) asm("{\n\t.reg .pred q0, q1;\n\tsetp.gt.f16x2 q0|q1, %4, %5;\n\tselp.u32 %0, 1, 0, q0;\n\tselp.u32 %1, 1, 0, q1;\n\t"
                 "setp.eq.f16x2 q0|q1, %4, %5;\n\tselp.u32 %2, 1, 0, q0;\n\tselp.u32 %3, 1, 0, q1;\n\t}"
                 : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(o), "r"(m));
    else asm("{\n\t.reg .pred q0, q1;\n\tsetp.lt.f16x2 q0|q1, %4, %5;\n\tselp.u32 %0, 1, 0, q0;\n\tselp.u32 %1, 1, 0, q1;\n\t"
             "setp.eq.f16x2 q0|q1, %4, %5;\n\tselp.u32 %2, 1, 0, q0;\n\tselp.u32 %3, 1, 0, q1;\n\t}"
             : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(o), "r"(m));
    b0 = x0; b1 = x1; e0 = y0; e1 = y1;
  }
  static __device__ __forceinline__ uint32_t splat(unsigned short v) { return (uint32_t)v | ((uint32_t)v << 16); }
  static __device__ __forceinline__ float half_to_float(uint32_t w, int hi) {
    return __half2float(__ushort_as_half((unsigned short)(hi ? (w >> 16) : (w & 0xffffu))));
  }
  static __device__ __forceinline__ uint32_t extreme(bool max_) { return max_ ? 0xFBFFFBFFu : 0x7BFF7BFFu; }  // -65504 / 65504
};

template <typename T, int RED, int LPR, int CH, int U> struct MinMax16Engine {
  using V = Vec<T>;
  using P = Pk<T>;
  static constexpr bool Q8 = false;
  static constexpr int VEC = 8;
  static constexpr int G = 32 / LPR;
  static constexpr int NA = VEC * CH;
  static constexpr bool ARG = true;
  static constexpr bool MAX = (RED == R_MAX);

  uint32_t pacc[NA / 2];
  int arg[NA];

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < NA / 2; i++) pacc[i] = P::extreme(MAX);
#pragma unroll
    for (int i = 0; i < NA; i++) arg[i] = 0x7fffffff;
  }
  __device__ __forceinline__ float acc_float(int i) const { return P::half_to_float(pacc[i >> 1], i & 1); }

  __device__ __forceinline__ void vec_step(int ch, unsigned short v, const uint4& d, int jabs) {
    const uint32_t v2 = P::splat(v);  // 1.0 when has_value=false => exact products
    const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint32_t p = P::mul(w[k], v2);
      const uint32_t m = P::template better<MAX>(p, pacc[ch * 4 + k]);
      if (m & 0xffffu) arg[ch * 8 + 2 * k] = jabs;
      if (m >> 16) arg[ch * 8 + 2 * k + 1] = jabs;
      pacc[ch * 4 + k] = (p & m) | (pacc[ch * 4 + k] & ~m);
    }
  }

  __device__ __forceinline__ void accumulate(IndexRing<T>& ring, int s, int e,
                                             const char* __restrict__ matb, uint32_t row_bytes,
                                             const bool (&col_ok)[CH], int lane, int g, uint64_t pol) {
    using VR = typename V::vraw;
    for (int j0 = s; j0 < e; j0 += U * G) {
      const int jend = min(e, j0 + U * G);
      ring.ensure(j0, jend, lane);
      const int slot0 = (j0 + g) & (kRing - 1);
      const uint32_t* pc = reinterpret_cast<const uint32_t*>(ring.s_col + slot0);
      const VR* pv = reinterpret_cast<const VR*>(ring.s_val) + slot0;
      const int jabs0 = (int)ring.base + j0 + g;
      const int nst = (jend - j0 + G - 1) / G;
      const int jrel = jend - j0 - g;
      uint4 d[U][CH];
      VR v[U];
      bool act[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (u >= nst) break;
        act[u] = u * G < jrel;
        const uint32_t c = pc[2 * u * G];
        v[u] = pv[u * G];
        const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
        for (int ch = 0; ch < CH; ch++)
          if (act[u] && col_ok[ch]) d[u][ch] = ldg128_hint(src + ch * (LPR * 16), pol);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (u >= nst) break;
#pragma unroll
        for (int ch = 0; ch < CH; ch++)
          if (act[u] && col_ok[ch]) vec_step(ch, v[u], d[u][ch], jabs0 + u * G);
      }
    }
  }

  __device__ __forceinline__ void reduce_groups() {
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
#pragma unroll
      for (int k = 0; k < NA / 2; k++) {
        const uint32_t o = __shfl_xor_sync(0xffffffffu, pacc[k], off);
        const int oa0 = __shfl_xor_sync(0xffffffffu, arg[2 * k], off);
        const int oa1 = __shfl_xor_sync(0xffffffffu, arg[2 * k + 1], off);
        bool b0, b1, e0, e1;
        P::template cmp<MAX>(o, pacc[k], b0, b1, e0, e1);
        const bool t0 = b0 || (e0 && oa0 < arg[2 * k]);
        const bool t1 = b1 || (e1 && oa1 < arg[2 * k + 1]);
        const uint32_t mask = (t0 ? 0x0000ffffu : 0u) | (t1 ? 0xffff0000u : 0u);
        pacc[k] = (o & mask) | (pacc[k] & ~mask);
        if (t0) arg[2 * k] = oa0;
        if (t1) arg[2 * k + 1] = oa1;
      }
    }
  }

  template <bool RES = false>  // no residual with min / max
  __device__ __forceinline__ void store_row(T* __restrict__ out_row, int64_t* __restrict__ arg_row,
                                            int64_t count, int64_t E, const bool (&col_ok)[CH], int li, bool,
                                            float* = nullptr, int = 0, const T* = nullptr, float = 0.f) {
    static_assert(!RES, "residual: sum / mean");
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
      uint4 o = make_uint4(pacc[ch * 4], pacc[ch * 4 + 1], pacc[ch * 4 + 2], pacc[ch * 4 + 3]);
      if (count == 0) o = make_uint4(0, 0, 0, 0);
      stg128_stream(out_row + koff, o);
      store_args<VEC>(arg_row + koff, &arg[ch * VEC], count, E);
    }
  }
};

// min/max over an fp8 operand compare in fp32 (the packed engine multiplies two values of the storage type)
template <typename T, int RED, int LPR, int CH, int U, typename X = T, bool HEADS = false> struct EngineFor {
  static_assert(!HEADS || (RED == R_SUM && std::is_same<X, T>::value), "per-head weights: sum over a T operand");
  using type = typename std::conditional<(RED != R_SUM && is_float16<T>::value && std::is_same<X, T>::value),
                                         MinMax16Engine<T, RED, LPR, CH, U>,
                                         RowEngine<T, RED, LPR, CH, U, X, HEADS>>::type;
};
// column kk of a multi-segment row (nseg segments, count = its degree): its partials folded in segment order (min/max:
// the smallest e wins ties), the mean's division applied. CG: read past L1 (partials written by other SMs during the
// same launch). RES: plus the row's residual (element type R, scale rs) in that column. The one definition of the fold:
// every combine of the SpMM forward calls it.
template <int RED, bool CG, bool RES = false, typename R = __nv_fp8_e4m3>
__device__ __forceinline__ float combine_col(const SpmmParams& p, const LongRow& L, int nseg, int64_t count,
                                             int64_t kk, int64_t& ar, float rs = 0.f) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const float* pv = (const float*)p.part_val;
  float a = CG ? __ldcg(pv + L.first_slot * p.K + kk) : pv[L.first_slot * p.K + kk];
  int64_t r = ARG ? (CG ? __ldcg(p.part_arg + L.first_slot * p.K + kk) : p.part_arg[L.first_slot * p.K + kk]) : 0;
  for (int sgi = 1; sgi < nseg; sgi++) {
    const float v = CG ? __ldcg(pv + (L.first_slot + sgi) * p.K + kk) : pv[(L.first_slot + sgi) * p.K + kk];
    if (RED == R_SUM) a += v;
    else {
      const int64_t va = CG ? __ldcg(p.part_arg + (L.first_slot + sgi) * p.K + kk)
                            : p.part_arg[(L.first_slot + sgi) * p.K + kk];
      const bool better = (RED == R_MIN) ? (v < a) : (v > a);
      if (better || (v == a && va < r)) { a = v; r = va; }
    }
  }
  ar = r;
  if (RED == R_SUM && p.mean) a = a / (float)(count != 0 ? count : 1);
  if constexpr (RES) a = res_add(a, rs, ResElem<R>::widen(__ldcs(res_at<R>(p, L.row_b, kk))));
  return a;
}

// combine the partials of one multi-segment row, in segment order, by ONE WARP (planned mode: the warp that finished
// the row's last segment); the partials were written by other SMs -> read them past L1. RES: plus the residual, of
// element type R.
template <typename T, int RED, bool RES = false, typename R = T>
__device__ __forceinline__ void combine_row_warp(const SpmmParams& p, const LongRow& L, int lane, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int nseg = (int)(L.nseg_count >> 40);
  const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
  const float rs = RES ? res_scale(p, L.row_b) : 0.f;
  for (int k = lane; k < kcols; k += 32) {
    const int64_t kk = p.k0 + k;
    if (kk >= p.K) break;
    int64_t ar;
    const float a = combine_col<RED, true, RES, R>(p, L, nseg, count, kk, ar, rs);
    ((T*)p.out)[L.row_b * p.K + kk] = Traits<T>::from_acc(a);
    if (ARG) p.arg_out[L.row_b * p.K + kk] = ar;
  }
}

// the same for an e4m3 result (QO): a first pass over the partials finds the row's amax, the second writes y / scale.
// RES: both passes add the residual, so the amax is taken over the values that are stored.
template <int RED, bool RES = false>
__device__ __forceinline__ void combine_row_warp_q8(const SpmmParams& p, const LongRow& L, int lane, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int nseg = (int)(L.nseg_count >> 40);
  const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
  const float rs = RES ? res_scale(p, L.row_b) : 0.f;
  float amax = 0.f;
  for (int k = lane; k < kcols; k += 32) {
    const int64_t kk = p.k0 + k;
    if (kk >= p.K) break;
    int64_t ar;
    amax = amax_nan(amax, fabsf(combine_col<RED, true, RES>(p, L, nseg, count, kk, ar, rs)));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = amax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  const float s = e4m3_row_scale(amax);
  if (lane == 0) p.out_scale[L.row_b] = s;
  for (int k = lane; k < kcols; k += 32) {
    const int64_t kk = p.k0 + k;
    if (kk >= p.K) break;
    int64_t ar;
    const float a = combine_col<RED, true, RES>(p, L, nseg, count, kk, ar, rs);
    ((uint8_t*)p.out)[L.row_b * p.K + kk] = e4m3_quant(a, s);
    if (ARG) p.arg_out[L.row_b * p.K + kk] = ar;
  }
}

// the fp32 partial of one segment of a multi-segment row, and its arg slots (min / max), into partial slot `slot`;
// written by group 0 after reduce_groups
template <int LPR, typename Eng, int CH>
__device__ __forceinline__ void store_partial(const SpmmParams& p, const Eng& eng, int64_t slot,
                                              const bool (&col_ok)[CH], int li) {
  constexpr int VEC = Eng::VEC;
  float* pv = (float*)p.part_val + slot * p.K + p.k0;
  int64_t* pa = Eng::ARG ? p.part_arg + slot * p.K + p.k0 : nullptr;
#pragma unroll
  for (int ch = 0; ch < CH; ch++) {
    if (!col_ok[ch]) continue;
    const int koff = (ch * LPR + li) * VEC;
#pragma unroll
    for (int i = 0; i < VEC; i++) {
      pv[koff + i] = eng.acc_float(ch * VEC + i);
      if (Eng::ARG) pa[koff + i] = stored_arg(eng.arg[ch * VEC + i], p.E);
    }
  }
}

// Where the final stores of rows r0 + rl of batch b go (T result: `out`, the ACC partial and arg_out, at column k0;
// QO: an e4m3 result, B == 1, one column tile). The two main kernels make one per work item, next to the gather base.
// store() is their final row store: the engine's store_row, or store_row_q8 for QO, called by the lanes that hold the
// row. The segment kernel and the planned drain store a whole-row segment with their own copy of the call: through
// RowOut the compiler orders their instructions differently (the e4m3-result min/max ones need more registers).
template <typename T, bool ACC, bool QO, bool RES, typename X> struct RowOut {
  T* outb;
  int64_t* argb;
  float* partb;
  int64_t r0;

  __device__ __forceinline__ RowOut(const SpmmParams& p, int64_t b, int64_t r0_) : r0(r0_) {
    outb = (T*)p.out + (b * p.M + r0) * p.K + p.k0;
    argb = p.arg_out ? p.arg_out + (b * p.M + r0) * p.K + p.k0 : nullptr;
    partb = ACC ? p.partial + (b * p.M + r0) * p.K + p.k0 : nullptr;
  }
  template <typename Eng, int CH>
  __device__ __forceinline__ void store(Eng& eng, const SpmmParams& p, int rl, int64_t count,
                                        const bool (&col_ok)[CH], int li) const {
    if constexpr (QO)
      eng.template store_row_q8<RES>((uint8_t*)p.out + (r0 + rl) * p.K, p.out_scale + r0 + rl,
                                     argb ? argb + (int64_t)rl * p.K : nullptr, count, p.E, col_ok, li, p.mean != 0,
                                     RES ? res_row<X>(p, r0 + rl) : nullptr, RES ? res_scale(p, r0 + rl) : 0.f);
    else
      eng.template store_row<RES>(outb + (int64_t)rl * p.K, argb ? argb + (int64_t)rl * p.K : nullptr, count, p.E,
                                  col_ok, li, p.mean != 0, ACC ? partb + (int64_t)rl * p.K : nullptr,
                                  ACC ? p.acc_mode : 0, RES ? res_row<X>(p, r0 + rl) : nullptr,
                                  RES ? res_scale(p, r0 + rl) : 0.f);
  }
};

// QO: e4m3 result with per-row scales (RowEngine::store_row_q8) instead of T. RES: plus an e4m3 residual per row.
// HEADS: per-head weights (tsb200_spmm_heads); the ring then streams the column words only.
template <typename T, int RED, int LPR, int CH, int U, int MINB, bool ACC = false, bool PLAN = false, typename X = T,
          bool QO = false, bool RES = false, bool HEADS = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_vec_kernel(const SpmmParams p) {
  using Eng = typename EngineFor<T, RED, LPR, CH, U, X, HEADS>::type;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.template bind<!HEADS>(p, s_col[warp], s_val[warp], lane);
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
  int hcol[HEADS ? CH : 1];
  uint32_t row_bytes;
  int64_t lane_off;
  lane_cols<X, LPR, VEC, CH, HEADS>(p, li, col_ok, hcol, row_bytes, lane_off);

  for (WorkItem it(p, lane); it.start(p, lane); it.advance()) {
    const int64_t a0 = __shfl_sync(0xffffffffu, it.rp0, 0);
    const int64_t base = a0 & ~(int64_t)31;
    const int s_rel = (int)(it.rp0 - base), e_rel = (int)(it.rp1 - base);
    const int deg = e_rel - s_rel;

    unsigned defer_mask;
    if constexpr (PLAN) {  // which rows are in the segment list was decided when the plan was built
      defer_mask = it.plan_defer_mask(p);
    } else {
      const bool defer = defer_row(deg, lane);
      defer_mask = __ballot_sync(0xffffffffu, defer);
      if (defer) push_row_segments(p, it.b, it.r0, lane, it.rp0, it.rp1, deg);  // rare
    }
    __syncwarp();

    ring.reset(base, __shfl_sync(0xffffffffu, it.rp1, 31));  // lanes >= nrows hold the item's end
    const char* matb = (const char*)p.mat + it.b * p.N * (int64_t)row_bytes + lane_off;
    asm volatile("" : "+l"(matb));  // keep the gather base in a register
    const RowOut<T, ACC, QO, RES, X> ro(p, it.b, it.r0);

    for (int rl = 0; rl < it.nrows; rl++) {
      if ((defer_mask >> rl) & 1u) continue;
      const int s = __shfl_sync(0xffffffffu, s_rel, rl);
      const int e = __shfl_sync(0xffffffffu, e_rel, rl);
      Eng eng;
      eng.init();
      set_scale(eng, p);
      set_heads<HEADS>(eng, p, hcol);
      eng.accumulate(ring, s, e, matb, row_bytes, col_ok, lane, g, pol);
      eng.reduce_groups();
      if (g == 0) ro.store(eng, p, rl, e - s, col_ok, li);
    }
  }

  if constexpr (PLAN) {
    // Planned mode: the row items are gone — this warp now takes segments of the long / over-budget rows from the
    // plan's list (all of them exist already: a ticket counter is the whole protocol). A multi-segment row is
    // combined by whichever warp finishes its last segment (counter per long row + fences, no waiting).
    constexpr int kcols = LPR * CH * VEC;
    while (true) {
      const unsigned int sidx = __shfl_sync(0xffffffffu, take_ticket(&p.counters[5], lane), 0);
      if ((int64_t)sidx >= p.n_seg) break;
      const Segment S = p.segs[sidx];
      const int64_t row = S.row_b;  // B == 1
      Eng eng;
      walk_segment<HEADS>(eng, p, S, 0, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
      if (S.slot < 0) {
        if constexpr (QO) {
          if (g == 0)
            eng.template store_row_q8<RES>((uint8_t*)p.out + row * p.K, p.out_scale + row,
                                           p.arg_out ? p.arg_out + row * p.K : nullptr, S.end - S.start, p.E, col_ok,
                                           li, p.mean != 0, RES ? res_row<X>(p, row) : nullptr,
                                           RES ? res_scale(p, row) : 0.f);
        } else {
          if (g == 0)
            eng.template store_row<RES>((T*)p.out + row * p.K + p.k0,
                                        p.arg_out ? p.arg_out + row * p.K + p.k0 : nullptr, S.end - S.start, p.E,
                                        col_ok, li, p.mean != 0, nullptr, 0, RES ? res_row<X>(p, row) : nullptr,
                                        RES ? res_scale(p, row) : 0.f);
        }
      } else {
        if (g == 0) store_partial<LPR>(p, eng, S.slot, col_ok, li);
        __syncwarp();
        __threadfence();  // this segment's partial is visible before its completion is counted
        const uint32_t lr = __ldg(p.seg_lr + sidx);
        unsigned int finished = 0;
        if (lane == 0) finished = atomicAdd(&p.long_done[lr], 1u);
        finished = __shfl_sync(0xffffffffu, finished, 0);
        const LongRow L = p.longs[lr];
        if ((int)finished == (int)(L.nseg_count >> 40) - 1) {
          __threadfence();
          if constexpr (QO) combine_row_warp_q8<RED, RES>(p, L, lane, kcols);
          else combine_row_warp<T, RED, RES, X>(p, L, lane, kcols);
        }
      }
      __syncwarp();
    }
  }
}

// ---- narrow dense rows (K*sizeof(T) <= 128 B): group-per-row SUM kernel ----------------------------
// With LPR <= 8 a row-at-a-time warp spends most of its instructions on per-row bookkeeping and on the
// cross-group reduction (the kernel becomes issue-bound). Here the G = 32/LPR lane groups of a warp each walk their OWN row: no cross-group
// reduction, per-row overhead amortised over G rows, U independent (index -> gather) chains in flight
// per lane. Indices are read straight from global memory (lanes of a group broadcast one address,
// consecutive nnz hit L1). Long rows / budget overflow still go to the segment queue.

// HEADS: the weight of entry j for this lane's chunk is val[j * heads + hcol], loaded in place of val[j].
template <typename T, int RED, int LPR, int U, int MINB, bool ACC = false, bool PLAN = false, typename X = T,
          bool QO = false, bool RES = false, bool HEADS = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_gpr_kernel(const SpmmParams p) {
  using V = Vec<T>;
  using Eng = typename EngineFor<T, RED, LPR, 1, U, X, HEADS>::type;  // per-lane state + update + store of one row
  using VR = typename V::vraw;
  constexpr int VEC = Eng::VEC;
  constexpr bool Q8 = Eng::Q8;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  const bool col_ok = p.k0 + li * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(X));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(X);
  const uint64_t pol = make_policy_evict_last();
  const T* __restrict__ val = (const T*)p.value;
  const bool has_val = val != nullptr;
  int hcol[1];
  head_cols<HEADS, LPR, VEC, 1>(hcol, p, li);
  const int hstride = HEADS ? p.heads : 1;  // value elements per entry

  for (WorkItem it(p, lane); it.start(p, lane); it.advance()) {
    const int64_t base = __shfl_sync(0xffffffffu, it.rp0, 0);
    const int s_rel = (int)(it.rp0 - base), e_rel = (int)(it.rp1 - base);
    const int deg = e_rel - s_rel;

    unsigned defer_mask;
    if constexpr (PLAN) {
      defer_mask = it.plan_defer_mask(p);
    } else {
      const bool defer = defer_row(deg, lane);
      defer_mask = __ballot_sync(0xffffffffu, defer);
      if (defer) push_row_segments(p, it.b, it.r0, lane, it.rp0, it.rp1, deg);
    }
    __syncwarp();

    const char* matb = (const char*)p.mat + it.b * p.N * (int64_t)row_bytes + lane_off;
    asm volatile("" : "+l"(matb));
    const int64_t* __restrict__ colb = p.col + base;
    const T* __restrict__ valb = has_val ? (HEADS ? val + base * hstride + hcol[0] : val + base) : nullptr;
    const RowOut<T, ACC, QO, RES, X> ro(p, it.b, it.r0);
    const bool col_ok_arr[1] = {col_ok};
    const int jbase = (int)base;  // absolute nnz index of ring-relative 0 (E < 2^31)

    for (int t = 0; t < it.nrows; t += G) {
      const int rl = t + g;  // this lane group's row
      int s = __shfl_sync(0xffffffffu, s_rel, rl & 31);
      int e = __shfl_sync(0xffffffffu, e_rel, rl & 31);
      const bool mine = rl < it.nrows && !((defer_mask >> (rl & 31)) & 1u);
      if (!mine) e = s;
      const int len = e - s;
      int maxlen = len;
#pragma unroll
      for (int off = LPR; off < 32; off <<= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, off));

      Eng eng;
      eng.init();
      set_scale(eng, p);
      // software pipeline: the (col, value) pairs of chunk k+1 are loaded while chunk k's gathers fly
      uint32_t cn[U];
      VR vn[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        cn[u] = 0;
        vn[u] = V::one();
        if (u < len) {
          cn[u] = (uint32_t)__ldg(colb + s + u);
          if constexpr (HEADS) {
            if (col_ok) vn[u] = load_vraw<T>(valb + (int64_t)(s + u) * hstride);
          } else {
            if (has_val) vn[u] = load_vraw<T>(valb + s + u);
          }
        }
      }
      for (int j0 = 0; j0 < maxlen; j0 += U) {
        uint4 d[U];
        VR v[U];
        float sc[U];
        bool act[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          act[u] = (j0 + u < len) && col_ok;
          v[u] = vn[u];
          if (act[u]) d[u] = ldg128_hint(matb + (uint64_t)cn[u] * row_bytes, pol);
          if constexpr (Q8) sc[u] = act[u] ? eng.row_scale(cn[u]) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int jn = j0 + U + u;
          if (jn < len) {
            cn[u] = (uint32_t)__ldg(colb + s + jn);
            if constexpr (HEADS) {
              if (col_ok) vn[u] = load_vraw<T>(valb + (int64_t)(s + jn) * hstride);
            } else {
              if (has_val) vn[u] = load_vraw<T>(valb + s + jn);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (!act[u]) continue;
          if constexpr (Q8) eng.step(0, v[u], sc[u], d[u], jbase + s + j0 + u);
          else if constexpr (RED == R_SUM) V::fma(eng.acc, v[u], d[u]);
          else if constexpr (is_float16<T>::value) eng.vec_step(0, v[u], d[u], jbase + s + j0 + u);
          else eng.minmax_step(eng.acc, eng.arg, V::vfloat(v[u]), d[u], jbase + s + j0 + u);
        }
      }
      // QO: `mine` is the same for the LPR lanes of a group, so the group's amax shuffle is complete
      if (mine) ro.store(eng, p, rl, len, col_ok_arr, li);
    }
  }
}

// one warp per queued segment
template <typename T, int RED, int LPR, int CH, int U, int MINB, bool ACC = false, typename X = T, bool QO = false,
          bool RES = false, bool HEADS = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_seg_kernel(const SpmmParams p) {
  using Eng = typename EngineFor<T, RED, LPR, CH, U, X, HEADS>::type;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.template bind<!HEADS>(p, s_col[warp], s_val[warp], lane);
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
  int hcol[HEADS ? CH : 1];
  uint32_t row_bytes;
  int64_t lane_off;
  lane_cols<X, LPR, VEC, CH, HEADS>(p, li, col_ok, hcol, row_bytes, lane_off);

  const int64_t nseg = p.plan_mask ? p.n_seg : min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    const int64_t b = S.row_b / p.M, row = S.row_b - b * p.M;
    Eng eng;
    walk_segment<HEADS>(eng, p, S, b, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
    if (g == 0) {
      if (S.slot < 0) {
        if constexpr (QO)
          eng.template store_row_q8<RES>((uint8_t*)p.out + row * p.K, p.out_scale + row,
                                         p.arg_out ? p.arg_out + row * p.K : nullptr, S.end - S.start, p.E, col_ok,
                                         li, p.mean != 0, RES ? res_row<X>(p, row) : nullptr,
                                         RES ? res_scale(p, row) : 0.f);
        else
          eng.template store_row<RES>((T*)p.out + (b * p.M + row) * p.K + p.k0,
                                      p.arg_out ? p.arg_out + (b * p.M + row) * p.K + p.k0 : nullptr,
                                      S.end - S.start, p.E, col_ok, li, p.mean != 0,
                                      ACC ? p.partial + (b * p.M + row) * p.K + p.k0 : nullptr, ACC ? p.acc_mode : 0,
                                      RES ? res_row<X>(p, row) : nullptr, RES ? res_scale(p, row) : 0.f);
      } else {
        store_partial<LPR>(p, eng, S.slot, col_ok, li);
      }
    }
    __syncwarp();
  }
}

// combine the partials of multi-segment rows, in segment order. RES: plus the residual (element type R), after the
// mean's division.
template <typename T, int RED, bool RES = false, typename R = T>
__global__ void spmm_combine_kernel(const SpmmParams p, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int64_t nlong = p.plan_mask ? p.n_long : min((int64_t)p.counters[2], p.long_cap);
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    const int nseg = (int)(L.nseg_count >> 40);
    const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
    const float rs = RES ? res_scale(p, L.row_b) : 0.f;
    for (int k = threadIdx.x; k < kcols; k += blockDim.x) {
      const int64_t kk = p.k0 + k;
      if (kk >= p.K) break;
      int64_t ar;
      float a = combine_col<RED, false, RES, R>(p, L, nseg, count, kk, ar, rs);
      if (RED == R_SUM && p.acc_mode) {
        float* pr = p.partial + L.row_b * p.K + kk;
        if (p.acc_mode != 1) a += *pr;
        if (p.acc_mode != 3) { *pr = a; continue; }
      }
      ((T*)p.out)[L.row_b * p.K + kk] = Traits<T>::from_acc(a);
      if (ARG) p.arg_out[L.row_b * p.K + kk] = ar;
    }
  }
}

// the same for an e4m3 result (QO): per row, a first pass over the partials and a block reduction find the row's amax,
// the second pass writes y / scale. RES: both passes add the residual.
constexpr int kCombineThreads = 128;
template <int RED, bool RES = false>
__global__ void __launch_bounds__(kCombineThreads) spmm_combine_q8_kernel(const SpmmParams p, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  __shared__ float s_amax[kCombineThreads / 32];
  const int64_t nlong = p.plan_mask ? p.n_long : min((int64_t)p.counters[2], p.long_cap);
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    const int nseg = (int)(L.nseg_count >> 40);
    const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
    const float rs = RES ? res_scale(p, L.row_b) : 0.f;
    float amax = 0.f;
    for (int k = threadIdx.x; k < kcols; k += kCombineThreads) {
      const int64_t kk = p.k0 + k;
      if (kk >= p.K) break;
      int64_t ar;
      amax = amax_nan(amax, fabsf(combine_col<RED, false, RES>(p, L, nseg, count, kk, ar, rs)));
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) amax = amax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, off));
    if ((threadIdx.x & 31) == 0) s_amax[threadIdx.x >> 5] = amax;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kCombineThreads / 32; w++) amax = amax_nan(amax, s_amax[w]);
    __syncthreads();  // s_amax is rewritten for the next row
    const float s = e4m3_row_scale(amax);
    if (threadIdx.x == 0) p.out_scale[L.row_b] = s;
    for (int k = threadIdx.x; k < kcols; k += kCombineThreads) {
      const int64_t kk = p.k0 + k;
      if (kk >= p.K) break;
      int64_t ar;
      const float a = combine_col<RED, false, RES>(p, L, nseg, count, kk, ar, rs);
      ((uint8_t*)p.out)[L.row_b * p.K + kk] = e4m3_quant(a, s);
      if (ARG) p.arg_out[L.row_b * p.K + kk] = ar;
    }
  }
}

// ---- generic fallback: warp per (b,row), lane per column, sequential nnz walk -------------------
// RES (tsb200_spmm_fw_res, B == 1, sum / mean): plus fl(res_scale[m * res_stride] * res[m, k]) in the accumulator type
// (res_scale acc_t: float32, float64 for fp64), after the mean's division.
template <typename T, int RED, bool RES = false>
__global__ void __launch_bounds__(256)
spmm_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                    const T* __restrict__ value, const T* __restrict__ mat, T* __restrict__ out,
                    int64_t* __restrict__ arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                    int64_t E, bool mean, const T* __restrict__ res = nullptr, const void* __restrict__ res_scale = nullptr,
                    int64_t res_stride = 0) {
  static_assert(!RES || RED == R_SUM, "residual: sum / mean");
  const bool HV = value != nullptr;
  using acc_t = typename Traits<T>::acc_t;
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = wid; i < B * M; i += nw) {
    const int64_t b = i / M, m = i - b * M;
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    const T* matb = mat + b * N * K;
    for (int64_t k = lane; k < K; k += 32) {
      acc_t a;
      if (RED == R_MIN) a = Traits<T>::to_acc(Traits<T>::highest());
      else if (RED == R_MAX) a = Traits<T>::to_acc(Traits<T>::lowest());
      else a = (acc_t)0;
      int64_t ar = E;
      for (int64_t e = rs; e < re; e++) {
        const int64_t c = col[e];
        const acc_t mv = Traits<T>::to_acc(matb[c * K + k]);
        acc_t pr;
        if (HV) {
          const acc_t vv = Traits<T>::to_acc(value[e]);
          if constexpr (std::is_same<acc_t, float>::value) pr = __fmul_rn(vv, mv);
          else if constexpr (std::is_same<acc_t, double>::value) pr = __dmul_rn(vv, mv);
          else pr = (acc_t)(vv * mv);
        } else {
          pr = mv;
        }
        if (RED == R_SUM) {
          if constexpr (std::is_same<acc_t, float>::value) a = __fadd_rn(a, pr);
          else if constexpr (std::is_same<acc_t, double>::value) a = __dadd_rn(a, pr);
          else a = (acc_t)(a + pr);
        } else {
          if constexpr (is_float16<T>::value) pr = Traits<T>::to_acc(Traits<T>::from_acc(pr));
          const bool better = (RED == R_MIN) ? (pr < a) : (pr > a);
          if (better) { a = pr; ar = e; }
        }
      }
      const int64_t cnt = re - rs;
      if (RED == R_SUM && mean) a = a / (acc_t)(cnt > 0 ? cnt : 1);
      if (ARG && cnt == 0) a = (acc_t)0;
      if constexpr (RES)
        a = res_add(a, __ldg((const acc_t*)res_scale + m * res_stride), ResElem<T>::widen(__ldcs(res + m * K + k)));
      out[i * K + k] = Traits<T>::from_acc(a);
      if (ARG) arg_out[i * K + k] = cnt > 0 ? ar : E;
    }
  }
}

// ---- dispatch ------------------------------------------------------------------------------------
static bool vec_eligible(int dtype, int64_t K, int64_t E, int64_t N, const void* value,
                         const void* mat, const void* out, const void* col, const void* arg_out) {
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return false;
  const int64_t row_bytes = K * (int64_t)dtype_size(dtype);
  return row_bytes % 16 == 0 && rowsplit_extents(E, N, row_bytes) &&
         rowsplit_aligned({mat, out, arg_out}, col, {value});
}

// R: the residual's element type (X) with a residual, else T, so that every product without one shares a combine kernel
template <typename T, int RED, bool QO, bool RES, typename X>
static void launch_combine(const SpmmParams& p, int kcols, cudaStream_t st) {
  using R = typename std::conditional<RES, X, T>::type;
  if constexpr (QO) spmm_combine_q8_kernel<RED, RES><<<num_sms() * 2, kCombineThreads, 0, st>>>(p, kcols);
  else spmm_combine_kernel<T, RED, RES, R><<<num_sms() * 2, 128, 0, st>>>(p, kcols);
}

template <typename T, int RED, bool ACC, int LPR, int CH, int U, int MINB = 1, bool GPR = false, bool PLAN = false,
          typename X = T, bool QO = false, bool RES = false, bool HEADS = false>
static int launch_vec(SpmmParams p, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(X);
  constexpr int kcols = LPR * CH * VEC;
  void (*kmain)(const SpmmParams);
  if constexpr (GPR) kmain = spmm_gpr_kernel<T, RED, LPR, U, MINB, ACC, PLAN, X, QO, RES, HEADS>;
  else kmain = spmm_vec_kernel<T, RED, LPR, CH, U, MINB, ACC, PLAN, X, QO, RES, HEADS>;
  constexpr int USEG = (U > LPR) ? LPR : U;  // the row engine needs U * (32 / LPR) <= 32
  auto* kseg = spmm_seg_kernel<T, RED, LPR, CH, USEG, MINB, ACC, X, QO, RES, HEADS>;
  static GridCache gc_main, gc_seg;  // per instantiation, per device
  for (int k0 = 0; k0 < p.K; k0 += kcols) {
    p.k0 = k0;
    if constexpr (PLAN) {
      // one memset (ticket counters + the per-long-row completion counters behind them), ONE kernel: the row items,
      // then the plan's segments, drained by the same warps. The group-per-row kernel has no index ring to drain
      // with, so for narrow dense rows the segment / combine kernels are still launched — when the plan says there
      // is something for them to do.
      const int grid_main = gc_main.get((const void*)kmain, kWarpsPerCta * 32);
      p.item_shift = item_shift_for(p.M * p.B, grid_main);
      const int64_t n_items = ((p.M + (1 << p.item_shift) - 1) >> p.item_shift) * p.B;
      TSB_CUDA_TRY(cudaMemsetAsync(p.counters, 0, 256 + (size_t)p.n_long * 4, st));
      int64_t work = (n_items + kWarpsPerCta - 1) / kWarpsPerCta;
      if (!GPR) work = max(work, (p.n_seg + kWarpsPerCta - 1) / kWarpsPerCta);
      const int gm = (int)max((int64_t)1, min((int64_t)grid_main, work));
      kmain<<<gm, kWarpsPerCta * 32, 0, st>>>(p);
      TSB_LAUNCH_CHECK();
      if (GPR && p.n_seg > 0) {
        const int grid_seg = gc_seg.get((const void*)kseg, kWarpsPerCta * 32);
        kseg<<<grid_seg, kWarpsPerCta * 32, 0, st>>>(p);
        TSB_LAUNCH_CHECK();
        if (p.n_long > 0) {
          launch_combine<T, RED, QO, RES, X>(p, kcols, st);
          TSB_LAUNCH_CHECK();
        }
      }
    } else {
      if (const int rc = launch_rowsplit(kmain, kseg, gc_main, gc_seg, p, st)) return rc;
      launch_combine<T, RED, QO, RES, X>(p, kcols, st);
      TSB_LAUNCH_CHECK();
    }
  }
  return 0;
}

// (LPR, CH) follow from the width of a dense row; (U, MINB) = gathers in flight per lane and CTAs
// per SM: the kernel is HBM-latency bound, so resident warps x gathers-in-flight wins (40 warps/SM x 4 x 16 B
// per lane; the register budget of MINB = 5 is the same 64K registers per SM on sm_90).
template <typename T, int RED, bool ACC = false, bool PLAN = false, typename X = T, bool QO = false,
          bool RES = false>
static int dispatch_shape(const SpmmParams& p, cudaStream_t st) {
  // fp8 operand: a vector is 16 columns, so a lane keeps twice the accumulators (and arg slots) of a 16-bit operand
  // and needs more registers per thread: its own (U, CTAs/SM) per shape (ptxas report and times in DESIGN §3.1)
  constexpr bool Q8 = !std::is_same<X, T>::value;
  constexpr bool MM = RED != R_SUM;
  constexpr int VEC = 16 / sizeof(X);
  const int64_t vecs = p.K / VEC;  // 16-byte vectors per dense row
  // narrow rows: group-per-row kernel (all reductions)
  // A residual of the operand's type spills every main kernel at the CTAs/SM of its shape (its 16-byte residual chunk
  // and scale live next to the accumulators), so those take the most CTAs/SM at which none spills: one less, and two
  // less for the 5-CTA shapes, which still spill at 4 (ptxas table in DESIGN §3.1).
  constexpr bool FRES = RES && !Q8;
  constexpr int GB = Q8 ? (MM ? 2 : 3) : (FRES ? 3 : 5);
  if (vecs <= 1) return launch_vec<T, RED, ACC, 1, 1, 4, GB, true, PLAN, X, QO, RES>(p, st);
  if (vecs <= 2) return launch_vec<T, RED, ACC, 2, 1, 4, GB, true, PLAN, X, QO, RES>(p, st);
  if (vecs <= 4) return launch_vec<T, RED, ACC, 4, 1, 4, GB, true, PLAN, X, QO, RES>(p, st);
  if (vecs <= 8) return launch_vec<T, RED, ACC, 8, 1, 4, GB, true, PLAN, X, QO, RES>(p, st);
  // 256-byte rows (F = 128 bf16): at MINB = 5 the 48-register budget spills (120 B of stack in the planned kernel);
  // 3 CTAs/SM with 6 gathers in flight per lane is 8 % faster at C2 on the H100 (sweep in DESIGN §3.1)
  // e4m3 result (QO): the quantising epilogue (row amax, IEEE divisions) spills the sum kernels of 256-, 512- and
  // 2048-byte rows at the CTAs/SM of the fp32 result; those take one CTA/SM less (ptxas table in DESIGN §3.1).
  // A residual (RES) spills the planned kernels of the same shapes at that occupancy, so it takes the QO shapes.
  constexpr bool LOW = MM || QO || RES;
  if (vecs <= 16)
    return launch_vec<T, RED, ACC, 16, 1, Q8 && !MM ? 4 : 6, (Q8 && LOW) || FRES ? 2 : 3, false, PLAN, X, QO, RES>(p,
                                                                                                               st);
  if (vecs <= 32)
    return launch_vec<T, RED, ACC, 32, 1, 4, Q8 ? (LOW ? 2 : 3) : (FRES ? 3 : 5), false, PLAN, X, QO, RES>(p, st);
  if (vecs <= 64)
    return launch_vec<T, RED, ACC, 32, 2, Q8 && MM ? 2 : 4, Q8 || FRES ? 2 : 3, false, PLAN, X, QO, RES>(p, st);
  // column-tiled beyond 128 vectors
  return launch_vec<T, RED, ACC, 32, 4, 2, Q8 ? (LOW ? 1 : 2) : (FRES ? 2 : 3), false, PLAN, X, QO, RES>(p, st);
}

template <typename T, bool PLAN = false, typename X = T, bool QO = false, bool RES = false>
static int dispatch_red_vec(SpmmParams p, int reduce, cudaStream_t st) {
  p.mean = (reduce == TSB200_MEAN);
  if constexpr (RES) {  // a residual is added to sums and means only
    if (reduce != TSB200_SUM && reduce != TSB200_MEAN) return TSB200_ERR_UNSUPPORTED;
    return dispatch_shape<T, R_SUM, false, PLAN, X, QO, true>(p, st);
  } else {
    switch (reduce) {
      case TSB200_SUM:
      case TSB200_MEAN: return dispatch_shape<T, R_SUM, false, PLAN, X, QO>(p, st);
      case TSB200_MIN: return dispatch_shape<T, R_MIN, false, PLAN, X, QO>(p, st);
      case TSB200_MAX: return dispatch_shape<T, R_MAX, false, PLAN, X, QO>(p, st);
    }
    return TSB200_ERR_INVALID_ARG;
  }
}

// per-head weights (tsb200_spmm_heads): the sum kernels' shapes; (U, CTAs/SM) as for one head unless the weight
// registers spill there (ptxas table in DESIGN §3.1)
template <typename T, bool PLAN>
static int dispatch_heads(const SpmmParams& p, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t vecs = p.K / VEC;
  if (vecs <= 1) return launch_vec<T, R_SUM, false, 1, 1, 4, 4, true, PLAN, T, false, false, true>(p, st);
  if (vecs <= 2) return launch_vec<T, R_SUM, false, 2, 1, 4, 4, true, PLAN, T, false, false, true>(p, st);
  if (vecs <= 4) return launch_vec<T, R_SUM, false, 4, 1, 4, 4, true, PLAN, T, false, false, true>(p, st);
  if (vecs <= 8) return launch_vec<T, R_SUM, false, 8, 1, 4, 4, true, PLAN, T, false, false, true>(p, st);
  if (vecs <= 16) return launch_vec<T, R_SUM, false, 16, 1, 6, 2, false, PLAN, T, false, false, true>(p, st);
  if (vecs <= 32) return launch_vec<T, R_SUM, false, 32, 1, 4, 4, false, PLAN, T, false, false, true>(p, st);
  if (vecs <= 64) return launch_vec<T, R_SUM, false, 32, 2, 4, 2, false, PLAN, T, false, false, true>(p, st);
  return launch_vec<T, R_SUM, false, 32, 4, 2, 2, false, PLAN, T, false, false, true>(p, st);
}

// ---- plan: the segment list of a matrix, built once (tsb200_spmm_plan) -----------------------------------------
// One warp per group of 32 rows: the rows defer_row defers become <= kSeg-nnz segments; also leaves one mask word per
// group. Its push writes the records of push_row_segments from 64-bit degrees, plus each segment's long row (seg_lr).
__global__ void __launch_bounds__(256)
spmm_plan_kernel(const int64_t* __restrict__ rowptr, int64_t M, uint32_t* __restrict__ mask, Segment* __restrict__ segs,
                 uint32_t* __restrict__ seg_lr, LongRow* __restrict__ longs, unsigned int* __restrict__ counters,
                 int64_t seg_cap, int64_t long_cap) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t ngroups = (M + 31) >> 5;
  for (int64_t grp = wid; grp < ngroups; grp += nw) {
    const int64_t r0 = grp << 5;
    const int nrows = (int)min((int64_t)32, M - r0);
    const int64_t rp0 = __ldg(rowptr + r0 + min(lane, nrows));
    const int64_t rp1 = __ldg(rowptr + r0 + min(lane + 1, nrows));
    const int64_t deg64 = rp1 - rp0;
    const bool defer = defer_row((int)min(deg64, (int64_t)0x3fffffff), lane);
    const unsigned defer_mask = __ballot_sync(0xffffffffu, defer);
    if (lane == 0) mask[grp] = defer_mask;
    if (defer) {
      const int64_t nseg = (deg64 + kSeg - 1) / kSeg;
      const unsigned seg0 = atomicAdd(&counters[1], (unsigned)nseg);
      int64_t slot0 = -1;
      unsigned lr = 0;
      if (nseg > 1) {
        slot0 = atomicAdd(&counters[3], (unsigned)nseg);
        lr = atomicAdd(&counters[2], 1u);
        if ((int64_t)lr < long_cap) {
          LongRow L;
          L.row_b = r0 + lane;
          L.first_slot = slot0;
          L.nseg_count = (nseg << 40) | deg64;
          longs[lr] = L;
        }
      }
      for (int64_t sgi = 0; sgi < nseg; sgi++) {
        if ((int64_t)seg0 + sgi < seg_cap) {
          Segment S;
          S.row_b = r0 + lane;
          S.start = rp0 + sgi * kSeg;
          S.end = min(rp1, S.start + kSeg);
          S.slot = slot0 < 0 ? -1 : slot0 + sgi;
          segs[seg0 + sgi] = S;
          seg_lr[seg0 + sgi] = lr;
        }
      }
    }
  }
}

// generic per-head SpMM (tsb200_spmm_heads off the vector path): warp per row, lane per column k of the H * D, the
// entries summed in order with one rounding per product and per sum, as spmm_generic_kernel does
template <typename T>
__global__ void __launch_bounds__(256)
spmm_heads_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                          const T* __restrict__ value, const T* __restrict__ mat, T* __restrict__ out, int64_t M,
                          int64_t H, int64_t D) {
  using acc_t = typename Traits<T>::acc_t;
  const int64_t K = H * D;
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t m = wid; m < M; m += nw) {
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    for (int64_t k = lane; k < K; k += 32) {
      const int64_t h = k / D;
      acc_t a = (acc_t)0;
      for (int64_t e = rs; e < re; e++) {
        const acc_t mv = Traits<T>::to_acc(mat[col[e] * K + k]);
        const acc_t vv = Traits<T>::to_acc(value[e * H + h]);
        if constexpr (std::is_same<acc_t, double>::value) a = __dadd_rn(a, __dmul_rn(vv, mv));
        else a = __fadd_rn(a, __fmul_rn(vv, mv));
      }
      out[m * K + k] = Traits<T>::from_acc(a);
    }
  }
}

template <typename T, int RED>
static int launch_generic(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                          void* out, int64_t* arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                          int64_t E, bool mean, cudaStream_t st) {
  spmm_generic_kernel<T, RED><<<warp_grid(B * M, 64), 256, 0, st>>>(rowptr, col, (const T*)value, (const T*)mat,
                                                                    (T*)out, arg_out, B, M, N, K, E, mean);
  TSB_LAUNCH_CHECK();
  return 0;
}

// ---- multi-aggregation SpMM (tsb200_spmm_fw_multi) -----------------------------------------------------------------
// One gather pass accumulates, per column, the four statistics every aggregator is formed from: the sum S, the sum of
// squares Q = sum fma(p, p, .) of the products p, and the min and max of the products rounded to T with their entries.
// S, min and max follow exactly the single-reduction engines (same lane layout per row width, same per-lane order,
// butterfly and segment fold), so the sum, mean, min and max slices are spmm's bits. The store epilogue writes only
// the requested statistics, each into its slice of out [M, A, K], and the args only where their pointer is set.
enum : int { R_VAR = TSB200_VAR, R_STD = TSB200_STD, kStats = 6 };

struct MultiOut {
  int64_t* arg_min;  // [M, K] or NULL: not stored
  int64_t* arg_max;
  int A;             // slices per row of `out`
  int8_t slice[kStats];  // slice of each aggregator code, -1 = not requested
};

// aggregator c of one column from its statistics over a row of `count` entries, in the accumulator type: the mean's
// IEEE division, var = max(fl(fl(Q / n) - fl(mu * mu)), 0) (no contraction, so a one-entry row gives exactly 0; NaN
// passes), std = sqrt(var) where var > 1e-5, else 0
template <typename A>
__device__ __forceinline__ A multi_stat(int c, A s, A q, A mn, A mx, int64_t count) {
  const A n = (A)(count > 0 ? count : 1);
  if (c == R_SUM) return s;
  if (c == R_MIN) return count == 0 ? (A)0 : mn;
  if (c == R_MAX) return count == 0 ? (A)0 : mx;
  const A mu = s / n;
  if (c == R_MEAN) return mu;
  A d;
  if constexpr (std::is_same<A, double>::value) d = __dsub_rn(q / n, __dmul_rn(mu, mu));
  else d = __fsub_rn(q / n, __fmul_rn(mu, mu));
  const A var = d < (A)0 ? (A)0 : d;
  if (c == R_VAR) return var;
  return var > (A)1e-5 ? sqrt(var) : (A)0;
}

// the per-lane state of the multi kernels: VEC * CH columns of S, Q, min, max and the two args
template <typename T, int LPR, int CH, int U> struct MultiEngine {
  using V = Vec<T>;
  static constexpr bool Q8 = false;
  static constexpr int VEC = V::VEC;
  static constexpr int G = 32 / LPR;
  static constexpr int NA = VEC * CH;

  float s[NA], q[NA], mn[NA], mx[NA];
  int amn[NA], amx[NA];

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < NA; i++) {
      s[i] = 0.f;
      q[i] = 0.f;
      mn[i] = Traits<T>::to_acc(Traits<T>::highest());
      mx[i] = Traits<T>::to_acc(Traits<T>::lowest());
      amn[i] = amx[i] = 0x7fffffff;
    }
  }

  // one gathered vector of one entry (raw value v, entry jabs): the sum as Vec<T>::fma, the min / max on the product
  // rounded to T as RowEngine::minmax_step (bit for bit the packed 16-bit engine's), Q on the fp32 product
  __device__ __forceinline__ void step(int ch, typename V::vraw v, const uint4& d, int jabs) {
    const float vf = V::vfloat(v);
    float f[VEC];
    V::unpack(d, f);
#pragma unroll
    for (int i = 0; i < VEC; i++) {
      const int a = ch * VEC + i;
      s[a] = fmaf(vf, f[i], s[a]);
      const float pr = __fmul_rn(vf, f[i]);
      q[a] = fmaf(pr, pr, q[a]);
      const float pm = V::round_prod(pr);
      if (pm < mn[a]) { mn[a] = pm; amn[a] = jabs; }
      if (pm > mx[a]) { mx[a] = pm; amx[a] = jabs; }
    }
  }

  // ring-relative nnz [s, e) of one row, G entries per step (one per lane group) and U steps per chunk, as
  // RowEngine::accumulate walks them
  __device__ __forceinline__ void accumulate(IndexRing<T>& ring, int s0, int e, const char* __restrict__ matb,
                                             uint32_t row_bytes, const bool (&col_ok)[CH], int lane, int g,
                                             uint64_t pol) {
    using VR = typename V::vraw;
    for (int j0 = s0; j0 < e; j0 += U * G) {
      const int jend = min(e, j0 + U * G);
      ring.ensure(j0, jend, lane);
      const int slot0 = (j0 + g) & (kRing - 1);
      const uint32_t* pc = reinterpret_cast<const uint32_t*>(ring.s_col + slot0);
      const VR* pv = reinterpret_cast<const VR*>(ring.s_val) + slot0;
      const int jabs0 = (int)ring.base + j0 + g;
      const int nst = (jend - j0 + G - 1) / G;
      const int jrel = jend - j0 - g;
      uint4 d[U][CH];
      VR v[U];
      bool act[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (u >= nst) break;
        act[u] = u * G < jrel;
        const uint32_t c = pc[2 * u * G];
        v[u] = pv[u * G];
        const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
        for (int ch = 0; ch < CH; ch++)
          if (act[u] && col_ok[ch]) d[u][ch] = ldg128_hint(src + ch * (LPR * 16), pol);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (u >= nst) break;
#pragma unroll
        for (int ch = 0; ch < CH; ch++)
          if (act[u] && col_ok[ch]) step(ch, v[u], d[u][ch], jabs0 + u * G);
      }
    }
  }

  // the butterfly of RowEngine::reduce_groups over the four statistics
  __device__ __forceinline__ void reduce_groups() {
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
#pragma unroll
      for (int i = 0; i < NA; i++) {
        s[i] += __shfl_xor_sync(0xffffffffu, s[i], off);
        q[i] += __shfl_xor_sync(0xffffffffu, q[i], off);
        const float on = __shfl_xor_sync(0xffffffffu, mn[i], off);
        const int oan = __shfl_xor_sync(0xffffffffu, amn[i], off);
        if (on < mn[i] || (on == mn[i] && oan < amn[i])) { mn[i] = on; amn[i] = oan; }
        const float ox = __shfl_xor_sync(0xffffffffu, mx[i], off);
        const int oax = __shfl_xor_sync(0xffffffffu, amx[i], off);
        if (ox > mx[i] || (ox == mx[i] && oax < amx[i])) { mx[i] = ox; amx[i] = oax; }
      }
    }
  }

  // final write of row `row` (count entries) by the lanes that hold it: each requested aggregator into its slice, the
  // args where their pointers are set
  __device__ __forceinline__ void store_row(const SpmmParams& p, const MultiOut& mo, int64_t row, int64_t count,
                                            const bool (&col_ok)[CH], int li) const {
    T* orow = (T*)p.out + row * mo.A * p.K + p.k0;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
#pragma unroll
      for (int c = 0; c < kStats; c++) {
        const int sl = mo.slice[c];
        if (sl < 0) continue;
        float f[VEC];
#pragma unroll
        for (int i = 0; i < VEC; i++) {
          const int a = ch * VEC + i;
          f[i] = multi_stat<float>(c, s[a], q[a], mn[a], mx[a], count);
        }
        stg128_stream(orow + sl * p.K + koff, V::pack(f));
      }
      if (mo.arg_min) store_args<VEC>(mo.arg_min + row * p.K + p.k0 + koff, &amn[ch * VEC], count, p.E);
      if (mo.arg_max) store_args<VEC>(mo.arg_max + row * p.K + p.k0 + koff, &amx[ch * VEC], count, p.E);
    }
  }

  // the partial of one segment into slot `slot`: four fp32 planes [slot][4][K] (S, Q, min, max) and two int64 arg
  // planes [slot][2][K] (min, max)
  __device__ __forceinline__ void store_partial(const SpmmParams& p, int64_t slot, const bool (&col_ok)[CH],
                                                int li) const {
    float* pv = (float*)p.part_val + slot * 4 * p.K + p.k0;
    int64_t* pa = p.part_arg + slot * 2 * p.K + p.k0;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
#pragma unroll
      for (int i = 0; i < VEC; i++) {
        const int a = ch * VEC + i;
        pv[koff + i] = s[a];
        pv[p.K + koff + i] = q[a];
        pv[2 * p.K + koff + i] = mn[a];
        pv[3 * p.K + koff + i] = mx[a];
        pa[koff + i] = stored_arg(amn[a], p.E);
        pa[p.K + koff + i] = stored_arg(amx[a], p.E);
      }
    }
  }
};

// column kk of a multi-segment row: its partials folded in segment order as combine_col folds them (the smallest e
// wins min / max ties), then every requested aggregator and arg stored. CG: read past L1 (planned drain).
template <typename T, bool CG>
__device__ __forceinline__ void combine_multi_col(const SpmmParams& p, const MultiOut& mo, const LongRow& L, int nseg,
                                                  int64_t count, int64_t kk) {
  const float* pv = (const float*)p.part_val;
  auto ldv = [&](int64_t sl, int st) {
    const float* a = pv + (sl * 4 + st) * p.K + kk;
    return CG ? __ldcg(a) : *a;
  };
  auto lda = [&](int64_t sl, int st) {
    const int64_t* a = p.part_arg + (sl * 2 + st) * p.K + kk;
    return CG ? __ldcg(a) : *a;
  };
  float s = ldv(L.first_slot, 0), q = ldv(L.first_slot, 1), mn = ldv(L.first_slot, 2), mx = ldv(L.first_slot, 3);
  int64_t amn = lda(L.first_slot, 0), amx = lda(L.first_slot, 1);
  for (int sgi = 1; sgi < nseg; sgi++) {
    const int64_t sl = L.first_slot + sgi;
    s += ldv(sl, 0);
    q += ldv(sl, 1);
    const float vn = ldv(sl, 2), vx = ldv(sl, 3);
    const int64_t an = lda(sl, 0), ax = lda(sl, 1);
    if (vn < mn || (vn == mn && an < amn)) { mn = vn; amn = an; }
    if (vx > mx || (vx == mx && ax < amx)) { mx = vx; amx = ax; }
  }
  T* orow = (T*)p.out + L.row_b * mo.A * p.K + kk;
#pragma unroll
  for (int c = 0; c < kStats; c++)
    if (mo.slice[c] >= 0) orow[mo.slice[c] * p.K] = Traits<T>::from_acc(multi_stat<float>(c, s, q, mn, mx, count));
  if (mo.arg_min) mo.arg_min[L.row_b * p.K + kk] = amn;
  if (mo.arg_max) mo.arg_max[L.row_b * p.K + kk] = amx;
}

// row-per-warp multi kernel: the work items of spmm_vec_kernel and, PLAN with DRAIN, its drain of the plan's segments
template <typename T, int LPR, int CH, int U, int MINB, bool PLAN, bool DRAIN>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_multi_vec_kernel(const SpmmParams p, const MultiOut mo) {
  using Eng = MultiEngine<T, LPR, CH, U>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.template bind<true>(p, s_col[warp], s_val[warp], lane);
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
  int hcol[1];
  uint32_t row_bytes;
  int64_t lane_off;
  lane_cols<T, LPR, VEC, CH, false>(p, li, col_ok, hcol, row_bytes, lane_off);

  for (WorkItem it(p, lane); it.start(p, lane); it.advance()) {
    const int64_t a0 = __shfl_sync(0xffffffffu, it.rp0, 0);
    const int64_t base = a0 & ~(int64_t)31;
    const int s_rel = (int)(it.rp0 - base), e_rel = (int)(it.rp1 - base);
    const int deg = e_rel - s_rel;
    unsigned defer_mask;
    if constexpr (PLAN) {
      defer_mask = it.plan_defer_mask(p);
    } else {
      const bool defer = defer_row(deg, lane);
      defer_mask = __ballot_sync(0xffffffffu, defer);
      if (defer) push_row_segments(p, it.b, it.r0, lane, it.rp0, it.rp1, deg);
    }
    __syncwarp();
    ring.reset(base, __shfl_sync(0xffffffffu, it.rp1, 31));
    const char* matb = (const char*)p.mat + lane_off;
    asm volatile("" : "+l"(matb));
    for (int rl = 0; rl < it.nrows; rl++) {
      if ((defer_mask >> rl) & 1u) continue;
      const int s = __shfl_sync(0xffffffffu, s_rel, rl);
      const int e = __shfl_sync(0xffffffffu, e_rel, rl);
      Eng eng;
      eng.init();
      eng.accumulate(ring, s, e, matb, row_bytes, col_ok, lane, g, pol);
      eng.reduce_groups();
      if (g == 0) eng.store_row(p, mo, it.r0 + rl, e - s, col_ok, li);
    }
  }

  if constexpr (PLAN && DRAIN) {  // the planned drain of spmm_vec_kernel
    constexpr int kcols = LPR * CH * VEC;
    while (true) {
      const unsigned int sidx = __shfl_sync(0xffffffffu, take_ticket(&p.counters[5], lane), 0);
      if ((int64_t)sidx >= p.n_seg) break;
      const Segment S = p.segs[sidx];
      Eng eng;
      walk_segment<false>(eng, p, S, 0, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
      if (S.slot < 0) {
        if (g == 0) eng.store_row(p, mo, S.row_b, S.end - S.start, col_ok, li);
      } else {
        if (g == 0) eng.store_partial(p, S.slot, col_ok, li);
        __syncwarp();
        __threadfence();
        const uint32_t lr = __ldg(p.seg_lr + sidx);
        unsigned int finished = 0;
        if (lane == 0) finished = atomicAdd(&p.long_done[lr], 1u);
        finished = __shfl_sync(0xffffffffu, finished, 0);
        const LongRow L = p.longs[lr];
        int nseg;
        int64_t count;
        long_row_counts(L, nseg, count);
        if ((int)finished == nseg - 1) {
          __threadfence();
          for (int k = lane; k < kcols && p.k0 + k < p.K; k += 32)
            combine_multi_col<T, true>(p, mo, L, nseg, count, p.k0 + k);
        }
      }
      __syncwarp();
    }
  }
}

// group-per-row multi kernel (narrow rows): the walk of spmm_gpr_kernel, each lane group over its own row
template <typename T, int LPR, int U, int MINB, bool PLAN>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_multi_gpr_kernel(const SpmmParams p, const MultiOut mo) {
  using V = Vec<T>;
  using Eng = MultiEngine<T, LPR, 1, U>;
  using VR = typename V::vraw;
  constexpr int VEC = Eng::VEC;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  const bool col_ok = p.k0 + li * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(T);
  const uint64_t pol = make_policy_evict_last();
  const T* __restrict__ val = (const T*)p.value;
  const bool has_val = val != nullptr;

  for (WorkItem it(p, lane); it.start(p, lane); it.advance()) {
    const int64_t base = __shfl_sync(0xffffffffu, it.rp0, 0);
    const int s_rel = (int)(it.rp0 - base), e_rel = (int)(it.rp1 - base);
    const int deg = e_rel - s_rel;
    unsigned defer_mask;
    if constexpr (PLAN) {
      defer_mask = it.plan_defer_mask(p);
    } else {
      const bool defer = defer_row(deg, lane);
      defer_mask = __ballot_sync(0xffffffffu, defer);
      if (defer) push_row_segments(p, it.b, it.r0, lane, it.rp0, it.rp1, deg);
    }
    __syncwarp();
    const char* matb = (const char*)p.mat + lane_off;
    asm volatile("" : "+l"(matb));
    const int64_t* __restrict__ colb = p.col + base;
    const T* __restrict__ valb = has_val ? val + base : nullptr;
    const bool col_ok_arr[1] = {col_ok};
    const int jbase = (int)base;

    for (int t = 0; t < it.nrows; t += G) {
      const int rl = t + g;
      int s = __shfl_sync(0xffffffffu, s_rel, rl & 31);
      int e = __shfl_sync(0xffffffffu, e_rel, rl & 31);
      const bool mine = rl < it.nrows && !((defer_mask >> (rl & 31)) & 1u);
      if (!mine) e = s;
      const int len = e - s;
      int maxlen = len;
#pragma unroll
      for (int off = LPR; off < 32; off <<= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, off));
      Eng eng;
      eng.init();
      uint32_t cn[U];
      VR vn[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        cn[u] = 0;
        vn[u] = V::one();
        if (u < len) {
          cn[u] = (uint32_t)__ldg(colb + s + u);
          if (has_val) vn[u] = load_vraw<T>(valb + s + u);
        }
      }
      for (int j0 = 0; j0 < maxlen; j0 += U) {
        uint4 d[U];
        VR v[U];
        bool act[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          act[u] = (j0 + u < len) && col_ok;
          v[u] = vn[u];
          if (act[u]) d[u] = ldg128_hint(matb + (uint64_t)cn[u] * row_bytes, pol);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int jn = j0 + U + u;
          if (jn < len) {
            cn[u] = (uint32_t)__ldg(colb + s + jn);
            if (has_val) vn[u] = load_vraw<T>(valb + s + jn);
          }
        }
#pragma unroll
        for (int u = 0; u < U; u++)
          if (act[u]) eng.step(0, v[u], d[u], jbase + s + j0 + u);
      }
      if (mine) eng.store_row(p, mo, it.r0 + rl, len, col_ok_arr, li);
    }
  }
}

// one warp per queued segment (spmm_seg_kernel)
template <typename T, int LPR, int CH, int U, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_multi_seg_kernel(const SpmmParams p, const MultiOut mo) {
  using Eng = MultiEngine<T, LPR, CH, U>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  IndexRing<T> ring;
  ring.template bind<true>(p, s_col[warp], s_val[warp], lane);
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
  int hcol[1];
  uint32_t row_bytes;
  int64_t lane_off;
  lane_cols<T, LPR, VEC, CH, false>(p, li, col_ok, hcol, row_bytes, lane_off);

  const int64_t nseg = p.plan_mask ? p.n_seg : min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    Eng eng;
    walk_segment<false>(eng, p, S, 0, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
    if (g == 0) {
      if (S.slot < 0) eng.store_row(p, mo, S.row_b, S.end - S.start, col_ok, li);
      else eng.store_partial(p, S.slot, col_ok, li);
    }
    __syncwarp();
  }
}

// the multi-segment rows' partials, in segment order (spmm_combine_kernel)
template <typename T>
__global__ void spmm_multi_combine_kernel(const SpmmParams p, const MultiOut mo, int kcols) {
  const int64_t nlong = p.plan_mask ? p.n_long : min((int64_t)p.counters[2], p.long_cap);
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    int nseg;
    int64_t count;
    long_row_counts(L, nseg, count);
    for (int k = threadIdx.x; k < kcols && p.k0 + k < p.K; k += blockDim.x)
      combine_multi_col<T, false>(p, mo, L, nseg, count, p.k0 + k);
  }
}

// generic multi kernel (fp64, partial widths, unaligned operands, E >= 2^31): warp per row, lane per column, the entries
// in order as spmm_generic_kernel walks them (one rounding per product and per sum), plus Q = sum fma(p, p, .)
template <typename T>
__global__ void __launch_bounds__(256)
spmm_multi_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                          const T* __restrict__ value, const T* __restrict__ mat, T* __restrict__ out, int64_t M,
                          int64_t K, int64_t E, const MultiOut mo) {
  using acc_t = typename Traits<T>::acc_t;
  constexpr bool F64 = std::is_same<acc_t, double>::value;
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t m = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < M; m += nw) {
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    for (int64_t k = lane; k < K; k += 32) {
      acc_t s = 0, q = 0;
      acc_t mn = Traits<T>::to_acc(Traits<T>::highest()), mx = Traits<T>::to_acc(Traits<T>::lowest());
      int64_t amn = E, amx = E;
      for (int64_t e = rs; e < re; e++) {
        const acc_t mv = Traits<T>::to_acc(mat[col[e] * K + k]);
        acc_t pr = mv;
        if (value) {
          if constexpr (F64) pr = __dmul_rn(Traits<T>::to_acc(value[e]), mv);
          else pr = __fmul_rn(Traits<T>::to_acc(value[e]), mv);
        }
        if constexpr (F64) { s = __dadd_rn(s, pr); q = fma(pr, pr, q); }
        else { s = __fadd_rn(s, pr); q = fmaf(pr, pr, q); }
        acc_t pm = pr;
        if constexpr (is_float16<T>::value) pm = Traits<T>::to_acc(Traits<T>::from_acc(pr));
        if (pm < mn) { mn = pm; amn = e; }
        if (pm > mx) { mx = pm; amx = e; }
      }
      const int64_t cnt = re - rs;
#pragma unroll
      for (int c = 0; c < kStats; c++)
        if (mo.slice[c] >= 0)
          out[(m * mo.A + mo.slice[c]) * K + k] = Traits<T>::from_acc(multi_stat<acc_t>(c, s, q, mn, mx, cnt));
      if (mo.arg_min) mo.arg_min[m * K + k] = cnt > 0 ? amn : E;
      if (mo.arg_max) mo.arg_max[m * K + k] = cnt > 0 ? amx : E;
    }
  }
}

// workspace of tsb200_spmm_fw_multi: the layouts of tsb200_spmm_fw (plan == NULL) or tsb200_spmm_fw_planned over 4 * K
// fp32 partial columns per slot, followed by 2 * K int64 arg columns per slot
struct MultiWs {
  size_t args, total;
};
static inline MultiWs multi_ws(int64_t K, int64_t E, bool planned, int64_t n_long, int64_t n_slot) {
  MultiWs L;
  const int64_t slots = planned ? (n_slot > 0 ? n_slot : 1) : ws_layout(1, K, E, false).slot_cap;
  L.args = planned ? planned_ws(4 * K, n_long, n_slot, false).total : ws_layout(1, 4 * K, E, false).total;
  L.total = L.args + align_up((size_t)slots * (size_t)(2 * K) * sizeof(int64_t), 256);
  return L;
}

template <typename T, int LPR, int CH, int U, int MINB, bool GPR, bool PLAN>
static int launch_multi(SpmmParams p, const MultiOut& mo, cudaStream_t st) {
  constexpr int kcols = LPR * CH * Vec<T>::VEC;
  // the planned drain spills the 16-bit kernel of the widest shape (four statistics of 32 columns per lane), so there
  // the plan's segments go to the segment and combine kernels, as for the group-per-row shapes
  constexpr bool DRAIN = !GPR && !(sizeof(T) == 2 && CH == 4);
  void (*kmain)(const SpmmParams, const MultiOut);
  if constexpr (GPR) kmain = spmm_multi_gpr_kernel<T, LPR, U, MINB, PLAN>;
  else kmain = spmm_multi_vec_kernel<T, LPR, CH, U, MINB, PLAN, DRAIN>;
  constexpr int USEG = (U > LPR) ? LPR : U;
  auto* kseg = spmm_multi_seg_kernel<T, LPR, CH, USEG, MINB>;
  static GridCache gc_main, gc_seg;
  for (int k0 = 0; k0 < p.K; k0 += kcols) {
    p.k0 = k0;
    if constexpr (PLAN) {  // as launch_vec: one kernel, plus segment / combine kernels when it does not drain
      const int grid_main = gc_main.get((const void*)kmain, kWarpsPerCta * 32);
      p.item_shift = item_shift_for(p.M, grid_main);
      const int64_t n_items = (p.M + (1 << p.item_shift) - 1) >> p.item_shift;
      TSB_CUDA_TRY(cudaMemsetAsync(p.counters, 0, 256 + (size_t)p.n_long * 4, st));
      int64_t work = (n_items + kWarpsPerCta - 1) / kWarpsPerCta;
      if (DRAIN) work = max(work, (p.n_seg + kWarpsPerCta - 1) / kWarpsPerCta);
      kmain<<<(int)max((int64_t)1, min((int64_t)grid_main, work)), kWarpsPerCta * 32, 0, st>>>(p, mo);
      TSB_LAUNCH_CHECK();
      if (!DRAIN && p.n_seg > 0) {
        kseg<<<gc_seg.get((const void*)kseg, kWarpsPerCta * 32), kWarpsPerCta * 32, 0, st>>>(p, mo);
        TSB_LAUNCH_CHECK();
        if (p.n_long > 0) {
          spmm_multi_combine_kernel<T><<<num_sms() * 2, 128, 0, st>>>(p, mo, kcols);
          TSB_LAUNCH_CHECK();
        }
      }
    } else {
      if (const int rc = launch_rowsplit(kmain, kseg, gc_main, gc_seg, p, st, mo)) return rc;
      spmm_multi_combine_kernel<T><<<num_sms() * 2, 128, 0, st>>>(p, mo, kcols);
      TSB_LAUNCH_CHECK();
    }
  }
  return 0;
}

// (LPR, CH) of dispatch_shape for each row width, so that every lane sums, compares and folds as the single-reduction
// kernels do; (U, CTAs/SM) the most CTAs/SM at which ptxas reports no spill for the four statistics (DESIGN §3.1)
// (the 16-bit wide shapes hold twice the columns per lane of fp32 ones, so they take fewer CTAs and gathers in flight)
template <typename T, bool PLAN>
static int dispatch_multi(const SpmmParams& p, const MultiOut& mo, cudaStream_t st) {
  constexpr bool W16 = sizeof(T) == 2;
  const int64_t vecs = p.K / Vec<T>::VEC;
  if (vecs <= 1) return launch_multi<T, 1, 1, 4, 2, true, PLAN>(p, mo, st);
  if (vecs <= 2) return launch_multi<T, 2, 1, 4, 2, true, PLAN>(p, mo, st);
  if (vecs <= 4) return launch_multi<T, 4, 1, 4, 2, true, PLAN>(p, mo, st);
  if (vecs <= 8) return launch_multi<T, 8, 1, 4, 2, true, PLAN>(p, mo, st);
  if (vecs <= 16) return launch_multi<T, 16, 1, 4, 2, false, PLAN>(p, mo, st);
  if (vecs <= 32) return launch_multi<T, 32, 1, 4, 2, false, PLAN>(p, mo, st);
  if (vecs <= 64) return launch_multi<T, 32, 2, 2, W16 ? 1 : 2, false, PLAN>(p, mo, st);
  return launch_multi<T, 32, 4, W16 ? 1 : 2, 1, false, PLAN>(p, mo, st);
}

}  // namespace tsb

using namespace tsb;

extern "C" size_t tsb200_spmm_fw_workspace_bytes(int64_t B, int64_t M, int64_t K, int64_t E, int dtype,
                                                 int reduce) {
  (void)M;
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return 0;
  if (B <= 0 || K <= 0 || E <= 0) return 0;
  return ws_layout(B, K, E, reduce == TSB200_MIN || reduce == TSB200_MAX).total;
}

extern "C" int tsb200_spmm_fw(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                              void* out, int64_t* arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                              int64_t E, int dtype, int reduce, void* workspace, size_t workspace_bytes,
                              void* stream) {
  if (B < 0 || M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if (reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  if (dtype_size(dtype) == 0) return TSB200_ERR_INVALID_ARG;
  const bool arg = (reduce == TSB200_MIN || reduce == TSB200_MAX);
  if (B * M * K == 0) return 0;  // nothing to write
  if (!rowptr || !out || (arg && !arg_out)) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col || !mat)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;

  if (E > 0 && vec_eligible(dtype, K, E, N, value, mat, out, col, arg_out)) {
    SpmmParams p{rowptr, col, value, mat, out, arg_out, B, M, N, K, E};
    if (const int rc = bind_unplanned(p, workspace, workspace_bytes, arg)) return rc;
    return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_red_vec<decltype(tag)>(p, reduce, st); });
  }

  return dispatch_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    switch (reduce) {
      case TSB200_SUM: return launch_generic<T, R_SUM>(rowptr, col, value, mat, out, arg_out, B, M, N, K, E, false, st);
      case TSB200_MEAN: return launch_generic<T, R_SUM>(rowptr, col, value, mat, out, arg_out, B, M, N, K, E, true, st);
      case TSB200_MIN: return launch_generic<T, R_MIN>(rowptr, col, value, mat, out, arg_out, B, M, N, K, E, false, st);
      case TSB200_MAX: return launch_generic<T, R_MAX>(rowptr, col, value, mat, out, arg_out, B, M, N, K, E, false, st);
    }
    return TSB200_ERR_INVALID_ARG;
  });
}

// One column block of a SUM SpMM whose blocks are launched separately (the dense operand arrives block by block):
// same kernels, the row results go through an fp32 partial instead of straight to `out`.
extern "C" int tsb200_spmm_fw_acc(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                  void* out, float* partial, int acc_mode, int64_t B, int64_t M, int64_t N,
                                  int64_t K, int64_t E, int dtype, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  if (B < 0 || M < 0 || N < 0 || K < 0 || E <= 0) return TSB200_ERR_INVALID_ARG;
  if (acc_mode < 1 || acc_mode > 3 || !partial || !rowptr || !col || !mat) return TSB200_ERR_INVALID_ARG;
  if (acc_mode == 3 && !out) return TSB200_ERR_INVALID_ARG;
  if (B * M * K == 0) return 0;
  if (((uintptr_t)partial & 15) || (K & 3)) return TSB200_ERR_UNSUPPORTED;
  // `out` is only dereferenced by the last block; alignment is checked against the partial for the others
  if (!vec_eligible(dtype, K, E, N, value, mat, acc_mode == 3 ? out : (void*)partial, col, nullptr))
    return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  SpmmParams p{rowptr, col, value, mat, out, nullptr, B, M, N, K, E};
  p.partial = partial; p.acc_mode = acc_mode;
  if (const int rc = bind_unplanned(p, workspace, workspace_bytes, false)) return rc;
  return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_shape<decltype(tag), R_SUM, true>(p, st); });
}

// ---- planned SpMM: the segment structure of a matrix is computed once and reused by every product --------------
extern "C" size_t tsb200_spmm_plan_bytes(int64_t M, int64_t E) {
  if (M < 0 || E < 0) return 0;
  return plan_layout(M, E).total;
}

extern "C" int tsb200_spmm_plan(const int64_t* rowptr, int64_t M, int64_t E, void* plan, size_t plan_bytes,
                                int64_t* counts_host, void* stream) {
  if (M < 0 || E < 0 || !rowptr || !plan) return TSB200_ERR_INVALID_ARG;
  const PlanLayout L = plan_layout(M, E);
  if (plan_bytes < L.total) return TSB200_ERR_WORKSPACE;
  if ((uintptr_t)plan & 255) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  char* pl = (char*)plan;
  TSB_CUDA_TRY(cudaMemsetAsync(pl + L.header, 0, 256, st));
  if (M > 0) {
    spmm_plan_kernel<<<warp_grid((M + 31) / 32, 16), 256, 0, st>>>(
        rowptr, M, (uint32_t*)(pl + L.mask), (Segment*)(pl + L.segs), (uint32_t*)(pl + L.seg_lr),
        (LongRow*)(pl + L.longs), (unsigned int*)(pl + L.header), L.seg_cap, L.long_cap);
    TSB_LAUNCH_CHECK();
  }
  if (counts_host) {  // [n_seg, n_long, n_slot] as uint32 counters 1..3 of the header; the caller widens them
    unsigned int h[4] = {0, 0, 0, 0};
    TSB_CUDA_TRY(cudaMemcpyAsync(h, pl + L.header, 16, cudaMemcpyDeviceToHost, st));
    TSB_CUDA_TRY(cudaStreamSynchronize(st));
    counts_host[0] = h[1];
    counts_host[1] = h[2];
    counts_host[2] = h[3];
  }
  return 0;
}

extern "C" size_t tsb200_spmm_fw_planned_workspace_bytes(int64_t K, int64_t n_long, int64_t n_slot, int reduce) {
  if (K < 0 || n_long < 0 || n_slot < 0) return 0;
  return planned_ws(K, n_long, n_slot, reduce == TSB200_MIN || reduce == TSB200_MAX).total;
}

extern "C" int tsb200_spmm_fw_planned(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                      void* out, int64_t* arg_out, int64_t M, int64_t N, int64_t K, int64_t E,
                                      int dtype, int reduce, const void* plan, size_t plan_bytes, int64_t n_seg,
                                      int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  if (M < 0 || N < 0 || K < 0 || E <= 0 || n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  const bool arg = (reduce == TSB200_MIN || reduce == TSB200_MAX);
  if (M * K == 0) return 0;
  if (!rowptr || !col || !mat || !out || !plan || (arg && !arg_out)) return TSB200_ERR_INVALID_ARG;
  if (!vec_eligible(dtype, K, E, N, value, mat, out, col, arg_out)) return TSB200_ERR_UNSUPPORTED;
  SpmmParams p{rowptr, col, value, mat, out, arg_out, 1, M, N, K, E};
  if (const int rc = bind_workspace(p, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, arg))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_red_vec<decltype(tag), true>(p, reduce, st); });
}

// ---- SpMM over an fp8 (e4m3) dense operand with per-tensor or per-row scales ----------------------------------------
// The same kernels, instantiated with X = __nv_fp8_e4m3: value / output type T = out_dtype, a dense row is K bytes.
// out_scale != NULL: e4m3 result with per-row scales (tsb200_spmm_fw_fp8_quant): T = float, `out` is e4m3 [M, K].
// res8 != NULL: plus an e4m3 residual with its own scales (tsb200_spmm_fw_fp8_res): the RES instantiations, sum / mean.
namespace tsb {
__global__ void fill_f32_kernel(float* __restrict__ p, int64_t n, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// An empty matrix with a residual: every row is y = +0, so the result is z = fl32(+0 + rho) (a -0 residual gives +0).
// One warp per row; an e4m3 result takes the row amax of z first (K <= 2048), then writes z / scale.
template <typename T, bool QO>
__global__ void __launch_bounds__(256) spmm_res_only_kernel(const SpmmParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t m = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < p.M; m += nw) {
    const float rs = res_scale(p, m);
    const uint8_t* r = res_at<__nv_fp8_e4m3>(p, m, 0);
    if constexpr (QO) {
      float amax = 0.f;
      for (int64_t k = lane; k < p.K; k += 32) amax = amax_nan(amax, fabsf(res_add(0.f, rs, e4m3_to_f32(__ldcs(r + k)))));
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) amax = amax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, off));
      const float s = e4m3_row_scale(amax);
      if (lane == 0) p.out_scale[m] = s;
      for (int64_t k = lane; k < p.K; k += 32) ((uint8_t*)p.out)[m * p.K + k] = e4m3_quant(res_add(0.f, rs, e4m3_to_f32(r[k])), s);
    } else {
      for (int64_t k = lane; k < p.K; k += 32)
        ((T*)p.out)[m * p.K + k] = Traits<T>::from_acc(res_add(0.f, rs, e4m3_to_f32(__ldcs(r + k))));
    }
  }
}

template <bool PLAN, bool QO, bool RES = false>
static int dispatch_fp8_out(const SpmmParams& p, int out_dtype, int reduce, cudaStream_t st) {
  if constexpr (QO) return dispatch_red_vec<float, PLAN, __nv_fp8_e4m3, true, RES>(p, reduce, st);
  return dispatch_vec_dtype(out_dtype, [&](auto tag) {
    return dispatch_red_vec<decltype(tag), PLAN, __nv_fp8_e4m3, false, RES>(p, reduce, st);
  });
}
template <bool PLAN, bool QO>
static int dispatch_fp8_res(const SpmmParams& p, int out_dtype, int reduce, cudaStream_t st) {
  if (p.res) return dispatch_fp8_out<PLAN, QO, true>(p, out_dtype, reduce, st);
  return dispatch_fp8_out<PLAN, QO>(p, out_dtype, reduce, st);
}

template <typename T, bool QO>
static int launch_res_only(const SpmmParams& p, cudaStream_t st) {
  const int64_t blocks = min((p.M * 32 + 255) / 256, (int64_t)num_sms() * 16);
  spmm_res_only_kernel<T, QO><<<(int)blocks, 256, 0, st>>>(p);
  TSB_LAUNCH_CHECK();
  return 0;
}

// An empty matrix with a residual of the operand's type T, rows of a multiple of 16 bytes (tsb200_spmm_fw_res, E == 0):
// z = fl32(+0 + fl32(s * r)) rounded once to T, one 16-byte chunk of the residual and of the result per thread and step.
template <typename T>
__global__ void __launch_bounds__(256) spmm_res_only_vec_kernel(const SpmmParams p) {
  constexpr int VEC = Vec<T>::VEC;
  const int64_t per_row = p.K / VEC, n = p.M * per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / per_row;
    float f[VEC];
#pragma unroll
    for (int j = 0; j < VEC; j++) f[j] = 0.f;
    res_add_vec<T>(f, res_at<T>(p, m, (i - m * per_row) * VEC), res_scale(p, m));
    stg128_stream((T*)p.out + i * VEC, Vec<T>::pack(f));
  }
}

template <typename T>
static int launch_res_only_vec(const SpmmParams& p, cudaStream_t st) {
  const int64_t chunks = p.M * (p.K / Vec<T>::VEC);
  spmm_res_only_vec_kernel<T><<<(int)min((chunks + 255) / 256, (int64_t)num_sms() * 16), 256, 0, st>>>(p);
  TSB_LAUNCH_CHECK();
  return 0;
}

template <bool QO>
static int spmm_fw_fp8_impl(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                            const float* scale, int64_t scale_stride, void* out, float* out_scale, int64_t* arg_out,
                            int64_t M, int64_t N, int64_t K, int64_t E, int out_dtype, int reduce, const void* plan,
                            size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                            size_t workspace_bytes, void* stream, const uint8_t* res8, const float* res_scale,
                            int64_t res_stride) {
  if (M < 0 || N < 0 || K < 0 || E < 0 || n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  if (scale_stride != 0 && scale_stride != 1) return TSB200_ERR_INVALID_ARG;
  if (out_dtype != TSB200_F32 && out_dtype != TSB200_F16 && out_dtype != TSB200_BF16) return TSB200_ERR_UNSUPPORTED;
  if (K % 16 != 0) return TSB200_ERR_UNSUPPORTED;
  // e4m3 result: a row's amax is taken inside one column tile of the kernels (at most 2048 fp8 columns)
  if (QO && K > 2048) return TSB200_ERR_UNSUPPORTED;
  const bool arg = (reduce == TSB200_MIN || reduce == TSB200_MAX);
  if (M == 0 || (!QO && K == 0)) return 0;
  if (!rowptr || !out || (QO && !out_scale) || (arg && !arg_out)) return TSB200_ERR_INVALID_ARG;
  if (QO && ((uintptr_t)out_scale & 3)) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  SpmmParams p{rowptr, col, value, mat, out, arg_out, 1, M, N, K, E};
  p.scale = scale; p.scale_stride = (uint32_t)scale_stride;
  p.out_scale = out_scale;
  p.res = res8; p.res_scale = res_scale; p.res_stride = (uint32_t)res_stride;
  if (res8) {
    if (!res_scale || (res_stride != 0 && res_stride != 1)) return TSB200_ERR_INVALID_ARG;
    if (arg) return TSB200_ERR_UNSUPPORTED;
    if (((uintptr_t)res8 & 15) || ((uintptr_t)res_scale & 3)) return TSB200_ERR_UNSUPPORTED;
    if (E == 0 && K > 0) {  // every row is empty: the result is the residual alone
      if ((uintptr_t)out & 15) return TSB200_ERR_UNSUPPORTED;
      if constexpr (QO) return launch_res_only<float, true>(p, st);
      return dispatch_vec_dtype(out_dtype, [&](auto tag) { return launch_res_only<decltype(tag), false>(p, st); });
    }
  }
  if (E == 0 || K == 0) {  // every row is empty: 0, arg_out = E = 0, and a scale of 1 (an amax of 0)
    if (K > 0) {
      TSB_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)(M * K) * (QO ? 1 : dtype_size(out_dtype)), st));
      if (arg) TSB_CUDA_TRY(cudaMemsetAsync(arg_out, 0, (size_t)(M * K) * sizeof(int64_t), st));
    }
    if (QO) {
      fill_f32_kernel<<<(int)min((M + 255) / 256, (int64_t)num_sms() * 8), 256, 0, st>>>(out_scale, M, 1.f);
      TSB_LAUNCH_CHECK();
    }
    return 0;
  }
  if (!col || !mat || !scale) return TSB200_ERR_INVALID_ARG;
  if (!rowsplit_extents(E, N, K) || !rowsplit_aligned({mat, out, arg_out}, col, {value, scale}))
    return TSB200_ERR_UNSUPPORTED;
  if (!workspace || ((uintptr_t)workspace & 255)) return TSB200_ERR_INVALID_ARG;
  // the workspace layouts of tsb200_spmm_fw_planned and, without a plan, tsb200_spmm_fw
  if (const int rc = bind_workspace(p, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, arg))
    return rc;
  return plan ? dispatch_fp8_res<true, QO>(p, out_dtype, reduce, st)
              : dispatch_fp8_res<false, QO>(p, out_dtype, reduce, st);
}
}  // namespace tsb

extern "C" int tsb200_spmm_fw_fp8(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                  const float* scale, int64_t scale_stride, void* out, int64_t* arg_out, int64_t M,
                                  int64_t N, int64_t K, int64_t E, int out_dtype, int reduce, const void* plan,
                                  size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return spmm_fw_fp8_impl<false>(rowptr, col, value, mat, scale, scale_stride, out, nullptr, arg_out, M, N, K, E,
                                 out_dtype, reduce, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes,
                                 stream, nullptr, nullptr, 0);
}

extern "C" int tsb200_spmm_fw_fp8_quant(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                        const float* scale, int64_t scale_stride, void* out8, float* out_scale,
                                        int64_t* arg_out, int64_t M, int64_t N, int64_t K, int64_t E, int reduce,
                                        const void* plan, size_t plan_bytes, int64_t n_seg, int64_t n_long,
                                        int64_t n_slot, void* workspace, size_t workspace_bytes, void* stream) {
  return spmm_fw_fp8_impl<true>(rowptr, col, value, mat, scale, scale_stride, out8, out_scale, arg_out, M, N, K, E,
                                TSB200_F32, reduce, plan, plan_bytes, n_seg, n_long, n_slot, workspace,
                                workspace_bytes, stream, nullptr, nullptr, 0);
}

extern "C" int tsb200_spmm_fw_fp8_res(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                      const float* scale, int64_t scale_stride, const void* res8,
                                      const float* res_scale, int64_t res_scale_stride, void* out, float* out_scale,
                                      int64_t* arg_out, int64_t M, int64_t N, int64_t K, int64_t E, int out_dtype,
                                      int reduce, const void* plan, size_t plan_bytes, int64_t n_seg, int64_t n_long,
                                      int64_t n_slot, void* workspace, size_t workspace_bytes, void* stream) {
  if (out_scale) {
    if (out_dtype != TSB200_F32) return TSB200_ERR_INVALID_ARG;  // an e4m3 result takes float32 values
    return spmm_fw_fp8_impl<true>(rowptr, col, value, mat, scale, scale_stride, out, out_scale, arg_out, M, N, K, E,
                                  TSB200_F32, reduce, plan, plan_bytes, n_seg, n_long, n_slot, workspace,
                                  workspace_bytes, stream, (const uint8_t*)res8, res_scale, res_scale_stride);
  }
  return spmm_fw_fp8_impl<false>(rowptr, col, value, mat, scale, scale_stride, out, nullptr, arg_out, M, N, K, E,
                                 out_dtype, reduce, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes,
                                 stream, (const uint8_t*)res8, res_scale, res_scale_stride);
}

// ---- SpMM with a residual of the operand's type (tsb200_spmm_fw_res) ------------------------------------------------
// The sum kernels with RES over a T operand (F32 / F16 / BF16 on the vector path, with a 16-byte aligned residual): each
// storing lane adds the 16-byte chunk of the residual row under its own result chunk. E == 0 on the same condition runs
// the residual-only vector kernel (also the one-pass s * g of the residual's gradient). Everything else runs the
// generic kernel with RES, whose +0 sum of an empty row gives the same z = fl(+0 + rho).
// The definition takes its C linkage from the declaration in tsb200.h (see the guard below).
int tsb200_spmm_fw_res(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat, const void* res,
                       const void* res_scale, int64_t res_scale_stride, void* out, int64_t M, int64_t N, int64_t K,
                       int64_t E, int dtype, int reduce, const void* plan, size_t plan_bytes, int64_t n_seg,
                       int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes, void* stream) {
  if (M < 0 || N < 0 || K < 0 || E < 0 || n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  if (dtype_size(dtype) == 0) return TSB200_ERR_INVALID_ARG;
  if (res_scale_stride != 0 && res_scale_stride != 1) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F64 && dtype != TSB200_F16 && dtype != TSB200_BF16)
    return TSB200_ERR_UNSUPPORTED;
  if (reduce == TSB200_MIN || reduce == TSB200_MAX) return TSB200_ERR_UNSUPPORTED;
  if (M * K == 0) return 0;  // nothing to write
  if (!rowptr || !out || !res || !res_scale) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col || !mat)) return TSB200_ERR_INVALID_ARG;
  if ((uintptr_t)res_scale & (dtype == TSB200_F64 ? 7 : 3)) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;

  if (vec_eligible(dtype, K, E, N, value, mat, out, col, nullptr) && !((uintptr_t)res & 15)) {
    SpmmParams p{rowptr, col, value, mat, out, nullptr, 1, M, N, K, E};
    p.res = res; p.res_scale = (const float*)res_scale; p.res_stride = (uint32_t)res_scale_stride;
    if (E == 0) return dispatch_vec_dtype(dtype, [&](auto tag) { return launch_res_only_vec<decltype(tag)>(p, st); });
    if (const int rc = bind_workspace(p, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, false))
      return rc;
    return dispatch_vec_dtype(dtype, [&](auto tag) {
      using T = decltype(tag);
      return plan ? dispatch_red_vec<T, true, T, false, true>(p, reduce, st)
                  : dispatch_red_vec<T, false, T, false, true>(p, reduce, st);
    });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    spmm_generic_kernel<T, R_SUM, true><<<warp_grid(M, 64), 256, 0, st>>>(
        rowptr, col, (const T*)value, (const T*)mat, (T*)out, nullptr, 1, M, N, K, E, reduce == TSB200_MEAN,
        (const T*)res, res_scale, res_scale_stride);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}
// Were the definition above ever to drift from the declaration in tsb200.h, it would become a second, C++ overload and
// the exported C symbol would be left undefined: taking the address of an overload set does not compile.
[[maybe_unused]] static constexpr auto tsb200_spmm_fw_res_declared_once = &tsb200_spmm_fw_res;

// ---- SpMM with per-head weights (tsb200_spmm_heads) -------------------------------------------------------------
// The sum kernels with HEADS = true over x [N, H * D]; with value == NULL every weight is 1 and the product is the
// plain sum (tsb200_spmm_fw / tsb200_spmm_fw_planned over K = H * D columns).
extern "C" int tsb200_spmm_heads(const int64_t* rowptr, const int64_t* col, const void* value, const void* x, void* out,
                                 int64_t M, int64_t N, int64_t H, int64_t D, int64_t E, int dtype, const void* plan,
                                 size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (M < 0 || N < 0 || H < 0 || D < 0 || E < 0 || n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F64 && dtype != TSB200_F16 && dtype != TSB200_BF16)
    return TSB200_ERR_UNSUPPORTED;
  if (H > 0 && D > ((int64_t)1 << 40) / H) return TSB200_ERR_UNSUPPORTED;
  const int64_t K = H * D;
  if (M * K == 0) return 0;  // nothing to write
  if (!rowptr || !out) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (E == 0) {  // every row is empty: +0
    TSB_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)(M * K) * dtype_size(dtype), st));
    return 0;
  }
  if (!col || !x) return TSB200_ERR_INVALID_ARG;
  if (!value) {
    if (plan) return tsb200_spmm_fw_planned(rowptr, col, nullptr, x, out, nullptr, M, N, K, E, dtype, TSB200_SUM, plan,
                                            plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, stream);
    return tsb200_spmm_fw(rowptr, col, nullptr, x, out, nullptr, 1, M, N, K, E, dtype, TSB200_SUM, workspace,
                          workspace_bytes, stream);
  }
  const size_t es = dtype_size(dtype);
  if ((D * (int64_t)es) % 16 == 0 && vec_eligible(dtype, K, E, N, value, x, out, col, nullptr) &&
      H * E < ((int64_t)1 << 31)) {
    SpmmParams p{rowptr, col, value, x, out, nullptr, 1, M, N, K, E};
    p.heads = (int)H;
    if (const int rc = bind_workspace(p, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, false))
      return rc;
    return dispatch_vec_dtype(dtype, [&](auto tag) {
      using T = decltype(tag);
      return plan ? dispatch_heads<T, true>(p, st) : dispatch_heads<T, false>(p, st);
    });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    spmm_heads_generic_kernel<T><<<warp_grid(M, 64), 256, 0, st>>>(rowptr, col, (const T*)value, (const T*)x,
                                                                   (T*)out, M, H, D);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

// ---- multi-aggregation SpMM (tsb200_spmm_fw_multi) ------------------------------------------------------------------
// The definitions take their C linkage from the declarations in tsb200.h (see tsb200_spmm_fw_res and the guards below).
size_t tsb200_spmm_fw_multi_workspace_bytes(int64_t K, int64_t E, int planned, int64_t n_long, int64_t n_slot) {
  if (K <= 0 || E <= 0 || n_long < 0 || n_slot < 0) return 0;
  return multi_ws(K, E, planned != 0, n_long, n_slot).total;
}

int tsb200_spmm_fw_multi(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                         const int* aggrs, int n_aggr, void* out, int64_t* arg_min, int64_t* arg_max, int64_t M,
                         int64_t N, int64_t K, int64_t E, int dtype, const void* plan, size_t plan_bytes, int64_t n_seg,
                         int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes, void* stream) {
  if (M < 0 || N < 0 || K < 0 || E < 0 || n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (!aggrs || n_aggr < 1 || n_aggr > kStats) return TSB200_ERR_INVALID_ARG;
  MultiOut mo{arg_min, arg_max, n_aggr, {-1, -1, -1, -1, -1, -1}};
  for (int a = 0; a < n_aggr; a++) {
    const int c = aggrs[a];
    if (c < TSB200_SUM || c > TSB200_STD || mo.slice[c] >= 0) return TSB200_ERR_INVALID_ARG;
    mo.slice[c] = (int8_t)a;
  }
  if ((arg_min && mo.slice[R_MIN] < 0) || (arg_max && mo.slice[R_MAX] < 0)) return TSB200_ERR_INVALID_ARG;
  if (dtype_size(dtype) == 0) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F64 && dtype != TSB200_F16 && dtype != TSB200_BF16)
    return TSB200_ERR_UNSUPPORTED;
  if (M * K == 0) return 0;  // nothing to write
  if (!rowptr || !out) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col || !mat)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;

  if (E > 0 && vec_eligible(dtype, K, E, N, value, mat, out, col, arg_min) && !((uintptr_t)arg_max & 15)) {
    SpmmParams p{rowptr, col, value, mat, out, nullptr, 1, M, N, K, E};
    // the fp32 planes bound as a workspace of 4 * K partial columns, the arg planes behind them
    const MultiWs L = multi_ws(K, E, plan != nullptr, n_long, n_slot);
    SpmmParams q = p;
    q.K = 4 * K;
    if (const int rc = bind_workspace(q, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, false))
      return rc;
    if (workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
    q.K = K;
    q.part_arg = (int64_t*)((char*)workspace + L.args);
    return dispatch_vec_dtype(dtype, [&](auto tag) {
      using T = decltype(tag);
      return plan ? dispatch_multi<T, true>(q, mo, st) : dispatch_multi<T, false>(q, mo, st);
    });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    spmm_multi_generic_kernel<T><<<warp_grid(M, 64), 256, 0, st>>>(rowptr, col, (const T*)value, (const T*)mat,
                                                                   (T*)out, M, K, E, mo);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}
[[maybe_unused]] static constexpr auto tsb200_spmm_fw_multi_declared_once = &tsb200_spmm_fw_multi;
[[maybe_unused]] static constexpr auto tsb200_spmm_fw_multi_workspace_bytes_declared_once =
    &tsb200_spmm_fw_multi_workspace_bytes;
