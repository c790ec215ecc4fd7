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
//   * anything the vector path cannot take (K*sizeof(T) % 16 != 0, integer / fp64 types,
//     unaligned pointers, E >= 2^31) goes to a generic lane-per-column kernel that walks the
//     nnz sequentially exactly like csrc/cpu/spmm_cpu.cpp:75-88 (bit-identical for fp32/fp64).
#include "spmm_common.cuh"

namespace tsb {

template <typename T, int RED, int LPR, int CH, int U> struct RowEngine {
  using V = Vec<T>;
  static constexpr int VEC = V::VEC;
  static constexpr int G = 32 / LPR;
  static constexpr int NA = VEC * CH;
  static constexpr bool ARG = (RED == R_MIN || RED == R_MAX);

  float acc[NA];
  int arg[ARG ? NA : 1];

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

  // one step of the min/max update (compare on the product rounded to the storage type)
  __device__ __forceinline__ void minmax_step(float* a, int* ar, typename V::vraw v, const uint4& d, int jabs) {
    float f[VEC];
    V::unpack(d, f);
    const float vf = V::vfloat(v);
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
      if (jend - j0 == U * G) {  // full chunk: every lane group has work in every step
#pragma unroll
        for (int u = 0; u < U; u++) {
          const uint32_t c = pc[2 * u * G];
          v[u] = pv[u * G];
          const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
          for (int ch = 0; ch < CH; ch++)
            if (col_ok[ch]) d[u][ch] = ldg128_hint(src + ch * (LPR * 16), pol);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (!col_ok[ch]) continue;
            if (RED == R_SUM) V::fma(&acc[ch * VEC], v[u], d[u][ch]);
            else minmax_step(&acc[ch * VEC], &arg[ch * VEC], v[u], d[u][ch], jabs0 + u * G);
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
          for (int ch = 0; ch < CH; ch++) {
            if (!(act[u] && col_ok[ch])) continue;
            if (RED == R_SUM) V::fma(&acc[ch * VEC], v[u], d[u][ch]);
            else minmax_step(&acc[ch * VEC], &arg[ch * VEC], v[u], d[u][ch], jabs0 + u * G);
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

  // final write of one row (group 0 lanes). count = row degree.
  __device__ __forceinline__ void store_row(T* __restrict__ out_row, int64_t* __restrict__ arg_row,
                                            int64_t count, int64_t E, const bool (&col_ok)[CH], int li,
                                            bool mean, float* __restrict__ part_row = nullptr, int acc_mode = 0) {
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
      stg128_stream(out_row + koff, V::pack(f));
      if (ARG) {
#pragma unroll
        for (int i = 0; i < VEC; i += 2) {
          longlong2 a2;
          a2.x = (count > 0 && arg[ch * VEC + i] != 0x7fffffff) ? (int64_t)arg[ch * VEC + i] : E;
          a2.y = (count > 0 && arg[ch * VEC + i + 1] != 0x7fffffff) ? (int64_t)arg[ch * VEC + i + 1] : E;
          stg128_stream(arg_row + koff + i, *reinterpret_cast<uint4*>(&a2));
        }
      }
    }
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

  __device__ __forceinline__ void store_row(T* __restrict__ out_row, int64_t* __restrict__ arg_row,
                                            int64_t count, int64_t E, const bool (&col_ok)[CH], int li, bool,
                                            float* = nullptr, int = 0) {
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
      uint4 o = make_uint4(pacc[ch * 4], pacc[ch * 4 + 1], pacc[ch * 4 + 2], pacc[ch * 4 + 3]);
      if (count == 0) o = make_uint4(0, 0, 0, 0);
      stg128_stream(out_row + koff, o);
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        longlong2 a2;
        a2.x = (count > 0 && arg[ch * VEC + i] != 0x7fffffff) ? (int64_t)arg[ch * VEC + i] : E;
        a2.y = (count > 0 && arg[ch * VEC + i + 1] != 0x7fffffff) ? (int64_t)arg[ch * VEC + i + 1] : E;
        stg128_stream(arg_row + koff + i, *reinterpret_cast<uint4*>(&a2));
      }
    }
  }
};

template <typename T, int RED, int LPR, int CH, int U> struct EngineFor {
  using type = typename std::conditional<(RED != R_SUM && is_float16<T>::value), MinMax16Engine<T, RED, LPR, CH, U>,
                                         RowEngine<T, RED, LPR, CH, U>>::type;
};

// combine the partials of one multi-segment row, in segment order, by ONE WARP (planned mode: the warp that finished
// the row's last segment); the partials were written by other SMs -> read them past L1
template <typename T, int RED>
__device__ __forceinline__ void combine_row_warp(const SpmmParams& p, const LongRow& L, int lane, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int nseg = (int)(L.nseg_count >> 40);
  const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
  for (int k = lane; k < kcols; k += 32) {
    const int64_t kk = p.k0 + k;
    if (kk >= p.K) break;
    float a = __ldcg((const float*)p.part_val + L.first_slot * p.K + kk);
    int64_t ar = ARG ? __ldcg(p.part_arg + L.first_slot * p.K + kk) : 0;
    for (int sgi = 1; sgi < nseg; sgi++) {
      const float v = __ldcg((const float*)p.part_val + (L.first_slot + sgi) * p.K + kk);
      if (RED == R_SUM) a += v;
      else {
        const int64_t va = __ldcg(p.part_arg + (L.first_slot + sgi) * p.K + kk);
        const bool better = (RED == R_MIN) ? (v < a) : (v > a);
        if (better || (v == a && va < ar)) { a = v; ar = va; }
      }
    }
    if (RED == R_SUM && p.mean) a = a / (float)(count > 0 ? count : 1);
    ((T*)p.out)[L.row_b * p.K + kk] = Traits<T>::from_acc(a);
    if (ARG) p.arg_out[L.row_b * p.K + kk] = ar;
  }
}

template <typename T, int RED, int LPR, int CH, int U, int MINB, bool ACC = false, bool PLAN = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_vec_kernel(const SpmmParams p) {
  using Eng = typename EngineFor<T, RED, LPR, CH, U>::type;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.s_col = s_col[warp];
  ring.s_val = s_val[warp];
  ring.has_val = p.value != nullptr;
  if (!ring.has_val) {  // has_value=false: the ring's value half is a constant 1
    using VR = typename Vec<T>::vraw;
    for (int i = lane; i < kRingAlloc; i += 32) reinterpret_cast<VR*>(s_val[warp])[i] = Vec<T>::one();
    __syncwarp();
  }
  ring.col = p.col;
  ring.val = (const T*)p.value;
  ring.limit = p.E;
  const uint64_t pol = make_policy_evict_last();

  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = p.k0 + (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(T);

  const int item_rows = 1 << p.item_shift;
  const int64_t nblk = (p.M + item_rows - 1) >> p.item_shift;
  const int64_t n_items = nblk * p.B;

  unsigned int item = 0;
  if (lane == 0) item = atomicAdd(&p.counters[0], 1u);
  item = __shfl_sync(0xffffffffu, item, 0);

  while ((int64_t)item < n_items) {
    unsigned int next_item = 0;
    if (lane == 0) next_item = atomicAdd(&p.counters[0], 1u);  // latency hidden behind this item

    const int64_t b = item / nblk, blk = item - b * nblk;
    const int64_t r0 = blk << p.item_shift;
    const int nrows = (int)min((int64_t)item_rows, p.M - r0);
    const int64_t rp0 = __ldg(p.rowptr + r0 + min(lane, nrows));
    const int64_t rp1 = __ldg(p.rowptr + r0 + min(lane + 1, nrows));
    const int64_t a0 = __shfl_sync(0xffffffffu, rp0, 0);
    const int64_t base = a0 & ~(int64_t)31;
    const int s_rel = (int)(rp0 - base), e_rel = (int)(rp1 - base);
    const int deg = e_rel - s_rel;

    unsigned defer_mask;
    if constexpr (PLAN) {  // which rows are in the segment list was decided when the plan was built
      const uint32_t w = __ldg(p.plan_mask + (r0 >> 5));
      defer_mask = (w >> (r0 & 31)) & (nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u));
    } else {
      // nnz budget: prefix sum of the degrees of the non-long rows
      const bool is_long = deg > kLongT;
      int cum = is_long ? 0 : deg;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, cum, off);
        if (lane >= off) cum += t;
      }
      const bool defer = (deg > 0) && (is_long || cum > kItemCap);
      defer_mask = __ballot_sync(0xffffffffu, defer);

      if (defer) {  // rare: push this row's segments
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
    }
    __syncwarp();

    ring.reset(base, __shfl_sync(0xffffffffu, rp1, 31));  // lanes >= nrows hold the item's end
    const char* matb = (const char*)p.mat + b * p.N * (int64_t)row_bytes + lane_off;
    asm volatile("" : "+l"(matb));  // keep the gather base in a register
    T* outb = (T*)p.out + (b * p.M + r0) * p.K + p.k0;
    int64_t* argb = p.arg_out ? p.arg_out + (b * p.M + r0) * p.K + p.k0 : nullptr;
    float* partb = ACC ? p.partial + (b * p.M + r0) * p.K + p.k0 : nullptr;

    for (int rl = 0; rl < nrows; rl++) {
      if ((defer_mask >> rl) & 1u) continue;
      const int s = __shfl_sync(0xffffffffu, s_rel, rl);
      const int e = __shfl_sync(0xffffffffu, e_rel, rl);
      Eng eng;
      eng.init();
      eng.accumulate(ring, s, e, matb, row_bytes, col_ok, lane, g, pol);
      eng.reduce_groups();
      if (g == 0) eng.store_row(outb + (int64_t)rl * p.K, argb ? argb + (int64_t)rl * p.K : nullptr, e - s, p.E, col_ok, li, p.mean != 0,
                                ACC ? partb + (int64_t)rl * p.K : nullptr, ACC ? p.acc_mode : 0);
    }
    item = __shfl_sync(0xffffffffu, next_item, 0);
  }

  if constexpr (PLAN) {
    // Planned mode: the row items are gone — this warp now takes segments of the long / over-budget rows from the
    // plan's list (all of them exist already: a ticket counter is the whole protocol). A multi-segment row is
    // combined by whichever warp finishes its last segment (counter per long row + fences, no waiting).
    constexpr int kcols = LPR * CH * VEC;
    while (true) {
      unsigned int sidx = 0;
      if (lane == 0) sidx = atomicAdd(&p.counters[5], 1u);
      sidx = __shfl_sync(0xffffffffu, sidx, 0);
      if ((int64_t)sidx >= p.n_seg) break;
      const Segment S = p.segs[sidx];
      const int64_t row = S.row_b;  // B == 1
      const int64_t base = S.start & ~(int64_t)31;
      ring.reset(base, S.end);
      const char* matb = (const char*)p.mat + lane_off;
      asm volatile("" : "+l"(matb));
      Eng eng;
      eng.init();
      eng.accumulate(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, pol);
      eng.reduce_groups();
      if (S.slot < 0) {
        if (g == 0)
          eng.store_row((T*)p.out + row * p.K + p.k0, p.arg_out ? p.arg_out + row * p.K + p.k0 : nullptr,
                        S.end - S.start, p.E, col_ok, li, p.mean != 0);
      } else {
        if (g == 0) {
          float* pv = (float*)p.part_val + S.slot * p.K + p.k0;
          int64_t* pa = Eng::ARG ? p.part_arg + S.slot * p.K + p.k0 : nullptr;
#pragma unroll
          for (int ch = 0; ch < CH; ch++) {
            if (!col_ok[ch]) continue;
            const int koff = (ch * LPR + li) * VEC;
#pragma unroll
            for (int i = 0; i < VEC; i++) {
              pv[koff + i] = eng.acc_float(ch * VEC + i);
              if (Eng::ARG) pa[koff + i] = eng.arg[ch * VEC + i] == 0x7fffffff ? p.E : (int64_t)eng.arg[ch * VEC + i];
            }
          }
        }
        __syncwarp();
        __threadfence();  // this segment's partial is visible before its completion is counted
        const uint32_t lr = __ldg(p.seg_lr + sidx);
        unsigned int finished = 0;
        if (lane == 0) finished = atomicAdd(&p.long_done[lr], 1u);
        finished = __shfl_sync(0xffffffffu, finished, 0);
        const LongRow L = p.longs[lr];
        if ((int)finished == (int)(L.nseg_count >> 40) - 1) {
          __threadfence();
          combine_row_warp<T, RED>(p, L, lane, kcols);
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
template <typename T> __device__ __forceinline__ typename Vec<T>::vraw load_vraw(const T* p);
template <> __device__ __forceinline__ float load_vraw<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ unsigned short load_vraw<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __ldg(reinterpret_cast<const unsigned short*>(p));
}
template <> __device__ __forceinline__ unsigned short load_vraw<__half>(const __half* p) {
  return __ldg(reinterpret_cast<const unsigned short*>(p));
}

template <typename T, int RED, int LPR, int U, int MINB, bool ACC = false, bool PLAN = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_gpr_kernel(const SpmmParams p) {
  using V = Vec<T>;
  using Eng = typename EngineFor<T, RED, LPR, 1, U>::type;  // per-lane state + update + store of one row
  using VR = typename V::vraw;
  constexpr int VEC = V::VEC;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  const bool col_ok = p.k0 + li * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(T);
  const uint64_t pol = make_policy_evict_last();
  const T* __restrict__ val = (const T*)p.value;
  const bool has_val = val != nullptr;

  const int item_rows = 1 << p.item_shift;
  const int64_t nblk = (p.M + item_rows - 1) >> p.item_shift;
  const int64_t n_items = nblk * p.B;

  unsigned int item = 0;
  if (lane == 0) item = atomicAdd(&p.counters[0], 1u);
  item = __shfl_sync(0xffffffffu, item, 0);

  while ((int64_t)item < n_items) {
    unsigned int next_item = 0;
    if (lane == 0) next_item = atomicAdd(&p.counters[0], 1u);

    const int64_t b = item / nblk, blk = item - b * nblk;
    const int64_t r0 = blk << p.item_shift;
    const int nrows = (int)min((int64_t)item_rows, p.M - r0);
    const int64_t rp0 = __ldg(p.rowptr + r0 + min(lane, nrows));
    const int64_t rp1 = __ldg(p.rowptr + r0 + min(lane + 1, nrows));
    const int64_t base = __shfl_sync(0xffffffffu, rp0, 0);
    const int s_rel = (int)(rp0 - base), e_rel = (int)(rp1 - base);
    const int deg = e_rel - s_rel;

    unsigned defer_mask;
    if constexpr (PLAN) {
      const uint32_t w = __ldg(p.plan_mask + (r0 >> 5));
      defer_mask = (w >> (r0 & 31)) & (nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u));
    } else {
      const bool is_long = deg > kLongT;
      int cum = is_long ? 0 : deg;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, cum, off);
        if (lane >= off) cum += t;
      }
      const bool defer = (deg > 0) && (is_long || cum > kItemCap);
      defer_mask = __ballot_sync(0xffffffffu, defer);
      if (defer) {
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
    
    }
    __syncwarp();

    const char* matb = (const char*)p.mat + b * p.N * (int64_t)row_bytes + lane_off;
    asm volatile("" : "+l"(matb));
    const int64_t* __restrict__ colb = p.col + base;
    const T* __restrict__ valb = has_val ? val + base : nullptr;
    T* outb = (T*)p.out + (b * p.M + r0) * p.K + p.k0;
    int64_t* argb = p.arg_out ? p.arg_out + (b * p.M + r0) * p.K + p.k0 : nullptr;
    float* partb = ACC ? p.partial + (b * p.M + r0) * p.K + p.k0 : nullptr;
    const bool col_ok_arr[1] = {col_ok};
    const int jbase = (int)base;  // absolute nnz index of ring-relative 0 (E < 2^31)

    for (int t = 0; t < nrows; t += G) {
      const int rl = t + g;  // this lane group's row
      int s = __shfl_sync(0xffffffffu, s_rel, rl & 31);
      int e = __shfl_sync(0xffffffffu, e_rel, rl & 31);
      const bool mine = rl < nrows && !((defer_mask >> (rl & 31)) & 1u);
      if (!mine) e = s;
      const int len = e - s;
      int maxlen = len;
#pragma unroll
      for (int off = LPR; off < 32; off <<= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, off));

      Eng eng;
      eng.init();

      // software pipeline: the (col, value) pairs of chunk k+1 are loaded while chunk k's gathers fly
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
        for (int u = 0; u < U; u++) {
          if (!act[u]) continue;
          if constexpr (RED == R_SUM) V::fma(eng.acc, v[u], d[u]);
          else if constexpr (is_float16<T>::value) eng.vec_step(0, v[u], d[u], jbase + s + j0 + u);
          else eng.minmax_step(eng.acc, eng.arg, v[u], d[u], jbase + s + j0 + u);
        }
      }
      if (mine) eng.store_row(outb + (int64_t)rl * p.K, argb ? argb + (int64_t)rl * p.K : nullptr, len, p.E, col_ok_arr, li,
                              p.mean != 0, ACC ? partb + (int64_t)rl * p.K : nullptr, ACC ? p.acc_mode : 0);
    }
    item = __shfl_sync(0xffffffffu, next_item, 0);
  }
}

// one warp per queued segment
template <typename T, int RED, int LPR, int CH, int U, int MINB, bool ACC = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_seg_kernel(const SpmmParams p) {
  using Eng = typename EngineFor<T, RED, LPR, CH, U>::type;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  __shared__ __align__(16) T s_val[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.s_col = s_col[warp];
  ring.s_val = s_val[warp];
  ring.has_val = p.value != nullptr;
  if (!ring.has_val) {  // has_value=false: the ring's value half is a constant 1
    using VR = typename Vec<T>::vraw;
    for (int i = lane; i < kRingAlloc; i += 32) reinterpret_cast<VR*>(s_val[warp])[i] = Vec<T>::one();
    __syncwarp();
  }
  ring.col = p.col;
  ring.val = (const T*)p.value;
  ring.limit = p.E;
  const uint64_t pol = make_policy_evict_last();

  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = p.k0 + (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(T);

  const int64_t nseg = p.plan_mask ? p.n_seg : min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    const int64_t b = S.row_b / p.M, row = S.row_b - b * p.M;
    const int64_t base = S.start & ~(int64_t)31;
    ring.reset(base, S.end);
    const char* matb = (const char*)p.mat + b * p.N * (int64_t)row_bytes + lane_off;
    asm volatile("" : "+l"(matb));
    Eng eng;
    eng.init();
    eng.accumulate(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, pol);
    eng.reduce_groups();
    if (g == 0) {
      if (S.slot < 0) {
        eng.store_row((T*)p.out + (b * p.M + row) * p.K + p.k0,
                      p.arg_out ? p.arg_out + (b * p.M + row) * p.K + p.k0 : nullptr,
                      S.end - S.start, p.E, col_ok, li, p.mean != 0,
                      ACC ? p.partial + (b * p.M + row) * p.K + p.k0 : nullptr, ACC ? p.acc_mode : 0);
      } else {
        float* pv = (float*)p.part_val + S.slot * p.K + p.k0;
        int64_t* pa = Eng::ARG ? p.part_arg + S.slot * p.K + p.k0 : nullptr;
#pragma unroll
        for (int ch = 0; ch < CH; ch++) {
          if (!col_ok[ch]) continue;
          const int koff = (ch * LPR + li) * VEC;
#pragma unroll
          for (int i = 0; i < VEC; i++) {
            pv[koff + i] = eng.acc_float(ch * VEC + i);
            if (Eng::ARG) pa[koff + i] = eng.arg[ch * VEC + i] == 0x7fffffff ? p.E : (int64_t)eng.arg[ch * VEC + i];
          }
        }
      }
    }
    __syncwarp();
  }
}

// combine the partials of multi-segment rows, in segment order.
template <typename T, int RED>
__global__ void spmm_combine_kernel(const SpmmParams p, int kcols) {
  constexpr bool ARG = (RED == R_MIN || RED == R_MAX);
  const int64_t nlong = p.plan_mask ? p.n_long : min((int64_t)p.counters[2], p.long_cap);
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    const int nseg = (int)(L.nseg_count >> 40);
    const int64_t count = L.nseg_count & (((int64_t)1 << 40) - 1);
    for (int k = threadIdx.x; k < kcols; k += blockDim.x) {
      const int64_t kk = p.k0 + k;
      if (kk >= p.K) break;
      float a = ((const float*)p.part_val)[L.first_slot * p.K + kk];
      int64_t ar = ARG ? p.part_arg[L.first_slot * p.K + kk] : 0;
      for (int sgi = 1; sgi < nseg; sgi++) {
        const float v = ((const float*)p.part_val)[(L.first_slot + sgi) * p.K + kk];
        if (RED == R_SUM) a += v;
        else {
          const int64_t va = p.part_arg[(L.first_slot + sgi) * p.K + kk];
          const bool better = (RED == R_MIN) ? (v < a) : (v > a);
          if (better || (v == a && va < ar)) { a = v; ar = va; }
        }
      }
      if (RED == R_SUM && p.mean) a = a / (float)(count > 0 ? count : 1);
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

// ---- generic fallback: warp per (b,row), lane per column, sequential nnz walk -------------------
template <typename T, int RED>
__global__ void __launch_bounds__(256)
spmm_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                    const T* __restrict__ value, const T* __restrict__ mat, T* __restrict__ out,
                    int64_t* __restrict__ arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                    int64_t E, bool mean) {
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
      out[i * K + k] = Traits<T>::from_acc(a);
      if (ARG) arg_out[i * K + k] = cnt > 0 ? ar : E;
    }
  }
}

// ---- dispatch ------------------------------------------------------------------------------------
static bool vec_eligible(int dtype, int64_t K, int64_t E, int64_t N, const void* value,
                         const void* mat, const void* out, const void* col, const void* arg_out) {
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return false;
  const size_t es = dtype_size(dtype);
  if ((K * es) % 16 != 0) return false;
  if (E >= ((int64_t)1 << 31) - 64) return false;
  if (N >= ((int64_t)1 << 32) || K * (int64_t)es >= ((int64_t)1 << 31)) return false;
  if (((uintptr_t)mat & 15) || ((uintptr_t)out & 15) || ((uintptr_t)col & 7)) return false;
  if (value && ((uintptr_t)value & 3)) return false;
  if (arg_out && ((uintptr_t)arg_out & 15)) return false;
  return true;
}

template <typename T, int RED, bool ACC, int LPR, int CH, int U, int MINB = 1, bool GPR = false, bool PLAN = false>
static int launch_vec(SpmmParams p, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  constexpr int kcols = LPR * CH * VEC;
  void (*kmain)(const SpmmParams);
  if constexpr (GPR) kmain = spmm_gpr_kernel<T, RED, LPR, U, MINB, ACC, PLAN>;
  else kmain = spmm_vec_kernel<T, RED, LPR, CH, U, MINB, ACC, PLAN>;
  constexpr int USEG = (U > LPR) ? LPR : U;  // the row engine needs U * (32 / LPR) <= 32
  auto* kseg = spmm_seg_kernel<T, RED, LPR, CH, USEG, MINB, ACC>;
  static GridCache gc_main, gc_seg;  // per instantiation, per device
  const int grid_main = gc_main.get((const void*)kmain, kWarpsPerCta * 32);
  // small matrices: shrink the work item so that every resident warp gets rows
  int64_t want = p.M * p.B / ((int64_t)grid_main * kWarpsPerCta * 2);
  p.item_shift = 0;
  while (p.item_shift < 5 && ((int64_t)2 << p.item_shift) <= want) p.item_shift++;
  const int64_t n_items = ((p.M + (1 << p.item_shift) - 1) >> p.item_shift) * p.B;
  for (int k0 = 0; k0 < p.K; k0 += kcols) {
    p.k0 = k0;
    if constexpr (PLAN) {
      // one memset (ticket counters + the per-long-row completion counters behind them), ONE kernel: the row items,
      // then the plan's segments, drained by the same warps. The group-per-row kernel has no index ring to drain
      // with, so for narrow dense rows the segment / combine kernels are still launched — when the plan says there
      // is something for them to do.
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
          spmm_combine_kernel<T, RED><<<num_sms() * 2, 128, 0, st>>>(p, kcols);
          TSB_LAUNCH_CHECK();
        }
      }
    } else {
      const int grid_seg = gc_seg.get((const void*)kseg, kWarpsPerCta * 32);
      TSB_CUDA_TRY(cudaMemsetAsync(p.counters, 0, 64, st));
      const int gm = (int)min((int64_t)grid_main, (n_items + kWarpsPerCta - 1) / kWarpsPerCta);
      kmain<<<gm, kWarpsPerCta * 32, 0, st>>>(p);
      TSB_LAUNCH_CHECK();
      kseg<<<grid_seg, kWarpsPerCta * 32, 0, st>>>(p);
      TSB_LAUNCH_CHECK();
      spmm_combine_kernel<T, RED><<<num_sms() * 2, 128, 0, st>>>(p, kcols);
      TSB_LAUNCH_CHECK();
    }
  }
  return 0;
}

// (LPR, CH) follow from the width of a dense row; (U, MINB) = gathers in flight per lane and CTAs
// per SM: the kernel is HBM-latency bound, so resident warps x gathers-in-flight wins (40 warps/SM x 4 x 16 B
// per lane; the register budget of MINB = 5 is the same 64K registers per SM on sm_90).
template <typename T, int RED, bool ACC = false, bool PLAN = false> static int dispatch_shape(const SpmmParams& p, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t vecs = p.K / VEC;  // 16-byte vectors per dense row
  // narrow rows: group-per-row kernel (all reductions)
  if (vecs <= 1) return launch_vec<T, RED, ACC, 1, 1, 4, 5, true, PLAN>(p, st);
  if (vecs <= 2) return launch_vec<T, RED, ACC, 2, 1, 4, 5, true, PLAN>(p, st);
  if (vecs <= 4) return launch_vec<T, RED, ACC, 4, 1, 4, 5, true, PLAN>(p, st);
  if (vecs <= 8) return launch_vec<T, RED, ACC, 8, 1, 4, 5, true, PLAN>(p, st);
  // 256-byte rows (F = 128 bf16): at MINB = 5 the 48-register budget spills (120 B of stack in the planned kernel);
  // 3 CTAs/SM with 6 gathers in flight per lane is 8 % faster at C2 on the H100 (sweep in DESIGN §3.1)
  if (vecs <= 16) return launch_vec<T, RED, ACC, 16, 1, 6, 3, false, PLAN>(p, st);
  if (vecs <= 32) return launch_vec<T, RED, ACC, 32, 1, 4, 5, false, PLAN>(p, st);
  if (vecs <= 64) return launch_vec<T, RED, ACC, 32, 2, 4, 3, false, PLAN>(p, st);
  return launch_vec<T, RED, ACC, 32, 4, 2, 3, false, PLAN>(p, st);  // column-tiled beyond 128 vectors
}

template <typename T, bool PLAN = false> static int dispatch_red_vec(SpmmParams p, int reduce, cudaStream_t st) {
  p.mean = (reduce == TSB200_MEAN);
  switch (reduce) {
    case TSB200_SUM:
    case TSB200_MEAN: return dispatch_shape<T, R_SUM, false, PLAN>(p, st);
    case TSB200_MIN: return dispatch_shape<T, R_MIN, false, PLAN>(p, st);
    case TSB200_MAX: return dispatch_shape<T, R_MAX, false, PLAN>(p, st);
  }
  return TSB200_ERR_INVALID_ARG;
}

// ---- plan: the segment list of a matrix, built once (tsb200_spmm_plan) -----------------------------------------
// One warp per group of 32 rows, the same rule as the unplanned main kernels (rows longer than kLongT nnz, and rows
// beyond the group's kItemCap-nnz budget, become <= kSeg-nnz segments); also leaves one mask word per group.
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
    const int deg = (int)min(deg64, (int64_t)0x3fffffff);
    const bool is_long = deg > kLongT;
    int cum = is_long ? 0 : deg;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, cum, off);
      if (lane >= off) cum += t;
    }
    const bool defer = (deg > 0) && (is_long || cum > kItemCap);
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

template <typename T, int RED>
static int launch_generic(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                          void* out, int64_t* arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                          int64_t E, bool mean, cudaStream_t st) {
  const int64_t warps = B * M;
  int64_t blocks = (warps + 7) / 8;
  if (blocks > (int64_t)num_sms() * 64) blocks = (int64_t)num_sms() * 64;
  if (blocks < 1) blocks = 1;
  spmm_generic_kernel<T, RED><<<(int)blocks, 256, 0, st>>>(rowptr, col, (const T*)value, (const T*)mat,
                                                           (T*)out, arg_out, B, M, N, K, E, mean);
  TSB_LAUNCH_CHECK();
  return 0;
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
    const WsLayout L = ws_layout(B, K, E, arg);
    if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
    if ((uintptr_t)workspace & 255) return TSB200_ERR_INVALID_ARG;
    char* ws = (char*)workspace;
    SpmmParams p;
    p.rowptr = rowptr; p.col = col; p.value = value; p.mat = mat; p.out = out; p.arg_out = arg_out;
    p.B = B; p.M = M; p.N = N; p.K = K; p.E = E; p.k0 = 0; p.mean = 0; p.item_shift = 5;
    p.partial = nullptr; p.acc_mode = 0;
    p.plan_mask = nullptr; p.seg_lr = nullptr; p.long_done = nullptr; p.n_seg = 0; p.n_long = 0;
    p.counters = (unsigned int*)(ws + L.counters);
    p.segs = (Segment*)(ws + L.segs);
    p.longs = (LongRow*)(ws + L.longs);
    p.part_val = ws + L.part_val;
    p.part_arg = arg ? (int64_t*)(ws + L.part_arg) : nullptr;
    p.seg_cap = L.seg_cap; p.long_cap = L.long_cap; p.slot_cap = L.slot_cap;
    switch (dtype) {
      case TSB200_F32: return dispatch_red_vec<float>(p, reduce, st);
      case TSB200_F16: return dispatch_red_vec<__half>(p, reduce, st);
      case TSB200_BF16: return dispatch_red_vec<__nv_bfloat16>(p, reduce, st);
    }
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
  const WsLayout L = ws_layout(B, K, E, false);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  if ((uintptr_t)workspace & 255) return TSB200_ERR_INVALID_ARG;
  char* ws = (char*)workspace;
  SpmmParams p;
  p.rowptr = rowptr; p.col = col; p.value = value; p.mat = mat; p.out = out; p.arg_out = nullptr;
  p.B = B; p.M = M; p.N = N; p.K = K; p.E = E; p.k0 = 0; p.mean = 0; p.item_shift = 5;
  p.partial = partial; p.acc_mode = acc_mode;
  p.plan_mask = nullptr; p.seg_lr = nullptr; p.long_done = nullptr; p.n_seg = 0; p.n_long = 0;
  p.counters = (unsigned int*)(ws + L.counters);
  p.segs = (Segment*)(ws + L.segs);
  p.longs = (LongRow*)(ws + L.longs);
  p.part_val = ws + L.part_val;
  p.part_arg = nullptr;
  p.seg_cap = L.seg_cap; p.long_cap = L.long_cap; p.slot_cap = L.slot_cap;
  switch (dtype) {
    case TSB200_F32: return dispatch_shape<float, R_SUM, true>(p, st);
    case TSB200_F16: return dispatch_shape<__half, R_SUM, true>(p, st);
    case TSB200_BF16: return dispatch_shape<__nv_bfloat16, R_SUM, true>(p, st);
  }
  return TSB200_ERR_UNSUPPORTED;
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
    int64_t blocks = (((M + 31) / 32) * 32 + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    spmm_plan_kernel<<<(int)blocks, 256, 0, st>>>(rowptr, M, (uint32_t*)(pl + L.mask), (Segment*)(pl + L.segs),
                                                 (uint32_t*)(pl + L.seg_lr), (LongRow*)(pl + L.longs),
                                                 (unsigned int*)(pl + L.header), L.seg_cap, L.long_cap);
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
  const PlanLayout PL = plan_layout(M, E);
  if (plan_bytes < PL.total) return TSB200_ERR_WORKSPACE;
  if (n_seg > PL.seg_cap || n_long > PL.long_cap) return TSB200_ERR_INVALID_ARG;
  const PlannedWs W = planned_ws(K, n_long, n_slot, arg);
  if (!workspace || workspace_bytes < W.total) return TSB200_ERR_WORKSPACE;
  if (((uintptr_t)workspace & 255) || ((uintptr_t)plan & 255)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const char* pl = (const char*)plan;
  SpmmParams p;
  p.rowptr = rowptr; p.col = col; p.value = value; p.mat = mat; p.out = out; p.arg_out = arg_out;
  p.B = 1; p.M = M; p.N = N; p.K = K; p.E = E; p.k0 = 0; p.mean = 0; p.item_shift = 5;
  p.partial = nullptr; p.acc_mode = 0;
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
  switch (dtype) {
    case TSB200_F32: return dispatch_red_vec<float, true>(p, reduce, st);
    case TSB200_F16: return dispatch_red_vec<__half, true>(p, reduce, st);
    case TSB200_BF16: return dispatch_red_vec<__nv_bfloat16, true>(p, reduce, st);
  }
  return TSB200_ERR_UNSUPPORTED;
}
