// spmm_bw.cu — SpMM backward kernels for sm_90a.
//
//  * tsb200_spmm_value_bw: SDDMM  out[e] = sum_b <mat[b,col[e],:], grad[b,row[e],:]>
//    replaces spmm_value_bw_cpu / spmm_value_bw_kernel
//    (csrc/cpu/spmm_cpu.cpp:103-152, csrc/cuda/spmm_cuda.cu:157-237).
//    nnz-parallel (perfect balance on power-law rows): a warp takes 32 consecutive nnz, reads
//    row/col coalesced, LPR lanes x 16 B cover one dense row, the 32/LPR lane groups work on
//    different nnz, results are gathered back to one lane per nnz for a coalesced store.
//    grad[row[e]] is re-read per nnz but consecutive nnz share the row => L1/L2 hits.
//  * tsb200_sddmm_fp8: the row-wise SDDMM kernels over two e4m3 operands with per-row or per-tensor scales.
//  * tsb200_spmm_minmax_bw: fused replacement of the 8-op ATen chain of SPMMMin/SPMMMax::backward
//    (csrc/spmm.cpp:204-242, 264-302): one pass over arg_out, atomics into zero-filled fp32/fp64
//    accumulators.
#include <cstdlib>

#include "spmm_common.cuh"

namespace tsb {

template <typename T, int VEC> struct Vec16;
template <> struct Vec16<float, 4> {
  static __device__ __forceinline__ float dot(const uint4& a, const uint4& b) {
    return __uint_as_float(a.x) * __uint_as_float(b.x) + __uint_as_float(a.y) * __uint_as_float(b.y) +
           __uint_as_float(a.z) * __uint_as_float(b.z) + __uint_as_float(a.w) * __uint_as_float(b.w);
  }
};
// bf16 / f16: both operands widened to fp32 (exact, Vec<T>::unpack), products of two 16-bit values are exact in
// fp32, so FFMA rounds once per term; even and odd lanes of the pairs accumulate separately, fp32 throughout.
template <typename T> __device__ __forceinline__ float dot16(const uint4& a, const uint4& b) {
  float x[8], y[8];
  Vec<T>::unpack(a, x);
  Vec<T>::unpack(b, y);
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    s0 = fmaf(x[2 * i], y[2 * i], s0);
    s1 = fmaf(x[2 * i + 1], y[2 * i + 1], s1);
  }
  return s0 + s1;
}
template <> struct Vec16<__nv_bfloat16, 8> {
  static __device__ __forceinline__ float dot(const uint4& a, const uint4& b) { return dot16<__nv_bfloat16>(a, b); }
};
template <> struct Vec16<__half, 8> {
  static __device__ __forceinline__ float dot(const uint4& a, const uint4& b) { return dot16<__half>(a, b); }
};
// e4m3 (tsb200_sddmm_fp8): 16 elements per vector, widened exactly (Vec<__nv_fp8_e4m3>::unpack); the product of two
// e4m3 values is exact in fp32, so as above FFMA rounds once per term, even and odd elements accumulated separately.
template <> struct Vec16<__nv_fp8_e4m3, 16> {
  static __device__ __forceinline__ float dot(const uint4& a, const uint4& b) {
    float x[16], y[16];
    Vec<__nv_fp8_e4m3>::unpack(a, x);
    Vec<__nv_fp8_e4m3>::unpack(b, y);
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      s0 = fmaf(x[2 * i], y[2 * i], s0);
      s1 = fmaf(x[2 * i + 1], y[2 * i + 1], s1);
    }
    return s0 + s1;
  }
};

// Reduce U per-lane partial sums over the W*2 lanes of a lane group with a halving butterfly:
// level l exchanges half of the values with the partner lane (xor W), so U values cost
// U/2 + U/4 + ... + 1 + log2(LPR/U) shuffles instead of U*log2(LPR). Afterwards lane `li` of the group
// holds the total of value index li / (LPR/U).
template <int U, int W> __device__ __forceinline__ float multi_reduce(const float (&p)[U], int li) {
  if constexpr (U == 1) {
    float t = p[0];
#pragma unroll
    for (int off = W; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
    return t;
  } else {
    const bool hi = (li & W) != 0;
    float q[U / 2];
#pragma unroll
    for (int i = 0; i < U / 2; i++) {
      const float send = hi ? p[i] : p[i + U / 2];
      const float keep = hi ? p[i + U / 2] : p[i];
      q[i] = keep + __shfl_xor_sync(0xffffffffu, send, W);
    }
    return multi_reduce<U / 2, W / 2>(q, li);
  }
}

// vector path: K*sizeof(T) % 16 == 0, 16 B aligned mat/grad, M,N < 2^32.
template <typename T, int LPR, int U>
__global__ void __launch_bounds__(256, 3)
value_bw_vec_kernel(const int64_t* __restrict__ row, const int64_t* __restrict__ rowptr,
                    const int64_t* __restrict__ col, const T* __restrict__ mat,
                    const T* __restrict__ grad, T* __restrict__ out, int64_t B, int64_t M, int64_t N,
                    int64_t K, int64_t E, bool mean) {
  constexpr int VEC = 16 / sizeof(T);
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int nvec = (int)(K / VEC);  // 16-byte vectors per dense row
  const uint32_t row_bytes = (uint32_t)(K * (int64_t)sizeof(T));
  const uint64_t pol = make_policy_evict_last();

  int64_t e0 = wid * 32;
  // software prefetch of the next batch's (row, col): hides the index latency behind the gathers
  uint32_t r_nxt = 0, c_nxt = 0;
  if (e0 + lane < E) { r_nxt = (uint32_t)__ldg(row + e0 + lane); c_nxt = (uint32_t)__ldg(col + e0 + lane); }
  for (; e0 < E; e0 += nw * 32) {
    const uint32_t r = r_nxt, c = c_nxt;
    const int64_t en = e0 + nw * 32 + lane;
    if (en < E) { r_nxt = (uint32_t)__ldg(row + en); c_nxt = (uint32_t)__ldg(col + en); }
    const int nvalid = (int)min((int64_t)32, E - e0);
    float res = 0.f;  // lane j ends up with the result of nnz e0 + j
    for (int64_t b = 0; b < B; b++) {
      const char* matb = (const char*)mat + b * N * (int64_t)row_bytes + li * 16;
      const char* gradb = (const char*)grad + b * M * (int64_t)row_bytes + li * 16;
#pragma unroll 1
      for (int s0 = 0; s0 < nvalid; s0 += U * G) {
        uint4 a[U], q[U];
        bool act[U];
        if (nvec <= LPR) {  // one vector per lane: issue every gather of the chunk before the math
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int j = s0 + u * G + g;
            const uint32_t rj = __shfl_sync(0xffffffffu, r, j & 31);
            const uint32_t cj = __shfl_sync(0xffffffffu, c, j & 31);
            act[u] = j < nvalid && li < nvec;
            if (act[u]) {
              a[u] = ldg128_hint(matb + (uint64_t)cj * row_bytes, pol);
              q[u] = ldg128(gradb + (uint64_t)rj * row_bytes);
            }
          }
        }
        float part[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int j = s0 + u * G + g;
          float sdot = 0.f;
          if (nvec <= LPR) {
            if (act[u]) sdot = Vec16<T, VEC>::dot(a[u], q[u]);
          } else {  // rows wider than LPR vectors: strided walk
            const uint32_t rj = __shfl_sync(0xffffffffu, r, j & 31);
            const uint32_t cj = __shfl_sync(0xffffffffu, c, j & 31);
            if (j < nvalid)
              for (int v = li; v < nvec; v += LPR)
                sdot += Vec16<T, VEC>::dot(ldg128_hint(matb + (uint64_t)cj * row_bytes + (v - li) * 16, pol),
                                           ldg128(gradb + (uint64_t)rj * row_bytes + (v - li) * 16));
          }
          part[u] = sdot;
        }
        // lane li of group g now gets the total of step u = li / (LPR/U); hand nnz jj = u*G + g to lane s0 + jj
        const float tot = multi_reduce<U, LPR / 2>(part, li);
        const int jj = lane - s0;
        const bool mine = jj >= 0 && jj < U * G;
        const int src = mine ? (jj % G) * LPR + (jj / G) * (LPR / U) : 0;
        const float got = __shfl_sync(0xffffffffu, tot, src);
        if (mine) res += got;
      }
    }
    if (lane < nvalid) {
      if (mean) {
        const int64_t cnt = __ldg(rowptr + r + 1) - __ldg(rowptr + r);
        res = res / (float)(cnt > 0 ? cnt : 1);
      }
      out[e0 + lane] = Traits<T>::from_acc(res);
    }
  }
}

// ---- row-wise SDDMM (B == 1) ---------------------------------------------------------------------
// Same work decomposition as the SpMM forward (spmm_fw.cu): a warp pulls 32-row items from an atomic
// counter, the item's column indices stream through the per-warp cp.async ring, rows that are too long
// (or overflow the item's nnz budget) are deferred as <= 256-nnz segments to a second kernel. Per row the
// grad vector is loaded ONCE into registers (16 B per lane and chunk), so only the dense-operand rows are
// gathered (half the L1/L2 traffic of the nnz-parallel kernel); every nnz's dot product is reduced over the
// LPR lanes with the halving butterfly and the chunk's results leave with one coalesced store.
// T = output type, X = type of both dense operands: T itself, or __nv_fp8_e4m3 (tsb200_sddmm_fp8). For e4m3 a vector
// is 16 columns, `scale` is the row operand's scale of the row, and the gathered row's scale bscale[c * bstride] is
// loaded next to its column word; after the reduction out = round_T(fl32(fl32(scale * bscale[c]) * dot)).
// HL > 0 (tsb200_sddmm_heads): the operands are [rows, H, D] with HL = D * sizeof(T) / 16 lanes per head (a power of
// two, <= LPR): each step's dot is reduced over the HL lanes of a head, and out is [E, H].
template <typename T, int LPR, int CH, int U, typename X = T, int HL = 0> struct SddmmEngine {
  static constexpr bool Q8 = !std::is_same<X, T>::value;
  static constexpr int VEC = 16 / sizeof(X);
  static constexpr int G = 32 / LPR;
  uint4 gq[CH];

  __device__ __forceinline__ void load_grad(const char* grad_row, const bool (&col_ok)[CH], int li) {
#pragma unroll
    for (int ch = 0; ch < CH; ch++)
      gq[ch] = col_ok[ch] ? ldg128(grad_row + (ch * LPR + li) * 16) : make_uint4(0, 0, 0, 0);
  }

  // ring-relative nnz [s, e) of one row -> out[absolute nnz]
  __device__ __forceinline__ void run(IndexRing<T>& ring, int s, int e, const char* __restrict__ matb,
                                      uint32_t row_bytes, const bool (&col_ok)[CH], int lane, int g, int li,
                                      uint64_t pol, T* __restrict__ out, float scale,
                                      const float* __restrict__ bscale = nullptr, uint32_t bstride = 0) {
    for (int j0 = s; j0 < e; j0 += U * G) {
      const int jend = min(e, j0 + U * G);
      ring.ensure(j0, jend, lane);
      const int slot0 = (j0 + g) & (kRing - 1);
      const uint32_t* pc = reinterpret_cast<const uint32_t*>(ring.s_col + slot0);
      const int nst = (jend - j0 + G - 1) / G;
      const int jrel = jend - j0 - g;
      uint4 d[U][CH];
      float part[U];
      float sc[U];  // Q8 only: scale of each step's gathered row
      // Branch-free chunk (the kernel is issue-bound, and branches around the inline-asm gathers cost issue slots):
      // the gathers are predicated inside the asm into zeroed
      // registers and the dot products run unconditionally (an inactive slot contributes 0). The ring slot is read
      // unconditionally — slots past the row's end hold stale but in-bounds column words, and the predicate keeps
      // them from being dereferenced.
#pragma unroll
      for (int u = 0; u < U; u++) {
        const bool act = (u < nst) && (u * G < jrel);
        const uint32_t c = pc[2 * u * G];
        const char* src = matb + (uint64_t)c * row_bytes;
#pragma unroll
        for (int ch = 0; ch < CH; ch++) {
          d[u][ch] = make_uint4(0, 0, 0, 0);
          ldg128_hint_pred(d[u][ch], src + ch * (LPR * 16), pol, act && col_ok[ch]);
        }
        if constexpr (Q8) sc[u] = act ? __ldg(bscale + (size_t)c * bstride) : 0.f;
      }
      if constexpr (HL > 0) {
        store_heads(d, col_ok, g, li, nst, jend - j0 - g, out + (ring.base + j0) * heads);
      } else {
#pragma unroll
        for (int u = 0; u < U; u++) {
          float sdot = 0.f;
#pragma unroll
          for (int ch = 0; ch < CH; ch++) sdot += Vec16<X, VEC>::dot(d[u][ch], gq[ch]);
          part[u] = sdot;
        }
        // lane li of group g gets the total of step li / (LPR/U); nnz t = u*G + g of the chunk goes to lane t
        float tot = multi_reduce<U, LPR / 2>(part, li);
        if constexpr (Q8) {  // the scale product, on the lane that holds the step's total
          const int ul = li / (LPR / U);
          float sb = sc[0];
#pragma unroll
          for (int u = 1; u < U; u++)
            if (ul == u) sb = sc[u];
          tot = __fmul_rn(__fmul_rn(scale, sb), tot);
        }
        const bool mine = lane < jend - j0;
        const int src_lane = mine ? (lane % G) * LPR + (lane / G) * (LPR / U) : 0;
        const float got = __shfl_sync(0xffffffffu, tot, src_lane);
        if constexpr (Q8) {
          if (mine) out[ring.base + j0 + lane] = Traits<T>::from_acc(got);
        } else {
          if (mine) out[ring.base + j0 + lane] = Traits<T>::from_acc(got * scale);
        }
      }
    }
  }

  // HL > 0: the scores of one chunk (nst steps; lane group g is active in step u iff u * G < jrel) into outc, the
  // chunk's first [H] row. Head h of a chunk-ch vector is (ch * LPR + li) / HL; the lane holding a (step, head)
  // total stores it, so a step's G * H scores leave as one contiguous run.
  int heads;
  __device__ __forceinline__ void store_heads(const uint4 (&d)[U][CH], const bool (&col_ok)[CH], int g, int li,
                                              int nst, int jrel, T* __restrict__ outc) {
    const int hl = li & (HL - 1);
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      const int h = (ch * LPR + li) / HL;
      float part[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        float sdot = 0.f;
        sdot += Vec16<X, VEC>::dot(d[u][ch], gq[ch]);
        part[u] = sdot;
      }
      if constexpr (U <= HL) {  // halving butterfly: lane hl of the head gets the total of step hl / (HL / U)
        const float tot = multi_reduce<U, HL / 2>(part, hl);
        const int u = hl / (HL / U);
        if (hl % (HL / U) == 0 && col_ok[ch] && u < nst && u * G < jrel)
          outc[(int64_t)(u * G + g) * heads + h] = Traits<T>::from_acc(tot * 1.f);
      } else {  // fewer lanes per head than steps: every step reduced on its own
#pragma unroll
        for (int u = 0; u < U; u++) {
          float t = part[u];
#pragma unroll
          for (int off = HL / 2; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
          if (hl == 0 && col_ok[ch] && u < nst && u * G < jrel)
            outc[(int64_t)(u * G + g) * heads + h] = Traits<T>::from_acc(t);
        }
      }
    }
  }
};

// X = e4m3: gscale[row * gstride] is the row operand's scale, p.scale[col * p.scale_stride] the gathered row's
template <typename T, int LPR, int CH, int U, int MINB, typename X = T, int HL = 0>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
sddmm_vec_kernel(const SpmmParams p, const X* __restrict__ grad, T* __restrict__ out, const float* __restrict__ gscale,
                 uint32_t gstride) {
  using Eng = SddmmEngine<T, LPR, CH, U, X, HL>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.template bind<false>(p, s_col[warp], nullptr, lane);
  const uint64_t pol = make_policy_evict_last();

  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(X));
  const char* matb = (const char*)p.mat + (int64_t)li * 16;
  asm volatile("" : "+l"(matb));

  const int item_rows = 1 << p.item_shift;
  const int64_t n_items = (p.M + item_rows - 1) >> p.item_shift;
  unsigned int item = __shfl_sync(0xffffffffu, take_ticket(&p.counters[0], lane), 0);
  while ((int64_t)item < n_items) {
    const unsigned int next_item = take_ticket(&p.counters[0], lane);
    const int64_t r0 = (int64_t)item << p.item_shift;
    const int nrows = (int)min((int64_t)item_rows, p.M - r0);
    const int64_t rp0 = __ldg(p.rowptr + r0 + min(lane, nrows));
    const int64_t rp1 = __ldg(p.rowptr + r0 + min(lane + 1, nrows));
    const int64_t a0 = __shfl_sync(0xffffffffu, rp0, 0);
    const int64_t base = a0 & ~(int64_t)31;
    const int s_rel = (int)(rp0 - base), e_rel = (int)(rp1 - base);
    const int deg = e_rel - s_rel;
    const bool defer = defer_row(deg, lane);
    const unsigned defer_mask = __ballot_sync(0xffffffffu, defer);
    if (defer) {
      const int nseg = (deg + kSeg - 1) / kSeg;
      const unsigned seg0 = atomicAdd(&p.counters[1], (unsigned)nseg);
      for (int sgi = 0; sgi < nseg; sgi++) {
        if ((int64_t)seg0 + sgi < p.seg_cap) {
          Segment S;
          S.row_b = r0 + lane;
          S.start = rp0 + (int64_t)sgi * kSeg;
          S.end = min(rp1, S.start + kSeg);
          S.slot = -1;
          p.segs[seg0 + sgi] = S;
        }
      }
    }
    __syncwarp();
    ring.reset(base, __shfl_sync(0xffffffffu, rp1, 31));
    for (int rl = 0; rl < nrows; rl++) {
      if ((defer_mask >> rl) & 1u) continue;
      const int s = __shfl_sync(0xffffffffu, s_rel, rl);
      const int e = __shfl_sync(0xffffffffu, e_rel, rl);
      if (e == s) continue;
      Eng eng;
      if constexpr (HL > 0) eng.heads = p.heads;
      eng.load_grad((const char*)grad + (r0 + rl) * (int64_t)row_bytes, col_ok, li);
      if constexpr (Eng::Q8) {
        const float scale = __ldg(gscale + (r0 + rl) * gstride);
        eng.run(ring, s, e, matb, row_bytes, col_ok, lane, g, li, pol, out, scale, p.scale, p.scale_stride);
      } else {
        const float scale = p.mean ? 1.f / (float)(e - s) : 1.f;
        eng.run(ring, s, e, matb, row_bytes, col_ok, lane, g, li, pol, out, scale);
      }
    }
    item = __shfl_sync(0xffffffffu, next_item, 0);
  }
}

template <typename T, int LPR, int CH, int U, int MINB, typename X = T, int HL = 0>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
sddmm_seg_kernel(const SpmmParams p, const X* __restrict__ grad, T* __restrict__ out, const float* __restrict__ gscale,
                 uint32_t gstride) {
  using Eng = SddmmEngine<T, LPR, CH, U, X, HL>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  IndexRing<T> ring;
  ring.template bind<false>(p, s_col[warp], nullptr, lane);
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(X));
  const char* matb = (const char*)p.mat + (int64_t)li * 16;
  asm volatile("" : "+l"(matb));

  const int64_t nseg = min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    const int64_t base = S.start & ~(int64_t)31;
    ring.reset(base, S.end);
    Eng eng;
    if constexpr (HL > 0) eng.heads = p.heads;
    eng.load_grad((const char*)grad + S.row_b * (int64_t)row_bytes, col_ok, li);
    if constexpr (Eng::Q8) {
      eng.run(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, li, pol, out,
              __ldg(gscale + S.row_b * gstride), p.scale, p.scale_stride);
    } else {
      float scale = 1.f;
      if (p.mean) {
        const int64_t cnt = __ldg(p.rowptr + S.row_b + 1) - __ldg(p.rowptr + S.row_b);
        scale = 1.f / (float)(cnt > 0 ? cnt : 1);
      }
      eng.run(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, li, pol, out, scale);
    }
    __syncwarp();
  }
}

template <typename T, int LPR, int CH, int U, int MINB, typename X = T, int HL = 0>
static int launch_sddmm(SpmmParams p, const void* grad, void* out, cudaStream_t st, const float* gscale = nullptr,
                        uint32_t gstride = 0) {
  static GridCache gc_main, gc_seg;  // per instantiation, per device
  return launch_rowsplit(sddmm_vec_kernel<T, LPR, CH, U, MINB, X, HL>, sddmm_seg_kernel<T, LPR, CH, U, MINB, X, HL>,
                         gc_main, gc_seg, p, st, (const X*)grad, (T*)out, gscale, gstride);
}

template <typename T> static int dispatch_sddmm(const SpmmParams& p, const void* grad, void* out, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t vecs = p.K / VEC;
  if (vecs <= 4) return launch_sddmm<T, 4, 1, 4, 5>(p, grad, out, st);
  if (vecs <= 8) return launch_sddmm<T, 8, 1, 4, 5>(p, grad, out, st);
  if (vecs <= 16) return launch_sddmm<T, 16, 1, 4, 5>(p, grad, out, st);
  if (vecs <= 32) return launch_sddmm<T, 32, 1, 4, 4>(p, grad, out, st);
  return launch_sddmm<T, 32, 2, 4, 3>(p, grad, out, st);  // up to 64 vectors
}

// per-head scores (tsb200_sddmm_heads): vecs = H * HL vectors per row, HL lanes per head; the single-head
// (LPR, CH, U) with one CTA/SM less (the per-head reduction and stores spill at the single-head occupancy)
template <typename T, int HL> static int dispatch_sddmm_heads_lpr(const SpmmParams& p, const void* a, void* out,
                                                                   cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t vecs = p.K / VEC;
  if constexpr (HL <= 4) if (vecs <= 4) return launch_sddmm<T, 4, 1, 4, 4, T, HL>(p, a, out, st);
  if constexpr (HL <= 8) if (vecs <= 8) return launch_sddmm<T, 8, 1, 4, 4, T, HL>(p, a, out, st);
  if constexpr (HL <= 16) if (vecs <= 16) return launch_sddmm<T, 16, 1, 4, 4, T, HL>(p, a, out, st);
  if (vecs <= 32) return launch_sddmm<T, 32, 1, 4, 3, T, HL>(p, a, out, st);
  return launch_sddmm<T, 32, 2, 4, 2, T, HL>(p, a, out, st);  // up to 64 vectors
}
template <typename T> static int dispatch_sddmm_heads(const SpmmParams& p, int hl, const void* a, void* out,
                                                      cudaStream_t st) {
  switch (hl) {
    case 1: return dispatch_sddmm_heads_lpr<T, 1>(p, a, out, st);
    case 2: return dispatch_sddmm_heads_lpr<T, 2>(p, a, out, st);
    case 4: return dispatch_sddmm_heads_lpr<T, 4>(p, a, out, st);
    case 8: return dispatch_sddmm_heads_lpr<T, 8>(p, a, out, st);
    case 16: return dispatch_sddmm_heads_lpr<T, 16>(p, a, out, st);
    case 32: return dispatch_sddmm_heads_lpr<T, 32>(p, a, out, st);
  }
  return TSB200_ERR_UNSUPPORTED;
}

// generic per-head SDDMM: warp per CSR row, per (entry, head) the lanes stride over the D columns and the warp
// reduces, as value_bw_generic_kernel does for one head
template <typename T>
__global__ void __launch_bounds__(256)
sddmm_heads_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                           const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int64_t M,
                           int64_t H, int64_t D) {
  using acc_t = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t K = H * D;
  for (int64_t m = wid; m < M; m += nw) {
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    for (int64_t e = rs; e < re; e++) {
      const T* bp = b + col[e] * K;
      for (int64_t h = 0; h < H; h++) {
        acc_t s = (acc_t)0;
        for (int64_t k = lane; k < D; k += 32)
          s += Traits<T>::to_acc(a[m * K + h * D + k]) * Traits<T>::to_acc(bp[h * D + k]);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) out[e * H + h] = Traits<T>::from_acc(s);
      }
    }
  }
}

// e4m3 operands, output type T: a vector is 16 columns, so a K-column row is K / 16 vectors (K <= 2048)
template <typename T>
static int dispatch_sddmm_fp8(const SpmmParams& p, const void* a8, void* out, cudaStream_t st, const float* a_scale,
                              uint32_t a_stride) {
  using X = __nv_fp8_e4m3;
  const int64_t vecs = p.K / 16;
  if (vecs <= 4) return launch_sddmm<T, 4, 1, 4, 4, X>(p, a8, out, st, a_scale, a_stride);
  if (vecs <= 8) return launch_sddmm<T, 8, 1, 4, 4, X>(p, a8, out, st, a_scale, a_stride);
  if (vecs <= 16) return launch_sddmm<T, 16, 1, 4, 4, X>(p, a8, out, st, a_scale, a_stride);
  if (vecs <= 32) return launch_sddmm<T, 32, 1, 4, 4, X>(p, a8, out, st, a_scale, a_stride);
  if (vecs <= 64) return launch_sddmm<T, 32, 2, 4, 3, X>(p, a8, out, st, a_scale, a_stride);
  return launch_sddmm<T, 32, 4, 2, 2, X>(p, a8, out, st, a_scale, a_stride);  // up to 128 vectors
}

// generic: warp per nnz, lanes stride over k (any dtype / alignment).
template <typename T>
__global__ void __launch_bounds__(256)
value_bw_generic_kernel(const int64_t* __restrict__ row, const int64_t* __restrict__ rowptr,
                        const int64_t* __restrict__ col, const T* __restrict__ mat,
                        const T* __restrict__ grad, T* __restrict__ out, int64_t B, int64_t M,
                        int64_t N, int64_t K, int64_t E, bool mean) {
  using acc_t = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t e = wid; e < E; e += nw) {
    const int64_t r = row[e], c = col[e];
    acc_t s = (acc_t)0;
    for (int64_t b = 0; b < B; b++) {
      const T* mp = mat + (b * N + c) * K;
      const T* gp = grad + (b * M + r) * K;
      for (int64_t k = lane; k < K; k += 32) s += Traits<T>::to_acc(mp[k]) * Traits<T>::to_acc(gp[k]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) {
      if (mean) {
        const int64_t cnt = rowptr[r + 1] - rowptr[r];
        s = s / (acc_t)(cnt > 0 ? cnt : 1);
      }
      out[e] = Traits<T>::from_acc(s);
    }
  }
}

// Fused min/max backward (csrc/spmm.cpp:204-242 as ONE pass over arg_out): every output element (r, k) routes
// grad_out[r, k] to value[arg] and to grad_mat[col[arg], k]. The scattered 4-byte reads of mat and atomics on
// grad_mat touch one 32-byte sector each; with both arrays far larger than L2 (C3: 512 MB each) every sector would
// be fetched from / written back to DRAM up to 8 times (~13 GB of traffic for 2 GB of data). So the element space
// is walked FEATURE-SLICE-major by a persistent grid: all CTAs work on the same 2^lsl-feature slice at the same
// time, and a slice of mat + grad_mat (N * 2^lsl * (s + 4) bytes, sized by the host to ~32 MB) stays L2-resident
// while the whole arg_out / grad_out slice streams through -- each DRAM byte moves once.
template <typename T, typename A>
__global__ void __launch_bounds__(256)
minmax_bw_kernel(const int64_t* __restrict__ col, const T* __restrict__ value, const T* __restrict__ mat,
                 const T* __restrict__ grad_out, const int64_t* __restrict__ arg_out,
                 A* __restrict__ grad_value, A* __restrict__ grad_mat, int64_t B, int64_t M, int64_t N,
                 int64_t K, int64_t E, int lsl) {
  const int64_t per_slice = (B * M) << lsl;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t kmask = ((int64_t)1 << lsl) - 1;
  for (int64_t k0 = 0; k0 < K; k0 += kmask + 1) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < per_slice; j += stride) {
      const int64_t r = j >> lsl;
      const int64_t k = k0 + (j & kmask);
      if (k >= K) continue;
      const int64_t i = r * K + k;
      const int64_t a = arg_out[i];
      if (a < 0 || a >= E) continue;  // sentinel E: empty row (csrc/spmm.cpp:270-271)
      const A g = (A)Traits<T>::to_acc(grad_out[i]);
      const int64_t c = col[a];
      const int64_t b = B == 1 ? 0 : r / M;
      const int64_t mi = (b * N + c) * K + k;
      if (grad_value) atomicAdd(grad_value + a, (A)Traits<T>::to_acc(mat[mi]) * g);
      if (grad_mat) atomicAdd(grad_mat + mi, value ? (A)Traits<T>::to_acc(value[a]) * g : g);
    }
  }
}

template <typename T, int LPR, int U>
static int launch_value_vec(const int64_t* row, const int64_t* rowptr, const int64_t* col, const void* mat,
                            const void* grad, void* out, int64_t B, int64_t M, int64_t N, int64_t K,
                            int64_t E, bool mean, cudaStream_t st) {
  int64_t blocks = (E + 255) / 256;  // 8 warps x 32 nnz per CTA pass
  const int64_t cap = (int64_t)num_sms() * 6;  // 3 resident CTAs/SM, 2 passes
  if (blocks > cap) blocks = cap;
  value_bw_vec_kernel<T, LPR, U><<<(int)blocks, 256, 0, st>>>(row, rowptr, col, (const T*)mat, (const T*)grad,
                                                             (T*)out, B, M, N, K, E, mean);
  TSB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
static int dispatch_value_vec(const int64_t* row, const int64_t* rowptr, const int64_t* col, const void* mat,
                              const void* grad, void* out, int64_t B, int64_t M, int64_t N, int64_t K,
                              int64_t E, bool mean, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const int64_t vecs = K / VEC;
#define TSB_ARGS row, rowptr, col, mat, grad, out, B, M, N, K, E, mean, st
  if (vecs <= 1) return launch_value_vec<T, 1, 1>(TSB_ARGS);
  if (vecs <= 4) return launch_value_vec<T, 4, 2>(TSB_ARGS);
  if (vecs <= 8) return launch_value_vec<T, 8, 2>(TSB_ARGS);
  if (vecs <= 16) return launch_value_vec<T, 16, 4>(TSB_ARGS);
  return launch_value_vec<T, 32, 4>(TSB_ARGS);
#undef TSB_ARGS
}

}  // namespace tsb

using namespace tsb;

extern "C" size_t tsb200_spmm_value_bw_workspace_bytes(int64_t B, int64_t M, int64_t K, int64_t E, int dtype) {
  (void)M;
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return 0;
  if (B != 1 || K <= 0 || E <= 0) return 0;
  return ws_layout(1, K, E, false, false).total;
}

extern "C" int tsb200_spmm_value_bw(const int64_t* row, const int64_t* rowptr, const int64_t* col,
                                    const void* mat, const void* grad, void* out, int64_t B, int64_t M,
                                    int64_t N, int64_t K, int64_t E, int dtype, int reduce, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (B < 0 || M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if (reduce != TSB200_SUM && reduce != TSB200_MEAN) return TSB200_ERR_INVALID_ARG;
  if (dtype_size(dtype) == 0) return TSB200_ERR_INVALID_ARG;
  if (E == 0) return 0;
  if (!row || !rowptr || !col || !out) return TSB200_ERR_INVALID_ARG;
  if (B * K > 0 && (!mat || !grad)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const bool mean = reduce == TSB200_MEAN;
  const int64_t row_bytes = K * (int64_t)dtype_size(dtype);
  // nnz-parallel vector kernel: 16-byte rows of mat and grad, gathered by 32-bit row and column indices
  const bool vec = (dtype == TSB200_F32 || dtype == TSB200_F16 || dtype == TSB200_BF16) && K > 0 &&
                   row_bytes % 16 == 0 && rowsplit_aligned({mat, grad}, nullptr) && M < ((int64_t)1 << 32) &&
                   N < ((int64_t)1 << 32) && row_bytes < ((int64_t)1 << 31);
  // row-wise path: single batch, >= 3 and <= 64 vectors per dense row, a workspace for the segment queue; a short
  // workspace falls back to the nnz-parallel kernel
  if (vec && B == 1 && row_bytes >= 3 * 16 && row_bytes <= 64 * 16 && rowsplit_extents(E, N, row_bytes, M) &&
      rowsplit_aligned({mat, grad}, col) && workspace && !((uintptr_t)workspace & 255)) {
    SpmmParams p{rowptr, col, nullptr, mat, nullptr, nullptr, 1, M, N, K, E};
    p.mean = mean ? 1 : 0;
    if (!bind_unplanned(p, workspace, workspace_bytes, false, false))
      return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_sddmm<decltype(tag)>(p, grad, out, st); });
  }
  if (vec)
    return dispatch_vec_dtype(dtype, [&](auto tag) {
      return dispatch_value_vec<decltype(tag)>(row, rowptr, col, mat, grad, out, B, M, N, K, E, mean, st);
    });
  return dispatch_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    value_bw_generic_kernel<T><<<warp_grid(E, 32), 256, 0, st>>>(row, rowptr, col, (const T*)mat, (const T*)grad,
                                                                 (T*)out, B, M, N, K, E, mean);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

// ---- SDDMM over two e4m3 operands with per-tensor or per-row scales ------------------------------------------------
// The row-wise kernels with X = __nv_fp8_e4m3 and T = out_dtype: `mat` is b8 [N, K] (gathered, p.scale = b_scale) and
// `grad` is a8 [M, K] (one row in registers per CSR row, its scale read once per row).
extern "C" size_t tsb200_sddmm_fp8_workspace_bytes(int64_t M, int64_t K, int64_t E) {
  (void)M;
  if (K <= 0 || E <= 0) return 0;
  return ws_layout(1, K, E, false, false).total;
}

extern "C" int tsb200_sddmm_fp8(const int64_t* rowptr, const int64_t* col, const void* a8, const float* a_scale,
                                int64_t a_scale_stride, const void* b8, const float* b_scale, int64_t b_scale_stride,
                                void* out, int64_t M, int64_t N, int64_t K, int64_t E, int out_dtype, void* workspace,
                                size_t workspace_bytes, void* stream) {
  if (M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if ((a_scale_stride != 0 && a_scale_stride != 1) || (b_scale_stride != 0 && b_scale_stride != 1))
    return TSB200_ERR_INVALID_ARG;
  if (out_dtype != TSB200_F32 && out_dtype != TSB200_F16 && out_dtype != TSB200_BF16) return TSB200_ERR_UNSUPPORTED;
  if (K % 16 != 0 || K > 2048) return TSB200_ERR_UNSUPPORTED;
  if (E == 0) return 0;
  if (!out) return TSB200_ERR_INVALID_ARG;
  const size_t es = dtype_size(out_dtype);
  if ((uintptr_t)out % es) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  if (K == 0) {  // every dot product is empty: +0
    TSB_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)E * es, st));
    return 0;
  }
  if (!rowptr || !col || !a8 || !a_scale || !b8 || !b_scale) return TSB200_ERR_INVALID_ARG;
  if (!rowsplit_extents(E, N, K, M) || !rowsplit_aligned({a8, b8}, col, {a_scale, b_scale}))
    return TSB200_ERR_UNSUPPORTED;
  if (!workspace || ((uintptr_t)workspace & 255)) return TSB200_ERR_INVALID_ARG;
  SpmmParams p{rowptr, col, nullptr, b8, nullptr, nullptr, 1, M, N, K, E};
  if (const int rc = bind_unplanned(p, workspace, workspace_bytes, false, false)) return rc;
  p.scale = b_scale; p.scale_stride = (uint32_t)b_scale_stride;
  return dispatch_vec_dtype(out_dtype, [&](auto tag) {
    return dispatch_sddmm_fp8<decltype(tag)>(p, a8, out, st, a_scale, (uint32_t)a_scale_stride);
  });
}

extern "C" int tsb200_spmm_minmax_bw(const int64_t* col, const void* value, const void* mat,
                                     const void* grad_out, const int64_t* arg_out, void* grad_value,
                                     void* grad_mat, int64_t B, int64_t M, int64_t N, int64_t K, int64_t E,
                                     int dtype, void* stream) {
  if (B < 0 || M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if (B * M * K == 0 || E == 0) return 0;
  if (!col || !grad_out || !arg_out) return TSB200_ERR_INVALID_ARG;
  if (grad_value && !mat) return TSB200_ERR_INVALID_ARG;
  if (!grad_value && !grad_mat) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    using A = typename std::conditional<std::is_same<T, double>::value, double, float>::type;
    // feature slice (scripts/sweep_minmax_bw.py): whole rows while mat + grad_mat fit in half of L2; otherwise
    // 256-byte slices of a row when both gradients are wanted, 128-byte slices (one L2 line; narrower slices waste
    // line capacity) for a single gradient
    int full = 0;
    while (((int64_t)1 << full) < K) full++;
    int lsl = full;
    int dev = 0, l2 = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) != cudaSuccess)
      l2 = 0;
    const double resident = (double)B * (double)N * (double)K * (double)(sizeof(T) + sizeof(A));
    if (resident > 0.5 * (double)l2) {
      const int slice_bytes = (grad_value && grad_mat) ? 256 : 128;
      lsl = 0;
      while ((size_t)(2u << lsl) * sizeof(T) <= (size_t)slice_bytes) lsl++;
      if (lsl > full) lsl = full;
    }
    if (const char* ev = getenv("TSB200_MMBW_LSL")) { lsl = atoi(ev); if (lsl > full) lsl = full; if (lsl < 0) lsl = 0; }
    // persistent grid: every CTA resident, so all of them walk the slices in step
    int per_sm = 8;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)minmax_bw_kernel<T, A>, 256, 0);
    if (per_sm < 1) per_sm = 1;
    int64_t blocks = ((B * M << lsl) + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * per_sm;
    if (blocks > cap) blocks = cap;
    minmax_bw_kernel<T, A><<<(int)blocks, 256, 0, st>>>(col, (const T*)value, (const T*)mat, (const T*)grad_out,
                                                       arg_out, (A*)grad_value, (A*)grad_mat, B, M, N, K, E, lsl);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

// ---- SDDMM with per-head scores (tsb200_sddmm_heads) ----------------------------------------------------------------
// out[e, h] = <a[row_e, h, :], b[col_e, h, :]>. Row-wise kernels when D * sizeof(T) / 16 = HL is a power of two and
// the row is at most 64 vectors with HL <= LPR; the generic kernel otherwise.
extern "C" int tsb200_sddmm_heads(const int64_t* rowptr, const int64_t* col, const void* a, const void* b, void* out,
                                  int64_t M, int64_t N, int64_t H, int64_t D, int64_t E, int dtype, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  if (M < 0 || N < 0 || H < 0 || D < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F64 && dtype != TSB200_F16 && dtype != TSB200_BF16)
    return TSB200_ERR_UNSUPPORTED;
  if (H > 0 && D > ((int64_t)1 << 40) / H) return TSB200_ERR_UNSUPPORTED;
  if (E * H == 0) return 0;  // nothing to write
  if (!out) return TSB200_ERR_INVALID_ARG;
  const size_t es = dtype_size(dtype);
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 0) {  // every dot product is empty: +0
    TSB_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)(E * H) * es, st));
    return 0;
  }
  if (!rowptr || !col || !a || !b) return TSB200_ERR_INVALID_ARG;
  const int64_t K = H * D;
  const int64_t hl = (D * (int64_t)es) % 16 == 0 ? D * (int64_t)es / 16 : 0;
  const int64_t vecs = hl * H;
  const int64_t lpr = vecs <= 4 ? 4 : vecs <= 8 ? 8 : vecs <= 16 ? 16 : 32;
  if (dtype != TSB200_F64 && hl > 0 && (hl & (hl - 1)) == 0 && hl <= lpr && vecs <= 64 && E * H < ((int64_t)1 << 40) &&
      rowsplit_extents(E, N, K * (int64_t)es, M) && rowsplit_aligned({a, b}, col) && !((uintptr_t)out % es) &&
      workspace && !((uintptr_t)workspace & 255)) {
    SpmmParams p{rowptr, col, nullptr, b, nullptr, nullptr, 1, M, N, K, E};
    p.heads = (int)H;
    if (const int rc = bind_unplanned(p, workspace, workspace_bytes, false, false)) return rc;
    return dispatch_vec_dtype(dtype,
                              [&](auto tag) { return dispatch_sddmm_heads<decltype(tag)>(p, (int)hl, a, out, st); });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    sddmm_heads_generic_kernel<T><<<warp_grid(M, 32), 256, 0, st>>>(rowptr, col, (const T*)a, (const T*)b, (T*)out,
                                                                    M, H, D);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}
