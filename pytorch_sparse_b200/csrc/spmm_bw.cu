// spmm_bw.cu — SpMM backward kernels for sm_90a.
//
//  * tsb200_spmm_value_bw: SDDMM  out[e] = sum_b <mat[b,col[e],:], grad[b,row[e],:]>
//    replaces spmm_value_bw_cpu / spmm_value_bw_kernel
//    (csrc/cpu/spmm_cpu.cpp:103-152, csrc/cuda/spmm_cuda.cu:157-237).
//    nnz-parallel (perfect balance on power-law rows): a warp takes 32 consecutive nnz, reads
//    row/col coalesced, LPR lanes x 16 B cover one dense row, the 32/LPR lane groups work on
//    different nnz, results are gathered back to one lane per nnz for a coalesced store.
//    grad[row[e]] is re-read per nnz but consecutive nnz share the row => L1/L2 hits.
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
template <typename T, int LPR, int CH, int U> struct SddmmEngine {
  static constexpr int VEC = 16 / sizeof(T);
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
                                      uint64_t pol, T* __restrict__ out, float scale) {
    for (int j0 = s; j0 < e; j0 += U * G) {
      const int jend = min(e, j0 + U * G);
      ring.ensure(j0, jend, lane);
      const int slot0 = (j0 + g) & (kRing - 1);
      const uint32_t* pc = reinterpret_cast<const uint32_t*>(ring.s_col + slot0);
      const int nst = (jend - j0 + G - 1) / G;
      const int jrel = jend - j0 - g;
      uint4 d[U][CH];
      float part[U];
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
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        float sdot = 0.f;
#pragma unroll
        for (int ch = 0; ch < CH; ch++) sdot += Vec16<T, VEC>::dot(d[u][ch], gq[ch]);
        part[u] = sdot;
      }
      // lane li of group g gets the total of step li / (LPR/U); nnz t = u*G + g of the chunk goes to lane t
      const float tot = multi_reduce<U, LPR / 2>(part, li);
      const bool mine = lane < jend - j0;
      const int src_lane = mine ? (lane % G) * LPR + (lane / G) * (LPR / U) : 0;
      const float got = __shfl_sync(0xffffffffu, tot, src_lane);
      if (mine) out[ring.base + j0 + lane] = Traits<T>::from_acc(got * scale);
    }
  }
};

template <typename T, int LPR, int CH, int U, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
sddmm_vec_kernel(const SpmmParams p, const T* __restrict__ grad, T* __restrict__ out) {
  using Eng = SddmmEngine<T, LPR, CH, U>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;

  IndexRing<T> ring;
  ring.s_col = s_col[warp];
  ring.s_val = nullptr;
  ring.has_val = false;
  ring.col = p.col;
  ring.val = nullptr;
  ring.limit = p.E;
  const uint64_t pol = make_policy_evict_last();

  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const char* matb = (const char*)p.mat + (int64_t)li * 16;
  asm volatile("" : "+l"(matb));

  const int item_rows = 1 << p.item_shift;
  const int64_t n_items = (p.M + item_rows - 1) >> p.item_shift;
  unsigned int item = 0;
  if (lane == 0) item = atomicAdd(&p.counters[0], 1u);
  item = __shfl_sync(0xffffffffu, item, 0);

  while ((int64_t)item < n_items) {
    unsigned int next_item = 0;
    if (lane == 0) next_item = atomicAdd(&p.counters[0], 1u);
    const int64_t r0 = (int64_t)item << p.item_shift;
    const int nrows = (int)min((int64_t)item_rows, p.M - r0);
    const int64_t rp0 = __ldg(p.rowptr + r0 + min(lane, nrows));
    const int64_t rp1 = __ldg(p.rowptr + r0 + min(lane + 1, nrows));
    const int64_t a0 = __shfl_sync(0xffffffffu, rp0, 0);
    const int64_t base = a0 & ~(int64_t)31;
    const int s_rel = (int)(rp0 - base), e_rel = (int)(rp1 - base);
    const int deg = e_rel - s_rel;
    const bool is_long = deg > kLongT;
    int cum = is_long ? 0 : deg;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, cum, off);
      if (lane >= off) cum += t;
    }
    const bool defer = (deg > 0) && (is_long || cum > kItemCap);
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
      eng.load_grad((const char*)grad + (r0 + rl) * (int64_t)row_bytes, col_ok, li);
      const float scale = p.mean ? 1.f / (float)(e - s) : 1.f;
      eng.run(ring, s, e, matb, row_bytes, col_ok, lane, g, li, pol, out, scale);
    }
    item = __shfl_sync(0xffffffffu, next_item, 0);
  }
}

template <typename T, int LPR, int CH, int U, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
sddmm_seg_kernel(const SpmmParams p, const T* __restrict__ grad, T* __restrict__ out) {
  using Eng = SddmmEngine<T, LPR, CH, U>;
  constexpr int VEC = Eng::VEC;
  __shared__ __align__(16) int64_t s_col[kWarpsPerCta][kRingAlloc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  IndexRing<T> ring;
  ring.s_col = s_col[warp];
  ring.s_val = nullptr;
  ring.has_val = false;
  ring.col = p.col;
  ring.val = nullptr;
  ring.limit = p.E;
  const uint64_t pol = make_policy_evict_last();
  bool col_ok[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) col_ok[ch] = (ch * LPR + li) * VEC < p.K;
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const char* matb = (const char*)p.mat + (int64_t)li * 16;
  asm volatile("" : "+l"(matb));

  const int64_t nseg = min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    const int64_t base = S.start & ~(int64_t)31;
    ring.reset(base, S.end);
    Eng eng;
    eng.load_grad((const char*)grad + S.row_b * (int64_t)row_bytes, col_ok, li);
    float scale = 1.f;
    if (p.mean) {
      const int64_t cnt = __ldg(p.rowptr + S.row_b + 1) - __ldg(p.rowptr + S.row_b);
      scale = 1.f / (float)(cnt > 0 ? cnt : 1);
    }
    eng.run(ring, (int)(S.start - base), (int)(S.end - base), matb, row_bytes, col_ok, lane, g, li, pol, out, scale);
    __syncwarp();
  }
}

template <typename T, int LPR, int CH, int U, int MINB>
static int launch_sddmm(SpmmParams p, const void* grad, void* out, cudaStream_t st) {
  auto* kmain = sddmm_vec_kernel<T, LPR, CH, U, MINB>;
  auto* kseg = sddmm_seg_kernel<T, LPR, CH, U, MINB>;
  static GridCache gc_main, gc_seg;  // per instantiation, per device
  const int grid_main = gc_main.get((const void*)kmain, kWarpsPerCta * 32);
  const int grid_seg = gc_seg.get((const void*)kseg, kWarpsPerCta * 32);
  int64_t want = p.M / ((int64_t)grid_main * kWarpsPerCta * 2);
  p.item_shift = 0;
  while (p.item_shift < 5 && ((int64_t)2 << p.item_shift) <= want) p.item_shift++;
  const int64_t n_items = (p.M + (1 << p.item_shift) - 1) >> p.item_shift;
  TSB_CUDA_TRY(cudaMemsetAsync(p.counters, 0, 64, st));
  const int gm = (int)min((int64_t)grid_main, (n_items + kWarpsPerCta - 1) / kWarpsPerCta);
  kmain<<<gm, kWarpsPerCta * 32, 0, st>>>(p, (const T*)grad, (T*)out);
  TSB_LAUNCH_CHECK();
  kseg<<<grid_seg, kWarpsPerCta * 32, 0, st>>>(p, (const T*)grad, (T*)out);
  TSB_LAUNCH_CHECK();
  return 0;
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
  const size_t es = dtype_size(dtype);
  const bool vec = (dtype == TSB200_F32 || dtype == TSB200_F16 || dtype == TSB200_BF16) && K > 0 &&
                   (K * es) % 16 == 0 && !((uintptr_t)mat & 15) && !((uintptr_t)grad & 15) &&
                   M < ((int64_t)1 << 32) && N < ((int64_t)1 << 32) && K * (int64_t)es < ((int64_t)1 << 31);
  // row-wise path: single batch, >= 3 and <= 64 vectors per dense row, a workspace for the segment queue
  const int64_t vecs = vec ? (K * (int64_t)es) / 16 : 0;
  if (vec && B == 1 && vecs >= 3 && vecs <= 64 && E < ((int64_t)1 << 31) - 64 && !((uintptr_t)col & 7) && workspace &&
      !((uintptr_t)workspace & 255)) {
    const WsLayout L = ws_layout(1, K, E, false, false);
    if (workspace_bytes >= L.total) {
      char* ws = (char*)workspace;
      SpmmParams p;
      p.rowptr = rowptr; p.col = col; p.value = nullptr; p.mat = mat; p.out = nullptr; p.arg_out = nullptr;
      p.B = 1; p.M = M; p.N = N; p.K = K; p.E = E; p.k0 = 0; p.mean = mean ? 1 : 0; p.item_shift = 5;
      p.partial = nullptr; p.acc_mode = 0;
      p.plan_mask = nullptr; p.seg_lr = nullptr; p.long_done = nullptr; p.n_seg = 0; p.n_long = 0;
      p.counters = (unsigned int*)(ws + L.counters);
      p.segs = (Segment*)(ws + L.segs);
      p.longs = (LongRow*)(ws + L.longs);
      p.part_val = nullptr; p.part_arg = nullptr;
      p.seg_cap = L.seg_cap; p.long_cap = L.long_cap; p.slot_cap = L.slot_cap;
      switch (dtype) {
        case TSB200_F32: return dispatch_sddmm<float>(p, grad, out, st);
        case TSB200_F16: return dispatch_sddmm<__half>(p, grad, out, st);
        case TSB200_BF16: return dispatch_sddmm<__nv_bfloat16>(p, grad, out, st);
      }
    }
  }
  if (vec) {
    switch (dtype) {
      case TSB200_F32: return dispatch_value_vec<float>(row, rowptr, col, mat, grad, out, B, M, N, K, E, mean, st);
      case TSB200_F16: return dispatch_value_vec<__half>(row, rowptr, col, mat, grad, out, B, M, N, K, E, mean, st);
      case TSB200_BF16:
        return dispatch_value_vec<__nv_bfloat16>(row, rowptr, col, mat, grad, out, B, M, N, K, E, mean, st);
    }
  }
  return dispatch_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    int64_t blocks = (E + 7) / 8;
    const int64_t cap = (int64_t)num_sms() * 32;
    if (blocks > cap) blocks = cap;
    value_bw_generic_kernel<T><<<(int)blocks, 256, 0, st>>>(row, rowptr, col, (const T*)mat, (const T*)grad,
                                                           (T*)out, B, M, N, K, E, mean);
    TSB_LAUNCH_CHECK();
    return 0;
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
