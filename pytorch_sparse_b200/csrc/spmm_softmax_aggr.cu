// spmm_softmax_aggr.cu — softmax-aggregation SpMM for sm_90a: per row m and column k the messages p_e = v_e x[col_e, k]
// summed with the weights softmax_e(t_k p_e) over the row's entries (tsb200_spmm_fw_softmax_aggr), and its backward
// (tsb200_spmm_softmax_aggr_bw_rows / _cols).
//
// The forward runs in the row-split kernels of the SpMM forward with one more engine, SoftmaxAggrEngine: every lane
// keeps an online softmax (mu, s, a) per column it owns. The lane layout (LPR, CH) per row width, the per-lane entry
// order, the butterfly over lane groups and the segment-order fold of deferred rows are those of the mean kernels, so
// with t = 0 (every weight exp(0) = 1, s = the degree) the result is bit for bit spmm's mean on the same path.
#include "spmm_common.cuh"

namespace tsb {

// exp of the fp32 kernels: ex2.approx.ftz of the argument scaled by log2(e) (one MUFU.EX2). exp(0) = 1 and
// exp(-inf) = +0 exactly; results below 2^-126 flush to +0.
__device__ __forceinline__ float smx_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(__fmul_rn(x, 1.4426950408889634f)));
  return y;
}
__device__ __forceinline__ double smx_exp(double x) { return exp(x); }

// the factor that moves a state kept relative to maximum m0 to maximum m (m >= m0): exactly 1 when the maximum is
// unchanged, which also keeps two empty states (-inf, 0, 0) from forming exp(-inf + inf)
template <typename A> __device__ __forceinline__ A smx_rescale(A m0, A m) { return m0 == m ? (A)1 : smx_exp(m0 - m); }

// (mu, s, a) <- the merge of itself and (om, os, oa): one IEEE product per term and one IEEE add, never contracted,
// so the merge is commutative (both lanes of a butterfly pair hold the same state) and t = 0 adds exactly as the
// mean's butterfly and fold do
__device__ __forceinline__ void smx_merge(float& mu, float& s, float& a, float om, float os, float oa) {
  const float m = fmaxf(mu, om);
  const float r0 = smx_rescale(mu, m), r1 = smx_rescale(om, m);
  s = __fadd_rn(__fmul_rn(s, r0), __fmul_rn(os, r1));
  a = __fadd_rn(__fmul_rn(a, r0), __fmul_rn(oa, r1));
  mu = m;
}

// one message p with scaled logit y = fl(t p) into the online state: a new maximum rescales s and a first, then the
// message adds w = exp(y - mu) to s and w p to a. mu is only ever replaced by a larger y, so it is never NaN; a NaN
// message makes s and a NaN.
template <typename A> __device__ __forceinline__ void smx_update(A& mu, A& s, A& a, A y, A p) {
  if (y > mu) {
    const A r = smx_exp(mu - y);
    s *= r;
    a *= r;
    mu = y;
  }
  const A w = smx_exp(y - mu);
  s += w;
  a = fma(w, p, a);
}

// the stored result of a row of `count` entries: a / s (one IEEE division), +0 for an empty row
template <typename A> __device__ __forceinline__ A smx_result(A s, A a, int64_t count) {
  if (count == 0) return (A)0;
  if constexpr (std::is_same<A, double>::value) return __ddiv_rn(a, s);
  else return __fdiv_rn(a, s);
}

// the temperature and the log-sum-exp result of a forward launch: t[k * t_stride] (fp32), lse [M, K] fp32 or NULL
struct SmxArgs {
  const float* t;
  float* lse;
  uint32_t t_stride;
};

// the per-lane state of the softmax-aggregation kernels: VEC * CH columns of (mu, s, a) and their temperatures
template <typename T, int LPR, int CH, int U> struct SoftmaxAggrEngine {
  using V = Vec<T>;
  static constexpr bool Q8 = false;
  static constexpr int VEC = V::VEC;
  static constexpr int G = 32 / LPR;
  static constexpr int NA = VEC * CH;

  float mu[NA], s[NA], a[NA], t[NA];

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < NA; i++) {
      mu[i] = -INFINITY;
      s[i] = 0.f;
      a[i] = 0.f;
    }
  }
  // the lane's temperatures, loaded once per kernel by load_t
  __device__ __forceinline__ void set_t(const float (&tv)[NA]) {
#pragma unroll
    for (int i = 0; i < NA; i++) t[i] = tv[i];
  }
  static __device__ __forceinline__ void load_t(float (&tv)[NA], const SmxArgs& sa, const SpmmParams& p,
                                                const bool (&col_ok)[CH], int li) {
#pragma unroll
    for (int ch = 0; ch < CH; ch++)
#pragma unroll
      for (int i = 0; i < VEC; i++)
        tv[ch * VEC + i] = col_ok[ch] ? __ldg(sa.t + (p.k0 + (ch * LPR + li) * VEC + i) * sa.t_stride) : 0.f;
  }

  // one gathered vector of one entry: p = fl(v x) (exact for 16-bit operands), y = fl(t p)
  __device__ __forceinline__ void step(int ch, typename V::vraw v, const uint4& d) {
    const float vf = V::vfloat(v);
    float f[VEC];
    V::unpack(d, f);
#pragma unroll
    for (int i = 0; i < VEC; i++) {
      const int c = ch * VEC + i;
      const float pr = __fmul_rn(vf, f[i]);
      smx_update(mu[c], s[c], a[c], __fmul_rn(t[c], pr), pr);
    }
  }

  // ring-relative nnz [s0, e) of one row, G entries per step (one per lane group) and U steps per chunk, as
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
          if (act[u] && col_ok[ch]) step(ch, v[u], d[u][ch]);
      }
    }
  }

  // the butterfly of RowEngine::reduce_groups over the (mu, s, a) states
  __device__ __forceinline__ void reduce_groups() {
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
#pragma unroll
      for (int i = 0; i < NA; i++) {
        const float om = __shfl_xor_sync(0xffffffffu, mu[i], off);
        const float os = __shfl_xor_sync(0xffffffffu, s[i], off);
        const float oa = __shfl_xor_sync(0xffffffffu, a[i], off);
        smx_merge(mu[i], s[i], a[i], om, os, oa);
      }
    }
  }

  // final write of row `row` (count entries) by the lanes that hold it: a / s as T, and mu + log(s) where lse is set
  __device__ __forceinline__ void store_row(const SpmmParams& p, const SmxArgs& sa, int64_t row, int64_t count,
                                            const bool (&col_ok)[CH], int li) const {
    T* orow = (T*)p.out + row * p.K + p.k0;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
      float f[VEC];
#pragma unroll
      for (int i = 0; i < VEC; i++) f[i] = smx_result(s[ch * VEC + i], a[ch * VEC + i], count);
      stg128_stream(orow + koff, V::pack(f));
      if (sa.lse) {
        float* lrow = sa.lse + row * p.K + p.k0 + koff;
#pragma unroll
        for (int i = 0; i < VEC; i += 4) {
          float4 l;
          l.x = mu[ch * VEC + i] + logf(s[ch * VEC + i]);
          l.y = mu[ch * VEC + i + 1] + logf(s[ch * VEC + i + 1]);
          l.z = mu[ch * VEC + i + 2] + logf(s[ch * VEC + i + 2]);
          l.w = mu[ch * VEC + i + 3] + logf(s[ch * VEC + i + 3]);
          stg128_stream(lrow + i, *reinterpret_cast<const uint4*>(&l));
        }
      }
    }
  }

  // the partial of one segment into slot `slot`: three fp32 planes [slot][3][K] (mu, s, a)
  __device__ __forceinline__ void store_partial(const SpmmParams& p, int64_t slot, const bool (&col_ok)[CH],
                                                int li) const {
    float* pv = (float*)p.part_val + slot * 3 * p.K + p.k0;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!col_ok[ch]) continue;
      const int koff = (ch * LPR + li) * VEC;
#pragma unroll
      for (int i = 0; i < VEC; i++) {
        pv[koff + i] = mu[ch * VEC + i];
        pv[p.K + koff + i] = s[ch * VEC + i];
        pv[2 * p.K + koff + i] = a[ch * VEC + i];
      }
    }
  }
};

// column kk of a multi-segment row: its partials merged in segment order, then the result and lse stored. CG: read
// past L1 (the planned drain combines partials other SMs wrote during the same launch).
template <typename T, bool CG>
__device__ __forceinline__ void combine_smx_col(const SpmmParams& p, const SmxArgs& sa, const LongRow& L, int nseg,
                                                int64_t count, int64_t kk) {
  const float* pv = (const float*)p.part_val;
  auto ld = [&](int64_t sl, int st) {
    const float* q = pv + (sl * 3 + st) * p.K + kk;
    return CG ? __ldcg(q) : *q;
  };
  float mu = ld(L.first_slot, 0), s = ld(L.first_slot, 1), a = ld(L.first_slot, 2);
  for (int sgi = 1; sgi < nseg; sgi++) {
    const int64_t sl = L.first_slot + sgi;
    smx_merge(mu, s, a, ld(sl, 0), ld(sl, 1), ld(sl, 2));
  }
  ((T*)p.out)[L.row_b * p.K + kk] = Traits<T>::from_acc(smx_result(s, a, count));
  if (sa.lse) sa.lse[L.row_b * p.K + kk] = mu + logf(s);
}

// row-per-warp kernel: the work items of spmm_vec_kernel and, PLAN with DRAIN, its drain of the plan's segments
template <typename T, int LPR, int CH, int U, int MINB, bool PLAN, bool DRAIN>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_smx_vec_kernel(const SpmmParams p, const SmxArgs sa) {
  using Eng = SoftmaxAggrEngine<T, LPR, CH, U>;
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
  float tv[Eng::NA];
  Eng::load_t(tv, sa, p, col_ok, li);

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
      eng.set_t(tv);
      eng.init();
      eng.accumulate(ring, s, e, matb, row_bytes, col_ok, lane, g, pol);
      eng.reduce_groups();
      if (g == 0) eng.store_row(p, sa, it.r0 + rl, e - s, col_ok, li);
    }
  }

  if constexpr (PLAN && DRAIN) {  // the planned drain of spmm_vec_kernel
    constexpr int kcols = LPR * CH * VEC;
    while (true) {
      const unsigned int sidx = __shfl_sync(0xffffffffu, take_ticket(&p.counters[5], lane), 0);
      if ((int64_t)sidx >= p.n_seg) break;
      const Segment S = p.segs[sidx];
      Eng eng;
      eng.set_t(tv);
      walk_segment<false>(eng, p, S, 0, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
      if (S.slot < 0) {
        if (g == 0) eng.store_row(p, sa, S.row_b, S.end - S.start, col_ok, li);
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
            combine_smx_col<T, true>(p, sa, L, nseg, count, p.k0 + k);
        }
      }
      __syncwarp();
    }
  }
}

// group-per-row kernel (narrow rows): the walk of spmm_gpr_kernel, each lane group over its own row
template <typename T, int LPR, int U, int MINB, bool PLAN>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_smx_gpr_kernel(const SpmmParams p, const SmxArgs sa) {
  using V = Vec<T>;
  using Eng = SoftmaxAggrEngine<T, LPR, 1, U>;
  using VR = typename V::vraw;
  constexpr int VEC = Eng::VEC;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPR, li = lane % LPR;
  const bool col_ok = p.k0 + li * VEC < p.K;
  const bool col_ok_arr[1] = {col_ok};
  const uint32_t row_bytes = (uint32_t)(p.K * (int64_t)sizeof(T));
  const int64_t lane_off = ((int64_t)p.k0 + (int64_t)li * VEC) * (int64_t)sizeof(T);
  const uint64_t pol = make_policy_evict_last();
  const T* __restrict__ val = (const T*)p.value;
  const bool has_val = val != nullptr;
  float tv[Eng::NA];
  Eng::load_t(tv, sa, p, col_ok_arr, li);

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
      eng.set_t(tv);
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
          if (act[u]) eng.step(0, v[u], d[u]);
      }
      if (mine) eng.store_row(p, sa, it.r0 + rl, len, col_ok_arr, li);
    }
  }
}

// one warp per queued segment (spmm_seg_kernel)
template <typename T, int LPR, int CH, int U, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_smx_seg_kernel(const SpmmParams p, const SmxArgs sa) {
  using Eng = SoftmaxAggrEngine<T, LPR, CH, U>;
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
  float tv[Eng::NA];
  Eng::load_t(tv, sa, p, col_ok, li);

  const int64_t nseg = p.plan_mask ? p.n_seg : min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    Eng eng;
    eng.set_t(tv);
    walk_segment<false>(eng, p, S, 0, ring, col_ok, hcol, row_bytes, lane_off, lane, g, pol);
    if (g == 0) {
      if (S.slot < 0) eng.store_row(p, sa, S.row_b, S.end - S.start, col_ok, li);
      else eng.store_partial(p, S.slot, col_ok, li);
    }
    __syncwarp();
  }
}

// the multi-segment rows' partials, in segment order (spmm_combine_kernel)
template <typename T>
__global__ void spmm_smx_combine_kernel(const SpmmParams p, const SmxArgs sa, int kcols) {
  const int64_t nlong = p.plan_mask ? p.n_long : min((int64_t)p.counters[2], p.long_cap);
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    int nseg;
    int64_t count;
    long_row_counts(L, nseg, count);
    for (int k = threadIdx.x; k < kcols && p.k0 + k < p.K; k += blockDim.x)
      combine_smx_col<T, false>(p, sa, L, nseg, count, p.k0 + k);
  }
}

// generic kernel (fp64, partial widths, unaligned operands, E >= 2^31, E == 0): warp per row, lane per column, the
// entries in order, in the accumulator type A (fp32, fp64 for fp64), with exp the fp32 kernels' (fp64: exp)
template <typename T>
__global__ void __launch_bounds__(256)
spmm_smx_generic_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                        const T* __restrict__ value, const T* __restrict__ mat,
                        const typename Traits<T>::acc_t* __restrict__ t, int64_t t_stride, T* __restrict__ out,
                        typename Traits<T>::acc_t* __restrict__ lse, int64_t M, int64_t K) {
  using A = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t m = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < M; m += nw) {
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    for (int64_t k = lane; k < K; k += 32) {
      const A tk = t[k * t_stride];
      A mu = -INFINITY, s = 0, a = 0;
      for (int64_t e = rs; e < re; e++) {
        const A mv = Traits<T>::to_acc(mat[col[e] * K + k]);
        A pr = mv;
        if (value) {
          if constexpr (std::is_same<A, double>::value) pr = __dmul_rn(Traits<T>::to_acc(value[e]), mv);
          else pr = __fmul_rn(Traits<T>::to_acc(value[e]), mv);
        }
        A y;
        if constexpr (std::is_same<A, double>::value) y = __dmul_rn(tk, pr);
        else y = __fmul_rn(tk, pr);
        smx_update(mu, s, a, y, pr);
      }
      out[m * K + k] = Traits<T>::from_acc(smx_result(s, a, re - rs));
      if (lse) lse[m * K + k] = mu + log(s);
    }
  }
}

// workspace of tsb200_spmm_fw_softmax_aggr: the layouts of tsb200_spmm_fw (plan == NULL) or tsb200_spmm_fw_planned
// over 3 * K fp32 partial columns per slot (mu, s, a)
static inline size_t smx_ws_bytes(int64_t K, int64_t E, bool planned, int64_t n_long, int64_t n_slot) {
  return planned ? planned_ws(3 * K, n_long, n_slot, false).total : ws_layout(1, 3 * K, E, false).total;
}

template <typename T, int LPR, int CH, int U, int MINB, bool GPR, bool PLAN>
static int launch_smx(SpmmParams p, const SmxArgs& sa, cudaStream_t st) {
  constexpr int kcols = LPR * CH * Vec<T>::VEC;
  // as the multi kernels: the 16-bit kernel of the widest shape sends the plan's segments to the segment and combine
  // kernels instead of draining them itself
  constexpr bool DRAIN = !GPR && !(sizeof(T) == 2 && CH == 4);
  void (*kmain)(const SpmmParams, const SmxArgs);
  if constexpr (GPR) kmain = spmm_smx_gpr_kernel<T, LPR, U, MINB, PLAN>;
  else kmain = spmm_smx_vec_kernel<T, LPR, CH, U, MINB, PLAN, DRAIN>;
  constexpr int USEG = (U > LPR) ? LPR : U;
  auto* kseg = spmm_smx_seg_kernel<T, LPR, CH, USEG, MINB>;
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
      kmain<<<(int)max((int64_t)1, min((int64_t)grid_main, work)), kWarpsPerCta * 32, 0, st>>>(p, sa);
      TSB_LAUNCH_CHECK();
      if (!DRAIN && p.n_seg > 0) {
        kseg<<<gc_seg.get((const void*)kseg, kWarpsPerCta * 32), kWarpsPerCta * 32, 0, st>>>(p, sa);
        TSB_LAUNCH_CHECK();
        if (p.n_long > 0) {
          spmm_smx_combine_kernel<T><<<num_sms() * 2, 128, 0, st>>>(p, sa, kcols);
          TSB_LAUNCH_CHECK();
        }
      }
    } else {
      if (const int rc = launch_rowsplit(kmain, kseg, gc_main, gc_seg, p, st, sa)) return rc;
      spmm_smx_combine_kernel<T><<<num_sms() * 2, 128, 0, st>>>(p, sa, kcols);
      TSB_LAUNCH_CHECK();
    }
  }
  return 0;
}

// (LPR, CH) of dispatch_shape for each row width, so that every lane sums and folds as the mean kernels do; (U,
// CTAs/SM) the most CTAs/SM at which ptxas reports no spill for three states and a temperature per column (DESIGN §3.1)
template <typename T, bool PLAN>
static int dispatch_smx(const SpmmParams& p, const SmxArgs& sa, cudaStream_t st) {
  constexpr bool W16 = sizeof(T) == 2;
  const int64_t vecs = p.K / Vec<T>::VEC;
  if (vecs <= 1) return launch_smx<T, 1, 1, 4, 2, true, PLAN>(p, sa, st);
  if (vecs <= 2) return launch_smx<T, 2, 1, 4, 2, true, PLAN>(p, sa, st);
  if (vecs <= 4) return launch_smx<T, 4, 1, 4, 2, true, PLAN>(p, sa, st);
  if (vecs <= 8) return launch_smx<T, 8, 1, 4, 2, true, PLAN>(p, sa, st);
  if (vecs <= 16) return launch_smx<T, 16, 1, 4, 2, false, PLAN>(p, sa, st);
  if (vecs <= 32) return launch_smx<T, 32, 1, 4, 2, false, PLAN>(p, sa, st);
  if (vecs <= 64) return launch_smx<T, 32, 2, 2, W16 ? 1 : 2, false, PLAN>(p, sa, st);
  return launch_smx<T, 32, 4, W16 ? 1 : 2, 1, false, PLAN>(p, sa, st);
}

// ---- backward ------------------------------------------------------------------------------------------------------
// With g = grad_out, o = out and l = lse of row r, the gradient of message e in column k is
//   d_e = g alpha_e (1 + t (p_e - o)),   alpha_e = exp(t p_e - l).
// Two row-split kernels take the vector path: the row-wise one (grad_value and the temperature plane U) over the CSR
// view, the column-wise one (grad_mat) over the CSC view, where colptr, row_csc and value[csr2csc] play the roles of
// rowptr, col and value. Both defer long rows (columns) by defer_row into the segment queue and fold a multi-segment
// row's partials in segment order; the generic kernels below take fp64 and everything else. Every sum runs in a fixed
// order in the accumulator type, with no atomics, so every gradient is reproducible bit for bit.
template <typename A> __device__ __forceinline__ A smx_alpha(A t, A pr, A l) {
  if constexpr (std::is_same<A, double>::value) return exp(__dmul_rn(t, pr) - l);
  else return smx_exp(__fmul_rn(t, pr) - l);
}

// the operands of a backward launch besides SpmmParams: the temperature, grad_out, the forward's out and lse (fp32),
// and the outputs grad_value (T [E], NULL: not wanted) and U (fp32 [M, K], NULL: not wanted). The column-wise kernel
// writes grad_mat through SpmmParams::out.
struct SmxBwArgs {
  const float* t;
  const void* g;
  const void* o;
  const float* lse;
  void* gv;
  float* U;
  uint32_t t_stride;
};

// VEC consecutive fp32 values of an fp32 row at column koff (16-byte loads)
__device__ __forceinline__ void ld_f32(const float* row, int koff, float* f, int n) {
  for (int i = 0; i < n; i += 4) {
    const uint4 q = ldg128(row + koff + i);
    f[i] = __uint_as_float(q.x); f[i + 1] = __uint_as_float(q.y);
    f[i + 2] = __uint_as_float(q.z); f[i + 3] = __uint_as_float(q.w);
  }
}

// One warp walks entries [s, e) of row r (COLS: of column r of the CSC view), G = 32 / LPR entries per step, one per
// lane group; the lanes of a group hold VEC * CH consecutive feature columns (the forward's lane layout). The row's
// own operands stay in registers: g, o and lse of row r (rows), or x[r] (columns); the other side is gathered per
// entry: x[col_e] (rows), or g, o and lse of row row_csc[j] (columns). acc gets this lane group's column sums:
// sum alpha (p - o)^2 (rows, when U is wanted) or sum v d (columns); the rows walk also writes grad_value[e] for every
// entry, the dot product <x[col_e], d_e> reduced over the group's lanes.
template <bool COLS, typename T, int LPR, int CH>
__device__ __forceinline__ void smx_bw_walk(const SpmmParams& p, const SmxBwArgs& ba, int64_t r, int64_t s, int64_t e,
                                            const bool (&col_ok)[CH], const float (&tv)[Vec<T>::VEC * CH], int li,
                                            int g, float (&acc)[Vec<T>::VEC * CH]) {
  using V = Vec<T>;
  constexpr int VEC = V::VEC, G = 32 / LPR, NA = VEC * CH;
  const int64_t rb = p.K * (int64_t)sizeof(T);
  float own0[NA], own1[NA], own2[NA];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) {
    const int koff = (ch * LPR + li) * VEC;
    if (!col_ok[ch]) continue;
    if constexpr (COLS) {
      V::unpack(ldg128((const char*)p.mat + r * rb + koff * (int64_t)sizeof(T)), &own0[ch * VEC]);
    } else {
      V::unpack(ldg128((const T*)ba.g + r * p.K + koff), &own0[ch * VEC]);
      V::unpack(ldg128((const T*)ba.o + r * p.K + koff), &own1[ch * VEC]);
      ld_f32(ba.lse + r * p.K, koff, &own2[ch * VEC], VEC);
    }
  }
#pragma unroll
  for (int i = 0; i < NA; i++) acc[i] = 0.f;
  const bool has_val = p.value != nullptr;
  const bool want_u = COLS || ba.U != nullptr, want_v = !COLS && ba.gv != nullptr;
  for (int64_t j0 = s; j0 < e; j0 += G) {
    const int64_t j = j0 + g;
    const bool act = j < e;
    uint32_t c = 0;
    float v = 1.f;
    if (act) {
      c = (uint32_t)__ldg(p.col + j);
      if (has_val) v = V::vfloat(load_vraw<T>((const T*)p.value + j));
    }
    float dot = 0.f;
#pragma unroll
    for (int ch = 0; ch < CH; ch++) {
      if (!(act && col_ok[ch])) continue;
      const int koff = (ch * LPR + li) * VEC;
      float x[VEC], gg[VEC], oo[VEC], ll[VEC];
      if constexpr (COLS) {
        V::unpack(ldg128((const T*)ba.g + (int64_t)c * p.K + koff), gg);
        V::unpack(ldg128((const T*)ba.o + (int64_t)c * p.K + koff), oo);
        ld_f32(ba.lse + (int64_t)c * p.K, koff, ll, VEC);
      } else {
        V::unpack(ldg128((const char*)p.mat + (int64_t)c * rb + koff * (int64_t)sizeof(T)), x);
      }
#pragma unroll
      for (int i = 0; i < VEC; i++) {
        const int a = ch * VEC + i;
        const float xi = COLS ? own0[a] : x[i];
        const float gi = COLS ? gg[i] : own0[a], oi = COLS ? oo[i] : own1[a], li_ = COLS ? ll[i] : own2[a];
        const float pr = __fmul_rn(v, xi);
        const float al = smx_alpha(tv[a], pr, li_);
        const float dp = pr - oi;
        if constexpr (COLS) {
          acc[a] = fmaf(v, gi * al * fmaf(tv[a], dp, 1.f), acc[a]);
        } else {
          if (want_u) acc[a] = fmaf(al * dp, dp, acc[a]);
          if (want_v) dot = fmaf(xi, gi * al * fmaf(tv[a], dp, 1.f), dot);
        }
      }
    }
    if (want_v) {
#pragma unroll
      for (int off = 1; off < LPR; off <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
      if (act && li == 0) ((T*)ba.gv)[j] = Traits<T>::from_acc(dot);
    }
  }
  // the lane groups' column sums, by the butterfly of RowEngine::reduce_groups
#pragma unroll
  for (int off = LPR; off < 32; off <<= 1)
#pragma unroll
    for (int i = 0; i < NA; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
}

// the result of row (column) r from the column sums of a whole row, by group 0: U[r] = g[r] * acc (rows) or
// grad_mat[r] = acc (columns); a segment of a multi-segment row stores acc as its fp32 partial in slot `slot`
template <bool COLS, typename T, int LPR, int CH>
__device__ __forceinline__ void smx_bw_store(const SpmmParams& p, const SmxBwArgs& ba, int64_t r, int64_t slot,
                                             const bool (&col_ok)[CH], int li, const float (&acc)[Vec<T>::VEC * CH]) {
  constexpr int VEC = Vec<T>::VEC;
  if (!COLS && !ba.U) return;
#pragma unroll
  for (int ch = 0; ch < CH; ch++) {
    if (!col_ok[ch]) continue;
    const int koff = (ch * LPR + li) * VEC;
    if (slot >= 0) {
      float* pv = (float*)p.part_val + slot * p.K + koff;
#pragma unroll
      for (int i = 0; i < VEC; i++) pv[i] = acc[ch * VEC + i];
    } else if constexpr (COLS) {
      stg128_stream((T*)p.out + r * p.K + koff, Vec<T>::pack(&acc[ch * VEC]));
    } else {
      float gg[VEC];
      Vec<T>::unpack(ldg128((const T*)ba.g + r * p.K + koff), gg);
#pragma unroll
      for (int i = 0; i < VEC; i++) ba.U[r * p.K + koff + i] = gg[i] * acc[ch * VEC + i];
    }
  }
}

// the lane's columns and temperatures of the backward kernels (one column tile: K * sizeof(T) <= 1024)
template <typename T, int LPR, int CH>
__device__ __forceinline__ void smx_bw_lane(const SpmmParams& p, const SmxBwArgs& ba, int li, bool (&col_ok)[CH],
                                            float (&tv)[Vec<T>::VEC * CH]) {
  constexpr int VEC = Vec<T>::VEC;
#pragma unroll
  for (int ch = 0; ch < CH; ch++) {
    col_ok[ch] = (ch * LPR + li) * VEC < p.K;
#pragma unroll
    for (int i = 0; i < VEC; i++)
      tv[ch * VEC + i] = col_ok[ch] ? __ldg(ba.t + ((ch * LPR + li) * VEC + i) * ba.t_stride) : 0.f;
  }
}

// main kernel: the work items of spmm_vec_kernel (unplanned), each row walked by the whole warp
template <bool COLS, typename T, int LPR, int CH, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_smx_bw_vec_kernel(const SpmmParams p, const SmxBwArgs ba) {
  constexpr int NA = Vec<T>::VEC * CH;
  const int lane = threadIdx.x & 31, g = lane / LPR, li = lane % LPR;
  bool col_ok[CH];
  float tv[NA];
  smx_bw_lane<T, LPR, CH>(p, ba, li, col_ok, tv);
  for (WorkItem it(p, lane); it.start(p, lane); it.advance()) {
    const int deg = (int)(it.rp1 - it.rp0);
    const bool defer = defer_row(deg, lane);
    const unsigned defer_mask = __ballot_sync(0xffffffffu, defer);
    if (defer) push_row_segments(p, it.b, it.r0, lane, it.rp0, it.rp1, deg);
    __syncwarp();
    for (int rl = 0; rl < it.nrows; rl++) {
      if ((defer_mask >> rl) & 1u) continue;
      const int64_t s = __shfl_sync(0xffffffffu, it.rp0, rl), e = __shfl_sync(0xffffffffu, it.rp1, rl);
      float acc[NA];
      smx_bw_walk<COLS, T, LPR, CH>(p, ba, it.r0 + rl, s, e, col_ok, tv, li, g, acc);
      if (g == 0) smx_bw_store<COLS, T, LPR, CH>(p, ba, it.r0 + rl, -1, col_ok, li, acc);
    }
  }
}

// one warp per queued segment (spmm_seg_kernel)
template <bool COLS, typename T, int LPR, int CH, int MINB>
__global__ void __launch_bounds__(kWarpsPerCta * 32, MINB)
spmm_smx_bw_seg_kernel(const SpmmParams p, const SmxBwArgs ba) {
  constexpr int NA = Vec<T>::VEC * CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane / LPR, li = lane % LPR;
  bool col_ok[CH];
  float tv[NA];
  smx_bw_lane<T, LPR, CH>(p, ba, li, col_ok, tv);
  const int64_t nseg = min((int64_t)p.counters[1], p.seg_cap);
  const int64_t wstride = (int64_t)gridDim.x * kWarpsPerCta;
  for (int64_t sidx = (int64_t)blockIdx.x * kWarpsPerCta + warp; sidx < nseg; sidx += wstride) {
    const Segment S = p.segs[sidx];
    float acc[NA];
    smx_bw_walk<COLS, T, LPR, CH>(p, ba, S.row_b, S.start, S.end, col_ok, tv, li, g, acc);
    if (g == 0) smx_bw_store<COLS, T, LPR, CH>(p, ba, S.row_b, S.slot, col_ok, li, acc);
    __syncwarp();
  }
}

// the multi-segment rows' partials, summed in segment order: U[r] = g[r] * sum (rows) or grad_mat[r] = sum (columns)
template <bool COLS, typename T>
__global__ void spmm_smx_bw_combine_kernel(const SpmmParams p, const SmxBwArgs ba) {
  if (!COLS && !ba.U) return;
  const int64_t nlong = min((int64_t)p.counters[2], p.long_cap);
  const float* pv = (const float*)p.part_val;
  for (int64_t li = blockIdx.x; li < nlong; li += gridDim.x) {
    const LongRow L = p.longs[li];
    int nseg;
    int64_t count;
    long_row_counts(L, nseg, count);
    for (int64_t k = threadIdx.x; k < p.K; k += blockDim.x) {
      float a = pv[L.first_slot * p.K + k];
      for (int sgi = 1; sgi < nseg; sgi++) a += pv[(L.first_slot + sgi) * p.K + k];
      if constexpr (COLS) ((T*)p.out)[L.row_b * p.K + k] = Traits<T>::from_acc(a);
      else ba.U[L.row_b * p.K + k] = Traits<T>::to_acc(((const T*)ba.g)[L.row_b * p.K + k]) * a;
    }
  }
}

template <bool COLS, typename T, int LPR, int CH, int MINB>
static int launch_smx_bw(SpmmParams p, const SmxBwArgs& ba, cudaStream_t st) {
  auto* kmain = spmm_smx_bw_vec_kernel<COLS, T, LPR, CH, MINB>;
  auto* kseg = spmm_smx_bw_seg_kernel<COLS, T, LPR, CH, MINB>;
  static GridCache gc_main, gc_seg;
  if (const int rc = launch_rowsplit(kmain, kseg, gc_main, gc_seg, p, st, ba)) return rc;
  spmm_smx_bw_combine_kernel<COLS, T><<<num_sms() * 2, 128, 0, st>>>(p, ba);
  TSB_LAUNCH_CHECK();
  return 0;
}

// the forward's (LPR, CH) for rows of up to 1024 bytes; (CTAs/SM) the most at which ptxas reports no spill (DESIGN §3.1)
template <bool COLS, typename T>
static int dispatch_smx_bw(const SpmmParams& p, const SmxBwArgs& ba, cudaStream_t st) {
  constexpr int MB = sizeof(T) == 4 ? 4 : 3;  // CTAs/SM of the one-chunk shapes
  const int64_t vecs = p.K / Vec<T>::VEC;
  if (vecs <= 1) return launch_smx_bw<COLS, T, 1, 1, MB>(p, ba, st);
  if (vecs <= 2) return launch_smx_bw<COLS, T, 2, 1, MB>(p, ba, st);
  if (vecs <= 4) return launch_smx_bw<COLS, T, 4, 1, MB>(p, ba, st);
  if (vecs <= 8) return launch_smx_bw<COLS, T, 8, 1, MB>(p, ba, st);
  if (vecs <= 16) return launch_smx_bw<COLS, T, 16, 1, MB>(p, ba, st);
  if (vecs <= 32) return launch_smx_bw<COLS, T, 32, 1, MB>(p, ba, st);
  return launch_smx_bw<COLS, T, 32, 2, 2>(p, ba, st);
}

// whether a backward call takes the row-split kernels: F32 / F16 / BF16, rows of 16 ... 1024 bytes, E > 0, the
// row-split extents (E entries, `gathered` rows of the gathered operands) and the 16-byte alignment of every dense
// operand
static bool smx_bw_vec(int dtype, int64_t K, int64_t E, int64_t gathered, const int64_t* col, const void* value,
                       std::initializer_list<const void*> rows) {
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return false;
  const int64_t row_bytes = K * (int64_t)dtype_size(dtype);
  return E > 0 && row_bytes % 16 == 0 && row_bytes <= 1024 && rowsplit_extents(E, gathered, row_bytes) &&
         rowsplit_aligned(rows, col, {value});
}

// generic row-wise kernel (fp64, rows not a multiple of 16 bytes or wider than 1024, unaligned operands, E >= 2^31):
// a warp per row, a lane per column. grad_value[e] = <x[col_e], d_e> (the lanes' columns summed, then a butterfly over
// the warp) and U[r, k] = g sum_e alpha_e (p_e - o)^2 (the temperature gradient per row and column, summed by the
// caller)
template <typename T>
__global__ void __launch_bounds__(256)
spmm_smx_bw_rows_kernel(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ col,
                        const T* __restrict__ value, const T* __restrict__ mat,
                        const typename Traits<T>::acc_t* __restrict__ t, int64_t t_stride,
                        const T* __restrict__ grad_out, const T* __restrict__ out,
                        const typename Traits<T>::acc_t* __restrict__ lse, T* __restrict__ grad_value,
                        typename Traits<T>::acc_t* __restrict__ U, int64_t M, int64_t K) {
  using A = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t m = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < M; m += nw) {
    const int64_t rs = rowptr[m], re = rowptr[m + 1];
    if (U) {
      for (int64_t k = lane; k < K; k += 32) {
        const A tk = t[k * t_stride], o = Traits<T>::to_acc(out[m * K + k]), l = lse[m * K + k];
        A u = 0;
        for (int64_t e = rs; e < re; e++) {
          const A mv = Traits<T>::to_acc(mat[col[e] * K + k]);
          const A pr = value ? Traits<T>::to_acc(value[e]) * mv : mv;
          const A dp = pr - o;
          u = fma(smx_alpha(tk, pr, l) * dp, dp, u);
        }
        U[m * K + k] = Traits<T>::to_acc(grad_out[m * K + k]) * u;
      }
    }
    if (grad_value) {
      for (int64_t e = rs; e < re; e++) {
        const int64_t c = col[e];
        const A v = value ? Traits<T>::to_acc(value[e]) : (A)1;
        A dot = 0;
        for (int64_t k = lane; k < K; k += 32) {
          const A tk = t[k * t_stride], o = Traits<T>::to_acc(out[m * K + k]), l = lse[m * K + k];
          const A g = Traits<T>::to_acc(grad_out[m * K + k]);
          const A mv = Traits<T>::to_acc(mat[c * K + k]);
          const A pr = v * mv;
          dot = fma(mv, g * smx_alpha(tk, pr, l) * fma(tk, pr - o, (A)1), dot);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
        if (lane == 0) grad_value[e] = Traits<T>::from_acc(dot);
      }
    }
  }
}

// generic column-wise kernel, on the CSC view (colptr, row_csc, value_csc = value[csr2csc]): grad_mat[n, k] =
// sum_j v_j d_j over the entries j of column n, with x[n, k] held in a register and g, o, lse of row row_csc[j]
// gathered
template <typename T>
__global__ void __launch_bounds__(256, 2)
spmm_smx_bw_cols_kernel(const int64_t* __restrict__ colptr, const int64_t* __restrict__ row_csc,
                        const T* __restrict__ value_csc, const T* __restrict__ mat,
                        const typename Traits<T>::acc_t* __restrict__ t, int64_t t_stride,
                        const T* __restrict__ grad_out, const T* __restrict__ out,
                        const typename Traits<T>::acc_t* __restrict__ lse, T* __restrict__ grad_mat, int64_t N,
                        int64_t K) {
  using A = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < N; n += nw) {
    const int64_t js = colptr[n], je = colptr[n + 1];
    for (int64_t k = lane; k < K; k += 32) {
      const A tk = t[k * t_stride], mv = Traits<T>::to_acc(mat[n * K + k]);
      A acc = 0;
      for (int64_t j = js; j < je; j++) {
        const int64_t r = row_csc[j];
        const A v = value_csc ? Traits<T>::to_acc(value_csc[j]) : (A)1;
        const A pr = v * mv;
        const A o = Traits<T>::to_acc(out[r * K + k]), l = lse[r * K + k], g = Traits<T>::to_acc(grad_out[r * K + k]);
        acc = fma(v, g * smx_alpha(tk, pr, l) * fma(tk, pr - o, (A)1), acc);
      }
      grad_mat[n * K + k] = Traits<T>::from_acc(acc);
    }
  }
}

// the argument checks shared by the three entry points: 0 or the error code
static int smx_check(int64_t M, int64_t N, int64_t K, int64_t E, int dtype, int64_t t_stride, const void* t) {
  if (M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  if (t_stride != 0 && t_stride != 1) return TSB200_ERR_INVALID_ARG;
  if (dtype_size(dtype) == 0) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F64 && dtype != TSB200_F16 && dtype != TSB200_BF16)
    return TSB200_ERR_UNSUPPORTED;
  if ((uintptr_t)t & (dtype == TSB200_F64 ? 7 : 3)) return TSB200_ERR_UNSUPPORTED;
  return 0;
}

}  // namespace tsb

using namespace tsb;

// The definitions take their C linkage from the declarations in tsb200.h; the guards below make any drift between the
// two a compile error (see tsb200_spmm_fw_res).
size_t tsb200_spmm_fw_softmax_aggr_workspace_bytes(int64_t K, int64_t E, int planned, int64_t n_long, int64_t n_slot) {
  if (K <= 0 || E <= 0 || n_long < 0 || n_slot < 0) return 0;
  return smx_ws_bytes(K, E, planned != 0, n_long, n_slot);
}

int tsb200_spmm_fw_softmax_aggr(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                const void* t, int64_t t_stride, void* out, void* lse, int64_t M, int64_t N, int64_t K,
                                int64_t E, int dtype, const void* plan, size_t plan_bytes, int64_t n_seg,
                                int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes,
                                void* stream) {
  if (n_seg < 0 || n_long < 0 || n_slot < 0) return TSB200_ERR_INVALID_ARG;
  if (const int rc = smx_check(M, N, K, E, dtype, t_stride, t)) return rc;
  if (M * K == 0) return 0;  // nothing to write
  if (!rowptr || !out || !t) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col || !mat)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;

  const int64_t row_bytes = K * (int64_t)dtype_size(dtype);
  if (E > 0 && (dtype == TSB200_F32 || dtype == TSB200_F16 || dtype == TSB200_BF16) && row_bytes % 16 == 0 &&
      rowsplit_extents(E, N, row_bytes) && rowsplit_aligned({mat, out, lse}, col, {value})) {
    SpmmParams p{rowptr, col, value, mat, out, nullptr, 1, M, N, K, E};
    // the partial planes bound as a workspace of 3 * K partial columns
    SpmmParams q = p;
    q.K = 3 * K;
    if (const int rc = bind_workspace(q, plan, plan_bytes, n_seg, n_long, n_slot, workspace, workspace_bytes, false))
      return rc;
    q.K = K;
    const SmxArgs sa{(const float*)t, (float*)lse, (uint32_t)t_stride};
    return dispatch_vec_dtype(dtype, [&](auto tag) {
      using T = decltype(tag);
      return plan ? dispatch_smx<T, true>(q, sa, st) : dispatch_smx<T, false>(q, sa, st);
    });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    using A = typename Traits<T>::acc_t;
    spmm_smx_generic_kernel<T><<<warp_grid(M, 64), 256, 0, st>>>(rowptr, col, (const T*)value, (const T*)mat,
                                                                 (const A*)t, t_stride, (T*)out, (A*)lse, M, K);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

size_t tsb200_spmm_softmax_aggr_bw_workspace_bytes(int64_t K, int64_t E) {
  if (K <= 0 || E <= 0) return 0;
  return ws_layout(1, K, E, false).total;
}

int tsb200_spmm_softmax_aggr_bw_rows(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                     const void* t, int64_t t_stride, const void* grad_out, const void* out,
                                     const void* lse, void* grad_value, void* U, int64_t M, int64_t N, int64_t K,
                                     int64_t E, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = smx_check(M, N, K, E, dtype, t_stride, t)) return rc;
  if (!grad_value && !U) return 0;  // no gradient wanted
  if (grad_value && !value) return TSB200_ERR_INVALID_ARG;
  if (M == 0 || (K == 0 && !grad_value)) return 0;
  if (!rowptr || !t || !grad_out || !out || !lse) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col || !mat)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (smx_bw_vec(dtype, K, E, N, col, value, {mat, grad_out, out, lse})) {
    SpmmParams p{rowptr, col, value, mat, nullptr, nullptr, 1, M, N, K, E};
    if (const int rc = bind_unplanned(p, workspace, workspace_bytes, false)) return rc;
    const SmxBwArgs ba{(const float*)t, grad_out, out, (const float*)lse, grad_value, (float*)U, (uint32_t)t_stride};
    return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_smx_bw<false, decltype(tag)>(p, ba, st); });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    using A = typename Traits<T>::acc_t;
    spmm_smx_bw_rows_kernel<T><<<warp_grid(M, 64), 256, 0, st>>>(
        rowptr, col, (const T*)value, (const T*)mat, (const A*)t, t_stride, (const T*)grad_out, (const T*)out,
        (const A*)lse, (T*)grad_value, (A*)U, M, K);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

int tsb200_spmm_softmax_aggr_bw_cols(const int64_t* colptr, const int64_t* row_csc, const void* value_csc,
                                     const void* mat, const void* t, int64_t t_stride, const void* grad_out,
                                     const void* out, const void* lse, void* grad_mat, int64_t M, int64_t N, int64_t K,
                                     int64_t E, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = smx_check(M, N, K, E, dtype, t_stride, t)) return rc;
  if (!grad_mat || N * K == 0) return 0;  // nothing wanted or nothing to write
  if (!colptr || !mat || !t) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!row_csc || !grad_out || !out || !lse)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (smx_bw_vec(dtype, K, E, M, row_csc, value_csc, {mat, grad_out, out, lse, grad_mat})) {
    // the CSC view walked as a CSR matrix of N rows whose entries gather rows of g, o and lse
    SpmmParams p{colptr, row_csc, value_csc, mat, grad_mat, nullptr, 1, N, M, K, E};
    if (const int rc = bind_unplanned(p, workspace, workspace_bytes, false)) return rc;
    const SmxBwArgs ba{(const float*)t, grad_out, out, (const float*)lse, nullptr, nullptr, (uint32_t)t_stride};
    return dispatch_vec_dtype(dtype, [&](auto tag) { return dispatch_smx_bw<true, decltype(tag)>(p, ba, st); });
  }
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    using A = typename Traits<T>::acc_t;
    spmm_smx_bw_cols_kernel<T><<<warp_grid(N, 64), 256, 0, st>>>(
        colptr, row_csc, (const T*)value_csc, (const T*)mat, (const A*)t, t_stride, (const T*)grad_out,
        (const T*)out, (const A*)lse, (T*)grad_mat, N, K);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

[[maybe_unused]] static constexpr auto tsb200_spmm_fw_softmax_aggr_declared_once = &tsb200_spmm_fw_softmax_aggr;
[[maybe_unused]] static constexpr auto tsb200_spmm_fw_softmax_aggr_workspace_bytes_declared_once =
    &tsb200_spmm_fw_softmax_aggr_workspace_bytes;
[[maybe_unused]] static constexpr auto tsb200_spmm_softmax_aggr_bw_rows_declared_once =
    &tsb200_spmm_softmax_aggr_bw_rows;
[[maybe_unused]] static constexpr auto tsb200_spmm_softmax_aggr_bw_cols_declared_once =
    &tsb200_spmm_softmax_aggr_bw_cols;
[[maybe_unused]] static constexpr auto tsb200_spmm_softmax_aggr_bw_workspace_bytes_declared_once =
    &tsb200_spmm_softmax_aggr_bw_workspace_bytes;
