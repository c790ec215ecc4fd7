// softmax.cu — softmax of a sparse matrix's stored values over each row (CSR segments) or column (CSC segments
// through csr2csc), one softmax per trailing value column, forward and backward (no counterpart in the reference).
//
// Mapping. A segment is the contiguous [n, D] block of a row's values (for columns: n rows of D values gathered
// through perm). D is cut into C = D / V chunks of V columns, V the widest power of two up to 16 bytes that divides
// D; a work item is one (segment, chunk) pair, and every lane of an item owns the chunk of its entries. One CTA of
// 256 threads takes 256 consecutive segments; by length n a segment goes to
//   short  (n <= 32):  8 lanes per item, 4 items per warp, each lane holding up to 4 entries in registers;
//   medium (n <= 128): a warp per item, each lane holding up to 4 entries in registers;
//   long   (n > 128):  the whole CTA per item, three passes over the block (max, sum, write; the later from L2).
// So a short or medium segment is read once and written once, and a hub row runs on a CTA while the other CTAs go on.
// The vector form loads and stores V-wide chunks when every operand is aligned to V elements; the scalar form runs
// the same arithmetic element by element, so alignment never changes a bit.
//
// Arithmetic, in A = fp32 (fp64 for fp64), per segment and column: m = max_j v_j with any NaN winning;
// e_j = exp(fl(v_j - m)) (expf / exp); S = sum_j e_j, each lane adding its entries in order and the lanes combined by
// a fixed butterfly (the CTA path: butterfly within a warp, then the warps in order); out_j = round(e_j / S) with an
// IEEE division. The order depends only on n and D. Backward: dot = sum_k alpha_k g_k by FMA in the same order,
// grad_j = round(alpha_j * (g_j - dot)). No atomics, no host synchronisation.
#include "common.cuh"

namespace tsb {

constexpr int kSoftmaxThreads = 256;   // threads per CTA = segments per CTA
constexpr int kShortLanes = 8;         // lanes per short item
constexpr int kHeld = 4;               // entries a lane holds in registers (short and medium)
constexpr int64_t kShortMax = kShortLanes * kHeld;  // 32
constexpr int64_t kMediumMax = 32 * kHeld;          // 128
constexpr unsigned kFull = 0xffffffffu;

template <typename A> __device__ __forceinline__ A nan_max(A a, A b) { return (b > a || b != b) ? b : a; }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float exp_acc(float x) { return expf(x); }
__device__ __forceinline__ double exp_acc(double x) { return exp(x); }

// V consecutive elements, loaded and stored as one V * sizeof(T)-byte access (VEC) or element by element.
template <typename T, int V, bool VEC> struct Chunk {
  using A = typename Traits<T>::acc_t;
  static constexpr int kBytes = V * (int)sizeof(T);
  using W = std::conditional_t<kBytes == 16, uint4,
            std::conditional_t<kBytes == 8, uint2, std::conditional_t<kBytes == 4, uint32_t, uint16_t>>>;
  static __device__ __forceinline__ void load(const T* __restrict__ p, A (&x)[V]) {
    T v[V];
    if constexpr (VEC) {
      const W w = *reinterpret_cast<const W*>(p);
      memcpy(v, &w, sizeof(W));
    } else {
#pragma unroll
      for (int i = 0; i < V; i++) v[i] = p[i];
    }
#pragma unroll
    for (int i = 0; i < V; i++) x[i] = Traits<T>::to_acc(v[i]);
  }
  static __device__ __forceinline__ void store(T* __restrict__ p, const A (&x)[V]) {
    T v[V];
#pragma unroll
    for (int i = 0; i < V; i++) v[i] = Traits<T>::from_acc(x[i]);
    if constexpr (VEC) {
      W w;
      memcpy(&w, v, sizeof(W));
      *reinterpret_cast<W*>(p) = w;
    } else {
#pragma unroll
      for (int i = 0; i < V; i++) p[i] = v[i];
    }
  }
};

// butterflies over groups of P lanes: every lane of the group ends with the same bits
template <int P, typename A, int V> __device__ __forceinline__ void group_max(A (&m)[V]) {
#pragma unroll
  for (int o = P / 2; o > 0; o >>= 1)
#pragma unroll
    for (int i = 0; i < V; i++) m[i] = nan_max(m[i], __shfl_xor_sync(kFull, m[i], o, P));
}
template <int P, typename A, int V> __device__ __forceinline__ void group_sum(A (&s)[V]) {
#pragma unroll
  for (int o = P / 2; o > 0; o >>= 1)
#pragma unroll
    for (int i = 0; i < V; i++) s[i] = s[i] + __shfl_xor_sync(kFull, s[i], o, P);
}

// CTA-wide combine of per-thread values: warp butterfly, then the warps in order. `red` holds 8 * V values; the
// trailing barrier lets the caller reuse it.
template <bool MAX, typename A, int V> __device__ __forceinline__ void cta_combine(A (&x)[V], A* red) {
  if constexpr (MAX) group_max<32>(x); else group_sum<32>(x);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < V; i++) red[w * V + i] = x[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < V; i++) {
    A a = red[i];
    for (int k = 1; k < kSoftmaxThreads / 32; k++) a = MAX ? nan_max(a, red[k * V + i]) : a + red[k * V + i];
    x[i] = a;
  }
  __syncthreads();
}

// The address of entry j's chunk: row b + j of the block, or row perm[b + j] for a column.
__device__ __forceinline__ int64_t entry_off(const int64_t* __restrict__ perm, int64_t b, int64_t j, int64_t D,
                                             int64_t c0) {
  const int64_t src = perm ? __ldg(perm + b + j) : b + j;
  return src * D + c0;
}

template <typename T, int V, bool VEC> struct SoftmaxFw {
  using A = typename Traits<T>::acc_t;
  using IO = Chunk<T, V, VEC>;
  static constexpr int kV = V;
  const int64_t* perm;
  const T* value;
  T* out;
  int64_t D;

  // one item on a group of P lanes (p = lane in group), n <= P * kHeld; n = 0 only joins the shuffles
  template <int P> __device__ __forceinline__ void regs(int64_t b, int n, int64_t c0, int p) const {
    A x[kHeld][V], m[V], s[V];
    int64_t off[kHeld];
#pragma unroll
    for (int i = 0; i < V; i++) { m[i] = -std::numeric_limits<A>::infinity(); s[i] = (A)0; }
#pragma unroll
    for (int r = 0; r < kHeld; r++) {
      off[r] = 0;
      if (p + r * P < n) {
        off[r] = entry_off(perm, b, p + r * P, D, c0);
        IO::load(value + off[r], x[r]);
#pragma unroll
        for (int i = 0; i < V; i++) m[i] = nan_max(m[i], x[r][i]);
      }
    }
    group_max<P>(m);
#pragma unroll
    for (int r = 0; r < kHeld; r++) {
      if (p + r * P < n) {
#pragma unroll
        for (int i = 0; i < V; i++) { x[r][i] = exp_acc(x[r][i] - m[i]); s[i] = s[i] + x[r][i]; }
      }
    }
    group_sum<P>(s);
#pragma unroll
    for (int r = 0; r < kHeld; r++) {
      if (p + r * P < n) {
#pragma unroll
        for (int i = 0; i < V; i++) x[r][i] = div_rn(x[r][i], s[i]);
        IO::store(out + off[r], x[r]);
      }
    }
  }

  __device__ __forceinline__ void cta(int64_t b, int64_t n, int64_t c0, A* red) const {
    A x[V], m[V], s[V];
#pragma unroll
    for (int i = 0; i < V; i++) { m[i] = -std::numeric_limits<A>::infinity(); s[i] = (A)0; }
#pragma unroll 4
    for (int64_t j = threadIdx.x; j < n; j += kSoftmaxThreads) {
      IO::load(value + entry_off(perm, b, j, D, c0), x);
#pragma unroll
      for (int i = 0; i < V; i++) m[i] = nan_max(m[i], x[i]);
    }
    cta_combine<true>(m, red);
#pragma unroll 4
    for (int64_t j = threadIdx.x; j < n; j += kSoftmaxThreads) {
      IO::load(value + entry_off(perm, b, j, D, c0), x);
#pragma unroll
      for (int i = 0; i < V; i++) s[i] = s[i] + exp_acc(x[i] - m[i]);
    }
    cta_combine<false>(s, red);
#pragma unroll 4
    for (int64_t j = threadIdx.x; j < n; j += kSoftmaxThreads) {
      const int64_t o = entry_off(perm, b, j, D, c0);
      IO::load(value + o, x);
#pragma unroll
      for (int i = 0; i < V; i++) x[i] = div_rn(exp_acc(x[i] - m[i]), s[i]);
      IO::store(out + o, x);
    }
  }
};

template <typename T, int V, bool VEC> struct SoftmaxBw {
  using A = typename Traits<T>::acc_t;
  using IO = Chunk<T, V, VEC>;
  static constexpr int kV = V;
  const int64_t* perm;
  const T* alpha;
  const T* grad_out;
  T* grad_in;
  int64_t D;

  template <int P> __device__ __forceinline__ void regs(int64_t b, int n, int64_t c0, int p) const {
    A a[kHeld][V], g[kHeld][V], dot[V];
    int64_t off[kHeld];
#pragma unroll
    for (int i = 0; i < V; i++) dot[i] = (A)0;
#pragma unroll
    for (int r = 0; r < kHeld; r++) {
      off[r] = 0;
      if (p + r * P < n) {
        off[r] = entry_off(perm, b, p + r * P, D, c0);
        IO::load(alpha + off[r], a[r]);
        IO::load(grad_out + off[r], g[r]);
#pragma unroll
        for (int i = 0; i < V; i++) dot[i] = fma(a[r][i], g[r][i], dot[i]);
      }
    }
    group_sum<P>(dot);
#pragma unroll
    for (int r = 0; r < kHeld; r++) {
      if (p + r * P < n) {
#pragma unroll
        for (int i = 0; i < V; i++) a[r][i] = a[r][i] * (g[r][i] - dot[i]);
        IO::store(grad_in + off[r], a[r]);
      }
    }
  }

  __device__ __forceinline__ void cta(int64_t b, int64_t n, int64_t c0, A* red) const {
    A a[V], g[V], dot[V];
#pragma unroll
    for (int i = 0; i < V; i++) dot[i] = (A)0;
#pragma unroll 4
    for (int64_t j = threadIdx.x; j < n; j += kSoftmaxThreads) {
      const int64_t o = entry_off(perm, b, j, D, c0);
      IO::load(alpha + o, a);
      IO::load(grad_out + o, g);
#pragma unroll
      for (int i = 0; i < V; i++) dot[i] = fma(a[i], g[i], dot[i]);
    }
    cta_combine<false>(dot, red);
#pragma unroll 4
    for (int64_t j = threadIdx.x; j < n; j += kSoftmaxThreads) {
      const int64_t o = entry_off(perm, b, j, D, c0);
      IO::load(alpha + o, a);
      IO::load(grad_out + o, g);
#pragma unroll
      for (int i = 0; i < V; i++) a[i] = a[i] * (g[i] - dot[i]);
      IO::store(grad_in + o, a);
    }
  }
};

// One CTA per 256 consecutive segments: warp w classifies segments 32w .. 32w + 31 of the block, runs the short
// items in groups of 8 lanes and the medium ones on the whole warp, then the CTA runs the long ones in order.
template <class Op>
__global__ void __launch_bounds__(kSoftmaxThreads, 2)
segment_softmax_kernel(const int64_t* __restrict__ ptr, int64_t S, Op op) {
  using A = typename Op::A;
  constexpr int V = Op::kV;
  __shared__ A red[(kSoftmaxThreads / 32) * V];
  __shared__ unsigned long_mask[kSoftmaxThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t C = op.D / V;
  const int64_t s0 = (int64_t)blockIdx.x * kSoftmaxThreads + w * 32;
  int64_t b = 0, n = 0;
  if (s0 + lane < S) {
    b = __ldg(ptr + s0 + lane);
    n = __ldg(ptr + s0 + lane + 1) - b;
  }
  const unsigned short_m = __ballot_sync(kFull, n > 0 && n <= kShortMax);
  const unsigned medium_m = __ballot_sync(kFull, n > kShortMax && n <= kMediumMax);
  const unsigned long_m = __ballot_sync(kFull, n > kMediumMax);

  // short: group g takes the (base + g)-th short segment of the warp, chunk by chunk; the loop bounds are uniform
  // over the warp
  const int group = lane / kShortLanes, p = lane % kShortLanes;
  const int n_short = __popc(short_m);
  for (int base = 0; base < n_short; base += 32 / kShortLanes) {
    const bool live = base + group < n_short;
    const int src = live ? (int)__fns(short_m, 0, base + group + 1) : 0;
    const int64_t sb = __shfl_sync(kFull, b, src);
    const int64_t nn = __shfl_sync(kFull, n, src);
    const int sn = live ? (int)nn : 0;
    for (int64_t k = 0; k < C; k++) op.template regs<kShortLanes>(sb, sn, k * V, p);
  }
  // medium: the whole warp per item
  for (unsigned mm = medium_m; mm; mm &= mm - 1) {
    const int src = __ffs(mm) - 1;
    const int64_t sb = __shfl_sync(kFull, b, src);
    const int sn = (int)__shfl_sync(kFull, n, src);
    for (int64_t k = 0; k < C; k++) op.template regs<32>(sb, sn, k * V, lane);
  }
  // long: the whole CTA per item, segments in order
  if (lane == 0) long_mask[w] = long_m;
  __syncthreads();
  for (int ww = 0; ww < kSoftmaxThreads / 32; ww++) {
    for (unsigned lm = long_mask[ww]; lm; lm &= lm - 1) {
      const int64_t seg = (int64_t)blockIdx.x * kSoftmaxThreads + ww * 32 + (__ffs(lm) - 1);
      const int64_t sb = __ldg(ptr + seg), sn = __ldg(ptr + seg + 1) - sb;
      for (int64_t k = 0; k < C; k++) op.cta(sb, sn, k * V, red);
    }
  }
}

// V: the widest power of two up to 16 bytes that divides D; the vector form when every operand is V-aligned.
template <typename T, template <typename, int, bool> class Op, typename... P>
static int launch_softmax(const int64_t* ptr, int64_t S, int64_t D, std::initializer_list<const void*> operands,
                          cudaStream_t st, P... args) {
  int V = 16 / (int)sizeof(T);
  while (D % V) V >>= 1;
  bool vec = V > 1;
  for (const void* q : operands) vec = vec && ((uintptr_t)q % ((uintptr_t)V * sizeof(T))) == 0;
  const int64_t blocks = (S + kSoftmaxThreads - 1) / kSoftmaxThreads;
  if (blocks >= ((int64_t)1 << 31)) return TSB200_ERR_UNSUPPORTED;
  auto go = [&](auto op) -> int {
    segment_softmax_kernel<<<(unsigned)blocks, kSoftmaxThreads, 0, st>>>(ptr, S, op);
    TSB_LAUNCH_CHECK();
    return 0;
  };
  auto pick = [&](auto vtag) -> int {
    constexpr int W = decltype(vtag)::value;
    if constexpr (W * sizeof(T) > 16) {
      return TSB200_ERR_UNSUPPORTED;
    } else if constexpr (W == 1) {
      return go(Op<T, 1, false>{args..., D});
    } else {
      return vec ? go(Op<T, W, true>{args..., D}) : go(Op<T, W, false>{args..., D});
    }
  };
  switch (V) {
    case 8: return pick(std::integral_constant<int, 8>{});
    case 4: return pick(std::integral_constant<int, 4>{});
    case 2: return pick(std::integral_constant<int, 2>{});
    default: return pick(std::integral_constant<int, 1>{});
  }
}

}  // namespace tsb

using namespace tsb;

extern "C" int tsb200_segment_softmax(const int64_t* ptr, const int64_t* perm, const void* value, void* out, int64_t S,
                                      int64_t E, int64_t D, int dtype, void* stream) {
  if (S < 0 || E < 0 || D < 0) return TSB200_ERR_INVALID_ARG;
  if (S == 0 || E == 0 || D == 0) return 0;
  if (!ptr || !value || !out) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    return launch_softmax<T, SoftmaxFw>(ptr, S, D, {value, out}, st, perm, (const T*)value, (T*)out);
  });
}

extern "C" int tsb200_segment_softmax_bw(const int64_t* ptr, const int64_t* perm, const void* out,
                                         const void* grad_out, void* grad_in, int64_t S, int64_t E, int64_t D,
                                         int dtype, void* stream) {
  if (S < 0 || E < 0 || D < 0) return TSB200_ERR_INVALID_ARG;
  if (S == 0 || E == 0 || D == 0) return 0;
  if (!ptr || !out || !grad_out || !grad_in) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    return launch_softmax<T, SoftmaxBw>(ptr, S, D, {out, grad_out, grad_in}, st, perm, (const T*)out,
                                        (const T*)grad_out, (T*)grad_in);
  });
}
