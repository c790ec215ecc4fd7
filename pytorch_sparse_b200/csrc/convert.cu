// convert.cu — CSR/COO/CSC format kernels for sm_90a.
//
//  * tsb200_ind2ptr / tsb200_ptr2ind replace torch.ops.torch_sparse.{ind2ptr,ptr2ind}
//    (csrc/convert.cpp:22-48, csrc/cpu/convert_cpu.cpp:7-57, csrc/cuda/convert_cuda.cu:9-67).
//    ind2ptr: one thread per pointer entry, lower_bound over the sorted indices (balanced for any
//    gap pattern; the reference's thread-per-nnz loop serialises on runs of empty rows).
//    ptr2ind: a warp owns 32 rows (pointers in registers) and writes their nnz range with
//    coalesced stores, resolving each nnz's row with a 5-step in-register binary search (the
//    reference is thread-per-row: uncoalesced and imbalanced, convert_cuda.cu:43-54).
//  * tsb200_csr2csc replaces SparseStorage.csr2csc()/colptr() (torch_sparse/storage.py:369-416):
//    because the COO is row-major sorted, argsort(col*M + row) == STABLE argsort(col), so the radix
//    sort runs on 32-bit column keys over ceil(log2 N) bits only (3 passes at N = 1M instead of 5+
//    on the 40-bit linearised key), with a 32-bit payload.
#include <cub/cub.cuh>

#include "common.cuh"

namespace tsb {

__global__ void ind2ptr_kernel(const int64_t* __restrict__ ind, int64_t E, int64_t M, int64_t* __restrict__ ptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m <= M; m += stride) {
    // ptr[m] = #{e : ind[e] < m}
    int64_t lo = 0, hi = E;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(ind + mid) < m) lo = mid + 1;
      else hi = mid;
    }
    ptr[m] = lo;
  }
}

__global__ void __launch_bounds__(256) ptr2ind_kernel(const int64_t* __restrict__ ptr, int64_t M, int64_t E,
                                                      int64_t* __restrict__ ind) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t nblk = (M + 31) >> 5;
  for (int64_t blk = wid; blk < nblk; blk += nw) {
    const int64_t r0 = blk << 5;
    const int nrows = (int)min((int64_t)32, M - r0);
    const int64_t p0 = __ldg(ptr + r0 + min(lane, nrows));  // start of row r0+lane (end for lanes >= nrows)
    const int64_t a0 = __shfl_sync(0xffffffffu, p0, 0);
    int64_t a1 = __ldg(ptr + r0 + nrows);
    if (a1 > E) a1 = E;
    for (int64_t pos = a0 + lane; pos - lane < a1; pos += 32) {
      // largest l in [0,nrows) with start[l] <= pos
      int l = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int cand = l + step;
        const int64_t sc = __shfl_sync(0xffffffffu, p0, cand & 31);
        if (cand < nrows && sc <= pos) l = cand;
      }
      if (pos < a1) ind[pos] = r0 + l;
    }
  }
}

__global__ void col_keys_kernel(const int64_t* __restrict__ col, int64_t E, uint32_t* __restrict__ keys,
                                uint32_t* __restrict__ vals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride) {
    keys[i] = (uint32_t)col[i];
    vals[i] = (uint32_t)i;
  }
}

__global__ void csc_finish_kernel(const uint32_t* __restrict__ perm, const int64_t* __restrict__ row, int64_t E,
                                  int64_t* __restrict__ csr2csc, int64_t* __restrict__ row_csc) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride) {
    const uint32_t p = perm[i];
    csr2csc[i] = (int64_t)p;
    if (row_csc) row_csc[i] = __ldg(row + p);
  }
}

__global__ void colptr_kernel(const uint32_t* __restrict__ sorted_col, int64_t E, int64_t N,
                              int64_t* __restrict__ colptr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n <= N; n += stride) {
    int64_t lo = 0, hi = E;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)__ldg(sorted_col + mid) < n) lo = mid + 1;
      else hi = mid;
    }
    colptr[n] = lo;
  }
}

// warp per segment, lanes stride the segment's entries, shuffle tree combine (sum in acc_t, in lane order).
template <typename T>
__global__ void __launch_bounds__(256)
segment_reduce_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ perm, const T* __restrict__ value,
                      T* __restrict__ out, int64_t* __restrict__ arg_out, int64_t S, int64_t D, int reduce) {
  using acc_t = typename Traits<T>::acc_t;
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t seg = wid; seg < S; seg += nw) {
    const int64_t b = __ldg(ptr + seg), e = __ldg(ptr + seg + 1);
    for (int64_t d = 0; d < D; d++) {
      acc_t a = (acc_t)0;
      bool have = false;
      // (jpos, asrc): position inside the segment and input position of this lane's current extreme; a tie between
      // lanes goes to the smaller position, so the arg is the FIRST entry of the segment that attains the extreme
      // (torch_scatter's strict-compare rule, same as csrc/cpu/reducer.h:57-70 for SpMM)
      int64_t jpos = -1, asrc = -1;
      int64_t j = b + lane;
      // the lane's first entry starts its running value. Min/max compare strictly from the SEGMENT's first entry, so
      // a NaN there wins and a NaN anywhere else never does: a lane skips a later NaN as its first entry (kept, no
      // compare would ever replace it, and it would win the combine).
      for (; j < e; j += 32) {
        const int64_t src = perm ? __ldg(perm + j) : j;
        const acc_t v = Traits<T>::to_acc(value[src * D + d]);
        if (v != v && j != b && (reduce == TSB200_MIN || reduce == TSB200_MAX)) continue;
        a = v; have = true; jpos = j; asrc = src;
        j += 32;
        break;
      }
      for (; j < e; j += 32) {
        const int64_t src = perm ? __ldg(perm + j) : j;
        const acc_t v = Traits<T>::to_acc(value[src * D + d]);
        if (reduce == TSB200_SUM || reduce == TSB200_MEAN) a = a + v;
        else if (reduce == TSB200_MIN) { if (v < a) { a = v; jpos = j; asrc = src; } }
        else { if (v > a) { a = v; jpos = j; asrc = src; } }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const acc_t o = __shfl_down_sync(0xffffffffu, a, off);
        const bool oh = __shfl_down_sync(0xffffffffu, (int)have, off) != 0;
        const int64_t oj = __shfl_down_sync(0xffffffffu, jpos, off);
        const int64_t os = __shfl_down_sync(0xffffffffu, asrc, off);
        if (oh) {
          if (!have) { a = o; have = true; jpos = oj; asrc = os; }
          else if (reduce == TSB200_SUM || reduce == TSB200_MEAN) a = a + o;
          else if (reduce == TSB200_MIN) { if (o < a || (o == a && oj < jpos)) { a = o; jpos = oj; asrc = os; } }
          else { if (o > a || (o == a && oj < jpos)) { a = o; jpos = oj; asrc = os; } }
        }
      }
      if (lane == 0) {
        // the sum starts at +0 (torch_scatter's does): x + 0 == x except that a run of -0 comes out +0
        if (reduce == TSB200_SUM || reduce == TSB200_MEAN) a = a + (acc_t)0;
        if (reduce == TSB200_MEAN && e > b) a = a / (acc_t)(e - b);
        out[seg * D + d] = Traits<T>::from_acc(have ? a : (acc_t)0);
        if (arg_out) arg_out[seg * D + d] = have ? asrc : (int64_t)-1;
      }
    }
  }
}

// Backward of the segment / run reductions (segment_reduce, coalesce): a pure gather, no atomics.
//   sum : grad_in[i,d] = grad_out[seg[i],d]            mean: ... / max(count[seg[i]],1)
//   min/max: grad_in[i,d] = (arg[seg[i],d] == i) ? grad_out[seg[i],d] : 0
// (torch_scatter's segment_csr / scatter backward as reached from torch_sparse/storage.py:451 and reduce.py:36-54.)
template <typename T>
__global__ void __launch_bounds__(256)
segment_reduce_bw_kernel(const int64_t* __restrict__ seg, const int64_t* __restrict__ count,
                         const int64_t* __restrict__ arg, const T* __restrict__ grad_out, T* __restrict__ grad_in,
                         int64_t E, int64_t D, int reduce) {
  using acc_t = typename Traits<T>::acc_t;
  const int64_t total = E * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int64_t i = t / D, d = t - i * D;
    const int64_t s = __ldg(seg + i);
    acc_t g = Traits<T>::to_acc(grad_out[s * D + d]);
    if (reduce == TSB200_MEAN) {
      const int64_t c = __ldg(count + s);
      g = g / (acc_t)(c > 0 ? c : 1);
    } else if (reduce == TSB200_MIN || reduce == TSB200_MAX) {
      if (__ldg(arg + s * D + d) != i) g = (acc_t)0;
    }
    grad_in[t] = Traits<T>::from_acc(g);
  }
}

static inline int grid1d(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)num_sms() * 32;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

static inline int bits_for(int64_t n) {  // number of bits needed to represent values in [0, n)
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < n) b++;
  return b;
}

struct CscLayout {
  size_t k0, k1, v0, v1, cub, total;
  size_t cub_bytes;
};
static CscLayout csc_layout(int64_t E) {
  CscLayout L;
  size_t off = 0;
  const size_t n = align_up((size_t)(E > 0 ? E : 1) * 4, 256);
  L.k0 = off; off += n;
  L.k1 = off; off += n;
  L.v0 = off; off += n;
  L.v1 = off; off += n;
  size_t tb = 0;
  cub::DoubleBuffer<uint32_t> dk(nullptr, nullptr), dv(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)(E > 0 ? E : 1), 0, 32, (cudaStream_t)0);
  L.cub_bytes = tb;
  L.cub = off; off += align_up(tb, 256);
  L.total = off;
  return L;
}

}  // namespace tsb

using namespace tsb;

extern "C" int tsb200_ind2ptr(const int64_t* ind, int64_t E, int64_t M, int64_t* ptr, void* stream) {
  if (E < 0 || M < 0 || !ptr || (E > 0 && !ind)) return TSB200_ERR_INVALID_ARG;
  ind2ptr_kernel<<<grid1d(M + 1, 256), 256, 0, (cudaStream_t)stream>>>(ind, E, M, ptr);
  TSB_LAUNCH_CHECK();
  return 0;
}

extern "C" int tsb200_ptr2ind(const int64_t* ptr, int64_t M, int64_t E, int64_t* ind, void* stream) {
  if (E < 0 || M < 0 || !ptr) return TSB200_ERR_INVALID_ARG;
  if (E == 0 || M == 0) return 0;
  if (!ind) return TSB200_ERR_INVALID_ARG;
  const int64_t nblk = (M + 31) >> 5;
  ptr2ind_kernel<<<grid1d(nblk * 32, 256), 256, 0, (cudaStream_t)stream>>>(ptr, M, E, ind);
  TSB_LAUNCH_CHECK();
  return 0;
}

extern "C" size_t tsb200_csr2csc_workspace_bytes(int64_t E, int64_t M, int64_t N) {
  (void)M; (void)N;
  if (E < 0) return 0;
  return csc_layout(E).total;
}

extern "C" int tsb200_csr2csc(const int64_t* row, const int64_t* col, int64_t E, int64_t M, int64_t N,
                              int64_t* csr2csc, int64_t* colptr, int64_t* row_csc, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (E < 0 || M < 0 || N < 0) return TSB200_ERR_INVALID_ARG;
  if (E >= ((int64_t)1 << 31) || N >= ((int64_t)1 << 32)) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  if (E == 0) {
    if (colptr) TSB_CUDA_TRY(cudaMemsetAsync(colptr, 0, (size_t)(N + 1) * 8, st));
    return 0;
  }
  if (!col || !csr2csc || (row_csc && !row)) return TSB200_ERR_INVALID_ARG;
  const CscLayout L = csc_layout(E);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  char* ws = (char*)workspace;
  uint32_t* k0 = (uint32_t*)(ws + L.k0); uint32_t* k1 = (uint32_t*)(ws + L.k1);
  uint32_t* v0 = (uint32_t*)(ws + L.v0); uint32_t* v1 = (uint32_t*)(ws + L.v1);
  col_keys_kernel<<<grid1d(E, 256), 256, 0, st>>>(col, E, k0, v0);
  TSB_LAUNCH_CHECK();
  cub::DoubleBuffer<uint32_t> dk(k0, k1), dv(v0, v1);
  size_t tb = L.cub_bytes;
  TSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, tb, dk, dv, (int)E, 0, bits_for(N), st));
  csc_finish_kernel<<<grid1d(E, 256), 256, 0, st>>>(dv.Current(), row, E, csr2csc, row_csc);
  TSB_LAUNCH_CHECK();
  if (colptr) {
    colptr_kernel<<<grid1d(N + 1, 256), 256, 0, st>>>(dk.Current(), E, N, colptr);
    TSB_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int tsb200_segment_reduce(const int64_t* ptr, const int64_t* perm, const void* value, void* out,
                                     int64_t* arg_out, int64_t S, int64_t D, int dtype, int reduce, void* stream) {
  if (S < 0 || D < 0 || reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  if (S == 0 || D == 0) return 0;
  if (!ptr || !out) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    segment_reduce_kernel<T><<<grid1d(S * 32, 256), 256, 0, st>>>(
        ptr, perm, (const T*)value, (T*)out, (reduce == TSB200_MIN || reduce == TSB200_MAX) ? arg_out : nullptr, S, D,
        reduce);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

extern "C" int tsb200_segment_reduce_bw(const int64_t* seg, const int64_t* count, const int64_t* arg,
                                        const void* grad_out, void* grad_in, int64_t E, int64_t S, int64_t D,
                                        int dtype, int reduce, void* stream) {
  if (E < 0 || S < 0 || D < 0 || reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  if (E == 0 || D == 0) return 0;
  if (!seg || !grad_out || !grad_in) return TSB200_ERR_INVALID_ARG;
  if (reduce == TSB200_MEAN && !count) return TSB200_ERR_INVALID_ARG;
  if ((reduce == TSB200_MIN || reduce == TSB200_MAX) && !arg) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_float_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    segment_reduce_bw_kernel<T><<<grid1d(E * D, 256), 256, 0, st>>>(seg, count, arg, (const T*)grad_out, (T*)grad_in,
                                                                   E, D, reduce);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}
