// coalesce.cu — COO coalesce for sm_90a.
//
// Replaces torch_sparse.coalesce -> SparseStorage.__init__ (sort) + SparseStorage.coalesce()
// (torch_sparse/coalesce.py:5-25, torch_sparse/storage.py:149-162, 436-466; value reduction =
// torch_scatter.segment_csr, call site storage.py:451).
//
// The reference issues ~12-15 ATen kernels, 3-4 host syncs and builds the linearised key twice.
// Here:  phase 1  key = row*N+col (+ "already sorted?" flag) -> [stable CUB radix sort over only
//                 the significant key bits, 32-bit payload] -> DeviceSelect over on-the-fly head flags gives the
//                 run starts and E' on the device (copied to pinned host memory);
//        phase 2  one kernel emits row'/col' from the run heads and reduces the values of each run
//                 in sorted (== input, the sort is stable) order.
// A stable sort makes the float 'add' order canonical (input order); the reference's order over
// duplicates is unspecified (non-stable Tensor.sort, torch_sparse/utils.py:19-20).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "common.cuh"

namespace tsb {

// ib > 0: "packed" mode — the input position i is stored in the low ib bits of the key word, so the radix
// sort moves 8-byte keys only (no payload); it sorts bits [ib, ib+key_bits) and, being stable, leaves equal
// keys in input order. ib == 0: separate 32-bit payload array (keys wider than 64 - bits(E)).
__global__ void coalesce_keys_kernel(const int64_t* __restrict__ row, const int64_t* __restrict__ col,
                                     int64_t E, int64_t N, uint64_t* __restrict__ keys,
                                     uint32_t* __restrict__ perm, int* __restrict__ unsorted, int ib) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride) {
    const uint64_t k = (uint64_t)(row[i] * N + col[i]);
    if (ib) keys[i] = (k << ib) | (uint64_t)i;
    else { keys[i] = k; perm[i] = (uint32_t)i; }
    if (i > 0) {
      const uint64_t kp = (uint64_t)(__ldg(row + i - 1) * N + __ldg(col + i - 1));
      bad |= k < kp;
    }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(unsorted, 1);
}

// head-of-run flag of sorted entry i, computed on the fly for DeviceSelect::Flagged (no flag array, no extra pass)
struct HeadFlag {
  const uint64_t* keys;
  int ib;
  __host__ __device__ __forceinline__ uint8_t operator()(uint32_t i) const {
    return (i == 0 || (keys[i] >> ib) != (keys[i - 1] >> ib)) ? 1 : 0;
  }
};

__global__ void copy_count_kernel(const int* __restrict__ n_sel, int64_t* __restrict__ out) { *out = (int64_t)*n_sel; }

// `sel` = {which key buffer, which payload buffer, ib}, written by the sort phase into the workspace: the
// consumers pick the sorted buffers on the device, so phase 2 needs no read-back and no host synchronisation
__global__ void widen_perm_kernel(const uint64_t* __restrict__ k0, const uint64_t* __restrict__ k1,
                                  const uint32_t* __restrict__ p0, const uint32_t* __restrict__ p1,
                                  const int* __restrict__ sel, int64_t E, int64_t* __restrict__ out) {
  const uint64_t* keys = sel[0] ? k1 : k0;
  const uint32_t* perm = sel[1] ? p1 : p0;
  const int ib = sel[2];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const uint64_t mask = ib ? (((uint64_t)1 << ib) - 1) : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += stride)
    out[i] = ib ? (int64_t)(keys[i] & mask) : (int64_t)perm[i];
}

enum { C_SUM = TSB200_SUM, C_MEAN = TSB200_MEAN, C_MIN = TSB200_MIN, C_MAX = TSB200_MAX };

template <typename T>
__global__ void __launch_bounds__(256)
coalesce_emit_kernel(const uint64_t* __restrict__ k0, const uint64_t* __restrict__ k1,
                     const uint32_t* __restrict__ p0, const uint32_t* __restrict__ p1, const int* __restrict__ sel,
                     const uint32_t* __restrict__ starts, int64_t E, int64_t N, int64_t n_unique,
                     const T* __restrict__ value_in, int64_t D, int reduce, int64_t* __restrict__ row_out,
                     int64_t* __restrict__ col_out, T* __restrict__ value_out, int64_t* __restrict__ perm_out,
                     int64_t* __restrict__ seg_out, int64_t* __restrict__ count_out, int64_t* __restrict__ arg_out) {
  using acc_t = typename Traits<T>::acc_t;
  const uint64_t* keys = sel[0] ? k1 : k0;
  const uint32_t* perm = sel[1] ? p1 : p0;
  const int ib = sel[2];
  const uint64_t pmask = ib ? (((uint64_t)1 << ib) - 1) : 0;
  auto perm_at = [&](int64_t j) -> int64_t { return ib ? (int64_t)(keys[j] & pmask) : (int64_t)perm[j]; };
  const int64_t total = n_unique * (value_in ? D : 1);
  const int64_t Dd = value_in ? D : 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int64_t seg = t / Dd, d = t - seg * Dd;
    const int64_t s = starts[seg];
    const int64_t e = (seg + 1 < n_unique) ? (int64_t)starts[seg + 1] : E;
    if (d == 0) {
      const uint64_t k = keys[s] >> ib;
      const uint64_t r = k / (uint64_t)N;
      if (row_out) row_out[seg] = (int64_t)r;
      if (col_out) col_out[seg] = (int64_t)(k - r * (uint64_t)N);
      if (perm_out) perm_out[seg] = perm_at(s);
      if (count_out) count_out[seg] = e - s;
      // run id of every INPUT entry: what the backward of the value reduction gathers through
      if (seg_out)
        for (int64_t j = s; j < e; j++) seg_out[perm_at(j)] = seg;
    }
    if (value_in) {
      int64_t first = perm_at(s);
      acc_t a = Traits<T>::to_acc(value_in[first * D + d]);
      for (int64_t j = s + 1; j < e; j++) {
        const int64_t pj = perm_at(j);
        const acc_t v = Traits<T>::to_acc(value_in[pj * D + d]);
        if (reduce == C_SUM || reduce == C_MEAN) a = a + v;
        else if (reduce == C_MIN) { if (v < a) { a = v; first = pj; } }   // strict: ties keep the earliest input entry
        else { if (v > a) { a = v; first = pj; } }
      }
      // the sum starts at +0 (torch_scatter's does): x + 0 == x except that a run of -0 comes out +0
      if (reduce == C_SUM || reduce == C_MEAN) a = a + (acc_t)0;
      if (reduce == C_MEAN) a = a / (acc_t)(e - s);
      value_out[seg * D + d] = Traits<T>::from_acc(a);
      if (arg_out) arg_out[seg * D + d] = first;
    }
  }
}

struct CoLayout {
  size_t k0, k1, p0, p1, starts, scalars, cub, total;
  size_t cub_bytes;
  // scalars: [0] int unsorted, [1] int n_selected, [2..3] int64 n_unique, [4] int keys_cur, [5] int perm_cur, [6] int ib
};
static CoLayout co_layout(int64_t E) {
  CoLayout L;
  const size_t n = (size_t)(E > 0 ? E : 1);
  size_t off = 0;
  L.scalars = off; off += 256;
  L.k0 = off; off += align_up(n * 8, 256);
  L.k1 = off; off += align_up(n * 8, 256);
  L.p0 = off; off += align_up(n * 4, 256);
  L.p1 = off; off += align_up(n * 4, 256);
  L.starts = off; off += align_up(n * 4, 256);
  size_t t1 = 0, t2 = 0;
  cub::DoubleBuffer<uint64_t> dk(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> dv(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, t1, dk, dv, (int)n, 0, 64, (cudaStream_t)0);
  {
    size_t t3 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t3, dk, (int)n, 0, 64, (cudaStream_t)0);
    if (t3 > t1) t1 = t3;
  }
  cub::DeviceSelect::Flagged(nullptr, t2, thrust::counting_iterator<uint32_t>(0),
                             thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), HeadFlag{nullptr, 0}),
                             (uint32_t*)nullptr, (int*)nullptr, (int)n, (cudaStream_t)0);
  L.cub_bytes = t1 > t2 ? t1 : t2;
  L.cub = off; off += align_up(L.cub_bytes, 256);
  L.total = off;
  return L;
}

static inline int cgrid(int64_t n) {
  int64_t b = (n + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 32;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace tsb

using namespace tsb;

extern "C" size_t tsb200_coalesce_workspace_bytes(int64_t E, int64_t M, int64_t N) {
  (void)M; (void)N;
  if (E < 0) return 0;
  return co_layout(E).total;
}

// NOTE: synchronises `stream` once internally (to skip the sort when the input is already
// sorted, like the reference's `(idx[1:] < idx[:-1]).any()` check, storage.py:154).
extern "C" int tsb200_coalesce_sort(const int64_t* row, const int64_t* col, int64_t E, int64_t M, int64_t N,
                                    void* workspace, size_t workspace_bytes, int64_t* n_unique_host,
                                    void* stream) {
  if (E < 0 || M < 0 || N < 0) return TSB200_ERR_INVALID_ARG;
  if (E >= ((int64_t)1 << 31)) return TSB200_ERR_UNSUPPORTED;
  // the key row*N + col is one 64-bit word: wider shapes would wrap it and merge distinct entries
  const unsigned __int128 maxkey = (unsigned __int128)(M > 0 ? M : 1) * (unsigned __int128)(N > 0 ? N : 1);
  if (maxkey > ((unsigned __int128)1 << 64)) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const CoLayout L = co_layout(E);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  char* ws = (char*)workspace;
  int* sc = (int*)(ws + L.scalars);
  int64_t* n_unique_dev = (int64_t*)(ws + L.scalars + 8);
  TSB_CUDA_TRY(cudaMemsetAsync(sc, 0, 256, st));
  if (E == 0) {
    if (n_unique_host) *n_unique_host = 0;
    return 0;
  }
  if (!row || !col) return TSB200_ERR_INVALID_ARG;
  uint64_t* k0 = (uint64_t*)(ws + L.k0); uint64_t* k1 = (uint64_t*)(ws + L.k1);
  uint32_t* p0 = (uint32_t*)(ws + L.p0); uint32_t* p1 = (uint32_t*)(ws + L.p1);
  // key width and packing decision
  int bits = 1;
  while (bits < 64 && ((unsigned __int128)1 << bits) < maxkey) bits++;
  int ebits = 1;
  while (((int64_t)1 << ebits) < E) ebits++;
  const int ib = (bits + ebits <= 64) ? ebits : 0;
  coalesce_keys_kernel<<<cgrid(E), 256, 0, st>>>(row, col, E, N, k0, p0, sc, ib);
  TSB_LAUNCH_CHECK();
  int unsorted = 0;
  TSB_CUDA_TRY(cudaMemcpyAsync(&unsorted, sc, sizeof(int), cudaMemcpyDeviceToHost, st));
  TSB_CUDA_TRY(cudaStreamSynchronize(st));
  int cur = 0;
  if (unsorted) {
    size_t tb = L.cub_bytes;
    if (ib) {
      cub::DoubleBuffer<uint64_t> dk(k0, k1);
      TSB_CUDA_TRY(cub::DeviceRadixSort::SortKeys(ws + L.cub, tb, dk, (int)E, ib, ib + bits, st));
      cur = (dk.Current() == k1) ? 1 : 0;
    } else {
      cub::DoubleBuffer<uint64_t> dk(k0, k1);
      cub::DoubleBuffer<uint32_t> dv(p0, p1);
      TSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, tb, dk, dv, (int)E, 0, bits, st));
      cur = (dk.Current() == k1) ? 1 : 0;  // CUB keeps keys and values in the same selector
    }
  }
  int h[3] = {cur, cur, ib};
  TSB_CUDA_TRY(cudaMemcpyAsync(sc + 4, h, sizeof(h), cudaMemcpyHostToDevice, st));
  const uint64_t* keys = cur ? k1 : k0;
  size_t tb = L.cub_bytes;
  TSB_CUDA_TRY(cub::DeviceSelect::Flagged(
      ws + L.cub, tb, thrust::counting_iterator<uint32_t>(0),
      thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), HeadFlag{keys, ib}),
      (uint32_t*)(ws + L.starts), sc + 1, (int)E, st));
  copy_count_kernel<<<1, 1, 0, st>>>(sc + 1, n_unique_dev);
  TSB_LAUNCH_CHECK();
  if (n_unique_host)
    TSB_CUDA_TRY(cudaMemcpyAsync(n_unique_host, n_unique_dev, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  return 0;
}

extern "C" int tsb200_coalesce_emit(int64_t E, int64_t N, int64_t n_unique, const void* value_in, int64_t D,
                                    int dtype, int reduce, int64_t* row_out, int64_t* col_out, void* value_out,
                                    int64_t* perm_out, int64_t* seg_out, int64_t* count_out, int64_t* arg_out,
                                    const void* workspace, void* stream) {
  if (E < 0 || N < 0 || n_unique < 0 || n_unique > E) return TSB200_ERR_INVALID_ARG;
  if (n_unique == 0) return 0;
  if (!workspace) return TSB200_ERR_WORKSPACE;
  if (value_in && (!value_out || D < 0)) return TSB200_ERR_INVALID_ARG;
  if (value_in && (reduce < TSB200_SUM || reduce > TSB200_MAX)) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const CoLayout L = co_layout(E);
  const char* ws = (const char*)workspace;
  // which half of the double buffers holds the sorted data was recorded by phase 1 in the workspace; the kernel
  // reads it there (no read-back, no synchronisation in phase 2)
  const uint64_t* k0 = (const uint64_t*)(ws + L.k0); const uint64_t* k1 = (const uint64_t*)(ws + L.k1);
  const uint32_t* p0 = (const uint32_t*)(ws + L.p0); const uint32_t* p1 = (const uint32_t*)(ws + L.p1);
  const int* sel = (const int*)(ws + L.scalars + 16);
  const uint32_t* starts = (const uint32_t*)(ws + L.starts);
  if (value_in && D == 0) value_in = nullptr;
  const int64_t total = n_unique * (value_in ? D : 1);
  if (!value_in) {
    coalesce_emit_kernel<float><<<cgrid(total), 256, 0, st>>>(k0, k1, p0, p1, sel, starts, E, N, n_unique, nullptr, 1,
                                                             reduce, row_out, col_out, nullptr, perm_out, seg_out,
                                                             count_out, nullptr);
    TSB_LAUNCH_CHECK();
    return 0;
  }
  return dispatch_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    coalesce_emit_kernel<T><<<cgrid(total), 256, 0, st>>>(k0, k1, p0, p1, sel, starts, E, N, n_unique,
                                                         (const T*)value_in, D, reduce, row_out, col_out,
                                                         (T*)value_out, perm_out, seg_out, count_out,
                                                         (reduce == C_MIN || reduce == C_MAX) ? arg_out : nullptr);
    TSB_LAUNCH_CHECK();
    return 0;
  });
}

extern "C" int tsb200_coalesce_perm(int64_t E, int64_t* perm_out, const void* workspace, void* stream) {
  if (E < 0) return TSB200_ERR_INVALID_ARG;
  if (E == 0) return 0;
  if (!workspace) return TSB200_ERR_WORKSPACE;
  if (!perm_out) return TSB200_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const CoLayout L = co_layout(E);
  const char* ws = (const char*)workspace;
  widen_perm_kernel<<<cgrid(E), 256, 0, st>>>((const uint64_t*)(ws + L.k0), (const uint64_t*)(ws + L.k1),
                                               (const uint32_t*)(ws + L.p0), (const uint32_t*)(ws + L.p1),
                                               (const int*)(ws + L.scalars + 16), E, perm_out);
  TSB_LAUNCH_CHECK();
  return 0;
}
