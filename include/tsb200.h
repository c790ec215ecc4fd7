/*
 * tsb200.h — C-ABI of libtsb200.so: the H100-native (sm_90a) implementation of the
 * torch_sparse sparse-matmul hot path (CSR SpMM fwd/bwd, COO coalesce, SpSpMM, CSR<->COO/CSC
 * format kernels).
 *
 * Conventions (all entry points):
 *   - extern "C", plain pointers + extents + enums + an opaque `stream` (a cudaStream_t cast to
 *     void*; NULL = legacy default stream). No torch / ATen types cross this boundary.
 *   - Every pointer is a DEVICE pointer unless the name ends in `_host`.
 *   - Indices are int64 (the reference asserts int64 everywhere: torch_sparse/storage.py:52,85,92).
 *   - The library never allocates output memory: the caller owns outputs and workspaces
 *     (`*_workspace_bytes` tells how much scratch a call needs). The only internal allocations
 *     are none; CUB temp storage lives inside the caller's workspace.
 *   - Every call is asynchronous on `stream` unless documented otherwise and returns an int:
 *       0                 success
 *       > 0               a cudaError_t raised by a launch / runtime call
 *       < 0               TSB200_ERR_* (argument / support errors; nothing was launched)
 *     `tsb200_strerror` maps any return value to text. Nothing throws.
 *   - Thread safety: stateless; re-entrant as long as callers use distinct workspaces.
 *
 * Each entry point names the reference interface (file:line under rusty1s/pytorch_sparse
 * @ 91feaa5, torch_sparse 0.6.18) that it replaces.
 */
#ifndef TSB200_H_
#define TSB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSB200_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define TSB200_API __attribute__((visibility("default")))
#else
#define TSB200_API
#endif

/* dense / value element types (the reference dispatches AT_DISPATCH_ALL_TYPES_AND2(Half,BFloat16),
 * csrc/cpu/spmm_cpu.cpp:47). */
typedef enum {
  TSB200_F32 = 0,
  TSB200_F64 = 1,
  TSB200_F16 = 2,
  TSB200_BF16 = 3,
  TSB200_I32 = 4,
  TSB200_I64 = 5,
  TSB200_I16 = 6,
  TSB200_I8 = 7,
  TSB200_U8 = 8
} tsb200_dtype;

/* reductions reachable from Python (csrc/cpu/reducer.h:6-11; mul/div are unreachable). */
typedef enum { TSB200_SUM = 0, TSB200_MEAN = 1, TSB200_MIN = 2, TSB200_MAX = 3 } tsb200_reduce;

#define TSB200_ERR_INVALID_ARG (-1)   /* NULL where required, negative extent, bad enum */
#define TSB200_ERR_UNSUPPORTED (-2)   /* dtype/reduce/extent combination not implemented */
#define TSB200_ERR_WORKSPACE (-3)     /* workspace too small */
#define TSB200_ERR_NO_DEVICE (-4)     /* no CUDA device / wrong architecture */

TSB200_API int tsb200_version(void);
TSB200_API const char* tsb200_strerror(int code);
/* 0 iff a CUDA device with compute capability 9.x is current. */
TSB200_API int tsb200_device_ok(void);
/* CUDA toolkit version the library was built with, CUDA_VERSION encoding (12090 = 12.9). Replaces
 * torch.ops.torch_sparse.cuda_version() (csrc/version.cpp:27-41), read by the import-time check at
 * torch_sparse/__init__.py:23-37. */
TSB200_API int tsb200_cuda_version(void);
/* Multiprocessor count of the current device (grids are sized from it at run time). */
TSB200_API int tsb200_sm_count(void);

/* ------------------------------------------------------------------------------------------
 * CSR SpMM forward.   Replaces spmm_fw -> spmm_cpu / spmm_cuda
 *   (csrc/spmm.cpp:22-35, csrc/cpu/spmm_cpu.cpp:8-101, csrc/cuda/spmm_cuda.cu:92-155).
 *   out[b,m,:] = reduce_{e in [rowptr[m], rowptr[m+1])} value[e] * mat[b, col[e], :]
 *   rowptr i64[M+1], col i64[E], value dtype[E] or NULL (has_value=false), mat dtype[B,N,K]
 *   contiguous, out dtype[B,M,K]; arg_out i64[B,M,K] required for MIN/MAX (NULL otherwise) and is
 *   fully written by the call (empty rows get the sentinel E, csrc/cpu/spmm_cpu.cpp:35), so the
 *   caller need not pre-fill it.
 *   Semantics kept from csrc/cpu/reducer.h:43-84: mean divides by max(count,1); min/max use a
 *   strict compare (ties keep the smallest e), empty rows write 0.
 *   F16/BF16/F32 accumulate in fp32 (the reference accumulates in the storage dtype); the
 *   min/max compare is done on the product rounded to the storage dtype, as the reference does.
 *   workspace: tsb200_spmm_fw_workspace_bytes(...) bytes (may be NULL if that returns 0).
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_spmm_fw_workspace_bytes(int64_t B, int64_t M, int64_t K, int64_t E, int dtype,
                                      int reduce);
TSB200_API int tsb200_spmm_fw(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                   void* out, int64_t* arg_out, int64_t B, int64_t M, int64_t N, int64_t K,
                   int64_t E, int dtype, int reduce, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ------------------------------------------------------------------------------------------
 * Planned SpMM (no counterpart in the reference; the analogue of the structure caches it keeps, csr2csc / colptr).
 *   The only data-dependent control decision of the forward kernel — which rows are too long (or overflow their
 *   32-row group's nnz budget) and are therefore cut into <= 256-nnz segments — depends on rowptr alone.
 *   tsb200_spmm_plan computes it once per matrix: a row mask, the segment list and the multi-segment rows, into
 *   `plan` (tsb200_spmm_plan_bytes(M, E) bytes, 256 B aligned), and returns the three counts
 *   counts_host[0..2] = {segments, multi-segment rows, partial slots} (synchronises `stream` once).
 *   tsb200_spmm_fw_planned then runs ANY product with that matrix (same semantics as tsb200_spmm_fw, B = 1,
 *   F32 / F16 / BF16 with K * sizeof(dtype) % 16 == 0) as one memset + ONE kernel: the warps process the row items
 *   and then drain the plan's segment list themselves; a multi-segment row is combined by the warp that finishes its
 *   last segment. (For K * sizeof(dtype) <= 128 B the segment / combine kernels are still separate launches, issued
 *   only when the plan holds segments.) workspace: tsb200_spmm_fw_planned_workspace_bytes(K, n_long, n_slot, reduce).
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_spmm_plan_bytes(int64_t M, int64_t E);
TSB200_API int tsb200_spmm_plan(const int64_t* rowptr, int64_t M, int64_t E, void* plan, size_t plan_bytes,
                                int64_t* counts_host, void* stream);
TSB200_API size_t tsb200_spmm_fw_planned_workspace_bytes(int64_t K, int64_t n_long, int64_t n_slot, int reduce);
TSB200_API int tsb200_spmm_fw_planned(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                      void* out, int64_t* arg_out, int64_t M, int64_t N, int64_t K, int64_t E,
                                      int dtype, int reduce, const void* plan, size_t plan_bytes, int64_t n_seg,
                                      int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes,
                                      void* stream);

/* One COLUMN BLOCK of a SUM SpMM (multi-GPU pipelining: the dense operand arrives block by block over NVLink and
 * block p of A's columns is multiplied as soon as block p of `mat` has landed; no counterpart in the reference, which
 * has no collectives — the partitioner semantics are torch_sparse/narrow.py:15-42). (rowptr, col, value) hold only the
 * entries of A whose column lies in the block (col still indexes the full `mat`). The launches of one product share
 * an fp32 `partial` [B, M, K]:  acc_mode 1 = first block (partial = A_p mat), 2 = partial += A_p mat,
 * 3 = last block: out = cast(partial + A_p mat). F32 / F16 / BF16 with K * sizeof(dtype) % 16 == 0 only; E > 0.
 * Workspace: tsb200_spmm_fw_workspace_bytes(B, M, K, E, dtype, TSB200_SUM). */
TSB200_API int tsb200_spmm_fw_acc(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                  void* out, float* partial, int acc_mode, int64_t B, int64_t M, int64_t N,
                                  int64_t K, int64_t E, int dtype, void* workspace, size_t workspace_bytes,
                                  void* stream);

/* ------------------------------------------------------------------------------------------
 * SpMM value gradient (SDDMM).  Replaces spmm_value_bw -> spmm_value_bw_cpu / _cuda
 *   (csrc/spmm.cpp:37-49, csrc/cpu/spmm_cpu.cpp:103-152, csrc/cuda/spmm_cuda.cu:196-237).
 *   out[e] = sum_b <mat[b,col[e],:], grad[b,row[e],:]>   (/ max(rowcount,1) for MEAN)
 *   reduce in {SUM, MEAN}. With a workspace of tsb200_spmm_value_bw_workspace_bytes(...) bytes (256 B aligned)
 *   and B == 1 the row-wise kernel is used (grad row in registers, only `mat` rows gathered, long rows split
 *   through a device-side segment queue); workspace == NULL selects the nnz-parallel kernel. Same results.
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_spmm_value_bw_workspace_bytes(int64_t B, int64_t M, int64_t K, int64_t E, int dtype);
TSB200_API int tsb200_spmm_value_bw(const int64_t* row, const int64_t* rowptr, const int64_t* col,
                         const void* mat, const void* grad, void* out, int64_t B, int64_t M,
                         int64_t N, int64_t K, int64_t E, int dtype, int reduce, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused min/max backward.  Replaces the ATen chain in SPMMMin/SPMMMax::backward
 *   (csrc/spmm.cpp:204-242, 264-302): for every (b,m,k) with a = arg_out[b,m,k] != E,
 *     grad_value[a]           += mat[b,col[a],k] * grad_out[b,m,k]      (if grad_value != NULL)
 *     grad_mat[b,col[a],k]    += value[a]       * grad_out[b,m,k]      (if grad_mat   != NULL;
 *                                 value == NULL means has_value=false, factor 1)
 *   grad_value (acc_dtype[E]) and grad_mat (acc_dtype[B,N,K]) must be ZERO-FILLED by the caller and
 *   are accumulated with atomics. acc element type: float for F16/BF16/F32, double for F64
 *   (the host layer casts back to the storage dtype). Floating dtypes only.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_minmax_bw(const int64_t* col, const void* value, const void* mat,
                          const void* grad_out, const int64_t* arg_out, void* grad_value,
                          void* grad_mat, int64_t B, int64_t M, int64_t N, int64_t K, int64_t E,
                          int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * ind2ptr / ptr2ind.  Replace torch.ops.torch_sparse.{ind2ptr,ptr2ind}
 *   (csrc/convert.cpp:22-48, csrc/cpu/convert_cpu.cpp:7-57, csrc/cuda/convert_cuda.cu:9-67).
 *   ind2ptr: ind i64[E] sorted ascending, values in [0,M) -> ptr i64[M+1], ptr[i] = #{e: ind[e] < i}
 *   ptr2ind: ptr i64[M+1] -> ind i64[E]
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_ind2ptr(const int64_t* ind, int64_t E, int64_t M, int64_t* ptr, void* stream);
TSB200_API int tsb200_ptr2ind(const int64_t* ptr, int64_t M, int64_t E, int64_t* ind, void* stream);

/* ------------------------------------------------------------------------------------------
 * CSR -> CSC permutation.  Replaces SparseStorage.csr2csc()/colptr()
 *   (torch_sparse/storage.py:369-385, 407-416):  csr2csc = argsort(col * M + row) (stable),
 *   colptr = ind2ptr(col[csr2csc], N).   row i64[E] (sorted), col i64[E].
 *   Outputs: csr2csc i64[E]; colptr i64[N+1] (may be NULL); row_csc i64[E] = row[csr2csc] (may be NULL).
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_csr2csc_workspace_bytes(int64_t E, int64_t M, int64_t N);
TSB200_API int tsb200_csr2csc(const int64_t* row, const int64_t* col, int64_t E, int64_t M, int64_t N,
                   int64_t* csr2csc, int64_t* colptr, int64_t* row_csc, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Segment reduce over a CSR pointer.  Replaces torch_scatter.segment_csr / scatter as called by the row and
 *   column reductions of torch_sparse/reduce.py:36-54 (`segment_csr(value, rowptr, None, reduce)` for dim=1,
 *   `scatter(value, col, 0, None, N, reduce)` for dim=0, which on the CSC view is a segment reduce over colptr).
 *   out[s, d] = reduce_{j in [ptr[s], ptr[s+1])} value[perm ? perm[j] : j, d];  empty segment -> 0.
 *   ptr i64[S+1]; perm i64[E] or NULL; value dtype[E, D]; out dtype[S, D]; reduce in {SUM, MEAN, MIN, MAX}.
 *   arg_out i64[S, D] (optional, MIN/MAX only): INPUT position (perm applied) of the first entry of the segment that
 *   attains the extreme (strict compare, like csrc/cpu/reducer.h:57-70), -1 for an empty segment.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_segment_reduce(const int64_t* ptr, const int64_t* perm, const void* value, void* out,
                                     int64_t* arg_out, int64_t S, int64_t D, int dtype, int reduce, void* stream);

/* ------------------------------------------------------------------------------------------
 * Backward of a segment / duplicate-run reduction (tsb200_segment_reduce, tsb200_coalesce_emit).  Replaces the
 *   autograd of torch_scatter.segment_csr / scatter that the reference's value reductions ride on
 *   (torch_sparse/storage.py:451, torch_sparse/reduce.py:36-54, torch_sparse/tensor.py:424-427).
 *   seg i64[E]: segment id of every INPUT entry;  count i64[S] (MEAN);  arg i64[S, D] (MIN/MAX, input positions);
 *   grad_out dtype[S, D] -> grad_in dtype[E, D] (fully written, no atomics):
 *     SUM  grad_in[i,d] = grad_out[seg[i],d]        MEAN  ... / max(count[seg[i]], 1)
 *     MIN/MAX  grad_in[i,d] = arg[seg[i],d] == i ? grad_out[seg[i],d] : 0
 *   Floating dtypes only.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_segment_reduce_bw(const int64_t* seg, const int64_t* count, const int64_t* arg,
                                        const void* grad_out, void* grad_in, int64_t E, int64_t S, int64_t D,
                                        int dtype, int reduce, void* stream);

/* ------------------------------------------------------------------------------------------
 * COO coalesce.  Replaces torch_sparse.coalesce -> SparseStorage.__init__ sort + .coalesce()
 *   (torch_sparse/coalesce.py:5-25, torch_sparse/storage.py:149-162, 436-466).
 *   Phase 1 (tsb200_coalesce_sort): key = row*N + col, stable radix sort with the original position
 *     as payload; head flags; returns in the workspace: sorted keys, perm, segment starts, and the
 *     number of unique keys E' which is ALSO copied asynchronously to *n_unique_host (pinned host
 *     int64, may be NULL). The caller synchronises the stream, reads E', allocates outputs.
 *   Phase 2 (tsb200_coalesce_emit): writes row'/col' i64[E'] and, if value_in != NULL, reduces
 *     value_in dtype[E, D] over each run of equal keys, in sorted (stable => input) order, into
 *     value_out dtype[E', D] with op in {SUM(add), MEAN, MIN, MAX} (torch_scatter.segment_csr
 *     semantics, call site storage.py:451). perm_out i64[E'] (optional) receives the input
 *     position of the first entry of each run. For the backward of the value reduction (tsb200_segment_reduce_bw)
 *     the call can also emit seg_out i64[E] (run id of every INPUT entry), count_out i64[E'] (run lengths) and
 *     arg_out i64[E', D] (MIN/MAX: input position of the earliest entry attaining the extreme); each may be NULL.
 *   The same workspace must be passed to both phases.
 *   Synchronisation: phase 1 synchronises `stream` once internally (it reads back an "input already sorted"
 *   flag to skip the sort, like the reference's check at storage.py:154); phase 2 and tsb200_coalesce_perm
 *   are fully asynchronous (they pick the sorted buffers from a selector phase 1 left in the workspace).
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_coalesce_workspace_bytes(int64_t E, int64_t M, int64_t N);
TSB200_API int tsb200_coalesce_sort(const int64_t* row, const int64_t* col, int64_t E, int64_t M, int64_t N,
                         void* workspace, size_t workspace_bytes, int64_t* n_unique_host,
                         void* stream);
TSB200_API int tsb200_coalesce_emit(int64_t E, int64_t N, int64_t n_unique, const void* value_in, int64_t D,
                         int dtype, int reduce, int64_t* row_out, int64_t* col_out,
                         void* value_out, int64_t* perm_out, int64_t* seg_out, int64_t* count_out,
                         int64_t* arg_out, const void* workspace, void* stream);

/* Full sorted permutation after tsb200_coalesce_sort: perm_out i64[E], perm_out[i] = input position of
 * the i-th entry in (row,col) order (stable). Replaces the sort-on-construct of SparseStorage.__init__
 * (torch_sparse/storage.py:149-162: `_, perm = index_sort(idx[1:], max_value)`). */
TSB200_API int tsb200_coalesce_perm(int64_t E, int64_t* perm_out, const void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * SpSpMM  C = A (MxKd) * B (KdxN), CSR x CSR -> CSR/COO with sorted unique columns per row and
 * structural zeros kept.  Replaces spspmm_sum -> torch.sparse.mm
 *   (torch_sparse/matmul.py:94-111, torch_sparse/spspmm.py:6-33).
 *   Phase 1 (symbolic): rowptr_c i64[M+1] (exclusive scan of the per-row unique column counts);
 *     nnz(C) is copied asynchronously to *nnz_c_host (pinned host int64, may be NULL).
 *   Phase 2 (numeric): col_c i64[nnz], row_c i64[nnz] (may be NULL), val_c dtype[nnz] (NULL when
 *     neither input has values; a NULL val_a / val_b means all-ones). dtype in {F32, F64}
 *     (torch.sparse.mm supports only these; test/test_matmul.py:56-57).
 *   Both phases need the same workspace. Both are asynchronous on `stream`.
 *   Preconditions (those of a SparseStorage CSR view): rowptr arrays are non-decreasing; for N > 2^18 (more than
 *   one column window) the columns of every B row must be sorted ascending — the first and last entry of a B row
 *   bound the windows a C row is searched in. A's rows need not be sorted; duplicates in either operand are legal
 *   (their products are accumulated).
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_spspmm_workspace_bytes(int64_t M, int64_t Kd, int64_t N, int64_t nnz_a,
                                     int64_t nnz_b);
TSB200_API int tsb200_spspmm_symbolic(const int64_t* rowptr_a, const int64_t* col_a, const int64_t* rowptr_b,
                           const int64_t* col_b, int64_t M, int64_t Kd, int64_t N, int64_t nnz_a,
                           int64_t nnz_b, int64_t* rowptr_c, void* workspace,
                           size_t workspace_bytes, int64_t* nnz_c_host, void* stream);
TSB200_API int tsb200_spspmm_numeric(const int64_t* rowptr_a, const int64_t* col_a, const void* val_a,
                          const int64_t* rowptr_b, const int64_t* col_b, const void* val_b,
                          int64_t M, int64_t Kd, int64_t N, int64_t nnz_a, int64_t nnz_b,
                          const int64_t* rowptr_c, int64_t* row_c, int64_t* col_c, void* val_c,
                          int dtype, void* workspace, size_t workspace_bytes, void* stream);

/* Single-pass SpSpMM (same contract and preconditions as the two phases above, half the work when the caller can
 * afford output arrays sized by an UPPER BOUND of nnz(C)):
 *   tsb200_spspmm_bound: the number of products sum_{e in A} |B row col_a[e]| >= nnz(C), copied asynchronously to
 *     *bound_host (pinned int64). workspace: the SpSpMM workspace (>= 256 bytes are used).
 *   tsb200_spspmm_fused: one kernel computes structure and values. Every output row is counted, then placed behind
 *     the rows before it through a decoupled look-back over per-row status words in the workspace (rows are handed
 *     out in increasing order to a resident persistent grid), so no symbolic pre-pass is needed. row_c / col_c /
 *     val_c hold `capacity` entries (capacity >= the bound is always enough); rowptr_c i64[M+1] is written;
 *     *nnz_c_host (pinned int64) receives nnz(C) asynchronously, or -1 if capacity was too small (nothing is written
 *     past `capacity`). Entries [nnz(C), capacity) of the arrays stay untouched. */
TSB200_API int tsb200_spspmm_bound(const int64_t* col_a, const int64_t* rowptr_b, int64_t nnz_a, void* workspace,
                                   size_t workspace_bytes, int64_t* bound_host, void* stream);
TSB200_API int tsb200_spspmm_fused(const int64_t* rowptr_a, const int64_t* col_a, const void* val_a,
                                   const int64_t* rowptr_b, const int64_t* col_b, const void* val_b, int64_t M,
                                   int64_t Kd, int64_t N, int64_t nnz_a, int64_t nnz_b, int64_t* rowptr_c,
                                   int64_t* row_c, int64_t* col_c, void* val_c, int64_t capacity, int dtype,
                                   void* workspace, size_t workspace_bytes, int64_t* nnz_c_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * Host-buffer SpMM (the end-to-end call a reference-side binding makes with CPU tensors):
 * all `_host` pointers are HOST memory (pinned for full speed, pageable works); the call stages
 * them to the current device, runs tsb200_spmm_fw and copies out (and arg_out) back. Synchronous.
 * Same semantics/argument meaning as tsb200_spmm_fw. Staging resources are kept per device: calls on different
 * devices run concurrently, calls on one device serialise; on an error return no copy of the call is in flight.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_fw_host(const int64_t* rowptr_host, const int64_t* col_host,
                        const void* value_host, const void* mat_host, void* out_host,
                        int64_t* arg_out_host, int64_t B, int64_t M, int64_t N, int64_t K,
                        int64_t E, int dtype, int reduce);

#ifdef __cplusplus
}
#endif
#endif /* TSB200_H_ */
