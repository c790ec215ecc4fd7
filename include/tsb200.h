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

/* ------------------------------------------------------------------------------------------
 * SpMM over an FP8 (e4m3) dense operand (no counterpart in the reference).  B = 1.
 *   out[m,:] = reduce_{e in row m} w_e * x8[col[e], :]   with   w_e = fl32(value[e] * scale[col[e] * scale_stride])
 *   x8 e4m3[N, K] (K % 16 == 0, 16-byte aligned), scale f32 (scale_stride 0: one scale for the whole operand, 1: one
 *   per dense row), value out_dtype[E] or NULL (1), out out_dtype[M, K] with out_dtype in {F32, F16, BF16},
 *   arg_out i64[M, K] for MIN/MAX. x8 elements widen to fp32 exactly. SUM/MEAN: fp32 FFMA of w_e * x8 over the row,
 *   MEAN divides by max(deg, 1), one rounding to out_dtype. MIN/MAX: strict compare of p = round_out(fl32(w_e * x8)),
 *   the smallest e wins ties, out = p; empty rows, NaN and +-0 as tsb200_spmm_fw.
 *   plan == NULL: unplanned, workspace tsb200_spmm_fw_workspace_bytes(1, M, K, E, out_dtype, reduce). Otherwise
 *   `plan` is a tsb200_spmm_plan of rowptr with its counts, workspace tsb200_spmm_fw_planned_workspace_bytes(K,
 *   n_long, n_slot, reduce); results as tsb200_spmm_fw_planned vs tsb200_spmm_fw. TSB200_ERR_UNSUPPORTED for
 *   K % 16 != 0, another out_dtype, or a misaligned pointer (x8 / out 16 B, col 8 B, value / scale 4 B, arg_out 16 B).
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_fw_fp8(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                  const float* scale, int64_t scale_stride, void* out, int64_t* arg_out, int64_t M,
                                  int64_t N, int64_t K, int64_t E, int out_dtype, int reduce, const void* plan,
                                  size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                  size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * SpMM from an FP8 (e4m3) operand to an FP8 (e4m3) result with per-row scales, so that multi-hop propagation
 * (X_{h+1} = A X_h) stays in e4m3 without a float copy of the hop (no counterpart in the reference).  B = 1.
 *   Let y be the F32 result of tsb200_spmm_fw_fp8 with the same arguments and out_dtype = TSB200_F32, on the same path
 *   (planned or unplanned; value f32[E] or NULL). Then, per row m:
 *     out_scale[m] = amax_k |y[m,k]| / 448 (IEEE fp32 division, round to nearest), or 1 when that amax is not > 0
 *                    (an all-zero or empty row, and a row holding NaN: the amax propagates NaN);
 *     out8[m,k]    = e4m3(y[m,k] / out_scale[m]) (IEEE division), rounded to nearest even with subnormals kept, as
 *                    torch's non-saturating float8_e4m3fn cast: |q| <= 464 rounds to at most 448, |q| > 464 and
 *                    +-inf become NaN, -0 stays -0. An inf row gets scale inf: finite entries become +-0, inf NaN.
 *   That is, bit for bit, torch's quantize_fp8(y, per_row=True) on the CPU. arg_out (MIN/MAX) is that call's arg_out.
 *   out8 e4m3[M, K] (16-byte aligned), out_scale f32[M]: valid x8 / scale operands of the next hop.
 *   Plan and workspace sizing as tsb200_spmm_fw_fp8 with out_dtype = TSB200_F32. E == 0: out8 = 0, out_scale = 1,
 *   arg_out = 0. TSB200_ERR_UNSUPPORTED for K % 16 != 0, K > 2048 (one column tile: the row amax is not taken across
 *   tiles), or a misaligned pointer (as tsb200_spmm_fw_fp8; out_scale 4 B).
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_fw_fp8_quant(const int64_t* rowptr, const int64_t* col, const void* value,
                                        const void* mat, const float* scale, int64_t scale_stride, void* out8,
                                        float* out_scale, int64_t* arg_out, int64_t M, int64_t N, int64_t K,
                                        int64_t E, int reduce, const void* plan, size_t plan_bytes, int64_t n_seg,
                                        int64_t n_long, int64_t n_slot, void* workspace, size_t workspace_bytes,
                                        void* stream);

/* ------------------------------------------------------------------------------------------
 * FP8 SpMM with a per-row e4m3 residual added in the store epilogue, for propagation with a fixed residual term
 * (APPNP: X_{h+1} = (1-a) A X_h + a H; label propagation: Y_{h+1} = a A Y_h + (1-a) Y_0) without leaving e4m3
 * (no counterpart in the reference).  B = 1, SUM / MEAN only.
 *   Let y[m,k] be the F32 value tsb200_spmm_fw_fp8 writes with the same arguments and out_dtype = TSB200_F32, on the
 *   same path (planned or unplanned): after the mean's division, +0 on an empty row. With
 *     rho[m,k] = fl32(res_scale[m * res_scale_stride] * e4m3(res8[m,k]))    (res_scale_stride 0 or 1)
 *     z[m,k]   = fl32(y[m,k] + rho[m,k])                                     (one IEEE add, no FMA contraction)
 *   out_scale == NULL: out out_dtype[M, K] = round_out(z) (round to nearest even), value out_dtype[E] or NULL.
 *   out_scale != NULL: the e4m3 result of tsb200_spmm_fw_fp8_quant with z in place of y (bit for bit torch's
 *   quantize_fp8(z, per_row=True) on the CPU); out e4m3[M, K], value f32[E] or NULL, out_dtype must be TSB200_F32,
 *   K <= 2048. NaN and +-inf propagate through z as IEEE says (a -0 residual on an empty row gives +0).
 *   res8 e4m3[M, K] contiguous, 16-byte aligned; res_scale f32, 4-byte aligned. The caller folds propagation weights
 *   into the entry values and res_scale. E == 0: z = fl32(+0 + rho).
 *   Plan and workspace sizing as tsb200_spmm_fw_fp8 (with out_dtype = TSB200_F32 for an e4m3 result).
 *   res8 == NULL: exactly tsb200_spmm_fw_fp8 (out_scale == NULL) or tsb200_spmm_fw_fp8_quant, MIN / MAX included.
 *   TSB200_ERR_UNSUPPORTED for MIN / MAX with a residual, a misaligned res8 (16 B) or res_scale (4 B), and as
 *   tsb200_spmm_fw_fp8 / _quant otherwise.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_fw_fp8_res(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                      const float* scale, int64_t scale_stride, const void* res8,
                                      const float* res_scale, int64_t res_scale_stride, void* out, float* out_scale,
                                      int64_t* arg_out, int64_t M, int64_t N, int64_t K, int64_t E, int out_dtype,
                                      int reduce, const void* plan, size_t plan_bytes, int64_t n_seg, int64_t n_long,
                                      int64_t n_slot, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * SpMM with a residual added in the store epilogue: out = A x + s * r, for propagation layers with a dense term
 * (APPNP, GCNII, GIN, residual connections, GCN self-loops as a per-row scale 1/d) without a second pass over the
 * result (no counterpart in the reference).  B = 1, SUM / MEAN only.
 *   Let y[m,k] be the fp32 (fp64 for F64) row result tsb200_spmm_fw / tsb200_spmm_fw_planned computes with the same
 *   arguments, on the same path: after the mean's division, +0 on an empty row. With s = res_scale[m * res_scale_stride]
 *   (res_scale_stride 0 or 1; float32, or float64 when dtype is F64):
 *     out[m,k] = round_dtype(fl(y[m,k] + fl(s * res[m,k])))   (one IEEE product and one IEEE add, no FMA contraction)
 *   rounded to nearest even. NaN and +-inf propagate as IEEE says; a -0 residual on an empty row gives +0.
 *   dtype F32 / F64 / F16 / BF16; res dtype[M, K] contiguous; value dtype[E] or NULL (1). E == 0: round(fl(+0 + s*r)).
 *   plan == NULL: workspace tsb200_spmm_fw_workspace_bytes(1, M, K, E, dtype, reduce). Otherwise `plan` is a
 *   tsb200_spmm_plan of rowptr with its counts, workspace tsb200_spmm_fw_planned_workspace_bytes(K, n_long, n_slot,
 *   reduce). Both are read on the vector path only (F32 / F16 / BF16, K * sizeof(dtype) % 16 == 0, the alignments of
 *   tsb200_spmm_fw and a 16-byte aligned res) with E > 0; any other call reads neither. With E == 0 on the vector
 *   path's conditions a residual-only kernel writes round(fl(+0 + s*r)) in one pass without reading rowptr (the
 *   residual's gradient s * g is formed this way); otherwise the generic kernel runs and reads rowptr.
 *   res == NULL: TSB200_ERR_INVALID_ARG (without a residual the call is tsb200_spmm_fw / _planned).
 *   TSB200_ERR_UNSUPPORTED for MIN / MAX, an integer dtype, or a res_scale not aligned to its element size.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_fw_res(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                  const void* res, const void* res_scale, int64_t res_scale_stride, void* out,
                                  int64_t M, int64_t N, int64_t K, int64_t E, int dtype, int reduce, const void* plan,
                                  size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                  size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-aggregation SpMM: several per-row aggregations of the messages p_e = value[e] * mat[col[e]] from one gather
 * pass, for PNA-style layers (no counterpart in the reference).  B = 1.
 *   aggrs[0..n_aggr) are distinct codes among TSB200_SUM, TSB200_MEAN, TSB200_MIN, TSB200_MAX, TSB200_VAR and
 *   TSB200_STD (1 <= n_aggr <= 6); out dtype[M, n_aggr, K] holds aggregator aggrs[a] of row m in out[m, a, :].
 *   SUM, MEAN, MIN, MAX (and arg_min / arg_max): bit for bit what tsb200_spmm_fw / tsb200_spmm_fw_planned returns
 *   with the same arguments, on the same path and at the same work-item size. With n = max(deg, 1), mu the fp32 (fp64
 *   for F64) mean and Q = sum_e fma(p_e, p_e, .) accumulated in the sum's order:
 *     VAR = max(fl(fl(Q / n) - fl(mu * mu)), 0)   (NaN passes)
 *     STD = sqrt(VAR) where VAR > 1e-5, else 0
 *   each rounded once to dtype. arg_min / arg_max int64[M, K] or NULL (not stored); each needs its aggregator.
 *   dtype F32 / F64 / F16 / BF16; value dtype[E] or NULL (1). E == 0: every aggregator 0, args 0.
 *   plan == NULL: workspace tsb200_spmm_fw_multi_workspace_bytes(K, E, 0, 0, 0). Otherwise `plan` is a tsb200_spmm_plan
 *   of rowptr with its counts, workspace tsb200_spmm_fw_multi_workspace_bytes(K, E, 1, n_long, n_slot). Both are read
 *   on the vector path only (F32 / F16 / BF16, K * sizeof(dtype) % 16 == 0, E > 0, the extents and alignments of
 *   tsb200_spmm_fw, arg_max 16-byte aligned); any other call runs the generic kernel, which reads neither.
 *   TSB200_ERR_INVALID_ARG for an empty, long, repeating or out-of-range aggrs, or an arg pointer without its aggregator;
 *   TSB200_ERR_UNSUPPORTED for an integer dtype.
 * ------------------------------------------------------------------------------------------ */
#define TSB200_VAR 4
#define TSB200_STD 5
TSB200_API size_t tsb200_spmm_fw_multi_workspace_bytes(int64_t K, int64_t E, int planned, int64_t n_long,
                                                       int64_t n_slot);
TSB200_API int tsb200_spmm_fw_multi(const int64_t* rowptr, const int64_t* col, const void* value, const void* mat,
                                    const int* aggrs, int n_aggr, void* out, int64_t* arg_min, int64_t* arg_max,
                                    int64_t M, int64_t N, int64_t K, int64_t E, int dtype, const void* plan,
                                    size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Softmax-aggregation SpMM: per row m and column k the messages p_e = value[e] * mat[col[e], k] weighted by a softmax
 * over the row's entries with a temperature t_k, as GENConv's softmax aggregation (no counterpart in the reference).
 * B = 1. With A the accumulator type (fp32; fp64 for F64):
 *     p_e = fl_A(v_e x[col_e, k])   (exact for F16 / BF16),   y_e = fl_A(t_k p_e)
 *     mu = max_e y_e,   w_e = exp(y_e - mu),   s = sum_e w_e,   a = sum_e w_e p_e
 *     out[m, k] = round(a / s)  (one IEEE division),   lse[m, k] = mu + log(s)  (type A)
 *   Every stored entry counts, duplicates included. An empty row gives out = +0 and lse = -inf. NaN in x, value or t
 *   propagates to the columns it reaches. Inputs whose t * p is not finite are outside this contract: they do not
 *   fault, and give NaN or an unspecified value. The kernels run the softmax online (rescaling s and a when mu
 *   grows); the fp32 exp is ex2.approx.ftz of a log2(e)-scaled argument (exp(0) = 1, exp(-inf) = +0). With t = 0 the
 *   result is bit for bit tsb200_spmm_fw / _planned MEAN on the same path and work-item size for F16 / BF16, and for
 *   F32 without values. A one-entry row gives round(p). Negative t is allowed (a soft minimum).
 *   mat dtype[N, K], value dtype[E] or NULL (1), t type A with t_stride 0 (one scalar) or 1 (one per column, [K]),
 *   out dtype[M, K], lse A[M, K] or NULL (not stored). dtype F32 / F64 / F16 / BF16.
 *   plan == NULL: workspace tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 0, 0, 0). Otherwise `plan` is a
 *   tsb200_spmm_plan of rowptr with its counts, workspace tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 1, n_long,
 *   n_slot). Both are read on the vector path only (F32 / F16 / BF16, K * sizeof(dtype) % 16 == 0, E > 0, the extents
 *   and alignments of tsb200_spmm_fw, lse 16-byte aligned); any other call runs the generic kernel, which reads neither.
 *   TSB200_ERR_INVALID_ARG for a negative extent or count, a NULL pointer that is needed or t_stride not 0 / 1;
 *   TSB200_ERR_UNSUPPORTED for an integer dtype or a t not aligned to its element size; TSB200_ERR_WORKSPACE for a
 *   missing or short workspace.
 *
 * Its backward. With g = grad_out, o = out and l = lse (the forward's) of row r, and alpha_e = exp(t p_e - l), the
 * gradient of message e is d_e = g alpha_e (1 + t (p_e - o)), per column.
 *   tsb200_spmm_softmax_aggr_bw_rows: grad_value[e] = <x[col_e], d_e> (dtype[E], needs value) and
 *     U[r, k] = g[r, k] sum_{e in row r} alpha_e (p_e - o[r, k])^2 (type A [M, K]; the temperature's gradient is
 *     U.sum(0), or U.sum() for one scalar). Either output may be NULL: it is not wanted.
 *   tsb200_spmm_softmax_aggr_bw_cols: grad_mat[n] = sum_{e in column n} v_e d_e (dtype[N, K]), on the CSC view:
 *     colptr[N + 1], row_csc[E] and value_csc = value[csr2csc] (or NULL) in place of rowptr, col and value. grad_mat
 *     NULL: nothing is launched.
 *   F32 / F16 / BF16 rows of 16 ... 1024 bytes (K * sizeof(dtype) a multiple of 16), E > 0, the extents of
 *   tsb200_spmm_fw and 16-byte aligned mat, grad_out, out, lse (and grad_mat) run row-split kernels: rows (columns)
 *   longer than 256 entries, or past a 32-row item's budget, are cut into segments whose fp32 partials are summed in
 *   segment order. They need workspace tsb200_spmm_softmax_aggr_bw_workspace_bytes(K, E), 256-byte aligned (one
 *   workspace serves either call). Any other call runs a generic kernel (a warp per row or column, a lane per feature
 *   column) and reads no workspace. No atomics: every gradient is the same bit for bit from run to run. Return codes
 *   as the forward's.
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_spmm_fw_softmax_aggr_workspace_bytes(int64_t K, int64_t E, int planned, int64_t n_long,
                                                              int64_t n_slot);
TSB200_API int tsb200_spmm_fw_softmax_aggr(const int64_t* rowptr, const int64_t* col, const void* value,
                                           const void* mat, const void* t, int64_t t_stride, void* out, void* lse,
                                           int64_t M, int64_t N, int64_t K, int64_t E, int dtype, const void* plan,
                                           size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot,
                                           void* workspace, size_t workspace_bytes, void* stream);
TSB200_API int tsb200_spmm_softmax_aggr_bw_rows(const int64_t* rowptr, const int64_t* col, const void* value,
                                                const void* mat, const void* t, int64_t t_stride, const void* grad_out,
                                                const void* out, const void* lse, void* grad_value, void* U, int64_t M,
                                                int64_t N, int64_t K, int64_t E, int dtype, void* workspace,
                                                size_t workspace_bytes, void* stream);
TSB200_API int tsb200_spmm_softmax_aggr_bw_cols(const int64_t* colptr, const int64_t* row_csc, const void* value_csc,
                                                const void* mat, const void* t, int64_t t_stride, const void* grad_out,
                                                const void* out, const void* lse, void* grad_mat, int64_t M, int64_t N,
                                                int64_t K, int64_t E, int dtype, void* workspace,
                                                size_t workspace_bytes, void* stream);
TSB200_API size_t tsb200_spmm_softmax_aggr_bw_workspace_bytes(int64_t K, int64_t E);

/* ------------------------------------------------------------------------------------------
 * FP8 (e4m3) quantisation of a float matrix: the operand of tsb200_spmm_fw_fp8, made without float temporaries (no
 * counterpart in the reference).
 *   x dtype[N, K] with dtype in {F32, F16, BF16}, row m at x + m * ld elements (ld >= K; the last dimension is
 *   contiguous, so a column slice of a wider matrix needs no copy). Per row (per_row = 1) or over the whole tensor
 *   (per_row = 0), with xf = fl32(x) (exact):
 *     amax  = max |xf|, NaN if any element is NaN;
 *     scale = amax / 448 (IEEE fp32 division) when amax > 0, otherwise 1 (all-zero, all -0 and NaN rows);
 *     x8    = e4m3(xf / scale) (IEEE division), rounded as torch's non-saturating float8_e4m3fn cast: nearest even,
 *             subnormals kept, -0 stays -0, |q| > 464 and +-inf become NaN (an inf row gets scale inf).
 *   That is, bit for bit, torch's quantize_fp8(x, per_row) on the CPU (NaN in any encoding), and the rounding of
 *   tsb200_spmm_fw_fp8_quant's e4m3 result.
 *   x8 e4m3[N, K] contiguous; scale f32[N] (per row) or f32[1] (per tensor), 4-byte aligned.
 *   Rows are read with 16-byte loads when x, ld * size and K * size are multiples of 16 bytes and x8 is 16-byte
 *   aligned, element by element otherwise; both give the same bits.
 *   workspace: per_row = 0 only, >= 4 bytes, 4-byte aligned (one amax word; the call clears it); may be NULL per row.
 *   No host synchronisation (CUDA-graph capturable): per row one kernel, per tensor a memset, an amax kernel and the
 *   quantise kernel.
 *   N == 0 per row: nothing is launched. TSB200_ERR_INVALID_ARG for a negative extent, ld < K, per_row not 0 / 1,
 *   NULL x / x8 / scale, K == 0 or (per tensor) N == 0 (the amax of no elements); TSB200_ERR_UNSUPPORTED for another
 *   dtype, K >= 2^31, or a misaligned x (element size), scale or workspace; TSB200_ERR_WORKSPACE for a missing or
 *   short per-tensor workspace.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_quantize_fp8(const void* x, int64_t N, int64_t K, int64_t ld, int dtype, int per_row, void* x8,
                                   float* scale, void* workspace, size_t workspace_bytes, void* stream);

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
 * SDDMM over two FP8 (e4m3) operands with per-tensor or per-row scales: edge scores <a[row_e], b[col_e]> of quantised
 * embeddings (no counterpart in the reference).  B = 1.
 *   For every entry e of the CSR structure (rowptr, col), row r, column c:
 *     d_e = sum_k a8[r,k] * b8[c,k]   (each product exact in fp32, the sum in fp32 in the kernel's lane order,
 *                                      starting from +0)
 *     s_e = fl32(a_scale[r * a_scale_stride] * b_scale[c * b_scale_stride])   (strides 0: one scale per operand)
 *     out[e] = round_out(fl32(s_e * d_e))   (round to nearest even; no FMA contraction)
 *   a8 e4m3[M, K], b8 e4m3[N, K], both contiguous and 16-byte aligned, K % 16 == 0 and K <= 2048; a_scale / b_scale
 *   f32, 4-byte aligned; out out_dtype[E] in CSR order, out_dtype in {F32, F16, BF16}. NaN in either operand or scale
 *   propagates; +-0 follows IEEE. The work decomposition is tsb200_spmm_value_bw's row-wise kernel: the a8 row is
 *   loaded once per CSR row, b8 rows are gathered; rows over 256 entries go through the device-side segment queue.
 *   workspace: tsb200_sddmm_fp8_workspace_bytes(M, K, E) bytes, 256 B aligned (0 when E == 0 or K == 0).
 *   E == 0: nothing is launched. K == 0: out = +0 (a memset). TSB200_ERR_INVALID_ARG for a negative extent, a scale
 *   stride other than 0 / 1, a NULL pointer, a missing or misaligned workspace; TSB200_ERR_UNSUPPORTED for another
 *   out_dtype, K % 16 != 0, K > 2048, E >= 2^31 - 64, M or N >= 2^32, or a misaligned pointer (a8 / b8 16 B, col 8 B,
 *   scales 4 B, out its element size); TSB200_ERR_WORKSPACE for a short workspace.
 * ------------------------------------------------------------------------------------------ */
TSB200_API size_t tsb200_sddmm_fp8_workspace_bytes(int64_t M, int64_t K, int64_t E);
TSB200_API int tsb200_sddmm_fp8(const int64_t* rowptr, const int64_t* col, const void* a8, const float* a_scale,
                                int64_t a_scale_stride, const void* b8, const float* b_scale, int64_t b_scale_stride,
                                void* out, int64_t M, int64_t N, int64_t K, int64_t E, int out_dtype, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-head SpMM and SDDMM: one weight per entry and head (graph attention; no counterpart in the reference).  B = 1.
 *   x, a, b are [rows, H, D] contiguous (row-major, K = H * D columns per row), dtype F32 / F64 / F16 / BF16.
 *   tsb200_spmm_heads:  out[m, h, :] = sum_{e in row m} value[e, h] * x[col_e, h, :]
 *     value dtype[E, H] or NULL (every weight 1: the plain sum over K = H * D columns); out dtype[M, H, D].
 *     fp32 accumulation (fp64 for F64), one rounding to dtype; an empty row gives +0. With
 *     D * sizeof(dtype) % 16 == 0 and 16-byte aligned x / out (col 8 B, value 4 B) the sum kernels of tsb200_spmm_fw
 *     run with each 16-byte chunk weighed by its own head's value; with H == 1 the bits are those of tsb200_spmm_fw
 *     (or tsb200_spmm_fw_planned). Otherwise a lane-per-column kernel sums every column in entry order.
 *     plan: NULL, or tsb200_spmm_plan's plan of (rowptr, E) with its counts, as for tsb200_spmm_fw_planned.
 *     workspace: tsb200_spmm_fw_workspace_bytes(1, M, H * D, E, dtype, TSB200_SUM) bytes without a plan,
 *     tsb200_spmm_fw_planned_workspace_bytes(H * D, n_long, n_slot, TSB200_SUM) with one; 256 B aligned.
 *   tsb200_sddmm_heads: out[e, h] = <a[row_e, h, :], b[col_e, h, :]>, a dtype[M, H, D], b dtype[N, H, D],
 *     out dtype[E, H] in CSR order; fp32 accumulation (fp64 for F64), one rounding. With HL = D * sizeof(dtype) / 16
 *     a power of two, H * HL <= 64 vectors, HL not above the row's lane count, 16-byte aligned a / b and a workspace of
 *     tsb200_spmm_value_bw_workspace_bytes(1, M, H * D, E, dtype) bytes (256 B aligned) the row-wise kernels of
 *     tsb200_spmm_value_bw run, each step's dot reduced over the HL lanes of its head; with H == 1 their bits are
 *     tsb200_spmm_value_bw's (reduce SUM) wherever both take the row-wise kernel. Otherwise a warp-per-row kernel.
 *   Nothing is launched when there is nothing to write (M * H * D == 0, resp. E * H == 0); E == 0 (spmm) or D == 0
 *   (sddmm) writes +0. TSB200_ERR_INVALID_ARG for a negative extent or count, a NULL pointer that is needed or a
 *   misaligned workspace; TSB200_ERR_UNSUPPORTED for another dtype or H * D >= 2^40; TSB200_ERR_WORKSPACE for a
 *   short workspace. The workspace and plan rules are tsb200_spmm_fw_planned's.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_spmm_heads(const int64_t* rowptr, const int64_t* col, const void* value, const void* x, void* out,
                                 int64_t M, int64_t N, int64_t H, int64_t D, int64_t E, int dtype, const void* plan,
                                 size_t plan_bytes, int64_t n_seg, int64_t n_long, int64_t n_slot, void* workspace,
                                 size_t workspace_bytes, void* stream);
TSB200_API int tsb200_sddmm_heads(const int64_t* rowptr, const int64_t* col, const void* a, const void* b, void* out,
                                  int64_t M, int64_t N, int64_t H, int64_t D, int64_t E, int dtype, void* workspace,
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
 *   SUM/MEAN start at +0 (torch_scatter's reducer does): a segment of -0 entries gives +0. MIN/MAX compare strictly
 *   from the segment's first entry: a NaN there is the result (arg = that entry), a NaN anywhere else never is.
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
 * Segment softmax over a CSR / CSC pointer (torch.sparse.softmax over a row or a column; no counterpart in the
 *   reference).  ptr i64[S+1] (rowptr, or colptr with perm = csr2csc); perm i64[E] or NULL; value, out dtype[E, D],
 *   dtype F32 / F64 / F16 / BF16. Segment s is the entries j in [ptr[s], ptr[s+1]), read from value[perm ? perm[j] : j]
 *   and written to out at the same position, so a column softmax comes back in CSR order. Per segment and column d,
 *   in A = fp32 (fp64 for F64):
 *     m = max_j v_j (any NaN gives NaN);  e_j = exp(fl(v_j - m));  S = sum_j e_j;  out_j = round(e_j / S) (IEEE
 *     division). The order of the sum depends only on the segment's length and D, never on another segment, the grid
 *     or the operands' alignment. A segment holding a NaN or +inf, or all -inf, gives NaN everywhere; a -inf entry
 *     next to finite ones gives +0; an empty segment writes nothing.
 *   tsb200_segment_softmax_bw: grad_in_j = round(out_j * (grad_out_j - sum_k out_k grad_out_k)), the dot in A by FMA
 *     in a fixed order; out is the forward's result, grad_out / grad_in dtype[E, D] addressed like value / out.
 *   No workspace, no atomics, no host synchronisation (graph-capturable). Returns TSB200_ERR_INVALID_ARG for a
 *   negative extent or a NULL pointer that is needed, 0 without a launch when S, E or D is 0, and
 *   TSB200_ERR_UNSUPPORTED for another dtype.
 * ------------------------------------------------------------------------------------------ */
TSB200_API int tsb200_segment_softmax(const int64_t* ptr, const int64_t* perm, const void* value, void* out, int64_t S,
                                      int64_t E, int64_t D, int dtype, void* stream);
TSB200_API int tsb200_segment_softmax_bw(const int64_t* ptr, const int64_t* perm, const void* out,
                                         const void* grad_out, void* grad_in, int64_t S, int64_t E, int64_t D,
                                         int dtype, void* stream);

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
 *     Same rules as tsb200_segment_reduce: SUM/MEAN start at +0 (a run of -0 gives +0); MIN/MAX compare strictly
 *     from the run's first entry (a NaN there is the result, a NaN later in the run never is).
 *   The key is one 64-bit word: tsb200_coalesce_sort returns TSB200_ERR_UNSUPPORTED for M * N > 2^64 (and for
 *   E >= 2^31).
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
