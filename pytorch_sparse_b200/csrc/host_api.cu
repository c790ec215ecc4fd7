// host_api.cu — library-level entry points of libtsb200: version / error text / device check and
// the HOST-buffer SpMM call (the end-to-end path a reference-side binding takes when it holds CPU
// tensors, cf. spmm_cpu(rowptr, col, value, mat, reduce), csrc/cpu/spmm_cpu.cpp:8-11).
//
// tsb200_spmm_fw_host pipelines PCIe against the kernel: `mat` goes up first, split over TWO upload
// streams (one DMA stream does not saturate the host link), then the CSR arrays in row chunks alternating
// between the two; each chunk's SpMM starts on a compute stream as soon as its indices have landed and its
// output rows are copied back on a fourth stream while later chunks are still uploading (the link is
// full duplex).
#include <cstdlib>
#include <mutex>

#include "common.cuh"

namespace tsb {

// One staging context PER DEVICE (streams, events and the device staging buffer belong to the device they were
// created on; callers on different devices run concurrently, callers on the same device serialise on `mu`).
struct HostCtx {
  std::mutex mu;
  char* buf = nullptr;
  size_t cap = 0;
  cudaStream_t s_up[2] = {nullptr, nullptr}, s_comp = nullptr, s_down = nullptr;
  static constexpr int kMaxChunks = 16;
  cudaEvent_t ev_up[kMaxChunks] = {}, ev_comp[kMaxChunks] = {}, ev_mat[2] = {}, ev_rowptr = nullptr;
  bool init = false;
};
static HostCtx g_host[kMaxDevices];

// Drain the four staging streams: on an error path the caller's host buffers and the shared device buffer must not
// be touched by copies still in flight after the call has returned.
static void host_drain(HostCtx& c) {
  if (!c.init) return;
  for (cudaStream_t s : {c.s_up[0], c.s_up[1], c.s_comp, c.s_down})
    if (s) cudaStreamSynchronize(s);
}

static int host_init(HostCtx& c) {
  if (c.init) return 0;
  for (int i = 0; i < 2; i++) {
    TSB_CUDA_TRY(cudaStreamCreateWithFlags(&c.s_up[i], cudaStreamNonBlocking));
    TSB_CUDA_TRY(cudaEventCreateWithFlags(&c.ev_mat[i], cudaEventDisableTiming));
  }
  TSB_CUDA_TRY(cudaStreamCreateWithFlags(&c.s_comp, cudaStreamNonBlocking));
  TSB_CUDA_TRY(cudaStreamCreateWithFlags(&c.s_down, cudaStreamNonBlocking));
  TSB_CUDA_TRY(cudaEventCreateWithFlags(&c.ev_rowptr, cudaEventDisableTiming));
  for (int i = 0; i < HostCtx::kMaxChunks; i++) {
    TSB_CUDA_TRY(cudaEventCreateWithFlags(&c.ev_up[i], cudaEventDisableTiming));
    TSB_CUDA_TRY(cudaEventCreateWithFlags(&c.ev_comp[i], cudaEventDisableTiming));
  }
  c.init = true;
  return 0;
}

}  // namespace tsb

using namespace tsb;

extern "C" int tsb200_version(void) { return TSB200_VERSION; }

// CUDA toolkit the library was compiled with, in CUDA_VERSION encoding (12090 = 12.9) — what the reference's
// torch.ops.torch_sparse.cuda_version() returns (csrc/version.cpp:27-41) and its import-time check compares with
// torch.version.cuda (torch_sparse/__init__.py:23-37).
extern "C" int tsb200_cuda_version(void) { return CUDART_VERSION; }

extern "C" int tsb200_sm_count(void) { return num_sms(); }

extern "C" const char* tsb200_strerror(int code) {
  switch (code) {
    case 0: return "success";
    case TSB200_ERR_INVALID_ARG: return "tsb200: invalid argument";
    case TSB200_ERR_UNSUPPORTED: return "tsb200: unsupported dtype/reduce/extent combination";
    case TSB200_ERR_WORKSPACE: return "tsb200: workspace missing or too small";
    case TSB200_ERR_NO_DEVICE: return "tsb200: no sm_90 CUDA device";
  }
  if (code > 0) return cudaGetErrorString((cudaError_t)code);
  return "tsb200: unknown error";
}

extern "C" int tsb200_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return TSB200_ERR_NO_DEVICE;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess)
    return TSB200_ERR_NO_DEVICE;
  return major == 9 ? 0 : TSB200_ERR_NO_DEVICE;
}

static int spmm_fw_host_locked(HostCtx& c, const int64_t* rowptr_host, const int64_t* col_host,
                               const void* value_host, const void* mat_host, void* out_host, int64_t* arg_out_host,
                               int64_t B, int64_t M, int64_t N, int64_t K, int64_t E, int dtype, int reduce);

extern "C" int tsb200_spmm_fw_host(const int64_t* rowptr_host, const int64_t* col_host, const void* value_host,
                                   const void* mat_host, void* out_host, int64_t* arg_out_host, int64_t B,
                                   int64_t M, int64_t N, int64_t K, int64_t E, int dtype, int reduce) {
  if (B < 0 || M < 0 || N < 0 || K < 0 || E < 0) return TSB200_ERR_INVALID_ARG;
  const size_t es = dtype_size(dtype);
  if (!es) return TSB200_ERR_INVALID_ARG;
  if (reduce < TSB200_SUM || reduce > TSB200_MAX) return TSB200_ERR_INVALID_ARG;
  const bool arg = reduce == TSB200_MIN || reduce == TSB200_MAX;
  if (B * M * K == 0) return 0;
  if (!rowptr_host || !out_host || (arg && !arg_out_host)) return TSB200_ERR_INVALID_ARG;
  if (E > 0 && (!col_host || !mat_host)) return TSB200_ERR_INVALID_ARG;
  if (int rc = tsb200_device_ok()) return rc;

  int dev = 0;
  TSB_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) return TSB200_ERR_NO_DEVICE;
  HostCtx& c = g_host[dev];
  std::lock_guard<std::mutex> lock(c.mu);
  int rc = host_init(c);
  if (!rc)
    rc = spmm_fw_host_locked(c, rowptr_host, col_host, value_host, mat_host, out_host, arg_out_host, B, M, N, K, E,
                             dtype, reduce);
  if (rc) host_drain(c);  // nothing of this call may still be in flight when the error is returned
  return rc;
}

static int spmm_fw_host_locked(HostCtx& c, const int64_t* rowptr_host, const int64_t* col_host,
                               const void* value_host, const void* mat_host, void* out_host, int64_t* arg_out_host,
                               int64_t B, int64_t M, int64_t N, int64_t K, int64_t E, int dtype, int reduce) {
  const size_t es = dtype_size(dtype);
  const bool arg = reduce == TSB200_MIN || reduce == TSB200_MAX;
  // device layout
  const size_t ws_bytes = tsb200_spmm_fw_workspace_bytes(B, M, K, E, dtype, reduce);
  size_t off = 0;
  const size_t o_rowptr = off; off += align_up((size_t)(M + 1) * 8, 256);
  const size_t o_col = off; off += align_up((size_t)(E > 0 ? E : 1) * 8 + 1024, 256);
  const size_t o_val = off; off += align_up((size_t)(E > 0 ? E : 1) * es + 1024, 256);
  const size_t o_mat = off; off += align_up((size_t)B * N * K * es, 256);
  const size_t o_out = off; off += align_up((size_t)B * M * K * es, 256);
  const size_t o_arg = off; off += arg ? align_up((size_t)B * M * K * 8, 256) : 0;
  const size_t o_ws = off; off += align_up(ws_bytes, 256);
  if (off > c.cap) {
    host_drain(c);
    if (c.buf) TSB_CUDA_TRY(cudaFree(c.buf));
    c.buf = nullptr; c.cap = 0;
    TSB_CUDA_TRY(cudaMalloc(&c.buf, off));
    c.cap = off;
  }
  char* d = c.buf;
  int64_t* d_rowptr = (int64_t*)(d + o_rowptr);
  int64_t* d_col = (int64_t*)(d + o_col);
  void* d_val = value_host ? (void*)(d + o_val) : nullptr;

  // dense operand: two halves on the two upload streams; rowptr rides on stream 0
  {
    const size_t mat_bytes = (size_t)B * N * K * es;
    const size_t half = align_up(mat_bytes / 2, 4096) < mat_bytes ? align_up(mat_bytes / 2, 4096) : mat_bytes;
    TSB_CUDA_TRY(cudaMemcpyAsync(d + o_mat, mat_host, half, cudaMemcpyHostToDevice, c.s_up[0]));
    if (mat_bytes > half)
      TSB_CUDA_TRY(cudaMemcpyAsync(d + o_mat + half, (const char*)mat_host + half, mat_bytes - half,
                                   cudaMemcpyHostToDevice, c.s_up[1]));
    TSB_CUDA_TRY(cudaMemcpyAsync(d_rowptr, rowptr_host, (size_t)(M + 1) * 8, cudaMemcpyHostToDevice, c.s_up[0]));
    TSB_CUDA_TRY(cudaEventRecord(c.ev_mat[0], c.s_up[0]));
    TSB_CUDA_TRY(cudaEventRecord(c.ev_mat[1], c.s_up[1]));
    TSB_CUDA_TRY(cudaStreamWaitEvent(c.s_comp, c.ev_mat[0], 0));
    TSB_CUDA_TRY(cudaStreamWaitEvent(c.s_comp, c.ev_mat[1], 0));
  }

  // chunking only pays (and only keeps out/arg_out contiguous per copy) for a single batch
  int nchunk = (B == 1 && M >= 4096 && E >= (1 << 20)) ? 8 : 1;
  if (const char* ev = getenv("TSB200_HOST_CHUNKS")) {  // tuning knob
    const int v = atoi(ev);
    if (v >= 1 && v <= HostCtx::kMaxChunks && B == 1) nchunk = v;
  }
  for (int ch = 0; ch < nchunk; ch++) {
    cudaStream_t up = c.s_up[ch & 1];
    const int64_t r0 = M * ch / nchunk, r1 = M * (ch + 1) / nchunk;
    const int64_t e0 = rowptr_host[r0], e1 = rowptr_host[r1];
    if (e1 > e0) {
      TSB_CUDA_TRY(cudaMemcpyAsync(d_col + e0, col_host + e0, (size_t)(e1 - e0) * 8, cudaMemcpyHostToDevice, up));
      if (value_host)
        TSB_CUDA_TRY(cudaMemcpyAsync((char*)d_val + e0 * es, (const char*)value_host + e0 * es,
                                     (size_t)(e1 - e0) * es, cudaMemcpyHostToDevice, up));
    }
    TSB_CUDA_TRY(cudaEventRecord(c.ev_up[ch], up));
    TSB_CUDA_TRY(cudaStreamWaitEvent(c.s_comp, c.ev_up[ch], 0));
    if (r1 > r0) {
      int rc = tsb200_spmm_fw(d_rowptr + r0, d_col, d_val, d + o_mat, d + o_out + (size_t)r0 * K * es,
                              arg ? (int64_t*)(d + o_arg) + r0 * K : nullptr, B, r1 - r0, N, K, E, dtype, reduce,
                              ws_bytes ? d + o_ws : nullptr, ws_bytes, c.s_comp);
      if (rc) return rc;
    }
    TSB_CUDA_TRY(cudaEventRecord(c.ev_comp[ch], c.s_comp));
    TSB_CUDA_TRY(cudaStreamWaitEvent(c.s_down, c.ev_comp[ch], 0));
    if (r1 > r0) {
      const size_t rows = (size_t)(nchunk == 1 ? B * M : (r1 - r0));
      TSB_CUDA_TRY(cudaMemcpyAsync((char*)out_host + (size_t)r0 * K * es, d + o_out + (size_t)r0 * K * es,
                                   rows * K * es, cudaMemcpyDeviceToHost, c.s_down));
      if (arg)
        TSB_CUDA_TRY(cudaMemcpyAsync(arg_out_host + r0 * K, (int64_t*)(d + o_arg) + r0 * K, rows * K * 8,
                                     cudaMemcpyDeviceToHost, c.s_down));
    }
  }
  TSB_CUDA_TRY(cudaStreamSynchronize(c.s_up[0]));
  TSB_CUDA_TRY(cudaStreamSynchronize(c.s_up[1]));
  TSB_CUDA_TRY(cudaStreamSynchronize(c.s_comp));
  TSB_CUDA_TRY(cudaStreamSynchronize(c.s_down));
  return 0;
}
