// quant.cu — tsb200_quantize_fp8: a bf16 / f16 / f32 matrix [N, K] (row stride ld) as an e4m3 matrix with a float32
// scale per row or per tensor, bit for bit torch's quantize_fp8 on the CPU. Streaming, nothing but x8 and the scales is
// written: a 16-byte aligned row of at most 2 KB is loaded into registers once (quantize_fp8_short_kernel); a longer or
// unaligned row is read once for its amax and once more, from L1 / L2, to be quantised (quantize_fp8_kernel). A
// per-tensor scale takes one more read of x (quantize_fp8_amax_kernel). The rounding helpers are the ones the
// e4m3-result SpMM epilogue uses (spmm_common.cuh), so both make the same bits from the same values.
#include "spmm_common.cuh"

namespace tsb {

constexpr int kQuantThreads = 256;

// A row is walked in units: W = Vec<T>::VEC elements (one 16-byte load) on the vector path, one element on the
// element-wise path taken by rows that are not 16-byte aligned. Both widenings to fp32 are exact.
template <typename T, int W> __device__ __forceinline__ void load_unit(const T* p, float* f) {
  if constexpr (W == 1) {
    f[0] = Traits<T>::to_acc(*p);
  } else {
    Vec<T>::unpack(ldg128(p), f);
  }
}

// W results divided by the scale, as W e4m3 bytes (one 8- or 4-byte store on the vector path)
template <int W> __device__ __forceinline__ void store_unit(uint8_t* q, const float* f, float s) {
  if constexpr (W == 1) {
    *q = e4m3_quant(f[0], s);
  } else {
    uint32_t w[W / 4];
#pragma unroll
    for (int j = 0; j < W / 4; j++)
      w[j] = e4m3x2(__fdiv_rn(f[4 * j], s), __fdiv_rn(f[4 * j + 1], s)) |
             (e4m3x2(__fdiv_rn(f[4 * j + 2], s), __fdiv_rn(f[4 * j + 3], s)) << 16);
    if constexpr (W == 8) {
      *reinterpret_cast<uint2*>(q) = make_uint2(w[0], w[1]);
    } else {
      *reinterpret_cast<uint32_t*>(q) = w[0];
    }
  }
}

// This lane's share of max |x| over one row: units gl, gl + G, ... of U. NaN propagates (amax_nan).
template <typename T, int W>
__device__ __forceinline__ float row_amax_part(const T* xr, int64_t U, int gl, int G, float m) {
#pragma unroll 2
  for (int64_t u = gl; u < U; u += G) {
    float f[W];
    load_unit<T, W>(xr + u * W, f);
#pragma unroll
    for (int i = 0; i < W; i++) m = amax_nan(m, fabsf(f[i]));
  }
  return m;
}

// Rows are handed to lane groups of G = 2^gshift lanes (the units of a row rounded up to a power of two, at most 32),
// grid-stride.
// amax_word == nullptr: one scale per row, from the row's amax (a shuffle over its group); otherwise one scale for the
// whole tensor, from the amax bits quantize_fp8_amax_kernel left in *amax_word, written to scale[0] by thread 0.
template <typename T, int W>
__global__ void __launch_bounds__(kQuantThreads)
    quantize_fp8_kernel(const T* __restrict__ x, int64_t N, int64_t K, int64_t ld, int gshift,
                        uint8_t* __restrict__ x8, float* __restrict__ scale, const uint32_t* __restrict__ amax_word) {
  const int G = 1 << gshift;
  const int lane = threadIdx.x & 31;
  const int gl = lane & (G - 1);
  const unsigned gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1) << (lane & ~(G - 1));
  const int64_t U = K / W;
  const int64_t rows_per_block = kQuantThreads >> gshift;
  float s = 1.f;
  if (amax_word) {
    s = e4m3_row_scale(__uint_as_float(*amax_word));
    if (blockIdx.x == 0 && threadIdx.x == 0) *scale = s;
  }
  for (int64_t row = (int64_t)blockIdx.x * rows_per_block + (threadIdx.x >> gshift); row < N;
       row += (int64_t)gridDim.x * rows_per_block) {
    const T* xr = x + row * ld;
    if (!amax_word) {
      float m = row_amax_part<T, W>(xr, U, gl, G, 0.f);
      for (int o = G >> 1; o > 0; o >>= 1) m = amax_nan(m, __shfl_xor_sync(gmask, m, o));
      s = e4m3_row_scale(m);
      if (gl == 0) scale[row] = s;
    }
    uint8_t* qr = x8 + row * K;
#pragma unroll 2
    for (int64_t u = gl; u < U; u += G) {
      float f[W];
      load_unit<T, W>(xr + u * W, f);
      store_unit<W>(qr + u * W, f, s);
    }
  }
}

// Rows of at most 2 KB on the vector path (NU = 1, 2 or 4 units per lane): a lane group takes RB = 4 / NU consecutive
// rows at a time and loads all its units of them into registers before it uses any, so every lane has four 16-byte
// loads in flight; each row is then reduced and quantised from the registers, read from memory once. Same arguments
// and results as quantize_fp8_kernel, which keeps one load in flight per lane on such rows.
template <typename T, int NU>
__global__ void __launch_bounds__(kQuantThreads)
    quantize_fp8_short_kernel(const T* __restrict__ x, int64_t N, int64_t K, int64_t ld, int gshift,
                              uint8_t* __restrict__ x8, float* __restrict__ scale,
                              const uint32_t* __restrict__ amax_word) {
  constexpr int W = Vec<T>::VEC;
  constexpr int RB = 4 / NU;
  const int G = 1 << gshift;
  const int lane = threadIdx.x & 31;
  const int gl = lane & (G - 1);
  const unsigned gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1) << (lane & ~(G - 1));
  const int U = (int)(K / W);
  const int64_t groups_per_block = kQuantThreads >> gshift;
  float s = 1.f;
  if (amax_word) {
    s = e4m3_row_scale(__uint_as_float(*amax_word));
    if (blockIdx.x == 0 && threadIdx.x == 0) *scale = s;
  }
  for (int64_t row0 = ((int64_t)blockIdx.x * groups_per_block + (threadIdx.x >> gshift)) * RB; row0 < N;
       row0 += (int64_t)gridDim.x * groups_per_block * RB) {
    uint4 d[RB][NU];
#pragma unroll
    for (int r = 0; r < RB; r++)
#pragma unroll
      for (int j = 0; j < NU; j++)
        if (row0 + r < N && gl + j * G < U) d[r][j] = ldg128(x + (row0 + r) * ld + (gl + j * G) * W);
#pragma unroll
    for (int r = 0; r < RB; r++) {
      if (row0 + r >= N) break;
      float f[W];
      if (!amax_word) {
        float m = 0.f;
#pragma unroll
        for (int j = 0; j < NU; j++) {
          if (gl + j * G >= U) continue;
          Vec<T>::unpack(d[r][j], f);
#pragma unroll
          for (int i = 0; i < W; i++) m = amax_nan(m, fabsf(f[i]));
        }
        for (int o = G >> 1; o > 0; o >>= 1) m = amax_nan(m, __shfl_xor_sync(gmask, m, o));
        s = e4m3_row_scale(m);
        if (gl == 0) scale[row0 + r] = s;
      }
#pragma unroll
      for (int j = 0; j < NU; j++) {
        if (gl + j * G >= U) continue;
        Vec<T>::unpack(d[r][j], f);
        store_unit<W>(x8 + (row0 + r) * K + (gl + j * G) * W, f, s);
      }
    }
  }
}

// Per-tensor amax: each thread takes the amax of its units over its rows, a warp reduces, and lane 0 folds it into
// *amax_word (zeroed before the launch) with atomicMax on the bits. |x| has a clear sign bit, so as unsigned integers
// the bits order like the values, with NaN above +inf: the word ends up NaN whenever any element is.
template <typename T, int W>
__global__ void __launch_bounds__(kQuantThreads)
    quantize_fp8_amax_kernel(const T* __restrict__ x, int64_t N, int64_t K, int64_t ld, int gshift,
                             uint32_t* __restrict__ amax_word) {
  const int G = 1 << gshift;
  const int gl = threadIdx.x & (G - 1);
  const int64_t U = K / W;
  const int64_t rows_per_block = kQuantThreads >> gshift;
  float m = 0.f;
  for (int64_t row = (int64_t)blockIdx.x * rows_per_block + (threadIdx.x >> gshift); row < N;
       row += (int64_t)gridDim.x * rows_per_block)
    m = row_amax_part<T, W>(x + row * ld, U, gl, G, m);
  for (int o = 16; o > 0; o >>= 1) m = amax_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax_word, __float_as_uint(m));
}

template <typename T, int NU>
static int quantize_fp8_short_run(const T* x, int64_t N, int64_t K, int64_t ld, int gshift, uint8_t* x8, float* scale,
                                  uint32_t* amax_word, cudaStream_t st) {
  static GridCache grid;
  const int64_t rows_per_block = (int64_t)(kQuantThreads >> gshift) * (4 / NU);
  const int64_t blocks = (N + rows_per_block - 1) / rows_per_block;
  const int g = (int)min(blocks, (int64_t)grid.get((const void*)quantize_fp8_short_kernel<T, NU>, kQuantThreads));
  quantize_fp8_short_kernel<T, NU><<<g, kQuantThreads, 0, st>>>(x, N, K, ld, gshift, x8, scale, amax_word);
  TSB_LAUNCH_CHECK();
  return 0;
}

template <typename T, int W>
static int quantize_fp8_run(const T* x, int64_t N, int64_t K, int64_t ld, uint8_t* x8, float* scale,
                            uint32_t* amax_word, cudaStream_t st) {
  const int64_t U = K / W;
  int gshift = 0;
  while (gshift < 5 && ((int64_t)1 << gshift) < U) gshift++;
  const int64_t rows_per_block = kQuantThreads >> gshift;
  const int64_t blocks = (N + rows_per_block - 1) / rows_per_block;
  if (amax_word) {
    static GridCache grid_amax;
    TSB_CUDA_TRY(cudaMemsetAsync(amax_word, 0, sizeof(uint32_t), st));
    const int g = (int)min(blocks, (int64_t)grid_amax.get((const void*)quantize_fp8_amax_kernel<T, W>, kQuantThreads));
    quantize_fp8_amax_kernel<T, W><<<g, kQuantThreads, 0, st>>>(x, N, K, ld, gshift, amax_word);
    TSB_LAUNCH_CHECK();
  }
  if constexpr (W > 1) {
    if (U <= 128) {
      const int64_t nu = (U + 31) / 32;
      if (nu == 1) return quantize_fp8_short_run<T, 1>(x, N, K, ld, gshift, x8, scale, amax_word, st);
      if (nu == 2) return quantize_fp8_short_run<T, 2>(x, N, K, ld, gshift, x8, scale, amax_word, st);
      return quantize_fp8_short_run<T, 4>(x, N, K, ld, gshift, x8, scale, amax_word, st);
    }
  }
  static GridCache grid_quant;
  const int g = (int)min(blocks, (int64_t)grid_quant.get((const void*)quantize_fp8_kernel<T, W>, kQuantThreads));
  quantize_fp8_kernel<T, W><<<g, kQuantThreads, 0, st>>>(x, N, K, ld, gshift, x8, scale, amax_word);
  TSB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
static int quantize_fp8_impl(const void* x, int64_t N, int64_t K, int64_t ld, void* x8, float* scale,
                             uint32_t* amax_word, cudaStream_t st) {
  if ((uintptr_t)x % sizeof(T)) return TSB200_ERR_UNSUPPORTED;
  constexpr int VEC = Vec<T>::VEC;
  const bool vec = (uintptr_t)x % 16 == 0 && (ld * (int64_t)sizeof(T)) % 16 == 0 &&
                   (K * (int64_t)sizeof(T)) % 16 == 0 && (uintptr_t)x8 % 16 == 0;
  if (vec) return quantize_fp8_run<T, VEC>((const T*)x, N, K, ld, (uint8_t*)x8, scale, amax_word, st);
  return quantize_fp8_run<T, 1>((const T*)x, N, K, ld, (uint8_t*)x8, scale, amax_word, st);
}

}  // namespace tsb

using namespace tsb;

extern "C" int tsb200_quantize_fp8(const void* x, int64_t N, int64_t K, int64_t ld, int dtype, int per_row, void* x8,
                                   float* scale, void* workspace, size_t workspace_bytes, void* stream) {
  if (N < 0 || K < 0 || ld < K || (per_row != 0 && per_row != 1)) return TSB200_ERR_INVALID_ARG;
  if (dtype != TSB200_F32 && dtype != TSB200_F16 && dtype != TSB200_BF16) return TSB200_ERR_UNSUPPORTED;
  if (K == 0 || (!per_row && N == 0)) return TSB200_ERR_INVALID_ARG;  // the amax of no elements
  if (N == 0) return 0;
  if (!x || !x8 || !scale) return TSB200_ERR_INVALID_ARG;
  if (K >= ((int64_t)1 << 31) || ((uintptr_t)scale & 3)) return TSB200_ERR_UNSUPPORTED;
  uint32_t* amax_word = nullptr;
  if (!per_row) {
    if (!workspace || workspace_bytes < sizeof(uint32_t)) return TSB200_ERR_WORKSPACE;
    if ((uintptr_t)workspace & 3) return TSB200_ERR_UNSUPPORTED;
    amax_word = (uint32_t*)workspace;
  }
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case TSB200_F32: return quantize_fp8_impl<float>(x, N, K, ld, x8, scale, amax_word, st);
    case TSB200_F16: return quantize_fp8_impl<__half>(x, N, K, ld, x8, scale, amax_word, st);
    case TSB200_BF16: return quantize_fp8_impl<__nv_bfloat16>(x, N, K, ld, x8, scale, amax_word, st);
  }
  return TSB200_ERR_UNSUPPORTED;
}
