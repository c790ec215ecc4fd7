// spspmm.cu — CSR x CSR -> CSR/COO sparse-sparse matmul for sm_90a.
//
// Replaces spspmm_sum -> torch.sparse.mm (torch_sparse/matmul.py:94-111; CPU: ATen sparse_matmul,
// CUDA: cuSPARSE SpGEMM), keeping its observable contract: output sorted by (row, col), unique,
// structural (numerical zeros are kept).
//
// Two-phase row-wise Gustavson with a per-CTA shared-memory BITMAP accumulator:
//   * a CTA owns one output row at a time (rows are handed out one per ticket from a global atomic
//     counter; the next row's ticket is taken while the current row runs and its A-row metadata is
//     prefetched, so the dependent global loads rowptr_a -> col_a -> rowptr_b of row r+1 overlap the work of row r);
//   * every product a_ik * b_kj sets bit j of a bitmap over a window of <= 2^18 columns (32 KB, XOR-swizzled
//     so that a thread can scan "its" 32 words with conflict-free LDS.128);
//   * one dense pass turns the bitmap into ranks (thread t owns words [32t, 32t+32): 8 x LDS.128 + popc,
//     one block scan): rank of column j = group prefix + popc(bits below j) => the output row comes out
//     ALREADY SORTED by column with no per-row sort and no hash probing;
//   * FLAT rows (single window, <= 128 A entries, <= 2048 products; every row of BASELINE's C4): the row's
//     products are numbered 0..P-1 through a prefix sum of the B-row lengths and dealt to the threads
//     (chunks of 32 round-robin over the warps, <= 8 products per thread), which keep them in REGISTERS across the passes, so B is read once per phase and every lane
//     is busy whatever the B-row lengths are. Bits are set with plain LDS/STS (a scattered warp-wide
//     shared-memory ATOMS.OR is serialised lane by lane);
//     two writers racing on one WORD can lose a bit, so after a barrier every product checks its own bit
//     and repairs a loss with an atomicOr (atomics only add bits, so the repair pass is race-free and only
//     the rare losers pay). The output row is staged in shared memory -- one word per slot carries the
//     column and the id of the product that wrote it last (= the slot's owner, which stores its value; the
//     rare other products of that column add theirs after a barrier) -- and leaves the SM as fully
//     coalesced streaming stores of row / col / val;
//   * other rows (GENERAL path) re-walk their products per pass (warp per A entry, lanes striding the B
//     row), window by window for matrices wider than one window (B rows are column-sorted, so only windows
//     between the row's smallest and largest product column are visited); bits via atomicOr, whose return
//     value tells the product whether it was the first on its column (the symbolic pass just counts those),
//     values with L2 atomics straight into val_c.
// Everything is HBM-bound on the 16+s bytes per output nonzero that must be written.
#include <cub/cub.cuh>

#include "common.cuh"

namespace tsb {

constexpr int kSpThreads = 256;
constexpr int kSpWarps = kSpThreads / 32;
constexpr int kFlatU = 8;                         // products per thread on the flat path
constexpr int kStageCap = kFlatU * kSpThreads;    // output entries staged in shared memory per row (2048)
constexpr int kMaxWindowLog2 = 18;
constexpr int kMaxWindowBits = 1 << kMaxWindowLog2;
constexpr int kClaimSlot = 3;                     // single-pass mode: schedule slot of the next row's ticket (SpNext)
constexpr int kABatch = 128;                      // A entries staged per batch
static_assert(kStageCap <= (1 << (32 - kMaxWindowLog2 - 1)), "owner id and column share one 32-bit word");

struct SpParams {
  const int64_t* rowptr_a; const int64_t* col_a; const void* val_a;
  const int64_t* rowptr_b; const int64_t* col_b; const void* val_b;
  int64_t M, N;
  int64_t* counts;          // symbolic: per-row nnz (accumulated at rowptr_c + 1, pre-zeroed)
  const int64_t* rowptr_c;  // numeric
  int64_t* row_c; int64_t* col_c; void* val_c;
  unsigned int* counter;
  unsigned long long* status;  // FUSED: per-row look-back words (zeroed by the host)
  int64_t capacity;            // FUSED: entries the output arrays can hold
  int* overflow;               // FUSED: set when a row would not fit
  // FUSED: kClaimSlot, read at run time: compiled in as a constant it made the C4 single pass take 8.4-8.7 ms instead
  // of 7.1-7.2 ms (one H100 80GB HBM3 at a 700 W power limit), although ptxas then reports no spills
  int claim_slot;
  int window_bits;  // power of two, 1024 .. 2^18
  int log2_wpt;     // log2(bitmap words per scan chunk), 2..5; chunks = (window_bits/32) >> log2_wpt <= 256
};

// bitmap word -> shared-memory word: XOR swizzle of the 16-byte group index inside each 32-word block with the
// block index, so that thread t reading group g of block t (chunk scans) is conflict-free without padding
__device__ __forceinline__ uint32_t sp_phys(uint32_t w) { return w ^ (((w >> 5) & 7u) << 2); }

__device__ __forceinline__ int popc4(const uint4 q) { return __popc(q.x) + __popc(q.y) + __popc(q.z) + __popc(q.w); }

// plain (non-atomic) bit set + repair, see the header comment
__device__ __forceinline__ void sp_mark(uint32_t* bitmap, uint32_t c0) {
  volatile uint32_t* a = bitmap + sp_phys(c0 >> 5);
  const uint32_t old = *a;
  *a = old | (1u << (c0 & 31u));
}
__device__ __forceinline__ void sp_verify(uint32_t* bitmap, uint32_t c0) {
  uint32_t* a = bitmap + sp_phys(c0 >> 5);
  const uint32_t bit = 1u << (c0 & 31u);
  if (!(*(volatile uint32_t*)a & bit)) atomicOr(a, bit);
}

// Rank (position in the sorted output row of this window) of window-relative column c0.
// ABS: pre4 holds absolute 16-bit prefixes (flat rows, <= 2048 outputs); otherwise chunk-relative + tbase.
template <bool ABS>
__device__ __forceinline__ uint32_t sp_rank(const uint32_t* bitmap, const uint16_t* pre4, const uint32_t* tbase,
                                            int lw, uint32_t c0) {
  const uint32_t w = c0 >> 5, g = w >> 2, k = w & 3u;
  const uint4 q = *reinterpret_cast<const uint4*>(&bitmap[sp_phys(g << 2)]);
  uint32_t below = 0, word = q.x;
  if (k > 0) { below += __popc(q.x); word = q.y; }
  if (k > 1) { below += __popc(q.y); word = q.z; }
  if (k > 2) { below += __popc(q.z); word = q.w; }
  uint32_t r = pre4[g] + below + __popc(word & ((1u << (c0 & 31u)) - 1u));
  if (!ABS) r += tbase[w >> lw];
  return r;
}

// Block-wide exclusive scan of one int per thread, ONE barrier; `total` = sum over the CTA.
__device__ __forceinline__ int sp_block_scan(int v, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, x, off);
    if (lane >= off) x += t;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  int woff = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kSpWarps; w++) {
    const int t = s_warp[w];
    if (w < warp) woff += t;
    total += t;
  }
  return woff + x - v;
}

// Dense rank pass, thread t owns chunk t (2^lw words = 2^(lw-2) groups of 4 words).
// ABS: every chunk is read, pre4 = absolute prefix per group (16 bit). Otherwise: only chunks whose touch flag
// is set are read, pre4 = prefix inside the chunk, tbase = exclusive prefix of the chunk.
// Returns the number of set bits. One barrier inside; the caller must barrier before sp_rank().
template <bool ABS>
__device__ __forceinline__ int sp_scan(const uint32_t* bitmap, uint16_t* pre4, uint32_t* tbase,
                                       const unsigned char* tflag, int lw, uint32_t nch, int* s_warp) {
  const int tid = threadIdx.x;
  const bool mine = (uint32_t)tid < nch && (ABS || tflag[tid]);
  const uint32_t w0 = mine ? (uint32_t)tid << lw : 0u;
  int total;
  if (lw == 5) {
    int c[8];
    int run = 0;
#pragma unroll
    for (int g = 0; g < 8; g++) {
      c[g] = mine ? popc4(*reinterpret_cast<const uint4*>(&bitmap[sp_phys(w0 + 4 * g)])) : 0;
      run += c[g];
    }
    const int base = sp_block_scan(run, s_warp, total);
    if (mine) {
      int r = ABS ? base : 0;
      uint32_t pk[4];
#pragma unroll
      for (int g = 0; g < 8; g += 2) {
        pk[g >> 1] = (uint32_t)r | ((uint32_t)(r + c[g]) << 16);
        r += c[g] + c[g + 1];
      }
      *reinterpret_cast<uint4*>(pre4 + (w0 >> 2)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
    if (!ABS && (uint32_t)tid < nch) tbase[tid] = (uint32_t)base;
  } else {
    const int ng = 1 << (lw - 2);
    int run = 0;
    if (mine)
      for (int g = 0; g < ng; g++) run += popc4(*reinterpret_cast<const uint4*>(&bitmap[sp_phys(w0 + 4 * g)]));
    const int base = sp_block_scan(run, s_warp, total);
    if (mine) {
      int r = ABS ? base : 0;
      for (int g = 0; g < ng; g++) {
        pre4[(w0 >> 2) + g] = (uint16_t)r;
        r += popc4(*reinterpret_cast<const uint4*>(&bitmap[sp_phys(w0 + 4 * g)]));
      }
    }
    if (!ABS && (uint32_t)tid < nch) tbase[tid] = (uint32_t)base;
  }
  return total;
}

// count the set bits of (and clear) the chunk this thread owns
__device__ __forceinline__ int sp_count_clear_chunk(uint32_t* bitmap, int lw) {
  const uint32_t w0 = (uint32_t)threadIdx.x << lw;
  const int ng = 1 << (lw - 2);
  int cnt = 0;
  if (lw == 5) {
#pragma unroll
    for (int g = 0; g < 8; g++) {
      uint4* qp = reinterpret_cast<uint4*>(&bitmap[sp_phys(w0 + 4 * g)]);
      cnt += popc4(*qp);
      *qp = make_uint4(0, 0, 0, 0);
    }
  } else {
    for (int g = 0; g < ng; g++) {
      uint4* qp = reinterpret_cast<uint4*>(&bitmap[sp_phys(w0 + 4 * g)]);
      cnt += popc4(*qp);
      *qp = make_uint4(0, 0, 0, 0);
    }
  }
  return cnt;
}

enum { SP_SYM = 0, SP_NUM = 1, SP_FUSED = 2 };

// ---- single-pass (FUSED) mode: per-row status words for the decoupled look-back ----------------------------
// status[i] = flag << 62 | value:  flag 0 = row not counted yet, 1 = value is the row's nnz (aggregate),
// 2 = value is the inclusive prefix (nnz of rows 0..i). One 64-bit word per row, written/read with relaxed
// gpu-scope accesses: flag and value travel in one word, and no other data is exchanged between CTAs.
constexpr unsigned long long kStAgg = 1ull << 62, kStPrefix = 2ull << 62, kStMask = (1ull << 62) - 1;

__device__ __forceinline__ unsigned long long sp_ld_status(const unsigned long long* q) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(q) : "memory");
  return v;
}
__device__ __forceinline__ void sp_st_status(unsigned long long* q, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(q), "l"(v) : "memory");
}

// One warp: number of output entries of all rows < i. Lane l inspects row j - l; a row that has published its
// inclusive prefix ends the walk. Rows are claimed in increasing order by CTAs that are running, and a row's
// aggregate depends on no other row, so every predecessor's status eventually becomes non-zero.
__device__ __forceinline__ int64_t sp_lookback(const unsigned long long* status, int64_t i, int lane) {
  int64_t excl = 0;
  for (int64_t j = i - 1; j >= 0; j -= 32) {
    const int64_t r = j - lane;
    unsigned long long st = kStPrefix;  // rows before row 0: inclusive prefix 0
    if (r >= 0) {
      st = sp_ld_status(status + r);
      while ((st >> 62) == 0) {
        __nanosleep(40);
        st = sp_ld_status(status + r);
      }
    }
    const unsigned pm = __ballot_sync(0xffffffffu, (st >> 62) == 2);
    long long v = (long long)(st & kStMask);
    if (pm && lane > __ffs(pm) - 1) v = 0;  // rows older than the nearest published prefix are inside it
#pragma unroll
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    excl += v;
    if (pm) break;
  }
  return excl;
}

// Single pass, warp 0 of a row with n > 0 output entries: finds the row's start by look-back, publishes its inclusive
// prefix and leaves the start in s_base, or -1 when the row does not fit into `capacity` (then the overflow flag is set
// and nothing of the row may be written; cannot happen with capacity >= the number of products).
__device__ __forceinline__ void sp_place(const SpParams& p, int64_t i, int64_t n, int lane, long long& s_base) {
  const int64_t base = sp_lookback(p.status, i, lane);
  if (lane == 0) {
    sp_st_status(p.status + i, kStPrefix | (unsigned long long)(base + n));
    const bool fits = base + n <= p.capacity;
    if (!fits) *p.overflow = 1;
    s_base = fits ? base : -1;
  }
}

__device__ __forceinline__ int sp_warp_sum(int v) {
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// symbolic: add the columns this warp's threads were first on to counts[i]
__device__ __forceinline__ void sp_store_count(const SpParams& p, int64_t i, int cnt) {
  cnt = sp_warp_sum(cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + i), (unsigned long long)cnt);
}

// The next row's A-row metadata, prefetched while the current row runs: B-row start, length and a_ik of A entry tid
template <typename T>
struct SpPrefetch {
  bool valid;
  int64_t bs;
  int len;
  T av;
};

// The next row, one row ahead: ticket taken at slot slot0 of the current row, read after the next barrier, then its loads
// rowptr_a -> col_a -> rowptr_b / val_a at the two slots after. Slot 0 = row start; in single-pass mode a later slot
// shortens the time from ticket to published nnz, which the rows behind the next row wait for.
template <bool NUMERIC, typename T>
struct SpNext {
  const SpParams& p;
  int slot0;              // the slot at which the next row's ticket is taken
  unsigned int* s_claim;  // row tickets: s_claim[par] the row being processed, s_claim[par ^ 1] the next one
  int par;
  SpPrefetch<T>& pf;
  int64_t row, s = 0, e = 0;  // the next row and its A-row extent
  bool do_pf = false;     // the next row is one A batch: its metadata is prefetched
  int64_t k = -1;         // column of the next row's A entry tid (-1: none)
  int stage = 0;          // 0 nothing yet, 1 ticket taken, 2 row known, 3 its col_a issued, 4 its rowptr_b issued

  __device__ __forceinline__ SpNext(const SpParams& p, int slot0, unsigned int* s_claim, int par, SpPrefetch<T>& pf)
      : p(p), slot0(slot0), s_claim(s_claim), par(par), pf(pf), row(p.M) {}
  __device__ __forceinline__ void take() {
    if (threadIdx.x == 0) s_claim[par ^ 1] = atomicAdd(p.counter, 1u);
    stage = 1;
  }
  __device__ __forceinline__ void read() {
    row = s_claim[par ^ 1];
    if (row < p.M) { s = p.rowptr_a[row]; e = p.rowptr_a[row + 1]; }
    stage = 2;
  }
  // the step due at slot `slot` of the current row
  __device__ __forceinline__ void at(int slot) {
    const int tid = threadIdx.x;
    if (stage == 0 && slot0 <= slot) {
      take();
    } else if (stage == 1) {
      read();
    } else if (stage == 2) {
      const int64_t nn = e - s;
      if (nn > 0 && nn <= kABatch) {
        do_pf = true;
        if (tid < nn) k = p.col_a[s + tid];
      }
      stage = 3;
    } else if (stage == 3) {
      if (do_pf) {
        if (k >= 0) {
          const T* va = reinterpret_cast<const T*>(p.val_a);
          pf.bs = p.rowptr_b[k];
          pf.len = (int)(p.rowptr_b[k + 1] - pf.bs);
          pf.av = (NUMERIC && va) ? va[s + tid] : (T)1;
        }
        pf.valid = true;
      }
      stage = 4;
    }
  }
  // what the current row's path did not reach: ticket and row extent are needed, the prefetch is not (see staging)
  __device__ __forceinline__ void finish() {
    if (stage == 0) take();
    if (stage == 1) {
      __syncthreads();
      read();
    }
  }
};

// The products of A row [a_s, a_e) on the general path. Its A entries are staged kABatch at a time in s_bs / s_len /
// s_av (a row of one batch was staged at its start); one warp per A entry, lanes striding its B row.
template <bool NUMERIC, typename T>
struct SpWalk {
  const SpParams& p;
  int64_t a_s, a_e;
  bool single_batch;
  int64_t* s_bs;
  int* s_len;
  T* s_av;
  uint64_t pol_b;

  // body(c, c0 = c - wlo, A entry in the staged batch, index into B) for every product with column c in [wlo, whi)
  template <typename Body>
  __device__ __forceinline__ void operator()(int64_t wlo, int64_t whi, Body&& body) const {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const T* va = reinterpret_cast<const T*>(p.val_a);
    for (int64_t ab = a_s; ab < a_e; ab += kABatch) {
      const int na = (int)min((int64_t)kABatch, a_e - ab);
      if (!single_batch) {
        __syncthreads();
        if (tid < na) {
          const int64_t k = p.col_a[ab + tid];
          const int64_t kb = p.rowptr_b[k];
          s_bs[tid] = kb;
          s_len[tid] = (int)(p.rowptr_b[k + 1] - kb);
          if (NUMERIC) s_av[tid] = va ? va[ab + tid] : (T)1;
        }
        __syncthreads();
      }
      for (int e = warp; e < na; e += kSpWarps) {
        const int64_t ebs = s_bs[e];
        const int elen = s_len[e];
        for (int f = lane; f < elen; f += 32) {
          const int64_t c = (int64_t)ldg64_hint(p.col_b + ebs + f, pol_b);
          if (c >= wlo && c < whi) body(c, (uint32_t)(c - wlo), e, ebs + f);
        }
      }
    }
  }
};

// Counting pass over the windows [win_lo, win_hi] (the whole job of the symbolic kernel; in single-pass mode it gives
// the row's nnz before anything is written): every product marks its column with atomicOr, whose return value tells it
// whether it was first. Returns the number of columns this thread was first on; the touched chunks are cleared again.
template <bool NUMERIC, typename T>
__device__ __forceinline__ int sp_count_pass(const SpWalk<NUMERIC, T>& walk, int64_t win_lo, int64_t win_hi,
                                             int64_t W, uint32_t* bitmap, unsigned char* tflag, int lw, uint32_t nch) {
  const int tid = threadIdx.x;
  int cnt = 0;
  for (int64_t win = win_lo; win <= win_hi; win++) {
    const int64_t wlo = win * W;
    walk(wlo, wlo + W, [&](int64_t, uint32_t c0, int, int64_t) {
      const uint32_t bit = 1u << (c0 & 31u);
      const uint32_t old = atomicOr(&bitmap[sp_phys(c0 >> 5)], bit);
      if (!(old & bit)) cnt++;
      tflag[c0 >> (5 + lw)] = 1;
    });
    __syncthreads();
    if ((uint32_t)tid < nch && tflag[tid]) {
      sp_count_clear_chunk(bitmap, lw);
      tflag[tid] = 0;
    }
    __syncthreads();
  }
  return cnt;
}

template <int MODE, typename T>
__global__ void __launch_bounds__(kSpThreads, MODE == SP_SYM ? 5 : (sizeof(T) == 8 ? 3 : 4)) spspmm_kernel(const SpParams p) {
  constexpr bool NUMERIC = MODE != SP_SYM;
  constexpr bool FUSED = MODE == SP_FUSED;
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t WW = (uint32_t)p.window_bits >> 5;   // bitmap words (>= 32)
  const int lw = p.log2_wpt;
  const uint32_t NCH = WW >> lw;                        // scan chunks (<= 256)
  uint32_t* bitmap = reinterpret_cast<uint32_t*>(smem);
  uint16_t* pre4 = reinterpret_cast<uint16_t*>(bitmap + WW);        // NUMERIC: WW/4 entries
  uint32_t* scol = reinterpret_cast<uint32_t*>(pre4 + (WW >> 2));   // NUMERIC: kStageCap entries
  T* acc = reinterpret_cast<T*>(scol + kStageCap);                  // NUMERIC: kStageCap entries (flat path)
  uint32_t* tbase = reinterpret_cast<uint32_t*>(acc);               // NUMERIC: 256 entries (general path, aliases acc)
  __shared__ int s_warp[kSpWarps];
  __shared__ unsigned int s_claim[2];               // row tickets: the row being processed / the next one
  __shared__ long long s_min, s_max, s_base;
  __shared__ int s_total;
  __shared__ int64_t s_bs[kABatch];
  __shared__ int s_len[kABatch];
  __shared__ int2 s_se[kABatch];                    // flat path: [first, last+1) product number of each A entry
  __shared__ unsigned char s_ent[kStageCap / 32];  // flat path: A entry that owns product 32*k
  __shared__ T s_av[NUMERIC ? kABatch : 1];
  __shared__ unsigned char tflag[kSpThreads];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t q = tid; q < WW; q += kSpThreads) bitmap[q] = 0;
  tflag[tid] = 0;
  if (tid == 0) s_claim[0] = atomicAdd(p.counter, 1u);

  const T* va = reinterpret_cast<const T*>(p.val_a);
  const T* vb = reinterpret_cast<const T*>(p.val_b);
  const int64_t W = p.window_bits;
  const bool multi_window = p.N > W;
  const bool has_val = NUMERIC && p.val_c != nullptr;
  T* val_c = reinterpret_cast<T*>(p.val_c);
  // B is re-read nnz(A)/Kd times while 20 bytes per output nonzero stream through L2: keep B's lines (evict_last)
  const uint64_t pol_b = make_policy_evict_last();

  SpPrefetch<T> pf{false, 0, 0, (T)1};

  __syncthreads();
  int par = 0;
  int64_t i = s_claim[0];
  int64_t a_s = 0, a_e = 0;
  if (i < p.M) { a_s = p.rowptr_a[i]; a_e = p.rowptr_a[i + 1]; }

  while (i < p.M) {
    const int64_t n_a = a_e - a_s;
    SpNext<NUMERIC, T> nx(p, FUSED ? p.claim_slot : 0, s_claim, par, pf);
    do {  // one row; `break` = done with it
      if (n_a <= 0) {  // empty row: counts[i] stays 0 (pre-zeroed) / status = aggregate 0; no output
        if (FUSED && tid == 0) sp_st_status(p.status + i, kStAgg);
        pf.valid = false;
        break;
      }
      nx.at(0);
      const int na0 = (int)min(n_a, (int64_t)kABatch);

      // ---- stage the (first batch of the) A-row metadata: start/length of each B row, a_ik; number the products ----
      int64_t bs = 0;
      int len = 0;
      T av = (T)1;
      if (pf.valid) { bs = pf.bs; len = pf.len; av = pf.av; }
      else if (tid < na0) {
        const int64_t k = p.col_a[a_s + tid];
        bs = p.rowptr_b[k];
        len = (int)(p.rowptr_b[k + 1] - bs);
        if (NUMERIC && va) av = va[a_s + tid];
      }
      if (tid >= na0) len = 0;
      if (tid < na0) {
        s_bs[tid] = bs;
        s_len[tid] = len;
        if (NUMERIC) s_av[tid] = av;
      }
      const int len_c = min(len, kStageCap + 1);  // keeps the sum in range; any clamped length disables the flat path
      int P;
      const int excl = sp_block_scan(len_c, s_warp, P);
      nx.at(1);  // (slot 0 ticket: the barrier inside the scan made it visible; the two rowptr_a loads are in flight)
      if (tid < na0) {
        s_se[tid] = make_int2(excl, excl + len_c);
        // the 32-aligned product numbers inside [excl, excl + len): this entry is where their chunk starts
        if (P <= kStageCap)
          for (int k = (excl + 31) >> 5; (k << 5) < excl + len_c; k++) s_ent[k] = (unsigned char)tid;
      }
      pf.valid = false;
      __syncthreads();  // s_bs / s_len / s_se / s_ent / s_av visible

      const bool flat = !multi_window && n_a <= kABatch && P <= kStageCap;
      if (flat) {
        // ================= flat row: products 0..P-1 dealt to the threads, kept in registers =================
        // product q lives in chunk q >> 5; chunk c is handled by warp c % 8 as its slot c / 8 (balanced to one chunk)
        uint32_t cc[kFlatU];  // window-relative column (18 bit) | rank << 18 once known; ~0 = no product
        T pv[kFlatU];
#pragma unroll
        for (int u = 0; u < kFlatU; u++) {
          cc[u] = 0xffffffffu;
          pv[u] = (T)0;
          const int q = ((warp + kSpWarps * u) << 5) + lane;
          if (((warp + kSpWarps * u) << 5) < P) {   // warp-uniform
            if (q < P) {
              int e = s_ent[warp + kSpWarps * u];
              int2 se = s_se[e];
              while (q >= se.y) se = s_se[++e];
              const int64_t idx = s_bs[e] + (q - se.x);
              cc[u] = (uint32_t)ldg64_hint(p.col_b + idx, pol_b);
              if (has_val) pv[u] = s_av[e] * (vb ? ldg_hint(vb + idx, pol_b) : (T)1);
            }
          }
        }
        nx.at(2);
#pragma unroll
        for (int u = 0; u < kFlatU; u++)
          if (cc[u] != 0xffffffffu) sp_mark(bitmap, cc[u]);
        __syncthreads();
        nx.at(3);
#pragma unroll
        for (int u = 0; u < kFlatU; u++)
          if (cc[u] != 0xffffffffu) sp_verify(bitmap, cc[u]);
        __syncthreads();
        nx.at(4);
        if (!NUMERIC) {
          sp_store_count(p, i, (uint32_t)tid < NCH ? sp_count_clear_chunk(bitmap, lw) : 0);
          break;  // the next row's staging barriers order the clears before its marks
        }
        const int wc = sp_scan<true>(bitmap, pre4, tbase, tflag, lw, NCH, s_warp);
        // single pass: the row's nnz is known now -> publish it, so that later rows can add it up while this
        // row is still ranking its products
        if (FUSED && tid == 0) sp_st_status(p.status + i, kStAgg | (unsigned long long)wc);
        __syncthreads();
        nx.at(5);
        // rank; every product writes (its id, its column) into the slot: the last writer owns the slot
#pragma unroll
        for (int u = 0; u < kFlatU; u++) {
          if (cc[u] != 0xffffffffu) {
            const uint32_t r = sp_rank<true>(bitmap, pre4, tbase, lw, cc[u]);
            const uint32_t q = (uint32_t)(((warp + kSpWarps * u) << 5) + lane);
            scol[r] = (q << kMaxWindowLog2) | cc[u];
            cc[u] |= r << kMaxWindowLog2;
          }
        }
        __syncthreads();
        nx.at(6);
        uint32_t dmask = 0;
        if (has_val) {
#pragma unroll
          for (int u = 0; u < kFlatU; u++) {
            if (cc[u] != 0xffffffffu) {
              const uint32_t r = cc[u] >> kMaxWindowLog2;
              const uint32_t q = (uint32_t)(((warp + kSpWarps * u) << 5) + lane);
              // + 0: the sum starts at +0 (as torch.sparse.mm's does), so an all -0 column stores +0
              if ((scol[r] >> kMaxWindowLog2) == q) acc[r] = pv[u] + (T)0;
              else dmask |= 1u << u;
            }
          }
        }
        if (FUSED && warp == 0 && wc > 0) sp_place(p, i, wc, lane, s_base);
        if (__syncthreads_or(dmask != 0)) {
#pragma unroll
          for (int u = 0; u < kFlatU; u++)
            if (dmask & (1u << u)) atomicAdd(&acc[cc[u] >> kMaxWindowLog2], pv[u]);
          __syncthreads();
        }
        nx.at(7);
        const int64_t ob = FUSED ? s_base : p.rowptr_c[i];
        const int nw = (FUSED && ob < 0) ? 0 : wc;  // a row that does not fit writes nothing
        for (int q = tid; q < nw; q += kSpThreads) {
          __stcs(p.col_c + ob + q, (int64_t)(scol[q] & (uint32_t)(kMaxWindowBits - 1)));
          if (p.row_c) __stcs(p.row_c + ob + q, i);
          if (has_val) __stcs(val_c + ob + q, acc[q]);
        }
#pragma unroll
        for (int u = 0; u < kFlatU; u++)
          if (cc[u] != 0xffffffffu) bitmap[sp_phys((cc[u] & (uint32_t)(kMaxWindowBits - 1)) >> 5)] = 0;
        break;  // the next row's staging barriers order the clears / staging reads before its writes
      }

      // ================= general row: products re-walked per pass, window by window =================
      nx.at(2);
      int64_t win_lo = 0, win_hi = 0;  // window index range [win_lo, win_hi]
      if (multi_window) {
        // B rows are column-sorted (SparseStorage invariant): first/last entry bound the row's columns
        if (tid == 0) { s_min = 0x7fffffffffffffffLL; s_max = -1; }
        __syncthreads();
        long long mn = 0x7fffffffffffffffLL, mx = -1;
        for (int64_t a = a_s + tid; a < a_e; a += kSpThreads) {
          const int64_t k = p.col_a[a];
          const int64_t kb = p.rowptr_b[k], ke = p.rowptr_b[k + 1];
          if (ke > kb) {
            mn = min(mn, (long long)p.col_b[kb]);
            mx = max(mx, (long long)p.col_b[ke - 1]);
          }
        }
        if (mx >= 0) { atomicMin(&s_min, mn); atomicMax(&s_max, mx); }
        __syncthreads();
        if (s_max < 0) { win_lo = 1; win_hi = 0; }
        else { win_lo = s_min / W; win_hi = s_max / W; }
        __syncthreads();
      }
      const SpWalk<NUMERIC, T> walk{p, a_s, a_e, n_a <= kABatch, s_bs, s_len, s_av, pol_b};
      int64_t done = 0;  // nnz of this row emitted by previous windows
      int64_t out0 = 0;
      if (MODE == SP_NUM) out0 = p.rowptr_c[i];

      if (!NUMERIC) {
        sp_store_count(p, i, sp_count_pass(walk, win_lo, win_hi, W, bitmap, tflag, lw, NCH));
        nx.at(3);
        break;
      }
      bool skip_row = false;
      if (FUSED) {
        if (tid == 0) s_total = 0;
        __syncthreads();
        const int cnt = sp_warp_sum(sp_count_pass(walk, win_lo, win_hi, W, bitmap, tflag, lw, NCH));
        if (lane == 0 && cnt) atomicAdd(&s_total, cnt);
        __syncthreads();
        const int total = s_total;
        if (warp == 0) {
          if (lane == 0) sp_st_status(p.status + i, kStAgg | (unsigned long long)total);
          if (total > 0) sp_place(p, i, total, lane, s_base);
        }
        __syncthreads();
        out0 = s_base;
        skip_row = total == 0 || out0 < 0;
      }
      if (!skip_row) {
        for (int64_t win = win_lo; win <= win_hi; win++) {
          const int64_t wlo = win * W, whi = wlo + W;
          // ---- mark ----
          walk(wlo, whi, [&](int64_t, uint32_t c0, int, int64_t) {
            atomicOr(&bitmap[sp_phys(c0 >> 5)], 1u << (c0 & 31u));
            tflag[c0 >> (5 + lw)] = 1;
          });
          __syncthreads();
          const int wc = sp_scan<false>(bitmap, pre4, tbase, tflag, lw, NCH, s_warp);
          const int64_t ob = out0 + done;
          const bool staged = wc <= kStageCap;  // columns staged in shared memory -> coalesced stores
          if (has_val)
            for (int q = tid; q < wc; q += kSpThreads) val_c[ob + q] = (T)0;
          __syncthreads();
          // ---- rank every product: column (same-value races are benign), value via L2 atomics ----
          walk(wlo, whi, [&](int64_t c, uint32_t c0, int e, int64_t b) {
            const uint32_t r = sp_rank<false>(bitmap, pre4, tbase, lw, c0);
            if (staged) {
              scol[r] = c0;
            } else {
              p.col_c[ob + r] = c;
              if (p.row_c) p.row_c[ob + r] = i;
            }
            if (has_val) atomicAdd(val_c + ob + r, s_av[e] * (vb ? ldg_hint(vb + b, pol_b) : (T)1));
          });
          __syncthreads();
          if (staged) {
            for (int q = tid; q < wc; q += kSpThreads) {
              __stcs(p.col_c + ob + q, wlo + (int64_t)scol[q]);
              if (p.row_c) __stcs(p.row_c + ob + q, i);
            }
          }
          // ---- clear touched chunks ----
          if ((uint32_t)tid < NCH && tflag[tid]) {
            sp_count_clear_chunk(bitmap, lw);
            tflag[tid] = 0;
          }
          done += wc;
          __syncthreads();
        }
      }
      nx.at(3);
    } while (false);
    nx.finish();
    i = nx.row;
    a_s = nx.s;
    a_e = nx.e;
    par ^= 1;
  }
}

// FUSED mode epilogue: rowptr_c from the per-row status words. Rows with output carry their inclusive prefix; rows
// without (aggregate 0) inherit the prefix of the nearest earlier row with output = a running maximum.
__global__ void sp_status_value_kernel(const unsigned long long* __restrict__ status, int64_t M, int64_t* __restrict__ v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += stride) {
    const unsigned long long st = status[i];
    v[i] = ((st >> 62) == 2) ? (int64_t)(st & kStMask) : 0;
  }
}

// sum over the entries of A of the length of the B row they select = number of products = upper bound of nnz(C)
__global__ void __launch_bounds__(256) sp_bound_kernel(const int64_t* __restrict__ col_a, int64_t nnz_a,
                                                       const int64_t* __restrict__ rowptr_b,
                                                       unsigned long long* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long s = 0;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz_a; e += stride) {
    const int64_t k = col_a[e];
    s += (unsigned long long)(rowptr_b[k + 1] - rowptr_b[k]);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// nnz(C) = rowptr_c[M], or -1 when the single pass raised `overflow` (a row did not fit into the caller's arrays;
// nothing was written past them)
__global__ void sp_finish_kernel(const int64_t* rowptr_c, int64_t M, const int* overflow, int64_t* nnz_dev) {
  *nnz_dev = (overflow && *overflow) ? (int64_t)-1 : rowptr_c[M];
}

static int window_bits_for(int64_t N) {
  int64_t w = 1024;
  while (w < N && w < kMaxWindowBits) w <<= 1;
  return (int)w;
}
static int log2_wpt_for(int window_bits) {
  int wpt = (window_bits >> 5) / kSpThreads;  // words per thread when every thread owns one chunk
  if (wpt < 4) wpt = 4;
  int lw = 2;
  while ((1 << lw) < wpt) lw++;
  return lw;  // 2..5 for windows up to 2^18
}
static size_t sp_smem_bytes(int window_bits, bool numeric, size_t elem) {
  const size_t WW = (size_t)window_bits >> 5;
  size_t b = WW * 4;
  if (numeric) b += WW / 4 * 2 + (size_t)kStageCap * 4 + (size_t)kStageCap * elem;  // acc also hosts tbase (1 KB)
  return b;
}

struct SpLayout {
  // the scalar block at `scalars`: row ticket (uint32), nnz(C) (int64), product bound (int64), overflow flag (int32)
  static constexpr size_t kTicket = 0, kNnz = 16, kBound = 32, kOverflow = 48, kScalarBytes = 256;
  size_t scalars, status, cub, total, cub_bytes;
};
static SpLayout sp_layout(int64_t M) {
  SpLayout L;
  size_t off = 0;
  L.scalars = off; off += SpLayout::kScalarBytes;
  L.status = off; off += align_up((size_t)(M > 0 ? M : 1) * 8, 256);
  size_t tb = 0, tb2 = 0;
  cub::DeviceScan::InclusiveSum(nullptr, tb, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(M > 0 ? M : 1),
                                (cudaStream_t)0);
  cub::DeviceScan::InclusiveScan(nullptr, tb2, (const int64_t*)nullptr, (int64_t*)nullptr, cub::Max(),
                                 (int)(M > 0 ? M : 1), (cudaStream_t)0);
  L.cub_bytes = tb > tb2 ? tb : tb2;
  L.cub = off; off += align_up(L.cub_bytes, 256);
  L.total = off;
  return L;
}

// what every kernel mode reads: the operands, the row ticket, the window and the scan-chunk width
static SpParams sp_bind(const int64_t* rowptr_a, const int64_t* col_a, const void* val_a, const int64_t* rowptr_b,
                        const int64_t* col_b, const void* val_b, int64_t M, int64_t N, char* scalars) {
  SpParams p{};
  p.rowptr_a = rowptr_a; p.col_a = col_a; p.val_a = val_a;
  p.rowptr_b = rowptr_b; p.col_b = col_b; p.val_b = val_b;
  p.M = M; p.N = N;
  p.counter = (unsigned int*)(scalars + SpLayout::kTicket);
  p.window_bits = window_bits_for(N);
  p.log2_wpt = log2_wpt_for(p.window_bits);
  return p;
}

template <int MODE, typename T> static int sp_launch(const SpParams& p, cudaStream_t st) {
  const size_t smem = sp_smem_bytes(p.window_bits, MODE != SP_SYM, sizeof(T));
  auto* k = spspmm_kernel<MODE, T>;
  TSB_CUDA_TRY(cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  TSB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k, kSpThreads, smem));
  if (per_sm < 1) per_sm = 1;
  // persistent grid, never larger than what is resident at once: in single-pass mode a row waits for the rows
  // before it, which must therefore belong to CTAs that are running
  int64_t grid = (int64_t)per_sm * num_sms();
  if (grid > p.M) grid = p.M;
  if (grid < 1) grid = 1;
  k<<<(int)grid, kSpThreads, smem, st>>>(p);
  TSB_LAUNCH_CHECK();
  return 0;
}

}  // namespace tsb

using namespace tsb;

extern "C" size_t tsb200_spspmm_workspace_bytes(int64_t M, int64_t Kd, int64_t N, int64_t nnz_a, int64_t nnz_b) {
  (void)Kd; (void)N; (void)nnz_a; (void)nnz_b;
  if (M < 0) return 0;
  return sp_layout(M).total;
}

extern "C" int tsb200_spspmm_symbolic(const int64_t* rowptr_a, const int64_t* col_a, const int64_t* rowptr_b,
                                      const int64_t* col_b, int64_t M, int64_t Kd, int64_t N, int64_t nnz_a,
                                      int64_t nnz_b, int64_t* rowptr_c, void* workspace, size_t workspace_bytes,
                                      int64_t* nnz_c_host, void* stream) {
  if (M < 0 || Kd < 0 || N < 0 || nnz_a < 0 || nnz_b < 0 || !rowptr_c) return TSB200_ERR_INVALID_ARG;
  if (M >= ((int64_t)1 << 31)) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const SpLayout L = sp_layout(M);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  char* ws = (char*)workspace;
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, SpLayout::kScalarBytes, st));
  TSB_CUDA_TRY(cudaMemsetAsync(rowptr_c, 0, (size_t)(M + 1) * 8, st));
  if (M == 0 || nnz_a == 0 || nnz_b == 0) {
    if (nnz_c_host) *nnz_c_host = 0;
    return 0;
  }
  if (!rowptr_a || !col_a || !rowptr_b || !col_b) return TSB200_ERR_INVALID_ARG;
  SpParams p = sp_bind(rowptr_a, col_a, nullptr, rowptr_b, col_b, nullptr, M, N, ws + L.scalars);
  p.counts = rowptr_c + 1;
  int rc = sp_launch<SP_SYM, float>(p, st);
  if (rc) return rc;
  size_t tb = L.cub_bytes;
  TSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, tb, rowptr_c + 1, rowptr_c + 1, (int)M, st));
  int64_t* nnz_dev = (int64_t*)(ws + L.scalars + SpLayout::kNnz);
  sp_finish_kernel<<<1, 1, 0, st>>>(rowptr_c, M, nullptr, nnz_dev);
  TSB_LAUNCH_CHECK();
  if (nnz_c_host) TSB_CUDA_TRY(cudaMemcpyAsync(nnz_c_host, nnz_dev, 8, cudaMemcpyDeviceToHost, st));
  return 0;
}

extern "C" int tsb200_spspmm_numeric(const int64_t* rowptr_a, const int64_t* col_a, const void* val_a,
                                     const int64_t* rowptr_b, const int64_t* col_b, const void* val_b, int64_t M,
                                     int64_t Kd, int64_t N, int64_t nnz_a, int64_t nnz_b, const int64_t* rowptr_c,
                                     int64_t* row_c, int64_t* col_c, void* val_c, int dtype, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  if (M < 0 || Kd < 0 || N < 0 || nnz_a < 0 || nnz_b < 0) return TSB200_ERR_INVALID_ARG;
  if (M == 0 || nnz_a == 0 || nnz_b == 0) return 0;
  if (!rowptr_a || !col_a || !rowptr_b || !col_b || !rowptr_c || !col_c) return TSB200_ERR_INVALID_ARG;
  if (val_c && dtype != TSB200_F32 && dtype != TSB200_F64) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const SpLayout L = sp_layout(M);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  char* ws = (char*)workspace;
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, SpLayout::kScalarBytes, st));
  SpParams p = sp_bind(rowptr_a, col_a, val_a, rowptr_b, col_b, val_b, M, N, ws + L.scalars);
  p.rowptr_c = rowptr_c; p.row_c = row_c; p.col_c = col_c; p.val_c = val_c;
  if (val_c && dtype == TSB200_F64) return sp_launch<SP_NUM, double>(p, st);
  return sp_launch<SP_NUM, float>(p, st);
}

extern "C" int tsb200_spspmm_bound(const int64_t* col_a, const int64_t* rowptr_b, int64_t nnz_a, void* workspace,
                                   size_t workspace_bytes, int64_t* bound_host, void* stream) {
  if (nnz_a < 0) return TSB200_ERR_INVALID_ARG;
  // only the scalar block is used, which sits at the start of every SpSpMM workspace
  if (!workspace || workspace_bytes < SpLayout::kScalarBytes) return TSB200_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* d = (unsigned long long*)((char*)workspace + SpLayout::kBound);
  TSB_CUDA_TRY(cudaMemsetAsync(d, 0, 8, st));
  if (nnz_a > 0) {
    if (!col_a || !rowptr_b) return TSB200_ERR_INVALID_ARG;
    int64_t blocks = (nnz_a + 1023) / 1024;
    const int64_t cap = (int64_t)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    sp_bound_kernel<<<(int)blocks, 256, 0, st>>>(col_a, nnz_a, rowptr_b, d);
    TSB_LAUNCH_CHECK();
  }
  if (bound_host) TSB_CUDA_TRY(cudaMemcpyAsync(bound_host, d, 8, cudaMemcpyDeviceToHost, st));
  return 0;
}

extern "C" int tsb200_spspmm_fused(const int64_t* rowptr_a, const int64_t* col_a, const void* val_a,
                                   const int64_t* rowptr_b, const int64_t* col_b, const void* val_b, int64_t M,
                                   int64_t Kd, int64_t N, int64_t nnz_a, int64_t nnz_b, int64_t* rowptr_c,
                                   int64_t* row_c, int64_t* col_c, void* val_c, int64_t capacity, int dtype,
                                   void* workspace, size_t workspace_bytes, int64_t* nnz_c_host, void* stream) {
  if (M < 0 || Kd < 0 || N < 0 || nnz_a < 0 || nnz_b < 0 || capacity < 0 || !rowptr_c) return TSB200_ERR_INVALID_ARG;
  if (M >= ((int64_t)1 << 31)) return TSB200_ERR_UNSUPPORTED;
  if (val_c && dtype != TSB200_F32 && dtype != TSB200_F64) return TSB200_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const SpLayout L = sp_layout(M);
  if (!workspace || workspace_bytes < L.total) return TSB200_ERR_WORKSPACE;
  char* ws = (char*)workspace;
  // the ticket and nnz(C), then the overflow flag; the product bound stays
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, SpLayout::kBound, st));
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars + SpLayout::kOverflow, 0, 8, st));
  TSB_CUDA_TRY(cudaMemsetAsync(rowptr_c, 0, (size_t)(M + 1) * 8, st));
  if (M == 0 || nnz_a == 0 || nnz_b == 0) {
    if (nnz_c_host) *nnz_c_host = 0;
    return 0;
  }
  if (!rowptr_a || !col_a || !rowptr_b || !col_b || (capacity > 0 && !col_c)) return TSB200_ERR_INVALID_ARG;
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.status, 0, (size_t)M * 8, st));
  SpParams p = sp_bind(rowptr_a, col_a, val_a, rowptr_b, col_b, val_b, M, N, ws + L.scalars);
  p.row_c = row_c; p.col_c = col_c; p.val_c = val_c;
  p.status = (unsigned long long*)(ws + L.status);
  p.capacity = capacity;
  p.overflow = (int*)(ws + L.scalars + SpLayout::kOverflow);
  p.claim_slot = kClaimSlot;
  int rc = (val_c && dtype == TSB200_F64) ? sp_launch<SP_FUSED, double>(p, st) : sp_launch<SP_FUSED, float>(p, st);
  if (rc) return rc;
  // rowptr_c[1 + i] = running maximum of the published inclusive prefixes
  int64_t blocks = (M + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  sp_status_value_kernel<<<(int)blocks, 256, 0, st>>>(p.status, M, rowptr_c + 1);
  TSB_LAUNCH_CHECK();
  size_t tb = L.cub_bytes;
  TSB_CUDA_TRY(cub::DeviceScan::InclusiveScan(ws + L.cub, tb, rowptr_c + 1, rowptr_c + 1, cub::Max(), (int)M, st));
  sp_finish_kernel<<<1, 1, 0, st>>>(rowptr_c, M, p.overflow, (int64_t*)(ws + L.scalars + SpLayout::kNnz));
  TSB_LAUNCH_CHECK();
  if (nnz_c_host)
    TSB_CUDA_TRY(cudaMemcpyAsync(nnz_c_host, ws + L.scalars + SpLayout::kNnz, 8, cudaMemcpyDeviceToHost, st));
  return 0;
}
