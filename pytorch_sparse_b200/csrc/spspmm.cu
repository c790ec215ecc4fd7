// spspmm.cu — CSR x CSR -> CSR/COO sparse-sparse matmul for sm_90a.
//
// Replaces spspmm_sum -> torch.sparse.mm (torch_sparse/matmul.py:94-111; CPU: ATen sparse_matmul,
// CUDA: cuSPARSE SpGEMM), keeping its observable contract: output sorted by (row, col), unique,
// structural (numerical zeros are kept).
//
// Two-phase row-wise Gustavson with a per-CTA shared-memory BITMAP accumulator:
//   * a CTA owns one output row at a time (rows are handed out in chunks of 8 from a global atomic
//     counter; the chunk's rowptr entries and the next row's A-row metadata are prefetched so the
//     dependent global loads rowptr_a -> col_a -> rowptr_b of row r+1 overlap the work of row r);
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
#include <cstdlib>

#include <cub/cub.cuh>

#include "common.cuh"

namespace tsb {

constexpr int kSpThreads = 256;
constexpr int kSpWarps = kSpThreads / 32;
constexpr int kFlatU = 8;                         // products per thread on the flat path
constexpr int kStageCap = kFlatU * kSpThreads;    // output entries staged in shared memory per row (2048)
constexpr int kMaxWindowLog2 = 18;
constexpr int kMaxWindowBits = 1 << kMaxWindowLog2;
constexpr int kClaimSlotDefault = 3;              // single-pass mode: schedule slot of the next row's ticket (see the kernel)
constexpr int kABatch = 128;                      // A entries staged per batch
static_assert(kStageCap <= (1 << (32 - kMaxWindowLog2 - 1)), "owner id and column share one 32-bit word");

struct SpParams {
  const int64_t* rowptr_a; const int64_t* col_a; const void* val_a;
  const int64_t* rowptr_b; const int64_t* col_b; const void* val_b;
  int64_t M, Kd, N;
  int64_t* counts;          // symbolic: per-row nnz (accumulated at rowptr_c + 1, pre-zeroed)
  const int64_t* rowptr_c;  // numeric
  int64_t* row_c; int64_t* col_c; void* val_c;
  unsigned int* counter;
  unsigned long long* status;  // FUSED: per-row look-back words (zeroed by the host)
  int64_t capacity;            // FUSED: entries the output arrays can hold
  int* overflow;               // FUSED: set when a row would not fit
  unsigned long long* dbg;     // FUSED: optional look-back statistics (steps, empty polls, look-backs)
  int claim_slot;              // where in a row's schedule the NEXT row's ticket is taken (0 = at the start)
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
__device__ __forceinline__ int64_t sp_lookback(const unsigned long long* status, int64_t i, int lane,
                                               unsigned long long* dbg) {
  int64_t excl = 0;
  unsigned steps = 0, polls = 0;
  for (int64_t j = i - 1; j >= 0; j -= 32) {
    const int64_t r = j - lane;
    unsigned long long st = kStPrefix;  // rows before row 0: inclusive prefix 0
    steps++;
    if (r >= 0) {
      st = sp_ld_status(status + r);
      while ((st >> 62) == 0) {
        polls++;
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
  if (dbg) {  // tuning aid (TSB200_SPSPMM_DEBUG): look-back steps and status polls that found nothing yet
#pragma unroll
    for (int off = 16; off; off >>= 1) polls += __shfl_xor_sync(0xffffffffu, polls, off);
    if (lane == 0) {
      atomicAdd(dbg, (unsigned long long)steps);
      atomicAdd(dbg + 1, (unsigned long long)polls);
      atomicAdd(dbg + 2, 1ull);
    }
  }
  return excl;
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

  // next row's A-row metadata, prefetched into registers while the current row is processed
  bool pf_valid = false;
  int64_t pf_bs = 0;
  int pf_len = 0;
  T pf_av = (T)1;

  __syncthreads();
  // Rows are handed out one at a time from a global ticket counter, one row AHEAD: the ticket of the next row is
  // taken when a row starts, so its rowptr_a -> col_a -> rowptr_b chain of dependent loads overlaps this row's work.
  int par = 0;
  int64_t i = s_claim[0];
  int64_t a_s = 0, a_e = 0;
  if (i < p.M) { a_s = p.rowptr_a[i]; a_e = p.rowptr_a[i + 1]; }

  // The next row's ticket is taken at schedule slot `cs` of the current row, read after the following barrier
  // (slot cs + 1), and its metadata chain is issued at slots cs + 2 / cs + 3. Slot 0 = row start (longest prefetch
  // distance); later slots shorten the time between taking a ticket and publishing that row's nnz, which is what
  // the rows behind it wait for in single-pass mode.
  const int cs = FUSED ? p.claim_slot : 0;
  while (i < p.M) {
    const int64_t n_a = a_e - a_s;
    int64_t nrow = p.M, nx_s = 0, nx_e = 0;   // the next row and its A-row extent
    bool do_pf = false;
    int64_t nk = -1;
    int stage = 0;  // 0 nothing yet, 1 ticket taken, 2 next row known, 3 its col_a issued, 4 its rowptr_b issued

#define SP_NEXT_ROW()                                              \
  nrow = s_claim[par ^ 1];                                         \
  if (nrow < p.M) { nx_s = p.rowptr_a[nrow]; nx_e = p.rowptr_a[nrow + 1]; }
#define SP_PF_STAGE1()                                             \
  {                                                                \
    const int64_t nn = nx_e - nx_s;                                \
    if (nn > 0 && nn <= kABatch) {                                 \
      do_pf = true;                                                \
      if (tid < nn) nk = p.col_a[nx_s + tid];                      \
    }                                                              \
  }
#define SP_PF_STAGE2()                                             \
  if (do_pf) {                                                     \
    if (nk >= 0) {                                                 \
      pf_bs = p.rowptr_b[nk];                                      \
      pf_len = (int)(p.rowptr_b[nk + 1] - pf_bs);                  \
      pf_av = (NUMERIC && va) ? va[nx_s + tid] : (T)1;             \
    }                                                              \
    pf_valid = true;                                               \
  }

#define SP_AT(S)                                                                             \
  {                                                                                          \
    if (stage == 0 && cs <= (S)) {                                                           \
      if (tid == 0) s_claim[par ^ 1] = atomicAdd(p.counter, 1u);                             \
      stage = 1;                                                                             \
    } else if (stage == 1) { SP_NEXT_ROW(); stage = 2; }                                     \
    else if (stage == 2) { SP_PF_STAGE1(); stage = 3; }                                      \
    else if (stage == 3) { SP_PF_STAGE2(); stage = 4; }                                      \
  }

    do {  // one row; `break` = done with it
      if (n_a <= 0) {  // empty row: counts[i] stays 0 (pre-zeroed) / status = aggregate 0; no output
        if (FUSED && tid == 0) sp_st_status(p.status + i, kStAgg);
        pf_valid = false;
        break;
      }
      SP_AT(0);
      const int na0 = (int)min(n_a, (int64_t)kABatch);

      // ---- stage the (first batch of the) A-row metadata: start/length of each B row, a_ik; number the products ----
      int64_t bs = 0;
      int len = 0;
      T av = (T)1;
      if (pf_valid) { bs = pf_bs; len = pf_len; av = pf_av; }
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
      SP_AT(1);   // (slot 0 ticket: the barrier inside the scan made it visible; the two rowptr_a loads are in flight)
      if (tid < na0) {
        s_se[tid] = make_int2(excl, excl + len_c);
        // the 32-aligned product numbers inside [excl, excl + len): this entry is where their chunk starts
        if (P <= kStageCap)
          for (int k = (excl + 31) >> 5; (k << 5) < excl + len_c; k++) s_ent[k] = (unsigned char)tid;
      }
      pf_valid = false;
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
        SP_AT(2);
#pragma unroll
        for (int u = 0; u < kFlatU; u++)
          if (cc[u] != 0xffffffffu) sp_mark(bitmap, cc[u]);
        __syncthreads();
        SP_AT(3);
#pragma unroll
        for (int u = 0; u < kFlatU; u++)
          if (cc[u] != 0xffffffffu) sp_verify(bitmap, cc[u]);
        __syncthreads();
        SP_AT(4);
        if (!NUMERIC) {
          int cnt = (uint32_t)tid < NCH ? sp_count_clear_chunk(bitmap, lw) : 0;
#pragma unroll
          for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
          if (lane == 0 && cnt) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + i), (unsigned long long)cnt);
          break;  // the next row's staging barriers order the clears before its marks
        }
        const int wc = sp_scan<true>(bitmap, pre4, tbase, tflag, lw, NCH, s_warp);
        // single pass: the row's nnz is known now -> publish it, so that later rows can add it up while this
        // row is still ranking its products
        if (FUSED && tid == 0) sp_st_status(p.status + i, kStAgg | (unsigned long long)wc);
        __syncthreads();
        SP_AT(5);
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
        SP_AT(6);
        uint32_t dmask = 0;
        if (has_val) {
#pragma unroll
          for (int u = 0; u < kFlatU; u++) {
            if (cc[u] != 0xffffffffu) {
              const uint32_t r = cc[u] >> kMaxWindowLog2;
              const uint32_t q = (uint32_t)(((warp + kSpWarps * u) << 5) + lane);
              if ((scol[r] >> kMaxWindowLog2) == q) acc[r] = pv[u];
              else dmask |= 1u << u;
            }
          }
        }
        if (FUSED && warp == 0 && wc > 0) {
          // where this row starts in the output: nnz of all earlier rows (decoupled look-back), then publish the
          // inclusive prefix for the rows behind
          const int64_t base = sp_lookback(p.status, i, lane, p.dbg);
          if (lane == 0) {
            sp_st_status(p.status + i, kStPrefix | (unsigned long long)(base + wc));
            s_base = base;
          }
        }
        if (__syncthreads_or(dmask != 0)) {
#pragma unroll
          for (int u = 0; u < kFlatU; u++)
            if (dmask & (1u << u)) atomicAdd(&acc[cc[u] >> kMaxWindowLog2], pv[u]);
          __syncthreads();
        }
        SP_AT(7);
        int64_t ob;
        if (FUSED) ob = s_base;
        else ob = p.rowptr_c[i];
        int nw = wc;
        if (FUSED && wc > 0 && ob + wc > p.capacity) {  // cannot happen with capacity >= sum of products; never write past it
          nw = 0;
          if (tid == 0) *p.overflow = 1;
        }
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
      SP_AT(2);
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
      const bool single_batch = n_a <= kABatch;
      int64_t done = 0;  // nnz of this row emitted by previous windows
      int64_t out0 = 0;
      if (MODE == SP_NUM) out0 = p.rowptr_c[i];
      int cnt = 0;       // symbolic: columns this thread was first on

      // walk every product of the row that falls into [wlo, whi); BODY sees c (column), c0 (window-relative),
      // e (A entry in the staged batch), ebs + f (index into B)
#define SP_WALK(BODY)                                                              \
  for (int64_t ab = a_s; ab < a_e; ab += kABatch) {                                \
    const int na = (int)min((int64_t)kABatch, a_e - ab);                           \
    if (!single_batch) {                                                           \
      __syncthreads();                                                             \
      if (tid < na) {                                                              \
        const int64_t k = p.col_a[ab + tid];                                       \
        const int64_t kb = p.rowptr_b[k];                                          \
        s_bs[tid] = kb;                                                            \
        s_len[tid] = (int)(p.rowptr_b[k + 1] - kb);                                \
        if (NUMERIC) s_av[tid] = va ? va[ab + tid] : (T)1;                         \
      }                                                                            \
      __syncthreads();                                                             \
    }                                                                              \
    for (int e = warp; e < na; e += kSpWarps) {                                    \
      const int64_t ebs = s_bs[e];                                                 \
      const int elen = s_len[e];                                                   \
      for (int f = lane; f < elen; f += 32) {                                      \
        const int64_t c = (int64_t)ldg64_hint(p.col_b + ebs + f, pol_b);           \
        if (c >= wlo && c < whi) {                                                 \
          const uint32_t c0 = (uint32_t)(c - wlo);                                 \
          BODY                                                                     \
        }                                                                          \
      }                                                                            \
    }                                                                              \
  }
      // counting pass (the whole job of the symbolic kernel; in single-pass mode it gives the row's nnz before
      // anything is written): mark with atomicOr, whose return value tells a product whether it was first
#define SP_COUNT_PASS()                                                            \
  for (int64_t win = win_lo; win <= win_hi; win++) {                               \
    const int64_t wlo = win * W, whi = wlo + W;                                    \
    SP_WALK({                                                                      \
      const uint32_t bit = 1u << (c0 & 31u);                                       \
      const uint32_t old = atomicOr(&bitmap[sp_phys(c0 >> 5)], bit);               \
      if (!(old & bit)) cnt++;                                                     \
      tflag[c0 >> (5 + lw)] = 1;                                                   \
    })                                                                             \
    __syncthreads();                                                               \
    if ((uint32_t)tid < NCH && tflag[tid]) {                                       \
      sp_count_clear_chunk(bitmap, lw);                                            \
      tflag[tid] = 0;                                                              \
    }                                                                              \
    __syncthreads();                                                               \
  }

      if (!NUMERIC) {
        SP_COUNT_PASS();
#pragma unroll
        for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
        if (lane == 0 && cnt) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + i), (unsigned long long)cnt);
        SP_AT(3);
        break;
      }
      bool skip_row = false;
      if (FUSED) {
        if (tid == 0) s_total = 0;
        __syncthreads();
        SP_COUNT_PASS();
#pragma unroll
        for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
        if (lane == 0 && cnt) atomicAdd(&s_total, cnt);
        __syncthreads();
        const int total = s_total;
        if (warp == 0) {
          if (lane == 0) sp_st_status(p.status + i, kStAgg | (unsigned long long)total);
          if (total > 0) {
            const int64_t base = sp_lookback(p.status, i, lane, p.dbg);
            if (lane == 0) {
              sp_st_status(p.status + i, kStPrefix | (unsigned long long)(base + total));
              s_base = base;
            }
          }
        }
        __syncthreads();
        out0 = s_base;
        if (total == 0) skip_row = true;
        else if (out0 + total > p.capacity) {
          skip_row = true;
          if (tid == 0) *p.overflow = 1;
        }
      }
      if (!skip_row) {
        for (int64_t win = win_lo; win <= win_hi; win++) {
          const int64_t wlo = win * W, whi = wlo + W;
          // ---- mark ----
          SP_WALK({
            atomicOr(&bitmap[sp_phys(c0 >> 5)], 1u << (c0 & 31u));
            tflag[c0 >> (5 + lw)] = 1;
          })
          __syncthreads();
          const int wc = sp_scan<false>(bitmap, pre4, tbase, tflag, lw, NCH, s_warp);
          const int64_t ob = out0 + done;
          const bool staged = wc <= kStageCap;  // columns staged in shared memory -> coalesced stores
          if (has_val)
            for (int q = tid; q < wc; q += kSpThreads) val_c[ob + q] = (T)0;
          __syncthreads();
          // ---- rank every product: column (same-value races are benign), value via L2 atomics ----
          SP_WALK({
            const uint32_t r = sp_rank<false>(bitmap, pre4, tbase, lw, c0);
            if (staged) {
              scol[r] = c0;
            } else {
              p.col_c[ob + r] = c;
              if (p.row_c) p.row_c[ob + r] = i;
            }
            if (has_val) atomicAdd(val_c + ob + r, s_av[e] * (vb ? ldg_hint(vb + ebs + f, pol_b) : (T)1));
          })
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
#undef SP_WALK
#undef SP_COUNT_PASS
      SP_AT(3);
    } while (false);
    // whatever part of the next-row schedule this row's path did not reach: the ticket and the row extent are
    // mandatory, the metadata prefetch is optional (a row without it loads its metadata at its start)
    if (stage == 0) {
      if (tid == 0) s_claim[par ^ 1] = atomicAdd(p.counter, 1u);
      stage = 1;
    }
    if (stage == 1) {
      __syncthreads();
      SP_NEXT_ROW();
    }
#undef SP_AT
#undef SP_PF_STAGE1
#undef SP_PF_STAGE2
#undef SP_NEXT_ROW
    i = nrow;
    a_s = nx_s;
    a_e = nx_e;
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

__global__ void sp_copy_last_kernel(const int64_t* rowptr_c, int64_t M, int64_t* nnz_dev) { *nnz_dev = rowptr_c[M]; }
// nnz(C), or -1 when a row did not fit into the caller's arrays (nothing was written past them)
__global__ void sp_finish_fused_kernel(const int64_t* rowptr_c, int64_t M, const int* overflow, int64_t* nnz_dev) {
  *nnz_dev = *overflow ? (int64_t)-1 : rowptr_c[M];
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

struct SpLayout { size_t scalars, status, cub, total, cub_bytes; };
static SpLayout sp_layout(int64_t M) {
  SpLayout L;
  size_t off = 0;
  L.scalars = off; off += 256;
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
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, 256, st));
  TSB_CUDA_TRY(cudaMemsetAsync(rowptr_c, 0, (size_t)(M + 1) * 8, st));
  if (M == 0 || nnz_a == 0 || nnz_b == 0) {
    if (nnz_c_host) *nnz_c_host = 0;
    return 0;
  }
  if (!rowptr_a || !col_a || !rowptr_b || !col_b) return TSB200_ERR_INVALID_ARG;
  SpParams p;
  p.rowptr_a = rowptr_a; p.col_a = col_a; p.val_a = nullptr;
  p.rowptr_b = rowptr_b; p.col_b = col_b; p.val_b = nullptr;
  p.M = M; p.Kd = Kd; p.N = N;
  p.counts = rowptr_c + 1; p.rowptr_c = nullptr; p.row_c = nullptr; p.col_c = nullptr; p.val_c = nullptr;
  p.counter = (unsigned int*)(ws + L.scalars);
  p.window_bits = window_bits_for(N);
  p.log2_wpt = log2_wpt_for(p.window_bits);
  p.status = nullptr; p.capacity = 0; p.overflow = nullptr; p.dbg = nullptr; p.claim_slot = 0;
  int rc = sp_launch<SP_SYM, float>(p, st);
  if (rc) return rc;
  size_t tb = L.cub_bytes;
  TSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, tb, rowptr_c + 1, rowptr_c + 1, (int)M, st));
  int64_t* nnz_dev = (int64_t*)(ws + L.scalars + 16);
  sp_copy_last_kernel<<<1, 1, 0, st>>>(rowptr_c, M, nnz_dev);
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
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, 256, st));
  SpParams p;
  p.rowptr_a = rowptr_a; p.col_a = col_a; p.val_a = val_a;
  p.rowptr_b = rowptr_b; p.col_b = col_b; p.val_b = val_b;
  p.M = M; p.Kd = Kd; p.N = N;
  p.counts = nullptr; p.rowptr_c = rowptr_c; p.row_c = row_c; p.col_c = col_c; p.val_c = val_c;
  p.counter = (unsigned int*)(ws + L.scalars);
  p.window_bits = window_bits_for(N);
  p.log2_wpt = log2_wpt_for(p.window_bits);
  p.status = nullptr; p.capacity = 0; p.overflow = nullptr; p.dbg = nullptr; p.claim_slot = 0;
  if (val_c && dtype == TSB200_F64) return sp_launch<SP_NUM, double>(p, st);
  return sp_launch<SP_NUM, float>(p, st);
}

extern "C" int tsb200_spspmm_bound(const int64_t* col_a, const int64_t* rowptr_b, int64_t nnz_a, void* workspace,
                                   size_t workspace_bytes, int64_t* bound_host, void* stream) {
  if (nnz_a < 0) return TSB200_ERR_INVALID_ARG;
  if (!workspace || workspace_bytes < 256) return TSB200_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* d = (unsigned long long*)((char*)workspace + 32);
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
  // scalars: [0] row ticket, [16] nnz(C) (int64), [32] product bound (tsb200_spspmm_bound), [48] overflow flag
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars, 0, 32, st));
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.scalars + 48, 0, 8, st));
  TSB_CUDA_TRY(cudaMemsetAsync(rowptr_c, 0, (size_t)(M + 1) * 8, st));
  int64_t* nnz_dev = (int64_t*)(ws + L.scalars + 16);
  if (M == 0 || nnz_a == 0 || nnz_b == 0) {
    if (nnz_c_host) { nnz_c_host[0] = 0; }
    return 0;
  }
  if (!rowptr_a || !col_a || !rowptr_b || !col_b || (capacity > 0 && !col_c)) return TSB200_ERR_INVALID_ARG;
  TSB_CUDA_TRY(cudaMemsetAsync(ws + L.status, 0, (size_t)M * 8, st));
  SpParams p;
  p.rowptr_a = rowptr_a; p.col_a = col_a; p.val_a = val_a;
  p.rowptr_b = rowptr_b; p.col_b = col_b; p.val_b = val_b;
  p.M = M; p.Kd = Kd; p.N = N;
  p.counts = nullptr; p.rowptr_c = nullptr; p.row_c = row_c; p.col_c = col_c; p.val_c = val_c;
  p.counter = (unsigned int*)(ws + L.scalars);
  p.status = (unsigned long long*)(ws + L.status);
  p.capacity = capacity;
  p.overflow = (int*)(ws + L.scalars + 48);
  p.dbg = nullptr;
  p.claim_slot = kClaimSlotDefault;
  if (const char* ev = getenv("TSB200_SPSPMM_CLAIM")) {  // tuning knob, 0..6
    const int v = atoi(ev);
    if (v >= 0 && v <= 6) p.claim_slot = v;
  }
  if (getenv("TSB200_SPSPMM_DEBUG")) {  // look-back statistics in scalars [64..88): steps, empty polls, look-backs
    p.dbg = (unsigned long long*)(ws + L.scalars + 64);
    TSB_CUDA_TRY(cudaMemsetAsync(p.dbg, 0, 24, st));
  }
  p.window_bits = window_bits_for(N);
  p.log2_wpt = log2_wpt_for(p.window_bits);
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
  sp_finish_fused_kernel<<<1, 1, 0, st>>>(rowptr_c, M, p.overflow, nnz_dev);
  TSB_LAUNCH_CHECK();
  if (nnz_c_host) TSB_CUDA_TRY(cudaMemcpyAsync(nnz_c_host, nnz_dev, 8, cudaMemcpyDeviceToHost, st));
  return 0;
}
