// spmv.cuh - merge-path CSR SpMV for sm_90a (fp64 values, int32 columns, int32/int64 row offsets).
//
// Replaces the operator of the reference, calcMatVecProd(...,'Strain') pcg_solver.py:242-300, on the
// assembled matrix A = K[Eff,Eff].
//
// Design (see DESIGN.md "SpMV"):
//   * plan time (once per matrix): a 2-D merge-path search over (row ends, nnz indices) cuts the
//     work into tiles of `tile_items` merge items; when no row is long, tile starts are snapped back
//     to a row boundary so that no row is split (no fix-up pass, bit-reproducible);
//   * run time, one CTA per tile: the tile's slice of `val` and `col` is brought into shared memory
//     by two TMA bulk copies (cp.async.bulk + mbarrier, L2 evict-first) - the streaming arrays never
//     pass through L1, which is left to the gather of x (ld.global.nc); the row offsets of the tile
//     are loaded meanwhile; then sub-warp groups of LANES lanes walk the rows of the tile, multiply
//     from shared memory against gathered x and finish each row with a shuffle reduction; row sums
//     are staged in shared memory and written to y coalesced, with an optional fused dot-product
//     epilogue  sum_r x[r]*y[r]  (the p.q of pcg_solver.py:487).
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace pcgb {

constexpr int kSpmvBlock = 256;
constexpr int kAlignMask = 7;      // tiles are staged from an 8-element aligned start
constexpr int kMaxRuns = 2048;     // staged-x plan: column runs per tile
constexpr int kMaxWin = 256;       // staged-x plan: x windows per tile
constexpr int kMaxXLen = 6144;     // staged-x plan: doubles of x staged per tile (48 KB)
constexpr int kVdictMax = 1024;    // value dictionary: at most this many distinct blocks (72 KB of shared memory per CTA)
constexpr int kVdictSlots = 4096;  // value dictionary: open-addressing hash table (load <= 1/4 at kVdictMax)

// per-tile descriptor of the persistent kernel: everything a producer warp needs in one 32-byte load
struct __align__(16) TileDesc {
  int64_t k0;   // first non-zero of the tile
  int cnt;      // non-zeros in the tile
  int r0;       // first row
  int R;        // rows with a segment here (incl. a partial last row); bit 31 = first row is a continuation
  int wb;       // first x window
  int nw;       // x windows
  int xlen;     // staged doubles of x
};

struct CsrPlan {
  int64_t nrows = 0, ncols = 0, nnz = 0;
  const void *rowptr = nullptr;
  bool rp64 = false;
  const int *col = nullptr;
  const double *val = nullptr;
  // plan
  int tile_items = 0, lanes = 0, ntiles = 0;
  bool snap = false, use_tma = true;
  int cap_nnz = 0, cap_rows = 0, smem_bytes = 0, max_row = 0;
  int *tile_row = nullptr;       // [ntiles+1]
  int64_t *tile_k = nullptr;     // [ntiles+1]
  double *carry = nullptr;       // [ntiles]   head-partial row sums (split mode)
  int nfix = 0;                  // rows that span more than one tile
  int *fix_row = nullptr, *fix_first = nullptr, *fix_cnt = nullptr;
  double *dot_partials = nullptr;  // [ntiles]  fused  x.y  partials
  // staged-x variant (k_spmv_staged): x windows per tile + 16-bit local column indices
  bool staged = false;
  uint16_t *lidx = nullptr;        // [nnz + 16]  position of col[k] inside the tile's staged x buffer
  int *tile_win = nullptr;         // [ntiles+1]  window range of each tile
  int *win_start = nullptr;        // [nwin]      first column of the window
  int *win_off = nullptr;          // [nwin]      offset of the window inside the staged buffer
  int *tile_xlen = nullptr;        // [ntiles]    staged doubles per tile
  int cap_x = 0, max_nw = 0, smem_staged = 0;
  int64_t nwin = 0;
  // persistent pipelined variant (k_spmv_persist)
  bool persist = false;
  struct TileDesc *tile_desc = nullptr;  // [ntiles]
  int stages = 0, stage_bytes = 0, smem_persist = 0, grid_persist = 0, ctas_per_sm = 1, persist_prod = 4;
  // column-triple index ("T3"): when every row is a sequence of aligned triples of consecutive staged positions
  // (3 dofs per node: hex / concrete), ONE 16-bit index is stored per triple -> 8 + 2/3 bytes per non-zero
  bool t3 = false;
  uint16_t *lidx3 = nullptr;       // [nnz/3 + 16]
  // node-block mode ("BSR-3"): 3 dofs per node give rows 3n, 3n+1, 3n+2 the SAME column pattern made of aligned column
  // triples; one thread then owns a whole 3x3 block (9 values, 3 x entries, ONE 16-bit staged position): 8 + 2/9 bytes per
  // non-zero from HBM, a third of the x gathers and a ninth of the index loads of the row-group consumer
  bool bsr = false;
  uint16_t *bidx = nullptr;        // [nnz/9 + 16]  staged x position of block t of node n at rowptr[3n]/9 + t
  int cap_blocks = 0, cap_nodes = 0, smem_bsr = 0, bsr_stage_bytes = 0, bsr_stages = 0, bsr_prod = 0, grid_bsr = 0, bsr_mode = 1, bsr_cw = 6;
  // value dictionary of the node-block kernel: when the matrix has few bitwise-distinct 3x3 blocks (a structured mesh of
  // one element type), each is stored once and every block position streams a 16-bit id instead of its 72 bytes of values
  int vd = 0;                      // distinct blocks D (0: no dictionary, the kernel streams val)
  uint16_t *bvid = nullptr;        // [nnz/9 + 16]  dictionary id of the block at bidx's position (plan time only)
  double *vdict = nullptr;         // [vd * 9]      the blocks, row-major
  int bsr_group = 0;               // tiles a CTA consumes between two barriers (k_spmv_bsr3_vd: one warp per tile)
  // index stream of k_spmv_bsr3_vd: per tile a segment list, then block words (staged position | id << 16); a run segment
  // (nodes whose blocks sit 3 staged doubles further on than their predecessor's, with the same ids) stores only its head
  uint32_t *vwords = nullptr;      // [nvwords + 8]
  int64_t *vtoff = nullptr;        // [ntiles + 1]  first word of each tile, by tile id
  int64_t nvwords = 0, run_nodes = 0;
  int cap_words = 0;               // words of the largest tile slice (16-byte aligned window)
  int *split_tile = nullptr;       // [ntiles]  tile id of desc_split[k]
  // interface-first split (multi-GPU overlap): tiles that own an interface row are listed first in desc_split
  struct TileDesc *desc_split = nullptr;  // [ntiles] permutation of tile_desc
  int nb_tiles = 0;                       // leading boundary tiles of desc_split
  double *dot_partials_split = nullptr;   // [2 * grid_persist]
  // the caller may drop `col` once the selected kernel no longer reads it (diag cached first)
  double *diag_cache = nullptr;
};

// ------------------------------------------------------------------ PTX wrappers (TMA bulk copy)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  // try_wait suspends the warp until the phase completes or the time hint (ns) expires: no hot spinning
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(1000000u)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// global -> shared bulk copy (UBLKCP), completion signalled on the mbarrier as transaction bytes
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}

// ------------------------------------------------------------------ plan kernels
template <typename RP>
__global__ void k_max_row(const RP *__restrict__ rowptr, int64_t nrows, int *out_max) {
  int m = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t len = (int64_t)rowptr[r + 1] - (int64_t)rowptr[r];
    m = max(m, (int)min(len, (int64_t)INT32_MAX));
  }
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(out_max, m);
}

// Merge-path split of diagonal d over (row_end = rowptr+1, nnz counting sequence): the largest i with
// row_end[r] <= d - r - 1 for all r < i.
template <typename RP>
__device__ __forceinline__ int64_t merge_path_rows(const RP *__restrict__ rowptr, int64_t nrows, int64_t nnz, int64_t d) {
  int64_t lo = d > nnz ? d - nnz : 0, hi = d < nrows ? d : nrows;
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if ((int64_t)rowptr[mid + 1] <= d - mid - 1) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

template <typename RP>
__global__ void k_partition(const RP *__restrict__ rowptr, int64_t nrows, int64_t nnz, int tile_items, int ntiles, int snap,
                            int *tile_row, int64_t *tile_k, int snap_unit = 1) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > ntiles) return;
  int64_t total = nrows + nnz;
  int64_t d = (int64_t)b * tile_items;
  if (d > total || b == ntiles) d = total;
  int64_t i = merge_path_rows(rowptr, nrows, nnz, d);
  int64_t j = d - i;
  if (snap) {
    if (i < nrows) i -= i % snap_unit;   // node-block mode: tiles start at a node (3 rows), never inside one
    j = (int64_t)rowptr[i];
  }
  tile_row[b] = (int)i;
  tile_k[b] = j;
}

template <typename RP>
__global__ void k_tile_stats(const RP *__restrict__ rowptr, const int *__restrict__ tile_row, const int64_t *__restrict__ tile_k,
                             int ntiles, int *max_cnt, int *max_rows, unsigned char *head_flag) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= ntiles) return;
  int64_t k0 = tile_k[b], k1 = tile_k[b + 1];
  int r0 = tile_row[b], r1 = tile_row[b + 1];
  int cnt = (int)(k1 - (k0 & ~(int64_t)kAlignMask));
  atomicMax(max_cnt, cnt);
  atomicMax(max_rows, r1 - r0 + 1);
  head_flag[b] = (int64_t)rowptr[r0] < k0 ? 1 : 0;
}

// ------------------------------------------------------------------ the SpMV kernel
template <int LANES, bool TMA, bool DOT, typename RP>
__global__ void __launch_bounds__(kSpmvBlock)
k_spmv_merge(const RP *__restrict__ rowptr, const int *__restrict__ col, const double *__restrict__ val,
             const double *__restrict__ x, double *__restrict__ y, const int *__restrict__ tile_row,
             const int64_t *__restrict__ tile_k, int64_t nrows, int64_t nnz, int cap_nnz, int cap_rows,
             double *__restrict__ carry, double *__restrict__ dot_partials, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;  // PCG state frozen (pcg_kernels.cuh): nothing to do
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double *sval = reinterpret_cast<double *>(smem_raw);
  double *srow = sval + cap_nnz;                          // cap_rows doubles
  int *scol = reinterpret_cast<int *>(srow + cap_rows);   // cap_nnz ints  (cap_nnz % 4 == 0, cap_rows % 2 == 0)
  int *soff = scol + cap_nnz;                             // cap_rows + 1 ints
  __shared__ uint64_t bar;
  __shared__ double red[32];

  const int tid = threadIdx.x;
  const int b = blockIdx.x;
  const int r0 = tile_row[b], r1 = tile_row[b + 1];
  const int64_t k0 = tile_k[b], k1 = tile_k[b + 1];
  const int64_t ka = k0 & ~(int64_t)kAlignMask;  // aligned start of the staged window (16 B for every array)
  const int k0l = (int)(k0 - ka), k1l = (int)(k1 - ka);
  const bool tail = (r1 < nrows) && (k1 > (int64_t)rowptr[r1]);
  const int R = r1 - r0 + (tail ? 1 : 0);  // rows that own at least a (possibly empty) segment here
  const bool head = (R > 0) && ((int64_t)rowptr[r0] < k0);

  // ---- stage val/col slices into shared memory
  if (TMA) {
    if (tid == 0) {
      mbar_init(&bar, 1);
      mbar_fence_init();
      int64_t kend = (k1 + kAlignMask) & ~(int64_t)kAlignMask;
      const int64_t lim = nnz & ~(int64_t)kAlignMask;
      if (kend > lim) kend = lim;
      const int nb = (int)(kend - ka);
      if (nb > 0) {
        const uint64_t pol = l2_evict_first_policy();
        mbar_expect_tx(&bar, (uint32_t)nb * 12u);
        bulk_g2s(sval, val + ka, (uint32_t)nb * 8u, &bar, pol);
        bulk_g2s(scol, col + ka, (uint32_t)nb * 4u, &bar, pol);
      } else {
        mbar_arrive(&bar);
      }
    }
    // the (at most 7) elements beyond the last full aligned group of the arrays
    {
      const int64_t lim = nnz & ~(int64_t)kAlignMask;
      int64_t kt = (lim > ka ? lim : ka) + tid;
      if (tid <= kAlignMask && kt >= lim && kt < k1) {
        sval[kt - ka] = val[kt];
        scol[kt - ka] = col[kt];
      }
    }
  } else {
#pragma unroll 4
    for (int j = k0l + tid; j < k1l; j += kSpmvBlock) {
      sval[j] = ld_stream(val + ka + j);
      scol[j] = ld_stream(col + ka + j);
    }
  }
  // ---- row offsets of the tile, relative to ka and clamped to the tile's nnz window
  for (int i = tid; i <= R; i += kSpmvBlock) {
    int64_t v = (int64_t)rowptr[r0 + i] - ka;
    v = v < k0l ? k0l : (v > k1l ? k1l : v);
    soff[i] = (int)v;
  }
  __syncthreads();
  if (TMA) mbar_wait(&bar, 0);

  // ---- segmented reduction: one group of LANES lanes per row, shuffle tree at the end
  constexpr int G = kSpmvBlock / LANES;
  const int gid = tid / LANES, gl = tid % LANES;
  // NOTE: the trip count is uniform over the CTA (i0, not i, is tested) because the shuffle
  // reduction below names all 32 lanes; lanes of a group past the last row just idle.
  for (int i0 = 0; i0 < R; i0 += G) {
    const int i = i0 + gid;
    const bool live = i < R;
    const int a = live ? soff[i] : 0, e = live ? soff[i + 1] : 0;
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
    int j = a + gl;
    for (; j + 3 * LANES < e; j += 4 * LANES) {
      const int c0 = scol[j], c1 = scol[j + LANES], c2 = scol[j + 2 * LANES], c3 = scol[j + 3 * LANES];
      const double v0 = sval[j], v1 = sval[j + LANES], v2 = sval[j + 2 * LANES], v3 = sval[j + 3 * LANES];
      const double x0 = __ldg(x + c0), x1 = __ldg(x + c1), x2 = __ldg(x + c2), x3 = __ldg(x + c3);
      acc0 = fma(v0, x0, acc0);
      acc1 = fma(v1, x1, acc1);
      acc2 = fma(v2, x2, acc2);
      acc3 = fma(v3, x3, acc3);
    }
    for (; j < e; j += LANES) acc0 = fma(sval[j], __ldg(x + scol[j]), acc0);
    double acc = group_sum<LANES>((acc0 + acc1) + (acc2 + acc3));
    if (live && gl == 0) srow[i] = acc;
  }
  __syncthreads();

  // ---- coalesced write-back (+ fused dot epilogue)
  double d = 0.0;
  for (int i = tid; i < R; i += kSpmvBlock) {
    const double s = srow[i];
    const int r = r0 + i;
    if (i == 0 && head) carry[b] = s;
    else y[r] = s;
    if (DOT) d = fma(s, __ldg(x + r), d);
  }
  if (DOT) {
    double v[1] = {d};
    block_sum<1, kSpmvBlock>(v, red);
    if (tid == 0) dot_partials[b] = v[0];
  }
}


// ------------------------------------------------------------------ staged-x variant: plan
// One CTA per tile.  Finds the maximal runs of consecutive columns in the tile, sorts them by first
// column, merges them (gap tolerance `gap`) into x windows, and rewrites every column index as a 16-bit
// position inside the concatenation of the tile's windows.
__global__ void __launch_bounds__(256)
k_plan_windows(const int *__restrict__ col, const int64_t *__restrict__ tile_k, int cap, int gap, int pass,
               const int *__restrict__ tile_win, uint16_t *__restrict__ lidx, int *__restrict__ win_start,
               int *__restrict__ win_off, int *__restrict__ tile_nw, int *__restrict__ tile_xlen, int *__restrict__ fail) {
  // pass 1: only count windows / staged length per tile;  pass 2: write the windows at tile_win[b] and lidx
  extern __shared__ int sm[];
  int *scol = sm;                 // cap
  int *rkey = scol + cap;         // kMaxRuns   first column of a run (sort key)
  int *rlen = rkey + kMaxRuns;    // kMaxRuns   run length
  int *rpos = rlen + kMaxRuns;    // kMaxRuns   position of the run head inside the tile
  int *wst = rpos + kMaxRuns;     // kMaxWin
  int *wof = wst + kMaxWin;       // kMaxWin + 1
  __shared__ int s_scan[256];
  __shared__ int s_nruns, s_nw, s_fail;
  const int tid = threadIdx.x, b = blockIdx.x;
  const int64_t k0 = tile_k[b], k1 = tile_k[b + 1];
  const int cnt = (int)(k1 - k0);
  if (tid == 0) { s_fail = 0; s_nw = 0; }
  for (int j = tid; j < cnt; j += 256) scol[j] = col[k0 + j];
  __syncthreads();
  // ---- run heads: one contiguous chunk per thread, exclusive scan of the head counts over the CTA
  const int per = (cnt + 255) / 256;
  const int lo = min(cnt, tid * per), hi = min(cnt, lo + per);
  int mine = 0;
  for (int j = lo; j < hi; ++j) mine += (j == 0 || scol[j] != scol[j - 1] + 1) ? 1 : 0;
  s_scan[tid] = mine;
  __syncthreads();
  if (tid == 0) {
    int acc = 0;
    for (int t = 0; t < 256; ++t) { const int v = s_scan[t]; s_scan[t] = acc; acc += v; }
    s_nruns = acc;
    if (acc > kMaxRuns) s_fail = 1;
  }
  __syncthreads();
  const int nruns = s_nruns;
  if (s_fail) {
    if (tid == 0) { atomicExch(fail, 1); if (pass == 1) { tile_nw[b] = 0; tile_xlen[b] = 0; } }
    return;
  }
  {
    int o = s_scan[tid];
    for (int j = lo; j < hi; ++j)
      if (j == 0 || scol[j] != scol[j - 1] + 1) { rkey[o] = scol[j]; rpos[o] = j; ++o; }
  }
  __syncthreads();
  for (int i = tid; i < nruns; i += 256) rlen[i] = ((i + 1 < nruns) ? rpos[i + 1] : cnt) - rpos[i];
  int np2 = 1;
  while (np2 < nruns) np2 <<= 1;
  for (int i = nruns + tid; i < np2; i += 256) { rkey[i] = INT32_MAX; rlen[i] = 0; }
  __syncthreads();
  // ---- bitonic sort of (rkey, rlen) by rkey
  for (int k = 2; k <= np2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < np2; i += 256) {
        const int l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const int a = rkey[i], c = rkey[l];
          if ((a > c) == up) {
            rkey[i] = c; rkey[l] = a;
            const int t = rlen[i]; rlen[i] = rlen[l]; rlen[l] = t;
          }
        }
      }
      __syncthreads();
    }
  // ---- merge the sorted runs into windows (sequential: a few hundred steps)
  if (tid == 0) {
    int nw = 0, xlen = 0, cs = 0, ce = -1;
    bool bad = false;
    for (int i = 0; i < nruns; ++i) {
      const int s = rkey[i], e = s + rlen[i];
      if (nw == 0 || s > ce + gap) {
        if (nw > 0) xlen += ce - cs;
        if (nw >= kMaxWin) { bad = true; break; }
        wst[nw] = s; wof[nw] = xlen; ++nw;
        cs = s; ce = e;
      } else if (e > ce) ce = e;
    }
    if (nw > 0) xlen += ce - cs;
    wof[nw] = xlen;
    if (bad || xlen > kMaxXLen) { s_fail = 1; atomicExch(fail, 1); nw = 0; xlen = 0; }
    s_nw = nw;
    if (pass == 1) { tile_nw[b] = nw; tile_xlen[b] = xlen; }
  }
  __syncthreads();
  if (s_fail || pass == 1) return;
  const int nw = s_nw, base = tile_win[b];
  for (int w = tid; w < nw; w += 256) { win_start[base + w] = wst[w]; win_off[base + w] = wof[w]; }
  // ---- local index of every entry: window by binary search over the window starts
  for (int j = tid; j < cnt; j += 256) {
    const int c = scol[j];
    int a = 0, z = nw - 1;
    while (a < z) {
      const int m = (a + z + 1) >> 1;
      if (wst[m] <= c) a = m; else z = m - 1;
    }
    lidx[k0 + j] = (uint16_t)(wof[a] + (c - wst[a]));
  }
}

// ------------------------------------------------------------------ staged-x variant: the kernel
// Same tile / row structure as k_spmv_merge, but (i) the gather of x goes to SHARED memory: the tile's x
// windows are copied in once, coalesced; (ii) the column stream is the 16-bit local index, so the kernel
// reads 10 bytes per non-zero from HBM instead of 12 and the 4-byte col array is not touched at all.
template <int LANES, bool DOT, typename RP>
__global__ void __launch_bounds__(kSpmvBlock)
k_spmv_staged(const RP *__restrict__ rowptr, const uint16_t *__restrict__ lidx, const double *__restrict__ val,
              const double *__restrict__ x, double *__restrict__ y, const int *__restrict__ tile_row,
              const int64_t *__restrict__ tile_k, const int *__restrict__ tile_win, const int *__restrict__ win_start,
              const int *__restrict__ win_off, const int *__restrict__ tile_xlen, int64_t nrows, int64_t nnz, int cap_nnz,
              int cap_rows, int cap_x, double *__restrict__ carry, double *__restrict__ dot_partials,
              const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double *sval = reinterpret_cast<double *>(smem_raw);               // cap_nnz
  double *sx = sval + cap_nnz;                                       // cap_x
  double *srow = sx + cap_x;                                         // cap_rows
  uint16_t *sidx = reinterpret_cast<uint16_t *>(srow + cap_rows);    // cap_nnz
  int *soff = reinterpret_cast<int *>(sidx + cap_nnz);               // cap_rows + 1
  __shared__ uint64_t bar;
  __shared__ double red[32];

  const int tid = threadIdx.x, b = blockIdx.x;
  const int r0 = tile_row[b], r1 = tile_row[b + 1];
  const int64_t k0 = tile_k[b], k1 = tile_k[b + 1];
  const int64_t ka = k0 & ~(int64_t)kAlignMask;
  const int k0l = (int)(k0 - ka), k1l = (int)(k1 - ka);
  const bool tail = (r1 < nrows) && (k1 > (int64_t)rowptr[r1]);
  const int R = r1 - r0 + (tail ? 1 : 0);
  const bool head = (R > 0) && ((int64_t)rowptr[r0] < k0);

  if (tid == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
    int64_t kend = (k1 + kAlignMask) & ~(int64_t)kAlignMask;
    const int64_t lim = nnz & ~(int64_t)kAlignMask;
    if (kend > lim) kend = lim;
    const int nb = (int)(kend - ka);
    if (nb > 0) {
      const uint64_t pol = l2_evict_first_policy();
      mbar_expect_tx(&bar, (uint32_t)nb * 10u);
      bulk_g2s(sval, val + ka, (uint32_t)nb * 8u, &bar, pol);
      bulk_g2s(sidx, lidx + ka, (uint32_t)nb * 2u, &bar, pol);
    } else {
      mbar_arrive(&bar);
    }
  }
  {
    const int64_t lim = nnz & ~(int64_t)kAlignMask;
    int64_t kt = (lim > ka ? lim : ka) + tid;
    if (tid <= kAlignMask && kt >= lim && kt < k1) {
      sval[kt - ka] = val[kt];
      sidx[kt - ka] = lidx[kt];
    }
  }
  // ---- x windows -> shared memory (one warp per window, coalesced)
  {
    const int wb = tile_win[b], nw = tile_win[b + 1] - wb, xlen = tile_xlen[b];
    const int warp = tid >> 5, lane = tid & 31;
    for (int w = warp; w < nw; w += kSpmvBlock / 32) {
      const int s = win_start[wb + w], o = win_off[wb + w];
      const int len = ((w + 1 < nw) ? win_off[wb + w + 1] : xlen) - o;
      for (int t = lane; t < len; t += 32) sx[o + t] = __ldg(x + s + t);
    }
  }
  for (int i = tid; i <= R; i += kSpmvBlock) {
    int64_t v = (int64_t)rowptr[r0 + i] - ka;
    v = v < k0l ? k0l : (v > k1l ? k1l : v);
    soff[i] = (int)v;
  }
  __syncthreads();
  mbar_wait(&bar, 0);

  constexpr int G = kSpmvBlock / LANES;
  const int gid = tid / LANES, gl = tid % LANES;
  for (int i0 = 0; i0 < R; i0 += G) {  // CTA-uniform trip count (full-mask shuffles below)
    const int i = i0 + gid;
    const bool live = i < R;
    const int a = live ? soff[i] : 0, e = live ? soff[i + 1] : 0;
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
    int j = a + gl;
    for (; j + 3 * LANES < e; j += 4 * LANES) {
      const double x0 = sx[sidx[j]], x1 = sx[sidx[j + LANES]], x2 = sx[sidx[j + 2 * LANES]], x3 = sx[sidx[j + 3 * LANES]];
      acc0 = fma(sval[j], x0, acc0);
      acc1 = fma(sval[j + LANES], x1, acc1);
      acc2 = fma(sval[j + 2 * LANES], x2, acc2);
      acc3 = fma(sval[j + 3 * LANES], x3, acc3);
    }
    for (; j < e; j += LANES) acc0 = fma(sval[j], sx[sidx[j]], acc0);
    double acc = group_sum<LANES>((acc0 + acc1) + (acc2 + acc3));
    if (live && gl == 0) srow[i] = acc;
  }
  __syncthreads();

  double d = 0.0;
  for (int i = tid; i < R; i += kSpmvBlock) {
    const double s = srow[i];
    const int r = r0 + i;
    if (i == 0 && head) carry[b] = s;
    else y[r] = s;
    if (DOT) d = fma(s, __ldg(x + r), d);
  }
  if (DOT) {
    double v[1] = {d};
    block_sum<1, kSpmvBlock>(v, red);
    if (tid == 0) dot_partials[b] = v[0];
  }
}


// ------------------------------------------------------------------ persistent, warp-specialised, pipelined variant
// One CTA = 8 consumer warps + kProd producer warps, kept resident (grid = SMs x CTAs/SM), looping over
// tiles c, c+grid, ... through a ring of `stages` shared-memory stages guarded by full/empty mbarriers:
//   producer warp (stage s):  wait empty[s] -> TMA bulk copies of val / 16-bit lidx -> copy the tile's x
//                             windows, x[r0..r0+R) and clamped row offsets into the stage -> arrive full[s]
//   consumer warps:           wait full[s] -> sub-warp groups reduce the rows out of shared memory,
//                             group leaders write y (and accumulate x.y) -> arrive empty[s]
// Consumers never wait on a global load; HBM streaming is entirely asynchronous (UBLKCP) and `stages` tiles deep.
constexpr int kProd = 4;          // at most this many producer warps (= min(4, stages)); stages % producers == 0
constexpr int kConsWarps = 8;
constexpr int kPersistThreads = (kConsWarps + kProd) * 32;

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <typename RP>
__global__ void k_build_desc(const RP *__restrict__ rowptr, const int *__restrict__ tile_row, const int64_t *__restrict__ tile_k,
                             const int *__restrict__ tile_win, const int *__restrict__ tile_xlen, int ntiles, int64_t nrows,
                             TileDesc *__restrict__ desc) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= ntiles) return;
  const int r0 = tile_row[b], r1 = tile_row[b + 1];
  const int64_t k0 = tile_k[b], k1 = tile_k[b + 1];
  const bool tail = (r1 < nrows) && (k1 > (int64_t)rowptr[r1]);
  const int R = r1 - r0 + (tail ? 1 : 0);
  const bool head = (R > 0) && ((int64_t)rowptr[r0] < k0);
  TileDesc d;
  d.k0 = k0; d.cnt = (int)(k1 - k0); d.r0 = r0; d.R = R | (head ? (int)0x80000000 : 0);
  d.wb = tile_win[b]; d.nw = tile_win[b + 1] - tile_win[b]; d.xlen = tile_xlen[b];
  desc[b] = d;
}

// cp.async (LDGSTS): asynchronous global -> shared copies issued by the producer lanes; their completion is
// reported to the stage's full barrier with cp.async.mbarrier.arrive.noinc (one arrival per lane).
template <int BYTES>
__device__ __forceinline__ void cp_async(void *dst_smem, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t *bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// T3 = column-triple index: sidx holds ONE 16-bit staged position per aligned triple of non-zeros (k0 % 3 == 0 for
// every tile because the plan is row-snapped and every row length is a multiple of 3); a lane owns whole triples:
// 1 index load + 3 value loads (stride 3 doubles across lanes: conflict-free over 16 lanes) + 3 x loads per 3 FMAs.
template <int LANES, bool DOT, bool T3, typename RP>
__global__ void __launch_bounds__(kPersistThreads)
k_spmv_persist(const RP *__restrict__ rowptr, const uint16_t *__restrict__ lidx, const double *__restrict__ val,
               const double *__restrict__ x, double *__restrict__ y, const TileDesc *__restrict__ desc,
               const int *__restrict__ win_start, const int *__restrict__ win_off, int ntiles, int64_t nnz, int cap_nnz,
               int cap_rows, int cap_x, int stages, int stage_bytes, double *__restrict__ carry,
               double *__restrict__ dot_partials, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t full_bar[8], empty_bar[8];
  __shared__ double red[32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    // full: 1 (TMA expect_tx arrive) + 32 (cp.async completion, one per producer lane) + 1 (producer's own stores)
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 34); mbar_init(&empty_bar[s], kConsWarps); }
    mbar_fence_init();
  }
  __syncthreads();

  // stage layout: sval[cap_nnz] f64 | sx[cap_x] f64 | srp[cap_rows+2] i64 | sidx (u16: cap_nnz, or cap_nnz/3+16 for T3) | meta[8] i32
  const int cap_idx = T3 ? (cap_nnz / 3 + 16) : cap_nnz;
  const size_t off_sx = (size_t)cap_nnz * 8, off_srp = off_sx + (size_t)cap_x * 8;
  const size_t off_sidx = off_srp + (size_t)(cap_rows + 2) * 8, off_meta = (off_sidx + (size_t)cap_idx * 2 + 15) & ~(size_t)15;

  if (warp >= kConsWarps) {
    // ================= producer warp p: tiles it = p, p + nprod, ... (stage = it % stages, stages % nprod == 0)
    const int nprod = (int)(blockDim.x >> 5) - kConsWarps;
    // Software-pipelined: the descriptor and the window descriptors of the NEXT tile are fetched while the
    // current one is being issued, so the only thing a stage waits for is its own TMA flight.
    const int p = warp - kConsWarps;
    const uint64_t pol = l2_evict_first_policy();
    int it = p;
    int tile = blockIdx.x + it * gridDim.x;
    bool have = tile < ntiles;
    int4 d0 = make_int4(0, 0, 0, 0), d1 = make_int4(0, 0, 0, 0);
    int ws = 0, wo = 0;
    if (have) {
      const int4 *dp = reinterpret_cast<const int4 *>(desc + tile);  // one 32-byte descriptor, broadcast load
      d0 = __ldg(dp); d1 = __ldg(dp + 1);
      if (lane < d1.z) { ws = __ldg(win_start + d1.y + lane); wo = __ldg(win_off + d1.y + lane); }
    }
    while (have) {
      const int s = it % stages;
      const uint32_t ph = (uint32_t)((it / stages) & 1);
      const int nit = it + nprod;
      const int ntile = blockIdx.x + nit * gridDim.x;
      const bool nhave = ntile < ntiles;
      int4 nd0 = make_int4(0, 0, 0, 0), nd1 = make_int4(0, 0, 0, 0);
      if (nhave) {
        const int4 *dp = reinterpret_cast<const int4 *>(desc + ntile);
        nd0 = __ldg(dp); nd1 = __ldg(dp + 1);
      }
      const int64_t k0 = ((int64_t)(uint32_t)d0.x) | ((int64_t)d0.y << 32);
      const int cnt = d0.z, r0 = d0.w, Rraw = d1.x, wb = d1.y, nw = d1.z, xlen = d1.w;
      const int R = Rraw & 0x7fffffff;
      unsigned char *base = smem_raw + (size_t)s * stage_bytes;
      double *sval = reinterpret_cast<double *>(base);
      double *sx = reinterpret_cast<double *>(base + off_sx);
      RP *srp = reinterpret_cast<RP *>(base + off_srp);
      uint16_t *sidx = reinterpret_cast<uint16_t *>(base + off_sidx);
      int *meta = reinterpret_cast<int *>(base + off_meta);
      const int64_t k1 = k0 + cnt;
      const int64_t ka = k0 & ~(int64_t)kAlignMask;
      mbar_wait(&empty_bar[s], ph ^ 1u);
      if (lane == 0) {
        int64_t kend = (k1 + kAlignMask) & ~(int64_t)kAlignMask;
        const int64_t lim = nnz & ~(int64_t)kAlignMask;
        if (kend > lim) kend = lim;
        const int nb = (int)(kend - ka);
        int toff = 0;
        if (T3) {
          // lidx3 is padded by 16 entries, so the aligned window [ta, tend) never leaves the array
          const int64_t t0 = k0 / 3, ta = t0 & ~(int64_t)kAlignMask;
          const int64_t tend = (t0 + cnt / 3 + kAlignMask) & ~(int64_t)kAlignMask;
          const uint32_t ib = (uint32_t)(tend - ta) * 2u;
          toff = (int)(t0 - ta);
          mbar_expect_tx(&full_bar[s], (nb > 0 ? (uint32_t)nb * 8u : 0u) + ib);
          if (nb > 0) bulk_g2s(sval, val + ka, (uint32_t)nb * 8u, &full_bar[s], pol);
          if (ib > 0) bulk_g2s(sidx, lidx + ta, ib, &full_bar[s], pol);
        } else if (nb > 0) {
          mbar_expect_tx(&full_bar[s], (uint32_t)nb * 10u);
          bulk_g2s(sval, val + ka, (uint32_t)nb * 8u, &full_bar[s], pol);
          bulk_g2s(sidx, lidx + ka, (uint32_t)nb * 2u, &full_bar[s], pol);
        } else {
          mbar_arrive(&full_bar[s]);
        }
        meta[0] = r0; meta[1] = Rraw; meta[2] = tile; meta[3] = cnt;
        meta[4] = (int)(k0 & 0xffffffff); meta[5] = (int)(k0 >> 32); meta[6] = toff;
      }
      {
        const int64_t lim = nnz & ~(int64_t)kAlignMask;
        const int64_t kt = (lim > ka ? lim : ka) + lane;
        if (lane <= kAlignMask && kt >= lim && kt < k1) {
          sval[kt - ka] = val[kt];
          if (!T3) sidx[kt - ka] = lidx[kt];
        }
      }
      // raw row offsets and the x entries of the tile's own rows: asynchronous copies
      for (int i = lane; i <= R; i += 32) cp_async<sizeof(RP)>(srp + i, rowptr + r0 + i);
      // x windows (descriptor w broadcast from the lane that fetched it)
      for (int w0 = 0; w0 < nw; w0 += 32) {
        if (w0 > 0) {
          ws = 0; wo = 0;
          if (w0 + lane < nw) { ws = __ldg(win_start + wb + w0 + lane); wo = __ldg(win_off + wb + w0 + lane); }
        }
        const int nwc = min(32, nw - w0);
        const int wo_next = (w0 + nwc < nw) ? __ldg(win_off + wb + w0 + nwc) : xlen;
        for (int w = 0; w < nwc; ++w) {
          const int s0 = __shfl_sync(0xffffffffu, ws, w), o0 = __shfl_sync(0xffffffffu, wo, w);
          const int o1n = __shfl_sync(0xffffffffu, wo, (w + 1) & 31);
          const int len = ((w + 1 < nwc) ? o1n : wo_next) - o0;
          for (int t = lane; t < len; t += 32) cp_async<8>(sx + o0 + t, x + s0 + t);
        }
      }
      // window descriptors of the next tile (its descriptor was requested at the top of this iteration)
      int nws = 0, nwo = 0;
      if (nhave && lane < nd1.z) { nws = __ldg(win_start + nd1.y + lane); nwo = __ldg(win_off + nd1.y + lane); }
      cp_async_arrive_noinc(&full_bar[s]);       // fires when this lane's cp.async copies have landed
      __syncwarp();
      if (lane == 0) mbar_arrive(&full_bar[s]);  // release: meta / tail stores of the warp
      d0 = nd0; d1 = nd1; ws = nws; wo = nwo; it = nit; tile = ntile; have = nhave;
    }
    return;
  }

  // ================= consumer warps
  constexpr int G = (kConsWarps * 32) / LANES;
  const int gid = tid / LANES, gl = tid % LANES;
  double dsum = 0.0;
  for (int it = 0;; ++it) {
    const int tile = blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int s = it % stages;
    const uint32_t ph = (uint32_t)((it / stages) & 1);
    const unsigned char *base = smem_raw + (size_t)s * stage_bytes;
    const double *sval = reinterpret_cast<const double *>(base);
    const double *sx = reinterpret_cast<const double *>(base + off_sx);
    const RP *srp = reinterpret_cast<const RP *>(base + off_srp);
    const uint16_t *sidx = reinterpret_cast<const uint16_t *>(base + off_sidx);
    const int *meta = reinterpret_cast<const int *>(base + off_meta);
    mbar_wait(&full_bar[s], ph);
    const int r0 = meta[0], Rraw = meta[1], cnt = meta[3];
    const int64_t k0 = ((int64_t)(uint32_t)meta[4]) | ((int64_t)meta[5] << 32);
    const int64_t ka = k0 & ~(int64_t)kAlignMask;
    const int k0l = (int)(k0 - ka), k1l = k0l + cnt;
    const int R = Rraw & 0x7fffffff;
    const bool head = Rraw < 0;
    const uint16_t *sidt = sidx + (T3 ? meta[6] : 0);   // T3: triple t of the tile sits at sidt[t]
    const double *svt = sval + k0l;                     //     and its values at svt[3 t .. 3 t + 2]
    for (int i0 = 0; i0 < R; i0 += G) {  // CTA-uniform trip count (full-mask shuffles)
      const int i = i0 + gid;  // (rows 8 apart per half-warp pair was tried: fewer bank conflicts, but slower - loses the x broadcast)
      const bool live = i < R;
      int a = 0, e = 0;
      double xr = 0.0;
      if (DOT && live && gl == 0) xr = __ldg(x + r0 + i);  // consumed after the row loop: latency hidden
      if (live) {
        const int64_t va = (int64_t)srp[i] - ka, ve = (int64_t)srp[i + 1] - ka;
        a = (int)(va < k0l ? k0l : (va > k1l ? k1l : va));
        e = (int)(ve < k0l ? k0l : (ve > k1l ? k1l : ve));
      }
      double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
      if (T3) {
        // row segment in triples of the tile
        const int ta = (int)((unsigned)(a - k0l) / 3u), te = (int)((unsigned)(e - k0l) / 3u);
        double acc4 = 0.0, acc5 = 0.0;
        int t = ta + gl;
        for (; t + LANES < te; t += 2 * LANES) {
          const int ia = sidt[t], ib = sidt[t + LANES];
          const double *va = svt + 3 * t, *vb = svt + 3 * (t + LANES);
          const double xa0 = sx[ia], xa1 = sx[ia + 1], xa2 = sx[ia + 2];
          const double xb0 = sx[ib], xb1 = sx[ib + 1], xb2 = sx[ib + 2];
          acc0 = fma(va[0], xa0, acc0);
          acc1 = fma(va[1], xa1, acc1);
          acc2 = fma(va[2], xa2, acc2);
          acc3 = fma(vb[0], xb0, acc3);
          acc4 = fma(vb[1], xb1, acc4);
          acc5 = fma(vb[2], xb2, acc5);
        }
        if (t < te) {
          const int ia = sidt[t];
          const double *va = svt + 3 * t;
          acc0 = fma(va[0], sx[ia], acc0);
          acc1 = fma(va[1], sx[ia + 1], acc1);
          acc2 = fma(va[2], sx[ia + 2], acc2);
        }
        acc0 += acc3; acc1 += acc4; acc2 += acc5; acc3 = 0.0;
      } else {
        int j = a + gl;
        for (; j + 3 * LANES < e; j += 4 * LANES) {
          const double x0 = sx[sidx[j]], x1 = sx[sidx[j + LANES]], x2 = sx[sidx[j + 2 * LANES]], x3 = sx[sidx[j + 3 * LANES]];
          acc0 = fma(sval[j], x0, acc0);
          acc1 = fma(sval[j + LANES], x1, acc1);
          acc2 = fma(sval[j + 2 * LANES], x2, acc2);
          acc3 = fma(sval[j + 3 * LANES], x3, acc3);
        }
        for (; j < e; j += LANES) acc0 = fma(sval[j], sx[sidx[j]], acc0);
      }
      const double acc = group_sum<LANES>((acc0 + acc1) + (acc2 + acc3));
      if (live && gl == 0) {
        if (i == 0 && head) carry[tile] = acc;
        else y[r0 + i] = acc;
        if (DOT) dsum = fma(acc, xr, dsum);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }
  if (DOT) {
    // block reduction over the consumer warps only (named barrier 1)
    double v = warp_sum(dsum);
    if (lane == 0) red[warp] = v;
    named_bar_sync(1, kConsWarps * 32);
    if (warp == 0) {
      double t = lane < kConsWarps ? red[lane] : 0.0;
      t = warp_sum(t);
      if (lane == 0) dot_partials[blockIdx.x] = t;
    }
  }
}

// ------------------------------------------------------------------ node-block ("BSR-3") persistent kernels
// Same tiles, x windows, TMA / mbarrier ring and producer warps as k_spmv_persist; the tile is a whole number of nodes
// (3 rows with one column pattern of aligned triples).  Two consumers, one per plan kind, share the producer and the
// 3x3 block product, and sum every row in the same order - partials of the node's blocks in block order, from 0.0 - so
// that y and x.y are the same bits whichever one runs:
//   k_spmv_bsr3     streams the values; the tile is a flat list of 3x3 blocks, one block per consumer thread per pass:
//     phase 1   thread b: node i by binary search in the node offsets, ONE 16-bit staged position -> x triple (3 LDS),
//               9 values at stride 3 doubles across the lanes (conflict-free), 9 FMAs -> 3 row partials to shared memory;
//     phase 2   (after one named barrier, scratch double-buffered by tile parity) thread r < R adds the partials of its
//               row in block order -> y[r]: fixed summation order, bit-reproducible, no shuffles, no atomics.
//     Per 9 non-zeros: 13 shared-memory loads + 3 stores instead of 27 loads, and 8 + 2/9 bytes from HBM instead of 10.
//   k_spmv_bsr3_vd  value dictionary: the stage holds the tile's 16-bit block ids where it held val, and every CTA keeps
//     the nvd distinct blocks in shared memory; a warp owns a whole tile (see there).  4 + 2/9 bytes per block from HBM.
constexpr int kBsrMaxStages = 16;   // ring of the dictionary kernel (mbarrier pairs)
constexpr int kVdStride = 10;       // doubles per dictionary entry in shared memory: 9 values + 1 pad -> five 16-byte loads

// the three row partials of a 3x3 block (rows L doubles apart) times an x triple
__device__ __forceinline__ void block3_rows(const double *pv, int L, double x0, double x1, double x2, double &p0, double &p1,
                                            double &p2) {
  const double a0 = pv[0], a1 = pv[1], a2 = pv[2];
  const double b0 = pv[L], b1 = pv[L + 1], b2 = pv[L + 2];
  const double c0 = pv[2 * L], c1 = pv[2 * L + 1], c2 = pv[2 * L + 2];
  p0 = fma(a2, x2, fma(a1, x1, a0 * x0));
  p1 = fma(b2, x2, fma(b1, x1, b0 * x0));
  p2 = fma(c2, x2, fma(c1, x1, c0 * x0));
}

// stage of the node-block ring: sval[cap_nnz] f64 | sx[cap_x] f64 | snp[cap_nodes+2] i64 | sbidx[cap_blocks+16] u16 | meta[8] i32
//                         VD:                      sx[cap_x] f64 | snp[cap_nodes+2] i64 | swords[cap_words] u32        | meta
struct Bsr3Stage {
  size_t off_sx, off_snp, off_sb, off_meta;
};
template <bool VD>
__device__ __forceinline__ Bsr3Stage bsr3_stage(int cap_nnz, int cap_x, int cap_nodes, int cap_idx) {
  // cap_idx: block indices (u16) of a tile, or VD: words (u32) of a tile's slice of the run-compressed stream
  const size_t sb_bytes = VD ? (size_t)cap_idx * 4 : ((size_t)(cap_idx + 16) * 2 + 15) & ~(size_t)15;
  Bsr3Stage L;
  L.off_sx = VD ? 0 : (size_t)cap_nnz * 8;
  L.off_snp = L.off_sx + (size_t)cap_x * 8;
  L.off_sb = L.off_snp + (size_t)(cap_nodes + 2) * 8;
  L.off_meta = L.off_sb + sb_bytes;
  return L;
}

// producer warp p of nprod (tiles it = p, p + nprod, ...; stage it % stages, stages % nprod == 0): TMA val + block indices
// (VD: the tile's slice of the word stream, found through the tile id: tile_ids[k] for a permuted descriptor list, else k),
// cp.async node offsets + x windows.  The descriptor and the window descriptors of the NEXT tile are fetched while the
// current one is being issued.
template <bool VD, typename RP>
__device__ __forceinline__ void bsr3_produce(int p, int nprod, unsigned char *smem_raw, const Bsr3Stage &SL, int stages,
                                             int stage_bytes, uint64_t *full_bar, uint64_t *empty_bar,
                                             const RP *__restrict__ rowptr, const uint16_t *__restrict__ bidx,
                                             const double *__restrict__ val, const uint32_t *__restrict__ vwords,
                                             const int64_t *__restrict__ vtoff, const int *__restrict__ tile_ids,
                                             const double *__restrict__ x, const TileDesc *__restrict__ desc,
                                             const int *__restrict__ win_start, const int *__restrict__ win_off, int ntiles,
                                             int64_t nnz) {
  const int lane = threadIdx.x & 31;
  const uint64_t pol = l2_evict_first_policy();
  int it = p;
  int tile = blockIdx.x + it * gridDim.x;
  bool have = tile < ntiles;
  int4 d0 = make_int4(0, 0, 0, 0), d1 = make_int4(0, 0, 0, 0);
  int ws = 0, wo = 0;
  int64_t vw0 = 0, vw1 = 0;   // VD: word range of the tile
  auto word_range = [&](int k, int64_t &a, int64_t &b) {
    const int g = tile_ids != nullptr ? __ldg(tile_ids + k) : k;
    a = __ldg(vtoff + g); b = __ldg(vtoff + g + 1);
  };
  if (have) {
    const int4 *dp = reinterpret_cast<const int4 *>(desc + tile);
    d0 = __ldg(dp); d1 = __ldg(dp + 1);
    if (lane < d1.z) { ws = __ldg(win_start + d1.y + lane); wo = __ldg(win_off + d1.y + lane); }
    if (VD) word_range(tile, vw0, vw1);
  }
  while (have) {
    const int s = it % stages;
    const uint32_t ph = (uint32_t)((it / stages) & 1);
    const int nit = it + nprod;
    const int ntile = blockIdx.x + nit * gridDim.x;
    const bool nhave = ntile < ntiles;
    int4 nd0 = make_int4(0, 0, 0, 0), nd1 = make_int4(0, 0, 0, 0);
    int64_t nvw0 = 0, nvw1 = 0;
    if (nhave) {
      const int4 *dp = reinterpret_cast<const int4 *>(desc + ntile);
      nd0 = __ldg(dp); nd1 = __ldg(dp + 1);
      if (VD) word_range(ntile, nvw0, nvw1);
    }
    const int64_t k0 = ((int64_t)(uint32_t)d0.x) | ((int64_t)d0.y << 32);
    const int cnt = d0.z, r0 = d0.w, R = d1.x & 0x3fffffff, uni = (d1.x >> 30) & 1, wb = d1.y, nw = d1.z, xlen = d1.w;
    unsigned char *base = smem_raw + (size_t)s * stage_bytes;
    double *sval = reinterpret_cast<double *>(base);
    double *sx = reinterpret_cast<double *>(base + SL.off_sx);
    RP *snp = reinterpret_cast<RP *>(base + SL.off_snp);
    uint16_t *sb = reinterpret_cast<uint16_t *>(base + SL.off_sb);
    int *meta = reinterpret_cast<int *>(base + SL.off_meta);
    const int64_t k1 = k0 + cnt;
    const int64_t ka = k0 & ~(int64_t)kAlignMask;
    mbar_wait(&empty_bar[s], ph ^ 1u);
    if (lane == 0) {
      // bidx is padded by 16 entries, vwords by 8: the aligned windows [ba, bend) and [wa, wend) never leave the arrays
      const int64_t b0 = k0 / 9, ba = b0 & ~(int64_t)kAlignMask;
      const int64_t bend = (b0 + cnt / 9 + kAlignMask) & ~(int64_t)kAlignMask;
      const uint32_t ib = (uint32_t)(bend - ba) * 2u;
      int sofs = (int)(b0 - ba);
      if (VD) {
        const int64_t wa = vw0 & ~(int64_t)3, wend = (vw1 + 3) & ~(int64_t)3;   // every tile has a header word: wend > wa
        const uint32_t wb = (uint32_t)(wend - wa) * 4u;
        sofs = (int)(vw0 - wa);
        mbar_expect_tx(&full_bar[s], wb);
        bulk_g2s(sb, vwords + wa, wb, &full_bar[s], pol);
      } else {
        int64_t kend = (k1 + kAlignMask) & ~(int64_t)kAlignMask;
        const int64_t lim = nnz & ~(int64_t)kAlignMask;
        if (kend > lim) kend = lim;
        const int nb = (int)(kend - ka);
        mbar_expect_tx(&full_bar[s], (nb > 0 ? (uint32_t)nb * 8u : 0u) + ib);
        if (nb > 0) bulk_g2s(sval, val + ka, (uint32_t)nb * 8u, &full_bar[s], pol);
        if (ib > 0) bulk_g2s(sb, bidx + ba, ib, &full_bar[s], pol);
      }
      meta[0] = r0; meta[1] = R; meta[2] = tile; meta[3] = cnt;
      meta[4] = (int)(k0 & 0xffffffff); meta[5] = (int)(k0 >> 32); meta[6] = sofs; meta[7] = uni;
    }
    if (!VD) {
      const int64_t lim = nnz & ~(int64_t)kAlignMask;
      const int64_t kt = (lim > ka ? lim : ka) + lane;
      if (lane <= kAlignMask && kt >= lim && kt < k1) sval[kt - ka] = val[kt];
    }
    // offsets of the first row of every node of the tile (+ the end): asynchronous copies
    for (int i = lane; i <= R / 3; i += 32) cp_async<sizeof(RP)>(snp + i, rowptr + r0 + 3 * i);
    for (int w0 = 0; w0 < nw; w0 += 32) {
      if (w0 > 0) {
        ws = 0; wo = 0;
        if (w0 + lane < nw) { ws = __ldg(win_start + wb + w0 + lane); wo = __ldg(win_off + wb + w0 + lane); }
      }
      const int nwc = min(32, nw - w0);
      const int wo_next = (w0 + nwc < nw) ? __ldg(win_off + wb + w0 + nwc) : xlen;
      for (int w = 0; w < nwc; ++w) {
        const int s0 = __shfl_sync(0xffffffffu, ws, w), o0 = __shfl_sync(0xffffffffu, wo, w);
        const int o1n = __shfl_sync(0xffffffffu, wo, (w + 1) & 31);
        const int len = ((w + 1 < nwc) ? o1n : wo_next) - o0;
        for (int t = lane; t < len; t += 32) cp_async<8>(sx + o0 + t, x + s0 + t);
      }
    }
    int nws = 0, nwo = 0;
    if (nhave && lane < nd1.z) { nws = __ldg(win_start + nd1.y + lane); nwo = __ldg(win_off + nd1.y + lane); }
    cp_async_arrive_noinc(&full_bar[s]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&full_bar[s]);
    d0 = nd0; d1 = nd1; ws = nws; wo = nwo; vw0 = nvw0; vw1 = nvw1; it = nit; tile = ntile; have = nhave;
  }
}

template <bool DOT, int CW, typename RP>
__global__ void __launch_bounds__((CW + 4) * 32)
k_spmv_bsr3(const RP *__restrict__ rowptr, const uint16_t *__restrict__ bidx, const double *__restrict__ val,
            const double *__restrict__ x, double *__restrict__ y, const TileDesc *__restrict__ desc,
            const int *__restrict__ win_start, const int *__restrict__ win_off, int ntiles, int64_t nnz, int cap_nnz,
            int cap_nodes, int cap_x, int cap_blocks, int stages, int stage_bytes, int mode, double *__restrict__ dot_partials,
            const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t full_bar[8], empty_bar[8];
  __shared__ double red[32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nprod = (int)(blockDim.x >> 5) - CW;   // producer warps; stages % nprod == 0

  if (tid == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 34); mbar_init(&empty_bar[s], CW); }
    mbar_fence_init();
  }
  __syncthreads();

  const Bsr3Stage SL = bsr3_stage<false>(cap_nnz, cap_x, cap_nodes, cap_blocks);
  // scratch behind the stages: row partials [2][3*cap_blocks] f64, node block offsets [2][cap_nodes+2] i32
  // (tried and rejected: a warp-segmented scan that leaves only a few partials per tile - no 25 KB scratch, larger stages - but
  //  35 shuffles per pass; 8 lanes per row in phase 2 serialises the two phases)
  // mode bit 1 (default): the row partials of a block OVERWRITE the block's own first-row values in the stage (the thread has all
  // nine values in registers by then) - no separate scratch, which buys a third stage per CTA; the stage is handed back to
  // the producer only after phase 2 has read the partials.
  const bool inplace = (mode & 2) != 0;
  const int part_len = inplace ? 0 : 3 * cap_blocks;
  double *spart = reinterpret_cast<double *>(smem_raw + (size_t)stages * stage_bytes);
  int *snbo = reinterpret_cast<int *>(spart + (size_t)2 * part_len);

  if (warp >= CW) {
    bsr3_produce<false, RP>(warp - CW, nprod, smem_raw, SL, stages, stage_bytes, full_bar, empty_bar, rowptr, bidx, val, nullptr,
                            nullptr, nullptr, x, desc, win_start, win_off, ntiles, nnz);
    return;
  }

  // ================= consumer warps (CW * 32 threads, tid = consumer thread id)
  constexpr int NT = CW * 32;
  double dsum = 0.0;
  for (int it = 0;; ++it) {
    const int tile = blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int s = it % stages;
    const uint32_t ph = (uint32_t)((it / stages) & 1);
    const int par = it & 1;
    const unsigned char *base = smem_raw + (size_t)s * stage_bytes;
    const double *sval = reinterpret_cast<const double *>(base);
    const double *sx = reinterpret_cast<const double *>(base + SL.off_sx);
    const RP *snp = reinterpret_cast<const RP *>(base + SL.off_snp);
    const uint16_t *sb = reinterpret_cast<const uint16_t *>(base + SL.off_sb);
    const int *meta = reinterpret_cast<const int *>(base + SL.off_meta);
    double *part = spart + (size_t)par * part_len;
    int *nbo = snbo + par * (cap_nodes + 2);
    mbar_wait(&full_bar[s], ph);
    const int r0 = meta[0], R = meta[1], cnt = meta[3];
    const int64_t k0 = ((int64_t)(uint32_t)meta[4]) | ((int64_t)meta[5] << 32);
    const int k0l = (int)(k0 & kAlignMask);
    const int NN = R / 3, NB = cnt / 9;
    const uint16_t *sbt = sb + meta[6];
    const double *svt = sval + k0l;
    // uniform tile (all nodes have the same number of blocks - the interior of a structured mesh): node = b / Lb, no look-ups
    const bool uni = (mode & 1) != 0 && meta[7] != 0 && NN > 0 && NB >= 2 * NN;   // (>= 2 blocks per node: the reciprocal fits 32 bits)
    const int Lbu = uni ? NB / NN : 0;
    const unsigned magic = uni ? (unsigned)((0xffffffffull + (unsigned)Lbu) / (unsigned)Lbu) : 0u;   // b / Lbu = (b * magic) >> 32 for b < 2^16
    // block offset of every node (kept for phase 2, which runs after the stage has been handed back)
    for (int i = tid; i <= NN; i += NT) nbo[i] = uni ? i * Lbu : (int)((int64_t)snp[i] - k0) / 9;
    // ---- phase 1: one 3x3 block per thread and pass
    for (int b = tid; b < NB; b += NT) {
      int noff, t3, L;
      if (uni) {
        const int i = (int)__umulhi((unsigned)b, magic);
        noff = i * 9 * Lbu; L = 3 * Lbu; t3 = 3 * (b - i * Lbu);
      } else {
        int lo = 0, hi = NN - 1;                     // node of block b: last i with (snp[i] - k0) <= 9 b
        const int kb = 9 * b;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if ((int)((int64_t)snp[mid] - k0) <= kb) lo = mid; else hi = mid - 1;
        }
        noff = (int)((int64_t)snp[lo] - k0);
        L = ((int)((int64_t)snp[lo + 1] - k0) - noff) / 3;   // non-zeros per row of this node
        t3 = (kb - noff) / 3;                                  // 3 t, t = b - noff / 9
      }
      const double *pv = svt + noff + t3;
      const int ii = sbt[b];
      double p0, p1, p2;
      block3_rows(pv, L, sx[ii], sx[ii + 1], sx[ii + 2], p0, p1, p2);
      double *pp = inplace ? const_cast<double *>(pv) : part + 3 * b;   // in place: positions 3t..3t+2 of the node's first row
      pp[0] = p0; pp[1] = p1; pp[2] = p2;
    }
    const bool has_rows = warp * 32 < R;            // this warp owns rows in phase 2
    if (!inplace || !has_rows) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);   // nothing more to read from the stage for this warp
    }
    named_bar_sync(1, NT);
    // ---- phase 2: one row per thread, partials added in block order.  Only the first warp(s) are busy here; the others
    //      already wait for / start on the next tile, so this overlaps with the next phase 1.
    for (int r = tid; r < R; r += NT) {
      const int i = r / 3, k = r - 3 * i;
      const int b0 = nbo[i], b1 = nbo[i + 1];
      double acc = 0.0;
      if (inplace) {
        const double *pr = svt + 9 * b0 + k;       // first row of node i: partial k of block t at 3 t + k
        for (int t = 0; t < b1 - b0; ++t) acc += pr[3 * t];
      } else {
        for (int b = b0; b < b1; ++b) acc += part[3 * b + k];
      }
      y[r0 + r] = acc;
      if (DOT) dsum = fma(acc, __ldg(x + r0 + r), dsum);
    }
    if (inplace && has_rows) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes to the stage before the next TMA fill
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }
  }
  if (DOT) {
    double v = warp_sum(dsum);
    if (lane == 0) red[warp] = v;
    named_bar_sync(1, NT);
    if (warp == 0) {
      double t = lane < CW ? red[lane] : 0.0;
      t = warp_sum(t);
      if (lane == 0) dot_partials[blockIdx.x] = t;
    }
  }
}

// Value-dictionary consumer.  The CTA takes its tiles (it = 0, 1, ... -> tile blockIdx.x + it * gridDim.x, as above) in
// groups of G consecutive ones:
//     phase A   warp g < G owns tile g of the group, with no CTA barrier: lane <-> node, the lane walks the node's blocks
//               in block order and keeps the three row sums in registers (acc += the block's row partial, from 0.0 - the
//               partial and the sum of k_spmv_bsr3 exactly), writes them to the group's y buffer and hands the stage back;
//     phase B   after ONE named barrier per group, the tiles of the group in tile order, thread r < R of the NT = CW * 32
//               consumer threads storing row r and adding x.y as k_spmv_bsr3's phase 2 does.
// So every consumer thread sees the same rows in the same order as there: y and every per-CTA x.y partial are the same
// bits, and G only sets how many stages are in flight.  The tile's index stream (k_vd_runs) is a segment list and block
// words (staged position | id << 16): a lane in a run segment reads its head's words, position + 3 per node after the
// head, so its word and dictionary loads are warp-wide broadcasts; a lane in an explicit segment reads its node's own words.
// Per 32 blocks (one warp step): one word load, 3 x loads at stride 3 doubles and five 16-byte dictionary loads.
// The y buffers are double-buffered by group parity: the barrier of group n + 1 orders phase B of group n before phase A
// of group n + 2.
template <bool DOT, int CW, typename RP>
__global__ void __launch_bounds__((CW + 4) * 32, 2)
k_spmv_bsr3_vd(const RP *__restrict__ rowptr, const uint32_t *__restrict__ vwords, const int64_t *__restrict__ vtoff,
               const int *__restrict__ tile_ids, const double *__restrict__ vdict, int nvd, const double *__restrict__ x,
               double *__restrict__ y, const TileDesc *__restrict__ desc, const int *__restrict__ win_start,
               const int *__restrict__ win_off, int ntiles, int cap_nodes, int cap_x, int cap_words, int stages, int stage_bytes,
               int group, double *__restrict__ dot_partials, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t full_bar[kBsrMaxStages], empty_bar[kBsrMaxStages];
  __shared__ int2 grows[2][kBsrMaxStages];   // (r0, R) of the tiles of a group, by group parity
  __shared__ double red[32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nprod = (int)(blockDim.x >> 5) - CW;   // producer warps; stages % nprod == 0, group <= stages

  if (tid == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 34); mbar_init(&empty_bar[s], 1); }
    mbar_fence_init();
  }
  __syncthreads();

  const Bsr3Stage SL = bsr3_stage<true>(0, cap_x, cap_nodes, cap_words);
  // behind the stages: y buffers [2][group][3 * cap_nodes] f64, then the dictionary [nvd][kVdStride] f64 (16 B aligned)
  const int ylen = 3 * cap_nodes;
  double *sy = reinterpret_cast<double *>(smem_raw + (size_t)stages * stage_bytes);
  double *sdict = sy + (size_t)2 * group * ylen;

  if (warp >= CW) {
    bsr3_produce<true, RP>(warp - CW, nprod, smem_raw, SL, stages, stage_bytes, full_bar, empty_bar, rowptr, nullptr, nullptr,
                           vwords, vtoff, tile_ids, x, desc, win_start, win_off, ntiles, 0);
    return;
  }

  constexpr int NT = CW * 32;
  // the dictionary, once per launch (from L2 after the first CTAs), while the producers fill the first stages
  for (int i = tid; i < kVdStride * nvd; i += NT) {
    const int e = i / kVdStride, c = i - kVdStride * e;
    sdict[i] = c < 9 ? __ldg(vdict + 9 * e + c) : 0.0;
  }
  named_bar_sync(1, NT);
  double dsum = 0.0;
  for (int g0 = 0; blockIdx.x + g0 * gridDim.x < ntiles; g0 += group) {
    const int par = (g0 / group) & 1;
    double *yg = sy + (size_t)par * group * ylen;
    // ---- phase A: warp g takes tile g0 + g of the group
    if (warp < group) {
      const int it = g0 + warp;
      const int tile = blockIdx.x + it * gridDim.x;
      if (tile < ntiles) {
        const int s = it % stages;
        const unsigned char *base = smem_raw + (size_t)s * stage_bytes;
        const double *sx = reinterpret_cast<const double *>(base + SL.off_sx);
        const RP *snp = reinterpret_cast<const RP *>(base + SL.off_snp);
        const int *meta = reinterpret_cast<const int *>(base + SL.off_meta);
        mbar_wait(&full_bar[s], (uint32_t)((it / stages) & 1));
        const int r0 = meta[0], R = meta[1];
        const int64_t k0 = ((int64_t)(uint32_t)meta[4]) | ((int64_t)meta[5] << 32);
        const uint32_t *swt = reinterpret_cast<const uint32_t *>(base + SL.off_sb) + meta[6];
        const int nseg = (int)swt[0];
        double *yt = yg + warp * ylen;
        for (int i = lane; i < R / 3; i += 32) {
          const int b0 = (int)((int64_t)snp[i] - k0) / 9, b1 = (int)((int64_t)snp[i + 1] - k0) / 9;
          int q = 0;   // segment of node i: the last one that starts at or before it
          for (int k = 1; k < nseg; ++k) q = (int)(swt[1 + 2 * k] & 0x7fffffffu) <= i ? k : q;
          const uint32_t head = swt[1 + 2 * q];
          const int sbase = (int)swt[2 + 2 * q];
          const bool run = (head >> 31) != 0;
          const uint32_t *wt = swt + sbase + (run ? 0 : b0);   // words of block 0 of the node (run: of its head)
          const int dpos = run ? 3 * (i - (int)(head & 0x7fffffffu)) : 0;
          double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0;
#pragma unroll 2
          for (int t = 0; t < b1 - b0; ++t) {
            const uint32_t w = wt[t];
            const int ii = (int)(w & 0xffffu) + dpos;
            const double2 *pv = reinterpret_cast<const double2 *>(sdict + kVdStride * (int)(w >> 16));
            const double2 v01 = pv[0], v23 = pv[1], v45 = pv[2], v67 = pv[3], v8 = pv[4];
            const double x0 = sx[ii], x1 = sx[ii + 1], x2 = sx[ii + 2];
            acc0 += fma(v23.x, x2, fma(v01.y, x1, v01.x * x0));
            acc1 += fma(v45.y, x2, fma(v45.x, x1, v23.y * x0));
            acc2 += fma(v8.x, x2, fma(v67.y, x1, v67.x * x0));
          }
          yt[3 * i] = acc0; yt[3 * i + 1] = acc1; yt[3 * i + 2] = acc2;
        }
        if (lane == 0) grows[par][warp] = make_int2(r0, R);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      }
    }
    named_bar_sync(1, NT);
    // ---- phase B: the tiles of the group in order, one row per consumer thread
    for (int g = 0; g < group && blockIdx.x + (g0 + g) * gridDim.x < ntiles; ++g) {
      const int2 rr = grows[par][g];
      const double *yt = yg + g * ylen;
      for (int r = tid; r < rr.y; r += NT) {
        const double acc = yt[r];
        y[rr.x + r] = acc;
        if (DOT) dsum = fma(acc, __ldg(x + rr.x + r), dsum);
      }
    }
  }
  if (DOT) {
    double v = warp_sum(dsum);
    if (lane == 0) red[warp] = v;
    named_bar_sync(1, NT);
    if (warp == 0) {
      double t = lane < CW ? red[lane] : 0.0;
      t = warp_sum(t);
      if (lane == 0) dot_partials[blockIdx.x] = t;
    }
  }
}

// ---- node-block plan helpers
// bit 30 of TileDesc.R: every row of the tile has the same length (uniform nodes -> no per-block node search in the kernel)
template <typename RP>
__global__ void k_mark_uniform(const RP *__restrict__ rowptr, TileDesc *__restrict__ desc, int ntiles, int *__restrict__ count) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= ntiles) return;
  const int r0 = desc[b].r0, R = desc[b].R & 0x3fffffff;
  if (R <= 0) return;
  const int64_t L0 = (int64_t)rowptr[r0 + 1] - (int64_t)rowptr[r0];
  bool uni = true;
  for (int i = 1; i < R; ++i) uni = uni && ((int64_t)rowptr[r0 + i + 1] - (int64_t)rowptr[r0 + i] == L0);
  if (uni) { desc[b].R |= 0x40000000; atomicAdd(count, 1); }
}

// eligibility: rows 3n, 3n+1, 3n+2 have one length (a multiple of 3) and one column pattern made of aligned consecutive triples
template <typename RP>
__global__ void k_check_bsr3(const RP *__restrict__ rowptr, const int *__restrict__ col, int64_t nnodes, int *__restrict__ fail,
                             unsigned long long *__restrict__ same_as_next) {
  for (int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; n < nnodes; n += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a0 = rowptr[3 * n], a1 = rowptr[3 * n + 1], a2 = rowptr[3 * n + 2], a3 = rowptr[3 * n + 3];
    const int64_t L = a1 - a0;
    if (a2 - a1 != L || a3 - a2 != L || L % 3 != 0) { *fail = 1; return; }
    // regularity of the mesh: how many nodes have as many blocks as their successor (structured meshes: almost all)
    if (n + 1 < nnodes && (int64_t)rowptr[3 * n + 4] - a3 == L) atomicAdd(same_as_next, 1ull);
    for (int64_t t = 0; t < L; t += 3) {
      const int c = col[a0 + t];
      if (col[a0 + t + 1] != c + 1 || col[a0 + t + 2] != c + 2) { *fail = 1; return; }
      if (col[a1 + t] != c || col[a2 + t] != c || col[a1 + t + 1] != c + 1 || col[a1 + t + 2] != c + 2 ||
          col[a2 + t + 1] != c + 1 || col[a2 + t + 2] != c + 2) { *fail = 1; return; }
    }
  }
}
// one 16-bit staged position per 3x3 block from the per-non-zero positions of the same tiles (rows of a node agree)
template <typename RP>
__global__ void k_build_bidx(const RP *__restrict__ rowptr, const uint16_t *__restrict__ lidx, int64_t nnodes,
                             uint16_t *__restrict__ bidx, int *__restrict__ fail) {
  for (int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; n < nnodes; n += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a0 = rowptr[3 * n], a1 = rowptr[3 * n + 1], a2 = rowptr[3 * n + 2];
    const int64_t L = a1 - a0;
    for (int64_t t = 0; t < L; t += 3) {
      const unsigned p = lidx[a0 + t];
      if (lidx[a0 + t + 1] != p + 1 || lidx[a0 + t + 2] != p + 2 || lidx[a1 + t] != p || lidx[a2 + t] != p) *fail = 1;
      bidx[a0 / 9 + t / 3] = (uint16_t)p;   // a0 % 9 == 0: blocks before node n = rowptr[3n] / 9
    }
  }
}

// ---- value dictionary plan helpers
// A block is keyed by its nine values as uint64 bit patterns (-0.0 and 0.0, or two NaN payloads, are different blocks).  A
// table slot holds the smallest (first-row position k << 24 | row length L) of the blocks with that value, so that the
// representative is the first occurrence whatever the order the threads arrive in: slots only go EMPTY -> key (CAS) and then
// down (atomicMin among equal blocks), so a stale non-empty read still names the right value.
constexpr unsigned long long kVdEmpty = ~0ull;
__device__ __forceinline__ void vd_block_bits(const double *__restrict__ val, int64_t k, int64_t L, unsigned long long w[9]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) w[3 * r + c] = (unsigned long long)__double_as_longlong(__ldg(val + k + r * L + c));
}
template <typename RP>
__global__ void k_vdict_insert(const RP *__restrict__ rowptr, const double *__restrict__ val, int64_t nnodes,
                               unsigned long long *__restrict__ table, uint16_t *__restrict__ bvid, int *__restrict__ count,
                               int *__restrict__ fail) {
  for (int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; n < nnodes; n += (int64_t)gridDim.x * blockDim.x) {
    if (*(volatile int *)fail) return;
    const int64_t a0 = rowptr[3 * n], L = (int64_t)rowptr[3 * n + 1] - a0;
    for (int64_t t3 = 0; t3 < L; t3 += 3) {
      unsigned long long w[9];
      vd_block_bits(val, a0 + t3, L, w);
      unsigned long long h = 0x9e3779b97f4a7c15ull;
#pragma unroll
      for (int j = 0; j < 9; ++j) { h ^= w[j]; h *= 0xff51afd7ed558ccdull; h ^= h >> 32; }
      const unsigned long long key = ((unsigned long long)(a0 + t3) << 24) | (unsigned long long)L;
      int probe = 0, slot = (int)(h & (kVdictSlots - 1));
      for (;; ++probe, slot = (slot + 1) & (kVdictSlots - 1)) {
        if (probe == kVdictSlots) { atomicExch(fail, 2); return; }
        unsigned long long v = *(volatile unsigned long long *)(table + slot);
        if (v == kVdEmpty) {
          v = atomicCAS(table + slot, kVdEmpty, key);
          if (v == kVdEmpty) {
            if (atomicAdd(count, 1) >= kVdictMax) { atomicExch(fail, 1); return; }
            break;
          }
        }
        unsigned long long u[9];
        vd_block_bits(val, (int64_t)(v >> 24), (int64_t)(v & 0xffffff), u);
        bool eq = true;
#pragma unroll
        for (int j = 0; j < 9; ++j) eq = eq && u[j] == w[j];
        if (eq) {
          if (key < v) atomicMin(table + slot, key);
          break;
        }
      }
      bvid[a0 / 9 + t3 / 3] = (uint16_t)slot;   // slot for now; k_vdict_finish maps it to the id
    }
  }
}
// slot -> id over all blocks, and the dictionary itself from the representatives (keys in id order)
__global__ void k_vdict_finish(uint16_t *__restrict__ bvid, int64_t nblk, const uint16_t *__restrict__ slot_id,
                               const double *__restrict__ val, const unsigned long long *__restrict__ rep, int nd,
                               double *__restrict__ vdict) {
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < nblk; g += (int64_t)gridDim.x * blockDim.x)
    bvid[g] = slot_id[bvid[g]];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 9 * nd) {
    const unsigned long long v = rep[i / 9];
    const int r = (i % 9) / 3, c = i % 3;
    vdict[i] = val[(int64_t)(v >> 24) + r * (int64_t)(v & 0xffffff) + c];
  }
}

// ---- run-compressed index stream of the dictionary kernel
// Within a tile, node i joins the run of node i - 1 when it has as many blocks and, block for block, the staged position
// + 3 and the same dictionary id (a structured mesh along its fastest axis).  The tile's slice of the stream is
//     nseg | nseg x (first node | run << 31, word base) | block words (bidx | bvid << 16)
// A run segment (a head and >= 1 node joining it) stores the head's words once at base; an explicit segment stores the
// words of all its nodes, node i's at base + (its first block in the tile).  More than kVdSegCap segments: the whole tile
// is one explicit segment.  words == nullptr: count only (words per tile -> tile_words, nodes in runs -> run_nodes).
constexpr int kVdSegCap = 8;
template <typename RP>
__global__ void k_vd_runs(const RP *__restrict__ rowptr, const TileDesc *__restrict__ desc, int ntiles,
                          const uint16_t *__restrict__ bidx, const uint16_t *__restrict__ bvid, const int64_t *__restrict__ vtoff,
                          uint32_t *__restrict__ words, int64_t *__restrict__ tile_words, unsigned long long *__restrict__ run_nodes) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= ntiles) return;
  const int64_t n0 = desc[b].r0 / 3;
  const int NN = (desc[b].R & 0x3fffffff) / 3;
  const int64_t kb0 = (int64_t)rowptr[3 * n0] / 9;   // first block of the tile
  auto blk = [&](int i) { return (int64_t)rowptr[3 * (n0 + i)] / 9; };
  auto joins = [&](int i) {   // node i (0 < i < NN) joins the run of node i - 1
    const int64_t a = blk(i - 1), c = blk(i), e = blk(i + 1);
    if (e - c != c - a) return false;
    for (int64_t t = 0; t < e - c; ++t)
      if ((unsigned)bidx[c + t] != (unsigned)bidx[a + t] + 3u || bvid[c + t] != bvid[a + t]) return false;
    return true;
  };
  int sfirst[kVdSegCap], nseg = 0;
  unsigned srun = 0;   // bit k: segment k is a run
  bool over = false;
  int64_t covered = 0;
  bool jcur = false, jnext = NN > 1 && joins(1);
  for (int i = 0; i < NN && !over; ++i) {
    const bool j = jcur;
    jcur = jnext;                                 // joins(i + 1)
    jnext = i + 2 < NN && joins(i + 2);
    if (j) { ++covered; continue; }               // in the current run
    const bool head = jcur;                       // starts a run
    if (!head && nseg > 0 && !((srun >> (nseg - 1)) & 1u)) continue;   // extends the current explicit segment
    if (nseg == kVdSegCap) { over = true; break; }
    sfirst[nseg] = i;
    if (head) { srun |= 1u << nseg; ++covered; }
    ++nseg;
  }
  if (over) { nseg = NN > 0 ? 1 : 0; sfirst[0] = 0; srun = 0; covered = 0; }
  // words: header, then per segment the head's blocks (run) or all its nodes' blocks (explicit)
  int64_t nw = 1 + 2 * nseg;
  for (int k = 0; k < nseg; ++k) {
    const int f = sfirst[k], l = k + 1 < nseg ? sfirst[k + 1] : NN;
    nw += ((srun >> k) & 1u) ? blk(f + 1) - blk(f) : blk(l) - blk(f);
  }
  if (words == nullptr) {
    tile_words[b] = nw;
    if (covered) atomicAdd(run_nodes, (unsigned long long)covered);
    return;
  }
  uint32_t *w = words + vtoff[b];
  w[0] = (uint32_t)nseg;
  int64_t o = 1 + 2 * nseg;
  for (int k = 0; k < nseg; ++k) {
    const int f = sfirst[k], l = k + 1 < nseg ? sfirst[k + 1] : NN;
    const bool run = (srun >> k) & 1u;
    const int64_t c0 = blk(f), c1 = run ? blk(f + 1) : blk(l);
    w[1 + 2 * k] = (uint32_t)f | (run ? 0x80000000u : 0u);
    w[2 + 2 * k] = (uint32_t)(int)(run ? o : o - (c0 - kb0));   // explicit: node i's words at base + (its block - kb0)
    for (int64_t t = c0; t < c1; ++t) w[o + t - c0] = (uint32_t)bidx[t] | ((uint32_t)bvid[t] << 16);
    o += c1 - c0;
  }
}

// ---- T3 plan helpers
// every row offset a multiple of 3  <=>  every row length a multiple of 3 (rowptr[0] = 0)
template <typename RP>
__global__ void k_rows_mod3(const RP *__restrict__ rowptr, int64_t nrows, int *__restrict__ fail) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= nrows; r += (int64_t)gridDim.x * blockDim.x)
    if (((int64_t)rowptr[r]) % 3 != 0) { *fail = 1; return; }
}
// one 16-bit staged position per aligned triple; fails unless the three positions are consecutive
__global__ void k_build_idx3(const uint16_t *__restrict__ lidx, int64_t ntrip, uint16_t *__restrict__ lidx3, int *__restrict__ fail) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < ntrip; t += (int64_t)gridDim.x * blockDim.x) {
    const unsigned a = lidx[3 * t], b = lidx[3 * t + 1], c = lidx[3 * t + 2];
    if (b != a + 1 || c != a + 2) *fail = 1;
    lidx3[t] = (uint16_t)a;
  }
}

// ---- interface-first split: flag the tiles that own at least one marked row
__global__ void k_mark_rows(const int *__restrict__ rows, int64_t count, unsigned char *__restrict__ rowflag) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < count) rowflag[rows[i]] = 1;
}
__global__ void k_flag_tiles(const TileDesc *__restrict__ desc, int ntiles, const unsigned char *__restrict__ rowflag,
                             unsigned char *__restrict__ tileflag) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= ntiles) return;
  const int r0 = desc[b].r0, R = desc[b].R & 0x3fffffff;   // bit 31: head continuation, bit 30: uniform nodes
  unsigned char f = 0;
  for (int i = 0; i < R; ++i) f |= rowflag[r0 + i];
  tileflag[b] = f;
}
__global__ void k_gather_desc(const TileDesc *__restrict__ desc, const int *__restrict__ perm, int ntiles, TileDesc *__restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < ntiles) out[b] = desc[perm[b]];
}

// rows that span several tiles: y[row] (written by the tile where the row starts) += carries, in tile order
__global__ void k_spmv_fixup(double *__restrict__ y, const double *__restrict__ carry, const int *__restrict__ fix_row,
                             const int *__restrict__ fix_first, const int *__restrict__ fix_cnt, int nfix) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nfix) return;
  const int row = fix_row[f], first = fix_first[f], cnt = fix_cnt[f];
  double s = y[row];
  for (int t = 0; t < cnt; ++t) s += carry[first + t];
  y[row] = s;
}

template <typename RP>
__global__ void k_csr_diag(const RP *__restrict__ rowptr, const int *__restrict__ col, const double *__restrict__ val,
                           int64_t nrows, double *__restrict__ diag) {
  // one 8-lane group per row
  const int64_t gidx = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 3;
  const int gl = threadIdx.x & 7;
  if (gidx >= nrows) return;
  double d = 0.0;
  for (int64_t k = (int64_t)rowptr[gidx] + gl; k < (int64_t)rowptr[gidx + 1]; k += 8)
    if (col[k] == gidx) d += val[k];
  d = group_sum<8>(d);
  if (gl == 0) diag[gidx] = d;
}

// ------------------------------------------------------------------ host side
inline int spmv_configure(const CsrPlan &P);
inline int env_int(const char *name, int dflt) {
  const char *s = getenv(name);
  return (s && *s) ? atoi(s) : dflt;
}

inline void free_plan(CsrPlan &P);

// device temporaries of the plan builder: freed on every exit path (the PCGB_CUDA macro returns early on errors)
struct DevTmp {
  void *p = nullptr;
  ~DevTmp() { if (p) cudaFree(p); }
  template <typename T> T *as() const { return static_cast<T *>(p); }
};

// Value dictionary of a node-block matrix (P.vd = D distinct blocks, P.bvid, P.vdict), or P.vd = 0 when it has more than
// kVdictMax distinct blocks.  Ids follow the first occurrence of each value, so the plan is deterministic.  mode 1 also
// refuses a dictionary that the grid's CTAs would load (once each per launch) in more bytes than half the values it replaces.
template <typename RP>
inline int build_vdict(CsrPlan &P, cudaStream_t st, int mode, int grid) {
  P.vd = 0;
  const int64_t nblk = P.nnz / 9, nnodes = P.nrows / 3;
  if (nblk == 0 || P.nnz >= (int64_t(1) << 40) || P.max_row >= (1 << 24)) return PCGB_OK;   // key = k << 24 | L
  DevTmp t_table, t_ctl, t_map;
  PCGB_CUDA(cudaMalloc(&t_table.p, kVdictSlots * sizeof(unsigned long long)));
  PCGB_CUDA(cudaMalloc(&t_ctl.p, 2 * sizeof(int)));
  PCGB_CUDA(cudaMemsetAsync(t_table.p, 0xff, kVdictSlots * sizeof(unsigned long long), st));
  PCGB_CUDA(cudaMemsetAsync(t_ctl.p, 0, 2 * sizeof(int), st));
  PCGB_CUDA(cudaMalloc(&P.bvid, ((size_t)nblk + 16) * sizeof(uint16_t)));
  PCGB_CUDA(cudaMemsetAsync(P.bvid + nblk, 0, 16 * sizeof(uint16_t), st));
  k_vdict_insert<RP><<<(int)std::min<int64_t>((nnodes + 127) / 128, (int64_t)num_sms() * 16), 128, 0, st>>>(
      static_cast<const RP *>(P.rowptr), P.val, nnodes, t_table.as<unsigned long long>(), P.bvid, t_ctl.as<int>(), t_ctl.as<int>() + 1);
  PCGB_CHECK_LAUNCH();
  int h_ctl[2] = {0, 0};
  std::vector<unsigned long long> table(kVdictSlots);
  PCGB_CUDA(cudaMemcpyAsync(h_ctl, t_ctl.p, sizeof(h_ctl), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaMemcpyAsync(table.data(), t_table.p, kVdictSlots * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  const int nd = h_ctl[0];
  if (h_ctl[1] != 0 || nd < 1 || nd > kVdictMax || (mode == 1 && nblk < 2 * (int64_t)nd * grid)) {
    cudaFree(P.bvid); P.bvid = nullptr;
    return PCGB_OK;
  }
  std::vector<std::pair<unsigned long long, int>> occ;   // (representative key, slot)
  for (int s = 0; s < kVdictSlots; ++s) if (table[(size_t)s] != kVdEmpty) occ.emplace_back(table[(size_t)s], s);
  std::sort(occ.begin(), occ.end());
  if ((int)occ.size() != nd) return fail(PCGB_ERR_CUDA, "value dictionary: %d slots for %d blocks", (int)occ.size(), nd);
  // one upload: slot -> id (u16 [kVdictSlots]) then the representatives in id order (u64 [nd])
  std::vector<unsigned char> buf((size_t)kVdictSlots * 2 + (size_t)nd * 8);
  uint16_t *slot_id = reinterpret_cast<uint16_t *>(buf.data());
  unsigned long long *rep = reinterpret_cast<unsigned long long *>(buf.data() + (size_t)kVdictSlots * 2);
  for (int s = 0; s < kVdictSlots; ++s) slot_id[s] = 0;
  for (int i = 0; i < nd; ++i) { slot_id[occ[(size_t)i].second] = (uint16_t)i; rep[i] = occ[(size_t)i].first; }
  PCGB_CUDA(cudaMalloc(&t_map.p, buf.size()));
  PCGB_CUDA(cudaMemcpyAsync(t_map.p, buf.data(), buf.size(), cudaMemcpyHostToDevice, st));
  PCGB_CUDA(cudaMalloc(&P.vdict, (size_t)nd * 9 * sizeof(double)));
  const int64_t work = std::max<int64_t>(nblk, 9 * (int64_t)nd);
  k_vdict_finish<<<(int)std::min<int64_t>((work + 255) / 256, (int64_t)num_sms() * 16), 256, 0, st>>>(
      P.bvid, nblk, t_map.as<uint16_t>(), P.val, reinterpret_cast<const unsigned long long *>(t_map.as<unsigned char>() + (size_t)kVdictSlots * 2),
      nd, P.vdict);
  PCGB_CHECK_LAUNCH();
  PCGB_CUDA(cudaStreamSynchronize(st));   // t_map is freed on return
  P.vd = nd;
  return PCGB_OK;
}

// The run-compressed index stream of the dictionary kernel (k_vd_runs) from bidx / bvid of the same tiles: P.vwords,
// P.vtoff, P.cap_words, P.run_nodes.  Frees bvid, which nothing reads afterwards.
template <typename RP>
inline int build_vd_runs(CsrPlan &P, cudaStream_t st) {
  const RP *rp = static_cast<const RP *>(P.rowptr);
  const int nt = P.ntiles;
  DevTmp t_nw, t_cov;
  PCGB_CUDA(cudaMalloc(&t_nw.p, (size_t)nt * sizeof(int64_t)));
  PCGB_CUDA(cudaMalloc(&t_cov.p, sizeof(unsigned long long)));
  PCGB_CUDA(cudaMemsetAsync(t_cov.p, 0, sizeof(unsigned long long), st));
  k_vd_runs<RP><<<(nt + 127) / 128, 128, 0, st>>>(rp, P.tile_desc, nt, P.bidx, P.bvid, nullptr, nullptr, t_nw.as<int64_t>(),
                                                  t_cov.as<unsigned long long>());
  PCGB_CHECK_LAUNCH();
  std::vector<int64_t> off((size_t)nt + 1);
  unsigned long long cov = 0;
  PCGB_CUDA(cudaMemcpyAsync(off.data(), t_nw.p, (size_t)nt * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaMemcpyAsync(&cov, t_cov.p, sizeof(cov), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  int64_t tot = 0, cap = 4;
  for (int b = 0; b < nt; ++b) {
    const int64_t w0 = tot;
    tot += off[(size_t)b];
    off[(size_t)b] = w0;
    cap = std::max(cap, ((tot + 3) & ~(int64_t)3) - (w0 & ~(int64_t)3));   // the producer's 16-byte aligned window
  }
  off[(size_t)nt] = tot;
  if (cap > (int64_t)1 << 20) return fail(PCGB_ERR_ARG, "SpMV tile index slice of %lld words", (long long)cap);
  PCGB_CUDA(cudaMalloc(&P.vwords, ((size_t)tot + 8) * sizeof(uint32_t)));
  PCGB_CUDA(cudaMemsetAsync(P.vwords + tot, 0, 8 * sizeof(uint32_t), st));
  PCGB_CUDA(cudaMalloc(&P.vtoff, ((size_t)nt + 1) * sizeof(int64_t)));
  PCGB_CUDA(cudaMemcpyAsync(P.vtoff, off.data(), ((size_t)nt + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  k_vd_runs<RP><<<(nt + 127) / 128, 128, 0, st>>>(rp, P.tile_desc, nt, P.bidx, P.bvid, P.vtoff, P.vwords, nullptr, nullptr);
  PCGB_CHECK_LAUNCH();
  PCGB_CUDA(cudaStreamSynchronize(st));   // `off` is read by the copy above
  P.nvwords = tot; P.cap_words = (int)cap; P.run_nodes = (int64_t)cov;
  cudaFree(P.bvid); P.bvid = nullptr;
  return PCGB_OK;
}

template <typename RP>
inline int build_plan_t(CsrPlan &P, cudaStream_t st, int bsr_tile = 0, int attempt = 0) {
  const RP *rp = static_cast<const RP *>(P.rowptr);
  DevTmp t_stats, t_head;
  PCGB_CUDA(cudaMalloc(&t_stats.p, 4 * sizeof(int)));
  int *const d_stats = t_stats.as<int>();
  PCGB_CUDA(cudaMemsetAsync(d_stats, 0, 4 * sizeof(int), st));
  if (P.nrows > 0) {
    int grid = (int)std::min<int64_t>((P.nrows + 255) / 256, (int64_t)num_sms() * 8);
    k_max_row<RP><<<grid, 256, 0, st>>>(rp, P.nrows, d_stats);
    PCGB_CHECK_LAUNCH();
  }
  int h_stats[4] = {0, 0, 0, 0};
  PCGB_CUDA(cudaMemcpyAsync(h_stats, d_stats, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  P.max_row = h_stats[0];

  const double avg = P.nrows ? (double)P.nnz / (double)P.nrows : 0.0;
  int lanes = avg <= 12.0 ? 4 : avg <= 85.0 ? 8 : avg <= 170.0 ? 16 : 32;
  lanes = env_int("PCGB_SPMV_LANES", lanes);
  if (lanes != 4 && lanes != 8 && lanes != 16 && lanes != 32) lanes = 16;
  // Tile size: the consumers walk the rows of a tile in passes of G = 256 / lanes rows; a tile should
  // fill ~90 % of a whole number of passes and four stages of two CTAs must fit in shared memory
  // (H100 stand-alone sweep, hex 128^3 with the node-block kernel off, 8 lanes, 4 stages: 1536 items 1.86-1.87 ms, 2048
  // 1.81 ms, 2304 1.79 ms; 2560 / 3072 items no longer fit two CTAs per SM and took 1.74 / 1.78 ms with one.  The 2304 cap
  // is carried over: a one-CTA ring has not been checked inside the PCG loop for this kernel, and for the node-block kernel
  // it was faster stand-alone but slower in the loop.)
  {
    const double per_pass = (256.0 / lanes) * (avg + 1.0);
    int npass = (int)(2048.0 / per_pass + 0.5);
    if (npass < 1) npass = 1;
    int t = (int)(0.9 * npass * per_pass);
    t = (t + 127) & ~127;
    if (t < 512) t = 512;
    if (t > 2304) t = 2304;
    P.tile_items = env_int("PCGB_SPMV_TILE", t);
  }
  if (P.tile_items < 256) P.tile_items = 256;
  P.lanes = lanes;
  P.use_tma = env_int("PCGB_SPMV_TMA", 1) != 0;
  // TMA bulk copies need 16-byte aligned global sources
  if ((reinterpret_cast<uintptr_t>(P.val) & 15) || (reinterpret_cast<uintptr_t>(P.col) & 15)) P.use_tma = false;
  // node-block mode: is this a 3-dofs-per-node matrix (rows 3n..3n+2 share one pattern of aligned column triples)?
  bool bsr_ok = false;
  if (P.use_tma && P.nrows > 0 && P.nrows % 3 == 0 && P.nnz % 9 == 0 && P.nnz > 0 && env_int("PCGB_SPMV_BSR", 1) != 0 &&
      env_int("PCGB_SPMV_STAGE", 1) != 0 && env_int("PCGB_SPMV_PERSIST", 1) != 0 && env_int("PCGB_SPMV_SNAP", 1) != 0) {
    unsigned long long *d_same = nullptr, h_same = 0;
    PCGB_CUDA(cudaMalloc(&d_same, sizeof(unsigned long long)));
    PCGB_CUDA(cudaMemsetAsync(d_same, 0, sizeof(unsigned long long), st));
    PCGB_CUDA(cudaMemsetAsync(d_stats + 3, 0, sizeof(int), st));
    k_check_bsr3<RP><<<(int)std::min<int64_t>((P.nrows / 3 + 127) / 128, (int64_t)num_sms() * 16), 128, 0, st>>>(rp, P.col, P.nrows / 3, d_stats + 3, d_same);
    cudaError_t ce_ = cudaGetLastError();
    if (ce_ == cudaSuccess) ce_ = cudaMemcpyAsync(h_stats + 3, d_stats + 3, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (ce_ == cudaSuccess) ce_ = cudaMemcpyAsync(&h_same, d_same, sizeof(h_same), cudaMemcpyDeviceToHost, st);
    if (ce_ == cudaSuccess) ce_ = cudaStreamSynchronize(st);
    cudaFree(d_same);
    PCGB_CUDA(ce_);
    // node-block kernel only for (mostly) regular node rows: on the octree model (concrete) the row-group kernel measured
    // faster (about half the SpMV time): irregular tiles need the per-block node search
    bsr_ok = h_stats[3] == 0 && (double)h_same >= 0.01 * env_int("PCGB_BSR_MIN_UNIFORM_PCT", 75) * (double)(P.nrows / 3);
    h_stats[3] = 0;
  }
  if (bsr_ok) {
    // one 3x3 block per consumer thread and pass (256 threads): a tile of at most 256 (or 512) blocks whatever the node snap does
    const int node_items = 3 * (P.max_row + 1);
    // two 3x3 blocks per consumer thread and pass in a 2-stage ring per CTA, two CTAs per SM, in-place row partials (default:
    // no scratch, two stages of ~53 KB per CTA in the 227 KB of an SM).  On H100 (hex 128^3) ONE CTA per SM with ~9000-item
    // tiles and 8 consumer warps was 1 % faster as a stand-alone SpMV (tools/spmv_sweep.py) but 7 % slower inside the PCG
    // loop (1.82 against 1.70 ms per iteration, bench.py), so two CTAs stay.
    // The tile is made as large as two CTAs per SM allow: start high and shrink by 4 % (re-plan) until the ring fits.
    int t = (env_int("PCGB_BSR_INPLACE", 1) != 0 ? 6100 : 4608) - node_items;
    if (bsr_tile > 0) t = bsr_tile;
    if (t < 2 * node_items) bsr_ok = false;                // rows too long for node-aligned tiles
    else P.tile_items = env_int("PCGB_SPMV_TILE", t);
    if (bsr_ok && P.tile_items < 2 * node_items) bsr_ok = false;
  }
  P.snap = bsr_ok || (P.max_row <= P.tile_items / 4 && env_int("PCGB_SPMV_SNAP", 1) != 0);

  const int64_t total = P.nrows + P.nnz;
  int64_t nt = (total + P.tile_items - 1) / P.tile_items;
  if (nt < 1) nt = 1;
  if (nt > INT32_MAX - 2) return fail(PCGB_ERR_ARG, "matrix too large for the tile index (ntiles=%lld)", (long long)nt);
  P.ntiles = (int)nt;
  PCGB_CUDA(cudaMalloc(&P.tile_row, (size_t)(P.ntiles + 1) * sizeof(int)));
  PCGB_CUDA(cudaMalloc(&P.tile_k, (size_t)(P.ntiles + 1) * sizeof(int64_t)));
  PCGB_CUDA(cudaMalloc(&P.carry, (size_t)P.ntiles * sizeof(double)));
  PCGB_CUDA(cudaMalloc(&P.dot_partials, (size_t)P.ntiles * sizeof(double)));
  PCGB_CUDA(cudaMemsetAsync(P.carry, 0, (size_t)P.ntiles * sizeof(double), st));
  PCGB_CUDA(cudaMalloc(&t_head.p, (size_t)P.ntiles));
  unsigned char *const d_head = t_head.as<unsigned char>();
  k_partition<RP><<<(P.ntiles + 1 + 255) / 256, 256, 0, st>>>(rp, P.nrows, P.nnz, P.tile_items, P.ntiles, P.snap ? 1 : 0,
                                                               P.tile_row, P.tile_k, bsr_ok ? 3 : 1);
  PCGB_CHECK_LAUNCH();
  k_tile_stats<RP><<<(P.ntiles + 255) / 256, 256, 0, st>>>(rp, P.tile_row, P.tile_k, P.ntiles, d_stats + 1, d_stats + 2, d_head);
  PCGB_CHECK_LAUNCH();
  PCGB_CUDA(cudaMemcpyAsync(h_stats, d_stats, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  P.cap_nnz = (h_stats[1] + 16 + 7) & ~7;
  P.cap_rows = (h_stats[2] + 2 + 1) & ~1;
  P.smem_bytes = P.cap_nnz * 12 + P.cap_rows * 8 + (P.cap_rows + 2) * 4;
  P.smem_bytes = (P.smem_bytes + 127) & ~127;
  if (P.smem_bytes > 200 * 1024)
    return fail(PCGB_ERR_ARG, "SpMV tile needs %d bytes of shared memory (tile_items=%d, max_row=%d)", P.smem_bytes,
                P.tile_items, P.max_row);

  // fix-up list for rows that span tiles (split mode only)
  P.nfix = 0;
  if (!P.snap) {
    std::vector<unsigned char> head(P.ntiles);
    std::vector<int> trow(P.ntiles + 1);
    PCGB_CUDA(cudaMemcpy(head.data(), d_head, (size_t)P.ntiles, cudaMemcpyDeviceToHost));
    PCGB_CUDA(cudaMemcpy(trow.data(), P.tile_row, (size_t)(P.ntiles + 1) * sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<int> frow, ffirst, fcnt;
    for (int b = 0; b < P.ntiles;) {
      if (!head[b]) { ++b; continue; }
      int e = b;
      while (e + 1 < P.ntiles && head[e + 1] && trow[e + 1] == trow[b]) ++e;
      frow.push_back(trow[b]); ffirst.push_back(b); fcnt.push_back(e - b + 1);
      b = e + 1;
    }
    P.nfix = (int)frow.size();
    if (P.nfix) {
      PCGB_CUDA(cudaMalloc(&P.fix_row, P.nfix * sizeof(int)));
      PCGB_CUDA(cudaMalloc(&P.fix_first, P.nfix * sizeof(int)));
      PCGB_CUDA(cudaMalloc(&P.fix_cnt, P.nfix * sizeof(int)));
      PCGB_CUDA(cudaMemcpy(P.fix_row, frow.data(), P.nfix * sizeof(int), cudaMemcpyHostToDevice));
      PCGB_CUDA(cudaMemcpy(P.fix_first, ffirst.data(), P.nfix * sizeof(int), cudaMemcpyHostToDevice));
      PCGB_CUDA(cudaMemcpy(P.fix_cnt, fcnt.data(), P.nfix * sizeof(int), cudaMemcpyHostToDevice));
    }
  }
  // ---- staged-x plan (k_spmv_staged): windows of x per tile + 16-bit local indices
  P.staged = false;
  if (P.use_tma && P.nnz > 0 && env_int("PCGB_SPMV_STAGE", 1) != 0) {
    const int gap = env_int("PCGB_SPMV_GAP", 8);
    const int plan_smem = (P.cap_nnz + 3 * kMaxRuns + 2 * kMaxWin + 8) * (int)sizeof(int);
    DevTmp t_fail, t_nw;
    PCGB_CUDA(cudaMalloc(&t_fail.p, sizeof(int)));
    int *const d_fail = t_fail.as<int>();
    PCGB_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), st));
    PCGB_CUDA(cudaMalloc(&t_nw.p, (size_t)P.ntiles * sizeof(int)));
    int *const d_nw = t_nw.as<int>();
    PCGB_CUDA(cudaMalloc(&P.tile_xlen, (size_t)P.ntiles * sizeof(int)));
    PCGB_CUDA(cudaFuncSetAttribute(k_plan_windows, cudaFuncAttributeMaxDynamicSharedMemorySize, plan_smem));
    k_plan_windows<<<P.ntiles, 256, plan_smem, st>>>(P.col, P.tile_k, P.cap_nnz, gap, 1, nullptr, nullptr, nullptr, nullptr, d_nw,
                                                     P.tile_xlen, d_fail);
    PCGB_CHECK_LAUNCH();
    std::vector<int> h_nw((size_t)P.ntiles), h_xl((size_t)P.ntiles);
    int h_fail = 0;
    PCGB_CUDA(cudaMemcpyAsync(&h_fail, d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
    PCGB_CUDA(cudaMemcpyAsync(h_nw.data(), d_nw, (size_t)P.ntiles * sizeof(int), cudaMemcpyDeviceToHost, st));
    PCGB_CUDA(cudaMemcpyAsync(h_xl.data(), P.tile_xlen, (size_t)P.ntiles * sizeof(int), cudaMemcpyDeviceToHost, st));
    PCGB_CUDA(cudaStreamSynchronize(st));
    if (!h_fail) {
      std::vector<int> h_tw((size_t)P.ntiles + 1);
      int64_t tot = 0;
      int mx = 0, mw = 0;
      for (int b = 0; b < P.ntiles; ++b) {
        h_tw[(size_t)b] = (int)tot;
        tot += h_nw[(size_t)b];
        mx = std::max(mx, h_xl[(size_t)b]);
        mw = std::max(mw, h_nw[(size_t)b]);
      }
      h_tw[(size_t)P.ntiles] = (int)tot;
      if (tot < INT32_MAX) {
        P.nwin = tot; P.max_nw = mw; P.cap_x = (mx + 2 + 1) & ~1;
        PCGB_CUDA(cudaMalloc(&P.tile_win, ((size_t)P.ntiles + 1) * sizeof(int)));
        PCGB_CUDA(cudaMalloc(&P.win_start, (size_t)std::max<int64_t>(tot, 1) * sizeof(int)));
        PCGB_CUDA(cudaMalloc(&P.win_off, (size_t)std::max<int64_t>(tot, 1) * sizeof(int)));
        PCGB_CUDA(cudaMalloc(&P.lidx, ((size_t)P.nnz + 16) * sizeof(uint16_t)));
        PCGB_CUDA(cudaMemcpyAsync(P.tile_win, h_tw.data(), ((size_t)P.ntiles + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
        k_plan_windows<<<P.ntiles, 256, plan_smem, st>>>(P.col, P.tile_k, P.cap_nnz, gap, 2, P.tile_win, P.lidx, P.win_start, P.win_off,
                                                         nullptr, nullptr, d_fail);
        PCGB_CHECK_LAUNCH();
        PCGB_CUDA(cudaStreamSynchronize(st));
        P.smem_staged = P.cap_nnz * 8 + P.cap_x * 8 + P.cap_rows * 8 + P.cap_nnz * 2 + (P.cap_rows + 2) * 4;
        P.smem_staged = (P.smem_staged + 127) & ~127;
        P.staged = P.smem_staged <= 200 * 1024;
        if (P.staged && env_int("PCGB_SPMV_PERSIST", 1) != 0) {
          // persistent pipelined kernel: descriptors + stage geometry
          PCGB_CUDA(cudaMalloc(&P.tile_desc, (size_t)P.ntiles * sizeof(TileDesc)));
          k_build_desc<RP><<<(P.ntiles + 255) / 256, 256, 0, st>>>(rp, P.tile_row, P.tile_k, P.tile_win, P.tile_xlen, P.ntiles, P.nrows,
                                                                  P.tile_desc);
          PCGB_CHECK_LAUNCH();
          PCGB_CUDA(cudaStreamSynchronize(st));
          // column-triple index: row-snapped plan, every row offset a multiple of 3, every aligned triple consecutive
          P.t3 = false;
          // Measured slower than the per-non-zero index on hex 128^3 with 8 lanes per row - the consumer is bound by
          // shared-memory wavefronts and per-row latency, not by the 13 % fewer HBM bytes - so the mode is OPT-IN
          // (PCGB_SPMV_T3=1) until the consumer is restructured.
          if (P.snap && P.nnz % 3 == 0 && P.nnz >= 3 && env_int("PCGB_SPMV_T3", 0) != 0) {
            PCGB_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), st));
            k_rows_mod3<RP><<<(int)std::min<int64_t>((P.nrows + 256) / 256, (int64_t)num_sms() * 8), 256, 0, st>>>(rp, P.nrows, d_fail);
            PCGB_CHECK_LAUNCH();
            const int64_t ntrip = P.nnz / 3;
            PCGB_CUDA(cudaMalloc(&P.lidx3, ((size_t)ntrip + 16) * sizeof(uint16_t)));
            PCGB_CUDA(cudaMemsetAsync(P.lidx3 + ntrip, 0, 16 * sizeof(uint16_t), st));
            k_build_idx3<<<(int)std::min<int64_t>((ntrip + 255) / 256, (int64_t)num_sms() * 16), 256, 0, st>>>(P.lidx, ntrip, P.lidx3, d_fail);
            PCGB_CHECK_LAUNCH();
            int h_f3 = 1;
            PCGB_CUDA(cudaMemcpyAsync(&h_f3, d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
            PCGB_CUDA(cudaStreamSynchronize(st));
            P.t3 = h_f3 == 0;
            if (!P.t3) { cudaFree(P.lidx3); P.lidx3 = nullptr; }
          }
          const int cap_idx = P.t3 ? (P.cap_nnz / 3 + 16) : P.cap_nnz;
          P.stage_bytes = P.cap_nnz * 8 + P.cap_x * 8 + (P.cap_rows + 2) * 8 + ((cap_idx * 2 + 15) & ~15) + 32;
          P.stage_bytes = (P.stage_bytes + 127) & ~127;
          int stages = env_int("PCGB_SPMV_STAGES", 4);
          if (stages < 1) stages = 1;
          if (stages > 8) stages = 8;
          P.persist_prod = stages >= kProd ? kProd : stages;
          stages -= stages % P.persist_prod;
          const int ctas = env_int("PCGB_SPMV_CTAS", 2);
          P.stages = stages;
          P.smem_persist = stages * P.stage_bytes;
          P.persist = P.smem_persist <= 200 * 1024 && P.dot_partials != nullptr;
          // resident CTAs per SM that really fit (227 KB of shared memory per SM, ~1 KB static per CTA)
          int fit = (227 * 1024) / (P.smem_persist + 2048);
          if (fit < 1) fit = 1;
          P.ctas_per_sm = std::min(ctas > 0 ? ctas : 1, fit);
          P.grid_persist = std::min(P.ntiles, num_sms() * P.ctas_per_sm);
          if (bsr_ok && P.dot_partials != nullptr) {
            // node-block index stream from the per-non-zero positions of the same (node-aligned) tiles
            PCGB_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), st));
            const int64_t nblk = P.nnz / 9;
            PCGB_CUDA(cudaMalloc(&P.bidx, ((size_t)nblk + 16) * sizeof(uint16_t)));
            PCGB_CUDA(cudaMemsetAsync(P.bidx + nblk, 0, 16 * sizeof(uint16_t), st));
            k_build_bidx<RP><<<(int)std::min<int64_t>((P.nrows / 3 + 127) / 128, (int64_t)num_sms() * 16), 128, 0, st>>>(rp, P.lidx, P.nrows / 3, P.bidx, d_fail);
            PCGB_CHECK_LAUNCH();
            int h_fb = 1;
            PCGB_CUDA(cudaMemcpyAsync(&h_fb, d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
            PCGB_CUDA(cudaStreamSynchronize(st));
            P.cap_blocks = (P.cap_nnz / 9 + 2 + 7) & ~7;
            P.cap_nodes = (P.cap_rows / 3 + 2 + 1) & ~1;
            const int sb_bytes = ((P.cap_blocks + 16) * 2 + 15) & ~15;
            P.bsr_stage_bytes = P.cap_nnz * 8 + P.cap_x * 8 + (P.cap_nodes + 2) * 8 + sb_bytes + 32;
            P.bsr_stage_bytes = (P.bsr_stage_bytes + 127) & ~127;
            const bool inplace = env_int("PCGB_BSR_INPLACE", 1) != 0;
            P.bsr_mode = (env_int("PCGB_BSR_UNI", 1) ? 1 : 0) | (inplace ? 2 : 0);
            P.bsr_cw = env_int("PCGB_BSR_CW", 6);
            if (P.bsr_cw != 8 && P.bsr_cw != 12) P.bsr_cw = 6;
            const int scratch = (inplace ? 0 : 6 * P.cap_blocks * 8) + 2 * (P.cap_nodes + 2) * 4 + 64;
            // 2 CTAs x 4 stages when they fit, else 2 CTAs x 2 stages (2 producer warps), else 1 CTA x 4 stages
            int bst = 2, bct = 2;
            if (2 * (2 * P.bsr_stage_bytes + scratch + 2048) > 227 * 1024) {
              if (h_fb == 0 && attempt < 8 && env_int("PCGB_SPMV_TILE", 0) == 0 && P.tile_items > 1536) {
                // two CTAs of two stages do not fit: plan again with a smaller tile (set-up cost only)
                const int smaller = (int)(P.tile_items * 0.96) & ~1;
                const void *rowptr = P.rowptr; const int *col = P.col; const double *val = P.val;
                const int64_t nr = P.nrows, nc = P.ncols, nz = P.nnz; const bool r64 = P.rp64;
                free_plan(P);
                P = CsrPlan();
                P.rowptr = rowptr; P.col = col; P.val = val; P.nrows = nr; P.ncols = nc; P.nnz = nz; P.rp64 = r64;
                return build_plan_t<RP>(P, st, smaller, attempt + 1);
              }
              bst = 4; bct = 1;
            }
            bst = env_int("PCGB_SPMV_STAGES", bst);
            bct = env_int("PCGB_SPMV_CTAS", bct);
            if (bst < 1) bst = 1;
            if (bst > 8) bst = 8;
            P.bsr_prod = bst >= 4 ? 4 : bst;                 // producer warps; stages % producers == 0
            bst -= bst % P.bsr_prod;
            P.bsr_stages = bst;
            P.smem_bsr = bst * P.bsr_stage_bytes + scratch;
            int bfit = (227 * 1024) / (P.smem_bsr + 2048);
            if (bfit < 1) bfit = 1;
            P.bsr = h_fb == 0 && P.smem_bsr <= 226 * 1024;
            if (P.bsr) {
              // uniform tiles (every node of the tile has the same number of blocks) take the search-free path
              PCGB_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), st));
              k_mark_uniform<RP><<<(P.ntiles + 255) / 256, 256, 0, st>>>(rp, P.tile_desc, P.ntiles, d_fail);
              PCGB_CHECK_LAUNCH();
              PCGB_CUDA(cudaStreamSynchronize(st));
              P.persist = true;
              P.ctas_per_sm = std::min(bct > 0 ? bct : 1, bfit);
              P.grid_bsr = std::min(P.ntiles, num_sms() * P.ctas_per_sm);
              // value dictionary (PCGB_SPMV_VDICT: 0 off, 1 when it pays, 2 whenever the blocks fit it).  The tiles, the grid and
              // the consumer warps stay those of the plan without one - they fix the order in which x.y is summed, so y and
              // x.y are the same bits either way; only the ring changes: a stage holds no values (sx | snp | the tile's
              // run-compressed block words | meta), and behind the ring sit the y buffers of two groups of tiles and the
              // dictionary (k_spmv_bsr3_vd).
              const int vd_mode = env_int("PCGB_SPMV_VDICT", 1);
              if (vd_mode != 0) PCGB_TRY(build_vdict<RP>(P, st, vd_mode, P.grid_bsr));
              if (P.vd) PCGB_TRY(build_vd_runs<RP>(P, st));
              if (P.vd) {
                // G warps consume G tiles at once, so the ring holds the G stages of a group plus at least two that the
                // producers fill for the next one, up to a whole second group: G = CW where G + 2 stages still fit the CTAs
                // per SM of the plan (hex 128^3: CW 6 and 8), else the largest G that does, and then the deepest even ring
                // up to 2 G + 2 that fits.  PCGB_SPMV_STAGES sets the ring instead, G = min(CW, stages).
                const int vstage = (P.cap_x * 8 + (P.cap_nodes + 2) * 8 + P.cap_words * 4 + 32 + 127) & ~127;
                auto ring_smem = [&](int g, int s) { return s * vstage + 2 * g * 3 * P.cap_nodes * 8 + kVdStride * 8 * P.vd; };
                auto ring_fits = [&](int smem) { return smem <= 226 * 1024 && (227 * 1024) / (smem + 2048) >= P.ctas_per_sm; };
                int vst = 0, vg = 0;
                const int env_st = env_int("PCGB_SPMV_STAGES", 0);
                if (env_st > 0) {
                  vst = std::min(env_st, kBsrMaxStages);
                  vg = std::min(P.bsr_cw, vst);
                  if (!ring_fits(ring_smem(vg, vst))) vst = 0;
                } else {
                  for (int g = P.bsr_cw; g >= 1 && vst == 0; --g)   // even rings (producer warps: see below)
                    for (int s = std::min((2 * g + 3) & ~1, kBsrMaxStages); s >= g + 2 && vst == 0; s -= 2)
                      if (ring_fits(ring_smem(g, s))) { vst = s; vg = g; }
                }
                if (vst > 0) {
                  P.bsr_stages = vst; P.bsr_group = vg; P.bsr_stage_bytes = vstage; P.smem_bsr = ring_smem(vg, vst);
                  P.bsr_prod = vst < 4 ? vst : vst % 4 == 0 ? 4 : vst % 2 == 0 ? 2 : 1;   // stages % producers == 0
                  cudaFree(P.bidx); P.bidx = nullptr;   // the word stream replaces it
                } else {
                  cudaFree(P.vdict); cudaFree(P.vwords); cudaFree(P.vtoff);
                  P.vdict = nullptr; P.vwords = nullptr; P.vtoff = nullptr; P.vd = 0;
                  P.nvwords = 0; P.run_nodes = 0; P.cap_words = 0;
                }
              }
              P.grid_persist = P.grid_bsr; P.smem_persist = P.smem_bsr; P.stages = P.bsr_stages; P.stage_bytes = P.bsr_stage_bytes;
              cudaFree(P.lidx); P.lidx = nullptr;           // the node-block kernel is the only consumer of the index stream now
              if (P.t3) { cudaFree(P.lidx3); P.lidx3 = nullptr; P.t3 = false; }
            } else {
              cudaFree(P.bidx); P.bidx = nullptr;
            }
          }
          if (P.persist) {
            PCGB_CUDA(cudaMalloc(&P.dot_partials_split, (size_t)2 * (size_t)std::max(P.grid_persist, 1) * sizeof(double)));
            if (P.t3 && !P.bsr) {
              cudaFree(P.lidx); P.lidx = nullptr;   // the persistent T3 kernel is the only consumer of the indices
              // lanes per row: a lane owns whole triples; 16 lanes at stride 3 doubles read the values conflict-free
              const double t_avg = avg / 3.0;
              int l3 = t_avg <= 6.0 ? 4 : t_avg <= 40.0 ? 8 : t_avg <= 80.0 ? 16 : 32;   // fewer, fatter row passes win (sweep r2a)
              l3 = env_int("PCGB_SPMV_LANES3", l3);
              if (l3 == 4 || l3 == 8 || l3 == 16 || l3 == 32) P.lanes = l3;
            }
          } else if (P.t3) {
            cudaFree(P.lidx3); P.lidx3 = nullptr; P.t3 = false;
          }
          if (!P.persist && P.bidx) { cudaFree(P.bidx); P.bidx = nullptr; P.bsr = false; }
        }
      }
    }
    if (!P.staged) {
      P.persist = false;
      cudaFree(P.tile_xlen); cudaFree(P.tile_win); cudaFree(P.win_start); cudaFree(P.win_off); cudaFree(P.lidx);
      P.tile_xlen = nullptr; P.tile_win = nullptr; P.win_start = nullptr; P.win_off = nullptr; P.lidx = nullptr;
    }
  }
  return spmv_configure(P);
}

template <int LANES, bool TMA, bool DOT, typename RP>
inline int launch_spmv_inst(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip) {
  auto kern = k_spmv_merge<LANES, TMA, DOT, RP>;
  if (P.ntiles == 0) return PCGB_OK;
  if (skip == reinterpret_cast<const int *>(1)) {  // configuration request from build_plan
    PCGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return PCGB_OK;
  }
  kern<<<P.ntiles, kSpmvBlock, P.smem_bytes, st>>>(static_cast<const RP *>(P.rowptr), P.col, P.val, x, y, P.tile_row, P.tile_k,
                                                   P.nrows, P.nnz, P.cap_nnz, P.cap_rows, P.carry, P.dot_partials, skip);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

template <bool TMA, bool DOT, typename RP>
inline int launch_spmv_lanes(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip) {
  switch (P.lanes) {
    case 4: return launch_spmv_inst<4, TMA, DOT, RP>(P, x, y, st, skip);
    case 8: return launch_spmv_inst<8, TMA, DOT, RP>(P, x, y, st, skip);
    case 32: return launch_spmv_inst<32, TMA, DOT, RP>(P, x, y, st, skip);
    default: return launch_spmv_inst<16, TMA, DOT, RP>(P, x, y, st, skip);
  }
}

template <int LANES, bool DOT, typename RP>
inline int launch_staged_inst(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip) {
  auto kern = k_spmv_staged<LANES, DOT, RP>;
  if (P.ntiles == 0) return PCGB_OK;
  if (skip == reinterpret_cast<const int *>(1)) {
    PCGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return PCGB_OK;
  }
  kern<<<P.ntiles, kSpmvBlock, P.smem_staged, st>>>(static_cast<const RP *>(P.rowptr), P.lidx, P.val, x, y, P.tile_row, P.tile_k, P.tile_win,
                                                    P.win_start, P.win_off, P.tile_xlen, P.nrows, P.nnz, P.cap_nnz, P.cap_rows, P.cap_x,
                                                    P.carry, P.dot_partials, skip);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

template <bool DOT, typename RP>
inline int launch_staged_lanes(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip) {
  switch (P.lanes) {
    case 4: return launch_staged_inst<4, DOT, RP>(P, x, y, st, skip);
    case 8: return launch_staged_inst<8, DOT, RP>(P, x, y, st, skip);
    case 32: return launch_staged_inst<32, DOT, RP>(P, x, y, st, skip);
    default: return launch_staged_inst<16, DOT, RP>(P, x, y, st, skip);
  }
}

// one launch of the persistent kernel over the tiles desc[0..ntiles) with `grid` resident CTAs; dot partials -> dotp[0..grid)
template <int LANES, bool DOT, bool T3, typename RP>
inline int launch_persist_inst(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip, const TileDesc *desc,
                               int ntiles, int grid, double *dotp) {
  auto kern = k_spmv_persist<LANES, DOT, T3, RP>;
  if (skip == reinterpret_cast<const int *>(1)) {
    PCGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return PCGB_OK;
  }
  if (ntiles == 0) return PCGB_OK;
  kern<<<grid, (kConsWarps + P.persist_prod) * 32, P.smem_persist, st>>>(static_cast<const RP *>(P.rowptr), T3 ? P.lidx3 : P.lidx, P.val, x, y, desc,
                                                       P.win_start, P.win_off, ntiles, P.nnz, P.cap_nnz, P.cap_rows, P.cap_x,
                                                       P.stages, P.stage_bytes, P.carry, dotp, skip);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

template <bool DOT, bool T3, typename RP>
inline int launch_persist_lanes(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip, const TileDesc *desc,
                                int ntiles, int grid, double *dotp) {
  switch (P.lanes) {
    case 4: return launch_persist_inst<4, DOT, T3, RP>(P, x, y, st, skip, desc, ntiles, grid, dotp);
    case 8: return launch_persist_inst<8, DOT, T3, RP>(P, x, y, st, skip, desc, ntiles, grid, dotp);
    case 32: return launch_persist_inst<32, DOT, T3, RP>(P, x, y, st, skip, desc, ntiles, grid, dotp);
    default: return launch_persist_inst<16, DOT, T3, RP>(P, x, y, st, skip, desc, ntiles, grid, dotp);
  }
}

template <bool DOT, int CW, typename RP, bool VD>
inline int launch_bsr_cw(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip, const TileDesc *desc,
                         int ntiles, int grid, double *dotp, const int *tile_ids) {
  if constexpr (VD) {
    auto kern = k_spmv_bsr3_vd<DOT, CW, RP>;
    if (skip == reinterpret_cast<const int *>(1)) {
      PCGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
      return PCGB_OK;
    }
    if (ntiles == 0) return PCGB_OK;
    kern<<<grid, (CW + P.bsr_prod) * 32, P.smem_bsr, st>>>(static_cast<const RP *>(P.rowptr), P.vwords, P.vtoff, tile_ids, P.vdict,
                                                           P.vd, x, y, desc, P.win_start, P.win_off, ntiles, P.cap_nodes, P.cap_x,
                                                           P.cap_words, P.bsr_stages, P.bsr_stage_bytes, P.bsr_group, dotp, skip);
  } else {
    auto kern = k_spmv_bsr3<DOT, CW, RP>;
    if (skip == reinterpret_cast<const int *>(1)) {
      PCGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
      return PCGB_OK;
    }
    if (ntiles == 0) return PCGB_OK;
    kern<<<grid, (CW + P.bsr_prod) * 32, P.smem_bsr, st>>>(static_cast<const RP *>(P.rowptr), P.bidx, P.val, x, y, desc, P.win_start,
                                                           P.win_off, ntiles, P.nnz, P.cap_nnz, P.cap_nodes, P.cap_x, P.cap_blocks,
                                                           P.bsr_stages, P.bsr_stage_bytes, P.bsr_mode, dotp, skip);
  }
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

template <bool DOT, typename RP, bool VD>
inline int launch_bsr_vd(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip, const TileDesc *desc,
                         int ntiles, int grid, double *dotp, const int *tile_ids) {
  // consumer warps per CTA: 6 by default; 8 and 12 are selectable with PCGB_BSR_CW.  On H100 (hex 128^3) the three are equal
  // within noise: 1.450-1.452 ms stand-alone (tools/spmv_sweep.py), 604-606 PCG it/s in bench.py.
  if (P.bsr_cw == 8) return launch_bsr_cw<DOT, 8, RP, VD>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
  if (P.bsr_cw == 12) return launch_bsr_cw<DOT, 12, RP, VD>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
  return launch_bsr_cw<DOT, 6, RP, VD>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
}

template <bool DOT, typename RP>
inline int launch_bsr_inst(const CsrPlan &P, const double *x, double *y, cudaStream_t st, const int *skip, const TileDesc *desc,
                           int ntiles, int grid, double *dotp, const int *tile_ids) {
  if (P.vd) return launch_bsr_vd<DOT, RP, true>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
  return launch_bsr_vd<DOT, RP, false>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
}

// tile_ids: tile id of every entry of desc (nullptr: desc is the plan's own tile order)
inline int launch_persist_any(const CsrPlan &P, const double *x, double *y, bool with_dot, cudaStream_t st, const int *skip,
                              const TileDesc *desc, int ntiles, int grid, double *dotp, const int *tile_ids) {
  if (P.ntiles == 0) return PCGB_OK;
  if (P.bsr) {
    if (P.rp64) return with_dot ? launch_bsr_inst<true, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids)
                                : launch_bsr_inst<false, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
    return with_dot ? launch_bsr_inst<true, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids)
                    : launch_bsr_inst<false, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp, tile_ids);
  }
  if (P.t3) {
    if (P.rp64) return with_dot ? launch_persist_lanes<true, true, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp)
                                : launch_persist_lanes<false, true, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp);
    return with_dot ? launch_persist_lanes<true, true, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp)
                    : launch_persist_lanes<false, true, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp);
  }
  if (P.rp64) return with_dot ? launch_persist_lanes<true, false, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp)
                              : launch_persist_lanes<false, false, int64_t>(P, x, y, st, skip, desc, ntiles, grid, dotp);
  return with_dot ? launch_persist_lanes<true, false, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp)
                  : launch_persist_lanes<false, false, int32_t>(P, x, y, st, skip, desc, ntiles, grid, dotp);
}

// y = A x ; with_dot additionally leaves per-tile partials of x.y in P.dot_partials.
// Returns the number of kernel launches through *launches.
inline int spmv_launch(const CsrPlan &P, const double *x, double *y, bool with_dot, cudaStream_t st, int *launches = nullptr,
                       const int *skip = nullptr) {
  int rc;
  if (P.persist) {
    rc = launch_persist_any(P, x, y, with_dot, st, skip, P.tile_desc, P.ntiles, P.grid_persist, P.dot_partials, nullptr);
  } else if (P.staged) {
    if (P.rp64) rc = with_dot ? launch_staged_lanes<true, int64_t>(P, x, y, st, skip) : launch_staged_lanes<false, int64_t>(P, x, y, st, skip);
    else rc = with_dot ? launch_staged_lanes<true, int32_t>(P, x, y, st, skip) : launch_staged_lanes<false, int32_t>(P, x, y, st, skip);
  } else if (P.rp64) {
    if (P.use_tma) rc = with_dot ? launch_spmv_lanes<true, true, int64_t>(P, x, y, st, skip) : launch_spmv_lanes<true, false, int64_t>(P, x, y, st, skip);
    else rc = with_dot ? launch_spmv_lanes<false, true, int64_t>(P, x, y, st, skip) : launch_spmv_lanes<false, false, int64_t>(P, x, y, st, skip);
  } else {
    if (P.use_tma) rc = with_dot ? launch_spmv_lanes<true, true, int32_t>(P, x, y, st, skip) : launch_spmv_lanes<true, false, int32_t>(P, x, y, st, skip);
    else rc = with_dot ? launch_spmv_lanes<false, true, int32_t>(P, x, y, st, skip) : launch_spmv_lanes<false, false, int32_t>(P, x, y, st, skip);
  }
  PCGB_TRY(rc);
  if (skip == reinterpret_cast<const int *>(1)) return PCGB_OK;
  int n = 1;
  if (P.nfix > 0) {
    k_spmv_fixup<<<(P.nfix + 127) / 128, 128, 0, st>>>(y, P.carry, P.fix_row, P.fix_first, P.fix_cnt, P.nfix);
    PCGB_CHECK_LAUNCH();
    ++n;
  }
  if (launches) *launches += n;
  return PCGB_OK;
}

// ---- interface-first split (multi-GPU overlap) ------------------------------------------------------------
// spmv_split_available(P): the persistent kernel is selected, no row spans tiles, and a boundary set was registered.
inline bool spmv_split_available(const CsrPlan &P) { return P.persist && P.nfix == 0 && P.desc_split != nullptr; }

// part 0: the tiles owning interface rows (launch BEFORE the halo pack); part 1: all other tiles (overlaps the
// transfer).  With with_dot the partials of part k land in dot_partials_split[k * grid_persist ...); the caller
// reduces spmv_split_dot_count(P) contiguous entries (unused slots are zero-filled at registration).
inline int spmv_launch_part(const CsrPlan &P, int part, const double *x, double *y, bool with_dot, cudaStream_t st,
                            int *launches = nullptr, const int *skip = nullptr) {
  const int nt = part == 0 ? P.nb_tiles : P.ntiles - P.nb_tiles;
  if (nt <= 0) return PCGB_OK;
  const TileDesc *desc = P.desc_split + (part == 0 ? 0 : P.nb_tiles);
  const int grid = std::min(nt, P.grid_persist);
  PCGB_TRY(launch_persist_any(P, x, y, with_dot, st, skip, desc, nt, grid, P.dot_partials_split + (size_t)part * P.grid_persist,
                              P.split_tile + (part == 0 ? 0 : P.nb_tiles)));
  if (launches) *launches += 1;
  return PCGB_OK;
}
inline int spmv_split_dot_count(const CsrPlan &P) { return 2 * P.grid_persist; }

// register the interface rows (device array of row indices) and build the boundary-first tile order
inline int spmv_set_boundary_rows(CsrPlan &P, const int *d_rows, int64_t count, cudaStream_t st) {
  if (!P.persist || P.nfix != 0 || P.ntiles == 0) return PCGB_OK;  // split not applicable: callers fall back to the serial order
  unsigned char *rowflag = nullptr, *tileflag = nullptr;
  int rc = PCGB_OK;
  std::vector<unsigned char> hflag((size_t)P.ntiles);
  std::vector<int> perm((size_t)P.ntiles);
  auto cleanup = [&]() { cudaFree(rowflag); cudaFree(tileflag); };
#define PCGB_SB(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup(); return fail(PCGB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } } while (0)
  PCGB_SB(cudaMalloc(&rowflag, (size_t)P.nrows + 1));
  PCGB_SB(cudaMalloc(&tileflag, (size_t)P.ntiles));
  PCGB_SB(cudaMemsetAsync(rowflag, 0, (size_t)P.nrows + 1, st));
  if (count > 0) k_mark_rows<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(d_rows, count, rowflag);
  k_flag_tiles<<<(P.ntiles + 255) / 256, 256, 0, st>>>(P.tile_desc, P.ntiles, rowflag, tileflag);
  PCGB_SB(cudaGetLastError());
  PCGB_SB(cudaMemcpyAsync(hflag.data(), tileflag, (size_t)P.ntiles, cudaMemcpyDeviceToHost, st));
  PCGB_SB(cudaStreamSynchronize(st));
  int nb = 0;
  for (int b = 0; b < P.ntiles; ++b) if (hflag[(size_t)b]) perm[(size_t)nb++] = b;
  int k = nb;
  for (int b = 0; b < P.ntiles; ++b) if (!hflag[(size_t)b]) perm[(size_t)k++] = b;
  if (!P.desc_split) PCGB_SB(cudaMalloc(&P.desc_split, (size_t)P.ntiles * sizeof(TileDesc)));
  if (!P.split_tile) PCGB_SB(cudaMalloc(&P.split_tile, (size_t)P.ntiles * sizeof(int)));   // the tile ids of desc_split
  PCGB_SB(cudaMemcpyAsync(P.split_tile, perm.data(), (size_t)P.ntiles * sizeof(int), cudaMemcpyHostToDevice, st));
  k_gather_desc<<<(P.ntiles + 255) / 256, 256, 0, st>>>(P.tile_desc, P.split_tile, P.ntiles, P.desc_split);
  PCGB_SB(cudaGetLastError());
  PCGB_SB(cudaMemsetAsync(P.dot_partials_split, 0, (size_t)2 * (size_t)std::max(P.grid_persist, 1) * sizeof(double), st));
  PCGB_SB(cudaStreamSynchronize(st));
#undef PCGB_SB
  P.nb_tiles = nb;
  cleanup();
  return rc;
}

// raise the dynamic shared memory limit of the instantiations this plan will launch (done once at
// plan time so that nothing but launches happens inside CUDA-graph capture)
inline int spmv_configure(const CsrPlan &P) {
  const int *cfg = reinterpret_cast<const int *>(1);
  PCGB_TRY(spmv_launch(P, nullptr, nullptr, false, 0, nullptr, cfg));
  PCGB_TRY(spmv_launch(P, nullptr, nullptr, true, 0, nullptr, cfg));
  return PCGB_OK;
}

inline void free_plan(CsrPlan &P) {
  cudaFree(P.tile_row); cudaFree(P.tile_k); cudaFree(P.carry); cudaFree(P.dot_partials);
  cudaFree(P.fix_row); cudaFree(P.fix_first); cudaFree(P.fix_cnt);
  cudaFree(P.tile_xlen); cudaFree(P.tile_win); cudaFree(P.win_start); cudaFree(P.win_off); cudaFree(P.lidx);
  cudaFree(P.tile_desc); cudaFree(P.lidx3); cudaFree(P.bidx); cudaFree(P.desc_split); cudaFree(P.dot_partials_split); cudaFree(P.diag_cache);
  cudaFree(P.bvid); cudaFree(P.vdict); cudaFree(P.vwords); cudaFree(P.vtoff); cudaFree(P.split_tile);
}

}  // namespace pcgb
