// assemble.cuh - device-side assembly of the sub-assembled stiffness matrix  A_i = K_i[Eff,Eff]  in CSR form from the
// reference's pattern groups (SURVEY.md 8(f2)):
//     K_i = sum_groups sum_e  P_e^T ( Ck_e . S_e . Ke_group . S_e ) P_e          (calcMatVecProd's operator, pcg_solver.py:263-300,
//                                                                                 type groups of partition_mesh.py:443-491)
// The reference never assembles (its operator is element-by-element); the CSR hot path needs the assembled form and the
// host cannot build it for large parts (a 128^3 METIS part is 1.2e9 element entries).  Everything below is hand-written,
// atomics-free in the arithmetic and bit-reproducible:
//   1. incidence lists  dof -> (group, element, local index), counted and filled per dof, then sorted per dof by
//      (group, element, local index) so that their order does not depend on the fill order;
//   2. symbolic pass, one warp per row: the columns of all incident elements are gathered into shared memory, sorted
//      (bitonic) and compacted to the distinct ascending columns -> row lengths -> row offsets (exclusive scan);
//   3. numeric pass, one warp per row: same column list, then for every incident element IN LIST ORDER the nd values
//      ((s_i s_j) Ke[i][j]) Ck_e are added into the row's shared-memory accumulator at the binary-searched position,
//      in ascending j.  An element may list the same free dof twice (the host COO assembly and the EBE operator sum
//      such repeats too); lanes of one pass that share a position are then added by the lowest of them in lane order
//      -> col / val written once, ascending.
// Both scans are checked against totals counted independently (atomics on the counts), so a wrong offset is reported
// instead of being used to size or index an allocation.
#pragma once
#include <vector>

#include "common.cuh"
#include "ebe.cuh"

namespace pcgb {

constexpr int kAsmMaxCand = 2048;   // candidate columns of one row (incident elements x pattern size): 8 KB + 16 KB smem per warp
constexpr int kAsmWarps = 4;

struct AsmGroup {
  int nd = 0;
  int64_t ne = 0;
  const int *idx = nullptr;             // [nd][ne] free-dof numbering, -1 = clamped
  const unsigned char *sign = nullptr;  // [nd][ne] or null
  const double *ck = nullptr;           // [ne]
  const double *ke = nullptr;           // [nd][nd] device
};

struct AsmPlan {
  int64_t n = 0;
  std::vector<AsmGroup> groups;
  AsmGroup *d_groups = nullptr;
  int64_t *d_inc_ptr = nullptr;            // [n+1]
  unsigned long long *d_inc = nullptr;     // [ninc]  (group << 48) | (element << 8) | local index
  int64_t ninc = 0, nnz = 0;
  int *d_fail = nullptr;
};

// ---- a plain three-kernel exclusive scan (int64), set-up code
__global__ void __launch_bounds__(1024) k_scan_block(const int64_t *__restrict__ in, int64_t n, int64_t *__restrict__ out, int64_t *__restrict__ bsum) {
  __shared__ int64_t sh[1024];
  const int64_t i = blockIdx.x * (int64_t)1024 + threadIdx.x;
  const int64_t v = i < n ? in[i] : 0;
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int64_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
    __syncthreads();
    sh[threadIdx.x] += t;
    __syncthreads();
  }
  if (i < n) out[i] = sh[threadIdx.x] - v;   // exclusive inside the block
  if (threadIdx.x == 1023) bsum[blockIdx.x] = sh[1023];
}
__global__ void __launch_bounds__(1024) k_scan_sums(int64_t *__restrict__ bsum, int64_t nb) {   // one CTA: exclusive scan of the block sums
  __shared__ int64_t sh[1024];
  __shared__ int64_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < nb; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = i < nb ? bsum[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int64_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < nb) bsum[i] = carry + sh[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += sh[1023];
    __syncthreads();
  }
}
__global__ void __launch_bounds__(1024) k_scan_add(int64_t *__restrict__ out, int64_t n, const int64_t *__restrict__ bsum, int64_t *__restrict__ total,
                                                  const int64_t *__restrict__ in) {
  const int64_t i = blockIdx.x * (int64_t)1024 + threadIdx.x;
  if (i < n) {
    out[i] += bsum[blockIdx.x];
    if (i == n - 1) *total = out[i] + in[i];
  }
}
// out[0..n) = exclusive scan of in[0..n), out[n] = total (in and out may not alias)
inline int exclusive_scan_i64(const int64_t *in, int64_t n, int64_t *out, cudaStream_t st) {
  if (n <= 0) { PCGB_CUDA(cudaMemsetAsync(out, 0, sizeof(int64_t), st)); return PCGB_OK; }
  const int64_t nb = (n + 1023) / 1024;
  int64_t *bsum = nullptr;
  PCGB_CUDA(cudaMalloc(&bsum, (size_t)nb * sizeof(int64_t)));
  k_scan_block<<<(unsigned)nb, 1024, 0, st>>>(in, n, out, bsum);
  k_scan_sums<<<1, 1024, 0, st>>>(bsum, nb);
  k_scan_add<<<(unsigned)nb, 1024, 0, st>>>(out, n, bsum, out + n, in);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(bsum);
  PCGB_CUDA(e);
  return PCGB_OK;
}

// ---- incidence lists
// cnt[d] += incidences of dof d; cnt[n] += all of them (the total the scan of cnt[0..n) must reach)
__global__ void k_asm_count(AsmGroup g, int64_t n, int64_t *__restrict__ cnt) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int d = t < g.ne * g.nd ? g.idx[t] : -1;
  if (d >= 0) atomicAdd(reinterpret_cast<unsigned long long *>(cnt + d), 1ull);
  const int c = __syncthreads_count(d >= 0);
  if (threadIdx.x == 0 && c > 0) atomicAdd(reinterpret_cast<unsigned long long *>(cnt + n), (unsigned long long)c);
}
__global__ void k_asm_fill(AsmGroup g, int gi, const int64_t *__restrict__ inc_ptr, int64_t *__restrict__ cursor,
                           unsigned long long *__restrict__ inc) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= g.ne * g.nd) return;
  const int d = g.idx[t];
  if (d < 0) return;
  const int64_t i = t / g.ne, e = t - i * g.ne;
  const unsigned long long slot = atomicAdd(reinterpret_cast<unsigned long long *>(cursor + d), 1ull);
  inc[inc_ptr[d] + (int64_t)slot] = ((unsigned long long)gi << 48) | ((unsigned long long)e << 8) | (unsigned long long)i;
}
// per dof: insertion sort of its (short) list -> order independent of the atomic fill order
// (K = the incidence keys here, the int32 slot positions of ebe_ordered.cuh)
template <typename K>
__global__ void k_asm_sort_inc(int64_t n, const int64_t *__restrict__ inc_ptr, K *__restrict__ inc) {
  const int64_t d = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (d >= n) return;
  const int64_t a = inc_ptr[d], b = inc_ptr[d + 1];
  for (int64_t i = a + 1; i < b; ++i) {
    const K key = inc[i];
    int64_t j = i - 1;
    while (j >= a && inc[j] > key) { inc[j + 1] = inc[j]; --j; }
    inc[j + 1] = key;
  }
}

// gather + sort + unique of the candidate columns of row `row` by one warp; returns the number of distinct columns
// (valid in all lanes), leaves them ascending in sc[0..nu); -1 when the candidates exceed kAsmMaxCand
__device__ __forceinline__ int asm_row_columns(const AsmGroup *__restrict__ groups, const int64_t *__restrict__ inc_ptr,
                                               const unsigned long long *__restrict__ inc, int64_t row, int *sc, int lane) {
  const int64_t a = inc_ptr[row], b = inc_ptr[row + 1];
  int total = 0;
  for (int64_t k = a; k < b; ++k) {
    const unsigned long long key = inc[k];
    const AsmGroup g = groups[key >> 48];
    const int64_t e = (int64_t)((key >> 8) & 0xffffffffffull);
    if (total + g.nd > kAsmMaxCand) return -1;
    for (int j = lane; j < g.nd; j += 32) {
      const int c = g.idx[(int64_t)j * g.ne + e];
      sc[total + j] = c >= 0 ? c : INT32_MAX;   // clamped columns sort to the end
    }
    total += g.nd;
  }
  int np2 = 32;
  while (np2 < total) np2 <<= 1;
  for (int i = total + lane; i < np2; i += 32) sc[i] = INT32_MAX;
  __syncwarp();
  for (int k = 2; k <= np2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < np2; i += 32) {
        const int l = i ^ j;
        if (l > i) {
          const int x = sc[i], y = sc[l];
          if ((x > y) == ((i & k) == 0)) { sc[i] = y; sc[l] = x; }
        }
      }
      __syncwarp();
    }
  // compact the distinct values (< INT32_MAX), warp-wide running offset
  int nu = 0;
  for (int base = 0; base < np2; base += 32) {
    const int i = base + lane;
    const int v = sc[i];
    const bool keep = v != INT32_MAX && (i == 0 || sc[i - 1] != v);
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    if (keep) sc[nu + __popc(m & ((1u << lane) - 1u))] = v;   // nu + rank <= i: never overwrites an unread entry of a later chunk
    nu += __popc(m);
    __syncwarp();
  }
  return nu;
}

__global__ void __launch_bounds__(kAsmWarps * 32)
k_asm_row_count(const AsmGroup *__restrict__ groups, const int64_t *__restrict__ inc_ptr, const unsigned long long *__restrict__ inc,
                int64_t n, int64_t *__restrict__ rowcount, int *__restrict__ fail) {   // rowcount[n] += sum of the row lengths
  extern __shared__ int asm_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int *sc = asm_smem + warp * kAsmMaxCand;
  unsigned long long sum = 0;
  for (int64_t row = blockIdx.x * (int64_t)kAsmWarps + warp; row < n; row += (int64_t)gridDim.x * kAsmWarps) {
    const int nu = asm_row_columns(groups, inc_ptr, inc, row, sc, lane);
    if (nu < 0) { if (lane == 0) *fail = 1; continue; }
    if (lane == 0) rowcount[row] = nu;
    sum += (unsigned)nu;
    __syncwarp();
  }
  if (lane == 0 && sum > 0) atomicAdd(reinterpret_cast<unsigned long long *>(rowcount + n), sum);
}

__global__ void __launch_bounds__(kAsmWarps * 32)
k_asm_row_fill(const AsmGroup *__restrict__ groups, const int64_t *__restrict__ inc_ptr, const unsigned long long *__restrict__ inc,
               int64_t n, const int64_t *__restrict__ rowptr, int *__restrict__ col, double *__restrict__ val) {
  extern __shared__ int asm_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int *sc = asm_smem + warp * kAsmMaxCand;
  double *sv = reinterpret_cast<double *>(asm_smem + kAsmWarps * kAsmMaxCand) + warp * kAsmMaxCand;
  for (int64_t row = blockIdx.x * (int64_t)kAsmWarps + warp; row < n; row += (int64_t)gridDim.x * kAsmWarps) {
    const int nu = asm_row_columns(groups, inc_ptr, inc, row, sc, lane);
    if (nu < 0) continue;
    for (int u = lane; u < nu; u += 32) sv[u] = 0.0;
    __syncwarp();
    const int64_t a = inc_ptr[row], b = inc_ptr[row + 1];
    for (int64_t k = a; k < b; ++k) {   // fixed order: (group, element, local index) ascending
      const unsigned long long key = inc[k];
      const AsmGroup g = groups[key >> 48];
      const int64_t e = (int64_t)((key >> 8) & 0xffffffffffull);
      const int i = (int)(key & 0xffull);
      const double ck = g.ck[e];
      const bool si = g.sign != nullptr && g.sign[(int64_t)i * g.ne + e] != 0;
      for (int j0 = 0; j0 < g.nd; j0 += 32) {
        const int j = j0 + lane;
        const int c = j < g.nd ? g.idx[(int64_t)j * g.ne + e] : -1;
        double v = 0.0;
        int lo = -1;                      // position of column c in the distinct ascending list, -1 = nothing to add
        if (c >= 0) {
          const bool sj = g.sign != nullptr && g.sign[(int64_t)j * g.ne + e] != 0;
          v = g.ke[i * g.nd + j];
          if (si != sj) v = -v;          // (s_i s_j) Ke[i][j]   (pcg_solver.py:278,280), times Ck_e (:279) in the fma below
          int hi = nu - 1;
          lo = 0;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (sc[mid] < c) lo = mid + 1; else hi = mid;
          }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, lo);
        // every term enters with one rounding, sv = fma(v, Ck_e, sv), in ascending j
        if (!__any_sync(0xffffffffu, lo >= 0 && peers != (1u << lane))) {
          if (lo >= 0) sv[lo] = fma(v, ck, sv[lo]);   // the columns of this pass are distinct
        } else {                          // a repeated column: its lowest lane adds the peers' terms in lane order
          double s = lo >= 0 ? sv[lo] : 0.0;
          for (int src = 0; src < 32; ++src) {
            const double w = __shfl_sync(0xffffffffu, v, src);
            if (((peers >> src) & 1u) && lo >= 0) s = fma(w, ck, s);
          }
          if (lo >= 0 && lane == __ffs(peers) - 1) sv[lo] = s;
        }
        __syncwarp();                     // a column repeated in the next pass reads this pass's sum
      }
    }
    const int64_t o = rowptr[row];
    for (int u = lane; u < nu; u += 32) { col[o + u] = sc[u]; val[o + u] = sv[u]; }
    __syncwarp();
  }
}

inline void asm_free(AsmPlan &P) {
  for (AsmGroup &g : P.groups) cudaFree(const_cast<double *>(g.ke));
  cudaFree(P.d_groups); cudaFree(P.d_inc_ptr); cudaFree(P.d_inc); cudaFree(P.d_fail);
  P.groups.clear();
  P.d_groups = nullptr; P.d_inc_ptr = nullptr; P.d_inc = nullptr; P.d_fail = nullptr;
}

// symbolic phase: incidence lists, row lengths -> d_rowptr[0..n] (int64, caller-owned), P.nnz
inline int asm_symbolic(AsmPlan &P, int64_t *d_rowptr, cudaStream_t st) {
  const int64_t n = P.n;
  int64_t *cnt = nullptr, *cursor = nullptr;
  cudaError_t ce = cudaSuccess;
  int rc = PCGB_OK;
  auto done = [&](int code) { cudaFree(cnt); cudaFree(cursor); return code; };
#define PCGB_AS(call) do { ce = (call); if (ce != cudaSuccess) return done(fail(PCGB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(ce))); } while (0)
  PCGB_AS(cudaMalloc(&cnt, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_AS(cudaMalloc(&cursor, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_AS(cudaMalloc(&P.d_inc_ptr, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_AS(cudaMalloc(&P.d_fail, sizeof(int)));
  PCGB_AS(cudaMemsetAsync(cnt, 0, (size_t)(n + 1) * sizeof(int64_t), st));
  PCGB_AS(cudaMemsetAsync(cursor, 0, (size_t)(n + 1) * sizeof(int64_t), st));
  PCGB_AS(cudaMemsetAsync(P.d_fail, 0, sizeof(int), st));
  PCGB_AS(cudaMalloc(&P.d_groups, std::max<size_t>(P.groups.size(), 1) * sizeof(AsmGroup)));
  if (!P.groups.empty()) PCGB_AS(cudaMemcpyAsync(P.d_groups, P.groups.data(), P.groups.size() * sizeof(AsmGroup), cudaMemcpyHostToDevice, st));
  for (const AsmGroup &g : P.groups) {
    const int64_t tot = g.ne * g.nd;
    if (tot > 0) k_asm_count<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(g, n, cnt);
  }
  PCGB_AS(cudaGetLastError());
  rc = exclusive_scan_i64(cnt, n, P.d_inc_ptr, st);
  if (rc != PCGB_OK) return done(rc);
  int64_t counted = 0;
  PCGB_AS(cudaMemcpyAsync(&P.ninc, P.d_inc_ptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_AS(cudaMemcpyAsync(&counted, cnt + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_AS(cudaStreamSynchronize(st));
  if (P.ninc != counted)
    return done(fail(PCGB_ERR_CUDA, "pcgb_assemble: incidence offsets end at %lld, but %lld incidences were counted", (long long)P.ninc, (long long)counted));
  PCGB_AS(cudaMalloc(&P.d_inc, std::max<size_t>((size_t)P.ninc, 1) * sizeof(unsigned long long)));
  for (size_t gi = 0; gi < P.groups.size(); ++gi) {
    const AsmGroup &g = P.groups[gi];
    const int64_t tot = g.ne * g.nd;
    if (tot > 0) k_asm_fill<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(g, (int)gi, P.d_inc_ptr, cursor, P.d_inc);
  }
  if (n > 0) k_asm_sort_inc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, P.d_inc_ptr, P.d_inc);
  PCGB_AS(cudaGetLastError());
  // row lengths (reuses cnt; cnt[n] collects their sum), then the row offsets
  PCGB_AS(cudaMemsetAsync(cnt + n, 0, sizeof(int64_t), st));
  const int smem = kAsmWarps * kAsmMaxCand * (int)sizeof(int);
  PCGB_AS(cudaFuncSetAttribute(k_asm_row_count, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const unsigned grid = (unsigned)std::min<int64_t>((n + kAsmWarps - 1) / kAsmWarps, (int64_t)num_sms() * 16);
  if (n > 0) k_asm_row_count<<<grid, kAsmWarps * 32, smem, st>>>(P.d_groups, P.d_inc_ptr, P.d_inc, n, cnt, P.d_fail);
  PCGB_AS(cudaGetLastError());
  int h_fail = 0;
  PCGB_AS(cudaMemcpyAsync(&h_fail, P.d_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCGB_AS(cudaStreamSynchronize(st));
  if (h_fail) return done(fail(PCGB_ERR_ARG, "pcgb_assemble: a row has more than %d candidate columns (incident elements x pattern size)", kAsmMaxCand));
  rc = exclusive_scan_i64(cnt, n, d_rowptr, st);
  if (rc != PCGB_OK) return done(rc);
  PCGB_AS(cudaMemcpyAsync(&P.nnz, d_rowptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_AS(cudaMemcpyAsync(&counted, cnt + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_AS(cudaStreamSynchronize(st));
  if (P.nnz != counted)
    return done(fail(PCGB_ERR_CUDA, "pcgb_assemble: row offsets end at %lld, but the row lengths sum to %lld", (long long)P.nnz, (long long)counted));
#undef PCGB_AS
  return done(PCGB_OK);
}

inline int asm_numeric(const AsmPlan &P, const int64_t *d_rowptr, int *d_col, double *d_val, cudaStream_t st) {
  if (P.n == 0) return PCGB_OK;
  const int smem = kAsmWarps * kAsmMaxCand * (int)(sizeof(int) + sizeof(double));
  PCGB_CUDA(cudaFuncSetAttribute(k_asm_row_fill, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const unsigned grid = (unsigned)std::min<int64_t>((P.n + kAsmWarps - 1) / kAsmWarps, (int64_t)num_sms() * 8);
  k_asm_row_fill<<<grid, kAsmWarps * 32, smem, st>>>(P.d_groups, P.d_inc_ptr, P.d_inc, P.n, d_rowptr, d_col, d_val);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

}  // namespace pcgb
