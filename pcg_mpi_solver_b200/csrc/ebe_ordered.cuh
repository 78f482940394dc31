// ebe_ordered.cuh - the matrix-free EBE operator with a fixed summation order (bit-reproducible), reachable from the
// PCG solve.  It is the reference's own two-phase form of calcMatVecProd (pcg_solver.py:263-300): every element product
// goes into one flat array (`Flat`, :279-297), then each dof sums its entries (`np.bincount(Flat_ElemLocDof, ...)`, :300).
//
//   phase 1  for group g, element e, local index a:   V[off_g + a*ne_g + e] = s_a * acc,
//              acc = fma(Ke[a][b], u_b, acc) over b = 0..nd-1 ascending from 0.0,  u_b = Ck_e * (s_b * x[idx_b])
//              (u_b = 0 for a clamped b).  The slot layout is the layout of idx itself, groups concatenated.
//              Slots of clamped a are not written (and never read).
//   phase 2  y_i = ((0.0 + V[p_1]) + V[p_2]) + ...  over the slots p_1 < p_2 < ... of dof i, i.e. the order in which
//              np.bincount visits them: (group, local index, element).  Every y_i is written exactly once; 0 when
//              no slot names dof i.
// Set-up (once per operator, on the device): per-dof slot lists - counts (k_asm_count), exclusive scan, a fill, and a
// per-dof sort by slot position.  Positions are unique, so the sorted lists do not depend on the (atomic) fill order.
// Kernels of phase 1 mirror ebe.cuh: k_ebo_t24 one thread per element with Ke in constant memory (c_ebe_ke24 slots),
// k_ebo_warp one warp per element for every other pattern (Ke from global memory, row a read by lane a).
#pragma once
#include <vector>

#include "common.cuh"
#include "ebe.cuh"
#include "assemble.cuh"

namespace pcgb {

struct EboPlan {
  EbePlan P;                     // groups, constant-memory slots and the warp-kernel block tables (as the atomic operator)
  std::vector<int64_t> off;      // slot offset of every group
  int64_t *d_off = nullptr;      // device copy (k_ebo_warp)
  int64_t nslots = 0;            // flat length sum nd*ne
  int64_t nfree = 0;             // slots of free (unclamped) local indices = entries of the per-dof lists
  double *v = nullptr;           // [nslots] element products
  int64_t *d_ptr = nullptr;      // [n+1] per-dof list offsets
  int *d_pos = nullptr;          // [nfree] slot positions, ascending per dof
};

template <bool SIGN>
__global__ void __launch_bounds__(128)
k_ebo_t24(const int *__restrict__ idx, const unsigned char *__restrict__ sign, const double *__restrict__ ck, int slot, int64_t ne,
          const double *__restrict__ x, double *__restrict__ v, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t e = blockIdx.x * (int64_t)128 + threadIdx.x;
  if (e >= ne) return;
  const double c = ck[e];
  int id[24];
  double u[24];
  unsigned sbits = 0;
#pragma unroll
  for (int b = 0; b < 24; ++b) {
    id[b] = idx[(int64_t)b * ne + e];
    double w = id[b] >= 0 ? __ldg(x + id[b]) : 0.0;
    if (SIGN && sign[(int64_t)b * ne + e]) { w = -w; sbits |= 1u << b; }   // pcg_solver.py:278
    u[b] = c * w;                                                          // :279  Ck * U
  }
#pragma unroll
  for (int a = 0; a < 24; ++a) {
    if (id[a] < 0) continue;
    double acc = 0.0;
#pragma unroll
    for (int b = 0; b < 24; ++b) acc = fma(c_ebe_ke24[slot][a * 24 + b], u[b], acc);   // :279  Ke @ (Ck * U)
    if (SIGN && ((sbits >> a) & 1u)) acc = -acc;                                        // :280
    v[(int64_t)a * ne + e] = acc;                                                       // :294-297  Flat
  }
}

__global__ void __launch_bounds__(kEbeWarpsPerBlock * 32)
k_ebo_warp(const EbeGroup *__restrict__ groups, const int64_t *__restrict__ off, const int *__restrict__ blk_group,
           const int64_t *__restrict__ blk_e0, const double *__restrict__ x, double *__restrict__ v, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  __shared__ double su[kEbeWarpsPerBlock][96];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gi = blk_group[blockIdx.x];
  const EbeGroup g = groups[gi];
  const int64_t e = blk_e0[blockIdx.x] + warp;
  if (e >= g.ne) return;
  const int nd = g.nd;
  const double c = g.ck[e];
  for (int b = lane; b < nd; b += 32) {
    const int id = g.idx[(int64_t)b * g.ne + e];
    double w = id >= 0 ? __ldg(x + id) : 0.0;
    if (g.sign != nullptr && g.sign[(int64_t)b * g.ne + e] != 0) w = -w;
    su[warp][b] = c * w;
  }
  __syncwarp();
  double *vg = v + off[gi];
  for (int a = lane; a < nd; a += 32) {
    const int id = g.idx[(int64_t)a * g.ne + e];
    if (id < 0) continue;
    double acc = 0.0;
    for (int b = 0; b < nd; ++b) acc = fma(__ldg(g.ke + (int64_t)a * nd + b), su[warp][b], acc);
    if (g.sign != nullptr && g.sign[(int64_t)a * g.ne + e] != 0) acc = -acc;
    vg[(int64_t)a * g.ne + e] = acc;
  }
}

// phase 2: one thread per dof, its slots in ascending position
__global__ void __launch_bounds__(256)
k_ebo_sum(int64_t n, const int64_t *__restrict__ ptr, const int *__restrict__ pos, const double *__restrict__ v,
          double *__restrict__ y, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t i = blockIdx.x * (int64_t)256 + threadIdx.x;
  if (i >= n) return;
  const int64_t a = ptr[i], b = ptr[i + 1];
  double acc = 0.0;
  for (int64_t k = a; k < b; ++k) acc += v[pos[k]];
  y[i] = acc;
}

// ---- set-up
// Each dof's list is filled from its end towards its start, so the fill order is never the ascending order by accident:
// a missing sort shows up as a wrong order instead of passing unnoticed.
__global__ void k_ebo_fill(const int *__restrict__ idx, int64_t tot, int64_t off, const int64_t *__restrict__ ptr,
                           int64_t *__restrict__ cursor, int *__restrict__ pos) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= tot) return;
  const int d = idx[t];
  if (d < 0) return;
  const unsigned long long k = atomicAdd(reinterpret_cast<unsigned long long *>(cursor + d), 1ull);
  pos[ptr[d + 1] - 1 - (int64_t)k] = (int)(off + t);
}

inline void ebo_free_lists(EboPlan &O) {
  cudaFree(O.d_off); cudaFree(O.v); cudaFree(O.d_ptr); cudaFree(O.d_pos);
  O.d_off = nullptr; O.v = nullptr; O.d_ptr = nullptr; O.d_pos = nullptr;
}

// the per-dof slot lists and the slot buffer of an operator whose groups are in O.P (set up by the caller)
inline int ebo_build_lists(EboPlan &O, cudaStream_t st) {
  const int64_t n = O.P.n;
  int64_t *cnt = nullptr, *cursor = nullptr;
  cudaError_t ce = cudaSuccess;
  auto done = [&](int code) { cudaFree(cnt); cudaFree(cursor); return code; };
#define PCGB_EO(call) do { ce = (call); if (ce != cudaSuccess) return done(fail(PCGB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(ce))); } while (0)
  PCGB_EO(cudaMalloc(&O.d_off, std::max<size_t>(O.off.size(), 1) * sizeof(int64_t)));
  if (!O.off.empty()) PCGB_EO(cudaMemcpy(O.d_off, O.off.data(), O.off.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
  PCGB_EO(cudaMalloc(&O.v, (size_t)std::max<int64_t>(O.nslots, 1) * sizeof(double)));
  PCGB_EO(cudaMalloc(&O.d_ptr, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_EO(cudaMalloc(&cnt, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_EO(cudaMalloc(&cursor, (size_t)(n + 1) * sizeof(int64_t)));
  PCGB_EO(cudaMemsetAsync(cnt, 0, (size_t)(n + 1) * sizeof(int64_t), st));
  PCGB_EO(cudaMemsetAsync(cursor, 0, (size_t)(n + 1) * sizeof(int64_t), st));
  for (const EbeGroup &g : O.P.groups) {
    const int64_t tot = g.ne * g.nd;
    AsmGroup ag;
    ag.nd = g.nd; ag.ne = g.ne; ag.idx = g.idx;
    if (tot > 0) k_asm_count<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(ag, n, cnt);
  }
  PCGB_EO(cudaGetLastError());
  int rc = exclusive_scan_i64(cnt, n, O.d_ptr, st);
  if (rc != PCGB_OK) return done(rc);
  int64_t counted = 0;
  PCGB_EO(cudaMemcpyAsync(&O.nfree, O.d_ptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_EO(cudaMemcpyAsync(&counted, cnt + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCGB_EO(cudaStreamSynchronize(st));
  if (O.nfree != counted || O.nfree > O.nslots)
    return done(fail(PCGB_ERR_CUDA, "pcgb_ebe_ordered_create: slot-list offsets end at %lld, but %lld free slots were counted (of %lld)",
                     (long long)O.nfree, (long long)counted, (long long)O.nslots));
  PCGB_EO(cudaMalloc(&O.d_pos, (size_t)std::max<int64_t>(O.nfree, 1) * sizeof(int)));
  for (size_t gi = 0; gi < O.P.groups.size(); ++gi) {
    const EbeGroup &g = O.P.groups[gi];
    const int64_t tot = g.ne * g.nd;
    if (tot > 0) k_ebo_fill<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(g.idx, tot, O.off[gi], O.d_ptr, cursor, O.d_pos);
  }
  if (n > 0) k_asm_sort_inc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, O.d_ptr, O.d_pos);
  PCGB_EO(cudaGetLastError());
  PCGB_EO(cudaStreamSynchronize(st));
#undef PCGB_EO
  return done(PCGB_OK);
}

inline int ebo_apply(const EboPlan &O, const double *x, double *y, cudaStream_t st, int *launches = nullptr, const int *skip = nullptr) {
  int nl = 0;
  for (size_t gi = 0; gi < O.P.groups.size(); ++gi) {
    const EbeGroup &g = O.P.groups[gi];
    if (g.nd != 24 || g.slot < 0 || g.ne == 0) continue;
    const unsigned grid = (unsigned)((g.ne + 127) / 128);
    double *vg = O.v + O.off[gi];
    if (g.sign) k_ebo_t24<true><<<grid, 128, 0, st>>>(g.idx, g.sign, g.ck, g.slot, g.ne, x, vg, skip);
    else k_ebo_t24<false><<<grid, 128, 0, st>>>(g.idx, nullptr, g.ck, g.slot, g.ne, x, vg, skip);
    PCGB_CHECK_LAUNCH();
    ++nl;
  }
  if (O.P.nblk_warp > 0) {
    k_ebo_warp<<<O.P.nblk_warp, kEbeWarpsPerBlock * 32, 0, st>>>(O.P.d_groups, O.d_off, O.P.d_blk_group, O.P.d_blk_e0, x, O.v, skip);
    PCGB_CHECK_LAUNCH();
    ++nl;
  }
  if (O.P.n > 0) {
    k_ebo_sum<<<(unsigned)((O.P.n + 255) / 256), 256, 0, st>>>(O.P.n, O.d_ptr, O.d_pos, O.v, y, skip);
    PCGB_CHECK_LAUNCH();
    ++nl;
  }
  if (launches) *launches += nl;
  return PCGB_OK;
}

}  // namespace pcgb
