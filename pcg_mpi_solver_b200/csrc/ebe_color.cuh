// ebe_color.cuh - operator-level variant (tests/test_gpu_ebe_colored.py):
// atomics-free, bit-reproducible variant of the matrix-free operator of ebe.cuh.  The host colours the elements
// (pcg_mpi_solver_b200/coloring.py: no two elements of a colour share a node) and passes every (pattern group,
// colour) slice as its own group, ordered by colour ("phase").  Inside one phase the scatter y[dof] += v needs no
// atomic; phases run as consecutive launches, so the summation order per dof is fixed (colour order) - the
// deterministic counterpart of np.bincount (pcg_solver.py:300).  Rationale: DESIGN.md section 6 item 1 - the 24
// fp64 RED per element are ~80 % of the first EBE kernel's time.
#pragma once
#include <vector>

#include "common.cuh"
#include "ebe.cuh"

namespace pcgb {

struct EbeLaunch {
  int kind;        // 0 = k_ebe_t24p on group `a` ; 1 = k_ebe_warp_p on blocks [a, b)
  int a, b;
};

struct EbeColorPlan {
  EbePlan P;                       // groups (one per pattern group x colour), device tables
  std::vector<EbeLaunch> launches; // in phase order
};

template <bool SIGN>
__global__ void __launch_bounds__(128)
k_ebe_t24p(const int *__restrict__ idx, const unsigned char *__restrict__ sign, const double *__restrict__ ck, int slot, int64_t ne,
           const double *__restrict__ x, double *__restrict__ y) {
  const int64_t e = blockIdx.x * (int64_t)128 + threadIdx.x;
  if (e >= ne) return;
  int id[24];
  double u[24];
  unsigned sbits = 0;
#pragma unroll
  for (int j = 0; j < 24; ++j) {
    id[j] = idx[(int64_t)j * ne + e];
    double v = id[j] >= 0 ? __ldg(x + id[j]) : 0.0;
    if (SIGN && sign[(int64_t)j * ne + e]) { v = -v; sbits |= 1u << j; }
    u[j] = v;
  }
  const double c = ck[e];
#pragma unroll
  for (int i = 0; i < 24; ++i) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < 24; ++j) acc = fma(c_ebe_ke24[slot][i * 24 + j], u[j], acc);
    acc *= c;
    if (SIGN && ((sbits >> i) & 1u)) acc = -acc;
    if (id[i] >= 0) y[id[i]] += acc;   // no other element of this colour touches this dof
  }
}

__global__ void __launch_bounds__(kEbeWarpsPerBlock * 32)
k_ebe_warp_p(const EbeGroup *__restrict__ groups, const int *__restrict__ blk_group, const int64_t *__restrict__ blk_e0, int blk0,
             const double *__restrict__ x, double *__restrict__ y) {
  __shared__ double su[kEbeWarpsPerBlock][96];
  __shared__ int sid[kEbeWarpsPerBlock][96];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int blk = blk0 + blockIdx.x;
  const EbeGroup g = groups[blk_group[blk]];
  const int64_t e = blk_e0[blk] + warp;
  if (e >= g.ne) return;
  const int nd = g.nd;
  for (int j = lane; j < nd; j += 32) {
    const int id = g.idx[(int64_t)j * g.ne + e];
    double v = id >= 0 ? __ldg(x + id) : 0.0;
    const bool s = g.sign != nullptr && g.sign[(int64_t)j * g.ne + e] != 0;
    su[warp][j] = s ? -v : v;
    sid[warp][j] = s ? (id | (int)0x40000000) : id;
  }
  __syncwarp();
  const double c = g.ck[e];
  for (int i = lane; i < nd; i += 32) {
    double acc = 0.0;
    for (int j = 0; j < nd; ++j) acc = fma(__ldg(g.ke + (int64_t)j * nd + i), su[warp][j], acc);
    acc *= c;
    int id = sid[warp][i];
    if (id >= 0) {
      if (id & 0x40000000) { acc = -acc; id &= 0x3fffffff; }
      y[id] += acc;
    }
  }
}

inline int ebe_color_apply(const EbeColorPlan &C, const double *x, double *y, cudaStream_t st) {
  const EbePlan &P = C.P;
  PCGB_CUDA(cudaMemsetAsync(y, 0, (size_t)P.n * sizeof(double), st));
  for (const EbeLaunch &L : C.launches) {
    if (L.kind == 0) {
      const EbeGroup &g = P.groups[(size_t)L.a];
      const unsigned grid = (unsigned)((g.ne + 127) / 128);
      if (g.sign) k_ebe_t24p<true><<<grid, 128, 0, st>>>(g.idx, g.sign, g.ck, g.slot, g.ne, x, y);
      else k_ebe_t24p<false><<<grid, 128, 0, st>>>(g.idx, nullptr, g.ck, g.slot, g.ne, x, y);
    } else {
      k_ebe_warp_p<<<L.b - L.a, kEbeWarpsPerBlock * 32, 0, st>>>(P.d_groups, P.d_blk_group, P.d_blk_e0, L.a, x, y);
    }
    PCGB_CHECK_LAUNCH();
  }
  return PCGB_OK;
}

}  // namespace pcgb
