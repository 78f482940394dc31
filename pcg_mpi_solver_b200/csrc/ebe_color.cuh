// ebe_color.cuh - operator-level variant (tests/test_gpu_ebe_colored.py, tests/test_gpu_ebe_color_edges.py):
// atomics-free, bit-reproducible variant of the matrix-free operator of ebe.cuh.  The host colours the elements
// (pcg_mpi_solver_b200/coloring.py: no two elements of a colour share a free dof) and passes every (pattern group,
// colour) slice as its own group, ordered by colour ("phase").  Inside one phase the scatter y[dof] += v needs no
// atomic; phases run as consecutive launches, so the summation order per dof is fixed (colour order) - the
// deterministic counterpart of np.bincount (pcg_solver.py:300).  Rationale: DESIGN.md section 6 item 1 - the 24
// fp64 RED per element are ~80 % of the first EBE kernel's time.
//
// The result, bit for bit (include/pcgb200.h): every free dof d starts from +0.0; colours are taken in ascending order,
// and for the one element e of the colour that touches d, every local index i with idx[i] = d in ascending i does
// y_d = y_d + v_{e,i}, where u_j = s_j x_j (0 for a clamped dof), acc = fma(Ke[i][j], u_j, acc) over j ascending from
// 0.0 and v = round(acc * Ck_e), negated when s_i is set.  Every operation of the scatter is an explicit __dmul_rn /
// __dadd_rn so that contraction cannot fuse it into an fma (hexop.cuh does the same).
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
  EbePlan P;                       // groups (one per pattern group x colour), device tables; each ke is Ke TRANSPOSED
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
    double v = __dmul_rn(acc, c);
    if (SIGN && ((sbits >> i) & 1u)) v = -v;
    if (id[i] >= 0) y[id[i]] = __dadd_rn(y[id[i]], v);   // no other element of this colour touches this dof; an element's
  }                                                        // own repeats come in ascending i from this one thread
}

// One warp per element.  The rows go to shared memory first; then the lane of a dof's FIRST local index adds every
// occurrence of that dof in ascending local index, so an element that lists a dof twice (in one 32-lane pass or in two)
// loses no update and sums it in the documented order.
__global__ void __launch_bounds__(kEbeWarpsPerBlock * 32)
k_ebe_warp_p(const EbeGroup *__restrict__ groups, const int *__restrict__ blk_group, const int64_t *__restrict__ blk_e0, int blk0,
             const double *__restrict__ x, double *__restrict__ y) {
  __shared__ double su[kEbeWarpsPerBlock][96];
  __shared__ double sv[kEbeWarpsPerBlock][96];
  __shared__ int sid[kEbeWarpsPerBlock][96];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int blk = blk0 + blockIdx.x;
  const EbeGroup g = groups[blk_group[blk]];
  const int64_t e = blk_e0[blk] + warp;
  if (e >= g.ne) return;
  const int nd = g.nd;
  unsigned sneg = 0;   // bit k: sign of local index lane + 32 k (the gather and the rows visit the same indices per lane)
  for (int j = lane, k = 0; j < nd; j += 32, ++k) {
    const int id = g.idx[(int64_t)j * g.ne + e];
    double v = id >= 0 ? __ldg(x + id) : 0.0;
    const bool s = g.sign != nullptr && g.sign[(int64_t)j * g.ne + e] != 0;
    su[warp][j] = s ? -v : v;
    sid[warp][j] = id;
    if (s) sneg |= 1u << k;
  }
  __syncwarp();
  const double c = g.ck[e];
  for (int i = lane, k = 0; i < nd; i += 32, ++k) {
    double acc = 0.0;
    for (int j = 0; j < nd; ++j) acc = fma(__ldg(g.ke + (int64_t)j * nd + i), su[warp][j], acc);   // ke = Ke^T: row i of Ke
    double v = __dmul_rn(acc, c);
    if ((sneg >> k) & 1u) v = -v;
    sv[warp][i] = v;
  }
  __syncwarp();
  for (int i = lane; i < nd; i += 32) {
    const int id = sid[warp][i];
    if (id < 0) continue;
    int j = 0;
    while (sid[warp][j] != id) ++j;
    if (j < i) continue;                 // not the first occurrence: that lane adds this one
    double yv = __dadd_rn(y[id], sv[warp][i]);
    for (j = i + 1; j < nd; ++j)
      if (sid[warp][j] == id) yv = __dadd_rn(yv, sv[warp][j]);
    y[id] = yv;
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
