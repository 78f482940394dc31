// hexgen.cuh - on-device generator of the sub-assembled stiffness matrix of a box of trilinear hex
// elements (benchmark configs C2 / C3 / C5 of BASELINE.json; SURVEY.md 8(d)).
//
// What it stands in for: the assembled form  A = K[Eff,Eff],  K = sum_e P_e^T (Ck_e Ke) P_e,  of the
// reference's element-by-element operator (pcg_solver.py:263-300) on a structured mesh where every
// element has the same pattern matrix Ke (24x24) and scale Ck (= E*h, ElemList_Ck).  A 256^3 block is
// 4.09e9 non-zeros (49 GB) and cannot be assembled on the host, hence a kernel.
//
// Numbering: local node (lx,ly,lz) of the box, x fastest; nodes whose GLOBAL x index is 0 are
// clamped and dropped; free dof = 3*freenode + dir.  Columns of a row are emitted in ascending order.
#pragma once
#include "common.cuh"

namespace pcgb {

__constant__ double c_hex_ke[24 * 24];

struct HexGeom {
  int nx, ny, nz;   // elements in the box
  int x_lo;         // 1 if the box touches the clamped face (global x index 0), else 0
  int nxf;          // free nodes per x line = nx + 1 - x_lo
  int64_t nfree_nodes;
};

inline HexGeom hex_geom(const pcgb_hex_box *b) {
  HexGeom g;
  g.nx = b->ne[0]; g.ny = b->ne[1]; g.nz = b->ne[2];
  g.x_lo = b->e0[0] == 0 ? 1 : 0;
  g.nxf = g.nx + 1 - g.x_lo;
  g.nfree_nodes = (int64_t)g.nxf * (g.ny + 1) * (g.nz + 1);
  return g;
}

// one thread per free node: number of (free, in-box) neighbour nodes -> 3 rows of 3*nb entries each
__global__ void k_hex_count(HexGeom g, int64_t *__restrict__ rowcount) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t == 0) rowcount[0] = 0;
  if (t >= g.nfree_nodes) return;
  const int fx = (int)(t % g.nxf);
  const int ly = (int)((t / g.nxf) % (g.ny + 1));
  const int lz = (int)(t / ((int64_t)g.nxf * (g.ny + 1)));
  const int lx = fx + g.x_lo;
  int nb = 0;
  for (int dz = -1; dz <= 1; ++dz)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int bx = lx + dx, by = ly + dy, bz = lz + dz;
        if (bx < g.x_lo || bx > g.nx || by < 0 || by > g.ny || bz < 0 || bz > g.nz) continue;
        ++nb;
      }
  for (int d = 0; d < 3; ++d) rowcount[1 + 3 * t + d] = 3 * nb;
}

// one warp per free node; lane = neighbour slot (27 of 32 lanes active); each active lane computes the
// 3x3 block coupling node a to neighbour b by summing the element matrices of the elements containing both.
__global__ void __launch_bounds__(256)
k_hex_fill(HexGeom g, double ck, const int64_t *__restrict__ rowptr, int *__restrict__ col, double *__restrict__ val) {
  const int64_t t = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= g.nfree_nodes) return;
  const int fx = (int)(t % g.nxf);
  const int ly = (int)((t / g.nxf) % (g.ny + 1));
  const int lz = (int)(t / ((int64_t)g.nxf * (g.ny + 1)));
  const int lx = fx + g.x_lo;
  const int dx = lane % 3 - 1, dy = (lane / 3) % 3 - 1, dz = lane / 9 - 1;
  const int bx = lx + dx, by = ly + dy, bz = lz + dz;
  const bool valid = lane < 27 && !(bx < g.x_lo || bx > g.nx || by < 0 || by > g.ny || bz < 0 || bz > g.nz);
  // slot of this neighbour inside the row = number of valid lanes below (ascending column order)
  const unsigned mask = __ballot_sync(0xffffffffu, valid);
  if (!valid) return;
  const int slot = __popc(mask & ((1u << lane) - 1u));
  double blk[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  // elements containing both a=(lx,ly,lz) and b: origin o with o<=min(a,b), o+1>=max(a,b), inside the box
  const int ox0 = max(max(lx, bx) - 1, 0), ox1 = min(min(lx, bx), g.nx - 1);
  const int oy0 = max(max(ly, by) - 1, 0), oy1 = min(min(ly, by), g.ny - 1);
  const int oz0 = max(max(lz, bz) - 1, 0), oz1 = min(min(lz, bz), g.nz - 1);
  for (int oz = oz0; oz <= oz1; ++oz)
    for (int oy = oy0; oy <= oy1; ++oy)
      for (int ox = ox0; ox <= ox1; ++ox) {
        const int la = (lx - ox) + 2 * (ly - oy) + 4 * (lz - oz);
        const int lb = (bx - ox) + 2 * (by - oy) + 4 * (bz - oz);
#pragma unroll
        for (int d = 0; d < 3; ++d)
#pragma unroll
          for (int e = 0; e < 3; ++e) blk[d * 3 + e] += c_hex_ke[(la * 3 + d) * 24 + lb * 3 + e];
      }
  const int64_t bnode = ((int64_t)bz * (g.ny + 1) + by) * g.nxf + (bx - g.x_lo);
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const int64_t base = rowptr[3 * t + d] + 3 * slot;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      col[base + e] = (int)(3 * bnode + e);
      val[base + e] = ck * blk[d * 3 + e];
    }
  }
}

// k_hex_fill for a heterogeneous box: the same rows, columns and element loop, but every element brings its own matrix.
// kElemMat = false: element e = (oz * ny + oy) * nx + ox of the box contributes ck[e] * Ke (Ke in c_hex_ke; a voxel model
// with one Young's modulus per element).  kElemMat = true: it contributes kel[576 e ..] (one row-major 24x24 matrix per
// element; the Galerkin coarse levels of the multigrid).  Each block entry is summed from 0.0 over the elements in
// (oz, oy, ox) ascending order.
template <bool kElemMat>
__global__ void __launch_bounds__(256)
k_hex_fill_var(HexGeom g, const double *__restrict__ ck, const double *__restrict__ kel, const int64_t *__restrict__ rowptr,
               int *__restrict__ col, double *__restrict__ val) {
  const int64_t t = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= g.nfree_nodes) return;
  const int fx = (int)(t % g.nxf);
  const int ly = (int)((t / g.nxf) % (g.ny + 1));
  const int lz = (int)(t / ((int64_t)g.nxf * (g.ny + 1)));
  const int lx = fx + g.x_lo;
  const int dx = lane % 3 - 1, dy = (lane / 3) % 3 - 1, dz = lane / 9 - 1;
  const int bx = lx + dx, by = ly + dy, bz = lz + dz;
  const bool valid = lane < 27 && !(bx < g.x_lo || bx > g.nx || by < 0 || by > g.ny || bz < 0 || bz > g.nz);
  const unsigned mask = __ballot_sync(0xffffffffu, valid);
  if (!valid) return;
  const int slot = __popc(mask & ((1u << lane) - 1u));
  double blk[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const int ox0 = max(max(lx, bx) - 1, 0), ox1 = min(min(lx, bx), g.nx - 1);
  const int oy0 = max(max(ly, by) - 1, 0), oy1 = min(min(ly, by), g.ny - 1);
  const int oz0 = max(max(lz, bz) - 1, 0), oz1 = min(min(lz, bz), g.nz - 1);
  for (int oz = oz0; oz <= oz1; ++oz)
    for (int oy = oy0; oy <= oy1; ++oy)
      for (int ox = ox0; ox <= ox1; ++ox) {
        const int la = (lx - ox) + 2 * (ly - oy) + 4 * (lz - oz);
        const int lb = (bx - ox) + 2 * (by - oy) + 4 * (bz - oz);
        const int64_t e = ((int64_t)oz * g.ny + oy) * g.nx + ox;
        if (kElemMat) {
          const double *k = kel + 576 * e;
#pragma unroll
          for (int d = 0; d < 3; ++d)
#pragma unroll
            for (int c = 0; c < 3; ++c) blk[d * 3 + c] += k[(la * 3 + d) * 24 + lb * 3 + c];
        } else {
          const double s = ck[e];
#pragma unroll
          for (int d = 0; d < 3; ++d)
#pragma unroll
            for (int c = 0; c < 3; ++c) blk[d * 3 + c] += s * c_hex_ke[(la * 3 + d) * 24 + lb * 3 + c];
        }
      }
  const int64_t bnode = ((int64_t)bz * (g.ny + 1) + by) * g.nxf + (bx - g.x_lo);
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const int64_t base = rowptr[3 * t + d] + 3 * slot;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      col[base + c] = (int)(3 * bnode + c);
      val[base + c] = blk[d * 3 + c];
    }
  }
}

// *bad = 1 when some v[i] is not a finite positive number (a per-element Ck field)
__global__ void k_field_check(int64_t n, const double *__restrict__ v, int *__restrict__ bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
    if (!(v[i] > 0.0) || !isfinite(v[i])) *bad = 1;
}

}  // namespace pcgb
