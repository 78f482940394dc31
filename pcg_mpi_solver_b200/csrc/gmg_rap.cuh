// gmg_rap.cuh - level 1 of the multigrid's "rap" field hierarchy (pcgb_mg_create_field_rap): y_1 = P^T A_0 P x_1 applied
// from the fine Ck field, with no level-1 matrix, and the set-up kernel that gives its diagonal.
//
// k_mg_rap1 is bit-identical to the three launches it fuses, with the fine operator applied as k_hexop<true> does:
//   u = k_mg_prolong_add of x_1 into a zero fine vector   (u_f = 0.0 + s_f, s_f the (z, y, x)-ordered sum of <= 8 terms)
//   v = k_hexop<true> of u with the fine Ck                 (hex_node_rows; 0.0 for clamped nodes and nodes outside the box)
//   y_1 = k_mg_restrict of v, own_f = NULL                  (<= 27 fine nodes in (dz, dy, dx) order from 0.0)
// The transfer weights are powers of two, so w v is exact (outside the subnormal range) and the explicit
// __dadd_rn(s, __dmul_rn(w, v)) here equals the transfer kernels' possibly contracted s += w * v.
//
// One CTA per brick of kRapBX x kRapBY x kRapBZ coarse nodes, in dynamic shared memory:
//   xs  coarse x on the brick plus a one-node halo (B + 2 per axis), 0.0 for clamped nodes and nodes outside the box
//   us  u on the 2B + 3 fine nodes per axis around the brick
//   cs  Ck of the 2B + 2 fine elements per axis those nodes touch, 0.0 outside the box
//   vs  v on the 2B + 1 fine nodes per axis the restriction reads; it shares memory with xs, which is dead once u is built
// Fine nodes whose v is computed by two bricks are computed twice (1.34x the fine work for 8 x 4 x 4), and no fine-size
// vector is needed.
#pragma once
#include "common.cuh"
#include "gmg.cuh"
#include "hexop.cuh"

namespace pcgb {

constexpr int kRapBX = 8, kRapBY = 4, kRapBZ = 4;                       // coarse nodes per brick
constexpr int kRapThreads = 352;                                          // 11 warps: 4 rounds over the 1377 v nodes
constexpr int kRapUX = 2 * kRapBX + 3, kRapUY = 2 * kRapBY + 3, kRapUZ = 2 * kRapBZ + 3;
constexpr int kRapVX = 2 * kRapBX + 1, kRapVY = 2 * kRapBY + 1, kRapVZ = 2 * kRapBZ + 1;
constexpr int kRapCX = 2 * kRapBX + 2, kRapCY = 2 * kRapBY + 2, kRapCZ = 2 * kRapBZ + 2;
constexpr int kRapXX = kRapBX + 2, kRapXY = kRapBY + 2, kRapXZ = kRapBZ + 2;
constexpr int kRapU = 3 * kRapUX * kRapUY * kRapUZ, kRapV = 3 * kRapVX * kRapVY * kRapVZ, kRapC = kRapCX * kRapCY * kRapCZ;
static_assert(3 * kRapXX * kRapXY * kRapXZ <= kRapV, "x_1 shares memory with v");
constexpr size_t kRapSmem = sizeof(double) * (kRapU + kRapV + kRapC);   // 102 624 bytes

struct RapShape {
  HexGeom gf, gc;       // the fine box and level 1
  int nbx, nby, nbz;    // bricks per axis (x over level 1's free nodes)
};

inline RapShape rap_shape(const HexGeom &gf, const HexGeom &gc) {
  RapShape s;
  s.gf = gf;
  s.gc = gc;
  s.nbx = (gc.nxf + kRapBX - 1) / kRapBX;
  s.nby = (gc.ny + 1 + kRapBY - 1) / kRapBY;
  s.nbz = (gc.nz + 1 + kRapBZ - 1) / kRapBZ;
  return s;
}

__global__ void __launch_bounds__(kRapThreads, 2)
k_mg_rap1(const __grid_constant__ HexKe ke, RapShape s, const double *__restrict__ ckf, const double *__restrict__ x1,
          double *__restrict__ y1, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  extern __shared__ double smem[];
  double *us = smem, *vs = smem + kRapU, *cs = vs + kRapV, *xs = vs;
  const HexGeom &gf = s.gf, &gc = s.gc;
  const int b = blockIdx.x;
  const int bx = b % s.nbx, by = (b / s.nbx) % s.nby, bz = b / (s.nbx * s.nby);
  const int cx0 = gc.x_lo + bx * kRapBX, cy0 = by * kRapBY, cz0 = bz * kRapBZ;   // first coarse node of the brick
  // x_1 on coarse nodes c0 - 1 .. c0 + B
  for (int t = threadIdx.x; t < 3 * kRapXX * kRapXY * kRapXZ; t += kRapThreads) {
    const int c = t % (3 * kRapXX), r = t / (3 * kRapXX);
    const int cx = cx0 - 1 + c / 3, cy = cy0 - 1 + r % kRapXY, cz = cz0 - 1 + r / kRapXY;
    double v = 0.0;
    if (cx >= gc.x_lo && cx <= gc.nx && cy >= 0 && cy <= gc.ny && cz >= 0 && cz <= gc.nz) v = x1[3 * mg_index(gc, cx, cy, cz) + c % 3];
    xs[t] = v;
  }
  // Ck on fine elements 2 c0 - 2 .. 2 c0 + 2B - 1
  const int ex0 = 2 * cx0 - 2, ey0 = 2 * cy0 - 2, ez0 = 2 * cz0 - 2;
  for (int t = threadIdx.x; t < kRapC; t += kRapThreads) {
    const int ox = ex0 + t % kRapCX, oy = ey0 + (t / kRapCX) % kRapCY, oz = ez0 + t / (kRapCX * kRapCY);
    double v = 0.0;
    if (ox >= 0 && ox < gf.nx && oy >= 0 && oy < gf.ny && oz >= 0 && oz < gf.nz) v = ckf[((int64_t)oz * gf.ny + oy) * gf.nx + ox];
    cs[t] = v;
  }
  __syncthreads();
  // u = P x_1 on fine nodes 2 c0 - 2 .. 2 c0 + 2B (k_mg_prolong_add into zeros)
  for (int t = threadIdx.x; t < kRapUX * kRapUY * kRapUZ; t += kRapThreads) {
    const int i = t % kRapUX, j = (t / kRapUX) % kRapUY, k = t / (kRapUX * kRapUY);
    const int fx = ex0 + i, fy = ey0 + j, fz = ez0 + k;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    const bool free_node = fx >= gf.x_lo && fx <= gf.nx && fy >= 0 && fy <= gf.ny && fz >= 0 && fz <= gf.nz;
    if (free_node) {
      const int nz = (fz & 1) ? 2 : 1, ny = (fy & 1) ? 2 : 1, nx = (fx & 1) ? 2 : 1;
      const double w = (nx == 2 ? 0.5 : 1.0) * (ny == 2 ? 0.5 : 1.0) * (nz == 2 ? 0.5 : 1.0);
      for (int kz = 0; kz < nz; ++kz) {
        const int cz = (fz >> 1) + kz;
        for (int ky = 0; ky < ny; ++ky) {
          const int cy = (fy >> 1) + ky;
          for (int kx = 0; kx < nx; ++kx) {
            const int cx = (fx >> 1) + kx;
            if (cx < gc.x_lo) continue;   // clamped coarse node
            const double *src = xs + 3 * (((cz - cz0 + 1) * kRapXY + (cy - cy0 + 1)) * kRapXX + (cx - cx0 + 1));
            s0 = __dadd_rn(s0, __dmul_rn(w, src[0]));
            s1 = __dadd_rn(s1, __dmul_rn(w, src[1]));
            s2 = __dadd_rn(s2, __dmul_rn(w, src[2]));
          }
        }
      }
      s0 = __dadd_rn(0.0, s0); s1 = __dadd_rn(0.0, s1); s2 = __dadd_rn(0.0, s2);   // the zero fine vector plus P x_1
    }
    us[3 * t] = s0; us[3 * t + 1] = s1; us[3 * t + 2] = s2;
  }
  __syncthreads();
  // v = A_0 u on the free fine nodes 2 c0 - 1 .. 2 c0 + 2B - 1 (k_hexop<true>'s per-node product)
  for (int t = threadIdx.x; t < kRapVX * kRapVY * kRapVZ; t += kRapThreads) {
    const int i = t % kRapVX, j = (t / kRapVX) % kRapVY, k = t / (kRapVX * kRapVY);
    const int fx = ex0 + 1 + i, fy = ey0 + 1 + j, fz = ez0 + 1 + k;
    if (fx < gf.x_lo || fx > gf.nx || fy < 0 || fy > gf.ny || fz < 0 || fz > gf.nz) continue;   // never restricted
    double r0, r1, r2;
    hex_node_rows(ke, gf, fx, fy, fz,
                  [&](int ax, int ay, int az) { return cs[((k + 1 - az) * kRapCY + (j + 1 - ay)) * kRapCX + (i + 1 - ax)]; },
                  [&](int dx, int dy, int dz) { return us + 3 * (((k + 1 + dz) * kRapUY + (j + 1 + dy)) * kRapUX + (i + 1 + dx)); },
                  r0, r1, r2);
    vs[3 * t] = r0; vs[3 * t + 1] = r1; vs[3 * t + 2] = r2;
  }
  __syncthreads();
  // y_1 = P^T v on the brick's coarse nodes (k_mg_restrict)
  for (int t = threadIdx.x; t < kRapBX * kRapBY * kRapBZ; t += kRapThreads) {
    const int cx = cx0 + t % kRapBX, cy = cy0 + (t / kRapBX) % kRapBY, cz = cz0 + t / (kRapBX * kRapBY);
    if (cx > gc.nx || cy > gc.ny || cz > gc.nz) continue;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int dz = -1; dz <= 1; ++dz) {
      const int fz = 2 * cz + dz;
      if (fz < 0 || fz > gf.nz) continue;
      for (int dy = -1; dy <= 1; ++dy) {
        const int fy = 2 * cy + dy;
        if (fy < 0 || fy > gf.ny) continue;
        for (int dx = -1; dx <= 1; ++dx) {
          const int fx = 2 * cx + dx;
          if (fx < gf.x_lo || fx > gf.nx) continue;
          const double w = (dx ? 0.5 : 1.0) * (dy ? 0.5 : 1.0) * (dz ? 0.5 : 1.0);
          const double *src = vs + 3 * (((fz - ez0 - 1) * kRapVY + (fy - ey0 - 1)) * kRapVX + (fx - ex0 - 1));
          s0 = __dadd_rn(s0, __dmul_rn(w, src[0]));
          s1 = __dadd_rn(s1, __dmul_rn(w, src[1]));
          s2 = __dadd_rn(s2, __dmul_rn(w, src[2]));
        }
      }
    }
    const int64_t c = mg_index(gc, cx, cy, cz);
    y1[3 * c] = s0; y1[3 * c + 1] = s1; y1[3 * c + 2] = s2;
  }
}

// Level-1 diagonal from a slab of its element matrices (kel: the elements of layers z0 .. z1 - 1, x fastest): one thread per
// free node of planes z0 .. z1, each of its three diagonal entries d += K_e[3 la + dir][3 la + dir] over the slab's elements
// at the node in (oz, oy, ox) ascending order.  Slabs run in ascending z on a zeroed d, so every entry is summed from 0.0 in
// the order of k_hex_fill_var<true>, and the diagonal is that of the level's CSR bit for bit.
__global__ void __launch_bounds__(256)
k_mg_rap_diag(HexGeom g, int z0, int z1, const double *__restrict__ kel, double *__restrict__ d) {
  const int64_t plane = (int64_t)g.nxf * (g.ny + 1);
  const int64_t t = z0 * plane + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (z1 + 1) * plane || t >= g.nfree_nodes) return;
  int lx, ly, lz;
  mg_node(g, t, lx, ly, lz);
  double r0 = d[3 * t], r1 = d[3 * t + 1], r2 = d[3 * t + 2];
  for (int oz = max(lz - 1, z0); oz <= min(lz, z1 - 1); ++oz)
    for (int oy = max(ly - 1, 0); oy <= min(ly, g.ny - 1); ++oy)
      for (int ox = max(lx - 1, 0); ox <= min(lx, g.nx - 1); ++ox) {
        const int la = (lx - ox) + 2 * (ly - oy) + 4 * (lz - oz);
        const double *k = kel + 576 * (((int64_t)(oz - z0) * g.ny + oy) * g.nx + ox);
        r0 += k[(3 * la + 0) * 25];
        r1 += k[(3 * la + 1) * 25];
        r2 += k[(3 * la + 2) * 25];
      }
  d[3 * t] = r0; d[3 * t + 1] = r1; d[3 * t + 2] = r2;
}

}  // namespace pcgb
