// hexop.cuh - the index-free matrix-free operator of a hex box (uniform Ck or one Ck per element): y = K_i x computed per
// node from the node's coordinates, bit-identical to the ordered EBE operator (ebe_ordered.cuh) on the box's single
// pattern group (hexmesh.hex_type_group).  It stands in for calcMatVecProd (pcg_solver.py:263-300) like that operator,
// without its index list, slot buffer and per-dof position lists.
//
// Numbering (hexgen.cuh): free node (lz, ly, fx), x fastest, lx = fx + x_lo; dof = 3 node + dir.  Element e = (oz ny + oy) nx
// + ox, local node l at (l&1, l>>1&1, l>>2&1).  For free dof (node, d) the ordered operator's slots are, in ascending
// position, the elements around the node in ascending local index la (each element holds the node at exactly one la):
//
//   y = 0.0;  for la = 0..7 with e = node - (la&1, la>>1&1, la>>2&1) inside the box:
//       acc = 0.0;  for b = 0..23:  acc = fma(Ke[3 la + d][b], Ck_e * x_b, acc)     (x_b = 0.0 for a clamped node)
//       y = y + acc
//
// which is k_ebo_t24's fma chain followed by k_ebo_sum's sum.  Every operation is an explicit __dmul_rn / __fma_rn /
// __dadd_rn so that contraction cannot change it.
//
// Kernel: one CTA per brick of kHxBX x kHxBY x kHxBZ nodes, one thread per node computing its three rows.  The CTA stages
// the brick's x plus a one-node halo (0.0 outside the free nodes) and, with a field, the brick's Ck in shared memory with
// plain coalesced loads, which works for every nxf.  la is the outer loop and fully unrolled, so la is uniform across a
// warp and every Ke entry is a compile-time offset into the kernel's 4608-byte __grid_constant__ parameter: a constant-bank
// operand of the DFMA.  Ke thus belongs to the launch (the handle's copy), not to c_hex_ke or the c_ebe_ke24 slots.
#pragma once
#include "common.cuh"
#include "hexgen.cuh"

namespace pcgb {

struct HexKe { double k[576]; };       // row-major 24x24 element matrix, passed by value to every launch
struct HexKeDiag { double k[24]; };    // its diagonal

constexpr int kHxBX = 32, kHxBY = 4, kHxBZ = 2;           // nodes per brick
constexpr int kHxThreads = kHxBX * kHxBY * kHxBZ;
constexpr int kHxSX = kHxBX + 2, kHxSY = kHxBY + 2, kHxSZ = kHxBZ + 2;   // staged nodes (one-node halo)

struct HexOpShape {
  HexGeom g;
  int nbx, nby, nbz;    // bricks per axis (x over the free nodes)
};

inline HexOpShape hexop_shape(const HexGeom &g, bool periodic = false) {
  HexOpShape s;
  s.g = g;
  s.nbx = (g.nxf + kHxBX - 1) / kHxBX;
  s.nby = (g.ny + (periodic ? 0 : 1) + kHxBY - 1) / kHxBY;
  s.nbz = (g.nz + (periodic ? 0 : 1) + kHxBZ - 1) / kHxBZ;
  return s;
}

// A periodic cell of ne[0] x ne[1] x ne[2] elements (the box must be the whole mesh: e0 = 0, ne = ng): x_lo = 0 and nxf = nx,
// every node free, nfree_nodes = nx ny nz
inline HexGeom periodic_geom(const pcgb_hex_box *b) {
  HexGeom g;
  g.nx = b->ne[0]; g.ny = b->ne[1]; g.nz = b->ne[2];
  g.x_lo = 0;
  g.nxf = g.nx;
  g.nfree_nodes = (int64_t)g.nx * g.ny * g.nz;
  return g;
}

// the coordinate c of a periodic axis of n nodes, for c in -1 .. n: -1 wraps to n - 1 and n to 0
__device__ __forceinline__ int hex_wrap(int c, int n) { return c < 0 ? c + n : c >= n ? c - n : c; }

// The three rows of free node (lx, ly, lz) of K x, in the order stated at the top of this file: la outer over the elements
// inside the box, b = (lb, e) inner with an fma chain from 0.0, then the element's sum added to the row.  ck_at(ax, ay, az)
// is the Ck of element node - (ax, ay, az); x_at(dx, dy, dz) points at the three staged x of node + (dx, dy, dz), d in
// {-1, 0, 1}, 0.0 for a clamped node or one outside the box.  k_hexop and the multigrid's fused level-1 product (gmg_rap.cuh)
// both call it, so their per-node arithmetic is one piece of code.  kAll: every element around the node exists (a periodic
// cell, whose ck_at and x_at wrap), so the inside test is dropped; the order is unchanged.
template <bool kAll = false, class CkAt, class XAt>
__device__ __forceinline__ void hex_node_rows(const HexKe &ke, const HexGeom &g, int lx, int ly, int lz, CkAt ck_at, XAt x_at,
                                              double &r0, double &r1, double &r2) {
  r0 = 0.0; r1 = 0.0; r2 = 0.0;
#pragma unroll
  for (int la = 0; la < 8; ++la) {
    const int ax = la & 1, ay = (la >> 1) & 1, az = la >> 2;
    const int ox = lx - ax, oy = ly - ay, oz = lz - az;
    if (!kAll && (ox < 0 || ox >= g.nx || oy < 0 || oy >= g.ny || oz < 0 || oz >= g.nz)) continue;
    const double c = ck_at(ax, ay, az);
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll
    for (int lb = 0; lb < 8; ++lb) {
      const double *xs = x_at((lb & 1) - ax, ((lb >> 1) & 1) - ay, (lb >> 2) - az);
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const double u = __dmul_rn(c, xs[e]);                                   // :279  Ck * U
        a0 = __fma_rn(ke.k[(3 * la + 0) * 24 + 3 * lb + e], u, a0);              // :279  Ke @ (Ck * U)
        a1 = __fma_rn(ke.k[(3 * la + 1) * 24 + 3 * lb + e], u, a1);
        a2 = __fma_rn(ke.k[(3 * la + 2) * 24 + 3 * lb + e], u, a2);
      }
    }
    r0 = __dadd_rn(r0, a0);                                                     // :300  np.bincount's order
    r1 = __dadd_rn(r1, a1);
    r2 = __dadd_rn(r2, a2);
  }
}

// kPeriodic: the periodic cell's numbering and staging (header); kPeriodic = false is the box's kernel unchanged
template <bool kField, bool kPeriodic = false>
__global__ void __launch_bounds__(kHxThreads)
k_hexop(const __grid_constant__ HexKe ke, HexOpShape s, double ck, const double *__restrict__ ckf, const double *__restrict__ x,
        double *__restrict__ y, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  __shared__ double sx[kHxSZ][kHxSY][kHxSX * 3];
  __shared__ double sc[kField ? kHxBZ + 1 : 1][kField ? kHxBY + 1 : 1][kField ? kHxBX + 1 : 1];
  const HexGeom &g = s.g;
  const int b = blockIdx.x;
  const int bx = b % s.nbx, by = (b / s.nbx) % s.nby, bz = b / (s.nbx * s.nby);
  const int lx0 = g.x_lo + bx * kHxBX, ly0 = by * kHxBY, lz0 = bz * kHxBZ;   // first node of the brick (lx counts the clamped line)
  for (int t = threadIdx.x; t < kHxSZ * kHxSY * kHxSX * 3; t += kHxThreads) {
    const int c = t % (kHxSX * 3), r = t / (kHxSX * 3);
    const int sy = r % kHxSY, sz = r / kHxSY;
    const int lx = lx0 - 1 + c / 3, ly = ly0 - 1 + sy, lz = lz0 - 1 + sz;
    double v = 0.0;
    if (kPeriodic) {   // nodes -1 .. n of each axis are read (wrapped); staged nodes beyond are never read
      if (lx <= g.nx && ly <= g.ny && lz <= g.nz)
        v = x[3 * (((int64_t)hex_wrap(lz, g.nz) * g.ny + hex_wrap(ly, g.ny)) * g.nx + hex_wrap(lx, g.nx)) + c % 3];
    } else if (lx >= g.x_lo && lx <= g.nx && ly >= 0 && ly <= g.ny && lz >= 0 && lz <= g.nz) {
      v = x[3 * (((int64_t)lz * (g.ny + 1) + ly) * g.nxf + (lx - g.x_lo)) + c % 3];
    }
    sx[sz][sy][c] = v;
  }
  if (kField) {
    for (int t = threadIdx.x; t < (kHxBZ + 1) * (kHxBY + 1) * (kHxBX + 1); t += kHxThreads) {
      const int i = t % (kHxBX + 1), r = t / (kHxBX + 1);
      const int j = r % (kHxBY + 1), k = r / (kHxBY + 1);
      const int ox = lx0 - 1 + i, oy = ly0 - 1 + j, oz = lz0 - 1 + k;
      double v = 0.0;
      if (kPeriodic) {   // elements -1 .. n - 1 are read (-1 wrapped)
        if (ox < g.nx && oy < g.ny && oz < g.nz)
          v = ckf[((int64_t)hex_wrap(oz, g.nz) * g.ny + hex_wrap(oy, g.ny)) * g.nx + hex_wrap(ox, g.nx)];
      } else if (ox >= 0 && ox < g.nx && oy >= 0 && oy < g.ny && oz >= 0 && oz < g.nz) {
        v = ckf[((int64_t)oz * g.ny + oy) * g.nx + ox];
      }
      sc[k][j][i] = v;
    }
  }
  __syncthreads();
  const int tx = threadIdx.x % kHxBX, ty = (threadIdx.x / kHxBX) % kHxBY, tz = threadIdx.x / (kHxBX * kHxBY);
  const int lx = lx0 + tx, ly = ly0 + ty, lz = lz0 + tz;
  if (kPeriodic ? (lx >= g.nx || ly >= g.ny || lz >= g.nz) : (lx > g.nx || ly > g.ny || lz > g.nz)) return;
  double r0, r1, r2;
  hex_node_rows<kPeriodic>(ke, g, lx, ly, lz,
                [&](int ax, int ay, int az) { return kField ? sc[kField ? tz + 1 - az : 0][kField ? ty + 1 - ay : 0][kField ? tx + 1 - ax : 0] : ck; },
                [&](int dx, int dy, int dz) { return &sx[tz + 1 + dz][ty + 1 + dy][3 * (tx + 1 + dx)]; }, r0, r1, r2);
  const int64_t node = kPeriodic ? ((int64_t)lz * g.ny + ly) * g.nx + lx : ((int64_t)lz * (g.ny + 1) + ly) * g.nxf + (lx - g.x_lo);
  y[3 * node + 0] = r0;
  y[3 * node + 1] = r1;
  y[3 * node + 2] = r2;
}

// the diagonal, as EbeMatrix._diag sums it (pcg_solver.py:282-287): d = 0.0; d = d + Ck_e Ke[3la+dir][3la+dir] in ascending la
// (periodic: over all 8 elements, wrapped, in the same order)
template <bool kField, bool kPeriodic = false>
__global__ void __launch_bounds__(256)
k_hexop_diag(const __grid_constant__ HexKeDiag kd, HexGeom g, double ck, const double *__restrict__ ckf, double *__restrict__ d) {
  const int64_t t = blockIdx.x * (int64_t)256 + threadIdx.x;
  if (t >= g.nfree_nodes) return;
  const int nyl = kPeriodic ? g.ny : g.ny + 1;   // node lines per axis
  const int fx = (int)(t % g.nxf);
  const int ly = (int)((t / g.nxf) % nyl);
  const int lz = (int)(t / ((int64_t)g.nxf * nyl));
  const int lx = fx + g.x_lo;
  double r0 = 0.0, r1 = 0.0, r2 = 0.0;
#pragma unroll
  for (int la = 0; la < 8; ++la) {
    int ox = lx - (la & 1), oy = ly - ((la >> 1) & 1), oz = lz - (la >> 2);
    if (kPeriodic) {
      ox = hex_wrap(ox, g.nx); oy = hex_wrap(oy, g.ny); oz = hex_wrap(oz, g.nz);
    } else if (ox < 0 || ox >= g.nx || oy < 0 || oy >= g.ny || oz < 0 || oz >= g.nz) {
      continue;
    }
    const double c = kField ? ckf[((int64_t)oz * g.ny + oy) * g.nx + ox] : ck;
    r0 = __dadd_rn(r0, __dmul_rn(c, kd.k[3 * la + 0]));
    r1 = __dadd_rn(r1, __dmul_rn(c, kd.k[3 * la + 1]));
    r2 = __dadd_rn(r2, __dmul_rn(c, kd.k[3 * la + 2]));
  }
  d[3 * t + 0] = r0;
  d[3 * t + 1] = r1;
  d[3 * t + 2] = r2;
}

// The macroscopic-strain load of a periodic cell, b = -K u_bar per node, u_bar = eps_bar x.  u_bar is taken relative to the
// node computed (Ke annihilates the constant u_bar(node) in exact arithmetic): u_bar(node + d) - u_bar(node) = eps_bar h d
// for d in {-1, 0, 1}^3, the 27-entry table below, so b depends on no absolute coordinate.  The rows are hex_node_rows<true>
// with x_at returning that table: the periodic operator's order exactly (la outer, Ck_e * u then the fma chain from 0.0,
// then the element sums from 0.0 in ascending la), then b = -row (exact).
struct HexUbar { double u[27][3]; };   // entry (dz + 1) 9 + (dy + 1) 3 + (dx + 1): eps_bar h d

template <bool kField>
__global__ void __launch_bounds__(256)
k_hexop_load(const __grid_constant__ HexKe ke, const __grid_constant__ HexUbar ub, HexGeom g, double ck, const double *__restrict__ ckf,
             double *__restrict__ b) {
  const int64_t t = blockIdx.x * (int64_t)256 + threadIdx.x;
  if (t >= g.nfree_nodes) return;
  const int lx = (int)(t % g.nx);
  const int ly = (int)((t / g.nx) % g.ny);
  const int lz = (int)(t / ((int64_t)g.nx * g.ny));
  double r0, r1, r2;
  hex_node_rows<true>(ke, g, lx, ly, lz,
                      [&](int ax, int ay, int az) {
                        return kField ? ckf[((int64_t)hex_wrap(lz - az, g.nz) * g.ny + hex_wrap(ly - ay, g.ny)) * g.nx + hex_wrap(lx - ax, g.nx)] : ck;
                      },
                      [&](int dx, int dy, int dz) { return ub.u[(dz + 1) * 9 + (dy + 1) * 3 + dx + 1]; }, r0, r1, r2);
  b[3 * t + 0] = -r0;
  b[3 * t + 1] = -r1;
  b[3 * t + 2] = -r2;
}

struct HexOp {
  HexOpShape s;
  HexKe ke;
  HexKeDiag kd;
  double ck = 0.0;                // uniform Ck (d_ck NULL)
  const double *d_ck = nullptr;   // per-element Ck (caller-owned), or NULL
  int64_t n = 0;                  // free dofs
  int64_t bytes = 0;              // algorithmic bytes per application: x and y once, the field once
  bool periodic = false;          // a periodic cell (periodic_geom numbering, k_hexop<., true>)
};

inline int hexop_apply(const HexOp &H, const double *x, double *y, cudaStream_t st, int *launches = nullptr, const int *skip = nullptr) {
  const unsigned grid = (unsigned)((int64_t)H.s.nbx * H.s.nby * H.s.nbz);
  if (H.periodic) {
    if (H.d_ck) k_hexop<true, true><<<grid, kHxThreads, 0, st>>>(H.ke, H.s, 0.0, H.d_ck, x, y, skip);
    else k_hexop<false, true><<<grid, kHxThreads, 0, st>>>(H.ke, H.s, H.ck, nullptr, x, y, skip);
  } else if (H.d_ck) {
    k_hexop<true><<<grid, kHxThreads, 0, st>>>(H.ke, H.s, 0.0, H.d_ck, x, y, skip);
  } else {
    k_hexop<false><<<grid, kHxThreads, 0, st>>>(H.ke, H.s, H.ck, nullptr, x, y, skip);
  }
  PCGB_CHECK_LAUNCH();
  if (launches) *launches += 1;
  return PCGB_OK;
}

inline int hexop_diag(const HexOp &H, double *d, cudaStream_t st) {
  const unsigned grid = (unsigned)((H.s.g.nfree_nodes + 255) / 256);
  if (H.periodic) {
    if (H.d_ck) k_hexop_diag<true, true><<<grid, 256, 0, st>>>(H.kd, H.s.g, 0.0, H.d_ck, d);
    else k_hexop_diag<false, true><<<grid, 256, 0, st>>>(H.kd, H.s.g, H.ck, nullptr, d);
  } else if (H.d_ck) {
    k_hexop_diag<true><<<grid, 256, 0, st>>>(H.kd, H.s.g, 0.0, H.d_ck, d);
  } else {
    k_hexop_diag<false><<<grid, 256, 0, st>>>(H.kd, H.s.g, H.ck, nullptr, d);
  }
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

// b = -K u_bar of a periodic cell (k_hexop_load) for the macroscopic strain `strain` (Voigt 11, 22, 33, 23, 13, 12 with
// engineering shears) and element edge h.  The table entry of d is u_i = (E_i0 h d0 + E_i1 h d1) + E_i2 h d2 with the tensor
// E (E_23 = 0.5 gamma_23, ...) and E_ij h one rounded product; d in {-1, 0, 1} makes each term exact.
inline int hexop_load(const HexOp &H, const double strain[6], double h, double *b, cudaStream_t st) {
  const double E[3][3] = {{strain[0], 0.5 * strain[5], 0.5 * strain[4]},
                          {0.5 * strain[5], strain[1], 0.5 * strain[3]},
                          {0.5 * strain[4], 0.5 * strain[3], strain[2]}};
  HexUbar ub;
  for (int dz = -1; dz <= 1; ++dz)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx)
        for (int i = 0; i < 3; ++i)
          ub.u[(dz + 1) * 9 + (dy + 1) * 3 + dx + 1][i] = (dx * (E[i][0] * h) + dy * (E[i][1] * h)) + dz * (E[i][2] * h);
  const unsigned grid = (unsigned)((H.s.g.nfree_nodes + 255) / 256);
  if (H.d_ck) k_hexop_load<true><<<grid, 256, 0, st>>>(H.ke, ub, H.s.g, 0.0, H.d_ck, b);
  else k_hexop_load<false><<<grid, 256, 0, st>>>(H.ke, ub, H.s.g, H.ck, nullptr, b);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

}  // namespace pcgb
