// gmg.cuh - kernels of the geometric multigrid preconditioner for hex-box operators (pcgb_mg_*).
//
// Levels are nested trilinear hex boxes: level l+1 has half the elements of level l per axis.  Every level uses the
// free-node numbering of hexgen.cuh (x fastest, nodes with global x index 0 clamped and dropped, dof = 3*node + dir).
// P is trilinear interpolation of the coarse free nodes onto the fine ones, direction by direction, with weights
// 1, 1/2, 1/4, 1/8; clamped nodes carry 0 on every level.  Both transfers are gathers with one thread per output
// node and a fixed summation order, so they are bit-reproducible (no atomics).
//
// Every kernel takes `skip` (the PCG control state, NULL outside the loop) and returns at once when *skip != 0, so
// the V-cycle can sit inside batched and graph-captured iterations like every other kernel of the loop.
#pragma once
#include "common.cuh"
#include "hexgen.cuh"
#include "pcg_kernels.cuh"

namespace pcgb {

// free node (fx, ly, lz) of a level -> (lx, ly, lz)
__device__ __forceinline__ void mg_node(const HexGeom &g, int64_t t, int &lx, int &ly, int &lz) {
  lx = (int)(t % g.nxf) + g.x_lo;
  ly = (int)((t / g.nxf) % (g.ny + 1));
  lz = (int)(t / ((int64_t)g.nxf * (g.ny + 1)));
}
__device__ __forceinline__ int64_t mg_index(const HexGeom &g, int lx, int ly, int lz) {
  return ((int64_t)lz * (g.ny + 1) + ly) * g.nxf + (lx - g.x_lo);
}

// A rank's box of a level inside the level's global box: local node (lx, ly, lz) is global node (e0 + l).  One rank:
// e0 = 0 and glob = the box itself, so the global free index of a dof is its local index.
struct MgPlace {
  HexGeom glob;
  int e0x, e0y, e0z;
};
__device__ __forceinline__ int64_t mg_global_node(const MgPlace &p, int lx, int ly, int lz) {
  return mg_index(p.glob, lx + p.e0x, ly + p.e0y, lz + p.e0z);
}

// r_c = P^T r_f: one thread per coarse free node; the <= 27 fine nodes 2*c + (dx, dy, dz), d in {-1, 0, 1}, are summed
// in (dz, dy, dx) ascending order from 0.0, each with weight prod_a (d_a == 0 ? 1 : 1/2).  Local indices serve a rank's
// box as well, because its fine e0 is twice its coarse e0.  own_f (NULL = every node): 0/1 ownership of the fine dofs;
// only owned fine nodes are summed (selected, not multiplied), so after the coarse level's exchange-add every fine node
// of the global box has been counted exactly once.
__global__ void __launch_bounds__(256)
k_mg_restrict(HexGeom gf, HexGeom gc, const double *__restrict__ rf, const double *__restrict__ own_f, double *__restrict__ rc,
              const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= gc.nfree_nodes) return;
  int cx, cy, cz;
  mg_node(gc, t, cx, cy, cz);
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
        const int64_t fi = mg_index(gf, fx, fy, fz);
        if (own_f != nullptr && own_f[3 * fi] == 0.0) continue;
        const double w = (dx ? 0.5 : 1.0) * (dy ? 0.5 : 1.0) * (dz ? 0.5 : 1.0);
        const double *src = rf + 3 * fi;
        s0 += w * src[0]; s1 += w * src[1]; s2 += w * src[2];
      }
    }
  }
  rc[3 * t] = s0; rc[3 * t + 1] = s1; rc[3 * t + 2] = s2;
}

// x_f += P e_c: one thread per fine free node; the <= 8 coarse nodes around it (per axis: c = f/2 for even f, else
// (f-1)/2 then (f+1)/2, each 1/2) are summed in (z, y, x) ascending order from 0.0, then added to x_f.
__global__ void __launch_bounds__(256)
k_mg_prolong_add(HexGeom gf, HexGeom gc, const double *__restrict__ ec, double *__restrict__ xf, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= gf.nfree_nodes) return;
  int fx, fy, fz;
  mg_node(gf, t, fx, fy, fz);
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  const int nz = (fz & 1) ? 2 : 1, ny = (fy & 1) ? 2 : 1, nx = (fx & 1) ? 2 : 1;
  for (int kz = 0; kz < nz; ++kz) {
    const int cz = (fz >> 1) + kz;
    for (int ky = 0; ky < ny; ++ky) {
      const int cy = (fy >> 1) + ky;
      for (int kx = 0; kx < nx; ++kx) {
        const int cx = (fx >> 1) + kx;
        if (cx < gc.x_lo) continue;   // clamped coarse node
        const double w = (nx == 2 ? 0.5 : 1.0) * (ny == 2 ? 0.5 : 1.0) * (nz == 2 ? 0.5 : 1.0);
        const double *src = ec + 3 * mg_index(gc, cx, cy, cz);
        s0 += w * src[0]; s1 += w * src[1]; s2 += w * src[2];
      }
    }
  }
  xf[3 * t] += s0; xf[3 * t + 1] += s1; xf[3 * t + 2] += s2;
}

// First Chebyshev step.  q == NULL (pre-smoother, x = 0 on entry): r = b.  Otherwise r = b - q with q = A x.
// Then d = inv_theta * (dinv * r) and x = d (q == NULL) or x += d.
__global__ void __launch_bounds__(256)
k_mg_cheb_first(int64_t n, const double *__restrict__ b, const double *__restrict__ q, const double *__restrict__ dinv,
                double inv_theta, double *__restrict__ r, double *__restrict__ d, double *__restrict__ x, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const double ri = q ? b[i] - q[i] : b[i];
    const double di = inv_theta * (dinv[i] * ri);
    r[i] = ri;
    d[i] = di;
    x[i] = q ? x[i] + di : di;
  }
}

// Later Chebyshev steps with q = A d: r -= q, then (unless last) d = c1 * d + c2 * (dinv * r) and x += d.
// `last` only updates the residual (the pre-smoother's r = b - A x handed to the restriction).
__global__ void __launch_bounds__(256)
k_mg_cheb_step(int64_t n, const double *__restrict__ q, const double *__restrict__ dinv, double c1, double c2, int last,
               double *__restrict__ r, double *__restrict__ d, double *__restrict__ x, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const double ri = r[i] - q[i];
    r[i] = ri;
    if (last) continue;
    const double di = c1 * d[i] + c2 * (dinv[i] * ri);
    d[i] = di;
    x[i] += di;
  }
}

// Fixed start vector of the Lanczos estimate: v_i = 1/2 + ((37 g + 11) mod 101) / 101 with g the dof's free index in the
// level's global box (g = i on one rank), so every rank's copy of a shared dof starts alike.
__global__ void k_mg_lanczos_start(HexGeom g, MgPlace p, double *__restrict__ v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < g.nfree_nodes; t += stride) {
    int lx, ly, lz;
    mg_node(g, t, lx, ly, lz);
    const int64_t gn = mg_global_node(p, lx, ly, lz);
    for (int d = 0; d < 3; ++d) v[3 * t + d] = 0.5 + (double)((37 * (3 * gn + d) + 11) % 101) / 101.0;
  }
}

// Lanczos on D^-1 A in the D inner product (v.D v = sum v^2 / dinv): w = (scale ? dinv * y : y) - alpha v - beta vp into
// w (which may be vp), and partials of w.D w over the owned dofs (own NULL = all).  v and vp may be NULL (start vector).
__global__ void __launch_bounds__(256)
k_mg_lanczos_w(int64_t n, const double *__restrict__ y, const double *__restrict__ v, const double *vp, const double *__restrict__ dinv,
               const double *__restrict__ own, double alpha, double beta, int scale, double *w, double *__restrict__ partials) {
  __shared__ double red[32];
  double s = 0.0;
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = blockIdx.x * (int64_t)256 + threadIdx.x; i < n; i += stride) {
    double wi = scale ? dinv[i] * y[i] : y[i];
    if (v) wi = wi - alpha * v[i] - beta * vp[i];
    w[i] = wi;
    if (own == nullptr || own[i] != 0.0) s = fma(wi, wi / dinv[i], s);
  }
  double vv[1] = {s};
  block_sum<1, 256>(vv, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = vv[0];
}

// next Lanczos vector: vp <- v, v <- w / beta (w held in vp)
__global__ void k_mg_lanczos_next(int64_t n, double inv_beta, double *__restrict__ v, double *__restrict__ vp) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const double wi = vp[i];
    vp[i] = v[i];
    v[i] = wi * inv_beta;
  }
}

// Gather of the last ranked level into its global box: one thread per global free node; the entry is this rank's copy
// when the rank owns it (selected on ownership, so a non-owned copy, NaN or not, never enters) and 0.0 otherwise.  The
// exchange-add over the all-to-all gather plan then completes the vector: one non-zero term per entry, exact in any order.
__global__ void __launch_bounds__(256)
k_mg_gather(HexGeom g, MgPlace p, const double *__restrict__ v, const double *__restrict__ own, double *__restrict__ out,
            const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= p.glob.nfree_nodes) return;
  int gx, gy, gz;
  mg_node(p.glob, t, gx, gy, gz);
  const int lx = gx - p.e0x, ly = gy - p.e0y, lz = gz - p.e0z;
  const bool in = lx >= g.x_lo && lx <= g.nx && ly >= 0 && ly <= g.ny && lz >= 0 && lz <= g.nz;
  const int64_t li = in ? mg_index(g, lx, ly, lz) : 0;
  for (int d = 0; d < 3; ++d) out[3 * t + d] = in && own[3 * li + d] != 0.0 ? v[3 * li + d] : 0.0;
}

// Scatter back: every local dof (owned or not) takes the global vector's entry, so the ranked vector is consistent.
__global__ void __launch_bounds__(256)
k_mg_scatter(HexGeom g, MgPlace p, const double *__restrict__ in, double *__restrict__ v, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= g.nfree_nodes) return;
  int lx, ly, lz;
  mg_node(g, t, lx, ly, lz);
  const int64_t gi = mg_global_node(p, lx, ly, lz);
  for (int d = 0; d < 3; ++d) v[3 * t + d] = in[3 * gi + d];
}

// Gather of a rank's element matrices at the last ranked level into the global box's (pcgb_mg_create_ranks_field): one
// thread per entry, element (X, Y, Z) of the rank's box g to global element e0 + (X, Y, Z) of p.glob, every other entry of
// kg left as the caller zeroed it.  The exchange-add over the all-to-all element plan then completes kg: every global
// element lies in exactly one rank's box, so each entry has one non-zero term and every rank holds the same matrices.
__global__ void __launch_bounds__(256)
k_mg_gather_elements(HexGeom g, MgPlace p, const double *__restrict__ kel, double *__restrict__ kg) {
  const int64_t n = 576 * (int64_t)g.nx * g.ny * g.nz;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t e = i / 576;
    const int X = (int)(e % g.nx), Y = (int)((e / g.nx) % g.ny), Z = (int)(e / ((int64_t)g.nx * g.ny));
    const int64_t E = ((int64_t)(Z + p.e0z) * p.glob.ny + (Y + p.e0y)) * p.glob.nx + (X + p.e0x);
    kg[576 * E + i % 576] = kel[i];
  }
}

// rz and the count of non-finite z entries of z = M r: (sum z*(r*w), #(!isfinite z)) into partials[0] / partials[kMaxVecGrid]
// (slots 3 and 4 of the iteration's partials).  A V-cycle spreads a NaN of the fine Minv over all of z, so NaN counts like
// inf here: the loop stops with flag 2 as MATLAB pcg does for a non-finite preconditioned residual.
__global__ void __launch_bounds__(256)
k_mg_rz(const int *__restrict__ skip, int64_t n, const double *__restrict__ r, const double *__restrict__ z,
        const double *__restrict__ w, double *__restrict__ partials) {
  if (skip != nullptr && *skip != 0) return;
  __shared__ double red[64];
  double s = 0.0, ninf = 0.0;
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = blockIdx.x * (int64_t)256 + threadIdx.x; i < n; i += stride) {
    const double ri = r[i], zi = z[i];
    if (!isfinite(zi)) ninf += 1.0;
    s = fma(zi, w ? ri * w[i] : ri, s);
  }
  double v[2] = {s, ninf};
  block_sum<2, 256>(v, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = v[0];
    partials[kMaxVecGrid + blockIdx.x] = v[1];
  }
}

// Weight of coarse corner k in the trilinear interpolation onto local node l of child c of a coarse element: child-c
// node l sits at p = c + (l&1, l>>1&1, l>>2&1) in {0,1,2}^3 (units of the fine spacing), and the weight is
// prod_a phi_{k_a}(p_a) with phi_0(p) = (2 - p) / 2, phi_1(p) = p / 2: one of 0, 1/8, 1/4, 1/2, 1, exact in binary.
__device__ __forceinline__ double mg_child_weight(int c, int l, int k) {
  double w = 1.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int p = ((c >> a) & 1) + ((l >> a) & 1);
    w *= ((k >> a) & 1) ? 0.5 * p : 0.5 * (2 - p);
  }
  return w;
}

// Galerkin element matrices of a coarse level: K_E = sum_c Q_c^T K_c Q_c over the 8 children c = cx + 2 cy + 4 cz of
// coarse element E = (X, Y, Z) (fine element (2X + cx, 2Y + cy, 2Z + cz)), Q_c the 24x24 interpolation of mg_child_weight
// (block-diagonal over the 3 directions).  K_c = ck[child] * Ke (Ke in c_hex_ke) when kf is NULL (the first coarse
// level, built from the fine field), else kf[576 child ..] (the level below's Galerkin matrices).  One CTA per coarse
// element, one thread per entry (i, j): T = K_c Q_c in shared memory (l ascending), then (Q_c^T T)[i][j] (l ascending),
// added to the entry in ascending c.  No atomics: a repeated set-up is bit-identical.  The result is written mirrored
// from its upper triangle, so every element matrix, and every CSR assembled from them, is exactly symmetric.
// Slabs (gmg_rap.cuh): CTA b builds coarse element E = e_off + b into kc[576 b ..], and child k is read at index k - child_off
// of ck / kf; both offsets are 0 for a whole level.
constexpr int kMgGalerkinThreads = 576;
__global__ void __launch_bounds__(kMgGalerkinThreads)
k_mg_galerkin(int cnx, int cny, int fnx, int fny, const double *__restrict__ ck, const double *__restrict__ kf, double *__restrict__ kc,
              int64_t e_off = 0, int64_t child_off = 0) {
  __shared__ double K[576], T[576];
  const int t = threadIdx.x, i = t / 24, j = t % 24;
  const int64_t E = blockIdx.x + e_off;
  const int X = (int)(E % cnx), Y = (int)((E / cnx) % cny), Z = (int)(E / ((int64_t)cnx * cny));
  double acc = 0.0;
  for (int c = 0; c < 8; ++c) {
    const int64_t child = ((int64_t)(2 * Z + (c >> 2)) * fny + (2 * Y + ((c >> 1) & 1))) * fnx + (2 * X + (c & 1)) - child_off;
    K[t] = kf ? kf[576 * child + t] : ck[child] * c_hex_ke[t];
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int l = 0; l < 8; ++l) s += mg_child_weight(c, l, j / 3) * K[i * 24 + 3 * l + j % 3];
    T[t] = s;
    __syncthreads();
    s = 0.0;
#pragma unroll
    for (int l = 0; l < 8; ++l) s += mg_child_weight(c, l, i / 3) * T[(3 * l + i % 3) * 24 + j];
    acc += s;
  }
  K[t] = acc;   // every thread is past its last read of K (the second barrier of c = 7)
  __syncthreads();
  kc[576 * (int64_t)blockIdx.x + t] = i <= j ? K[t] : K[j * 24 + i];
}

// ---- boxes of any size (pcgb_mg_create_any).  Every axis of a level is coarsened on its own: halved (ne >= 3; coarse node
// j sits at fine node s(j) = min(2j, ne), so an odd axis ends in a coarse element one fine element wide at its high end) or
// kept (ne <= 2; s(j) = j).  `keep` holds one bit per axis (x = 1, y = 2, z = 4).  P is the tensor product of the three 1-D
// interpolations between consecutive s(j), with weights 0, 1/2 and 1 (exact in binary); clamped nodes carry 0 as above.
// A level with every axis halved and every ne even uses k_mg_restrict / k_mg_prolong_add / k_mg_galerkin themselves.

// coarse position of coarse node j on an axis of nf fine elements
__device__ __forceinline__ int mg_any_pos(int j, int nf, bool keep) { return keep ? j : min(2 * j, nf); }

// r_c = P^T r_f for any axis modes: one thread per coarse free node; per axis the fine nodes s(j) + d, d in {-1, 0, 1}, that
// lie strictly inside the coarse elements on either side (weight 1/2; only an element two fine elements wide has one) and
// s(j) itself (weight 1), summed in (dz, dy, dx) ascending order from 0.0.  A kept axis contributes d = 0 only.
__global__ void __launch_bounds__(256)
k_mg_restrict_any(HexGeom gf, HexGeom gc, int keep, const double *__restrict__ rf, double *__restrict__ rc, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= gc.nfree_nodes) return;
  int c[3];
  mg_node(gc, t, c[0], c[1], c[2]);
  const int nf[3] = {gf.nx, gf.ny, gf.nz}, ncm[3] = {gc.nx, gc.ny, gc.nz};
  int s[3], lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const bool k = (keep >> a) & 1;
    s[a] = mg_any_pos(c[a], nf[a], k);
    lo[a] = c[a] > 0 && s[a] - mg_any_pos(c[a] - 1, nf[a], k) == 2 ? -1 : 0;
    hi[a] = c[a] < ncm[a] && mg_any_pos(c[a] + 1, nf[a], k) - s[a] == 2 ? 1 : 0;
  }
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int dz = lo[2]; dz <= hi[2]; ++dz) {
    for (int dy = lo[1]; dy <= hi[1]; ++dy) {
      for (int dx = lo[0]; dx <= hi[0]; ++dx) {
        const int fx = s[0] + dx;
        if (fx < gf.x_lo) continue;
        const double w = (dx ? 0.5 : 1.0) * (dy ? 0.5 : 1.0) * (dz ? 0.5 : 1.0);
        const double *src = rf + 3 * mg_index(gf, fx, s[1] + dy, s[2] + dz);
        s0 += w * src[0]; s1 += w * src[1]; s2 += w * src[2];
      }
    }
  }
  rc[3 * t] = s0; rc[3 * t + 1] = s1; rc[3 * t + 2] = s2;
}

// x_f += P e_c for any axis modes: one thread per fine free node; per axis the coarse node at the fine node (weight 1) or
// the two around it (an interior node of a two-wide coarse element, 1/2 each), summed in (z, y, x) ascending order from
// 0.0, then added to x_f.
__global__ void __launch_bounds__(256)
k_mg_prolong_add_any(HexGeom gf, HexGeom gc, int keep, const double *__restrict__ ec, double *__restrict__ xf, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= gf.nfree_nodes) return;
  int f[3];
  mg_node(gf, t, f[0], f[1], f[2]);
  const int nf[3] = {gf.nx, gf.ny, gf.nz};
  int c0[3], m[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if ((keep >> a) & 1) { c0[a] = f[a]; m[a] = 1; }
    else if ((f[a] & 1) == 0) { c0[a] = f[a] >> 1; m[a] = 1; }
    else if (f[a] == nf[a]) { c0[a] = (f[a] + 1) >> 1; m[a] = 1; }   // the high end of an odd axis: a coarse node
    else { c0[a] = f[a] >> 1; m[a] = 2; }
  }
  const double w = (m[0] == 2 ? 0.5 : 1.0) * (m[1] == 2 ? 0.5 : 1.0) * (m[2] == 2 ? 0.5 : 1.0);
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int kz = 0; kz < m[2]; ++kz) {
    for (int ky = 0; ky < m[1]; ++ky) {
      for (int kx = 0; kx < m[0]; ++kx) {
        const int cx = c0[0] + kx;
        if (cx < gc.x_lo) continue;   // clamped coarse node
        const double *src = ec + 3 * mg_index(gc, cx, c0[1] + ky, c0[2] + kz);
        s0 += w * src[0]; s1 += w * src[1]; s2 += w * src[2];
      }
    }
  }
  xf[3 * t] += s0; xf[3 * t + 1] += s1; xf[3 * t + 2] += s2;
}

// mg_child_weight for coarse elements of width w_a in {1, 2} fine elements per axis (bit a of `thin`: w_a = 1, so c_a = 0):
// phi_0(p) = (w - p) / w, phi_1(p) = p / w.  A width-2 axis performs mg_child_weight's arithmetic.
__device__ __forceinline__ double mg_child_weight_any(int c, int l, int k, int thin) {
  double w = 1.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int p = ((c >> a) & 1) + ((l >> a) & 1);
    if ((thin >> a) & 1) w *= ((k >> a) & 1) ? (double)p : (double)(1 - p);
    else w *= ((k >> a) & 1) ? 0.5 * p : 0.5 * (2 - p);
  }
  return w;
}

// k_mg_galerkin for any axis modes: coarse element (X, Y, Z) covers fine elements s(X) .. s(X+1) - 1 per axis (one or two),
// and K_E = sum_c Q_c^T K_c Q_c over the children that exist, c = cx + 2 cy + 4 cz ascending, with mg_child_weight_any.
// When every axis is two wide this is k_mg_galerkin's arithmetic in k_mg_galerkin's order.  Every thread of a CTA skips the
// same children, so the barriers stay uniform.
__global__ void __launch_bounds__(kMgGalerkinThreads)
k_mg_galerkin_any(int cnx, int cny, int fnx, int fny, int fnz, int keep, const double *__restrict__ ck, const double *__restrict__ kf,
                  double *__restrict__ kc) {
  __shared__ double K[576], T[576];
  const int t = threadIdx.x, i = t / 24, j = t % 24;
  const int64_t E = blockIdx.x;
  const int C[3] = {(int)(E % cnx), (int)((E / cnx) % cny), (int)(E / ((int64_t)cnx * cny))};
  const int nf[3] = {fnx, fny, fnz};
  int f0[3], m[3], thin = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const bool k = (keep >> a) & 1;
    f0[a] = mg_any_pos(C[a], nf[a], k);
    m[a] = mg_any_pos(C[a] + 1, nf[a], k) - f0[a];
    if (m[a] == 1) thin |= 1 << a;
  }
  double acc = 0.0;
  for (int c = 0; c < 8; ++c) {
    if ((c & 1) >= m[0] || ((c >> 1) & 1) >= m[1] || (c >> 2) >= m[2]) continue;
    const int64_t child = ((int64_t)(f0[2] + (c >> 2)) * fny + (f0[1] + ((c >> 1) & 1))) * fnx + (f0[0] + (c & 1));
    K[t] = kf ? kf[576 * child + t] : ck[child] * c_hex_ke[t];
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int l = 0; l < 8; ++l) s += mg_child_weight_any(c, l, j / 3, thin) * K[i * 24 + 3 * l + j % 3];
    T[t] = s;
    __syncthreads();
    s = 0.0;
#pragma unroll
    for (int l = 0; l < 8; ++l) s += mg_child_weight_any(c, l, i / 3, thin) * T[(3 * l + i % 3) * 24 + j];
    acc += s;
  }
  K[t] = acc;   // every thread is past its last read of K (the second barrier of the last child)
  __syncthreads();
  kc[576 * E + t] = i <= j ? K[t] : K[j * 24 + i];
}

// dense[i][col] = val of the coarsest level's CSR (dense zero-filled before)
__global__ void k_mg_densify(int64_t n, const int64_t *__restrict__ rowptr, const int *__restrict__ col, const double *__restrict__ val,
                             double *__restrict__ dense) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int64_t k = rowptr[i]; k < rowptr[i + 1]; ++k) dense[i * n + col[k]] = val[k];
}

constexpr int kMgCholThreads = 1024;

// In-place dense Cholesky A = L L^T in one CTA, right-looking, columns in ascending order: L is left in the lower
// triangle and mirrored into the upper one (a[k][i] = L[i][k]) so both substitutions read rows.  *bad = 1 when a
// pivot is not positive (or not finite).
__global__ void __launch_bounds__(kMgCholThreads) k_mg_chol_factor(int n, double *__restrict__ a, int *__restrict__ bad) {
  __shared__ double piv;
  for (int k = 0; k < n; ++k) {
    if (threadIdx.x == 0) {
      const double akk = a[(int64_t)k * n + k];
      if (!(akk > 0.0) || !isfinite(akk)) *bad = 1;
      piv = sqrt(akk);
      a[(int64_t)k * n + k] = piv;
    }
    __syncthreads();
    const double dk = piv;
    for (int i = k + 1 + threadIdx.x; i < n; i += blockDim.x) {
      const double l = a[(int64_t)i * n + k] / dk;
      a[(int64_t)i * n + k] = l;
      a[(int64_t)k * n + i] = l;
    }
    __syncthreads();
    // trailing update of the lower triangle: a[i][j] -= L[i][k] * L[j][k] for k < j <= i, one warp per row
    const int lane = threadIdx.x & 31;
    for (int i = k + 1 + (threadIdx.x >> 5); i < n; i += blockDim.x >> 5) {
      const double lik = a[(int64_t)k * n + i];
      for (int j = k + 1 + lane; j <= i; j += 32) a[(int64_t)i * n + j] -= lik * a[(int64_t)k * n + j];
    }
    __syncthreads();
  }
}

// z = A^-1 r with the factor of k_mg_chol_factor, in one CTA: forward substitution L y = r column by column (column j of L
// = row j of the mirrored upper triangle), then L^T z = y from the last column down.  Every entry is updated in a fixed
// column order.  n <= kMgMaxCoarse.
constexpr int kMgMaxCoarse = 1536;
__global__ void __launch_bounds__(kMgCholThreads)
k_mg_chol_solve(int n, const double *__restrict__ a, const double *__restrict__ r, double *__restrict__ z, const int *__restrict__ skip) {
  if (skip != nullptr && *skip != 0) return;
  __shared__ double y[kMgMaxCoarse];
  for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = r[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    const double yj = y[j] / a[(int64_t)j * n + j];
    __syncthreads();
    if (threadIdx.x == 0) y[j] = yj;
    for (int i = j + 1 + threadIdx.x; i < n; i += blockDim.x) y[i] -= a[(int64_t)j * n + i] * yj;
    __syncthreads();
  }
  for (int j = n - 1; j >= 0; --j) {
    const double zj = y[j] / a[(int64_t)j * n + j];
    __syncthreads();
    if (threadIdx.x == 0) y[j] = zj;
    for (int i = threadIdx.x; i < j; i += blockDim.x) y[i] -= a[(int64_t)j * n + i] * zj;
    __syncthreads();
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) z[i] = y[i];
}

}  // namespace pcgb
