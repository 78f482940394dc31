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
