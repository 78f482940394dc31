// fields.cuh - strains and stresses of a hex box recovered on the device from its displacement: element strain and stress,
// principal values, and their nodal averages (updateElemStrain, pcg_solver.py:601-618; getNodalPS, :730-814;
// getPrincipalStress / getPrincipalStrain, file_operations.py:251-301).
//
// Numbering (hexgen.cuh / hexop.cuh): element e = (oz ny + oy) nx + ox (the flattened order of an E field of shape
// (ne[2], ne[1], ne[0])); local node l at (l&1, l>>1&1, l>>2&1), sign s_a(l) = +1 when bit a of l is set, else -1.  x is
// the free-dof vector of the box (free node (lz, ly, fx), x fastest, lx = fx + x_lo; dof = 3 node + dir); a node on the
// clamped line (global x index 0) has u = 0.0.
//
// Arithmetic contract (every operation an explicit __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn, left to right, so that no
// contraction can change it; element strain and stress are bit-identical to a numpy restatement of the same operations):
//   strain   the Q1 gradient at the centroid (on a brick the element's volume-averaged strain; the centroid B matrix stands
//            for the reference's strain modes Se, 1/h for Ce).  q = 0.25 / h (host double).  For a, i in 0..2:
//              acc = 0.0;  for l = 0..7: acc = acc + u_l,i if s_a(l) > 0 else acc - u_l,i;   g[a][i] = acc q
//            Voigt order (11, 22, 33, 23, 13, 12) of file_operations.py:259-264, tensor (not engineering) shears:
//              e11 = g00, e22 = g11, e33 = g22, e23 = 0.5 (g12 + g21), e13 = 0.5 (g02 + g20), e12 = 0.5 (g01 + g10)
//   stress   sigma = E_e D eps with the lambda, mu of hexmesh.hex_element_stiffness(1, nu) (host doubles lam, m2 = 2 mu):
//              tr = (e11 + e22) + e33;  s_ii = E_e (lam tr + m2 e_ii);  s_ij = E_e (m2 e_ij)
//            E_e is the uniform E or the field entry (not Ck / h).  The damage factor (1 - Omega) of pcg_solver.py:755 is 1:
//            the builder sets Omega = 0 (partition_mesh.py:482).
//   principal values of a symmetric tensor s (stress, or strain for getPrincipalStrain), the invariant form of
//            getPrincipalStress:
//              I1 = (s11 + s22) + s33
//              I2 = s11 s22 + s22 s33 + s33 s11 - s12^2 - s23^2 - s13^2
//              I3 = s11 s22 s33 - s11 s23^2 - s22 s13^2 - s33 s12^2 + 2 s12 s23 s13
//              J2 = I1^2 - 3 I2,  B = 0.5 (2 I1^3 - 9 I1 I2 + 27 I3) / (J2 sqrt(J2)) clamped to [-1, 1],  Phi = acos(B) / 3
//              P_k = I1 / 3 + (2/3) sqrt(J2) cos(Phi + 2 pi k / 3),  k = 0, 1, 2
//            out: P1 = max P_k, P3 = min P_k, P2 = (I1 - P1) - P3 clamped to [P3, P1] (the clamp acts only where two
//            values coincide and rounding would put P2 outside them, so P1 >= P2 >= P3 always holds).  J2 sqrt(J2) is the
//            reference's J2^1.5, both correctly rounded.  Two deviations from the reference: no 1e-24 max|S| term in J2 (a
//            maximum over the whole part, which made each element depend on the partition), and where J2 sqrt(J2) <= 0 (a
//            hydrostatic state up to rounding, the zero tensor included) every P_k is I1 / 3, where the reference gives
//            NaN once rounding makes J2 negative.  acos and cos are CUDA's, so principal values agree with a host
//            restatement to the accuracy of those functions, not bit for bit.
//   nodal    over every node of the box, clamped line included, node = (lz (ny + 1) + ly) (nx + 1) + lx:
//              sum_k = 0.0 + P_k(e) ..., count = 0.0 + 1.0 ... over the elements e = node - (la&1, la>>1&1, la>>2&1) inside
//              the box in ascending la (np.bincount's order on the hex type group, pcg_solver.py:764-771, as in k_hexop)
//            written node-major as (sum_0, sum_1, sum_2, count); across ranks the halo plan adds the neighbours' copies in
//            neighbour order after the node's own value (:804-809); then out_k = sum_k / (count + 1e-15) (:811).
//
// Kernels: k_fields_elem, one CTA per brick of kFdBX x kFdBY x kFdBZ elements, one thread per element; the CTA stages the
// brick's nodes (one more per axis) of x in shared memory with plain coalesced loads, as k_hexop does.  kOut selects the
// outputs at compile time, so a pass without principal values has no trigonometry.  k_fields_nodal sums a scratch copy of
// the element principal values per node; k_fields_divide finishes the average.  Offsets are 64-bit throughout.
//
// Periodic cells (kPeriodic, DESIGN §2.13; the numbering of hexop.cuh's periodic cells: node = (lz ny + ly) nx + lx, node
// coordinates wrapped modulo the cell): x is the periodic fluctuation u~; the staging wraps node nx to 0 (and so on), and
// the macroscopic strain eps_bar (Voigt, tensor shears) is added to the centroid strain, eps_k = g-strain_k + eps_bar_k;
// the stress law and principal values are then the code above, unchanged.  Nodal averages are not defined for them.
//   average  k_fields_average: the same element pass, fused with a deterministic two-stage reduction of the 12 values
//            (eps_0..5, sigma_0..5) and no per-element output.  Stage 1: thread t = tx + 32 ty + 128 tz of brick b holds its
//            element's values (0.0 for a thread outside the cell); for w = 128, 64, ..., 1: v[t] = v[t] + v[t + w] (t < w);
//            partial[b] = v[0].  Stage 2 (k_fields_average_final, one CTA of 256 threads): with c = ceil(nb / 256), thread t
//            sums acc = 0.0 + partial[t c] + partial[t c + 1] + ... (ascending b, b < nb), the same halving tree over the 256
//            sums follows, and mean = sum / (nx ny nz).  On a brick the centroid strain is the element's volume average
//            and E is constant per element, so the plain mean of the element stresses is the exact volume average of the
//            finite-element stress field.  The result is bit-reproducible: no atomics, a fixed order.
#pragma once
#include "common.cuh"
#include "hexgen.cuh"

namespace pcgb {

constexpr int kFdBX = 32, kFdBY = 4, kFdBZ = 2;          // elements per brick
constexpr int kFdThreads = kFdBX * kFdBY * kFdBZ;
constexpr int kFdSX = kFdBX + 1, kFdSY = kFdBY + 1, kFdSZ = kFdBZ + 1;   // staged nodes
constexpr int kFdStrain = 1, kFdStress = 2, kFdPS = 4, kFdPE = 8;         // output bits of k_fields_elem

struct FieldsMacro { double e[6]; };   // the macroscopic strain of a periodic cell (Voigt, tensor shears); unread otherwise

struct FieldsShape {
  HexGeom g;
  int nbx, nby, nbz;   // bricks per axis
  double q;            // 0.25 / h
  double E, lam, m2;   // uniform E (d_E NULL), lambda and 2 mu of hex_element_stiffness(1, nu)
};

// P1 >= P2 >= P3 of the symmetric tensor s (Voigt 11, 22, 33, 23, 13, 12)
__device__ __forceinline__ void principal3(const double (&s)[6], double *p) {
  constexpr double a1 = 1.0 / 3.0;
  constexpr double c2 = 2.0 * a1 * 3.14159265358979323846, c4 = 4.0 * a1 * 3.14159265358979323846;
  const double s11 = s[0], s22 = s[1], s33 = s[2], s23 = s[3], s13 = s[4], s12 = s[5];
  const double s12_2 = __dmul_rn(s12, s12), s23_2 = __dmul_rn(s23, s23), s13_2 = __dmul_rn(s13, s13);
  const double I1 = __dadd_rn(__dadd_rn(s11, s22), s33);
  const double I2 = __dsub_rn(__dsub_rn(__dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(s11, s22), __dmul_rn(s22, s33)), __dmul_rn(s33, s11)),
                                                  s12_2), s23_2), s13_2);
  const double I3 = __dadd_rn(__dsub_rn(__dsub_rn(__dsub_rn(__dmul_rn(__dmul_rn(s11, s22), s33), __dmul_rn(s11, s23_2)),
                                                  __dmul_rn(s22, s13_2)), __dmul_rn(s33, s12_2)),
                              __dmul_rn(__dmul_rn(__dmul_rn(2.0, s12), s23), s13));
  const double I1_2 = __dmul_rn(I1, I1), I1_3 = __dmul_rn(I1_2, I1);
  const double J2 = __dsub_rn(I1_2, __dmul_rn(3.0, I2));
  const double c = __dmul_rn(a1, I1);
  double p0 = c, p1 = c, p2 = c;
  const double rj = sqrt(J2 > 0.0 ? J2 : 0.0);
  const double den = __dmul_rn(J2, rj);
  if (den > 0.0) {
    const double num = __dadd_rn(__dsub_rn(__dmul_rn(2.0, I1_3), __dmul_rn(__dmul_rn(9.0, I1), I2)), __dmul_rn(27.0, I3));
    double br = __ddiv_rn(__dmul_rn(0.5, num), den);
    br = fmin(fmax(br, -1.0), 1.0);
    const double phi = __dmul_rn(a1, acos(br));
    const double f = __dmul_rn(2.0 * a1, rj);
    p0 = __dadd_rn(c, __dmul_rn(f, cos(phi)));
    p1 = __dadd_rn(c, __dmul_rn(f, cos(__dadd_rn(phi, c2))));
    p2 = __dadd_rn(c, __dmul_rn(f, cos(__dadd_rn(phi, c4))));
  }
  const double hi = fmax(fmax(p0, p1), p2), lo = fmin(fmin(p0, p1), p2);
  p[0] = hi;
  p[1] = fmin(fmax(__dsub_rn(__dsub_rn(I1, hi), lo), lo), hi);
  p[2] = lo;
}

// The brick's nodes of x (one more than its elements per axis) into sx: 0.0 on the clamped line and outside the box, or, on
// a periodic cell, node n of an axis wrapped to 0
template <bool kPeriodic>
__device__ __forceinline__ void fields_stage(const HexGeom &g, const double *__restrict__ x, int ox0, int oy0, int oz0,
                                             double (&sx)[kFdSZ][kFdSY][kFdSX * 3]) {
  for (int t = threadIdx.x; t < kFdSZ * kFdSY * kFdSX * 3; t += kFdThreads) {
    const int c = t % (kFdSX * 3), r = t / (kFdSX * 3);
    const int sy = r % kFdSY, sz = r / kFdSY;
    const int lx = ox0 + c / 3, ly = oy0 + sy, lz = oz0 + sz;
    double v = 0.0;
    if (kPeriodic) {
      if (lx <= g.nx && ly <= g.ny && lz <= g.nz)
        v = x[3 * (((int64_t)(lz == g.nz ? 0 : lz) * g.ny + (ly == g.ny ? 0 : ly)) * g.nx + (lx == g.nx ? 0 : lx)) + c % 3];
    } else if (lx >= g.x_lo && lx <= g.nx && ly <= g.ny && lz <= g.nz) {
      v = x[3 * (((int64_t)lz * (g.ny + 1) + ly) * g.nxf + (lx - g.x_lo)) + c % 3];
    }
    sx[sz][sy][c] = v;
  }
}

// the centroid strain of element (tx, ty, tz) of the staged brick (header: strain), plus eps_bar on a periodic cell
template <bool kPeriodic>
__device__ __forceinline__ void fields_strain(const double (&sx)[kFdSZ][kFdSY][kFdSX * 3], int tx, int ty, int tz, double q,
                                              const FieldsMacro &m, double (&eps)[6]) {
  double gr[3][3];   // gr[a][i] = d u_i / d x_a
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      double acc = 0.0;
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        const double u = sx[tz + (l >> 2)][ty + ((l >> 1) & 1)][3 * (tx + (l & 1)) + i];
        acc = ((l >> a) & 1) ? __dadd_rn(acc, u) : __dsub_rn(acc, u);
      }
      gr[a][i] = __dmul_rn(acc, q);
    }
  eps[0] = gr[0][0];
  eps[1] = gr[1][1];
  eps[2] = gr[2][2];
  eps[3] = __dmul_rn(0.5, __dadd_rn(gr[1][2], gr[2][1]));
  eps[4] = __dmul_rn(0.5, __dadd_rn(gr[0][2], gr[2][0]));
  eps[5] = __dmul_rn(0.5, __dadd_rn(gr[0][1], gr[1][0]));
  if (kPeriodic) {
#pragma unroll
    for (int k = 0; k < 6; ++k) eps[k] = __dadd_rn(eps[k], m.e[k]);
  }
}

// sigma = E D eps (header: stress)
__device__ __forceinline__ void fields_stress(const FieldsShape &s, double E, const double (&eps)[6], double (&sg)[6]) {
  const double tr = __dadd_rn(__dadd_rn(eps[0], eps[1]), eps[2]);
  const double ltr = __dmul_rn(s.lam, tr);
#pragma unroll
  for (int k = 0; k < 3; ++k) sg[k] = __dmul_rn(E, __dadd_rn(ltr, __dmul_rn(s.m2, eps[k])));
#pragma unroll
  for (int k = 3; k < 6; ++k) sg[k] = __dmul_rn(E, __dmul_rn(s.m2, eps[k]));
}

template <int kOut, bool kField, bool kPeriodic = false>
__global__ void __launch_bounds__(kFdThreads)
k_fields_elem(FieldsShape s, const double *__restrict__ Ef, const double *__restrict__ x, double *__restrict__ strain,
              double *__restrict__ stress, double *__restrict__ ps, double *__restrict__ pe, const FieldsMacro m) {
  __shared__ double sx[kFdSZ][kFdSY][kFdSX * 3];
  const HexGeom &g = s.g;
  const int b = blockIdx.x;
  const int bx = b % s.nbx, by = (b / s.nbx) % s.nby, bz = b / (s.nbx * s.nby);
  const int ox0 = bx * kFdBX, oy0 = by * kFdBY, oz0 = bz * kFdBZ;   // first element of the brick = its first node
  fields_stage<kPeriodic>(g, x, ox0, oy0, oz0, sx);
  __syncthreads();
  const int tx = threadIdx.x % kFdBX, ty = (threadIdx.x / kFdBX) % kFdBY, tz = threadIdx.x / (kFdBX * kFdBY);
  const int ox = ox0 + tx, oy = oy0 + ty, oz = oz0 + tz;
  if (ox >= g.nx || oy >= g.ny || oz >= g.nz) return;
  const int64_t e = ((int64_t)oz * g.ny + oy) * g.nx + ox;
  double eps[6];
  fields_strain<kPeriodic>(sx, tx, ty, tz, s.q, m, eps);
  if (kOut & kFdStrain) {
#pragma unroll
    for (int k = 0; k < 6; ++k) strain[6 * e + k] = eps[k];
  }
  if (kOut & kFdPE) {
    double p[3];
    principal3(eps, p);
#pragma unroll
    for (int k = 0; k < 3; ++k) pe[3 * e + k] = p[k];
  }
  if (kOut & (kFdStress | kFdPS)) {
    double sg[6];
    fields_stress(s, kField ? Ef[e] : s.E, eps, sg);
    if (kOut & kFdStress) {
#pragma unroll
      for (int k = 0; k < 6; ++k) stress[6 * e + k] = sg[k];
    }
    if (kOut & kFdPS) {
      double p[3];
      principal3(sg, p);
#pragma unroll
      for (int k = 0; k < 3; ++k) ps[3 * e + k] = p[k];
    }
  }
}

constexpr int kFdAvg = 12;   // averaged values: strain 0..5, stress 0..5

// v[k][t] = v[k][t] + v[k][t + w] for w = 128, 64, ..., 1 over the CTA's 256 threads (header: average); the sums end in v[k][0]
__device__ __forceinline__ void fields_tree(double (&v)[kFdAvg][kFdThreads]) {
#pragma unroll
  for (int w = kFdThreads / 2; w >= 1; w >>= 1) {
    __syncthreads();
    if ((int)threadIdx.x < w) {
#pragma unroll
      for (int k = 0; k < kFdAvg; ++k) v[k][threadIdx.x] = __dadd_rn(v[k][threadIdx.x], v[k][threadIdx.x + w]);
    }
  }
  __syncthreads();
}

// stage 1 of the average on a periodic cell: the element pass of k_fields_elem<., ., true>, then brick b's 12 sums into
// partial[12 b + k]
template <bool kField>
__global__ void __launch_bounds__(kFdThreads)
k_fields_average(FieldsShape s, const double *__restrict__ Ef, const double *__restrict__ x, const FieldsMacro m,
                 double *__restrict__ partial) {
  __shared__ double sx[kFdSZ][kFdSY][kFdSX * 3];
  __shared__ double v[kFdAvg][kFdThreads];
  const HexGeom &g = s.g;
  const int b = blockIdx.x;
  const int bx = b % s.nbx, by = (b / s.nbx) % s.nby, bz = b / (s.nbx * s.nby);
  const int ox0 = bx * kFdBX, oy0 = by * kFdBY, oz0 = bz * kFdBZ;
  fields_stage<true>(g, x, ox0, oy0, oz0, sx);
  __syncthreads();
  const int tx = threadIdx.x % kFdBX, ty = (threadIdx.x / kFdBX) % kFdBY, tz = threadIdx.x / (kFdBX * kFdBY);
  const int ox = ox0 + tx, oy = oy0 + ty, oz = oz0 + tz;
  if (ox < g.nx && oy < g.ny && oz < g.nz) {
    double eps[6], sg[6];
    fields_strain<true>(sx, tx, ty, tz, s.q, m, eps);
    fields_stress(s, kField ? Ef[((int64_t)oz * g.ny + oy) * g.nx + ox] : s.E, eps, sg);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      v[k][threadIdx.x] = eps[k];
      v[6 + k][threadIdx.x] = sg[k];
    }
  } else {
#pragma unroll
    for (int k = 0; k < kFdAvg; ++k) v[k][threadIdx.x] = 0.0;
  }
  fields_tree(v);
  if (threadIdx.x < kFdAvg) partial[(int64_t)kFdAvg * b + threadIdx.x] = v[threadIdx.x][0];
}

// stage 2: one CTA; thread t sums partials t c .. t c + c - 1 in ascending order, the tree sums the 256, out = sum / ne
__global__ void __launch_bounds__(kFdThreads)
k_fields_average_final(int64_t nb, double ne, const double *__restrict__ partial, double *__restrict__ out) {
  __shared__ double v[kFdAvg][kFdThreads];
  const int64_t c = (nb + kFdThreads - 1) / kFdThreads;
  const int64_t b0 = c * threadIdx.x, b1 = b0 + c < nb ? b0 + c : nb;
  double acc[kFdAvg];
#pragma unroll
  for (int k = 0; k < kFdAvg; ++k) acc[k] = 0.0;
  for (int64_t b = b0; b < b1; ++b)
#pragma unroll
    for (int k = 0; k < kFdAvg; ++k) acc[k] = __dadd_rn(acc[k], partial[kFdAvg * b + k]);
#pragma unroll
  for (int k = 0; k < kFdAvg; ++k) v[k][threadIdx.x] = acc[k];
  fields_tree(v);
  if (threadIdx.x < kFdAvg) out[threadIdx.x] = __ddiv_rn(v[threadIdx.x][0], ne);
}

// one thread per node of the box: (sum_0, sum_1, sum_2, count) of the element values pv (ne x 3) around it, ascending la
__global__ void __launch_bounds__(256)
k_fields_nodal(HexGeom g, const double *__restrict__ pv, double *__restrict__ work) {
  const int64_t t = blockIdx.x * (int64_t)256 + threadIdx.x;
  const int64_t nnodes = (int64_t)(g.nx + 1) * (g.ny + 1) * (g.nz + 1);
  if (t >= nnodes) return;
  const int lx = (int)(t % (g.nx + 1));
  const int ly = (int)((t / (g.nx + 1)) % (g.ny + 1));
  const int lz = (int)(t / ((int64_t)(g.nx + 1) * (g.ny + 1)));
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, cnt = 0.0;
#pragma unroll
  for (int la = 0; la < 8; ++la) {
    const int ox = lx - (la & 1), oy = ly - ((la >> 1) & 1), oz = lz - (la >> 2);
    if (ox < 0 || ox >= g.nx || oy < 0 || oy >= g.ny || oz < 0 || oz >= g.nz) continue;
    const double *p = pv + 3 * (((int64_t)oz * g.ny + oy) * g.nx + ox);
    s0 = __dadd_rn(s0, p[0]);
    s1 = __dadd_rn(s1, p[1]);
    s2 = __dadd_rn(s2, p[2]);
    cnt = __dadd_rn(cnt, 1.0);
  }
  work[4 * t + 0] = s0;
  work[4 * t + 1] = s1;
  work[4 * t + 2] = s2;
  work[4 * t + 3] = cnt;
}

// out = sum / (count + 1e-15) per node (pcg_solver.py:811)
__global__ void __launch_bounds__(256)
k_fields_divide(int64_t nnodes, const double *__restrict__ work, double *__restrict__ out) {
  const int64_t t = blockIdx.x * (int64_t)256 + threadIdx.x;
  if (t >= nnodes) return;
  const double d = __dadd_rn(work[4 * t + 3], 1e-15);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * t + k] = __ddiv_rn(work[4 * t + k], d);
}

inline FieldsShape fields_shape(const HexGeom &g) {
  FieldsShape s{};
  s.g = g;
  s.nbx = (g.nx + kFdBX - 1) / kFdBX;
  s.nby = (g.ny + kFdBY - 1) / kFdBY;
  s.nbz = (g.nz + kFdBZ - 1) / kFdBZ;
  return s;
}

template <int kOut, bool kPeriodic>
inline void fields_elem_launch(const FieldsShape &s, const FieldsMacro &m, const double *Ef, const double *x, double *strain,
                               double *stress, double *ps, double *pe, cudaStream_t st) {
  const unsigned grid = (unsigned)((int64_t)s.nbx * s.nby * s.nbz);
  if (Ef) k_fields_elem<kOut, true, kPeriodic><<<grid, kFdThreads, 0, st>>>(s, Ef, x, strain, stress, ps, pe, m);
  else k_fields_elem<kOut, false, kPeriodic><<<grid, kFdThreads, 0, st>>>(s, nullptr, x, strain, stress, ps, pe, m);
}

// the element pass for the outputs that are not NULL (at least one); m (the macroscopic strain) only with periodic
inline int fields_elem(const FieldsShape &s, const double *Ef, const double *x, double *strain, double *stress, double *ps, double *pe,
                       cudaStream_t st, bool periodic = false, const FieldsMacro &m = FieldsMacro{}) {
  using L = void (*)(const FieldsShape &, const FieldsMacro &, const double *, const double *, double *, double *, double *, double *,
                     cudaStream_t);
#define PCGB_FD_ROW(P)                                                                                                              \
  {nullptr, fields_elem_launch<1, P>, fields_elem_launch<2, P>, fields_elem_launch<3, P>, fields_elem_launch<4, P>,             \
   fields_elem_launch<5, P>, fields_elem_launch<6, P>, fields_elem_launch<7, P>, fields_elem_launch<8, P>,                      \
   fields_elem_launch<9, P>, fields_elem_launch<10, P>, fields_elem_launch<11, P>, fields_elem_launch<12, P>,                   \
   fields_elem_launch<13, P>, fields_elem_launch<14, P>, fields_elem_launch<15, P>}
  static const L table[2][16] = {PCGB_FD_ROW(false), PCGB_FD_ROW(true)};
#undef PCGB_FD_ROW
  const int out = (strain ? kFdStrain : 0) | (stress ? kFdStress : 0) | (ps ? kFdPS : 0) | (pe ? kFdPE : 0);
  if (out == 0) return PCGB_OK;
  table[periodic ? 1 : 0][out](s, m, Ef, x, strain, stress, ps, pe, st);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

// The volume averages of strain and stress over a periodic cell (header: average): out[0..5] strain, out[6..11] stress,
// device; partial holds 12 doubles per brick
inline int fields_average(const FieldsShape &s, const FieldsMacro &m, const double *Ef, const double *x, double *partial, double *out,
                          cudaStream_t st) {
  const int64_t nb = (int64_t)s.nbx * s.nby * s.nbz;
  if (Ef) k_fields_average<true><<<(unsigned)nb, kFdThreads, 0, st>>>(s, Ef, x, m, partial);
  else k_fields_average<false><<<(unsigned)nb, kFdThreads, 0, st>>>(s, nullptr, x, m, partial);
  PCGB_CHECK_LAUNCH();
  k_fields_average_final<<<1, kFdThreads, 0, st>>>(nb, (double)((int64_t)s.g.nx * s.g.ny * s.g.nz), partial, out);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

}  // namespace pcgb
