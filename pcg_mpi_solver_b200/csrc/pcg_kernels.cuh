// pcg_kernels.cuh - fused vector kernels and the device-resident control state of the PCG loop.
//
// Reference semantics: PCG(RefMeshPart), pcg_solver.py:356-598 (a transliteration of MATLAB pcg).
// One reference iteration (pcg_solver.py:438-562) maps onto
//     k_pupdate      z = Minv.*r ; p = z (+ beta p)                       (:446-479)
//     k_spmv_merge   q = A p  with fused  p.q  partials                    (:482-487)
//     k_reduce<1>    pq -> alpha  (+ breakdown checks)                     (:488-498)
//     k_update       r -= alpha q ; partial sums of p.p, x.x, r.r, z'.r' ; x += alpha p   (:501-516)
//     k_reduce<5>    norms, stagnation, convergence trigger, min-residual bookkeeping,
//                    and the head of the next iteration (rho, beta)       (:504-562, :446-478)
// All scalars live in `PcgCtrl` in device memory; every kernel returns immediately once
// ctrl->state != ST_RUN, so the host may enqueue batches of iterations without synchronising and
// still stop at exactly the iteration the reference would stop at.
#pragma once
#include "common.cuh"

namespace pcgb {

enum PcgState : int { ST_RUN = 0, ST_TRIGGER = 1, ST_BREAK = 2, ST_EXHAUSTED = 3 };

struct PcgCtrl {
  double rho, rho_prev, alpha, beta, pq;
  double normr, normp, normx, normr_act, normrmin;
  double tolb, n2b, eps;
  int state, flag, iter, stag, moresteps, imin;
  int xcur, xmin;  // which of the two x buffers holds X / XMin (zero-copy min-residual tracking, :555-558)
  int maxiter, maxstag, fixed_iters;
  int alias;       // 1 while XMin is still the SAME array as X: the reference binds MP_XMin = MP_X (pcg_solver.py:379-380)
                   // and updates MP_X in place (:516), so XMin follows X until the first np.array(MP_X) copy (:557)
};

constexpr int kVecBlock = 256;
constexpr int kMaxVecGrid = 2048;  // partial-sum slots per reduced quantity

inline int vec_grid(int64_t n) {
  int64_t g = (n + kVecBlock * 4 - 1) / (kVecBlock * 4);
  int64_t cap = (int64_t)num_sms() * 8;
  if (cap > kMaxVecGrid) cap = kMaxVecGrid;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

// ---- generic weighted dot: partials[b] = sum a*b*w over the block's grid-stride share
__global__ void __launch_bounds__(kVecBlock)
k_dot_w(int64_t n, const double *__restrict__ a, const double *__restrict__ b, const double *__restrict__ w,
        double *__restrict__ partials) {
  __shared__ double red[32];
  double s = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kVecBlock;
  for (int64_t i = blockIdx.x * (int64_t)kVecBlock + threadIdx.x; i < n; i += stride) {
    double bw = w ? b[i] * w[i] : b[i];
    s = fma(a[i], bw, s);
  }
  double v[1] = {s};
  block_sum<1, kVecBlock>(v, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

// rz partials and inf count for z = Minv.*r :  (sum z*(r*w), #inf(z))   (pcg_solver.py:447-448,462)
__global__ void __launch_bounds__(kVecBlock)
k_rz(int64_t n, const double *__restrict__ r, const double *__restrict__ minv, const double *__restrict__ w,
     double *__restrict__ partials /* [2][kMaxVecGrid] */) {
  __shared__ double red[64];
  double s = 0.0, ninf = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kVecBlock;
  for (int64_t i = blockIdx.x * (int64_t)kVecBlock + threadIdx.x; i < n; i += stride) {
    const double ri = r[i];
    const double zi = minv ? minv[i] * ri : ri;
    if (isinf(zi)) ninf += 1.0;
    s = fma(zi, w ? ri * w[i] : ri, s);
  }
  double v[2] = {s, ninf};
  block_sum<2, kVecBlock>(v, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = v[0];
    partials[kMaxVecGrid + blockIdx.x] = v[1];
  }
}

// r = b - q   (true residual, pcg_solver.py:414,531,572) with partials of sum r*r*w
__global__ void __launch_bounds__(kVecBlock)
k_residual(int64_t n, const double *__restrict__ b, const double *__restrict__ q, const double *__restrict__ w,
           double *__restrict__ r, double *__restrict__ partials) {
  __shared__ double red[32];
  double s = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kVecBlock;
  for (int64_t i = blockIdx.x * (int64_t)kVecBlock + threadIdx.x; i < n; i += stride) {
    const double ri = b[i] - q[i];
    r[i] = ri;
    s = fma(ri, w ? ri * w[i] : ri, s);
  }
  double v[1] = {s};
  block_sum<1, kVecBlock>(v, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

// ---- p = z + beta p  (z = Minv.*r);  p = z on the first iteration   (pcg_solver.py:446-479)
__global__ void __launch_bounds__(kVecBlock)
k_pupdate(const PcgCtrl *__restrict__ ctrl, int64_t n, const double *__restrict__ r, const double *__restrict__ minv,
          double *__restrict__ p) {
  if (ctrl->state != ST_RUN) return;
  const bool first = ctrl->iter == 0;
  const double beta = ctrl->beta;
  const int64_t stride = (int64_t)gridDim.x * kVecBlock;
  for (int64_t i = blockIdx.x * (int64_t)kVecBlock + threadIdx.x; i < n; i += stride) {
    const double zi = minv ? minv[i] * r[i] : r[i];
    p[i] = first ? zi : fma(beta, p[i], zi);
  }
}

// ---- fused update  (pcg_solver.py:501-516 plus z/rho of the next iteration, :447,462)
//   r -= alpha q ; sums of p*p*w, x*x*w (x BEFORE its update, :505 vs :516), r*r*w, z*(r*w), #inf(z);
//   x_new = x + alpha p written to the buffer that does not hold XMin.
__global__ void __launch_bounds__(kVecBlock)
k_update(const PcgCtrl *__restrict__ ctrl, int64_t n, double *__restrict__ r, const double *__restrict__ q,
         const double *__restrict__ p, const double *__restrict__ minv, const double *__restrict__ w,
         double *xb0, double *xb1, double *__restrict__ partials /* [5][kMaxVecGrid] */) {
  if (ctrl->state != ST_RUN) return;
  __shared__ double red[5 * 32];
  const double alpha = ctrl->alpha;
  const int cur = ctrl->xcur;
  const int dst = (!ctrl->alias && cur == ctrl->xmin) ? (cur ^ 1) : cur;   // aliased: in place, XMin follows X
  const double *xs = cur ? xb1 : xb0;
  double *xd = dst ? xb1 : xb0;
  double spp = 0.0, sxx = 0.0, srr = 0.0, srz = 0.0, ninf = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kVecBlock;
  for (int64_t i = blockIdx.x * (int64_t)kVecBlock + threadIdx.x; i < n; i += stride) {
    const double pi = p[i], xi = xs[i];
    const double ri = fma(-alpha, q[i], r[i]);
    r[i] = ri;
    const double wi = w ? w[i] : 1.0;
    spp = fma(pi, pi * wi, spp);
    sxx = fma(xi, xi * wi, sxx);
    const double rw = ri * wi;
    srr = fma(ri, rw, srr);
    const double zi = minv ? minv[i] * ri : ri;
    if (isinf(zi)) ninf += 1.0;
    srz = fma(zi, rw, srz);
    xd[i] = fma(alpha, pi, xi);
  }
  double v[5] = {spp, sxx, srr, srz, ninf};
  block_sum<5, kVecBlock>(v, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 5; ++k) partials[k * kMaxVecGrid + blockIdx.x] = v[k];
  }
}

// ------------------------------------------------------------------ scalar control logic
// alpha = rho / pq with the breakdown checks of pcg_solver.py:492-498
__device__ __forceinline__ void ctrl_alpha(PcgCtrl *c, double pq) {
  c->pq = pq;
  if (pq <= 0.0 || isinf(pq)) { c->flag = 4; c->state = ST_BREAK; return; }
  const double alpha = c->rho / pq;
  if (isinf(alpha)) { c->flag = 4; c->state = ST_BREAK; return; }
  c->alpha = alpha;
}

// head of an iteration: rho / beta checks (pcg_solver.py:446-478); `rz`, `ninf` belong to the current r
__device__ __forceinline__ void ctrl_head(PcgCtrl *c, double rz, double ninf) {
  if (ninf > 0.0) { c->flag = 2; c->state = ST_BREAK; return; }
  c->rho_prev = c->rho;
  c->rho = rz;
  if (rz == 0.0 || isinf(rz)) { c->flag = 4; c->state = ST_BREAK; return; }
  if (c->iter > 0) {
    const double beta = rz / c->rho_prev;
    if (beta == 0.0 || isinf(beta)) { c->flag = 4; c->state = ST_BREAK; return; }
    c->beta = beta;
  }
}

// advance the loop variable (for i in range(MaxIter), :438) and run the head of the next iteration
__device__ __forceinline__ void ctrl_next(PcgCtrl *c, double rz, double ninf) {
  if (c->iter + 1 >= c->maxiter) { c->state = ST_EXHAUSTED; return; }
  c->iter += 1;
  ctrl_head(c, rz, ninf);
}

// tail of an iteration after the norms are known (pcg_solver.py:504-562)
__device__ __forceinline__ void ctrl_norms(PcgCtrl *c, double pp, double xx, double rr, double rz, double ninf, double *resvec) {
  // the x buffer switch performed by k_update
  if (!c->alias && c->xcur == c->xmin) c->xcur ^= 1;
  const double normp = sqrt(pp), normx = sqrt(xx), normr = sqrt(rr);
  c->normp = normp; c->normx = normx; c->normr = normr;
  if (normp * fabs(c->alpha) < c->eps * normx) c->stag += 1;  // :512-513
  else c->stag = 0;
  c->normr_act = normr;                                          // :518
  if (resvec) resvec[c->iter + 1] = normr;
  if (!c->fixed_iters && (normr <= c->tolb || c->stag >= c->maxstag || c->moresteps > 0)) {
    c->state = ST_TRIGGER;  // host recomputes the true residual (:527-552)
    return;
  }
  if (normr < c->normrmin) {  // :555-558, zero-copy: XMin is whichever buffer holds X now
    c->normrmin = normr;
    c->xmin = c->xcur;
    c->imin = c->iter;
    c->alias = 0;             // XMin = np.array(MP_X): from here on XMin is a frozen copy
  }
  if (!c->fixed_iters && c->stag >= c->maxstag) { c->flag = 3; c->state = ST_BREAK; return; }  // :560-562
  ctrl_next(c, rz, ninf);
}

// Sum NV rows of per-block partials (fixed order -> deterministic) into out[0..NV).
// MODE 0: only reduce.  MODE 1: reduce + alpha logic.  MODE 2: reduce + norms logic.
template <int NV, int MODE>
__global__ void __launch_bounds__(256)
k_reduce(PcgCtrl *ctrl, const double *__restrict__ partials, int count, int row_stride, double *__restrict__ out, double *resvec) {
  if (MODE != 0 && ctrl->state != ST_RUN) return;
  __shared__ double red[NV * 32];
  double v[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double s = 0.0;
    for (int i = threadIdx.x; i < count; i += 256) s += partials[(size_t)k * row_stride + i];
    v[k] = s;
  }
  block_sum<NV, 256>(v, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) out[k] = v[k];
    if (MODE == 1) ctrl_alpha(ctrl, v[0]);
    if (MODE == 2) ctrl_norms(ctrl, v[0], v[1 % NV], v[2 % NV], v[3 % NV], v[4 % NV], resvec);
  }
}

// first level of a two-level sum over many partials (one CTA per 4096 entries, fixed order)
__global__ void __launch_bounds__(256) k_stage_reduce(const double *__restrict__ in, int count, double *__restrict__ out) {
  __shared__ double red[32];
  const int lo = blockIdx.x * 4096, hi = min(count, lo + 4096);
  double s = 0.0;
  for (int i = lo + threadIdx.x; i < hi; i += 256) s += in[i];
  double v[1] = {s};
  block_sum<1, 256>(v, red);
  if (threadIdx.x == 0) out[blockIdx.x] = v[0];
}

// control logic on already all-reduced values (multi-GPU path: partial reduce -> ncclAllReduce -> this)
__global__ void k_ctrl_alpha(PcgCtrl *ctrl, const double *__restrict__ red) {
  if (ctrl->state != ST_RUN) return;
  ctrl_alpha(ctrl, red[0]);
}
__global__ void k_ctrl_norms(PcgCtrl *ctrl, const double *__restrict__ red, double *resvec) {
  if (ctrl->state != ST_RUN) return;
  ctrl_norms(ctrl, red[0], red[1], red[2], red[3], red[4], resvec);
}
// resume after a host-side verification step / initial set-up: run the head of iteration ctrl->iter
__global__ void k_ctrl_head(PcgCtrl *ctrl, const double *__restrict__ red /* rz, ninf */, int advance) {
  if (ctrl->state != ST_RUN) return;
  if (advance) ctrl_next(ctrl, red[0], red[1]);
  else ctrl_head(ctrl, red[0], red[1]);
}

// ---- opt-in trace of the control steps (pcgb_solver_set_trace): one fixed-size record per step, appended in order.
// Records hold the reduced values the step consumed and the whole PcgCtrl after it, so a host restatement of the
// control logic can replay the loop bit for bit (tests/pcg_shadow.py).  Nothing here runs unless tracing is on.
enum PcgTraceKind : int { TR_HEAD = 0, TR_ITER = 1, TR_VERIFY = 2, TR_RESUME = 3, TR_FINAL = 4 };
// in[] / local[] slots: 0 pq | 1 pp | 2 xx | 3 rr | 4 rz | 5 ninf | 6 b.b | 7 r0.r0   (unused slots are 0)
//   HEAD (iteration 0) and RESUME (head after a failed verification): rz, ninf (+ b.b, r0.r0 for HEAD)
//   ITER: pq, pp, xx, rr, rz, ninf      VERIFY: rr = sum (b - A x_cur)^2 w      FINAL: rr of b - A x_min (0 when flag 0)
struct PcgTraceRec {
  int kind, rank, pad0, pad1;
  double in[8];     // what the step consumed (all-reduced over the ranks)
  double local[8];  // this rank's value of the same slots before the all-reduce (= in on one rank)
  PcgCtrl ctrl;     // control state after the step
};
struct PcgTraceHdr {
  unsigned long long total;  // records produced by the solve (those past the capacity are dropped)
  int frozen;                // the last record left the loop stopped: later no-op iterations write nothing
  int pad[13];
};
static_assert(sizeof(PcgTraceHdr) == 64, "trace header layout");

__device__ __forceinline__ PcgTraceRec *trace_slot(PcgTraceHdr *hdr, PcgTraceRec *rec, long long cap, int state) {
  const unsigned long long k = hdr->total;
  hdr->total = k + 1;
  hdr->frozen = state != ST_RUN;
  return k < (unsigned long long)cap ? rec + k : nullptr;
}

// record of a device-side step (HEAD / ITER / RESUME) from the control block and the reduced scalars in red[0..8)
__global__ void k_trace_step(PcgTraceHdr *hdr, PcgTraceRec *rec, long long cap, int rank, int kind, const PcgCtrl *ctrl,
                             const double *red, const double *local, double bb, double r0r0) {
  if (kind == TR_ITER && hdr->frozen) return;   // the iteration did not run
  PcgTraceRec *t = trace_slot(hdr, rec, cap, ctrl->state);
  if (!t) return;
  double in[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int mask;
  if (kind == TR_ITER) { for (int k = 0; k < 6; ++k) in[k] = red[k]; mask = 0x3f; }
  else { in[4] = red[6]; in[5] = red[7]; in[6] = bb; in[7] = r0r0; mask = 0x30; }
  t->kind = kind; t->rank = rank; t->pad0 = 0; t->pad1 = 0;
  for (int k = 0; k < 8; ++k) {
    t->in[k] = in[k];
    t->local[k] = local ? (((mask >> k) & 1) ? local[k] : 0.0) : in[k];
  }
  t->ctrl = *ctrl;
}

// record of a host-side step (VERIFY / FINAL): the host's control block by value; snap_tail (may be NULL) receives
// xcur, xmin, alias of that control block
__global__ void k_trace_host(PcgTraceHdr *hdr, PcgTraceRec *rec, long long cap, int rank, int kind, PcgCtrl c, double rr,
                             const double *local, double *snap_tail) {
  if (snap_tail) { snap_tail[0] = c.xcur; snap_tail[1] = c.xmin; snap_tail[2] = c.alias; }
  PcgTraceRec *t = trace_slot(hdr, rec, cap, c.state);
  if (!t) return;
  t->kind = kind; t->rank = rank; t->pad0 = 0; t->pad1 = 0;
  for (int k = 0; k < 8; ++k) { t->in[k] = k == 3 ? rr : 0.0; t->local[k] = k == 3 ? (local ? local[3] : rr) : 0.0; }
  t->ctrl = c;
}

// out[0] = sqrt(in[0])  (ResVec[0] = ||r0|| without a host round trip)
__global__ void k_sqrt_store(const double *__restrict__ in, double *__restrict__ out) { out[0] = sqrt(in[0]); }

// ---- simple elementwise kernels exposed through the C ABI
__global__ void k_axpby(int64_t n, double a, const double *__restrict__ x, double b, double *__restrict__ y) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
    y[i] = b == 0.0 ? a * x[i] : fma(a, x[i], b * y[i]);
}
__global__ void k_mul(int64_t n, const double *__restrict__ x, const double *__restrict__ y, double *__restrict__ z) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) z[i] = x[i] * y[i];
}
__global__ void k_reciprocal(int64_t n, const double *__restrict__ d, double *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) out[i] = 1.0 / d[i];
}

// ---- halo pack / unpack-add  (pcg_solver.py:304-312, 332-334)
__global__ void k_halo_pack(int64_t m, const int *__restrict__ idx, const double *__restrict__ y, double *__restrict__ send) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < m) send[i] = y[idx[i]];
}
// one thread per distinct interface dof: y[dof] += sum of its received copies, in neighbour order
__global__ void k_halo_unpack_add(int64_t ndof, const int *__restrict__ dof, const int *__restrict__ ptr,
                                  const int *__restrict__ pos, const double *__restrict__ recv, double *__restrict__ y) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= ndof) return;
  double s = y[dof[t]];
  for (int k = ptr[t]; k < ptr[t + 1]; ++k) s += recv[pos[k]];
  y[dof[t]] = s;
}

}  // namespace pcgb
