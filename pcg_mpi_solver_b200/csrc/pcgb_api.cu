// pcgb_api.cu - C ABI of libpcgb200.so (see include/pcgb200.h) and the host side of the PCG loop.
// sm_90a only.  No CPU fallback: every compute entry point requires a CUDA device.
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "spmv.cuh"
#include "pcg_kernels.cuh"
#include "comm.cuh"
#include "hexgen.cuh"
#include "ebe.cuh"
#include "ebe_color.cuh"
#include "assemble.cuh"
#include "ebe_ordered.cuh"
#include "gmg.cuh"
#include "hexop.cuh"
#include "gmg_rap.cuh"
#include "fields.cuh"

using namespace pcgb;

struct pcgb_csr_s {
  CsrPlan P;
};

struct pcgb_ebe_s {
  EbePlan P;
  int device = 0;
};

struct pcgb_asm_s {
  AsmPlan P;
};

struct pcgb_ebe2_s {
  EbeColorPlan C;
  int device = 0;
};

struct pcgb_ebe_ordered_s {
  EboPlan O;
  int device = 0;
};

struct pcgb_hexop_s {
  HexOp H;
};

struct pcgb_fields_s {
  FieldsShape s;
  const double *d_E = nullptr;   // per-element E (caller-owned), or NULL
  int64_t ne = 0, nnodes = 0, n = 0;   // elements, nodes (clamped line included), free dofs
};

// What may differ between two solves on one handle and changes the captured iterations (the operator, the x buffers and
// PCGB_FORK are fixed when the solver is created).
struct GraphKey {
  const void *minv = nullptr, *w = nullptr, *resvec = nullptr;
  int iters = 0;
  bool peer = false;              // peer transport
  bool split = false;             // the product runs interface-first (split_product)
  const void *trace = nullptr;    // trace buffer and capacity (kernel arguments of the captured trace records; NULL = tracing off)
  long long trace_cap = 0;
  const void *mg = nullptr;       // multigrid preconditioner of the captured V-cycles (NULL = diagonal Minv)
  bool operator==(const GraphKey &o) const {
    return minv == o.minv && w == o.w && resvec == o.resvec && iters == o.iters && peer == o.peer && split == o.split &&
           trace == o.trace && trace_cap == o.trace_cap && mg == o.mg;
  }
};

// The solver's operator K: exactly one handle is set.  rows() and apply() are the only code that asks which; the iteration's
// product reads A for the CSR dot partials and the interface-first split.
struct FineOp {
  pcgb_csr_t A = nullptr;
  pcgb_ebe_t E = nullptr;           // opt-in matrix-free operator
  pcgb_ebe_ordered_t O = nullptr;   // opt-in matrix-free operator with a fixed summation order
  pcgb_hexop_t H = nullptr;         // opt-in index-free operator of a hex box (the ordered operator's bits)
  int64_t rows() const { return A ? A->P.nrows : E ? E->P.n : O ? O->O.P.n : H->H.n; }
  // y = K x, without the interface sum
  int apply(const double *x, double *y, cudaStream_t st, int *nl, const int *skip) const {
    if (E) return ebe_apply(E->P, x, y, st, nl, skip);
    if (O) return ebo_apply(O->O, x, y, st, nl, skip);
    if (H) return hexop_apply(H->H, x, y, st, nl, skip);
    return spmv_launch(A->P, x, y, false, st, nl, skip);
  }
};

struct pcgb_solver_s {
  FineOp op;
  pcgb_halo_t halo = nullptr;
  pcgb_comm_t comm = nullptr;
  int64_t n = 0;
  double *r = nullptr, *p = nullptr, *q = nullptr, *xalt = nullptr, *xown = nullptr;
  double *partials = nullptr;   // [5][kMaxVecGrid]
  double *stage = nullptr;      // first-level sums of the SpMV dot partials
  int stage_cap = 0;
  double *red = nullptr;        // [8] device scalars: [0]=pq, [1..5]=pp,xx,rr,rz,ninf ; [6..7] scratch
  PcgCtrl *d_ctrl = nullptr;
  PcgCtrl *h_ctrl = nullptr;    // pinned
  double *h_red = nullptr;      // pinned [8]
  cudaStream_t own = nullptr;   // the solve runs here: the caller's stream may be the legacy stream, which cannot be captured
  cudaStream_t side = nullptr;  // fork of the iteration: the halo unpack-add runs beside the p.q all-reduce
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr, ev_l0 = nullptr, ev_l1 = nullptr, ev_s0 = nullptr, ev_s1 = nullptr;
  std::vector<cudaEvent_t> ev_k;  // SpMV brackets (time_kernels)
  cudaGraphExec_t gexec = nullptr;
  GraphKey gkey;
  int launches = 0;             // launches issued outside graphs (running counter per solve)
  int launches_per_iter = 0;
  bool fork_halo = true;        // PCGB_FORK=0 keeps the unpack on the main stream
  // opt-in trace of the control steps (pcgb_solver_set_trace); all NULL = off, and the loop is launched exactly as without it
  PcgTraceHdr *trace = nullptr;
  long long trace_cap = 0;
  double *snapshot = nullptr;   // [5][n] + 3: r, p, q, x buffer 0, x buffer 1, then xcur, xmin, alias at the loop exit
  double *tr_local = nullptr;   // [8] device: this rank's sums before the all-reduce (multi-rank traces)
  // multigrid handles built on this solver: destroying the solver first detaches them, so a later pcgb_mg_destroy (a
  // garbage collector may finalise the two in either order) does not read the freed solver
  std::vector<pcgb_mg_t> mgs;
};
void mg_detach(pcgb_mg_t mg);

static int require_device() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return fail(PCGB_ERR_NODEVICE, "no CUDA device visible: libpcgb200 has no CPU fallback");
  }
  return PCGB_OK;
}

namespace {
template <typename T>
cudaError_t upload(T **d, const std::vector<T> &v) {
  cudaError_t e = cudaMalloc(d, std::max<size_t>(v.size(), 1) * sizeof(T));
  if (e != cudaSuccess || v.empty()) return e;
  return cudaMemcpy(*d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
}
// blob of a halo plan: IPC handle | m | per source rank r: {offset of r's segment in my receive buffer (doubles, -1 = not a
// neighbour), my neighbour slot of r, number of shared entries}
struct HaloBlobHead { unsigned char handle[PCGB_IPC_BLOB_BYTES]; int64_t m; };
struct HaloBlobRank { int64_t off, slot, cnt; };
}  // namespace

// Constant-memory slots of the 24-dof pattern matrices (c_ebe_ke24) are a per-device resource shared by every EBE
// operator of the process: slots are de-duplicated by content and reference-counted, so a second operator can never
// overwrite the matrices of a live one; when all slots are taken the group runs on the warp kernel (Ke from global memory).
namespace {
struct EbeSlot { int refs = 0; double ke[576]; };
struct EbeSlotTable { EbeSlot slot[kEbeMaxSlots]; };
std::mutex g_ebe_slot_mutex;
EbeSlotTable *ebe_slot_table(int device) {
  static std::vector<EbeSlotTable *> tabs;
  if (device < 0) return nullptr;
  if ((int)tabs.size() <= device) tabs.resize((size_t)device + 1, nullptr);
  if (!tabs[(size_t)device]) tabs[(size_t)device] = new EbeSlotTable();
  return tabs[(size_t)device];
}
// returns the slot holding `ke` (acquiring a reference) or -1 when the table is full
int ebe_slot_acquire(const double *ke) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  std::lock_guard<std::mutex> lock(g_ebe_slot_mutex);
  EbeSlotTable *t = ebe_slot_table(dev);
  int free_slot = -1;
  for (int k = 0; k < kEbeMaxSlots; ++k) {
    if (t->slot[k].refs > 0 && memcmp(t->slot[k].ke, ke, sizeof(t->slot[k].ke)) == 0) { t->slot[k].refs += 1; return k; }
    if (t->slot[k].refs == 0 && free_slot < 0) free_slot = k;
  }
  if (free_slot < 0) return -1;
  if (cudaMemcpyToSymbol(c_ebe_ke24, ke, 576 * sizeof(double), (size_t)free_slot * 576 * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  memcpy(t->slot[free_slot].ke, ke, sizeof(t->slot[free_slot].ke));
  t->slot[free_slot].refs = 1;
  return free_slot;
}
void ebe_slot_release(int device, int slot) {
  if (slot < 0 || slot >= kEbeMaxSlots) return;
  std::lock_guard<std::mutex> lock(g_ebe_slot_mutex);
  EbeSlotTable *t = ebe_slot_table(device);
  if (t && t->slot[slot].refs > 0) t->slot[slot].refs -= 1;
}
}  // namespace

extern "C" {

int pcgb_version(void) { return PCGB_VERSION; }
void pcgb_abi_sizes(int32_t out[4]) {
  out[0] = (int32_t)sizeof(pcgb_options); out[1] = (int32_t)sizeof(pcgb_result);
  out[2] = (int32_t)sizeof(pcgb_hex_box); out[3] = (int32_t)sizeof(pcgb_ebe_group);
}
const char *pcgb_last_error(void) { return last_error().c_str(); }
int pcgb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// ------------------------------------------------------------------------------------ CSR
int pcgb_csr_create(int64_t nrows, int64_t ncols, int64_t nnz, const void *d_rowptr, int rowptr_is_64, const int32_t *d_col,
                    const double *d_val, void *stream, pcgb_csr_t *out) {
  if (!out || nrows < 0 || ncols < 0 || nnz < 0 || !d_rowptr) return fail(PCGB_ERR_ARG, "pcgb_csr_create: bad argument");
  if (nrows > INT32_MAX - 8 || ncols > INT32_MAX - 8) return fail(PCGB_ERR_ARG, "pcgb_csr_create: more than 2^31 rows/cols");
  if (!rowptr_is_64 && nnz > INT32_MAX) return fail(PCGB_ERR_ARG, "pcgb_csr_create: nnz >= 2^31 needs 64-bit row offsets");
  PCGB_TRY(require_device());
  pcgb_csr_t A = new pcgb_csr_s();
  A->P.nrows = nrows; A->P.ncols = ncols; A->P.nnz = nnz;
  A->P.rowptr = d_rowptr; A->P.rp64 = rowptr_is_64 != 0; A->P.col = d_col; A->P.val = d_val;
  int rc = A->P.rp64 ? build_plan_t<int64_t>(A->P, (cudaStream_t)stream) : build_plan_t<int32_t>(A->P, (cudaStream_t)stream);
  if (rc != PCGB_OK) { free_plan(A->P); delete A; return rc; }
  *out = A;
  return PCGB_OK;
}

int pcgb_csr_destroy(pcgb_csr_t A) {
  if (!A) return PCGB_OK;
  free_plan(A->P);
  delete A;
  return PCGB_OK;
}

int pcgb_spmv(pcgb_csr_t A, const double *d_x, double *d_y, void *stream) {
  if (!A || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_spmv: null argument");
  return spmv_launch(A->P, d_x, d_y, false, (cudaStream_t)stream);
}

static int csr_diag_compute(const CsrPlan &P, double *d_diag, cudaStream_t st) {
  if (P.nrows == 0) return PCGB_OK;
  if (!P.col) return fail(PCGB_ERR_ARG, "pcgb_csr_diag: the column array was released and no diagonal is cached");
  const unsigned grid = (unsigned)((P.nrows * 8 + 255) / 256);
  if (P.rp64) k_csr_diag<int64_t><<<grid, 256, 0, st>>>((const int64_t *)P.rowptr, P.col, P.val, P.nrows, d_diag);
  else k_csr_diag<int32_t><<<grid, 256, 0, st>>>((const int32_t *)P.rowptr, P.col, P.val, P.nrows, d_diag);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_csr_diag(pcgb_csr_t A, double *d_diag, void *stream) {
  if (!A || !d_diag) return fail(PCGB_ERR_ARG, "pcgb_csr_diag: null argument");
  const CsrPlan &P = A->P;
  if (P.diag_cache) {
    PCGB_CUDA(cudaMemcpyAsync(d_diag, P.diag_cache, (size_t)P.nrows * sizeof(double), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return PCGB_OK;
  }
  return csr_diag_compute(P, d_diag, (cudaStream_t)stream);
}

/* The selected SpMV kernel may not read d_col at all (the persistent staged-x kernel works on its own 16-bit index
 * stream).  pcgb_csr_release_col caches the diagonal (the one other consumer) and drops the library's reference, after
 * which the caller may free d_col (2 GB at 128^3, 16 GB at 256^3).  Returns PCGB_ERR_ARG if the plan still needs it. */
int pcgb_csr_release_col(pcgb_csr_t A, void *stream) {
  if (!A) return fail(PCGB_ERR_ARG, "pcgb_csr_release_col: null argument");
  CsrPlan &P = A->P;
  if (!P.col) return PCGB_OK;
  if (!P.persist) return fail(PCGB_ERR_ARG, "pcgb_csr_release_col: the selected SpMV kernel reads the column array");
  if (!P.diag_cache && P.nrows > 0) {
    PCGB_CUDA(cudaMalloc(&P.diag_cache, (size_t)P.nrows * sizeof(double)));
    int rc = csr_diag_compute(P, P.diag_cache, (cudaStream_t)stream);
    if (rc == PCGB_OK && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) rc = fail(PCGB_ERR_CUDA, "pcgb_csr_release_col: sync failed");
    if (rc != PCGB_OK) { cudaFree(P.diag_cache); P.diag_cache = nullptr; return rc; }
  }
  P.col = nullptr;
  return PCGB_OK;
}

int64_t pcgb_spmv_bytes(pcgb_csr_t A) {
  if (!A) return 0;
  const CsrPlan &P = A->P;
  return 12 * P.nnz + (P.rp64 ? 8 : 4) * (P.nrows + 1) + 8 * P.ncols + 8 * P.nrows;
}

/* bytes the selected kernel actually streams from HBM per SpMV: values 8 B per non-zero + the index stream
 * (4 B columns for the L1-gather kernel, 2 B staged positions, 2/3 B with the column-triple index, or 2/9 B per 3x3
 * block) + row offsets, x, y and the tile / window tables.  With a value dictionary the values are the dictionary, which
 * every resident CTA loads once, and the index stream is the run-compressed block words (4 B each) + 8 B per tile. */
int64_t pcgb_spmv_stream_bytes(pcgb_csr_t A) {
  if (!A) return 0;
  const CsrPlan &P = A->P;
  const int64_t val_bytes = P.vd ? 72 * (int64_t)P.vd * P.grid_persist : 8 * P.nnz;
  const int64_t idx_bytes = P.vd ? 4 * P.nvwords + 8 * (int64_t)P.ntiles
                                 : P.bsr ? (2 * P.nnz) / 9 : (P.persist && P.t3) ? (2 * P.nnz) / 3 : (P.staged ? 2 * P.nnz : 4 * P.nnz);
  return val_bytes + idx_bytes + (P.rp64 ? 8 : 4) * (P.nrows + 1) + 8 * P.ncols + 8 * P.nrows +
         (P.staged ? 8 * P.nwin + 8 * (int64_t)P.ntiles : 0) + (P.persist ? 32 : 12) * (int64_t)P.ntiles;
}

int pcgb_csr_value_dict(pcgb_csr_t A) { return A ? A->P.vd : 0; }

/* share of the nodes whose blocks the dictionary kernel reads through a run head (0 without a dictionary) */
double pcgb_csr_run_share(pcgb_csr_t A) {
  if (!A || A->P.vd == 0 || A->P.nrows < 3) return 0.0;
  return (double)A->P.run_nodes / (double)(A->P.nrows / 3);
}

int pcgb_csr_vd_plan(pcgb_csr_t A, int64_t out[8]) {
  if (!A || !out) return fail(PCGB_ERR_ARG, "pcgb_csr_vd_plan: null argument");
  const CsrPlan &P = A->P;
  for (int i = 0; i < 8; ++i) out[i] = 0;
  if (P.vd == 0) return PCGB_OK;
  out[0] = P.bsr_stages; out[1] = P.bsr_group; out[2] = P.bsr_prod; out[3] = P.bsr_cw;
  out[4] = P.cap_words; out[5] = P.nvwords; out[6] = P.cap_nodes; out[7] = P.ctas_per_sm;
  return PCGB_OK;
}

int pcgb_csr_plan_info(pcgb_csr_t A, int64_t info[16]) {
  if (!A || !info) return fail(PCGB_ERR_ARG, "pcgb_csr_plan_info: null argument");
  const CsrPlan &P = A->P;
  info[0] = P.ntiles; info[1] = P.tile_items; info[2] = P.lanes; info[3] = P.snap ? 1 : 0;
  info[4] = P.nfix; info[5] = P.staged ? P.smem_staged : P.smem_bytes; info[6] = P.max_row; info[7] = P.use_tma ? 1 : 0;
  info[8] = P.persist ? 2 : (P.staged ? 1 : 0); info[9] = P.nwin; info[10] = P.cap_x; info[11] = P.max_nw;
  if (P.persist) info[5] = P.smem_persist;
  info[12] = P.bsr ? 2 : (P.t3 ? 1 : 0); info[13] = P.desc_split ? P.nb_tiles : -1; info[14] = P.persist ? P.grid_persist : 0; info[15] = P.col ? 0 : 1;
  return PCGB_OK;
}

/* Interface-first split of the SpMV (multi-GPU overlap, SURVEY 8(e) "order boundary rows first, launch exchange, compute
 * interior rows"): d_rows = the distinct local rows that take part in the interface exchange.  The solver registers
 * them itself from its halo plan; the two entry points below exist so that the split can be tested on one GPU. */
int pcgb_csr_set_boundary_rows(pcgb_csr_t A, const int32_t *d_rows, int64_t count, void *stream) {
  if (!A || count < 0 || (count > 0 && !d_rows)) return fail(PCGB_ERR_ARG, "pcgb_csr_set_boundary_rows: bad argument");
  return spmv_set_boundary_rows(A->P, d_rows, count, (cudaStream_t)stream);
}
/* y = A x as two launches (interface tiles, then the rest); out_dot (device, may be NULL) receives x.y */
int pcgb_spmv_split(pcgb_csr_t A, const double *d_x, double *d_y, double *d_out_dot, void *stream) {
  if (!A || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_spmv_split: null argument");
  const CsrPlan &P = A->P;
  if (!spmv_split_available(P)) return fail(PCGB_ERR_ARG, "pcgb_spmv_split: no split plan (persistent kernel + registered boundary rows needed)");
  cudaStream_t st = (cudaStream_t)stream;
  PCGB_TRY(spmv_launch_part(P, 0, d_x, d_y, d_out_dot != nullptr, st));
  PCGB_TRY(spmv_launch_part(P, 1, d_x, d_y, d_out_dot != nullptr, st));
  if (d_out_dot) {
    k_reduce<1, 0><<<1, 256, 0, st>>>(nullptr, P.dot_partials_split, spmv_split_dot_count(P), 0, d_out_dot, nullptr);
    PCGB_CHECK_LAUNCH();
  }
  return PCGB_OK;
}

// ------------------------------------------------------------------------------------ vector kernels
// sum `nv` (1, 2 or 5) rows, `row_stride` apart, of the partials of `count` blocks into d_out[0 .. nv)
static int reduce_rows(const double *partials, int count, int row_stride, int nv, double *d_out, cudaStream_t st) {
  switch (nv) {
    case 1: k_reduce<1, 0><<<1, 256, 0, st>>>(nullptr, partials, count, row_stride, d_out, nullptr); break;
    case 2: k_reduce<2, 0><<<1, 256, 0, st>>>(nullptr, partials, count, row_stride, d_out, nullptr); break;
    default: k_reduce<5, 0><<<1, 256, 0, st>>>(nullptr, partials, count, row_stride, d_out, nullptr); break;
  }
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_dot_w(int64_t n, const double *d_a, const double *d_b, const double *d_w, double *d_out, void *stream) {
  if (n < 0 || !d_out || (n > 0 && (!d_a || !d_b))) return fail(PCGB_ERR_ARG, "pcgb_dot_w: bad argument");
  PCGB_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  // stream-ordered scratch on the CURRENT device: no state shared between calls, streams or devices
  double *scratch = nullptr;
  PCGB_CUDA(cudaMallocAsync(&scratch, kMaxVecGrid * sizeof(double), st));
  const int grid = vec_grid(n);
  k_dot_w<<<grid, kVecBlock, 0, st>>>(n, d_a, d_b, d_w, scratch);
  int rc = cudaGetLastError() == cudaSuccess ? reduce_rows(scratch, grid, kMaxVecGrid, 1, d_out, st) : fail(PCGB_ERR_CUDA, "pcgb_dot_w: launch failed");
  cudaFreeAsync(scratch, st);
  return rc;
}

int pcgb_axpby(int64_t n, double a, const double *d_x, double b, double *d_y, void *stream) {
  if (n < 0 || (n > 0 && (!d_x || !d_y))) return fail(PCGB_ERR_ARG, "pcgb_axpby: bad argument");
  if (n == 0) return PCGB_OK;
  k_axpby<<<vec_grid(n), kVecBlock, 0, (cudaStream_t)stream>>>(n, a, d_x, b, d_y);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_mul(int64_t n, const double *d_x, const double *d_y, double *d_z, void *stream) {
  if (n < 0 || (n > 0 && (!d_x || !d_y || !d_z))) return fail(PCGB_ERR_ARG, "pcgb_mul: bad argument");
  if (n == 0) return PCGB_OK;
  k_mul<<<vec_grid(n), kVecBlock, 0, (cudaStream_t)stream>>>(n, d_x, d_y, d_z);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_reciprocal(int64_t n, const double *d_d, double *d_out, void *stream) {
  if (n < 0 || (n > 0 && (!d_d || !d_out))) return fail(PCGB_ERR_ARG, "pcgb_reciprocal: bad argument");
  if (n == 0) return PCGB_OK;
  k_reciprocal<<<vec_grid(n), kVecBlock, 0, (cudaStream_t)stream>>>(n, d_d, d_out);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

// ------------------------------------------------------------------------------------ communicator
int pcgb_comm_unique_id(unsigned char id[PCGB_UNIQUE_ID_BYTES]) {
  NcclApi *api = nullptr;
  PCGB_TRY(nccl_api(&api));
  ncclUniqueId uid;
  PCGB_NCCL(api, api->GetUniqueId(&uid));
  static_assert(sizeof(uid) == PCGB_UNIQUE_ID_BYTES, "ncclUniqueId size");
  memcpy(id, &uid, sizeof(uid));
  return PCGB_OK;
}

int pcgb_comm_create(int rank, int nranks, const unsigned char *id, pcgb_comm_t *out) {
  if (!out || rank < 0 || rank >= nranks) return fail(PCGB_ERR_ARG, "pcgb_comm_create: bad argument");
  if (!id && nranks > kMaxPeers) return fail(PCGB_ERR_ARG, "pcgb_comm_create: a peer-only communicator holds at most %d ranks", kMaxPeers);
  PCGB_TRY(require_device());
  pcgb_comm_t c = new pcgb_comm_s();
  c->rank = rank; c->nranks = nranks;
  cudaGetDevice(&c->device);
  int rc = PCGB_OK;
  if (id) {
    NcclApi *api = nullptr;
    rc = nccl_api(&api);
    if (rc == PCGB_OK) {
      ncclUniqueId uid;
      memcpy(&uid, id, sizeof(uid));
      c->api = api;
      int e = api->CommInitRank(&c->comm, nranks, uid, rank);
      if (e != ncclSuccess) rc = fail(PCGB_ERR_NCCL, "ncclCommInitRank -> %s", api->GetErrorString ? api->GetErrorString(e) : "error");
    }
  }
  // the peer window: zeroed before anyone can import it
  cudaError_t ce = cudaSuccess;
  if (rc == PCGB_OK && nranks <= kMaxPeers) {
    if ((ce = cudaMalloc(&c->win, kWinBytes)) == cudaSuccess && (ce = cudaMemset(c->win, 0, kWinBytes)) == cudaSuccess &&
        (ce = cudaMalloc(&c->d_status, sizeof(int))) == cudaSuccess && (ce = cudaMemset(c->d_status, 0, sizeof(int))) == cudaSuccess &&
        (ce = cudaMallocHost(&c->h_status, sizeof(int))) == cudaSuccess)
      ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) rc = fail(PCGB_ERR_CUDA, "pcgb_comm_create: window allocation -> %s", cudaGetErrorString(ce));
  }
  const char *tr = getenv("PCGB_COMM");
  c->transport = (tr && (tr[0] == 'n' || tr[0] == 'N')) ? PCGB_TRANSPORT_NCCL : PCGB_TRANSPORT_PEER;
  if (rc != PCGB_OK) { pcgb_comm_destroy(c); return rc; }
  *out = c;
  return PCGB_OK;
}

int pcgb_comm_destroy(pcgb_comm_t c) {
  if (!c) return PCGB_OK;
  for (int r = 0; r < kMaxPeers; ++r)
    if (c->peer[r]) cudaIpcCloseMemHandle(c->peer[r]);
  cudaFree(c->win); cudaFree(c->d_status);
  if (c->h_status) cudaFreeHost(c->h_status);
  if (c->comm && c->api && c->api->CommDestroy) c->api->CommDestroy(c->comm);
  delete c;
  return PCGB_OK;
}

/* Peer windows: every rank exports the CUDA IPC handle of its window, the host code all-gathers the blobs over ANY
 * side channel (torch.distributed object collectives, mpi4py allgather, ...) and every rank imports them.  From then
 * on the all-reduces and the halo exchange of this communicator are the library's own kernels over NVLink peer memory
 * (csrc/peer.cuh) unless PCGB_COMM=nccl / pcgb_comm_set_transport(c, 0) keeps NCCL. */
int pcgb_comm_window_export(pcgb_comm_t c, unsigned char blob[PCGB_IPC_BLOB_BYTES]) {
  if (!c || !blob) return fail(PCGB_ERR_ARG, "pcgb_comm_window_export: null argument");
  if (!c->win) return fail(PCGB_ERR_ARG, "pcgb_comm_window_export: communicator has no window (more than %d ranks)", kMaxPeers);
  static_assert(sizeof(cudaIpcMemHandle_t) == PCGB_IPC_BLOB_BYTES, "cudaIpcMemHandle_t size");
  cudaIpcMemHandle_t h;
  PCGB_CUDA(cudaIpcGetMemHandle(&h, c->win));
  memcpy(blob, &h, sizeof(h));
  return PCGB_OK;
}

int pcgb_comm_window_import(pcgb_comm_t c, const unsigned char *blobs) {
  if (!c || !blobs) return fail(PCGB_ERR_ARG, "pcgb_comm_window_import: null argument");
  if (!c->win) return fail(PCGB_ERR_ARG, "pcgb_comm_window_import: communicator has no window");
  for (int r = 0; r < c->nranks; ++r) {
    if (r == c->rank || c->peer[r]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, blobs + (size_t)r * PCGB_IPC_BLOB_BYTES, sizeof(h));
    void *ptr = nullptr;
    PCGB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer[r] = static_cast<unsigned long long *>(ptr);
  }
  c->peer_ready = true;
  return PCGB_OK;
}

int pcgb_comm_transport(pcgb_comm_t c) { return c && c->use_peer() ? PCGB_TRANSPORT_PEER : PCGB_TRANSPORT_NCCL; }
int pcgb_comm_set_transport(pcgb_comm_t c, int transport) {
  if (!c || (transport != PCGB_TRANSPORT_NCCL && transport != PCGB_TRANSPORT_PEER)) return fail(PCGB_ERR_ARG, "pcgb_comm_set_transport: bad argument");
  if (transport == PCGB_TRANSPORT_PEER && !c->peer_ready) return fail(PCGB_ERR_ARG, "pcgb_comm_set_transport: peer windows have not been imported");
  if (transport == PCGB_TRANSPORT_NCCL && !c->api) return fail(PCGB_ERR_ARG, "pcgb_comm_set_transport: communicator was created without NCCL");
  c->transport = transport;
  return PCGB_OK;
}
/* 0 = healthy; non-zero after a peer kernel gave up waiting for another rank (sticky) */
int pcgb_comm_status(pcgb_comm_t c, void *stream) {
  if (!c || !c->d_status) return 0;
  if (cudaMemcpyAsync(c->h_status, c->d_status, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream) != cudaSuccess ||
      cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
    return -1;
  return *c->h_status;
}

int pcgb_allreduce_sum(pcgb_comm_t c, double *d_buf, int count, void *stream) {
  if (!c || !d_buf || count < 0) return fail(PCGB_ERR_ARG, "pcgb_allreduce_sum: bad argument");
  return allreduce_sum(c, d_buf, count, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ halo plan

int pcgb_halo_create(pcgb_comm_t c, int n_nbr, const int32_t *nbr_rank, const int64_t *nbr_ptr, const int64_t *idx_host,
                     int64_t nlocal, pcgb_halo_t *out) {
  if (!out || n_nbr < 0 || (n_nbr > 0 && (!c || !nbr_rank || !nbr_ptr))) return fail(PCGB_ERR_ARG, "pcgb_halo_create: bad argument");
  PCGB_TRY(require_device());
  // The whole table is checked before anything is allocated.  Neighbours are distinct and so are the indices of one list
  // (a repeated index would be added twice where the reference's y[list] += recv adds it once).
  if (n_nbr > 0 && nbr_ptr[0] != 0) return fail(PCGB_ERR_ARG, "pcgb_halo_create: nbr_ptr[0] must be 0");
  std::vector<char> listed(c ? (size_t)c->nranks : 0, 0);
  std::vector<int> kept;   // slots with a non-empty list, in the caller's order
  for (int j = 0; j < n_nbr; ++j) {
    if (nbr_rank[j] < 0 || nbr_rank[j] >= c->nranks || nbr_rank[j] == c->rank || nbr_ptr[j + 1] < nbr_ptr[j])
      return fail(PCGB_ERR_ARG, "pcgb_halo_create: bad neighbour table at slot %d", j);
    if (listed[(size_t)nbr_rank[j]]) return fail(PCGB_ERR_ARG, "pcgb_halo_create: neighbour rank %d is listed twice", nbr_rank[j]);
    listed[(size_t)nbr_rank[j]] = 1;
    if (nbr_ptr[j + 1] > nbr_ptr[j]) kept.push_back(j);
  }
  const int64_t m = n_nbr > 0 ? nbr_ptr[n_nbr] : 0;
  if (m > INT32_MAX) return fail(PCGB_ERR_ARG, "pcgb_halo_create: too many shared dofs");
  if (m > 0 && !idx_host) return fail(PCGB_ERR_ARG, "pcgb_halo_create: null index array");
  std::vector<int> idx((size_t)m), ent_nbr((size_t)m), sorted;
  for (int jj = 0; jj < (int)kept.size(); ++jj) {
    const int j = kept[(size_t)jj];
    for (int64_t k = nbr_ptr[j]; k < nbr_ptr[j + 1]; ++k) {
      if (idx_host[k] < 0 || idx_host[k] >= nlocal) return fail(PCGB_ERR_ARG, "pcgb_halo_create: index %lld out of range", (long long)idx_host[k]);
      idx[(size_t)k] = (int)idx_host[k];
      ent_nbr[(size_t)k] = jj;
    }
    sorted.assign(idx.begin() + nbr_ptr[j], idx.begin() + nbr_ptr[j + 1]);
    std::sort(sorted.begin(), sorted.end());
    const auto dup = std::adjacent_find(sorted.begin(), sorted.end());
    if (dup != sorted.end())
      return fail(PCGB_ERR_ARG, "pcgb_halo_create: index %d appears twice in the list of neighbour rank %d", *dup, nbr_rank[j]);
  }
  // An empty list is dropped.  Both sides of an interface list the same number of entries, so both drop it, and a rank
  // whose lists are all empty has no neighbours: nobody waits for an exchange it never starts (m == 0 sends nothing).
  pcgb_halo_t h = new pcgb_halo_s();
  h->comm = c; h->n_nbr = (int)kept.size(); h->m = m; h->nlocal = nlocal;
  h->nbr_ptr.assign(1, 0);
  for (int j : kept) { h->nbr_rank.push_back(nbr_rank[j]); h->nbr_ptr.push_back(nbr_ptr[j + 1]); }
  std::vector<int> nptr(h->nbr_ptr.begin(), h->nbr_ptr.end());
  // group the receive positions by dof, neighbour order inside a dof (stable: k ascending = neighbour ascending)
  std::vector<int> order((size_t)m);
  for (int64_t k = 0; k < m; ++k) order[(size_t)k] = (int)k;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return idx[a] < idx[b]; });
  std::vector<int> dof, ptr, pos((size_t)m);
  for (int64_t s = 0; s < m; ++s) {
    const int k = order[(size_t)s];
    if (s == 0 || idx[k] != idx[order[(size_t)s - 1]]) { dof.push_back(idx[k]); ptr.push_back((int)s); }
    pos[(size_t)s] = k;
  }
  ptr.push_back((int)m);
  h->ndof = (int64_t)dof.size();
  // receive block shared with the neighbours: [2][m] doubles + [n_nbr][2] flags (peer transport)
  h->blk_bytes = (size_t)2 * (size_t)m * sizeof(double) + (size_t)2 * (size_t)std::max(h->n_nbr, 1) * sizeof(unsigned long long);
  cudaError_t ce = cudaSuccess;
  if ((ce = upload(&h->d_idx, idx)) == cudaSuccess && (ce = upload(&h->d_dof, dof)) == cudaSuccess &&
      (ce = upload(&h->d_ptr, ptr)) == cudaSuccess && (ce = upload(&h->d_pos, pos)) == cudaSuccess &&
      (ce = upload(&h->d_nbr_ptr, nptr)) == cudaSuccess && (ce = upload(&h->d_ent_nbr, ent_nbr)) == cudaSuccess &&
      (ce = cudaMalloc(&h->d_send, std::max<size_t>((size_t)m, 1) * sizeof(double))) == cudaSuccess &&
      (ce = cudaMalloc(&h->d_recv, std::max<size_t>((size_t)m, 1) * sizeof(double))) == cudaSuccess &&
      (ce = cudaMalloc(&h->blk, h->blk_bytes)) == cudaSuccess && (ce = cudaMemset(h->blk, 0, h->blk_bytes)) == cudaSuccess &&
      (ce = cudaMalloc(&h->d_epoch, 2 * sizeof(unsigned long long))) == cudaSuccess &&
      (ce = cudaMemset(h->d_epoch, 0, 2 * sizeof(unsigned long long))) == cudaSuccess)
    ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) {
    const int rc = fail(PCGB_ERR_CUDA, "pcgb_halo_create: %s", cudaGetErrorString(ce));
    pcgb_halo_destroy(h);
    return rc;
  }
  *out = h;
  return PCGB_OK;
}

int pcgb_halo_destroy(pcgb_halo_t h) {
  if (!h) return PCGB_OK;
  for (void *p : h->opened) cudaIpcCloseMemHandle(p);
  cudaFree(h->d_idx); cudaFree(h->d_dof); cudaFree(h->d_ptr); cudaFree(h->d_pos); cudaFree(h->d_send); cudaFree(h->d_recv);
  cudaFree(h->blk); cudaFree(h->d_nbr_ptr); cudaFree(h->d_ent_nbr); cudaFree(h->d_remote); cudaFree(h->d_remote_m);
  cudaFree(h->d_remote_flag); cudaFree(h->d_epoch);
  delete h;
  return PCGB_OK;
}

/* Peer transport of the halo: export / all-gather (host side channel) / import, like the communicator window.
 * Every rank of the communicator takes part, also one without neighbours. */
int64_t pcgb_halo_blob_bytes(pcgb_halo_t h) {
  if (!h || !h->comm) return 0;
  return (int64_t)(sizeof(HaloBlobHead) + (size_t)h->comm->nranks * sizeof(HaloBlobRank));
}

int pcgb_halo_export(pcgb_halo_t h, unsigned char *blob) {
  if (!h || !blob || !h->comm) return fail(PCGB_ERR_ARG, "pcgb_halo_export: null argument");
  HaloBlobHead head;
  memset(&head, 0, sizeof(head));
  cudaIpcMemHandle_t ih;
  PCGB_CUDA(cudaIpcGetMemHandle(&ih, h->blk));
  memcpy(head.handle, &ih, sizeof(ih));
  head.m = h->m;
  memcpy(blob, &head, sizeof(head));
  std::vector<HaloBlobRank> tab((size_t)h->comm->nranks, HaloBlobRank{-1, -1, 0});
  for (int j = 0; j < h->n_nbr; ++j) tab[(size_t)h->nbr_rank[j]] = HaloBlobRank{h->nbr_ptr[j], j, h->nbr_ptr[j + 1] - h->nbr_ptr[j]};
  memcpy(blob + sizeof(head), tab.data(), tab.size() * sizeof(HaloBlobRank));
  return PCGB_OK;
}

int pcgb_halo_import(pcgb_halo_t h, const unsigned char *blobs) {
  if (!h || !blobs || !h->comm) return fail(PCGB_ERR_ARG, "pcgb_halo_import: null argument");
  if (h->peer_ready) return PCGB_OK;
  const size_t stride = (size_t)pcgb_halo_blob_bytes(h);
  const int me = h->comm->rank;
  std::vector<double *> remote((size_t)h->n_nbr, nullptr);
  std::vector<int64_t> remote_m((size_t)h->n_nbr, 0);
  std::vector<unsigned long long *> remote_flag((size_t)h->n_nbr, nullptr);
  for (int j = 0; j < h->n_nbr; ++j) {
    const unsigned char *b = blobs + (size_t)h->nbr_rank[j] * stride;
    HaloBlobHead head;
    HaloBlobRank mine;
    memcpy(&head, b, sizeof(head));
    memcpy(&mine, b + sizeof(head) + (size_t)me * sizeof(HaloBlobRank), sizeof(mine));
    const int64_t cnt = h->nbr_ptr[j + 1] - h->nbr_ptr[j];
    if (mine.off < 0 || mine.cnt != cnt)
      return fail(PCGB_ERR_ARG, "pcgb_halo_import: rank %d shares %lld dofs with rank %d but that rank lists %lld for us (interface lists must match)",
                  me, (long long)cnt, h->nbr_rank[j], (long long)mine.cnt);
    cudaIpcMemHandle_t ih;
    memcpy(&ih, head.handle, sizeof(ih));
    void *ptr = nullptr;
    PCGB_CUDA(cudaIpcOpenMemHandle(&ptr, ih, cudaIpcMemLazyEnablePeerAccess));
    h->opened.push_back(ptr);
    remote[(size_t)j] = static_cast<double *>(ptr) + mine.off;
    remote_m[(size_t)j] = head.m;
    remote_flag[(size_t)j] = reinterpret_cast<unsigned long long *>(static_cast<unsigned char *>(ptr) + (size_t)2 * (size_t)head.m * sizeof(double)) + 2 * mine.slot;
  }
  PCGB_CUDA(upload(&h->d_remote, remote));
  PCGB_CUDA(upload(&h->d_remote_m, remote_m));
  PCGB_CUDA(upload(&h->d_remote_flag, remote_flag));
  h->peer_ready = true;
  return PCGB_OK;
}

int pcgb_halo_exchange_add(pcgb_halo_t h, double *d_y, void *stream) {
  if (!h || !d_y) return fail(PCGB_ERR_ARG, "pcgb_halo_exchange_add: null argument");
  return halo_exchange_add(h, d_y, (cudaStream_t)stream);
}

int64_t pcgb_halo_bytes(pcgb_halo_t h) { return h ? h->m * 8 : 0; }

}  // extern "C"

// The caller's pattern group g: a size of 1..max_nd, at most max_ne elements, and the arrays its elements need.
static int check_group(const pcgb_ebe_group &src, int g, int max_nd, int64_t max_ne, const char *who) {
  if (src.nd <= 0 || src.nd > max_nd || src.ne < 0 || src.ne > max_ne || !src.ke_host || (src.ne > 0 && (!src.d_idx || !src.d_ck)))
    return fail(PCGB_ERR_ARG, "%s: group %d: pattern size must be 1..%d and arrays non-null", who, g, max_nd);
  return PCGB_OK;
}

// device copy of the group's pattern matrix Ke (nd x nd), or of its transpose
static int upload_ke(const pcgb_ebe_group &src, const double **d_ke, const char *who, bool transpose = false) {
  const size_t bytes = (size_t)src.nd * src.nd * sizeof(double);
  std::vector<double> kt;
  const double *h = src.ke_host;
  if (transpose) {
    kt.resize((size_t)src.nd * src.nd);
    for (int i = 0; i < src.nd; ++i)
      for (int j = 0; j < src.nd; ++j) kt[(size_t)j * src.nd + i] = src.ke_host[(size_t)i * src.nd + j];
    h = kt.data();
  }
  double *d = nullptr;
  cudaError_t ce = cudaMalloc(&d, bytes);
  if (ce == cudaSuccess) ce = cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) { cudaFree(d); return fail(PCGB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(ce)); }
  *d_ke = d;
  return PCGB_OK;
}

// Groups of an EBE plan (atomic, ordered or coloured operator): device copies of Ke, constant-memory slots of the 24-dof
// patterns, the warp-kernel block tables (blocks in group order).  On failure P holds what was acquired so far, which
// ebe_plan_free releases.  ke_transposed: the device copies hold Ke^T, so that a warp kernel reading column i of the copy
// (coalesced across lanes) gets row i of Ke.
static int ebe_plan_build(EbePlan &P, int64_t n, int ngroups, const pcgb_ebe_group *groups, const char *who,
                          bool ke_transposed = false) {
  P.n = n;
  std::vector<int> blk_group;
  std::vector<int64_t> blk_e0;
  P.bytes = 16 * n;
  for (int g = 0; g < ngroups; ++g) {
    const pcgb_ebe_group &src = groups[g];
    PCGB_TRY(check_group(src, g, 96, INT64_MAX, who));
    EbeGroup eg;
    eg.nd = src.nd; eg.ne = src.ne; eg.idx = src.d_idx; eg.sign = src.d_sign; eg.ck = src.d_ck;
    PCGB_TRY(upload_ke(src, &eg.ke, who, ke_transposed));
    if (src.nd == 24) eg.slot = ebe_slot_acquire(src.ke_host);
    if (eg.slot < 0)
      for (int64_t e0 = 0; e0 < src.ne; e0 += kEbeWarpsPerBlock) { blk_group.push_back((int)P.groups.size()); blk_e0.push_back(e0); }
    P.bytes += src.ne * ((int64_t)src.nd * (4 + (src.d_sign ? 1 : 0)) + 8);
    P.groups.push_back(eg);
  }
  P.nblk_warp = (int)blk_group.size();
  cudaError_t ce = cudaSuccess;
  if ((ce = upload(&P.d_groups, P.groups)) != cudaSuccess || (ce = upload(&P.d_blk_group, blk_group)) != cudaSuccess ||
      (ce = upload(&P.d_blk_e0, blk_e0)) != cudaSuccess)
    return fail(PCGB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(ce));
  return PCGB_OK;
}

static void ebe_plan_free(EbePlan &P, int device) {
  for (EbeGroup &g : P.groups) {
    cudaFree(const_cast<double *>(g.ke));
    ebe_slot_release(device, g.slot);
  }
  cudaFree(P.d_groups); cudaFree(P.d_blk_group); cudaFree(P.d_blk_e0);
}

extern "C" {

// ------------------------------------------------------------------------------------ EBE operator (opt-in, f1)
int pcgb_ebe_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, pcgb_ebe_t *out) {
  if (!out || n < 0 || ngroups < 0 || (ngroups > 0 && !groups)) return fail(PCGB_ERR_ARG, "pcgb_ebe_create: bad argument");
  if (n >= (1 << 30)) return fail(PCGB_ERR_ARG, "pcgb_ebe_create: more than 2^30 dofs");
  PCGB_TRY(require_device());
  pcgb_ebe_t E = new pcgb_ebe_s();
  cudaGetDevice(&E->device);
  const int rc = ebe_plan_build(E->P, n, ngroups, groups, "pcgb_ebe_create");
  if (rc != PCGB_OK) { pcgb_ebe_destroy(E); return rc; }
  *out = E;
  return PCGB_OK;
}

int pcgb_ebe_destroy(pcgb_ebe_t E) {
  if (!E) return PCGB_OK;
  ebe_plan_free(E->P, E->device);
  delete E;
  return PCGB_OK;
}

int pcgb_ebe_apply(pcgb_ebe_t E, const double *d_x, double *d_y, void *stream) {
  if (!E || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_ebe_apply: null argument");
  return ebe_apply(E->P, d_x, d_y, (cudaStream_t)stream);
}

int64_t pcgb_ebe_bytes(pcgb_ebe_t E) { return E ? E->P.bytes : 0; }

// ------------------------------------------------------------------------------------ ordered EBE operator (bit-reproducible)
int pcgb_ebe_ordered_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, pcgb_ebe_ordered_t *out) {
  if (!out || n < 0 || ngroups < 0 || (ngroups > 0 && !groups)) return fail(PCGB_ERR_ARG, "pcgb_ebe_ordered_create: bad argument");
  if (n >= (1 << 30)) return fail(PCGB_ERR_ARG, "pcgb_ebe_ordered_create: more than 2^30 dofs");
  // every refusal happens here, before anything is allocated
  int64_t nslots = 0;
  for (int g = 0; g < ngroups; ++g) {
    const pcgb_ebe_group &src = groups[g];
    PCGB_TRY(check_group(src, g, 96, INT64_MAX, "pcgb_ebe_ordered_create"));
    if (src.ne > INT32_MAX || (nslots += (int64_t)src.nd * src.ne) > INT32_MAX)
      return fail(PCGB_ERR_ARG, "pcgb_ebe_ordered_create: 2^31 or more element slots (slot positions are int32)");
  }
  PCGB_TRY(require_device());
  pcgb_ebe_ordered_t O = new pcgb_ebe_ordered_s();
  cudaGetDevice(&O->device);
  EboPlan &Q = O->O;
  int rc = ebe_plan_build(Q.P, n, ngroups, groups, "pcgb_ebe_ordered_create");
  if (rc == PCGB_OK) {
    for (const EbeGroup &g : Q.P.groups) { Q.off.push_back(Q.nslots); Q.nslots += (int64_t)g.nd * g.ne; }
    rc = ebo_build_lists(Q, nullptr);
  }
  if (rc != PCGB_OK) { pcgb_ebe_ordered_destroy(O); return rc; }
  // phase 1 as the atomic operator (indices, signs, Ck, x, y) plus the products written; phase 2 reads them back with their
  // positions and the list offsets (y is already counted)
  Q.P.bytes += 8 * Q.nfree + 12 * Q.nfree + 8 * (n + 1);
  *out = O;
  return PCGB_OK;
}

int pcgb_ebe_ordered_destroy(pcgb_ebe_ordered_t O) {
  if (!O) return PCGB_OK;
  ebe_plan_free(O->O.P, O->device);
  ebo_free_lists(O->O);
  delete O;
  return PCGB_OK;
}

int pcgb_ebe_ordered_apply(pcgb_ebe_ordered_t O, const double *d_x, double *d_y, void *stream) {
  if (!O || (O->O.P.n > 0 && (!d_x || !d_y))) return fail(PCGB_ERR_ARG, "pcgb_ebe_ordered_apply: null argument");   // n = 0: no vector
  return ebo_apply(O->O, d_x, d_y, (cudaStream_t)stream);
}

int64_t pcgb_ebe_ordered_bytes(pcgb_ebe_ordered_t O) { return O ? O->O.P.bytes : 0; }

// ------------------------------------------------------------------------------------ device assembly (f2)
int pcgb_assemble_symbolic(int64_t n, int ngroups, const pcgb_ebe_group *groups, int64_t *d_rowptr, int64_t *nnz_out, void *stream,
                           pcgb_asm_t *out) {
  if (!out || !d_rowptr || !nnz_out || n < 0 || ngroups < 0 || (ngroups > 0 && !groups)) return fail(PCGB_ERR_ARG, "pcgb_assemble_symbolic: bad argument");
  if (n >= (1ll << 31) - 8 || ngroups >= 65536) return fail(PCGB_ERR_ARG, "pcgb_assemble_symbolic: too many rows / pattern groups");
  PCGB_TRY(require_device());
  pcgb_asm_t a = new pcgb_asm_s();
  a->P.n = n;
  int rc = PCGB_OK;
  for (int g = 0; g < ngroups && rc == PCGB_OK; ++g) {
    const pcgb_ebe_group &src = groups[g];
    AsmGroup ag;
    ag.nd = src.nd; ag.ne = src.ne; ag.idx = src.d_idx; ag.sign = src.d_sign; ag.ck = src.d_ck;
    if ((rc = check_group(src, g, 255, (1ll << 40) - 1, "pcgb_assemble_symbolic")) == PCGB_OK &&
        (rc = upload_ke(src, &ag.ke, "pcgb_assemble_symbolic")) == PCGB_OK)
      a->P.groups.push_back(ag);
  }
  if (rc == PCGB_OK) rc = asm_symbolic(a->P, d_rowptr, (cudaStream_t)stream);
  if (rc != PCGB_OK) { pcgb_assemble_destroy(a); return rc; }
  *nnz_out = a->P.nnz;
  *out = a;
  return PCGB_OK;
}

int pcgb_assemble_numeric(pcgb_asm_t a, const int64_t *d_rowptr, int32_t *d_col, double *d_val, void *stream) {
  if (!a || !d_rowptr || (a->P.nnz > 0 && (!d_col || !d_val))) return fail(PCGB_ERR_ARG, "pcgb_assemble_numeric: null argument");
  return asm_numeric(a->P, d_rowptr, d_col, d_val, (cudaStream_t)stream);
}

int pcgb_assemble_destroy(pcgb_asm_t a) {
  if (!a) return PCGB_OK;
  asm_free(a->P);
  delete a;
  return PCGB_OK;
}

// ------------------------------------------------------------------------------------ coloured EBE operator (operator level)
// groups[] holds one entry per (pattern group, colour), sorted by colour; phase[g] is the colour.  Pattern matrices of
// the 24-dof groups are de-duplicated into the constant-memory slots by content of ke_host.  The colouring itself is
// trusted (EbeMatrixColored checks it on the host).
int pcgb_ebe2_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, const int32_t *phase, pcgb_ebe2_t *out) {
  if (!out || n < 0 || ngroups < 0 || (ngroups > 0 && (!groups || !phase))) return fail(PCGB_ERR_ARG, "pcgb_ebe2_create: bad argument");
  if (n >= (1 << 30)) return fail(PCGB_ERR_ARG, "pcgb_ebe2_create: more than 2^30 dofs");
  PCGB_TRY(require_device());
  for (int g = 1; g < ngroups; ++g)
    if (phase[g] < phase[g - 1]) return fail(PCGB_ERR_ARG, "pcgb_ebe2_create: groups must be sorted by phase (colour)");
  pcgb_ebe2_t E = new pcgb_ebe2_s();
  cudaGetDevice(&E->device);
  const int rc = ebe_plan_build(E->C.P, n, ngroups, groups, "pcgb_ebe2_create", true);
  if (rc != PCGB_OK) { pcgb_ebe2_destroy(E); return rc; }
  // Launches in colour order: the colour's t24 groups in group order, then one warp launch over the colour's blocks, which
  // are contiguous in the block tables because the groups arrive sorted by colour.  A t24 launch and a warp launch of one
  // colour may touch the same dofs only if the colouring was done per pattern group; the Python side colours ALL elements
  // of the subdomain together and checks that no free dof is shared inside a colour, so they cannot.
  int blk = 0;
  for (int g = 0; g < ngroups;) {
    const int blk0 = blk;
    for (const int c = phase[g]; g < ngroups && phase[g] == c; ++g) {
      const EbeGroup &eg = E->C.P.groups[(size_t)g];
      if (eg.slot < 0) blk += (int)((eg.ne + kEbeWarpsPerBlock - 1) / kEbeWarpsPerBlock);
      else if (eg.ne > 0) E->C.launches.push_back({0, g, 0});
    }
    if (blk > blk0) E->C.launches.push_back({1, blk0, blk});
  }
  *out = E;
  return PCGB_OK;
}

int pcgb_ebe2_destroy(pcgb_ebe2_t E) {
  if (!E) return PCGB_OK;
  ebe_plan_free(E->C.P, E->device);
  delete E;
  return PCGB_OK;
}

int pcgb_ebe2_apply(pcgb_ebe2_t E, const double *d_x, double *d_y, void *stream) {
  if (!E || (E->C.P.n > 0 && (!d_x || !d_y))) return fail(PCGB_ERR_ARG, "pcgb_ebe2_apply: null argument");   // n = 0: no vector
  return ebe_color_apply(E->C, d_x, d_y, (cudaStream_t)stream);
}

int pcgb_ebe2_launches(pcgb_ebe2_t E) { return E ? (int)E->C.launches.size() : 0; }

// ------------------------------------------------------------------------------------ solver
static int solver_create_common(FineOp op, pcgb_halo_t halo, pcgb_comm_t comm, pcgb_solver_t *out) {
  if (halo && !comm) comm = halo->comm;
  PCGB_TRY(require_device());
  pcgb_solver_t s = new pcgb_solver_s();
  s->op = op; s->halo = halo; s->comm = comm; s->n = op.rows();
  s->fork_halo = env_int("PCGB_FORK", 1) != 0;
  const size_t nb = (size_t)(s->n > 0 ? s->n : 1) * sizeof(double);
  s->stage_cap = ((op.A ? op.A->P.ntiles : 0) + 4095) / 4096 + 1;
  cudaError_t ce = cudaSuccess;
  int rc = PCGB_OK;
  if ((ce = cudaMalloc(&s->r, nb)) == cudaSuccess && (ce = cudaMalloc(&s->p, nb)) == cudaSuccess &&
      (ce = cudaMalloc(&s->q, nb)) == cudaSuccess && (ce = cudaMalloc(&s->xalt, nb)) == cudaSuccess &&
      (ce = cudaMalloc(&s->xown, nb)) == cudaSuccess && (ce = cudaMemset(s->p, 0, nb)) == cudaSuccess &&
      (ce = cudaMalloc(&s->partials, 5 * kMaxVecGrid * sizeof(double))) == cudaSuccess &&
      (ce = cudaMalloc(&s->stage, (size_t)s->stage_cap * sizeof(double))) == cudaSuccess &&
      (ce = cudaMalloc(&s->red, 8 * sizeof(double))) == cudaSuccess && (ce = cudaMemset(s->red, 0, 8 * sizeof(double))) == cudaSuccess &&
      (ce = cudaMalloc(&s->d_ctrl, sizeof(PcgCtrl))) == cudaSuccess && (ce = cudaMallocHost(&s->h_ctrl, sizeof(PcgCtrl))) == cudaSuccess &&
      (ce = cudaMallocHost(&s->h_red, 8 * sizeof(double))) == cudaSuccess &&
      (ce = cudaStreamCreateWithFlags(&s->own, cudaStreamNonBlocking)) == cudaSuccess &&
      (ce = cudaStreamCreateWithFlags(&s->side, cudaStreamNonBlocking)) == cudaSuccess &&
      (ce = cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming)) == cudaSuccess &&
      (ce = cudaEventCreateWithFlags(&s->ev_join, cudaEventDisableTiming)) == cudaSuccess &&
      (ce = cudaEventCreateWithFlags(&s->ev_in, cudaEventDisableTiming)) == cudaSuccess &&
      (ce = cudaEventCreateWithFlags(&s->ev_out, cudaEventDisableTiming)) == cudaSuccess &&
      (ce = cudaEventCreate(&s->ev_l0)) == cudaSuccess && (ce = cudaEventCreate(&s->ev_l1)) == cudaSuccess &&
      (ce = cudaEventCreate(&s->ev_s0)) == cudaSuccess)
    ce = cudaEventCreate(&s->ev_s1);
  if (ce != cudaSuccess) rc = fail(PCGB_ERR_CUDA, "pcgb_solver_create: %s", cudaGetErrorString(ce));
  // interface-first tile order: the tiles owning exchanged rows run first, their values travel while the rest computes
  // Opt-in (PCGB_OVERLAP=1): with the peer-store halo the exchange costs a few microseconds and is not worth a second
  // persistent launch (measured slower than the unsplit launch at 2 GPUs, 128^3 per GPU).
  if (rc == PCGB_OK && op.A && halo && halo->ndof > 0 && env_int("PCGB_OVERLAP", 0) != 0)
    rc = spmv_set_boundary_rows(op.A->P, halo->d_dof, halo->ndof, s->own);
  if (rc != PCGB_OK) { pcgb_solver_destroy(s); return rc; }
  *out = s;
  return PCGB_OK;
}

int pcgb_solver_create(pcgb_csr_t A, pcgb_halo_t halo, pcgb_comm_t comm, pcgb_solver_t *out) {
  if (!A || !out) return fail(PCGB_ERR_ARG, "pcgb_solver_create: null argument");
  if (A->P.nrows != A->P.ncols) return fail(PCGB_ERR_ARG, "pcgb_solver_create: operator must be square");
  return solver_create_common(FineOp{A}, halo, comm, out);
}

int pcgb_solver_create_ebe(pcgb_ebe_t E, pcgb_halo_t halo, pcgb_comm_t comm, pcgb_solver_t *out) {
  if (!E || !out) return fail(PCGB_ERR_ARG, "pcgb_solver_create_ebe: null argument");
  return solver_create_common(FineOp{nullptr, E}, halo, comm, out);
}

int pcgb_solver_create_ebe_ordered(pcgb_ebe_ordered_t O, pcgb_halo_t halo, pcgb_comm_t comm, pcgb_solver_t *out) {
  if (!O || !out) return fail(PCGB_ERR_ARG, "pcgb_solver_create_ebe_ordered: null argument");
  return solver_create_common(FineOp{nullptr, nullptr, O}, halo, comm, out);
}

// the index-free hex-box operator (pcg_solver.py:263-300 in the ordered operator's order)
int pcgb_solver_create_hexop(pcgb_hexop_t H, pcgb_halo_t halo, pcgb_comm_t comm, pcgb_solver_t *out) {
  if (!H || !out) return fail(PCGB_ERR_ARG, "pcgb_solver_create_hexop: null argument");
  return solver_create_common(FineOp{nullptr, nullptr, nullptr, H}, halo, comm, out);
}

int pcgb_solver_destroy(pcgb_solver_t s) {
  if (!s) return PCGB_OK;
  for (pcgb_mg_t mg : s->mgs) mg_detach(mg);
  if (s->gexec) cudaGraphExecDestroy(s->gexec);
  if (s->own) cudaStreamDestroy(s->own);
  if (s->side) cudaStreamDestroy(s->side);
  if (s->ev_fork) cudaEventDestroy(s->ev_fork);
  if (s->ev_join) cudaEventDestroy(s->ev_join);
  if (s->ev_in) cudaEventDestroy(s->ev_in);
  if (s->ev_out) cudaEventDestroy(s->ev_out);
  if (s->ev_l0) cudaEventDestroy(s->ev_l0);
  if (s->ev_l1) cudaEventDestroy(s->ev_l1);
  if (s->ev_s0) cudaEventDestroy(s->ev_s0);
  if (s->ev_s1) cudaEventDestroy(s->ev_s1);
  for (cudaEvent_t e : s->ev_k) cudaEventDestroy(e);
  cudaFree(s->r); cudaFree(s->p); cudaFree(s->q); cudaFree(s->xalt); cudaFree(s->xown); cudaFree(s->partials); cudaFree(s->stage);
  cudaFree(s->red); cudaFree(s->d_ctrl); cudaFree(s->tr_local);
  if (s->h_ctrl) cudaFreeHost(s->h_ctrl);
  if (s->h_red) cudaFreeHost(s->h_red);
  delete s;
  return PCGB_OK;
}

int64_t pcgb_trace_record_bytes(void) { return (int64_t)sizeof(PcgTraceRec); }

int pcgb_solver_set_trace(pcgb_solver_t s, void *d_trace, int64_t capacity, double *d_snapshot) {
  if (!s || capacity < 0) return fail(PCGB_ERR_ARG, "pcgb_solver_set_trace: bad argument");
  if (d_trace && !s->tr_local) PCGB_CUDA(cudaMalloc(&s->tr_local, 8 * sizeof(double)));
  s->trace = static_cast<PcgTraceHdr *>(d_trace);
  s->trace_cap = d_trace ? capacity : 0;
  s->snapshot = d_trace ? d_snapshot : nullptr;
  return PCGB_OK;
}

}  // extern "C"

// ---- host helpers of the solve -------------------------------------------------------------
namespace {

inline bool multi_rank(pcgb_solver_t s) { return s->comm && s->comm->nranks > 1; }
inline bool peer_path(pcgb_solver_t s) { return multi_rank(s) && s->comm->use_peer() && (!s->halo || s->halo->m == 0 || s->halo->use_peer()); }

// y = A x + interface sum  (calcMPFint, pcg_solver.py:339-342)
int op_apply(pcgb_solver_t s, const double *x, double *y, cudaStream_t st) {
  PCGB_TRY(s->op.apply(x, y, st, &s->launches, nullptr));
  if (s->halo) PCGB_TRY(halo_exchange_add(s->halo, y, st, &s->launches));
  return PCGB_OK;
}

// sum `nv` (<= 2) rows of s->partials over blocks and ranks into the device scalars s->red[dst .. dst+nv)
int reduce_to_device(pcgb_solver_t s, int count, int nv, int dst, cudaStream_t st) {
  PCGB_TRY(reduce_rows(s->partials, count, kMaxVecGrid, nv, s->red + dst, st));
  s->launches += 1;
  if (multi_rank(s)) {
    PCGB_TRY(allreduce_sum(s->comm, s->red + dst, nv, st));
    if (s->comm->use_peer()) s->launches += 1;
  }
  return PCGB_OK;
}

// q = A x ; r = b - q ; sum r*r*w over all ranks -> s->red[dst] (device)
int true_residual_dev(pcgb_solver_t s, const double *b, const double *w, const double *x, int dst, cudaStream_t st) {
  PCGB_TRY(op_apply(s, x, s->q, st));
  const int grid = vec_grid(s->n);
  k_residual<<<grid, kVecBlock, 0, st>>>(s->n, b, s->q, w, s->r, s->partials);
  PCGB_CHECK_LAUNCH();
  s->launches += 1;
  return reduce_to_device(s, grid, 1, dst, st);
}

// host copy of s->red[6..8) (one synchronisation)
int fetch_red(pcgb_solver_t s, cudaStream_t st) {
  PCGB_CUDA(cudaMemcpyAsync(s->h_red, s->red + 6, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  return PCGB_OK;
}

// r = b - A x ; returns sqrt(sum r*r*w) over all ranks
int true_residual(pcgb_solver_t s, const double *b, const double *w, const double *x, double *normr, cudaStream_t st) {
  PCGB_TRY(true_residual_dev(s, b, w, x, 6, st));
  PCGB_TRY(fetch_red(s, st));
  *normr = std::sqrt(s->h_red[0]);
  return PCGB_OK;
}

// ---- trace (pcgb_solver_set_trace): extra launches only when tracing is on
inline int trace_rank(pcgb_solver_t s) { return s->comm ? s->comm->rank : 0; }
// this rank's sum of `nv` rows of the partials of `count` blocks into tr_local[dst..) (the same code as the local half of the
// all-reduce, hence the same bits)
int trace_local(pcgb_solver_t s, const double *partials, int count, int row_stride, int nv, int dst, cudaStream_t st, int *nl) {
  if (!s->trace || !multi_rank(s)) return PCGB_OK;
  PCGB_TRY(reduce_rows(partials, count, row_stride, nv, s->tr_local + dst, st));
  *nl += 1;
  return PCGB_OK;
}
int trace_step(pcgb_solver_t s, int kind, double bb, double r0r0, cudaStream_t st, int *nl) {
  if (!s->trace) return PCGB_OK;
  k_trace_step<<<1, 1, 0, st>>>(s->trace, reinterpret_cast<PcgTraceRec *>(s->trace + 1), s->trace_cap, trace_rank(s), kind,
                                s->d_ctrl, s->red, multi_rank(s) ? s->tr_local : nullptr, bb, r0r0);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return PCGB_OK;
}
// has_local: tr_local[3] holds this rank's share of rr (false when rr is not a reduced sum, e.g. 0 for a converged finalisation)
int trace_host(pcgb_solver_t s, int kind, const PcgCtrl &c, double rr, bool has_local, double *snap_tail, cudaStream_t st) {
  if (!s->trace) return PCGB_OK;
  k_trace_host<<<1, 1, 0, st>>>(s->trace, reinterpret_cast<PcgTraceRec *>(s->trace + 1), s->trace_cap, trace_rank(s), kind, c,
                                rr, multi_rank(s) && has_local ? s->tr_local : nullptr, snap_tail);
  PCGB_CHECK_LAUNCH();
  s->launches += 1;
  return PCGB_OK;
}

}  // namespace

// ---- geometric multigrid preconditioner (pcgb_mg_*): one symmetric V-cycle z = M r
// Across ranks (pcgb_mg_create_ranks) levels 0 .. la are ranked: each rank holds its own box, vectors are consistent (every
// copy of a shared dof holds the full value) and every operator application and restriction is followed by the level's
// exchange-add.  Level la is not smoothed: its vector is gathered into the global box, which levels la+1 .. hold as a
// replicated one-rank hierarchy on every rank.  One rank: la = -1 and every level is a whole box.

// What a level applies: the solver's operator (level 0), the level's CSR matrix, the index-free operator of its box
// (pcgb_mg_create_index_free / _ranks_index_free: Ke, uniform Ck = E 2^glev h), P^T A_0 P from the fine Ck field (level 1
// of pcgb_mg_create_field_rap), or nothing (the gathered level and the coarsest level).
enum class MgOp { None, Fine, Csr, Hex, Rap };

struct MgLevel {
  HexGeom g{};
  MgPlace place{};             // the box inside the level's global box (one rank: the box itself at e0 = 0)
  int glev = 0;                // level of the global hierarchy (spacing 2^glev h)
  pcgb_halo_t halo = nullptr;  // ranked levels: exchange-add of the level (level 0: the solver's halo; not owned)
  double *own = nullptr;       // ranked levels: 0/1 ownership of the dofs (copy)
  int64_t n = 0;
  MgOp op = MgOp::None;
  void *rowptr = nullptr;   // Csr: device-generated CSR (int32 offsets below 2^31 non-zeros)
  int *col = nullptr;
  double *val = nullptr;
  CsrPlan P;
  HexOp H;                  // Hex
  RapShape R{};             // Rap: y = P^T A_0 P x by k_mg_rap1 from Ke and the fine Ck field, no matrix
  HexKe ke{};
  const double *ck_fine = nullptr;
  double *dinv = nullptr;                                    // inverse diagonal (level 0: a copy of the caller's Minv)
  double *b = nullptr, *x = nullptr;                         // right-hand side and correction (level 0: the caller's r and z)
  double *r = nullptr, *d = nullptr, *q = nullptr;           // smoother residual, direction, operator product
  double lambda = 0.0, inv_theta = 0.0;
  std::vector<double> c1, c2;                                // Chebyshev recurrence of steps 1 .. degree-1
  // the coarsening from this level to the next (pcgb_mg_create_any): any = some axis is kept or odd, so the transfers
  // and the Galerkin products take the *_any kernels with `keep` (bit a: axis a kept); otherwise every ne is halved
  bool any = false;
  int keep = 0;
};

struct pcgb_mg_s {
  pcgb_solver_t s = nullptr;
  std::vector<MgLevel> lv;
  int degree = 2;
  double lo = 0.25;
  int la = -1;                     // gathered ranked level (-1: one rank)
  pcgb_halo_t gather = nullptr;    // all-to-all plan over the global box of level la (not owned)
  int nc = 0;
  double *chol = nullptr;   // coarsest level: dense Cholesky factor, L in the lower triangle mirrored into the upper
  double *z = nullptr;      // z = M r of the PCG loop
  double *partials = nullptr, *red = nullptr, *h_red = nullptr;
  int *d_bad = nullptr;
  int64_t bytes = 0;
  // field hierarchies (pcgb_mg_create_field): the fine per-element Ck, the Galerkin element matrices of the level being
  // built (freed once the next level's exist), their peak device bytes and the device time of k_mg_galerkin.  Across
  // ranks (pcgb_mg_create_ranks_field) also the all-to-all plan over the element matrices of level la's global box, used
  // by the set-up only (not owned, not kept after create)
  const double *ck_fine = nullptr;
  pcgb_halo_t kel_gather = nullptr;
  double *kel = nullptr;
  int64_t kel_peak = 0;
  double galerkin_ms = 0.0;
};

void mg_detach(pcgb_mg_t mg) { mg->s = nullptr; }

namespace {

constexpr int kMgLanczosSteps = 20;

// whether level l is smoothed: every level above the coarsest but the gathered one
bool mg_smoothed(pcgb_mg_t mg, int l) { return l >= 0 && l + 1 < (int)mg->lv.size() && l != mg->la; }

// y = A x on level l, the rank's local product (no exchange-add)
int level_apply(pcgb_mg_t mg, int l, const double *x, double *y, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &L = mg->lv[(size_t)l];
  switch (L.op) {
    case MgOp::Fine: return mg->s->op.apply(x, y, st, nl, skip);
    case MgOp::Csr: return spmv_launch(L.P, x, y, false, st, nl, skip);
    case MgOp::Hex: return hexop_apply(L.H, x, y, st, nl, skip);
    case MgOp::Rap:
      k_mg_rap1<<<(unsigned)((int64_t)L.R.nbx * L.R.nby * L.R.nbz), kRapThreads, kRapSmem, st>>>(L.ke, L.R, L.ck_fine, x, y, skip);
      PCGB_CHECK_LAUNCH();
      if (nl) *nl += 1;
      return PCGB_OK;
    case MgOp::None: break;
  }
  return fail(PCGB_ERR_ARG, "level %d has no operator", l);
}

// y = A x on level l, then the level's exchange-add on a ranked level.  The exchange runs whatever the loop state, like
// the fine halo of the iteration: every rank enqueues the same exchanges and all ranks stop at the same iteration.
int mg_op(pcgb_mg_t mg, int l, const double *x, double *y, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &L = mg->lv[(size_t)l];
  PCGB_TRY(level_apply(mg, l, x, y, st, nl, skip));
  return L.halo ? halo_exchange_add(L.halo, y, st, nl) : PCGB_OK;
}

// Chebyshev smoothing of D^-1 A on level l: zero_start: x = S b (no operator application for x = 0); otherwise
// x += S (b - A x).  S is the same polynomial in both forms, so pre- and post-smoothing keep the V-cycle symmetric.
// resid (pre-smoother): one more product leaves r = b - A x for the restriction.
int mg_smooth(pcgb_mg_t mg, int l, const double *b, double *x, bool zero_start, bool resid, cudaStream_t st, int *nl, const int *skip) {
  MgLevel &L = mg->lv[(size_t)l];
  const int grid = vec_grid(L.n);
  if (!zero_start) PCGB_TRY(mg_op(mg, l, x, L.q, st, nl, skip));
  k_mg_cheb_first<<<grid, 256, 0, st>>>(L.n, b, zero_start ? nullptr : L.q, L.dinv, L.inv_theta, L.r, L.d, x, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  for (int j = 0; j < (int)L.c1.size() + (resid ? 1 : 0); ++j) {
    const bool last = j == (int)L.c1.size();
    PCGB_TRY(mg_op(mg, l, L.d, L.q, st, nl, skip));
    k_mg_cheb_step<<<grid, 256, 0, st>>>(L.n, L.q, L.dinv, last ? 0.0 : L.c1[(size_t)j], last ? 0.0 : L.c2[(size_t)j], last ? 1 : 0,
                                         L.r, L.d, x, skip);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
  }
  return PCGB_OK;
}

inline unsigned mg_node_grid(const HexGeom &g) { return (unsigned)((g.nfree_nodes + 255) / 256); }

int mg_coarse_solve(pcgb_mg_t mg, const double *r, double *z, cudaStream_t st, int *nl, const int *skip) {
  k_mg_chol_solve<<<1, kMgCholThreads, 0, st>>>(mg->nc, mg->chol, r, z, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return PCGB_OK;
}

// r_c = P^T r_f from level l to l+1; on a ranked level each rank sums its owned fine nodes and the coarse level's
// exchange-add completes the sum
int mg_restrict(pcgb_mg_t mg, int l, const double *rf, double *rc, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &A = mg->lv[(size_t)l], &C = mg->lv[(size_t)l + 1];
  if (A.any) k_mg_restrict_any<<<mg_node_grid(C.g), 256, 0, st>>>(A.g, C.g, A.keep, rf, rc, skip);
  else k_mg_restrict<<<mg_node_grid(C.g), 256, 0, st>>>(A.g, C.g, rf, A.own, rc, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return C.halo ? halo_exchange_add(C.halo, rc, st, nl) : PCGB_OK;
}

// x_f += P e_c from level l+1 to l
int mg_prolong_add(pcgb_mg_t mg, int l, const double *ec, double *xf, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &A = mg->lv[(size_t)l], &C = mg->lv[(size_t)l + 1];
  if (A.any) k_mg_prolong_add_any<<<mg_node_grid(A.g), 256, 0, st>>>(A.g, C.g, A.keep, ec, xf, skip);
  else k_mg_prolong_add<<<mg_node_grid(A.g), 256, 0, st>>>(A.g, C.g, ec, xf, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return PCGB_OK;
}

// level la's ranked vector -> the global box of level la (replicated on every rank), and back
int mg_gather(pcgb_mg_t mg, const double *v, double *out, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &A = mg->lv[(size_t)mg->la];
  k_mg_gather<<<(unsigned)((A.place.glob.nfree_nodes + 255) / 256), 256, 0, st>>>(A.g, A.place, v, A.own, out, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return halo_exchange_add(mg->gather, out, st, nl);
}
int mg_scatter(pcgb_mg_t mg, const double *in, double *v, cudaStream_t st, int *nl, const int *skip) {
  const MgLevel &A = mg->lv[(size_t)mg->la];
  k_mg_scatter<<<mg_node_grid(A.g), 256, 0, st>>>(A.g, A.place, in, v, skip);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return PCGB_OK;
}

// z = M r: pre-smooth and restrict down to the coarsest level, solve there, prolong and post-smooth back up.  Across ranks
// the gathered level la is not smoothed: its vector goes into the replicated hierarchy below it and comes back out.
int mg_vcycle(pcgb_mg_t mg, const double *rin, double *zout, cudaStream_t st, int *nl, const int *skip) {
  const int L = (int)mg->lv.size();
  for (int l = 0; l + 1 < L; ++l) {
    MgLevel &A = mg->lv[(size_t)l], &C = mg->lv[(size_t)l + 1];
    if (l == mg->la) {
      PCGB_TRY(mg_gather(mg, A.b, C.b, st, nl, skip));
      continue;
    }
    PCGB_TRY(mg_smooth(mg, l, l ? A.b : rin, l ? A.x : zout, true, true, st, nl, skip));
    PCGB_TRY(mg_restrict(mg, l, A.r, C.b, st, nl, skip));
  }
  PCGB_TRY(mg_coarse_solve(mg, mg->lv.back().b, mg->lv.back().x, st, nl, skip));
  for (int l = L - 2; l >= 0; --l) {
    MgLevel &A = mg->lv[(size_t)l], &C = mg->lv[(size_t)l + 1];
    if (l == mg->la) {
      PCGB_TRY(mg_scatter(mg, C.x, A.x, st, nl, skip));
      continue;
    }
    double *x = l ? A.x : zout;
    PCGB_TRY(mg_prolong_add(mg, l, C.x, x, st, nl, skip));
    PCGB_TRY(mg_smooth(mg, l, l ? A.b : rin, x, false, false, st, nl, skip));
  }
  return PCGB_OK;
}

// z = M r of the solver's current residual, then the (rz, #non-finite z) partials into partials rows dst, dst+1
int mg_rz(pcgb_solver_t s, pcgb_mg_t mg, const double *w, double *partials, cudaStream_t st, int *nl, const int *skip) {
  PCGB_TRY(mg_vcycle(mg, s->r, mg->z, st, nl, skip));
  k_mg_rz<<<vec_grid(s->n), 256, 0, st>>>(skip, s->n, s->r, mg->z, w, partials);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  return PCGB_OK;
}

// Head of an iteration (pcg_solver.py:446-469) with the loop state c: rho = z.r, with z = Minv .* r or, with mg, z = M r
// by the V-cycle (the same launches as inside the iteration).  resume = 0 for iteration 0 (the trace record carries bb and
// r0r0), 1 after a failed verification.
int enqueue_head(pcgb_solver_t s, const PcgCtrl &c, const double *minv, const double *w, pcgb_mg_t mg, int resume, double bb,
                 double r0r0, cudaStream_t st) {
  const int grid = vec_grid(s->n);
  *s->h_ctrl = c;
  // (pinned source, stream-ordered: the next write to h_ctrl is the D2H copy of fetch_ctrl on the same stream)
  PCGB_CUDA(cudaMemcpyAsync(s->d_ctrl, s->h_ctrl, sizeof(PcgCtrl), cudaMemcpyHostToDevice, st));
  if (mg) {
    PCGB_TRY(mg_rz(s, mg, w, s->partials, st, &s->launches, &s->d_ctrl->state));
  } else {
    k_rz<<<grid, kVecBlock, 0, st>>>(s->n, s->r, minv, w, s->partials);
    PCGB_CHECK_LAUNCH();
    s->launches += 1;
  }
  PCGB_TRY(reduce_to_device(s, grid, 2, 6, st));
  k_ctrl_head<<<1, 1, 0, st>>>(s->d_ctrl, s->red + 6, resume);
  PCGB_CHECK_LAUNCH();
  s->launches += 1;
  PCGB_TRY(trace_local(s, s->partials, grid, kMaxVecGrid, 2, 4, st, &s->launches));
  return trace_step(s, resume ? TR_RESUME : TR_HEAD, bb, r0r0, st, &s->launches);
}

// ev[0..kEvPerIter): optional events at the phase boundaries of an iteration (time_kernels):
//   0 start | 1 after p-update | 2 after SpMV (interface tiles when split) | 3 after halo pack | 4 after the interior tiles |
//   5 after the p.q reduction + all-reduce + alpha | 6 after halo unpack-add | 7 after the fused update | 8 after the norms reduction
constexpr int kEvPerIter = 9;
#define PCGB_MARK(k) do { if (ev) PCGB_CUDA(cudaEventRecord(ev[k], st)); } while (0)

// the CSR product of an iteration runs interface-first: interface tiles -> halo pack -> interior tiles
inline bool split_product(pcgb_solver_t s, bool peer) {
  return peer && s->op.A && s->halo && s->halo->m > 0 && spmv_split_available(s->op.A->P);
}

// q = K p of an iteration (marks 2-4) and the partials of p.q it leaves: *src, *count.  *packed: the halo pack of q is
// enqueued.  In the multi-GPU case the partials are those of the UNASSEMBLED local product, whose rank sum equals the
// reference's weighted dot of the assembled q (p is consistent on shared dofs and K = sum of the subdomain matrices); see
// DESIGN.md.
int enqueue_product(pcgb_solver_t s, bool peer, cudaStream_t st, int *nl, cudaEvent_t *ev, const double **src, int *count,
                    bool *packed) {
  const int *skip = &s->d_ctrl->state;
  *packed = false;
  if (!s->op.A) {  // matrix-free operator: product, then a separate unweighted dot of the local product
    PCGB_TRY(s->op.apply(s->p, s->q, st, nl, skip));
    PCGB_MARK(2); PCGB_MARK(3); PCGB_MARK(4);
    const int vg = vec_grid(s->n);
    k_dot_w<<<vg, kVecBlock, 0, st>>>(s->n, s->p, s->q, nullptr, s->partials);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
    *src = s->partials; *count = vg;
    return PCGB_OK;
  }
  const CsrPlan &P = s->op.A->P;
  if (split_product(s, peer)) {   // the peer stores of the pack fly over NVLink; the unpack follows the p.q all-reduce
    PCGB_TRY(spmv_launch_part(P, 0, s->p, s->q, true, st, nl, skip));
    PCGB_MARK(2);
    PCGB_TRY(halo_pack(s->halo, s->q, st, nl));
    PCGB_MARK(3);
    PCGB_TRY(spmv_launch_part(P, 1, s->p, s->q, true, st, nl, skip));
    PCGB_MARK(4);
    *src = P.dot_partials_split; *count = spmv_split_dot_count(P); *packed = true;
    return PCGB_OK;
  }
  PCGB_TRY(spmv_launch(P, s->p, s->q, true, st, nl, skip));
  PCGB_MARK(2);
  if (peer && s->halo) { PCGB_TRY(halo_pack(s->halo, s->q, st, nl)); *packed = true; }
  PCGB_MARK(3); PCGB_MARK(4);
  // per-tile partials -> (stage) -> scalar
  *src = P.dot_partials;
  *count = P.persist ? P.grid_persist : P.ntiles;
  if (*count > 8192) {
    const int sb = (*count + 4095) / 4096;
    k_stage_reduce<<<sb, 256, 0, st>>>(P.dot_partials, *count, s->stage);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
    *src = s->stage; *count = sb;
  }
  return PCGB_OK;
}

// p.q over blocks and ranks into red[0] and alpha (mark 5), then the halo unpack-add of q (mark 6)
int pq_reduce(pcgb_solver_t s, bool peer, const double *src, int count, bool packed, cudaStream_t st, int *nl, cudaEvent_t *ev) {
  if (peer) {
    // own kernels over peer memory: the all-reduce is fused into the reduction kernel, the scalar logic follows in the same CTA
    if (s->halo && !packed) PCGB_TRY(halo_pack(s->halo, s->q, st, nl));
    // fork: the unpack-add of the interface values (waits for the neighbours' stores) runs beside the p.q all-reduce (waits
    // for the other ranks' sums); both only need the pack above, which never waits - so no order of execution can deadlock
    const bool fork = s->halo && s->halo->m > 0 && s->side != nullptr && s->fork_halo;
    if (fork) {
      PCGB_CUDA(cudaEventRecord(s->ev_fork, st));
      PCGB_CUDA(cudaStreamWaitEvent(s->side, s->ev_fork, 0));
      PCGB_TRY(halo_unpack(s->halo, s->q, s->side, nl));
      PCGB_CUDA(cudaEventRecord(s->ev_join, s->side));
    }
    k_reduce_ar<1, 1><<<1, 256, 0, st>>>(s->comm->window(), s->d_ctrl, src, count, 0, s->red, nullptr);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
    PCGB_TRY(trace_local(s, src, count, 0, 1, 0, st, nl));   // before k_update: the EBE dot partials share s->partials
    PCGB_MARK(5);
    if (fork) PCGB_CUDA(cudaStreamWaitEvent(st, s->ev_join, 0));
    else if (s->halo) PCGB_TRY(halo_unpack(s->halo, s->q, st, nl));
  } else if (!multi_rank(s)) {
    k_reduce<1, 1><<<1, 256, 0, st>>>(s->d_ctrl, src, count, 0, s->red, nullptr);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
    PCGB_MARK(5);
  } else {
    // NCCL transport: reduction, ncclAllReduce and the scalar logic are three stream operations; the halo is serial
    k_reduce<1, 0><<<1, 256, 0, st>>>(s->d_ctrl, src, count, 0, s->red, nullptr);
    PCGB_CHECK_LAUNCH();
    PCGB_TRY(trace_local(s, src, count, 0, 1, 0, st, nl));
    PCGB_TRY(allreduce_sum(s->comm, s->red, 1, st));
    k_ctrl_alpha<<<1, 1, 0, st>>>(s->d_ctrl, s->red);
    PCGB_CHECK_LAUNCH();
    *nl += 2;
    PCGB_MARK(5);
    if (s->halo) PCGB_TRY(halo_exchange_add(s->halo, s->q, st, nl));
  }
  PCGB_MARK(6);
  return PCGB_OK;
}

// pp, xx, rr, rz, #inf over blocks and ranks into red[1..6) and the control step that consumes them (mark 8)
int norms_reduce(pcgb_solver_t s, bool peer, double *resvec, cudaStream_t st, int *nl, cudaEvent_t *ev) {
  const int vg = vec_grid(s->n);
  if (peer) {
    k_reduce_ar<5, 2><<<1, 256, 0, st>>>(s->comm->window(), s->d_ctrl, s->partials, vg, kMaxVecGrid, s->red + 1, resvec);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
    PCGB_MARK(8);
    return trace_local(s, s->partials, vg, kMaxVecGrid, 5, 1, st, nl);
  }
  if (!multi_rank(s)) {
    k_reduce<5, 2><<<1, 256, 0, st>>>(s->d_ctrl, s->partials, vg, kMaxVecGrid, s->red + 1, resvec);
    PCGB_CHECK_LAUNCH();
    *nl += 1;
  } else {
    k_reduce<5, 0><<<1, 256, 0, st>>>(s->d_ctrl, s->partials, vg, kMaxVecGrid, s->red + 1, nullptr);
    PCGB_CHECK_LAUNCH();
    PCGB_TRY(trace_local(s, s->partials, vg, kMaxVecGrid, 5, 1, st, nl));
    PCGB_TRY(allreduce_sum(s->comm, s->red + 1, 5, st));
    k_ctrl_norms<<<1, 1, 0, st>>>(s->d_ctrl, s->red + 1, resvec);
    PCGB_CHECK_LAUNCH();
    *nl += 2;
  }
  PCGB_MARK(8);
  return PCGB_OK;
}

// one PCG iteration enqueued on st (pcg_solver.py:438-562); every kernel no-ops once the state is frozen.
// mg (one rank only): z = M r by a V-cycle instead of z = Minv .* r: p is updated from the z of the previous iteration
// (k_pupdate with z in place of r and no Minv), k_update runs without Minv and its z sums (rows 3, 4) are replaced by
// k_mg_rz after the V-cycle on the new r.
int enqueue_iteration(pcgb_solver_t s, const double *minv, const double *w, double *resvec, cudaStream_t st, int *nl,
                      cudaEvent_t *ev, pcgb_mg_t mg) {
  const int vg = vec_grid(s->n);
  const bool peer = peer_path(s);
  PCGB_MARK(0);
  k_pupdate<<<vg, kVecBlock, 0, st>>>(s->d_ctrl, s->n, mg ? mg->z : s->r, mg ? nullptr : minv, s->p);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  PCGB_MARK(1);
  const double *pq_src = nullptr;
  int pq_cnt = 0;
  bool packed = false;
  PCGB_TRY(enqueue_product(s, peer, st, nl, ev, &pq_src, &pq_cnt, &packed));
  PCGB_TRY(pq_reduce(s, peer, pq_src, pq_cnt, packed, st, nl, ev));
  k_update<<<vg, kVecBlock, 0, st>>>(s->d_ctrl, s->n, s->r, s->q, s->p, mg ? nullptr : minv, w, s->xown, s->xalt, s->partials);
  PCGB_CHECK_LAUNCH();
  *nl += 1;
  if (mg) PCGB_TRY(mg_rz(s, mg, w, s->partials + 3 * kMaxVecGrid, st, nl, &s->d_ctrl->state));
  PCGB_MARK(7);
  PCGB_TRY(norms_reduce(s, peer, resvec, st, nl, ev));
  return trace_step(s, TR_ITER, 0.0, 0.0, st, nl);
}
#undef PCGB_MARK

int fetch_ctrl(pcgb_solver_t s, cudaStream_t st) {
  PCGB_CUDA(cudaMemcpyAsync(s->h_ctrl, s->d_ctrl, sizeof(PcgCtrl), cudaMemcpyDeviceToHost, st));
  if (s->comm && s->comm->d_status) PCGB_CUDA(cudaMemcpyAsync(s->comm->h_status, s->comm->d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  if (s->comm && s->comm->d_status && *s->comm->h_status != 0)
    return fail(PCGB_ERR_COMM, "a peer-memory exchange timed out waiting for another rank (rank %d of %d)", s->comm->rank, s->comm->nranks);
  return PCGB_OK;
}

}  // namespace

extern "C" {

int pcgb_apply(pcgb_solver_t s, const double *d_x, double *d_y, void *stream) {
  if (!s || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_apply: null argument");
  return op_apply(s, d_x, d_y, (cudaStream_t)stream);
}

static int solve_on(pcgb_solver_t s, const double *d_b, const double *d_minv, const double *d_w, double *d_x,
                    const pcgb_options *opt, double *d_resvec, pcgb_result *res, cudaStream_t st, pcgb_mg_t mg) {
  const int64_t n = s->n;
  const int vg = vec_grid(n);
  memset(res, 0, sizeof(*res));
  s->launches = 0;
  int64_t matvecs = 0, graph_launch_kernels = 0;
  const int maxstag = opt->max_stag > 0 ? opt->max_stag : 3;
  const int64_t nglob = opt->n_global > 0 ? opt->n_global : n;
  // the loop works on the solver's own pair of x buffers (graph / kernel arguments never change between solves)
  double *const xw = s->xown;
  double *xbuf[2] = {xw, s->xalt};
  PCGB_CUDA(cudaEventRecord(s->ev_s0, st));
  if (s->trace) PCGB_CUDA(cudaMemsetAsync(s->trace, 0, sizeof(PcgTraceHdr), st));

  // ---- ||b||  (pcg_solver.py:381-384) and the initial residual (:408-418) with ONE host synchronisation:
  //      sum b*b*w -> red[7], r = b - A x0 and sum r*r*w -> red[6]
  k_dot_w<<<vg, kVecBlock, 0, st>>>(n, d_b, d_b, d_w, s->partials);
  PCGB_CHECK_LAUNCH();
  s->launches += 1;
  PCGB_TRY(reduce_to_device(s, vg, 1, 7, st));
  if (opt->x0_zero) {
    // the caller states x0 = 0: A x0 = 0 exactly, hence r = b and ||r|| = ||b|| bit for bit - no operator application
    PCGB_CUDA(cudaMemsetAsync(xw, 0, (size_t)n * sizeof(double), st));
    PCGB_CUDA(cudaMemcpyAsync(s->r, d_b, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    PCGB_CUDA(cudaMemcpyAsync(s->red + 6, s->red + 7, sizeof(double), cudaMemcpyDeviceToDevice, st));
  } else {
    PCGB_CUDA(cudaMemcpyAsync(xw, d_x, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    PCGB_TRY(true_residual_dev(s, d_b, d_w, xw, 6, st));
    ++matvecs;
  }
  if (d_resvec) {  // ResVec[0] = sqrt(red[6]) (:431), computed on the device
    k_sqrt_store<<<1, 1, 0, st>>>(s->red + 6, d_resvec);
    PCGB_CHECK_LAUNCH();
  }
  PCGB_TRY(fetch_red(s, st));
  const double n2b = std::sqrt(s->h_red[1]);
  const double normr = std::sqrt(s->h_red[0]);
  const double tolb = opt->tol * n2b;
  res->normb = n2b;
  if (n2b == 0.0) {  // :387-395 - returns the initial guess, flag 0, relres 0, iter 0
    res->flag = 0; res->relres = 0.0; res->iters = 0; res->launches = s->launches;
    return PCGB_OK;
  }
  if (!opt->fixed_iters && normr <= tolb) {  // :421-426
    res->flag = 0; res->relres = normr / n2b; res->iters = 0; res->matvecs = matvecs; res->launches = s->launches;
    return PCGB_OK;
  }
  // ---- loop state (:399-406)
  int64_t mm = nglob / 50;
  if (mm > 5) mm = 5;
  if (nglob - opt->maxiter < mm) mm = nglob - opt->maxiter;
  const int64_t maxmsteps = mm;
  PcgCtrl c;
  memset(&c, 0, sizeof(c));
  c.rho = 1.0; c.rho_prev = 1.0; c.alpha = 0.0; c.beta = 0.0;
  c.normr = normr; c.normr_act = normr; c.normrmin = normr;
  c.tolb = tolb; c.n2b = n2b; c.eps = 2.220446049250313e-16;
  c.state = ST_RUN; c.flag = 1; c.iter = 0; c.stag = 0; c.moresteps = 0; c.imin = 0; c.xcur = 0; c.xmin = 0;
  c.alias = 1;   // MP_XMin = MP_X (:379-380): the same array until the first improvement is recorded
  c.maxiter = opt->maxiter; c.maxstag = maxstag; c.fixed_iters = opt->fixed_iters ? 1 : 0;
  PCGB_TRY(enqueue_head(s, c, d_minv, d_w, mg, 0, s->h_red[1], s->h_red[0], st));

  int batch = opt->check_every > 0 ? opt->check_every : 16;
  if (batch > opt->maxiter) batch = opt->maxiter;
  const bool want_graph = opt->use_graph != 0 && !opt->time_kernels;
  size_t ktimed = 0;           // iterations whose SpMV launches carry event brackets
  PCGB_CUDA(cudaEventRecord(s->ev_l0, st));
  int flag = 1;
  int too_small = 0;

  for (;;) {
    // ---- enqueue `batch` iterations
    if (want_graph && batch > 1) {
      const bool peer = peer_path(s);
      const GraphKey key{d_minv, d_w, d_resvec, batch, peer, split_product(s, peer), s->trace, s->trace_cap, mg};
      if (!s->gexec || !(s->gkey == key)) {
        if (s->gexec) { cudaGraphExecDestroy(s->gexec); s->gexec = nullptr; }
        cudaGraph_t graph = nullptr;
        PCGB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        int rc = PCGB_OK, nl = 0;
        for (int k = 0; k < batch && rc == PCGB_OK; ++k) rc = enqueue_iteration(s, d_minv, d_w, d_resvec, st, &nl, nullptr, mg);
        cudaError_t ce = cudaStreamEndCapture(st, &graph);
        if (rc != PCGB_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
        PCGB_CUDA(ce);
        PCGB_CUDA(cudaGraphInstantiate(&s->gexec, graph, 0));
        cudaGraphDestroy(graph);
        s->gkey = key;
        s->launches_per_iter = nl / batch;
      }
      PCGB_CUDA(cudaGraphLaunch(s->gexec, st));
      graph_launch_kernels += (int64_t)s->launches_per_iter * batch;
    } else {
      for (int k = 0; k < batch; ++k) {
        int nl = 0;
        cudaEvent_t *ev = nullptr;
        if (opt->time_kernels && ktimed < 1024) {
          while (s->ev_k.size() < (size_t)kEvPerIter * (ktimed + 1)) { cudaEvent_t e; PCGB_CUDA(cudaEventCreate(&e)); s->ev_k.push_back(e); }
          ev = &s->ev_k[(size_t)kEvPerIter * ktimed]; ++ktimed;
        }
        PCGB_TRY(enqueue_iteration(s, d_minv, d_w, d_resvec, st, &nl, ev, mg));
        s->launches += nl;
      }
    }
    PCGB_TRY(fetch_ctrl(s, st));
    c = *s->h_ctrl;
    if (c.state == ST_RUN) continue;
    if (c.state == ST_TRIGGER) {
      // ---- verification with the true residual (:527-552)
      double normr_act = 0.0;
      PCGB_TRY(true_residual(s, d_b, d_w, xbuf[c.xcur], &normr_act, st));
      const double rr_act = s->h_red[0];
      PCGB_TRY(trace_local(s, s->partials, vg, kMaxVecGrid, 1, 3, st, &s->launches));
      ++matvecs;
      c.normr_act = normr_act;
      if (normr_act <= tolb) {                                  // :540-543
        flag = 0; c.flag = 0;
        PCGB_TRY(trace_host(s, TR_VERIFY, c, rr_act, true, nullptr, st));
        break;
      }
      if (c.stag >= maxstag && c.moresteps == 0) c.stag = 0;   // :545
      c.moresteps += 1;                                         // :546
      if (c.moresteps >= maxmsteps) {                           // :548-552 (the reference raises here)
        too_small = 1; flag = 3; c.flag = 3;
        PCGB_TRY(trace_host(s, TR_VERIFY, c, rr_act, true, nullptr, st));
        break;
      }
      if (normr_act < c.normrmin) { c.normrmin = normr_act; c.xmin = c.xcur; c.imin = c.iter; c.alias = 0; }  // :555-558
      if (c.stag >= maxstag) {                                  // :560-562
        flag = 3; c.flag = 3;
        PCGB_TRY(trace_host(s, TR_VERIFY, c, rr_act, true, nullptr, st));
        break;
      }
      // continue with the replaced residual: head of the next iteration
      c.state = ST_RUN;
      PCGB_TRY(trace_host(s, TR_VERIFY, c, rr_act, true, nullptr, st));
      PCGB_TRY(enqueue_head(s, c, d_minv, d_w, mg, 1, 0.0, 0.0, st));
      batch = 1;  // MoreSteps > 0: every further iteration is verified (:527)
      continue;
    }
    flag = c.flag;  // ST_BREAK (2,3,4) or ST_EXHAUSTED (1)
    break;
  }
  PCGB_CUDA(cudaEventRecord(s->ev_l1, st));
  if (s->snapshot) {  // the loop's vectors before the finalisation overwrites r and q
    const double *src[5] = {s->r, s->p, s->q, xbuf[0], xbuf[1]};
    for (int k = 0; k < 5; ++k)
      PCGB_CUDA(cudaMemcpyAsync(s->snapshot + (size_t)k * n, src[k], (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  }

  // ---- finalisation (:566-584)
  const int i = c.iter;
  int iter_out;
  double relres;
  int xout;
  if (flag == 0) {
    relres = c.normr_act / n2b;
    iter_out = i;
    xout = c.xcur;
    PCGB_TRY(trace_host(s, TR_FINAL, c, 0.0, false, s->snapshot ? s->snapshot + 5 * n : nullptr, st));
  } else {
    // XMin is the current iterate while it is still aliased to X (no improvement recorded yet): c.xmin == c.xcur then
    double normr_min = 0.0;
    PCGB_TRY(true_residual(s, d_b, d_w, xbuf[c.xmin], &normr_min, st));
    if (s->trace) {
      PCGB_TRY(trace_local(s, s->partials, vg, kMaxVecGrid, 1, 3, st, &s->launches));
      PCGB_TRY(trace_host(s, TR_FINAL, c, s->h_red[0], true, s->snapshot ? s->snapshot + 5 * n : nullptr, st));
    }
    ++matvecs;
    if (normr_min < c.normr_act) { iter_out = c.imin; relres = normr_min / n2b; }
    else { iter_out = i; relres = c.normr_act / n2b; }
    xout = c.xmin;  // the reference exports XMin on this path in both cases (:569, :598)
  }
  iter_out += 1;  // :584
  PCGB_CUDA(cudaMemcpyAsync(d_x, xbuf[xout], (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  PCGB_CUDA(cudaEventRecord(s->ev_s1, st));
  PCGB_CUDA(cudaEventSynchronize(s->ev_s1));
  {
    float ms = 0.f;
    PCGB_CUDA(cudaEventElapsedTime(&ms, s->ev_l0, s->ev_l1));
    res->loop_ms = ms;
    res->loop_iters = c.iter + 1;
    PCGB_CUDA(cudaEventElapsedTime(&ms, s->ev_s0, s->ev_l0));
    res->setup_ms = ms;
    PCGB_CUDA(cudaEventElapsedTime(&ms, s->ev_l1, s->ev_s1));
    res->final_ms = ms;
    // phase sums over the bracketed iterations: p-update | SpMV | halo pack | p.q reduce + all-reduce | halo unpack |
    // fused update | norms reduce + all-reduce   (phase_ms[7] = their total)
    double tot = 0.0;
    static const int seg[7][2] = {{0, 1}, {1, 2}, {2, 3}, {4, 5}, {5, 6}, {6, 7}, {7, 8}};
    for (size_t k = 0; k < ktimed; ++k) {
      const cudaEvent_t *e = &s->ev_k[(size_t)kEvPerIter * k];
      float t = 0.f;
      for (int ph = 0; ph < 7; ++ph) {
        PCGB_CUDA(cudaEventElapsedTime(&t, e[seg[ph][0]], e[seg[ph][1]]));
        res->phase_ms[ph] += t;
      }
      PCGB_CUDA(cudaEventElapsedTime(&t, e[3], e[4]));   // interior tiles of a split SpMV (zero-length otherwise)
      res->phase_ms[1] += t;
      PCGB_CUDA(cudaEventElapsedTime(&t, e[0], e[8]));
      res->phase_ms[7] += t;
    }
    tot = res->phase_ms[1];
    res->spmv_ms = tot; res->spmv_timed = (int64_t)ktimed;
  }
  res->flag = flag; res->iters = iter_out; res->relres = relres; res->imin = c.imin; res->stag = c.stag;
  res->moresteps = c.moresteps; res->too_small_tol = too_small;
  // matvecs inside the loop = iterations started
  res->matvecs = matvecs + (int64_t)(c.iter + 1);
  res->launches = s->launches + graph_launch_kernels;
  return PCGB_OK;
}

// order the solver's own stream after the caller's stream, run, and order the caller's stream after us
static int solve_fenced(pcgb_solver_t s, pcgb_mg_t mg, const double *d_b, const double *d_minv, const double *d_w, double *d_x,
                        const pcgb_options *opt, double *d_resvec, pcgb_result *res, void *stream) {
  cudaStream_t user = (cudaStream_t)stream;
  PCGB_CUDA(cudaEventRecord(s->ev_in, user));
  PCGB_CUDA(cudaStreamWaitEvent(s->own, s->ev_in, 0));
  PCGB_TRY(solve_on(s, d_b, d_minv, d_w, d_x, opt, d_resvec, res, s->own, mg));
  PCGB_CUDA(cudaEventRecord(s->ev_out, s->own));
  PCGB_CUDA(cudaStreamWaitEvent(user, s->ev_out, 0));
  return PCGB_OK;
}

int pcgb_solve(pcgb_solver_t s, const double *d_b, const double *d_minv, const double *d_w, double *d_x,
               const pcgb_options *opt, double *d_resvec, pcgb_result *res, void *stream) {
  if (!s || !d_b || !d_x || !opt || !res) return fail(PCGB_ERR_ARG, "pcgb_solve: null argument");
  if (opt->maxiter <= 0) return fail(PCGB_ERR_ARG, "pcgb_solve: maxiter must be positive");
  return solve_fenced(s, nullptr, d_b, d_minv, d_w, d_x, opt, d_resvec, res, stream);
}

// ------------------------------------------------------------------------------------ geometric multigrid (hex boxes)
int pcgb_mg_destroy(pcgb_mg_t mg) {
  if (!mg) return PCGB_OK;
  // The solver's cached graph of MG iterations holds this handle's buffers and coefficients as kernel arguments, and its key
  // knows the handle only by address, which a later pcgb_mg_create may receive again: drop the graph with the handle.
  pcgb_solver_t s = mg->s;
  if (s && s->gexec && s->gkey.mg == mg) {
    cudaGraphExecDestroy(s->gexec);
    s->gexec = nullptr;
    s->gkey = {};
  }
  if (s) s->mgs.erase(std::remove(s->mgs.begin(), s->mgs.end(), mg), s->mgs.end());
  for (size_t l = 0; l < mg->lv.size(); ++l) {
    MgLevel &L = mg->lv[l];
    if (L.op == MgOp::Csr) free_plan(L.P);
    cudaFree(L.rowptr); cudaFree(L.col); cudaFree(L.val); cudaFree(L.dinv); cudaFree(L.own);
    if (l > 0) { cudaFree(L.b); cudaFree(L.x); }
    cudaFree(L.r); cudaFree(L.d); cudaFree(L.q);
  }
  cudaFree(mg->chol); cudaFree(mg->z); cudaFree(mg->partials); cudaFree(mg->red); cudaFree(mg->d_bad); cudaFree(mg->kel);
  if (mg->h_red) cudaFreeHost(mg->h_red);
  delete mg;
  return PCGB_OK;
}

namespace {
// Stiffness matrix of level L's box as device CSR (int64 row offsets; the caller frees them): k_hex_count, a host scan,
// k_hex_fill with Ck = ck, or (kel != NULL) k_hex_fill_var from the level's per-element matrices
int mg_hex_csr(const HexGeom &g, const double *ke_host, double ck, int64_t **rp, int **col, double **val, int64_t *nnz,
               const double *kel = nullptr) {
  const int64_t n = 3 * g.nfree_nodes;
  std::vector<int64_t> cnt((size_t)n + 1);
  PCGB_CUDA(cudaMalloc(rp, (size_t)(n + 1) * sizeof(int64_t)));
  k_hex_count<<<(unsigned)((g.nfree_nodes + 255) / 256), 256>>>(g, *rp);
  PCGB_CHECK_LAUNCH();
  PCGB_CUDA(cudaMemcpy(cnt.data(), *rp, cnt.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
  for (size_t i = 1; i < cnt.size(); ++i) cnt[i] += cnt[i - 1];
  *nnz = cnt.back();
  PCGB_CUDA(cudaMemcpy(*rp, cnt.data(), cnt.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
  PCGB_CUDA(cudaMalloc(col, (size_t)*nnz * sizeof(int)));
  PCGB_CUDA(cudaMalloc(val, (size_t)*nnz * sizeof(double)));
  if (kel) {
    k_hex_fill_var<true><<<(unsigned)((g.nfree_nodes * 32 + 255) / 256), 256>>>(g, nullptr, kel, *rp, *col, *val);
  } else {
    PCGB_CUDA(cudaMemcpyToSymbol(c_hex_ke, ke_host, 24 * 24 * sizeof(double)));
    k_hex_fill<<<(unsigned)((g.nfree_nodes * 32 + 255) / 256), 256>>>(g, ck, *rp, *col, *val);
  }
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

// The index-free operator of box g: Ke (row-major 24x24) and its diagonal by value, Ck uniform or (d_ck) per element
HexOp hexop_of(const HexGeom &g, const double *ke_host, double ck, const double *d_ck) {
  HexOp H;
  H.s = hexop_shape(g);
  std::memcpy(H.ke.k, ke_host, sizeof(H.ke.k));
  for (int a = 0; a < 24; ++a) H.kd.k[a] = ke_host[a * 24 + a];
  H.ck = d_ck ? 0.0 : ck;
  H.d_ck = d_ck;
  H.n = 3 * g.nfree_nodes;
  H.bytes = 16 * H.n + (d_ck ? 8 * (int64_t)g.nx * g.ny * g.nz : 0);
  return H;
}

// Field hierarchies: the Galerkin element matrices of level l (l >= 1) from those of level l - 1 (level 1: from the fine
// Ck field and Ke), into mg->kel; the level below's matrices are freed once these exist, so at most two levels' are held.
int mg_galerkin_level(pcgb_mg_t mg, int l, const double *ke_host) {
  const HexGeom &F = mg->lv[(size_t)l - 1].g, &C = mg->lv[(size_t)l].g;
  const int64_t nce = (int64_t)C.nx * C.ny * C.nz;
  const int64_t prev = l > 1 ? 576 * sizeof(double) * (int64_t)F.nx * F.ny * F.nz : 0;
  double *kc = nullptr;
  PCGB_CUDA(cudaMalloc(&kc, (size_t)nce * 576 * sizeof(double)));
  mg->kel_peak = std::max(mg->kel_peak, prev + nce * 576 * (int64_t)sizeof(double));
  if (l == 1) PCGB_CUDA(cudaMemcpyToSymbol(c_hex_ke, ke_host, 24 * 24 * sizeof(double)));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, 0);
  const MgLevel &FL = mg->lv[(size_t)l - 1];
  if (FL.any)
    k_mg_galerkin_any<<<(unsigned)nce, kMgGalerkinThreads>>>(C.nx, C.ny, F.nx, F.ny, F.nz, FL.keep, mg->ck_fine, l > 1 ? mg->kel : nullptr, kc);
  else
    k_mg_galerkin<<<(unsigned)nce, kMgGalerkinThreads>>>(C.nx, C.ny, F.nx, F.ny, mg->ck_fine, l > 1 ? mg->kel : nullptr, kc);
  const cudaError_t le = cudaGetLastError();
  cudaEventRecord(e1, 0);
  const cudaError_t se = cudaEventSynchronize(e1);
  float ms = 0.0f;
  if (le == cudaSuccess && se == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(mg->kel);
  mg->kel = kc;
  if (le != cudaSuccess || se != cudaSuccess) return fail(PCGB_ERR_CUDA, "pcgb_mg_create_field: Galerkin kernel failed: %s",
                                                          cudaGetErrorString(le != cudaSuccess ? le : se));
  mg->galerkin_ms += ms;
  return PCGB_OK;
}

// Field hierarchies across ranks: the rank's element matrices of level la (mg->kel) into a zeroed array of the whole global
// box of la, completed by one exchange-add over mg->kel_gather; it replaces mg->kel as the matrices of level la + 1.
int mg_gather_elements(pcgb_mg_t mg) {
  const MgLevel &A = mg->lv[(size_t)mg->la];
  const int64_t nel = (int64_t)A.g.nx * A.g.ny * A.g.nz;
  const int64_t nge = (int64_t)A.place.glob.nx * A.place.glob.ny * A.place.glob.nz;
  double *kg = nullptr;
  PCGB_CUDA(cudaMalloc(&kg, (size_t)nge * 576 * sizeof(double)));
  mg->kel_peak = std::max(mg->kel_peak, (nel + nge) * 576 * (int64_t)sizeof(double));
  cudaError_t e = cudaMemset(kg, 0, (size_t)nge * 576 * sizeof(double));
  if (e == cudaSuccess) {
    k_mg_gather_elements<<<(unsigned)std::min<int64_t>((576 * nel + 255) / 256, 65536), 256>>>(A.g, A.place, mg->kel, kg);
    e = cudaGetLastError();
  }
  cudaFree(mg->kel);   // stream-ordered after the gather on the legacy stream
  mg->kel = kg;
  if (e != cudaSuccess) return fail(PCGB_ERR_CUDA, "pcgb_mg_create_ranks_field: element gather failed: %s", cudaGetErrorString(e));
  return halo_exchange_add(mg->kel_gather, kg, 0);
}

// largest slab of level-1 element matrices a rap set-up holds (at least one pair of element layers)
constexpr int64_t kMgRapSlabBytes = int64_t(1) << 30;

// Rap hierarchies: level 1 applied by k_mg_rap1, and level 2's Galerkin element matrices (into mg->kel) built without holding
// level 1's.  In ascending z, a slab of level-1 element layers (an even number, at most kMgRapSlabBytes, at least 2) is built
// from the fine field with k_mg_galerkin, its diagonal entries are added into level 1's diagonal (L1.r, zeroed), and each
// finished pair of layers gives one layer of level-2 matrices, k_mg_galerkin from the slab.  Every level-1 matrix is the
// field hierarchy's bit for bit, so are the level-2 matrices and the diagonal.  Across ranks the boxes are the rank's and the
// field its slice: L1.r is the rank's part of the diagonal, which mg_build exchange-adds like every ranked level's.
int mg_rap_level1(pcgb_mg_t mg, const double *ke_host) {
  MgLevel &L1 = mg->lv[1];
  const HexGeom &G0 = mg->lv[0].g, &G1 = L1.g, &G2 = mg->lv[2].g;
  const int64_t layer = (int64_t)G1.nx * G1.ny, layer2 = (int64_t)G2.nx * G2.ny;
  const int64_t layer_bytes = 576 * (int64_t)sizeof(double) * layer;
  const int per = (int)std::min<int64_t>(G1.nz, std::max<int64_t>(2, (kMgRapSlabBytes / layer_bytes) & ~int64_t(1)));
  const int64_t bytes2 = 576 * (int64_t)sizeof(double) * layer2 * G2.nz;
  L1.R = rap_shape(G0, G1);
  std::memcpy(L1.ke.k, ke_host, sizeof(L1.ke.k));
  L1.ck_fine = mg->ck_fine;
  PCGB_CUDA(cudaFuncSetAttribute(k_mg_rap1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRapSmem));
  PCGB_CUDA(cudaMemcpyToSymbol(c_hex_ke, ke_host, 24 * 24 * sizeof(double)));
  PCGB_CUDA(cudaMemset(L1.r, 0, (size_t)L1.n * sizeof(double)));
  PCGB_CUDA(cudaMalloc(&mg->kel, (size_t)bytes2));   // freed by the build or by pcgb_mg_destroy
  double *slab = nullptr;
  PCGB_CUDA(cudaMalloc(&slab, (size_t)(per * layer_bytes)));
  mg->kel_peak = std::max(mg->kel_peak, bytes2 + per * layer_bytes);
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaError_t err = cudaSuccess;
  for (int z0 = 0; z0 < G1.nz && err == cudaSuccess; z0 += per) {
    const int k = std::min(per, G1.nz - z0);   // even: G1.nz and per are
    cudaEventRecord(e0, 0);
    k_mg_galerkin<<<(unsigned)(k * layer), kMgGalerkinThreads>>>(G1.nx, G1.ny, G0.nx, G0.ny, mg->ck_fine, nullptr, slab, z0 * layer, 0);
    k_mg_galerkin<<<(unsigned)(k / 2 * layer2), kMgGalerkinThreads>>>(G2.nx, G2.ny, G1.nx, G1.ny, nullptr, slab,
                                                                      mg->kel + 576 * (z0 / 2) * layer2, z0 / 2 * layer2, z0 * layer);
    cudaEventRecord(e1, 0);
    const int64_t nodes = (int64_t)G1.nxf * (G1.ny + 1) * (k + 1);
    k_mg_rap_diag<<<(unsigned)((nodes + 255) / 256), 256>>>(G1, z0, z0 + k, slab, L1.r);
    err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaEventSynchronize(e1);
    float ms = 0.0f;
    if (err == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
    mg->galerkin_ms += ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  cudaFree(slab);
  return err == cudaSuccess ? PCGB_OK
                            : fail(PCGB_ERR_CUDA, "pcgb_mg_create_field_rap: level-1 set-up failed: %s", cudaGetErrorString(err));
}

// largest eigenvalue of the symmetric tridiagonal matrix (diagonal a, off-diagonal b) by bisection on the Sturm count
double tridiag_max_eig(const std::vector<double> &a, const std::vector<double> &b) {
  const size_t k = a.size();
  double lo = 0.0, hi = 0.0;
  for (size_t i = 0; i < k; ++i) {
    const double r = (i > 0 ? std::fabs(b[i - 1]) : 0.0) + (i + 1 < k ? std::fabs(b[i]) : 0.0);
    if (!std::isfinite(a[i]) || !std::isfinite(r)) return NAN;
    lo = i ? std::min(lo, a[i] - r) : a[i] - r;
    hi = i ? std::max(hi, a[i] + r) : a[i] + r;
  }
  for (int it = 0; it < 200 && lo < hi; ++it) {
    const double mid = 0.5 * (lo + hi);
    if (mid <= lo || mid >= hi) break;
    size_t below = 0;   // eigenvalues < mid: sign changes of the LDL^T pivots of T - mid I
    double d = 1.0;
    for (size_t i = 0; i < k; ++i) {
      d = a[i] - mid - (i ? b[i - 1] * b[i - 1] / d : 0.0);
      if (d == 0.0) d = -1e-300;
      if (d < 0.0) ++below;
    }
    if (below == k) hi = mid; else lo = mid;
  }
  return hi;
}

// largest eigenvalue of D^-1 A on level l: kMgLanczosSteps Lanczos steps (D inner product) from a fixed start vector, the
// largest eigenvalue of their tridiagonal matrix.  Then the Chebyshev coefficients of the level.  On a ranked level the
// vectors stay consistent (mg_op exchanges), the inner products sum the owned dofs and are all-reduced (one value per
// step), and the start vector is indexed by the global free dof, so lambda is the same number on every rank.
int mg_estimate(pcgb_mg_t mg, int l) {
  MgLevel &L = mg->lv[(size_t)l];
  const int grid = vec_grid(L.n);
  const bool ranked = l <= mg->la;
  int nl = 0;
  auto fetch = [&](double *out) -> int {
    k_reduce<1, 0><<<1, 256>>>(nullptr, mg->partials, grid, kMaxVecGrid, mg->red, nullptr);
    PCGB_CHECK_LAUNCH();
    if (ranked) PCGB_TRY(allreduce_sum(mg->s->comm, mg->red, 1, 0));
    PCGB_CUDA(cudaMemcpy(mg->h_red, mg->red, sizeof(double), cudaMemcpyDeviceToHost));
    *out = mg->h_red[0];
    return PCGB_OK;
  };
  PCGB_CUDA(cudaMemset(L.d, 0, (size_t)L.n * sizeof(double)));
  k_mg_lanczos_start<<<grid, 256>>>(L.g, L.place, L.q);
  k_mg_lanczos_w<<<grid, 256>>>(L.n, L.q, nullptr, nullptr, L.dinv, L.own, 0.0, 0.0, 0, L.r, mg->partials);
  PCGB_CHECK_LAUNCH();
  double bb = 0.0;
  PCGB_TRY(fetch(&bb));
  double beta = std::sqrt(bb);
  k_mg_lanczos_next<<<grid, 256>>>(L.n, 1.0 / beta, L.d, L.r);   // v1 = start / |start|_D, v0 = 0
  PCGB_CHECK_LAUNCH();
  std::vector<double> al, be;
  beta = 0.0;
  for (int it = 0; it < kMgLanczosSteps; ++it) {
    PCGB_TRY(mg_op(mg, l, L.d, L.q, 0, &nl, nullptr));
    k_dot_w<<<grid, kVecBlock>>>(L.n, L.d, L.q, L.own, mg->partials);
    PCGB_CHECK_LAUNCH();
    double alpha = 0.0;
    PCGB_TRY(fetch(&alpha));
    al.push_back(alpha);
    if (it + 1 == kMgLanczosSteps) break;
    k_mg_lanczos_w<<<grid, 256>>>(L.n, L.q, L.d, L.r, L.dinv, L.own, alpha, beta, 1, L.r, mg->partials);
    PCGB_CHECK_LAUNCH();
    PCGB_TRY(fetch(&bb));
    beta = std::sqrt(bb);
    if (!(beta > 0.0) || !std::isfinite(beta)) {   // invariant subspace (or a non-finite Minv)
      if (!std::isfinite(beta)) al.back() = NAN;
      break;
    }
    be.push_back(beta);
    k_mg_lanczos_next<<<grid, 256>>>(L.n, 1.0 / beta, L.d, L.r);
    PCGB_CHECK_LAUNCH();
  }
  L.lambda = tridiag_max_eig(al, be);
  // Chebyshev on [lo, 1.1] * lambda: theta = centre, delta = half width, sigma = theta / delta
  const double a = mg->lo * L.lambda, b = 1.1 * L.lambda;
  const double theta = 0.5 * (b + a), delta = 0.5 * (b - a), sigma = theta / delta;
  double rho = 1.0 / sigma;
  L.inv_theta = 1.0 / theta;
  for (int j = 1; j < mg->degree; ++j) {
    const double rn = 1.0 / (2.0 * sigma - rho);
    L.c1.push_back(rn * rho);
    L.c2.push_back(2.0 * rn / delta);
    rho = rn;
  }
  return PCGB_OK;
}

// whole boxes below geo.back(): halve every ne while all are even and the halves stay >= 2
void mg_whole_box_levels(std::vector<HexGeom> &geo) {
  for (;;) {
    const HexGeom g = geo.back();
    if (g.nx % 2 || g.ny % 2 || g.nz % 2 || g.nx < 4 || g.ny < 4 || g.nz < 4) break;
    pcgb_hex_box cb{};
    const int ne[3] = {g.nx / 2, g.ny / 2, g.nz / 2};
    for (int a = 0; a < 3; ++a) { cb.ne[a] = ne[a]; cb.ng[a] = ne[a]; cb.e0[a] = 0; }
    geo.push_back(hex_geom(&cb));
  }
}

// whole boxes below geo.back() under the rule of pcgb_mg_create_any: every axis with ne >= 3 becomes (ne + 1) / 2 elements,
// the others are kept, while some axis has ne >= 3.  keep[l] is the kept-axis mask from level l to l + 1 and any[l] whether
// that coarsening leaves the even rule (an axis kept or odd).  Stops past max_levels (the caller refuses that depth).
void mg_any_box_levels(std::vector<HexGeom> &geo, std::vector<int> &keep, std::vector<char> &any, size_t max_levels) {
  while (geo.size() <= max_levels) {
    const HexGeom g = geo.back();
    const int ne[3] = {g.nx, g.ny, g.nz};
    if (ne[0] <= 2 && ne[1] <= 2 && ne[2] <= 2) break;
    pcgb_hex_box cb{};
    int k = 0;
    bool odd = false;
    for (int a = 0; a < 3; ++a) {
      if (ne[a] <= 2) k |= 1 << a;
      odd = odd || (ne[a] > 2 && ne[a] % 2);
      cb.ne[a] = ne[a] <= 2 ? ne[a] : (ne[a] + 1) / 2;
      cb.ng[a] = cb.ne[a];
      cb.e0[a] = 0;
    }
    keep.push_back(k);
    any.push_back(k != 0 || odd);
    geo.push_back(hex_geom(&cb));
  }
}

// largest global box a multi-rank hierarchy gathers onto every rank
constexpr int64_t kMgMaxGathered = 1 << 17;
// most elements of that box whose matrices a multi-rank field hierarchy gathers (4608 bytes each, and a plan of
// (ranks - 1) * 576 entries per element)
constexpr int64_t kMgMaxGatheredElements = 4096;

// Builds the levels whose geometry (g, place, glev) and halos the caller has set in mg->lv.  coarse: what the smoothed
// coarse levels apply (Rap: level 1, with CSR matrices below it).  own: ownership weights of the ranked levels 0 .. la
// (copied).
int mg_build(pcgb_mg_t mg, MgOp coarse, const double *ke_host, double E, double h, const double *d_minv_fine,
             const double *const *own) {
  const int nlev = (int)mg->lv.size();
  auto alloc = [&](double **p, int64_t n) -> cudaError_t {
    mg->bytes += 8 * n;
    return cudaMalloc(p, (size_t)std::max<int64_t>(n, 1) * sizeof(double));
  };
  // set-up runs on the legacy stream, which does not wait for non-blocking streams: finish whatever work of the caller may
  // still be writing d_minv_fine (or the operator's arrays) before the first read
  PCGB_CUDA(cudaDeviceSynchronize());
  PCGB_CUDA(cudaMallocHost(&mg->h_red, 4 * sizeof(double)));
  PCGB_CUDA(cudaMalloc(&mg->partials, kMaxVecGrid * sizeof(double)));
  PCGB_CUDA(cudaMalloc(&mg->red, 4 * sizeof(double)));
  PCGB_CUDA(cudaMalloc(&mg->d_bad, sizeof(int)));
  PCGB_CUDA(cudaMemset(mg->d_bad, 0, sizeof(int)));
  for (int l = 0; l < nlev; ++l) {
    MgLevel &L = mg->lv[(size_t)l];
    L.n = 3 * L.g.nfree_nodes;
    const double ck = E * h * (double)(1ll << L.glev);
    L.op = l == 0 ? MgOp::Fine : l == mg->la || l == nlev - 1 ? MgOp::None : coarse == MgOp::Rap && l > 1 ? MgOp::Csr : coarse;
    if (l == 0) {
      PCGB_CUDA(alloc(&mg->z, L.n));
    } else {
      PCGB_CUDA(alloc(&L.b, L.n));
      PCGB_CUDA(alloc(&L.x, L.n));
    }
    if (l <= mg->la) {
      PCGB_CUDA(alloc(&L.own, L.n));
      PCGB_CUDA(cudaMemcpy(L.own, own[l], (size_t)L.n * sizeof(double), cudaMemcpyDeviceToDevice));
      if (l == mg->la) {   // gathered: no operator, no smoother
        if (mg->ck_fine) {   // field: the rank's Galerkin element matrices, gathered into level la + 1's global box
          // (rap with la = 2: level 2's matrices are already in mg->kel, from mg_rap_level1)
          if (!(coarse == MgOp::Rap && l <= 2)) PCGB_TRY(mg_galerkin_level(mg, l, ke_host));
          PCGB_TRY(mg_gather_elements(mg));
        }
        continue;
      }
    }
    // field: the level's Galerkin element matrices (level la + 1, the global box of la, holds the gathered ones)
    // (rap: levels 1 and 2 come from mg_rap_level1)
    if (mg->ck_fine && l > 0 && l != mg->la + 1 && !(coarse == MgOp::Rap && l <= 2)) PCGB_TRY(mg_galerkin_level(mg, l, ke_host));
    if (l == nlev - 1) {   // coarsest: dense Cholesky factor of its matrix
      int64_t *rp = nullptr, nnz = 0;
      int *col = nullptr;
      double *val = nullptr;
      int rc = mg_hex_csr(L.g, ke_host, ck, &rp, &col, &val, &nnz, mg->kel);
      mg->nc = (int)L.n;
      if (rc == PCGB_OK && alloc(&mg->chol, L.n * L.n) == cudaSuccess && cudaMemset(mg->chol, 0, (size_t)(L.n * L.n) * sizeof(double)) == cudaSuccess) {
        k_mg_densify<<<(unsigned)((L.n + 255) / 256), 256>>>(L.n, rp, col, val, mg->chol);
        k_mg_chol_factor<<<1, kMgCholThreads>>>(mg->nc, mg->chol, mg->d_bad);
        if (cudaGetLastError() != cudaSuccess) rc = fail(PCGB_ERR_CUDA, "pcgb_mg_create: coarse factorisation launch failed");
      } else if (rc == PCGB_OK) {
        rc = fail(PCGB_ERR_CUDA, "pcgb_mg_create: coarse matrix allocation failed");
      }
      cudaDeviceSynchronize();
      cudaFree(rp); cudaFree(col); cudaFree(val);
      cudaFree(mg->kel);
      mg->kel = nullptr;
      PCGB_TRY(rc);
      int bad = 0;
      PCGB_CUDA(cudaMemcpy(&bad, mg->d_bad, sizeof(int), cudaMemcpyDeviceToHost));
      if (bad) return fail(PCGB_ERR_ARG, "pcgb_mg_create: the coarsest matrix is not positive definite");
      break;
    }
    PCGB_CUDA(alloc(&L.r, L.n));
    PCGB_CUDA(alloc(&L.d, L.n));
    PCGB_CUDA(alloc(&L.q, L.n));
    PCGB_CUDA(alloc(&L.dinv, L.n));
    if (l == 0) {   // D^-1 is the caller's Minv
      PCGB_CUDA(cudaMemcpy(L.dinv, d_minv_fine, (size_t)L.n * sizeof(double), cudaMemcpyDeviceToDevice));
    } else {
      // the level's operator, and the rank's part of its diagonal into L.r
      if (L.op == MgOp::Rap) {
        PCGB_TRY(mg_rap_level1(mg, ke_host));
      } else if (L.op == MgOp::Hex) {
        L.H = hexop_of(L.g, ke_host, ck, nullptr);
        PCGB_TRY(hexop_diag(L.H, L.r, 0));
      } else {
        int64_t *rp = nullptr, nnz = 0;
        const int rc = mg_hex_csr(L.g, ke_host, ck, &rp, &L.col, &L.val, &nnz, mg->kel);
        L.rowptr = rp;
        PCGB_TRY(rc);
        mg->bytes += 12 * nnz + 8 * (L.n + 1);
        L.P.nrows = L.n; L.P.ncols = L.n; L.P.nnz = nnz; L.P.rowptr = rp; L.P.rp64 = true; L.P.col = L.col; L.P.val = L.val;
        if (nnz < INT32_MAX) {   // int32 row offsets, as the fine hex matrices use below 2^31 non-zeros
          std::vector<int64_t> r64((size_t)L.n + 1);
          PCGB_CUDA(cudaMemcpy(r64.data(), rp, r64.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
          std::vector<int32_t> r32(r64.begin(), r64.end());
          int32_t *rp32 = nullptr;
          PCGB_CUDA(upload(&rp32, r32));
          cudaFree(rp);
          L.rowptr = rp32; L.P.rowptr = rp32; L.P.rp64 = false;
          mg->bytes -= 4 * (L.n + 1);
        }
        PCGB_TRY(L.P.rp64 ? build_plan_t<int64_t>(L.P, 0) : build_plan_t<int32_t>(L.P, 0));
        PCGB_TRY(csr_diag_compute(L.P, L.r, 0));
      }
      if (L.halo) PCGB_TRY(halo_exchange_add(L.halo, L.r, 0));   // assembled diagonal of a ranked level
      k_reciprocal<<<vec_grid(L.n), 256>>>(L.n, L.r, L.dinv);
      PCGB_CHECK_LAUNCH();
    }
    PCGB_TRY(mg_estimate(mg, l));
  }
  PCGB_CUDA(cudaDeviceSynchronize());
  return PCGB_OK;
}
}  // namespace

namespace {
// *bad = whether some of the n entries of d_v is not a finite positive number (synchronises `st`)
int field_bad(int64_t n, const double *d_v, cudaStream_t st, const char *who, int *bad) {
  int *d_flag = nullptr;
  PCGB_CUDA(cudaMalloc(&d_flag, sizeof(int)));
  cudaMemsetAsync(d_flag, 0, sizeof(int), st);
  k_field_check<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, 4096)), 256, 0, st>>>(n, d_v, d_flag);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(bad, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(d_flag);
  return e == cudaSuccess ? PCGB_OK : fail(PCGB_ERR_CUDA, "%s: field check failed: %s", who, cudaGetErrorString(e));
}

// ---- checks and tail shared by mg_create_one and mg_create_ranks
int mg_check_ranges(int degree, double lo, double E, double h, const char *who) {
  if (degree >= 1 && lo > 0.0 && lo < 1.1 && E > 0.0 && h > 0.0) return PCGB_OK;
  return fail(PCGB_ERR_ARG, "%s: degree >= 1, 0 < lo < 1.1, E > 0 and h > 0 required", who);
}

int mg_check_rows(pcgb_solver_t s, const pcgb_hex_box *box, const char *who) {
  const int64_t n = 3 * hex_geom(box).nfree_nodes;
  if (n == s->n) return PCGB_OK;
  return fail(PCGB_ERR_ARG, "%s: the solver's operator has %lld rows, the box %lld", who, (long long)s->n, (long long)n);
}

// geo: the whole-box levels from the global box down; nlev: the levels of the whole hierarchy
int mg_check_levels(const std::vector<HexGeom> &geo, size_t nlev, const char *who) {
  if (3 * geo.back().nfree_nodes > kMgMaxCoarse)
    return fail(PCGB_ERR_ARG, "%s: the coarsest level has %lld dofs (at most %d)", who, (long long)(3 * geo.back().nfree_nodes), kMgMaxCoarse);
  if (nlev > PCGB_MG_MAX_LEVELS) return fail(PCGB_ERR_ARG, "%s: more than %d levels", who, PCGB_MG_MAX_LEVELS);
  return PCGB_OK;
}

// the caller's fine Ck field of nel elements
int mg_check_field(int64_t nel, const double *d_ck_fine, const char *who) {
  // the check runs on the legacy stream, which does not wait for non-blocking streams: finish whatever work of the caller
  // may still be writing d_ck_fine first
  PCGB_CUDA(cudaDeviceSynchronize());
  int bad = 0;
  PCGB_TRY(field_bad(nel, d_ck_fine, 0, who, &bad));
  return bad ? fail(PCGB_ERR_ARG, "%s: every Ck of the field must be finite and positive", who) : PCGB_OK;
}

// Builds the hierarchy the caller has laid out in mg, forgets the caller's field and element plan (not used after create; a
// rap level 1 keeps the field, as the caller does), and registers the handle with the solver; destroys it on failure.
int mg_finish(pcgb_mg_t mg, MgOp coarse, const double *ke_host, double E, double h, const double *d_minv_fine,
              const double *const *own, pcgb_mg_t *out) {
  const int rc = mg_build(mg, coarse, ke_host, E, h, d_minv_fine, own);
  mg->ck_fine = nullptr;
  mg->kel_gather = nullptr;
  if (rc != PCGB_OK) { pcgb_mg_destroy(mg); return rc; }
  mg->s->mgs.push_back(mg);
  *out = mg;
  return PCGB_OK;
}

// pcgb_mg_create (d_ck_fine NULL: Ck = E 2^l h on level l; coarse Hex: pcgb_mg_create_index_free), pcgb_mg_create_field
// (field: Galerkin levels from d_ck_fine, which must be given; coarse Rap: pcgb_mg_create_field_rap) and pcgb_mg_create_any
// (any_rule: the coarsening of mg_any_box_levels, Galerkin levels from d_ck_fine or, NULL, Ck = E h)
int mg_create_one(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, double E, double h, bool field,
                  const double *d_ck_fine, const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out, const char *who,
                  bool any_rule = false, MgOp coarse = MgOp::Csr) {
  PCGB_TRY(require_device());
  if (!s || !box || !ke_host || !d_minv_fine || !out || (field && !d_ck_fine)) return fail(PCGB_ERR_ARG, "%s: null argument", who);
  if (s->halo || s->comm) return fail(PCGB_ERR_ARG, "%s: one rank only (the solver has a halo plan or a communicator)", who);
  PCGB_TRY(mg_check_ranges(degree, lo, E, h, who));
  for (int a = 0; a < 3; ++a)
    if (box->e0[a] != 0 || box->ng[a] != box->ne[a] || box->ne[a] <= 0)
      return fail(PCGB_ERR_ARG, "%s: the box must be the whole mesh (e0 = 0, ng = ne)", who);
  PCGB_TRY(mg_check_rows(s, box, who));
  std::vector<HexGeom> geo{hex_geom(box)};
  std::vector<int> keep;
  std::vector<char> any;
  if (any_rule) {
    mg_any_box_levels(geo, keep, any, PCGB_MG_MAX_LEVELS);
    if (geo.size() < 2) return fail(PCGB_ERR_ARG, "%s: the box does not coarsen (some ne must be >= 3)", who);
  } else {
    mg_whole_box_levels(geo);
    if (geo.size() < 2) return fail(PCGB_ERR_ARG, "%s: the box does not coarsen (every ne must be even and >= 4)", who);
  }
  if (coarse == MgOp::Rap && geo.size() < 3)
    return fail(PCGB_ERR_ARG, "%s: the hierarchy has %d levels (at least 3, so that level 1 is smoothed)", who, (int)geo.size());
  PCGB_TRY(mg_check_levels(geo, geo.size(), who));
  if (d_ck_fine) PCGB_TRY(mg_check_field((int64_t)geo[0].nx * geo[0].ny * geo[0].nz, d_ck_fine, who));
  // a uniform box under the any rule: Galerkin levels from Ck = E h on every fine element (freed once the levels exist)
  double *ck_uniform = nullptr;
  if (any_rule && !d_ck_fine) {
    PCGB_CUDA(cudaDeviceSynchronize());
    const std::vector<double> ckh((size_t)geo[0].nx * geo[0].ny * geo[0].nz, E * h);
    PCGB_CUDA(upload(&ck_uniform, ckh));
    d_ck_fine = ck_uniform;
  }
  pcgb_mg_t mg = new pcgb_mg_s();
  mg->s = s; mg->degree = degree; mg->lo = lo; mg->ck_fine = d_ck_fine;
  mg->lv.resize(geo.size());
  for (size_t l = 0; l < geo.size(); ++l) {
    MgLevel &L = mg->lv[l];
    L.g = geo[l]; L.glev = (int)l; L.place = MgPlace{geo[l], 0, 0, 0};
    if (l < any.size()) { L.any = any[l] != 0; L.keep = keep[l]; }
  }
  const int rc = mg_finish(mg, coarse, ke_host, E, h, d_minv_fine, nullptr, out);
  cudaFree(ck_uniform);
  return rc;
}
}  // namespace

int pcgb_mg_create(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, double E, double h, const double *d_minv_fine,
                   int degree, double lo, pcgb_mg_t *out) {
  return mg_create_one(s, box, ke_host, E, h, false, nullptr, d_minv_fine, degree, lo, out, "pcgb_mg_create");
}

int pcgb_mg_create_index_free(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, double E, double h,
                              const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_one(s, box, ke_host, E, h, false, nullptr, d_minv_fine, degree, lo, out, "pcgb_mg_create_index_free", false,
                       MgOp::Hex);
}

int pcgb_mg_create_field(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine,
                         const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_one(s, box, ke_host, 1.0, 1.0, true, d_ck_fine, d_minv_fine, degree, lo, out, "pcgb_mg_create_field");
}

int pcgb_mg_create_field_rap(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine,
                             const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_one(s, box, ke_host, 1.0, 1.0, true, d_ck_fine, d_minv_fine, degree, lo, out, "pcgb_mg_create_field_rap", false,
                       MgOp::Rap);
}

int pcgb_mg_create_any(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine, double E, double h,
                       const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_one(s, box, ke_host, E, h, false, d_ck_fine, d_minv_fine, degree, lo, out, "pcgb_mg_create_any", true);
}

int pcgb_mg_level_box(pcgb_mg_t mg, int level, int32_t *ne) {
  if (!mg || !ne) return fail(PCGB_ERR_ARG, "pcgb_mg_level_box: null argument");
  if (level < 0 || level >= (int)mg->lv.size())
    return fail(PCGB_ERR_ARG, "pcgb_mg_level_box: level %d outside 0 .. %d", level, (int)mg->lv.size() - 1);
  const HexGeom &g = mg->lv[(size_t)level].g;
  ne[0] = g.nx; ne[1] = g.ny; ne[2] = g.nz;
  return PCGB_OK;
}

int pcgb_mg_level_csr(pcgb_mg_t mg, int level, int64_t *d_rowptr, int32_t *d_col, double *d_val, int64_t *nnz, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !nnz) return fail(PCGB_ERR_ARG, "pcgb_mg_level_csr: null argument");
  if (level == 0 || !mg_smoothed(mg, level))
    return fail(PCGB_ERR_ARG, "pcgb_mg_level_csr: level %d has no coarse CSR (levels 1 .. %d, not the gathered one)", level,
                (int)mg->lv.size() - 2);
  const MgLevel &L = mg->lv[(size_t)level];
  if (L.op == MgOp::Hex) return fail(PCGB_ERR_ARG, "pcgb_mg_level_csr: level %d is index-free (no CSR)", level);
  if (L.op == MgOp::Rap) return fail(PCGB_ERR_ARG, "pcgb_mg_level_csr: level %d is applied as P^T A P from the fine field (no CSR)", level);
  *nnz = L.P.nnz;
  if (!d_rowptr && !d_col && !d_val) return PCGB_OK;
  if (!d_rowptr || !d_col || !d_val) return fail(PCGB_ERR_ARG, "pcgb_mg_level_csr: give all three buffers or none");
  const cudaStream_t st = (cudaStream_t)stream;
  std::vector<int64_t> r64((size_t)L.n + 1);
  if (L.P.rp64) {
    PCGB_CUDA(cudaMemcpy(r64.data(), L.rowptr, r64.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
  } else {
    std::vector<int32_t> r32(r64.size());
    PCGB_CUDA(cudaMemcpy(r32.data(), L.rowptr, r32.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    std::copy(r32.begin(), r32.end(), r64.begin());
  }
  PCGB_CUDA(cudaMemcpyAsync(d_rowptr, r64.data(), r64.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  PCGB_CUDA(cudaMemcpyAsync(d_col, L.col, (size_t)L.P.nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  PCGB_CUDA(cudaMemcpyAsync(d_val, L.val, (size_t)L.P.nnz * sizeof(double), cudaMemcpyDeviceToDevice, st));
  PCGB_CUDA(cudaStreamSynchronize(st));
  return PCGB_OK;
}

int pcgb_mg_level_apply(pcgb_mg_t mg, int level, const double *d_x, double *d_y, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_mg_level_apply: null argument");
  if (level == 0 || !mg_smoothed(mg, level))
    return fail(PCGB_ERR_ARG, "pcgb_mg_level_apply: level %d has no coarse operator (levels 1 .. %d, not the gathered one)", level,
                (int)mg->lv.size() - 2);
  const MgLevel &L = mg->lv[(size_t)level];
  const uintptr_t x0 = (uintptr_t)d_x, y0 = (uintptr_t)d_y, nb = (uintptr_t)L.n * sizeof(double);
  if (x0 < y0 + nb && y0 < x0 + nb) return fail(PCGB_ERR_ARG, "pcgb_mg_level_apply: x and y overlap");
  return level_apply(mg, level, d_x, d_y, (cudaStream_t)stream, nullptr, nullptr);
}

int pcgb_mg_level_dinv(pcgb_mg_t mg, int level, double *d_out, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !d_out) return fail(PCGB_ERR_ARG, "pcgb_mg_level_dinv: null argument");
  if (!mg_smoothed(mg, level))
    return fail(PCGB_ERR_ARG, "pcgb_mg_level_dinv: level %d is not smoothed (levels 0 .. %d, not the gathered one)", level,
                (int)mg->lv.size() - 2);
  const MgLevel &L = mg->lv[(size_t)level];
  PCGB_CUDA(cudaMemcpyAsync(d_out, L.dinv, (size_t)L.n * sizeof(double), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return PCGB_OK;
}

int pcgb_mg_setup_info(pcgb_mg_t mg, double *galerkin_ms, int64_t *element_matrix_peak_bytes) {
  if (!mg) return fail(PCGB_ERR_ARG, "pcgb_mg_setup_info: null argument");
  if (galerkin_ms) *galerkin_ms = mg->galerkin_ms;
  if (element_matrix_peak_bytes) *element_matrix_peak_bytes = mg->kel_peak;
  return PCGB_OK;
}

namespace {
// pcgb_mg_create_ranks, (coarse Hex) pcgb_mg_create_ranks_index_free and (field: d_ck_fine and kel_gather, which must be
// given) pcgb_mg_create_ranks_field (coarse Rap: pcgb_mg_create_ranks_field_rap, level 1 applied by k_mg_rap1 on the rank's
// level-1 box from the rank's Ck slice, its local product completed by the level's exchange-add like every ranked level's)
int mg_create_ranks(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos, pcgb_halo_t gather,
                    const double *const *d_own, const double *ke_host, double E, double h, const double *d_minv_fine, int degree,
                    double lo, pcgb_mg_t *out, MgOp coarse, const char *who, bool field = false, const double *d_ck_fine = nullptr,
                    pcgb_halo_t kel_gather = nullptr) {
  PCGB_TRY(require_device());
  if (!s || !box || !level_halos || !gather || !d_own || !ke_host || !d_minv_fine || !out || (field && (!d_ck_fine || !kel_gather)))
    return fail(PCGB_ERR_ARG, "%s: null argument", who);
  if (!s->comm || s->comm->nranks < 2) return fail(PCGB_ERR_ARG, "%s: the solver has no communicator of 2 or more ranks", who);
  PCGB_TRY(mg_check_ranges(degree, lo, E, h, who));
  for (int a = 0; a < 3; ++a)
    if (box->ne[a] <= 0 || box->e0[a] < 0 || box->e0[a] + box->ne[a] > box->ng[a])
      return fail(PCGB_ERR_ARG, "%s: the box does not lie in the mesh", who);
  PCGB_TRY(mg_check_rows(s, box, who));
  if (n_ranked < 1) return fail(PCGB_ERR_ARG, "%s: the fine level does not coarsen (n_ranked >= 1 required)", who);
  if (coarse == MgOp::Rap && n_ranked < 2)
    return fail(PCGB_ERR_ARG, "%s: n_ranked is %d (at least 2, so that level 1 is smoothed, not gathered)", who, n_ranked);
  // ranked levels 0 .. la: the rank's box halved la times, and the global box around it
  const int la = n_ranked;
  std::vector<pcgb_hex_box> rb{*box};
  for (int l = 1; l <= la; ++l) {
    const pcgb_hex_box &p = rb.back();
    pcgb_hex_box c = p;
    for (int a = 0; a < 3; ++a) {
      if (p.ne[a] % 2 || p.ne[a] < 4 || p.e0[a] % 2 || p.ng[a] % 2)
        return fail(PCGB_ERR_ARG, "%s: level %d cannot be halved (ne even and >= 4, e0 and ng even)", who, l - 1);
      c.ng[a] = p.ng[a] / 2; c.e0[a] = p.e0[a] / 2; c.ne[a] = p.ne[a] / 2;
    }
    rb.push_back(c);
  }
  for (int l = 1; l <= la; ++l) {
    const pcgb_halo_t hl = level_halos[l - 1];
    if (!hl || hl->comm != s->comm || hl->nlocal != 3 * hex_geom(&rb[(size_t)l]).nfree_nodes)
      return fail(PCGB_ERR_ARG, "%s: the halo of level %d is missing, on another communicator or not of the level's size", who, l);
  }
  pcgb_hex_box gb = rb.back();
  for (int a = 0; a < 3; ++a) { gb.e0[a] = 0; gb.ne[a] = gb.ng[a]; }
  std::vector<HexGeom> geo{hex_geom(&gb)};
  const int64_t ng_dofs = 3 * geo[0].nfree_nodes;
  if (ng_dofs > kMgMaxGathered)
    return fail(PCGB_ERR_ARG, "%s: the gathered level has %lld dofs (at most %lld)", who, (long long)ng_dofs, (long long)kMgMaxGathered);
  if (gather->comm != s->comm || gather->nlocal != ng_dofs || gather->n_nbr != s->comm->nranks - 1 ||
      gather->m != (int64_t)(s->comm->nranks - 1) * ng_dofs)
    return fail(PCGB_ERR_ARG, "%s: the gather plan must list all %lld dofs of the gathered level for every other rank", who,
                (long long)ng_dofs);
  for (int l = 0; l <= la; ++l)
    if (!d_own[l]) return fail(PCGB_ERR_ARG, "%s: null ownership weights of level %d", who, l);
  mg_whole_box_levels(geo);
  PCGB_TRY(mg_check_levels(geo, (size_t)la + 1 + geo.size(), who));
  if (field) {
    const int64_t nge = (int64_t)geo[0].nx * geo[0].ny * geo[0].nz;
    if (nge > kMgMaxGatheredElements)
      return fail(PCGB_ERR_ARG, "%s: the gathered level has %lld elements (at most %lld)", who, (long long)nge,
                  (long long)kMgMaxGatheredElements);
    if (kel_gather->comm != s->comm || kel_gather->nlocal != 576 * nge || kel_gather->n_nbr != s->comm->nranks - 1 ||
        kel_gather->m != (int64_t)(s->comm->nranks - 1) * 576 * nge)
      return fail(PCGB_ERR_ARG, "%s: the element plan must list all %lld entries of the gathered level's element matrices for "
                  "every other rank", who, (long long)(576 * nge));
    PCGB_TRY(mg_check_field((int64_t)box->ne[0] * box->ne[1] * box->ne[2], d_ck_fine, who));
  }
  pcgb_mg_t mg = new pcgb_mg_s();
  mg->s = s; mg->degree = degree; mg->lo = lo; mg->la = la; mg->gather = gather;
  mg->ck_fine = d_ck_fine; mg->kel_gather = kel_gather;
  mg->lv.resize((size_t)la + 1 + geo.size());
  for (int l = 0; l <= la; ++l) {
    MgLevel &L = mg->lv[(size_t)l];
    const pcgb_hex_box &b = rb[(size_t)l];
    pcgb_hex_box whole = b;
    for (int a = 0; a < 3; ++a) { whole.e0[a] = 0; whole.ne[a] = whole.ng[a]; }
    L.g = hex_geom(&b); L.glev = l; L.place = MgPlace{hex_geom(&whole), b.e0[0], b.e0[1], b.e0[2]};
    L.halo = l ? level_halos[l - 1] : s->halo;
  }
  for (size_t k = 0; k < geo.size(); ++k) {
    MgLevel &L = mg->lv[(size_t)la + 1 + k];
    L.g = geo[k]; L.glev = la + (int)k; L.place = MgPlace{geo[k], 0, 0, 0};
  }
  return mg_finish(mg, coarse, ke_host, E, h, d_minv_fine, d_own, out);
}
}  // namespace

int pcgb_mg_create_ranks(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos, pcgb_halo_t gather,
                         const double *const *d_own, const double *ke_host, double E, double h, const double *d_minv_fine,
                         int degree, double lo, pcgb_mg_t *out) {
  return mg_create_ranks(s, box, n_ranked, level_halos, gather, d_own, ke_host, E, h, d_minv_fine, degree, lo, out, MgOp::Csr,
                         "pcgb_mg_create_ranks");
}

int pcgb_mg_create_ranks_index_free(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                                    pcgb_halo_t gather, const double *const *d_own, const double *ke_host, double E, double h,
                                    const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_ranks(s, box, n_ranked, level_halos, gather, d_own, ke_host, E, h, d_minv_fine, degree, lo, out, MgOp::Hex,
                         "pcgb_mg_create_ranks_index_free");
}

int pcgb_mg_create_ranks_field(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                               pcgb_halo_t gather, pcgb_halo_t kel_gather, const double *const *d_own, const double *ke_host,
                               const double *d_ck_fine, const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_ranks(s, box, n_ranked, level_halos, gather, d_own, ke_host, 1.0, 1.0, d_minv_fine, degree, lo, out, MgOp::Csr,
                         "pcgb_mg_create_ranks_field", true, d_ck_fine, kel_gather);
}

int pcgb_mg_create_ranks_field_rap(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                                   pcgb_halo_t gather, pcgb_halo_t kel_gather, const double *const *d_own, const double *ke_host,
                                   const double *d_ck_fine, const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out) {
  return mg_create_ranks(s, box, n_ranked, level_halos, gather, d_own, ke_host, 1.0, 1.0, d_minv_fine, degree, lo, out, MgOp::Rap,
                         "pcgb_mg_create_ranks_field_rap", true, d_ck_fine, kel_gather);
}

int pcgb_mg_apply(pcgb_mg_t mg, const double *d_r, double *d_z, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !d_r || !d_z) return fail(PCGB_ERR_ARG, "pcgb_mg_apply: null argument");
  // the pre-smoother writes z while the post-smoother still reads r as the fine right-hand side
  const uintptr_t r0 = (uintptr_t)d_r, z0 = (uintptr_t)d_z, nb = (uintptr_t)mg->lv[0].n * sizeof(double);
  if (r0 < z0 + nb && z0 < r0 + nb) return fail(PCGB_ERR_ARG, "pcgb_mg_apply: r and z overlap");
  int nl = 0;
  return mg_vcycle(mg, d_r, d_z, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_info(pcgb_mg_t mg, int32_t *nlevels, int64_t *n_level, double *lambda, int64_t *bytes) {
  PCGB_TRY(require_device());
  if (!mg) return fail(PCGB_ERR_ARG, "pcgb_mg_info: null argument");
  if (nlevels) *nlevels = (int32_t)mg->lv.size();
  for (size_t l = 0; l < mg->lv.size(); ++l) {
    if (n_level) n_level[l] = mg->lv[l].n;
    if (lambda) lambda[l] = mg->lv[l].lambda;
  }
  if (bytes) *bytes = mg->bytes;
  return PCGB_OK;
}

int pcgb_mg_restrict(pcgb_mg_t mg, int level, const double *d_fine, double *d_coarse, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !mg_smoothed(mg, level) || !d_fine || !d_coarse)
    return fail(PCGB_ERR_ARG, "pcgb_mg_restrict: bad argument");
  int nl = 0;
  return mg_restrict(mg, level, d_fine, d_coarse, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_prolong_add(pcgb_mg_t mg, int level, const double *d_coarse, double *d_fine, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !mg_smoothed(mg, level) || !d_fine || !d_coarse)
    return fail(PCGB_ERR_ARG, "pcgb_mg_prolong_add: bad argument");
  int nl = 0;
  return mg_prolong_add(mg, level, d_coarse, d_fine, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_smooth(pcgb_mg_t mg, int level, const double *d_b, double *d_x, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !mg_smoothed(mg, level) || !d_b || !d_x)
    return fail(PCGB_ERR_ARG, "pcgb_mg_smooth: bad argument");
  int nl = 0;
  return mg_smooth(mg, level, d_b, d_x, false, false, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_info_ranks(pcgb_mg_t mg, int32_t *gather_level, int64_t *n_gathered) {
  if (!mg) return fail(PCGB_ERR_ARG, "pcgb_mg_info_ranks: null argument");
  if (gather_level) *gather_level = mg->la;
  if (n_gathered) *n_gathered = mg->la >= 0 ? mg->lv[(size_t)mg->la + 1].n : 0;
  return PCGB_OK;
}

int pcgb_mg_gather(pcgb_mg_t mg, const double *d_ranked, double *d_global, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || mg->la < 0 || !d_ranked || !d_global) return fail(PCGB_ERR_ARG, "pcgb_mg_gather: bad argument (or a one-rank handle)");
  int nl = 0;
  return mg_gather(mg, d_ranked, d_global, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_scatter(pcgb_mg_t mg, const double *d_global, double *d_ranked, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || mg->la < 0 || !d_ranked || !d_global) return fail(PCGB_ERR_ARG, "pcgb_mg_scatter: bad argument (or a one-rank handle)");
  int nl = 0;
  return mg_scatter(mg, d_global, d_ranked, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_mg_coarse_solve(pcgb_mg_t mg, const double *d_r, double *d_z, void *stream) {
  PCGB_TRY(require_device());
  if (!mg || !d_r || !d_z) return fail(PCGB_ERR_ARG, "pcgb_mg_coarse_solve: null argument");
  int nl = 0;
  return mg_coarse_solve(mg, d_r, d_z, (cudaStream_t)stream, &nl, nullptr);
}

int pcgb_solve_mg(pcgb_solver_t s, pcgb_mg_t mg, const double *d_b, const double *d_w, double *d_x, const pcgb_options *opt,
                  double *d_resvec, pcgb_result *res, void *stream) {
  PCGB_TRY(require_device());
  if (!s || !mg || !d_b || !d_x || !opt || !res) return fail(PCGB_ERR_ARG, "pcgb_solve_mg: null argument");
  if (mg->s != s) return fail(PCGB_ERR_ARG, "pcgb_solve_mg: the preconditioner was built for another solver");
  if (opt->maxiter <= 0) return fail(PCGB_ERR_ARG, "pcgb_solve_mg: maxiter must be positive");
  return solve_fenced(s, mg, d_b, nullptr, d_w, d_x, opt, d_resvec, res, stream);
}

// ------------------------------------------------------------------------------------ hex generator
int64_t pcgb_hex_nrows(const pcgb_hex_box *box) {
  if (!box) return 0;
  return 3 * hex_geom(box).nfree_nodes;
}

int pcgb_hex_count(const pcgb_hex_box *box, int64_t *d_rowcount, void *stream) {
  if (!box || !d_rowcount) return fail(PCGB_ERR_ARG, "pcgb_hex_count: null argument");
  PCGB_TRY(require_device());
  HexGeom g = hex_geom(box);
  if (g.nx <= 0 || g.ny <= 0 || g.nz <= 0 || g.nfree_nodes <= 0) return fail(PCGB_ERR_ARG, "pcgb_hex_count: empty box");
  k_hex_count<<<(unsigned)((g.nfree_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, d_rowcount);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_hex_fill(const pcgb_hex_box *box, const double *ke_host, double ck, const int64_t *d_rowptr, int32_t *d_col,
                  double *d_val, void *stream) {
  if (!box || !ke_host || !d_rowptr || !d_col || !d_val) return fail(PCGB_ERR_ARG, "pcgb_hex_fill: null argument");
  PCGB_TRY(require_device());
  HexGeom g = hex_geom(box);
  PCGB_CUDA(cudaMemcpyToSymbolAsync(c_hex_ke, ke_host, 24 * 24 * sizeof(double), 0, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  const int64_t threads = g.nfree_nodes * 32;
  k_hex_fill<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, ck, d_rowptr, d_col, d_val);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

int pcgb_hex_field_check(const pcgb_hex_box *box, const double *d_ck, void *stream) {
  if (!box || !d_ck) return fail(PCGB_ERR_ARG, "pcgb_hex_field_check: null argument");
  PCGB_TRY(require_device());
  HexGeom g = hex_geom(box);
  if (g.nx <= 0 || g.ny <= 0 || g.nz <= 0) return fail(PCGB_ERR_ARG, "pcgb_hex_field_check: empty box");
  int bad = 0;
  PCGB_TRY(field_bad((int64_t)g.nx * g.ny * g.nz, d_ck, (cudaStream_t)stream, "pcgb_hex_field_check", &bad));
  return bad ? fail(PCGB_ERR_ARG, "pcgb_hex_field_check: every Ck of the field must be finite and positive") : PCGB_OK;
}

int pcgb_hex_fill_field(const pcgb_hex_box *box, const double *ke_host, const double *d_ck, const int64_t *d_rowptr, int32_t *d_col,
                        double *d_val, void *stream) {
  if (!box || !ke_host || !d_ck || !d_rowptr || !d_col || !d_val) return fail(PCGB_ERR_ARG, "pcgb_hex_fill_field: null argument");
  PCGB_TRY(require_device());
  HexGeom g = hex_geom(box);
  if (g.nx <= 0 || g.ny <= 0 || g.nz <= 0 || g.nfree_nodes <= 0) return fail(PCGB_ERR_ARG, "pcgb_hex_fill_field: empty box");
  const cudaStream_t st = (cudaStream_t)stream;
  int bad = 0;
  PCGB_TRY(field_bad((int64_t)g.nx * g.ny * g.nz, d_ck, st, "pcgb_hex_fill_field", &bad));
  if (bad) return fail(PCGB_ERR_ARG, "pcgb_hex_fill_field: every Ck of the field must be finite and positive");
  PCGB_CUDA(cudaMemcpyToSymbolAsync(c_hex_ke, ke_host, 24 * 24 * sizeof(double), 0, cudaMemcpyHostToDevice, st));
  const int64_t threads = g.nfree_nodes * 32;
  k_hex_fill_var<false><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(g, d_ck, nullptr, d_rowptr, d_col, d_val);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

// ------------------------------------------------------------------------------------ index-free hex-box operator
// calcMatVecProd (pcg_solver.py:263-300) on a structured box, every index computed from the node's coordinates; the
// product and the diagonal (updatePreconditioner, :282-287) are bit-identical to the ordered EBE operator's on
// hexmesh.hex_type_group(box).
int pcgb_hexop_create(const pcgb_hex_box *box, const double *ke_host, double ck, const double *d_ck, pcgb_hexop_t *out) {
  if (!box || !ke_host || !out) return fail(PCGB_ERR_ARG, "pcgb_hexop_create: null argument");
  *out = nullptr;
  for (int a = 0; a < 3; ++a)
    if (box->ne[a] <= 0 || box->e0[a] < 0 || (int64_t)box->e0[a] + box->ne[a] > box->ng[a])
      return fail(PCGB_ERR_ARG, "pcgb_hexop_create: the box must have ne > 0 and lie inside its global mesh on every axis");
  if (!d_ck && !(std::isfinite(ck) && ck > 0.0)) return fail(PCGB_ERR_ARG, "pcgb_hexop_create: Ck must be finite and positive");
  PCGB_TRY(require_device());
  const HexOp H = hexop_of(hex_geom(box), ke_host, ck, d_ck);
  const HexGeom &g = H.s.g;
  if ((int64_t)H.s.nbx * H.s.nby * H.s.nbz >= (int64_t)1 << 31) return fail(PCGB_ERR_ARG, "pcgb_hexop_create: box too large");
  if (d_ck) {
    // the check runs on the legacy stream, which does not wait for non-blocking streams: finish the caller's writes first
    PCGB_CUDA(cudaDeviceSynchronize());
    int bad = 0;
    PCGB_TRY(field_bad((int64_t)g.nx * g.ny * g.nz, d_ck, 0, "pcgb_hexop_create", &bad));
    if (bad) return fail(PCGB_ERR_ARG, "pcgb_hexop_create: every Ck of the field must be finite and positive");
  }
  pcgb_hexop_t h = new pcgb_hexop_s();
  h->H = H;
  *out = h;
  return PCGB_OK;
}

int pcgb_hexop_destroy(pcgb_hexop_t H) {
  delete H;
  return PCGB_OK;
}

int pcgb_hexop_apply(pcgb_hexop_t H, const double *d_x, double *d_y, void *stream) {
  if (!H || !d_x || !d_y) return fail(PCGB_ERR_ARG, "pcgb_hexop_apply: null argument");
  const uintptr_t x0 = (uintptr_t)d_x, y0 = (uintptr_t)d_y, nb = (uintptr_t)H->H.n * sizeof(double);
  if (x0 < y0 + nb && y0 < x0 + nb) return fail(PCGB_ERR_ARG, "pcgb_hexop_apply: x and y overlap (each y is written from x around it)");
  return hexop_apply(H->H, d_x, d_y, (cudaStream_t)stream);
}

int pcgb_hexop_diag(pcgb_hexop_t H, double *d_diag, void *stream) {
  if (!H || !d_diag) return fail(PCGB_ERR_ARG, "pcgb_hexop_diag: null argument");
  return hexop_diag(H->H, d_diag, (cudaStream_t)stream);
}

int64_t pcgb_hexop_bytes(pcgb_hexop_t H) { return H ? H->H.bytes : 0; }

// ------------------------------------------------------------------------------------ strain and stress recovery
// updateElemStrain (pcg_solver.py:601-618), getNodalPS (:730-814) and getPrincipalStress / getPrincipalStrain
// (file_operations.py:251-301) on a hex box; the arithmetic contract is in fields.cuh.
int pcgb_fields_create(const pcgb_hex_box *box, double h, double E, double nu, const double *d_E, pcgb_fields_t *out) {
  if (!box || !out) return fail(PCGB_ERR_ARG, "pcgb_fields_create: null argument");
  *out = nullptr;
  for (int a = 0; a < 3; ++a)
    if (box->ne[a] <= 0 || box->e0[a] < 0 || (int64_t)box->e0[a] + box->ne[a] > box->ng[a])
      return fail(PCGB_ERR_ARG, "pcgb_fields_create: the box must have ne > 0 and lie inside its global mesh on every axis");
  if (!(std::isfinite(h) && h > 0.0) || !(std::isfinite(E) && E > 0.0) || !(nu > -1.0 && nu < 0.5))
    return fail(PCGB_ERR_ARG, "pcgb_fields_create: h and E must be finite and positive and -1 < nu < 0.5");
  PCGB_TRY(require_device());
  const HexGeom g = hex_geom(box);
  FieldsShape s = fields_shape(g);
  if ((int64_t)s.nbx * s.nby * s.nbz >= (int64_t)1 << 31) return fail(PCGB_ERR_ARG, "pcgb_fields_create: box too large");
  const int64_t ne = (int64_t)g.nx * g.ny * g.nz;
  if (d_E) {
    // the check runs on the legacy stream, which does not wait for non-blocking streams: finish the caller's writes first
    PCGB_CUDA(cudaDeviceSynchronize());
    int bad = 0;
    PCGB_TRY(field_bad(ne, d_E, 0, "pcgb_fields_create", &bad));
    if (bad) return fail(PCGB_ERR_ARG, "pcgb_fields_create: every E of the field must be finite and positive");
  }
  // lambda and mu as hexmesh.hex_element_stiffness(1.0, nu) computes them
  const double one = 1.0;
  s.q = 0.25 / h;
  s.E = E;
  s.lam = one * nu / ((1 + nu) * (1 - 2 * nu));
  s.m2 = 2 * (one / (2 * (1 + nu)));
  pcgb_fields_t F = new pcgb_fields_s();
  F->s = s;
  F->d_E = d_E;
  F->ne = ne;
  F->nnodes = (int64_t)(g.nx + 1) * (g.ny + 1) * (g.nz + 1);
  F->n = 3 * g.nfree_nodes;
  *out = F;
  return PCGB_OK;
}

int pcgb_fields_destroy(pcgb_fields_t F) {
  delete F;
  return PCGB_OK;
}

static bool overlap(const double *a, int64_t na, const double *b, int64_t nb) {
  if (!a || !b) return false;
  const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
  return a0 < b0 + (uintptr_t)nb * sizeof(double) && b0 < a0 + (uintptr_t)na * sizeof(double);
}

int pcgb_fields_element(pcgb_fields_t F, const double *d_x, double *d_strain, double *d_stress, double *d_ps, double *d_pe, void *stream) {
  if (!F || !d_x) return fail(PCGB_ERR_ARG, "pcgb_fields_element: null argument");
  const int64_t ne = F->ne;
  if (overlap(d_x, F->n, d_strain, 6 * ne) || overlap(d_x, F->n, d_stress, 6 * ne) || overlap(d_x, F->n, d_ps, 3 * ne) ||
      overlap(d_x, F->n, d_pe, 3 * ne))
    return fail(PCGB_ERR_ARG, "pcgb_fields_element: x overlaps an output");
  return fields_elem(F->s, F->d_E, d_x, d_strain, d_stress, d_ps, d_pe, (cudaStream_t)stream);
}

int pcgb_fields_nodal(pcgb_fields_t F, const double *d_x, int kind, pcgb_halo_t halo, double *d_work, double *d_out, void *stream) {
  if (!F || !d_x || !d_work || !d_out) return fail(PCGB_ERR_ARG, "pcgb_fields_nodal: null argument");
  if (kind != 0 && kind != 1) return fail(PCGB_ERR_ARG, "pcgb_fields_nodal: kind must be 0 (stress) or 1 (strain)");
  const int64_t nn = F->nnodes;
  if (halo && halo->nlocal != 4 * nn)
    return fail(PCGB_ERR_ARG, "pcgb_fields_nodal: the halo plan exchanges %lld entries, the box needs 4 per node (%lld)",
                (long long)halo->nlocal, (long long)(4 * nn));
  if (overlap(d_x, F->n, d_work, 4 * nn) || overlap(d_x, F->n, d_out, 3 * nn) || overlap(d_work, 4 * nn, d_out, 3 * nn))
    return fail(PCGB_ERR_ARG, "pcgb_fields_nodal: x, work and out must not overlap");
  const cudaStream_t st = (cudaStream_t)stream;
  double *pv = nullptr;   // the element principal values, 3 per element, for this call only
  PCGB_CUDA(cudaMallocAsync((void **)&pv, (size_t)(3 * F->ne) * sizeof(double), st));
  int rc = fields_elem(F->s, F->d_E, d_x, nullptr, nullptr, kind == 0 ? pv : nullptr, kind == 1 ? pv : nullptr, st);
  if (rc == PCGB_OK) {
    k_fields_nodal<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(F->s.g, pv, d_work);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(PCGB_ERR_CUDA, "pcgb_fields_nodal: %s", cudaGetErrorString(e));
  }
  const cudaError_t fe = cudaFreeAsync(pv, st);
  if (rc != PCGB_OK) return rc;
  if (fe != cudaSuccess) return fail(PCGB_ERR_CUDA, "pcgb_fields_nodal: %s", cudaGetErrorString(fe));
  if (halo) PCGB_TRY(halo_exchange_add(halo, d_work, st));
  k_fields_divide<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(nn, d_work, d_out);
  PCGB_CHECK_LAUNCH();
  return PCGB_OK;
}

}  // extern "C"
