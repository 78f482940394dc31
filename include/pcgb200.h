/* pcgb200.h - C ABI of libpcgb200.so: the H100 (sm_90a) implementation of the PCG inner
 * iteration of ankitskr/PCG-MPI-solver (reference: src/solver/pcg_solver.py).
 *
 * The reference is pure Python (numpy + mpi4py) and has no FFI of its own; the functions
 * below are what a ctypes binding of its hot path binds.  Each entry point cites the
 * reference code it replaces (file:line in the reference repository).
 *
 * Conventions
 *   - every pointer named d_* is a DEVICE pointer owned by the caller (torch tensors in the
 *     Python host code); the library never copies between host and device behind the
 *     caller's back, except the few control scalars pcgb_solve reads back to steer the loop;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - return value: 0 = ok, negative = error (see pcgb_last_error()); the MATLAB-style
 *     solver status (0..4, pcg_solver.py:399,449,468,477,493,497,541,561) is returned
 *     separately through pcgb_result;
 *   - handles are opaque; a handle may be used by one host thread at a time.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef PCGB200_H
#define PCGB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCGB_VERSION 200 /* 0.2.0 */

typedef struct pcgb_csr_s *pcgb_csr_t;     /* device CSR matrix + merge-path SpMV plan          */
typedef struct pcgb_comm_s *pcgb_comm_t;   /* communicator: peer-memory windows (+ NCCL), one rank = one GPU */
typedef struct pcgb_halo_s *pcgb_halo_t;   /* interface ("halo") exchange-add plan              */
typedef struct pcgb_solver_s *pcgb_solver_t; /* PCG workspace bound to one operator             */
typedef struct pcgb_ebe_s *pcgb_ebe_t;     /* opt-in matrix-free element-by-element operator (f1) */
typedef struct pcgb_asm_s *pcgb_asm_t;     /* device assembly of K_i[Eff,Eff] from the pattern groups (symbolic phase state) */
typedef struct pcgb_ebe2_s *pcgb_ebe2_t;   /* coloured (atomics-free, bit-reproducible) variant of the EBE operator */
typedef struct pcgb_ebe_ordered_s *pcgb_ebe_ordered_t; /* EBE operator with a fixed summation order (bit-reproducible, solver-ready) */
typedef struct pcgb_hexop_s *pcgb_hexop_t; /* index-free matrix-free operator of a hex box (the ordered operator's bits) */
typedef struct pcgb_mg_s *pcgb_mg_t;       /* geometric multigrid preconditioner of a hex-box solver (one V-cycle) */
typedef struct pcgb_fields_s *pcgb_fields_t; /* strain / stress recovery of a hex box (element fields, nodal averages) */

/* error codes */
#define PCGB_OK 0
#define PCGB_ERR_ARG (-1)
#define PCGB_ERR_CUDA (-2)
#define PCGB_ERR_NCCL (-3)
#define PCGB_ERR_NODEVICE (-4)
#define PCGB_ERR_COMM (-5) /* a peer-memory exchange timed out waiting for another rank */

int pcgb_version(void);
/* sizeof(pcgb_options), sizeof(pcgb_result), sizeof(pcgb_hex_box), sizeof(pcgb_ebe_group): lets a binding verify its struct layouts */
void pcgb_abi_sizes(int32_t out[4]);
const char *pcgb_last_error(void); /* thread-local message of the last failing call */
int pcgb_device_count(void);       /* number of visible CUDA devices (0 on a CPU box) */

/* ---------------------------------------------------------------- CSR operator (a2, a7)
 * Replaces calcMatVecProd(..., 'Strain') (pcg_solver.py:242-300) on the free ("Eff") dofs:
 * A = K[Eff,Eff] assembled to CSR (SURVEY Fact 1), so the P_unq[LocDofEff] scatter /
 * Q_unq[LocDofEff] gather around the matvec (pcg_solver.py:482-484) disappear.
 * fp64 values, int32 column indices, row offsets int32 or int64 (int64 is mandatory once
 * nnz >= 2^31, e.g. the 256^3 block).  Arrays stay owned by the caller and must outlive the
 * handle.  pcgb_csr_create builds the merge-path tile plan (device-side searches).
 */
int pcgb_csr_create(int64_t nrows, int64_t ncols, int64_t nnz, const void *d_rowptr, int rowptr_is_64,
                    const int32_t *d_col, const double *d_val, void *stream, pcgb_csr_t *out);
int pcgb_csr_destroy(pcgb_csr_t A);
/* y = A x  (one launch of the merge-path kernel, plus a fix-up launch only if rows are split) */
int pcgb_spmv(pcgb_csr_t A, const double *d_x, double *d_y, void *stream);
/* d[i] = A[i,i]  (Jacobi diagonal, replaces calcMatVecProd(...,'Preconditioner'), pcg_solver.py:282-287) */
int pcgb_csr_diag(pcgb_csr_t A, double *d_diag, void *stream);
/* The persistent staged-x SpMV kernel reads its own 16-bit index stream, never d_col.  pcgb_csr_release_col caches the
 * diagonal and drops the library's reference to d_col; the caller may then free it (2 GB at 128^3, 16 GB at 256^3).
 * PCGB_ERR_ARG when the selected kernel still needs the column array. */
int pcgb_csr_release_col(pcgb_csr_t A, void *stream);
/* Interface-first split of the SpMV for the multi-GPU overlap (SURVEY 8(e): "order boundary rows first, launch exchange,
 * compute interior rows"): d_rows = distinct local rows taking part in the interface exchange (pcg_solver.py:304-312).
 * Tiles owning such a row run in a first launch, all others in a second one.  pcgb_solver_create registers the rows
 * of its halo plan itself; these two entry points make the split testable on one GPU.  d_out_dot (may be NULL) = x.y */
int pcgb_csr_set_boundary_rows(pcgb_csr_t A, const int32_t *d_rows, int64_t count, void *stream);
int pcgb_spmv_split(pcgb_csr_t A, const double *d_x, double *d_y, double *d_out_dot, void *stream);
/* Algorithmic bytes of one SpMV: 12*nnz + R*(nrows+1) + 8*ncols + 8*nrows (SURVEY 8(d)). */
int64_t pcgb_spmv_bytes(pcgb_csr_t A);
/* Bytes the selected kernel really streams from HBM (the staged-x kernel reads 16-bit local column
 * indices: 10 B per non-zero instead of 12; with the column-triple index 8 + 2/3 B). */
int64_t pcgb_spmv_stream_bytes(pcgb_csr_t A);
/* plan introspection for tests / DESIGN.md: tiles, tile items, lanes, snap, split rows, smem bytes,
 * max row, tma, staged, x windows, staged doubles per tile (cap), max windows per tile, column-triple index (0/1),
 * interface tiles (-1 = no split registered), resident CTAs of the persistent kernel, column array released (0/1) */
int pcgb_csr_plan_info(pcgb_csr_t A, int64_t info[16]);
/* Distinct 3x3 blocks D of the value dictionary of the node-block kernel, 0 when the plan has none.  With D > 0 the SpMV
 * streams a 16-bit block id per block instead of its 72 bytes of values and reads the values from a D-entry copy in
 * shared memory: products bit-identical to the kernel that streams the values.  The plan builds one for node-block
 * matrices with at most 1024 bitwise-distinct blocks (a structured mesh of one element type) when the values it replaces
 * outweigh the per-CTA dictionary loads; PCGB_SPMV_VDICT=0 disables it, =2 drops the size condition.  d_val is still
 * read by pcgb_csr_diag and must stay allocated. */
int pcgb_csr_value_dict(pcgb_csr_t A);
/* With a dictionary, the index stream holds per tile a list of at most 8 segments of consecutive nodes.  In a run segment
 * every node has the blocks of the one before it, 3 staged x entries further on with the same ids, and only the head's
 * block words are stored.  Returns the share of the nodes that lie in run segments (0 without a dictionary). */
double pcgb_csr_run_share(pcgb_csr_t A);
/* The ring of the dictionary kernel, all zeros when the plan has no dictionary: out = {stages, tiles per group G,
 * producer warps, consumer warps CW, words of the largest tile slice (cap_words), words of the index stream (nvwords),
 * nodes per tile stage (cap_nodes), resident CTAs per SM}. */
int pcgb_csr_vd_plan(pcgb_csr_t A, int64_t out[8]);

/* ---------------------------------------------------------------- vector kernels (a4-a10)
 * out[0] = sum_i a[i]*b[i]*w[i]   (w may be NULL = all ones).  np.dot(a, b*w) of
 * pcg_solver.py:381,415,462,487,504-506,532,573.  Deterministic two-level reduction.  */
int pcgb_dot_w(int64_t n, const double *d_a, const double *d_b, const double *d_w, double *d_out, void *stream);
/* y[i] = a*x[i] + b*y[i] */
int pcgb_axpby(int64_t n, double a, const double *d_x, double b, double *d_y, void *stream);
/* z[i] = x[i]*y[i] */
int pcgb_mul(int64_t n, const double *d_x, const double *d_y, double *d_z, void *stream);
/* out[i] = 1/d[i]  (updatePreconditioner, pcg_solver.py:351) */
int pcgb_reciprocal(int64_t n, const double *d_d, double *d_out, void *stream);

/* ---------------------------------------------------------------- communicator (a13)
 * Replaces mpi4py COMM_WORLD (pcg_solver.py:968-970).  Two transports for the data path:
 *   PEER (default)  the library's own kernels over CUDA-IPC mapped peer memory (NVLink / NVSwitch): the all-reduce is
 *                   fused into the reduction kernel of the iteration, the halo values are stored straight into the
 *                   neighbours' receive buffers (csrc/peer.cuh).  Needs the window exchange below.
 *   NCCL            ncclAllReduce / ncclSend / ncclRecv (baseline and fallback; PCGB_COMM=nccl selects it).
 * NCCL is resolved at run time with dlopen("libnccl.so.2") so the library loads on a box without NCCL.  Rank 0 obtains a
 * unique id and the host code broadcasts it (torch.distributed / mpi4py / any side channel).  id == NULL creates a
 * peer-only communicator (no NCCL at all; at most 16 ranks).                                                     */
#define PCGB_UNIQUE_ID_BYTES 128
#define PCGB_IPC_BLOB_BYTES 64
#define PCGB_TRANSPORT_NCCL 0
#define PCGB_TRANSPORT_PEER 1
int pcgb_comm_unique_id(unsigned char id[PCGB_UNIQUE_ID_BYTES]);
int pcgb_comm_create(int rank, int nranks, const unsigned char *id /* [PCGB_UNIQUE_ID_BYTES] or NULL */, pcgb_comm_t *out);
int pcgb_comm_destroy(pcgb_comm_t c);
/* window exchange: export -> all-gather the blobs over the host side channel (rank order) -> import */
int pcgb_comm_window_export(pcgb_comm_t c, unsigned char blob[PCGB_IPC_BLOB_BYTES]);
int pcgb_comm_window_import(pcgb_comm_t c, const unsigned char *blobs /* nranks * PCGB_IPC_BLOB_BYTES */);
int pcgb_comm_transport(pcgb_comm_t c);                  /* transport the data path uses right now */
int pcgb_comm_set_transport(pcgb_comm_t c, int transport);
int pcgb_comm_status(pcgb_comm_t c, void *stream);       /* 0 healthy; != 0 after a peer exchange timed out (sticky) */
/* in-place sum of `count` doubles over all ranks (MPI_SUM, pcg_solver.py:622-628); rank-ordered, bit-identical on every rank */
int pcgb_allreduce_sum(pcgb_comm_t c, double *d_buf, int count, void *stream);

/* ---------------------------------------------------------------- halo exchange-add (a14)
 * Replaces the pack / Isend / Recv / Waitall / += of pcg_solver.py:303-334.
 *   nbr_rank[j]        neighbour j's rank              (NbrMPIdVector)
 *   nbr_ptr[j..j+1]    range of neighbour j in idx     (host array, n_nbr+1 entries)
 *   idx[k]             local row index (in the Eff numbering of A) of the k-th shared dof,
 *                      ordered by ascending GLOBAL node id then direction on both sides
 *                      (OvrlpLocalDofVecList, partition_mesh.py:822-827)
 * Lists are positional pairs: entry t of my list for rank s and entry t of s's list for me
 * name the same dof, so both lists have the same length.  nbr_ptr[0] is 0, the neighbour
 * ranks are distinct (not this rank, in 0..nranks-1), and the indices of one list are
 * distinct and in 0..nlocal-1; anything else is PCGB_ERR_ARG before anything is allocated.
 * An empty list is dropped (both sides drop it alike), so a rank whose lists are all empty
 * has no neighbours and nobody waits for it.
 * The exchange computes, for every shared dof, y[dof] first, then the neighbours' copies
 * added in the caller's neighbour order j = 0..n_nbr-1 (one per list the dof is in), i.e.
 * the summation order of the reference loop at pcg_solver.py:333-334 (deterministic).    */
int pcgb_halo_create(pcgb_comm_t c, int n_nbr, const int32_t *nbr_rank, const int64_t *nbr_ptr,
                     const int64_t *idx_host, int64_t nlocal, pcgb_halo_t *out);
int pcgb_halo_destroy(pcgb_halo_t h);
/* peer transport: every rank exports its receive block, the host all-gathers the blobs (pcgb_halo_blob_bytes each, rank
 * order) and imports them; the import checks that both sides of every interface list the same number of shared dofs */
int64_t pcgb_halo_blob_bytes(pcgb_halo_t h);
int pcgb_halo_export(pcgb_halo_t h, unsigned char *blob);
int pcgb_halo_import(pcgb_halo_t h, const unsigned char *blobs);
/* y[idx] += (values of the same dofs on the neighbours) */
int pcgb_halo_exchange_add(pcgb_halo_t h, double *d_y, void *stream);
int64_t pcgb_halo_bytes(pcgb_halo_t h); /* bytes sent (= received) per exchange by this rank */

/* ---------------------------------------------------------------- PCG (a1, a4-a13)
 * Replaces PCG(RefMeshPart) (pcg_solver.py:356-598): Jacobi-PCG with MATLAB `pcg`
 * semantics on the free dofs of one subdomain.                                         */
typedef struct pcgb_options {
  double tol;           /* GlobData['Tol']                                                 */
  int32_t maxiter;      /* GlobData['MaxIter']                                             */
  int64_t n_global;     /* GlobData['GlobNDofEff'] (only used for MaxMSteps, :404)          */
  int32_t max_stag;     /* MaxStagSteps = 3 (:403); <=0 selects 3                           */
  int32_t check_every;  /* iterations enqueued between host polls of the device state; <=0 = 16 */
  int32_t use_graph;    /* capture the batch of iterations in a CUDA graph (1) or launch directly (0) */
  int32_t fixed_iters;  /* benchmark mode: ignore convergence, run exactly maxiter iterations */
  int32_t record_resvec; /* keep ||r|| per iteration (reference has this commented out, :428-434) */
  int32_t time_kernels; /* bracket every SpMV launch of the loop with CUDA events (forces direct launches) */
  int32_t x0_zero;      /* the caller guarantees d_x is all zeros on entry: r0 = b exactly, the initial operator application is skipped */
} pcgb_options;

typedef struct pcgb_result {
  int32_t flag;       /* 0 converged, 1 maxiter, 2 precond inf, 3 stagnation, 4 breakdown       */
  int32_t iters;      /* `Iter` after the +1 of pcg_solver.py:584                                */
  double relres;      /* RelRes                                                                  */
  double normb;       /* NormRefLoadVector (n2b)                                                 */
  int32_t imin;       /* iMin                                                                    */
  int32_t stag;       /* Stag at exit                                                            */
  int32_t moresteps;  /* MoreSteps at exit                                                       */
  int32_t too_small_tol; /* 1 if the reference would have raised Warning('PCG : TooSmallTolerance') (:549) */
  int64_t matvecs;    /* operator applications performed                                         */
  int64_t launches;   /* CUDA kernel launches issued by this solve (bench 'gpu_launches')        */
  double loop_ms;     /* device time of the iteration loop only (CUDA events on the solver stream)  */
  double spmv_ms;     /* sum of the SpMV launch durations inside the loop (time_kernels only)        */
  int64_t spmv_timed; /* number of SpMV launches in spmv_ms                                         */
  int64_t loop_iters; /* iterations executed inside the timed loop                                  */
  double setup_ms;    /* device time from the entry of the solve to the start of the loop (||b||, r0, rho0) */
  double final_ms;    /* device time from the end of the loop to the copy-out of x (finalisation matvec)    */
  double phase_ms[8]; /* time_kernels: sums over the bracketed iterations of p-update | SpMV | halo pack | p.q reduce+all-reduce |
                         halo unpack-add | fused update | norms reduce+all-reduce | whole iteration                  */
} pcgb_result;

int pcgb_solver_create(pcgb_csr_t A, pcgb_halo_t halo /* may be NULL */, pcgb_comm_t comm /* may be NULL */,
                       pcgb_solver_t *out);
int pcgb_solver_destroy(pcgb_solver_t s);
/* d_b: right-hand side Fext[LocDofEff]; d_minv: inverse diagonal (InvDiagPreCondVector0) or
 * NULL = identity (ExistDP0 False); d_w: DofWeightVector_Eff or NULL = ones;
 * d_x: in = initial guess X0, out = solution (X, or XMin on the non-converged path, :569-582).
 * d_resvec: optional device buffer of maxiter+2 doubles when record_resvec is set.
 * Weights: d_w weights ||b||, every norm and z.r (:381, :462, :504-506, :532).  p.q is always the UNWEIGHTED sum of the
 * local products p_i.(K_i p_i), fused into the operator: over several ranks that equals the reference's weighted dot of
 * the assembled q (p is consistent on shared dofs).  On ONE rank with w != 1 the reference would weight p.q too
 * (:487) and this solver does not, so alpha differs from the reference there; one rank has no shared dofs and its
 * natural weights are all 1.                                                                    */
int pcgb_solve(pcgb_solver_t s, const double *d_b, const double *d_minv, const double *d_w, double *d_x,
               const pcgb_options *opt, double *d_resvec, pcgb_result *res, void *stream);
/* Opt-in trace of the loop (tests / debugging).  d_trace (device, NULL = off) = a 64-byte header {uint64 records
 * produced; int32 scratch ...} followed by `capacity` records of pcgb_trace_record_bytes() bytes; records past the
 * capacity are dropped (the header still counts them).  One record per control step, in order: the head of
 * iteration 0, every iteration, every host verification, the head that follows a failed verification, and the
 * finalisation.  Each holds the reduced values the step consumed (and, over several ranks, this rank's local value
 * before the all-reduce, recomputed from the same partials) and the whole control block after the step
 * (layout: struct PcgTraceRec, csrc/pcg_kernels.cuh).  d_snapshot (device, may be NULL) = 5*n + 3 doubles: r, p, q
 * and the two x buffers when the loop exits, before the finalisation, then xcur, xmin, alias.  The setting stays
 * on the handle until changed; with tracing off the solve launches exactly what it launches without this call. */
int pcgb_solver_set_trace(pcgb_solver_t s, void *d_trace, int64_t capacity, double *d_snapshot);
int64_t pcgb_trace_record_bytes(void);
/* y = A x followed by the interface sum: calcMPFint (pcg_solver.py:339-342) on Eff dofs */
int pcgb_apply(pcgb_solver_t s, const double *d_x, double *d_y, void *stream);

/* ---------------------------------------------------------------- opt-in: matrix-free EBE operator (f1)
 * The reference's own operator form: calcMatVecProd(...,'Strain'), pcg_solver.py:263-300, on the GPU, one
 * pattern group per reference type group (partition_mesh.py:470-491).  Parity-tested (tests/test_gpu_ebe.py);
 * opt-in - the assembled CSR path is the default.  d_idx is [nd][ne] int32 in the FREE-dof numbering
 * (-1 = clamped dof), d_sign [nd][ne] uint8 or NULL, d_ck [ne], ke_host the nd x nd pattern matrix (host).  */
typedef struct pcgb_ebe_group {
  int32_t nd;
  int64_t ne;
  const int32_t *d_idx;
  const unsigned char *d_sign;
  const double *d_ck;
  const double *ke_host;
} pcgb_ebe_group;
int pcgb_ebe_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, pcgb_ebe_t *out);
int pcgb_ebe_destroy(pcgb_ebe_t E);
int pcgb_ebe_apply(pcgb_ebe_t E, const double *d_x, double *d_y, void *stream); /* y = K_i x (no interface sum) */
int64_t pcgb_ebe_bytes(pcgb_ebe_t E);                                            /* algorithmic bytes per application */
int pcgb_solver_create_ebe(pcgb_ebe_t E, pcgb_halo_t halo /* may be NULL */, pcgb_comm_t comm /* may be NULL */,
                           pcgb_solver_t *out);

/* ---------------------------------------------------------------- opt-in: ordered matrix-free EBE operator
 * The same operator as pcgb_ebe_create (same group layout), applied in the reference's own two phases
 * (calcMatVecProd, pcg_solver.py:279-300) with no atomics in the arithmetic, so every application and every solve is
 * bit-reproducible:
 *   phase 1  every group g, element e and local index a writes one product into a slot buffer laid out like the
 *            reference's `Flat`: slot = off_g + a*ne_g + e (off_g = sum of nd*ne over the groups before g), value
 *            s_a * acc with acc = fma(Ke[a][b], u_b, acc) over b = 0..nd-1 ascending, starting from 0.0, and
 *            u_b = Ck_e * (s_b * x[idx_b]) (0 for a clamped b).  Ke is row-major, Ke[a][b] = ke_host[a*nd + b].
 *   phase 2  y_i = ((0.0 + v_1) + v_2) + ... over the slots of dof i in ascending slot position, i.e. in
 *            (group, local index, element) order - the order in which np.bincount visits `Flat` (:300).  Every y_i is
 *            written, 0 when no slot names dof i.
 * Create builds per-dof slot lists on the device (count, scan, fill, per-dof sort) and synchronises the device.
 * PCGB_ERR_ARG, before anything is allocated: n >= 2^30, a pattern size outside 1..96, null arrays, or 2^31 or more
 * slots in all (slot positions are int32).  The slot buffer costs 8 bytes per slot, the lists 4 bytes per free slot. */
int pcgb_ebe_ordered_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, pcgb_ebe_ordered_t *out);
int pcgb_ebe_ordered_destroy(pcgb_ebe_ordered_t O);
int pcgb_ebe_ordered_apply(pcgb_ebe_ordered_t O, const double *d_x, double *d_y, void *stream); /* y = K_i x (no interface sum) */
int64_t pcgb_ebe_ordered_bytes(pcgb_ebe_ordered_t O);                                         /* algorithmic bytes per application */
int pcgb_solver_create_ebe_ordered(pcgb_ebe_ordered_t O, pcgb_halo_t halo /* may be NULL */, pcgb_comm_t comm /* may be NULL */,
                                   pcgb_solver_t *out);

/* ---------------------------------------------------------------- device assembly of the CSR operator (f2)
 * A_i = K_i[Eff,Eff] = sum_e P_e^T (Ck_e S_e Ke S_e) P_e  from the reference's pattern type groups (partition_mesh.py:443-491;
 * the operator calcMatVecProd applies element by element, pcg_solver.py:263-300), assembled on the device with hand-written
 * kernels (csrc/assemble.cuh): incidence lists per dof -> per-row sorted distinct columns (symbolic) -> per-row
 * accumulation in a fixed element order (numeric).  No atomics in the arithmetic: bit-reproducible.  `groups` uses the same
 * layout as the EBE operator (d_idx in the free-dof numbering, -1 = clamped).  Two phases because the caller owns the
 * output arrays: symbolic fills d_rowptr[0..n] (int64) and reports nnz; numeric fills d_col / d_val (ascending columns). */
int pcgb_assemble_symbolic(int64_t n, int ngroups, const pcgb_ebe_group *groups, int64_t *d_rowptr, int64_t *nnz_out, void *stream,
                           pcgb_asm_t *out);
int pcgb_assemble_numeric(pcgb_asm_t a, const int64_t *d_rowptr, int32_t *d_col, double *d_val, void *stream);
int pcgb_assemble_destroy(pcgb_asm_t a);

/* Operator-level (not reachable from pcgb_solve; tests/test_gpu_ebe_colored.py, tests/test_gpu_ebe_color_edges.py): the
 * same operator with an atomics-free deterministic scatter.  groups[] = one entry per (pattern group, colour) slice, sorted
 * by colour (PCGB_ERR_ARG otherwise); phase[g] = colour of entry g.  No two elements of one colour may share a free dof;
 * create TRUSTS the caller's phases to be such a colouring and does not check it (EbeMatrixColored checks it on the host).
 * Ke is row-major, Ke[i][j] = ke_host[i*nd + j], and need not be symmetric.  Apply gives, bit for bit:
 *   for every free dof d, y_d starts from +0.0; the colours are taken in ascending order, and for the one element e of
 *   that colour that touches d, every local index i with idx[i] = d, in ascending i, does y_d = y_d + v_{e,i}, where
 *     u_j = s_j x_j (0.0 for a clamped dof),  acc = fma(Ke[i][j], u_j, acc) over j ascending from 0.0,
 *     v_{e,i} = round(acc * Ck_e), negated when s_i is set.
 *   Every y_d is written, +0.0 when no element touches d.                                                         */
int pcgb_ebe2_create(int64_t n, int ngroups, const pcgb_ebe_group *groups, const int32_t *phase, pcgb_ebe2_t *out);
int pcgb_ebe2_destroy(pcgb_ebe2_t E);
int pcgb_ebe2_apply(pcgb_ebe2_t E, const double *d_x, double *d_y, void *stream);
int pcgb_ebe2_launches(pcgb_ebe2_t E); /* kernel launches per application */

/* ---------------------------------------------------------------- structured hex generator
 * On-device generator of the sub-assembled stiffness matrix of one box of trilinear hex
 * elements (benchmark configs C2/C3/C5; SURVEY 8(d)).  The box holds elements
 * [e0[a], e0[a]+ne[a]) of a global ng[0] x ng[1] x ng[2] mesh; nodes with global x index 0
 * are clamped (removed from the Eff numbering).  ke is the 24x24 element matrix (host
 * pointer, row-major, local node l at offsets (l&1, l>>1&1, l>>2&1), 3 dofs per node) and ck
 * the per-element scale (ElemList_Ck = E*h).  Free dof numbering: x fastest, then y, z, then
 * direction.  pcgb_hex_count writes rowcount[i+1] (int64, rowcount[0] = 0) so that an
 * inclusive scan by the caller yields the row offsets.                                     */
typedef struct pcgb_hex_box {
  int32_t ng[3];
  int32_t e0[3];
  int32_t ne[3];
} pcgb_hex_box;
int64_t pcgb_hex_nrows(const pcgb_hex_box *box);
int pcgb_hex_count(const pcgb_hex_box *box, int64_t *d_rowcount, void *stream);
int pcgb_hex_fill(const pcgb_hex_box *box, const double *ke_host, double ck, const int64_t *d_rowptr,
                  int32_t *d_col, double *d_val, void *stream);
/* The same rows and columns for a voxel model: element e of the box (e = (z * ne[1] + y) * ne[0] + x, x fastest, the
 * element order of hexmesh.hex_type_group) has its own scale d_ck[e] (device, ne[0]*ne[1]*ne[2] doubles; Ck = E_e h),
 * as every element of the reference's concrete model carries its own ElemList_Ck (partition_mesh.py:437-479).  Each
 * 3x3 block is sum_e d_ck[e] Ke[la, lb] over the elements of pcgb_hex_fill, in the same order, summed from 0.0.
 * PCGB_ERR_ARG (before the fill; the check synchronises `stream`): an entry of d_ck that is not finite and positive. */
int pcgb_hex_fill_field(const pcgb_hex_box *box, const double *ke_host, const double *d_ck, const int64_t *d_rowptr,
                        int32_t *d_col, double *d_val, void *stream);
/* The same check of d_ck on its own (PCGB_ERR_ARG for an entry that is not finite and positive; synchronises `stream`), so
 * a caller can refuse a field before it allocates the CSR arrays. */
int pcgb_hex_field_check(const pcgb_hex_box *box, const double *d_ck, void *stream);

/* ---------------------------------------------------------------- opt-in: index-free matrix-free operator of a hex box
 * y = K_i x of `box` (the pcgb_hex_* numbering, no interface sum) with every index computed from the node's coordinates:
 * no index list, slot buffer, position list or atomics.  Bit-identical to pcgb_ebe_ordered_create on the box's single
 * pattern group (Ke, Ck per element in the order of pcgb_hex_fill_field): for free dof (node, d)
 *   y = 0.0;  for la = 0..7 ascending with element e = node - (la&1, la>>1&1, la>>2&1) inside the box:
 *             acc = 0.0;  for b = 0..23: acc = fma(Ke[3 la + d][b], Ck_e * x_b, acc)   (x_b = 0.0 for a clamped node);
 *             y = y + acc
 * (calcMatVecProd, pcg_solver.py:263-300, in np.bincount's order).  Ck_e = ck, or d_ck[e] when d_ck is not NULL (device,
 * ne[0]*ne[1]*ne[2] doubles, caller-owned: it must outlive the handle).  ke_host (24x24, row-major) is copied into the
 * handle and passed with every launch, so no other operator or generator can change it.
 * pcgb_hexop_create refuses with PCGB_ERR_ARG, holding no device memory: a box with some ne <= 0 or outside its global
 * mesh, a uniform ck that is not finite and positive, a field entry that is not (checked on the device after a device
 * synchronise).  The handle itself holds no device memory.
 * pcgb_hexop_apply refuses overlapping x and y (each y is computed from x around it).  pcgb_hexop_diag writes the
 * diagonal d = 0.0 + Ck_e Ke[3la+d][3la+d] + ... in ascending la (pcg_solver.py:282-287, np.bincount's order).
 * pcgb_hexop_bytes: algorithmic bytes per application (x and y once, 8 per element with a field). */
int pcgb_hexop_create(const pcgb_hex_box *box, const double *ke_host, double ck, const double *d_ck /* NULL = uniform */,
                      pcgb_hexop_t *out);
int pcgb_hexop_destroy(pcgb_hexop_t H);
int pcgb_hexop_apply(pcgb_hexop_t H, const double *d_x, double *d_y, void *stream);
int pcgb_hexop_diag(pcgb_hexop_t H, double *d_diag, void *stream);
int64_t pcgb_hexop_bytes(pcgb_hexop_t H);
int pcgb_solver_create_hexop(pcgb_hexop_t H, pcgb_halo_t halo /* may be NULL */, pcgb_comm_t comm /* may be NULL */,
                             pcgb_solver_t *out);

/* ---------------------------------------------------------------- opt-in: geometric multigrid preconditioner (hex boxes)
 * z = M r is one symmetric V-cycle over nested hex boxes (across ranks: pcgb_mg_create_ranks below), for a one-rank solver whose operator (CSR, EBE or ordered EBE) is
 * the stiffness matrix of `box` in the pcgb_hex_* numbering.  Level l+1 halves every ne of level l while all ne are even and
 * the halves stay >= 2; its matrix is generated on the device at spacing 2^l h (Ck = E 2^l h), which for nested Q1 spaces
 * equals the Galerkin product P^T A P.  P is trilinear interpolation of the free nodes, direction by direction (weights 1,
 * 1/2, 1/4, 1/8); restriction (P^T, <= 27 fine nodes in (dz, dy, dx) ascending order) and prolongation (<= 8 coarse nodes
 * in ascending order, added to x) are gathers without atomics.  Every level but the coarsest smooths with a degree-`degree`
 * Chebyshev polynomial in D^-1 A on [lo, 1.1] * lambda, lambda the largest eigenvalue of the tridiagonal matrix of 20
 * Lanczos steps on D^-1 A (D inner product) from the fixed start vector v_i = 1/2 + ((37 i + 11) mod 101) / 101.  The pre-smoother starts from x = 0 and the
 * post-smoother applies the same polynomial to b - A x, so M is symmetric.  The coarsest level (at most 1536 dofs) is
 * solved with a dense Cholesky factor computed on the device at create.  D^-1 of the fine level is a copy of
 * d_minv_fine (n doubles); the coarse levels use their own diagonals.
 * PCGB_ERR_ARG before anything is allocated: a solver with a halo plan or communicator, a box with e0 != 0 or ng != ne, a
 * box that does not coarsen at least once, a coarsest level above 1536 dofs, degree < 1, lo outside (0, 1.1), E or h <= 0,
 * or an operator whose size is not the box's.  PCGB_ERR_ARG after allocation, with every allocation given back: a coarsest
 * matrix whose Cholesky factorisation meets a pivot that is not positive (e.g. nu >= 0.5).  The solver must outlive the handle; destroying the handle also drops the
 * solver's cached graph of MG iterations.  Create synchronises the device first (d_minv_fine may come from any stream)
 * and again before it returns.                                                                                          */
#define PCGB_MG_MAX_LEVELS 32
int pcgb_mg_create(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, double E, double h, const double *d_minv_fine,
                   int degree, double lo, pcgb_mg_t *out);
int pcgb_mg_destroy(pcgb_mg_t mg);
/* z = M r (one V-cycle).  PCGB_ERR_ARG, before any launch, when [d_r, d_r + n) and [d_z, d_z + n) overlap (z = r included):
 * the pre-smoother writes z while the post-smoother still reads r. */
int pcgb_mg_apply(pcgb_mg_t mg, const double *d_r, double *d_z, void *stream);
/* levels; n per level, lambda per level (0 for the coarsest) into arrays of PCGB_MG_MAX_LEVELS entries; device bytes the
 * hierarchy allocated (vectors, coarse CSR, dense factor; the coarse SpMV plans' tile tables are not counted).  Any may be NULL. */
int pcgb_mg_info(pcgb_mg_t mg, int32_t *nlevels, int64_t *n_level, double *lambda, int64_t *bytes);
/* the V-cycle's parts, for tests: r_c = P^T r_f and x_f += P e_c between `level` and level+1; one smoothing
 * x += S (b - A x) on `level` (x = 0 gives the pre-smoother's x = S b); z = A_c^-1 r on the coarsest level */
int pcgb_mg_restrict(pcgb_mg_t mg, int level, const double *d_fine, double *d_coarse, void *stream);
int pcgb_mg_prolong_add(pcgb_mg_t mg, int level, const double *d_coarse, double *d_fine, void *stream);
int pcgb_mg_smooth(pcgb_mg_t mg, int level, const double *d_b, double *d_x, void *stream);
int pcgb_mg_coarse_solve(pcgb_mg_t mg, const double *d_r, double *d_z, void *stream);
/* pcgb_solve with z = M r instead of z = Minv .* r: the same loop, options, result and trace.  z counts as infinite
 * (flag 2) when any entry is not finite, since a V-cycle spreads one NaN over all of z.  res->matvecs counts the solver
 * operator's applications by the loop itself (one per iteration plus the true residuals), as in pcgb_solve; the
 * V-cycles' own products (2 * degree of the fine operator per cycle, plus the coarse levels) are not in it.  With
 * time_kernels, phase_ms[5] ("fused update") includes the V-cycle that follows the update.                        */
int pcgb_solve_mg(pcgb_solver_t s, pcgb_mg_t mg, const double *d_b, const double *d_w, double *d_x, const pcgb_options *opt,
                  double *d_resvec, pcgb_result *res, void *stream);
/* The same preconditioner across ranks, for a solver with a communicator of 2 or more ranks whose boxes tile the global mesh
 * (the domain decomposition of pcg_solver.py, whose Jacobi z = Minv .* r it replaces).  Collective: every rank calls it with
 * the same n_ranked.  Levels 0 .. la (la = n_ranked) are ranked: level l holds the rank's box halved l times (ng, e0, ne
 * all halved; each halving needs ne even and >= 4 and e0, ng even), its sub-assembled matrix at spacing 2^l h, halo plan
 * level_halos[l-1] (level 0: the solver's) and 0/1 ownership weights d_own[l] (n_l doubles, copied; the owner of a shared
 * dof is the lowest rank).  Every product and restriction on a ranked level is followed by its exchange-add, so vectors
 * stay consistent; restriction sums the owned fine nodes only; lambda comes from all-reduced, owner-weighted Lanczos sums
 * from the start vector at the GLOBAL free index g (so the one-rank lambda of the global mesh, to rounding).  Level la is
 * not smoothed: its owned entries are gathered into the global box of level la (k_mg_gather, then `gather`, a plan that
 * lists all of that box's dofs for every other rank: one non-zero term per entry, so every rank holds the same vector
 * bit for bit), which continues on every rank as the one-rank hierarchy above (whole boxes, dense Cholesky at the
 * bottom); its result is copied back out to level la.  The global boxes are those of pcgb_mg_create on the global mesh.
 * PCGB_ERR_ARG before anything is allocated: no multi-rank communicator, a box outside the mesh, an operator whose size
 * is not the box's, n_ranked < 1, a level that cannot be halved, a halo of the wrong size or communicator, a gather
 * plan that is not all-to-all over the gathered box, a gathered box above 2^17 dofs, a coarsest level above 1536 dofs,
 * the scalar arguments of pcgb_mg_create.  The halo plans must outlive the handle.  pcgb_mg_restrict on a ranked level
 * includes the coarse exchange-add; restrict / prolong_add / smooth refuse level la (use gather / scatter).        */
int pcgb_mg_create_ranks(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos, pcgb_halo_t gather,
                         const double *const *d_own, const double *ke_host, double E, double h, const double *d_minv_fine,
                         int degree, double lo, pcgb_mg_t *out);
/* The one-rank preconditioner for a voxel model (pcgb_hex_fill_field; the reference's per-element ElemList_Ck,
 * partition_mesh.py:437-479): d_ck_fine holds the fine box's Ck per element in the order of pcgb_hex_fill_field, and
 * the coarse matrices are Galerkin products instead of rediscretisations, which equal P^T A P only for a constant Ck.
 * Coarse element (X,Y,Z) has children (2X+cx, 2Y+cy, 2Z+cz), c in {0,1}^3; Q_c is the 24x24 trilinear interpolation
 * from its 8 corners onto child c's nodes (child node l at p = c + (l&1, l>>1&1, l>>2&1), weight from corner k
 * prod_a phi_{k_a}(p_a), phi_0(p) = (2-p)/2, phi_1(p) = p/2, exact in binary).  Level 1: K_E = sum_c Q_c^T (Ck_c Ke) Q_c;
 * level l+1: K_E = sum_c Q_c^T K_child(c) Q_c; each level is assembled from its element matrices like pcgb_hex_fill
 * (same rows, columns and element order), clamped nodes dropped, which is P_free^T A P_free with the P of
 * pcgb_mg_restrict / pcgb_mg_prolong_add.  Fixed summation order, no atomics: a repeated create is bit-identical.  The
 * element matrices take 4608 bytes per coarse element and live on the device only while the next level is built
 * (pcgb_mg_setup_info).  Smoothers, lambda, D^-1, the coarse Cholesky factor, pcgb_mg_apply and pcgb_solve_mg are
 * those of pcgb_mg_create.  Refusals: those of pcgb_mg_create, and PCGB_ERR_ARG, before anything is allocated, for an
 * entry of d_ck_fine that is not finite and positive (a device check, after a device synchronise, so d_ck_fine may come
 * from any stream).  d_ck_fine is not read after create returns. */
int pcgb_mg_create_field(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine,
                         const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* The voxel-model preconditioner across ranks: pcgb_mg_create_ranks (same boxes, levels, halo plans, ownership weights,
 * gather plan, collective call and V-cycle) with the Galerkin element matrices of pcgb_mg_create_field instead of
 * rediscretisations, for the domain decomposition of a heterogeneous model (the reference's per-element ElemList_Ck,
 * partition_mesh.py:437-479, split over ranks; it replaces the diagonal preconditioner of pcg_solver.py:346-352 and
 * 446-454).  d_ck_fine: the rank's fine Ck per element of `box`, in the order of pcgb_hex_fill_field.  Each rank builds
 * the element matrices of its own boxes only (levels 1 .. la, k_mg_galerkin from that element's eight children, so each
 * is bit-identical to the one-rank matrix of the same element of the global mesh); levels 1 .. la-1 are assembled into
 * the rank's sub-assembled CSR.  Level la's matrices are written into a zeroed array of the whole global box of level la
 * and completed by one exchange-add over kel_gather, a plan over 576 * (elements of that box) entries that lists all of
 * them for every other rank: one non-zero term per entry, so every rank holds the same matrices bit for bit.  They are
 * the matrices of level la + 1, from which the replicated levels continue as in pcgb_mg_create_field; their CSR and
 * lambda are those of the one-rank field hierarchy of the global mesh.  kel_gather is only used during the call (the
 * caller may destroy it when create returns); its buffers grow with (ranks - 1) * 576 * elements, so the gathered box
 * may hold at most 4096 elements.  Refusals: those of pcgb_mg_create_ranks (without E and h), and PCGB_ERR_ARG before
 * anything is allocated for a null d_ck_fine or kel_gather, an element plan that is not all-to-all over the gathered
 * box's matrices, a gathered box above 4096 elements, and an entry of d_ck_fine that is not finite and positive (a
 * device check after a device synchronise; it sees the rank's own entries only, so a caller checks the global field
 * before the collective call, as multigrid.HexMultigrid does).  d_ck_fine is not read after create returns. */
int pcgb_mg_create_ranks_field(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                               pcgb_halo_t gather, pcgb_halo_t kel_gather, const double *const *d_own, const double *ke_host,
                               const double *d_ck_fine, const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* The one-rank preconditioner for a box of any size, uniform or a voxel model; like pcgb_mg_create and
 * pcgb_mg_create_field it replaces the diagonal preconditioner of pcg_solver.py:346-352 and 446-454.  Every axis of a
 * level is coarsened on its own while some axis has ne >= 3: an axis with ne >= 3 is halved to (ne + 1) / 2 elements,
 * coarse node j at fine node s(j) = min(2j, ne), so an odd axis ends in a coarse element one fine element wide at its high
 * end; an axis with ne <= 2 is kept (s(j) = j).  The coarsest level has at most 2x2x2 elements (54 dofs).  Fine node i
 * between s(j) and s(j+1) takes weight (s(j+1) - i) / (s(j+1) - s(j)) from coarse node j and the rest from j + 1 (0, 1/2
 * or 1); P is the tensor product of the three 1-D maps, clamped nodes dropped.  The coarse levels are Galerkin products of
 * element matrices as in pcgb_mg_create_field, a coarse element having 1 or 2 children per axis, phi_0(p) = (w - p) / w,
 * phi_1(p) = p / w with w its width in fine elements; the fine elements carry d_ck_fine (as in pcgb_mg_create_field) or,
 * d_ck_fine NULL, Ck = E h.  A level whose axes are all halved from even ne uses exactly the kernels of
 * pcgb_mg_create_field (so an all-even box gives its hierarchy bit for bit); only levels with an odd or kept axis use the
 * transfers and Galerkin products for any widths.  Element matrices are always built: 4608 bytes per level-1 element at
 * the peak (pcgb_mg_setup_info).  PCGB_ERR_ARG before anything is allocated: the refusals of pcgb_mg_create_field but the
 * coarsening rule's (a box with every ne <= 2, more than PCGB_MG_MAX_LEVELS levels), and E or h <= 0. */
int pcgb_mg_create_any(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine, double E, double h,
                       const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* pcgb_mg_create and pcgb_mg_create_ranks with index-free coarse levels: the same hierarchy, arguments, refusals and
 * synchronisation, the same replacement of the diagonal preconditioner (pcg_solver.py:346-352 and 446-454), but every
 * smoothed level l >= 1 (across ranks: the ranked levels 1 .. la-1 and the replicated levels above the coarsest) applies
 * its box with the index-free operator of pcgb_hexop_create (Ke = ke_host, Ck = E 2^glev h, glev the level of the global
 * hierarchy; calcMatVecProd, pcg_solver.py:263-300, per node) instead of a device-generated CSR matrix and SpMV plan.
 * D^-1 of such a level is 1 / its pcgb_hexop_diag diagonal (pcg_solver.py:282-287), after the level's exchange-add on a
 * ranked level.  Lambda, smoothers, transfers, gather / scatter and the coarsest level's dense Cholesky factor are
 * unchanged, so the V-cycle equals pcgb_mg_create's to rounding.  The hierarchy holds only vectors and that factor:
 * pcgb_mg_info's bytes are 8 (5 n_0 + 6 sum n_l over the smoothed coarse levels + 2 n_c + n_c^2) on one rank (across
 * ranks also n_l ownership weights per ranked level and 2 n_la for the gathered level).  pcgb_mg_level_csr refuses its
 * levels.                                                                                                               */
int pcgb_mg_create_index_free(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, double E, double h,
                              const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
int pcgb_mg_create_ranks_index_free(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                                    pcgb_halo_t gather, const double *const *d_own, const double *ke_host, double E, double h,
                                    const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* pcgb_mg_create_field with a matrix-free level 1, for voxel models whose level-1 Galerkin matrices do not fit on the
 * device (at 512^3 they take 77 GB as element matrices, 49 GB as CSR).  Arguments, checks and refusals are those of
 * pcgb_mg_create_field, plus PCGB_ERR_ARG before anything is allocated for a box whose hierarchy has fewer than 3 levels
 * (level 1 would be the coarsest, not smoothed).  Level 1 applies y_1 = P^T A_0 P x_1 in one kernel (k_mg_rap1) from
 * d_ck_fine and ke_host, bit-identical to pcgb_mg_prolong_add of x_1 into a zero fine vector, the index-free fine
 * operator of pcgb_hexop_create with d_ck_fine, and pcgb_mg_restrict; it holds no matrix.  Levels >= 2 are those of
 * pcgb_mg_create_field bit for bit (CSR, D^-1, lambda, coarsest factor): level 2's element matrices are built from slabs
 * of level-1 element layers (at most 1 GiB, at least two layers) in ascending z, so level 1's are never held whole, and
 * level 1's D^-1 is the field hierarchy's bit for bit.  d_ck_fine is read by every V-cycle: it must outlive the handle.
 * pcgb_mg_level_csr refuses level 1; pcgb_mg_setup_info reports the level-2 matrices plus the slab (or, when larger, the
 * level-2 and level-3 matrices) and the device time of the Galerkin kernels. */
int pcgb_mg_create_field_rap(pcgb_solver_t s, const pcgb_hex_box *box, const double *ke_host, const double *d_ck_fine,
                             const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* pcgb_mg_create_ranks_field with the matrix-free level 1 of pcgb_mg_create_field_rap, for partitioned voxel models whose
 * rank boxes are too large for the level-1 Galerkin matrices.  Arguments, collective contract and refusals are those of
 * pcgb_mg_create_ranks_field, plus PCGB_ERR_ARG before anything is allocated for n_ranked < 2 (level 1 would be the
 * gathered level, which is not smoothed).  Ranked level 1 applies y_1 = P^T A_0 P x_1 by k_mg_rap1 on the rank's level-1
 * box from the rank's d_ck_fine, restricting without ownership weights: fine elements outside the box contribute 0.0,
 * and every fine node of a box with even e0 interpolates from coarse nodes of the box only, so the level's exchange-add
 * completes the assembled product.  Level 1's diagonal is summed from slabs of the rank's level-1 element matrices as in
 * pcgb_mg_create_field_rap, then exchange-added, so its D^-1 is pcgb_mg_create_ranks_field's bit for bit; so are every
 * level >= 2 (ranked CSR, gathered element matrices, replicated levels) and every lambda from level 2 on.  d_ck_fine is
 * read by every V-cycle: it must outlive the handle.  pcgb_mg_level_csr refuses level 1; pcgb_mg_setup_info reports the
 * rank's peak of element matrices, the gathered level's included. */
int pcgb_mg_create_ranks_field_rap(pcgb_solver_t s, const pcgb_hex_box *box, int n_ranked, const pcgb_halo_t *level_halos,
                                   pcgb_halo_t gather, pcgb_halo_t kel_gather, const double *const *d_own, const double *ke_host,
                                   const double *d_ck_fine, const double *d_minv_fine, int degree, double lo, pcgb_mg_t *out);
/* For tests: the inverse diagonal of smoothed level `level` (0 .. nlevels - 2, not the gathered level of a multi-rank
 * handle; level 0: the copy of d_minv_fine) of any handle into d_out (n_l doubles), ordered on `stream`.  PCGB_ERR_ARG
 * for any other level. */
int pcgb_mg_level_dinv(pcgb_mg_t mg, int level, double *d_out, void *stream);
/* For tests: y = A_l x on smoothed coarse level `level` (1 <= level < nlevels - 1, not the gathered level of a multi-rank
 * handle) of either kind, the local product without the level's exchange-add.  PCGB_ERR_ARG for any other level and,
 * before any launch, when [d_x, d_x + n_l) and [d_y, d_y + n_l) overlap. */
int pcgb_mg_level_apply(pcgb_mg_t mg, int level, const double *d_x, double *d_y, void *stream);
/* The element counts of level `level` (0 .. nlevels - 1) of any handle into ne[3] (x, y, z); PCGB_ERR_ARG outside. */
int pcgb_mg_level_box(pcgb_mg_t mg, int level, int32_t *ne);
/* For tests: level `level`'s CSR (1 <= level < nlevels - 1, the smoothed coarse levels) into caller buffers: int64 row
 * offsets (n + 1), int32 columns and values (nnz each).  With all three buffers NULL only *nnz is written.  Synchronises
 * `stream`.  PCGB_ERR_ARG for level 0 (the solver's operator), the coarsest level (held as a dense factor), the
 * gathered level of a multi-rank handle, every level of an index-free hierarchy and level 1 of a rap hierarchy. */
int pcgb_mg_level_csr(pcgb_mg_t mg, int level, int64_t *d_rowptr, int32_t *d_col, double *d_val, int64_t *nnz, void *stream);
/* Set-up costs of a field hierarchy (0 for the others): device time of the Galerkin kernels in ms, and the peak device
 * bytes of element matrices held at once during create.  Either may be NULL. */
int pcgb_mg_setup_info(pcgb_mg_t mg, double *galerkin_ms, int64_t *element_matrix_peak_bytes);
/* la (-1 for a one-rank handle) and the dofs of its gathered global box; pcgb_mg_info lists levels 0 .. la, then the
 * replicated levels (lambda 0 for level la and the coarsest) */
int pcgb_mg_info_ranks(pcgb_mg_t mg, int32_t *gather_level, int64_t *n_gathered);
/* level la's ranked vector into its global box on every rank (gather + exchange), and the rank's entries back out */
int pcgb_mg_gather(pcgb_mg_t mg, const double *d_ranked, double *d_global, void *stream);
int pcgb_mg_scatter(pcgb_mg_t mg, const double *d_global, double *d_ranked, void *stream);

/* ---------------------------------------------------------------- strain and stress recovery of a hex box
 * Replaces updateElemStrain (pcg_solver.py:601-618), getPrincipalStress / getPrincipalStrain (file_operations.py:251-301)
 * and getNodalPS (pcg_solver.py:730-814) with its exchange (:784-809) for the boxes of the pcgb_hex_* numbering; the
 * arithmetic contract (centroid Q1 gradient, stress law, invariant-form principal values and their two deviations, the
 * fixed nodal summation order) is the header comment of csrc/fields.cuh.  d_x: the box's free-dof vector (n =
 * pcgb_hex_nrows doubles, clamped nodes u = 0).  Elements e = (z ne[1] + y) ne[0] + x; nodes of the whole box, clamped
 * line included: node = (z (ne[1]+1) + y) (ne[0]+1) + x.
 * pcgb_fields_create: h the element edge, E the uniform Young's modulus, nu Poisson's ratio (lambda and mu of the Q1
 * matrix's D); d_E (device, ne[0]*ne[1]*ne[2] doubles, caller-owned, must outlive the handle) replaces E per element.
 * PCGB_ERR_ARG, holding no device memory: a box with some ne <= 0 or outside its global mesh, h or E not finite and
 * positive, nu outside (-1, 0.5), an entry of d_E that is not finite and positive (checked on the device after a device
 * synchronise).  The handle holds no device memory.
 * pcgb_fields_element: one pass over the box writing the outputs that are not NULL, element-major: strain (6 per element,
 * Voigt 11, 22, 33, 23, 13, 12, tensor shears), stress (6), principal stress (3: P1 >= P2 >= P3), principal strain (3).
 * PCGB_ERR_ARG when x overlaps an output.
 * pcgb_fields_nodal: the nodal average of the principal stresses (kind 0) or strains (kind 1): d_work (4 doubles per node)
 * receives (sum_0, sum_1, sum_2, count) over the node's elements, then, with a halo plan (pcgb_halo_create over the 4 *
 * nodes entries of d_work, listing 4 node + k, k = 0..3, of each shared node), the neighbours' copies; d_out (3 per node)
 * = sum / (count + 1e-15).  Scratch of 3 doubles per element is allocated and freed on `stream` within the call.
 * PCGB_ERR_ARG before any launch: kind not 0 or 1, a halo whose vector length is not 4 * nodes, x, work and out
 * overlapping. */
int pcgb_fields_create(const pcgb_hex_box *box, double h, double E, double nu, const double *d_E /* NULL = uniform E */,
                       pcgb_fields_t *out);
int pcgb_fields_destroy(pcgb_fields_t F);
int pcgb_fields_element(pcgb_fields_t F, const double *d_x, double *d_strain, double *d_stress, double *d_ps, double *d_pe,
                        void *stream);
int pcgb_fields_nodal(pcgb_fields_t F, const double *d_x, int kind /* 0 stress, 1 strain */, pcgb_halo_t halo /* NULL on one rank */,
                      double *d_work /* 4 per node */, double *d_out /* 3 per node */, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PCGB200_H */
