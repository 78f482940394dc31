// comm.cuh - NCCL communicator + interface ("halo") exchange plan.
//
// Replaces the mpi4py traffic of the hot path: the three allreduces per iteration
// (MPI_SUM, pcg_solver.py:622-628) and the neighbour exchange-add of the matvec
// (pcg_solver.py:303-334).  NCCL is bound at run time (dlopen) so that libpcgb200.so loads on
// machines without NCCL and picks up the copy torch already mapped into the process.
#pragma once
#include <dlfcn.h>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "pcg_kernels.cuh"
#include "peer.cuh"

namespace pcgb {

// minimal NCCL ABI (stable since NCCL 2.x): types and enum values from nccl.h
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclFloat64 = 8 };
enum { ncclSum = 0 };

struct NcclApi {
  void *handle = nullptr;
  int (*GetUniqueId)(ncclUniqueId *) = nullptr;
  int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Send)(const void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Recv)(void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  int (*GetVersion)(int *) = nullptr;
};

inline int nccl_api(NcclApi **out) {
  static NcclApi api;
  static std::once_flag once;
  static std::string load_error;
  std::call_once(once, []() {
    const char *names[] = {getenv("PCGB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
      if (!n || !*n) continue;
      api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
      const char *e = dlerror();
      if (e) load_error = e;
    }
    if (api.handle) {
#define PCGB_SYM(field, name) *(void **)(&api.field) = dlsym(api.handle, name)
      PCGB_SYM(GetUniqueId, "ncclGetUniqueId");
      PCGB_SYM(CommInitRank, "ncclCommInitRank");
      PCGB_SYM(CommDestroy, "ncclCommDestroy");
      PCGB_SYM(AllReduce, "ncclAllReduce");
      PCGB_SYM(Send, "ncclSend");
      PCGB_SYM(Recv, "ncclRecv");
      PCGB_SYM(GroupStart, "ncclGroupStart");
      PCGB_SYM(GroupEnd, "ncclGroupEnd");
      PCGB_SYM(GetErrorString, "ncclGetErrorString");
      PCGB_SYM(GetVersion, "ncclGetVersion");
#undef PCGB_SYM
    }
  });
  if (!api.handle || !api.CommInitRank || !api.AllReduce || !api.Send || !api.Recv)
    return fail(PCGB_ERR_NCCL, "NCCL not available: dlopen(libnccl.so.2) failed (%s)", load_error.empty() ? "missing symbols" : load_error.c_str());
  *out = &api;
  return PCGB_OK;
}

#define PCGB_NCCL(api, call)                                                                   \
  do {                                                                                         \
    int e_ = (call);                                                                           \
    if (e_ != ::pcgb::ncclSuccess)                                                             \
      return ::pcgb::fail(PCGB_ERR_NCCL, "%s:%d %s -> %s", __FILE__, __LINE__, #call,          \
                          (api)->GetErrorString ? (api)->GetErrorString(e_) : "nccl error");   \
  } while (0)

}  // namespace pcgb

// Transport of the data path: PEER = the library's own kernels over CUDA-IPC mapped peer memory (peer.cuh, default as
// soon as the windows have been exchanged), NCCL = ncclAllReduce / ncclSend / ncclRecv (bootstrap-free fallback and
// the comparison baseline; PCGB_COMM=nccl keeps it even when windows exist).
// (PCGB_TRANSPORT_NCCL / PCGB_TRANSPORT_PEER are defined in pcgb200.h)

struct pcgb_comm_s {
  pcgb::NcclApi *api = nullptr;      // null for a peer-only communicator (created without a unique id)
  pcgb::ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  int device = 0;
  // peer window
  unsigned long long *win = nullptr;                       // local window (cudaMalloc, exported through cudaIpcGetMemHandle)
  unsigned long long *peer[pcgb::kMaxPeers] = {nullptr};   // opened windows of the other ranks
  bool peer_ready = false;
  int transport = PCGB_TRANSPORT_NCCL;
  int *d_status = nullptr;                                 // sticky time-out flag of the peer kernels
  int *h_status = nullptr;                                 // pinned mirror

  pcgb::PeerWin window() const {
    pcgb::PeerWin w;
    w.rank = rank; w.nranks = nranks;
    for (int r = 0; r < pcgb::kMaxPeers; ++r) w.base[r] = r < nranks ? (r == rank ? win : peer[r]) : nullptr;
    w.epoch = win + pcgb::kWinArBytes / 8;
    w.status = d_status;
    return w;
  }
  bool use_peer() const { return peer_ready && transport == PCGB_TRANSPORT_PEER; }
};

struct pcgb_halo_s {
  pcgb_comm_t comm = nullptr;
  int n_nbr = 0;
  std::vector<int> nbr_rank;
  std::vector<int64_t> nbr_ptr;
  int64_t m = 0;          // total shared entries (with multiplicity over neighbours)
  int64_t ndof = 0;       // distinct interface dofs
  int64_t nlocal = 0;     // length of the vectors it exchanges
  int *d_idx = nullptr;   // [m]   gather index for the pack
  int *d_dof = nullptr;   // [ndof] distinct dofs
  int *d_ptr = nullptr;   // [ndof+1]
  int *d_pos = nullptr;   // [m]   positions in the receive buffer, neighbour order per dof
  double *d_send = nullptr, *d_recv = nullptr;   // NCCL transport staging
  // peer transport: one IPC-exported block  [ recv 2*m doubles | flags n_nbr*2 u64 ]  + local bookkeeping
  unsigned char *blk = nullptr;
  size_t blk_bytes = 0;
  std::vector<void *> opened;                    // neighbour blocks opened with cudaIpcOpenMemHandle
  int *d_nbr_ptr = nullptr, *d_ent_nbr = nullptr;
  double **d_remote = nullptr;
  int64_t *d_remote_m = nullptr;
  unsigned long long **d_remote_flag = nullptr;
  unsigned long long *d_epoch = nullptr;         // [0] epoch, [1] pack completion counter
  bool peer_ready = false;

  pcgb::PeerHalo peer_view() const {
    pcgb::PeerHalo v;
    v.n_nbr = n_nbr; v.m = m; v.nbr_ptr = d_nbr_ptr; v.ent_nbr = d_ent_nbr; v.remote = d_remote; v.remote_m = d_remote_m;
    v.remote_flag = d_remote_flag; v.recv = reinterpret_cast<double *>(blk);
    v.flags = reinterpret_cast<unsigned long long *>(blk + (size_t)2 * (size_t)m * sizeof(double));
    v.epoch = d_epoch; v.done = reinterpret_cast<unsigned int *>(d_epoch + 1); v.status = comm ? comm->d_status : nullptr;
    return v;
  }
  bool use_peer() const { return peer_ready && comm && comm->use_peer(); }
};

namespace pcgb {

// y[idx] += neighbours' copies.  Peer transport: pack (stores into the neighbours' buffers) and unpack are separate so
// that the solver can put the interior SpMV tiles between them (halo_pack / halo_unpack); NCCL transport: serial.
inline int halo_pack(pcgb_halo_t h, const double *y, cudaStream_t st, int *launches = nullptr) {
  if (!h || h->m == 0) return PCGB_OK;
  k_halo_pack_peer<<<(unsigned)((h->m + 256 * kPackPerThread - 1) / (256 * kPackPerThread)), 256, 0, st>>>(h->peer_view(), h->d_idx, y);
  PCGB_CHECK_LAUNCH();
  if (launches) *launches += 1;
  return PCGB_OK;
}
inline int halo_unpack(pcgb_halo_t h, double *y, cudaStream_t st, int *launches = nullptr) {
  if (!h || h->m == 0) return PCGB_OK;
  k_halo_unpack_peer<<<(unsigned)((h->ndof + 255) / 256), 256, 0, st>>>(h->peer_view(), h->ndof, h->d_dof, h->d_ptr, h->d_pos, y);
  PCGB_CHECK_LAUNCH();
  if (launches) *launches += 1;
  return PCGB_OK;
}

inline int halo_exchange_add(pcgb_halo_t h, double *y, cudaStream_t st, int *launches = nullptr) {
  if (!h || h->m == 0) return PCGB_OK;
  if (h->use_peer()) {
    PCGB_TRY(halo_pack(h, y, st, launches));
    return halo_unpack(h, y, st, launches);
  }
  if (!h->comm || !h->comm->api) return fail(PCGB_ERR_NCCL, "halo exchange: neither peer windows nor NCCL are available");
  NcclApi *api = h->comm->api;
  k_halo_pack<<<(unsigned)((h->m + 255) / 256), 256, 0, st>>>(h->m, h->d_idx, y, h->d_send);
  PCGB_CHECK_LAUNCH();
  PCGB_NCCL(api, api->GroupStart());
  for (int j = 0; j < h->n_nbr; ++j) {
    const int64_t o = h->nbr_ptr[j], c = h->nbr_ptr[j + 1] - o;
    PCGB_NCCL(api, api->Send(h->d_send + o, (size_t)c, ncclFloat64, h->nbr_rank[j], h->comm->comm, st));
    PCGB_NCCL(api, api->Recv(h->d_recv + o, (size_t)c, ncclFloat64, h->nbr_rank[j], h->comm->comm, st));
  }
  PCGB_NCCL(api, api->GroupEnd());
  k_halo_unpack_add<<<(unsigned)((h->ndof + 255) / 256), 256, 0, st>>>(h->ndof, h->d_dof, h->d_ptr, h->d_pos, h->d_recv, y);
  PCGB_CHECK_LAUNCH();
  if (launches) *launches += 2;
  return PCGB_OK;
}

// in-place sum of count <= 8 doubles over the ranks (MPI_SUM, pcg_solver.py:622-628)
inline int allreduce_sum(pcgb_comm_t c, double *d_buf, int count, cudaStream_t st) {
  if (c->use_peer() && count <= kArMaxVals) {
    k_allreduce_peer<<<1, 32, 0, st>>>(c->window(), d_buf, count);
    PCGB_CHECK_LAUNCH();
    return PCGB_OK;
  }
  if (!c->api) return fail(PCGB_ERR_NCCL, "allreduce: peer windows not exchanged and no NCCL communicator");
  PCGB_NCCL(c->api, c->api->AllReduce(d_buf, d_buf, (size_t)count, ncclFloat64, ncclSum, c->comm, st));
  return PCGB_OK;
}

}  // namespace pcgb
