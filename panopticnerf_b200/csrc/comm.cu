// comm.cu — the multi-GPU entry points of the C ABI (SURVEY.md 8(b) "Multi-GPU entry", 8(e)): one NCCL
// communicator per context and ONE all-gather of the rendered per-ray tiles (image / label tiles) over NVLink.
// Rays shard with no data-path collective; this gather is the only exchange step on the path.  Data-parallel
// training (lib/train/data_parallel.py) reuses the same all-gather for its gradients and counts, and a broadcast once
// at start-up.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, the soname both the system package and the PyTorch wheel
// install): libpnr keeps loading on boxes without NCCL, and inside a PyTorch process the already-loaded copy is
// reused instead of a second NCCL being pulled in.
#include <dlfcn.h>
#include <mutex>
#include "common.cuh"

namespace pnr {

// Minimal NCCL surface, declared here so that no NCCL header version is baked in (the ABI of these six
// functions has been stable across NCCL 2.x).
struct NcclUniqueId { char internal[PNR_COMM_ID_BYTES]; };
typedef struct ncclComm* NcclComm;
typedef int NcclResult;   // 0 = ncclSuccess
enum { kNcclUint8 = 1 };  // ncclUint8

struct NcclApi {
  NcclResult (*GetUniqueId)(NcclUniqueId*) = nullptr;
  NcclResult (*CommInitRank)(NcclComm*, int, NcclUniqueId, int) = nullptr;
  NcclResult (*CommDestroy)(NcclComm) = nullptr;
  NcclResult (*AllGather)(const void*, void*, size_t, int, NcclComm, cudaStream_t) = nullptr;
  NcclResult (*Broadcast)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(NcclResult) = nullptr;
  NcclResult (*GetVersion)(int*) = nullptr;
  bool ok = false;
  char why[256] = "";
};

static NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
      snprintf(api.why, sizeof(api.why), "libnccl.so.2 not found (%s)", dlerror());
      return;
    }
    auto sym = [&](const char* name) -> void* {
      void* p = dlsym(h, name);
      if (!p && !api.why[0]) snprintf(api.why, sizeof(api.why), "libnccl lacks %s", name);
      return p;
    };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
    api.Broadcast = (decltype(api.Broadcast))sym("ncclBroadcast");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Broadcast &&
             api.GetErrorString;
  });
  return api;
}

#define PNR_NCCL(call)                                                                            \
  do {                                                                                            \
    NcclResult r__ = (call);                                                                      \
    if (r__ != 0)                                                                                 \
      return ::pnr::set_error(PNR_ERR_CUDA, "%s failed: %s", #call, nccl().GetErrorString(r__)); \
  } while (0)

struct Comm {
  NcclComm comm = nullptr;
  int rank = 0, world = 1, device = 0;
};

}  // namespace pnr

using namespace pnr;

struct pnr_comm : Comm {};

extern "C" int pnr_comm_available(void) { return nccl().ok ? 1 : 0; }

extern "C" int pnr_comm_unique_id(uint8_t* id_out) {
  PNR_CHECK_ARG(id_out, "pnr_comm_unique_id: null pointer");
  if (!nccl().ok) return set_error(PNR_ERR_UNSUPPORTED, "pnr_comm_unique_id: NCCL unavailable: %s", nccl().why);
  NcclUniqueId id;
  PNR_NCCL(nccl().GetUniqueId(&id));
  memcpy(id_out, id.internal, PNR_COMM_ID_BYTES);
  return PNR_OK;
}

extern "C" int pnr_comm_init(pnr_comm** out, const uint8_t* id, int32_t rank, int32_t world, int32_t device) {
  PNR_CHECK_ARG(out && id, "pnr_comm_init: null pointer");
  PNR_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "pnr_comm_init: rank %d of %d", rank, world);
  if (!nccl().ok) return set_error(PNR_ERR_UNSUPPORTED, "pnr_comm_init: NCCL unavailable: %s", nccl().why);
  int ndev = 0;
  PNR_CUDA(cudaGetDeviceCount(&ndev));
  PNR_CHECK_ARG(device >= 0 && device < ndev, "pnr_comm_init: device %d of %d", device, ndev);
  DeviceGuard guard(device);
  NcclUniqueId uid;
  memcpy(uid.internal, id, PNR_COMM_ID_BYTES);
  pnr_comm* c = new pnr_comm();
  c->rank = rank; c->world = world; c->device = device;
  const NcclResult r = nccl().CommInitRank(&c->comm, world, uid, rank);
  if (r != 0) {
    delete c;
    return set_error(PNR_ERR_CUDA, "ncclCommInitRank(rank %d of %d) failed: %s", rank, world, nccl().GetErrorString(r));
  }
  *out = c;
  return PNR_OK;
}

extern "C" int pnr_comm_destroy(pnr_comm* comm) {
  if (!comm) return PNR_OK;
  DeviceGuard guard(comm->device);
  if (comm->comm) nccl().CommDestroy(comm->comm);
  delete comm;
  return PNR_OK;
}

// recv [world * bytes_per_rank] <- every rank's send [bytes_per_rank], in rank order; in place when
// send == recv + rank * bytes_per_rank.  Asynchronous on `stream`.
extern "C" int pnr_allgather_outputs(pnr_comm* comm, const void* send, void* recv, size_t bytes_per_rank,
                                     void* stream) {
  PNR_CHECK_ARG(comm, "pnr_allgather_outputs: null communicator");
  if (bytes_per_rank == 0) return PNR_OK;
  PNR_CHECK_ARG(send && recv, "pnr_allgather_outputs: null pointer");
  DeviceGuard guard(comm->device);
  PNR_NCCL(nccl().AllGather(send, recv, bytes_per_rank, kNcclUint8, comm->comm, (cudaStream_t)stream));
  return PNR_OK;
}

// buf [bytes] <- root's buf on every rank, in place.  Asynchronous on `stream`.
extern "C" int pnr_broadcast(pnr_comm* comm, void* buf, size_t bytes, int32_t root, void* stream) {
  PNR_CHECK_ARG(comm, "pnr_broadcast: null communicator");
  PNR_CHECK_ARG(root >= 0 && root < comm->world, "pnr_broadcast: root %d of %d", root, comm->world);
  if (bytes == 0) return PNR_OK;
  PNR_CHECK_ARG(buf, "pnr_broadcast: null pointer");
  DeviceGuard guard(comm->device);
  PNR_NCCL(nccl().Broadcast(buf, buf, bytes, kNcclUint8, root, comm->comm, (cudaStream_t)stream));
  return PNR_OK;
}
