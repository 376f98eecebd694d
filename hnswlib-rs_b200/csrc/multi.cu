// Multi-GPU search behind the C ABI (SURVEY §8e): the frozen index is replicated, queries are sharded.
//
// The reference's parallel_search (/root/reference/src/hnsw.rs:1612-1635) is ONE call that fans a batch out over the
// host's cores; here the same call fans it out over the GPUs of the box.  Two ways to get the replicas:
//   * one process, N devices (hnsw_b200_replicate): the library creates a replica Index per extra device, one
//     ncclCommInitAll communicator, and broadcasts every blob of the frozen index with grouped ncclBroadcast calls
//     over NVLink.  Afterwards search_flat / parallel_search_neighbours_<ty> split the batch into contiguous shards
//     (host_search.cu): one worker thread per device runs its shard (H2D, kernel, D2H) and writes its slice of the
//     caller's output, so there is no result gather at all for host results;
//   * one process per GPU (hnsw_b200_nccl_*): the host exchanges an ncclUniqueId by its own means (MPI, a TCP store,
//     torch.distributed ...), every rank opens the communicator on its handle's device, the building rank broadcasts
//     header + blobs, and device-resident answers can be all-gathered on a caller-chosen stream.
// NCCL is bound at run time (dlopen of libnccl.so.2): the library itself links nothing but cudart, and a host that
// already loaded an NCCL (torch) shares it.
#include <dlfcn.h>
#include <nccl.h>

#include "index.h"

namespace hb {

// ------------------------------------------------------------------------------------------------ NCCL binding
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommInitRankConfig)(ncclComm_t*, int, ncclUniqueId, int, ncclConfig_t*);  // may be null (NCCL < 2.17)
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  const char* (*GetErrorString)(ncclResult_t);
  bool ok = false;
  std::string why;
};

static NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // an NCCL the host already loaded (e.g. torch's)
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
      api.why = std::string("libnccl.so.2 not found: ") + dlerror();
      return;
    }
#define HB_SYM(field, name)                                          \
  api.field = reinterpret_cast<decltype(api.field)>(dlsym(h, name)); \
  if (!api.field) {                                                  \
    api.why = std::string("NCCL symbol missing: ") + name;           \
    return;                                                          \
  }
    HB_SYM(GetUniqueId, "ncclGetUniqueId")
    HB_SYM(CommInitRank, "ncclCommInitRank")
    HB_SYM(CommInitAll, "ncclCommInitAll")
    HB_SYM(CommDestroy, "ncclCommDestroy")
    HB_SYM(Broadcast, "ncclBroadcast")
    HB_SYM(AllGather, "ncclAllGather")
    HB_SYM(GroupStart, "ncclGroupStart")
    HB_SYM(GroupEnd, "ncclGroupEnd")
    HB_SYM(GetErrorString, "ncclGetErrorString")
#undef HB_SYM
    api.CommInitRankConfig = reinterpret_cast<decltype(api.CommInitRankConfig)>(dlsym(h, "ncclCommInitRankConfig"));
    api.ok = true;
  });
  return api;
}

#define HB_NCCL(call)                                                                                       \
  do {                                                                                                      \
    ncclResult_t r__ = (call);                                                                              \
    if (r__ != ncclSuccess) return fail(std::string("NCCL error: ") + nccl().GetErrorString(r__) + " at " #call); \
  } while (0)

void Index::drop_replicas() {
  DeviceRestore keep;
  workers_.resize(0);
  if (nccl().ok)
    for (void* c : comms_)
      if (c) nccl().CommDestroy((ncclComm_t)c);
  comms_.clear();
  replicas_.clear();
  replica_devices_.clear();
}

// broadcast the blobs of `this` (communicator rank 0) to the replicas (ranks 1..), then rebuild their host mirrors
int Index::broadcast_to_replicas() {
  DeviceRestore keep;
  NcclApi& nc = nccl();
  uint64_t header[16];
  blob_header(header);
  int r;
  for (auto& rep : replicas_) {
    if (rep->n != 0) {  // a stale copy: start from an empty index of the same configuration
      const int dev = rep->device;
      rep.reset(new Index(M, max_elements, max_layer, ef_c, metric, dtype, dev));
      if (!rep->ok()) return fail("replica: " + rep->err());
    }
    if ((r = rep->blob_alloc(header))) return fail("replica: " + rep->err());
  }
  HB_CUDA(cudaSetDevice(device));
  HB_CUDA(cudaStreamSynchronize(stream_));
  for (int b = 0; b < blob_count(); ++b) {
    void* src = nullptr;
    uint64_t bytes = 0;
    if ((r = blob_info(b, &src, &bytes))) return r;
    if (bytes == 0) continue;
    HB_NCCL(nc.GroupStart());
    HB_NCCL(nc.Broadcast(src, src, bytes, ncclChar, 0, (ncclComm_t)comms_[0], stream_));
    for (size_t i = 0; i < replicas_.size(); ++i) {
      void* dst = nullptr;
      uint64_t rb = 0;
      if (replicas_[i]->blob_info(b, &dst, &rb) || rb != bytes) {
        nc.GroupEnd();
        return fail("replica blob shape differs from the source index");
      }
      HB_NCCL(nc.Broadcast(dst, dst, bytes, ncclChar, 0, (ncclComm_t)comms_[i + 1], replicas_[i]->stream_));
    }
    HB_NCCL(nc.GroupEnd());
  }
  HB_CUDA(cudaSetDevice(device));
  HB_CUDA(cudaStreamSynchronize(stream_));
  for (auto& rep : replicas_) {
    HB_CUDA(cudaSetDevice(rep->device));
    HB_CUDA(cudaStreamSynchronize(rep->stream_));
    if ((r = rep->blob_commit())) return fail("replica: " + rep->err());
    rep->searching = true;
  }
  HB_CUDA(cudaSetDevice(device));
  replicas_stale_ = false;
  return 0;
}

int Index::replicate(int ndev, const int* devices) {
  DeviceRestore keep;
  if (ndev < 1 || !devices) return fail("replicate: need at least one device");
  if (devices[0] != device) return fail("replicate: devices[0] must be the device that holds the index");
  NcclApi& nc = nccl();
  if (ndev > 1 && !nc.ok) return fail("replicate: " + nc.why);
  int have = 0;
  HB_CUDA(cudaGetDeviceCount(&have));
  for (int i = 0; i < ndev; ++i) {
    if (devices[i] < 0 || devices[i] >= have) return fail("replicate: device index out of range");
    for (int j = 0; j < i; ++j)
      if (devices[j] == devices[i]) return fail("replicate: a device is named twice");
  }
  drop_replicas();
  if (ndev == 1) return 0;
  for (int i = 1; i < ndev; ++i) {
    replicas_.emplace_back(new Index(M, max_elements, max_layer, ef_c, metric, dtype, devices[i]));
    if (!replicas_.back()->ok()) {
      const std::string why = replicas_.back()->err();
      drop_replicas();
      return fail("replicate: " + why);
    }
  }
  replica_devices_.assign(devices, devices + ndev);
  std::vector<ncclComm_t> cs(ndev);
  const ncclResult_t ir = nc.CommInitAll(cs.data(), ndev, devices);
  if (ir != ncclSuccess) {
    drop_replicas();  // no half-made replica set: the handle goes on answering from its own device
    return fail(std::string("replicate: ncclCommInitAll: ") + nc.GetErrorString(ir));
  }
  comms_.assign(cs.begin(), cs.end());
  workers_.resize(ndev - 1);
  int r = broadcast_to_replicas();
  if (r) drop_replicas();
  HB_CUDA(cudaSetDevice(device));
  return r;
}

// tickets of submitted batches (hnsw_b200_search_flat_submit / _wait)
int64_t Index::park_ticket(Ticket&& t) {
  std::lock_guard<std::mutex> lk(ticket_mu_);
  const int64_t id = next_ticket_++;
  tickets_[id] = std::move(t);
  return id;
}
bool Index::take_ticket(int64_t id, Ticket& out) {
  std::lock_guard<std::mutex> lk(ticket_mu_);
  auto it = tickets_.find(id);
  if (it == tickets_.end()) return false;
  out = std::move(it->second);
  tickets_.erase(it);
  return true;
}

// ------------------------------------------------------------------------------------------------ one process per GPU
int Index::nccl_unique_id(unsigned char* out128) {
  NcclApi& nc = nccl();
  if (!nc.ok) return -1;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  if (nc.GetUniqueId(&id) != ncclSuccess) return -1;
  memcpy(out128, &id, 128);
  return 0;
}

int Index::nccl_init(int nranks, int rank, const unsigned char* id128) {
  DeviceRestore keep;
  NcclApi& nc = nccl();
  if (!nc.ok) return fail("nccl_init: " + nc.why);
  if (nranks < 1 || rank < 0 || rank >= nranks) return fail("nccl_init: bad rank");
  if (comm_) {
    nc.CommDestroy((ncclComm_t)comm_);
    comm_ = nullptr;
  }
  HB_CUDA(cudaSetDevice(device));
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  ncclComm_t c;
  if (nc.CommInitRankConfig) {
    // the gathers of this communicator run next to search kernels that fill every SM: keep them to a few CTAs, so that a
    // gather waiting for its peers does not park thousands of threads
    ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
    cfg.minCTAs = 1;
    cfg.maxCTAs = 2;
    HB_NCCL(nc.CommInitRankConfig(&c, nranks, id, rank, &cfg));
  } else {
    HB_NCCL(nc.CommInitRank(&c, nranks, id, rank));
  }
  comm_ = c;
  nranks_ = nranks;
  rank_ = rank;
  return 0;
}

int Index::nccl_broadcast_index(int root) {
  DeviceRestore keep;
  NcclApi& nc = nccl();
  if (!comm_) return fail("nccl_broadcast_index: call hnsw_b200_nccl_init first");
  if (root < 0 || root >= nranks_) return fail("nccl_broadcast_index: bad root");
  HB_CUDA(cudaSetDevice(device));
  DevBuf hdr;
  HB_CUDA(cudaMalloc(&hdr.p, 16 * sizeof(uint64_t)));
  uint64_t* d_hdr = (uint64_t*)hdr.p;
  uint64_t header[16];
  if (rank_ == root) {
    blob_header(header);
    HB_CUDA(cudaMemcpyAsync(d_hdr, header, sizeof(header), cudaMemcpyHostToDevice, stream_));
  }
  HB_NCCL(nc.Broadcast(d_hdr, d_hdr, sizeof(header), ncclChar, root, (ncclComm_t)comm_, stream_));
  HB_CUDA(cudaMemcpyAsync(header, d_hdr, sizeof(header), cudaMemcpyDeviceToHost, stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  int r;
  if (rank_ != root && (r = blob_alloc(header))) return r;
  for (int b = 0; b < blob_count(); ++b) {
    void* ptr = nullptr;
    uint64_t bytes = 0;
    if ((r = blob_info(b, &ptr, &bytes))) return r;
    if (bytes) HB_NCCL(nc.Broadcast(ptr, ptr, bytes, ncclChar, root, (ncclComm_t)comm_, stream_));
  }
  HB_CUDA(cudaStreamSynchronize(stream_));
  if (rank_ != root) {
    if ((r = blob_commit())) return r;
    searching = true;
  }
  return 0;
}

int Index::nccl_allgather(const void* d_send, void* d_recv, size_t bytes_per_rank, cudaStream_t s) {
  DeviceRestore keep;
  NcclApi& nc = nccl();
  if (!comm_) return fail("nccl_allgather: call hnsw_b200_nccl_init first");
  HB_CUDA(cudaSetDevice(device));
  HB_NCCL(nc.AllGather(d_send, d_recv, bytes_per_rank, ncclChar, (ncclComm_t)comm_, s ? s : stream_));
  return 0;
}

void Index::nccl_destroy() {
  if (comm_ && nccl().ok) nccl().CommDestroy((ncclComm_t)comm_);
  comm_ = nullptr;
}

}  // namespace hb
