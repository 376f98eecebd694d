// Host side of the engine: owns the HBM-resident index, schedules insert batches and query
// launches.  Replaces, above the kernels, what PointIndexation / Hnsw::new / parallel_insert /
// parallel_search do on the CPU in the reference (/root/reference/src/hnsw.rs:395-557, 739-905,
// 1224-1238, 1612-1635): point bookkeeping (level draw, PointId ranks, entry point), and the
// rayon fan-out, which here is a persistent-warp kernel launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <functional>
#include <map>
#include <memory>
#include <condition_variable>
#include <mutex>
#include <shared_mutex>
#include <tuple>
#include <string>
#include <thread>
#include <vector>

#include "kernels.h"

namespace hb {

struct SplitMix64 {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double unif() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

// restores the calling thread's current device on scope exit (the library switches devices when it works on replicas;
// a host that tracks the current device itself, e.g. torch, must find it unchanged after every call)
struct DeviceRestore {
  int prev = -1;
  DeviceRestore() { cudaGetDevice(&prev); }
  ~DeviceRestore() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// in an Index member: a failed CUDA call returns its status (-2) with the message set
#define HB_CUDA(call)                                     \
  do {                                                    \
    cudaError_t e__ = (call);                             \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)

struct DevBuf {  // device memory freed on scope exit, so that no early return leaks it
  void* p = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { cudaFree(p); }
};

// The device arrays that hold the graph.  Replication blob i is array i, in this order (the order is part of the blob
// protocol between processes); the per-point insert locks come last and are not replicated.
struct GraphStore {
  enum Array { VEC, ADJ0, ADJU, UP_OFF, PLEVEL, LEVEL, ORIGIN, ADJ0_D, ADJU_D, LOCKS, COUNT };
  static constexpr int BLOBS = LOCKS;
  // elements per point: a vector row (row_bytes), a layer-0 list (2M), one; or per upper-layer list: a list (M)
  enum Row { VEC_ROW, LIST0, ONE, LISTU };
  struct Desc {
    int elem;  // bytes per element
    Row row;
    int fill;  // byte new space is filled with
  };
  static constexpr Desc DESC[COUNT] = {
      {1, VEC_ROW, 0},   // VEC: zero padded to whole 128-byte lines
      {4, LIST0, 0xFF},  // ADJ0: neighbour ids, INVALID_ID = empty slot
      {4, LISTU, 0xFF},  // ADJU
      {4, ONE, 0xFF},    // UP_OFF: the point's first upper-layer list, INVALID_ID = none
      {1, ONE, 0},       // PLEVEL
      {1, ONE, 0},       // LEVEL
      {8, ONE, 0},       // ORIGIN
      {4, LIST0, 0},     // ADJ0_D: neighbour distances
      {4, LISTU, 0},     // ADJU_D
      {4, ONE, 0},       // LOCKS
  };
  void* p[COUNT] = {};
  size_t cap = 0, cap_ul = 0;  // points / upper-layer lists allocated
  template <class T>
  T* at(Array a) const { return static_cast<T*>(p[a]); }
};

struct DumpDescription {  // Description, /root/reference/src/hnswio.rs:846-870
  int format_version = 0;
  uint8_t dumpmode = 0, max_nb_connection = 0, nb_layer = 0;
  double level_scale = 1.0;
  uint64_t ef = 0, nb_point = 0, dimension = 0;
  std::string distname, t_name;
  long header_bytes = 0;
};
int read_description(const std::string& graph_path, DumpDescription& out, std::string& err);
int metric_from_name(const std::string& name);       // "DistL2" -> METRIC_L2; -1 if unknown
int metric_from_type_name(const std::string& full);  // the same on the last `::` segment of a type path
int dtype_from_type_name(const std::string& s);

class Index;

// The points an exact scan (exact_knn_kernel, aux.cu) covers: `ids`, n sorted internal ids on the scanning device, or
// every stored point (ids == nullptr)
struct ExactScan {
  const uint32_t* ids = nullptr;
  size_t n = 0;
};

// rows [first, first + count) of an exact launch with a filter per query, all scanning the same points
struct ExactGroup {
  size_t first, count;
  ExactScan scan;
};

// Resident filters (hnsw_b200_filter_new, filter_store.cu): a FilterT materialised once per handle, as one bitmap per
// partition (one for an ordinary handle) over the points stored when it was made.  The host copy stays; each device a
// search uses it on gets one device copy, made at its first use there.  Ids are unique over all handles, so an id that
// belongs to another handle is unknown here.  A search takes the handle's lock shared and uses a filter under it; free
// takes it exclusively, so a filter is never freed while a search holds it.
class FilterStore {
 public:
  struct Filter {
    std::vector<std::vector<uint32_t>> bits;  // [partition] bit per internal id (make_filter_bits)
    std::vector<size_t> counts;               // [partition] points stored when the filter was made
    std::map<std::pair<int, int>, void*> dev;  // (partition, device) -> device copy of bits[partition]
    // (partition, device) -> the admitted internal ids of bits[partition], sorted, on the device, and their count; made
    // at the first exact search with the filter there
    std::map<std::pair<int, int>, std::pair<void*, size_t>> ids;
  };
  FilterStore() = default;
  FilterStore(const FilterStore&) = delete;
  FilterStore& operator=(const FilterStore&) = delete;
  ~FilterStore();  // frees every device copy (the owner has synchronised its streams)
  int64_t add(Filter&& f);
  bool has(int64_t id);
  // the device copy of partition p's bitmap on rx's device (copied there on first use), after checking that the filter
  // exists and that rx, partition p of `nparts`, still holds the points the filter was made over; if not, rx's error.
  // With `list`, the sorted id list of the admitted points instead (made and copied there on first use).
  int use(int64_t id, int p, int nparts, const Index* rx, const uint32_t** d_bits, ExactScan* list = nullptr);
  void erase(int64_t id);  // frees its device copies; the caller waited for every search that may read them

 private:
  std::mutex mu_;
  std::map<int64_t, Filter> f_;
};

class Partitions;  // partition.cu: the points of one handle split over several Index objects
struct PartitionsDeleter {
  void operator()(Partitions* p) const;
};

// One thread that runs the closures its owner hands it, one at a time.
struct Worker {
  std::thread th;
  std::mutex m;
  std::condition_variable cv;
  std::function<void()> job;
  bool has_job = false, done = true, quit = false;
  Worker();
  ~Worker();
  void submit(std::function<void()> j);
  void wait();
};

// The worker threads of a fan-out over devices (replicas) or partitions: run(n, job) runs job(0) on the calling thread
// and job(i) on worker i - 1, all at once, waits for every one and returns the first i whose job failed (-1: none).
// One run at a time (a worker holds one job); `mu` is the lock run takes.
class WorkerGroup {
 public:
  void resize(size_t n);  // n workers
  int run(int n, const std::function<int(int)>& job);
  std::mutex mu;

 private:
  std::vector<std::unique_ptr<Worker>> w_;
};

// ---- host searches (host_search.cu)
// Where a host search writes its [nq][k] answer slots and counts[nq]: either the reference entry points' answer blocks
// (`nb`: Neighbour_api with the internal id in its tail padding) or hnsw_b200_search_flat's arrays (internal and pid
// optional).
struct AnswerArrays {
  NeighbourOut* nb = nullptr;
  uint64_t* ids = nullptr;
  float* dist = nullptr;
  uint32_t* internal = nullptr;
  int32_t* pid = nullptr;
  int32_t* counts = nullptr;
  const size_t* perm = nullptr;  // row j of the batch is written to row perm[j] (nullptr: to row j)
};

// The filter of a search: none, a FilterT (mode != 0, as make_filter_bits reads it: 1 sorted origin-id list, 2 callback),
// or one of the handle's resident filters (the id *resident).
struct FilterArg {
  int mode = 0;
  const uint64_t* ids = nullptr;
  size_t nids = 0;
  int (*fn)(uint64_t, void*) = nullptr;
  void* ctx = nullptr;
  const int64_t* resident = nullptr;
};

// One host search batch: flat queries or one pointer per query (rows), k answers each into `out`.  `exact`: the exact
// scan of the points the filter admits (ef unused) instead of the graph search.
struct HostBatch {
  const void* queries = nullptr;
  const void* const* rows = nullptr;
  size_t nq = 0;
  int d = 0;
  size_t k = 0, ef = 0;
  FilterArg filter;
  AnswerArrays out;
  bool exact = false;
  const int64_t* per_query = nullptr;  // [nq]: each query's resident filter, or -1 for none (then `filter` is unused)
};

// A leg's share of a batch with a filter per query, whose rows the driver sorted by filter (resolve_per_query): the
// leg's first `plain` rows have no filter.  Graph search: its row plain + i uses bitmap table[sel[i]].  Exact scan:
// `groups`, its rows by the points they scan (every point for the plain rows).
struct LegFilters {
  bool on = false;
  size_t plain = 0;
  std::vector<const uint32_t*> table;
  std::vector<uint32_t> sel;
  std::vector<ExactGroup> groups;
};

// One Index's part of a batch: queries [first, first + count) searched on rx (the handle, a replica, or partition `part`)
// on its leased context ctx, with the filter bits resolve_filter gave it, or for an exact batch the points to scan
struct Leg {
  Index* rx = nullptr;
  int part = 0;
  size_t first = 0, count = 0;
  int ctx = -1;  // -1: not leased
  const uint32_t* host_bits = nullptr;
  const uint32_t* dev_bits = nullptr;
  ExactScan scan;
  bool begun = false;  // enqueued
  int rc = 0;
  LegFilters pq;
};

class Index {
 public:
  Index(int M, size_t max_elements, int max_layer, int ef_c, int metric, int dtype, int device);
  ~Index();
  bool ok() const { return ok_; }

  // ---- configuration (Hnsw::new and setters, hnsw.rs:771-905)
  int M, max_layer, ef_c, metric, dtype, es, device;  // es = bytes per element
  size_t max_elements;
  bool extend_candidates = false, keep_pruned = false, searching = false;
  int link_mode = 0;      // hnsw_b200_set_link_mode: 0 back-links under the new point's level (hnsw.rs:1257), 1 per layer
  bool tie_std_ = false;  // hnsw_b200_set_tie_mode: equal-distance ties resolved like the reference's std BinaryHeaps (search_std.cu)
  double level_scale;  // 1/ln(M) * factor
  SplitMix64 rng{397};
  uint32_t batch_ratio = 16, batch_max = 16384;

  // ---- state
  int dim = 0, row_bytes = 0;  // row_bytes = dim*es rounded up to whole 128-byte lines
  size_t n = 0;          // points stored (all linked: inserts are synchronous per call)
  size_t n_ul = 0;       // upper lists allocated
  size_t layer_count[MAX_LAYERS];
  uint32_t entry = INVALID_ID;
  int entry_level = -1;
  std::vector<uint8_t> h_level, h_plevel;
  std::vector<int32_t> h_rank;
  std::vector<uint64_t> h_origin;
  std::vector<uint32_t> h_upoff;

  // ---- operations (return 0 or a negative status; message in err())
  int set_dim(int d);
  int draw_level();
  int insert_batch(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
                   const int32_t* levels);
  int import_graph(const void* vecs, size_t n_new, int d, const uint64_t* origin, const uint8_t* levels,
                   int64_t entry_id, int nlayers, const uint64_t* const* offsets, const uint32_t* const* ids,
                   const float* const* dists);
  // host queries (flat or row pointers) on leased context c, answers left in the context's pinned buffer (valid until
  // it is released).  The filter is either host bits, uploaded into the context for this call, or d_filter_bits already
  // on this device (a resident filter); at most one of the two is non-null.  With `scan`, the exact scan of those points
  // instead of the graph search (no filter bits, ef unused).  With `pq` (pq->on; no filter bits and no scan), a filter
  // per query.
  int search_host_begin(int c, const void* queries, const void* const* rows, size_t nq, int d, size_t k, size_t ef,
                        const uint32_t* filter_bits_host, const uint32_t* d_filter_bits, const ExactScan* scan = nullptr,
                        const LegFilters* pq = nullptr);
  int search_host_finish(int c, const NeighbourOut** out, const int32_t** counts);
  // host search batches (host_search.cu): synchronous, or submitted now and collected by finish_batch
  struct Ticket {
    std::vector<Leg> legs;
    size_t k = 0;
    AnswerArrays out;
  };
  int search_batch(const HostBatch& b);
  int64_t submit_batch(const HostBatch& b);  // a ticket id, or < 0
  int finish_batch(Ticket& t);
  // submitted-but-not-waited host searches: anything that changes the graph waits for them (drain_pending)
  std::atomic<int> pending_{0};
  void drain_pending() const {
    while (pending_.load() != 0) std::this_thread::yield();
  }
  // the filter bits of legs[0, n): a FilterT's host bits, made on the calling thread once per partition (a replica
  // shares the handle's internal ids, and so its bits) into `bits`, or a resident filter's copy on each leg's device.
  // Nonzero when a leg could not have them; that leg's rc is set (legs_fail reports it).  `exact`: each leg's ExactScan
  // instead (the resident filter's id list on the leg's device, or every point).
  int resolve_filter(const FilterArg& f, bool exact, Leg* legs, size_t n, std::vector<std::vector<uint32_t>>& bits);
  // a batch with a filter per query: every entry of filters[0, nq) is -1 or a live, current filter of this handle (else
  // the first bad position is refused), and `perm` orders the rows stably by filter, the unfiltered ones first
  int sort_per_query(const int64_t* filters, size_t nq, std::vector<size_t>& perm);
  // each leg's LegFilters for the rows sorted by filter (sorted[j]: the filter of sorted row j), on its partition and
  // device; nonzero when a leg could not have them, with that leg's rc set
  int resolve_per_query(const std::vector<int64_t>& sorted, bool exact, Leg* legs, size_t n);
  // device queries in, device answers out; the filter is none or a resident filter.  `exact`: the exact scan (ef unused).
  int search_device(const FilterArg& f, bool exact, const void* d_queries, size_t nq, size_t k, size_t ef, NeighbourOut* d_out,
                    int32_t* d_counts, bool sync, float* kernel_ms);
  // filter materialisation: bit per internal id from a sorted origin-id list or a callback
  int make_filter_bits(int mode, const uint64_t* sorted_ids, size_t nids, int (*fn)(uint64_t, void*), void* ctx,
                       std::vector<uint32_t>& bits) const;
  // resident filters of this handle; free_filter waits for the asynchronous device-resident launches that may still read
  // the filter (the caller holds the handle exclusively, so no other search and no submitted batch is left)
  FilterStore filters;
  // a resident filter over every stored point (every partition's, on a partitioned handle): its id (>= 0), or < 0
  int64_t new_filter(int mode, const uint64_t* sorted_ids, size_t nids, int (*fn)(uint64_t, void*), void* ctx);
  int free_filter(int64_t id);

  int export_layer(int layer, uint64_t* offsets, uint32_t* ids, float* dists, int64_t* total) const;
  int export_vectors(void* out) const;
  // FlatNeighborhood (/root/reference/src/flatten.rs:50-126): per point, the neighbours of ALL layers merged and
  // sorted by distance; CSR over internal ids, neighbours named by origin id
  int flatten(std::vector<uint64_t>& offsets, std::vector<uint64_t>& nb_origin, std::vector<float>& nb_dist) const;
  // dump / reload in the reference's two-file format (hnswio.cu)
  int file_dump(const std::string& dir, const std::string& basename, bool overwrite, std::string* used_basename);
  int load_dump(const std::string& dir, const std::string& basename);
  int enable_stats(bool on);
  int get_stats(uint64_t* out4, bool reset);

  // replication blobs
  int blob_header(uint64_t* h16) const;
  int blob_alloc(const uint64_t* h16);
  int blob_count() const { return GraphStore::BLOBS; }
  int blob_info(int i, void** p, uint64_t* bytes) const;
  int blob_commit();

  // ---- multi-GPU (multi.cu).  One process, N devices: replicate() builds a copy of the frozen index on every listed
  // device (NCCL broadcast), and a host search batch is split into contiguous shards over them, one worker thread per
  // device (host_search.cu).  One process per GPU: nccl_init() + nccl_broadcast_index() + nccl_allgather().
  int replicate(int ndev, const int* devices);
  size_t replica_count() const { return replicas_.size(); }
  int64_t park_ticket(Ticket&& t);
  bool take_ticket(int64_t id, Ticket& out);
  void drop_replicas();
  static int nccl_unique_id(unsigned char* out128);
  int nccl_init(int nranks, int rank, const unsigned char* id128);
  int nccl_broadcast_index(int root);
  int nccl_allgather(const void* d_send, void* d_recv, size_t bytes_per_rank, cudaStream_t s);
  void nccl_destroy();

  // ---- search contexts.  Everything a running search owns besides the (read-only) graph: stream, work counter,
  // status flag, visited tables, staging buffers.  Up to NCTX searches are in flight at once: calls from several host
  // threads (the reference serves concurrent searches, hnsw.rs:830-833) and consecutive asynchronous device-resident
  // launches, whose last queries then overlap the next launch's first (a launch ends with a few long searches that
  // leave most SMs idle).
  struct VisitedPool {
    uint32_t* tab = nullptr;
    uint32_t* epoch = nullptr;
    size_t slots = 0, cap = 0;
    int id_bits = 0;
  };
  struct SearchCtx {
    cudaStream_t stream = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr, ev0 = nullptr, ev1 = nullptr;
    unsigned int* d_counter = nullptr;
    int* d_status = nullptr;
    VisitedPool vis, fvis;  // unfiltered / filtered searches
    void *d_fbits = nullptr, *d_cbuf = nullptr;  // the call's filter bits (or its per-query bitmap table and selectors) / C
    size_t d_fbits_bytes = 0, d_cbuf_bytes = 0;
    void *d_xq = nullptr, *d_xpart = nullptr;  // exact scan: the host batch's queries on the device / tickets and slice lists
    size_t d_xq_bytes = 0, d_xpart_bytes = 0;
    void *h_pin = nullptr, *h_res = nullptr;  // pinned, mapped: query staging / answers
    size_t h_pin_bytes = 0, h_res_bytes = 0;
    bool busy = false;
    struct Pending {  // a host search enqueued by search_host_begin, completed by search_host_finish
      const void* d_queries = nullptr;
      const uint32_t* dfb = nullptr;
      bool exact = false;  // an exact scan: no status, nothing to re-run
      // a filter per query: rows [0, plain) unfiltered, the others on the device bitmap table / selectors
      bool per_query = false;
      size_t plain = 0;
      const uint32_t* const* ftab = nullptr;
      const uint32_t* fsel = nullptr;
      NeighbourOut *k_out = nullptr, *hout = nullptr;
      int32_t *k_cnt = nullptr, *hcnt = nullptr, *hstatus = nullptr;
      size_t nq = 0, k = 0, ef = 0;
      bool enqueued = false;
    } pend;
  };
  static constexpr int NCTX = 4;    // leased by synchronous calls (host threads)
  static constexpr int NASYNC = 2;  // alternated by asynchronous device-resident launches (never leased)
  int acquire_ctx();            // blocks until a context is free
  void release_ctx(int c);
  SearchCtx& ctx(int c) { return ctx_[c]; }
  struct CtxLease {             // RAII: a context leased for the scope
    Index* ix;
    int c;
    explicit CtxLease(Index* i) : ix(i), c(i->acquire_ctx()) {}
    ~CtxLease() { ix->release_ctx(c); }
    CtxLease(const CtxLease&) = delete;
    CtxLease& operator=(const CtxLease&) = delete;
  };

  int dist_batch(const void* queries, size_t nq, int d, const uint32_t* cand, size_t m, float* out);
  int bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist);

  std::string err() const;
  GraphView view() const;
  cudaStream_t stream() const { return stream_; }
  int join();                           // the handle's stream waits for every asynchronous launch enqueued so far
  int stream_wait_last(cudaStream_t s);  // `s` waits for the most recent asynchronous launch
  int set_stream(cudaStream_t s);   // run on a caller-owned stream (e.g. torch's current stream); nullptr = own stream
  int check_status();               // synchronise; 0 ok, 1 = a visited table overflowed since the last check
  // the C ABI allows calls from many host threads (hnsw.rs:830-833): searches share the graph, anything that changes it
  // (insert, import, load, replicate) holds it exclusively
  mutable std::shared_mutex mu;

  // ---- partitions (partition.cu).  A partitioned handle keeps its settings and level RNG here and its points in `parts`;
  // each partition is an Index of its own whose `owner` is that handle (the C ABI serves it read-only, as a view).
  std::unique_ptr<Partitions, PartitionsDeleter> parts;
  const Index* owner = nullptr;

 private:
  friend class Partitions;
  friend class FilterStore;
  int fail(const std::string& m) const;
  int cuda_fail(cudaError_t e, const char* what) const;
  // ---- graph store
  size_t row_size(int a) const;  // bytes of array a per point (per upper-layer list for ADJU, ADJU_D)
  int grow_store(bool per_list, size_t cap, size_t keep);
  int ensure_points(size_t need);
  int ensure_upper(size_t need_lists);
  // ---- point ledger: the host mirrors (h_level ... h_upoff) and the per-layer counts
  void resize_points(size_t count);
  void rank_points();  // layer_count and h_rank from h_level, in internal-id order
  int upload_points(size_t first, size_t count);  // level, plevel, origin, up_off of [first, first + count)
  // ---- graph export
  struct ListRef {  // a point's list at one layer: adj0 (layer 0) or adjU from element `at`, `cap` slots (0: none)
    size_t at, cap;
  };
  ListRef list_of(size_t p, int layer) const;
  struct LayerCsr {  // one layer over internal ids: point p's neighbours are ids / dists [off[p], off[p + 1])
    std::vector<uint64_t> off;
    std::vector<uint32_t> ids;
    std::vector<float> dists;
  };
  int export_layers(int lo, int hi, std::vector<LayerCsr>& out) const;  // out[l - lo] for layers lo..hi
  int top_layer() const;  // highest layer any point is present at
  // ---- insert launch
  struct InsertShape {
    int q_kind, q_smem;
    size_t smem_per_warp;
  };
  InsertShape insert_shape() const;
  int ensure_visited(VisitedPool& v, size_t slots, size_t cap_entries, cudaStream_t st);
  int fill_visited_cfg(VisitedPool& v, VisitedCfg& c, cudaStream_t st);
  int ensure_scratch(void** p, size_t* cur, size_t need, cudaStream_t st);
  int ensure_pinned(void** p, size_t* cur, size_t need, unsigned int flags);
  int grow_plevel(uint32_t id, int new_plevel);
  int run_insert_range(size_t first, size_t count, size_t mask_off);
  int check_insert_fit();
  void rollback_points(size_t keep);

  // ---- host search batches (host_search.cu)
  int plan(size_t nq, std::vector<Leg>& legs);
  void begin_leg(const HostBatch& b, Leg& l);
  void release_leg(Leg& l);
  int end_leg(Leg& l, size_t k, const AnswerArrays& out);
  int legs_fail(const Leg* legs, size_t n, bool replicas_first);

  int broadcast_to_replicas();
  std::vector<std::unique_ptr<Index>> replicas_;  // replicas_[i] lives on replica_devices_[i + 1]
  WorkerGroup workers_;                           // worker i serves replicas_[i]
  std::vector<void*> comms_;                      // ncclComm_t per device, rank 0 = this index
  std::vector<int> replica_devices_;
  bool replicas_stale_ = false;                   // the index changed after the last broadcast
  void* comm_ = nullptr;                          // ncclComm_t of the one-process-per-GPU mode
  int nranks_ = 1, rank_ = 0;

  bool ok_ = false;
  bool poisoned_ = false;  // a CUDA failure interrupted an insert: the graph may hold half-written links
  std::string poison_msg_;
  mutable std::string err_;
  mutable std::mutex err_mu_;
  cudaStream_t stream_ = nullptr, own_stream_ = nullptr;
  int sm_count_ = 0;

  GraphStore graph_;

  VisitedPool vis_;  // visited tables of the insert kernel (searches: SearchCtx)
  SearchCtx ctx_[NCTX + NASYNC];
  // d_ftab / d_fsel: a filter per query, query i on bitmap d_ftab[d_fsel[i]] (then d_filter_bits is null)
  int search_on_ctx(SearchCtx& c, const void* d_queries, size_t nq, size_t k, size_t ef_arg, const uint32_t* d_filter_bits,
                    NeighbourOut* d_out, int32_t* d_counts, bool sync, float* kernel_ms,
                    const uint32_t* const* d_ftab = nullptr, const uint32_t* d_fsel = nullptr);
  // the exact k nearest of device queries among scan's points (aux.cu); the slices' scratch is sized before the launch.
  // With `groups` (a filter per query), each group's rows among that group's points instead of scan's.
  int exact_on_ctx(SearchCtx& c, const void* d_queries, size_t nq, size_t k, const ExactScan& scan, NeighbourOut* d_out,
                   int32_t* d_counts, bool sync, float* kernel_ms, const std::vector<ExactGroup>* groups = nullptr);
  // the graph search of a per-query leg on context c: the plain rows' launch, then the filtered rows' launch
  int per_query_on_ctx(SearchCtx& c, bool sync);
  std::mutex ctx_mu_;
  std::condition_variable ctx_cv_;
  std::mutex ticket_mu_;
  std::map<int64_t, Ticket> tickets_;
  int64_t next_ticket_ = 0;
  int last_async_ = -1;
  unsigned ctx_rr_ = 0;        // round robin of the asynchronous device-resident launches
  std::mutex occ_mu_;

  // small device scratch (insert path; searches: SearchCtx)
  unsigned int* d_counter_ = nullptr;
  int* d_status_ = nullptr;
  unsigned long long* d_stats_ = nullptr;
  bool stats_on_ = false;
  std::atomic<uint64_t> stat_queries_{0};

  // staging of the insert path
  void* h_pin_ = nullptr;
  size_t h_pin_bytes_ = 0;
  // (kernel, queue kind, queue slots, warps per CTA, d4, shared memory per CTA) -> CTAs per SM
  std::map<std::tuple<QueryKernel, int, int, int, int, size_t>, int> occ_cache_;
  void* d_mask_ = nullptr;
  size_t d_mask_bytes_ = 0;
};

}  // namespace hb
