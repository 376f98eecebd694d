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
#include <unordered_map>
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

// One allocation, owned: device memory (cudaMalloc) or, Pinned, page-locked host memory (cudaHostAlloc with the
// caller's flags).  It is made on the current device and freed on that device, the caller's current device kept; an
// empty one makes no CUDA call.  reset frees, then allocates exactly `bytes`; contents are not kept.  A failed
// allocation leaves it empty (size 0), so that the next call allocates again.  A move swaps: the moved-from object
// frees what the target held.
template <bool Pinned>
class CudaBuffer {
 public:
  CudaBuffer() = default;
  CudaBuffer(CudaBuffer&& o) noexcept { *this = std::move(o); }
  CudaBuffer& operator=(CudaBuffer&& o) noexcept {
    std::swap(p_, o.p_), std::swap(bytes_, o.bytes_), std::swap(dev_, o.dev_);
    return *this;
  }
  ~CudaBuffer() { release(); }
  cudaError_t reset(size_t bytes, unsigned int flags = 0);
  size_t size() const { return bytes_; }
  template <class T = void>
  T* as() const { return static_cast<T*>(p_); }

 private:
  void release();
  void* p_ = nullptr;
  size_t bytes_ = 0;
  int dev_ = -1;
};

struct DeviceBuffer : CudaBuffer<false> {
  // at least `need` bytes: a smaller buffer is replaced by max(need, 4 KB) once `st`, which may still read it, is idle
  cudaError_t grow(size_t need, cudaStream_t st);
};

struct PinnedBuffer : CudaBuffer<true> {
  cudaError_t grow(size_t need, unsigned int flags) { return need <= size() ? cudaSuccess : reset(need, flags); }
};

// A stream or an event, owned: created on the current device and destroyed on it, the caller's current device kept;
// it reads as its handle.  An empty one makes no CUDA call.
template <class H, cudaError_t (*Create)(H*, unsigned int), cudaError_t (*Destroy)(H)>
class CudaHandle {
 public:
  CudaHandle() = default;
  CudaHandle(const CudaHandle&) = delete;
  CudaHandle& operator=(const CudaHandle&) = delete;
  ~CudaHandle() {
    if (!h_) return;
    DeviceRestore keep;
    cudaSetDevice(dev_);
    Destroy(h_);
  }
  cudaError_t create(unsigned int flags) {
    cudaError_t e = cudaGetDevice(&dev_);
    if (e == cudaSuccess && (e = Create(&h_, flags)) != cudaSuccess) h_ = nullptr;
    return e;
  }
  operator H() const { return h_; }

 private:
  H h_ = nullptr;
  int dev_ = -1;
};
using Stream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;

// The device arrays that hold the graph.  Replication blob i is array i, in this order (the order is part of the blob
// protocol between processes); the per-point insert locks, labels and attributes come last and are not replicated.
struct GraphStore {
  enum Array { VEC, ADJ0, ADJU, UP_OFF, PLEVEL, LEVEL, ORIGIN, ADJ0_D, ADJU_D, LOCKS, LABEL, ATTR, COUNT };
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
      {4, ONE, 0xFF},    // LABEL: the point's label, LABEL_NONE = none
      {8, ONE, 0},       // ATTR: the point's attribute, attr_bias(value), 0 = none (attr_bias(ATTR_NONE))
  };
  DeviceBuffer p[COUNT];
  size_t cap = 0, cap_ul = 0;  // points / upper-layer lists allocated
  template <class T>
  T* at(Array a) const { return p[a].as<T>(); }
};

// A value per point kept next to the graph (labels.cu): graph store array `array` and its host mirror, `none` for every
// point until it is set; `version` counts the calls that changed it (a replica: the handle's version it copied).
template <class T>
struct PointColumn {
  GraphStore::Array array;
  T none;
  std::vector<T> host{};
  uint64_t version = 0;
};

// The deleted points of one Index (deleted.cu): a bit per internal id on the host and on the device, `count` bits set;
// `version` counts the calls that changed it (a replica: the handle's version it copied).  The device bitmap covers the
// graph store's capacity and grows with it, zero-filled (Index::ensure_points), so that a new point is live.
struct DeletedSet {
  std::vector<uint32_t> host{};
  DeviceBuffer dev{};
  size_t count = 0;
  uint64_t version = 0;
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
// A reference-format pair read into memory (Index::parse_dump): its points in file order (layer by layer, by PointId
// rank within a layer), their vectors, and each layer's lists as CSR over those file positions
struct ParsedDump {
  DumpDescription de;
  size_t n = 0;
  int d = 0;
  std::vector<uint64_t> origin;
  std::vector<uint8_t> levels;
  std::vector<unsigned char> vecs;  // [n][d] elements
  int64_t entry = -1;
  int nlayers = 1;  // layers [0, nlayers) hold lists
  std::vector<std::vector<uint64_t>> off;  // [layer][n + 1]
  std::vector<std::vector<uint32_t>> ids;
  std::vector<std::vector<float>> dists;
};
int metric_from_name(const std::string& name);       // "DistL2" -> METRIC_L2; -1 if unknown
int metric_from_type_name(const std::string& full);  // the same on the last `::` segment of a type path
int dtype_from_type_name(const std::string& s);

class Index;

// The points an exact scan (exact_knn_kernel, aux.cu) covers: `ids`, n distinct internal ids on the scanning device in
// any order, or every stored point (ids == nullptr)
struct ExactScan {
  const uint32_t* ids = nullptr;
  size_t n = 0;
};

// rows [first, first + count) of an exact launch, all scanning the same points
struct ExactGroup {
  size_t first, count;
  ExactScan scan;
};

// The restriction of one search launch, as SearchParams reads it: none (sel, filter.ptr and filter.attr null), `filter`
// for every row, or row i under table[sel[i]]; the Index's deleted points, which no row admits (nullptr: none); and the
// rows [0, live_rows) of the live run (LegPlan::Run::live)
struct LaunchFilter {
  RowFilter filter{nullptr, nullptr, LABEL_NONE, 0, nullptr, 0, 0};
  const RowFilter* table = nullptr;
  const uint32_t* sel = nullptr;
  const uint32_t* deleted = nullptr;
  uint32_t live_rows = 0;
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
    std::vector<size_t> admitted;             // [partition] points it admits (bits set in bits[partition])
    std::map<std::pair<int, int>, DeviceBuffer> dev;  // (partition, device) -> device copy of bits[partition]
    // (partition, device) -> the admitted internal ids of bits[partition], sorted, on the device, and their count; made
    // at the first exact search with the filter there
    std::map<std::pair<int, int>, std::pair<DeviceBuffer, size_t>> ids;
  };
  int64_t add(Filter&& f);
  bool has(int64_t id);
  // the device copy of partition p's bitmap on rx's device (copied there on first use), after checking that the filter
  // exists and that rx, partition p of `nparts`, still holds the points the filter was made over; if not, rx's error.
  // With `list`, the sorted id list of the admitted points instead (made and copied there on first use).
  int use(int64_t id, int p, int nparts, const Index* rx, const uint32_t** d_bits, ExactScan* list = nullptr);
  // the number of points partition p's bitmap admits, after use's checks
  int admitted(int64_t id, int p, int nparts, const Index* rx, size_t* count);
  void erase(int64_t id);  // frees its device copies; the caller waited for every search that may read them

 private:
  std::mutex mu_;
  std::map<int64_t, Filter> f_;
  Filter* current(int64_t id, int p, int nparts, const Index* rx);  // use's checks (the caller holds mu_); nullptr: rx's error
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
// optional).  A radius batch also writes each row's total, the number of its points within its radius (optional).
struct AnswerArrays {
  NeighbourOut* nb = nullptr;
  uint64_t* ids = nullptr;
  float* dist = nullptr;
  uint32_t* internal = nullptr;
  int32_t* pid = nullptr;
  int32_t* counts = nullptr;
  const size_t* perm = nullptr;  // row j of the batch is written to row perm[j] (nullptr: to row j)
  uint64_t* total = nullptr;
  int32_t* exact = nullptr;  // a planned batch: per row, the legs that scanned it exactly (optional)
};

// What the rows of a batch may return: every point (NONE); the points a FilterT admits (FILTER_T: `mode` 1 sorted
// origin-id list, 2 callback, as make_filter_bits reads it); one resident filter for every row (RESIDENT); a resident
// filter per row, -1 = none (ROW_FILTERS); or a set of labels per row (a label per row: sets of one), row i's the values
// qset[qset_off[i], qset_off[i + 1]) in any order and with repeats, {LABEL_NONE} = none (ROW_LABEL_SETS), each within an
// attribute range when qrange is set: row i's [qrange[2i], qrange[2i + 1]], inclusive, [INT64_MIN, INT64_MAX] = none.
struct Restriction {
  enum Kind { NONE, FILTER_T, RESIDENT, ROW_FILTERS, ROW_LABEL_SETS } kind = NONE;
  int mode = 0;
  const uint64_t* ids = nullptr;
  size_t nids = 0;
  int (*fn)(uint64_t, void*) = nullptr;
  void* ctx = nullptr;
  int64_t resident = -1;
  const int64_t* filters = nullptr;  // [nq]
  const uint64_t* qset_off = nullptr;  // [nq + 1]
  const uint32_t* qset = nullptr;
  const int64_t* qrange = nullptr;  // [2 nq]
  bool per_row() const { return kind == ROW_FILTERS || kind == ROW_LABEL_SETS; }
};

// The distinct (label set, range) pairs of a ROW_LABEL_SETS batch (Index::sort_rows): set j is values[off[j], off[j + 1]),
// ascending and without repeats, within the biased attribute range [range[2j], range[2j + 1]] (attr_bias; lo >= 1), or
// with no range when that is (0, ~0)
struct LabelSets {
  std::vector<uint32_t> values;
  std::vector<size_t> off;
  std::vector<uint64_t> range;
};

// What each row of a host batch brings in, a column per field (nullptr: absent): its query (flat, a row pointer, or by
// stored point the stored vector of qids[i], an insertion rank, a partitioned handle's global one); the id it leaves out
// (skip, ~0: none; qids itself for exclude_self; write_row, search_core.cuh); in an exact batch the radius it holds
// the points within (>= 0, not NaN), reporting how many of its points are; and the points it never returns (excluded:
// an ExcludedRow per row into excluded_ids[0, nexcluded_ids), the one list of every row's ascending, distinct internal
// ids, which stays in place when the rows are permuted or sliced).  A new column is a field here and in SearchCtx::Rows,
// a line in sorted_rows and leg_rows (host_search.cu), and an entry in search_host_begin's staging list.
struct HostRows {
  const void* queries = nullptr;
  const void* const* rows = nullptr;
  const uint64_t* qids = nullptr;
  const uint64_t* skip = nullptr;
  const float* radius = nullptr;
  const ExcludedRow* excluded = nullptr;
  const uint32_t* excluded_ids = nullptr;
  size_t nexcluded_ids = 0;
};

// The caller's excluded points of a batch: row i's are the distinct values of ids[off[i], off[i + 1]) in any order,
// insertion ranks (a partitioned handle's global ones); off == nullptr: none (Index::exclusion_lists reads them)
struct Exclusions {
  const uint64_t* off = nullptr;
  const uint64_t* ids = nullptr;
};

// What each row of a leg takes out (search_host_finish): k answer slots and a count per row, and a radius batch's
// totals, in the context's pinned result buffer (valid until it is released); rc: 0, or the leg's failure
struct HostAnswers {
  const NeighbourOut* slots = nullptr;
  const int32_t* counts = nullptr;
  const uint32_t* totals = nullptr;
  int rc = 0;
};

// One host search batch: the rows `in`, k answers each into `out`.  `exact`: the exact scan of the points each row may
// return (ef unused) instead of the graph search.  `excluded`: each row's points left out on top of its restriction
// (made into in.excluded when the batch is planned).  `stored`: a store-level scan (hnsw_b200_bruteforce), which returns
// deleted points too.
struct HostBatch {
  HostRows in;
  size_t nq = 0;
  int d = 0;
  size_t k = 0, ef = 0;
  Restriction restriction;
  bool exact = false;
  AnswerArrays out;
  Exclusions excluded;
  bool stored = false;
  bool planned = false;  // each row on the graph or by the exact scan, per leg, by the planned rule (exact unset)
};

// A leg's restriction (Index::resolve): its rows [0, plain) are unrestricted, and `runs` cover the rest, each a range of
// consecutive rows under one restriction: a bitmap (a resident filter's on the leg's device, or a FilterT's host bits,
// uploaded into the context when the leg begins) or a label set on `labels` (the label array on the leg's device), the
// latter within an attribute range on `attrs` unless its lo is 0.  In an exact batch its points are slices [slice,
// slice + nslices): a filter's id list, or a label set's and range's slices of an exact-scan order.  A batch-wide filter
// is a plan with no prefix and one run over every row.  Graph rows that exclude points and have no other restriction
// are a run over every point (`every`), so that they run in the filtered kernel, which reads their lists.  On an Index
// with deleted points (`deleted`, its bitmap on the leg's device) a graph leg has no unrestricted prefix: those rows are
// a run over every point that stops by the live rule (`live`, SearchParams::live_rows).
struct LegPlan {
  struct Run {
    size_t first, count;
    bool every = false;
    bool live = false;
    const uint32_t* bits = nullptr;
    const uint32_t* host_bits = nullptr;
    const uint32_t* set = nullptr;  // the run's label set, nset values of a LabelSets
    uint32_t nset = 0;
    uint64_t lo = 0, hi = 0;  // the run's attribute range, biased bounds of a LabelSets (lo == 0: none)
    size_t slice = 0, nslices = 0;
  };
  bool exact = false;
  size_t plain = 0;
  std::vector<Run> runs;
  std::vector<ExactScan> slices;
  const uint32_t* labels = nullptr;
  const uint64_t* attrs = nullptr;  // the attribute array on the leg's device, when a run has a range
  const uint32_t* deleted = nullptr;
};

// A planned leg's rows split by the planned rule (Index::split_legs): rows[0] the leg rows that take the graph search,
// rows[1] those that take the exact scan, each ascending and under its own plan.  The parts run one after the other on
// the leg's one context, the graph part first (`running`: the part begun there), and their answers are gathered into
// `slots` and `counts` in leg-row order, so that the leg's answers read as an unsplit leg's.
struct LegSplit {
  bool on = false;
  std::vector<size_t> rows[2];
  LegPlan plan[2];
  int running = 0;
  std::vector<NeighbourOut> slots;
  std::vector<int32_t> counts;
};

// One Index's part of a batch: queries [first, first + count) searched on rx (the handle, a replica, or partition `part`)
// on its leased context ctx, under its plan (a planned batch: its split's plans)
struct Leg {
  Index* rx = nullptr;
  int part = 0;
  size_t first = 0, count = 0;
  int ctx = -1;  // -1: not leased
  bool begun = false;  // enqueued
  int rc = 0;
  LegPlan plan;
  LegSplit split;
};

// A handle's settings (its setters, hnsw.rs:810-905).  One value, on the handle; its partitions and replicas read it
// through Index::settings(), so a setting made before or after partitioning or replicating applies to all of them.
struct Settings {
  bool extend_candidates = false, keep_pruned = false;
  int link_mode = 0;       // hnsw_b200_set_link_mode: 0 back-links under the new point's level (hnsw.rs:1257), 1 per layer
  bool tie_std = false;    // hnsw_b200_set_tie_mode: equal-distance ties resolved like the reference's std BinaryHeaps (search_std.cu)
  int visited_stages = 0;  // hnsw_b200_set_visited_stages: 0 auto (first stage when the tables outgrow L2), 1 always, 2 never
  bool stats = false;      // hnsw_b200_enable_stats: launches add their work to the counters of the Index they run on
  double level_scale;      // 1/ln(M) * factor (the Index constructor sets factor 1)
  uint32_t batch_ratio = 16, batch_max = 16384;  // hnsw_b200_set_insert_batching
};

class Index {
 public:
  Index(int M, size_t max_elements, int max_layer, int ef_c, int metric, int dtype, int device);
  // a partition or replica of `handle` on `device`, sized for max_elements points: the handle's configuration, and the
  // handle's settings through settings()
  Index(Index* handle, size_t max_elements, int device);
  ~Index();
  bool ok() const { return ok_; }

  // ---- configuration (Hnsw::new, hnsw.rs:771-790)
  int M, max_layer, ef_c, metric, dtype, es, device;  // es = bytes per element
  size_t max_elements;
  SplitMix64 rng{397};
  // the settings of the handle this Index serves: its own on a handle, the handle's on a partition or a replica
  const Settings& settings() const { return handle_->settings_; }
  Settings& settings() { return handle_->settings_; }

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
  // a batch of the handle's, in dimension d: split over the partitions by placement (Partitions::insert), or set_dim and
  // insert_batch on an unpartitioned handle
  int insert(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
             const int32_t* levels, int d);
  int import_graph(const void* vecs, size_t n_new, int d, const uint64_t* origin, const uint8_t* levels,
                   int64_t entry_id, int nlayers, const uint64_t* const* offsets, const uint32_t* const* ids,
                   const float* const* dists);
  // the rows `in` of one leg (by stored point: ranks of this Index) on leased context c under the leg's plan, answers
  // left in the context's pinned buffer
  int search_host_begin(int c, const HostRows& in, size_t nq, int d, size_t k, size_t ef, const LegPlan& plan);
  HostAnswers search_host_finish(int c);
  // host search batches (host_search.cu): synchronous, or submitted now and collected by finish_batch.  A ticket is a
  // batch `b` planned into legs, with what the legs read until they are collected: a per-row batch's caller row of each
  // sorted row (out.perm) and its sorted rows, a FilterT's host bits per partition, a label-set batch's sets, and the
  // rows' excluded points.
  struct Ticket {
    std::vector<Leg> legs;
    HostBatch b;
    std::vector<size_t> perm;
    std::vector<unsigned char> rows;      // a per-row batch: its HostRows columns in sorted-row order
    std::vector<unsigned char> gathered;  // a partitioned batch by stored point: the query rows read from their partitions
    std::vector<std::vector<uint32_t>> bits;
    LabelSets sets;
    std::vector<ExcludedRow> xrows;  // per caller row, into xids (exclusion_lists)
    std::vector<uint32_t> xids;
    std::vector<int32_t> exact;  // a planned batch: per batch row, the legs that scan it exactly
  };
  int search_batch(const HostBatch& b);
  int run_batch(Ticket& t);  // the planned legs of t begun, collected and written
  int64_t submit_batch(const HostBatch& b);  // a ticket id, or < 0
  int finish_batch(Ticket& t);
  // submitted-but-not-waited host searches: anything that changes the graph waits for them (drain_pending)
  std::atomic<int> pending_{0};
  void drain_pending() const {
    while (pending_.load() != 0) std::this_thread::yield();
  }
  // the plan of each of legs[0, n) under `rs`; `sorted` holds a per-row restriction's keys (a filter id or a set of
  // `sets`, -1: none, EVERY_POINT: rows that only exclude points) in the order the legs run the rows (sort_rows,
  // prepare_batch), also for an unrestricted graph batch with excluded points.  A FilterT's host bits are made on the calling
  // thread once per partition (a replica shares the handle's internal ids, and so its bits) into `bits`; a resident
  // filter is its copy on each leg's device; a label set needs the label array on the leg's device.  `exact`: each
  // run's slices (a filter's id list on the leg's device; a label set's scan_slices).  Nonzero when a leg could not have
  // its plan; that leg's rc is set (legs_fail reports it).  Unless `stored`, a leg on an Index with deleted points
  // carries their bitmap, and its unrestricted graph rows become a live run (LegPlan).
  int resolve(const Restriction& rs, bool exact, const std::vector<int64_t>& sorted, Leg* legs, size_t n,
              std::vector<std::vector<uint32_t>>& bits, const LabelSets* sets = nullptr, bool stored = false);
  // a per-row restriction: every filter of rs.filters[0, nq) is -1 or a live, current filter of this handle (else the
  // first bad position is refused), and `perm` orders the rows stably by filter, the unfiltered ones first; label sets,
  // each made ascending without repeats into `sets`, by set in lexicographic order, {LABEL_NONE} first (a decreasing
  // offset, or LABEL_NONE with another label, refuses the first such row).  sorted[j]: the filter or set of sorted row
  // j (-1: none).
  int sort_rows(const Restriction& rs, size_t nq, std::vector<size_t>& perm, std::vector<int64_t>& sorted,
                LabelSets& sets);
  // the excluded points of rows [0, nq) as t.xrows / t.xids: each row's ranks checked below nb_point, then sorted and
  // de-duplicated.  A decreasing offset refuses its row; the first rank out of range refuses its row and position.
  int exclusion_lists(const Exclusions& x, size_t nq, Ticket& t);
  // the key sort_rows' keys leave free, which resolve makes a run over every point (LegPlan::Run::every)
  static constexpr int64_t EVERY_POINT = -2;
  // out[i]: the points row i of rs admits (none, a resident filter, or label sets with optional ranges), summed over the
  // holders, deleted points included; sort_rows' and the filters' checks refuse as a search would
  int count_admitted(const Restriction& rs, size_t nq, uint64_t* out);
  // the points that the row key `key` of rs (sort_rows' keys; -1 and EVERY_POINT: every point) admits on holder p:
  // its n, a resident filter's count, or the lengths of a label set's scan_slices
  int admitted(const Restriction& rs, int64_t key, const LabelSets& sets, int p, size_t* count);

  // ---- point labels and attributes (labels.cu): a u32 label per point, LABEL_NONE = none, and an int64 attribute per
  // point, stored as attr_bias(value), 0 = none (ATTR_NONE)
  PointColumn<uint32_t> labels{GraphStore::LABEL, LABEL_NONE};
  PointColumn<uint64_t> attrs{GraphStore::ATTR, attr_bias(ATTR_NONE)};
  // c's values of the points [first, first + count) of this Index (the caller checked the range): value(i) for point
  // first + i.  Copied on the handle's stream and waited for, so that no search launched after this returns reads the old
  // values.
  template <class T, class F>
  int set_points(PointColumn<T>& c, size_t first, size_t count, F value) {
    if (count == 0) return 0;
    HB_CUDA(cudaSetDevice(device));
    for (size_t i = 0; i < count; ++i) c.host[first + i] = value(i);
    HB_CUDA(cudaMemcpyAsync(graph_.at<T>(c.array) + first, c.host.data() + first, count * sizeof(T), cudaMemcpyHostToDevice,
                            stream_));
    HB_CUDA(cudaStreamSynchronize(stream_));
    ++c.version;
    return 0;
  }
  // column `col`'s array on this Index's device, as current as src's (src == this: its own; a replica: its copy of the
  // handle's, refreshed when the handle's changed)
  template <class T>
  int on_device(PointColumn<T> Index::*col, const Index* src, const T** d);
  // the points of one run, appended to `slices`: those whose label is one of set[0, nset) (ascending; {LABEL_NONE}: any
  // label) and, unless lo is 0, whose attribute is in the biased range [lo, hi] (lo >= 1).  They are slices of one
  // exact-scan order (rebuilt when a column it is keyed on changed): per label of the set, its group, narrowed to the
  // range by binary search in a value-keyed order; slices that follow each other in the order are joined.
  int scan_slices(const uint32_t* set, size_t nset, uint64_t lo, uint64_t hi, std::vector<ExactScan>& slices);

  // ---- deleted points (deleted.cu): points that no search returns, by internal id of this Index.  They stay in the
  // graph and in the store, route searches and inserts, and are counted by nb_point.
  DeletedSet deleted;
  // the points ids[0, n) (the caller checked them below n) marked deleted (on) or live; the changed words are copied to
  // the device and waited for, after the asynchronous device-resident launches that may read the bitmap are done
  int mark_deleted(const uint64_t* ids, size_t count, bool on);
  // the deleted-point bitmap on this Index's device as current as src's (src == this: its own; a replica: its copy of
  // the handle's, refreshed when the handle's changed), or nullptr when src has no deleted point
  int deleted_on_device(const Index* src, const uint32_t** d);
  // the batch b with device rows in and device answers out (b.in: queries, or qids and skip; b.out: nb and counts); the
  // restriction is none or a resident filter
  int search_device(const HostBatch& b, bool sync, float* kernel_ms);
  // the stored vectors of ranks[0, n) into out[n][dim], a partitioned handle's global ranks each from its partition (the
  // caller checked the ranks)
  int get_vectors(const uint64_t* ranks, size_t n, void* out) const;
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
  int load_dump(const std::string& dir, const std::string& basename);  // parse_dump + import_dump, as the reference reloads
  int parse_dump(const std::string& dir, const std::string& basename, ParsedDump& out) const;
  int import_dump(const ParsedDump& p);  // import_graph of p's points, internal ids in p's order
  // saved indexes (saved.cu): the handle's pair(s) and a manifest of what the pairs do not hold (ranks, columns, deleted
  // points, settings, level RNG), so that restore gives back the same index.  save refuses before it writes anything;
  // restore returns a new handle, or nullptr with `err` set, leaving nothing behind.
  int save(const std::string& dir, const std::string& basename, bool overwrite, std::string* used_basename);
  static Index* restore(const std::string& dir, const std::string& basename, int ndev, const int* devices, int device,
                        std::string& err);
  // the work counters summed over the holders (a query counts once per partition) and the replicas
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
    DeviceBuffer tab, epoch;
    size_t slots = 0, cap = 0;  // cap: the full stage; a slot also holds a first stage (visited_first_stage)
    int id_bits = 0;
    bool staged = false;  // the layout of the last launch: [first stage + full stage] per slot, or the full stage alone
  };
  struct SearchCtx {
    Stream stream;
    Event fork, join, ev0, ev1;
    DeviceBuffer d_counter, d_status;  // unsigned int, int
    VisitedPool vis, fvis;  // unfiltered / filtered searches
    // what the call's restriction uploads (stage_plan; exact: its label sets' joined id lists) / C
    DeviceBuffer d_fbits, d_cbuf;
    DeviceBuffer d_xq, d_xpart;  // exact scan: the host batch's queries on the device / tickets and slice lists
    PinnedBuffer h_pin, h_res;   // pinned, mapped: query staging / answers
    bool busy = false;
    // The per-row device arrays of a launch: queries (by stored point q_ids, stored rows), the id each row leaves out
    // (skip: the launch searches k + 1), a radius launch's radii and totals, k answer slots and a count per row, and each
    // row's excluded points (into excluded_ids, which does not move with the rows)
    struct Rows {
      const void* d_queries = nullptr;
      const uint64_t* q_ids = nullptr;
      const uint64_t* skip = nullptr;
      const float* radius = nullptr;
      uint32_t* totals = nullptr;
      NeighbourOut* out = nullptr;
      int32_t* counts = nullptr;
      const ExcludedRow* excluded = nullptr;
      const uint32_t* excluded_ids = nullptr;
      Rows from(size_t j, size_t q_bytes, size_t k) const {  // the same rows from row j on: only present arrays move
        return {d_queries ? (const char*)d_queries + j * q_bytes : nullptr, q_ids ? q_ids + j : nullptr, skip ? skip + j : nullptr,
                radius ? radius + j : nullptr, totals ? totals + j : nullptr, out ? out + j * k : nullptr,
                counts ? counts + j : nullptr, excluded ? excluded + j : nullptr, excluded_ids};
      }
    };
    // The launches of one leg on the context (run_plan): its rows, and the device view of the leg's plan (stage_plan).
    // Graph: rows [0, plain) unrestricted, the others under `filter`.  Exact: the rows by the points they scan, none of
    // filter.deleted.
    struct Launch {
      Rows rows;
      size_t nq = 0, k = 0, ef = 0;
      bool exact = false;
      size_t plain = 0;
      LaunchFilter filter;
      std::vector<ExactGroup> groups;
    };
    struct Pending {  // a host search enqueued by search_host_begin, completed by search_host_finish
      Launch run;
      HostAnswers ans;
      int32_t* hstatus = nullptr;
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
  // each partition is an Index of its own whose `owner` is that handle (the C ABI serves it read-only, as a view).  A
  // replica has no owner: it is never handed out.
  std::unique_ptr<Partitions, PartitionsDeleter> parts;
  const Index* owner = nullptr;
  bool partitioned() const { return parts != nullptr; }
  // the Index objects that hold the handle's points: its partitions in partition order, or the handle itself
  const std::vector<Index*>& holders() const;
  // the handle's status for a failure r of holders()[p]: r itself, or on a partitioned handle its error "partition p
  // (device D): why"
  int holder_fail(int p, int r) const;
  size_t nb_point() const;  // over the holders
  int max_level() const;    // the highest level a point has, 0 when there is none

 private:
  friend class Partitions;
  friend class FilterStore;
  int fail(const std::string& m) const;
  int cuda_fail(cudaError_t e, const char* what) const;
  Settings settings_;       // a handle's settings (unused on a partition or a replica)
  Index* handle_ = this;    // the handle whose settings_ settings() reads
  std::vector<Index*> self_{this};  // holders() of an unpartitioned handle
  int own_stats(uint64_t* out4, bool reset);  // this Index's counters
  // ---- graph store
  size_t row_size(int a) const;  // bytes of array a per point (per upper-layer list for ADJU, ADJU_D)
  int grow_store(bool per_list, size_t cap, size_t keep);
  int ensure_points(size_t need);
  int grow_deleted(size_t cap);  // the deleted-point bitmap to `cap` points, the new bits zero (deleted.cu)
  int ensure_upper(size_t need_lists);
  // ---- point ledger: the host mirrors (h_level ... h_upoff) and the per-layer counts
  void resize_points(size_t count);
  void rank_points();  // layer_count and h_rank from h_level, in internal-id order
  int upload_points(size_t first, size_t count);  // level, plevel, origin, up_off, label, attr of [first, first + count)
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
  int fill_visited_cfg(VisitedPool& v, VisitedCfg& c, bool staged, cudaStream_t st);
  bool visited_staged(size_t slots, size_t cap, size_t need, bool first_fits) const;
  int grow_plevel(uint32_t id, int new_plevel);
  int run_insert_range(size_t first, size_t count, size_t mask_off);
  int check_insert_fit();
  void rollback_points(size_t keep);

  // ---- host search batches (host_search.cu)
  int plan(size_t nq, std::vector<Leg>& legs);
  int prepare_batch(const HostBatch& call, Ticket& t, bool replicas_first);
  // a planned batch's legs split by the planned rule (t.exact counts the exact rows), each part resolved on its own
  int split_legs(Ticket& t, const std::vector<int64_t>& sorted);
  void begin_leg(const HostBatch& b, Leg& l);
  void start_leg(const HostBatch& b, Leg& l);  // enqueues the leg, or its running part
  // a begun leg's answers: a planned leg's parts collected one after the other into its split
  HostAnswers collect_leg(const HostBatch& b, Leg& l);
  void release_leg(Leg& l);
  int end_leg(Leg& l, const HostBatch& b);
  int legs_fail(const Leg* legs, size_t n, bool replicas_first);

  // ---- exact-scan orders (labels.cu): the internal ids of this Index's points that have what the order is keyed on (a
  // label, an attribute, or both), in groups per label (groups[label] = (offset, count)) laid out in ascending label
  // order; a value-only order is one group, LABEL_NONE's.  Within a group the ids ascend, or in a value-keyed order go
  // by (value, id), whose biased values stay on the host for the binary searches.  The ids go to the device.  Made from
  // the columns at the first exact search that needs the order after a column it is keyed on changed (the versions it
  // was made at, ~0: never).  A point added since has neither a label nor an attribute, so inserts leave it current.
  struct ScanOrder {
    bool by_label, by_value;
    DeviceBuffer d_ids{};
    uint64_t label_version = ~0ull, attr_version = ~0ull;
    std::unordered_map<uint32_t, std::pair<uint32_t, uint32_t>> groups{};
    std::vector<uint64_t> values{};
  };
  ScanOrder by_label_{true, false}, by_value_{false, true}, by_label_value_{true, true};
  int make_order(ScanOrder& o);
  // label_mu_ guards the orders and a replica's copy of the labels and attributes
  std::mutex label_mu_;

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
  cudaStream_t stream_ = nullptr;  // own_stream_, or the caller's (set_stream)
  Stream own_stream_;
  int sm_count_ = 0;
  size_t l2_bytes_ = 0;

  GraphStore graph_;

  VisitedPool vis_;  // visited tables of the insert kernel (searches: SearchCtx)
  SearchCtx ctx_[NCTX + NASYNC];
  // one graph search launch of rows [0, nq) of r (the filtered kernel when `f` restricts it; SearchParams)
  int search_on_ctx(SearchCtx& c, const SearchCtx::Rows& r, size_t nq, size_t k, size_t ef_arg, const LaunchFilter& f,
                    bool sync, float* kernel_ms);
  // the exact k nearest of rows [0, nq) of r, each group's rows among that group's points (aux.cu; the slices' scratch
  // sized before the launch); radius mode (r.radius): only those within each row's radius, their number into r.totals
  int exact_on_ctx(SearchCtx& c, const SearchCtx::Rows& r, size_t nq, size_t k, const std::vector<ExactGroup>& groups,
                   const uint32_t* deleted, bool sync, float* kernel_ms);
  // the device view of a leg's plan in `run`, with what it needs uploaded into context c
  int stage_plan(SearchCtx& c, const LegPlan& plan, SearchCtx::Launch& run);
  // the launches of `run` on context c, after what they share (the checks, a radius launch's totals zeroed, an empty
  // index's empty rows): the unrestricted rows as an ordinary unfiltered launch, then the restricted ones in one
  // filtered launch (exact: one launch over the groups).  Both share the context's status, so an overflow in either
  // re-runs both (sync: growing the tables).
  int run_plan(SearchCtx& c, const SearchCtx::Launch& run, bool sync, float* kernel_ms);
  std::mutex ctx_mu_;
  std::condition_variable ctx_cv_;
  std::mutex ticket_mu_;
  std::map<int64_t, Ticket> tickets_;
  int64_t next_ticket_ = 0;
  int last_async_ = -1;
  unsigned ctx_rr_ = 0;        // round robin of the asynchronous device-resident launches
  std::mutex occ_mu_;

  // small device scratch (insert path; searches: SearchCtx)
  DeviceBuffer d_counter_, d_status_, d_stats_;  // unsigned int, int, unsigned long long[4]
  std::atomic<uint64_t> stat_queries_{0};

  PinnedBuffer h_pin_;  // staging of the insert path
  // (kernel, queue kind, queue slots, warps per CTA, d4, shared memory per CTA) -> CTAs per SM
  std::map<std::tuple<QueryKernel, int, int, int, int, size_t>, int> occ_cache_;
  DeviceBuffer d_mask_;
};

}  // namespace hb
