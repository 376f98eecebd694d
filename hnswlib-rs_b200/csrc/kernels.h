// Host-visible declarations of the kernel launchers (search.cu, build.cu, aux.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "common.cuh"

namespace hb {

enum DType : int { DT_F32 = 0, DT_U8 = 1, DT_U16 = 2, DT_U32 = 3, DT_I32 = 4 };
inline int dtype_size(int dt) { return dt == DT_U8 ? 1 : dt == DT_U16 ? 2 : 4; }

constexpr int SEARCH_THREADS = 256;  // 8 warps = 8 queries in flight per CTA
constexpr int BUILD_THREADS = 128;   // 4 warps = 4 inserts in flight per CTA
constexpr int LEAN_THREADS = 32;      // lean kernel (search_lean.cuh): one warp per CTA, so that a finished query frees its slot at once
constexpr size_t SMEM_BUDGET = 220 * 1024;  // dynamic shared memory one CTA may ask for (an H100 SM offers 227 KB)
// 20 one-warp CTAs per SM, <= 96 registers per thread, no spills.  With two-stage visited tables, H100 SXM 80 GB at a 700 W
// power limit, bench.py c2, one run each: 4.60 M queries/s at 20 (96 registers, 0 spill bytes; one launch of 100 000
// queries 22.0 ms), 4.74 M at 24 (80 registers, 26 bytes spilled; 21.6 ms), 4.59 M at 28 (72 registers, 70 bytes spilled;
// 22.8 ms).  24 is not taken: it spills in the production kernel.  (The sweep with full-size tables, 400 W: 25.8 ms at 20,
// 26.7 at 24, 28.3 at 28, 32.4 at 32.)  With the first stage in shared memory (8 960 bytes per CTA at c2) the production
// kernel has 95 registers and 0 spill bytes, and the runtime grants 20 CTAs per SM, as without the window.
constexpr int LEAN_MIN_BLOCKS = 20;

// Visited tables (Visited, common.cuh): a search starts in a first stage of cap / VISITED_FIRST_DIV entries and moves to
// the full stage of `cap` entries when the first one is 3/4 full.  H100 SXM 80 GB, 700 W, bench.py c2 (cap = 8 192): 4.35 M
// queries/s at cap / 8 (65-74 % of queries move), 4.60 M at cap / 4 (7-10 % move), 4.54 M at cap / 2 (none moves); 4.21 M
// with one full-size table per slot.  Those first stages were global (~23 MB per search context resident in L2); the lean
// kernel's first stage is now in shared memory (8 KB per warp at c2, none in L2): 4.58-4.59 -> 5.72-5.73 M queries/s,
// same card and power limit, one session.
constexpr int VISITED_FIRST_DIV = 4;
inline size_t visited_first_stage(size_t cap) { return cap / VISITED_FIRST_DIV; }
inline size_t visited_slot_entries(size_t cap) { return cap + visited_first_stage(cap); }

// One answer slot.  Same 16-byte layout as the reference's #[repr(C)] Neighbour_api {id: usize, d: f32}
// (/root/reference/src/libext.rs:64-71); the internal id rides in what is tail padding there.
struct NeighbourOut {
  uint64_t origin;
  float dist;
  uint32_t internal;
};

// the restriction of one row of a filtered launch, two parts that both must admit a point:
//   * none (ptr == nullptr), a bitmap over internal ids (label == LABEL_NONE), or the label array and the one label the
//     row admits (set == nullptr), or the label array and the row's set, set[0, nset) ascending (set is not nullptr,
//     also when the set is empty, and label is then any value but LABEL_NONE);
//   * none (attr == nullptr), or the attribute array (attr_bias values) and the range lo <= attr[p] <= hi, biased
//     bounds with lo >= 1, so that a point without an attribute (0) is never in it;
// and the row's own excluded points, excl[0, nexcl) ascending and distinct, which it never admits (nexcl == 0: none),
// with xep the search's entry point when it is one of them or a deleted point (else INVALID_ID).  Those three are filled
// per row by the filtered kernel (excl / nexcl from SearchParams::excluded) and are never part of a run's entry.
struct RowFilter {
  const uint32_t* ptr;
  const uint32_t* set;
  uint32_t label;
  uint32_t nset;
  const uint64_t* attr;
  uint64_t lo, hi;
  const uint32_t* excl;
  uint32_t nexcl;
  uint32_t xep;
};

// One row's excluded points (hnsw_b200_search_*_excluding): ids[off, off + n) of its launch's concatenated id list,
// internal ids of the searched Index, ascending and distinct
struct ExcludedRow {
  uint32_t off, n;
};

struct SearchParams {
  GraphView g;
  const void* queries;  // device, raw element bytes, row i at i * q_stride_bytes
  int q_bytes;          // bytes of one query = dim * sizeof(T)
  int q_stride_bytes;
  uint32_t nq;
  int k;
  int ef;      // already max(ef_arg, k), hnsw.rs:1531
  int layer0;  // lowest layer holding a point of exactly that level (hnsw.rs:1534-1540), normally 0
  VisitedCfg vis;
  unsigned int* work_counter;
  NeighbourOut* out_nb;  // [nq][k]
  int32_t* out_count;    // [nq]
  const RowFilter* filter_table;  // filtered search: one entry per run of rows
  unsigned long long* stats;    // nullptr or [3]: evals, expansions, adjacency ids read
  int* status;                  // set to 1 on visited-table overflow
  int smem_per_warp;
  int threads;  // threads per CTA of this launch (a multiple of 32)
  int q_smem;  // queue slots in shared memory
  int q_kind;  // QueueSel kind
  uint64_t* cbuf;  // filtered search only: candidate queue C, [slots][ccap] keys
  uint32_t ccap;
  // filtered search: query i's restriction is filter_table[filter_sel[i]], or `filter` when filter_sel is nullptr
  const uint32_t* filter_sel;  // [nq]
  RowFilter filter;
  // a search by stored point: query i is row q_ids[i] of g.vec instead of `queries` (query_row, search_core.cuh)
  const uint64_t* q_ids;
  // nullptr, or per row the id the row leaves out (~0: none): k is knbn + 1 and each row knbn wide (write_row)
  const uint64_t* skip_ids;
  // filtered search: nullptr, or per row its excluded points in excluded_ids (RowFilter::excl)
  const ExcludedRow* excluded;
  const uint32_t* excluded_ids;
  // filtered search: nullptr, or the searched Index's deleted points, one bit per internal id, which no row admits; and
  // how many leading rows are the live run (LegPlan::Run::live), searched by the live stop rule: when the nearest
  // candidate is farther than W's farthest member the search returns W, as an unfiltered search does, instead of
  // dropping W's non-admitted members and expanding on.  (Fields after every other kernel's, and not on RowFilter, which
  // SearchParams holds by value: the lean, std-tie and generic kernels keep their parameter offsets.)
  const uint32_t* deleted;
  uint32_t live_rows;
};

// whether bit `id` of the deleted-point bitmap `bits` is set
__device__ __forceinline__ bool is_deleted(const uint32_t* bits, uint32_t id) { return (__ldg(bits + (id >> 5)) >> (id & 31)) & 1u; }

// the label of a point that has none (hnsw_b200_set_labels): no label admits it
constexpr uint32_t LABEL_NONE = 0xFFFFFFFFu;

// A point's int64 attribute (hnsw_b200_set_attributes) is stored as its bits with the sign bit flipped, so that the
// unsigned order of the stored values is the signed order of the attributes and HNSW_B200_ATTR_NONE (INT64_MIN), the
// attribute of a point that has none, is 0: the byte the graph store fills new space with.
__host__ __device__ constexpr uint64_t attr_bias(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }
__host__ __device__ constexpr int64_t attr_unbias(uint64_t b) { return (int64_t)(b ^ 0x8000000000000000ull); }
constexpr int64_t ATTR_NONE = (int64_t)0x8000000000000000ull;

// rows of up to 512 bytes are (partly) staged by TMA: STAGE_ROWS rows + an mbarrier per warp
__host__ __device__ inline size_t stage_bytes(int d4) { return d4 <= 32 ? (size_t)STAGE_ROWS * d4 * 16 : 0; }

// ---- per-warp shared-memory layouts: the byte offset of each region and the total, rounded to 128 bytes.  The host sizes
// a launch from `bytes` (query_smem_per_warp, Index::insert_shape), the kernel takes its regions from the offsets.
__host__ __device__ constexpr size_t round128(size_t b) { return (b + 127) & ~(size_t)127; }

// generic and filtered kernels (search.cu, filter.cu): [TMA stage][query][queue keys][chunk ids][chunk distances][mbarrier]
struct QueryLayout {
  size_t stage, query, queue, cand_id, cand_d, bar, bytes;
};
__host__ __device__ inline QueryLayout query_layout(int d4, int q_smem) {
  QueryLayout l;
  l.stage = 0;
  l.query = stage_bytes(d4);
  l.queue = l.query + (size_t)d4 * 16;
  l.cand_id = l.queue + (size_t)q_smem * 8;
  l.cand_d = l.cand_id + 64 * 4;  // 64 slots reserved, 32 used (one chunk of neighbours)
  l.bar = l.cand_d + 64 * 4;
  l.bytes = round128(l.bar + 16);
  return l;
}

// std-tie kernel (search_std.cu): [query][W heap, q_smem 8-byte items][chunk ids][chunk distances]
struct StdLayout {
  size_t query, heap, cand_id, cand_d, bytes;
};
__host__ __device__ inline StdLayout std_layout(int d4, int q_smem) {
  StdLayout l;
  l.query = 0;
  l.heap = (size_t)d4 * 16;
  l.cand_id = l.heap + (size_t)q_smem * 8;
  l.cand_d = l.cand_id + 32 * 4;
  l.bytes = round128(l.cand_d + 32 * 4);
  return l;
}

// lean kernel (search_lean.cuh): [queue keys, also the query's staging buffer][chunk ids][chunk distances]
// [visited first stage, `small` words (VisitedCfg.small; none for a single-stage launch)]
struct LeanLayout {
  uint32_t queue, cand_id, cand_d, visited, bytes;
};
__host__ __device__ constexpr LeanLayout lean_layout(int q_smem, uint32_t small = 0) {
  const uint32_t cand_id = (uint32_t)q_smem * 8, cand_d = cand_id + 32 * 4, visited = cand_d + 32 * 4;
  return LeanLayout{0, cand_id, cand_d, visited, (uint32_t)round128(visited + (size_t)small * 4)};
}

// insert kernel (build.cu): [TMA stage][new point][point of a selection step][queue keys][chunk ids][chunk distances]
// [mbarrier][selected ids][selected distances][distances of a selection step][discarded positions, u16]
struct InsertLayout {
  size_t stage, query, point, queue, cand_id, cand_d, bar, sel_id, sel_d, tmp, disc, bytes;
};
__host__ __device__ inline InsertLayout insert_layout(int d4, int ef_c, int deg0, int q_smem) {
  InsertLayout l;
  l.stage = 0;
  l.query = stage_bytes(d4);
  l.point = l.query + (size_t)d4 * 16;
  l.queue = l.point + (size_t)d4 * 16;
  l.cand_id = l.queue + (size_t)q_smem * 8;
  l.cand_d = l.cand_id + 64 * 4;
  l.bar = l.cand_d + 64 * 4;
  l.sel_id = l.bar + 16;
  l.sel_d = l.sel_id + (size_t)deg0 * 4;
  l.tmp = l.sel_d + (size_t)deg0 * 4;
  l.disc = l.tmp + (size_t)deg0 * 4;
  l.bytes = round128(l.disc + (size_t)ef_c * 2);
  return l;
}

// exact k-NN kernel (aux.cu), per CTA: [query tile, tq rows][row ring, stages x rows][tq queues of k keys]
// [candidates, tq x rows keys][tq queue thresholds][tq candidate counts][tq queue lengths][stages mbarriers]
struct ExactLayout {
  size_t query, ring, queue, cand, thr, ccount, qn, bar, bytes;
};
__host__ __device__ inline ExactLayout exact_layout(int d4, int k, int tq, int rows, int stages) {
  ExactLayout l;
  l.query = 0;
  l.ring = (size_t)tq * d4 * 16;
  l.queue = l.ring + (size_t)stages * rows * d4 * 16;
  l.cand = l.queue + (size_t)tq * k * 8;
  l.thr = l.cand + (size_t)tq * rows * 8;
  l.ccount = l.thr + (size_t)tq * 8;
  l.qn = l.ccount + (size_t)tq * 4;
  l.bar = (l.qn + (size_t)tq * 4 + 15) & ~(size_t)15;
  l.bytes = round128(l.bar + (size_t)stages * 8);
  return l;
}

// one tile of an exact launch whose tiles differ (a filter per query): queries [q0, q0 + nq) of the launch, scanned over
// `list` (npts distinct internal ids, in any order) or, with list == nullptr, over the points 0 .. npts - 1
struct ExactTile {
  uint32_t q0, nq;
  const uint32_t* list;
  uint32_t npts;
};

// Queue kind for a given ef (see QueueSel): compile-time chunked shared-memory queue up to ef = 256, generic beyond.
// (A register-resident variant spilled at 64 registers/thread, and a speculative two-candidates-per-iteration loop was
// exact but slower; both were removed.)
inline int queue_kind(int ef, int metric, int dtype) {
  const bool common = dtype == DT_F32 && (metric == METRIC_L1 || metric == METRIC_L2 || metric == METRIC_DOT || metric == METRIC_COSINE);
  if (!common || ef > 256) return 0;
  if (ef <= 32) return 101;
  if (ef <= 64) return 102;
  if (ef <= 128) return 104;
  return 108;
}
inline int queue_slots(int kind, int ef) { return kind >= 100 ? 32 * (kind - 100) : ef; }

// ---- lean kernel (search_lean.cuh): rows of 128 / 256 / 512 bytes (compile-time chunk count), ef <= 128, no filter
inline int lean_queue_slots(int ef) { return ef <= 64 ? 64 : (ef <= 128 ? 128 : 0); }
inline bool lean_eligible(int d4, int ef) { return (d4 == 8 || d4 == 16 || d4 == 32) && lean_queue_slots(ef) != 0; }

// ---- the query kernels.  Lean (search_lean.cuh) whenever it applies, else the generic warp kernel (search.cu), the
// filtered kernel (filter.cu), or with tie mode "std" the reference's heaps replayed literally (search_std.cu).
enum class QueryKernel { Lean, Generic, Filtered, StdTie };
// queue slots in shared memory (q_kind: QueueSel kind, used by the generic kernel only)
inline int query_queue_slots(QueryKernel kind, int q_kind, int ef) {
  switch (kind) {
    case QueryKernel::Lean: return lean_queue_slots(ef);
    case QueryKernel::StdTie: return ef + 2;  // the W heap holds at most ef + 1 items (push, then pop when over ef)
    default: return queue_slots(q_kind, ef);
  }
}
inline size_t query_smem_per_warp(QueryKernel kind, int d4, int q_smem) {
  switch (kind) {
    case QueryKernel::Lean: return lean_layout(q_smem).bytes;
    case QueryKernel::StdTie: return std_layout(d4, q_smem).bytes;
    default: return query_layout(d4, q_smem).bytes;
  }
}
inline int query_threads(QueryKernel kind) { return kind == QueryKernel::Lean ? LEAN_THREADS : SEARCH_THREADS; }

// Launch shape for a kernel built for up to `max_warps` warps per CTA: fewer warps when one warp's share of shared
// memory is large (wide rows, big ef).  warps == 0: a single warp does not fit.
struct CtaShape {
  int warps;
  size_t smem;
};
inline CtaShape cta_shape(size_t smem_per_warp, int max_warps) {
  int w = max_warps;
  while (w > 1 && smem_per_warp * w > SMEM_BUDGET) w >>= 1;
  if (smem_per_warp * w > SMEM_BUDGET) return {0, 0};
  return {w, smem_per_warp * w};
}

struct InsertParams {
  GraphView g;
  uint32_t first;   // internal id of the first point of the batch
  uint32_t count;   // points in the batch
  const uint16_t* layer_mask;  // [count] bit l set <=> some point of exact level l exists when this point searches
  int ef_c;
  int keep_pruned;
  int extend;  // extend_candidates flag (hnsw.rs:858), only with ef_c > 2M
  int link_mode;  // phase B target layer: 0 the new point's level (hnsw.rs:1257), 1 the layer being linked
  VisitedCfg vis;
  unsigned int* work_counter;
  int* locks;  // [capacity] per-point spin locks (phase B)
  unsigned long long* stats;
  int* status;
  int smem_per_warp;
  int threads;  // threads per CTA of the search phase (a multiple of 32)
  int q_smem;
  int q_kind;
};

// The kernel this host thread last launched through launch_kernel (hnsw_b200_last_kernel reports its name), so that a
// test can tell which template instantiation served a call.
inline thread_local const void* last_launched_kernel = nullptr;
// its dynamic shared memory and threads per CTA (hnsw_b200_last_kernel_shape)
inline thread_local size_t last_launched_smem = 0;
inline thread_local int last_launched_threads = 0;

// Every launcher below sets the kernel's dynamic shared-memory limit to `smem`, then either launches it (blocks_per_sm ==
// nullptr) or only reports how many CTAs of `threads` threads fit on one SM.
template <class P>
cudaError_t launch_kernel(void (*kern)(P), const P& p, int grid, int threads, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  if (blocks_per_sm) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, kern, threads, smem);
  kern<<<grid, threads, smem, st>>>(p);
  last_launched_kernel = reinterpret_cast<const void*>(kern);
  last_launched_smem = smem;
  last_launched_threads = threads;
  return cudaGetLastError();
}

cudaError_t launch_insert_search(const InsertParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                                 int* blocks_per_sm);
cudaError_t launch_insert_link(const InsertParams& p, int grid, cudaStream_t st);

cudaError_t launch_search_filtered(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                                   int* blocks_per_sm);
cudaError_t launch_search(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm);
cudaError_t launch_search_std(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                              int* blocks_per_sm);
cudaError_t launch_search_lean(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                               int* blocks_per_sm);
cudaError_t launch_search_lean_u8(const SearchParams& p, int metric, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm);
cudaError_t launch_search_lean_u16(const SearchParams& p, int metric, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm);

inline cudaError_t launch_query(QueryKernel kind, const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                                int* blocks_per_sm) {
  switch (kind) {
    case QueryKernel::Lean: return launch_search_lean(p, metric, dtype, grid, smem, st, blocks_per_sm);
    case QueryKernel::Generic: return launch_search(p, metric, dtype, grid, smem, st, blocks_per_sm);
    case QueryKernel::Filtered: return launch_search_filtered(p, metric, dtype, grid, smem, st, blocks_per_sm);
    case QueryKernel::StdTie: return launch_search_std(p, metric, dtype, grid, smem, st, blocks_per_sm);
  }
  return cudaErrorInvalidValue;
}

// ---- (metric, element type) -> distance functor.  f is called as f(OpTag<Op>{}) and returns cudaError_t.
template <class Op>
struct OpTag {
  typedef Op type;
};
// CH-specialised kernels (compile-time row length) are only built for the common f32 metrics
template <class Op>
struct Specialise {
  static constexpr bool value = false;
};
template <> struct Specialise<OpL1> { static constexpr bool value = true; };
template <> struct Specialise<OpL2> { static constexpr bool value = true; };
template <> struct Specialise<OpDot> { static constexpr bool value = true; };
template <> struct Specialise<OpCosine> { static constexpr bool value = true; };

// (metric, element type) pairs the lean kernel (search_lean.cuh) is instantiated for
inline bool lean_op_supported(int metric, int dtype) {
  if (dtype == DT_F32) return metric == METRIC_L1 || metric == METRIC_L2 || metric == METRIC_DOT || metric == METRIC_COSINE;
  if (dtype == DT_U8 || dtype == DT_U16)
    return metric == METRIC_L1 || metric == METRIC_L2 || metric == METRIC_HAMMING || metric == METRIC_JACCARD;
  return false;
}

// WITH_JACCARD is a template parameter so that the Jaccard kernels of an element type without DistJaccard (i32) are
// not compiled at all
template <class T, bool WITH_JACCARD, class F>
cudaError_t dispatch_int(int metric, F&& f) {
  switch (metric) {
    case METRIC_L1: return f(OpTag<OpCast<T, OpL1>>{});
    case METRIC_L2: return f(OpTag<OpCast<T, OpL2>>{});
    case METRIC_HAMMING: return f(OpTag<OpHamming<T>>{});
    case METRIC_JACCARD:
      if constexpr (WITH_JACCARD) return f(OpTag<OpJaccard<T>>{});
      break;
  }
  return cudaErrorInvalidValue;
}

template <class F>
cudaError_t dispatch_op(int metric, int dtype, F&& f) {
  switch (dtype) {
    case DT_F32:
      switch (metric) {
        case METRIC_L1: return f(OpTag<OpL1>{});
        case METRIC_L2: return f(OpTag<OpL2>{});
        case METRIC_DOT: return f(OpTag<OpDot>{});
        case METRIC_COSINE: return f(OpTag<OpCosine>{});
        case METRIC_HELLINGER: return f(OpTag<OpHellinger>{});
        case METRIC_JEFFREYS: return f(OpTag<OpJeffreys>{});
        case METRIC_JENSENSHANNON: return f(OpTag<OpJS>{});
      }
      break;
    case DT_U8: return dispatch_int<uint8_t, true>(metric, f);
    case DT_U16: return dispatch_int<uint16_t, true>(metric, f);
    case DT_U32: return dispatch_int<uint32_t, true>(metric, f);
    case DT_I32: return dispatch_int<int32_t, false>(metric, f);
  }
  return cudaErrorInvalidValue;
}

// which (metric, dtype) pairs exist (mirrors init_hnsw_{f32,i32,u32,u16,u8} in /root/reference/src/libext.rs)
inline bool metric_supported(int metric, int dtype) {
  if (dtype == DT_F32)
    return metric == METRIC_L1 || metric == METRIC_L2 || metric == METRIC_DOT || metric == METRIC_COSINE ||
           metric == METRIC_HELLINGER || metric == METRIC_JEFFREYS || metric == METRIC_JENSENSHANNON;
  if (metric == METRIC_L1 || metric == METRIC_L2 || metric == METRIC_HAMMING) return true;
  return metric == METRIC_JACCARD && dtype != DT_I32;
}

}  // namespace hb
