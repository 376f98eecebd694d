// A partitioned index: the points of one handle split over P Index objects ("partitions"), each on its own device or
// several on one.  The g-th point inserted goes to partition g % P as its local id g / P; every query searches every
// partition and the P answer lists are merged.  This adds capacity (P devices' HBM for one index), where replication
// (multi.cu) adds throughput.  DESIGN.md §6 "Partitioned index" states the rules.
#pragma once
#include "index.h"

namespace hb {

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
};

// PointId (level, rank) of internal id `it` of `rx`, hnsw.rs:46; (-1, -1) for an empty slot
inline void point_id(const Index* rx, uint32_t it, int32_t* pid2) {
  pid2[0] = it != INVALID_ID ? (int32_t)rx->h_level[it] : -1;
  pid2[1] = it != INVALID_ID ? rx->h_rank[it] : -1;
}

// slot s of `out` from answer e of index rx, reported with internal id `internal` (a partitioned handle's global rank)
inline void put_answer(const AnswerArrays& out, size_t s, const Index* rx, const NeighbourOut& e, uint32_t internal) {
  if (out.nb) {
    out.nb[s] = NeighbourOut{e.origin, e.dist, internal};
    return;
  }
  out.ids[s] = e.origin;
  out.dist[s] = e.dist;
  if (out.internal) out.internal[s] = internal;
  if (out.pid) point_id(rx, e.internal, out.pid + 2 * s);
}

class Partitions {
 public:
  static constexpr int MAX_PARTS = 64;
  // splits the empty handle `parent` into nparts partitions, partition p on devices[p] (devices[0] = parent->device)
  static int create(Index* parent, int nparts, const int* devices);
  int count() const { return (int)ix_.size(); }
  Index* part(int p) const { return ix_[p].get(); }
  // a C ABI handle on partition p: the address of a pointer to it, which is the layout of every handle
  const void* view_handle(int p) const { return &views_[p]; }

  // every partition's lock in partition order (the caller holds the handle's own first); exclusive also waits for
  // submitted searches on the partitions' views
  std::vector<std::shared_lock<std::shared_mutex>> lock_shared() const;
  std::vector<std::unique_lock<std::shared_mutex>> lock_exclusive() const;

  size_t nb_point() const;
  int max_level() const;
  // a batch in the engine's insert form (flat `vecs` with `stride` elements per row, or `rows`), split by placement
  int insert(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
             const int32_t* levels, int d);
  // every query on every partition with the caller's k and ef, merged into `out`.  The filter is the FilterT arguments
  // (filter_mode 1, 2) or `resident`, the id of one of the handle's resident filters (filter_mode 0).
  int search(const void* queries, const void* const* rows, size_t nq, int d, size_t k, size_t ef, int filter_mode,
             const uint64_t* filter_ids, size_t nfilter, int (*fn)(uint64_t, void*), void* ctx, const int64_t* resident,
             const AnswerArrays& out);
  // exact k nearest over all partitions, merged like search; out_ids are global insertion ranks
  int bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist);
  int get_stats(uint64_t* out4, bool reset);

 private:
  explicit Partitions(Index* parent) : parent_(parent) {}
  int fail(int p, const std::string& why) const;
  // job(p) for every partition at once: partition 0 on the calling thread, partition p > 0 on worker p - 1
  int fan_out(const std::function<int(int)>& job);
  size_t expected_count(int p, size_t total) const { return (total + count() - 1 - p) / count(); }

  Index* parent_;
  std::vector<std::unique_ptr<Index>> ix_;
  std::vector<std::unique_ptr<Index::Worker>> workers_;
  std::vector<Index*> views_;
  std::string broken_;  // set when a failed insert left the partitions at counts the placement rule does not give
  std::mutex fan_mu_;   // one fan-out at a time: a worker holds one job
};

}  // namespace hb
