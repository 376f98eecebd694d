// A partitioned index: the points of one handle split over P Index objects ("partitions"), each on its own device or
// several on one.  The g-th point inserted goes to partition g % P as its local id g / P; every query searches every
// partition and the P answer lists are merged.  This adds capacity (P devices' HBM for one index), where replication
// (multi.cu) adds throughput.  DESIGN.md §6 "Partitioned index" states the rules.
#pragma once
#include <algorithm>

#include "index.h"

namespace hb {

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
  // exact k nearest over all partitions, merged like a search (host_search.cu); out_ids are global insertion ranks
  int bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist);
  int get_stats(uint64_t* out4, bool reset);
  // the handle's error "partition p (device D): why"
  int fail(int p, const std::string& why) const;

 private:
  explicit Partitions(Index* parent) : parent_(parent) {}
  size_t expected_count(int p, size_t total) const { return (total + count() - 1 - p) / count(); }

  Index* parent_;
  std::vector<std::unique_ptr<Index>> ix_;
  WorkerGroup workers_;  // worker p - 1 serves partition p
  std::vector<Index*> views_;
  std::string broken_;  // set when a failed insert left the partitions at counts the placement rule does not give
};

// Merge rule: the first min(k, sum of counts) entries of the P ascending lists of one query, ordered by (distance,
// partition, position in that partition's list).  dist(p, i) is entry i of list p; emit(j, p, i) writes output slot j.
template <class Dist, class Emit>
size_t merge_lists(int P, size_t k, const int32_t* cnt, const Dist& dist, const Emit& emit) {
  int pos[Partitions::MAX_PARTS] = {};
  size_t total = 0;
  for (int p = 0; p < P; ++p) total += (size_t)cnt[p];
  total = std::min(total, k);
  for (size_t j = 0; j < total; ++j) {
    int best = -1;
    float bd = 0.f;
    for (int p = 0; p < P; ++p) {
      if (pos[p] >= cnt[p]) continue;
      const float dp = dist(p, pos[p]);
      if (best < 0 || dp < bd) {
        best = p;
        bd = dp;
      }
    }
    emit(j, best, pos[best]++);
  }
  return total;
}

}  // namespace hb
