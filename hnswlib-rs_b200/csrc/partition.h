// A partitioned index: the points of one handle split over P Index objects ("partitions"), each on its own device or
// several on one.  The g-th point inserted goes to partition g % P as its local id g / P; every query searches every
// partition and the P answer lists are merged.  This adds capacity (P devices' HBM for one index), where replication
// (multi.cu) adds throughput.  DESIGN.md §6 "Partitioned index" states the rules.
#pragma once
#include <algorithm>

#include "index.h"

namespace hb {

// The placement rule over P partitions (P = 1: an unpartitioned handle, where a rank is its own local id).  Global rank
// g is local id g / P of partition g % P.
struct Placed {
  int part;
  uint64_t local;
};
inline Placed place(uint64_t g, uint64_t P) { return {(int)(g % P), g / P}; }
inline uint64_t global_rank(int part, uint64_t local, uint64_t P) { return local * P + (uint64_t)part; }
// f(p, lo, count, at, step) for each partition p that holds some of the ranks [first, first + n): its local ids lo ..
// lo + count - 1 are the ranks first + at, first + at + step, ...  Returns the first nonzero f, or 0.
template <class F>
int for_each_share(uint64_t first, uint64_t n, uint64_t P, const F& f) {
  for (uint64_t p = 0; p < P; ++p) {
    const uint64_t g0 = first + (p + P - first % P) % P;  // the first rank of partition p in the range
    if (g0 >= first + n) continue;
    if (int r = f((int)p, g0 / P, (first + n - g0 + P - 1) / P, g0 - first, P)) return r;
  }
  return 0;
}

class Partitions {
 public:
  static constexpr int MAX_PARTS = 64;
  // splits the empty handle `parent` into nparts partitions, partition p on devices[p] (devices[0] = parent->device)
  static int create(Index* parent, int nparts, const int* devices);
  int count() const { return (int)ix_.size(); }
  Index* part(int p) const { return ix_[p].get(); }
  const std::vector<Index*>& all() const { return views_; }
  // a C ABI handle on partition p: the address of a pointer to it, which is the layout of every handle
  const void* view_handle(int p) const { return &views_[p]; }

  // a batch in the engine's insert form (flat `vecs` with `stride` elements per row, or `rows`), split by placement
  int insert(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
             const int32_t* levels, int d);
  // the handle's error "partition p (device D): why"
  int fail(int p, const std::string& why) const;
  // job(p) for every partition at once, one per worker; the first failure as fail(p, that partition's error)
  int run(const std::function<int(int)>& job);
  // why a failed insert left the partitions unusable for inserts ("" while they are not)
  const std::string& broken() const { return broken_; }

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
