// Partitioned index (partition.h): placement, the fan-out of inserts and brute-force searches over the partitions.  No
// kernel of its own: every partition runs the ordinary insert kernels on its own stream.  Searches run through the host
// search driver (host_search.cu), which merges the partitions' answers.
#include "partition.h"

#include <algorithm>
#include <cstring>

namespace hb {

void PartitionsDeleter::operator()(Partitions* p) const { delete p; }

int Partitions::fail(int p, const std::string& why) const {
  return parent_->fail("partition " + std::to_string(p) + " (device " + std::to_string(ix_[p]->device) + "): " + why);
}

int Partitions::create(Index* parent, int nparts, const int* devices) {
  DeviceRestore keep;
  if (parent->owner) return parent->fail("partition: a partition view cannot be partitioned");
  if (parent->parts) return parent->fail("partition: the handle is already partitioned");
  if (parent->n != 0) return parent->fail("partition: the handle must be empty");
  if (parent->replica_count() || parent->comm_) return parent->fail("partition: the handle is replicated or NCCL-initialised");
  if (nparts < 1 || nparts > MAX_PARTS || !devices) return parent->fail("partition: nparts must be in [1, 64]");
  if (devices[0] != parent->device) return parent->fail("partition: devices[0] must be the handle's device");
  int have = 0;
  if (cudaGetDeviceCount(&have) != cudaSuccess) return parent->fail("partition: cudaGetDeviceCount failed");
  for (int p = 0; p < nparts; ++p)
    if (devices[p] < 0 || devices[p] >= have) return parent->fail("partition: device index out of range");
  std::unique_ptr<Partitions, PartitionsDeleter> ps(new Partitions(parent));
  const size_t cap = (parent->max_elements + nparts - 1) / nparts;
  for (int p = 0; p < nparts; ++p) {
    std::unique_ptr<Index> ix(new Index(parent->M, cap, parent->max_layer, parent->ef_c, parent->metric, parent->dtype, devices[p]));
    if (!ix->ok()) return parent->fail("partition " + std::to_string(p) + ": " + ix->err());
    // the settings made on the handle so far; the level RNG stays with the handle (levels are drawn in global order)
    ix->extend_candidates = parent->extend_candidates;
    ix->keep_pruned = parent->keep_pruned;
    ix->link_mode = parent->link_mode;
    ix->searching = parent->searching;
    ix->tie_std_ = parent->tie_std_;
    ix->visited_stages_ = parent->visited_stages_;
    ix->level_scale = parent->level_scale;
    ix->batch_ratio = parent->batch_ratio;
    ix->batch_max = parent->batch_max;
    ix->stats_on_ = parent->stats_on_;
    if (parent->dim) ix->set_dim(parent->dim);
    ix->owner = parent;
    ps->ix_.push_back(std::move(ix));
  }
  ps->workers_.resize(nparts - 1);
  for (auto& ix : ps->ix_) ps->views_.push_back(ix.get());
  parent->parts = std::move(ps);
  return 0;
}

std::vector<std::shared_lock<std::shared_mutex>> Partitions::lock_shared() const {
  std::vector<std::shared_lock<std::shared_mutex>> l;
  for (auto& ix : ix_) l.emplace_back(ix->mu);
  return l;
}
std::vector<std::unique_lock<std::shared_mutex>> Partitions::lock_exclusive() const {
  std::vector<std::unique_lock<std::shared_mutex>> l;
  for (auto& ix : ix_) {
    l.emplace_back(ix->mu);
    ix->drain_pending();
  }
  return l;
}

size_t Partitions::nb_point() const {
  size_t s = 0;
  for (auto& ix : ix_) s += ix->n;
  return s;
}
int Partitions::max_level() const {
  int m = 0;
  for (auto& ix : ix_) m = std::max(m, ix->entry_level);
  return m;
}

int Partitions::insert(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
                       const int32_t* levels, int d) {
  if (n_new == 0) return 0;
  if (!broken_.empty()) return parent_->fail(broken_);
  const int P = count();
  int r;
  // ---- checks: nothing below changes a partition's points before all of them pass
  if ((r = parent_->set_dim(d))) return r;
  for (auto& ix : ix_) ix->set_dim(d);  // cannot fail: a partition's dimension is 0 or the handle's
  for (int p = 0; p < P; ++p)
    if ((r = ix_[p]->check_insert_fit())) return fail(p, ix_[p]->err());
  const size_t before = nb_point();
  if (before + n_new >= (size_t)INVALID_ID) return parent_->fail("a partitioned handle holds fewer than 2^32 - 1 points");
  // levels in global insertion order from the handle's RNG, clamped as Index::insert_batch clamps them; origin ids
  // default to the global rank
  std::vector<int32_t> lv(n_new);
  for (size_t i = 0; i < n_new; ++i) lv[i] = std::min(std::max(levels ? levels[i] : parent_->draw_level(), 0), parent_->max_layer - 1);
  // partition p's share: the points i = first[p], first[p] + P, ... of the batch
  std::vector<size_t> first(P), share(P);
  std::vector<std::vector<uint64_t>> og(P);
  std::vector<std::vector<int32_t>> pl(P);
  std::vector<std::vector<const void*>> pr(P);
  for (int p = 0; p < P; ++p) {
    first[p] = (size_t)((p - (int)(before % P) + P) % P);
    share[p] = first[p] < n_new ? (n_new - first[p] + P - 1) / P : 0;
    size_t need_ul = 0;
    for (size_t i = first[p]; i < n_new; i += P) {
      og[p].push_back(ids ? ids[i] : (uint64_t)(before + i));
      pl[p].push_back(lv[i]);
      if (rows) pr[p].push_back(rows[i]);
      need_ul += lv[i];
    }
    Index* ix = ix_[p].get();
    if (!share[p]) continue;
    if (cudaSetDevice(ix->device) != cudaSuccess) return fail(p, "cudaSetDevice failed");
    if ((r = ix->ensure_points(ix->n + share[p])) || (r = ix->ensure_upper(ix->n_ul + need_ul + 2 * MAX_LAYERS)))
      return fail(p, ix->err());
  }
  cudaSetDevice(parent_->device);
  // ---- every partition inserts its share at once
  const size_t row = stride * parent_->es;
  const int bad = workers_.run(P, [&](int p) {
    const void* v = rows ? nullptr : (const void*)((const char*)vecs + first[p] * row);
    return ix_[p]->insert_batch(v, share[p], stride * P, rows ? pr[p].data() : nullptr, og[p].data(), pl[p].data());
  });
  r = bad < 0 ? 0 : fail(bad, ix_[bad]->err());
  if (r) {
    bool unchanged = true;
    for (int p = 0; p < P; ++p) unchanged = unchanged && ix_[p]->n == expected_count(p, before);
    if (!unchanged) {
      broken_ = "a failed insert left this partitioned handle's partitions at uneven counts; it refuses further inserts "
                "(searches still work).  The failure: " + parent_->err();
    }
  }
  return r;
}

int Partitions::bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist) {
  if (nq == 0 || k == 0) return 0;
  if (d != parent_->dim) return parent_->fail("query length differs from the index dimension");
  const int P = count();
  std::vector<std::vector<uint32_t>> ids(P);
  std::vector<std::vector<float>> ds(P);
  const int bad = workers_.run(P, [&](int p) {
    if (ix_[p]->n == 0) return 0;  // an empty partition answers nothing
    ids[p].resize(nq * k);
    ds[p].resize(nq * k);
    return ix_[p]->bruteforce(queries, nq, d, k, ids[p].data(), ds[p].data());
  });
  if (bad >= 0) return fail(bad, ix_[bad]->err());
  int32_t cnt[MAX_PARTS];
  for (size_t q = 0; q < nq; ++q) {
    const size_t o = q * k;
    for (int p = 0; p < P; ++p) {  // a list ends at its first empty slot
      cnt[p] = 0;
      if (!ids[p].empty())
        while ((size_t)cnt[p] < k && ids[p][o + cnt[p]] != INVALID_ID) cnt[p]++;
    }
    const size_t total = merge_lists(
        P, k, cnt, [&](int p, int i) { return ds[p][o + i]; },
        [&](size_t j, int p, int i) {
          out_ids[o + j] = ids[p][o + i] * (uint32_t)P + (uint32_t)p;
          out_dist[o + j] = ds[p][o + i];
        });
    for (size_t j = total; j < k; ++j) {
      out_ids[o + j] = INVALID_ID;
      out_dist[o + j] = __builtin_inff();
    }
  }
  return 0;
}

int Partitions::get_stats(uint64_t* out4, bool reset) {
  DeviceRestore keep;
  for (int i = 0; i < 4; ++i) out4[i] = 0;
  for (int p = 0; p < count(); ++p) {
    uint64_t s[4];
    if (ix_[p]->get_stats(s, reset)) return fail(p, ix_[p]->err());
    for (int i = 0; i < 4; ++i) out4[i] += s[i];
  }
  return 0;
}

}  // namespace hb
