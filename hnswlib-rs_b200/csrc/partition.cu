// Partitioned index (partition.h): placement and the fan-out of inserts over the partitions.  No kernel of its own: every
// partition runs the ordinary insert kernels on its own stream.  Searches, brute-force ones included, run through the
// host search driver (host_search.cu), which merges the partitions' answers.
#include "partition.h"

#include <algorithm>
#include <cstring>

namespace hb {

void PartitionsDeleter::operator()(Partitions* p) const { delete p; }

const std::vector<Index*>& Index::holders() const { return parts ? parts->all() : self_; }

int Index::holder_fail(int p, int r) const { return parts ? parts->fail(p, holders()[p]->err()) : r; }

int Index::insert(const void* vecs, size_t n_new, size_t stride, const void* const* rows, const uint64_t* ids,
                  const int32_t* levels, int d) {
  if (parts) return parts->insert(vecs, n_new, stride, rows, ids, levels, d);
  int r;
  if ((r = set_dim(d))) return r;
  return insert_batch(vecs, n_new, stride, rows, ids, levels);
}

int Partitions::fail(int p, const std::string& why) const {
  return parent_->fail("partition " + std::to_string(p) + " (device " + std::to_string(ix_[p]->device) + "): " + why);
}

int Partitions::run(const std::function<int(int)>& job) {
  const int bad = workers_.run(count(), job);
  return bad < 0 ? 0 : fail(bad, ix_[bad]->err());
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
    // the level RNG stays with the handle (levels are drawn in global order)
    std::unique_ptr<Index> ix(new Index(parent, cap, devices[p]));
    if (!ix->ok()) return parent->fail("partition " + std::to_string(p) + ": " + ix->err());
    if (parent->dim) ix->set_dim(parent->dim);
    ix->owner = parent;
    ps->ix_.push_back(std::move(ix));
  }
  ps->workers_.resize(nparts - 1);
  for (auto& ix : ps->ix_) ps->views_.push_back(ix.get());
  parent->parts = std::move(ps);
  return 0;
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
  const size_t before = parent_->nb_point();
  if (before + n_new >= (size_t)INVALID_ID) return parent_->fail("a partitioned handle holds fewer than 2^32 - 1 points");
  // levels in global insertion order from the handle's RNG, clamped as Index::insert_batch clamps them; origin ids
  // default to the global rank
  std::vector<int32_t> lv(n_new);
  for (size_t i = 0; i < n_new; ++i) lv[i] = std::min(std::max(levels ? levels[i] : parent_->draw_level(), 0), parent_->max_layer - 1);
  // partition p's share: the points i = first[p], first[p] + P, ... of the batch (none: share[p] = 0)
  std::vector<size_t> first(P), share(P);
  std::vector<std::vector<uint64_t>> og(P);
  std::vector<std::vector<int32_t>> pl(P);
  std::vector<std::vector<const void*>> pr(P);
  r = for_each_share(before, n_new, P, [&](int p, uint64_t, uint64_t cnt, uint64_t at, uint64_t step) {
    first[p] = at;
    share[p] = cnt;
    size_t need_ul = 0;
    for (size_t i = at; i < n_new; i += step) {
      og[p].push_back(ids ? ids[i] : (uint64_t)(before + i));
      pl[p].push_back(lv[i]);
      if (rows) pr[p].push_back(rows[i]);
      need_ul += lv[i];
    }
    Index* ix = ix_[p].get();
    if (cudaSetDevice(ix->device) != cudaSuccess) return fail(p, "cudaSetDevice failed");
    if (ix->ensure_points(ix->n + cnt) || ix->ensure_upper(ix->n_ul + need_ul + 2 * MAX_LAYERS)) return fail(p, ix->err());
    return 0;
  });
  if (r) return r;
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

}  // namespace hb
