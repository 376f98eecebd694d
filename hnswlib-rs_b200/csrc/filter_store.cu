// Resident filters (index.h FilterStore): a FilterT materialised once and kept on every device that searches with it.
// No kernel of its own: a search with a resident filter runs the same filtered query kernel a per-call filter runs, on
// a bitmap that is already on the device instead of one uploaded for the call.  An exact search with it runs the exact
// scan over the filter's sorted id list, made from the bitmap at the first exact search on a device.
#include "index.h"

namespace hb {

static std::atomic<int64_t> g_next_filter{0};  // over all handles: another handle's id is unknown to this one

static std::string unknown_filter(int64_t id) {
  return "filter " + std::to_string(id) + " is not a live filter of this handle (freed, or made on another handle)";
}

// a copy of `words` on `device`, never null: an empty id list is not a null list (every point)
static cudaError_t upload(const std::vector<uint32_t>& words, int device, DeviceBuffer& out) {
  DeviceRestore keep;
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess || (e = out.reset(std::max<size_t>(1, words.size()) * 4)) != cudaSuccess)
    return e;
  return cudaMemcpy(out.as(), words.data(), words.size() * 4, cudaMemcpyHostToDevice);
}

int64_t FilterStore::add(Filter&& f) {
  std::lock_guard<std::mutex> lk(mu_);
  const int64_t id = g_next_filter++;
  f_.emplace(id, std::move(f));
  return id;
}

bool FilterStore::has(int64_t id) {
  std::lock_guard<std::mutex> lk(mu_);
  return f_.count(id) != 0;
}

FilterStore::Filter* FilterStore::current(int64_t id, int p, int nparts, const Index* rx) {
  auto it = f_.find(id);
  if (it == f_.end()) return rx->fail(unknown_filter(id)), nullptr;
  Filter& f = it->second;
  // the kernel reads one bit per stored point: a bitmap made over fewer points than the index now holds is refused
  if ((int)f.counts.size() != nparts)
    return rx->fail("filter " + std::to_string(id) + " was made before the handle was partitioned: make a new filter"), nullptr;
  if (f.counts[p] != rx->n)
    return rx->fail("filter " + std::to_string(id) + " is stale: it covers " + std::to_string(f.counts[p]) + " points and the " +
                    (nparts > 1 ? "partition" : "index") + " now holds " + std::to_string(rx->n) + ": make a new filter"),
           nullptr;
  return &f;
}

int FilterStore::admitted(int64_t id, int p, int nparts, const Index* rx, size_t* count) {
  std::lock_guard<std::mutex> lk(mu_);
  const Filter* f = current(id, p, nparts, rx);
  if (!f) return -1;
  *count = f->admitted[p];
  return 0;
}

int FilterStore::use(int64_t id, int p, int nparts, const Index* rx, const uint32_t** d_bits, ExactScan* list) {
  std::lock_guard<std::mutex> lk(mu_);
  Filter* fp = current(id, p, nparts, rx);
  if (!fp) return -1;
  Filter& f = *fp;
  const std::pair<int, int> key(p, rx->device);
  if (list) {
    auto l = f.ids.find(key);
    if (l == f.ids.end()) {  // first exact search on this device: the admitted ids in order, kept until the filter is freed
      const std::vector<uint32_t>& b = f.bits[p];
      std::vector<uint32_t> ids;
      for (size_t i = 0; i < f.counts[p]; ++i)
        if ((b[i >> 5] >> (i & 31)) & 1u) ids.push_back((uint32_t)i);
      DeviceBuffer copy;
      if (cudaError_t e = upload(ids, rx->device, copy)) return rx->cuda_fail(e, "filter id list upload");
      l = f.ids.emplace(key, std::make_pair(std::move(copy), ids.size())).first;
    }
    list->ids = l->second.first.as<const uint32_t>();
    list->n = l->second.second;
    return 0;
  }
  auto d = f.dev.find(key);
  if (d == f.dev.end()) {  // first use on this device: one copy, kept until the filter is freed
    DeviceBuffer copy;
    if (cudaError_t e = upload(f.bits[p], rx->device, copy)) return rx->cuda_fail(e, "filter upload");
    d = f.dev.emplace(key, std::move(copy)).first;
  }
  *d_bits = d->second.as<const uint32_t>();
  return 0;
}

void FilterStore::erase(int64_t id) {  // each device copy is freed on its device
  std::lock_guard<std::mutex> lk(mu_);
  f_.erase(id);
}

int64_t Index::new_filter(int mode, const uint64_t* sorted_ids, size_t nids, int (*fn)(uint64_t, void*), void* ctx) {
  if (mode != 1 && mode != 2) return fail("filter_mode must be 1 (sorted origin-id list) or 2 (callback)");
  if (mode == 1 && nids && !sorted_ids) return fail("filter_ids is NULL");
  const std::vector<Index*>& part = holders();
  const int P = (int)part.size();
  FilterStore::Filter f;
  f.bits.resize(P);
  for (int p = 0; p < P; ++p) {  // on the calling thread: a callback runs once per stored point in all
    if (part[p]->make_filter_bits(mode, sorted_ids, nids, fn, ctx, f.bits[p])) return fail(part[p]->err());
    f.counts.push_back(part[p]->n);
    size_t admitted = 0;
    for (uint32_t w : f.bits[p]) admitted += __builtin_popcount(w);
    f.admitted.push_back(admitted);
  }
  const int64_t id = filters.add(std::move(f));
  // the copy on the device of every partition now, so that no search pays for it
  for (int p = 0; p < P; ++p) {
    const uint32_t* d = nullptr;
    if (filters.use(id, p, P, part[p], &d)) {
      filters.erase(id);
      return fail(part[p]->err());
    }
  }
  return id;
}

int Index::free_filter(int64_t id) {
  if (!filters.has(id)) return fail(unknown_filter(id));
  // an asynchronous search_device / search_exact_device launch may still read the bitmap or the id list: wait for the contexts those launches run on
  DeviceRestore keep;
  HB_CUDA(cudaSetDevice(device));
  for (int i = NCTX; i < NCTX + NASYNC; ++i) HB_CUDA(cudaStreamSynchronize(ctx_[i].stream));
  filters.erase(id);
  return 0;
}

}  // namespace hb
