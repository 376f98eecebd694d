// Deleted points (index.h "deleted points"): a bit per point that keeps it out of every search's answers.  No kernel of
// its own.  The filtered query kernel (filter.cu) rejects a deleted point where it rejects an excluded one, and the exact
// scan (aux.cu) where it tests a key's excluded list.  Unrestricted graph rows of an Index with deleted points run in
// the filtered kernel as a run over every point with the live stop rule (Index::resolve, RowFilter::live).  An update
// changes the host bits and copies the words it changed.
#include <algorithm>

#include "index.h"

namespace hb {

int Index::grow_deleted(size_t cap) {
  const size_t bytes = (cap + 31) / 32 * 4;
  if (bytes <= deleted.dev.size()) return 0;
  DeviceBuffer grown;
  HB_CUDA(grown.reset(bytes));
  HB_CUDA(cudaMemsetAsync(grown.as(), 0, bytes, stream_));
  if (deleted.dev.size())
    HB_CUDA(cudaMemcpyAsync(grown.as(), deleted.dev.as(), deleted.dev.size(), cudaMemcpyDeviceToDevice, stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  deleted.dev = std::move(grown);  // the old bitmap is freed with `grown`
  return 0;
}

int Index::mark_deleted(const uint64_t* ids, size_t count, bool on) {
  DeviceRestore keep;
  HB_CUDA(cudaSetDevice(device));
  // an asynchronous search_device / search_exact_device launch may still read the bitmap: wait for the contexts those
  // launches run on (the caller holds the Index exclusively, so no other search and no submitted batch is left)
  for (int i = NCTX; i < NCTX + NASYNC; ++i) HB_CUDA(cudaStreamSynchronize(ctx_[i].stream));
  DeletedSet& s = deleted;
  s.host.resize((n + 31) / 32, 0u);
  size_t lo = s.host.size(), hi = 0;  // the changed words [lo, hi]
  for (size_t i = 0; i < count; ++i) {
    const size_t w = ids[i] >> 5;
    const uint32_t m = 1u << (ids[i] & 31);
    if (((s.host[w] & m) != 0) == on) continue;  // already so: nothing to do
    s.host[w] ^= m;
    s.count += on ? 1 : -1;
    lo = std::min(lo, w);
    hi = std::max(hi, w);
  }
  if (lo > hi) return 0;
  HB_CUDA(cudaMemcpyAsync(deleted.dev.as<uint32_t>() + lo, s.host.data() + lo, (hi - lo + 1) * 4, cudaMemcpyHostToDevice,
                          stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  ++s.version;
  return 0;
}

// A replica holds the handle's internal ids, so a copy of the handle's bits is its set.  The set changes only under the
// handle's exclusive lock, so a search that finds the copy current uses it unchanged.
int Index::deleted_on_device(const Index* src, const uint32_t** d) {
  const DeletedSet& s = src->deleted;
  *d = nullptr;
  if (s.count == 0) return 0;
  if (src != this) {
    std::lock_guard<std::mutex> lk(label_mu_);
    if (deleted.version != s.version) {
      DeviceRestore keep;
      HB_CUDA(cudaSetDevice(device));
      if ((size_t)deleted.dev.size() < s.host.size() * 4) return fail("the deleted-point bitmap is smaller than the handle's");
      deleted.host = s.host;
      HB_CUDA(cudaMemcpyAsync(deleted.dev.as(), deleted.host.data(), deleted.host.size() * 4, cudaMemcpyHostToDevice, stream_));
      HB_CUDA(cudaStreamSynchronize(stream_));
      deleted.count = s.count;
      deleted.version = s.version;
    }
  }
  *d = deleted.dev.as<const uint32_t>();
  return 0;
}

}  // namespace hb
