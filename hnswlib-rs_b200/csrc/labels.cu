// Point labels (index.h "point labels"): one u32 per point, next to the graph, that a search can restrict each query to.
// No kernel of its own.  A graph search with a label per query runs the filtered query kernel (filter.cu), whose
// admission test reads the label array instead of a bitmap.  An exact search runs the exact scan over one slice per
// label of a CSR of internal ids grouped by label, made on the host.
#include <algorithm>

#include "index.h"

namespace hb {

using GS = GraphStore;

int Index::set_labels(size_t first, size_t count, const uint32_t* labels) {
  if (count == 0) return 0;
  HB_CUDA(cudaSetDevice(device));
  std::copy(labels, labels + count, h_label.begin() + first);
  // on the handle's stream and waited for, so that no search launched after this call returns reads the old labels
  HB_CUDA(cudaMemcpyAsync(graph_.at<uint32_t>(GS::LABEL) + first, h_label.data() + first, count * 4, cudaMemcpyHostToDevice,
                          stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  ++label_version;
  return 0;
}

// A replica holds the handle's internal ids, so a copy of the handle's whole label array is its label array.  Labels
// change only under the handle's exclusive lock, so a search that finds the copy current uses it unchanged.
int Index::labels_on_device(const Index* src, const uint32_t** d_labels) {
  if (src != this) {
    std::lock_guard<std::mutex> lk(label_mu_);
    if (label_version != src->label_version) {
      DeviceRestore keep;
      HB_CUDA(cudaSetDevice(device));
      h_label = src->h_label;
      if (n) {
        HB_CUDA(cudaMemcpyAsync(graph_.at<uint32_t>(GS::LABEL), h_label.data(), n * 4, cudaMemcpyHostToDevice, stream_));
        HB_CUDA(cudaStreamSynchronize(stream_));
      }
      label_version = src->label_version;
    }
  }
  *d_labels = graph_.at<uint32_t>(GS::LABEL);
  return 0;
}

int Index::label_scan(uint32_t label, ExactScan* scan) {
  std::lock_guard<std::mutex> lk(label_mu_);
  LabelCsr& c = label_csr_;
  if (c.version != label_version) {
    // counts per label, then each group's offset, then the ids in ascending order into their groups
    c.groups.clear();
    size_t total = 0;
    for (size_t i = 0; i < n; ++i)
      if (h_label[i] != LABEL_NONE) {
        c.groups[h_label[i]].second++;
        total++;
      }
    uint32_t off = 0;
    for (auto& g : c.groups) {
      g.second.first = off;
      off += g.second.second;
    }
    std::vector<uint32_t> ids(total);
    std::unordered_map<uint32_t, uint32_t> at;
    for (const auto& g : c.groups) at[g.first] = g.second.first;
    for (size_t i = 0; i < n; ++i)
      if (h_label[i] != LABEL_NONE) ids[at[h_label[i]]++] = (uint32_t)i;
    DeviceRestore keep;
    HB_CUDA(cudaSetDevice(device));
    const size_t need = std::max<size_t>(total, 1) * 4;  // never null: a null list means every point
    if (need > c.bytes) {
      HB_CUDA(cudaStreamSynchronize(stream_));
      cudaFree(c.d_ids);
      c.d_ids = nullptr;
      c.bytes = 0;
      HB_CUDA(cudaMalloc(&c.d_ids, need));
      c.bytes = need;
    }
    if (total) {
      HB_CUDA(cudaMemcpyAsync(c.d_ids, ids.data(), total * 4, cudaMemcpyHostToDevice, stream_));
      HB_CUDA(cudaStreamSynchronize(stream_));
    }
    c.version = label_version;
  }
  auto g = c.groups.find(label);
  const uint32_t off = g == c.groups.end() ? 0 : g->second.first, cnt = g == c.groups.end() ? 0 : g->second.second;
  scan->ids = (const uint32_t*)c.d_ids + off;
  scan->n = cnt;
  return 0;
}

}  // namespace hb
