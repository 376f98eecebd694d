// Point labels (index.h "point labels"): one u32 per point, next to the graph, that a search can restrict each query to.
// No kernel of its own.  A graph search with a label set per query runs the filtered query kernel (filter.cu), whose
// admission test reads the label array and looks the point's label up in the query's set (or compares it, when every
// set is one label).  An exact search scans a label set's slices of a CSR of internal ids grouped by label, made on
// the host, joined into one list by copies when there are several (stage_plan).
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

int Index::label_set_scan(const uint32_t* set, size_t nset, std::vector<ExactScan>& slices) {
  std::lock_guard<std::mutex> lk(label_mu_);
  LabelCsr& c = label_csr_;
  if (c.version != label_version) {
    // counts per label, then each group's offset in ascending label order (so that a label set's adjacent labels are
    // one slice), then the ids in ascending order into their groups
    c.groups.clear();
    size_t total = 0;
    for (size_t i = 0; i < n; ++i)
      if (h_label[i] != LABEL_NONE) {
        c.groups[h_label[i]].second++;
        total++;
      }
    std::vector<uint32_t> order;
    order.reserve(c.groups.size());
    for (const auto& g : c.groups) order.push_back(g.first);
    std::sort(order.begin(), order.end());
    uint32_t off = 0;
    for (uint32_t L : order) {
      auto& g = c.groups[L];
      g.first = off;
      off += g.second;
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
  const size_t first = slices.size();
  for (size_t j = 0; j < nset; ++j) {
    auto g = c.groups.find(set[j]);  // a group holds at least one point
    if (g == c.groups.end()) continue;
    const ExactScan s{(const uint32_t*)c.d_ids + g->second.first, g->second.second};
    if (slices.size() > first && slices.back().ids + slices.back().n == s.ids)
      slices.back().n += s.n;
    else
      slices.push_back(s);
  }
  return 0;
}

}  // namespace hb
