// Point labels and attributes (index.h "point labels", "point attributes"): one u32 label and one int64 attribute per
// point, next to the graph, that a search can restrict each query to.  No kernel of its own.  A graph search with a
// label set per query runs the filtered query kernel (filter.cu), whose admission test reads the label array and looks
// the point's label up in the query's set (or compares it, when every set is one label), and with a range compares the
// point's attribute with its bounds.  An exact search scans a label set's slices of a CSR of internal ids grouped by
// label, or a range's slices of the points sorted by attribute (alone, or within each label), made on the host and
// joined into one list by copies when there are several (stage_plan).
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

int Index::set_attributes(size_t first, size_t count, const int64_t* values) {
  if (count == 0) return 0;
  HB_CUDA(cudaSetDevice(device));
  for (size_t i = 0; i < count; ++i) h_attr[first + i] = attr_bias(values[i]);
  // on the handle's stream and waited for, as set_labels does
  HB_CUDA(cudaMemcpyAsync(graph_.at<uint64_t>(GS::ATTR) + first, h_attr.data() + first, count * 8, cudaMemcpyHostToDevice,
                          stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  ++attr_version;
  return 0;
}

// labels_on_device's twin: attributes, too, change only under the handle's exclusive lock
int Index::attrs_on_device(const Index* src, const uint64_t** d_attrs) {
  if (src != this) {
    std::lock_guard<std::mutex> lk(label_mu_);
    if (attr_version != src->attr_version) {
      DeviceRestore keep;
      HB_CUDA(cudaSetDevice(device));
      h_attr = src->h_attr;
      if (n) {
        HB_CUDA(cudaMemcpyAsync(graph_.at<uint64_t>(GS::ATTR), h_attr.data(), n * 8, cudaMemcpyHostToDevice, stream_));
        HB_CUDA(cudaStreamSynchronize(stream_));
      }
      attr_version = src->attr_version;
    }
  }
  *d_attrs = graph_.at<uint64_t>(GS::ATTR);
  return 0;
}

// o made current (the caller holds label_mu_): the points with an attribute (and, by_label, a label) sorted by (value,
// id), or by (label, value, id) with each label's group
int Index::make_attr_order(AttrOrder& o, bool by_label) {
  if (o.version == attr_version && (!by_label || o.lversion == label_version)) return 0;
  std::vector<uint32_t> ids;
  for (size_t i = 0; i < n; ++i)
    if (h_attr[i] != 0 && (!by_label || h_label[i] != LABEL_NONE)) ids.push_back((uint32_t)i);
  auto key = [&](uint32_t i) { return std::make_tuple(by_label ? h_label[i] : 0u, h_attr[i], i); };
  std::sort(ids.begin(), ids.end(), [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
  o.values.resize(ids.size());
  o.groups.clear();
  for (size_t j = 0; j < ids.size(); ++j) {
    o.values[j] = h_attr[ids[j]];
    if (by_label) {
      auto g = o.groups.emplace(h_label[ids[j]], std::make_pair((uint32_t)j, 0u)).first;
      g->second.second++;
    }
  }
  DeviceRestore keep;
  HB_CUDA(cudaSetDevice(device));
  const size_t need = std::max<size_t>(ids.size(), 1) * 4;  // never null: a null list means every point
  if (need > o.bytes) {
    HB_CUDA(cudaStreamSynchronize(stream_));
    cudaFree(o.d_ids);
    o.d_ids = nullptr;
    o.bytes = 0;
    HB_CUDA(cudaMalloc(&o.d_ids, need));
    o.bytes = need;
  }
  if (!ids.empty()) {
    HB_CUDA(cudaMemcpyAsync(o.d_ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, stream_));
    HB_CUDA(cudaStreamSynchronize(stream_));
  }
  o.version = attr_version;
  o.lversion = label_version;
  return 0;
}

int Index::attr_range_scan(const uint32_t* set, size_t nset, uint64_t lo, uint64_t hi, std::vector<ExactScan>& slices) {
  std::lock_guard<std::mutex> lk(label_mu_);
  const bool by_label = !(nset == 1 && set[0] == LABEL_NONE);
  AttrOrder& o = by_label ? by_label_value_ : by_value_;
  int r;
  if ((r = make_attr_order(o, by_label))) return r;
  // the values of [b, e) in [lo, hi], as a slice of the order
  auto slice = [&](size_t b, size_t e) {
    const auto v = o.values.begin();
    const size_t s = std::lower_bound(v + b, v + e, lo) - v, t = lo > hi ? s : std::upper_bound(v + s, v + e, hi) - v;
    return ExactScan{(const uint32_t*)o.d_ids + s, t - s};
  };
  if (!by_label) {
    slices.push_back(slice(0, o.values.size()));
    return 0;
  }
  const size_t first = slices.size();
  for (size_t j = 0; j < nset; ++j) {
    auto g = o.groups.find(set[j]);
    if (g == o.groups.end()) continue;
    const ExactScan s = slice(g->second.first, (size_t)g->second.first + g->second.second);
    if (s.n == 0) continue;
    if (slices.size() > first && slices.back().ids + slices.back().n == s.ids)
      slices.back().n += s.n;
    else
      slices.push_back(s);
  }
  return 0;
}

}  // namespace hb
