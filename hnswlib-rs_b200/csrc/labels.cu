// Point labels and attributes (index.h "point labels and attributes"): one u32 label and one int64 attribute per point,
// next to the graph, that a search can restrict each query to.  No kernel of its own.  A graph search with a label set
// per query runs the filtered query kernel (filter.cu), whose admission test reads the label array and looks the
// point's label up in the query's set (or compares it, when every set is one label), and with a range compares the
// point's attribute with its bounds.  An exact search scans slices of an order of the internal ids made on the host: a
// label set's groups of the ids by label, a range's slice of the ids by value, or both's slices of the ids by label and
// value, joined into one list by copies when there are several (stage_plan).
#include <algorithm>

#include "index.h"

namespace hb {

// A replica holds the handle's internal ids, so a copy of the handle's whole column is its column.  Columns change only
// under the handle's exclusive lock, so a search that finds the copy current uses it unchanged.
template <class T>
int Index::on_device(PointColumn<T> Index::*col, const Index* src, const T** d) {
  PointColumn<T>& c = this->*col;
  if (src != this) {
    std::lock_guard<std::mutex> lk(label_mu_);
    const PointColumn<T>& s = src->*col;
    if (c.version != s.version) {
      DeviceRestore keep;
      HB_CUDA(cudaSetDevice(device));
      c.host = s.host;
      if (n) {
        HB_CUDA(cudaMemcpyAsync(graph_.at<T>(c.array), c.host.data(), n * sizeof(T), cudaMemcpyHostToDevice, stream_));
        HB_CUDA(cudaStreamSynchronize(stream_));
      }
      c.version = s.version;
    }
  }
  *d = graph_.at<T>(c.array);
  return 0;
}
template int Index::on_device(PointColumn<uint32_t> Index::*, const Index*, const uint32_t**);
template int Index::on_device(PointColumn<uint64_t> Index::*, const Index*, const uint64_t**);

// o made current (the caller holds label_mu_).  Counts per group, then each group's offset in ascending label order (so
// that a label set's adjacent labels are one slice), then the ids in ascending order into their groups; a value-keyed
// order then sorts each group by (value, id).
int Index::make_order(ScanOrder& o) {
  if ((!o.by_label || o.label_version == labels.version) && (!o.by_value || o.attr_version == attrs.version)) return 0;
  const std::vector<uint32_t>& lab = labels.host;
  const std::vector<uint64_t>& val = attrs.host;
  auto member = [&](size_t i) { return (!o.by_label || lab[i] != LABEL_NONE) && (!o.by_value || val[i] != 0); };
  auto group = [&](size_t i) { return o.by_label ? lab[i] : LABEL_NONE; };
  o.groups.clear();
  size_t total = 0;
  for (size_t i = 0; i < n; ++i)
    if (member(i)) {
      o.groups[group(i)].second++;
      total++;
    }
  std::vector<uint32_t> order;
  order.reserve(o.groups.size());
  for (const auto& g : o.groups) order.push_back(g.first);
  std::sort(order.begin(), order.end());
  uint32_t off = 0;
  for (uint32_t L : order) {
    auto& g = o.groups[L];
    g.first = off;
    off += g.second;
  }
  std::vector<uint32_t> ids(total);
  std::unordered_map<uint32_t, uint32_t> at;
  for (const auto& g : o.groups) at[g.first] = g.second.first;
  for (size_t i = 0; i < n; ++i)
    if (member(i)) ids[at[group(i)]++] = (uint32_t)i;
  if (o.by_value) {
    for (const auto& g : o.groups)
      std::sort(ids.begin() + g.second.first, ids.begin() + g.second.first + g.second.second,
                [&](uint32_t a, uint32_t b) { return std::make_pair(val[a], a) < std::make_pair(val[b], b); });
    o.values.resize(total);
    for (size_t j = 0; j < total; ++j) o.values[j] = val[ids[j]];
  }
  DeviceRestore keep;
  HB_CUDA(cudaSetDevice(device));
  HB_CUDA(o.d_ids.grow(std::max<size_t>(total, 1) * 4, stream_));  // never null: a null list means every point
  if (total) {
    HB_CUDA(cudaMemcpyAsync(o.d_ids.as(), ids.data(), total * 4, cudaMemcpyHostToDevice, stream_));
    HB_CUDA(cudaStreamSynchronize(stream_));
  }
  o.label_version = labels.version;
  o.attr_version = attrs.version;
  return 0;
}

int Index::scan_slices(const uint32_t* set, size_t nset, uint64_t lo, uint64_t hi, std::vector<ExactScan>& slices) {
  std::lock_guard<std::mutex> lk(label_mu_);
  ScanOrder& o = lo == 0 ? by_label_ : nset == 1 && set[0] == LABEL_NONE ? by_value_ : by_label_value_;
  int r;
  if ((r = make_order(o))) return r;
  const size_t first = slices.size();
  for (size_t j = 0; j < nset; ++j) {
    auto g = o.groups.find(set[j]);  // a group holds at least one point
    if (g == o.groups.end()) continue;
    size_t b = g->second.first, e = b + g->second.second;
    if (o.by_value) {  // the group's values in [lo, hi]
      const auto v = o.values.begin();
      b = std::lower_bound(v + b, v + e, lo) - v;
      e = std::upper_bound(v + b, v + e, hi) - v;
      if (b == e) continue;
    }
    const ExactScan s{o.d_ids.as<const uint32_t>() + b, e - b};
    if (slices.size() > first && slices.back().ids + slices.back().n == s.ids)
      slices.back().n += s.n;
    else
      slices.push_back(s);
  }
  return 0;
}

}  // namespace hb
