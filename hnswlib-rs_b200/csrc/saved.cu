// Saved indexes (DESIGN.md "Saved indexes", under SURVEY §8 row f2): a handle written as the reference-format pair of
// each Index that holds its points (hnswio.cu's writer, unchanged) and one manifest, <base>.hnsw.b200, of what the pairs
// do not hold, written last.  Restore parses each pair with hnswio.cu's parser, puts its points back in insertion-rank
// order, imports them, and then sets the columns, the deleted points, the settings and the level RNG.  Host side only.
//
// Manifest, version 1, native endian (little-endian hosts), no padding:
//   u32 magic "HBSV", u32 version, u32 dtype, u32 metric, u32 M, u32 max_layer, u64 dim, u64 ef_c, u64 max_elements,
//   u32 link_mode, u32 visited_stages, u32 batch_ratio, u32 batch_max, u8 extend_candidates, u8 keep_pruned, u8 tie_std,
//   u8 columns (1 labels, 2 attributes, 4 deleted points), f64 level_scale, u64 level RNG state, u64 P, u64 count[P];
//   per partition with points: u64 graph size, u64 graph checksum, u64 data size, u64 data checksum, u64 rank[count]
//   (the local insertion rank of the pair's points in file order);
//   u32 label[n], i64 attribute[n], u8 deleted[(n + 7) / 8] (bit g % 8 of byte g / 8), each only when its column bit is
//   set, all by global insertion rank; u64 checksum of every byte before it.
// A checksum (Sum64) is mix64(length + sum over the bytes' little-endian u64 words w_i, the last zero-padded, of
// mix64(w_i ^ i * 0x9E3779B97F4A7C15)), mod 2^64: it finds a changed, truncated or replaced file, not a forged one.
#include <sys/stat.h>

#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "partition.h"

namespace hb {

namespace {

constexpr uint32_t MANIFEST_MAGIC = 0x56534248;  // "HBSV"
constexpr uint32_t MANIFEST_VERSION = 1;
enum Columns : uint8_t { HAS_LABELS = 1, HAS_ATTRS = 2, HAS_DELETED = 4 };

uint64_t mix64(uint64_t z) {  // the SplitMix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct Sum64 {
  uint64_t acc = 0, words = 0, bytes = 0;
  void add(const unsigned char* p, size_t len) {  // len is a multiple of 8 except at the last call
    for (size_t at = 0; at < len; at += 8) {
      uint64_t w = 0;
      memcpy(&w, p + at, std::min<size_t>(8, len - at));
      acc += mix64(w ^ (words++ * 0x9E3779B97F4A7C15ull));
    }
    bytes += len;
  }
  uint64_t value() const { return mix64(acc + bytes); }
};

bool file_sum(const std::string& path, uint64_t* size, uint64_t* sum) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  std::vector<unsigned char> buf((size_t)8 << 20);
  Sum64 s;
  size_t got;
  while ((got = fread(buf.data(), 1, buf.size(), f)) > 0) s.add(buf.data(), got);
  const bool ok = !ferror(f);
  fclose(f);
  *size = s.bytes;
  *sum = s.value();
  return ok;
}

bool exists(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0;
}

// partition p's pair of a save of P partitions: <base>-p<p>, or <base> itself when the handle is not partitioned
std::string pair_base(const std::string& base, int p, int P) { return P == 1 ? base : base + "-p" + std::to_string(p); }

struct Out {
  std::vector<unsigned char> b;
  template <class T>
  void put(const T& v) {
    bytes(&v, sizeof(T));
  }
  void bytes(const void* p, size_t n) { b.insert(b.end(), (const unsigned char*)p, (const unsigned char*)p + n); }
};
struct In {
  const unsigned char* p;
  size_t n, at = 0;
  bool ok = true;
  size_t left() const { return n - at; }
  template <class T>
  T get() {
    T v{};
    bytes(&v, sizeof(T));
    return v;
  }
  void bytes(void* dst, size_t len) {
    if (!ok || len > left()) {
      ok = false;
      return;
    }
    memcpy(dst, p + at, len);
    at += len;
  }
};

struct Manifest {
  uint32_t dtype = 0, metric = 0, M = 0, max_layer = 0;
  uint64_t dim = 0, ef_c = 0, max_elements = 0;
  Settings set{};
  uint64_t rng = 0;
  uint8_t columns = 0;
  std::vector<uint64_t> counts;
  struct Pair {
    uint64_t gsize = 0, gsum = 0, dsize = 0, dsum = 0;
    std::vector<uint64_t> rank;  // rank[f]: the local insertion rank of the pair's f-th point
  };
  std::vector<Pair> pairs;
  std::vector<uint32_t> labels;
  std::vector<int64_t> attrs;
  std::vector<uint8_t> deleted;
};

std::vector<unsigned char> write_manifest(const Manifest& m) {
  Out o;
  o.put(MANIFEST_MAGIC);
  o.put(MANIFEST_VERSION);
  o.put(m.dtype);
  o.put(m.metric);
  o.put(m.M);
  o.put(m.max_layer);
  o.put(m.dim);
  o.put(m.ef_c);
  o.put(m.max_elements);
  o.put((uint32_t)m.set.link_mode);
  o.put((uint32_t)m.set.visited_stages);
  o.put(m.set.batch_ratio);
  o.put(m.set.batch_max);
  o.put((uint8_t)m.set.extend_candidates);
  o.put((uint8_t)m.set.keep_pruned);
  o.put((uint8_t)m.set.tie_std);
  o.put(m.columns);
  o.put(m.set.level_scale);
  o.put(m.rng);
  o.put((uint64_t)m.counts.size());
  for (uint64_t c : m.counts) o.put(c);
  for (size_t p = 0; p < m.counts.size(); ++p) {
    if (!m.counts[p]) continue;
    const Manifest::Pair& pr = m.pairs[p];
    o.put(pr.gsize);
    o.put(pr.gsum);
    o.put(pr.dsize);
    o.put(pr.dsum);
    o.bytes(pr.rank.data(), pr.rank.size() * 8);
  }
  if (m.columns & HAS_LABELS) o.bytes(m.labels.data(), m.labels.size() * 4);
  if (m.columns & HAS_ATTRS) o.bytes(m.attrs.data(), m.attrs.size() * 8);
  if (m.columns & HAS_DELETED) o.bytes(m.deleted.data(), m.deleted.size());
  Sum64 s;
  s.add(o.b.data(), o.b.size());
  o.put(s.value());
  return o.b;
}

// "" when buf is a whole, consistent manifest (into m), else why not
std::string read_manifest(const std::vector<unsigned char>& buf, Manifest& m) {
  In h{buf.data(), buf.size()};
  const uint32_t magic = h.get<uint32_t>(), version = h.get<uint32_t>();
  if (!h.ok) return "truncated manifest";
  if (magic != MANIFEST_MAGIC) return "not a saved-index manifest (bad magic)";
  if (version != MANIFEST_VERSION)
    return "manifest version " + std::to_string(version) + " (this library reads version " + std::to_string(MANIFEST_VERSION) + ")";
  if (buf.size() < 16) return "truncated manifest";
  uint64_t stored;
  memcpy(&stored, buf.data() + buf.size() - 8, 8);
  Sum64 s;
  s.add(buf.data(), buf.size() - 8);
  if (s.value() != stored) return "manifest checksum mismatch (the manifest is truncated or was changed after the save)";
  In in{buf.data(), buf.size() - 8};
  in.at = 8;
  m.dtype = in.get<uint32_t>();
  m.metric = in.get<uint32_t>();
  m.M = in.get<uint32_t>();
  m.max_layer = in.get<uint32_t>();
  m.dim = in.get<uint64_t>();
  m.ef_c = in.get<uint64_t>();
  m.max_elements = in.get<uint64_t>();
  m.set.link_mode = (int)in.get<uint32_t>();
  m.set.visited_stages = (int)in.get<uint32_t>();
  m.set.batch_ratio = in.get<uint32_t>();
  m.set.batch_max = in.get<uint32_t>();
  m.set.extend_candidates = in.get<uint8_t>() != 0;
  m.set.keep_pruned = in.get<uint8_t>() != 0;
  m.set.tie_std = in.get<uint8_t>() != 0;
  m.columns = in.get<uint8_t>();
  m.set.level_scale = in.get<double>();
  m.set.stats = false;
  m.rng = in.get<uint64_t>();
  const uint64_t P = in.get<uint64_t>();
  if (!in.ok) return "truncated manifest";
  if (m.dtype > DT_I32 || m.metric > METRIC_JENSENSHANNON || !metric_supported((int)m.metric, (int)m.dtype))
    return "unknown element type or distance";
  if (m.M < 2 || m.M > 256 || m.max_layer != MAX_LAYERS || m.dim == 0 || m.dim > ((uint64_t)1 << 24) || m.ef_c == 0 ||
      m.ef_c > (1u << 30))
    return "bad configuration (M, max_layer, dimension or ef_construction)";
  if (m.set.link_mode > 1 || m.set.visited_stages < 0 || m.set.visited_stages > 2 || m.set.batch_ratio == 0 ||
      m.set.batch_max == 0 || !(m.set.level_scale > 0) || (m.columns & ~7u))
    return "bad settings";
  if (P < 1 || P > (uint64_t)Partitions::MAX_PARTS) return "bad partition count";
  if (in.left() < P * 8) return "truncated manifest";
  m.counts.resize(P);
  uint64_t total = 0;
  for (uint64_t& c : m.counts) {
    c = in.get<uint64_t>();
    if (c >= ((uint64_t)1 << 31)) return "bad point count";
    total += c;
  }
  if (total == 0) return "no points";
  for (uint64_t p = 0; p < P; ++p)
    if (m.counts[p] != (total + P - 1 - p) / P) return "the partitions' point counts do not follow the placement rule";
  m.pairs.resize(P);
  for (uint64_t p = 0; p < P; ++p) {
    const uint64_t c = m.counts[p];
    if (!c) continue;
    Manifest::Pair& pr = m.pairs[p];
    pr.gsize = in.get<uint64_t>();
    pr.gsum = in.get<uint64_t>();
    pr.dsize = in.get<uint64_t>();
    pr.dsum = in.get<uint64_t>();
    if (!in.ok || in.left() < c * 8) return "truncated manifest";
    pr.rank.resize(c);
    in.bytes(pr.rank.data(), c * 8);
    std::vector<bool> seen(c, false);
    for (uint64_t r : pr.rank) {
      if (r >= c || seen[r]) return "the rank list of partition " + std::to_string(p) + " is not a permutation";
      seen[r] = true;
    }
  }
  const uint64_t want = (m.columns & HAS_LABELS ? total * 4 : 0) + (m.columns & HAS_ATTRS ? total * 8 : 0) +
                        (m.columns & HAS_DELETED ? (total + 7) / 8 : 0);
  if (in.left() != want) return in.left() < want ? "truncated manifest" : "trailing bytes in the manifest";
  if (m.columns & HAS_LABELS) {
    m.labels.resize(total);
    in.bytes(m.labels.data(), total * 4);
  }
  if (m.columns & HAS_ATTRS) {
    m.attrs.resize(total);
    in.bytes(m.attrs.data(), total * 8);
  }
  if (m.columns & HAS_DELETED) {
    m.deleted.resize((total + 7) / 8);
    in.bytes(m.deleted.data(), m.deleted.size());
  }
  return in.ok ? "" : "truncated manifest";
}

// d's points moved into insertion-rank order: the point at file position f goes to rank[f], and every list, list entry
// and the entry point follow it
void to_rank_order(ParsedDump& d, const std::vector<uint64_t>& rank) {
  const size_t N = d.n, row = d.vecs.size() / N;
  std::vector<uint64_t> origin(N), file_of(N);
  std::vector<uint8_t> levels(N);
  std::vector<unsigned char> vecs(d.vecs.size());
  for (size_t f = 0; f < N; ++f) {
    const uint64_t r = rank[f];
    file_of[r] = f;
    origin[r] = d.origin[f];
    levels[r] = d.levels[f];
    memcpy(vecs.data() + r * row, d.vecs.data() + f * row, row);
  }
  for (int l = 0; l < d.nlayers; ++l) {
    std::vector<uint64_t> off(N + 1, 0);
    std::vector<uint32_t> ids;
    std::vector<float> ds;
    ids.reserve(d.ids[l].size());
    ds.reserve(d.ids[l].size());
    for (size_t r = 0; r < N; ++r) {
      off[r] = ids.size();
      const size_t f = file_of[r];
      for (uint64_t j = d.off[l][f]; j < d.off[l][f + 1]; ++j) {
        ids.push_back((uint32_t)rank[d.ids[l][j]]);
        ds.push_back(d.dists[l][j]);
      }
    }
    off[N] = ids.size();
    d.off[l].swap(off);
    d.ids[l].swap(ids);
    d.dists[l].swap(ds);
  }
  d.origin.swap(origin);
  d.levels.swap(levels);
  d.vecs.swap(vecs);
  d.entry = (int64_t)rank[d.entry];
}

}  // namespace

// ------------------------------------------------------------------------------------------------ save
int Index::save(const std::string& dir, const std::string& basename, bool overwrite, std::string* used) {
  if (owner) return fail("save: a partition view cannot be saved; save its partitioned handle");
  if (parts && !parts->broken().empty()) return fail("save: " + parts->broken());
  const std::vector<Index*>& hs = holders();
  const int P = (int)hs.size();
  const size_t total = nb_point();
  if (total == 0) return fail("save: entry point not initialized (the index holds no point)");
  if (max_layer != MAX_LAYERS) return fail("save: nb_layer != NB_MAX_LAYER (hnswio.rs:893-896)");
  for (int p = 0; p < P; ++p)
    if (hs[p]->poisoned_) return holder_fail(p, hs[p]->fail(hs[p]->poison_msg_));
  // the set's files; with overwrite off, a basename none of them exists under (DumpInit, hnswio.rs:150-236)
  auto files = [&](const std::string& b) {
    std::vector<std::string> f;
    for (int p = 0; p < P; ++p)
      if (hs[p]->n) {
        f.push_back(dir + "/" + pair_base(b, p, P) + ".hnsw.graph");
        f.push_back(dir + "/" + pair_base(b, p, P) + ".hnsw.data");
      }
    f.push_back(dir + "/" + b + ".hnsw.b200");
    return f;
  };
  auto any_exists = [&](const std::string& b) {
    for (const std::string& f : files(b))
      if (exists(f)) return true;
    return false;
  };
  std::string base = basename;
  if (!overwrite && any_exists(base)) {
    std::mt19937_64 rng(std::random_device{}());
    do base = basename + "-" + std::to_string(rng() % 10000);
    while (any_exists(base));
  }
  const std::vector<std::string> written = files(base);
  const std::string mpath = written.back();
  // an earlier manifest goes first, so that a save interrupted below leaves no manifest over changed pairs
  remove(mpath.c_str());
  auto undo = [&](int r) {
    for (const std::string& f : written) remove(f.c_str());
    return r;
  };
  Manifest m;
  m.dtype = (uint32_t)dtype;
  m.metric = (uint32_t)metric;
  m.M = (uint32_t)M;
  m.max_layer = (uint32_t)max_layer;
  m.dim = (uint64_t)dim;
  m.ef_c = (uint64_t)ef_c;
  m.max_elements = (uint64_t)max_elements;
  m.set = settings();
  m.rng = rng.s;  // a partition's own RNG is never drawn: Partitions::insert passes every level
  m.counts.resize(P);
  m.pairs.resize(P);
  for (int p = 0; p < P; ++p) {
    Index* x = hs[p];
    m.counts[p] = x->n;
    if (!x->n) continue;
    const std::string pb = dir + "/" + pair_base(base, p, P);
    if (int r = x->file_dump(dir, pair_base(base, p, P), true, nullptr)) return undo(holder_fail(p, r));
    Manifest::Pair& pr = m.pairs[p];
    if (!file_sum(pb + ".hnsw.graph", &pr.gsize, &pr.gsum) || !file_sum(pb + ".hnsw.data", &pr.dsize, &pr.dsum))
      return undo(fail("save: could not read back " + pb + ".hnsw.graph / .hnsw.data"));
    pr.rank.reserve(x->n);
    for (int lay = 0; lay < MAX_LAYERS; ++lay)  // file_dump's order: layer by layer, insertion order within a layer
      for (size_t i = 0; i < x->n; ++i)
        if (x->h_level[i] == lay) pr.rank.push_back(i);
  }
  // the columns by global rank, each only when some point has a value
  auto value = [&](uint64_t g) {
    const Placed at = place(g, P);
    return std::make_pair(hs[at.part], (size_t)at.local);
  };
  bool any_label = false, any_attr = false, any_deleted = false;
  for (const Index* x : hs) {
    for (uint32_t v : x->labels.host) any_label = any_label || v != LABEL_NONE;
    for (uint64_t v : x->attrs.host) any_attr = any_attr || v != attr_bias(ATTR_NONE);
    any_deleted = any_deleted || x->deleted.count > 0;
  }
  m.columns = (any_label ? HAS_LABELS : 0) | (any_attr ? HAS_ATTRS : 0) | (any_deleted ? HAS_DELETED : 0);
  if (any_label) m.labels.resize(total);
  if (any_attr) m.attrs.resize(total);
  if (any_deleted) m.deleted.assign((total + 7) / 8, 0);
  for (uint64_t g = 0; g < total; ++g) {
    const auto xp = value(g);
    const Index* x = xp.first;
    const size_t i = xp.second;
    if (any_label) m.labels[g] = x->labels.host[i];
    if (any_attr) m.attrs[g] = attr_unbias(x->attrs.host[i]);
    if (any_deleted && i / 32 < x->deleted.host.size() && ((x->deleted.host[i / 32] >> (i % 32)) & 1u))
      m.deleted[g / 8] |= (uint8_t)(1u << (g % 8));
  }
  const std::vector<unsigned char> bytes = write_manifest(m);
  FILE* f = fopen(mpath.c_str(), "wb");
  if (!f) return undo(fail("save: could not open " + mpath));
  const bool ok = fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
  if (fclose(f) != 0 || !ok) return undo(fail("save: write error on " + mpath));
  if (used) *used = base;
  return 0;
}

// ------------------------------------------------------------------------------------------------ restore
Index* Index::restore(const std::string& dir, const std::string& basename, int ndev, const int* devices, int device,
                      std::string& err) {
  const std::string mpath = dir + "/" + basename + ".hnsw.b200";
  auto refuse = [&](const std::string& why) -> Index* {
    err = "restore: " + why;
    return nullptr;
  };
  std::vector<unsigned char> buf;
  {
    FILE* f = fopen(mpath.c_str(), "rb");
    if (!f) return refuse("could not open the manifest " + mpath);
    unsigned char chunk[1 << 16];
    size_t got;
    while ((got = fread(chunk, 1, sizeof chunk, f)) > 0) buf.insert(buf.end(), chunk, chunk + got);
    const bool bad = ferror(f);
    fclose(f);
    if (bad) return refuse("read error on " + mpath);
  }
  Manifest m;
  const std::string why = read_manifest(buf, m);
  if (!why.empty()) return refuse(mpath + ": " + why);
  const int P = (int)m.counts.size();
  if (P == 1 ? (ndev != 0 && ndev != 1) : ndev != P)
    return refuse(mpath + " holds " + std::to_string(P) + " partition(s): ndev must be " + (P == 1 ? "0 or 1" : std::to_string(P)) +
                  ", not " + std::to_string(ndev));
  if (ndev > 0 && !devices) return refuse("devices is NULL");
  for (int p = 0; p < P; ++p) {  // every pair as the manifest recorded it, before anything is allocated
    if (!m.counts[p]) continue;
    const std::string pb = dir + "/" + pair_base(basename, p, P);
    const Manifest::Pair& pr = m.pairs[p];
    const std::pair<std::string, const uint64_t*> two[2] = {{pb + ".hnsw.graph", &pr.gsize}, {pb + ".hnsw.data", &pr.dsize}};
    for (const auto& fs : two) {
      uint64_t size = 0, sum = 0;
      if (!file_sum(fs.first, &size, &sum)) return refuse("could not read " + fs.first);
      if (size != fs.second[0])
        return refuse(fs.first + ": " + std::to_string(size) + " bytes, the manifest says " + std::to_string(fs.second[0]));
      if (sum != fs.second[1]) return refuse(fs.first + ": checksum differs from the manifest's (changed or replaced after the save)");
    }
  }
  DeviceRestore keep;
  std::unique_ptr<Index> ix(new Index((int)m.M, (size_t)m.max_elements, (int)m.max_layer, (int)m.ef_c, (int)m.metric,
                                      (int)m.dtype, ndev ? devices[0] : device));
  if (!ix->ok()) return refuse(ix->err());
  if (P > 1 && Partitions::create(ix.get(), P, devices)) return refuse(ix->err());
  const std::vector<Index*>& hs = ix->holders();
  // ---- the pairs, parsed, put in rank order and imported, every partition at once
  auto load = [&](int p) -> int {
    Index* x = hs[p];
    if (!m.counts[p]) return 0;
    const std::string pb = pair_base(basename, p, P);
    ParsedDump d;
    if (int r = x->parse_dump(dir, pb, d)) return r;
    if (d.n != m.counts[p] || (uint64_t)d.d != m.dim)
      return x->fail(dir + "/" + pb + ".hnsw.graph holds " + std::to_string(d.n) + " points of dimension " + std::to_string(d.d) +
                     ", the manifest " + std::to_string(m.counts[p]) + " of dimension " + std::to_string(m.dim));
    to_rank_order(d, m.pairs[p].rank);
    return x->import_dump(d);
  };
  if ((P > 1 ? ix->parts->run(load) : load(0)) != 0) return refuse(ix->err());
  for (Index* x : hs) x->set_dim((int)m.dim);  // also the partitions without a point
  ix->set_dim((int)m.dim);
  // ---- the columns and the deleted points, each holder its share by placement
  for (int p = 0; p < P; ++p) {
    Index* x = hs[p];
    const size_t cnt = m.counts[p];
    auto g = [&](size_t i) { return (size_t)global_rank(p, i, P); };
    int r = 0;
    if (m.columns & HAS_LABELS) r = x->set_points(x->labels, 0, cnt, [&](size_t i) { return m.labels[g(i)]; });
    if (!r && (m.columns & HAS_ATTRS)) r = x->set_points(x->attrs, 0, cnt, [&](size_t i) { return attr_bias(m.attrs[g(i)]); });
    if (!r && (m.columns & HAS_DELETED)) {
      std::vector<uint64_t> ids;
      for (size_t i = 0; i < cnt; ++i)
        if ((m.deleted[g(i) / 8] >> (g(i) % 8)) & 1u) ids.push_back(i);
      r = x->mark_deleted(ids.data(), ids.size(), true);
    }
    if (r) {
      ix->holder_fail(p, r);
      return refuse(ix->err());
    }
  }
  ix->settings_ = m.set;
  ix->rng.s = m.rng;
  return ix.release();
}

}  // namespace hb
