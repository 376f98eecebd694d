// Dump / reload in the reference's on-disk format (SURVEY §8 row f2), host-side only.
//   writer: /root/reference/src/hnswio.rs:878-919 (Description::dump), 1063-1115 (dump_point),
//           1303-1340 (PointIndexation::dump), 1355-1387 (Hnsw::dump), 150-236 (DumpInit naming)
//   reader: /root/reference/src/hnswio.rs:937-1042 (load_description), 1221-1289 (load_point_graph),
//           1119-1178 (load_point_data), 615-784 (load_point_indexation)
// Native-endian, usize = 8 bytes.  <base>.hnsw.graph holds the description and the adjacency (neighbours named
// by DataId + PointId(level, rank) + distance), <base>.hnsw.data the vectors in the same point order.
// A graph dumped by the reference can be loaded here and searched on the GPU, and vice versa.
#include <sys/stat.h>

#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "index.h"

namespace hb {

static const uint32_t MAGICPOINT = 0x000a678f;    // hnswio.rs:47
static const uint32_t MAGICDESCR_2 = 0x002a677f;  // :49 (bincode-encoded vectors: not readable here)
static const uint32_t MAGICDESCR_3 = 0x002a6771;  // :56
static const uint32_t MAGICDESCR_4 = 0x002a6779;  // :60
static const uint32_t MAGICLAYER = 0x000a676f;    // :63
static const uint32_t MAGICDATAP = 0xa67f0000;    // :65

// the anndists distance types, by metric id: the C ABI names them bare, a dump by their full type path
static const char* const METRIC_NAMES[] = {"DistL1",      "DistL2",        "DistDot",      "DistCosine",       "DistHamming",
                                           "DistJaccard", "DistHellinger", "DistJeffreys", "DistJensenShannon"};
static_assert(sizeof(METRIC_NAMES) / sizeof(METRIC_NAMES[0]) == METRIC_JENSENSHANNON + 1, "one name per metric id");

static std::string metric_type_name(int metric) {  // std::any::type_name::<D>()
  if (metric < 0 || metric > METRIC_JENSENSHANNON) return "?";
  return std::string("anndists::dist::distances::") + METRIC_NAMES[metric];
}
static const char* dtype_type_name(int dt) {
  switch (dt) {
    case DT_F32: return "f32";
    case DT_U8: return "u8";
    case DT_U16: return "u16";
    case DT_U32: return "u32";
    case DT_I32: return "i32";
  }
  return "?";
}
int metric_from_name(const std::string& name) {
  for (int m = 0; m <= METRIC_JENSENSHANNON; ++m)
    if (name == METRIC_NAMES[m]) return m;
  return -1;
}
int metric_from_type_name(const std::string& full) {
  const size_t p = full.rfind("::");
  return metric_from_name(p == std::string::npos ? full : full.substr(p + 2));
}
int dtype_from_type_name(const std::string& s) {
  if (s == "f32") return DT_F32;
  if (s == "u8") return DT_U8;
  if (s == "u16") return DT_U16;
  if (s == "u32") return DT_U32;
  if (s == "i32") return DT_I32;
  return -1;
}

struct Writer {
  FILE* f = nullptr;
  bool ok = true;
  template <class T>
  void put(const T& v) {
    if (ok && fwrite(&v, sizeof(T), 1, f) != 1) ok = false;
  }
  void bytes(const void* p, size_t n) {
    if (ok && n && fwrite(p, 1, n, f) != n) ok = false;
  }
};
struct Reader {
  FILE* f = nullptr;
  bool ok = true;
  template <class T>
  T get() {
    T v{};
    if (ok && fread(&v, sizeof(T), 1, f) != 1) ok = false;
    return v;
  }
  void bytes(void* p, size_t n) {
    if (ok && n && fread(p, 1, n, f) != n) ok = false;
  }
};

static bool exists(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0;
}

// ------------------------------------------------------------------------------------------------ dump
int Index::file_dump(const std::string& dir, const std::string& basename_default, bool overwrite, std::string* used) {
  if (poisoned_) return fail(poison_msg_);
  if (max_layer != MAX_LAYERS) return fail("dump of Description, nb_layer != NB_MAX_LAYER (hnswio.rs:893-896)");
  if (n == 0 || entry == INVALID_ID) return fail("entry point not initialized (hnswio.rs:1323-1325)");
  // DumpInit::new (hnswio.rs:150-236): keep an existing data file when overwrite is false
  std::string base = basename_default;
  if (!overwrite && exists(dir + "/" + base + ".hnsw.data")) {
    std::mt19937_64 rng(std::random_device{}());
    for (;;) {
      base = basename_default + "-" + std::to_string(rng() % 10000);
      if (!exists(dir + "/" + base + ".hnsw.data")) break;
    }
  }
  // ---- gather the graph on the host
  std::vector<LayerCsr> layers;
  int r;
  if ((r = export_layers(0, top_layer(), layers))) return r;
  std::vector<unsigned char> vecs(n * (size_t)dim * es);
  if ((r = export_vectors(vecs.data()))) return r;
  std::vector<std::vector<uint32_t>> by_level(MAX_LAYERS);  // points_by_layer: rank order == insertion order
  for (size_t p = 0; p < n; ++p) by_level[h_level[p]].push_back((uint32_t)p);

  Writer g, d;
  g.f = fopen((dir + "/" + base + ".hnsw.graph").c_str(), "wb");
  d.f = fopen((dir + "/" + base + ".hnsw.data").c_str(), "wb");
  if (!g.f || !d.f) {
    if (g.f) fclose(g.f);
    if (d.f) fclose(d.f);
    return fail("DumpInit: could not open dump files in " + dir);
  }
  // ---- Description (hnswio.rs:878-919), format v4
  g.put<uint32_t>(MAGICDESCR_4);
  g.put<uint8_t>(1);                 // DumpMode::Full
  g.put<uint8_t>((uint8_t)M);        // get_max_nb_connection() as u8 (256 wraps to 0 upstream too)
  g.put<double>(level_scale);        // v4: level scale
  g.put<uint8_t>((uint8_t)max_layer);
  g.put<uint64_t>((uint64_t)ef_c);
  g.put<uint64_t>((uint64_t)n);
  g.put<uint64_t>((uint64_t)dim);
  const std::string dn = metric_type_name(metric), tn = dtype_type_name(dtype);
  g.put<uint64_t>(dn.size());
  g.bytes(dn.data(), dn.size());
  g.put<uint64_t>(tn.size());
  g.bytes(tn.data(), tn.size());
  // ---- data header (hnswio.rs:1382-1383)
  d.put<uint32_t>(MAGICDATAP);
  d.put<uint64_t>((uint64_t)dim);
  // ---- PointIndexation::dump (hnswio.rs:1303-1340)
  g.put<uint8_t>((uint8_t)max_layer);
  for (int lay = 0; lay < max_layer; ++lay) {
    g.put<uint32_t>(MAGICLAYER);
    g.put<uint64_t>(by_level[lay].size());
    for (uint32_t p : by_level[lay]) {  // dump_point, hnswio.rs:1063-1115
      g.put<uint32_t>(MAGICPOINT);
      g.put<uint64_t>(h_origin[p]);
      g.put<uint8_t>(h_level[p]);
      g.put<int32_t>(h_rank[p]);
      for (int l = 0; l < MAX_LAYERS; ++l) {
        uint64_t b = 0, e = 0;
        if (l < (int)layers.size()) {  // above the top layer every list is empty
          b = layers[l].off[p];
          e = layers[l].off[p + 1];
        }
        g.put<uint64_t>(e - b);
        for (uint64_t j = b; j < e; ++j) {
          const uint32_t q = layers[l].ids[j];
          g.put<uint64_t>(h_origin[q]);
          g.put<uint8_t>(h_level[q]);
          g.put<int32_t>(h_rank[q]);
          g.put<float>(layers[l].dists[j]);
        }
      }
      d.put<uint32_t>(MAGICDATAP);
      d.put<uint64_t>(h_origin[p]);
      d.put<uint64_t>((uint64_t)dim * es);
      d.bytes(vecs.data() + (size_t)p * dim * es, (size_t)dim * es);
    }
  }
  g.put<uint64_t>(h_origin[entry]);
  g.put<uint8_t>(h_level[entry]);
  g.put<int32_t>(h_rank[entry]);
  const bool ok = g.ok && d.ok;
  if (fclose(g.f) != 0 || fclose(d.f) != 0 || !ok) return fail("write error while dumping");
  if (used) *used = base;
  return 0;
}

// ------------------------------------------------------------------------------------------------ description
int read_description(const std::string& graph_path, DumpDescription& out, std::string& err) {
  Reader r;
  r.f = fopen(graph_path.c_str(), "rb");
  if (!r.f) {
    err = "could not open file " + graph_path;
    return -1;
  }
  const uint32_t magic = r.get<uint32_t>();
  if (magic == MAGICDESCR_2) out.format_version = 2;
  else if (magic == MAGICDESCR_3) out.format_version = 3;
  else if (magic == MAGICDESCR_4) out.format_version = 4;
  else {
    fclose(r.f);
    err = "bad magic at descr beginning";
    return -1;
  }
  out.dumpmode = r.get<uint8_t>();
  out.max_nb_connection = r.get<uint8_t>();
  out.level_scale = out.format_version == 4 ? r.get<double>() : 1.0;
  out.nb_layer = r.get<uint8_t>();
  out.ef = r.get<uint64_t>();
  out.nb_point = r.get<uint64_t>();
  out.dimension = r.get<uint64_t>();
  uint64_t len = r.get<uint64_t>();
  if (!r.ok || len > 256) {
    fclose(r.f);
    err = "bad length for distance name";
    return -1;
  }
  out.distname.resize(len);
  r.bytes(&out.distname[0], len);
  len = r.get<uint64_t>();
  if (!r.ok || len > 256) {
    fclose(r.f);
    err = "bad length for T name";
    return -1;
  }
  out.t_name.resize(len);
  r.bytes(&out.t_name[0], len);
  out.header_bytes = ftell(r.f);
  fclose(r.f);
  if (!r.ok) {
    err = "truncated description";
    return -1;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ load
int Index::load_dump(const std::string& dir, const std::string& basename) {
  if (n != 0) return fail("load needs an empty index");
  const std::string gpath = dir + "/" + basename + ".hnsw.graph", dpath = dir + "/" + basename + ".hnsw.data";
  DumpDescription de;
  std::string e;
  if (read_description(gpath, de, e)) return fail(e);
  if (de.format_version == 2) return fail("dump format v2 (bincode-encoded vectors) is not supported; re-dump with hnsw_rs >= 0.2");
  if (de.dumpmode != 1) return fail("only DumpMode::Full dumps can be reloaded");
  if (dtype_from_type_name(de.t_name) != dtype) return fail("dump holds element type '" + de.t_name + "', handle type differs");
  if (metric_from_type_name(de.distname) != metric) return fail("dump was built with distance '" + de.distname + "'");
  const int dumpM = de.max_nb_connection == 0 ? 256 : de.max_nb_connection;
  if (dumpM != M) return fail("dump max_nb_connection differs from the handle's");
  Reader g, d;
  g.f = fopen(gpath.c_str(), "rb");
  d.f = fopen(dpath.c_str(), "rb");
  if (!g.f || !d.f) {
    if (g.f) fclose(g.f);
    if (d.f) fclose(d.f);
    return fail("could not open " + gpath + " / " + dpath);
  }
  fseek(g.f, de.header_bytes, SEEK_SET);
  auto bail = [&](const std::string& m) {
    fclose(g.f);
    fclose(d.f);
    return fail(m);
  };
  if (d.get<uint32_t>() != MAGICDATAP) return bail("bad magic at data beginning");
  const uint64_t ddim = d.get<uint64_t>();
  if (ddim != de.dimension) return bail("data dimension differs between graph and data files");
  const size_t N = (size_t)de.nb_point, D = (size_t)de.dimension, ES = (size_t)dtype_size(dtype);
  {  // a corrupt header must not size the allocations below: every point costs >= 20 + D*ES bytes of .hnsw.data and
     // >= 17 bytes of .hnsw.graph
    struct stat sd, sg;
    if (stat(dpath.c_str(), &sd) != 0 || stat(gpath.c_str(), &sg) != 0) return bail("cannot stat the dump files");
    if (D == 0 || D > ((size_t)1 << 24) || N > (size_t)sd.st_size / (20 + D * ES) + 1 || N > (size_t)sg.st_size / 17 + 1)
      return bail("dump header (nb_point, dimension) is inconsistent with the file sizes");
  }
  const int nb_layer = g.get<uint8_t>();
  if (nb_layer > MAX_LAYERS) return bail("nb_layer > 16");
  struct Nb {
    uint8_t level;
    int32_t rank;
    float dist;
  };
  std::vector<uint64_t> origin;
  std::vector<uint8_t> levels;
  std::vector<unsigned char> vecs;
  origin.reserve(N);
  levels.reserve(N);
  vecs.reserve(N * D * ES);
  std::vector<std::vector<std::vector<Nb>>> lists(MAX_LAYERS);  // [layer][point] -> neighbours
  std::vector<size_t> layer_start(MAX_LAYERS + 1, 0);
  for (int lay = 0; lay < nb_layer; ++lay) {
    if (g.get<uint32_t>() != MAGICLAYER) return bail("bad magic at layer beginning");
    const uint64_t np = g.get<uint64_t>();
    layer_start[lay] = origin.size();
    for (uint64_t j = 0; j < np; ++j) {
      if (g.get<uint32_t>() != MAGICPOINT) return bail("bad magic at point beginning");
      const uint64_t oid = g.get<uint64_t>();
      const uint8_t lv = g.get<uint8_t>();
      const int32_t rk = g.get<int32_t>();
      if (!g.ok || lv != lay || rk != (int32_t)j) return bail("point id incoherent with its position in the dump");
      origin.push_back(oid);
      levels.push_back(lv);
      for (int l = 0; l < de.nb_layer; ++l) {
        const uint64_t nn = g.get<uint64_t>();
        if (!g.ok || nn > 100000) return bail("corrupt neighbour count");
        if (l >= MAX_LAYERS) return bail("nb_layer > 16");
        if (lists[l].size() < origin.size()) lists[l].resize(origin.size());
        std::vector<Nb>& dst = lists[l][origin.size() - 1];
        dst.resize(nn);
        for (uint64_t t = 0; t < nn; ++t) {
          (void)g.get<uint64_t>();  // neighbour DataId (the PointId below identifies it)
          dst[t].level = g.get<uint8_t>();
          dst[t].rank = g.get<int32_t>();
          dst[t].dist = g.get<float>();
        }
      }
      if (d.get<uint32_t>() != MAGICDATAP) return bail("bad magic in data file");
      if (d.get<uint64_t>() != oid) return bail("origin_id incoherent between graph and data");
      const uint64_t blen = d.get<uint64_t>();
      if (!d.ok || blen != D * ES) return bail("vector byte length differs from dimension * sizeof(T)");
      const size_t at = vecs.size();
      vecs.resize(at + blen);
      d.bytes(vecs.data() + at, blen);
    }
  }
  layer_start[nb_layer] = origin.size();
  for (int l = nb_layer + 1; l <= MAX_LAYERS; ++l) layer_start[l] = origin.size();
  const uint64_t e_oid = g.get<uint64_t>();
  const uint8_t e_lv = g.get<uint8_t>();
  const int32_t e_rk = g.get<int32_t>();
  (void)e_oid;
  const bool okr = g.ok && d.ok;
  fclose(g.f);
  fclose(d.f);
  if (!okr) return fail("truncated dump");
  if (origin.size() != N) return fail("nb_point of the description differs from the points found");
  auto id_of = [&](uint8_t lv, int32_t rk) -> int64_t {
    if (lv >= MAX_LAYERS || rk < 0) return -1;
    const size_t id = layer_start[lv] + (size_t)rk;
    return id < layer_start[lv + 1] ? (int64_t)id : -1;
  };
  const int64_t entry_id = id_of(e_lv, e_rk);
  if (entry_id < 0) return fail("entry point of the dump not found");
  // ---- CSR per layer, neighbours resolved through their PointId (hnswio.rs:700-735)
  std::vector<std::vector<uint64_t>> off(MAX_LAYERS);
  std::vector<std::vector<uint32_t>> ids(MAX_LAYERS);
  std::vector<std::vector<float>> ds(MAX_LAYERS);
  int nl = 0;
  for (int l = 0; l < MAX_LAYERS; ++l) {
    off[l].assign(N + 1, 0);
    lists[l].resize(N);
    for (size_t p = 0; p < N; ++p) {
      off[l][p] = ids[l].size();
      for (const Nb& nb : lists[l][p]) {
        const int64_t q = id_of(nb.level, nb.rank);
        if (q < 0) return fail("neighbour PointId of the dump not found");
        ids[l].push_back((uint32_t)q);
        ds[l].push_back(nb.dist);
      }
    }
    off[l][N] = ids[l].size();
    if (!ids[l].empty()) nl = l + 1;
  }
  nl = std::max(nl, 1);
  std::vector<const uint64_t*> po(nl);
  std::vector<const uint32_t*> pi(nl);
  std::vector<const float*> pd(nl);
  for (int l = 0; l < nl; ++l) {
    po[l] = off[l].data();
    pi[l] = ids[l].data();
    pd[l] = ds[l].data();
  }
  ef_c = (int)de.ef;
  // the reference re-applies the stored scale as a FACTOR of 1/ln(M) on reload (hnswio.rs:773-777 with
  // hnsw.rs:339-352): levels drawn for points inserted after a reload follow that law, mirrored here
  level_scale = (1.0 / std::log((double)M)) * de.level_scale;
  int r = import_graph(vecs.data(), N, (int)D, origin.data(), levels.data(), entry_id, nl, po.data(), pi.data(), pd.data());
  if (r) return r;
  if (ef_c > 2 * M) extend_candidates = true;  // hnswio.rs:510,599: reloaded indexes extend candidates
  return 0;
}

}  // namespace hb
