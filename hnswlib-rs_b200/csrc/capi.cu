// extern "C" surface of libhnsw_b200.so: the reference's libext.rs symbols (f32) + extensions.
// Declarations and the reference file:line each one replaces are in include/hnsw_b200.h.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <exception>
#include <cstring>
#include <mutex>
#include <numeric>
#include <shared_mutex>
#include <string>
#include <vector>

#include "../../include/hnsw_b200.h"
#include "index.h"
#include "partition.h"

using hb::Index;
using hb::NeighbourOut;
using hb::AnswerArrays;
using hb::Restriction;
using hb::HostBatch;

// every typed handle of libext.rs (HnswApif32, HnswApii32, HnswApiu32, HnswApiu16, HnswApiu8) has this layout
struct HnswApif32 { Index* ix; };
struct HnswApii32 { Index* ix; };
struct HnswApiu32 { Index* ix; };
struct HnswApiu16 { Index* ix; };
struct HnswApiu8 { Index* ix; };
struct AnyApi { Index* ix; };

static thread_local std::string g_err;
static int g_device = 0;

static_assert(sizeof(Neighbour_api) == 16, "Neighbour_api must match #[repr(C)] {usize, f32}");
static_assert(sizeof(NeighbourOut) == sizeof(Neighbour_api), "device answer slot must alias Neighbour_api");
static_assert(sizeof(Neighbourhood_api) == 16 && sizeof(Vec_api_Neighbourhood_api) == 16, "libext.rs struct layouts");

static int set_err(const std::string& m) {
  g_err = m;
  return -1;
}
static int pass(Index* ix, int r) {
  if (r) g_err = ix->err();
  return r;
}
// Refuses the first of v[0, n) that is not below have = nb_point, naming it `what`[i]
static int not_below(const std::string& what, const uint64_t* v, uint64_t n, uint64_t have) {
  for (uint64_t i = 0; i < n; ++i)
    if (v[i] >= have)
      return set_err(what + "[" + std::to_string(i) + "] = " + std::to_string(v[i]) + " is not below nb_point = " +
                     std::to_string(have));
  return 0;
}

// The locks of one call on handle h, held for the guard's scope: the handle's `mu`, then on a partitioned handle every
// partition's in partition order, all shared (searches, read-only queries) or all exclusive (anything that may change
// the index).  Exclusive also waits for the searches submitted on each (drain_pending).  A NULL handle is refused, and
// the guard reads as a null Index*.
enum Mode { SHARED, EXCLUSIVE };
class Locked {
 public:
  Locked(const void* h, Mode mode) : ix_(h ? ((const AnyApi*)h)->ix : nullptr) {
    if (!ix_) {
      set_err("NULL handle");
      return;
    }
    take(ix_, mode);
    for (Index* x : ix_->holders())
      if (x != ix_) take(x, mode);
  }
  operator Index*() const { return ix_; }
  Index* operator->() const { return ix_; }

 private:
  void take(Index* x, Mode mode) {
    if (mode == SHARED) {
      shared_.emplace_back(x->mu);
      return;
    }
    exclusive_.emplace_back(x->mu);
    x->drain_pending();
  }
  Index* ix_;
  std::vector<std::shared_lock<std::shared_mutex>> shared_;
  std::vector<std::unique_lock<std::shared_mutex>> exclusive_;
};

// Partitioned handles (partition.h) and their views.  A view serves read-only calls only; a call the partitioned handle
// cannot serve is refused before it changes anything.
#define HB_NOT_VIEW(ix) \
  if ((ix)->owner) return set_err("a partition view is read-only")
#define HB_NOT_PARTITIONED(ix, what) \
  if ((ix)->partitioned()) return set_err(std::string(what) + " is not available on a partitioned handle")

static int metric_from_name(const uint8_t* name, size_t len) {
  return hb::metric_from_name(std::string((const char*)name, len));
}

static void* make_index(int dtype, size_t max_nb_conn, size_t ef_const, size_t namelen, const uint8_t* cdistname,
                        size_t max_elements, size_t max_layer) {
  if (!cdistname) {
    set_err("distance name is NULL");
    return nullptr;
  }
  const int metric = metric_from_name(cdistname, namelen);
  if (metric < 0 || !hb::metric_supported(metric, dtype)) {  // libext.rs:520-523: unknown distance => null
    set_err("unknown / unsupported distance name '" + std::string((const char*)cdistname, namelen) + "' for this element type");
    return nullptr;
  }
  if (max_nb_conn < 2 || max_nb_conn > 256) {  // hnsw.rs:784-787 caps at 256; ln(1) = 0 breaks the level law
    set_err("max_nb_connection must be in [2, 256]");
    return nullptr;
  }
  if (ef_const == 0 || max_layer == 0) {
    set_err("ef_construction and max_layer must be positive");
    return nullptr;
  }
  Index* ix = new Index((int)max_nb_conn, max_elements, (int)max_layer, (int)ef_const, metric, dtype, g_device);
  if (!ix->ok()) {
    set_err(ix->err());
    delete ix;
    return nullptr;
  }
  return new AnyApi{ix};
}

// ---- generic bodies of the reference entry points (element type = the handle's)
static void insert_any(void* hv, size_t len, const void* data, size_t id) {
  AnyApi* h = (AnyApi*)hv;
  if (!h || !data) {
    set_err("insert: NULL argument");
    return;
  }
  if (h->ix->owner) {
    set_err("insert: a partition view is read-only");
    return;
  }
  Locked ix(h, EXCLUSIVE);
  uint64_t id64 = id;
  pass(ix, ix->insert(data, 1, len, nullptr, &id64, nullptr, (int)len));
}

static void parallel_insert_any(void* hv, size_t nb_vec, size_t vec_len, const void* const* datas, const size_t* ids) {
  AnyApi* h = (AnyApi*)hv;
  if (!h || !datas || !ids) {
    set_err("parallel_insert: NULL argument");
    return;
  }
  if (h->ix->owner) {
    set_err("parallel_insert: a partition view is read-only");
    return;
  }
  Locked ix(h, EXCLUSIVE);
  std::vector<uint64_t> id64(ids, ids + nb_vec);
  pass(ix, ix->insert(nullptr, nb_vec, vec_len, datas, id64.data(), nullptr, (int)vec_len));
}

static const Neighbourhood_api* search_any(const void* hv, size_t len, const void* data, size_t knbn, size_t ef_search) {
  const AnyApi* h = (const AnyApi*)hv;
  if (!h || !data || knbn == 0) {
    set_err("search_neighbours: bad argument");
    return nullptr;
  }
  Locked ix(h, SHARED);
  Neighbour_api* nb = (Neighbour_api*)malloc(sizeof(Neighbour_api) * knbn);
  int32_t cnt = 0;
  const AnswerArrays ans{(NeighbourOut*)nb, nullptr, nullptr, nullptr, nullptr, &cnt};
  if (pass(ix, ix->search_batch(HostBatch{{data}, 1, (int)len, knbn, ef_search, Restriction(), false, ans}))) {
    free(nb);
    return nullptr;
  }
  Neighbourhood_api* out = (Neighbourhood_api*)malloc(sizeof(Neighbourhood_api));
  out->nbgh = cnt;
  out->neighbours = nb;
  return out;
}

struct VecApiBox {
  Vec_api_Neighbourhood_api v;  // first member: the pointer handed to the caller
  Neighbourhood_api* hoods;
  Neighbour_api* block;
};

static const Vec_api_Neighbourhood_api* parallel_search_any(const void* hv, size_t nb_vec, int64_t vec_len,
                                                            const void* const* data, size_t knbn, size_t ef_search) {
  const AnyApi* h = (const AnyApi*)hv;
  if (!h || (!data && nb_vec) || knbn == 0) {
    set_err("parallel_search_neighbours: bad argument");
    return nullptr;
  }
  Locked ix(h, SHARED);
  VecApiBox* box = (VecApiBox*)malloc(sizeof(VecApiBox));
  box->hoods = (Neighbourhood_api*)malloc(sizeof(Neighbourhood_api) * (nb_vec ? nb_vec : 1));
  box->block = (Neighbour_api*)malloc(sizeof(Neighbour_api) * (nb_vec ? nb_vec * knbn : 1));
  std::vector<int32_t> cnt(nb_vec);
  const AnswerArrays out{(NeighbourOut*)box->block, nullptr, nullptr, nullptr, nullptr, cnt.data()};
  // with replicas, every device answers its slice of the batch in place
  if (pass(ix, ix->search_batch(HostBatch{{nullptr, data}, nb_vec, (int)vec_len, knbn, ef_search, Restriction(), false, out}))) {
    free(box->hoods);
    free(box->block);
    free(box);
    return nullptr;
  }
  for (size_t i = 0; i < nb_vec; ++i) {  // input order, hnsw.rs:1622-1633
    box->hoods[i].nbgh = cnt[i];
    box->hoods[i].neighbours = box->block + i * knbn;
  }
  box->v.len = (int64_t)nb_vec;
  box->v.ptr = box->hoods;
  return &box->v;
}

static void drop_any(const void* p) {
  const AnyApi* h = (const AnyApi*)p;
  if (!h) return;
  if (h->ix->owner) {  // a partition view is freed with its partitioned handle
    set_err("drop: a partition view is not a handle of its own");
    return;
  }
  delete h->ix;
  delete h;
}

static int64_t file_dump_any(const void* hv, size_t namelen, const uint8_t* filename);

extern "C" {

// libext.rs generates one set of entry points per element type with macros (generate_insert!, ... :106-275,
// instantiated :770-771, 829-835, 898-904, 1044-1048, 1112-1116); so do we.
#define HB_TYPED_API(SUF, CT, DT)                                                                                      \
  const HnswApi##SUF* init_hnsw_##SUF(size_t max_nb_conn, size_t ef_const, size_t namelen, const uint8_t* cdistname) { \
    return (const HnswApi##SUF*)make_index(DT, max_nb_conn, ef_const, namelen, cdistname, 10000, 16);                   \
  }                                                                                                                    \
  const HnswApi##SUF* init_hnsw_ptrdist_##SUF(size_t, size_t, float (*)(const CT*, const CT*, unsigned long long)) {   \
    set_err("init_hnsw_ptrdist: a host distance callback cannot run inside a CUDA kernel; use a named distance");      \
    return nullptr;                                                                                                    \
  }                                                                                                                    \
  void insert_##SUF(HnswApi##SUF* h, size_t len, const CT* data, size_t id) { insert_any(h, len, data, id); }          \
  void parallel_insert_##SUF(HnswApi##SUF* h, size_t nb_vec, size_t vec_len, const CT** datas, const size_t* ids) {    \
    parallel_insert_any(h, nb_vec, vec_len, (const void* const*)datas, ids);                                           \
  }                                                                                                                    \
  const Neighbourhood_api* search_neighbours_##SUF(const HnswApi##SUF* h, size_t len, const CT* data, size_t knbn,     \
                                                   size_t ef_search) {                                                 \
    return search_any(h, len, data, knbn, ef_search);                                                                  \
  }                                                                                                                    \
  const Vec_api_Neighbourhood_api* parallel_search_neighbours_##SUF(const HnswApi##SUF* h, size_t nb_vec,              \
                                                                    int64_t vec_len, const CT** data, size_t knbn,     \
                                                                    size_t ef_search) {                                \
    return parallel_search_any(h, nb_vec, vec_len, (const void* const*)data, knbn, ef_search);                         \
  }                                                                                                                    \
  int64_t file_dump_##SUF(const HnswApi##SUF* h, size_t namelen, const uint8_t* filename) {                            \
    return file_dump_any(h, namelen, filename);                                                                        \
  }

HB_TYPED_API(f32, float, hb::DT_F32)
HB_TYPED_API(i32, int32_t, hb::DT_I32)
HB_TYPED_API(u32, uint32_t, hb::DT_U32)
HB_TYPED_API(u16, uint16_t, hb::DT_U16)
HB_TYPED_API(u8, uint8_t, hb::DT_U8)
#undef HB_TYPED_API

const HnswApif32* new_hnsw_f32(size_t max_nb_conn, size_t ef_const, size_t namelen, const uint8_t* cdistname,
                               size_t max_elements, size_t max_layer) {
  return (const HnswApif32*)make_index(hb::DT_F32, max_nb_conn, ef_const, namelen, cdistname, max_elements, max_layer);
}
const HnswApiu16* new_hnsw_u16(size_t max_nb_conn, size_t ef_const, size_t namelen, const uint8_t* cdistname,
                               size_t max_elements, size_t max_layer) {  // libext.rs:964-1028
  return (const HnswApiu16*)make_index(hb::DT_U16, max_nb_conn, ef_const, namelen, cdistname, max_elements, max_layer);
}
void drop_hnsw_f32(const HnswApif32* p) { drop_any(p); }  // libext.rs:626-630
void drop_hnsw_u16(const HnswApiu16* p) { drop_any(p); }  // libext.rs:636-640
void hnsw_b200_drop(const void* p) { drop_any(p); }       // upstream exports no drop for i32/u32/u8
// typed constructor with max_elements / max_layer for every element type (upstream has it for f32 and u16 only)
void* hnsw_b200_new(int dtype, size_t max_nb_conn, size_t ef_const, size_t namelen, const uint8_t* cdistname,
                    size_t max_elements, size_t max_layer) {
  if (dtype < 0 || dtype > 4) {
    set_err("dtype must be 0 f32, 1 u8, 2 u16, 3 u32, 4 i32");
    return nullptr;
  }
  return make_index(dtype, max_nb_conn, ef_const, namelen, cdistname, max_elements, max_layer);
}

}  // extern "C"

// generate_file_dump!, libext.rs:257-275: dump into "." with the given basename; 1 on success, -1 on failure
static int64_t file_dump_any(const void* hv, size_t namelen, const uint8_t* filename) {
  const AnyApi* h = (const AnyApi*)hv;
  if (!h || !filename) {
    set_err("file_dump: NULL argument");
    return -1;
  }
  Locked ix(h, SHARED);
  HB_NOT_PARTITIONED(ix, "file_dump (dump each partition_view)");
  std::string used;
  // api.rs:76-78: the reference refuses to overwrite only while a dump is memory-mapped; nothing is mapped here
  if (pass(ix, ix->file_dump(".", std::string((const char*)filename, namelen), true, &used))) return -1;
  return 1;
}

// HnswIo (hnswio.rs:300-380) reduced to what the C ABI needs: directory + basename
struct HnswIo {
  std::string dir, basename;
};

static void* load_any_unguarded(HnswIo* io, int dtype, int metric);
// nothing may unwind through the C boundary: a dump that makes an allocation fail returns NULL like the reference does
static void* load_any(HnswIo* io, int dtype, int metric) {
  try {
    return load_any_unguarded(io, dtype, metric);
  } catch (const std::exception& e) {
    set_err(std::string("load_hnswdump: ") + e.what());
    return nullptr;
  }
}
static void* load_any_unguarded(HnswIo* io, int dtype, int metric) {
  if (!io) {
    set_err("load_hnswdump: NULL HnswIo");
    return nullptr;
  }
  hb::DumpDescription de;
  std::string e;
  if (hb::read_description(io->dir + "/" + io->basename + ".hnsw.graph", de, e)) {
    set_err(e);
    return nullptr;
  }
  const int M = de.max_nb_connection == 0 ? 256 : de.max_nb_connection;
  Index* ix = new Index(M, (size_t)de.nb_point, 16, (int)de.ef, metric, dtype, g_device);
  if (!ix->ok() || ix->load_dump(io->dir, io->basename)) {
    set_err(ix->err());
    delete ix;
    return nullptr;  // libext.rs:297-300: failed reload => null
  }
  return new AnyApi{ix};
}

extern "C" {

// get_hnswio, libext.rs:27-33: dump basename, files looked up in the current directory
HnswIo* get_hnswio(uint64_t flen, const uint8_t* name) {
  if (!name) return nullptr;
  return new HnswIo{".", std::string((const char*)name, (size_t)flen)};
}
HnswIo* hnsw_b200_get_hnswio(const char* dir, const char* basename) {
  if (!dir || !basename) return nullptr;
  return new HnswIo{dir, basename};
}
void hnsw_b200_free_hnswio(HnswIo* io) { delete io; }

// generate_loadhnsw!, libext.rs:280-451: one loader per (element type, distance) pair upstream instantiates
#define HB_LOADER(SUF, DIST, DT, METRIC)                                             \
  const HnswApi##SUF* load_hnswdump_##SUF##_##DIST(HnswIo* io) {                     \
    return (const HnswApi##SUF*)load_any(io, DT, METRIC);                            \
  }
HB_LOADER(f32, DistL1, hb::DT_F32, hb::METRIC_L1)
HB_LOADER(f32, DistL2, hb::DT_F32, hb::METRIC_L2)
HB_LOADER(f32, DistCosine, hb::DT_F32, hb::METRIC_COSINE)
HB_LOADER(f32, DistDot, hb::DT_F32, hb::METRIC_DOT)
HB_LOADER(f32, DistJensenShannon, hb::DT_F32, hb::METRIC_JENSENSHANNON)
HB_LOADER(f32, DistJeffreys, hb::DT_F32, hb::METRIC_JEFFREYS)
HB_LOADER(i32, DistL1, hb::DT_I32, hb::METRIC_L1)
HB_LOADER(i32, DistL2, hb::DT_I32, hb::METRIC_L2)
HB_LOADER(i32, DistHamming, hb::DT_I32, hb::METRIC_HAMMING)
HB_LOADER(u32, DistL1, hb::DT_U32, hb::METRIC_L1)
HB_LOADER(u32, DistL2, hb::DT_U32, hb::METRIC_L2)
HB_LOADER(u32, DistHamming, hb::DT_U32, hb::METRIC_HAMMING)
HB_LOADER(u32, DistJaccard, hb::DT_U32, hb::METRIC_JACCARD)
HB_LOADER(u16, DistL1, hb::DT_U16, hb::METRIC_L1)
HB_LOADER(u16, DistL2, hb::DT_U16, hb::METRIC_L2)
HB_LOADER(u16, DistHamming, hb::DT_U16, hb::METRIC_HAMMING)
HB_LOADER(u8, DistL1, hb::DT_U8, hb::METRIC_L1)
HB_LOADER(u8, DistL2, hb::DT_U8, hb::METRIC_L2)
HB_LOADER(u8, DistHamming, hb::DT_U8, hb::METRIC_HAMMING)
HB_LOADER(u8, DistJaccard, hb::DT_U8, hb::METRIC_JACCARD)
#undef HB_LOADER

// load any (element type, distance) by name: dtype 0 f32, 1 u8, 2 u16, 3 u32, 4 i32
void* hnsw_b200_load_dump(HnswIo* io, int dtype, size_t namelen, const uint8_t* cdistname) {
  if (!cdistname) return nullptr;
  const int metric = metric_from_name(cdistname, namelen);
  if (metric < 0 || !hb::metric_supported(metric, dtype)) {
    set_err("unknown / unsupported distance name for this element type");
    return nullptr;
  }
  return load_any(io, dtype, metric);
}

int hnsw_b200_file_dump(const void* h, const char* dir, const char* basename, int overwrite, char* used_basename,
                        size_t used_cap) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "file_dump (dump each partition_view)");
  if (!dir || !basename) return set_err("NULL path");
  std::string used;
  int r = pass(ix, ix->file_dump(dir, basename, overwrite != 0, &used));
  if (r) return r;
  if (used_basename && used_cap) {
    strncpy(used_basename, used.c_str(), used_cap - 1);
    used_basename[used_cap - 1] = 0;
  }
  return 0;
}

int hnsw_b200_save(const void* h, const char* dir, const char* basename, int overwrite, char* used_basename,
                   size_t used_cap) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  if (!dir || !basename) return set_err("NULL path");
  std::string used;
  if (pass(ix, ix->save(dir, basename, overwrite != 0, &used))) return -1;
  if (used_basename && used_cap) {
    strncpy(used_basename, used.c_str(), used_cap - 1);
    used_basename[used_cap - 1] = 0;
  }
  return 0;
}

void* hnsw_b200_restore(const char* dir, const char* basename, int ndev, const int* devices) {
  if (!dir || !basename) {
    set_err("restore: NULL path");
    return nullptr;
  }
  try {  // nothing may unwind through the C boundary (an allocation sized by the files may fail)
    std::string e;
    Index* ix = Index::restore(dir, basename, ndev, devices, g_device, e);
    if (!ix) {
      set_err(e);
      return nullptr;
    }
    return new AnyApi{ix};
  } catch (const std::exception& ex) {
    set_err(std::string("restore: ") + ex.what());
    return nullptr;
  }
}

// load_hnsw_description, libext.rs:1170-1232.  `name` = path of the .hnsw.graph file.  Release with
// hnsw_b200_free_description (upstream leaks it).
const DescriptionFFI* load_hnsw_description(size_t flen, const uint8_t* name) {
  if (!name) return nullptr;
  hb::DumpDescription de;
  std::string e;
  if (hb::read_description(std::string((const char*)name, flen), de, e)) {
    set_err(e);
    return nullptr;
  }
  DescriptionFFI* d = (DescriptionFFI*)calloc(1, sizeof(DescriptionFFI));
  d->dumpmode = 1;  // upstream hard-codes 1 here ("CAVEAT", libext.rs:1196)
  d->max_nb_connection = de.max_nb_connection;
  d->nb_layer = de.nb_layer;
  d->ef = (size_t)de.ef;
  d->nb_point = (size_t)de.nb_point;  // upstream leaves this field at 0; filled here
  d->data_dimension = (size_t)de.dimension;
  char* dn = (char*)malloc(de.distname.size() + 1);
  memcpy(dn, de.distname.c_str(), de.distname.size() + 1);
  char* tn = (char*)malloc(de.t_name.size() + 1);
  memcpy(tn, de.t_name.c_str(), de.t_name.size() + 1);
  d->distname_len = de.distname.size();
  d->distname = (const uint8_t*)dn;
  d->t_name_len = de.t_name.size();
  d->t_name = (const uint8_t*)tn;
  return d;
}
void hnsw_b200_free_description(const DescriptionFFI* d) {
  if (!d) return;
  free((void*)d->distname);
  free((void*)d->t_name);
  free((void*)d);
}

void init_rust_log(void) {}

// ------------------------------------------------------------------ extensions
const char* hnsw_b200_last_error(void) { return g_err.c_str(); }

int hnsw_b200_last_kernel(char* buf, size_t cap) {
  if (buf && cap) buf[0] = '\0';
  if (!hb::last_launched_kernel) return 0;
  const char* name = nullptr;
  cudaError_t e = cudaFuncGetName(&name, hb::last_launched_kernel);
  if (e != cudaSuccess || !name) return set_err(std::string("cudaFuncGetName: ") + cudaGetErrorString(e));
  const size_t len = strlen(name);
  if (buf && cap) {
    const size_t m = len < cap - 1 ? len : cap - 1;
    memcpy(buf, name, m);
    buf[m] = '\0';
  }
  return (int)len;
}

int hnsw_b200_last_kernel_shape(int64_t* out3) {
  if (!out3) return set_err("NULL output");
  out3[0] = out3[1] = out3[2] = 0;
  if (!hb::last_launched_kernel) return 0;
  int bps = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, hb::last_launched_kernel, hb::last_launched_threads,
                                                                hb::last_launched_smem);
  if (e != cudaSuccess) return set_err(std::string("cudaOccupancyMaxActiveBlocksPerMultiprocessor: ") + cudaGetErrorString(e));
  out3[0] = (int64_t)hb::last_launched_smem;
  out3[1] = hb::last_launched_threads;
  out3[2] = bps;
  return 1;
}

int hnsw_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int hnsw_b200_set_device(int device) {
  int n = hnsw_b200_device_count();
  if (device < 0 || device >= n) return set_err("device index out of range");
  g_device = device;
  return 0;
}

void hnsw_b200_free_neighbourhood(const Neighbourhood_api* p) {
  if (!p) return;
  free((void*)p->neighbours);
  free((void*)p);
}

void hnsw_b200_free_vec_api(const Vec_api_Neighbourhood_api* p) {
  if (!p) return;
  VecApiBox* box = (VecApiBox*)p;
  free(box->hoods);
  free(box->block);
  free(box);
}


int hnsw_b200_set_extend_candidates(void* h, int flag) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (flag && ix->ef_c <= 2 * ix->M)
    return set_err("extend_candidates needs ef_construction > 2*max_nb_connection in this engine (otherwise the "
                   "extension set of hnsw.rs:1336-1362 is not provably empty)");
  ix->settings().extend_candidates = flag != 0;
  return 0;
}
int hnsw_b200_get_extend_candidates(const void* h) {
  if (!h) return set_err("NULL handle");
  return ((const AnyApi*)h)->ix->settings().extend_candidates ? 1 : 0;
}
int hnsw_b200_set_keeping_pruned(void* h, int flag) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  ix->settings().keep_pruned = flag != 0;
  return 0;
}
int hnsw_b200_modify_level_scale(void* h, double scale) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (ix->nb_point() > 0) return set_err("modify_level_scale: index already holds points (hnsw.rs:881-888)");
  if (!(scale >= 0.2 && scale <= 1.0)) return set_err("modify_level_scale: factor must be in [0.2, 1]");  // hnsw.rs:889-900
  ix->settings().level_scale = scale / std::log((double)ix->M);
  return 0;
}
int hnsw_b200_set_tie_mode(void* h, int mode) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (mode != 0 && mode != 1) return set_err("tie mode must be 0 (distance, id) or 1 (reference std heaps)");
  ix->settings().tie_std = mode == 1;
  return 0;
}
int hnsw_b200_set_visited_stages(void* h, int mode) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (mode < 0 || mode > 2) return set_err("visited stages must be 0 (auto), 1 (always) or 2 (never)");
  ix->settings().visited_stages = mode;
  return 0;
}
int hnsw_b200_set_link_mode(void* h, int mode) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (mode != 0 && mode != 1) return set_err("link mode must be 0 (reference: new point's level) or 1 (per layer)");
  ix->settings().link_mode = mode;
  return 0;
}
int hnsw_b200_get_link_mode(const void* h) {
  if (!h) return set_err("NULL handle");
  return ((const AnyApi*)h)->ix->settings().link_mode;
}
int hnsw_b200_set_searching_mode(void* h, int) {  // nothing in this engine depends on the mode
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  return 0;
}
int hnsw_b200_set_level_seed(void* h, uint64_t seed) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  ix->rng.s = seed;  // a partitioned handle draws every level itself, in global insertion order
  return 0;
}
uint64_t hnsw_b200_get_nb_point(const void* h) { return h ? ((const AnyApi*)h)->ix->nb_point() : 0; }
int hnsw_b200_get_max_level_observed(const void* h) { return h ? ((const AnyApi*)h)->ix->max_level() : 0; }
int hnsw_b200_get_dim(const void* h) { return h ? ((const AnyApi*)h)->ix->dim : 0; }
int hnsw_b200_set_insert_batching(void* h, uint32_t ratio, uint32_t max_batch) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (ratio == 0 || max_batch == 0) return set_err("ratio and max_batch must be positive");
  ix->settings().batch_ratio = ratio;
  ix->settings().batch_max = max_batch;
  return 0;
}

int hnsw_b200_partition(void* h, int nparts, const int* devices) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  return pass(ix, hb::Partitions::create(ix, nparts, devices));
}
int hnsw_b200_partition_count(const void* h) {
  if (!h) return set_err("NULL handle");
  const Index* ix = ((const AnyApi*)h)->ix;
  return ix->parts ? ix->parts->count() : 1;
}
const void* hnsw_b200_partition_view(const void* h, int p) {
  if (!h) {
    set_err("NULL handle");
    return nullptr;
  }
  const Index* ix = ((const AnyApi*)h)->ix;
  if (!ix->parts || p < 0 || p >= ix->parts->count()) {
    set_err("partition_view: no such partition");
    return nullptr;
  }
  return ix->parts->view_handle(p);
}

int hnsw_b200_insert_flat(void* h, const void* vecs, uint64_t n, uint64_t dim, const uint64_t* ids,
                          const int32_t* levels) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (n == 0) return 0;
  if (!vecs) return set_err("vecs is NULL");
  return pass(ix, ix->insert(vecs, n, dim, nullptr, ids, levels, (int)dim));
}

// ---- searches.  Every search entry point below is one Request, which search() checks and runs on the handle held
// shared (Locked):
//   * HOST: host rows in, host answers out, through the host batch driver; a partitioned handle searches every partition;
//   * SUBMIT: the same, split in two (hnsw_b200_search_flat_wait collects it), so that one host thread keeps several
//     batches in flight.  With replicas (hnsw_b200_replicate) every device gets its contiguous share enqueued at submit
//     time.  Refused on a partitioned handle;
//   * DEVICE: device rows in, device answers out (b.out.nb, b.out.counts), `sync` and `kernel_ms` as
//     hnsw_b200_search_device takes them (the other two ignore them).  Refused on a partitioned handle.
// By stored point (b.in.qids) the queries are the stored vectors of qids[0, nq), each below nb_point, in the handle's
// dimension.
namespace {
enum Via { HOST, SUBMIT, DEVICE };

static Restriction label_sets(const uint64_t* off, const uint32_t* set, const int64_t* range) {
  return {.kind = Restriction::ROW_LABEL_SETS, .qset_off = off, .qset = set, .qrange = range};
}

// Label sets of one label per query, for the calls that give no offsets: query i's set is {labels[i]}, or {LABEL_NONE}
// (any label) when labels is NULL; the offsets 0, 1, ..., nq, and the nq LABEL_NONE values, are kept here
struct OneLabelSets {
  std::vector<uint64_t> off;
  std::vector<uint32_t> none;
  Restriction rows(uint64_t nq, const uint32_t* labels, const int64_t* qrange) {
    off.resize(nq + 1);
    std::iota(off.begin(), off.end(), (uint64_t)0);
    if (!labels) none.assign(nq, hb::LABEL_NONE);
    return label_sets(off.data(), labels ? labels : none.data(), qrange);
  }
};

// How a call reads its restriction.  FIXED: b.restriction as the entry point made it.  LABELS: a label per query,
// query i's set {qlabels[i]}.  ROWS: a resident filter (`filter`; -1: none) or label sets (qset_off, qset) and ranges
// (qrange) per query, but not both; a range without sets is a range within {LABEL_NONE}.
enum Takes { FIXED, LABELS, ROWS };
// The arguments a call refuses as NULL when nq > 0: b.in.qids, qlabels, qrange, b.excluded (else only one of its two
// arrays NULL is refused), b.in.radius
enum Need { QIDS = 1, QLABELS = 2, QRANGE = 4, QX = 8, RADIUS = 16 };

// One search call as its entry point received it: the entry point's name (as refusals name it), how it runs, its batch
// (with the excluded lists and the radii as passed), and its restriction's arguments as passed.  `early`: nq == 0
// returns 0 before the handle is locked; otherwise a HOST call returns 0 under the lock, and SUBMIT and DEVICE go on.
struct Request {
  const char* name;
  Via via = HOST;
  HostBatch b;
  Takes takes = FIXED;
  int need = 0;
  bool early = false;
  int64_t filter = -1;
  const uint32_t* qlabels = nullptr;
  const int64_t* qrange = nullptr;
  const uint64_t* qset_off = nullptr;
  const uint32_t* qset = nullptr;
  int sync = 1;
  float* kernel_ms = nullptr;
  OneLabelSets one{};          // the offsets of LABELS, and of ranges without sets
  std::vector<float> radii{};  // b.in.radius as run: -0 read as 0, whose key is the smallest
};

// The checks of q that need no lock, in the header's order, and the restriction they leave in q.b.restriction: a NULL
// handle, nq == 0 (early: 1, nothing to run), the NULL arguments, the radii (NaN or negative: refused), and a resident
// filter together with sets or ranges.  -1: refused, 0: go on.
static int prepare(const void* h, Request& q) {
  HostBatch& b = q.b;
  auto refuse = [&](const std::string& what) { return set_err(std::string(q.name) + ": " + what); };
  if (!h) return set_err("NULL handle");
  if (b.nq == 0 && q.early) return 1;
  if (b.nq) {
    if ((q.need & QIDS) && !b.in.qids) return refuse("qids is NULL");
    if ((q.need & QLABELS) && !q.qlabels) return set_err("qlabels is NULL");
    if ((q.need & QRANGE) && !q.qrange) return set_err("qrange is NULL");
    if (((q.need & QX) || b.excluded.ids) && !b.excluded.off) return refuse("qx_off is NULL");
    if (((q.need & QX) || b.excluded.off) && !b.excluded.ids) return refuse("qx is NULL");
    if (q.need & RADIUS) {
      if (!b.in.radius) return refuse("radius is NULL");
      q.radii.resize(b.nq);
      for (uint64_t i = 0; i < b.nq; ++i) {
        const float r = b.in.radius[i];
        if (std::isnan(r) || r < 0)
          return refuse("radius[" + std::to_string(i) + "] = " + std::to_string(r) + " is " + (std::isnan(r) ? "NaN" : "negative"));
        q.radii[i] = r == 0 ? 0.0f : r;
      }
      b.in.radius = q.radii.data();
    }
  }
  if (q.takes == LABELS) b.restriction = q.one.rows(b.nq, q.qlabels, nullptr);
  if (q.takes == ROWS) {
    if (q.filter != -1 && (q.qrange || q.qset_off || q.qset))
      return refuse("a resident filter cannot be combined with label sets or ranges");
    if (q.qset_off || q.qset) b.restriction = label_sets(q.qset_off, q.qset, q.qrange);
    else if (q.qrange) b.restriction = q.one.rows(b.nq, nullptr, q.qrange);
    else if (q.filter != -1) b.restriction = {.kind = Restriction::RESIDENT, .resident = q.filter};
  }
  return 0;
}

// A per-row restriction without its arrays is refused
static int missing_rows(const Restriction& rs) {
  if (rs.kind == Restriction::ROW_FILTERS && !rs.filters) return set_err("filters is NULL");
  if (rs.kind == Restriction::ROW_LABEL_SETS && !rs.qset_off) return set_err("qset_off is NULL");
  if (rs.kind == Restriction::ROW_LABEL_SETS && !rs.qset) return set_err("qset is NULL");
  return 0;
}

// q checked and run: prepare's checks, then under the lock a partitioned handle (SUBMIT, DEVICE), nq == 0 (HOST: 0),
// qids below nb_point, the restriction's and the answers' arrays.  A radius call with knbn == 0 counts only: the scan
// runs at k = 1 into scratch rows, the caller's row arrays may be NULL, and every count is 0.  SUBMIT returns the ticket.
static int64_t search(const void* h, Request q) {
  if (const int s = prepare(h, q)) return s < 0 ? -1 : 0;
  HostBatch& b = q.b;
  Locked ix(h, SHARED);
  if (!ix) return -1;
  if (q.via != HOST) HB_NOT_PARTITIONED(ix, q.name);
  if (q.via == DEVICE) return pass(ix, ix->search_device(b, q.sync != 0, q.kernel_ms));
  if (q.via == HOST && b.nq == 0) return 0;
  if (b.in.qids) {
    if (not_below(std::string(q.name) + ": qids", b.in.qids, b.nq, ix->nb_point())) return -1;
    b.d = ix->dim;
  }
  if (missing_rows(b.restriction)) return -1;
  const bool count_only = b.in.radius && b.k == 0;
  std::vector<uint64_t> scratch_ids(count_only ? b.nq : 0);
  std::vector<float> scratch_dist(count_only ? b.nq : 0);
  if (count_only) {
    b.k = 1;
    b.out.ids = scratch_ids.data();
    b.out.dist = scratch_dist.data();
    b.out.internal = nullptr;
    b.out.pid = nullptr;
  }
  if (!(b.in.queries || b.in.qids) || !b.out.ids || !b.out.dist || !b.out.counts || b.k == 0 || b.nq == 0)
    return set_err("bad argument");
  if (q.via == SUBMIT) {
    const int64_t t = ix->submit_batch(b);
    if (t < 0) g_err = ix->err();
    return t;
  }
  const int rc = pass(ix, ix->search_batch(b));
  if (rc == 0 && count_only) std::fill(b.out.counts, b.out.counts + b.nq, 0);
  return rc;
}
static AnswerArrays columns(uint64_t* ids, float* dist, uint32_t* internal, int32_t* pid, int32_t* counts) {
  return {.ids = ids, .dist = dist, .internal = internal, .pid = pid, .counts = counts};
}
static AnswerArrays on_device(void* d_out, int32_t* d_counts) {
  return {.nb = (NeighbourOut*)d_out, .counts = d_counts};
}
static hb::HostRows by_id(const uint64_t* qids, int exclude_self) {
  return {.qids = qids, .skip = exclude_self ? qids : nullptr};
}
}  // namespace

// hnsw_b200_search_flat and _search_flat_filtered: the filter is the FilterT arguments (filter_mode 1, 2) or one of the
// handle's resident filters.  The kernels and the answers are the same.
int hnsw_b200_search_flat(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                          uint64_t ef_search, int filter_mode, const uint64_t* filter_ids, uint64_t nfilter,
                          hnsw_b200_filter_fn fn, void* ctx, uint64_t* out_ids, float* out_dist,
                          uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  const Restriction filter = filter_mode ? Restriction{.kind = Restriction::FILTER_T, .mode = filter_mode, .ids = filter_ids,
                                                       .nids = nfilter, .fn = fn, .ctx = ctx} : Restriction();
  return (int)search(h, {.name = "search_flat", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn, .ef = ef_search,
                         .restriction = filter, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}
int hnsw_b200_search_flat_filtered(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim,
                                   uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                   uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_filtered", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .restriction = {.kind = Restriction::RESIDENT, .resident = filter},
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}

int64_t hnsw_b200_search_flat_submit(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                                     uint64_t ef_search, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                     int32_t* out_pid, int32_t* out_counts) {
  return search(h, {.name = "search_flat_submit", .via = SUBMIT, .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                    .ef = ef_search, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}
int64_t hnsw_b200_search_flat_submit_filtered(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim,
                                              uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                              uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return search(h, {.name = "search_flat_submit_filtered", .via = SUBMIT, .b = {.in = {queries}, .nq = nq, .d = (int)dim,
                    .k = knbn, .ef = ef_search, .restriction = {.kind = Restriction::RESIDENT, .resident = filter},
                    .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}

int hnsw_b200_search_flat_wait(const void* h, int64_t ticket) {
  if (!h) return set_err("NULL handle");
  Index* ix = ((const AnyApi*)h)->ix;  // no lock: a writer holding the index exclusively is waiting for this very call
  hb::DeviceRestore keep;
  Index::Ticket t;
  if (!ix->take_ticket(ticket, t)) return set_err("bad ticket");
  const int r = pass(ix, ix->finish_batch(t));  // sharded: every replica's leg is collected by that replica's worker
  ix->pending_.fetch_sub(1);
  return r;
}

int hnsw_b200_search_device(const void* h, const void* d_queries, uint64_t nq, uint64_t knbn,
                            uint64_t ef_search, void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  return (int)search(h, {.name = "search_device", .via = DEVICE, .b = {.in = {d_queries}, .nq = nq, .k = knbn,
                         .ef = ef_search, .out = on_device(d_out, d_counts)}, .sync = sync, .kernel_ms = kernel_ms});
}
int hnsw_b200_search_device_filtered(const void* h, int64_t filter, const void* d_queries, uint64_t nq, uint64_t knbn,
                                     uint64_t ef_search, void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  return (int)search(h, {.name = "search_device_filtered", .via = DEVICE, .b = {.in = {d_queries}, .nq = nq, .k = knbn,
                         .ef = ef_search, .restriction = {.kind = Restriction::RESIDENT, .resident = filter},
                         .out = on_device(d_out, d_counts)}, .sync = sync, .kernel_ms = kernel_ms});
}

// Exact search: the exact scan of the points a resident filter admits (filter >= 0) or of every point (-1), through the
// same batch driver and device-resident path as the graph searches
int hnsw_b200_search_exact(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                           uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn, .exact = true,
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}, .takes = ROWS,
                         .filter = filter});
}

// A filter per query: filters[i] is a resident filter of the handle or -1; the graph search (ef_search) or the exact
// scan.  One batch, every entry checked before anything runs.
int hnsw_b200_search_flat_per_query(const void* h, const int64_t* filters, const void* queries, uint64_t nq, uint64_t dim,
                                    uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                    uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_per_query", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .restriction = {.kind = Restriction::ROW_FILTERS, .filters = filters},
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}
int hnsw_b200_search_exact_per_query(const void* h, const int64_t* filters, const void* queries, uint64_t nq, uint64_t dim,
                                     uint64_t knbn, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                     int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_per_query", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .restriction = {.kind = Restriction::ROW_FILTERS, .filters = filters}, .exact = true,
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}

// Point labels (and attributes), addressed by insertion rank; on a partitioned handle each partition holds its share of
// a range by the placement rule (partition.h).
static int label_range(const Index* ix, uint64_t first, uint64_t n, const char* what = "labels") {
  const uint64_t have = ix->nb_point();
  if (first > have || n > have - first)
    return set_err(std::string(what) + " [" + std::to_string(first) + ", " + std::to_string(first + n) + ") are out of range: the " +
                   (ix->owner ? "partition" : "index") + " holds " + std::to_string(have) + " points");
  return 0;
}
// set_labels / set_attributes: column `col` of the points [first, first + n) set to value(0), ..., value(n - 1), under
// the handle's locks taken exclusively; a partition's share is every P-th value.
// get_labels / get_attributes: out[i] = value(x, p) for the point p of Index x that is point first + i, under the
// handle's locks taken shared.
extern "C++" {
namespace {
template <class T, class F>
int set_per_point(void* h, uint64_t first, uint64_t n, const void* values, const char* what, const char* null_msg,
                  hb::PointColumn<T> Index::*col, F value) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  if (label_range(ix, first, n, what)) return -1;
  if (n == 0) return 0;
  if (!values) return set_err(null_msg);
  hb::DeviceRestore keep;
  const std::vector<Index*>& hs = ix->holders();
  return hb::for_each_share(first, n, hs.size(), [&](int p, uint64_t lo, uint64_t cnt, uint64_t at, uint64_t step) {
    const int r = hs[p]->set_points(hs[p]->*col, lo, cnt, [&](size_t i) { return value(at + i * step); });
    return pass(ix, r ? ix->holder_fail(p, r) : 0);
  });
}
template <class T, class F>
int get_per_point(const void* h, uint64_t first, uint64_t n, T* out, const char* what, F value) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  if (label_range(ix, first, n, what)) return -1;
  if (n == 0) return 0;
  if (!out) return set_err("out is NULL");
  const std::vector<Index*>& hs = ix->holders();
  return hb::for_each_share(first, n, hs.size(), [&](int p, uint64_t lo, uint64_t cnt, uint64_t at, uint64_t step) {
    for (uint64_t i = 0; i < cnt; ++i) out[at + i * step] = value(hs[p], lo + i);
    return 0;
  });
}
}  // namespace
}  // extern "C++"
int hnsw_b200_set_labels(void* h, uint64_t first, uint64_t n, const uint32_t* labels) {
  return set_per_point(h, first, n, labels, "labels", "labels is NULL", &Index::labels,
                       [&](size_t i) { return labels[i]; });
}
int hnsw_b200_get_labels(const void* h, uint64_t first, uint64_t n, uint32_t* out) {
  return get_per_point(h, first, n, out, "labels", [](const Index* x, size_t p) { return x->labels.host[p]; });
}

// Point attributes: addressed as labels are, stored biased
int hnsw_b200_set_attributes(void* h, uint64_t first, uint64_t n, const int64_t* values) {
  return set_per_point(h, first, n, values, "attributes", "values is NULL", &Index::attrs,
                       [&](size_t i) { return hb::attr_bias(values[i]); });
}
int hnsw_b200_get_attributes(const void* h, uint64_t first, uint64_t n, int64_t* out) {
  return get_per_point(h, first, n, out, "attributes",
                       [](const Index* x, size_t p) { return hb::attr_unbias(x->attrs.host[p]); });
}

// Deleted points: the ranks split by placement, each partition's share marked on it, under the handle's locks taken
// exclusively; every rank is checked before anything changes.  get_deleted reads as get_labels does.
static int mark_deleted(void* h, const uint64_t* ranks, uint64_t n, bool on) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  if (n && !ranks) return set_err("ranks is NULL");
  if (not_below("ranks", ranks, n, ix->nb_point())) return -1;
  HB_NOT_VIEW(ix);
  if (n == 0) return 0;
  hb::DeviceRestore keep;
  const std::vector<Index*>& hs = ix->holders();
  const uint64_t P = hs.size();
  std::vector<std::vector<uint64_t>> local(P);
  for (uint64_t i = 0; i < n; ++i) {
    const hb::Placed at = hb::place(ranks[i], P);
    local[at.part].push_back(at.local);
  }
  for (uint64_t p = 0; p < P; ++p)
    if (const int r = hs[p]->mark_deleted(local[p].data(), local[p].size(), on)) return pass(ix, ix->holder_fail((int)p, r));
  return 0;
}
int hnsw_b200_delete_points(void* h, const uint64_t* ranks, uint64_t n) { return mark_deleted(h, ranks, n, true); }
int hnsw_b200_restore_points(void* h, const uint64_t* ranks, uint64_t n) { return mark_deleted(h, ranks, n, false); }
int hnsw_b200_get_deleted(const void* h, uint64_t first, uint64_t n, uint8_t* out) {
  return get_per_point(h, first, n, out, "deleted points", [](const Index* x, size_t p) {
    const std::vector<uint32_t>& w = x->deleted.host;
    return (uint8_t)(p / 32 < w.size() ? (w[p / 32] >> (p % 32)) & 1u : 0u);
  });
}
int64_t hnsw_b200_get_nb_deleted(const void* h) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  int64_t total = 0;
  for (const Index* x : ix->holders()) total += (int64_t)x->deleted.count;
  return total;
}

// A label per query: labels[i] is the label query i is restricted to, or LABEL_NONE for none; the graph search
// (ef_search) or the exact scan.  Query i's label set is {qlabels[i]}.
int hnsw_b200_search_flat_labeled(const void* h, const uint32_t* qlabels, const void* queries, uint64_t nq, uint64_t dim,
                                  uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                  uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_labeled", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = LABELS, .need = QLABELS, .qlabels = qlabels});
}
int hnsw_b200_search_exact_labeled(const void* h, const uint32_t* qlabels, const void* queries, uint64_t nq, uint64_t dim,
                                   uint64_t knbn, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                   int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_labeled", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .exact = true, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = LABELS, .need = QLABELS, .qlabels = qlabels});
}

// A label set per query: query i is restricted to the points whose label is one of qset[qset_off[i], qset_off[i + 1])
// ({LABEL_NONE}: every point); the graph search (ef_search) or the exact scan.
int hnsw_b200_search_flat_label_sets(const void* h, const uint64_t* qset_off, const uint32_t* qset, const void* queries,
                                     uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t ef_search, uint64_t* out_ids,
                                     float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_label_sets", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .restriction = label_sets(qset_off, qset, nullptr),
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}
int hnsw_b200_search_exact_label_sets(const void* h, const uint64_t* qset_off, const uint32_t* qset, const void* queries,
                                      uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t* out_ids, float* out_dist,
                                      uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_label_sets", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .restriction = label_sets(qset_off, qset, nullptr), .exact = true,
                         .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)}});
}

// Attribute ranges.  Query i is restricted to the points whose attribute is in [qrange[2i], qrange[2i + 1]]
// ([INT64_MIN, INT64_MAX]: every point, also those without one) and whose label is one of qset[qset_off[i],
// qset_off[i + 1]) ({LABEL_NONE}: any; qset_off and qset both NULL: {LABEL_NONE} for every query); the graph search
// (ef_search) or the exact scan.
int hnsw_b200_search_flat_ranges(const void* h, const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset,
                                 const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t ef_search,
                                 uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                                 int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_ranges", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = ROWS, .need = QRANGE, .qrange = qrange, .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_exact_ranges(const void* h, const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset,
                                  const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t* out_ids,
                                  float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_ranges", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .exact = true, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = ROWS, .need = QRANGE, .qrange = qrange, .qset_off = qset_off, .qset = qset});
}

int hnsw_b200_search_exact_device(const void* h, int64_t filter, const void* d_queries, uint64_t nq, uint64_t knbn,
                                  void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  return (int)search(h, {.name = "search_exact_device", .via = DEVICE, .b = {.in = {d_queries}, .nq = nq, .k = knbn,
                         .exact = true, .out = on_device(d_out, d_counts)}, .takes = ROWS, .filter = filter,
                         .sync = sync, .kernel_ms = kernel_ms});
}

// Search by stored point (b.in.qids, and b.in.skip for exclude_self), under a ROWS restriction
int hnsw_b200_search_flat_by_id(const void* h, const uint64_t* qids, uint64_t nq, uint64_t knbn, uint64_t ef_search,
                                int exclude_self, int64_t filter, const int64_t* qrange, const uint64_t* qset_off,
                                const uint32_t* qset, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_by_id", .b = {.in = by_id(qids, exclude_self), .nq = nq, .k = knbn,
                         .ef = ef_search, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = ROWS, .need = QIDS, .early = true, .filter = filter, .qrange = qrange,
                         .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_exact_by_id(const void* h, const uint64_t* qids, uint64_t nq, uint64_t knbn, int exclude_self,
                                 int64_t filter, const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset,
                                 uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                                 int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_by_id", .b = {.in = by_id(qids, exclude_self), .nq = nq, .k = knbn,
                         .exact = true, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts)},
                         .takes = ROWS, .need = QIDS, .early = true, .filter = filter, .qrange = qrange,
                         .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_device_by_id(const void* h, int exact, int64_t filter, const uint64_t* d_qids, uint64_t nq,
                                  uint64_t knbn, uint64_t ef_search, int exclude_self, void* d_out, int32_t* d_counts,
                                  int sync, float* kernel_ms) {
  return (int)search(h, {.name = "search_device_by_id", .via = DEVICE, .b = {.in = by_id(d_qids, exclude_self), .nq = nq,
                         .k = knbn, .ef = exact ? 0 : ef_search, .exact = exact != 0, .out = on_device(d_out, d_counts)},
                         .takes = ROWS, .need = QIDS, .early = true, .filter = filter, .sync = sync,
                         .kernel_ms = kernel_ms});
}

// Excluded points per query: host queries under a ROWS restriction, row i without the points of qx[qx_off[i],
// qx_off[i + 1]) (insertion ranks; their check against nb_point runs under the handle's lock, Index::exclusion_lists)
int hnsw_b200_search_flat_excluding(const void* h, const uint64_t* qx_off, const uint64_t* qx, int64_t filter,
                                    const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset,
                                    const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t ef_search,
                                    uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                                    int32_t* out_counts) {
  return (int)search(h, {.name = "search_flat_excluding", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts),
                         .excluded = {qx_off, qx}}, .takes = ROWS, .need = QX, .early = true, .filter = filter,
                         .qrange = qrange, .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_exact_excluding(const void* h, const uint64_t* qx_off, const uint64_t* qx, int64_t filter,
                                     const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset,
                                     const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t* out_ids,
                                     float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return (int)search(h, {.name = "search_exact_excluding", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .exact = true, .out = columns(out_ids, out_dist, out_internal, out_pid, out_counts),
                         .excluded = {qx_off, qx}}, .takes = ROWS, .need = QX, .early = true, .filter = filter,
                         .qrange = qrange, .qset_off = qset_off, .qset = qset});
}

// Planned search: count_admitted reads its restriction as the by-id calls do; the planned calls run each row on the graph
// or by the exact scan per leg (Index::split_legs), under a ROWS restriction and, with qx_off and qx, each row's
// excluded points; out_exact (may be NULL) is written once the batch succeeded
int hnsw_b200_count_admitted(const void* h, int64_t filter, const int64_t* qrange, const uint64_t* qset_off,
                             const uint32_t* qset, uint64_t nq, uint64_t* out_count) {
  Request q{.name = "count_admitted", .b = {.nq = nq}, .takes = ROWS, .early = true, .filter = filter, .qrange = qrange,
            .qset_off = qset_off, .qset = qset};
  if (const int s = prepare(h, q)) return s < 0 ? -1 : 0;
  if (missing_rows(q.b.restriction)) return -1;
  if (!out_count) return set_err("count_admitted: out_count is NULL");
  Locked ix(h, SHARED);
  if (!ix) return -1;
  return pass(ix, ix->count_admitted(q.b.restriction, nq, out_count));
}
int hnsw_b200_search_planned(const void* h, const uint64_t* qx_off, const uint64_t* qx, int64_t filter,
                             const int64_t* qrange, const uint64_t* qset_off, const uint32_t* qset, const void* queries,
                             uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t ef_search, uint64_t* out_ids,
                             float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts,
                             int32_t* out_exact) {
  return (int)search(h, {.name = "search_planned", .b = {.in = {queries}, .nq = nq, .d = (int)dim, .k = knbn,
                         .ef = ef_search, .out = {.ids = out_ids, .dist = out_dist, .internal = out_internal,
                         .pid = out_pid, .counts = out_counts, .exact = out_exact}, .excluded = {qx_off, qx},
                         .planned = true}, .takes = ROWS, .early = true, .filter = filter, .qrange = qrange,
                         .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_planned_by_id(const void* h, const uint64_t* qids, uint64_t nq, uint64_t knbn, uint64_t ef_search,
                                   int exclude_self, int64_t filter, const int64_t* qrange, const uint64_t* qset_off,
                                   const uint32_t* qset, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                   int32_t* out_pid, int32_t* out_counts, int32_t* out_exact) {
  return (int)search(h, {.name = "search_planned_by_id", .b = {.in = by_id(qids, exclude_self), .nq = nq, .k = knbn,
                         .ef = ef_search, .out = {.ids = out_ids, .dist = out_dist, .internal = out_internal,
                         .pid = out_pid, .counts = out_counts, .exact = out_exact}, .planned = true}, .takes = ROWS,
                         .need = QIDS, .early = true, .filter = filter, .qrange = qrange, .qset_off = qset_off,
                         .qset = qset});
}

// Radius search: the exact scan of host queries or of stored points, under a ROWS restriction, each row cut at its
// radius and its total of points within it into out_total (may be NULL); knbn == 0 counts only (search)
int hnsw_b200_search_exact_radius(const void* h, int64_t filter, const int64_t* qrange, const uint64_t* qset_off,
                                  const uint32_t* qset, const void* queries, uint64_t nq, uint64_t dim,
                                  const float* radius, uint64_t knbn, uint64_t* out_ids, float* out_dist,
                                  uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts, uint64_t* out_total) {
  return (int)search(h, {.name = "search_exact_radius", .b = {.in = {.queries = queries, .radius = radius}, .nq = nq,
                         .d = (int)dim, .k = knbn, .exact = true, .out = {.ids = out_ids, .dist = out_dist,
                         .internal = out_internal, .pid = out_pid, .counts = out_counts, .total = out_total}},
                         .takes = ROWS, .need = RADIUS, .early = true, .filter = filter, .qrange = qrange,
                         .qset_off = qset_off, .qset = qset});
}
int hnsw_b200_search_exact_radius_by_id(const void* h, const uint64_t* qids, uint64_t nq, const float* radius,
                                        uint64_t knbn, int exclude_self, int64_t filter, const int64_t* qrange,
                                        const uint64_t* qset_off, const uint32_t* qset, uint64_t* out_ids,
                                        float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                                        int32_t* out_counts, uint64_t* out_total) {
  return (int)search(h, {.name = "search_exact_radius_by_id", .b = {.in = {.qids = qids, .skip = exclude_self ? qids :
                         nullptr, .radius = radius}, .nq = nq, .k = knbn, .exact = true, .out = {.ids = out_ids,
                         .dist = out_dist, .internal = out_internal, .pid = out_pid, .counts = out_counts,
                         .total = out_total}}, .takes = ROWS, .need = QIDS | RADIUS, .early = true, .filter = filter,
                         .qrange = qrange, .qset_off = qset_off, .qset = qset});
}

int hnsw_b200_get_vectors(const void* h, const uint64_t* ranks, uint64_t n, void* out) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  if (n == 0) return 0;
  if (!ranks) return set_err("get_vectors: ranks is NULL");
  if (!out) return set_err("get_vectors: out is NULL");
  if (not_below("get_vectors: ranks", ranks, n, ix->nb_point())) return -1;
  hb::DeviceRestore keep;
  return pass(ix, ix->get_vectors(ranks, n, out));
}

int64_t hnsw_b200_filter_new(const void* h, int filter_mode, const uint64_t* filter_ids, uint64_t nfilter,
                             hnsw_b200_filter_fn fn, void* ctx) {
  Locked ix(h, SHARED);  // shared: the points cannot change while the bitmap is made
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  const int64_t id = ix->new_filter(filter_mode, filter_ids, nfilter, fn, ctx);
  if (id < 0) g_err = ix->err();
  return id;
}
int hnsw_b200_filter_free(const void* h, int64_t filter) {
  Locked ix(h, EXCLUSIVE);  // exclusive: waits for every search under the shared lock and every outstanding ticket
  if (!ix) return -1;
  return pass(ix, ix->free_filter(filter));
}

int hnsw_b200_join(void* h) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  return pass(ix, ix->join());
}
int hnsw_b200_stream_wait_last(void* h, void* cuda_stream) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  return pass(ix, ix->stream_wait_last((cudaStream_t)cuda_stream));
}
int hnsw_b200_set_stream(void* h, void* cuda_stream) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  return pass(ix, ix->set_stream((cudaStream_t)cuda_stream));
}
int hnsw_b200_check_status(void* h) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  int r = ix->check_status();
  if (r < 0) g_err = ix->err();
  return r;
}

int hnsw_b200_enable_stats(void* h, int enable) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  ix->settings().stats = enable != 0;
  return 0;
}
int hnsw_b200_get_stats(const void* h, uint64_t* out4, int reset) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  return pass(ix, ix->get_stats(out4, reset != 0));
}

int hnsw_b200_export_points(const void* h, uint8_t* levels, int32_t* ranks, uint64_t* origin, int64_t* entry) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "export_points (export each partition_view)");
  for (size_t i = 0; i < ix->n; ++i) {
    if (levels) levels[i] = ix->h_level[i];
    if (ranks) ranks[i] = ix->h_rank[i];
    if (origin) origin[i] = ix->h_origin[i];
  }
  if (entry) *entry = ix->entry == hb::INVALID_ID ? -1 : (int64_t)ix->entry;
  return 0;
}
int hnsw_b200_export_vectors(const void* h, void* out) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "export_vectors (export each partition_view)");
  return pass(ix, ix->export_vectors(out));
}
// FlatNeighborhood::from(&hnsw) + get_neighbours(DataId) (flatten.rs:93-126): neighbours of `origin_id` over all
// layers, ascending distance.  Returns the number written (<= cap), -1 when the id is unknown.
int64_t hnsw_b200_flat_neighbours(const void* h, uint64_t origin_id, Neighbour_api* out, uint64_t cap) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "flatten (flatten each partition_view)");
  std::vector<uint64_t> off, nbo;
  std::vector<float> nbd;
  if (pass(ix, ix->flatten(off, nbo, nbd))) return -1;
  for (size_t p = 0; p < ix->n; ++p)
    if (ix->h_origin[p] == origin_id) {
      uint64_t c = 0;
      for (uint64_t j = off[p]; j < off[p + 1] && c < cap; ++j, ++c) out[c] = Neighbour_api{(size_t)nbo[j], nbd[j]};
      return (int64_t)c;
    }
  set_err("unknown origin id");
  return -1;
}
// whole flattened graph: offsets[nb_point+1] (internal-id order), neighbour origin ids and distances; pass NULL
// arrays to get the total neighbour count only
int64_t hnsw_b200_flatten(const void* h, uint64_t* offsets, uint64_t* nb_origin, float* nb_dist) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "flatten (flatten each partition_view)");
  std::vector<uint64_t> off, nbo;
  std::vector<float> nbd;
  if (pass(ix, ix->flatten(off, nbo, nbd))) return -1;
  if (offsets) memcpy(offsets, off.data(), off.size() * 8);
  if (nb_origin) memcpy(nb_origin, nbo.data(), nbo.size() * 8);
  if (nb_dist) memcpy(nb_dist, nbd.data(), nbd.size() * 4);
  return (int64_t)nbo.size();
}

int64_t hnsw_b200_layer_edges(const void* h, int layer) {
  Locked ix(h, SHARED);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "layer_edges (export each partition_view)");
  int64_t total = 0;
  if (pass(ix, ix->export_layer(layer, nullptr, nullptr, nullptr, &total))) return -1;
  return total;
}
int hnsw_b200_export_layer(const void* h, int layer, uint64_t* offsets, uint32_t* ids, float* dists) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "export_layer (export each partition_view)");
  return pass(ix, ix->export_layer(layer, offsets, ids, dists, nullptr));
}
int hnsw_b200_import_graph(void* h, const void* vecs, uint64_t n, uint64_t dim, const uint64_t* origin,
                           const uint8_t* levels, int64_t entry, int nlayers, const uint64_t* const* offsets,
                           const uint32_t* const* ids, const float* const* dists) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "import_graph");
  return pass(ix, ix->import_graph(vecs, n, (int)dim, origin, levels, entry, nlayers, offsets, ids, dists));
}

int hnsw_b200_blob_header(const void* h, uint64_t* header16) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "blob_header");
  return ix->blob_header(header16);
}
int hnsw_b200_blob_alloc(void* h, const uint64_t* header16) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "blob_alloc");
  return pass(ix, ix->blob_alloc(header16));
}
int hnsw_b200_blob_count(const void* h) {
  if (!h) return 0;
  HB_NOT_PARTITIONED(((const AnyApi*)h)->ix, "blob_count");
  return ((const AnyApi*)h)->ix->blob_count();
}
int hnsw_b200_blob_info(const void* h, int i, void** dev_ptr, uint64_t* nbytes) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "blob_info");
  return pass(ix, ix->blob_info(i, dev_ptr, nbytes));
}
int hnsw_b200_blob_commit(void* h) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "blob_commit");
  return pass(ix, ix->blob_commit());
}

// ---- multi-GPU (multi.cu)
int hnsw_b200_replicate(void* h, int ndev, const int* devices) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "replicate");
  return pass(ix, ix->replicate(ndev, devices));
}
int hnsw_b200_replica_count(const void* h) { return h ? (int)((const AnyApi*)h)->ix->replica_count() : 0; }
int hnsw_b200_nccl_unique_id(uint8_t* id128) {
  if (!id128) return set_err("NULL argument");
  return Index::nccl_unique_id(id128) ? set_err("NCCL is not available (libnccl.so.2)") : 0;
}
int hnsw_b200_nccl_init(void* h, int nranks, int rank, const uint8_t* id128) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "nccl_init");
  if (!id128) return set_err("NULL argument");
  return pass(ix, ix->nccl_init(nranks, rank, id128));
}
int hnsw_b200_nccl_broadcast_index(void* h, int root) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "nccl_broadcast_index");
  return pass(ix, ix->nccl_broadcast_index(root));
}
int hnsw_b200_nccl_allgather(void* h, const void* d_send, void* d_recv, uint64_t bytes_per_rank, void* cuda_stream) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "nccl_allgather");
  return pass(ix, ix->nccl_allgather(d_send, d_recv, bytes_per_rank, (cudaStream_t)cuda_stream));
}

int hnsw_b200_dist_batch(const void* h, const void* queries, uint64_t nq, uint64_t dim, const uint32_t* cand,
                         uint64_t m, float* out) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  HB_NOT_PARTITIONED(ix, "dist_batch");
  return pass(ix, ix->dist_batch(queries, nq, (int)dim, cand, m, out));
}
int hnsw_b200_bruteforce(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t k,
                         uint32_t* out_ids, float* out_dist) {
  Locked ix(h, EXCLUSIVE);
  if (!ix) return -1;
  // a partitioned handle's ids are global insertion ranks (the partitions' answers merged like a search's)
  return pass(ix, ix->bruteforce(queries, nq, (int)dim, k, out_ids, out_dist));
}

}  // extern "C"
