// extern "C" surface of libhnsw_b200.so: the reference's libext.rs symbols (f32) + extensions.
// Declarations and the reference file:line each one replaces are in include/hnsw_b200.h.
#include <cstdlib>
#include <exception>
#include <cstring>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <vector>

#include "../../include/hnsw_b200.h"
#include "index.h"
#include "partition.h"

using hb::Index;
using hb::NeighbourOut;
using hb::AnswerArrays;
using hb::FilterArg;
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

// HB_H: exclusive access (anything that may change the index); HB_HS: shared access (searches, read-only queries)
#define HB_H(h) \
  if (!(h)) return set_err("NULL handle"); \
  Index* ix = ((const AnyApi*)(h))->ix;    \
  std::unique_lock<std::shared_mutex> g__(ix->mu); \
  ix->drain_pending()
#define HB_HS(h) \
  if (!(h)) return set_err("NULL handle"); \
  Index* ix = ((const AnyApi*)(h))->ix;    \
  std::shared_lock<std::shared_mutex> g__(ix->mu)

// Partitioned handles (partition.h) and their views.  A view serves read-only calls only; a call the partitioned handle
// cannot serve is refused before it changes anything.  A partitioned call holds the handle's lock, then every
// partition's in partition order (HB_PARTS_SHARED for searches, HB_PARTS_EXCLUSIVE for inserts and settings).
#define HB_NOT_VIEW(ix) \
  if ((ix)->owner) return set_err("a partition view is read-only")
#define HB_NOT_PARTITIONED(ix, what) \
  if ((ix)->parts) return set_err(std::string(what) + " is not available on a partitioned handle")
#define HB_PARTS_SHARED(ix) const auto pl__ = (ix)->parts->lock_shared()
#define HB_PARTS_SHARED_IF(ix) \
  const auto pl__ = (ix)->parts ? (ix)->parts->lock_shared() : std::vector<std::shared_lock<std::shared_mutex>>()
#define HB_PARTS_EXCLUSIVE(ix) const auto pl__ = (ix)->parts->lock_exclusive()

// a setting: on a partitioned handle it is applied to the handle and to every partition
static void apply(Index* ix, const std::function<void(Index*)>& set) {
  set(ix);
  if (!ix->parts) return;
  HB_PARTS_EXCLUSIVE(ix);
  for (int p = 0; p < ix->parts->count(); ++p) set(ix->parts->part(p));
}
static uint64_t nb_point(const Index* ix) { return ix->parts ? ix->parts->nb_point() : ix->n; }

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
  std::unique_lock<std::shared_mutex> g(h->ix->mu);
  h->ix->drain_pending();
  uint64_t id64 = id;
  if (h->ix->parts) {
    HB_PARTS_EXCLUSIVE(h->ix);
    pass(h->ix, h->ix->parts->insert(data, 1, len, nullptr, &id64, nullptr, (int)len));
    return;
  }
  if (pass(h->ix, h->ix->set_dim((int)len))) return;
  pass(h->ix, h->ix->insert_batch(data, 1, len, nullptr, &id64, nullptr));
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
  std::unique_lock<std::shared_mutex> g(h->ix->mu);
  h->ix->drain_pending();
  std::vector<uint64_t> id64(ids, ids + nb_vec);
  if (h->ix->parts) {
    HB_PARTS_EXCLUSIVE(h->ix);
    pass(h->ix, h->ix->parts->insert(nullptr, nb_vec, vec_len, datas, id64.data(), nullptr, (int)vec_len));
    return;
  }
  if (pass(h->ix, h->ix->set_dim((int)vec_len))) return;
  pass(h->ix, h->ix->insert_batch(nullptr, nb_vec, vec_len, datas, id64.data(), nullptr));
}

static const Neighbourhood_api* search_any(const void* hv, size_t len, const void* data, size_t knbn, size_t ef_search) {
  const AnyApi* h = (const AnyApi*)hv;
  if (!h || !data || knbn == 0) {
    set_err("search_neighbours: bad argument");
    return nullptr;
  }
  std::shared_lock<std::shared_mutex> g(h->ix->mu);
  HB_PARTS_SHARED_IF(h->ix);
  Neighbour_api* nb = (Neighbour_api*)malloc(sizeof(Neighbour_api) * knbn);
  int32_t cnt = 0;
  const AnswerArrays ans{(NeighbourOut*)nb, nullptr, nullptr, nullptr, nullptr, &cnt};
  if (pass(h->ix, h->ix->search_batch(HostBatch{data, nullptr, 1, (int)len, knbn, ef_search, FilterArg(), ans}))) {
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
  std::shared_lock<std::shared_mutex> g(h->ix->mu);
  HB_PARTS_SHARED_IF(h->ix);
  VecApiBox* box = (VecApiBox*)malloc(sizeof(VecApiBox));
  box->hoods = (Neighbourhood_api*)malloc(sizeof(Neighbourhood_api) * (nb_vec ? nb_vec : 1));
  box->block = (Neighbour_api*)malloc(sizeof(Neighbour_api) * (nb_vec ? nb_vec * knbn : 1));
  std::vector<int32_t> cnt(nb_vec);
  const AnswerArrays out{(NeighbourOut*)box->block, nullptr, nullptr, nullptr, nullptr, cnt.data()};
  // with replicas, every device answers its slice of the batch in place
  if (pass(h->ix, h->ix->search_batch(HostBatch{nullptr, data, nb_vec, (int)vec_len, knbn, ef_search, FilterArg(), out}))) {
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
  HB_NOT_PARTITIONED(h->ix, "file_dump (dump each partition_view)");
  std::shared_lock<std::shared_mutex> g(h->ix->mu);
  std::string used;
  // api.rs:76-78: the reference refuses to overwrite only while a dump is memory-mapped; nothing is mapped here
  if (pass(h->ix, h->ix->file_dump(".", std::string((const char*)filename, namelen), true, &used))) return -1;
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
  HB_H(h);
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
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (flag && ix->ef_c <= 2 * ix->M)
    return set_err("extend_candidates needs ef_construction > 2*max_nb_connection in this engine (otherwise the "
                   "extension set of hnsw.rs:1336-1362 is not provably empty)");
  apply(ix, [=](Index* x) { x->extend_candidates = flag != 0; });
  return 0;
}
int hnsw_b200_get_extend_candidates(const void* h) {
  if (!h) return set_err("NULL handle");
  return ((const AnyApi*)h)->ix->extend_candidates ? 1 : 0;
}
int hnsw_b200_set_keeping_pruned(void* h, int flag) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  apply(ix, [=](Index* x) { x->keep_pruned = flag != 0; });
  return 0;
}
int hnsw_b200_modify_level_scale(void* h, double scale) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (nb_point(ix) > 0) return set_err("modify_level_scale: index already holds points (hnsw.rs:881-888)");
  if (!(scale >= 0.2 && scale <= 1.0)) return set_err("modify_level_scale: factor must be in [0.2, 1]");  // hnsw.rs:889-900
  apply(ix, [=](Index* x) { x->level_scale = scale / std::log((double)x->M); });
  return 0;
}
int hnsw_b200_set_tie_mode(void* h, int mode) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (mode != 0 && mode != 1) return set_err("tie mode must be 0 (distance, id) or 1 (reference std heaps)");
  apply(ix, [=](Index* x) { x->tie_std_ = mode == 1; });
  return 0;
}
int hnsw_b200_set_link_mode(void* h, int mode) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (mode != 0 && mode != 1) return set_err("link mode must be 0 (reference: new point's level) or 1 (per layer)");
  apply(ix, [=](Index* x) { x->link_mode = mode; });
  return 0;
}
int hnsw_b200_get_link_mode(const void* h) {
  if (!h) return set_err("NULL handle");
  return ((const AnyApi*)h)->ix->link_mode;
}
int hnsw_b200_set_searching_mode(void* h, int flag) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  apply(ix, [=](Index* x) { x->searching = flag != 0; });
  return 0;
}
int hnsw_b200_set_level_seed(void* h, uint64_t seed) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  ix->rng.s = seed;  // a partitioned handle draws every level itself, in global insertion order
  return 0;
}
uint64_t hnsw_b200_get_nb_point(const void* h) { return h ? nb_point(((const AnyApi*)h)->ix) : 0; }
int hnsw_b200_get_max_level_observed(const void* h) {
  if (!h) return 0;
  const Index* ix = ((const AnyApi*)h)->ix;
  return ix->parts ? ix->parts->max_level() : std::max(ix->entry_level, 0);
}
int hnsw_b200_get_dim(const void* h) { return h ? ((const AnyApi*)h)->ix->dim : 0; }
int hnsw_b200_set_insert_batching(void* h, uint32_t ratio, uint32_t max_batch) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (ratio == 0 || max_batch == 0) return set_err("ratio and max_batch must be positive");
  apply(ix, [=](Index* x) {
    x->batch_ratio = ratio;
    x->batch_max = max_batch;
  });
  return 0;
}

int hnsw_b200_partition(void* h, int nparts, const int* devices) {
  HB_H(h);
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
  HB_H(h);
  HB_NOT_VIEW(ix);
  if (n == 0) return 0;
  if (!vecs) return set_err("vecs is NULL");
  if (ix->parts) {
    HB_PARTS_EXCLUSIVE(ix);
    return pass(ix, ix->parts->insert(vecs, n, dim, nullptr, ids, levels, (int)dim));
  }
  int r;
  if ((r = pass(ix, ix->set_dim((int)dim)))) return r;
  return pass(ix, ix->insert_batch(vecs, n, dim, nullptr, ids, levels));
}

// hnsw_b200_search_flat and _search_flat_filtered: the filter is the FilterT arguments (filter_mode 1, 2) or, when
// `resident` is set, one of the handle's resident filters (filter_mode 0).  The kernels and the answers are the same.
static int search_flat_any(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn, uint64_t ef_search,
                           int filter_mode, const uint64_t* filter_ids, uint64_t nfilter, hnsw_b200_filter_fn fn, void* ctx,
                           const int64_t* resident, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                           int32_t* out_pid, int32_t* out_counts) {
  HB_HS(h);
  if (nq == 0) return 0;
  if (!queries || !out_ids || !out_dist || !out_counts || knbn == 0) return set_err("bad argument");
  HB_PARTS_SHARED_IF(ix);
  const FilterArg f{filter_mode, filter_ids, nfilter, fn, ctx, resident};
  const AnswerArrays out{nullptr, out_ids, out_dist, out_internal, out_pid, out_counts};
  return pass(ix, ix->search_batch(HostBatch{queries, nullptr, nq, (int)dim, knbn, ef_search, f, out}));
}

int hnsw_b200_search_flat(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                          uint64_t ef_search, int filter_mode, const uint64_t* filter_ids, uint64_t nfilter,
                          hnsw_b200_filter_fn fn, void* ctx, uint64_t* out_ids, float* out_dist,
                          uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return search_flat_any(h, queries, nq, dim, knbn, ef_search, filter_mode, filter_ids, nfilter, fn, ctx, nullptr, out_ids,
                         out_dist, out_internal, out_pid, out_counts);
}
int hnsw_b200_search_flat_filtered(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim,
                                   uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                   uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return search_flat_any(h, queries, nq, dim, knbn, ef_search, 0, nullptr, 0, nullptr, nullptr, &filter, out_ids, out_dist,
                         out_internal, out_pid, out_counts);
}

// Submit / wait: the same search with the call split in two, so that one host thread keeps several batches in flight
// (batch i+1 is enqueued before batch i's answers are collected).  Unfiltered, or with a resident filter.  With replicas
// (hnsw_b200_replicate) the batch is sharded like a search_flat call: every device gets its contiguous share enqueued at
// submit time.
static int64_t submit_any(const void* h, const int64_t* resident, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                          uint64_t ef_search, uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                          int32_t* out_counts) {
  HB_HS(h);
  HB_NOT_PARTITIONED(ix, resident ? "search_flat_submit_filtered" : "search_flat_submit");
  if (!queries || !out_ids || !out_dist || !out_counts || knbn == 0 || nq == 0) return set_err("bad argument");
  const FilterArg f{0, nullptr, 0, nullptr, nullptr, resident};
  const AnswerArrays out{nullptr, out_ids, out_dist, out_internal, out_pid, out_counts};
  const int64_t t = ix->submit_batch(HostBatch{queries, nullptr, nq, (int)dim, knbn, ef_search, f, out});
  if (t < 0) g_err = ix->err();
  return t;
}

int64_t hnsw_b200_search_flat_submit(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                                     uint64_t ef_search, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                     int32_t* out_pid, int32_t* out_counts) {
  return submit_any(h, nullptr, queries, nq, dim, knbn, ef_search, out_ids, out_dist, out_internal, out_pid, out_counts);
}
int64_t hnsw_b200_search_flat_submit_filtered(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim,
                                              uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                              uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return submit_any(h, &filter, queries, nq, dim, knbn, ef_search, out_ids, out_dist, out_internal, out_pid, out_counts);
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

static int search_device_any(const void* h, const int64_t* resident, const void* d_queries, uint64_t nq, uint64_t knbn,
                             uint64_t ef_search, void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  HB_HS(h);
  HB_NOT_PARTITIONED(ix, resident ? "search_device_filtered" : "search_device");
  const FilterArg f{0, nullptr, 0, nullptr, nullptr, resident};
  return pass(ix, ix->search_device(f, false, d_queries, nq, knbn, ef_search, (NeighbourOut*)d_out, d_counts, sync != 0,
                                    kernel_ms));
}
int hnsw_b200_search_device(const void* h, const void* d_queries, uint64_t nq, uint64_t knbn,
                            uint64_t ef_search, void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  return search_device_any(h, nullptr, d_queries, nq, knbn, ef_search, d_out, d_counts, sync, kernel_ms);
}
int hnsw_b200_search_device_filtered(const void* h, int64_t filter, const void* d_queries, uint64_t nq, uint64_t knbn,
                                     uint64_t ef_search, void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  return search_device_any(h, &filter, d_queries, nq, knbn, ef_search, d_out, d_counts, sync, kernel_ms);
}

// Exact search: the exact scan of the points a resident filter admits (filter >= 0) or of every point (-1), through the
// same batch driver and device-resident path as the graph searches
int hnsw_b200_search_exact(const void* h, int64_t filter, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                           uint64_t* out_ids, float* out_dist, uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  HB_HS(h);
  if (nq == 0) return 0;
  if (!queries || !out_ids || !out_dist || !out_counts || knbn == 0) return set_err("bad argument");
  HB_PARTS_SHARED_IF(ix);
  FilterArg f;
  if (filter != -1) f.resident = &filter;
  HostBatch b{queries, nullptr, nq, (int)dim, knbn, 0, f, AnswerArrays{nullptr, out_ids, out_dist, out_internal, out_pid, out_counts}};
  b.exact = true;
  return pass(ix, ix->search_batch(b));
}

// A filter per query: filters[i] is a resident filter of the handle or -1; the graph search (ef_search) or the exact
// scan (exact).  One batch, every entry checked before anything runs.
static int per_query_any(const void* h, const int64_t* filters, const void* queries, uint64_t nq, uint64_t dim, uint64_t knbn,
                         uint64_t ef_search, bool exact, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                         int32_t* out_pid, int32_t* out_counts) {
  HB_HS(h);
  if (nq == 0) return 0;
  if (!filters) return set_err("filters is NULL");
  if (!queries || !out_ids || !out_dist || !out_counts || knbn == 0) return set_err("bad argument");
  HB_PARTS_SHARED_IF(ix);
  HostBatch b{queries, nullptr, nq, (int)dim, knbn, ef_search, FilterArg(),
              AnswerArrays{nullptr, out_ids, out_dist, out_internal, out_pid, out_counts}};
  b.exact = exact;
  b.per_query = filters;
  return pass(ix, ix->search_batch(b));
}
int hnsw_b200_search_flat_per_query(const void* h, const int64_t* filters, const void* queries, uint64_t nq, uint64_t dim,
                                    uint64_t knbn, uint64_t ef_search, uint64_t* out_ids, float* out_dist,
                                    uint32_t* out_internal, int32_t* out_pid, int32_t* out_counts) {
  return per_query_any(h, filters, queries, nq, dim, knbn, ef_search, false, out_ids, out_dist, out_internal, out_pid,
                       out_counts);
}
int hnsw_b200_search_exact_per_query(const void* h, const int64_t* filters, const void* queries, uint64_t nq, uint64_t dim,
                                     uint64_t knbn, uint64_t* out_ids, float* out_dist, uint32_t* out_internal,
                                     int32_t* out_pid, int32_t* out_counts) {
  return per_query_any(h, filters, queries, nq, dim, knbn, 0, true, out_ids, out_dist, out_internal, out_pid, out_counts);
}

int hnsw_b200_search_exact_device(const void* h, int64_t filter, const void* d_queries, uint64_t nq, uint64_t knbn,
                                  void* d_out, int32_t* d_counts, int sync, float* kernel_ms) {
  HB_HS(h);
  HB_NOT_PARTITIONED(ix, "search_exact_device");
  FilterArg f;
  if (filter != -1) f.resident = &filter;
  return pass(ix, ix->search_device(f, true, d_queries, nq, knbn, 0, (NeighbourOut*)d_out, d_counts, sync != 0, kernel_ms));
}

int64_t hnsw_b200_filter_new(const void* h, int filter_mode, const uint64_t* filter_ids, uint64_t nfilter,
                             hnsw_b200_filter_fn fn, void* ctx) {
  HB_HS(h);  // shared: the points cannot change while the bitmap is made
  HB_NOT_VIEW(ix);
  if (ix->parts) {
    HB_PARTS_SHARED(ix);
    const int64_t id = ix->new_filter(filter_mode, filter_ids, nfilter, fn, ctx);
    if (id < 0) g_err = ix->err();
    return id;
  }
  const int64_t id = ix->new_filter(filter_mode, filter_ids, nfilter, fn, ctx);
  if (id < 0) g_err = ix->err();
  return id;
}
int hnsw_b200_filter_free(const void* h, int64_t filter) {
  HB_H(h);  // exclusive: waits for every search under the shared lock and every outstanding ticket
  return pass(ix, ix->free_filter(filter));
}

int hnsw_b200_join(void* h) {
  HB_HS(h);
  return pass(ix, ix->join());
}
int hnsw_b200_stream_wait_last(void* h, void* cuda_stream) {
  HB_HS(h);
  return pass(ix, ix->stream_wait_last((cudaStream_t)cuda_stream));
}
int hnsw_b200_set_stream(void* h, void* cuda_stream) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  return pass(ix, ix->set_stream((cudaStream_t)cuda_stream));
}
int hnsw_b200_check_status(void* h) {
  HB_H(h);
  int r = ix->check_status();
  if (r < 0) g_err = ix->err();
  return r;
}

int hnsw_b200_enable_stats(void* h, int enable) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  apply(ix, [=](Index* x) { x->enable_stats(enable != 0); });
  return 0;
}
int hnsw_b200_get_stats(const void* h, uint64_t* out4, int reset) {
  HB_H(h);
  if (ix->parts) {  // the sum over the partitions: out4[3] counts a query once per partition
    HB_PARTS_EXCLUSIVE(ix);
    return pass(ix, ix->parts->get_stats(out4, reset != 0));
  }
  return pass(ix, ix->get_stats(out4, reset != 0));
}

int hnsw_b200_export_points(const void* h, uint8_t* levels, int32_t* ranks, uint64_t* origin, int64_t* entry) {
  HB_H(h);
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
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "export_vectors (export each partition_view)");
  return pass(ix, ix->export_vectors(out));
}
// FlatNeighborhood::from(&hnsw) + get_neighbours(DataId) (flatten.rs:93-126): neighbours of `origin_id` over all
// layers, ascending distance.  Returns the number written (<= cap), -1 when the id is unknown.
int64_t hnsw_b200_flat_neighbours(const void* h, uint64_t origin_id, Neighbour_api* out, uint64_t cap) {
  if (!h) return set_err("NULL handle");
  Index* ix = ((const AnyApi*)h)->ix;
  HB_NOT_PARTITIONED(ix, "flatten (flatten each partition_view)");
  std::shared_lock<std::shared_mutex> g(ix->mu);
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
  if (!h) return set_err("NULL handle");
  Index* ix = ((const AnyApi*)h)->ix;
  HB_NOT_PARTITIONED(ix, "flatten (flatten each partition_view)");
  std::shared_lock<std::shared_mutex> g(ix->mu);
  std::vector<uint64_t> off, nbo;
  std::vector<float> nbd;
  if (pass(ix, ix->flatten(off, nbo, nbd))) return -1;
  if (offsets) memcpy(offsets, off.data(), off.size() * 8);
  if (nb_origin) memcpy(nb_origin, nbo.data(), nbo.size() * 8);
  if (nb_dist) memcpy(nb_dist, nbd.data(), nbd.size() * 4);
  return (int64_t)nbo.size();
}

int64_t hnsw_b200_layer_edges(const void* h, int layer) {
  if (!h) return set_err("NULL handle");
  Index* ix = ((const AnyApi*)h)->ix;
  HB_NOT_PARTITIONED(ix, "layer_edges (export each partition_view)");
  std::shared_lock<std::shared_mutex> g(ix->mu);
  int64_t total = 0;
  if (pass(ix, ix->export_layer(layer, nullptr, nullptr, nullptr, &total))) return -1;
  return total;
}
int hnsw_b200_export_layer(const void* h, int layer, uint64_t* offsets, uint32_t* ids, float* dists) {
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "export_layer (export each partition_view)");
  return pass(ix, ix->export_layer(layer, offsets, ids, dists, nullptr));
}
int hnsw_b200_import_graph(void* h, const void* vecs, uint64_t n, uint64_t dim, const uint64_t* origin,
                           const uint8_t* levels, int64_t entry, int nlayers, const uint64_t* const* offsets,
                           const uint32_t* const* ids, const float* const* dists) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "import_graph");
  return pass(ix, ix->import_graph(vecs, n, (int)dim, origin, levels, entry, nlayers, offsets, ids, dists));
}

int hnsw_b200_blob_header(const void* h, uint64_t* header16) {
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "blob_header");
  return ix->blob_header(header16);
}
int hnsw_b200_blob_alloc(void* h, const uint64_t* header16) {
  HB_H(h);
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
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "blob_info");
  return pass(ix, ix->blob_info(i, dev_ptr, nbytes));
}
int hnsw_b200_blob_commit(void* h) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "blob_commit");
  return pass(ix, ix->blob_commit());
}

// ---- multi-GPU (multi.cu)
int hnsw_b200_replicate(void* h, int ndev, const int* devices) {
  HB_H(h);
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
  HB_H(h);
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "nccl_init");
  if (!id128) return set_err("NULL argument");
  return pass(ix, ix->nccl_init(nranks, rank, id128));
}
int hnsw_b200_nccl_broadcast_index(void* h, int root) {
  HB_H(h);
  HB_NOT_VIEW(ix);
  HB_NOT_PARTITIONED(ix, "nccl_broadcast_index");
  return pass(ix, ix->nccl_broadcast_index(root));
}
int hnsw_b200_nccl_allgather(void* h, const void* d_send, void* d_recv, uint64_t bytes_per_rank, void* cuda_stream) {
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "nccl_allgather");
  return pass(ix, ix->nccl_allgather(d_send, d_recv, bytes_per_rank, (cudaStream_t)cuda_stream));
}

int hnsw_b200_dist_batch(const void* h, const void* queries, uint64_t nq, uint64_t dim, const uint32_t* cand,
                         uint64_t m, float* out) {
  HB_H(h);
  HB_NOT_PARTITIONED(ix, "dist_batch");
  return pass(ix, ix->dist_batch(queries, nq, (int)dim, cand, m, out));
}
int hnsw_b200_bruteforce(const void* h, const void* queries, uint64_t nq, uint64_t dim, uint64_t k,
                         uint32_t* out_ids, float* out_dist) {
  HB_H(h);
  if (ix->parts) {  // every partition's exact answers, merged like a search; ids are global insertion ranks
    HB_PARTS_EXCLUSIVE(ix);
    return pass(ix, ix->parts->bruteforce(queries, nq, (int)dim, k, out_ids, out_dist));
  }
  return pass(ix, ix->bruteforce(queries, nq, (int)dim, k, out_ids, out_dist));
}

}  // extern "C"
