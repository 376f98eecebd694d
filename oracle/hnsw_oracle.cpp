// TEST INFRASTRUCTURE ONLY.  This file is the parity ORACLE and the `cpu_baseline` of
// bench.py.  It is never linked into, loaded by, or called from the product library
// (hnswlib-rs_b200/lib/libhnsw_b200.so); only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load liboracle.so.
//
// PARITY UNPINNED: the reference (jean-pierreBoth/hnswlib-rs, Rust) cannot be compiled in
// this container (no cargo/rustc, no vendored crates), its tests hold no golden vectors and
// all of its test inputs are unseeded (SURVEY.md §4, §8c).  This file is therefore a
// line-by-line CPU restatement of the algorithm, pinned only by (i) the property checks the
// reference's own tests assert (self-query distance 0, always-false filter => empty,
// single-admit filter => <=1 hit, answers in input order, ...), and (ii) unit checks of the
// Rust-std heap semantics in rheap.h.
//
// What is restated (reference file:line):
//   search_layer                       /root/reference/src/hnsw.rs:922-1064
//   search_filter / search             /root/reference/src/hnsw.rs:1487-1599
//   parallel_search ordering contract  /root/reference/src/hnsw.rs:1612-1635
//   insert_slice                       /root/reference/src/hnsw.rs:1077-1215
//   select_neighbours                  /root/reference/src/hnsw.rs:1299-1421
//   reverse_update_neighborhood_simple /root/reference/src/hnsw.rs:1241-1289
//   LayerGenerator::generate           /root/reference/src/hnsw.rs:363-374
//   generate_new_point / check_entry_point  /root/reference/src/hnsw.rs:503-557
//   FilterT for sorted Vec<usize> / closures /root/reference/src/filter.rs:7-24
//   parallel_insert (racy, per-point locks) /root/reference/src/hnsw.rs:1224-1238
//
// It also restates the engine's own insert rule where it departs from the reference (Index::insert_batched, see its
// comment): batch-synchronous inserts, each batch searching the graph as it stood when the batch began, and link mode 1
// (back-links filed in the layer they were made in).  Serial mode-1 builds are restated by tests/linkgraph.py instead.
//
// Two comparison modes:
//   MODE_STD : items compare by distance only, queues are Rust-std BinaryHeaps (rheap.h) —
//              the literal reference behaviour incl. its tie handling.
//   MODE_DET : every comparison uses the total order (distance, internal id).  This is the
//              order the CUDA kernels implement; GPU results must equal MODE_DET exactly.
//              MODE_DET == MODE_STD whenever no two compared distances are bit-equal.
//
// Internal id of a point = its insertion rank (0-based).  PointId(level, rank-in-level) of the
// reference is kept per point for the Neighbour output.
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "distances.h"
#include "rheap.h"

namespace oracle {

enum Mode : int { MODE_STD = 0, MODE_DET = 1 };
static const int NB_LAYER_MAX = 16;  // /root/reference/src/hnsw.rs:42

struct Item {
  float kd;     // signed key distance exactly as the reference stores it (+d in W, -d in C)
  uint32_t id;  // internal id
};

// Ord of PointWithOrder = dist_to_ref.partial_cmp (hnsw.rs:273-297); MODE_DET breaks ties by id.
struct ItemCmp {
  int mode;
  bool neg;  // heap stores -d (nearest = max)
  int operator()(const Item& a, const Item& b) const {
    if (a.kd < b.kd) return -1;
    if (a.kd > b.kd) return 1;
    if (mode == MODE_STD || a.id == b.id) return 0;
    // total order on (d, id): in a positive heap larger id = larger; in a negative heap
    // (stored -d) the nearer item must be the larger one, and nearer = smaller id on ties.
    if (!neg) return a.id < b.id ? -1 : 1;
    return a.id < b.id ? 1 : -1;
  }
};
typedef RHeap<Item, ItemCmp> Heap;

struct Edge {
  uint32_t id;
  float d;  // distance to the owner of the list
};

struct SpinLock {
  std::atomic_flag f = ATOMIC_FLAG_INIT;
  void lock() { while (f.test_and_set(std::memory_order_acquire)) { } }
  void unlock() { f.clear(std::memory_order_release); }
};

struct Node {
  uint64_t origin = 0;
  uint8_t level = 0;
  int32_t rank = -1;
  SpinLock lk;
  std::vector<Edge> nb[NB_LAYER_MAX];  // hnsw.rs:176-188: 16 lists per point
};

struct Counters {
  std::atomic<uint64_t> evals{0}, expansions{0}, adj_read{0}, queries{0};
  std::atomic<uint64_t> spec_ok{0}, spec_total{0};  // study: how often the 2nd-nearest candidate is expanded next
};

typedef int (*filter_fn_t)(uint64_t origin_id, void* ctx);

struct Filter {
  const uint64_t* sorted_ids = nullptr;
  size_t n = 0;
  filter_fn_t fn = nullptr;
  void* ctx = nullptr;
  bool active = false;
  bool pass(uint64_t id) const {
    if (fn) return fn(id, ctx) != 0;
    return std::binary_search(sorted_ids, sorted_ids + n, id);  // filter.rs:11-15
  }
};

struct Neighbour {  // hnsw.rs:98-107
  uint64_t origin;
  float dist;
  uint8_t level;
  int32_t rank;
  uint32_t internal;
};

// splitmix64 -> uniform [0,1) f64.  The reference draws from StdRng seeded through
// Xoshiro256PlusPlus::seed_from_u64(397) (hnsw.rs:329-331); that stream needs the `rand`
// crate, so only the LAW (hnsw.rs:363-374) is restated, with our own documented generator.
struct SplitMix {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double unif() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

static const size_t BLOCK_SHIFT = 14;
static const size_t BLOCK = (size_t)1 << BLOCK_SHIFT;

template <class T>
class Index {
 public:
  Index(int M, size_t max_elements, int max_layer, int ef_c, int metric, int dim)
      : M_(M), ef_c_(ef_c), metric_(metric), dim_(dim) {
    (void)max_elements;  // allocation hint only in the reference (hnsw.rs:452-461)
    max_layer_ = std::min(max_layer, NB_LAYER_MAX);  // hnsw.rs:778
    scale_ = 1.0 / std::log((double)M);              // hnsw.rs:327
    rng_.s = 397;
    for (int l = 0; l < NB_LAYER_MAX; ++l) layer_count_[l] = 0;
    vblocks_.reserve(1 << 18);
    nblocks_.reserve(1 << 18);
  }
  ~Index() {
    for (T* p : vblocks_) free(p);
    for (Node* p : nblocks_) delete[] p;
  }

  // ---- options (hnsw.rs:834-905)
  int mode = MODE_STD;
  int order = ORDER_REF;
  bool extend_candidates = false;  // hnsw.rs:781
  bool keep_pruned = false;        // hnsw.rs:782
  Counters cnt;

  void modify_level_scale(double f) { scale_ = f / std::log((double)M_); }  // hnsw.rs:876-905 (law only)
  void set_seed(uint64_t s) { rng_.s = s; }
  size_t size() const { return n_.load(std::memory_order_acquire); }
  int dim() const { return dim_; }
  int M() const { return M_; }
  int max_layer() const { return max_layer_; }
  int64_t entry() const { return entry_.load(std::memory_order_acquire); }
  size_t layer_count(int l) const { return layer_count_[l].load(); }

  const T* vec(uint32_t id) const { return vblocks_[id >> BLOCK_SHIFT] + (size_t)(id & (BLOCK - 1)) * dim_; }
  Node& node(uint32_t id) const { return nblocks_[id >> BLOCK_SHIFT][id & (BLOCK - 1)]; }

  float dist(const T* a, const T* b) {
    return eval_dist<T>(metric_, order, a, b, (size_t)dim_);
  }

  // LayerGenerator::generate, hnsw.rs:363-374
  int draw_level() {
    double xsi = rng_.unif();
    if (xsi <= 0.) xsi = 1e-300;
    double level = -std::log(xsi) * scale_;
    size_t ulevel = (size_t)std::floor(level);
    if (ulevel >= (size_t)max_layer_) ulevel = (size_t)(rng_.next() % (uint64_t)max_layer_);
    return (int)ulevel;
  }

  // ------------------------------------------------------------------ search_layer
  // hnsw.rs:922-1064.  Returns the positive-distance heap W.
  struct Scratch {
    std::vector<uint32_t> stamp;
    uint32_t epoch = 0;
    std::vector<Edge> list;
    uint64_t evals = 0, expansions = 0, adj_read = 0, spec_ok = 0, spec_total = 0;
    int64_t predicted = -1;
    void begin(size_t n) {
      if (stamp.size() < n) stamp.resize(n + n / 2 + 1024, 0);
      if (++epoch == 0) { std::fill(stamp.begin(), stamp.end(), 0); epoch = 1; }
    }
    bool visit(uint32_t id) {  // true if newly visited
      if (id >= stamp.size()) stamp.resize((size_t)id + (size_t)id / 2 + 1024, 0);  // index grew under a racing insert
      if (stamp[id] == epoch) return false;
      stamp[id] = epoch;
      return true;
    }
  };

  // `mask` (batched inserts): bit l says whether layer l counts as non-empty for this search, in place of layer_count_
  Heap search_layer(const T* q, uint32_t ep, size_t ef, int layer, const Filter* filter, Scratch& sc,
                    bool locked, const uint16_t* mask = nullptr) {
    Heap W(ItemCmp{mode, false});
    const bool empty = mask ? !((*mask >> layer) & 1u) : layer_count_[layer].load(std::memory_order_acquire) == 0;
    if (empty) return W;  // 942-946
    // (947-950: negative rank cannot happen for a stored point)
    sc.begin(size());
    float d0 = dist(q, vec(ep));  // 952
    sc.evals++;
    sc.visit(ep);  // 955-956
    Heap C(ItemCmp{mode, true});
    C.push(Item{-d0, ep});  // 960-963
    W.push(Item{d0, ep});   // 964-967  (unfiltered)
    const bool has_filter = filter && filter->active;
    sc.predicted = -1;
    while (!C.empty()) {  // 969
      Item c = C.pop();   // 971
      if (sc.predicted >= 0) { sc.spec_total++; if ((int64_t)c.id == sc.predicted) sc.spec_ok++; }
      sc.predicted = C.empty() ? -1 : (int64_t)C.peek().id;  // nearest remaining candidate BEFORE c's neighbours are seen
      // 973 unwraps W.peek(): the reference would PANIC on an empty W here (reachable only with a filter, ef == 1 and
      // an entry point that fails it); the restatement and the engine return the empty W instead.
      if (W.empty()) return W;
      const Item& f = W.peek();  // 973
      bool stop;
      if (mode == MODE_STD) stop = (-c.kd) > f.kd;  // 981
      else if (has_filter) stop = (-c.kd) > f.kd;  // with a filter the rule only prunes W: distances, as the reference
      else stop = ItemCmp{MODE_DET, false}(Item{-c.kd, c.id}, f) > 0;
      if (stop) {
        if (!has_filter) return W;  // 992-993
        if (W.size() >= ef)         // 994-1000
          W.retain([&](const Item& p) { return filter->pass(node(p.id).origin); });
      }
      // 1006: read lock on c's neighbours; copy the list so evals run outside the lock
      Node& cn = node(c.id);
      if (locked) cn.lk.lock();
      sc.list = cn.nb[layer];
      if (locked) cn.lk.unlock();
      sc.expansions++;
      sc.adj_read += sc.list.size();
      for (const Edge& e : sc.list) {  // 1013
        if (!sc.visit(e.id)) continue;  // 1016-1017
        if (W.empty()) return W;        // 1019-1024
        const Item f2 = W.peek();
        float de = dist(q, vec(e.id));  // 1026
        sc.evals++;
        bool closer;
        if (mode == MODE_STD) closer = de < f2.kd;
        else closer = ItemCmp{MODE_DET, false}(Item{de, e.id}, f2) < 0;
        if (closer || W.size() < ef) {  // 1028
          C.push(Item{-de, e.id});      // 1035-1036
          if (!has_filter) {
            W.push(Item{de, e.id});     // 1038
          } else if (filter->pass(node(e.id).origin)) {  // 1040-1049
            if (W.size() == 1) {
              uint64_t only = node(W.peek().id).origin;
              if (!filter->pass(only)) W.clear();
            }
            W.push(Item{de, e.id});
          }
          if (W.size() > ef) W.pop();  // 1051-1053
        }
      }
    }
    return W;  // 1063
  }

  // ------------------------------------------------------------------ search_filter
  // hnsw.rs:1487-1580
  size_t search(const T* q, size_t knbn, size_t ef_arg, const Filter* filter, Neighbour* out, Scratch& sc) {
    int64_t ep64 = entry();
    if (ep64 < 0) return 0;  // 1498-1503
    uint32_t ep = (uint32_t)ep64;
    float best = dist(q, vec(ep));  // 1506
    sc.evals++;
    uint32_t pivot = ep;
    int ep_level = node(ep).level;
    for (int layer = ep_level; layer >= 1; --layer) {  // 1511
      bool changed = false;
      uint32_t new_pivot = pivot;
      const std::vector<Edge>& nbs = node(pivot).nb[layer];
      sc.adj_read += nbs.size();
      for (const Edge& n : nbs) {  // 1516
        float t = dist(q, vec(n.id));  // 1518
        sc.evals++;
        if (t < best) { new_pivot = n.id; changed = true; best = t; }  // 1519-1523 (strict, first min)
      }
      if (changed) pivot = new_pivot;  // 1526-1528
    }
    size_t ef = std::max(ef_arg, knbn);  // 1531
    int layer_to_search = 0;             // 1534-1540
    while (layer_to_search < NB_LAYER_MAX - 1 && layer_count_[layer_to_search].load() == 0) layer_to_search++;
    Heap W = search_layer(q, pivot, ef, layer_to_search, filter, sc, false);  // 1542
    std::vector<Item> sorted = W.into_sorted_vec();  // 1544
    size_t last = std::min(std::min(knbn, ef), sorted.size());  // 1547
    size_t n = 0;
    const bool has_filter = filter && filter->active;
    for (size_t i = 0; i < last; ++i) {  // 1549-1579
      const Node& nd = node(sorted[i].id);
      if (has_filter && !filter->pass(nd.origin)) continue;
      out[n++] = Neighbour{nd.origin, sorted[i].kd, nd.level, nd.rank, sorted[i].id};
    }
    return n;
  }

  void flush(Scratch& sc, uint64_t nq) {
    cnt.evals += sc.evals; cnt.expansions += sc.expansions; cnt.adj_read += sc.adj_read; cnt.queries += nq;
    cnt.spec_ok += sc.spec_ok; cnt.spec_total += sc.spec_total;
    sc.evals = sc.expansions = sc.adj_read = sc.spec_ok = sc.spec_total = 0;
  }

  // parallel_search: answers in INPUT order whatever the completion order (hnsw.rs:1622-1633)
  void search_batch(const T* qs, size_t nq, size_t knbn, size_t ef, const Filter* filter, int nthreads,
                    Neighbour* out, int32_t* counts) {
    std::atomic<size_t> next{0};
    auto work = [&]() {
      Scratch sc;
      size_t done = 0;
      for (;;) {
        size_t b = next.fetch_add(16);
        if (b >= nq) break;
        size_t e = std::min(nq, b + 16);
        for (size_t i = b; i < e; ++i) {
          counts[i] = (int32_t)search(qs + i * (size_t)dim_, knbn, ef, filter, out + i * knbn, sc);
          ++done;
        }
      }
      flush(sc, done);
    };
    if (nthreads <= 1) { work(); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) th.emplace_back(work);
    for (auto& t : th) t.join();
  }

  // ------------------------------------------------------------------ insert
  // generate_new_point, hnsw.rs:503-531 (level passed in so that batch draws stay in order)
  uint32_t new_point(const T* v, uint64_t origin, int level, size_t* rank_out) {
    std::lock_guard<std::mutex> g(glock_);
    size_t id = n_.load(std::memory_order_relaxed);
    if ((id >> BLOCK_SHIFT) >= vblocks_.size()) {
      vblocks_.push_back((T*)malloc(BLOCK * (size_t)dim_ * sizeof(T)));
      nblocks_.push_back(new Node[BLOCK]);
    }
    memcpy(vblocks_[id >> BLOCK_SHIFT] + (id & (BLOCK - 1)) * (size_t)dim_, v, (size_t)dim_ * sizeof(T));
    Node& nd = nblocks_[id >> BLOCK_SHIFT][id & (BLOCK - 1)];
    nd.origin = origin;
    nd.level = (uint8_t)level;
    nd.rank = (int32_t)layer_count_[level].load();  // 511
    layer_count_[level].fetch_add(1, std::memory_order_release);  // 516
    n_.store(id + 1, std::memory_order_release);   // 520-523
    *rank_out = id + 1;
    return (uint32_t)id;
  }

  void check_entry_point(uint32_t p) {  // hnsw.rs:534-557
    std::lock_guard<std::mutex> g(elock_);
    int64_t e = entry_.load();
    if (e < 0 || node(p).level > node((uint32_t)e).level) entry_.store((int64_t)p, std::memory_order_release);
  }

  // select_neighbours, hnsw.rs:1299-1421.  `cand` is the negative heap (nearest = max).
  void select_neighbours(const T* q, Heap& cand, size_t nb, bool extend_asked, int layer, bool keep_pr,
                         std::vector<Edge>& out, Scratch& sc, bool locked) {
    out.clear();
    bool extend = false;
    if (cand.size() <= nb) {  // 1318
      if (!extend_asked) {
        while (!cand.empty()) { Item p = cand.pop(); out.push_back(Edge{p.id, -p.kd}); }  // 1321-1326
        return;
      }
      extend = true;  // 1329
    }
    if (extend) {  // 1336-1362.  The reference iterates hashbrown maps (random order); here the
      // new candidates are visited in ascending id order (tie order is unspecified upstream).
      std::vector<uint32_t> cset;
      for (const Item& c : cand.items()) cset.push_back(c.id);
      std::sort(cset.begin(), cset.end());
      std::vector<uint32_t> fresh;
      for (uint32_t p : cset) {
        Node& pn = node(p);
        if (locked) pn.lk.lock();
        sc.list = pn.nb[layer];
        if (locked) pn.lk.unlock();
        for (const Edge& e : sc.list)
          if (!std::binary_search(cset.begin(), cset.end(), e.id)) fresh.push_back(e.id);
      }
      std::sort(fresh.begin(), fresh.end());
      fresh.erase(std::unique(fresh.begin(), fresh.end()), fresh.end());
      for (uint32_t p : fresh) {
        float d = dist(q, vec(p));  // 1359
        sc.evals++;
        cand.push(Item{-d, p});     // 1360
      }
    }
    Heap discarded(ItemCmp{mode, true});
    while (!cand.empty() && out.size() < nb) {  // 1365
      Item e = cand.pop();
      bool ins = true;
      const T* ev = vec(e.id);
      for (const Edge& d : out) {  // 1373-1375
        float dd = dist(ev, vec(d.id));
        sc.evals++;
        if (dd <= -e.kd) { ins = false; break; }
      }
      if (ins) out.push_back(Edge{e.id, -e.kd});          // 1379-1382
      else if (keep_pr) discarded.push(e);               // 1387-1392
    }
    if (keep_pr) {  // 1399-1409
      while (!discarded.empty() && out.size() < nb) {
        Item b = discarded.pop();
        out.push_back(Edge{b.id, -b.kd});
      }
    }
  }

  void sort_edges(std::vector<Edge>& v) {  // sort_unstable by distance (hnsw.rs:1195,1280)
    if (mode == MODE_STD)
      std::stable_sort(v.begin(), v.end(), [](const Edge& a, const Edge& b) { return a.d < b.d; });
    else
      std::sort(v.begin(), v.end(), [](const Edge& a, const Edge& b) { return a.d < b.d || (a.d == b.d && a.id < b.id); });
  }

  // reverse_update_neighborhood_simple, hnsw.rs:1241-1289.  link_mode1: each back-link goes to the layer it was made in
  // (the engine's link mode 1, csrc/build.cu insert_link_kernel) instead of the new point's level.
  void reverse_update(uint32_t np, bool locked, bool link_mode1 = false) {
    Node& nn = node(np);
    int level = nn.level;
    for (int l = level; l >= 0; --l) {  // 1248
      std::vector<Edge> mine;
      if (locked) nn.lk.lock();
      mine = nn.nb[l];
      if (locked) nn.lk.unlock();
      for (const Edge& q : mine) {  // 1249
        if (q.id == np) continue;   // 1250
        Node& qn = node(q.id);
        if (locked) qn.lk.lock();
        int l_n = link_mode1 ? l : level;  // 1257: the NEW point's level, not l
        std::vector<Edge>& tgt = qn.nb[l_n];
        bool already = false;
        for (const Edge& o : tgt) if (o.id == np) { already = true; break; }  // 1258-1267
        if (!already) {
          tgt.push_back(Edge{np, q.d});  // 1268
          size_t thr = l_n > 0 ? (size_t)M_ : (size_t)2 * M_;  // 1272-1276
          bool shrink = tgt.size() > thr;
          sort_edges(tgt);               // 1280
          if (shrink) tgt.pop_back();    // 1281-1283
        }
        if (locked) qn.lk.unlock();
      }
    }
  }

  // insert_slice, hnsw.rs:1077-1215
  void insert(const T* v, uint64_t origin, int level, Scratch& sc, bool locked) {
    size_t point_rank;
    uint32_t np = new_point(v, origin, level, &point_rank);
    int64_t ep64 = entry();
    if (ep64 >= 0 && point_rank == 1) return;  // 1096-1102
    if (ep64 < 0) { check_entry_point(np); return; }  // 1106-1109
    insert_search(np, (uint32_t)ep64, sc, locked, nullptr, false);
    reverse_update(np, locked);  // 1210
    check_entry_point(np);       // 1212
  }

  // The part of insert_slice between generate_new_point and reverse_update (hnsw.rs:1103-1205): descent from `ep`, then
  // search and selection per layer, writing the stored point np's own lists.  `mask` as in search_layer; link_mode1
  // drops the descent's push into np's lists above its level (1140-1144), as the engine's link mode 1 does.
  void insert_search(uint32_t np, uint32_t ep, Scratch& sc, bool locked, const uint16_t* mask, bool link_mode1) {
    Node& nn = node(np);
    const T* v = vec(np);
    const int level = nn.level;
    int max_level_observed = node(ep).level;  // 1103
    float dist_to_entry = dist(v, vec(ep));   // 1110-1112
    sc.evals++;
    for (int l = max_level_observed; l >= level + 1; --l) {  // 1114
      Heap sp = search_layer(v, ep, 1, l, nullptr, sc, locked, mask);
      if (sp.size() > 1) { fprintf(stderr, "oracle: search_layer(ef=1) returned %zu\n", sp.size()); abort(); }  // 1128
      if (!sp.empty()) {
        Item r = sp.pop();
        if (locked) nn.lk.lock();
        if (!link_mode1 && nn.nb[l].size() < (size_t)(uint8_t)M_)
          nn.nb[l].push_back(Edge{r.id, r.kd});  // 1140-1144 (list ABOVE level)
        if (locked) nn.lk.unlock();
        float t = dist(v, vec(r.id));  // 1146
        sc.evals++;
        if (t < dist_to_entry) { ep = r.id; dist_to_entry = t; }  // 1147-1150
      }
    }
    std::vector<Edge> sel;
    for (int l = level; l >= 0; --l) {  // 1158
      Heap sp = search_layer(v, ep, (size_t)ef_c_, l, nullptr, sc, locked, mask);  // 1161
      // from_positive_binaryheap_to_negative_binary_heap, 1664-1681: iterate in heap-vector order
      Heap neg(ItemCmp{mode, true});
      for (const Item& p : sp.items()) neg.push(Item{-p.kd, p.id});
      if (!neg.empty()) {  // 1174
        size_t nb_conn = l == 0 ? (size_t)2 * M_ : (size_t)M_;  // 1177-1183
        bool ext = l == 0 ? extend_candidates : false;
        select_neighbours(v, neg, nb_conn, ext, l, keep_pruned, sel, sc, locked);
        sort_edges(sel);  // 1195
        if (locked) nn.lk.lock();
        nn.nb[l] = sel;   // 1197
        if (locked) nn.lk.unlock();
        if (!sel.empty()) ep = sel[0].id;  // 1201-1203
      }
    }
  }

  // The engine's batched insert (csrc/index.cu Index::insert_batch, csrc/build.cu), restated: the points go in as the
  // batches sizes[0..nbatches) that partition [0, n).  Per batch:
  //   * store every point in order (new_point); point i's layer mask is taken right after its own new_point: layer l
  //     counts as non-empty iff a point of level l was stored up to and including i (Index::insert_batch's masks[i]);
  //   * phase A (insert_search) for every point against the graph as it stood when the batch began: no list names a
  //     point of the batch yet, so the phase is read-only on other points' lists and runs on nthreads threads;
  //   * phase B (reverse_update) for every point, in insertion order, or in a permutation drawn from order_seed != 0;
  //   * check_entry_point for every point.
  // The reference instead races whole inserts on a rayon pool (hnsw.rs:1224-1238).  Batches the engine never makes are
  // refused: a first point into an empty index that is not alone, and a batch of several points with one above the
  // entry level (the engine cuts a batch before such a point and runs it alone).  link_mode1 as in insert_search and
  // reverse_update.
  void insert_batched(const T* vs, const uint64_t* ids, const int* levels, size_t n, const uint64_t* sizes,
                      size_t nbatches, int nthreads, bool link_mode1, uint64_t order_seed) {
    size_t done = 0;
    for (size_t b = 0; b < nbatches; ++b) {
      const size_t cnt = (size_t)sizes[b];
      if (cnt == 0 || done + cnt > n) {
        fprintf(stderr, "oracle: insert_batched: batch %zu of %zu points does not fit the %zu points left\n", b, cnt, n - done);
        abort();
      }
      const int64_t e = entry();
      if (e < 0 && cnt != 1) {
        fprintf(stderr, "oracle: insert_batched: the first point into an empty index must be alone in its batch\n");
        abort();
      }
      if (e >= 0 && cnt > 1)
        for (size_t i = done; i < done + cnt; ++i)
          if (levels[i] > node((uint32_t)e).level) {
            fprintf(stderr, "oracle: insert_batched: point %zu of level %d shares batch %zu above the entry level %d\n", i,
                    levels[i], b, (int)node((uint32_t)e).level);
            abort();
          }
      std::vector<uint32_t> pts(cnt);
      std::vector<uint16_t> masks(cnt);
      for (size_t i = 0; i < cnt; ++i) {
        size_t r;
        pts[i] = new_point(vs + (done + i) * (size_t)dim_, ids[done + i], levels[done + i], &r);
        uint16_t m = 0;
        for (int l = 0; l < NB_LAYER_MAX; ++l)
          if (layer_count_[l].load() > 0) m |= (uint16_t)(1u << l);
        masks[i] = m;
      }
      if (e >= 0) {
        std::atomic<size_t> next{0};
        auto work = [&]() {
          Scratch sc;
          for (size_t i; (i = next.fetch_add(1)) < cnt;) insert_search(pts[i], (uint32_t)e, sc, false, &masks[i], link_mode1);
          flush(sc, 0);
        };
        const size_t nth = std::min<size_t>((size_t)std::max(nthreads, 1), cnt);
        if (nth <= 1) {
          work();
        } else {
          std::vector<std::thread> th;
          for (size_t t = 0; t < nth; ++t) th.emplace_back(work);
          for (auto& t : th) t.join();
        }
        std::vector<uint32_t> order(pts);
        if (order_seed) {  // Fisher-Yates over splitmix64
          SplitMix g{order_seed};
          for (size_t i = cnt; i > 1; --i) std::swap(order[i - 1], order[g.next() % i]);
        }
        for (uint32_t p : order) reverse_update(p, false, link_mode1);
      }
      for (uint32_t p : pts) check_entry_point(p);
      done += cnt;
    }
    if (done != n) {
      fprintf(stderr, "oracle: insert_batched: the batches hold %zu of %zu points\n", done, n);
      abort();
    }
  }

  // parallel_insert: rayon par_iter of insert (hnsw.rs:1224-1238).  Levels are drawn up front in
  // input order so that a run is reproducible up to the thread race on the graph itself.
  void insert_batch(const T* vs, const uint64_t* ids, size_t n, int nthreads) {
    std::vector<int> levels(n);
    for (size_t i = 0; i < n; ++i) levels[i] = draw_level();
    insert_batch_levels(vs, ids, levels.data(), n, nthreads);
  }
  void insert_batch_levels(const T* vs, const uint64_t* ids, const int* levels, size_t n, int nthreads) {
    if (nthreads <= 1) {
      Scratch sc;
      for (size_t i = 0; i < n; ++i) insert(vs + i * (size_t)dim_, ids[i], levels[i], sc, false);
      flush(sc, 0);
      return;
    }
    std::atomic<size_t> next{0};
    size_t start = 0;
    {   // the very first points go in serially so that an entry point exists
      Scratch sc;
      while (start < n && size() < 64) { insert(vs + start * (size_t)dim_, ids[start], levels[start], sc, false); ++start; }
      flush(sc, 0);
    }
    next = start;
    auto work = [&]() {
      Scratch sc;
      for (;;) {
        size_t i = next.fetch_add(1);
        if (i >= n) break;
        insert(vs + i * (size_t)dim_, ids[i], levels[i], sc, true);
      }
      flush(sc, 0);
    };
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) th.emplace_back(work);
    for (auto& t : th) t.join();
  }

  // ------------------------------------------------------------------ import (graph built elsewhere)
  // Points are appended with their level/rank/origin; adjacency given per layer as CSR.
  void import_points(const T* vs, const uint64_t* origin, const uint8_t* levels, size_t n, int64_t entry_id) {
    for (size_t i = 0; i < n; ++i) {
      size_t r;
      new_point(vs + i * (size_t)dim_, origin[i], levels[i], &r);
    }
    entry_.store(entry_id);
  }
  void import_layer(int layer, const uint64_t* offsets, const uint32_t* ids, const float* dists, size_t n) {
    for (size_t i = 0; i < n; ++i) {
      std::vector<Edge>& l = node((uint32_t)i).nb[layer];
      l.clear();
      for (uint64_t j = offsets[i]; j < offsets[i + 1]; ++j) l.push_back(Edge{ids[j], dists ? dists[j] : 0.f});
    }
  }

 private:
  int M_, max_layer_, ef_c_, metric_, dim_;
  double scale_;
  SplitMix rng_;
  std::mutex glock_, elock_;
  std::atomic<size_t> n_{0};
  std::atomic<int64_t> entry_{-1};
  std::atomic<size_t> layer_count_[NB_LAYER_MAX];
  std::vector<T*> vblocks_;
  std::vector<Node*> nblocks_;
};

}  // namespace oracle

// ======================================================================== C ABI (ctypes)
using namespace oracle;

struct OracleHandle {
  int dtype;  // 0 f32, 1 u8, 2 u16, 3 u32, 4 i32
  void* idx;
};

#define DISPATCH(h, CALL)                                                   \
  switch ((h)->dtype) {                                                     \
    case 0: { auto* ix = (Index<float>*)(h)->idx; CALL; } break;            \
    case 1: { auto* ix = (Index<uint8_t>*)(h)->idx; CALL; } break;          \
    case 2: { auto* ix = (Index<uint16_t>*)(h)->idx; CALL; } break;         \
    case 3: { auto* ix = (Index<uint32_t>*)(h)->idx; CALL; } break;         \
    case 4: { auto* ix = (Index<int32_t>*)(h)->idx; CALL; } break;          \
  }

template <class T>
static void do_search_batch(Index<T>* ix, const void* qs, size_t nq, size_t k, size_t ef, const Filter* f, int nth,
                            uint64_t* out_origin, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                            int32_t* counts) {
  std::vector<Neighbour> tmp(nq * k);
  ix->search_batch((const T*)qs, nq, k, ef, f, nth, tmp.data(), counts);
  for (size_t i = 0; i < nq; ++i)
    for (size_t j = 0; j < k; ++j) {
      size_t o = i * k + j;
      if ((int32_t)j < counts[i]) {
        out_origin[o] = tmp[o].origin;
        out_dist[o] = tmp[o].dist;
        if (out_internal) out_internal[o] = tmp[o].internal;
        if (out_pid) { out_pid[2 * o] = tmp[o].level; out_pid[2 * o + 1] = tmp[o].rank; }
      } else {
        out_origin[o] = ~0ull;
        out_dist[o] = INFINITY;
        if (out_internal) out_internal[o] = 0xFFFFFFFFu;
        if (out_pid) { out_pid[2 * o] = -1; out_pid[2 * o + 1] = -1; }
      }
    }
}

// Memory placement for the CPU baseline: interleave the calling thread's future allocations over all NUMA nodes
// (set_mempolicy(MPOL_INTERLEAVE)), as a multi-threaded build would spread them by first touch; on = 0 restores the
// default policy.  Returns 0 on success, -1 when the kernel refuses (single node, container policy): harmless.
static int set_interleave(int on) {
#ifdef SYS_set_mempolicy
  unsigned long mask[16];
  for (int i = 0; i < 16; ++i) mask[i] = ~0ul;
  long r = on ? syscall(SYS_set_mempolicy, 3 /*MPOL_INTERLEAVE*/, mask, 1024ul) : syscall(SYS_set_mempolicy, 0, nullptr, 0ul);
  if (r != 0 && on) {  // retry with a small node mask (kernels reject bits beyond the possible nodes on some configs)
    for (int nodes = 8; nodes >= 2 && r != 0; nodes /= 2) {
      unsigned long m1 = (1ul << nodes) - 1;
      r = syscall(SYS_set_mempolicy, 3, &m1, (unsigned long)nodes + 1);
    }
  }
  return r == 0 ? 0 : -1;
#else
  (void)on;
  return -1;
#endif
}

extern "C" {

int oracle_numa_interleave(int on) { return set_interleave(on); }

void* oracle_new(int dtype, int M, uint64_t max_elements, int max_layer, int ef_c, int metric, int dim) {
  OracleHandle* h = new OracleHandle{dtype, nullptr};
  switch (dtype) {
    case 0: h->idx = new Index<float>(M, max_elements, max_layer, ef_c, metric, dim); break;
    case 1: h->idx = new Index<uint8_t>(M, max_elements, max_layer, ef_c, metric, dim); break;
    case 2: h->idx = new Index<uint16_t>(M, max_elements, max_layer, ef_c, metric, dim); break;
    case 3: h->idx = new Index<uint32_t>(M, max_elements, max_layer, ef_c, metric, dim); break;
    case 4: h->idx = new Index<int32_t>(M, max_elements, max_layer, ef_c, metric, dim); break;
    default: delete h; return nullptr;
  }
  return h;
}

void oracle_free(void* hv) {
  OracleHandle* h = (OracleHandle*)hv;
  if (!h) return;
  DISPATCH(h, delete ix);
  delete h;
}

// opt: 0 mode, 1 order, 2 extend_candidates, 3 keep_pruned, 4 level_scale (as double), 5 seed
void oracle_set_option(void* hv, int opt, double val) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    switch (opt) {
      case 0: ix->mode = (int)val; break;
      case 1: ix->order = (int)val; break;
      case 2: ix->extend_candidates = val != 0; break;
      case 3: ix->keep_pruned = val != 0; break;
      case 4: ix->modify_level_scale(val); break;
      case 5: ix->set_seed((uint64_t)val); break;
    }
  });
}

uint64_t oracle_size(void* hv) {
  OracleHandle* h = (OracleHandle*)hv;
  uint64_t n = 0;
  DISPATCH(h, n = ix->size());
  return n;
}

int64_t oracle_entry(void* hv) {
  OracleHandle* h = (OracleHandle*)hv;
  int64_t e = -1;
  DISPATCH(h, e = ix->entry());
  return e;
}

// levels == NULL: draw from the level law.  nthreads > 1: racy parallel insert like rayon.
void oracle_insert_batch(void* hv, const void* vs, const uint64_t* ids, const int32_t* levels, uint64_t n, int nthreads) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    typedef typename std::remove_pointer<decltype(ix->vec(0))>::type CT;
    typedef typename std::remove_const<CT>::type T;
    if (levels) ix->insert_batch_levels((const T*)vs, ids, (const int*)levels, n, nthreads);
    else ix->insert_batch((const T*)vs, ids, n, nthreads);
  });
}

// the engine's batch-synchronous insert (Index::insert_batched): sizes[0..nbatches) partition the n points; link_mode
// 0 or 1; order_seed != 0 links each batch's points in a random order (the graph must not depend on it)
void oracle_insert_batched(void* hv, const void* vs, const uint64_t* ids, const int32_t* levels, uint64_t n,
                           const uint64_t* sizes, uint64_t nbatches, int nthreads, int link_mode, uint64_t order_seed) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    typedef typename std::remove_const<typename std::remove_pointer<decltype(ix->vec(0))>::type>::type T;
    ix->insert_batched((const T*)vs, ids, (const int*)levels, n, sizes, nbatches, nthreads, link_mode != 0, order_seed);
  });
}

void oracle_draw_levels(void* hv, int32_t* out, uint64_t n) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, { for (uint64_t i = 0; i < n; ++i) out[i] = ix->draw_level(); });
}

// filter: sorted origin-id array (may be NULL with nfilter = 0 and use_filter = 1 => always false),
// or a callback.  use_filter = 0 => no filter.
void oracle_search_batch(void* hv, const void* qs, uint64_t nq, uint64_t k, uint64_t ef, int use_filter,
                         const uint64_t* filter_ids, uint64_t nfilter, filter_fn_t fn, void* ctx, int nthreads,
                         uint64_t* out_origin, float* out_dist, uint32_t* out_internal, int32_t* out_pid,
                         int32_t* counts) {
  OracleHandle* h = (OracleHandle*)hv;
  Filter f;
  f.active = use_filter != 0;
  f.sorted_ids = filter_ids;
  f.n = nfilter;
  f.fn = fn;
  f.ctx = ctx;
  DISPATCH(h, do_search_batch(ix, qs, nq, k, ef, use_filter ? &f : nullptr, nthreads, out_origin, out_dist,
                              out_internal, out_pid, counts));
}

uint64_t oracle_spec_counters(void* hv, uint64_t* out2) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, { out2[0] = ix->cnt.spec_ok; out2[1] = ix->cnt.spec_total; });
  return 0;
}

// evals, expansions, adjacency ids read, queries; reset when `reset` != 0
void oracle_counters(void* hv, uint64_t* out4, int reset) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    out4[0] = ix->cnt.evals; out4[1] = ix->cnt.expansions; out4[2] = ix->cnt.adj_read; out4[3] = ix->cnt.queries;
    if (reset) { ix->cnt.evals = 0; ix->cnt.expansions = 0; ix->cnt.adj_read = 0; ix->cnt.queries = 0; }
  });
}

// ---- export: per point (level, rank, origin); per layer CSR (offsets[N+1], ids, dists)
void oracle_export_points(void* hv, uint8_t* levels, int32_t* ranks, uint64_t* origin) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    size_t n = ix->size();
    for (size_t i = 0; i < n; ++i) {
      const Node& nd = ix->node((uint32_t)i);
      if (levels) levels[i] = nd.level;
      if (ranks) ranks[i] = nd.rank;
      if (origin) origin[i] = nd.origin;
    }
  });
}

uint64_t oracle_layer_edges(void* hv, int layer) {
  OracleHandle* h = (OracleHandle*)hv;
  uint64_t tot = 0;
  DISPATCH(h, { size_t n = ix->size(); for (size_t i = 0; i < n; ++i) tot += ix->node((uint32_t)i).nb[layer].size(); });
  return tot;
}

void oracle_export_layer(void* hv, int layer, uint64_t* offsets, uint32_t* ids, float* dists) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    size_t n = ix->size();
    uint64_t o = 0;
    for (size_t i = 0; i < n; ++i) {
      offsets[i] = o;
      for (const Edge& e : ix->node((uint32_t)i).nb[layer]) { ids[o] = e.id; if (dists) dists[o] = e.d; ++o; }
    }
    offsets[n] = o;
  });
}

void oracle_export_vectors(void* hv, void* out) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    size_t n = ix->size();
    size_t rb = (size_t)ix->dim() * sizeof(*ix->vec(0));
    for (size_t i = 0; i < n; ++i) memcpy((char*)out + i * rb, ix->vec((uint32_t)i), rb);
  });
}

void oracle_import_points(void* hv, const void* vs, const uint64_t* origin, const uint8_t* levels, uint64_t n, int64_t entry) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, {
    typedef typename std::remove_const<typename std::remove_pointer<decltype(ix->vec(0))>::type>::type T;
    ix->import_points((const T*)vs, origin, levels, n, entry);
  });
}

void oracle_import_layer(void* hv, int layer, const uint64_t* offsets, const uint32_t* ids, const float* dists, uint64_t n) {
  OracleHandle* h = (OracleHandle*)hv;
  DISPATCH(h, ix->import_layer(layer, offsets, ids, dists, n));
}

// ---- stand-alone distance (for unit tests of the metric restatements)
float oracle_dist(int dtype, int metric, int order, const void* a, const void* b, uint64_t d) {
  switch (dtype) {
    case 0: return eval_dist<float>(metric, order, (const float*)a, (const float*)b, d);
    case 1: return eval_dist<uint8_t>(metric, order, (const uint8_t*)a, (const uint8_t*)b, d);
    case 2: return eval_dist<uint16_t>(metric, order, (const uint16_t*)a, (const uint16_t*)b, d);
    case 3: return eval_dist<uint32_t>(metric, order, (const uint32_t*)a, (const uint32_t*)b, d);
    case 4: return eval_dist<int32_t>(metric, order, (const int32_t*)a, (const int32_t*)b, d);
  }
  return NAN;
}

// ---- the natural logarithm each order uses: device_logf in ORDER_GPU, the C library's in ORDER_REF
void oracle_logf(int order, const float* x, float* out, uint64_t n) {
  for (uint64_t i = 0; i < n; ++i) out[i] = order == ORDER_GPU ? device_logf(x[i]) : std::log(x[i]);
}

// ---- exact brute force (ground truth for recall): ascending (dist, id), nthreads workers
void oracle_bruteforce(int dtype, int metric, int order, const void* base, uint64_t n, const void* qs, uint64_t nq,
                       uint64_t d, uint64_t k, int nthreads, uint32_t* out_ids, float* out_dist) {
  auto run = [&](auto tag) {
    typedef decltype(tag) T;
    const T* B = (const T*)base;
    const T* Q = (const T*)qs;
    std::atomic<size_t> next{0};
    auto work = [&]() {
      std::vector<std::pair<float, uint32_t>> heap;
      for (;;) {
        size_t i = next.fetch_add(1);
        if (i >= nq) break;
        heap.clear();
        for (size_t j = 0; j < n; ++j) {
          float dd = eval_dist<T>(metric, order, Q + i * d, B + j * d, d);
          std::pair<float, uint32_t> it(dd, (uint32_t)j);
          if (heap.size() < k) { heap.push_back(it); std::push_heap(heap.begin(), heap.end()); }
          else if (it < heap.front()) { std::pop_heap(heap.begin(), heap.end()); heap.back() = it; std::push_heap(heap.begin(), heap.end()); }
        }
        std::sort_heap(heap.begin(), heap.end());
        for (size_t j = 0; j < k; ++j) {
          out_ids[i * k + j] = j < heap.size() ? heap[j].second : 0xFFFFFFFFu;
          out_dist[i * k + j] = j < heap.size() ? heap[j].first : INFINITY;
        }
      }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < std::max(1, nthreads); ++t) th.emplace_back(work);
    for (auto& t : th) t.join();
  };
  switch (dtype) {
    case 0: run(float()); break;
    case 1: run(uint8_t()); break;
    case 2: run(uint16_t()); break;
    case 3: run(uint32_t()); break;
    case 4: run(int32_t()); break;
  }
}

// ---- Rust-std BinaryHeap restatement exposed for unit tests: ops[i] >= 0 pushes (key = vals[i], id = ops[i]);
// ops[i] == -1 pops.  Pop results are appended to out_ids; finally into_sorted_vec ids follow.  Returns count.
uint64_t oracle_rheap_script(const int64_t* ops, const float* vals, uint64_t nops, int mode, int neg, int64_t* out_ids) {
  Heap h(ItemCmp{mode, neg != 0});
  uint64_t o = 0;
  for (uint64_t i = 0; i < nops; ++i) {
    if (ops[i] >= 0) h.push(Item{vals[i], (uint32_t)ops[i]});
    else if (!h.empty()) out_ids[o++] = h.pop().id;
  }
  std::vector<Item> s = h.into_sorted_vec();
  for (const Item& it : s) out_ids[o++] = it.id;
  return o;
}

}  // extern "C"
