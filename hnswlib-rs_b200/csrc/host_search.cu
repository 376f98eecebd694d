// Host search batches (index.h "host searches"): every host entry point's batch is planned into legs, each leg is begun
// and finished on its Index, and the answers are written into the caller's AnswerArrays.  No kernel of its own: a leg
// runs the ordinary query kernels, or for an exact batch the exact scan (aux.cu), through search_host_begin / finish.
//
// A leg is leased, begun, finished and written, and its context released.  Every begun leg is collected, also after
// another leg failed, and a leg whose enqueue failed has its stream synchronised before its context is released.  Who
// runs each step depends on the call:
//   * one leg (an unpartitioned handle, no sharding): the calling thread does everything;
//   * sharded over replicas (synchronous): each leg's worker leases, stages, searches and writes its slice;
//   * partitioned: the calling thread leases the P contexts in partition order, begins all P legs, collects them and merges;
//   * submit / wait: the calling thread begins the legs at submit; at wait the root's leg is collected by the caller and
//     each replica's leg by that replica's worker.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <set>

#include "../../include/hnsw_b200.h"
#include "index.h"
#include "partition.h"

namespace hb {

// ------------------------------------------------------------------------------------------------ worker threads
Worker::Worker() {
  th = std::thread([this] {
    std::unique_lock<std::mutex> lk(m);
    for (;;) {
      cv.wait(lk, [this] { return has_job || quit; });
      if (quit) return;
      auto j = std::move(job);
      has_job = false;
      lk.unlock();
      j();
      lk.lock();
      done = true;
      cv.notify_all();
    }
  });
}
void Worker::submit(std::function<void()> j) {
  std::unique_lock<std::mutex> lk(m);
  job = std::move(j);
  has_job = true;
  done = false;
  cv.notify_all();
}
void Worker::wait() {
  std::unique_lock<std::mutex> lk(m);
  cv.wait(lk, [this] { return done; });
}
Worker::~Worker() {
  {
    std::unique_lock<std::mutex> lk(m);
    quit = true;
    cv.notify_all();
  }
  th.join();
}

void WorkerGroup::resize(size_t n) {
  w_.resize(n);
  for (auto& w : w_)
    if (!w) w.reset(new Worker());
}

int WorkerGroup::run(int n, const std::function<int(int)>& job) {
  DeviceRestore keep;
  std::lock_guard<std::mutex> one(mu);
  std::vector<int> rc(n, 0);
  for (int i = 1; i < n; ++i) {
    int* out = &rc[i];
    w_[i - 1]->submit([=, &job] { *out = job(i); });
  }
  rc[0] = job(0);
  for (int i = 1; i < n; ++i) w_[i - 1]->wait();
  for (int i = 0; i < n; ++i)
    if (rc[i]) return i;
  return -1;
}

// ------------------------------------------------------------------------------------------------ answers
// PointId (level, rank) of internal id `it` of `rx`, hnsw.rs:46; (-1, -1) for an empty slot
static inline void point_id(const Index* rx, uint32_t it, int32_t* pid2) {
  pid2[0] = it != INVALID_ID ? (int32_t)rx->h_level[it] : -1;
  pid2[1] = it != INVALID_ID ? rx->h_rank[it] : -1;
}

// rows [first, first + count) of `out` from one leg's answers `ans` (k slots each, as the kernels left them: the slots
// beyond a query's count hold (~0, +inf, INVALID_ID)), and a radius batch's totals: plain copies
static void put_rows(const AnswerArrays& out, const Index* rx, size_t first, size_t count, size_t k, const HostAnswers& ans) {
  if (count == 0) return;
  memcpy(out.counts + first, ans.counts, count * sizeof(int32_t));
  if (out.total && ans.totals)
    for (size_t i = 0; i < count; ++i) out.total[first + i] = ans.totals[i];
  const size_t o = first * k, tot = count * k;
  if (out.nb) {
    memcpy(out.nb + o, ans.slots, tot * sizeof(NeighbourOut));
    return;
  }
  if (out.ids) {
    uint64_t* ids = out.ids + o;
    for (size_t s = 0; s < tot; ++s) ids[s] = ans.slots[s].origin;
  }
  float* dist = out.dist + o;
  for (size_t s = 0; s < tot; ++s) dist[s] = ans.slots[s].dist;
  if (out.internal) {
    uint32_t* internal = out.internal + o;
    for (size_t s = 0; s < tot; ++s) internal[s] = ans.slots[s].internal;
  }
  if (out.pid) {
    int32_t* pid = out.pid + 2 * o;
    for (size_t s = 0; s < tot; ++s) point_id(rx, ans.slots[s].internal, pid + 2 * s);
  }
}

// queries [first, first + count) of the batch from one leg's answers, each to its row of `out` (out.perm)
static void put_slice(const AnswerArrays& out, const Index* rx, size_t first, size_t count, size_t k, const HostAnswers& a) {
  if (!out.perm) return put_rows(out, rx, first, count, k, a);
  for (size_t i = 0; i < count; ++i)
    put_rows(out, rx, out.perm[first + i], 1, k, {a.slots + i * k, a.counts + i, a.totals ? a.totals + i : nullptr});
}

// slot s of `out` from answer e of index rx, reported with internal id `internal` (a partitioned handle's global rank)
static inline void put_answer(const AnswerArrays& out, size_t s, const Index* rx, const NeighbourOut& e, uint32_t internal) {
  if (out.nb) {
    out.nb[s] = NeighbourOut{e.origin, e.dist, internal};
    return;
  }
  if (out.ids) out.ids[s] = e.origin;
  out.dist[s] = e.dist;
  if (out.internal) out.internal[s] = internal;
  if (out.pid) point_id(rx, e.internal, out.pid + 2 * s);
}

// every query of the batch from the answers of P partition legs, merged by merge_lists, to its row of `out` (out.perm);
// the slots past a query's count are padded with (~0, +inf, INVALID_ID) and PointId (-1, -1).  A radius batch's total is
// the sum of the partitions'.  a[p]: leg p's answers.
static void put_merged(const AnswerArrays& out, const std::vector<Leg>& legs, size_t nq, size_t k,
                       const std::vector<HostAnswers>& a) {
  const int P = (int)legs.size();
  const NeighbourOut pad{~0ull, __builtin_inff(), INVALID_ID};
  int32_t cnt[Partitions::MAX_PARTS];
  for (size_t q = 0; q < nq; ++q) {
    for (int p = 0; p < P; ++p) cnt[p] = a[p].counts[q];
    const size_t o = q * k, row = out.perm ? out.perm[q] : q, w = row * k;
    const size_t total = merge_lists(
        P, k, cnt, [&](int p, int i) { return a[p].slots[o + i].dist; },
        [&](size_t j, int p, int i) {
          const NeighbourOut& e = a[p].slots[o + i];
          put_answer(out, w + j, legs[p].rx, e, (uint32_t)global_rank(p, e.internal, P));
        });
    for (size_t j = total; j < k; ++j) put_answer(out, w + j, nullptr, pad, INVALID_ID);
    out.counts[row] = (int32_t)total;
    if (out.total && a[0].totals) {
      uint64_t sum = 0;
      for (int p = 0; p < P; ++p) sum += a[p].totals[q];
      out.total[row] = sum;
    }
  }
}

// ------------------------------------------------------------------------------------------------ legs
// The legs of an nq-query batch: every query on every partition of a partitioned handle; contiguous shards over the
// handle and its replicas when there are replicas and every device gets a worthwhile share (a stale replica set is
// re-broadcast first); otherwise the whole batch on the handle.
int Index::plan(size_t nq, std::vector<Leg>& legs) {
  if (parts) {
    for (int p = 0; p < parts->count(); ++p) legs.push_back(Leg{parts->part(p), p, 0, nq});
    return 0;
  }
  const size_t ndev = replicas_.size() + 1;
  if (ndev == 1 || nq < 64 * ndev) {
    legs.push_back(Leg{this, 0, 0, nq});
    return 0;
  }
  {
    // one re-broadcast at a time; the copies go stale only under the handle's exclusive lock, which no search overlaps
    std::lock_guard<std::mutex> one(workers_.mu);
    if (replicas_stale_) {
      int r = broadcast_to_replicas();
      if (r) return r;
    }
  }
  const size_t per = (nq + ndev - 1) / ndev;
  for (size_t i = 0; i < ndev; ++i) {
    const size_t first = std::min(nq, i * per);
    legs.push_back(Leg{i ? replicas_[i - 1].get() : this, 0, first, std::min(nq, (i + 1) * per) - first});
  }
  return 0;
}

int Index::resolve(const Restriction& rs, bool exact, const std::vector<int64_t>& sorted, Leg* legs, size_t n,
                   std::vector<std::vector<uint32_t>>& bits, const LabelSets* sets, bool stored) {
  const std::vector<Index*>& hs = holders();
  const int P = (int)hs.size();
  if (rs.kind == Restriction::FILTER_T) {
    bits.resize(P);
    for (int p = 0; p < P; ++p) {
      Index* rx = hs[p];
      if (rx->make_filter_bits(rs.mode, rs.ids, rs.nids, rs.fn, rs.ctx, bits[p])) {
        for (Leg* l = legs; l < legs + n; ++l)
          if (l->rx == rx) l->rc = -1;
        return -1;
      }
    }
  }
  // run u of leg l under `key`, a resident filter, a label set or every point; exact: its slices appended to the plan's
  auto restrict_run = [&](Leg& l, int64_t key, LegPlan::Run& u) {
    if (rs.kind == Restriction::FILTER_T) {
      u.host_bits = bits[l.part].data();
      return 0;
    }
    std::vector<ExactScan>& slices = l.plan.slices;
    u.slice = slices.size();
    int r = 0;
    if (key == EVERY_POINT) {  // graph batches only: an exact batch applies its lists in the scan (prepare_batch)
      u.every = true;
    } else if (rs.kind == Restriction::ROW_LABEL_SETS) {
      u.set = sets->values.data() + sets->off[key];
      u.nset = (uint32_t)(sets->off[key + 1] - sets->off[key]);
      u.lo = sets->range[2 * key];
      u.hi = sets->range[2 * key + 1];
      r = exact ? l.rx->scan_slices(u.set, u.nset, u.lo, u.hi, slices) : 0;
    } else {
      ExactScan list;
      r = filters.use(key, l.part, P, l.rx, &u.bits, exact ? &list : nullptr);
      if (!r && exact) slices.push_back(list);
    }
    u.nslices = slices.size() - u.slice;
    return r;
  };
  // a graph leg with deleted points: its unrestricted rows [0, plain) become one run over every point with the live
  // stop rule, ahead of the leg's other runs
  auto live_run = [](LegPlan& pl) {
    if (pl.exact || !pl.deleted || !pl.plain) return;
    LegPlan::Run u{0, pl.plain};
    u.every = u.live = true;
    pl.runs.push_back(u);
    pl.plain = 0;
  };
  int r = 0;
  for (Leg* l = legs; l < legs + n; ++l) {  // every leg, so that the caller reports the failure it chooses
    LegPlan& pl = l->plan;
    pl.exact = exact;
    // labels, attributes and deleted points: the leg's own, or on a replica its copies of the handle's, made current first
    const Index* src = parts ? l->rx : this;
    if (!stored && l->rx->deleted_on_device(src, &pl.deleted)) {
      r = l->rc = -1;
      continue;
    }
    if (!rs.per_row() && sorted.empty()) {  // every row unrestricted, or one run over every row
      LegPlan::Run u{0, l->count};
      if (rs.kind == Restriction::NONE) {
        pl.plain = l->count;
        live_run(pl);
      } else if (restrict_run(*l, rs.resident, u)) {
        r = l->rc = -1;
      } else {
        pl.runs.push_back(u);
      }
      continue;
    }
    const int64_t* key = sorted.data() + l->first;
    while (pl.plain < l->count && key[pl.plain] == -1) ++pl.plain;
    if (rs.kind == Restriction::ROW_LABEL_SETS && pl.plain < l->count &&
        (l->rx->on_device(&Index::labels, src, &pl.labels) || (rs.qrange && l->rx->on_device(&Index::attrs, src, &pl.attrs)))) {
      r = l->rc = -1;
      continue;
    }
    const size_t restricted = pl.plain;
    live_run(pl);
    for (size_t j = restricted, e; j < l->count; j = e) {  // one run per filter or label set
      for (e = j + 1; e < l->count && key[e] == key[j];) ++e;
      LegPlan::Run u{j, e - j};
      if (restrict_run(*l, key[j], u)) {
        r = l->rc = -1;
        break;
      }
      pl.runs.push_back(u);
    }
  }
  return r;
}

// sort_rows for label sets, or the refusal of the first bad row: the rows copied into one array (a longer row sorted and
// de-duplicated), their indices sorted once, and one walk over them that numbers the distinct (set, range) pairs into
// `sets`.
static std::string label_set_rows(const Restriction& rs, size_t nq, std::vector<size_t>& perm,
                                  std::vector<int64_t>& sorted, LabelSets& sets) {
  std::vector<uint32_t> v;  // row i's set is v[at[i], at[i + 1])
  v.reserve(nq);
  std::vector<size_t> at(nq + 1);
  // key[i]: -1 for {LABEL_NONE} (the only accepted set that holds it), 0 for the empty set, else 1 + the set's smallest
  // value; rows of one key are ordered by the rest of their sets, which only rows of several labels have (`longer`),
  // then by their ranges
  std::vector<int64_t> key(nq);
  // row i's range, biased: (0, ~0) for none, which sorts first; else lo >= 1, and (1, 0) for every empty one
  std::vector<uint64_t> rg(2 * nq);
  bool longer = false;
  for (size_t i = 0; i < nq; ++i) {
    const uint64_t lo = rs.qset_off[i], hi = rs.qset_off[i + 1];
    if (hi < lo)
      return "label set " + std::to_string(i) + ": qset_off[" + std::to_string(i + 1) + "] = " + std::to_string(hi) +
             " is below qset_off[" + std::to_string(i) + "] = " + std::to_string(lo);
    at[i] = v.size();
    v.insert(v.end(), rs.qset + lo, rs.qset + hi);
    if (hi - lo > 1) {
      std::sort(v.begin() + at[i], v.end());
      v.erase(std::unique(v.begin() + at[i], v.end()), v.end());
      if (v.size() - at[i] > 1 && v.back() == LABEL_NONE)
        return "label set " + std::to_string(i) + " holds LABEL_NONE together with another label";
      longer |= v.size() - at[i] > 1;
    }
    key[i] = at[i] == v.size() ? 0 : v[at[i]] == LABEL_NONE ? -1 : 1 + (int64_t)v[at[i]];
    const int64_t* q = rs.qrange ? rs.qrange + 2 * i : nullptr;
    uint64_t blo = 0, bhi = ~0ull;
    if (q && (q[0] != INT64_MIN || q[1] != INT64_MAX)) {
      blo = std::max<uint64_t>(attr_bias(q[0]), 1);  // ATTR_NONE is no value: a range never admits a point without one
      bhi = attr_bias(q[1]);
      if (blo > bhi) blo = 1, bhi = 0;
    }
    rg[2 * i] = blo;
    rg[2 * i + 1] = bhi;
  }
  at[nq] = v.size();
  auto less = [&](size_t a, size_t b) {
    if (key[a] != key[b]) return key[a] < key[b];
    if (longer && key[a] > 0) {
      const auto a0 = v.begin() + at[a] + 1, a1 = v.begin() + at[a + 1], b0 = v.begin() + at[b] + 1, b1 = v.begin() + at[b + 1];
      if (std::lexicographical_compare(a0, a1, b0, b1)) return true;
      if (std::lexicographical_compare(b0, b1, a0, a1)) return false;
    }
    return std::make_pair(rg[2 * a], rg[2 * a + 1]) < std::make_pair(rg[2 * b], rg[2 * b + 1]);
  };
  perm.resize(nq);
  std::iota(perm.begin(), perm.end(), (size_t)0);
  std::stable_sort(perm.begin(), perm.end(), less);
  sorted.resize(nq);
  sets.values.clear();
  sets.off.assign(1, 0);
  sets.range.clear();
  for (size_t j = 0; j < nq; ++j) {
    const size_t i = perm[j];
    if (key[i] == -1 && rg[2 * i] == 0) {  // every point
      sorted[j] = -1;
      continue;
    }
    if (j == 0 || less(perm[j - 1], i)) {  // a (set, range) the sorted rows have not had yet
      sets.values.insert(sets.values.end(), v.begin() + at[i], v.begin() + at[i + 1]);
      sets.off.push_back(sets.values.size());
      sets.range.insert(sets.range.end(), {rg[2 * i], rg[2 * i + 1]});
    }
    sorted[j] = (int64_t)sets.off.size() - 2;
  }
  return {};
}

// Every filter is checked on every partition before anything runs, so that a bad entry refuses the whole call, named by
// its first position.  The sort is stable: rows of one filter keep their order, and -1 (no filter) sorts first.
int Index::sort_rows(const Restriction& rs, size_t nq, std::vector<size_t>& perm, std::vector<int64_t>& sorted,
                     LabelSets& sets) {
  if (rs.kind == Restriction::ROW_LABEL_SETS) {
    const std::string e = label_set_rows(rs, nq, perm, sorted, sets);
    return e.empty() ? 0 : fail(e);
  }
  const std::vector<Index*>& hs = holders();
  const int P = (int)hs.size();
  const int64_t* fid = rs.filters;
  std::set<int64_t> checked;
  for (size_t i = 0; i < nq; ++i) {
    if (fid[i] == -1 || checked.count(fid[i])) continue;
    for (int p = 0; p < P; ++p) {
      const uint32_t* bits = nullptr;
      if (filters.use(fid[i], p, P, hs[p], &bits))
        return fail("filters[" + std::to_string(i) + "] = " + std::to_string(fid[i]) + ": " + hs[p]->err());
    }
    checked.insert(fid[i]);
  }
  perm.resize(nq);
  std::iota(perm.begin(), perm.end(), (size_t)0);
  std::stable_sort(perm.begin(), perm.end(), [&](size_t a, size_t b) { return fid[a] < fid[b]; });
  sorted.resize(nq);
  for (size_t j = 0; j < nq; ++j) sorted[j] = fid[perm[j]];
  return 0;
}

// Row i's list is copied, sorted and de-duplicated (as label_set_rows treats a set) after its ranks are checked.  The
// ranks are this Index's: a partitioned handle's global ones, split per partition by leg_rows.
int Index::exclusion_lists(const Exclusions& x, size_t nq, Ticket& t) {
  const uint64_t have = nb_point();
  t.xrows.resize(nq);
  t.xids.clear();
  for (size_t i = 0; i < nq; ++i) {
    const uint64_t lo = x.off[i], hi = x.off[i + 1];
    if (hi < lo)
      return fail("excluded list " + std::to_string(i) + ": qx_off[" + std::to_string(i + 1) + "] = " + std::to_string(hi) +
                  " is below qx_off[" + std::to_string(i) + "] = " + std::to_string(lo));
    for (uint64_t j = lo; j < hi; ++j)
      if (x.ids[j] >= have)
        return fail("excluded list " + std::to_string(i) + ": qx[" + std::to_string(j) + "] = " + std::to_string(x.ids[j]) +
                    " is not below nb_point = " + std::to_string(have));
    const size_t at = t.xids.size();
    t.xids.insert(t.xids.end(), x.ids + lo, x.ids + hi);  // below nb_point, so below 2^32
    if (hi - lo > 1) {
      std::sort(t.xids.begin() + at, t.xids.end());
      t.xids.erase(std::unique(t.xids.begin() + at, t.xids.end()), t.xids.end());
    }
    if (t.xids.size() > UINT32_MAX) return fail("the excluded lists hold more than 2^32 - 1 distinct ids in all");
    t.xrows[i] = ExcludedRow{(uint32_t)at, (uint32_t)(t.xids.size() - at)};
  }
  return 0;
}

int Index::admitted(const Restriction& rs, int64_t key, const LabelSets& sets, int p, size_t* count) {
  Index* rx = holders()[p];
  if (rs.kind == Restriction::RESIDENT) return filters.admitted(rs.resident, p, (int)holders().size(), rx, count);
  if (rs.kind != Restriction::ROW_LABEL_SETS || key < 0) {
    *count = rx->n;
    return 0;
  }
  std::vector<ExactScan> slices;
  const size_t at = sets.off[key];
  if (int r = rx->scan_slices(sets.values.data() + at, sets.off[key + 1] - at, sets.range[2 * key], sets.range[2 * key + 1],
                              slices))
    return r;
  *count = 0;
  for (const ExactScan& x : slices) *count += x.n;
  return 0;
}

// The rows sorted as a search sorts them, so that each distinct key is counted once per holder
int Index::count_admitted(const Restriction& rs, size_t nq, uint64_t* out) {
  std::vector<size_t> perm;
  std::vector<int64_t> sorted;
  LabelSets sets;
  int r;
  if (rs.per_row() && (r = sort_rows(rs, nq, perm, sorted, sets))) return r;
  std::vector<uint64_t> c(nq, 0);
  for (int p = 0; p < (int)holders().size(); ++p) {
    size_t n = 0;
    for (size_t j = 0; j < nq; ++j) {
      const int64_t key = sorted.empty() ? -1 : sorted[j];
      if ((j == 0 || (!sorted.empty() && key != sorted[j - 1])) && (r = admitted(rs, key, sets, p, &n)))
        return holder_fail(p, r);
      c[perm.empty() ? j : perm[j]] += n;
    }
  }
  std::copy(c.begin(), c.end(), out);
  return 0;
}

// Row j of leg l takes the exact scan when the scan can hold its k' keys (k, plus 1 with exclude_self) at this dimension
// and c^2 <= GAMMA n e D, in 128-bit integers: c the points its restriction admits on the leg's holder, n the points
// stored there, e = max(ef, k') the ef the graph search runs at, D = 2 M the layer-0 list capacity.  A graph search over a
// fraction s = c / n of the points reads about e D / s rows, the exact scan c rows: the two meet at c^2 = GAMMA n e D.
// The counts are the holder's, so that a replica's leg decides as the handle does.
int Index::split_legs(Ticket& t, const std::vector<int64_t>& sorted) {
  const HostBatch& b = t.b;
  const size_t kq = b.k + (b.in.skip ? 1 : 0);
  t.exact.assign(b.nq, 0);
  int r = 0;
  for (Leg& l : t.legs) {
    Index* cx = holders()[l.part];
    // exact_shape's least shape; a k' of more keys than the budget has bytes never fits (and stays within int)
    const bool fits = kq <= SMEM_BUDGET && exact_layout(cx->row_bytes / 16, (int)kq, 1, 1, 2).bytes <= SMEM_BUDGET;
    const unsigned __int128 bound =
        (unsigned __int128)HNSW_B200_PLANNED_GAMMA * cx->n * std::max(b.ef, kq) * (2 * (unsigned __int128)cx->M);
    LegSplit& s = l.split;
    s.on = true;
    size_t c = 0;
    for (size_t j = 0; j < l.count; ++j) {
      const int64_t key = sorted.empty() ? -1 : sorted[l.first + j];
      if ((j == 0 || (!sorted.empty() && key != sorted[l.first + j - 1])) &&
          (l.rc = admitted(b.restriction, key, t.sets, l.part, &c)))
        break;
      const bool exact = fits && (unsigned __int128)c * c <= bound;
      s.rows[exact].push_back(j);
      t.exact[l.first + j] += exact;
    }
    for (int e = 0; e < 2 && !l.rc; ++e) {  // the exact part reads a graph batch's EVERY_POINT rows as unrestricted
      if (s.rows[e].empty()) continue;
      std::vector<int64_t> keys;
      if (!sorted.empty())
        for (size_t j : s.rows[e]) keys.push_back(e && sorted[l.first + j] == EVERY_POINT ? -1 : sorted[l.first + j]);
      Leg part{l.rx, l.part, 0, s.rows[e].size()};
      if (resolve(b.restriction, e == 1, keys, &part, 1, t.bits, &t.sets)) l.rc = part.rc;
      s.plan[e] = std::move(part.plan);
    }
    if (l.rc) r = -1;
  }
  return r;
}

// The handle's error for the first failed leg of legs[0, n) (0 if none failed): in leg order, or the replicas' before the
// root's (replicas_first, the synchronous sharded search's order).  A partition's and a replica's message name it.
int Index::legs_fail(const Leg* legs, size_t n, bool replicas_first) {
  for (size_t j = 0; j < n; ++j) {
    const Leg& l = legs[replicas_first ? (j + 1) % n : j];
    if (!l.rc) continue;
    if (l.rx == this) return l.rc;
    if (parts) return parts->fail(l.part, l.rx->err());
    return fail("device " + std::to_string(l.rx->device) + ": " + l.rx->err());
  }
  return 0;
}

// The batch's rows in sorted-row order (row j: caller row perm[j]): every present column copied in that order into
// `store`, flat queries as row pointers into them (q_bytes apart), skip still the ids when it was, and the excluded ids
// where they were
static HostRows sorted_rows(const HostRows& in, const std::vector<size_t>& perm, size_t q_bytes,
                            std::vector<unsigned char>& store) {
  const size_t nq = perm.size();
  // room for every column, 8-byte ones first
  store.resize(nq * (sizeof(void*) + 2 * sizeof(uint64_t) + sizeof(ExcludedRow) + sizeof(float)));
  unsigned char* at = store.data();
  auto column = [&](auto value) {  // the next column of `store`: row j holds value(perm[j])
    unsigned char* c = at;
    for (size_t j = 0; j < nq; ++j, at += sizeof(value(0))) {
      const auto v = value(perm[j]);
      memcpy(at, &v, sizeof(v));
    }
    return c;
  };
  HostRows s;
  if (in.queries || in.rows)
    s.rows = (const void* const*)column([&](size_t i) {
      return in.rows ? in.rows[i] : (const void*)((const char*)in.queries + i * q_bytes);
    });
  if (in.qids) s.qids = (const uint64_t*)column([&](size_t i) { return in.qids[i]; });
  if (in.skip) s.skip = in.skip == in.qids ? s.qids : (const uint64_t*)column([&](size_t i) { return in.skip[i]; });
  if (in.excluded) s.excluded = (const ExcludedRow*)column([&](size_t i) { return in.excluded[i]; });
  if (in.radius) s.radius = (const float*)column([&](size_t i) { return in.radius[i]; });
  s.excluded_ids = in.excluded_ids;
  s.nexcluded_ids = in.nexcluded_ids;
  return s;
}

// Leg l's rows: rows [l.first, l.first + l.count) of the batch's, flat queries q_bytes apart.  A batch by stored point on
// a partitioned handle (P partitions; 0: none) runs on its rows gathered into the queries, and a row leaves out its
// point only on the partition that holds it, as that partition's local id (made in `local`).  On a partitioned handle
// a row's excluded points are those of its list that the leg's partition holds, as its local ids (made in `xrows` and
// `xids`; the list ascends, and so does its part: local id g / P of global rank g).
static HostRows leg_rows(const HostRows& in, const Leg& l, size_t q_bytes, uint64_t P, std::vector<uint64_t>& local,
                         std::vector<ExcludedRow>& xrows, std::vector<uint32_t>& xids) {
  const size_t j = l.first;
  HostRows s{in.queries ? (const char*)in.queries + j * q_bytes : nullptr, in.rows ? in.rows + j : nullptr,
             in.qids ? in.qids + j : nullptr, in.skip ? in.skip + j : nullptr, in.radius ? in.radius + j : nullptr,
             in.excluded ? in.excluded + j : nullptr, in.excluded_ids, in.nexcluded_ids};
  if (P && s.excluded) {
    xrows.resize(l.count);
    for (size_t i = 0; i < l.count; ++i) {
      const ExcludedRow x = s.excluded[i];
      const size_t at = xids.size();
      for (uint32_t e = 0; e < x.n; ++e) {
        const Placed g = place(s.excluded_ids[x.off + e], P);
        if (g.part == l.part) xids.push_back((uint32_t)g.local);
      }
      xrows[i] = ExcludedRow{(uint32_t)at, (uint32_t)(xids.size() - at)};
    }
    s.excluded = xrows.data();
    s.excluded_ids = xids.data();
    s.nexcluded_ids = xids.size();
  }
  if (P && s.qids) {
    if (s.skip) {
      local.resize(l.count);
      for (size_t i = 0; i < l.count; ++i) {
        const Placed at = place(s.skip[i], P);
        local[i] = at.part == l.part ? at.local : ~0ull;
      }
      s.skip = local.data();
    }
    s.qids = nullptr;
  }
  return s;
}

void Index::begin_leg(const HostBatch& b, Leg& l) {
  if (l.ctx < 0) l.ctx = l.rx->acquire_ctx();
  LegSplit& s = l.split;
  if (s.on) {
    s.running = s.rows[0].empty() && !s.rows[1].empty();
    s.slots.resize(l.count * b.k);
    s.counts.resize(l.count);
  }
  start_leg(b, l);
}

// A planned part runs on its rows gathered from the leg's (sorted_rows), so that its answers are its rows' in order
void Index::start_leg(const HostBatch& b, Leg& l) {
  std::vector<uint64_t> local;
  std::vector<ExcludedRow> xrows;
  std::vector<uint32_t> xids;
  std::vector<unsigned char> part;
  const size_t q_bytes = (size_t)b.d * es;
  const HostRows in = leg_rows(b.in, l, q_bytes, parts ? parts->count() : 0, local, xrows, xids);
  const LegSplit& s = l.split;
  if (s.on) {
    const std::vector<size_t>& rows = s.rows[s.running];
    l.rc = l.rx->search_host_begin(l.ctx, sorted_rows(in, rows, q_bytes, part), rows.size(), b.d, b.k, b.ef,
                                   s.plan[s.running]);
  } else {
    l.rc = l.rx->search_host_begin(l.ctx, in, l.count, b.d, b.k, b.ef, l.plan);
  }
  l.begun = l.rc == 0;
}

// A planned leg: each part's answers scattered to its rows, then the exact part begun and collected after the graph
// part, on the same context (a second lease while holding one could deadlock two callers).  Only the pending part is
// re-run when its visited tables overflow (search_host_finish), so an exact row runs and is written once.
HostAnswers Index::collect_leg(const HostBatch& b, Leg& l) {
  HostAnswers a = l.rx->search_host_finish(l.ctx);
  LegSplit& s = l.split;
  if (!s.on) return a;
  for (;;) {
    if (a.rc) return a;
    const std::vector<size_t>& rows = s.rows[s.running];
    for (size_t i = 0; i < rows.size(); ++i) {
      s.counts[rows[i]] = a.counts[i];
      memcpy(s.slots.data() + rows[i] * b.k, a.slots + i * b.k, b.k * sizeof(NeighbourOut));
    }
    if (s.running == 1 || s.rows[1].empty()) break;
    s.running = 1;
    start_leg(b, l);
    if (l.rc) return HostAnswers{nullptr, nullptr, nullptr, l.rc};
    a = l.rx->search_host_finish(l.ctx);
  }
  return HostAnswers{s.slots.data(), s.counts.data(), nullptr, 0};
}

void Index::release_leg(Leg& l) {
  if (l.ctx < 0) return;
  if (!l.begun && l.rc) {  // the enqueue failed: nothing of it may still run once the context is released
    cudaSetDevice(l.rx->device);
    cudaStreamSynchronize(l.rx->ctx(l.ctx).stream);
  }
  l.rx->release_ctx(l.ctx);
  l.ctx = -1;
}

// collects a leg, writes its slice of b.out and releases its context
int Index::end_leg(Leg& l, const HostBatch& b) {
  if (l.begun) {
    const HostAnswers a = collect_leg(b, l);
    l.rc = a.rc;
    if (!l.rc) put_slice(b.out, l.rx, l.first, l.count, b.k, a);
  }
  release_leg(l);
  return l.rc;
}

// ------------------------------------------------------------------------------------------------ batches
// The batch `call` planned into t's legs, each with its plan; t.b is the batch as the legs run it.  A per-row
// restriction: the batch is planned over the rows sorted by filter or label set (sorted_rows), and each answer goes
// back to its caller's row.  A batch by stored point on a partitioned handle has its rows gathered from their
// partitions first, since no device reads another partition's store, and is then searched as host queries.  Excluded
// points ride with their rows; in a graph batch the unrestricted rows that exclude points are moved from the
// unrestricted prefix into a run over every point, after the rows that stay there.  A leg that could not have its plan
// is reported in leg order, or the replicas' first.
int Index::prepare_batch(const HostBatch& call, Ticket& t, bool replicas_first) {
  if (parts && dim != 0 && call.d != dim) return fail("query length differs from the index dimension");
  int r;
  HostBatch& b = t.b;
  b = call;
  if (parts && call.in.qids) {
    t.gathered.resize(call.nq * (size_t)dim * es);
    if ((r = get_vectors(call.in.qids, call.nq, t.gathered.data()))) return r;
    b.in.queries = t.gathered.data();
  }
  const Restriction& rs = call.restriction;
  if (call.excluded.off) {
    if ((r = exclusion_lists(call.excluded, call.nq, t))) return r;
    b.in.excluded = t.xrows.data();
    b.in.excluded_ids = t.xids.data();
    b.in.nexcluded_ids = t.xids.size();
  }
  const bool every = call.excluded.off && !call.exact && (rs.kind == Restriction::NONE || rs.per_row());
  std::vector<int64_t> sorted;
  if (rs.per_row() || every) {
    if (rs.per_row() && (r = sort_rows(rs, call.nq, t.perm, sorted, t.sets))) return r;
    if (!rs.per_row()) {
      t.perm.resize(call.nq);
      std::iota(t.perm.begin(), t.perm.end(), (size_t)0);
      sorted.assign(call.nq, -1);
    }
    if (every) {
      size_t plain = 0;
      while (plain < call.nq && sorted[plain] == -1) ++plain;
      const auto listed = std::stable_partition(t.perm.begin(), t.perm.begin() + plain,
                                                [&](size_t i) { return t.xrows[i].n == 0; });
      std::fill(sorted.begin() + (listed - t.perm.begin()), sorted.begin() + plain, EVERY_POINT);
    }
    b.in = sorted_rows(b.in, t.perm, (size_t)b.d * es, t.rows);
    b.out.perm = t.perm.data();
  }
  if ((r = plan(b.nq, t.legs))) return r;
  if (b.planned ? split_legs(t, sorted)
                : resolve(b.restriction, b.exact, sorted, t.legs.data(), t.legs.size(), t.bits, &t.sets, b.stored))
    return legs_fail(t.legs.data(), t.legs.size(), replicas_first && !parts);
  return 0;
}

// A planned batch writes each row's exact count (out.exact) once every leg succeeded
int Index::search_batch(const HostBatch& call) {
  if (call.nq == 0) return 0;
  Ticket t;
  int r;
  if ((r = prepare_batch(call, t, true)) || (r = run_batch(t))) return r;
  const AnswerArrays& out = t.b.out;
  if (out.exact)
    for (size_t j = 0; j < t.exact.size(); ++j) out.exact[out.perm ? out.perm[j] : j] = t.exact[j];
  return 0;
}

int Index::run_batch(Ticket& t) {
  const HostBatch& b = t.b;
  std::vector<Leg>& legs = t.legs;
  const int n = (int)legs.size();
  const bool sharded = n > 1 && !parts;
  if (n == 1 && !parts) {
    begin_leg(b, legs[0]);
    return end_leg(legs[0], b);
  }
  if (sharded) {  // leg i on worker i - 1
    workers_.run(n, [&](int i) {
      begin_leg(b, legs[i]);
      return end_leg(legs[i], b);
    });
    return legs_fail(legs.data(), n, true);
  }
  // partitioned: the P searches run at once, on one device or several; the answers stay in the leased contexts until
  // the merge is done.  A failed enqueue is reported ahead of any collection failure.
  DeviceRestore keep;
  for (Leg& l : legs) l.ctx = l.rx->acquire_ctx();
  int bad = -1;
  for (int p = 0; p < n && bad < 0; ++p) {
    begin_leg(b, legs[p]);
    if (legs[p].rc) bad = p;
  }
  std::vector<HostAnswers> a(n);
  for (int p = 0; p < n; ++p) {
    if (legs[p].begun) {
      a[p] = collect_leg(b, legs[p]);
      legs[p].rc = a[p].rc;
    }
    if (legs[p].rc && bad < 0) bad = p;
  }
  if (bad < 0) put_merged(b.out, legs, b.nq, b.k, a);
  for (Leg& l : legs) release_leg(l);
  return bad < 0 ? 0 : legs_fail(&legs[bad], 1, false);
}

int64_t Index::submit_batch(const HostBatch& call) {
  DeviceRestore keep;  // the legs switch to their devices on the calling thread
  Ticket t;
  int r;
  if ((r = prepare_batch(call, t, false))) return r;
  int bad = -1;
  for (size_t i = 0; i < t.legs.size() && bad < 0; ++i) {  // one after the other, on the calling thread
    begin_leg(t.b, t.legs[i]);
    if (t.legs[i].rc) bad = (int)i;
  }
  if (bad >= 0) {
    for (Leg& l : t.legs) end_leg(l, t.b);  // collect what was enqueued before the failure
    return legs_fail(&t.legs[bad], 1, false);
  }
  pending_.fetch_add(1);
  return park_ticket(std::move(t));
}

int Index::finish_batch(Ticket& t) {
  if (t.legs.size() == 1) return end_leg(t.legs[0], t.b);
  workers_.run((int)t.legs.size(), [&](int i) { return end_leg(t.legs[i], t.b); });
  return legs_fail(t.legs.data(), t.legs.size(), false);
}

}  // namespace hb
