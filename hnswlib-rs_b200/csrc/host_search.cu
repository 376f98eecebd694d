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

// rows [first, first + count) of `out` from one leg's answers (k slots each, as the kernels left them: the slots beyond a
// query's count hold (~0, +inf, INVALID_ID)): plain copies
static void put_rows(const AnswerArrays& out, const Index* rx, size_t first, size_t count, size_t k, const NeighbourOut* a,
                     const int32_t* cnts) {
  if (count == 0) return;
  memcpy(out.counts + first, cnts, count * sizeof(int32_t));
  const size_t o = first * k, tot = count * k;
  if (out.nb) {
    memcpy(out.nb + o, a, tot * sizeof(NeighbourOut));
    return;
  }
  if (out.ids) {
    uint64_t* ids = out.ids + o;
    for (size_t s = 0; s < tot; ++s) ids[s] = a[s].origin;
  }
  float* dist = out.dist + o;
  for (size_t s = 0; s < tot; ++s) dist[s] = a[s].dist;
  if (out.internal) {
    uint32_t* internal = out.internal + o;
    for (size_t s = 0; s < tot; ++s) internal[s] = a[s].internal;
  }
  if (out.pid) {
    int32_t* pid = out.pid + 2 * o;
    for (size_t s = 0; s < tot; ++s) point_id(rx, a[s].internal, pid + 2 * s);
  }
}

// queries [first, first + count) of the batch from one leg's answers, each to its row of `out` (out.perm)
static void put_slice(const AnswerArrays& out, const Index* rx, size_t first, size_t count, size_t k, const NeighbourOut* a,
                      const int32_t* cnts) {
  if (!out.perm) return put_rows(out, rx, first, count, k, a, cnts);
  for (size_t i = 0; i < count; ++i) put_rows(out, rx, out.perm[first + i], 1, k, a + i * k, cnts + i);
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
// the slots past a query's count are padded with (~0, +inf, INVALID_ID) and PointId (-1, -1)
static void put_merged(const AnswerArrays& out, const std::vector<Leg>& legs, size_t nq, size_t k,
                       const std::vector<const NeighbourOut*>& a, const std::vector<const int32_t*>& c) {
  const int P = (int)legs.size();
  const NeighbourOut pad{~0ull, __builtin_inff(), INVALID_ID};
  int32_t cnt[Partitions::MAX_PARTS];
  for (size_t q = 0; q < nq; ++q) {
    for (int p = 0; p < P; ++p) cnt[p] = c[p][q];
    const size_t o = q * k, row = out.perm ? out.perm[q] : q, w = row * k;
    const size_t total = merge_lists(
        P, k, cnt, [&](int p, int i) { return a[p][o + i].dist; },
        [&](size_t j, int p, int i) {
          const NeighbourOut& e = a[p][o + i];
          put_answer(out, w + j, legs[p].rx, e, e.internal * (uint32_t)P + (uint32_t)p);
        });
    for (size_t j = total; j < k; ++j) put_answer(out, w + j, nullptr, pad, INVALID_ID);
    out.counts[row] = (int32_t)total;
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

int Index::resolve_filter(const FilterArg& f, bool exact, Leg* legs, size_t n, std::vector<std::vector<uint32_t>>& bits) {
  const int P = parts ? parts->count() : 1;
  int r = 0;
  if (f.mode) {
    bits.resize(P);
    for (int p = 0; p < P; ++p) {
      Index* rx = parts ? parts->part(p) : this;
      if (rx->make_filter_bits(f.mode, f.ids, f.nids, f.fn, f.ctx, bits[p])) {
        for (Leg* l = legs; l < legs + n; ++l)
          if (l->rx == rx) l->rc = -1;
        return -1;
      }
    }
    for (size_t i = 0; i < n; ++i) legs[i].host_bits = bits[legs[i].part].data();
  }
  for (Leg* l = legs; f.resident && l < legs + n; ++l)  // every leg, so that the caller reports the failure it chooses
    if (filters.use(*f.resident, l->part, P, l->rx, &l->dev_bits, exact ? &l->scan : nullptr)) r = l->rc = -1;
  return r;
}

// Every filter is checked on every partition before anything runs, so that a bad entry refuses the whole call, named by
// its first position.  The sort is stable: rows of one filter keep their order, and -1 (no filter) sorts first.  A label
// needs no check; LABEL_NONE sorts first as -1.
int Index::sort_per_query(const HostBatch& b, std::vector<size_t>& perm, std::vector<int64_t>& sorted) {
  const int P = parts ? parts->count() : 1;
  const size_t nq = b.nq;
  std::vector<int64_t> key;
  const int64_t* fid = b.per_query;
  if (b.labels) {
    key.resize(nq);
    for (size_t i = 0; i < nq; ++i) key[i] = b.labels[i] == LABEL_NONE ? -1 : (int64_t)b.labels[i];
    fid = key.data();
  }
  std::set<int64_t> checked;
  for (size_t i = 0; !b.labels && i < nq; ++i) {
    if (fid[i] == -1 || checked.count(fid[i])) continue;
    for (int p = 0; p < P; ++p) {
      Index* rx = parts ? parts->part(p) : this;
      const uint32_t* bits = nullptr;
      if (filters.use(fid[i], p, P, rx, &bits))
        return fail("filters[" + std::to_string(i) + "] = " + std::to_string(fid[i]) + ": " + rx->err());
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

int Index::resolve_per_query(const std::vector<int64_t>& sorted, bool labels, bool exact, Leg* legs, size_t n) {
  const int P = parts ? parts->count() : 1;
  int r = 0;
  for (Leg* l = legs; l < legs + n; ++l) {  // every leg, so that the caller reports the failure it chooses
    LegFilters& q = l->pq;
    const int64_t* f = sorted.data() + l->first;
    q.on = true;
    while (q.plain < l->count && f[q.plain] == -1) ++q.plain;
    // labels: the leg's own, or on a replica its copy of the handle's, made current first.  The graph search reads the
    // label array and each row's label; the exact scan, a slice per label of the leg's CSR.
    if (labels && q.plain < l->count && l->rx->labels_on_device(parts ? l->rx : this, &q.labels)) {
      r = l->rc = -1;
      continue;
    }
    if (exact && q.plain) q.groups.push_back(ExactGroup{0, q.plain, ExactScan()});
    for (size_t j = q.plain, e; j < l->count; j = e) {  // one run of rows per filter or label
      for (e = j + 1; e < l->count && f[e] == f[j];) ++e;
      ExactScan s;
      const uint32_t* bits = nullptr;
      if (labels) {
        if (!exact) {
          q.sel.insert(q.sel.end(), e - j, (uint32_t)f[j]);
          continue;
        }
        if (l->rx->label_scan((uint32_t)f[j], &s)) {
          r = l->rc = -1;
          break;
        }
      } else if (filters.use(f[j], l->part, P, l->rx, &bits, exact ? &s : nullptr)) {
        r = l->rc = -1;
        break;
      }
      if (exact) {
        q.groups.push_back(ExactGroup{j, e - j, s});
      } else {
        q.sel.insert(q.sel.end(), e - j, (uint32_t)q.table.size());
        q.table.push_back(bits);
      }
    }
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

void Index::begin_leg(const HostBatch& b, Leg& l) {
  if (l.ctx < 0) l.ctx = l.rx->acquire_ctx();
  const void* q = b.rows ? nullptr : (const char*)b.queries + l.first * (size_t)b.d * es;
  l.rc = l.rx->search_host_begin(l.ctx, q, b.rows ? b.rows + l.first : nullptr, l.count, b.d, b.k, b.ef, l.host_bits,
                                 l.dev_bits, b.exact ? &l.scan : nullptr, l.pq.on ? &l.pq : nullptr);
  l.begun = l.rc == 0;
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

// collects a leg, writes its slice of `out` and releases its context
int Index::end_leg(Leg& l, size_t k, const AnswerArrays& out) {
  if (l.begun) {
    const NeighbourOut* a = nullptr;
    const int32_t* c = nullptr;
    l.rc = l.rx->search_host_finish(l.ctx, &a, &c);
    if (!l.rc) put_slice(out, l.rx, l.first, l.count, k, a, c);
  }
  release_leg(l);
  return l.rc;
}

// ------------------------------------------------------------------------------------------------ batches
int Index::search_batch(const HostBatch& call) {
  if (call.nq == 0) return 0;
  if (parts && dim != 0 && call.d != dim) return fail("query length differs from the index dimension");
  int r;
  // a filter or a label per query: the batch is planned over the rows sorted by filter or label, gathered through row
  // pointers, and each answer goes back to its caller's row
  HostBatch b = call;
  std::vector<size_t> perm;
  std::vector<const void*> rows;
  std::vector<int64_t> sorted;
  const bool per_row = call.per_query || call.labels;
  if (per_row) {
    if ((r = sort_per_query(call, perm, sorted))) return r;
    rows.resize(call.nq);
    for (size_t j = 0; j < call.nq; ++j)
      rows[j] = call.rows ? call.rows[perm[j]] : (const char*)call.queries + perm[j] * (size_t)call.d * es;
    b.rows = rows.data();
    b.out.perm = perm.data();
  }
  std::vector<Leg> legs;
  std::vector<std::vector<uint32_t>> bits;
  if ((r = plan(b.nq, legs))) return r;
  const int n = (int)legs.size();
  const bool sharded = n > 1 && !parts;
  if (per_row ? resolve_per_query(sorted, b.labels != nullptr, b.exact, legs.data(), n)
              : resolve_filter(b.filter, b.exact, legs.data(), n, bits))
    return legs_fail(legs.data(), n, sharded);
  if (n == 1 && !parts) {
    begin_leg(b, legs[0]);
    return end_leg(legs[0], b.k, b.out);
  }
  if (sharded) {  // leg i on worker i - 1
    workers_.run(n, [&](int i) {
      begin_leg(b, legs[i]);
      return end_leg(legs[i], b.k, b.out);
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
  std::vector<const NeighbourOut*> a(n);
  std::vector<const int32_t*> c(n);
  for (int p = 0; p < n; ++p) {
    if (legs[p].begun) legs[p].rc = legs[p].rx->search_host_finish(legs[p].ctx, &a[p], &c[p]);
    if (legs[p].rc && bad < 0) bad = p;
  }
  if (bad < 0) put_merged(b.out, legs, b.nq, b.k, a, c);
  for (Leg& l : legs) release_leg(l);
  return bad < 0 ? 0 : legs_fail(&legs[bad], 1, false);
}

int64_t Index::submit_batch(const HostBatch& b) {
  DeviceRestore keep;  // the legs switch to their devices on the calling thread
  Ticket t;
  t.k = b.k;
  t.out = b.out;
  std::vector<std::vector<uint32_t>> bits;
  int r;
  if ((r = plan(b.nq, t.legs))) return r;
  if (resolve_filter(b.filter, b.exact, t.legs.data(), t.legs.size(), bits)) return legs_fail(t.legs.data(), t.legs.size(), false);
  int bad = -1;
  for (size_t i = 0; i < t.legs.size() && bad < 0; ++i) {  // one after the other, on the calling thread
    begin_leg(b, t.legs[i]);
    if (t.legs[i].rc) bad = (int)i;
  }
  if (bad >= 0) {
    for (Leg& l : t.legs) end_leg(l, t.k, t.out);  // collect what was enqueued before the failure
    return legs_fail(&t.legs[bad], 1, false);
  }
  pending_.fetch_add(1);
  return park_ticket(std::move(t));
}

int Index::finish_batch(Ticket& t) {
  if (t.legs.size() == 1) return end_leg(t.legs[0], t.k, t.out);
  workers_.run((int)t.legs.size(), [&](int i) { return end_leg(t.legs[i], t.k, t.out); });
  return legs_fail(t.legs.data(), t.legs.size(), false);
}

}  // namespace hb
