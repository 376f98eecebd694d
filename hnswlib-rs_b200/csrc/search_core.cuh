// search_layer on a warp: the ef-bounded best-first expansion of one layer.
// Restates /root/reference/src/hnsw.rs:922-1064 (search_layer) for one warp that owns the whole
// queue state of one query; used by the query kernel (search.cu) and the insert kernel (build.cu).
// Also the per-query scaffold the query kernels share: the work counter (all four), the upper-layer descent and the counter
// flush (the warp kernels search.cu, filter.cu, search_std.cu), the answer write-out (all but the filtered kernel, which
// compacts its answers).  The scaffold functions (and Visited) take the caller's lane, because the lean kernel
// (search_lean.cuh) pins its lane; a layer search (search_layer here, search_layer_filtered in filter.cu) is a warp kernel's
// own loop, not scaffold, and takes the lane once at its top.
#pragma once
#include "kernels.h"

namespace hb {

struct WarpSmem {
  uint4* q4;          // query row, d4 16-byte chunks (zero padded)
  uint64_t* wbuf;     // queue keys, capacity >= ef
  uint32_t* cand_id;  // one chunk of neighbours: 32 ids
  float* cand_d;      // and their distances
};

// One chunk of up to 32 candidates of a warp kernel, scored by warp_dists into WarpSmem (see descend()).
template <class Op, int CH, int U>
struct WarpChunk {
  const GraphView& g;
  const WarpSmem& s;
  int lane;
  __device__ __forceinline__ void score(uint32_t id, int cnt) const {
    __syncwarp();  // earlier reads of the chunk happen-before the writes below
    if (lane < cnt) s.cand_id[lane] = id;
    __syncwarp();
    warp_dists<Op, CH, U>(reinterpret_cast<const uint4*>(g.vec), g.d4, g.dim, s.q4, s.cand_id, cnt, s.cand_d);
    __syncwarp();
  }
  __device__ __forceinline__ float dist(int j) const { return s.cand_d[j]; }
  __device__ __forceinline__ uint32_t id(int j) const { return s.cand_id[j]; }
};

struct Stats {
  unsigned evals, expansions, adj;
};

// Unfiltered search_layer.  On return Q (in s.wbuf) holds min(ef, reached) keys ascending by
// (dist, id).  Equivalence with the two-heap reference loop (no filter):
//   * accept rule `d < d(f) || |W| < ef` + bounded W  == keep the ef smallest keys seen (SortedQueue)
//   * C.pop() nearest-first + stop when d(c) > d(f)   == expand the nearest unexpanded entry of W until none is left:
//     a candidate evicted from W has key > every key of the (full) W, and f only decreases afterwards,
//     so it would trip the stop rule the moment it is popped.
// Ties on distance are ordered by id (oracle MODE_DET).
template <class Op, int CH, int U, class Queue>
__device__ __forceinline__ void search_layer(const GraphView& g, const WarpSmem& s, Stage& stg, const VisitedCfg& vc,
                                             Visited& vis, Queue& Q, uint32_t ep, int ef, int layer, Stats& st, bool& overflow) {
  const int lane = lane_id();
  const uint4* vec4 = reinterpret_cast<const uint4*>(g.vec);
  vis.begin(vc, ep, lane);  // hnsw.rs:955-956
  WarpChunk<Op, CH, U>{g, s, lane}.score(ep, 1);  // hnsw.rs:952
  st.evals += 1;
  const float d0 = Op::post(s.cand_d[0]);
  Q.reset(s.wbuf, ef);
  Q.push_first(make_key(d0, ep));  // hnsw.rs:958-967 (ep enters W and C)
  for (;;) {
    const int idx = Q.first_unexpanded();  // C.pop(): nearest candidate (hnsw.rs:971)
    if (idx < 0) break;                    // C empty (969) or stop rule (981-993), see header
    const uint32_t c = key_id(Q.get(idx));
    int cap;
    const uint32_t* ids = list_ids(g, c, layer, cap);  // hnsw.rs:1006
    {  // pull the adjacency rows of the two most likely next candidates towards L2 while this one is expanded
      int n1, n2, n3;
      Q.next3(idx + 1, n1, n2, n3);
      const uint32_t c1 = n1 >= 0 ? key_id(Q.get(n1)) : INVALID_ID;
      const uint32_t c2 = n2 >= 0 ? key_id(Q.get(n2)) : INVALID_ID;
      const uint32_t pc = lane == 0 ? c1 : (lane == 1 ? c2 : INVALID_ID);
      if (pc != INVALID_ID) {
        int pcap;
        const uint32_t* pids = list_ids(g, pc, layer, pcap);
        if (pids) asm volatile("prefetch.global.L2 [%0];" ::"l"(pids));
      }
    }
    Q.mark_expanded(idx);
    st.expansions += 1;
    for (int base = 0; base < cap; base += 32) {  // hnsw.rs:1013, 32 neighbours at a time
      const uint32_t nid = (base + lane < cap) ? ids[base + lane] : INVALID_ID;
      const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
      st.adj += __popc(valid);
      const bool fresh = vis.test_and_set(vc, lane, nid, nid != INVALID_ID);  // hnsw.rs:1016-1017
      const unsigned m = __ballot_sync(FULL, fresh);
      const int cnt = __popc(m);
      if (cnt) {
        const int pos = __popc(m & ((1u << lane) - 1u));
        if (fresh) s.cand_id[pos] = nid;
        __syncwarp();
        warp_dists_staged<Op, CH, U>(vec4, g.d4, g.dim, s.q4, s.cand_id, cnt, s.cand_d, stg);  // hnsw.rs:1026
        __syncwarp();
        st.evals += cnt;
        const uint64_t key = lane < cnt ? make_key(Op::post(s.cand_d[lane]), s.cand_id[lane]) : ~0ull;
        unsigned acc = __ballot_sync(FULL, lane < cnt && Q.accepts(key));  // hnsw.rs:1028
        while (acc) {
          const int j = __ffs(acc) - 1;
          acc &= acc - 1;
          const uint64_t kj = __shfl_sync(FULL, key, j);
          if (Q.accepts(kj)) Q.insert(kj);  // hnsw.rs:1035-1053
        }
      }
      if (valid != FULL) break;  // lists are dense prefixes terminated by INVALID_ID
    }
    if (vis.grow_or_overflow(vc, lane)) {
      overflow = true;
      break;
    }
  }
}

// the next work item of this warp from a launch's work counter (warp-uniform)
__device__ __forceinline__ uint32_t next_item(unsigned int* work_counter, int lane) {
  uint32_t i = 0;
  if (lane == 0) i = atomicAdd(work_counter, 1u);
  return __shfl_sync(FULL, i, 0);
}

struct Entry {
  uint32_t pivot;  // entry point of the lowest layer
  float best;      // its distance
};

// Upper-layer descent (hnsw.rs:1498-1529): from the graph's entry point, ONE pass over pivot.neighbours[layer] per
// layer, moving to the first minimum of the list when it is strictly below the best distance so far.
// How one chunk is scored is the parameter: ch.score(id, cnt) puts the ids of lanes i < cnt in slots 0..cnt-1 and scores
// them, ch.dist(j) / ch.id(j) read slot j back (distance before Op::post).
template <class Op, class Chunk>
__device__ __forceinline__ Entry descend(const GraphView& g, int lane, Stats& st, const Chunk& ch) {
  uint32_t pivot = g.entry;
  ch.score(pivot, 1);  // hnsw.rs:1506
  st.evals += 1;
  float best = Op::post(ch.dist(0));
  for (int layer = g.entry_level; layer >= 1; --layer) {
    int cap;
    const uint32_t* ids = list_ids(g, pivot, layer, cap);
    uint32_t new_pivot = pivot;
    for (int b = 0; b < cap; b += 32) {
      const uint32_t nid = (b + lane < cap) ? ids[b + lane] : INVALID_ID;
      const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
      const int cnt = __popc(valid);  // dense prefix
      if (cnt) {
        ch.score(nid, cnt);  // hnsw.rs:1518
        st.evals += cnt;
        st.adj += cnt;
        // strict `<` scanned in list order == first minimum of the list, if below `best`
        uint64_t key = lane < cnt ? (((uint64_t)__float_as_uint(Op::post(ch.dist(lane))) << 32) | (uint32_t)lane) : ~0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const uint64_t other = __shfl_xor_sync(FULL, key, o);
          key = other < key ? other : key;
        }
        const float dmin = __uint_as_float((uint32_t)(key >> 32));
        if (dmin < best) {
          best = dmin;
          new_pivot = ch.id((uint32_t)key & 31u);
        }
      }
      if (valid != FULL) break;
    }
    pivot = new_pivot;  // hnsw.rs:1526-1528
  }
  return Entry{pivot, best};
}

// Where query qi of a launch is: row q_ids[qi] of the store for a search by stored point (rows are zero padded to whole
// lines, so staging one gives the bytes its vector would), else row qi of `queries`, `stride` bytes apart.
__device__ __forceinline__ const char* query_row(const GraphView& g, const uint64_t* q_ids, const void* queries, size_t stride,
                                                 uint32_t qi) {
  if (q_ids) return reinterpret_cast<const char*>(g.vec) + (size_t)q_ids[qi] * ((size_t)g.d4 * 16);
  return reinterpret_cast<const char*>(queries) + (size_t)qi * stride;
}

// x is one of the sorted values v[0, n): a binary search in global memory
__device__ __forceinline__ bool in_sorted(const uint32_t* v, uint32_t n, uint32_t x) {
  while (n) {
    const uint32_t h = n >> 1, m = __ldg(v + h);
    if (m == x) return true;
    if (m < x) {
      v += h + 1;
      n -= h + 1;
    } else {
      n = h;
    }
  }
  return false;
}

// Row qi of a launch's answers from its keys key_at(0 .. count - 1), ascending: those keep(id) admits, as (origin,
// distance, internal id), then (~0, +inf, INVALID_ID) to the row's width, and their count.  Without skip ids a row is k
// wide.  With them (a search by stored point that leaves the point out) the launch searched k = knbn + 1 and a row is
// k - 1 wide: the key whose id is skip[qi] is left out and the rest cut to that width, which is the k-row without that
// entry, or without its last one when it does not hold it.
template <class KeyAt, class Keep>
__device__ __forceinline__ void write_row(NeighbourOut* out, int32_t* counts, const uint64_t* origin, int k,
                                          const uint64_t* skip, uint32_t qi, int lane, int count, KeyAt&& key_at, Keep&& keep) {
  const uint64_t skip_id = skip ? skip[qi] : ~0ull;
  const int w = skip ? k - 1 : k;
  NeighbourOut* o = out + (size_t)qi * w;
  int n = 0;
  for (int b = 0; b < count && n < w; b += 32) {  // warp-uniform trip count
    const int j = b + lane;
    uint64_t key = 0;
    bool in = false;
    if (j < count) {
      key = key_at(j);
      in = key_id(key) != skip_id && keep(key_id(key));
    }
    const unsigned m = __ballot_sync(FULL, in);
    const int at = n + __popc(m & ((1u << lane) - 1u));
    if (in && at < w) {
      const uint32_t id = key_id(key);
      o[at] = NeighbourOut{origin[id], key_dist(key), id};
    }
    n += __popc(m);
  }
  n = min(n, w);
  for (int j = n + lane; j < w; j += 32) o[j] = NeighbourOut{~0ull, __int_as_float(0x7f800000), INVALID_ID};
  if (lane == 0) counts[qi] = n;
  __syncwarp();
}

struct KeepAll {
  __device__ __forceinline__ bool operator()(uint32_t) const { return true; }
};

// The answers of query qi (hnsw.rs:1544-1579): key_at(j) for j < count, ascending (write_row).  A query whose visited
// table overflowed answers nothing and raises the launch's status flag (the host re-runs it).
template <class KeyAt>
__device__ __forceinline__ void write_answers(const SearchParams& p, int lane, uint32_t qi, bool overflow, int count, KeyAt&& key_at) {
  if (overflow) {
    if (lane == 0) atomicExch(p.status, 1);
    count = 0;
  }
  write_row(p.out_nb, p.out_count, p.g.origin, p.k, p.skip_ids, qi, lane, count, key_at, KeepAll());
}

// the traversal counters of one warp into the launch's totals (the counters are warp-uniform)
__device__ __forceinline__ void flush_stats(unsigned long long* stats, const Stats& st, int lane) {
  if (stats && lane == 0) {
    atomicAdd(stats + 0, (unsigned long long)st.evals);
    atomicAdd(stats + 1, (unsigned long long)st.expansions);
    atomicAdd(stats + 2, (unsigned long long)st.adj);
  }
}

}  // namespace hb
