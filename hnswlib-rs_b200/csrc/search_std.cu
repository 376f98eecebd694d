// Query kernel, std-tie form (opt-in: hnsw_b200_set_tie_mode(h, 1)).
//
// The reference keeps search_layer's two queues in Rust-std BinaryHeaps whose Ord compares the DISTANCE only
// (/root/reference/src/hnsw.rs:273-297, 940-1053, 1544).  With metrics that tie all the time (Hamming, Jaccard, integer
// L1) which of several equal-distance points is evicted, popped first or returned is decided by the heap's sift rules.
// The production kernels order ties by (distance, id) instead, a total order that never disagrees with the reference on
// data without ties.  This kernel replays the reference literally, so that the neighbour IDS are those of the
// reference on tie-heavy data as well (BASELINE.json: "identical neighbour-id sets for integer Hamming/Jaccard"):
//   * W and C are binary heaps with std's algorithms: push = sift_up stopping on `elem <= parent`; pop = swap the
//     last element into the root, sift_down_to_bottom (always descend, the right child when `left <= right`), sift_up;
//     into_sorted_vec = swap(0, end) + sift_down_range.  One lane runs them (W in shared memory, C in the per-warp global
//     scratch the filtered kernel also uses); the warp does the row gathers and distance sums as everywhere else;
//   * neighbours are taken in LIST ORDER, one at a time, against the bound as it is at that moment
//     (hnsw.rs:1013-1053): `d < f.dist || |W| < ef` -> C.push, W.push, W.pop when |W| > ef;
//   * stop rule `-(c.dist) > f.dist` (hnsw.rs:981), result = W.into_sorted_vec() truncated (hnsw.rs:1544-1547).
// Distances are computed in the kernels' summation order; for the integer metrics this mode is meant for they are exact
// in any order.  It is several times slower than the production kernels (one lane drives the heaps).
#include "kernels.h"
#include "search_core.cuh"

namespace hb {

struct SItem {
  float kd;     // signed key distance exactly as the reference stores it (+d in W, -d in C)
  uint32_t id;  // internal id
};
// PointWithOrder's Ord = dist_to_ref.partial_cmp (hnsw.rs:273-297): the id takes no part
__device__ __forceinline__ bool s_le(const SItem& a, const SItem& b) { return !(a.kd > b.kd); }
__device__ __forceinline__ bool s_lt(const SItem& a, const SItem& b) { return a.kd < b.kd; }
__device__ __forceinline__ bool s_ge(const SItem& a, const SItem& b) { return !(a.kd < b.kd); }

// Rust std alloc::collections::binary_heap, restated (cf. oracle/rheap.h, which pins the same rules on the CPU)
struct StdHeap {
  SItem* v;
  int n;
  __device__ int sift_up(int start, int pos) {
    const SItem elt = v[pos];
    while (pos > start) {
      const int parent = (pos - 1) / 2;
      if (s_le(elt, v[parent])) break;
      v[pos] = v[parent];
      pos = parent;
    }
    v[pos] = elt;
    return pos;
  }
  __device__ void sift_down_range(int pos, int end) {
    const SItem elt = v[pos];
    int child = 2 * pos + 1;
    const int lim = end >= 2 ? end - 2 : 0;  // end.saturating_sub(2)
    while (child <= lim && end >= 2) {
      if (s_le(v[child], v[child + 1])) child += 1;
      if (s_ge(elt, v[child])) {
        v[pos] = elt;
        return;
      }
      v[pos] = v[child];
      pos = child;
      child = 2 * pos + 1;
    }
    if (end >= 1 && child == end - 1 && s_lt(elt, v[child])) {
      v[pos] = v[child];
      pos = child;
    }
    v[pos] = elt;
  }
  __device__ void sift_down_to_bottom(int pos) {
    const int end = n, start = pos;
    const SItem elt = v[pos];
    int child = 2 * pos + 1;
    const int lim = end >= 2 ? end - 2 : 0;
    while (child <= lim && end >= 2) {
      if (s_le(v[child], v[child + 1])) child += 1;
      v[pos] = v[child];
      pos = child;
      child = 2 * pos + 1;
    }
    if (end >= 1 && child == end - 1) {
      v[pos] = v[child];
      pos = child;
    }
    v[pos] = elt;
    sift_up(start, pos);
  }
  __device__ void push(const SItem& it) {
    const int old = n;
    v[n++] = it;
    sift_up(0, old);
  }
  __device__ SItem pop() {
    SItem item = v[n - 1];
    n -= 1;
    if (n > 0) {
      const SItem root = v[0];
      v[0] = item;
      item = root;
      sift_down_to_bottom(0);
    }
    return item;
  }
  __device__ void into_sorted() {  // ascending, in place
    int end = n;
    while (end > 1) {
      end -= 1;
      const SItem t = v[0];
      v[0] = v[end];
      v[end] = t;
      sift_down_range(0, end);
    }
  }
};

template <class Op>
__global__ void __launch_bounds__(SEARCH_THREADS) search_std_kernel(SearchParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GraphView& g = p.g;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  const StdLayout L = std_layout(g.d4, p.q_smem);
  const WarpSmem s{reinterpret_cast<uint4*>(base + L.query), nullptr, reinterpret_cast<uint32_t*>(base + L.cand_id),
                   reinterpret_cast<float*>(base + L.cand_d)};
  SItem* wv = reinterpret_cast<SItem*>(base + L.heap);
  const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + warp;  // the host launches fewer warps per CTA when shared memory is short
  Visited vis;
  vis.init(p.vis, slot);
  SItem* cv = reinterpret_cast<SItem*>(p.cbuf + (size_t)slot * p.ccap);
  Stats st{0, 0, 0};
  const uint4* vec4 = reinterpret_cast<const uint4*>(g.vec);
  const int ef = p.ef;

  for (;;) {
    const uint32_t qi = next_item(p.work_counter, lane);
    if (qi >= p.nq) break;
    stage_row_bytes(s.q4, query_row(g, p.q_ids, p.queries, p.q_stride_bytes, qi), p.q_bytes, g.d4 * 16);
    int count = 0;
    bool overflow = false;
    StdHeap W{wv, 0}, C{cv, 0};
    if (g.entry != INVALID_ID) {
      // ---- descent (hnsw.rs:1498-1529): strict '<' in list order, distances only: as in every kernel
      const Entry e = descend<Op>(g, lane, st, WarpChunk<Op, 0, 2>{g, s, lane});
      const uint32_t pivot = e.pivot;
      const float best = e.best;
      // ---- search_layer, literally (hnsw.rs:940-1063)
      vis.begin(p.vis, pivot, lane);  // 955-956
      st.evals += 1;                  // 952: dist(q, ep), the value is `best`
      int wn = 0;
      if (lane == 0) {
        C.push(SItem{-best, pivot});  // 960-963
        W.push(SItem{best, pivot});   // 964-967
        wn = W.n;
      }
      for (;;) {
        uint32_t c = INVALID_ID;
        if (lane == 0 && C.n > 0) {       // 969
          const SItem ci = C.pop();       // 971
          const SItem f = W.v[0];         // 973
          if (!((-ci.kd) > f.kd)) c = ci.id;  // 981: stop when the nearest candidate is farther than W's farthest
        }
        c = __shfl_sync(FULL, c, 0);
        if (c == INVALID_ID) break;  // C empty, or the stop rule
        st.expansions += 1;
        int cap;
        const uint32_t* ids = list_ids(g, c, p.layer0, cap);  // 1006
        for (int b = 0; b < cap; b += 32) {  // 1013
          const uint32_t nid = (b + lane < cap) ? ids[b + lane] : INVALID_ID;
          const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
          st.adj += __popc(valid);
          const bool fresh = vis.test_and_set(p.vis, lane, nid, nid != INVALID_ID);  // 1016-1017
          const unsigned m = __ballot_sync(FULL, fresh);
          const int cnt = __popc(m);
          if (cnt) {
            const int pos = __popc(m & ((1u << lane) - 1u));  // lane order == list order
            if (fresh) s.cand_id[pos] = nid;
            __syncwarp();
            warp_dists<Op, 0, 2>(vec4, g.d4, g.dim, s.q4, s.cand_id, cnt, s.cand_d);  // 1026
            __syncwarp();
            st.evals += cnt;
            if (lane == 0) {
              for (int i = 0; i < cnt; ++i) {
                const float de = Op::post(s.cand_d[i]);
                const SItem f2 = W.v[0];  // 1019-1024
                if (de < f2.kd || W.n < ef) {  // 1028
                  if (C.n >= (int)p.ccap) {
                    overflow = true;
                    break;
                  }
                  C.push(SItem{-de, s.cand_id[i]});  // 1035-1036
                  W.push(SItem{de, s.cand_id[i]});   // 1038
                  if (W.n > ef) W.pop();           // 1051-1053
                }
              }
            }
            __syncwarp();
          }
          if (valid != FULL) break;
        }
        overflow = __shfl_sync(FULL, (int)overflow, 0) != 0 || vis.grow_or_overflow(p.vis, lane);
        if (overflow) break;
      }
      if (lane == 0) {
        W.into_sorted();  // 1544
        wn = W.n;
      }
      wn = __shfl_sync(FULL, wn, 0);
      __syncwarp();
      count = min(p.k, min(ef, wn));  // 1547
    }
    write_answers(p, lane, qi, overflow, count, [&](int j) { return make_key(wv[j].kd, wv[j].id); });
  }
  vis.save(p.vis, slot, lane);
  flush_stats(p.stats, st, lane);
}

cudaError_t launch_search_std(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                              int* blocks_per_sm) {
  return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    using Op = typename decltype(tag)::type;
    return launch_kernel(search_std_kernel<Op>, p, grid, p.threads, smem, st, blocks_per_sm);
  });
}

}  // namespace hb
