// Filtered query kernel: search_filter with Some(filter) (/root/reference/src/hnsw.rs:1487-1580) and the
// filter branches of search_layer (/root/reference/src/hnsw.rs:981-1001, 1037-1050).
//
// With a filter the reference's loop differs from the unfiltered one in ways that break the
// "C is the unexpanded part of W" argument of search_core.cuh:
//   * W only receives candidates that pass the filter (plus the unfiltered entry point), but C receives
//     every accepted candidate, so C is not a subset of W;
//   * the stop rule does not return: when d(c) > d(f) it only drops non-passing points from W (if |W| >= ef)
//     and keeps expanding, until C is empty.
// So here C is a real queue: an unsorted array of keys per warp in global memory, pop = warp-wide min scan
// (consumed entries are overwritten with ~0).  W is the same sorted shared-memory array as elsewhere.
// The FilterT predicate (filter.rs:7-24) is a device bitmap over internal ids, materialised by the host.
#include "kernels.h"
#include "search_core.cuh"

namespace hb {

__device__ __forceinline__ bool filter_pass(const uint32_t* bits, uint32_t id) {
  return (__ldg(bits + (id >> 5)) >> (id & 31)) & 1u;
}

// keeps the keys w[0, n) whose points pass the filter, in order, at the front of w; returns how many there are
__device__ __forceinline__ int keep_passing(uint64_t* w, int n, const uint32_t* fbits) {
  const int lane = lane_id();
  int out = 0;
  for (int b = 0; b < n; b += 32) {
    const int i = b + lane;
    uint64_t v = 0;
    bool keep = false;
    if (i < n) {
      v = w[i];
      keep = filter_pass(fbits, key_id(v));
    }
    const unsigned m = __ballot_sync(FULL, keep);
    __syncwarp();
    if (keep) w[out + __popc(m & ((1u << lane) - 1u))] = v;
    out += __popc(m);
    __syncwarp();
  }
  return out;
}

template <class Op, int CH, int U>
__device__ __forceinline__ void search_layer_filtered(const GraphView& g, const WarpSmem& s, const VisitedCfg& vc, Visited& vis,
                                                      SortedQueue& W, uint64_t* cbuf, uint32_t ccap,
                                                      const uint32_t* const* fslot, uint32_t ep, int ef, int layer, Stats& st, bool& overflow) {
  const int lane = lane_id();
  const uint4* vec4 = reinterpret_cast<const uint4*>(g.vec);
  vis.begin(vc, ep, lane);  // hnsw.rs:955-956
  WarpChunk<Op, CH, U>{g, s, lane}.score(ep, 1);  // hnsw.rs:952
  st.evals += 1;
  const float d0 = Op::post(s.cand_d[0]);
  W.reset(s.wbuf, ef);
  if (lane == 0) {
    s.wbuf[0] = make_key(d0, ep);  // ep enters W unfiltered (hnsw.rs:964-967)
    cbuf[0] = make_key(d0, ep);    // and C (960-963)
  }
  W.n = 1;
  uint32_t cn = 1;
  __syncwarp();
  for (;;) {
    // ---- C.pop(): nearest candidate (hnsw.rs:971)
    uint64_t best = ~0ull;
    uint32_t bpos = 0;
    for (uint32_t b = 0; b < cn; b += 32) {
      const uint32_t i = b + lane;
      const uint64_t v = i < cn ? __ldcg(cbuf + i) : ~0ull;
      if (v < best) {
        best = v;
        bpos = i;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t ov = __shfl_xor_sync(FULL, best, o);
      const uint32_t op = __shfl_xor_sync(FULL, bpos, o);
      if (ov < best) {
        best = ov;
        bpos = op;
      }
    }
    if (best == ~0ull) break;  // C is empty (969)
    if (lane == 0) __stcg(cbuf + bpos, ~0ull);
    // trim consumed entries at the tail so the scan stays short
    if (bpos == cn - 1) cn -= 1;
    __syncwarp();
    // The reference unwraps W.peek() here (973) and would panic on an empty W (possible only when the
    // entry point fails the filter, ef == 1 and it was retained away); we return the empty W instead.
    if (W.n == 0) break;
    const uint64_t fkey = W.w[W.n - 1] & ~1ull;
    // 981: the reference compares DISTANCES here (-(c.dist) > f.dist); with equal distances a larger id must not
    // trigger the retain pass (Hamming / Jaccard / integer L1 tie often)
    if ((best >> 32) > (fkey >> 32) && W.n >= ef) W.n = keep_passing(W.w, W.n, *fslot);  // 994-1000
    const uint32_t c = key_id(best);
    int cap;
    const uint32_t* ids = list_ids(g, c, layer, cap);  // 1006
    st.expansions += 1;
    bool done = false;
    for (int base = 0; base < cap && !done; base += 32) {
      const uint32_t nid = (base + lane < cap) ? ids[base + lane] : INVALID_ID;
      const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
      st.adj += __popc(valid);
      const bool fresh = vis.test_and_set(vc, lane, nid, nid != INVALID_ID);  // 1016-1017
      const unsigned m = __ballot_sync(FULL, fresh);
      const int cnt = __popc(m);
      if (cnt) {
        const int pos = __popc(m & ((1u << lane) - 1u));
        if (fresh) s.cand_id[pos] = nid;
        __syncwarp();
        warp_dists<Op, CH, U>(vec4, g.d4, g.dim, s.q4, s.cand_id, cnt, s.cand_d);  // 1026
        __syncwarp();
        st.evals += cnt;
        const uint32_t my_id = lane < cnt ? s.cand_id[lane] : 0u;
        const uint64_t key = lane < cnt ? make_key(Op::post(s.cand_d[lane]), my_id) : ~0ull;
        const bool my_pass = lane < cnt && filter_pass(*fslot, my_id);
        const unsigned passmask = __ballot_sync(FULL, my_pass);
        for (int j = 0; j < cnt; ++j) {  // strictly in list order: the accept rule sees the W of that moment
          if (W.n == 0) {                // 1019-1024
            done = true;
            break;
          }
          const uint64_t kj = __shfl_sync(FULL, key, j);
          if (W.n < ef || kj < (W.w[W.n - 1] & ~1ull)) {  // 1028
            if (cn >= ccap) {
              overflow = true;
              done = true;
              break;
            }
            if (lane == 0) __stcg(cbuf + cn, kj);  // 1035-1036: every accepted candidate goes to C
            cn += 1;
            if ((passmask >> j) & 1u) {  // 1040-1049
              if (W.n == 1 && !filter_pass(*fslot, key_id(W.w[0]))) W.n = 0;
              __syncwarp();
              W.insert(kj);  // push, and pop the farthest when over ef (1051-1053)
            }
          }
        }
        __syncwarp();
      }
      if (valid != FULL) break;
    }
    if (done && W.n == 0) break;
    if (overflow || vis.overflowing(vc)) {
      overflow = true;
      break;
    }
  }
}

template <class Op, int CH, int U>
__global__ void __launch_bounds__(SEARCH_THREADS) search_filter_kernel(SearchParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GraphView& g = p.g;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  const QueryLayout L = query_layout(g.d4, p.q_smem);  // search.cu's layout; the stage is unused here
  const WarpSmem s{reinterpret_cast<uint4*>(base + L.query), reinterpret_cast<uint64_t*>(base + L.queue),
                   reinterpret_cast<uint32_t*>(base + L.cand_id), reinterpret_cast<float*>(base + L.cand_d)};
  const uint32_t** fslot = reinterpret_cast<const uint32_t**>(base + L.bar);
  const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + warp;  // the host launches fewer warps per CTA when shared memory is short
  Visited vis;
  vis.init(p.vis, slot);
  uint64_t* cbuf = p.cbuf + (size_t)slot * p.ccap;
  SortedQueue W;
  Stats st{0, 0, 0};

  for (;;) {
    const uint32_t qi = next_item(p.work_counter, lane);
    if (qi >= p.nq) break;
    stage_row_bytes(s.q4, reinterpret_cast<const char*>(p.queries) + (size_t)qi * p.q_stride_bytes, p.q_bytes, g.d4 * 16);
    // this query's bitmap: the launch's one filter, or its own entry of the filter table.  It is kept in the warp's
    // mbarrier slot (unused by this kernel) and read at each use, so that the search loop holds no extra register.
    if (lane == 0) *fslot = p.filter_sel ? p.filter_table[p.filter_sel[qi]] : p.filter_bits;
    __syncwarp();
    int count = 0;
    bool overflow = false;
    W.reset(s.wbuf, p.ef);
    if (g.entry != INVALID_ID) {
      // the filter plays no role in the descent (hnsw.rs:1511-1529)
      const Entry e = descend<Op>(g, lane, st, WarpChunk<Op, CH, U>{g, s, lane});
      search_layer_filtered<Op, CH, U>(g, s, p.vis, vis, W, cbuf, p.ccap, fslot, e.pivot, p.ef, p.layer0, st, overflow);
      count = min(p.k, min(p.ef, W.n));  // hnsw.rs:1547
    }
    if (overflow) {
      if (lane == 0) atomicExch(p.status, 1);
      count = 0;
    }
    // post-filter AFTER truncation (hnsw.rs:1549-1563): only the entry point can fail here
    const size_t ob = (size_t)qi * p.k;
    int outn = 0;
    for (int b = 0; b < count; b += 32) {
      const int j = b + lane;
      uint64_t key = 0;
      bool keep = false;
      if (j < count) {
        key = W.w[j];
        keep = filter_pass(*fslot, key_id(key));
      }
      const unsigned m = __ballot_sync(FULL, keep);
      if (keep) {
        const uint32_t id = key_id(key);
        p.out_nb[ob + outn + __popc(m & ((1u << lane) - 1u))] = NeighbourOut{g.origin[id], key_dist(key), id};
      }
      outn += __popc(m);
    }
    for (int j = outn + lane; j < p.k; j += 32) p.out_nb[ob + j] = NeighbourOut{~0ull, __int_as_float(0x7f800000), INVALID_ID};
    if (lane == 0) p.out_count[qi] = outn;
    __syncwarp();
  }
  vis.save(p.vis, slot, lane);
  flush_stats(p.stats, st, lane);
}

template <class Op>
static cudaError_t launch_filter_for_op(const SearchParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  if constexpr (Specialise<Op>::value) {
    if (p.g.d4 / 8 == 4) return launch_kernel(search_filter_kernel<Op, 4, 2>, p, grid, p.threads, smem, st, blocks_per_sm);
  }
  return launch_kernel(search_filter_kernel<Op, 0, 2>, p, grid, p.threads, smem, st, blocks_per_sm);
}

cudaError_t launch_search_filtered(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                                   int* blocks_per_sm) {
  return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    using Op = typename decltype(tag)::type;
    return launch_filter_for_op<Op>(p, grid, smem, st, blocks_per_sm);
  });
}

}  // namespace hb
