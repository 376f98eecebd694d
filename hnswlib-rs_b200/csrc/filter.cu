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
// The FilterT predicate (filter.rs:7-24) is a device bitmap over internal ids, materialised by the host, or a point
// label: the predicate label(p) == L, or label(p) in a set S of labels, over the label array of the graph store; and,
// alone or with a label part, a range lo <= attr(p) <= hi over the attribute array of the graph store.  A row may also
// name points it never admits (its excluded list, binary-searched), on top of its run's predicate or alone, and no row
// admits a deleted point (the Index's deleted-point bitmap).  Unrestricted rows of an Index with deleted points run here
// too, as a run that admits every point and stops by the live rule (SearchParams::live_rows).
#include "kernels.h"
#include "search_core.cuh"

namespace hb {

__device__ __noinline__ bool in_sorted_call(const uint32_t* v, uint32_t n, uint32_t x) { return in_sorted(v, n, x); }

// Kernels whose register allocation (ptxas -v) stays the one they had before label sets only when the set lookup is a
// call: the generic u32 / i32 Hamming and L2 and u8 / u16 Jaccard ones.  Inlined, they spill more (Hamming: 76 registers
// and no spill became 64 and 40 bytes, measurably slower); every other kernel keeps its allocation with the lookup
// inlined, and the f32 L2 one only then.
template <class Op> struct SetLookupCall { static constexpr bool value = false; };
template <> struct SetLookupCall<OpHamming<int32_t>> { static constexpr bool value = true; };
template <> struct SetLookupCall<OpHamming<uint32_t>> { static constexpr bool value = true; };
template <> struct SetLookupCall<OpCast<int32_t, OpL2>> { static constexpr bool value = true; };
template <> struct SetLookupCall<OpCast<uint32_t, OpL2>> { static constexpr bool value = true; };
template <> struct SetLookupCall<OpJaccard<uint8_t>> { static constexpr bool value = true; };
template <> struct SetLookupCall<OpJaccard<uint16_t>> { static constexpr bool value = true; };
// A row's excluded points (RowFilter::excl) are looked up once per point, where it is scored: for a chunk of fresh
// neighbours before their distances (excluded_flags), and for the entry point when the search starts (xep).  Every
// other point of W entered it past that test, so W's later tests (keep_passing, the single-element clear, write_row's
// post-filter) only compare the id with xep (member_pass).  A lookup inside filter_pass at those sites made the generic
// u16 L1 and u32 Jaccard kernels spill (78 / 74 registers became 64 and 100 / 84 bytes spilled, inlined or called
// alike).  A deleted point is looked up at the same two places, and its flag shares the excluded one.  With the bitmap
// probe next to it, the generic u16 L1 kernel keeps its allocation (78 registers, no spill) only with the list lookup a
// call (inlined: 64 registers and 100 bytes spilled).
template <class Op> struct ExclLookupCall { static constexpr bool value = SetLookupCall<Op>::value; };
template <> struct ExclLookupCall<OpCast<uint16_t, OpL1>> { static constexpr bool value = true; };
template <class Op>
__device__ __forceinline__ bool in_excluded(const RowFilter* f, uint32_t id) {
  if constexpr (ExclLookupCall<Op>::value) return in_sorted_call(f->excl, f->nexcl, id);
  return in_sorted(f->excl, f->nexcl, id);
}

// A row's RowFilter in the warp's shared memory, with what the kernel adds per row: the Index's deleted points
// (SearchParams::deleted), whether the row is in the live run (SearchParams::live_rows), and whether it removes any
// point (excluded or deleted ones), the one word the chunk loop reads before and after the distances
struct RowSlot : RowFilter {
  const uint32_t* del;
  uint32_t live;
  uint32_t drops;
};

// the row never admits point id: it is deleted, or one of the row's excluded points
template <class Op>
__device__ __forceinline__ bool removed(const RowSlot* f, uint32_t id) {
  return (f->del && is_deleted(f->del, id)) || (f->nexcl && in_excluded<Op>(f, id));
}

// the admission test of the run's predicate: the point's attribute against the query's range, then its label against
// the query's label or set, or its bit of the bitmap
template <class Op>
__device__ __forceinline__ bool filter_pass(const RowFilter* f, uint32_t id) {
  const uint64_t* attr = f->attr;
  if (attr) {
    const uint64_t v = __ldg(attr + id);
    if (v < f->lo || v > f->hi) return false;
  }
  if (!f->ptr) return true;
  const uint32_t want = f->label;
  if (want != LABEL_NONE) {
    const uint32_t lab = __ldg(f->ptr + id);
    const uint32_t* set = f->set;
    if (!set) return lab == want;
    if constexpr (SetLookupCall<Op>::value) return in_sorted_call(set, f->nset, lab);
    return in_sorted(set, f->nset, lab);
  }
  return (__ldg(f->ptr + (id >> 5)) >> (id & 31)) & 1u;
}

// the admission test of a member of W: not the excluded entry point, and the run's predicate
template <class Op>
__device__ __forceinline__ bool member_pass(const RowFilter* f, uint32_t id) {
  return id != f->xep && filter_pass<Op>(f, id);
}

// keeps the keys w[0, n) whose points pass the filter, in order, at the front of w; returns how many there are
template <class Op>
__device__ __forceinline__ int keep_passing(uint64_t* w, int n, const RowFilter* fslot) {
  const int lane = lane_id();
  int out = 0;
  for (int b = 0; b < n; b += 32) {
    const int i = b + lane;
    uint64_t v = 0;
    bool keep = false;
    if (i < n) {
      v = w[i];
      keep = member_pass<Op>(fslot, key_id(v));
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
                                                      RowSlot* fslot, uint32_t ep, int ef, int layer,
                                                      Stats& st, bool& overflow) {
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
  // ep enters W before any test; if the row excludes it or it is deleted, every later test of W's members rejects it
  // (member_pass)
  if (lane == 0 && removed<Op>(fslot, ep)) fslot->xep = ep;
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
    const bool stop = (best >> 32) > (fkey >> 32);
    const bool live_stop = stop && fslot->live;
    if (stop && !live_stop && W.n >= ef) W.n = keep_passing<Op>(W.w, W.n, fslot);  // 994-1000
    const uint32_t c = key_id(best);
    int cap;
    const uint32_t* ids = list_ids(g, c, layer, cap);  // 1006
    // a live row returns W here, as without a filter (992-993): c is not expanded and C is emptied, so the next pop
    // ends the search.  (An early break here cost 11 filtered kernels their register allocation; this form keeps it.)
    if (live_stop) cn = 0;
    st.expansions += !live_stop;
    bool done = live_stop;
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
        // the chunk's excluded or deleted flags, in the unused upper half of the candidate-id region (nothing stays in a
        // register across the distances)
        uint32_t* const excluded_flags = s.cand_id + 32;
        if (fresh && fslot->drops) excluded_flags[pos] = removed<Op>(fslot, nid);
        __syncwarp();
        warp_dists<Op, CH, U>(vec4, g.d4, g.dim, s.q4, s.cand_id, cnt, s.cand_d);  // 1026
        __syncwarp();
        st.evals += cnt;
        const uint32_t my_id = lane < cnt ? s.cand_id[lane] : 0u;
        const uint64_t key = lane < cnt ? make_key(Op::post(s.cand_d[lane]), my_id) : ~0ull;
        const bool my_pass =
            lane < cnt && !(fslot->drops && excluded_flags[lane]) && filter_pass<Op>(fslot, my_id);
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
              if (W.n == 1 && !member_pass<Op>(fslot, key_id(W.w[0]))) W.n = 0;
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
    if (overflow || vis.grow_or_overflow(vc, lane)) {
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
  // the query's filter, read at each use so that the search loop holds no register for it: in the upper half of the
  // candidate-distance region, whose first 32 of 64 reserved entries are all this kernel scores into
  static_assert(sizeof(RowSlot) <= 32 * 4, "a RowSlot fits the upper half of the candidate-distance region");
  RowSlot* fslot = reinterpret_cast<RowSlot*>(base + L.cand_d + 32 * 4);
  const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + warp;  // the host launches fewer warps per CTA when shared memory is short
  Visited vis;
  vis.init(p.vis, slot);
  uint64_t* cbuf = p.cbuf + (size_t)slot * p.ccap;
  SortedQueue W;
  Stats st{0, 0, 0};

  for (;;) {
    const uint32_t qi = next_item(p.work_counter, lane);
    if (qi >= p.nq) break;
    stage_row_bytes(s.q4, query_row(g, p.q_ids, p.queries, p.q_stride_bytes, qi), p.q_bytes, g.d4 * 16);
    if (lane == 0) {
      *static_cast<RowFilter*>(fslot) = p.filter_sel ? p.filter_table[p.filter_sel[qi]] : p.filter;
      fslot->xep = INVALID_ID;
      fslot->del = p.deleted;
      fslot->live = qi < p.live_rows;
      if (p.excluded) {  // the row's own part: its excluded points
        const ExcludedRow x = p.excluded[qi];
        fslot->excl = p.excluded_ids + x.off;
        fslot->nexcl = x.n;
      }
      fslot->drops = fslot->nexcl || p.deleted;
    }
    __syncwarp();
    int count = 0;
    bool overflow = false;
    W.reset(s.wbuf, p.ef);
    if (g.entry != INVALID_ID) {
      // the filter plays no role in the descent (hnsw.rs:1511-1529)
      const Entry e = descend<Op>(g, lane, st, WarpChunk<Op, CH, U>{g, s, lane});
      search_layer_filtered<Op, CH, U>(g, s, p.vis, vis, W, cbuf, p.ccap, fslot, e.pivot, p.ef, p.layer0, st,
                                       overflow);
      count = min(p.k, min(p.ef, W.n));  // hnsw.rs:1547
    }
    if (overflow) {
      if (lane == 0) atomicExch(p.status, 1);
      count = 0;
    }
    // post-filter AFTER truncation (hnsw.rs:1549-1563): only the entry point can fail here
    write_row(p.out_nb, p.out_count, g.origin, p.k, p.skip_ids, qi, lane, count, [&](int j) { return W.w[j]; },
              [&](uint32_t id) { return member_pass<Op>(fslot, id); });
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
