// Query kernel, lean form: one warp per query, persistent warps pulling query indices from a counter.
//
// Restates /root/reference/src/hnsw.rs:1487-1580 (search_filter without a filter: entry fetch, one hop per
// upper layer, search_layer on the lowest populated layer, ascending top-k), hnsw.rs:922-1064 (search_layer) and the
// batch contract of parallel_search (hnsw.rs:1612-1635: one answer per query, in input order).
//
// Same algorithm and the same arithmetic as search.cu / search_core.cuh (bit-identical answers and traversal
// counters); what differs is what one expansion costs.  The step time of this kernel is the length of the warp's
// dependent instruction chain (~10 cycles per instruction with the few warps an SM holds), not the memory latency,
// so everything here is about issuing fewer instructions per expansion:
//   * C (the reference's candidate heap) is a BIT MASK in registers over the positions of the sorted array W:
//     "pop the nearest candidate" is a find-first-set, "push" is a shift-and-or at the insertion position; no scans
//     of the queue, no expanded flag inside the keys to maintain;
//   * the lane's chunks of the query live in registers for the whole search, W / row ids / distances are addressed
//     through 32-bit shared-memory window addresses computed once (pin());
//   * rows are fetched by plain 128-bit loads, 8 rows in flight per warp, and the lines of the rows beyond the first
//     eight are prefetched to L2 the moment the list is known, so that only the first pass pays the HBM latency
//     (issuing one bulk copy per row costs ~8 instructions per row: the copy engine takes uniform operands);
//   * two rows per lane group are reduced with one transposed reduction (3 shuffles for 2 rows, same sums);
//   * a staged launch keeps the visited set's first stage in the warp's shared memory (VisitedT<FirstStage::Shared>):
//     a probe is a shared-memory load, and a query that never moves touches no table line in L2;
//   * the traversal counters are a template parameter: the production instantiation does not carry them.
#pragma once
#include "kernels.h"
#include "lean_common.cuh"
#include "search_core.cuh"

namespace hb {

struct NoHook {
  __device__ __forceinline__ void operator()() const {}
};

// 8 lanes per row, rows base+4u+r (u < 2, r = lane group) per pass; results (before Op::post) to da[].
// `hook` runs once, after the loads of the first pass are issued and before they are used: whatever it loads
// travels together with the rows.
template <class Op, int CH, class Hook>
__device__ __forceinline__ void lean_score(const char* vecb, const uint4 (&qv)[CH], uint32_t ca, uint32_t da, int cnt, int dim,
                                           int g, int r, uint64_t pol_rows, Hook&& hook) {
  typedef typename Op::red_t red_t;
  constexpr uint32_t row_bytes = (uint32_t)CH * 128u;
  for (int base = 0; base < cnt; base += 8) {
    uint4 x[2][CH];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int idx = base + 4 * u + r;
      const uint32_t id = lds32(ca + 4 * (idx < cnt ? idx : cnt - 1));
      const uint4* row = reinterpret_cast<const uint4*>(vecb + (size_t)id * row_bytes) + g;
#pragma unroll
      for (int i = 0; i < CH; ++i) x[u][i] = ldg_stream(row + 8 * i, pol_rows);
    }
    if (base == 0) hook();
    red_t a[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      typename Op::acc_t acc = Op::zero();
#pragma unroll
      for (int i = 0; i < CH; ++i) Op::chunk(acc, qv[i], x[u][i]);
      a[u] = Op::fold(acc);
    }
    // transposed first butterfly step: lanes with bit 2 clear finish row u = 0, the others row u = 1 (same pairs
    // of partial sums as reduce8: bit-identical)
    const bool h4 = (g & 4) != 0;
    red_t s = radd(h4 ? a[1] : a[0], rshfl(h4 ? a[0] : a[1], 4));
    s = radd(s, rshfl(s, 2));
    s = radd(s, rshfl(s, 1));
    const int idx = base + 4 * (g >> 2) + r;
    if ((g & 3) == 0 && idx < cnt) sts32(da + 4 * idx, __float_as_uint(Op::finish(s, dim)));
  }
}

// W: sorted keys in shared memory, QC = 32 * NCH slots, slots >= ef hold ~0 (compare above every key).
// One merge per 32-neighbour chunk instead of one sorted insert per accepted neighbour (hnsw.rs:1028-1053).  The
// accepted set A = {key < the bound before the chunk} contains every key the one-at-a-time loop would push (the bound
// only tightens), and what that loop leaves is the `cap` smallest of W u A, which is what is built here: an old entry
// moves up by the number of accepted keys below it, an accepted key lands at (its rank in A) + (old entries below
// it), entries that land at >= cap fall off.  The unexpanded mask C follows the entries.
template <int NCH, class MaskT>
__device__ __forceinline__ void lean_merge(uint32_t wa, int lane, uint64_t key, unsigned accmask, int cap, int& n,
                                           uint64_t& thr, MaskT& open) {
  const bool accepted = (accmask >> lane) & 1u;
  uint64_t cur[NCH];
  int lb[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    cur[c] = lds64(wa + 8 * (32 * c + lane));
    lb[c] = 0;
  }
  int np = 0;  // an accepted key lands at (old entries below it) + (accepted keys below it)
  for (unsigned rem = accmask; rem; rem &= rem - 1) {
    const int j = __ffs(rem) - 1;
    const uint64_t kj = __shfl_sync(FULL, key, j);
    int below = (accepted && key < kj) ? 1 : 0;  // keys are distinct: ids are (the visited set admits an id once)
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const bool lt = cur[c] < kj;
      below += lt ? 1 : 0;
      lb[c] += lt ? 0 : 1;
    }
    below = __reduce_add_sync(FULL, below);
    if (lane == j) np = below;
  }
  __syncwarp();  // every lane holds its old entries: the slots may be rewritten
  uint32_t bits[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) bits[c] = 0;
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int ni = 32 * c + lane + lb[c];
    if (ni < cap && cur[c] != ~0ull) {
      if (lb[c] > 0) sts64(wa + 8 * ni, cur[c]);
      if (open.test(32 * c + lane)) {
#pragma unroll
        for (int w = 0; w < NCH; ++w)
          if ((ni >> 5) == w) bits[w] |= 1u << (ni & 31);
      }
    }
  }
  if (accepted && np < cap) {
    sts64(wa + 8 * np, key);
#pragma unroll
    for (int w = 0; w < NCH; ++w)
      if ((np >> 5) == w) bits[w] |= 1u << (np & 31);
  }
#pragma unroll
  for (int w = 0; w < NCH; ++w) bits[w] = __reduce_or_sync(FULL, bits[w]);
  open.set_words(bits);
  __syncwarp();
  n += __popc(accmask);
  n = n < cap ? n : cap;
  thr = lds64(wa + 8 * (cap - 1));
}

template <class Op, int CH, int QC, bool STATS>
__global__ void __launch_bounds__(LEAN_THREADS, LEAN_MIN_BLOCKS) search_lean_kernel(SearchParams p) {
  typedef typename MaskSel<QC>::type MaskT;
  constexpr int NCH = QC / 32;
  constexpr LeanLayout L = lean_layout(QC);
  static_assert(CH * 128 <= QC * 8, "the query is staged in the queue buffer");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const GraphView& G = p.g;
  const int lane = (int)pin(threadIdx.x & 31);
  const int g = lane & 7, r = lane >> 3;
  // the warp's region is p.smem_per_warp bytes: lean_layout(QC, p.vis.small)
  const uint32_t wa = pin(smem_u32(smem_raw) + (uint32_t)(threadIdx.x >> 5) * (uint32_t)p.smem_per_warp + L.queue);
  const uint32_t ca = wa + L.cand_id, da = wa + L.cand_d;
  const char* const vecb = reinterpret_cast<const char*>(G.vec);
  constexpr uint32_t row_bytes = (uint32_t)CH * 128u;
  const uint64_t pol_rows = l2_policy_evict_first();

  const uint32_t slot = blockIdx.x * (LEAN_THREADS / 32) + (threadIdx.x >> 5);
  VisitedT<FirstStage::Shared> vis;  // first stage in the warp's shared memory, full stage in its global slot
  vis.init(p.vis, slot, wa - L.queue + L.visited, lane);
  unsigned evals = 0, expans = 0, adjr = 0;
  const int cap = p.ef;

  for (;;) {
    const uint32_t qi = next_item(p.work_counter, lane);
    if (qi >= p.nq) break;
    // ---- the lane's chunks of the query (zero padded) -> registers, through the queue buffer
    {
      const char* src = query_row(G, p.q_ids, p.queries, p.q_stride_bytes, qi);
      const int nw = p.q_bytes >> 2;
      if ((reinterpret_cast<size_t>(src) & 3) == 0) {
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
        for (int i = lane; i < CH * 32; i += 32) {
          uint32_t v = 0;
          if (i < nw) v = s32[i];
          else if ((i << 2) < p.q_bytes)
            for (int b = 0; b < (p.q_bytes & 3); ++b) v |= (uint32_t)(uint8_t)src[(nw << 2) + b] << (8 * b);
          sts32(wa + 4 * i, v);
        }
      } else {
        for (int i = lane; i < CH * 32; i += 32) {
          uint32_t v = 0;
          for (int b = 0; b < 4; ++b)
            if ((i << 2) + b < p.q_bytes) v |= (uint32_t)(uint8_t)src[(i << 2) + b] << (8 * b);
          sts32(wa + 4 * i, v);
        }
      }
    }
    __syncwarp();
    uint4 qv[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) qv[i] = lds128(wa + 16 * (g + 8 * i));
    __syncwarp();

    // ---- descent: ONE pass over pivot.neighbours[layer] per layer (hnsw.rs:1498-1529).  descend() (search_core.cuh) with
    // lean_score as its chunk scorer computes the same, but the compiler then schedules and allocates this kernel differently
    // (more registers in most instantiations, spills in the Jaccard ones with 512-byte rows); this copy keeps its code as tuned.
    uint32_t pivot = G.entry;
    if (lane == 0) sts32(ca, pivot);
    __syncwarp();
    lean_score<Op, CH>(vecb, qv, ca, da, 1, G.dim, g, r, pol_rows, NoHook());  // hnsw.rs:1506
    __syncwarp();
    if (STATS) evals += 1;
    float best = Op::post(__uint_as_float(lds32(da)));
    for (int layer = G.entry_level; layer >= 1; --layer) {
      int lcap;
      const uint32_t* ids = list_ids(G, pivot, layer, lcap);
      uint32_t new_pivot = pivot;
      for (int b = 0; b < lcap; b += 32) {
        const uint32_t nid = (b + lane < lcap) ? ids[b + lane] : INVALID_ID;
        const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
        const int cnt = __popc(valid);  // dense prefix
        if (cnt) {
          __syncwarp();
          if (lane < cnt) sts32(ca + 4 * lane, nid);
          __syncwarp();
          lean_score<Op, CH>(vecb, qv, ca, da, cnt, G.dim, g, r, pol_rows, NoHook());  // hnsw.rs:1518
          __syncwarp();
          if (STATS) {
            evals += cnt;
            adjr += cnt;
          }
          // strict `<` scanned in list order == first minimum of the list, if below `best`
          uint64_t key = lane < cnt ? (((uint64_t)__float_as_uint(Op::post(__uint_as_float(lds32(da + 4 * lane)))) << 32) | (uint32_t)lane) : ~0ull;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const uint64_t other = __shfl_xor_sync(FULL, key, o);
            key = other < key ? other : key;
          }
          const float dmin = __uint_as_float((uint32_t)(key >> 32));
          if (dmin < best) {
            best = dmin;
            new_pivot = lds32(ca + 4 * ((uint32_t)key & 31u));
          }
        }
        if (valid != FULL) break;
      }
      pivot = new_pivot;  // hnsw.rs:1526-1528
    }

    // ---- search_layer on the lowest populated layer (hnsw.rs:1531-1542, 940-1057)
    vis.begin(p.vis, pivot, lane);  // hnsw.rs:955-956
#pragma unroll
    for (int c = 0; c < NCH; ++c) sts64(wa + 8 * (32 * c + lane), ~0ull);
    __syncwarp();
    if (lane == 0) sts64(wa, make_key(best, pivot));  // the layer's entry enters W and C (hnsw.rs:958-967)
    __syncwarp();
    if (STATS) evals += 1;  // search_layer's own evaluation of its entry point (hnsw.rs:952): the value is `best`
    int n = 1;
    MaskT open;
    open.set_only(0);
    uint64_t thr = lds64(wa + 8 * (cap - 1));
    bool overflow = false;
    // look-ahead: while the rows of an expansion are in flight, the adjacency chunk of the candidate that will be
    // popped next if no nearer one turns up (the first unexpanded entry now) and its first visited probe are loaded
    bool pre_ok = false;
    uint32_t pre_c = INVALID_ID, pre_nid = INVALID_ID, pre_h = 0, pre_cv = 0;
    while (!open.none()) {
      // C.pop(): nearest unexpanded entry of W (hnsw.rs:971); "C empty or d(c) > d(f)" == none left (search_core.cuh)
      const int idx = open.first();
      open.drop_first();
      const uint32_t c = key_id(lds64(wa + 8 * idx));
      if (STATS) expans += 1;
      int lcap;
      const uint32_t* ids = list_ids(G, c, p.layer0, lcap);  // hnsw.rs:1006
      const bool hit = pre_ok && pre_c == c;
      pre_ok = false;
      {  // pull the adjacency rows of the two candidates after the next towards L2 while this one is expanded
        MaskT o2 = open;
        o2.drop_first();
        if (lane == 1) o2.drop_first();
        if (lane < 2 && !o2.none()) {
          const uint32_t pc = key_id(lds64(wa + 8 * o2.first()));
          int pcap;
          const uint32_t* pids = list_ids(G, pc, p.layer0, pcap);
          if (pids) asm volatile("prefetch.global.L2 [%0];" ::"l"(pids));
        }
      }
      for (int b = 0; b < lcap; b += 32) {  // hnsw.rs:1013, 32 neighbours at a time
        const bool use_pre = hit && b == 0;
        uint32_t nid = pre_nid;
        if (!use_pre) nid = (b + lane < lcap) ? ids[b + lane] : INVALID_ID;
        const unsigned valid = __ballot_sync(FULL, nid != INVALID_ID);
        if (STATS) adjr += __popc(valid);
        const bool fresh = vis.test_and_set(p.vis, lane, nid, nid != INVALID_ID, use_pre, pre_h, pre_cv);  // hnsw.rs:1016-1017
        const unsigned m = __ballot_sync(FULL, fresh);
        const int cnt = __popc(m);
        const bool last = valid != FULL || b + 32 >= lcap;
        auto lookahead = [&]() {
          if (last && !open.none()) {
            pre_c = key_id(lds64(wa + 8 * open.first()));
            int pcap;
            const uint32_t* pids = list_ids(G, pre_c, p.layer0, pcap);
            pre_nid = (lane < pcap) ? pids[lane] : INVALID_ID;
            pre_h = vis.home(pre_nid);
            pre_cv = 0;
            if (pre_nid != INVALID_ID) pre_cv = vis.probe(p.vis, pre_h, l2_policy_evict_last());
            pre_ok = true;
          }
        };
        if (cnt) {
          const int at = __popc(m & ((1u << lane) - 1u));
          if (fresh) sts32(ca + 4 * at, nid);
          __syncwarp();
          // lines of the rows beyond the first pass (8 rows) -> L2
          for (int l = 8 * CH + lane; l < cnt * CH; l += 32)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(vecb + (size_t)lds32(ca + 4 * (l / CH)) * row_bytes + (uint32_t)(l % CH) * 128u));
          lean_score<Op, CH>(vecb, qv, ca, da, cnt, G.dim, g, r, pol_rows, lookahead);  // hnsw.rs:1026
          __syncwarp();
          if (STATS) evals += cnt;
          uint64_t key = ~0ull;
          if (lane < cnt) key = make_key(Op::post(__uint_as_float(lds32(da + 4 * lane))), lds32(ca + 4 * lane));
          const unsigned acc = __ballot_sync(FULL, key < thr);  // hnsw.rs:1028 (a queue that is not full has thr = ~0)
          if (acc) lean_merge<NCH>(wa, lane, key, acc, cap, n, thr, open);
        } else {
          lookahead();
        }
        if (last) break;  // lists are dense prefixes terminated by INVALID_ID
      }
      if (vis.grow_or_overflow(p.vis, lane, pre_ok)) {
        overflow = true;
        break;
      }
    }
    // ---- ascending top-k (hnsw.rs:1544-1579); the queue is already sorted
    write_answers(p, lane, qi, overflow, n < p.k ? n : p.k, [&](int j) { return lds64(wa + 8 * j); });  // hnsw.rs:1547 (n <= ef)
  }
  vis.save(p.vis, slot, lane);
  if (STATS && p.stats && lane == 0) {
    atomicAdd(p.stats + 0, (unsigned long long)evals);
    atomicAdd(p.stats + 1, (unsigned long long)expans);
    atomicAdd(p.stats + 2, (unsigned long long)adjr);
  }
}

// A launch whose `smem` holds a visited first stage asks for the largest shared-memory carveout, so that the windows do
// not cost CTAs per SM (c2: 20 CTAs x (8 960 + 1 024 reserved) bytes = 195 KB); one without leaves the split to the driver.
template <class Op, int CH, int QC>
static cudaError_t launch_lean_kernel(const SearchParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  void (*kern)(SearchParams) = p.stats ? search_lean_kernel<Op, CH, QC, true> : search_lean_kernel<Op, CH, QC, false>;
  const int carveout = smem > lean_layout(QC).bytes ? (int)cudaSharedmemCarveoutMaxShared : (int)cudaSharedmemCarveoutDefault;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
  if (e != cudaSuccess) return e;
  return launch_kernel(kern, p, grid, LEAN_THREADS, smem, st, blocks_per_sm);
}

template <class Op, int QC>
static cudaError_t launch_lean_for_op(const SearchParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  const int ch = p.g.d4 / 8;
  if (ch == 1) return launch_lean_kernel<Op, 1, QC>(p, grid, smem, st, blocks_per_sm);
  if (ch == 2) return launch_lean_kernel<Op, 2, QC>(p, grid, smem, st, blocks_per_sm);
  if (ch == 4) return launch_lean_kernel<Op, 4, QC>(p, grid, smem, st, blocks_per_sm);
  return cudaErrorInvalidValue;
}

// one translation unit per element type instantiates the kernels (search_lean_f32.cu, search_lean_u8.cu, search_lean_u16.cu)
template <class Op>
static cudaError_t launch_lean_op(const SearchParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  if (p.q_smem == 64) return launch_lean_for_op<Op, 64>(p, grid, smem, st, blocks_per_sm);
  if (p.q_smem == 128) return launch_lean_for_op<Op, 128>(p, grid, smem, st, blocks_per_sm);
  return cudaErrorInvalidValue;
}

}  // namespace hb
