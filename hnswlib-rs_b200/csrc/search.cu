// Query kernel: one warp per query, persistent warps pulling query indices from a counter.
// Restates /root/reference/src/hnsw.rs:1487-1580 (search_filter: entry fetch, one-hop-per-layer
// descent, layer-0 search_layer, ascending top-k extraction) and the batch contract of
// parallel_search (hnsw.rs:1612-1635: one answer per query, in input order).
#include "kernels.h"
#include "search_core.cuh"

namespace hb {

template <class Op, int CH, int U, int NS>
__global__ void __launch_bounds__(SEARCH_THREADS, 4) search_kernel(SearchParams p) {
  using Queue = typename QueueSel<NS>::type;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GraphView& g = p.g;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  const QueryLayout L = query_layout(g.d4, p.q_smem);
  const WarpSmem s{reinterpret_cast<uint4*>(base + L.query), reinterpret_cast<uint64_t*>(base + L.queue),
                   reinterpret_cast<uint32_t*>(base + L.cand_id), reinterpret_cast<float*>(base + L.cand_d)};
  Stage stg;
  stg.buf = stage_bytes(g.d4) ? reinterpret_cast<uint4*>(base + L.stage) : nullptr;
  stg.bar = reinterpret_cast<uint64_t*>(base + L.bar);
  stg.phase = 0;
  if (lane == 0) mbar_init(stg.bar, 1);
  __syncwarp();

  const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + warp;  // the host launches fewer warps per CTA when shared memory is short
  Visited vis;
  vis.init(p.vis, slot);
  Queue Q;
  Q.reset(s.wbuf, p.ef);
  Stats st{0, 0, 0};

  for (;;) {
    const uint32_t qi = next_item(p.work_counter, lane);
    if (qi >= p.nq) break;
    // stage the query (zero padded to d_pad)
    stage_row_bytes(s.q4, query_row(g, p.q_ids, p.queries, p.q_stride_bytes, qi), p.q_bytes, g.d4 * 16);
    int count = 0;
    bool overflow = false;
    if (g.entry != INVALID_ID) {  // hnsw.rs:1498-1503
      const Entry e = descend<Op>(g, lane, st, WarpChunk<Op, CH, U>{g, s, lane});
      // ---- layer-0 (lowest populated layer) search, hnsw.rs:1531-1542
      search_layer<Op, CH, U, Queue>(g, s, stg, p.vis, vis, Q, e.pivot, p.ef, p.layer0, st, overflow);
      count = min(p.k, min(p.ef, Q.n));  // hnsw.rs:1547
    }
    write_answers(p, lane, qi, overflow, count, [&](int j) { return Q.local(j); });  // the queue is already sorted
  }
  vis.save(p.vis, slot, lane);
  flush_stats(p.stats, st, lane);
}

// Compile-time row length (CH chunks of 128 bytes) only where the lean kernel cannot take the search: a 256-slot queue
// (ef 129-256) or the generic one (ef > 256).  With a 32 / 64 / 128-slot queue the generic kernel runs only on an index
// without an entry point, whose answers are empty.
template <class Op, int NS>
static cudaError_t launch_for_op(const SearchParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  const int ch = p.g.d4 / 8;
  if constexpr (Specialise<Op>::value && (NS == 0 || NS == 108)) {
    if (ch == 1) return launch_kernel(search_kernel<Op, 1, 4, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
    if (ch == 2) return launch_kernel(search_kernel<Op, 2, 4, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
    if (ch == 4) return launch_kernel(search_kernel<Op, 4, 2, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
  }
  return launch_kernel(search_kernel<Op, 0, 2, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
}

cudaError_t launch_search(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    using Op = typename decltype(tag)::type;
    if constexpr (Specialise<Op>::value) {
      if (p.q_kind == 101) return launch_for_op<Op, 101>(p, grid, smem, st, blocks_per_sm);
      if (p.q_kind == 102) return launch_for_op<Op, 102>(p, grid, smem, st, blocks_per_sm);
      if (p.q_kind == 104) return launch_for_op<Op, 104>(p, grid, smem, st, blocks_per_sm);
      if (p.q_kind == 108) return launch_for_op<Op, 108>(p, grid, smem, st, blocks_per_sm);
    }
    return launch_for_op<Op, 0>(p, grid, smem, st, blocks_per_sm);
  });
}

}  // namespace hb
