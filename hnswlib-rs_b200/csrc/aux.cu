// Stand-alone kernels on the index's point store:
//   dist_batch_kernel — K1: queries x candidate ids -> distances.  The batched form of
//                       Distance<T>::eval (crate anndists; call sites /root/reference/src/hnsw.rs:1026,1518).
//   exact_knn_kernel  — K5: exact k nearest neighbours of a batch over every stored point or a sorted id list, the GPU
//                       counterpart of brute_force_neighbours in /root/reference/tests/serpar.rs:42-70 (recall ground
//                       truth), and the exact search over a resident filter (hnsw_b200_search_exact).
#include "index.h"
#include "kernels.h"

namespace hb {

struct AuxParams {
  GraphView g;
  const void* queries;  // [nq][q_bytes] raw element bytes
  int q_bytes;
  uint32_t nq;
  const uint32_t* cand;  // [nq][m]
  uint32_t m;
  float* out;            // [nq][m]
  int smem_per_warp;
};

template <class Op, int CH, int U>
__global__ void __launch_bounds__(256) dist_batch_kernel(AuxParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  uint4* q4 = reinterpret_cast<uint4*>(base);
  uint32_t* cid = reinterpret_cast<uint32_t*>(base + (size_t)p.g.d4 * 16);
  float* cd = reinterpret_cast<float*>(cid + 32);
  const uint4* vec4 = reinterpret_cast<const uint4*>(p.g.vec);
  const uint32_t wstride = gridDim.x * 8;
  for (uint32_t qi = blockIdx.x * 8 + warp; qi < p.nq; qi += wstride) {
    __syncwarp();
    stage_row_bytes(q4, reinterpret_cast<const char*>(p.queries) + (size_t)qi * p.q_bytes, p.q_bytes, p.g.d4 * 16);
    for (uint32_t b = 0; b < p.m; b += 32) {
      const int cnt = min(32u, p.m - b);
      if (lane < cnt) cid[lane] = p.cand[(size_t)qi * p.m + b + lane];
      __syncwarp();
      warp_dists<Op, CH, U>(vec4, p.g.d4, p.g.dim, q4, cid, cnt, cd);
      __syncwarp();
      if (lane < cnt) p.out[(size_t)qi * p.m + b + lane] = Op::post(cd[lane]);
      __syncwarp();
    }
  }
}

template <class Op>
static cudaError_t launch_dist_batch_for_op(const AuxParams& p, int grid, size_t smem, cudaStream_t st) {
  const int ch = p.g.d4 / 8;
  if constexpr (Specialise<Op>::value) {
    if (ch == 1) return launch_kernel(dist_batch_kernel<Op, 1, 4>, p, grid, 256, smem, st, nullptr);
    if (ch == 4) return launch_kernel(dist_batch_kernel<Op, 4, 2>, p, grid, 256, smem, st, nullptr);
  }
  return launch_kernel(dist_batch_kernel<Op, 0, 2>, p, grid, 256, smem, st, nullptr);
}

// ------------------------------------------------------------------------------------------------ exact k-NN scan
// A CTA owns a tile of tq queries (staged once in shared memory, zero padded) and one slice of the point list, which it
// streams through a ring of `stages` blocks of `rows` rows, one cp.async.bulk per row.  Every staged row is scored
// against every query of the tile by an 8-lane group with warp_dists' lane / chunk order, so each distance is
// bit-identical to warp_dists'.  A key that beats its query's threshold goes to a per-query candidate list; after each
// block the warp that owns the query (query % 8) merges the list into the query's sorted queue.  With slices > 1 every
// CTA leaves its top k in `part` and the last CTA of a tile to finish (ticket) merges the slices' lists.
struct ExactParams {
  GraphView g;
  const void* queries;   // device, [nq][q_bytes] raw element bytes
  int q_bytes;
  uint32_t nq;
  const uint32_t* list;  // sorted internal ids, or nullptr: the points 0 .. npts - 1
  uint32_t npts;
  int k;
  int tq, rows, stages;  // queries per tile, rows per ring block (divides 32), ring blocks
  int slices;            // CTAs per tile, each over a contiguous part of the point list
  uint64_t* part;        // slices > 1: [tiles][slices][tq][k] keys (~0 = none)
  unsigned* tickets;     // slices > 1: [tiles], zero at launch; the merging CTA leaves them zero
  NeighbourOut* out;     // [nq][k]
  int32_t* counts;       // [nq]
  const ExactTile* tiles;  // nullptr: tile t is queries [t * tq, t * tq + tq) over (list, npts); else tile t is tiles[t]
};

// keys[0, c) (~0 = none) into the warp's sorted queue Q, 32 at a time: those Q accepts, inserted in lane order.  The keys
// are in shared memory, or (global) in global memory written by other CTAs, read from L2.
__device__ __forceinline__ void queue_offer(SortedQueue& Q, const uint64_t* keys, int c, bool global) {
  const int lane = lane_id();
  for (int base = 0; base < c; base += 32) {
    const bool in = base + lane < c;
    const uint64_t key = !in ? ~0ull : global ? __ldcg(reinterpret_cast<const unsigned long long*>(keys) + base + lane) : keys[base + lane];
    unsigned acc = __ballot_sync(FULL, in && key != ~0ull && Q.accepts(key));
    while (acc) {
      const int j = __ffs(acc) - 1;
      acc &= acc - 1;
      const uint64_t kj = __shfl_sync(FULL, key, j);
      if (Q.accepts(kj)) Q.insert(kj);
    }
  }
  __syncwarp();
}

template <class Op, int CH>
__global__ void __launch_bounds__(256, 2) exact_knn_kernel(ExactParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ int last_cta;
  const int d4 = p.g.d4, tq = p.tq, B = p.rows, NS = p.stages, k = p.k;
  const ExactLayout L = exact_layout(d4, k, tq, B, NS);
  uint4* qs = reinterpret_cast<uint4*>(smem_raw + L.query);
  uint4* ring = reinterpret_cast<uint4*>(smem_raw + L.ring);
  uint64_t* queue = reinterpret_cast<uint64_t*>(smem_raw + L.queue);
  uint64_t* cand = reinterpret_cast<uint64_t*>(smem_raw + L.cand);
  uint64_t* thr = reinterpret_cast<uint64_t*>(smem_raw + L.thr);
  int* ccount = reinterpret_cast<int*>(smem_raw + L.ccount);
  int* qn = reinterpret_cast<int*>(smem_raw + L.qn);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + L.bar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tile = blockIdx.x / p.slices, slice = blockIdx.x % p.slices;
  uint32_t q0 = tile * tq, npts = p.npts;
  int nqt = (int)min((uint32_t)tq, p.nq - q0);
  const uint32_t* list = p.list;
  if (p.tiles) {  // a tile of its own size over its own points; its slices split those points
    const ExactTile t = p.tiles[tile];
    q0 = t.q0;
    nqt = (int)t.nq;
    list = t.list;
    npts = t.npts;
  }
  const uint32_t per = (npts + p.slices - 1) / p.slices;
  const uint32_t lo = min(npts, slice * per), hi = min(npts, lo + per);
  const uint32_t nblk = (hi - lo + B - 1) / B;
  const uint32_t row_bytes = (uint32_t)d4 * 16u;
  const uint4* vec4 = reinterpret_cast<const uint4*>(p.g.vec);

  if (threadIdx.x == 0)
    for (int s = 0; s < NS; ++s) mbar_init(bar + s, 1);
  for (int q = warp; q < tq; q += 8)
    stage_row_bytes(qs + (size_t)q * d4, reinterpret_cast<const char*>(p.queries) + (size_t)(q < nqt ? q0 + q : 0) * p.q_bytes,
                    q < nqt ? p.q_bytes : 0, (int)row_bytes);
  for (int q = threadIdx.x; q < tq; q += blockDim.x) {
    thr[q] = ~0ull;
    ccount[q] = 0;
    qn[q] = 0;
  }
  __syncthreads();

  // warp 0: block b of the slice into ring slot b % NS, one bulk copy per row (lane i: row i)
  auto issue = [&](uint32_t b) {
    const uint32_t first = lo + b * B;
    const int cnt = (int)min((uint32_t)B, hi - first);
    uint64_t* br = bar + b % NS;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the slot's earlier generic reads precede the async writes
    if (lane == 0) mbar_expect_tx(br, row_bytes * cnt);
    __syncwarp();
    if (lane < cnt) {
      const uint32_t id = list ? __ldg(list + first + lane) : first + lane;
      bulk_g2s(ring + ((size_t)(b % NS) * B + lane) * d4, vec4 + (size_t)id * d4, row_bytes, br, l2_policy_evict_first());
    }
  };
  if (warp == 0)
    for (uint32_t b = 0; b < nblk && b < (uint32_t)NS; ++b) issue(b);

  // 8-lane group `grp` scores row rs of each block against queries ph, ph + nph, ... (a warp-uniform trip count)
  const int grp = threadIdx.x >> 3, g = lane & 7;
  const int rs = grp % B, ph = grp / B, nph = 32 / B;
  const int qsteps = (tq + nph - 1) / nph;
  for (uint32_t b = 0; b < nblk; ++b) {
    const int slot = (int)(b % NS);
    mbar_wait(bar + slot, (b / NS) & 1u);
    const uint32_t first = lo + b * B;
    const bool row_ok = rs < (int)min((uint32_t)B, hi - first);
    const uint32_t id = !row_ok ? 0u : list ? __ldg(list + first + rs) : first + rs;
    const uint4* row = ring + ((size_t)slot * B + (row_ok ? rs : 0)) * d4 + g;
    uint4 x[CH > 0 ? CH : 1];
    if constexpr (CH > 0) {
#pragma unroll
      for (int i = 0; i < CH; ++i) x[i] = row[8 * i];
    }
    for (int j = 0; j < qsteps; ++j) {
      const int q = ph + j * nph;
      const uint4* qv = qs + (size_t)(q < tq ? q : 0) * d4 + g;
      typename Op::acc_t a = Op::zero();
      if constexpr (CH > 0) {
#pragma unroll
        for (int i = 0; i < CH; ++i) Op::chunk(a, qv[8 * i], x[i]);
      } else {
        const int nch = d4 >> 3;
#pragma unroll 4
        for (int i = 0; i < nch; ++i) Op::chunk(a, qv[8 * i], row[8 * i]);
      }
      const float dist = reduce8<Op>(a, p.g.dim);
      if (g == 0 && row_ok && q < nqt) {
        const uint64_t key = make_key(Op::post(dist), id);
        if (key < thr[q]) cand[q * B + atomicAdd(&ccount[q], 1)] = key;
      }
    }
    __syncthreads();  // the slot is read and the candidates are in
    if (warp == 0 && b + NS < nblk) issue(b + NS);
    for (int q = warp; q < nqt; q += 8) {
      const int c = ccount[q];
      if (c == 0) continue;
      SortedQueue Q;
      Q.w = queue + (size_t)q * k;
      Q.n = qn[q];
      Q.cap = k;
      queue_offer(Q, cand + q * B, c, false);
      if (lane == 0) {
        qn[q] = Q.n;
        thr[q] = Q.n < k ? ~0ull : Q.w[k - 1];
        ccount[q] = 0;
      }
    }
    __syncthreads();
  }

  // answers: (origin, distance, internal id) for the first n keys, then (~0, +inf, INVALID_ID)
  auto write = [&](int q, const uint64_t* w, int n) {
    NeighbourOut* o = p.out + (size_t)(q0 + q) * k;
    for (int j = lane; j < k; j += 32) {
      if (j < n) {
        const uint32_t it = key_id(w[j]);
        o[j] = NeighbourOut{p.g.origin[it], key_dist(w[j]), it};
      } else {
        o[j] = NeighbourOut{~0ull, __int_as_float(0x7f800000), INVALID_ID};
      }
    }
    if (lane == 0) p.counts[q0 + q] = n;
  };
  if (p.slices == 1) {
    for (int q = warp; q < nqt; q += 8) write(q, queue + (size_t)q * k, qn[q]);
    return;
  }
  uint64_t* tile_part = p.part + (size_t)tile * p.slices * tq * k;
  for (int q = warp; q < nqt; q += 8)
    for (int j = lane; j < k; j += 32) tile_part[((size_t)slice * tq + q) * k + j] = j < qn[q] ? queue[(size_t)q * k + j] : ~0ull;
  __threadfence();  // this slice's list is visible before its ticket
  __syncthreads();
  if (threadIdx.x == 0) last_cta = atomicAdd(p.tickets + tile, 1u) == (unsigned)p.slices - 1;
  __syncthreads();
  if (!last_cta) return;
  __threadfence();  // every other slice's list is read after its ticket
  for (int q = warp; q < nqt; q += 8) {
    SortedQueue Q;
    Q.reset(queue + (size_t)q * k, k);
    for (int s = 0; s < p.slices; ++s) queue_offer(Q, tile_part + ((size_t)s * tq + q) * k, k, true);
    write(q, Q.w, Q.n);
  }
  if (threadIdx.x == 0) p.tickets[tile] = 0;
}

template <class Op>
static cudaError_t launch_exact_for_op(const ExactParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  const int ch = p.g.d4 / 8;
  if constexpr (Specialise<Op>::value) {
    if (ch == 1) return launch_kernel(exact_knn_kernel<Op, 1>, p, grid, 256, smem, st, blocks_per_sm);
    if (ch == 4) return launch_kernel(exact_knn_kernel<Op, 4>, p, grid, 256, smem, st, blocks_per_sm);
  }
  return launch_kernel(exact_knn_kernel<Op, 0>, p, grid, 256, smem, st, blocks_per_sm);
}

// The tile and ring of a launch: the whole tile (up to 32 queries) with a ring of >= 8 rows inside half of SMEM_BUDGET
// (two CTAs per SM) if possible, else the largest tile and ring that fit SMEM_BUDGET.  False if not even one query with
// a two-row ring fits.
static bool exact_shape(int d4, size_t k, size_t nq, ExactParams& p, size_t& smem) {
  static const int RING[][2] = {{32, 3}, {32, 2}, {16, 2}, {8, 2}, {4, 2}, {2, 2}, {1, 2}};
  const int tq_max = (int)std::min<size_t>(32, nq);
  for (int pass = 0; pass < 2; ++pass) {
    const size_t budget = pass == 0 ? SMEM_BUDGET / 2 : SMEM_BUDGET;
    for (int tq = tq_max; tq >= 1; tq = pass == 0 ? 0 : tq / 2)
      for (const auto& r : RING) {
        if (pass == 0 && r[0] < 8) break;
        const size_t b = exact_layout(d4, (int)k, tq, r[0], r[1]).bytes;
        if (b > budget) continue;
        p.tq = tq;
        p.rows = r[0];
        p.stages = r[1];
        smem = b;
        return true;
      }
  }
  return false;
}

int Index::exact_on_ctx(SearchCtx& c, const void* d_queries, size_t nq, size_t k, const ExactScan& scan, NeighbourOut* d_out,
                        int32_t* d_counts, bool sync, float* kernel_ms, const std::vector<ExactGroup>* groups) {
  if (k == 0) return fail("knbn must be positive");
  if (poisoned_) return fail(poison_msg_);
  cudaStream_t st = c.stream;
  if (dim == 0) {  // empty index: every answer is empty
    HB_CUDA(cudaMemsetAsync(d_counts, 0, nq * sizeof(int32_t), st));
    if (sync) HB_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
  ExactParams p{};
  p.g = view();
  p.queries = d_queries;
  p.q_bytes = dim * es;
  p.nq = (uint32_t)nq;
  p.list = scan.ids;
  p.npts = (uint32_t)(scan.ids ? scan.n : n);
  p.k = (int)k;
  size_t widest_group = nq;
  if (groups) {
    widest_group = 0;
    for (const ExactGroup& gr : *groups) widest_group = std::max(widest_group, gr.count);
  }
  size_t smem = 0;
  if (!exact_shape(p.g.d4, k, widest_group, p, smem)) return fail("k / dimension too large for the exact search kernel");
  auto launch = [&](int grid, int* blocks_per_sm) {
    return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
      return launch_exact_for_op<typename decltype(tag)::type>(p, grid, smem, st, blocks_per_sm);
    });
  };
  // groups: tiles of up to tq rows of one group each, every tile over its group's points
  std::vector<ExactTile> tl;
  if (groups)
    for (const ExactGroup& gr : *groups)
      for (size_t q = 0; q < gr.count; q += p.tq)
        tl.push_back(ExactTile{(uint32_t)(gr.first + q), (uint32_t)std::min<size_t>(p.tq, gr.count - q), gr.scan.ids,
                               (uint32_t)(gr.scan.ids ? gr.scan.n : n)});
  const size_t tiles = groups ? tl.size() : (nq + p.tq - 1) / p.tq;
  if (tiles == 0) return 0;
  double mean = p.npts, widest = p.npts;  // points a tile scans: on average, and at most
  if (groups) {
    mean = widest = 0;
    for (const ExactTile& t : tl) {
      mean += t.npts;
      widest = std::max(widest, (double)t.npts);
    }
    mean /= (double)tiles;
  }
  // slices: the CTAs of a launch run in waves of `slots` (CTAs per SM x SMs), and a CTA's time is about its share of its
  // tile's points.  S minimises the launch time in units of one unsplit CTA over the widest tile: the waves the tiles
  // fill, each as long as a slice of the mean tile, but no less than one slice of the widest tile,
  //   cost(S) = max(ceil(tiles * S / slots) * mean, widest) / (S * widest).
  // With equal tiles that is waves / S (few queries: S ~ slots / tiles; a tile count just above a whole number of waves:
  // a few slices even out the last wave); with a filter per query one wide tile among narrow ones is split while the
  // narrow ones fill the waves.  Each slice of the widest tile keeps >= 1024 points, and the smallest S within 2 % of the
  // best is taken, since every slice adds a list to merge.
  int bps = 0;
  HB_CUDA(launch(0, &bps));
  if (bps < 1) return fail("exact search kernel does not fit on an SM");
  const size_t slots = (size_t)sm_count_ * bps;
  const size_t smax = std::max<size_t>(1, std::min<size_t>((size_t)widest / 1024, 4 * slots));
  auto cost = [&](size_t S) {
    return widest <= 0 ? 1.0 / (double)S
                       : std::max((double)((tiles * S + slots - 1) / slots) * mean, widest) / ((double)S * widest);
  };
  double best = cost(1);
  for (size_t S = 2; S <= smax; ++S) best = std::min(best, cost(S));
  p.slices = 1;
  while (cost(p.slices) > best * 1.02) ++p.slices;
  // scratch: [tile table][tickets][slice lists]
  const size_t tile_bytes = round128(tl.size() * sizeof(ExactTile));
  const size_t tick_bytes = p.slices > 1 ? round128(tiles * 4) : 0;
  const size_t part_bytes = p.slices > 1 ? tiles * p.slices * p.tq * k * 8 : 0;
  if (tile_bytes + tick_bytes + part_bytes) {
    int r;
    if ((r = ensure_scratch(&c.d_xpart, &c.d_xpart_bytes, tile_bytes + tick_bytes + part_bytes, st))) return r;
  }
  if (groups) {
    p.tiles = (const ExactTile*)c.d_xpart;
    HB_CUDA(cudaMemcpyAsync(c.d_xpart, tl.data(), tl.size() * sizeof(ExactTile), cudaMemcpyHostToDevice, st));
  }
  if (p.slices > 1) {
    p.tickets = (unsigned*)((char*)c.d_xpart + tile_bytes);
    p.part = (uint64_t*)((char*)c.d_xpart + tile_bytes + tick_bytes);
    HB_CUDA(cudaMemsetAsync(p.tickets, 0, tiles * 4, st));
  }
  p.out = d_out;
  p.counts = d_counts;
  HB_CUDA(cudaEventRecord(c.ev0, st));
  HB_CUDA(launch((int)(tiles * p.slices), nullptr));
  HB_CUDA(cudaEventRecord(c.ev1, st));
  if (sync) {
    HB_CUDA(cudaStreamSynchronize(st));
    if (kernel_ms) HB_CUDA(cudaEventElapsedTime(kernel_ms, c.ev0, c.ev1));
  }
  return 0;
}
int Index::dist_batch(const void* queries, size_t nq, int d, const uint32_t* cand, size_t m, float* out) {
  if (nq == 0 || m == 0) return 0;
  if (d != dim) return fail("query length differs from the index dimension");
  for (size_t i = 0; i < nq * m; ++i)
    if (cand[i] >= n) return fail("candidate id out of range");
  HB_CUDA(cudaSetDevice(device));
  DevBuf dq, dc, dout;
  HB_CUDA(cudaMalloc(&dq.p, nq * d * es));
  HB_CUDA(cudaMalloc(&dc.p, nq * m * 4));
  HB_CUDA(cudaMalloc(&dout.p, nq * m * 4));
  HB_CUDA(cudaMemcpyAsync(dq.p, queries, nq * d * es, cudaMemcpyHostToDevice, stream_));
  HB_CUDA(cudaMemcpyAsync(dc.p, cand, nq * m * 4, cudaMemcpyHostToDevice, stream_));
  AuxParams p{};
  p.g = view();
  p.queries = dq.p;
  p.q_bytes = d * es;
  p.nq = (uint32_t)nq;
  p.cand = (const uint32_t*)dc.p;
  p.m = (uint32_t)m;
  p.out = (float*)dout.p;
  p.smem_per_warp = p.g.d4 * 16 + 256;
  const size_t smem = (size_t)p.smem_per_warp * 8;
  const int grid = (int)std::min<size_t>((size_t)sm_count_ * 8, (nq + 7) / 8);
  HB_CUDA(dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    return launch_dist_batch_for_op<typename decltype(tag)::type>(p, grid, smem, stream_);
  }));
  HB_CUDA(cudaMemcpyAsync(out, dout.p, nq * m * 4, cudaMemcpyDeviceToHost, stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  return 0;
}

// the exact scan over every stored point, through the host batch driver; internal ids and distances only
int Index::bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist) {
  if (nq == 0 || k == 0) return 0;
  if (d != dim) return fail("query length differs from the index dimension");
  std::vector<int32_t> counts(nq);
  HostBatch b;
  b.queries = queries;
  b.nq = nq;
  b.d = d;
  b.k = k;
  b.exact = true;
  b.out.internal = out_ids;
  b.out.dist = out_dist;
  b.out.counts = counts.data();
  return search_batch(b);
}

}  // namespace hb
