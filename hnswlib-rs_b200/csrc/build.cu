// Batched insert kernels.  One warp owns one new point.
//   phase A (insert_search_kernel): upper-layer ef=1 descent, per-layer search_layer(ef_construction),
//            heuristic neighbour selection, write of the new point's own lists
//            == /root/reference/src/hnsw.rs:1110-1205 (insert_slice) + 1299-1421 (select_neighbours)
//   phase B (insert_link_kernel): reverse links under a per-point lock
//            == /root/reference/src/hnsw.rs:1241-1289 (reverse_update_neighborhood_simple),
//            including its quirk that every back-link is filed under the NEW point's level (1257); with
//            link mode 1 (hnsw_b200_set_link_mode) each back-link is filed in the layer it was made in instead.
// The reference races inserts under parking_lot locks on a rayon pool (hnsw.rs:1224-1238); here a
// batch of inserts searches the graph as it stood at the start of the batch (phase A is read-only
// on other points' lists) and links afterwards; see DESIGN.md "batched insert".
#include "kernels.h"
#include "search_core.cuh"

namespace hb {

// dists from the vector of point `e` to kept[0..cnt): stage e's row as the "query"
template <class Op, int CH, int U>
__device__ __forceinline__ void dists_from_point(const GraphView& g, uint4* qe4, uint32_t e, const uint32_t* kept,
                                                 int cnt, float* out) {
  const uint4* vec4 = reinterpret_cast<const uint4*>(g.vec);
  const int lane = lane_id();
  __syncwarp();
  for (int i = lane; i < g.d4; i += 32) qe4[i] = __ldg(vec4 + (size_t)e * g.d4 + i);
  __syncwarp();
  warp_dists<Op, CH, U>(vec4, g.d4, g.dim, qe4, kept, cnt, out);
  __syncwarp();
}

template <class Op, int CH, int U, int NS>
__global__ void __launch_bounds__(BUILD_THREADS) insert_search_kernel(InsertParams p) {
  using Queue = typename QueueSel<NS>::type;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GraphView& g = p.g;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  const InsertLayout L = insert_layout(g.d4, p.ef_c, g.deg0, p.q_smem);
  const WarpSmem s{reinterpret_cast<uint4*>(base + L.query), reinterpret_cast<uint64_t*>(base + L.queue),
                   reinterpret_cast<uint32_t*>(base + L.cand_id), reinterpret_cast<float*>(base + L.cand_d)};
  Stage stg;
  stg.buf = stage_bytes(g.d4) ? reinterpret_cast<uint4*>(base + L.stage) : nullptr;
  stg.bar = reinterpret_cast<uint64_t*>(base + L.bar);
  stg.phase = 0;
  if (lane == 0) mbar_init(stg.bar, 1);
  __syncwarp();
  uint4* qe4 = reinterpret_cast<uint4*>(base + L.point);
  uint32_t* sel_id = reinterpret_cast<uint32_t*>(base + L.sel_id);
  float* sel_d = reinterpret_cast<float*>(base + L.sel_d);
  float* tmp = reinterpret_cast<float*>(base + L.tmp);
  uint16_t* disc = reinterpret_cast<uint16_t*>(base + L.disc);

  const uint32_t slot = blockIdx.x * (blockDim.x >> 5) + warp;
  Visited vis;
  vis.init(p.vis, slot);
  Queue Q;
  Q.reset(s.wbuf, p.ef_c);
  Stats st{0, 0, 0};
  const uint4* vec4 = reinterpret_cast<const uint4*>(g.vec);

  for (;;) {
    const uint32_t wi = next_item(p.work_counter, lane);
    if (wi >= p.count) break;
    const uint32_t x = p.first + wi;
    const int lv = g.level[x];
    const unsigned mask = p.layer_mask[wi];
    for (int i = lane; i < g.d4; i += 32) s.q4[i] = __ldg(vec4 + (size_t)x * g.d4 + i);
    __syncwarp();

    bool overflow = false;
    uint32_t cur = g.entry;
    WarpChunk<Op, CH, U>{g, s, lane}.score(cur, 1);  // dist_to_entry, hnsw.rs:1110-1112
    float dist_to_entry = Op::post(s.cand_d[0]);
    // ---- layers above the new point's level: ef = 1 (hnsw.rs:1114-1155).  The reference also pushes
    // the result into new_point.neighbours[l] for l above its level (1140-1144); that list can never
    // be traversed (DESIGN.md "lists above a point's level") and is not materialised.
    for (int l = g.entry_level; l > lv; --l) {
      if (!((mask >> l) & 1u)) continue;  // points_by_layer[l].is_empty() => empty result (942-946)
      search_layer<Op, CH, U, Queue>(g, s, stg, p.vis, vis, Q, cur, 1, l, st, overflow);
      if (overflow) break;
      const uint64_t k0 = Q.get(0);
      const float t = key_dist(k0);  // == dist(data, ep) recomputed at 1146
      if (t < dist_to_entry) {       // 1147-1150
        cur = key_id(k0);
        dist_to_entry = t;
      }
    }
    // ---- layers level..0: ef_construction search + selection (hnsw.rs:1158-1205)
    for (int l = lv; l >= 0 && !overflow; --l) {
      if (!((mask >> l) & 1u)) continue;
      search_layer<Op, CH, U, Queue>(g, s, stg, p.vis, vis, Q, cur, p.ef_c, l, st, overflow);
      if (overflow) break;
      const int n = Q.n;
      const int nb = (l == 0) ? g.deg0 : g.M;  // 1177-1183
      int cnt = 0;
      // extend_candidates (1318-1362, layer 0 only): with |cand| <= nb the reference adds the neighbours of the
      // candidates that are not candidates themselves, then runs the heuristic instead of taking everything.
      // When |cand| < ef_construction the search ended because every reachable node was visited, accepted
      // (|W| < ef) and expanded, so those neighbours are all candidates already and the extension set is
      // empty; the host only allows the flag when ef_construction > 2*max_nb_connection >= |cand|.
      const bool heuristic_on_few = p.extend && l == 0;
      if (n <= nb && !heuristic_on_few) {
        // 1318-1327: few candidates, take them all nearest first
        for (int i = lane; i < n; i += 32) {
          const uint64_t k = Q.local(i);
          sel_id[i] = key_id(k);
          sel_d[i] = key_dist(k);
        }
        cnt = n;
        __syncwarp();
      } else {
        int ndisc = 0;
        for (int i = 0; i < n && cnt < nb; ++i) {  // 1365: pop nearest while |out| < nb
          const uint64_t k = Q.get(i);
          const uint32_t e = key_id(k);
          const float de = key_dist(k);
          bool keep = true;
          if (cnt > 0) {  // 1372-1376: reject when some kept d has dist(e,d) <= dist(e,q)
            dists_from_point<Op, CH, U>(g, qe4, e, sel_id, cnt, tmp);
            st.evals += cnt;
            for (int b = 0; b < cnt; b += 32) {
              const bool bad = (b + lane < cnt) && (Op::post(tmp[b + lane]) <= de);
              if (__any_sync(FULL, bad)) {
                keep = false;
                break;
              }
            }
          }
          __syncwarp();
          if (keep) {
            if (lane == 0) {
              sel_id[cnt] = e;
              sel_d[cnt] = de;
            }
            cnt++;
          } else if (p.keep_pruned) {  // 1387-1392
            if (lane == 0) disc[ndisc] = (uint16_t)i;
            ndisc++;
          }
          __syncwarp();
        }
        if (p.keep_pruned && cnt < nb && ndisc > 0) {
          // 1399-1409: back-fill with the nearest discarded ones, then the caller sorts (1195).
          // Kept and discarded are both ascending sub-sequences of Q, so a merge by key restores order.
          const int take = min(ndisc, nb - cnt);
          // serial merge, executed uniformly by the warp (take <= nb, rare option); lane 0 writes
          {
            int a = cnt - 1, b = take - 1, o = cnt + take - 1;
            while (b >= 0) {
              const uint64_t kb = Q.get(disc[b]) & ~1ull;
              const bool from_a = a >= 0 && make_key(sel_d[a], sel_id[a]) > kb;
              __syncwarp();
              if (lane == 0) {
                sel_id[o] = from_a ? sel_id[a] : key_id(kb);
                sel_d[o] = from_a ? sel_d[a] : key_dist(kb);
              }
              __syncwarp();
              if (from_a) --a; else --b;
              --o;
            }
          }
          cnt += take;
          __syncwarp();
        }
      }
      // own list of layer l (hnsw.rs:1197), ascending, INVALID padded
      const List own = list_at(g, x, l);
      for (int i = lane; i < own.cap; i += 32) {
        own.ids[i] = i < cnt ? sel_id[i] : INVALID_ID;
        own.dists[i] = i < cnt ? sel_d[i] : 0.f;
      }
      if (cnt > 0) cur = sel_id[0];  // 1201-1203
      __syncwarp();
    }
    if (overflow && lane == 0) atomicExch(p.status, 1);
  }
  vis.save(p.vis, slot, lane);
  flush_stats(p.stats, st, lane);
}

// ------------------------------------------------------------------------------------------------
// phase B
__device__ __forceinline__ void lock_point(int* locks, uint32_t q) {
  if (lane_id() == 0) {
    while (atomicCAS(locks + q, 0, 1) != 0) {
      __nanosleep(64);
    }
    __threadfence();
  }
  __syncwarp();
}
__device__ __forceinline__ void unlock_point(int* locks, uint32_t q) {
  __syncwarp();
  if (lane_id() == 0) {
    __threadfence();
    atomicExch(locks + q, 0);
  }
  __syncwarp();
}

// add (x, d) to the sorted list ids/ds of capacity cap; drop the farthest when over capacity
// (push + sort_unstable + pop, hnsw.rs:1268-1284).  Warp-collective, list is locked.
__device__ __forceinline__ void list_add_sorted(uint32_t* ids, float* ds, int cap, uint32_t x, float d) {
  const int lane = lane_id();
  const uint64_t key = make_key(d, x);
  int n = 0, pos = 0;
  bool already = false;
  for (int b = 0; b < cap; b += 32) {
    const int i = b + lane;
    uint32_t id = INVALID_ID;
    float di = 0.f;
    if (i < cap) {
      id = __ldcg(ids + i);
      di = __ldcg(ds + i);
    }
    const bool valid = id != INVALID_ID;
    n += __popc(__ballot_sync(FULL, valid));
    pos += __popc(__ballot_sync(FULL, valid && make_key(di, id) < key));
    already |= __any_sync(FULL, valid && id == x) != 0;
  }
  if (already) return;  // hnsw.rs:1258-1267
  if (n == cap && pos == cap) return;  // pushed then popped again
  const int new_n = n < cap ? n + 1 : cap;
  int top = new_n - 1;
  while (top > pos) {
    const int lo = top - 31 > pos + 1 ? top - 31 : pos + 1;
    const int i = lo + lane;
    uint32_t vi = 0;
    float vd = 0.f;
    if (i <= top) {
      vi = __ldcg(ids + i - 1);
      vd = __ldcg(ds + i - 1);
    }
    __syncwarp();
    if (i <= top) {
      __stcg(ids + i, vi);
      __stcg(ds + i, vd);
    }
    __syncwarp();
    top = lo - 1;
  }
  if (lane == 0) {
    __stcg(ids + pos, x);
    __stcg(ds + pos, d);
  }
  __syncwarp();
}

__global__ void __launch_bounds__(BUILD_THREADS) insert_link_kernel(InsertParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GraphView& g = p.g;
  const uint32_t wstride = gridDim.x * (BUILD_THREADS / 32);
  for (uint32_t wi = blockIdx.x * (BUILD_THREADS / 32) + warp; wi < p.count; wi += wstride) {
    const uint32_t x = p.first + wi;
    const int L = g.level[x];
    for (int l = L; l >= 0; --l) {  // hnsw.rs:1248
      const List own = list_at(g, x, l);
      for (int j = 0; j < own.cap; ++j) {  // hnsw.rs:1249
        const uint32_t q = own.ids[j];
        if (q == INVALID_ID) break;
        if (q == x) continue;  // 1250
        const float d = own.dists[j];
        // target list: q.neighbours[L] with L = the NEW point's level (1257), or in link mode 1 q.neighbours[l];
        // 2*max_nb_connection slots at layer 0 (1272-1276).  Above plevel[q] it is a list no search can ever read, and
        // is not materialised.  In mode 1 q was visited at layer l, so plevel[q] >= l and the list always exists.
        const List t = list_at(g, q, p.link_mode ? l : L);
        if (!t.ids) continue;
        lock_point(p.locks, q);
        list_add_sorted(t.ids, t.dists, t.cap, x, d);
        unlock_point(p.locks, q);
      }
    }
  }
  (void)lane;
}

template <class Op, int NS>
static cudaError_t launch_insert_for_op(const InsertParams& p, int grid, size_t smem, cudaStream_t st, int* blocks_per_sm) {
  const int ch = p.g.d4 / 8;
  if constexpr (Specialise<Op>::value) {
    if (ch == 1) return launch_kernel(insert_search_kernel<Op, 1, 4, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
    if (ch == 2) return launch_kernel(insert_search_kernel<Op, 2, 4, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
    if (ch == 4) return launch_kernel(insert_search_kernel<Op, 4, 2, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
  }
  return launch_kernel(insert_search_kernel<Op, 0, 2, NS>, p, grid, p.threads, smem, st, blocks_per_sm);
}

cudaError_t launch_insert_search(const InsertParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                                 int* blocks_per_sm) {
  return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    using Op = typename decltype(tag)::type;
    if constexpr (Specialise<Op>::value) {
      if (p.q_kind == 108) return launch_insert_for_op<Op, 108>(p, grid, smem, st, blocks_per_sm);
      if (p.q_kind == 104) return launch_insert_for_op<Op, 104>(p, grid, smem, st, blocks_per_sm);
    }
    return launch_insert_for_op<Op, 0>(p, grid, smem, st, blocks_per_sm);
  });
}

cudaError_t launch_insert_link(const InsertParams& p, int grid, cudaStream_t st) {
  insert_link_kernel<<<grid, BUILD_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace hb
