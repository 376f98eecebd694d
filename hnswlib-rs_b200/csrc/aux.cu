// Stand-alone kernels on the index's point store:
//   dist_batch_kernel  — K1: queries x candidate ids -> distances.  The batched form of
//                        Distance<T>::eval (crate anndists; call sites /root/reference/src/hnsw.rs:1026,1518).
//   bruteforce_kernel  — K5: exact k nearest neighbours by linear scan, the GPU counterpart of
//                        brute_force_neighbours in /root/reference/tests/serpar.rs:42-70 (recall ground truth).
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
  int k;
  uint32_t* out_ids;     // [nq][k]
  float* out_dist;       // [nq][k]
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

template <class Op, int CH, int U>
__global__ void __launch_bounds__(256) bruteforce_kernel(AuxParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* base = smem_raw + (size_t)warp * p.smem_per_warp;
  uint4* q4 = reinterpret_cast<uint4*>(base);
  uint32_t* cid = reinterpret_cast<uint32_t*>(base + (size_t)p.g.d4 * 16);
  float* cd = reinterpret_cast<float*>(cid + 32);
  uint64_t* wbuf = reinterpret_cast<uint64_t*>(cd + 32);
  const uint4* vec4 = reinterpret_cast<const uint4*>(p.g.vec);
  const uint32_t wstride = gridDim.x * 8;
  SortedQueue Q;
  for (uint32_t qi = blockIdx.x * 8 + warp; qi < p.nq; qi += wstride) {
    __syncwarp();
    stage_row_bytes(q4, reinterpret_cast<const char*>(p.queries) + (size_t)qi * p.q_bytes, p.q_bytes, p.g.d4 * 16);
    Q.reset(wbuf, p.k);
    for (uint32_t b = 0; b < p.g.n; b += 32) {
      const int cnt = min(32u, p.g.n - b);
      cid[lane] = b + lane;
      __syncwarp();
      warp_dists<Op, CH, U>(vec4, p.g.d4, p.g.dim, q4, cid, cnt, cd);
      __syncwarp();
      const uint64_t key = lane < cnt ? make_key(Op::post(cd[lane]), b + lane) : ~0ull;
      unsigned acc = __ballot_sync(FULL, lane < cnt && Q.accepts(key));
      while (acc) {
        const int j = __ffs(acc) - 1;
        acc &= acc - 1;
        const uint64_t kj = __shfl_sync(FULL, key, j);
        if (Q.accepts(kj)) Q.insert(kj);
      }
      __syncwarp();
    }
    for (int j = lane; j < p.k; j += 32) {
      p.out_ids[(size_t)qi * p.k + j] = j < Q.n ? key_id(Q.w[j]) : INVALID_ID;
      p.out_dist[(size_t)qi * p.k + j] = j < Q.n ? key_dist(Q.w[j]) : __int_as_float(0x7f800000);
    }
  }
}

template <class Op, int CH, int U>
static cudaError_t launch_aux_kernel(const AuxParams& p, bool brute, int grid, size_t smem, cudaStream_t st) {
  return launch_kernel(brute ? bruteforce_kernel<Op, CH, U> : dist_batch_kernel<Op, CH, U>, p, grid, 256, smem, st, nullptr);
}

template <class Op>
static cudaError_t launch_aux_for_op(const AuxParams& p, bool brute, int grid, size_t smem, cudaStream_t st) {
  const int ch = p.g.d4 / 8;
  if constexpr (Specialise<Op>::value) {
    if (ch == 1) return launch_aux_kernel<Op, 1, 4>(p, brute, grid, smem, st);
    if (ch == 4) return launch_aux_kernel<Op, 4, 2>(p, brute, grid, smem, st);
  }
  return launch_aux_kernel<Op, 0, 2>(p, brute, grid, smem, st);
}

static cudaError_t launch_aux(const AuxParams& p, int metric, int dtype, bool brute, int grid, size_t smem, cudaStream_t st) {
  return dispatch_op(metric, dtype, [&](auto tag) -> cudaError_t {
    using Op = typename decltype(tag)::type;
    return launch_aux_for_op<Op>(p, brute, grid, smem, st);
  });
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
  HB_CUDA(launch_aux(p, metric, dtype, false, grid, smem, stream_));
  HB_CUDA(cudaMemcpyAsync(out, dout.p, nq * m * 4, cudaMemcpyDeviceToHost, stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  return 0;
}

int Index::bruteforce(const void* queries, size_t nq, int d, size_t k, uint32_t* out_ids, float* out_dist) {
  if (nq == 0 || k == 0) return 0;
  if (d != dim) return fail("query length differs from the index dimension");
  AuxParams p{};
  p.g = view();
  p.q_bytes = d * es;
  p.nq = (uint32_t)nq;
  p.k = (int)k;
  p.smem_per_warp = (int)(((size_t)p.g.d4 * 16 + 256 + k * 8 + 15) & ~(size_t)15);
  const size_t smem = (size_t)p.smem_per_warp * 8;  // the kernel indexes its 8 warps itself
  if (smem > SMEM_BUDGET) return fail("k / dimension too large for the brute-force kernel");
  HB_CUDA(cudaSetDevice(device));
  DevBuf dq, dids, dd;
  HB_CUDA(cudaMalloc(&dq.p, nq * d * es));
  HB_CUDA(cudaMalloc(&dids.p, nq * k * 4));
  HB_CUDA(cudaMalloc(&dd.p, nq * k * 4));
  HB_CUDA(cudaMemcpyAsync(dq.p, queries, nq * d * es, cudaMemcpyHostToDevice, stream_));
  p.queries = dq.p;
  p.out_ids = (uint32_t*)dids.p;
  p.out_dist = (float*)dd.p;
  const int grid = (int)std::min<size_t>((size_t)sm_count_ * 4, (nq + 7) / 8);
  HB_CUDA(launch_aux(p, metric, dtype, true, grid, smem, stream_));
  HB_CUDA(cudaMemcpyAsync(out_ids, dids.p, nq * k * 4, cudaMemcpyDeviceToHost, stream_));
  HB_CUDA(cudaMemcpyAsync(out_dist, dd.p, nq * k * 4, cudaMemcpyDeviceToHost, stream_));
  HB_CUDA(cudaStreamSynchronize(stream_));
  return 0;
}

}  // namespace hb
