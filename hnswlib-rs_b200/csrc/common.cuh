// Device-side building blocks of the H100 HNSW engine (sm_90a).
//
// Replaces, on the hot path of jean-pierreBoth/hnswlib-rs:
//   Point / PointWithOrder / PointIndexation pointer graph  (/root/reference/src/hnsw.rs:164-173,265-271,395-408)
//     -> GraphView: flat 128B-aligned point store + fixed-stride adjacency in HBM
//   Distance<T>::eval (crate anndists; call sites hnsw.rs:952,1026,1506,1518)
//     -> warp_dists<>: 8 lanes per row, float4 loads, xor-butterfly reduce
//   hashbrown visited map (hnsw.rs:955-956,1016-1017)  -> Visited: per-warp epoch-tagged open-addressing table
//   std BinaryHeap W and C (hnsw.rs:940-1053)           -> SortedQueue: one sorted array of (dist,id,expanded) keys
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace hb {

constexpr uint32_t INVALID_ID = 0xFFFFFFFFu;
constexpr unsigned FULL = 0xFFFFFFFFu;
constexpr int MAX_LAYERS = 16;  // NB_LAYER_MAX, hnsw.rs:42

enum Metric : int {
  METRIC_L1 = 0,
  METRIC_L2 = 1,
  METRIC_DOT = 2,
  METRIC_COSINE = 3,
  METRIC_HAMMING = 4,
  METRIC_JACCARD = 5,
  METRIC_HELLINGER = 6,
  METRIC_JEFFREYS = 7,
  METRIC_JENSENSHANNON = 8,
};

// ------------------------------------------------------------------------------------------------
// HBM layout of the index.  Internal id = insertion rank.  Rows of `vec` are d_pad floats
// (d rounded up to 32 floats = 128 B, zero padded) so that a row is a whole number of cache lines
// and 8 lanes x float4 cover exactly one line.
// Layer 0 adjacency: adj0[id][deg0] (deg0 = 2*max_nb_connection), INVALID_ID-terminated, with the
// distance-to-owner of each link in adj0_d (needed by the insert path only).
// Layers >= 1: a point owns `plevel[id]` consecutive lists of M slots starting at list index
// up_off[id] in adjU (list for layer l is up_off[id] + l - 1).  plevel >= level; it exceeds the
// point's own level only for former entry points (see DESIGN.md "lists above a point's level").
struct GraphView {
  const void* vec;  // rows of element type T (f32, i32, u32, u16, u8), zero padded to whole 128-byte lines
  int d4;           // 16-byte chunks per row (multiple of 8)
  int dim;          // true number of elements per vector
  uint32_t* adj0;
  float* adj0_d;
  int deg0;
  uint32_t* adjU;
  float* adjU_d;
  int M;
  const uint32_t* up_off;
  const uint8_t* plevel;
  const uint8_t* level;
  const uint64_t* origin;
  uint32_t n;
  uint32_t entry;  // INVALID_ID when empty
  int entry_level;
};

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// L2 cache policies (createpolicy): vector rows stream through once per query (evict_first), the per-warp visited
// tables are re-read for the whole search (evict_last), so that 6 GB of rows per launch do not push them out of L2.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint4 ldg_stream(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint32_t ld_keep(const uint32_t* p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.cg.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint4 ld_keep4(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.cg.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_keep(uint32_t* p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.cg.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}

// The list of (p, layer): pointer to its ids and its capacity, or nullptr / 0 above plevel[p], where the point owns no list.
// The one place a list's address is worked out; list_at adds the distances, which sit at the same offset.
__device__ __forceinline__ const uint32_t* list_ids(const GraphView& g, uint32_t p, int layer, int& cap) {
  if (layer == 0) {
    cap = g.deg0;
    return g.adj0 + (size_t)p * g.deg0;
  }
  if (layer > (int)g.plevel[p]) {
    cap = 0;
    return nullptr;
  }
  cap = g.M;
  return g.adjU + ((size_t)g.up_off[p] + (layer - 1)) * g.M;
}
struct List {
  uint32_t* ids;  // nullptr above plevel[p]
  float* dists;   // distance of each link to p
  int cap;
};
__device__ __forceinline__ List list_at(const GraphView& g, uint32_t p, int layer) {
  List l;
  l.ids = const_cast<uint32_t*>(list_ids(g, p, layer, l.cap));
  l.dists = !l.ids ? nullptr : layer == 0 ? g.adj0_d + (l.ids - g.adj0) : g.adjU_d + (l.ids - g.adjU);
  return l;
}

// ------------------------------------------------------------------------------------------------
// Distance functors.  BIT-EXACT SUMMATION ORDER (mirrored by oracle/distances.h accumulate_gpu):
// lane g (0..7) of a row group owns float4 chunks g, g+8, g+16, ...; inside a chunk x,y,z,w in that
// order; fused multiply-add where a product is accumulated; then partials are combined with a
// 4,2,1 xor butterfly and finished (sqrt / 1-x / ...).  Zero padding adds exact zeros.
// f32 L2 / L1 / Dot keep two partial sums per lane (elements x,z and y,w of each chunk) that are added before
// the butterfly; every other op keeps one.  The two sums are independent dependency chains, so the FMA latency of
// one overlaps the other.
__device__ __forceinline__ float fold2(float2 a) { return __fadd_rn(a.x, a.y); }

// L2 / L1 / Dot accumulate TWO partial sums per lane: .x takes the elements x and z of every 16-byte chunk,
// .y takes y and w; fold() adds them before the butterfly.
// (The scalar step() is the single-accumulator form used for integer element types, OpCast.)
struct OpL2 {
  typedef float2 acc_t;
  typedef float red_t;
  static __device__ __forceinline__ acc_t zero() { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ void step(float& a, float q, float x) {
    float df = __fsub_rn(q, x);
    a = __fmaf_rn(df, df, a);
  }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a.x, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a.y, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a.x, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a.y, __uint_as_float(q.w), __uint_as_float(x.w));
  }
  static __device__ __forceinline__ red_t fold(acc_t a) { return fold2(a); }
  static __device__ __forceinline__ red_t comb(red_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  // finish() runs once per row pass in every lane, post() once per candidate: the square root is deferred to post()
  static __device__ __forceinline__ float finish(red_t a, int) { return a; }
  static __device__ __forceinline__ float post(float v) { return __fsqrt_rn(v); }
};
struct OpL1 {
  typedef float2 acc_t;
  typedef float red_t;
  static __device__ __forceinline__ acc_t zero() { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ void step(float& a, float q, float x) { a = __fadd_rn(a, fabsf(__fsub_rn(q, x))); }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a.x, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a.y, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a.x, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a.y, __uint_as_float(q.w), __uint_as_float(x.w));
  }
  static __device__ __forceinline__ red_t fold(acc_t a) { return fold2(a); }
  static __device__ __forceinline__ red_t comb(red_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  static __device__ __forceinline__ float finish(red_t a, int) { return a; }
  static __device__ __forceinline__ float post(float v) { return v; }
};
struct OpDot {
  typedef float2 acc_t;
  typedef float red_t;
  static __device__ __forceinline__ acc_t zero() { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    a.x = __fmaf_rn(__uint_as_float(q.x), __uint_as_float(x.x), a.x);
    a.y = __fmaf_rn(__uint_as_float(q.y), __uint_as_float(x.y), a.y);
    a.x = __fmaf_rn(__uint_as_float(q.z), __uint_as_float(x.z), a.x);
    a.y = __fmaf_rn(__uint_as_float(q.w), __uint_as_float(x.w), a.y);
  }
  static __device__ __forceinline__ red_t fold(acc_t a) { return fold2(a); }
  static __device__ __forceinline__ red_t comb(red_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  static __device__ __forceinline__ float finish(red_t a, int) { return fmaxf(__fsub_rn(1.0f, a), 0.f); }
  static __device__ __forceinline__ float post(float v) { return v; }
};
struct Cos3 {
  double ab, aa, bb;
};
struct OpCosine {  // f64 accumulation like anndists DistCosine
  typedef Cos3 acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return Cos3{0., 0., 0.}; }
  static __device__ __forceinline__ void step(acc_t& a, float q, float x) {
    double dq = (double)q, dx = (double)x;
    a.ab = __fma_rn(dq, dx, a.ab);
    a.aa = __fma_rn(dq, dq, a.aa);
    a.bb = __fma_rn(dx, dx, a.bb);
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) {
    Cos3 r;
    r.ab = __dadd_rn(a.ab, __shfl_xor_sync(FULL, a.ab, off));
    r.aa = __dadd_rn(a.aa, __shfl_xor_sync(FULL, a.aa, off));
    r.bb = __dadd_rn(a.bb, __shfl_xor_sync(FULL, a.bb, off));
    return r;
  }
  static __device__ __forceinline__ float finish(acc_t a, int) {
    if (a.aa > 0. && a.bb > 0.) {
      double r = __dsub_rn(1., __ddiv_rn(a.ab, __dsqrt_rn(__dmul_rn(a.aa, a.bb))));
      return (float)(r > 0. ? r : 0.);
    }
    return 0.f;
  }
  static __device__ __forceinline__ float post(float v) { return v; }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a, __uint_as_float(q.w), __uint_as_float(x.w));
  }
};
struct OpHellinger {
  typedef float acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return 0.f; }
  static __device__ __forceinline__ void step(acc_t& a, float q, float x) { a = __fadd_rn(a, __fsqrt_rn(__fmul_rn(q, x))); }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  static __device__ __forceinline__ float finish(acc_t a, int) { return __fsqrt_rn(fmaxf(__fsub_rn(1.0f, a), 0.f)); }
  static __device__ __forceinline__ float post(float v) { return v; }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a, __uint_as_float(q.w), __uint_as_float(x.w));
  }
};
struct OpJeffreys {
  typedef float acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return 0.f; }
  static __device__ __forceinline__ void step(acc_t& a, float q, float x) {
    float qm = fmaxf(q, 1e-30f), xm = fmaxf(x, 1e-30f);
    a = __fadd_rn(a, __fmul_rn(__fsub_rn(q, x), logf(__fdiv_rn(qm, xm))));
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  static __device__ __forceinline__ float finish(acc_t a, int) { return a; }
  static __device__ __forceinline__ float post(float v) { return v; }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a, __uint_as_float(q.w), __uint_as_float(x.w));
  }
};
struct OpJS {
  typedef float acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return 0.f; }
  static __device__ __forceinline__ void step(acc_t& a, float q, float x) {
    float m = __fmul_rn(0.5f, __fadd_rn(q, x));
    float t = 0.f;
    if (q > 0.f) t = __fadd_rn(t, __fmul_rn(q, logf(__fdiv_rn(q, m))));
    if (x > 0.f) t = __fadd_rn(t, __fmul_rn(x, logf(__fdiv_rn(x, m))));
    a = __fadd_rn(a, t);
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) { return __fadd_rn(a, __shfl_xor_sync(FULL, a, off)); }
  static __device__ __forceinline__ float finish(acc_t a, int) { return __fsqrt_rn(fmaxf(__fmul_rn(0.5f, a), 0.f)); }
  static __device__ __forceinline__ float post(float v) { return v; }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    step(a, __uint_as_float(q.x), __uint_as_float(x.x));
    step(a, __uint_as_float(q.y), __uint_as_float(x.y));
    step(a, __uint_as_float(q.z), __uint_as_float(x.z));
    step(a, __uint_as_float(q.w), __uint_as_float(x.w));
  }
};

// ---- integer element types (SURVEY §8 row f1): a 16-byte chunk holds 4 (i32/u32), 8 (u16) or 16 (u8) elements.
// L1/L2 cast every element to f32 (as anndists does for integer T) and accumulate like the f32 ops, elements of a
// chunk in memory order.  Hamming counts differing elements, Jaccard sums min and max, both in exact integers.
template <class T>
struct Elems;
template <>
struct Elems<uint32_t> {
  static constexpr int N = 4;
  static __device__ __forceinline__ float get(const uint4& v, int i) { return (float)(i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w); }
};
template <>
struct Elems<int32_t> {
  static constexpr int N = 4;
  static __device__ __forceinline__ float get(const uint4& v, int i) { return (float)(int32_t)(i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w); }
};
template <>
struct Elems<uint16_t> {
  static constexpr int N = 8;
  static __device__ __forceinline__ float get(const uint4& v, int i) {
    const uint32_t w = (i >> 1) == 0 ? v.x : (i >> 1) == 1 ? v.y : (i >> 1) == 2 ? v.z : v.w;
    return (float)((w >> (16 * (i & 1))) & 0xFFFFu);
  }
};
template <>
struct Elems<uint8_t> {
  static constexpr int N = 16;
  static __device__ __forceinline__ float get(const uint4& v, int i) {
    const uint32_t w = (i >> 2) == 0 ? v.x : (i >> 2) == 1 ? v.y : (i >> 2) == 2 ? v.z : v.w;
    return (float)((w >> (8 * (i & 3))) & 0xFFu);
  }
};

template <class T, class FOp>  // FOp = OpL1 / OpL2 on the elements cast to f32
struct OpCast {
  typedef float acc_t;
  typedef float red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return 0.f; }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
#pragma unroll
    for (int i = 0; i < Elems<T>::N; ++i) FOp::step(a, Elems<T>::get(q, i), Elems<T>::get(x, i));
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) { return FOp::comb(a, off); }
  static __device__ __forceinline__ float finish(acc_t a, int d) { return FOp::finish(a, d); }
  static __device__ __forceinline__ float post(float v) { return FOp::post(v); }
};

template <class T>
struct OpHamming {  // DistHamming: #{a_i != b_i} / len
  typedef uint32_t acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return 0u; }
  static __device__ __forceinline__ uint32_t ne(uint32_t a, uint32_t b) {
    if (sizeof(T) == 1) return __popc(__vcmpne4(a, b) & 0x01010101u);
    if (sizeof(T) == 2) return __popc(__vcmpne2(a, b) & 0x00010001u);
    return a != b ? 1u : 0u;
  }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    a += ne(q.x, x.x) + ne(q.y, x.y) + ne(q.z, x.z) + ne(q.w, x.w);
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) { return a + __shfl_xor_sync(FULL, a, off); }
  static __device__ __forceinline__ float finish(acc_t a, int d) { return __fdiv_rn((float)a, (float)d); }
  static __device__ __forceinline__ float post(float v) { return v; }
};

struct MinMax64 {
  unsigned long long mn, mx;
};
template <class T>
struct OpJaccard {  // weighted Jaccard: 1 - sum min / sum max, integer sums, f64 division
  typedef MinMax64 acc_t;
  typedef acc_t red_t;
  static __device__ __forceinline__ red_t fold(acc_t a) { return a; }
  static __device__ __forceinline__ acc_t zero() { return MinMax64{0ull, 0ull}; }
  static __device__ __forceinline__ void word(acc_t& a, uint32_t q, uint32_t x) {
    if (sizeof(T) == 1) {
      a.mn += __vsadu4(__vminu4(q, x), 0u);
      a.mx += __vsadu4(__vmaxu4(q, x), 0u);
    } else if (sizeof(T) == 2) {
      a.mn += __vsadu2(__vminu2(q, x), 0u);
      a.mx += __vsadu2(__vmaxu2(q, x), 0u);
    } else {
      a.mn += q < x ? q : x;
      a.mx += q < x ? x : q;
    }
  }
  static __device__ __forceinline__ void chunk(acc_t& a, const uint4& q, const uint4& x) {
    word(a, q.x, x.x);
    word(a, q.y, x.y);
    word(a, q.z, x.z);
    word(a, q.w, x.w);
  }
  static __device__ __forceinline__ acc_t comb(acc_t a, int off) {
    return MinMax64{a.mn + __shfl_xor_sync(FULL, a.mn, off), a.mx + __shfl_xor_sync(FULL, a.mx, off)};
  }
  static __device__ __forceinline__ float finish(acc_t a, int) {
    if (a.mx == 0ull) return 0.f;
    return (float)__dsub_rn(1.0, __ddiv_rn((double)a.mn, (double)a.mx));
  }
  static __device__ __forceinline__ float post(float v) { return v; }
};

template <class Op>
__device__ __forceinline__ float reduce8(typename Op::acc_t acc, int dim) {
  typename Op::red_t a = Op::fold(acc);
  a = Op::comb(a, 4);
  a = Op::comb(a, 2);
  a = Op::comb(a, 1);
  return Op::finish(a, dim);
}

// ------------------------------------------------------------------------------------------------
// warp_dists: distances from the query (float4 view in shared memory, d4 chunks) to `n` rows named
// by ids[] (shared memory), results to out[] (shared memory).  8 lanes per row, 4 rows per pass,
// U passes in flight; CH = d4/8 when known at compile time (CH float4 loads per lane per row),
// CH = 0 for the generic loop.  Every load instruction covers 4 rows x 128 B contiguous.
template <class Op, int CH, int U>
__device__ __forceinline__ void warp_dists(const uint4* __restrict__ vec, int d4, int dim, const uint4* q4,
                                           const uint32_t* ids, int n, float* out) {
  const int lane = lane_id();
  const int g = lane & 7, r = lane >> 3;
  const uint64_t pol = l2_policy_evict_first();
  if constexpr (CH > 0) {
    uint4 qv[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) qv[i] = q4[g + 8 * i];
    for (int base = 0; base < n; base += 4 * U) {
      const uint4* row[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        int idx = base + u * 4 + r;
        uint32_t id = ids[idx < n ? idx : n - 1];
        row[u] = vec + (size_t)id * d4 + g;
      }
      uint4 x[U][CH];
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int i = 0; i < CH; ++i) x[u][i] = ldg_stream(row[u] + 8 * i, pol);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        typename Op::acc_t a = Op::zero();
#pragma unroll
        for (int i = 0; i < CH; ++i) Op::chunk(a, qv[i], x[u][i]);
        float dist = reduce8<Op>(a, dim);
        int idx = base + u * 4 + r;
        if (g == 0 && idx < n) out[idx] = dist;
      }
    }
  } else {
    const int nch = d4 >> 3;
    for (int base = 0; base < n; base += 4 * U) {
      const uint4* row[U];
      typename Op::acc_t a[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        int idx = base + u * 4 + r;
        uint32_t id = ids[idx < n ? idx : n - 1];
        row[u] = vec + (size_t)id * d4 + g;
        a[u] = Op::zero();
      }
#pragma unroll 4
      for (int i = 0; i < nch; ++i) {
        uint4 qv = q4[g + 8 * i];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          uint4 x = ldg_stream(row[u] + 8 * i, pol);
          Op::chunk(a[u], qv, x);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float dist = reduce8<Op>(a[u], dim);
        int idx = base + u * 4 + r;
        if (g == 0 && idx < n) out[idx] = dist;
      }
    }
  }
}

// copy one query/point row of `nbytes` raw bytes into the warp's shared-memory row buffer, zero padding to row_bytes
__device__ __forceinline__ void stage_row_bytes(void* dst, const void* src, int nbytes, int row_bytes) {
  const int lane = lane_id();
  uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
  const int nw = nbytes >> 2;
  if ((reinterpret_cast<size_t>(src) & 3) == 0) {
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
    for (int i = lane; i < (row_bytes >> 2); i += 32) d32[i] = i < nw ? s32[i] : 0u;
    __syncwarp();
    const uint8_t* s8 = reinterpret_cast<const uint8_t*>(src);
    uint8_t* d8 = reinterpret_cast<uint8_t*>(dst);
    for (int i = (nw << 2) + lane; i < nbytes; i += 32) d8[i] = s8[i];
  } else {
    const uint8_t* s8 = reinterpret_cast<const uint8_t*>(src);
    uint8_t* d8 = reinterpret_cast<uint8_t*>(dst);
    for (int i = lane; i < row_bytes; i += 32) d8[i] = i < nbytes ? s8[i] : (uint8_t)0;
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// TMA staging: rows copied HBM -> shared memory by the bulk-copy engine (cp.async.bulk, SASS UBLKCP), completion
// signalled on an mbarrier.  One lane issues one 1-D bulk copy per row, so a row in flight costs no registers.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}

constexpr int STAGE_ROWS = 8;  // rows of a chunk fetched by TMA; the rest of the chunk goes through registers

struct Stage {
  uint4* buf;    // [STAGE_ROWS][d4] or nullptr (rows too long to stage)
  uint64_t* bar;  // mbarrier, arrival count 1
  uint32_t phase;
};

// Hybrid row fetch: rows [0, min(n,8)) by TMA into shared memory, rows [8, n) through registers (warp_dists),
// all in flight together; then the staged rows are reduced from shared memory with the same lane/chunk mapping,
// so every distance is bit-identical to the pure register path.
template <class Op, int CH, int U>
__device__ __forceinline__ void warp_dists_staged(const uint4* __restrict__ vec, int d4, int dim, const uint4* q4,
                                                  const uint32_t* ids, int n, float* out, Stage& st) {
  if constexpr (CH == 0) {
    warp_dists<Op, CH, U>(vec, d4, dim, q4, ids, n, out);
  } else {
    const int lane = lane_id();
    const int nst = n < STAGE_ROWS ? n : STAGE_ROWS;
    const uint32_t row_bytes = (uint32_t)d4 * 16u;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic reads of the stage precede the async writes
    if (lane == 0) mbar_expect_tx(st.bar, row_bytes * nst);
    __syncwarp();
    if (lane < nst) bulk_g2s(st.buf + (size_t)lane * d4, vec + (size_t)ids[lane] * d4, row_bytes, st.bar, l2_policy_evict_first());
    if (n > STAGE_ROWS) warp_dists<Op, CH, U>(vec, d4, dim, q4, ids + STAGE_ROWS, n - STAGE_ROWS, out + STAGE_ROWS);
    const int g = lane & 7, r = lane >> 3;
    uint4 qv[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) qv[i] = q4[g + 8 * i];
    mbar_wait(st.bar, st.phase);
    st.phase ^= 1u;
#pragma unroll
    for (int pass = 0; pass < STAGE_ROWS / 4; ++pass) {
      const int row = pass * 4 + r;
      if (pass * 4 < nst) {
        const uint4* src = st.buf + (size_t)(row < nst ? row : nst - 1) * d4 + g;
        typename Op::acc_t a = Op::zero();
#pragma unroll
        for (int i = 0; i < CH; ++i) {
          const uint4 x = src[8 * i];
          Op::chunk(a, qv[i], x);
        }
        const float dist = reduce8<Op>(a, dim);
        if (g == 0 && row < nst) out[row] = dist;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Visited set: one open-addressing table per resident warp ("warp slot") in global memory (L2
// resident).  Entry = (epoch << id_bits) | id; an entry whose epoch differs from the current one is
// free, so a new search only bumps the epoch instead of clearing.  Exact (no false positives).
struct VisitedCfg {
  uint32_t* tables;   // [n_slots][cap]
  uint32_t* epochs;   // [n_slots] persisted across launches
  uint32_t cap;       // power of two
  int shift;          // 32 - log2(cap)
  int id_bits;        // bits needed for ids
};

// The state of one warp's set is what changes during a search: table pointer, epoch, insert count.  Capacity, hash shift
// and the epoch / id split are read from the launch's VisitedCfg (kernel parameters) where they are used.  Every
// function is warp-collective and takes the caller's lane (the lean kernel pins it, see lean_common.cuh pin()).
struct Visited {
  uint32_t* tab;
  uint32_t epoch;
  uint32_t used;  // insertions of the current search (warp-uniform)

  __device__ __forceinline__ void init(const VisitedCfg& c, uint32_t slot) {
    tab = c.tables + (size_t)slot * c.cap;
    epoch = c.epochs[slot];
    used = 0;
  }
  __device__ __forceinline__ void save(const VisitedCfg& c, uint32_t slot, int lane) const {
    if (lane == 0) c.epochs[slot] = epoch;
  }
  static __device__ __forceinline__ uint32_t home(const VisitedCfg& c, uint32_t id) { return (id * 2654435761u) >> c.shift; }
  // Start a new search from `entry` (hnsw.rs:955-956): bump the epoch instead of clearing the table (cleared only when the
  // epoch wraps), then record the entry.  The table holds nothing of the new epoch yet, so the entry's home slot is free.
  __device__ __forceinline__ void begin(const VisitedCfg& c, uint32_t entry, int lane) {
    const uint32_t epoch_max = (c.id_bits >= 32) ? 0u : ((1u << (32 - c.id_bits)) - 1u);
    if (epoch >= epoch_max) {
      for (uint32_t i = lane; i < c.cap; i += 32) tab[i] = 0u;
      epoch = 0;
    }
    epoch += 1;
    used = 1;
    __syncwarp();
    if (lane == 0) st_keep(tab + home(c, entry), (epoch << c.id_bits) | entry, l2_policy_evict_last());
    __syncwarp();
  }
  // Test-and-set of up to 32 ids (one per lane, `valid` lanes only).  Returns true in the lanes whose id was not yet in
  // the set (it is afterwards).  The table is private to this warp, so no atomics are needed: lanes that find the same
  // free slot in the same round elect the lowest lane (match_any); the others probe on.  One L2 round trip per round,
  // and almost always one round.  The first probe may have been done ahead of time (`pre`: slot pre_h was read as
  // pre_cv after the last store to the table).
  __device__ __forceinline__ bool test_and_set(const VisitedCfg& c, int lane, uint32_t id, bool valid, bool pre = false,
                                               uint32_t pre_h = 0, uint32_t pre_cv = 0) {
    const uint32_t want = (epoch << c.id_bits) | id;
    const uint64_t pol_keep = l2_policy_evict_last();
    uint32_t h = pre ? pre_h : home(c, id);
    bool pending = valid, fresh = false, first = pre;
    while (__any_sync(FULL, pending)) {
      uint32_t cur = 0;
      if (pending) cur = first ? pre_cv : ld_keep(tab + h, pol_keep);
      first = false;
      bool claim = false;
      if (pending) {
        if (cur == want) {
          pending = false;  // already visited
        } else if ((cur >> c.id_bits) != epoch) {
          claim = true;  // stale or empty slot
        } else {
          h = (h + 1) & (c.cap - 1);
        }
      }
      const unsigned claimers = __ballot_sync(FULL, claim);
      if (claim) {
        const unsigned same = __match_any_sync(claimers, h);
        const int leader = __ffs(same) - 1;
        const uint32_t lead_id = __shfl_sync(claimers, id, leader);
        if (lane == leader) {
          st_keep(tab + h, want, pol_keep);
          fresh = true;
          pending = false;
        } else if (lead_id == id) {
          pending = false;  // the same id twice in one chunk: the leader records it
        } else {
          h = (h + 1) & (c.cap - 1);
        }
      }
      __syncwarp();  // orders this round's stores before the next round's loads
    }
    used += __popc(__ballot_sync(FULL, fresh));  // warp-uniform count
    return fresh;
  }
  __device__ __forceinline__ bool overflowing(const VisitedCfg& c) const { return used >= c.cap - (c.cap >> 2); }
};

// ------------------------------------------------------------------------------------------------
// Queue keys: (float bits of distance << 32) | (id << 1) | expanded.  Distances are >= 0 so the
// unsigned order of the bits is the numeric order; ties on distance order by id: the total order
// (dist, id) of the oracle's MODE_DET.
__device__ __forceinline__ uint64_t make_key(float d, uint32_t id) {
  return ((uint64_t)__float_as_uint(d) << 32) | ((uint64_t)id << 1);
}
__device__ __forceinline__ float key_dist(uint64_t k) { return __uint_as_float((uint32_t)(k >> 32)); }
__device__ __forceinline__ uint32_t key_id(uint64_t k) { return ((uint32_t)k) >> 1; }

// One sorted array (ascending) in shared memory standing for both reference queues: W = the array,
// C = its not-yet-expanded entries (entries evicted from W can never be expanded again, see
// DESIGN.md "one array for W and C").  All functions are warp-collective.
struct SortedQueue {
  uint64_t* w;
  int n;
  int cap;  // ef

  __device__ __forceinline__ void reset(uint64_t* buf, int ef) {
    w = buf;
    n = 0;
    cap = ef;
  }
  __device__ __forceinline__ uint64_t get(int i) const { return w[i]; }
  __device__ __forceinline__ uint64_t local(int i) const { return w[i]; }  // i == lane (mod 32)
  __device__ __forceinline__ void mark_expanded(int i) {
    __syncwarp();
    if (lane_id() == 0) w[i] |= 1ull;
    __syncwarp();
  }
  __device__ __forceinline__ void push_first(uint64_t key) {
    if (lane_id() == 0) w[0] = key;
    n = 1;
    __syncwarp();
  }
  // index of the nearest unexpanded entry, or -1
  __device__ __forceinline__ int first_unexpanded() const {
    const int lane = lane_id();
    for (int base = 0; base < n; base += 32) {
      int i = base + lane;
      bool open = (i < n) && ((w[i] & 1ull) == 0ull);
      unsigned m = __ballot_sync(FULL, open);
      if (m) return base + __ffs(m) - 1;
    }
    return -1;
  }
  // index of the first unexpanded entry at or after `from`, or -1
  __device__ __forceinline__ int next_unexpanded(int from) const {
    const int lane = lane_id();
    for (int base = from & ~31; base < n; base += 32) {
      int i = base + lane;
      bool open = (i < n) && (i >= from) && ((w[i] & 1ull) == 0ull);
      unsigned m = __ballot_sync(FULL, open);
      if (m) return base + __ffs(m) - 1;
    }
    return -1;
  }
  __device__ __forceinline__ void next3(int from, int& a, int& b, int& c) const {
    a = next_unexpanded(from);
    b = a >= 0 ? next_unexpanded(a + 1) : -1;
    c = b >= 0 ? next_unexpanded(b + 1) : -1;
  }
  __device__ __forceinline__ bool accepts(uint64_t key) const { return n < cap || key < (w[n - 1] & ~1ull); }
  // insert key (expanded bit clear) keeping order; drops the largest entry when full. Caller checked accepts().
  __device__ __forceinline__ void insert(uint64_t key) {
    const int lane = lane_id();
    int pos = 0;
    for (int base = 0; base < n; base += 32) {
      int i = base + lane;
      bool less = (i < n) && (w[i] < key);
      pos += __popc(__ballot_sync(FULL, less));
    }
    const int new_n = n < cap ? n + 1 : cap;
    // shift (pos, new_n-1] right by one; chunks are handled top-down so that a chunk's sources are
    // read before a lower chunk overwrites them
    int top = new_n - 1;
    while (top > pos) {
      int lo = top - 31 > pos + 1 ? top - 31 : pos + 1;  // chunk [lo, top]
      int i = lo + lane;
      uint64_t v = 0;
      if (i <= top) v = w[i - 1];
      __syncwarp();
      if (i <= top) w[i] = v;
      __syncwarp();
      top = lo - 1;
    }
    __syncwarp();  // reads of the queue by other lanes (accepts, rank) happen-before the write below
    if (lane == 0) w[pos] = key;
    __syncwarp();
    n = new_n;
  }
};

// SortedQueue with a compile-time number of 32-entry chunks (capacity 32*NCH >= ef): no loops, no bounds tests
// (unused slots hold ~0, which compares above every key and reads as "expanded"), one __syncwarp per update.
template <int NCH>
struct SmemQueueN {
  uint64_t* w;
  int n;
  int cap;

  __device__ __forceinline__ void reset(uint64_t* buf, int ef) {
    w = buf;
    n = 0;
    cap = ef;
    const int lane = lane_id();
    __syncwarp();
#pragma unroll
    for (int c = 0; c < NCH; ++c) w[32 * c + lane] = ~0ull;
    __syncwarp();
  }
  __device__ __forceinline__ uint64_t get(int i) const { return w[i]; }
  __device__ __forceinline__ uint64_t local(int i) const { return w[i]; }
  __device__ __forceinline__ void mark_expanded(int i) {
    __syncwarp();  // other lanes' reads of the queue (scans, get) happen-before this write (racecheck: WAR hazard)
    if (lane_id() == 0) w[i] |= 1ull;
    __syncwarp();
  }
  __device__ __forceinline__ void push_first(uint64_t key) {
    if (lane_id() == 0) w[0] = key;
    n = 1;
    __syncwarp();
  }
  __device__ __forceinline__ int first_unexpanded() const { return next_unexpanded(0); }
  __device__ __forceinline__ int next_unexpanded(int from) const {
    const int lane = lane_id();
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int i = 32 * c + lane;
      const unsigned m = __ballot_sync(FULL, ((w[i] & 1ull) == 0ull) && i >= from);
      if (m) return 32 * c + __ffs(m) - 1;
    }
    return -1;
  }
  // first three unexpanded indices at or after `from` in one pass over the queue (-1 when absent)
  __device__ __forceinline__ void next3(int from, int& a, int& b, int& c) const {
    const int lane = lane_id();
    unsigned m[NCH];
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int i = 32 * ch + lane;
      m[ch] = __ballot_sync(FULL, ((w[i] & 1ull) == 0ull) && i >= from);
    }
    int out[3] = {-1, -1, -1};
    int k = 0;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      unsigned mm = m[ch];
      while (mm && k < 3) {
        out[k++] = 32 * ch + __ffs(mm) - 1;
        mm &= mm - 1;
      }
    }
    a = out[0];
    b = out[1];
    c = out[2];
  }
  // when the queue is not full its last slot holds ~0, so one comparison covers both cases
  __device__ __forceinline__ bool accepts(uint64_t key) const { return key < (w[cap - 1] & ~1ull); }
  __device__ __forceinline__ void insert(uint64_t key) {
    const int lane = lane_id();
    uint64_t cur[NCH], prev[NCH];
    int pos = 0;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int i = 32 * c + lane;
      cur[c] = w[i];
      prev[c] = i > 0 ? w[i - 1] : 0ull;
      pos += __popc(__ballot_sync(FULL, cur[c] < key));
    }
    __syncwarp();  // every lane has read its sources
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int i = 32 * c + lane;
      uint64_t nv = i > pos ? prev[c] : key;
      if (i >= cap) nv = ~0ull;
      if (i >= pos) w[i] = nv;
    }
    __syncwarp();
    n = n < cap ? n + 1 : cap;
  }
};

// queue kinds: 0 = generic SortedQueue (any ef), 100 + NCH = SmemQueueN<NCH> (ef <= 32*NCH)
template <int KIND>
struct QueueSel;
template <> struct QueueSel<0> { typedef SortedQueue type; };
template <> struct QueueSel<101> { typedef SmemQueueN<1> type; };
template <> struct QueueSel<102> { typedef SmemQueueN<2> type; };
template <> struct QueueSel<104> { typedef SmemQueueN<4> type; };
template <> struct QueueSel<108> { typedef SmemQueueN<8> type; };

}  // namespace hb
