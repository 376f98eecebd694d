// Building blocks of the lean query kernel (search_lean.cuh): the reduction arithmetic of the distance functors by type, the "still unexpanded" bit masks that stand for the reference's candidate heap C
// (/root/reference/src/hnsw.rs:940-1001).  Shared-memory access through pinned 32-bit window addresses is in common.cuh.
#pragma once
#include "common.cuh"

namespace hb {

// ---- reduction arithmetic of the Ops' partial sums, by type (same operations as every Op::comb)
__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ uint32_t radd(uint32_t a, uint32_t b) { return a + b; }
__device__ __forceinline__ Cos3 radd(const Cos3& a, const Cos3& b) {
  return Cos3{__dadd_rn(a.ab, b.ab), __dadd_rn(a.aa, b.aa), __dadd_rn(a.bb, b.bb)};
}
__device__ __forceinline__ MinMax64 radd(const MinMax64& a, const MinMax64& b) { return MinMax64{a.mn + b.mn, a.mx + b.mx}; }
__device__ __forceinline__ float rshfl(float a, int off) { return __shfl_xor_sync(FULL, a, off); }
__device__ __forceinline__ uint32_t rshfl(uint32_t a, int off) { return __shfl_xor_sync(FULL, a, off); }
__device__ __forceinline__ Cos3 rshfl(const Cos3& a, int off) {
  return Cos3{__shfl_xor_sync(FULL, a.ab, off), __shfl_xor_sync(FULL, a.aa, off), __shfl_xor_sync(FULL, a.bb, off)};
}
__device__ __forceinline__ MinMax64 rshfl(const MinMax64& a, int off) {
  return MinMax64{__shfl_xor_sync(FULL, a.mn, off), __shfl_xor_sync(FULL, a.mx, off)};
}

// ---- the "still unexpanded" mask over queue positions: bit p set <=> W[p] has not been expanded yet
struct Mask64 {
  uint64_t m;
  __device__ __forceinline__ bool none() const { return m == 0; }
  __device__ __forceinline__ int first() const { return __ffsll((long long)m) - 1; }  // -1 when none
  __device__ __forceinline__ void drop_first() { m &= m - 1; }
  __device__ __forceinline__ void set_only(int p) { m = 1ull << p; }
  __device__ __forceinline__ bool test(int p) const { return (m >> p) & 1ull; }
  __device__ __forceinline__ void set_words(const uint32_t (&w)[2]) { m = (uint64_t)w[0] | ((uint64_t)w[1] << 32); }
};
struct Mask128 {
  uint64_t lo, hi;
  __device__ __forceinline__ bool none() const { return (lo | hi) == 0; }
  __device__ __forceinline__ int first() const {
    return lo ? __ffsll((long long)lo) - 1 : (hi ? 63 + __ffsll((long long)hi) : -1);
  }
  __device__ __forceinline__ void drop_first() {
    if (lo) lo &= lo - 1;
    else hi &= hi - 1;
  }
  __device__ __forceinline__ void set_only(int p) {
    lo = p < 64 ? 1ull << p : 0ull;
    hi = p < 64 ? 0ull : 1ull << (p - 64);
  }
  __device__ __forceinline__ bool test(int p) const { return ((p < 64 ? lo : hi) >> (p & 63)) & 1ull; }
  __device__ __forceinline__ void set_words(const uint32_t (&w)[4]) {
    lo = (uint64_t)w[0] | ((uint64_t)w[1] << 32);
    hi = (uint64_t)w[2] | ((uint64_t)w[3] << 32);
  }
};
template <int QC>
struct MaskSel;
template <> struct MaskSel<64> { typedef Mask64 type; };
template <> struct MaskSel<128> { typedef Mask128 type; };

}  // namespace hb
