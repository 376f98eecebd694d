// Lean query kernel (search_lean.cuh), f32 instantiations: DistL1, DistL2, DistDot, DistCosine.
#include "search_lean.cuh"

namespace hb {

cudaError_t launch_search_lean_f32(const SearchParams& p, int metric, int grid, size_t smem, cudaStream_t st,
                                   int* blocks_per_sm) {
  switch (metric) {
    case METRIC_L2: return launch_lean_op<OpL2>(p, grid, smem, st, blocks_per_sm);
    case METRIC_L1: return launch_lean_op<OpL1>(p, grid, smem, st, blocks_per_sm);
    case METRIC_DOT: return launch_lean_op<OpDot>(p, grid, smem, st, blocks_per_sm);
    case METRIC_COSINE: return launch_lean_op<OpCosine>(p, grid, smem, st, blocks_per_sm);
  }
  return cudaErrorInvalidValue;
}

// the lean kernel covers: f32 with L1 / L2 / Dot / Cosine, u8 and u16 with L1 / L2 / Hamming / Jaccard
cudaError_t launch_search_lean(const SearchParams& p, int metric, int dtype, int grid, size_t smem, cudaStream_t st,
                               int* blocks_per_sm) {
  if (dtype == DT_F32) return launch_search_lean_f32(p, metric, grid, smem, st, blocks_per_sm);
  if (dtype == DT_U8) return launch_search_lean_u8(p, metric, grid, smem, st, blocks_per_sm);
  if (dtype == DT_U16) return launch_search_lean_u16(p, metric, grid, smem, st, blocks_per_sm);
  return cudaErrorInvalidValue;
}

}  // namespace hb
