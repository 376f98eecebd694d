// Lean query kernel (search_lean.cuh), u16 instantiations: DistL1, DistL2 (elements cast to f32), DistHamming, DistJaccard.
#include "search_lean.cuh"

namespace hb {

cudaError_t launch_search_lean_u16(const SearchParams& p, int metric, int grid, size_t smem, cudaStream_t st,
                                   int* blocks_per_sm) {
  switch (metric) {
    case METRIC_L1: return launch_lean_op<OpCast<uint16_t, OpL1>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_L2: return launch_lean_op<OpCast<uint16_t, OpL2>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_HAMMING: return launch_lean_op<OpHamming<uint16_t>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_JACCARD: return launch_lean_op<OpJaccard<uint16_t>>(p, grid, smem, st, blocks_per_sm);
  }
  return cudaErrorInvalidValue;
}

}  // namespace hb
