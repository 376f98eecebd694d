// Lean query kernel (search_lean.cuh), u8 instantiations: DistL1, DistL2 (elements cast to f32), DistHamming, DistJaccard.
#include "search_lean.cuh"

namespace hb {

cudaError_t launch_search_lean_u8(const SearchParams& p, int metric, int grid, size_t smem, cudaStream_t st,
                                   int* blocks_per_sm) {
  switch (metric) {
    case METRIC_L1: return launch_lean_op<OpCast<uint8_t, OpL1>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_L2: return launch_lean_op<OpCast<uint8_t, OpL2>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_HAMMING: return launch_lean_op<OpHamming<uint8_t>>(p, grid, smem, st, blocks_per_sm);
    case METRIC_JACCARD: return launch_lean_op<OpJaccard<uint8_t>>(p, grid, smem, st, blocks_per_sm);
  }
  return cudaErrorInvalidValue;
}

}  // namespace hb
