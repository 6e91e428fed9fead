// flood_profiled.cu — the persistent kernel with device cycle counters (ffn_engine_profile).
#define FFN_KNS profiled
#define FFN_PROFILE 1
#include "flood_kernel.cuh"

namespace ffn {
namespace profiled {

template __global__ void ffn_flood_kernel<false>(const __grid_constant__ KParams p);
template __global__ void ffn_flood_kernel<true>(const __grid_constant__ KParams p);

// Called at launch time, not from a static initializer: this translation unit's static initialisation registers the
// kernels.
const void* flood_kernel(bool split) {
  return split ? reinterpret_cast<const void*>(ffn_flood_kernel<true>) : reinterpret_cast<const void*>(ffn_flood_kernel<false>);
}

}  // namespace profiled
}  // namespace ffn
