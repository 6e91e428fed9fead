// flood_plain.cu — the product build of the persistent kernel: flood_kernel.cuh without device cycle counters.
#define FFN_KNS plain
#define FFN_PROFILE 0
#include "flood_kernel.cuh"

namespace ffn {
namespace plain {

template __global__ void ffn_flood_kernel<false>(const __grid_constant__ KParams p);
template __global__ void ffn_flood_kernel<true>(const __grid_constant__ KParams p);

// Called at launch time, not from a static initializer: this translation unit's static initialisation registers the
// kernels.
const void* flood_kernel(bool split) {
  return split ? reinterpret_cast<const void*>(ffn_flood_kernel<true>) : reinterpret_cast<const void*>(ffn_flood_kernel<false>);
}

}  // namespace plain
}  // namespace ffn
