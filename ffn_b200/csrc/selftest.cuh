// selftest.cuh — known-answer test of the sm_90a wgmma descriptors (host driver: ffn_selftest_wgmma in engine.cu).
// Not part of the product path: it pins the wgmma descriptor conventions the conv kernel relies on
// (K-major, no-swizzle core matrices; shifted start addresses = convolution taps).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "sm90.cuh"

namespace ffn {
namespace selftest {

// ---- D[128 x 96] = A[128 x K] * B[96 x K]^T with explicit descriptors ------------
// Two warpgroups, 64 rows each, like the conv kernel's consumers.  A in smem: [k-chunk][row] 16-byte
// units (row pitch 16 B, chunk pitch a_lbo); start address shifted by `a_shift_rows` rows (a
// convolution tap).  B: [k-chunk][12 n-groups][8][8].
__global__ void wgmma_kat_kernel(const __half* a_g, int a_rows_total, const __half* b_g, int kchunks,
                                 int a_shift_rows, uint32_t a_lbo, uint32_t a_sbo, uint32_t b_lbo, uint32_t b_sbo,
                                 float* d_out) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __half* a_s = reinterpret_cast<__half*>(smem);
  __half* b_s = a_s + (size_t)kchunks * a_rows_total * 8;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < kchunks * a_rows_total * 8; i += blockDim.x) a_s[i] = a_g[i];
  for (int i = tid; i < kchunks * 96 * 8; i += blockDim.x) b_s[i] = b_g[i];
  sm90::fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor core (async proxy)
  __syncthreads();
  const int row0 = (warp >> 2) * 64;
  float d[48];
  for (int i = 0; i < 48; ++i) d[i] = 0.f;
  sm90::wgmma_fence();
  for (int j = 0; j < kchunks / 2; ++j) {
    const uint32_t a_addr = sm90::smem_u32(a_s) + (uint32_t)((2 * j) * a_rows_total + a_shift_rows + row0) * 16;
    const uint32_t b_addr = sm90::smem_u32(b_s) + (uint32_t)(2 * j) * 12 * 128;
    sm90::wgmma_m64n96k16(d, sm90::wgmma_desc(a_addr, a_lbo, a_sbo), sm90::wgmma_desc(b_addr, b_lbo, b_sbo), j > 0 ? 1u : 0u);
  }
  sm90::wgmma_commit();
  sm90::wgmma_wait_all();
  for (int i = 0; i < 48; ++i) {
    const int row = row0 + (warp & 3) * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
    const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    d_out[(size_t)row * 96 + col] = d[i];
  }
}

}  // namespace selftest
}  // namespace ffn
