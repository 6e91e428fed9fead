// selftest.cuh — known-answer test of the sm_90a wgmma descriptors.
// Not part of the product path: it pins the wgmma descriptor conventions the conv kernel relies on
// (K-major, no-swizzle core matrices; shifted start addresses = convolution taps).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

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

inline float host_half_round(float v) { return __half2float(__float2half_rn(v)); }

#define ST_CUDA(expr)                                                                      \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      *err = std::string(#expr) + ": " + cudaGetErrorString(e__);                          \
      return 1;                                                                            \
    }                                                                                      \
  } while (0)

inline int run_kat(double* out, std::string* err) {
  const int K = 64, kch = K / 8, rows_total = 256;   // A window has room for shifts up to 127 rows
  std::vector<float> a((size_t)rows_total * K), b((size_t)96 * K);
  unsigned s = 12345u;
  auto rnd = [&]() {
    s = s * 1664525u + 1013904223u;
    return (float)((int)((s >> 20) & 15) - 8) * 0.125f;
  };
  for (auto& v : a) v = rnd();
  for (auto& v : b) v = rnd();
  std::vector<__half> ah((size_t)kch * rows_total * 8), bh((size_t)kch * 96 * 8);
  for (int r = 0; r < rows_total; ++r)
    for (int k = 0; k < K; ++k) ah[((size_t)(k / 8) * rows_total + r) * 8 + k % 8] = __float2half_rn(a[(size_t)r * K + k]);
  for (int n = 0; n < 96; ++n)
    for (int k = 0; k < K; ++k)
      bh[(((size_t)(k / 8)) * 12 + n / 8) * 64 + (n % 8) * 8 + k % 8] = __float2half_rn(b[(size_t)n * K + k]);
  __half *d_a = nullptr, *d_b = nullptr;
  float* d_d = nullptr;
  ST_CUDA(cudaMalloc(&d_a, ah.size() * 2));
  ST_CUDA(cudaMalloc(&d_b, bh.size() * 2));
  ST_CUDA(cudaMalloc(&d_d, 128 * 96 * 4));
  ST_CUDA(cudaMemcpy(d_a, ah.data(), ah.size() * 2, cudaMemcpyHostToDevice));
  ST_CUDA(cudaMemcpy(d_b, bh.data(), bh.size() * 2, cudaMemcpyHostToDevice));
  // the swapped-descriptor case strides 8-row groups by a_lbo / b_lbo and reaches ~58 KB past the operand base:
  // allocate that much so the wrong answer is a wrong number, not an out-of-range shared-memory read
  const int smem = 64 * 1024;
  ST_CUDA(cudaFuncSetAttribute(wgmma_kat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const uint32_t a_lbo = rows_total * 16, a_sbo = 128, b_lbo = 12 * 128, b_sbo = 128;
  struct Case { int shift; bool swapped; };
  const Case cases[4] = {{0, false}, {3, false}, {35, false}, {0, true}};
  for (int ci = 0; ci < 4; ++ci) {
    const Case& c = cases[ci];
    ST_CUDA(cudaMemset(d_d, 0xff, 128 * 96 * 4));
    wgmma_kat_kernel<<<1, 256, smem>>>(d_a, rows_total, d_b, kch, c.shift, c.swapped ? a_sbo : a_lbo,
                                       c.swapped ? a_lbo : a_sbo, c.swapped ? b_sbo : b_lbo,
                                       c.swapped ? b_lbo : b_sbo, d_d);
    ST_CUDA(cudaGetLastError());
    ST_CUDA(cudaDeviceSynchronize());
    std::vector<float> d(128 * 96);
    ST_CUDA(cudaMemcpy(d.data(), d_d, d.size() * 4, cudaMemcpyDeviceToHost));
    double worst = 0;
    for (int r = 0; r < 128; ++r)
      for (int n = 0; n < 96; ++n) {
        double ref = 0;
        for (int k = 0; k < K; ++k) ref += (double)a[(size_t)(r + c.shift) * K + k] * (double)b[(size_t)n * K + k];
        const double e = std::fabs(ref - (double)d[(size_t)r * 96 + n]);
        if (!(e <= worst)) worst = std::isnan(e) ? 1e30 : e;
      }
    out[ci] = worst;
  }
  cudaFree(d_a);
  cudaFree(d_b);
  cudaFree(d_d);
  return 0;
}

inline int run(int device, double* out, int n_out, std::string* err) {
  ST_CUDA(cudaSetDevice(device));
  for (int i = 0; i < n_out; ++i) out[i] = -1.0;
  return run_kat(out, err);
}

}  // namespace selftest
}  // namespace ffn
