// train_kernels.cuh — one training step of ConvStack3DFFNModel on the device (namespace trk): forward pass with saved
// state, sigmoid cross-entropy head, input and weight gradients of the 3x3x3 convolutions on the tensor cores (bf16
// operands, fp32 accumulation, wgmma), deterministic reductions and the clipped optimizer update.
//
// Row space.  Every patch is stored zero-padded by one voxel on each side, (Z+2)(Y+2)(X+2) rows of 32 channels, the
// patches of a batch back to back after `guard` zero rows.  Tap (kz, ky, kx) of a SAME 3x3x3 convolution is then the
// constant row offset (kz-1) P2 + (ky-1) P + (kx-1) (P = X+2, P2 = (Y+2) P): no tap needs a mask.  Rows that are not
// inside a patch (its padding, the tail of the last tile) are written as zero by every kernel, so they supply the
// zero padding of the next convolution and add nothing to a weight gradient.
//
// bf16 operands are stored as [chunk][row][8] (chunk = 8 channels, 16 bytes per row): a tap is a shifted start
// address of a wgmma shared-memory descriptor, as in the flood kernel.  fp32 tensors (residual stream and its
// gradient) are [row][32].  The ReLU derivative of a convolution's input is one bit per channel, a uint32 per row.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include "sm90.cuh"

namespace trk {

constexpr int kTileRows = 128;     // output rows of one forward / dgrad tile (two consumer warpgroups of 64)
constexpr int kConvThreads = 256;
constexpr int kSplitRows = 1024;   // rows of one weight-gradient partial sum: fixed, so the sum order is too
constexpr int kKTile = 128;        // rows staged per weight-gradient k-tile
constexpr int kWgradThreads = 384; // one warpgroup per dx tap
constexpr int kHeadThreads = 256;
constexpr int kHeadCols = 65;      // head partials: 32 bias sums of the last conv, 32 conv_lom weight sums, 1 bias sum

enum { kFwdA = 0, kFwdB = 1, kBwdA = 2, kBwdB = 3 };
enum { kSgd = 0, kMomentum = 1, kAdam = 2 };

struct TGeom {
  int Z, Y, X;        // field of view
  int P, P2, Vp, V;   // padded row pitch, padded plane pitch, padded patch rows, voxels per patch
  int guard;          // zero rows before the first patch (>= P2 + P + 1)
  int batch;
  int data_rows;      // batch * Vp rounded up to kSplitRows: the rows every kernel covers
  int rows;           // rows allocated
};

// Voxel index of row r, or -1 when r is not inside a patch.
__device__ __forceinline__ int row_voxel(const TGeom& g, int r) {
  const int q = r - g.guard;
  if (q < 0 || q >= g.batch * g.Vp) return -1;
  const int b = q / g.Vp, rem = q - b * g.Vp;
  const int z = rem / g.P2, rem2 = rem - z * g.P2;
  const int y = rem2 / g.P, x = rem2 - y * g.P;
  if (z < 1 || z > g.Z || y < 1 || y > g.Y || x < 1 || x > g.X) return -1;
  return ((b * g.Z + z - 1) * g.Y + y - 1) * g.X + x - 1;
}

__device__ __forceinline__ int voxel_row(const TGeom& g, int v) {
  const int b = v / g.V, rem = v - b * g.V;
  const int yx = g.Y * g.X;
  const int z = rem / yx, y = (rem - z * yx) / g.X, x = rem - z * yx - y * g.X;
  return g.guard + b * g.Vp + (z + 1) * g.P2 + (y + 1) * g.P + x + 1;
}

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// D[64 x 32] (+)= A[64 x 16] * B[16 x 32], bf16 operands from shared memory, fp32 accumulators.  kTA / kTB = 1 read A /
// B MN-major (transposed), 0 K-major.  Fragment: d[4 nb + e] = D[16 w + l/4 + 8 (e/2)][8 nb + 2 (l%4) + e%2].
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n32k16_bf16(float (&d)[16], uint64_t ad, uint64_t bd, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(ad), "l"(bd), "r"(acc), "n"(kTA), "n"(kTB));
}

// Copies `rows` 16-byte rows of each of `chunks` chunks (global pitch gpitch rows, shared pitch spitch rows) with all
// threads of the block.
__device__ __forceinline__ void stage_rows(uint4* dst, const uint4* src, int chunks, int rows, int gpitch, int spitch) {
  for (int i = threadIdx.x; i < chunks * rows; i += blockDim.x) {
    const int c = i / rows, r = i - c * rows;
    dst[c * spitch + r] = src[(size_t)c * gpitch + r];
  }
}

// ------------------------------------------------------------------------------------------------------ weights
// fp32 DHWIO masters -> bf16 B operands.  Forward: per tap [k-chunk][n/8][n%8][k%8] with n = output, k = input channel
// (K-major).  dgrad: the same layout of W[26 - tap] transposed (n = input, k = output channel), so that the input
// gradient is the forward template run on the output gradient.
__global__ void pack_weights(const float* __restrict__ w, int cin, int kc, __nv_bfloat16* __restrict__ fwd,
                             __nv_bfloat16* __restrict__ dgrad) {
  const int n_el = 27 * cin * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += gridDim.x * blockDim.x) {
    const int tap = i / (cin * 32), ci = (i / 32) % cin, co = i % 32;
    const __nv_bfloat16 v = __float2bfloat16_rn(w[i]);
    fwd[(size_t)tap * kc * 256 + ((ci / 8) * 4 + co / 8) * 64 + (co % 8) * 8 + ci % 8] = v;
    if (dgrad) dgrad[(size_t)(26 - tap) * 4 * 256 + ((co / 8) * 4 + ci / 8) * 64 + (ci % 8) * 8 + co % 8] = v;
  }
}

// concat(image, seed) as the bf16 operand of conv0_a: channel 0 image, channel 1 seed (convstack_3d.py:86).
__global__ void stage_input(TGeom g, const float* __restrict__ image, const float* __restrict__ seed,
                            __nv_bfloat16* __restrict__ x0) {
  const int n = g.batch * g.V;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const int r = voxel_row(g, v);
    reinterpret_cast<__nv_bfloat162*>(x0)[(size_t)r * 4] = __floats2bfloat162_rn(image[v], seed[v]);
  }
}

// ------------------------------------------------------------------------------------------------------ convolution
// One SAME 3x3x3 convolution of 32 output channels over 128-row tiles: forward (weights `w` = forward pack, input the
// layer's bf16 operand) or input gradient (dgrad pack, input the bf16 output gradient).  Epilogues:
//   kFwdA  t = acc + bias:          next operand bf16(relu(t)), next mask t > 0
//   kFwdB  s = acc + bias (+ res):  res = s; next operand bf16(relu(s)) unless last; next mask s > 0
//   kBwdA  g = acc * mask:          g_out bf16(g), bias partial sums of g
//   kBwdB  G = res + acc * mask:    res = G; g_out bf16(G), bias partial sums of G
struct ConvArgs {
  const __nv_bfloat16* x;   // [KC][rows][8]
  const __nv_bfloat16* w;   // [27][KC][4][8][8]
  const float* bias;        // forward
  float* res;               // [rows][32]: residual stream (forward) or its gradient (kBwdB)
  const uint32_t* mask_in;  // backward: ReLU derivative of this convolution's input
  uint32_t* mask_out;       // forward: ReLU derivative of the next convolution's input
  __nv_bfloat16* out;       // [4][rows][8]: next operand (forward, may be null) or output gradient (backward)
  float* bias_part;         // backward: [tiles][32]
  int add_res;              // kFwdB: add the residual stream
  TGeom g;
};

template <int KC, int KIND>
__global__ void __launch_bounds__(kConvThreads) conv(ConvArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ float red[8][32];
  const TGeom& g = a.g;
  const int Rw = kTileRows + 2 * (g.P + 1);   // rows of one dz window
  uint4* ws = reinterpret_cast<uint4*>(smem);
  uint4* win = reinterpret_cast<uint4*>(smem + 27 * KC * 512);
  stage_rows(ws, reinterpret_cast<const uint4*>(a.w), 1, 27 * KC * 32, 0, 0);

  const int tid = threadIdx.x, wg = tid / 128, warp = (tid / 32) % 4, lane = tid % 32, q = lane % 4;
  const uint32_t w_addr = sm90::smem_u32(ws);
  const uint32_t a_addr = sm90::smem_u32(win) + wg * 64 * 16;
  const int ntiles = g.data_rows / kTileRows;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int r0 = g.guard + t * kTileRows;
    for (int dz = 0; dz < 3; ++dz)
      stage_rows(win + dz * KC * Rw, reinterpret_cast<const uint4*>(a.x) + r0 + (dz - 1) * g.P2 - (g.P + 1), KC, Rw,
                 g.rows, Rw);
    __syncthreads();
    fence_proxy_async_smem();
    float d[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) d[i] = 0.f;
    sm90::wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const int dz = tap / 9, dy = (tap / 3) % 3, dx = tap % 3;
      const uint32_t at = a_addr + (uint32_t)((dz * KC * Rw + dy * g.P + dx) * 16);
#pragma unroll
      for (int kk = 0; kk < KC / 2; ++kk) {
        const uint64_t ad = sm90::wgmma_desc(at + kk * 2 * Rw * 16, Rw * 16, 128);
        const uint64_t bd = sm90::wgmma_desc(w_addr + (tap * KC + 2 * kk) * 512, 512, 128);
        wgmma_m64n32k16_bf16<0, 0>(d, ad, bd, (tap | kk) ? 1u : 0u);
      }
    }
    sm90::wgmma_commit();
    sm90::wgmma_wait_all();

    float csum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) csum[i] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + wg * 64 + warp * 16 + lane / 4 + 8 * h;
      const bool in = row_voxel(g, r) >= 0;
      uint32_t bits = 0;
      uint32_t relu_grad = 0;
      if (KIND == kBwdA || KIND == kBwdB) relu_grad = in ? a.mask_in[r] : 0u;
#pragma unroll
      for (int nb = 0; nb < 4; ++nb) {
        const int c = 8 * nb + 2 * q;
        float v0 = d[4 * nb + 2 * h], v1 = d[4 * nb + 2 * h + 1];
        float2* res2 = reinterpret_cast<float2*>(a.res + (size_t)r * 32 + c);
        if (KIND == kFwdA || KIND == kFwdB) {
          v0 = __fadd_rn(v0, a.bias[c]);
          v1 = __fadd_rn(v1, a.bias[c + 1]);
          if (KIND == kFwdB && a.add_res) {
            const float2 s = *res2;
            v0 = __fadd_rn(v0, s.x);
            v1 = __fadd_rn(v1, s.y);
          }
          if (!in) v0 = v1 = 0.f;
          if (KIND == kFwdB) *res2 = make_float2(v0, v1);
          bits |= (uint32_t)(v0 > 0.f) << c | (uint32_t)(v1 > 0.f) << (c + 1);
          if (a.out)
            reinterpret_cast<__nv_bfloat162*>(a.out)[((size_t)nb * g.rows + r) * 4 + q] =
                __floats2bfloat162_rn(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
        } else {
          v0 = (relu_grad >> c & 1u) ? v0 : 0.f;
          v1 = (relu_grad >> (c + 1) & 1u) ? v1 : 0.f;
          if (KIND == kBwdB) {
            const float2 s = *res2;
            v0 = __fadd_rn(s.x, v0);
            v1 = __fadd_rn(s.y, v1);
            if (!in) v0 = v1 = 0.f;
            *res2 = make_float2(v0, v1);
          }
          reinterpret_cast<__nv_bfloat162*>(a.out)[((size_t)nb * g.rows + r) * 4 + q] = __floats2bfloat162_rn(v0, v1);
          csum[2 * nb] = __fadd_rn(csum[2 * nb], v0);
          csum[2 * nb + 1] = __fadd_rn(csum[2 * nb + 1], v1);
        }
      }
      if (KIND == kFwdA || KIND == kFwdB) {
        bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
        bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
        if (q == 0) a.mask_out[r] = bits;
      }
    }
    if (KIND == kBwdA || KIND == kBwdB) {
      // column sums of the tile in a fixed order: the 16 rows of a warp by a butterfly over lane / 4, then the 8 warps
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float s = csum[i];
        s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 4));
        s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 8));
        s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 16));
        if (lane < 4) red[tid / 32][8 * (i / 2) + 2 * q + i % 2] = s;
      }
      __syncthreads();
      if (tid < 32) {
        float s = 0.f;
        for (int w8 = 0; w8 < 8; ++w8) s = __fadd_rn(s, red[w8][tid]);
        a.bias_part[(size_t)t * 32 + tid] = s;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------ weight gradient
// dW[tap][ci][co] = sum over rows r of x[r + off(tap)][ci] * g[r][co].  One CTA per kSplitRows rows writes its partial
// sum; reduce_partials adds the partials in split order.  The MMA reads both operands MN-major (transposed) straight from
// the [chunk][row][8] tiles: M = (two or four dz/dy tap-row windows) x (input channels), N = 32 output channels, K = rows.
// Warpgroup w takes dx = w - 1.
template <int KC>
struct WgradShape {
  static constexpr int kWinPerMma = 8 / KC;                           // 64 / (8 KC) windows per M = 64
  static constexpr int kMmas = (9 + kWinPerMma - 1) / kWinPerMma;
  static constexpr int kWindows = kMmas * kWinPerMma;                 // the windows past 9 are never loaded, never read out
  static constexpr int kWinRows = kKTile + 2;
  static constexpr int kSmem = kWindows * KC * kWinRows * 16 + 4 * kKTile * 16;
};

template <int KC>
__global__ void __launch_bounds__(kWgradThreads) wgrad(const __nv_bfloat16* __restrict__ x,
                                                       const __nv_bfloat16* __restrict__ gout, float* __restrict__ part,
                                                       TGeom g, int cin) {
  using S = WgradShape<KC>;
  extern __shared__ __align__(128) unsigned char smem[];
  uint4* win = reinterpret_cast<uint4*>(smem);
  uint4* gs = win + S::kWindows * KC * S::kWinRows;
  const int tid = threadIdx.x, wg = tid / 128, warp = (tid / 32) % 4, lane = tid % 32, q = lane % 4;
  const uint32_t win_addr = sm90::smem_u32(win) + wg * 16, g_addr = sm90::smem_u32(gs);
  constexpr uint32_t Pc = S::kWinRows * 16;
  float d[S::kMmas][16];
#pragma unroll
  for (int j = 0; j < S::kMmas; ++j)
#pragma unroll
    for (int i = 0; i < 16; ++i) d[j][i] = 0.f;
  const int split = blockIdx.x;
  for (int kt = 0; kt < kSplitRows / kKTile; ++kt) {
    const int k0 = g.guard + split * kSplitRows + kt * kKTile;
    stage_rows(gs, reinterpret_cast<const uint4*>(gout) + k0, 4, kKTile, g.rows, kKTile);
    for (int w9 = 0; w9 < 9; ++w9)
      stage_rows(win + w9 * KC * S::kWinRows,
                 reinterpret_cast<const uint4*>(x) + k0 + (w9 / 3 - 1) * g.P2 + (w9 % 3 - 1) * g.P - 1, KC,
                 S::kWinRows, g.rows, S::kWinRows);
    __syncthreads();
    fence_proxy_async_smem();
    sm90::wgmma_fence();
#pragma unroll
    for (int j = 0; j < S::kMmas; ++j)
#pragma unroll
      for (int ks = 0; ks < kKTile / 16; ++ks) {
        const uint64_t ad = sm90::wgmma_desc(win_addr + j * S::kWinPerMma * KC * Pc + ks * 256, 128, Pc);
        const uint64_t bd = sm90::wgmma_desc(g_addr + ks * 256, 128, kKTile * 16);
        wgmma_m64n32k16_bf16<1, 1>(d[j], ad, bd, 1u);
      }
    sm90::wgmma_commit();
    sm90::wgmma_wait_all();
    __syncthreads();
  }
  const size_t n_el = (size_t)27 * cin * 32;
#pragma unroll
  for (int j = 0; j < S::kMmas; ++j)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int m = warp * 16 + lane / 4 + 8 * ((i % 4) / 2);
      const int n = 8 * (i / 4) + 2 * q + i % 2;
      const int window = j * S::kWinPerMma + m / (8 * KC), ci = m % (8 * KC);
      if (window < 9 && ci < cin) part[split * n_el + ((size_t)(window * 3 + wg) * cin + ci) * 32 + n] = d[j][i];
    }
}

// out[c] = sum over p = 0, 1, ... of part[p][c], in that order.
__global__ void reduce_partials(const float* __restrict__ part, int nparts, int ncols, float* __restrict__ out) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ncols; c += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s = __fadd_rn(s, part[(size_t)p * ncols + c]);
    out[c] = s;
  }
}

// ------------------------------------------------------------------------------------------------------ head
// Per voxel: logits = seed + (b_lom + <relu(s), w_lom>) (model.py:176-177), the weighted sigmoid cross-entropy
// max(x, 0) - x z + log1p(exp(-|x|)) (float64 sum per block) and d loss / d logits = (sigmoid(x) - z) (w / N).  Then the
// conv_lom backward: the residual gradient dl w_lom masked by s > 0 (fp32 and bf16) and the block's column sums of it
// (the last conv's bias gradient), of relu(s) dl (conv_lom's weight gradient) and of dl (its bias gradient).
struct HeadArgs {
  const float *seed, *labels, *loss_weights;   // loss_weights may be null (all 1)
  const float* res;                             // s of the last conv, [rows][32]
  const uint32_t* mask;                         // s > 0
  const float* lom;                             // w_lom[32], b_lom
  float inv_n;
  float *logits, *dlogits;
  float* gres;                                  // [rows][32]
  __nv_bfloat16* gout;                          // [4][rows][8]
  float* part;                                  // [blocks][kHeadCols]
  double* loss_part;                            // [blocks]
  TGeom g;
};

__global__ void __launch_bounds__(kHeadThreads) head(HeadArgs a) {
  __shared__ float red[kHeadThreads / 32][kHeadCols];
  __shared__ double lred[kHeadThreads / 32];
  const TGeom& g = a.g;
  const int v = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x % 32, warp = threadIdx.x / 32;
  const bool in = v < g.batch * g.V;
  float s[32];
  float dl = 0.f;
  double pl = 0.0;
  int r = 0;
  if (in) {
    r = voxel_row(g, v);
    const float4* s4 = reinterpret_cast<const float4*>(a.res + (size_t)r * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 t = s4[i];
      s[4 * i] = t.x; s[4 * i + 1] = t.y; s[4 * i + 2] = t.z; s[4 * i + 3] = t.w;
    }
    float dot = 0.f;
#pragma unroll
    for (int c = 0; c < 32; ++c) dot = __fadd_rn(dot, __fmul_rn(fmaxf(s[c], 0.f), a.lom[c]));
    const float x = __fadd_rn(a.seed[v], __fadd_rn(a.lom[32], dot));
    const float z = a.labels[v], w = a.loss_weights ? a.loss_weights[v] : 1.f;
    const float l = __fadd_rn(__fsub_rn(fmaxf(x, 0.f), __fmul_rn(x, z)), log1pf(expf(-fabsf(x))));
    pl = (double)__fmul_rn(l, w);
    const float sig = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
    dl = __fmul_rn(__fsub_rn(sig, z), __fmul_rn(w, a.inv_n));
    a.logits[v] = x;
    a.dlogits[v] = dl;
  } else {
#pragma unroll
    for (int c = 0; c < 32; ++c) s[c] = 0.f;
  }
  const uint32_t m = in ? a.mask[r] : 0u;
  float gcol[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) gcol[c] = (m >> c & 1u) ? __fmul_rn(dl, a.lom[c]) : 0.f;
  if (in) {
    float4* g4 = reinterpret_cast<float4*>(a.gres + (size_t)r * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) g4[i] = make_float4(gcol[4 * i], gcol[4 * i + 1], gcol[4 * i + 2], gcol[4 * i + 3]);
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) {
      __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(a.gout) + ((size_t)nb * g.rows + r) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = __floats2bfloat162_rn(gcol[8 * nb + 2 * k], gcol[8 * nb + 2 * k + 1]);
    }
  }
  // fixed-order block sums: butterfly within the warp, then the warps in order
  auto warp_sum = [&](float x) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) x = __fadd_rn(x, __shfl_xor_sync(0xffffffffu, x, o));
    return x;
  };
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const float a0 = warp_sum(gcol[c]);
    const float a1 = warp_sum(__fmul_rn(fmaxf(s[c], 0.f), dl));
    if (lane == 0) { red[warp][c] = a0; red[warp][32 + c] = a1; }
  }
  const float a2 = warp_sum(dl);
  double lp = pl;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) lp += __shfl_xor_sync(0xffffffffu, lp, o);
  if (lane == 0) { red[warp][64] = a2; lred[warp] = lp; }
  __syncthreads();
  if (threadIdx.x < kHeadCols) {
    float t = 0.f;
    for (int w8 = 0; w8 < kHeadThreads / 32; ++w8) t = __fadd_rn(t, red[w8][threadIdx.x]);
    a.part[(size_t)blockIdx.x * kHeadCols + threadIdx.x] = t;
  }
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w8 = 0; w8 < kHeadThreads / 32; ++w8) t += lred[w8];
    a.loss_part[blockIdx.x] = t;
  }
}

// ------------------------------------------------------------------------------------------------------ update
// Clip every gradient entry to +-clip (clip <= 0: none; model.py:127-157), then one optimizer step in fp32 with every
// operation rounded on its own (no contraction), as TF1's ApplyGradientDescent / ApplyMomentum / ApplyAdam state them:
//   sgd       w -= lr g
//   momentum  a = a m + g;  w -= a lr
//   adam      m += (g - m)(1 - b1);  v += (g g - v)(1 - b2);  w -= (m alpha) / (sqrt(v) + eps)
// with alpha = lr sqrt(1 - b2^t) / (1 - b1^t) formed on the host.
struct UpdateArgs {
  float *w, *a, *b;
  const float* grad;
  int n, optimizer;
  float clip, lr, momentum, one_minus_b1, one_minus_b2, alpha, eps;
};

__global__ void update(UpdateArgs u) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < u.n; i += gridDim.x * blockDim.x) {
    float g = u.grad[i];
    if (u.clip > 0.f) g = fminf(fmaxf(g, -u.clip), u.clip);
    float w = u.w[i];
    if (u.optimizer == kSgd) {
      w = __fsub_rn(w, __fmul_rn(u.lr, g));
    } else if (u.optimizer == kMomentum) {
      const float a = __fadd_rn(__fmul_rn(u.a[i], u.momentum), g);
      u.a[i] = a;
      w = __fsub_rn(w, __fmul_rn(a, u.lr));
    } else {
      float m = u.a[i], v = u.b[i];
      m = __fadd_rn(m, __fmul_rn(__fsub_rn(g, m), u.one_minus_b1));
      v = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(g, g), v), u.one_minus_b2));
      u.a[i] = m;
      u.b[i] = v;
      w = __fsub_rn(w, __fdiv_rn(__fmul_rn(m, u.alpha), __fadd_rn(__fsqrt_rn(v), u.eps)));
    }
    u.w[i] = w;
  }
}

}  // namespace trk
