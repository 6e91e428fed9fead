// seed_kernels.cuh — PolicyPeaks on the device (SURVEY.md 8f rank 1): once the flood fill runs at
// thousands of FoV steps/s the host seed policy (Sobel -> adaptive threshold -> Euclidean distance
// transform -> local maxima; ffn/inference/seed.py:142-199) dominates the end-to-end time.
// Every stage is an HBM-bound grid-stride or line-parallel kernel over the canvas:
//   sobel_mag      27-point stencil, reflect boundary           8 B/voxel  (read f32/u8, write f32)
//   gauss_pass x3  1-D correlation, radius 33, reflect          8 B/voxel per pass
//   edges_kernel   edges > threshold, masks                     9 B/voxel
//   edt_x / edt_line x2  exact squared EDT (two sweeps, then lower envelope of parabolas per line)
//   peaks_kernel   7x7x7 maximum of (distance, tie-break noise) keys, plateau-free arg-max test; like
//                  peak_local_max's default exclude_border=True (seed.py:191) it drops every peak closer than
//                  3 voxels to the array border on any axis, whatever the canvas margin
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

namespace ffn {
namespace seedk {

constexpr float kBig = 1e18f;

__device__ __forceinline__ int reflect(int i, int n) {   // scipy 'reflect': d c b a | a b c d | d c b a
  if (n == 1) return 0;
  const int period = 2 * n;
  i = i % period;
  if (i < 0) i += period;
  return i < n ? i : period - 1 - i;
}

__device__ __forceinline__ float load_image(const void* img, int is_u8, float mean, float stddev, size_t i) {
  if (is_u8) return __fdiv_rn(__fsub_rn((float)reinterpret_cast<const uint8_t*>(img)[i], mean), stddev);
  return reinterpret_cast<const float*>(img)[i];
}

// ndimage.generic_gradient_magnitude(image, ndimage.sobel): per axis a derivative [-1, 0, 1] along the
// axis and [1, 2, 1] smoothing along the other two (ascending axis order), each 1-D pass accumulated in
// float64 and stored as float32 exactly like ndimage.correlate1d; then float32 squares, sum and sqrt.
__device__ __forceinline__ float smooth3(float a, float b, float c) {
  return (float)((double)b * 2.0 + ((double)a + (double)c));
}

__global__ void sobel_mag(const void* img, int is_u8, float mean, float stddev, float* out, int sz, int sy, int sx) {
  const size_t n = (size_t)sz * sy * sx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % sx), y = (int)((i / sx) % sy), z = (int)(i / ((size_t)sx * sy));
    float v[3][3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int zz = reflect(z + a - 1, sz);
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int yy = reflect(y + b - 1, sy);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int xx = reflect(x + c - 1, sx);
          v[a][b][c] = load_image(img, is_u8, mean, stddev, ((size_t)zz * sy + yy) * sx + xx);
        }
      }
    }
    float t[3], g[3];
    // axis 0 (z): derivative along z, smooth along y, then along x
#pragma unroll
    for (int c = 0; c < 3; ++c) t[c] = smooth3(v[2][0][c] - v[0][0][c], v[2][1][c] - v[0][1][c], v[2][2][c] - v[0][2][c]);
    g[0] = smooth3(t[0], t[1], t[2]);
    // axis 1 (y): derivative along y, smooth along z, then along x
#pragma unroll
    for (int c = 0; c < 3; ++c) t[c] = smooth3(v[0][2][c] - v[0][0][c], v[1][2][c] - v[1][0][c], v[2][2][c] - v[2][0][c]);
    g[1] = smooth3(t[0], t[1], t[2]);
    // axis 2 (x): derivative along x, smooth along z, then along y
#pragma unroll
    for (int b = 0; b < 3; ++b) t[b] = smooth3(v[0][b][2] - v[0][b][0], v[1][b][2] - v[1][b][0], v[2][b][2] - v[2][b][0]);
    g[2] = smooth3(t[0], t[1], t[2]);
    float acc = __fmul_rn(g[0], g[0]);
    acc = __fadd_rn(acc, __fmul_rn(g[1], g[1]));
    acc = __fadd_rn(acc, __fmul_rn(g[2], g[2]));
    out[i] = sqrtf(acc);
  }
}

// One separable pass of ndimage.gaussian_filter (mode='reflect'): float64 accumulation over the symmetric
// pairs from the outermost tap inwards (ndimage.correlate1d's symmetric branch), float32 store.
// weights[0..radius]: weights[0] is the centre tap; normalised on the host.
__global__ void gauss_pass(const float* in, float* out, const double* weights, int radius, int axis, int sz, int sy,
                           int sx) {
  const size_t n = (size_t)sz * sy * sx;
  const int len = axis == 0 ? sz : (axis == 1 ? sy : sx);
  const size_t st = axis == 0 ? (size_t)sy * sx : (axis == 1 ? (size_t)sx : 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % sx), y = (int)((i / sx) % sy), z = (int)(i / ((size_t)sx * sy));
    const int pos = axis == 0 ? z : (axis == 1 ? y : x);
    const size_t base = i - (size_t)pos * st;
    double acc = (double)in[i] * weights[0];
    if (pos >= radius && pos + radius < len) {
      for (int k = radius; k >= 1; --k)
        acc += ((double)in[i - (size_t)k * st] + (double)in[i + (size_t)k * st]) * weights[k];
    } else {
      for (int k = radius; k >= 1; --k)
        acc += ((double)in[base + (size_t)reflect(pos - k, len) * st] + (double)in[base + (size_t)reflect(pos + k, len) * st]) *
               weights[k];
    }
    out[i] = (float)acc;
  }
}

// filt_edges = edges > thresh (| masks); the distance transform input is 0 at edges, "infinite" elsewhere.
__global__ void edges_kernel(const float* edges, const float* thresh, const uint8_t* mask, const uint8_t* seed_mask,
                             float* d, size_t n, unsigned long long* n_free) {
  unsigned long long local = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const bool edge = edges[i] > thresh[i] || (mask && mask[i]) || (seed_mask && seed_mask[i]);
    d[i] = edge ? 0.f : kBig;
    local += edge ? 0 : 1;
  }
  if (local) atomicAdd(n_free, local);
}

// First EDT pass along x: squared distance (in physical units) to the nearest zero of the same x-line.
__global__ void edt_x(float* d, int sz, int sy, int sx, float wx) {
  const size_t lines = (size_t)sz * sy;
  for (size_t l = (size_t)blockIdx.x * blockDim.x + threadIdx.x; l < lines; l += (size_t)gridDim.x * blockDim.x) {
    float* row = d + l * sx;
    float dist = kBig;
    for (int x = 0; x < sx; ++x) {
      dist = row[x] == 0.f ? 0.f : (dist >= kBig ? kBig : dist + wx);
      row[x] = dist;
    }
    dist = kBig;
    for (int x = sx - 1; x >= 0; --x) {
      dist = row[x] == 0.f ? 0.f : (dist >= kBig ? kBig : dist + wx);
      const float m = fminf(row[x], dist);
      row[x] = m >= kBig ? kBig : m * m;
    }
  }
}

// Later EDT passes (axis = 1: y, axis = 0: z): D(q) = min_p f(p) + (w (q - p))^2 via the lower envelope of
// parabolas (Felzenszwalb & Huttenlocher).  One thread per line; the envelope arrays live in global
// scratch laid out [k][line] so that neighbouring threads touch neighbouring addresses.
__global__ void edt_line(float* d, int axis, int sz, int sy, int sx, float w, int* vbuf, double* zbuf) {
  const int len = axis == 0 ? sz : sy;
  const size_t st = axis == 0 ? (size_t)sy * sx : (size_t)sx;
  const size_t lines = axis == 0 ? (size_t)sy * sx : (size_t)sz * sx;
  const double w2 = (double)w * (double)w;
  for (size_t l = (size_t)blockIdx.x * blockDim.x + threadIdx.x; l < lines; l += (size_t)gridDim.x * blockDim.x) {
    size_t base;
    if (axis == 0) {
      base = l;                                            // (y, x) fixed
    } else {
      const size_t z = l / sx, x = l % sx;
      base = z * (size_t)sy * sx + x;                      // (z, x) fixed
    }
    int k = -1;
    for (int q = 0; q < len; ++q) {
      const float fq = d[base + (size_t)q * st];
      if (fq >= kBig) continue;
      double s = -CUDART_INF;
      while (k >= 0) {
        const int vk = vbuf[(size_t)k * lines + l];
        const double fv = (double)d[base + (size_t)vk * st];   // still the INPUT value: outputs are written later
        s = (((double)fq + w2 * q * q) - (fv + w2 * vk * vk)) / (2.0 * w2 * (q - vk));
        if (s <= zbuf[(size_t)k * lines + l]) {
          --k;
          s = -CUDART_INF;
        } else {
          break;
        }
      }
      ++k;
      vbuf[(size_t)k * lines + l] = q;
      zbuf[(size_t)k * lines + l] = s;
    }
    if (k < 0) continue;   // no finite value on this line: stays "infinite"
    // The outputs overwrite the inputs, so cache the envelope's f(v) first.
    const int nk = k + 1;
    for (int j = 0; j < nk; ++j) {
      const int vj = vbuf[(size_t)j * lines + l];
      zbuf[(size_t)(len + j) * lines + l] = (double)d[base + (size_t)vj * st];
    }
    int j = 0;
    for (int q = 0; q < len; ++q) {
      while (j + 1 < nk && zbuf[(size_t)(j + 1) * lines + l] < (double)q) ++j;
      const int vj = vbuf[(size_t)j * lines + l];
      const double dq = (double)(q - vj);
      d[base + (size_t)q * st] = (float)(w2 * dq * dq + zbuf[(size_t)(len + j) * lines + l]);
    }
  }
}

// dt = sqrt(squared distance); excluded voxels and "infinite" distances become -1 (seed.py:187-188).
__global__ void finish_dt(float* d, const int* seg, const uint8_t* mask, const uint8_t* seed_mask, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const bool excl = (seg && seg[i] > 0) || (mask && mask[i]) || (seed_mask && seed_mask[i]);
    const float v = d[i];
    d[i] = (excl || v >= kBig) ? -1.f : sqrtf(v);
  }
}

// peak_local_max(dt + noise * 1e-4, min_distance = 3, threshold_abs = 0): a voxel is a seed iff its key
// (dt, noise) is the maximum of its 7x7x7 neighbourhood (edge-clamped), dt + 1e-4 * noise > 0, and it lies at
// least `radius` voxels from the array border on every axis (exclude_border=True).
// Comparing (dt, noise) lexicographically equals comparing the float64 sums because distinct dt
// values differ by far more than 1e-4.
__global__ void peaks_kernel(const float* dt, const double* noise, int sz, int sy, int sx, int radius, int* coords,
                             unsigned long long cap, unsigned long long* count) {
  const size_t n = (size_t)sz * sy * sx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % sx), y = (int)((i / sx) % sy), z = (int)(i / ((size_t)sx * sy));
    if (z < radius || z >= sz - radius || y < radius || y >= sy - radius || x < radius || x >= sx - radius) continue;
    const float v = dt[i];
    const double nv = noise ? noise[i] : 0.0;
    if (!((double)v + nv * 1e-4 > 0.0)) continue;
    bool is_max = true;
    for (int dz = -radius; dz <= radius && is_max; ++dz) {
      const int zz = min(max(z + dz, 0), sz - 1);
      for (int dy = -radius; dy <= radius && is_max; ++dy) {
        const int yy = min(max(y + dy, 0), sy - 1);
        const size_t rb = ((size_t)zz * sy + yy) * sx;
        for (int dx = -radius; dx <= radius; ++dx) {
          const int xx = min(max(x + dx, 0), sx - 1);
          const size_t j = rb + xx;
          const float u = dt[j];
          if (u > v || (u == v && noise && noise[j] > nv)) {
            is_max = false;
            break;
          }
        }
      }
    }
    if (!is_max) continue;
    const unsigned long long slot = atomicAdd(count, 1ull);
    if (slot < cap) {
      coords[3 * slot + 0] = z;
      coords[3 * slot + 1] = y;
      coords[3 * slot + 2] = x;
    }
  }
}

// ---- PolicyPeaks2d / PolicyFillEmptySpace / PolicyMaxPeaks (seed.py:202-352) -------------------------------
//   sobel_mag2d      9-point stencil per z-slice, reflect boundary      8 B/voxel
//   gauss_pass x2    axes 1 and 2 only (2-D gaussian per slice)         8 B/voxel per pass
//   edges_kernel     movement mask only (seed_mask = NULL)              9 B/voxel
//   empty_input      seg == 0 -> EDT input                              8 B/voxel
//   masked_image     image with excluded voxels set to 0                10-13 B/voxel
//   edt_x, edt_line  as above (2-D: x and y sweeps only), then dt_finish 8 B/voxel
//   peak_keys        float64 key = (double)value + noise * 1e-4, min/max 20 B/voxel (12 with a noise plane in L2)
//   slice_min_keys   2-D threshold_abs=None only: each z-slice's minimum key  8 B/voxel
//   box_max x2-3     separable (2r+1) maximum of the keys, one axis each 16 B/voxel per pass
//   peaks_select     key == box maximum, threshold, border              16 B/voxel

// ndimage.generic_gradient_magnitude(slice, ndimage.sobel) on every z-slice: per in-plane axis the derivative
// along it and [1, 2, 1] smoothing along the other, each 1-D pass stored as float32 (see sobel_mag).
__global__ void sobel_mag2d(const void* img, int is_u8, float mean, float stddev, float* out, int sz, int sy, int sx) {
  const size_t n = (size_t)sz * sy * sx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % sx), y = (int)((i / sx) % sy), z = (int)(i / ((size_t)sx * sy));
    const size_t zb = (size_t)z * sy * sx;
    float v[3][3];
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const int yy = reflect(y + b - 1, sy);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[b][c] = load_image(img, is_u8, mean, stddev, zb + (size_t)yy * sx + reflect(x + c - 1, sx));
    }
    // axis y: derivative along y, smooth along x; axis x: derivative along x, smooth along y
    const float gy = smooth3(v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]);
    const float gx = smooth3(v[0][2] - v[0][0], v[1][2] - v[1][0], v[2][2] - v[2][0]);
    out[i] = sqrtf(__fadd_rn(__fmul_rn(gy, gy), __fmul_rn(gx, gx)));
  }
}

// edt.edt(segmentation == 0): labelled voxels (including the -1 markers) are the background.
__global__ void empty_input(const int* seg, float* d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d[i] = seg[i] == 0 ? kBig : 0.f;
}

// Squared distance -> distance; "infinite" (no background voxel on the slice / canvas) -> +inf, never a peak.
__global__ void dt_finish(float* d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = d[i];
    d[i] = v >= kBig ? CUDART_INF_F : sqrtf(v);
  }
}

// img = image.astype(float32); img[get_exclusion_mask()] = 0 (seed.py:343-345).
__global__ void masked_image(const void* img, int is_u8, float mean, float stddev, const int* seg, const uint8_t* mask,
                             const uint8_t* seed_mask, float* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const bool excl = seg[i] > 0 || (mask && mask[i]) || (seed_mask && seed_mask[i]);
    out[i] = excl ? 0.f : load_image(img, is_u8, mean, stddev, i);
  }
}

// Order-preserving map of a double onto uint64, so that atomicMin / atomicMax order keys.
__device__ __forceinline__ unsigned long long ordered_bits(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double from_ordered_bits(unsigned long long u) {
  return __longlong_as_double((long long)((u >> 63) ? (u & 0x7fffffffffffffffull) : ~u));
}

// key = values + noise * 1e-4 exactly as numpy forms it (float32 -> float64, one multiply and one add, each
// rounded to nearest; no FMA).  noise[i % noise_period] (period = Y*X for the per-slice plane, 0 = no noise).
// minmax[0] / [1] receive the ordered bits of the minimum / maximum finite key (threshold_abs=None and
// threshold_rel of peak_local_max).
__global__ void peak_keys(const float* values, const double* noise, size_t noise_period, double* keys, size_t n,
                          unsigned long long* minmax) {
  unsigned long long lo = ~0ull, hi = 0ull;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double k = (double)values[i];
    if (noise_period) k = __dadd_rn(k, __dmul_rn(noise[i % noise_period], 1e-4));
    keys[i] = k;
    if (isfinite(k)) {
      const unsigned long long o = ordered_bits(k);
      lo = o < lo ? o : lo;
      hi = o > hi ? o : hi;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const unsigned long long l2 = __shfl_down_sync(0xffffffffu, lo, off), h2 = __shfl_down_sync(0xffffffffu, hi, off);
    lo = l2 < lo ? l2 : lo;
    hi = h2 > hi ? h2 : hi;
  }
  if ((threadIdx.x & 31) == 0 && lo <= hi) {
    atomicMin(&minmax[0], lo);
    atomicMax(&minmax[1], hi);
  }
}

// threshold_abs=None of PolicyPeaks2d: peak_local_max runs once per z-slice (PolicyPeaks2d), so the threshold is
// each slice's own minimum key.  One block per slice; slice_min[z] (preset to ~0) receives its ordered bits.
__global__ void slice_min_keys(const double* keys, size_t slice_n, unsigned long long* slice_min) {
  const double* s = keys + (size_t)blockIdx.x * slice_n;
  unsigned long long lo = ~0ull;
  for (size_t i = threadIdx.x; i < slice_n; i += blockDim.x) {
    const double k = s[i];
    if (isfinite(k)) {
      const unsigned long long o = ordered_bits(k);
      lo = o < lo ? o : lo;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const unsigned long long l2 = __shfl_down_sync(0xffffffffu, lo, off);
    lo = l2 < lo ? l2 : lo;
  }
  if ((threadIdx.x & 31) == 0 && lo != ~0ull) atomicMin(&slice_min[blockIdx.x], lo);
}

// One separable pass of ndimage.maximum_filter(size = 2 radius + 1, mode='nearest') along `axis`: with edge
// clamping the window maximum is the maximum over the window's part inside the array.  Exact (max is
// associative), so three passes equal the (2r+1)^3 box; 15 cached loads per voxel at radius 7.
__global__ void box_max(const double* in, double* out, int radius, int axis, int sz, int sy, int sx) {
  const size_t n = (size_t)sz * sy * sx;
  const int len = axis == 0 ? sz : (axis == 1 ? sy : sx);
  const size_t st = axis == 0 ? (size_t)sy * sx : (axis == 1 ? (size_t)sx : 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % sx), y = (int)((i / sx) % sy), z = (int)(i / ((size_t)sx * sy));
    const int pos = axis == 0 ? z : (axis == 1 ? y : x);
    const int lo = max(pos - radius, 0), hi = min(pos + radius, len - 1);
    const double* base = in + (i - (size_t)pos * st);
    double m = base[(size_t)lo * st];
    for (int q = lo + 1; q <= hi; ++q) m = fmax(m, base[(size_t)q * st]);
    out[i] = m;
  }
}

// peak_local_max by its documented definition: key == maximum of its box, key > max(threshold_abs,
// threshold_rel * max key) (threshold_abs = the minimum key when abs_is_min; the minimum key of the voxel's z-slice
// when slice_min is given), finite, and at least border[a] voxels from the array border on every axis a.  Appends
// (z, y, x) to coords (up to cap); *count = peaks.
__global__ void peaks_select(const double* keys, const double* boxmax, double threshold_abs, int abs_is_min, int use_rel,
                             double threshold_rel, const unsigned long long* minmax, const unsigned long long* slice_min,
                             int bz, int by, int bx, int sz, int sy, int sx, int* coords, unsigned long long cap,
                             unsigned long long* count) {
  double thr = abs_is_min ? from_ordered_bits(minmax[0]) : threshold_abs;
  const double thr_rel = use_rel ? __dmul_rn(threshold_rel, from_ordered_bits(minmax[1])) : -CUDART_INF;
  thr = fmax(thr, thr_rel);
  const size_t n = (size_t)sz * sy * sx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const double k = keys[i];
    const int z = (int)(i / ((size_t)sx * sy));
    const double t = slice_min ? fmax(from_ordered_bits(slice_min[z]), thr_rel) : thr;
    if (!(isfinite(k) && k > t && k == boxmax[i])) continue;
    const int x = (int)(i % sx), y = (int)((i / sx) % sy);
    if (z < bz || z >= sz - bz || y < by || y >= sy - by || x < bx || x >= sx - bx) continue;
    const unsigned long long slot = atomicAdd(count, 1ull);
    if (slot < cap) {
      coords[3 * slot + 0] = z;
      coords[3 * slot + 1] = y;
      coords[3 * slot + 2] = x;
    }
  }
}

}  // namespace seedk
}  // namespace ffn
