// partition_kernels.cuh — partition map of a labelled volume (compute_partitions.py:115-204) on the device.
// For every voxel of a kept label in the VALID region, the number of voxels of the same label in the (2r+1)^3
// local-object-mask box, quantized by the thresholds; 255 where the box holds a masked voxel or the voxel lies in an
// exclusion sphere.  Passes (V: voxels of the volume, B: voxels of the labels' grown boxes, O: output voxels):
//   compact_ids      uint64 label -> compact id by binary search, dust cleared,   12 B/V, + 8 B/V with dust
//                    and per-label bounding boxes (warp-aggregated atomics)      (unique ids in L2)
//   count_x          per grown box: x-window count of `compact == k`               4 B/B read, 4 B/B written
//   count_y          y-window sum of count_x                                        4 B/B read, 4 B/B written
//   count_z          z-window sum of count_y at the label's VALID voxels, quantized 8 B/B read, 1 B written per voxel
//   box_any x3       separable any() of the mask over the box (mask only)          2 B/V per pass
//   finish           mask / exclusion spheres -> 255, 256-bin histogram            2 B/O (3 B/O with a mask)
// Labels are disjoint, so the count passes of different labels never write the same output voxel.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ffn {
namespace ptk {

typedef unsigned long long u64;

constexpr int kDust = -2;     // run code of an id cleared as dust (set to 0 in the labels)
constexpr int kSkipped = -1;  // run code of 0 and of an id outside the whitelist

// One label's grown box within a group.  `line[p]` is the first line of this box in pass p's numbering of the
// group's lines: pass 0 numbers (z, y) x-lines, pass 1 (z, x) y-lines, pass 2 (y, x) z-lines.
struct LabelBox {
  int k;           // compact id
  int lo[3];       // box start (z, y, x) in the volume
  int n[3];        // box extent
  int pad;
  long long off;   // first scratch voxel of the box
  long long line[3];
};

struct Geometry {
  int s[3];        // volume extent (z, y, x)
  int r[3];        // LOM radius (z, y, x)
  int o[3];        // VALID extent, s - 2 r
};

// Exclusion sphere in output-voxel terms: voxel o is inside when (o_x + corner_x - x)^2 + ... <= r^2, in int64
// (wrapping, as numpy) when `integer`, else in float64 summed left to right without contraction.
struct Sphere {
  long long c[3];  // x, y, z
  long long r2;
  double fc[3];
  double fr2;
  int integer;
  int pad;
};

// labels -> compact id (kSkipped for none), dust written back as 0, and each compact id's bounding box.  Every lane
// of a warp runs the same number of iterations, so a warp whose voxels share one id reduces its box with one set of
// atomics.
__global__ void compact_ids(u64* labels, size_t n, const u64* uniq, int nruns, const int* code, int* compact,
                            int* bmin, int* bmax, int sy, int sx) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t n_round = (n + 31) & ~(size_t)31;
  const unsigned full = 0xffffffffu;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    int k = kSkipped;
    unsigned z = 0, y = 0, x = 0;
    if (i < n) {
      const u64 lab = labels[i];
      int lo = 0, hi = nruns;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (uniq[mid] < lab) lo = mid + 1; else hi = mid;
      }
      const int c = code[lo];
      if (c == kDust) labels[i] = 0;
      k = c >= 0 ? c : kSkipped;
      compact[i] = k;
      x = (unsigned)(i % sx);
      y = (unsigned)((i / sx) % sy);
      z = (unsigned)(i / ((size_t)sx * sy));
    }
    const int k0 = __shfl_sync(full, k, 0);
    if (__all_sync(full, k == k0)) {
      if (k0 < 0) continue;
      const unsigned zl = __reduce_min_sync(full, z), yl = __reduce_min_sync(full, y), xl = __reduce_min_sync(full, x);
      const unsigned zh = __reduce_max_sync(full, z), yh = __reduce_max_sync(full, y), xh = __reduce_max_sync(full, x);
      if ((threadIdx.x & 31) == 0) {
        atomicMin(&bmin[3 * k0], (int)zl);
        atomicMin(&bmin[3 * k0 + 1], (int)yl);
        atomicMin(&bmin[3 * k0 + 2], (int)xl);
        atomicMax(&bmax[3 * k0], (int)zh);
        atomicMax(&bmax[3 * k0 + 1], (int)yh);
        atomicMax(&bmax[3 * k0 + 2], (int)xh);
      }
    } else if (k >= 0) {
      atomicMin(&bmin[3 * k], (int)z);
      atomicMin(&bmin[3 * k + 1], (int)y);
      atomicMin(&bmin[3 * k + 2], (int)x);
      atomicMax(&bmax[3 * k], (int)z);
      atomicMax(&bmax[3 * k + 1], (int)y);
      atomicMax(&bmax[3 * k + 2], (int)x);
    }
  }
}

// The box holding line `l` of pass P: the last box whose first line is <= l.
template <int P>
__device__ __forceinline__ int box_of(const LabelBox* boxes, int nb, long long l) {
  int lo = 0, hi = nb - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (boxes[mid].line[P] <= l) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// A[z, y, x] = #{x' in [x - rx, x + rx] : compact(z, y, x') == k} over the box, one thread per x-line.
__global__ void count_x(const int* __restrict__ compact, const LabelBox* boxes, int nb, long long nlines, Geometry g,
                        int* __restrict__ A) {
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    const LabelBox b = boxes[box_of<0>(boxes, nb, l)];
    const long long t = l - b.line[0];
    const int z = (int)(t / b.n[1]), y = (int)(t % b.n[1]);
    const int* row = compact + ((size_t)(b.lo[0] + z) * g.s[1] + (b.lo[1] + y)) * g.s[2] + b.lo[2];
    int* out = A + b.off + ((long long)z * b.n[1] + y) * b.n[2];
    const int nx = b.n[2], r = g.r[2], k = b.k;
    int sum = 0;
    for (int x = 0; x <= r && x < nx; ++x) sum += row[x] == k;
    for (int x = 0; x < nx; ++x) {
      out[x] = sum;
      if (x + r + 1 < nx) sum += row[x + r + 1] == k;
      if (x - r >= 0) sum -= row[x - r] == k;
    }
  }
}

// B[z, y, x] = sum of A[z, y', x] over y' in [y - ry, y + ry], one thread per (z, x) line.
__global__ void count_y(const int* __restrict__ A, const LabelBox* boxes, int nb, long long nlines, Geometry g,
                        int* __restrict__ B) {
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    const LabelBox b = boxes[box_of<1>(boxes, nb, l)];
    const long long t = l - b.line[1];
    const int z = (int)(t / b.n[2]), x = (int)(t % b.n[2]);
    const long long base = b.off + (long long)z * b.n[1] * b.n[2] + x;
    const int ny = b.n[1], r = g.r[1], st = b.n[2];
    int sum = 0;
    for (int y = 0; y <= r && y < ny; ++y) sum += A[base + (long long)y * st];
    for (int y = 0; y < ny; ++y) {
      B[base + (long long)y * st] = sum;
      if (y + r + 1 < ny) sum += A[base + (long long)(y + r + 1) * st];
      if (y - r >= 0) sum -= A[base + (long long)(y - r) * st];
    }
  }
}

// Quantized fraction: i + 1 for the first threshold (in list order) above count / fov, else nth + 1.
__device__ __forceinline__ unsigned char quantize(int count, double fov, const double* th, int nth) {
  const double f = __ddiv_rn((double)count, fov);
  for (int i = 0; i < nth; ++i)
    if (f < th[i]) return (unsigned char)(i + 1);
  return (unsigned char)(nth + 1);
}

// The z-window sum of B at every voxel of the box's label inside the VALID region, quantized into `out` (VALID
// coordinates), one thread per (y, x) line.
__global__ void count_z(const int* __restrict__ B, const int* __restrict__ compact, const LabelBox* boxes, int nb,
                        long long nlines, Geometry g, double fov, const double* th, int nth,
                        unsigned char* __restrict__ out) {
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    const LabelBox b = boxes[box_of<2>(boxes, nb, l)];
    const long long t = l - b.line[2];
    const int y = (int)(t / b.n[2]), x = (int)(t % b.n[2]);
    const int vy = b.lo[1] + y, vx = b.lo[2] + x;
    const long long st = (long long)b.n[1] * b.n[2];
    const long long base = b.off + (long long)y * b.n[2] + x;
    const int nz = b.n[0], r = g.r[0], k = b.k;
    const bool line_valid = vy >= g.r[1] && vy < g.s[1] - g.r[1] && vx >= g.r[2] && vx < g.s[2] - g.r[2];
    int sum = 0;
    for (int z = 0; z <= r && z < nz; ++z) sum += B[base + z * st];
    for (int z = 0; z < nz; ++z) {
      const int vz = b.lo[0] + z;
      if (line_valid && vz >= r && vz < g.s[0] - r &&
          compact[((size_t)vz * g.s[1] + vy) * g.s[2] + vx] == k)
        out[((size_t)(vz - r) * g.o[1] + (vy - g.r[1])) * g.o[2] + (vx - g.r[2])] = quantize(sum, fov, th, nth);
      if (z + r + 1 < nz) sum += B[base + (z + r + 1) * st];
      if (z - r >= 0) sum -= B[base + (z - r) * st];
    }
  }
}

// out = any(in over [i, i + 2r]) along `axis` (VALID: out extent = in extent - 2r on that axis), one thread per line.
__global__ void box_any(const unsigned char* __restrict__ in, unsigned char* __restrict__ out, int axis, int r,
                        int d0, int d1, int d2) {
  const int din[3] = {d0, d1, d2};
  int dout[3] = {d0, d1, d2};
  dout[axis] -= 2 * r;
  const long long sin[3] = {(long long)d1 * d2, d2, 1};
  const long long sout[3] = {(long long)dout[1] * dout[2], dout[2], 1};
  const int a1 = axis == 0 ? 1 : 0, a2 = axis == 2 ? 1 : 2;   // the other two axes, a2 the faster one
  const long long nlines = (long long)dout[a1] * dout[a2];
  const int len = dout[axis];
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    const long long c1 = l / dout[a2], c2 = l % dout[a2];
    const unsigned char* src = in + c1 * sin[a1] + c2 * sin[a2];
    unsigned char* dst = out + c1 * sout[a1] + c2 * sout[a2];
    const long long si = sin[axis], so = sout[axis];
    int cnt = 0;
    for (int t = 0; t < 2 * r && t < din[axis]; ++t) cnt += src[t * si] != 0;
    for (int i = 0; i < len; ++i) {
      cnt += src[(i + 2 * r) * si] != 0;
      dst[i * so] = cnt > 0;
      cnt -= src[i * si] != 0;
    }
  }
}

__device__ __forceinline__ bool in_sphere(const Sphere& s, long long hx, long long hy, long long hz) {
  if (s.integer) {
    const u64 dx = (u64)hx - (u64)s.c[0], dy = (u64)hy - (u64)s.c[1], dz = (u64)hz - (u64)s.c[2];
    return (long long)(dx * dx + dy * dy + dz * dz) <= s.r2;
  }
  const double dx = __dsub_rn((double)hx, s.fc[0]), dy = __dsub_rn((double)hy, s.fc[1]);
  const double dz = __dsub_rn((double)hz, s.fc[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) <= s.fr2;
}

// 255 where the LOM box holds a masked voxel (masked != null) or the voxel lies in an exclusion sphere; the histogram
// of the final values.
__global__ void finish(unsigned char* out, size_t nout, const unsigned char* masked, const Sphere* spheres,
                       int nspheres, Geometry g, unsigned long long* hist) {
  __shared__ unsigned int h[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nout; i += (size_t)gridDim.x * blockDim.x) {
    unsigned char v = out[i];
    bool excl = masked && masked[i];
    if (!excl && nspheres) {
      const long long hx = (long long)(i % g.o[2]) + g.r[2];
      const long long hy = (long long)((i / g.o[2]) % g.o[1]) + g.r[1];
      const long long hz = (long long)(i / ((size_t)g.o[2] * g.o[1])) + g.r[0];
      for (int s = 0; s < nspheres && !excl; ++s) excl = in_sphere(spheres[s], hx, hy, hz);
    }
    if (excl) {
      v = 255;
      out[i] = v;
    }
    atomicAdd(&h[v], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (h[i]) atomicAdd(&hist[i], (unsigned long long)h[i]);
}

}  // namespace ptk
}  // namespace ffn
