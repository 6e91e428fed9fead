// reseg_kernels.cuh — scoring of resegmentation results (ffn/inference/resegmentation_analysis.py:97-260) on the device.
// A batch holds items of one kind whose boxes share one extent, back to back.  HBM-bound passes:
//   pair_prepare      labels + 2 probability boxes -> 4 masks as distance keys, per-item counts   10 B read + 32 B written / voxel
//   nid_x, nid_line   (decision_kernels.cuh, one id: key = squared distance) x, y, z over the 4 masks 16 / 32 / 32 B per mask voxel
//   edt_max           largest key per mask                                                         8 B / mask voxel
//   endpoint_prepare  labels + 1 probability box -> sort values (item, mask), per-item counts       9 B read + 4 B written / voxel
//   2 radix sorts     (label, then item; stable) + run heads + scan + rows: the overlap counts of ComputeOverlapCounts
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ffn {
namespace rsk {

typedef unsigned long long u64;

constexpr u64 kInf = ~0ull;    // a voxel of the mask before the transform, or one no voxel outside the mask reaches
constexpr int kPairCounts = 10; // |seg0| |seg1| |r0| |r1| |r0 s0| |r0 s1| |r1 s0| |r1 s1| |r0 r1| |r0 or r1|

__device__ __forceinline__ u64 warp_sum(u64 v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ u64 warp_max(u64 v) {
  for (int o = 16; o > 0; o >>= 1) {
    const u64 w = __shfl_down_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// Per item (blockIdx.y, strided): seg0 = label == id_a, seg1 = label == id_b, reseg_k = table[probs_k].  Writes the four
// masks as distance-transform keys (0 outside the mask, kInf inside), mask-major per item, and adds the item's counts.
__global__ void pair_prepare(const u64* labels, const unsigned char* probs, const u64* ids, const unsigned char* table,
                             long long nitems, long long nbox, u64* keys, u64* counts) {
  __shared__ unsigned char tab[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = table[i];
  __syncthreads();
  for (long long it = blockIdx.y; it < nitems; it += gridDim.y) {
    const u64 ida = ids[2 * it], idb = ids[2 * it + 1];
    const u64* lab = labels + it * nbox;
    const unsigned char* p0 = probs + 2 * it * nbox;
    const unsigned char* p1 = p0 + nbox;
    u64* k0 = keys + 4 * it * nbox;
    u64 c[kPairCounts] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nbox; v += (long long)gridDim.x * blockDim.x) {
      const u64 l = lab[v];
      const bool s0 = l == ida, s1 = l == idb, r0 = tab[p0[v]] != 0, r1 = tab[p1[v]] != 0;
      k0[v] = s0 ? kInf : 0;
      k0[nbox + v] = s1 ? kInf : 0;
      k0[2 * nbox + v] = r0 ? kInf : 0;
      k0[3 * nbox + v] = r1 ? kInf : 0;
      c[0] += s0; c[1] += s1; c[2] += r0; c[3] += r1;
      c[4] += r0 && s0; c[5] += r0 && s1; c[6] += r1 && s0; c[7] += r1 && s1;
      c[8] += r0 && r1; c[9] += r0 || r1;
    }
#pragma unroll
    for (int j = 0; j < kPairCounts; ++j) {
      const u64 s = warp_sum(c[j]);
      if ((threadIdx.x & 31) == 0 && s) atomicAdd(&counts[it * kPairCounts + j], s);
    }
  }
}

// Largest key of each box (blockIdx.y, strided) of `nbox` keys.
__global__ void edt_max(const u64* keys, long long nboxes, long long nbox, u64* out) {
  for (long long b = blockIdx.y; b < nboxes; b += gridDim.y) {
    const u64* k = keys + b * nbox;
    u64 m = 0;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nbox; v += (long long)gridDim.x * blockDim.x)
      m = k[v] > m ? k[v] : m;
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&out[b], m);
  }
}

// Endpoint items: vals = item << 1 | mask (the second sort's key and the mask bit it carries), and per item |seg0|
// (label == id_a) and |mask|.
__global__ void endpoint_prepare(const u64* labels, const unsigned char* probs, const u64* ids, const unsigned char* table,
                                 long long nitems, long long nbox, unsigned* vals, u64* counts) {
  __shared__ unsigned char tab[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = table[i];
  __syncthreads();
  for (long long it = blockIdx.y; it < nitems; it += gridDim.y) {
    const u64 ida = ids[2 * it];
    const u64* lab = labels + it * nbox;
    const unsigned char* p = probs + it * nbox;
    unsigned* o = vals + it * nbox;
    u64 cs = 0, cr = 0;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nbox; v += (long long)gridDim.x * blockDim.x) {
      const unsigned r = tab[p[v]] != 0;
      o[v] = (unsigned)it << 1 | r;
      cs += lab[v] == ida;
      cr += r;
    }
    cs = warp_sum(cs);
    cr = warp_sum(cr);
    if ((threadIdx.x & 31) == 0 && cs) atomicAdd(&counts[2 * it], cs);
    if ((threadIdx.x & 31) == 0 && cr) atomicAdd(&counts[2 * it + 1], cr);
  }
}

// After sorting by (item, label): flags the first voxel of every (item, label) run and extracts the mask bits.
__global__ void run_heads(const unsigned* vals, const u64* labels, int n, unsigned char* head, unsigned* bits) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned v = vals[i];
    head[i] = i == 0 || (v >> 1) != (vals[i - 1] >> 1) || labels[i] != labels[i - 1];
    bits[i] = v & 1u;
  }
}

// One row per run: its item, label, mask voxels (from the inclusive scan of the mask bits) and voxels.
__global__ void run_rows(const int* heads, int nruns, int n, const unsigned* vals, const u64* labels,
                         const unsigned* scan, FfnResegOverlap* rows) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nruns; r += gridDim.x * blockDim.x) {
    const int s = heads[r], e = r + 1 < nruns ? heads[r + 1] : n;
    FfnResegOverlap row;
    row.item = (int64_t)(vals[s] >> 1);
    row.id = labels[s];
    row.num_overlapping = (int64_t)scan[e - 1] - (s > 0 ? (int64_t)scan[s - 1] : 0);
    row.num_original = e - s;
    rows[r] = row;
  }
}

struct Overlapping {
  __host__ __device__ bool operator()(const FfnResegOverlap& r) const { return r.num_overlapping > 0; }
};

}  // namespace rsk
}  // namespace ffn
