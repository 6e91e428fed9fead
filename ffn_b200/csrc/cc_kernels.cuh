// cc_kernels.cuh — connected components of a label volume (ffn/inference/segmentation.py:89-178) on the device.
// Union-find over int32 parents in which every root is the smallest linear index of its set, so components are
// numbered in C order of their first voxel whatever the thread schedule.  Background voxels get parent -1.  Passes
// (n < 2^31 voxels, so parents, ranks and counts are int32; loop indices are 64-bit, as i + stride can pass 2^31;
// bytes are HBM traffic per voxel, neighbour reads hit L1 / L2):
//   init             parent = start of the voxel's x-run within its warp, or the voxel before the warp    8 B read, 4 B written
//   merge<C>         union with every same-id backward neighbour but x - 1 (atomicMin linking)      8 B + 4 B and the tree walks
//   flatten_count    parent = root; voxels per root with one atomicAdd per distinct root per warp   4 B read, 4 B written
//   scan of the root flags (CUB) -> rank of every root                                               4 B read, 4 B written
//   write_labels     rank + 1 of the voxel's root, or 0 (background, dust); first and number of 0s  4 B read, 8 B written
//   select / gather  table of the kept roots (only when a table is wanted)                           4 B read
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_reduce.cuh>

namespace ffn {
namespace cck {

typedef unsigned long long u64;

constexpr int kBlock = 256;

struct Shape {
  int sz, sy, sx;
};

// Root of i.  Parents change under other threads' unions, so every read goes to memory.
__device__ __forceinline__ int find_root(const int* parent, int i) {
  const volatile int* p = parent;
  int q = p[i];
  while (q != i) {
    i = q;
    q = p[i];
  }
  return i;
}

// Lock-free union (Playne & Hawick 2018): the larger root is linked under the smaller one.  When another thread
// relinked that root first, atomicMin still only lowers its parent, and the loop goes on from the new parent.
__device__ __forceinline__ void unite(int* parent, int a, int b) {
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(parent + b, a);
    if (old == b) return;
    b = old;
  }
}

// parent[i]: -1 for background; otherwise the last run start at or before i within i's warp (a run is a maximal
// x-run of one id), or i - 1 when the run began before the warp.  Trees along x are at most sx / 32 + 1 deep, and
// merge needs no x - 1 union.  Every lane of a warp runs the same iterations, for the ballot.
__global__ void init(const u64* labels, int n, int sx, int* parent, int* first_zero) {
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) *first_zero = 0x7fffffff;
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x - lane; base < n;
       base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + lane;
    const bool valid = i < n;
    u64 v = 0;
    bool cont = false;
    if (valid) {
      v = labels[i];
      cont = v != 0 && i % sx != 0 && labels[i - 1] == v;
    }
    const unsigned starts = __ballot_sync(0xffffffffu, !cont);
    if (!valid) continue;
    int p = (int)i;
    if (v == 0) {
      p = -1;
    } else if (cont) {
      const unsigned m = starts & (0xffffffffu >> (31 - lane));
      p = (int)(m ? base + 31 - __clz(m) : base - 1);
    }
    parent[i] = p;
  }
}

// One thread per voxel: union with each backward neighbour (smaller linear index) of the same non-zero id under
// C = 1, 2, 3 (6-, 18-, 26-connectivity), except x - 1, which init linked.  A union that the voxel before it in the
// row also does, one step to the left, is skipped: both voxels and both neighbours are then in two joined x-runs.
template <int C>
__global__ void merge(const u64* labels, Shape s, int* parent) {
  const int n = s.sz * s.sy * s.sx;
  const int plane = s.sy * s.sx;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)t;
    const u64 v = labels[i];
    if (v == 0) continue;
    const int z = i / plane;
    const int r = i - z * plane;
    const int y = r / s.sx;
    const int x = r - y * s.sx;
    const bool left = x > 0 && labels[i - 1] == v;
#pragma unroll
    for (int dz = -1; dz <= 0; ++dz) {
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy) {
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          if (dz == 0 && (dy > 0 || (dy == 0 && dx >= 0))) continue;   // forward, or the voxel itself
          if (dz == 0 && dy == 0) continue;                             // x - 1: linked by init
          if ((dz != 0) + (dy != 0) + (dx != 0) > C) continue;
          if (z + dz < 0 || y + dy < 0 || y + dy >= s.sy || x + dx < 0 || x + dx >= s.sx) continue;
          const int j = i + dz * plane + dy * s.sx + dx;
          if (labels[j] != v) continue;
          if (left && x + dx > 0 && labels[j - 1] == v) continue;
          unite(parent, i, j);
        }
      }
    }
  }
}

// parent = root for every foreground voxel, and count[root] += 1 with one atomic per distinct root of a warp, so a
// component that fills the volume costs n / 32 atomics, not n.
__global__ void flatten_count(int* parent, int n, int* count) {
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x - lane; base < n;
       base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + lane;
    int r = -1;
    if (i < n && parent[i] >= 0) {
      r = find_root(parent, (int)i);
      parent[i] = r;
    }
    const unsigned group = __match_any_sync(0xffffffffu, r);
    if (r >= 0 && lane == __ffs(group) - 1) atomicAdd(count + r, __popc(group));
  }
}

// 1 for the root of a component, in the scan that numbers them.
struct IsRoot {
  const int* parent;
  __host__ __device__ int operator()(int i) const { return parent[i] == i; }
};

// A component that stays: its root, with at least min_size voxels (any size when min_size <= 0).
struct KeptRoot {
  const int* parent;
  const int* count;
  long long min_size;
  __host__ __device__ bool operator()(int i) const {
    return parent[i] == i && (min_size <= 0 || (long long)count[i] >= min_size);
  }
};

// out[i] = rank of the root + 1, or 0 for background and dust; first_zero / n_zero: the smallest index and the
// number of output zeros.
__global__ void __launch_bounds__(kBlock) write_labels(const int* parent, const int* rank, const int* count, int n,
                                                       long long min_size, u64* out, int* first_zero, int* n_zero) {
  int first = 0x7fffffff, zeros = 0;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)t;
    const int r = parent[i];
    u64 v = 0;
    if (r >= 0 && (min_size <= 0 || (long long)count[r] >= min_size)) v = (u64)rank[r] + 1;
    if (v == 0) {
      first = min(first, i);
      ++zeros;
    }
    out[i] = v;
  }
  typedef cub::BlockReduce<int, kBlock> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  first = Reduce(tmp).Reduce(first, cub::Min());
  __syncthreads();
  zeros = Reduce(tmp).Sum(zeros);
  if (threadIdx.x == 0) {
    if (first != 0x7fffffff) atomicMin(first_zero, first);
    if (zeros) atomicAdd(n_zero, zeros);
  }
}

// Table row k of the kept roots (ascending, so in id order): id, original id, voxel count.
__global__ void gather_rows(const int* roots, int nkept, const int* rank, const int* count, const u64* labels,
                            u64* ids, u64* orig, long long* counts) {
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nkept;
       k += (long long)gridDim.x * blockDim.x) {
    const int r = roots[k];
    ids[k] = (u64)rank[r] + 1;
    orig[k] = labels[r];
    counts[k] = count[r];
  }
}

}  // namespace cck
}  // namespace ffn
