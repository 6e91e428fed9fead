// consensus_kernels.cuh — split consensus of two segmentations (ffn/inference/segmentation.py:181-290) on the device.
// Every voxel gets the joint key a32 | b32 << 32 of its two 32-bit ids; the sorted unique keys are the overlapping
// (a, b) pairs in the reference's b-major, a-minor order, and every pair gets one output id.  HBM-bound passes:
//   compaction (only an array whose max id is above 2^32 - 1): radix sort + unique, then a rank by binary search
//   joint_keys       a, b -> key                                                   24 B/voxel (+ sorted ids in L2)
//   radix sort + run-length encode of the keys -> pairs and their counts
//   regroup / partner_pack / mark_partner / pair_flags / pair_labels              per pair, not per voxel
//   relabel          key -> output id by binary search among the pairs             16 B/voxel (+ pairs in L2)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ffn {
namespace csk {

typedef unsigned long long u64;

// First index of `v` in the sorted unique ids (remap_input's rank); v is always present.
__device__ __forceinline__ u64 rank_of(const u64* ids, int nids, u64 v) {
  int lo = 0, hi = nids;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < v) lo = mid + 1; else hi = mid;
  }
  return (u64)lo;
}

// key = a32 | b32 << 32.  An array with sorted unique ids (ua / ub non-null) is remapped to rank + shift, shift = 1
// when 0 is not among its ids; otherwise its ids already fit in 32 bits.
__global__ void joint_keys(const u64* a, const u64* b, size_t n, const u64* ua, int nua, unsigned sa, const u64* ub,
                           int nub, unsigned sb, u64* keys) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const u64 x = ua ? rank_of(ua, nua, a[i]) + sa : a[i];
    const u64 y = ub ? rank_of(ub, nub, b[i]) + sb : b[i];
    keys[i] = x | y << 32;
  }
}

// The pairs regrouped by a: key a << 32 | b, value the pair's index in b-major order.
__global__ void regroup(const u64* pairs, int np, u64* swapped, int* idx) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < np; j += gridDim.x * blockDim.x) {
    const u64 p = pairs[j];
    swapped[j] = p << 32 | p >> 32;
    idx[j] = j;
  }
}

// In a-major order: the a of each pair and count << 32 | ~b, whose maximum over one a is the largest overlap, the
// smallest b on equal counts (the first strictly larger count in b order wins in the reference).
__global__ void partner_pack(const u64* swapped, const int* idx, const int* counts, int np, unsigned* a_of, u64* pack) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
    const u64 s = swapped[k];
    a_of[k] = (unsigned)(s >> 32);
    pack[k] = (u64)(unsigned)counts[idx[k]] << 32 | (u64)(~(unsigned)s);
  }
}

// partner[j] = 1 for the pair j (b-major index) that is its a's largest overlap.  best[r] is the maximum pack of
// the r-th a in ascending order (ua_red), found by binary search.
__global__ void mark_partner(const unsigned* a_of, const u64* pack, const int* idx, const unsigned* ua_red,
                             const u64* best, int nu, int np, unsigned char* partner) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
    const unsigned a = a_of[k];
    int lo = 0, hi = nu;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ua_red[mid] < a) lo = mid + 1; else hi = mid;
    }
    partner[idx[k]] = pack[k] == best[lo];
  }
}

// 1 for a pair that takes a new id: large enough, a != 0 and not its a's largest overlap.
__global__ void pair_flags(const u64* pairs, const int* counts, const unsigned char* partner, int np,
                           long long min_size, int* flags) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < np; j += gridDim.x * blockDim.x)
    flags[j] = !((long long)counts[j] < min_size || (unsigned)pairs[j] == 0) && !partner[j];
}

// Output id per pair: 0 when too small or a == 0; a's original id for its largest overlap; otherwise
// max_id + 1 + (new ids before it in key order).
__global__ void pair_labels(const u64* pairs, const int* counts, const unsigned char* partner, const int* rank,
                            int np, long long min_size, const u64* ua, unsigned sa, u64 max_id, u64* labels) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < np; j += gridDim.x * blockDim.x) {
    const u64 a = (unsigned)pairs[j];
    u64 out;
    if ((long long)counts[j] < min_size || a == 0) out = 0;
    else if (partner[j]) out = ua ? ua[a - sa] : a;
    else out = max_id + 1 + (u64)rank[j];
    labels[j] = out;
  }
}

// Every voxel takes the output id of its pair.
__global__ void relabel(const u64* keys, size_t n, const u64* pairs, int np, const u64* labels, u64* out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = labels[rank_of(pairs, np, keys[i])];
}

}  // namespace csk
}  // namespace ffn
