// consensus.cu — split consensus of two segmentations on the device (ffn_split_intersection).

#include <string>

#include <cub/cub.cuh>

#include "../../include/ffn_b200.h"
#include "consensus_kernels.cuh"
#include "host.cuh"

using namespace ffn;

extern "C" {

namespace {
struct MaxU64 {
  __device__ __forceinline__ unsigned long long operator()(unsigned long long x, unsigned long long y) const {
    return x > y ? x : y;
  }
};
}  // namespace

int ffn_split_intersection(int device, int64_t n, uint64_t* a, const uint64_t* b, int64_t min_size) {
  using csk::u64;
  if (n < 0 || (n > 0 && (!a || !b))) return fail("bad argument");
  if (n >= (1ll << 31)) return fail("split consensus supports volumes of fewer than 2^31 voxels");
  if (n == 0) return 0;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int blocks = prop.multiProcessorCount * 16;
  const int ni = (int)n;
  int np = ni;   // an upper bound until the (a, b) pairs are counted
  DevBufs bufs;

  u64 *d_a = nullptr, *d_b = nullptr, *d_tmp = nullptr, *d_max = nullptr;
  int* d_num = nullptr;
  if (bufs.get(&d_a, n) || bufs.get(&d_b, n) || bufs.get(&d_tmp, n) || bufs.get(&d_max, 2) || bufs.get(&d_num, 2))
    return 1;
  u64 *d_pairs = nullptr, *d_sw = nullptr, *d_sw2 = nullptr, *d_pack = nullptr, *d_best = nullptr, *d_lab = nullptr;
  int *d_counts = nullptr, *d_idx = nullptr, *d_idx2 = nullptr, *d_flags = nullptr, *d_rank = nullptr;
  unsigned *d_aof = nullptr, *d_ured = nullptr;
  unsigned char* d_partner = nullptr;
  // The CUB calls (max_of, sort_keys and unique run on several arrays), sized for n items: no later call has more.
  auto max_of = [&](u64* in, u64* out) {
    return [=](void* t, size_t& b) { return cub::DeviceReduce::Max(t, b, in, out, ni, st); };
  };
  auto sort_keys = [&](u64* in, u64* out) {
    return [=](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, in, out, ni, 0, 64, st); };
  };
  auto unique = [&](u64* out) {
    return [=](void* t, size_t& b) { return cub::DeviceSelect::Unique(t, b, d_tmp, out, d_num, ni, st); };
  };
  auto rle = [&](void* t, size_t& b) {
    return cub::DeviceRunLengthEncode::Encode(t, b, d_b, d_pairs, d_counts, d_num, ni, st);
  };
  auto sort_pairs = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, d_sw, d_sw2, d_idx, d_idx2, np, 0, 64, st);
  };
  auto reduce_best = [&](void* t, size_t& b) {
    return cub::DeviceReduce::ReduceByKey(t, b, d_aof, d_ured, d_pack, d_best, d_num + 1, MaxU64(), np, st);
  };
  auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_flags, d_rank, np, st); };
  CubTemp temp;
  if (temp.alloc(bufs, max_of(d_a, d_max), sort_keys(d_a, d_tmp), unique(d_a), rle, sort_pairs, reduce_best, scan))
    return 1;
  CUDA_OK(cudaMemcpyAsync(d_a, a, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_b, b, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(temp.run(max_of(d_a, d_max)));
  CUDA_OK(temp.run(max_of(d_b, d_max + 1)));
  u64 maxes[2] = {0, 0};
  CUDA_OK(cudaMemcpyAsync(maxes, d_max, sizeof(maxes), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  const u64 max_id = maxes[0];

  // remap_input: sorted unique ids of an array whose ids do not fit in 32 bits, and the +1 shift when 0 is absent.
  u64* uniq[2] = {nullptr, nullptr};
  int nuniq[2] = {0, 0};
  unsigned shift[2] = {0, 0};
  for (int k = 0; k < 2; ++k) {
    if (maxes[k] <= 0xffffffffull) continue;
    CUDA_OK(temp.run(sort_keys(k ? d_b : d_a, d_tmp)));
    if (bufs.get(&uniq[k], n)) return 1;
    CUDA_OK(temp.run(unique(uniq[k])));
    u64 first = 0;
    CUDA_OK(cudaMemcpyAsync(&nuniq[k], d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(&first, uniq[k], sizeof(u64), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    shift[k] = first != 0;
  }

  // Joint keys (kept in d_tmp for the relabel), sorted into d_b, then the unique pairs and their counts.
  csk::joint_keys<<<blocks, 256, 0, st>>>(d_a, d_b, (size_t)n, uniq[0], nuniq[0], shift[0], uniq[1], nuniq[1],
                                          shift[1], d_tmp);
  CUDA_OK(cudaGetLastError());
  if (uniq[1]) bufs.release(uniq[1]);
  CUDA_OK(temp.run(sort_keys(d_tmp, d_b)));
  if (bufs.get(&d_pairs, n) || bufs.get(&d_counts, n)) return 1;
  CUDA_OK(temp.run(rle));
  CUDA_OK(cudaMemcpyAsync(&np, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_b);

  // Largest overlap per a: the pairs regrouped by a (a-major sort), then a maximum of count << 32 | ~b per a.
  if (bufs.get(&d_sw, np) || bufs.get(&d_sw2, np) || bufs.get(&d_pack, np) || bufs.get(&d_best, np) ||
      bufs.get(&d_lab, np) || bufs.get(&d_idx, np) || bufs.get(&d_idx2, np) || bufs.get(&d_flags, np) ||
      bufs.get(&d_rank, np) || bufs.get(&d_aof, np) || bufs.get(&d_ured, np) || bufs.get(&d_partner, np))
    return 1;
  csk::regroup<<<blocks, 256, 0, st>>>(d_pairs, np, d_sw, d_idx);
  CUDA_OK(temp.run(sort_pairs));
  csk::partner_pack<<<blocks, 256, 0, st>>>(d_sw2, d_idx2, d_counts, np, d_aof, d_pack);
  CUDA_OK(temp.run(reduce_best));
  int nu = 0;
  CUDA_OK(cudaMemcpyAsync(&nu, d_num + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  csk::mark_partner<<<blocks, 256, 0, st>>>(d_aof, d_pack, d_idx2, d_ured, d_best, nu, np, d_partner);

  // New ids in key order, then the output id of every pair.
  csk::pair_flags<<<blocks, 256, 0, st>>>(d_pairs, d_counts, d_partner, np, (long long)min_size, d_flags);
  CUDA_OK(temp.run(scan));
  int last[2] = {0, 0};
  CUDA_OK(cudaMemcpyAsync(&last[0], d_flags + np - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(&last[1], d_rank + np - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  const u64 n_new = (u64)last[0] + (u64)last[1];
  if (n_new > ~0ull - max_id)
    return fail("split consensus: max id " + std::to_string(max_id) + " + " + std::to_string(n_new) +
                " new ids does not fit in 64 bits");
  csk::pair_labels<<<blocks, 256, 0, st>>>(d_pairs, d_counts, d_partner, d_rank, np, (long long)min_size, uniq[0],
                                           shift[0], max_id, d_lab);
  csk::relabel<<<blocks, 256, 0, st>>>(d_tmp, (size_t)n, d_pairs, np, d_lab, d_a);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(a, d_a, n * sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
