// clean_up.cu — connected-component clean-up of a segmentation on the device (ffn_clean_up).

#include <cub/cub.cuh>

#include "../../include/ffn_b200.h"
#include "cc_kernels.cuh"
#include "host.cuh"

using namespace ffn;

extern "C" {

int ffn_clean_up(int device, const FfnCleanUpDesc* desc, uint64_t* labels, uint64_t* ids, uint64_t* orig_ids,
                 int64_t* counts, int64_t cap, int64_t* n_ids) {
  using cck::u64;
  const bool table = ids || orig_ids || counts;
  if (!desc || !n_ids || cap < 0 || (cap > 0 && !table)) return fail("bad argument");
  const int sz = desc->shape_zyx[0], sy = desc->shape_zyx[1], sx = desc->shape_zyx[2];
  if (sz < 0 || sy < 0 || sx < 0) return fail("shape must not be negative");
  if (desc->connectivity < 1 || desc->connectivity > 3) return fail("connectivity must be 1, 2 or 3");
  // Every extent is below 2^31, and sz * sy is checked before it is multiplied by sx, so no product wraps.
  size_t n = 0;
  if (sz && sy && sx) {
    if ((size_t)sz * sy >= (1ull << 31) || (size_t)sz * sy * sx >= (1ull << 31))
      return fail("connected components support volumes of fewer than 2^31 voxels");
    n = (size_t)sz * sy * sx;
  }
  *n_ids = 0;
  if (n == 0) return 0;
  if (!labels) return fail("bad argument");
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int blocks = prop.multiProcessorCount * 16;
  const int ni = (int)n;
  const long long min_size = desc->min_size;
  DevBufs bufs;

  u64 *d_lab = nullptr, *d_out = nullptr;
  int *d_par = nullptr, *d_cnt = nullptr, *d_rank = nullptr, *d_roots = nullptr, *d_misc = nullptr;
  // d_misc: [0] first output zero, [1] output zeros, [2] kept components
  if (bufs.get(&d_lab, n) || bufs.get(&d_out, n) || bufs.get(&d_par, n) || bufs.get(&d_cnt, n, true) ||
      bufs.get(&d_rank, n) || bufs.get(&d_misc, 3, true) || (table && bufs.get(&d_roots, n)))
    return 1;
  cub::CountingInputIterator<int> index(0);
  cub::TransformInputIterator<int, cck::IsRoot, cub::CountingInputIterator<int>> is_root(index, cck::IsRoot{d_par});
  auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, is_root, d_rank, ni, st); };
  auto select = [&](void* t, size_t& b) {
    return cub::DeviceSelect::If(t, b, index, d_roots, d_misc + 2, ni, cck::KeptRoot{d_par, d_cnt, min_size}, st);
  };
  CubTemp temp;
  if (table ? temp.alloc(bufs, scan, select) : temp.alloc(bufs, scan)) return 1;
  CUDA_OK(cudaMemcpyAsync(d_lab, labels, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  const cck::Shape shape{sz, sy, sx};
  cck::init<<<blocks, cck::kBlock, 0, st>>>(d_lab, ni, sx, d_par, d_misc);
  switch (desc->connectivity) {
    case 1: cck::merge<1><<<blocks, cck::kBlock, 0, st>>>(d_lab, shape, d_par); break;
    case 2: cck::merge<2><<<blocks, cck::kBlock, 0, st>>>(d_lab, shape, d_par); break;
    default: cck::merge<3><<<blocks, cck::kBlock, 0, st>>>(d_lab, shape, d_par); break;
  }
  cck::flatten_count<<<blocks, cck::kBlock, 0, st>>>(d_par, ni, d_cnt);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(temp.run(scan));
  cck::write_labels<<<blocks, cck::kBlock, 0, st>>>(d_par, d_rank, d_cnt, ni, min_size, d_out, d_misc, d_misc + 1);
  CUDA_OK(cudaGetLastError());
  if (table) CUDA_OK(temp.run(select));
  int misc[3] = {0, 0, 0};
  CUDA_OK(cudaMemcpyAsync(misc, d_misc, sizeof(misc), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  const int first_zero = misc[1] > 0 ? misc[0] : -1;

  // The table: the 0 row first when the output has a 0, then the kept components in id order.  A table larger than
  // cap leaves everything unwritten, so the caller can repeat the call on the same input with cap = *n_ids.
  if (table) {
    const int nkept = misc[2];
    const int z = first_zero >= 0;
    *n_ids = (int64_t)nkept + z;
    if (*n_ids > cap) return 0;
    u64 *d_ids = nullptr, *d_orig = nullptr;
    long long* d_counts = nullptr;
    if (bufs.get(&d_ids, nkept) || bufs.get(&d_orig, nkept) || bufs.get(&d_counts, nkept)) return 1;
    cck::gather_rows<<<blocks, cck::kBlock, 0, st>>>(d_roots, nkept, d_rank, d_cnt, d_lab, d_ids, d_orig, d_counts);
    CUDA_OK(cudaGetLastError());
    if (ids && nkept) CUDA_OK(cudaMemcpyAsync(ids + z, d_ids, nkept * sizeof(u64), cudaMemcpyDeviceToHost, st));
    if (orig_ids && nkept) CUDA_OK(cudaMemcpyAsync(orig_ids + z, d_orig, nkept * sizeof(u64), cudaMemcpyDeviceToHost, st));
    if (counts && nkept) CUDA_OK(cudaMemcpyAsync(counts + z, d_counts, nkept * sizeof(long long), cudaMemcpyDeviceToHost, st));
    if (z) {
      if (ids) ids[0] = 0;
      if (orig_ids) orig_ids[0] = labels[first_zero];   // labels still holds the input
      if (counts) counts[0] = misc[1];
    }
  }
  CUDA_OK(cudaMemcpyAsync(labels, d_out, n * sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
