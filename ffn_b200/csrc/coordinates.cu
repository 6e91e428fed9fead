// coordinates.cu — training coordinates from partition maps on the device: the rows of a partition map
// (ffn_partition_rows) and their serialised records (ffn_coordinate_records).

#include <algorithm>
#include <vector>

#include <cub/cub.cuh>

#include "../../include/ffn_b200.h"
#include "coordinate_kernels.cuh"
#include "host.cuh"

using namespace ffn;

extern "C" {

int ffn_partition_rows(int device, const FfnPartitionRowsDesc* desc, const uint8_t* volume, int64_t* rows,
                       int64_t counts[256]) {
  if (!desc || !volume || !rows || !counts) return fail("bad argument");
  cok::Crop c{};
  size_t nvol = 1;
  long long ncrop = 1;
  for (int a = 0; a < 3; ++a) {
    const int s = desc->shape_zyx[a], lo = desc->crop_start_zyx[a], n = desc->crop_shape_zyx[a];
    if (s < 0 || lo < 0 || n < 0 || (int64_t)lo + n > s) return fail("the crop must lie inside the volume");
    c.n[a] = n;
    c.lo[a] = lo;
    nvol *= (size_t)s;
    ncrop *= n;
  }
  if (ncrop >= (1ll << 31)) return fail("partition crops must have fewer than 2^31 voxels");
  c.sy = desc->shape_zyx[2];
  c.sz = (long long)desc->shape_zyx[1] * desc->shape_zyx[2];
  c.size = ncrop;
  std::fill(counts, counts + 256, (int64_t)0);
  if (ncrop == 0) return 0;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int ntiles = (int)((ncrop + cok::kTile - 1) / cok::kTile);
  const size_t nhist = (size_t)256 * ntiles;
  DevBufs bufs;
  unsigned char* d_vol = nullptr;
  int *d_hist = nullptr, *d_base = nullptr;
  unsigned long long* d_counts = nullptr;
  longlong2* d_rows = nullptr;
  auto scan = [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_hist, d_base, (int64_t)nhist, st);
  };
  CubTemp temp;
  if (bufs.get(&d_vol, nvol) || bufs.get(&d_hist, nhist) || bufs.get(&d_base, nhist) || bufs.get(&d_counts, 256) ||
      temp.alloc(bufs, scan))
    return 1;
  CUDA_OK(cudaMemcpyAsync(d_vol, volume, nvol, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(d_counts, 0, 256 * sizeof(unsigned long long), st));
  cok::bucket_hist<<<ntiles, cok::kThreads, 0, st>>>(d_vol, c, ntiles, d_hist, d_counts);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(temp.run(scan));
  CUDA_OK(cudaMemcpyAsync(counts, d_counts, 256 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_hist);
  bufs.release(temp.p);
  const long long kept = ncrop - counts[cok::kIgnore];
  if (bufs.get(&d_rows, kept)) return 1;
  cok::bucket_scatter<<<ntiles, cok::kThreads, 0, st>>>(d_vol, c, ntiles, d_base, desc->volume_index, d_rows);
  CUDA_OK(cudaGetLastError());
  if (kept > 0)
    CUDA_OK(cudaMemcpyAsync(rows, d_rows, kept * sizeof(longlong2), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaGetLastError());
  return 0;
}

int ffn_coordinate_records(int device, const FfnCoordinateDesc* desc, const int64_t* rows, int64_t n_rows,
                           uint8_t* out, int64_t out_capacity, int64_t* out_bytes) {
  if (!desc || !out_bytes || n_rows < 0 || (n_rows > 0 && (!rows || !out)) || desc->n_volumes < 0 ||
      (desc->n_volumes > 0 && !desc->volumes) || desc->names_bytes < 0 || (desc->names_bytes > 0 && !desc->names))
    return fail("bad argument");
  if (n_rows >= (1ll << 38)) return fail("too many rows in one call");
  std::vector<cok::Volume> vols(desc->n_volumes);
  for (int i = 0; i < desc->n_volumes; ++i) {
    const FfnCoordinateVolume& v = desc->volumes[i];
    for (int a = 0; a < 3; ++a) {
      if (v.crop_shape_zyx[a] < 0 || v.margin_zyx[a] < 0 || (int64_t)v.margin_zyx[a] + v.crop_shape_zyx[a] >= (1ll << 31))
        return fail("crop shapes and margins must be non-negative and their sum below 2^31");
      vols[i].n[a] = v.crop_shape_zyx[a];
      vols[i].margin[a] = v.margin_zyx[a];
    }
    if (v.name_offset < 0 || v.name_length < 0 || v.name_offset > desc->names_bytes ||
        v.name_length > desc->names_bytes - v.name_offset)
      return fail("a volume name lies outside the names");
    vols[i].name_off = v.name_offset;
    vols[i].name_len = v.name_length;
  }
  *out_bytes = 0;
  if (n_rows == 0) return 0;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const long long nblocks = (n_rows + cok::kThreads - 1) / cok::kThreads;
  DevBufs bufs;
  longlong2* d_rows = nullptr;
  cok::Volume* d_vols = nullptr;
  unsigned char *d_names = nullptr, *d_out = nullptr;
  cok::u64 *d_sums = nullptr, *d_offs = nullptr;
  int* d_bad = nullptr;
  auto scan = [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_sums, d_offs, (int64_t)nblocks + 1, st);
  };
  CubTemp temp;
  if (bufs.get(&d_rows, n_rows) || bufs.get(&d_vols, vols.size()) || bufs.get(&d_names, desc->names_bytes) ||
      bufs.get(&d_sums, nblocks + 1) || bufs.get(&d_offs, nblocks + 1) || bufs.get(&d_bad, 1) || temp.alloc(bufs, scan))
    return 1;
  CUDA_OK(cudaMemcpyAsync(d_rows, rows, n_rows * sizeof(longlong2), cudaMemcpyHostToDevice, st));
  if (!vols.empty())
    CUDA_OK(cudaMemcpyAsync(d_vols, vols.data(), vols.size() * sizeof(cok::Volume), cudaMemcpyHostToDevice, st));
  if (desc->names_bytes)
    CUDA_OK(cudaMemcpyAsync(d_names, desc->names, desc->names_bytes, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(d_sums + nblocks, 0, sizeof(cok::u64), st));
  CUDA_OK(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
  cok::record_sums<<<(unsigned)nblocks, cok::kThreads, 0, st>>>(d_rows, n_rows, d_vols, desc->n_volumes, d_sums, d_bad);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(temp.run(scan));
  cok::u64 total = 0;
  int bad = 0;
  CUDA_OK(cudaMemcpyAsync(&total, d_offs + nblocks, sizeof(total), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  if (bad) return fail("a row's volume or flat index lies outside the volume table");
  *out_bytes = (int64_t)total;
  if ((int64_t)total > out_capacity) return fail("the output buffer is smaller than the records");
  if (bufs.get(&d_out, total)) return 1;
  cok::write_records<<<(unsigned)nblocks, cok::kThreads, 0, st>>>(d_rows, n_rows, d_vols, desc->n_volumes, d_names,
                                                                  d_offs, d_out);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
