// partitions.cu — the partition map of a labelled volume on the device (ffn_compute_partitions).

#include <algorithm>
#include <vector>

#include <cub/cub.cuh>

#include "../../include/ffn_b200.h"
#include "host.cuh"
#include "partition_kernels.cuh"

using namespace ffn;

extern "C" {

int ffn_compute_partitions(int device, const FfnPartitionDesc* desc, uint64_t* labels, const uint8_t* mask,
                           uint8_t* out, int64_t counts[256]) {
  using ptk::u64;
  if (!desc || !labels || !out || !counts || desc->n_thresholds < 0 || (desc->n_thresholds > 0 && !desc->thresholds) ||
      desc->n_spheres < 0 || (desc->n_spheres > 0 && !desc->spheres) || desc->n_whitelist < 0 ||
      (desc->n_whitelist > 0 && !desc->whitelist))
    return fail("bad argument");
  ptk::Geometry g{};
  size_t n = 1, nout = 1;
  for (int a = 0; a < 3; ++a) {
    g.s[a] = desc->shape_zyx[a];
    g.r[a] = desc->lom_radius_zyx[a];
    if (g.s[a] < 0) return fail("shape must not be negative");
    if (g.r[a] < 0) return fail("the LOM radius must not be negative");
    g.o[a] = (int)std::max<int64_t>((int64_t)g.s[a] - 2 * (int64_t)g.r[a], 0);
    n *= (size_t)g.s[a];
    nout *= (size_t)g.o[a];
  }
  if (n >= (1ull << 31)) return fail("partition maps support volumes of fewer than 2^31 voxels");
  std::fill(counts, counts + 256, (int64_t)0);
  if (desc->n_labels_out) *desc->n_labels_out = 0;
  if (n == 0) return 0;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int blocks = prop.multiProcessorCount * 16;
  const int ni = (int)n;
  DevBufs bufs;

  // Compaction: sorted unique ids and their counts.
  u64 *d_lab = nullptr, *d_sorted = nullptr, *d_unique = nullptr;
  unsigned* d_cnt = nullptr;
  int* d_num = nullptr;
  if (bufs.get(&d_lab, n) || bufs.get(&d_sorted, n) || bufs.get(&d_unique, n) || bufs.get(&d_cnt, n) ||
      bufs.get(&d_num, 1))
    return 1;
  auto sort = [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, d_lab, d_sorted, ni, 0, 64, st); };
  auto rle = [&](void* t, size_t& b) {
    return cub::DeviceRunLengthEncode::Encode(t, b, d_sorted, d_unique, d_cnt, d_num, ni, st);
  };
  CubTemp temp;
  if (temp.alloc(bufs, sort, rle)) return 1;
  CUDA_OK(cudaMemcpyAsync(d_lab, labels, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(temp.run(sort));
  CUDA_OK(temp.run(rle));
  int nruns = 0;
  CUDA_OK(cudaMemcpyAsync(&nruns, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  std::vector<u64> ids(nruns);
  std::vector<unsigned> sizes(nruns);
  CUDA_OK(cudaMemcpyAsync(ids.data(), d_unique, nruns * sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(sizes.data(), d_cnt, nruns * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_sorted);
  bufs.release(d_cnt);
  bufs.release(temp.p);

  // Run codes: dust (cleared), skipped (0, or outside the whitelist) or the compact id, in uint64 id order.
  std::vector<u64> white(desc->whitelist, desc->whitelist + desc->n_whitelist);
  std::sort(white.begin(), white.end());
  std::vector<int> code(nruns);
  int nk = 0;
  bool dust = false;
  for (int i = 0; i < nruns; ++i) {
    if (ids[i] != 0 && desc->min_size > 0 && (int64_t)sizes[i] < desc->min_size) {
      code[i] = ptk::kDust;
      dust = true;
    } else if (ids[i] == 0 || (desc->use_whitelist && !std::binary_search(white.begin(), white.end(), ids[i]))) {
      code[i] = ptk::kSkipped;
    } else {
      code[i] = nk++;
    }
  }
  if (desc->n_labels_out) *desc->n_labels_out = nk;
  int *d_code = nullptr, *d_compact = nullptr, *d_bmin = nullptr, *d_bmax = nullptr;
  if (bufs.get(&d_code, nruns) || bufs.get(&d_compact, n) || bufs.get(&d_bmin, 3 * (size_t)nk) ||
      bufs.get(&d_bmax, 3 * (size_t)nk))
    return 1;
  CUDA_OK(cudaMemcpyAsync(d_code, code.data(), nruns * sizeof(int), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(d_bmin, 0x7f, 3 * (size_t)nk * sizeof(int), st));
  CUDA_OK(cudaMemsetAsync(d_bmax, 0xff, 3 * (size_t)nk * sizeof(int), st));
  ptk::compact_ids<<<blocks, 256, 0, st>>>(d_lab, n, d_unique, nruns, d_code, d_compact, d_bmin, d_bmax, g.s[1], g.s[2]);
  CUDA_OK(cudaGetLastError());
  if (dust) CUDA_OK(cudaMemcpyAsync(labels, d_lab, n * sizeof(u64), cudaMemcpyDeviceToHost, st));
  std::vector<int> bmin(3 * (size_t)nk), bmax(3 * (size_t)nk);
  if (nk > 0) {
    CUDA_OK(cudaMemcpyAsync(bmin.data(), d_bmin, bmin.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(bmax.data(), d_bmax, bmax.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_lab);
  bufs.release(d_unique);
  bufs.release(d_code);
  if (nout == 0) {
    CUDA_OK(cudaGetLastError());
    return 0;
  }

  unsigned char* d_out = nullptr;
  if (bufs.get(&d_out, nout)) return 1;
  CUDA_OK(cudaMemsetAsync(d_out, 0, nout, st));

  // Grown boxes: the windows of a label's voxels inside the VALID region, i.e. its box clipped to [r, s - r) and
  // grown by r.  A label with no voxel there writes nothing and is left out.
  std::vector<ptk::LabelBox> boxes;
  std::vector<long long> vols;
  for (int k = 0; k < nk; ++k) {
    ptk::LabelBox b{};
    b.k = k;
    bool empty = false;
    for (int a = 0; a < 3; ++a) {
      const int lo = std::max(bmin[3 * k + a], g.r[a]), hi = std::min(bmax[3 * k + a] + 1, g.s[a] - g.r[a]);
      empty |= lo >= hi;
      b.lo[a] = lo - g.r[a];
      b.n[a] = hi - lo + 2 * g.r[a];
    }
    if (empty) continue;
    boxes.push_back(b);
    vols.push_back((long long)b.n[0] * b.n[1] * b.n[2]);
  }
  // Groups whose two int32 scratch arrays fit the budget, in label order.
  long long budget = desc->scratch_bytes;
  if (budget <= 0) {
    size_t free_b = 0, total_b = 0;
    CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
    budget = (long long)(free_b / 4);
  }
  const long long per_vox = 2 * (long long)sizeof(int);
  std::vector<size_t> group_start{0};
  long long gvol = 0, max_gvol = 0;
  for (size_t j = 0; j < boxes.size(); ++j) {
    if (j > group_start.back() && (gvol + vols[j]) * per_vox > budget) {
      group_start.push_back(j);
      gvol = 0;
    }
    ptk::LabelBox& b = boxes[j];
    if (j > group_start.back()) {   // the first box of a group starts at scratch voxel 0 and line 0
      const ptk::LabelBox& p = boxes[j - 1];
      b.off = p.off + vols[j - 1];
      b.line[0] = p.line[0] + (long long)p.n[0] * p.n[1];
      b.line[1] = p.line[1] + (long long)p.n[0] * p.n[2];
      b.line[2] = p.line[2] + (long long)p.n[1] * p.n[2];
    }
    gvol += vols[j];
    max_gvol = std::max(max_gvol, gvol);
  }
  group_start.push_back(boxes.size());

  if (!boxes.empty()) {
    ptk::LabelBox* d_boxes = nullptr;
    double* d_th = nullptr;
    int *d_A = nullptr, *d_B = nullptr;
    if (bufs.get(&d_boxes, boxes.size()) || bufs.get(&d_th, desc->n_thresholds) || bufs.get(&d_A, max_gvol) ||
        bufs.get(&d_B, max_gvol))
      return 1;
    CUDA_OK(cudaMemcpyAsync(d_boxes, boxes.data(), boxes.size() * sizeof(ptk::LabelBox), cudaMemcpyHostToDevice, st));
    if (desc->n_thresholds)
      CUDA_OK(cudaMemcpyAsync(d_th, desc->thresholds, desc->n_thresholds * sizeof(double), cudaMemcpyHostToDevice, st));
    const double fov = (double)(2 * g.r[0] + 1) * (double)(2 * g.r[1] + 1) * (double)(2 * g.r[2] + 1);
    auto grid_for = [&](long long lines) { return (int)std::min<long long>((lines + 255) / 256, blocks * 2); };
    for (size_t gi = 0; gi + 1 < group_start.size(); ++gi) {
      const size_t j0 = group_start[gi], j1 = group_start[gi + 1];
      const ptk::LabelBox& last = boxes[j1 - 1];
      const int nb = (int)(j1 - j0);
      const long long lx = last.line[0] + (long long)last.n[0] * last.n[1];
      const long long ly = last.line[1] + (long long)last.n[0] * last.n[2];
      const long long lz = last.line[2] + (long long)last.n[1] * last.n[2];
      ptk::count_x<<<grid_for(lx), 256, 0, st>>>(d_compact, d_boxes + j0, nb, lx, g, d_A);
      ptk::count_y<<<grid_for(ly), 256, 0, st>>>(d_A, d_boxes + j0, nb, ly, g, d_B);
      ptk::count_z<<<grid_for(lz), 256, 0, st>>>(d_B, d_compact, d_boxes + j0, nb, lz, g, fov, d_th,
                                                  desc->n_thresholds, d_out);
      CUDA_OK(cudaGetLastError());
    }
    CUDA_OK(cudaStreamSynchronize(st));
    bufs.release(d_A);
    bufs.release(d_B);
  }
  bufs.release(d_compact);

  // Mask: any() over the LOM box, one axis at a time (x, then y, then z).
  unsigned char* d_masked = nullptr;
  if (mask) {
    unsigned char *d_m0 = nullptr, *d_m1 = nullptr;
    if (bufs.get(&d_m0, n) || bufs.get(&d_m1, n)) return 1;
    CUDA_OK(cudaMemcpyAsync(d_m0, mask, n, cudaMemcpyHostToDevice, st));
    ptk::box_any<<<blocks, 256, 0, st>>>(d_m0, d_m1, 2, g.r[2], g.s[0], g.s[1], g.s[2]);
    ptk::box_any<<<blocks, 256, 0, st>>>(d_m1, d_m0, 1, g.r[1], g.s[0], g.s[1], g.o[2]);
    ptk::box_any<<<blocks, 256, 0, st>>>(d_m0, d_m1, 0, g.r[0], g.s[0], g.o[1], g.o[2]);
    CUDA_OK(cudaGetLastError());
    d_masked = d_m1;
  }
  ptk::Sphere* d_sph = nullptr;
  unsigned long long* d_hist = nullptr;
  if (bufs.get(&d_sph, desc->n_spheres) || bufs.get(&d_hist, 256)) return 1;
  std::vector<ptk::Sphere> sph(desc->n_spheres);
  for (int s = 0; s < desc->n_spheres; ++s) {
    const FfnExclusionSphere& e = desc->spheres[s];
    for (int a = 0; a < 3; ++a) {
      sph[s].c[a] = e.c_xyz[a];
      sph[s].fc[a] = e.f_xyz[a];
    }
    sph[s].r2 = e.r2;
    sph[s].fr2 = e.f_r2;
    sph[s].integer = e.integer;
  }
  if (!sph.empty())
    CUDA_OK(cudaMemcpyAsync(d_sph, sph.data(), sph.size() * sizeof(ptk::Sphere), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(d_hist, 0, 256 * sizeof(unsigned long long), st));
  ptk::finish<<<blocks, 256, 0, st>>>(d_out, nout, d_masked, d_sph, desc->n_spheres, g, d_hist);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(out, d_out, nout, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(counts, d_hist, 256 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
