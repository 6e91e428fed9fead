// resegmentation.cu — the device side of resegmentation: the decision points of a segmentation
// (ffn_decision_points) and the scoring of resegmentation results (ffn_reseg_eval).  Both use the nearest-id
// transform of decision_kernels.cuh, so both live in the one translation unit that includes it.

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include <cub/cub.cuh>

#include "../../include/ffn_b200.h"
#include "decision_kernels.cuh"
#include "host.cuh"
#include "reseg_kernels.cuh"

using namespace ffn;

extern "C" {

int ffn_decision_points(int device, const FfnDecisionPointDesc* desc, uint64_t* labels, FfnDecisionPoint* out,
                        int64_t cap, int64_t* n_out) {
  using dpk::u64;
  if (!desc || !labels || !n_out || cap < 0 || (cap > 0 && !out)) return fail("bad argument");
  const int sz = desc->shape_zyx[0], sy = desc->shape_zyx[1], sx = desc->shape_zyx[2];
  if (sz < 1 || sy < 1 || sx < 1) return fail("shape must be positive");
  const size_t n = (size_t)sz * sy * sx;
  if (n >= (1ull << 31)) return fail("decision points support volumes of fewer than 2^31 voxels");
  const int w[3] = {desc->voxel_size_xyz[2], desc->voxel_size_xyz[1], desc->voxel_size_xyz[0]};   // z, y, x
  for (int a = 0; a < 3; ++a) {
    if (w[a] < 1) return fail("voxel sizes must be positive integers");
    if (desc->box_start_zyx[a] < 0 || desc->box_size_zyx[a] < 0 ||
        (int64_t)desc->box_start_zyx[a] + desc->box_size_zyx[a] > desc->shape_zyx[a])
      return fail("subvolume box lies outside the volume");
  }
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int blocks = prop.multiProcessorCount * 16;
  DevBufs bufs;

  // Compaction: sorted unique ids and their counts; the kept ids (non-zero, not dust) in uint64 order.
  u64 *d_lab = nullptr, *d_sorted = nullptr, *d_unique = nullptr;
  unsigned* d_counts = nullptr;
  unsigned char* d_flags = nullptr;
  int* d_num = nullptr;   // [0] runs, [1] kept ids
  int nruns = (int)n;     // an upper bound until the run-length encoding has counted them
  if (bufs.get(&d_lab, n) || bufs.get(&d_sorted, n) || bufs.get(&d_unique, n) || bufs.get(&d_counts, n) ||
      bufs.get(&d_num, 2))
    return 1;
  u64* const d_kept = d_sorted;   // the sorted copy is no longer needed once the runs are encoded
  auto sort = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortKeys(t, b, d_lab, d_sorted, (int)n, 0, 64, st);
  };
  auto rle = [&](void* t, size_t& b) {
    return cub::DeviceRunLengthEncode::Encode(t, b, d_sorted, d_unique, d_counts, d_num, (int)n, st);
  };
  auto select = [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, d_unique, d_flags, d_kept, d_num + 1, nruns, st);
  };
  CubTemp temp;
  if (temp.alloc(bufs, sort, rle, select)) return 1;
  CUDA_OK(cudaMemcpyAsync(d_lab, labels, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(temp.run(sort));
  CUDA_OK(temp.run(rle));
  u64 first_id = 0;
  CUDA_OK(cudaMemcpyAsync(&nruns, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(&first_id, d_unique, sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  if (bufs.get(&d_flags, nruns)) return 1;
  dpk::flag_kept<<<blocks, 256, 0, st>>>(d_unique, d_counts, nruns, desc->dust_threshold, d_flags);
  CUDA_OK(temp.run(select));
  int nkept = 0;
  CUDA_OK(cudaMemcpyAsync(&nkept, d_num + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_unique);
  bufs.release(d_counts);
  bufs.release(temp.p);
  bufs.release(d_flags);
  const bool dust_cleared = nkept < nruns - (first_id == 0 ? 1 : 0);

  // Key range: every finite key (D + 1) * M - 1 must stay below kInf.
  int log_m = 0;
  while ((1ull << log_m) <= (u64)nkept) ++log_m;
  const u64 m = 1ull << log_m;
  unsigned __int128 dmax = 0;
  for (int a = 0; a < 3; ++a) {
    const unsigned __int128 e = (unsigned __int128)w[a] * (unsigned __int128)(desc->shape_zyx[a] - 1);
    dmax += e * e;
  }
  if (dmax >= ((unsigned __int128)1 << 64) || ((dmax + 1) << log_m) >= ((unsigned __int128)1 << 64))
    return fail("voxel size and extent too large for exact 64-bit distance keys: (D_max + 1) * M = (" +
                std::to_string((double)dmax) + " + 1) * " + std::to_string(m) + " does not fit in 64 bits");

  u64 *keys = nullptr, *keys2 = nullptr;
  if (bufs.get(&keys, n)) return 1;
  dpk::init_keys<<<blocks, 256, 0, st>>>(d_lab, d_kept, nkept, keys, n);
  CUDA_OK(cudaGetLastError());
  if (dust_cleared) CUDA_OK(cudaMemcpyAsync(labels, d_lab, n * sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(d_lab);
  *n_out = 0;
  dpk::PairGeom g{};
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = desc->box_start_zyx[a];
    g.size[a] = desc->box_size_zyx[a];
  }
  if (nkept == 0 || (size_t)g.size[0] * g.size[1] * g.size[2] == 0) return 0;

  // Exact nearest-id transform: x sweeps in place, then y (keys -> keys2) and z (keys2 -> keys).
  int *sbuf = nullptr, *tbuf = nullptr;
  if (bufs.get(&keys2, n) || bufs.get(&sbuf, n) || bufs.get(&tbuf, n)) return 1;
  dpk::nid_x<<<blocks, 128, 0, st>>>(keys, sz, sy, sx, m * (u64)w[2] * (u64)w[2], m);
  dpk::nid_line<<<blocks, 128, 0, st>>>(keys, keys2, 1, sz, sy, sx, m * (u64)w[1] * (u64)w[1], sbuf, tbuf);
  dpk::nid_line<<<blocks, 128, 0, st>>>(keys2, keys, 0, sz, sy, sx, m * (u64)w[0] * (u64)w[0], sbuf, tbuf);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(st));
  bufs.release(keys2);
  bufs.release(sbuf);
  bufs.release(tbuf);

  // Pair search; a table that fills up is discarded and rebuilt four times larger.
  g.sy = sy;
  g.sx = sx;
  g.m = m;
  g.log_m = log_m;
  g.use_max_distance = desc->use_max_distance;
  g.max_distance = desc->max_distance;
  dpk::PairTable t{};
  u64* tmem = nullptr;
  u64* d_misc = nullptr;   // [0] reserved slots, [1] overflow flag, [2] emitted pairs
  if (bufs.get(&d_misc, 3)) return 1;
  for (u64 tcap = 4096;; tcap *= 4) {
    if (bufs.get(&tmem, 8 * tcap)) return 1;
    t.key = tmem;
    t.dist = tmem + tcap;
    t.cnt = tmem + 2 * tcap;
    t.sum = tmem + 3 * tcap;
    t.c2 = tmem + 6 * tcap;
    t.ord = tmem + 7 * tcap;
    t.cap = tcap;
    t.limit = tcap / 2;
    t.used = d_misc;
    t.overflow = (int*)(d_misc + 1);
    CUDA_OK(cudaMemsetAsync(d_misc, 0, 3 * sizeof(u64), st));
    dpk::table_init<<<blocks, 256, 0, st>>>(t);
    dpk::pair_pass<1><<<blocks, 256, 0, st>>>(keys, g, t);
    CUDA_OK(cudaGetLastError());
    u64 misc[2] = {0, 0};
    CUDA_OK(cudaMemcpyAsync(misc, d_misc, sizeof(misc), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (misc[1] == 0) break;
    bufs.release(tmem);
  }
  dpk::pair_pass<2><<<blocks, 256, 0, st>>>(keys, g, t);
  dpk::pair_pass<3><<<blocks, 256, 0, st>>>(keys, g, t);
  dpk::pair_pass<4><<<blocks, 256, 0, st>>>(keys, g, t);
  FfnDecisionPoint* d_out = nullptr;
  if (bufs.get(&d_out, t.limit)) return 1;
  dpk::emit_pairs<<<blocks, 256, 0, st>>>(t, d_kept, g.size[1], g.size[2], d_out, d_misc + 2);
  CUDA_OK(cudaGetLastError());
  u64 npairs = 0;
  CUDA_OK(cudaMemcpyAsync(&npairs, d_misc + 2, sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  std::vector<FfnDecisionPoint> host(npairs);
  CUDA_OK(cudaMemcpyAsync(host.data(), d_out, npairs * sizeof(FfnDecisionPoint), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  std::sort(host.begin(), host.end(), [](const FfnDecisionPoint& p, const FfnDecisionPoint& q) {
    return p.id_a < q.id_a || (p.id_a == q.id_a && p.id_b < q.id_b);
  });
  *n_out = (int64_t)npairs;
  std::copy(host.begin(), host.begin() + std::min<int64_t>(cap, (int64_t)npairs), out);
  return 0;
}

int ffn_reseg_eval(int device, const FfnResegEvalDesc* desc, const uint64_t* labels, const uint8_t* probs,
                   const uint64_t* ids, const uint8_t mask_table[256], FfnResegStats* stats_out,
                   FfnResegOverlap* overlaps_out, int64_t cap, int64_t* n_overlaps) {
  using rsk::u64;
  if (!desc || !n_overlaps || !stats_out || cap < 0 || (cap > 0 && !overlaps_out) || desc->num_items < 0 ||
      (desc->num_items > 0 && (!labels || !probs || !ids || !mask_table)))
    return fail("bad argument");
  const int bz = desc->box_zyx[0], by = desc->box_zyx[1], bx = desc->box_zyx[2];
  if (bz < 1 || by < 1 || bx < 1) return fail("box extent must be positive");
  const long long nitems = desc->num_items, nbox = (long long)bz * by * bx;
  const bool pair = desc->pair != 0;
  if (nitems > 0 && nbox > ((1ll << 31) - 1) / (nitems * (pair ? 4 : 1)))
    return fail("resegmentation analysis supports batches of fewer than 2^31 mask voxels (four masks per pair item)");
  const int w[3] = {desc->voxel_size_zyx[0], desc->voxel_size_zyx[1], desc->voxel_size_zyx[2]};
  unsigned __int128 dmax = 0;   // covers the no-background value, which uses the full z extent
  for (int a = 0; a < 3; ++a) {
    if (pair && w[a] < 1) return fail("voxel sizes must be positive integers");
    const unsigned __int128 e = (unsigned __int128)(pair ? w[a] : 0) * (unsigned __int128)desc->box_zyx[a];
    dmax += e * e;
  }
  if (dmax >= ((unsigned __int128)1 << 63)) return fail("voxel size and box too large for exact 64-bit squared distances");
  *n_overlaps = 0;
  if (nitems == 0) return 0;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const int blocks = prop.multiProcessorCount * 16;
  // Items (grid y) x blocks per box (grid x): about 16 resident blocks per SM over the whole batch.
  const dim3 item_grid((unsigned)std::max<long long>(1, std::min<long long>((nbox + 1023) / 1024,
                                                                              std::max<long long>(1, blocks / nitems))),
                       (unsigned)std::min<long long>(nitems, 65535));
  const size_t n = (size_t)(nitems * nbox);
  const int nprob = pair ? 2 : 1;
  DevBufs bufs;
  u64 *d_lab = nullptr, *d_ids = nullptr, *d_counts = nullptr;
  unsigned char *d_probs = nullptr, *d_table = nullptr;
  const int ncounts = pair ? rsk::kPairCounts : 2;
  if (bufs.get(&d_lab, n) || bufs.get(&d_probs, n * nprob) || bufs.get(&d_table, 256) ||
      bufs.get(&d_counts, (size_t)nitems * ncounts) || bufs.get(&d_ids, 2 * nitems))
    return 1;
  CUDA_OK(cudaMemcpyAsync(d_lab, labels, n * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_ids, ids, 2 * nitems * sizeof(u64), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_probs, probs, n * nprob, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_table, mask_table, 256, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(d_counts, 0, (size_t)nitems * ncounts * sizeof(u64), st));
  std::vector<u64> counts((size_t)nitems * ncounts);
  std::memset(stats_out, 0, (size_t)nitems * sizeof(FfnResegStats));

  if (pair) {
    // Four masks per item, then the exact squared EDT of every mask at once: with a single id, the nearest-id keys of
    // decision_kernels.cuh are plain squared distances (M = 1).  Boxes are stacked along z for the x and y passes and
    // seen as (masks, Z, Y * X) for the z pass, so that no line crosses a box.
    const long long nmasks = 4 * nitems;
    const size_t nk = (size_t)nmasks * nbox;
    u64 *keys = nullptr, *keys2 = nullptr, *d_max = nullptr;
    int *sbuf = nullptr, *tbuf = nullptr;
    if (bufs.get(&keys, nk) || bufs.get(&keys2, nk) || bufs.get(&sbuf, nk) ||
        bufs.get(&tbuf, nk) || bufs.get(&d_max, nmasks))
      return 1;
    CUDA_OK(cudaMemsetAsync(d_max, 0, nmasks * sizeof(u64), st));
    rsk::pair_prepare<<<item_grid, 256, 0, st>>>(d_lab, d_probs, d_ids, d_table, nitems, nbox, keys, d_counts);
    const int zs = (int)(nmasks * bz);
    dpk::nid_x<<<blocks, 128, 0, st>>>(keys, zs, by, bx, (u64)w[2] * (u64)w[2], 1);
    dpk::nid_line<<<blocks, 128, 0, st>>>(keys, keys2, 1, zs, by, bx, (u64)w[1] * (u64)w[1], sbuf, tbuf);
    dpk::nid_line<<<blocks, 128, 0, st>>>(keys2, keys, 1, (int)nmasks, bz, by * bx, (u64)w[0] * (u64)w[0], sbuf, tbuf);
    const dim3 mask_grid(item_grid.x, (unsigned)std::min<long long>(nmasks, 65535));
    rsk::edt_max<<<mask_grid, 256, 0, st>>>(keys, nmasks, nbox, d_max);
    CUDA_OK(cudaGetLastError());
    std::vector<u64> maxes(nmasks);
    CUDA_OK(cudaMemcpyAsync(maxes.data(), d_max, nmasks * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(counts.data(), d_counts, counts.size() * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    // No voxel outside the mask: scipy's feature transform then points every voxel at (-1, 0, 0).
    const u64 full = (u64)bz * bz * w[0] * w[0] + (u64)(by - 1) * (by - 1) * w[1] * w[1] +
                     (u64)(bx - 1) * (bx - 1) * w[2] * w[2];
    for (long long it = 0; it < nitems; ++it) {
      const u64* c = &counts[it * rsk::kPairCounts];
      FfnResegStats& s = stats_out[it];
      s.n_seg[0] = (int64_t)c[0];
      s.n_seg[1] = (int64_t)c[1];
      s.n_reseg[0] = (int64_t)c[2];
      s.n_reseg[1] = (int64_t)c[3];
      s.n_reseg_seg[0][0] = (int64_t)c[4];
      s.n_reseg_seg[0][1] = (int64_t)c[5];
      s.n_reseg_seg[1][0] = (int64_t)c[6];
      s.n_reseg_seg[1][1] = (int64_t)c[7];
      s.n_inter = (int64_t)c[8];
      s.n_union = (int64_t)c[9];
      for (int k = 0; k < 4; ++k) s.max_edt2[k] = maxes[4 * it + k] == rsk::kInf ? full : maxes[4 * it + k];
    }
    return 0;
  }

  // Endpoint: |mask| per item, and the voxels of every (item, label) split by mask, by sorting on label and then
  // (stably) on item.
  if (nitems >= (1ll << 30)) return fail("too many endpoint items");
  int ibits = 1;
  while ((1ll << ibits) < nitems) ++ibits;
  const int ni = (int)n;
  int nruns = ni;   // an upper bound until the runs are counted: at most one row per voxel
  u64* d_lab2 = nullptr;
  unsigned *d_vals = nullptr, *d_vals2 = nullptr, *d_scan = nullptr;
  unsigned char* d_head = nullptr;
  int *d_heads = nullptr, *d_num = nullptr;
  FfnResegOverlap *d_all = nullptr, *d_kept = nullptr;
  if (bufs.get(&d_lab2, n) || bufs.get(&d_vals, n) || bufs.get(&d_vals2, n) || bufs.get(&d_scan, n) ||
      bufs.get(&d_head, n) || bufs.get(&d_heads, n) || bufs.get(&d_num, 2))
    return 1;
  rsk::endpoint_prepare<<<item_grid, 256, 0, st>>>(d_lab, d_probs, d_ids, d_table, nitems, nbox, d_vals, d_counts);
  auto sort_label = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, d_lab, d_lab2, d_vals, d_vals2, ni, 0, 64, st);
  };
  auto sort_item = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, d_vals2, d_vals, d_lab2, d_lab, ni, 1, 1 + ibits, st);
  };
  auto select_heads = [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, cub::CountingInputIterator<int>(0), d_head, d_heads, d_num, ni, st);
  };
  auto scan = [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, d_vals2, d_scan, ni, st); };
  auto select_rows = [&](void* t, size_t& b) {
    return cub::DeviceSelect::If(t, b, d_all, d_kept, d_num + 1, nruns, rsk::Overlapping(), st);
  };
  CubTemp temp;
  if (temp.alloc(bufs, sort_label, sort_item, select_heads, scan, select_rows)) return 1;
  CUDA_OK(temp.run(sort_label));
  CUDA_OK(temp.run(sort_item));
  // Sorted by (item, label): d_vals = item << 1 | mask, d_lab = label.
  rsk::run_heads<<<blocks, 256, 0, st>>>(d_vals, d_lab, ni, d_head, d_vals2);
  CUDA_OK(temp.run(select_heads));
  CUDA_OK(temp.run(scan));
  CUDA_OK(cudaMemcpyAsync(&nruns, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(counts.data(), d_counts, counts.size() * sizeof(u64), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  if (bufs.get(&d_all, nruns) || bufs.get(&d_kept, nruns)) return 1;
  rsk::run_rows<<<blocks, 256, 0, st>>>(d_heads, nruns, ni, d_vals, d_lab, d_scan, d_all);
  CUDA_OK(temp.run(select_rows));
  CUDA_OK(cudaGetLastError());
  int nkept = 0;
  CUDA_OK(cudaMemcpyAsync(&nkept, d_num + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  const int64_t m = std::min<int64_t>(cap, nkept);
  if (m > 0) CUDA_OK(cudaMemcpyAsync(overlaps_out, d_kept, m * sizeof(FfnResegOverlap), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  for (long long it = 0; it < nitems; ++it) {
    stats_out[it].n_seg[0] = (int64_t)counts[2 * it];
    stats_out[it].n_reseg[0] = (int64_t)counts[2 * it + 1];
  }
  *n_overlaps = nkept;
  return 0;
}

}  // extern "C"
