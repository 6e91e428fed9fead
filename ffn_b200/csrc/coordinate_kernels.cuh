// coordinate_kernels.cuh — training coordinates from partition maps (build_coordinates.py:61-112) on the device.
// Passes (C: voxels of one crop, K: kept voxels (value != 255), R: records of a chunk):
//   bucket_hist      per 4096-voxel tile of the crop: 256-bin histogram (value-major), and the crop's counts  1 B/C
//   (cub scan)       exclusive sum over the value-major tile histograms = base of every (value, tile)        8 B per tile and value
//   bucket_scatter   stable counting-sort scatter: (volume, flat) int64 rows grouped by value, 255 dropped   1 B/C read, 16 B/K
//   record_sums      per block of records: the bytes of its TFRecord frames                                   16 B/R read
//   (cub scan)       exclusive sum over the block sums
//   write_records    unravel, Example payload, CRC-32C frames, written at the block offset + block scan      16 B/R read, ~70 B/R
// The crop is read in place from the uploaded volume: flat crop index f -> (z, y, x) -> volume offset.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

namespace ffn {
namespace cok {

typedef unsigned long long u64;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPerLane = 16;
constexpr int kTile = kThreads * kPerLane;   // voxels per tile; warp w owns [w * 512, (w + 1) * 512) of it
constexpr int kIgnore = 255;                 // IGNORE_PARTITION: counted, never written as a row

struct Crop {
  int n[3];          // crop extent (z, y, x)
  int lo[3];         // crop start in the volume
  long long sy, sz;  // volume strides (elements) of y and z
  long long size;    // n[0] * n[1] * n[2] (< 2^31)
};

// The value at flat crop index f, or 256 past the end of the crop.  Lane l of warp w loads voxels
// tile * kTile + w * 512 + j * 32 + l, so a warp reads 32 consecutive crop voxels per step and steps in flat order.
__device__ __forceinline__ void load_tile(const unsigned char* __restrict__ vol, const Crop& c, int tile,
                                          int key[kPerLane]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long base = (long long)tile * kTile + warp * (kPerLane * 32) + lane;
#pragma unroll
  for (int j = 0; j < kPerLane; ++j) {
    const long long f = base + j * 32;
    key[j] = 256;
    if (f < c.size) {
      const int x = (int)(f % c.n[2]);
      const long long zy = f / c.n[2];
      const int y = (int)(zy % c.n[1]), z = (int)(zy / c.n[1]);
      key[j] = vol[(long long)(c.lo[0] + z) * c.sz + (long long)(c.lo[1] + y) * c.sy + (c.lo[2] + x)];
    }
  }
}

// hist[v * ntiles + tile] = voxels of value v in the tile (every v, zeros included); counts[v] += the same.
__global__ void __launch_bounds__(kThreads) bucket_hist(const unsigned char* __restrict__ vol, Crop c, int ntiles,
                                                        int* __restrict__ hist, unsigned long long* counts) {
  __shared__ int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  int key[kPerLane];
  load_tile(vol, c, blockIdx.x, key);
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < kPerLane; ++j) {
    const unsigned peers = __match_any_sync(0xffffffffu, key[j]);
    if (key[j] < 256 && (__ffs(peers) - 1) == (int)lane) atomicAdd(&h[key[j]], __popc(peers));
  }
  __syncthreads();
  const int v = threadIdx.x;
  hist[(long long)v * ntiles + blockIdx.x] = h[v];
  if (h[v]) atomicAdd(&counts[v], (unsigned long long)h[v]);
}

// rows[base[v * ntiles + tile] + rank] = (volume, f) for every voxel of value v != 255, where rank counts the voxels
// of v before f in the tile: per-warp histograms are scanned in warp order, and inside a warp's 32-voxel step the
// lanes of one value (__match_any_sync) rank by lane, so each bucket stays in ascending flat order.
__global__ void __launch_bounds__(kThreads) bucket_scatter(const unsigned char* __restrict__ vol, Crop c, int ntiles,
                                                           const int* __restrict__ base, long long volume,
                                                           longlong2* __restrict__ rows) {
  __shared__ int wbase[kWarps][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kWarps * 256; i += kThreads) (&wbase[0][0])[i] = 0;
  __syncthreads();
  int key[kPerLane];
  load_tile(vol, c, blockIdx.x, key);
  const unsigned lt = (1u << lane) - 1;
#pragma unroll
  for (int j = 0; j < kPerLane; ++j) {
    const unsigned peers = __match_any_sync(0xffffffffu, key[j]);
    if (key[j] < kIgnore && (__ffs(peers) - 1) == lane) wbase[warp][key[j]] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {
    const int v = threadIdx.x;
    int run = v < kIgnore ? base[(long long)v * ntiles + blockIdx.x] : 0;
    for (int w = 0; w < kWarps; ++w) {
      const int n = wbase[w][v];
      wbase[w][v] = run;
      run += n;
    }
  }
  __syncthreads();
  const long long f0 = (long long)blockIdx.x * kTile + warp * (kPerLane * 32) + lane;
#pragma unroll
  for (int j = 0; j < kPerLane; ++j) {
    const int k = key[j];
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    if (k < kIgnore) rows[wbase[warp][k] + __popc(peers & lt)] = make_longlong2(volume, f0 + j * 32);
    __syncwarp();
    if (k < kIgnore && (__ffs(peers) - 1) == lane) wbase[warp][k] += __popc(peers);
    __syncwarp();
  }
}

// ---- TFRecord frames of tf.train.Example {center: Int64List, label_volume_name: BytesList} ----------------------
// Protobuf's deterministic encoding (map entries in key order) of
//   Example   { 1: Features }
//   Features  { 1: map entry {1: "center", 2: Feature {3: Int64List {1: packed [x, y, z]}}},
//               1: map entry {1: "label_volume_name", 2: Feature {1: BytesList {1: name}}} }
// framed as u64 length | u32 masked CRC-32C of the length | payload | u32 masked CRC-32C of the payload.

struct Volume {
  int n[3];             // crop extent (z, y, x)
  int margin[3];        // (z, y, x)
  long long name_off;   // into the names blob
  long long name_len;
};

__device__ __forceinline__ int varint_size(u64 v) {
  int n = 1;
  while (v >= 128) {
    v >>= 7;
    ++n;
  }
  return n;
}

struct Record {
  u64 c[3];        // center (x, y, z)
  int vol;
  int packed;      // bytes of the packed center values
  long long e2;    // label_volume_name map entry
  long long feats; // Features
  long long payload;
};

// Decodes row i; false when its volume index or flat index is outside the table.
__device__ __forceinline__ bool make_record(const longlong2 row, const Volume* vols, int nvol, Record& r) {
  if (row.x < 0 || row.x >= nvol) return false;
  const Volume v = vols[row.x];
  const long long size = (long long)v.n[0] * v.n[1] * v.n[2];
  if (row.y < 0 || row.y >= size) return false;
  const long long f = row.y;
  r.vol = (int)row.x;
  r.c[0] = (u64)(v.margin[2] + f % v.n[2]);
  r.c[1] = (u64)(v.margin[1] + (f / v.n[2]) % v.n[1]);
  r.c[2] = (u64)(v.margin[0] + f / ((long long)v.n[2] * v.n[1]));
  r.packed = varint_size(r.c[0]) + varint_size(r.c[1]) + varint_size(r.c[2]);
  // center entry: 0a 06 "center" 12 <4 + packed> 1a <2 + packed> 0a <packed> values  (packed <= 15: 1-byte lengths)
  const long long e1 = 14 + r.packed;
  const long long bl = 1 + varint_size(v.name_len) + v.name_len;
  const long long f2 = 1 + varint_size(bl) + bl;
  r.e2 = 19 + 1 + varint_size(f2) + f2;
  r.feats = 1 + varint_size(e1) + e1 + 1 + varint_size(r.e2) + r.e2;
  r.payload = 1 + varint_size(r.feats) + r.feats;
  return true;
}

__device__ __forceinline__ unsigned masked(unsigned crc) { return ((crc >> 15) | (crc << 17)) + 0xa282ead8u; }

// Byte writer that folds every byte into a running CRC-32C (table in shared memory).
struct Writer {
  unsigned char* p;
  unsigned crc;
  const unsigned* table;
  __device__ __forceinline__ void byte(unsigned b) {
    *p++ = (unsigned char)b;
    crc = table[(crc ^ b) & 0xffu] ^ (crc >> 8);
  }
  __device__ __forceinline__ void varint(u64 v) {
    while (v >= 128) {
      byte((unsigned)(v & 0x7f) | 0x80u);
      v >>= 7;
    }
    byte((unsigned)v);
  }
  __device__ __forceinline__ void raw32(unsigned v) {
    for (int i = 0; i < 4; ++i) *p++ = (unsigned char)(v >> (8 * i));
  }
};

__device__ __forceinline__ void crc_table(unsigned* t) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = (unsigned)i;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u)));
    t[i] = c;
  }
}

// sums[b] = bytes of the frames of block b's records; bad[0] = 1 when a row is outside the volume table.
__global__ void __launch_bounds__(kThreads) record_sums(const longlong2* __restrict__ rows, long long n,
                                                        const Volume* vols, int nvol, u64* sums, int* bad) {
  typedef cub::BlockReduce<u64, kThreads> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  u64 bytes = 0;
  if (i < n) {
    Record r;
    if (make_record(rows[i], vols, nvol, r)) bytes = 16 + r.payload;
    else atomicExch(bad, 1);
  }
  const u64 total = Reduce(tmp).Sum(bytes);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) write_records(const longlong2* __restrict__ rows, long long n,
                                                          const Volume* vols, int nvol,
                                                          const unsigned char* __restrict__ names,
                                                          const u64* __restrict__ block_off,
                                                          unsigned char* __restrict__ out) {
  typedef cub::BlockScan<u64, kThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ unsigned table[256];
  crc_table(table);
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  Record r;
  const bool ok = i < n && make_record(rows[i], vols, nvol, r);
  u64 off = 0;
  Scan(tmp).ExclusiveSum(ok ? (u64)(16 + r.payload) : 0ull, off);
  __syncthreads();   // the table
  if (!ok) return;
  Writer w{out + block_off[blockIdx.x] + off, ~0u, table};
  for (int k = 0; k < 8; ++k) w.byte((unsigned)((u64)r.payload >> (8 * k)) & 0xffu);
  w.raw32(masked(~w.crc));
  w.crc = ~0u;
  w.byte(0x0a);
  w.varint(r.feats);
  w.byte(0x0a);
  w.varint(14 + r.packed);
  w.byte(0x0a);
  w.byte(6);
  const char center[] = "center";
  for (int k = 0; k < 6; ++k) w.byte((unsigned char)center[k]);
  w.byte(0x12);
  w.byte(4 + r.packed);
  w.byte(0x1a);
  w.byte(2 + r.packed);
  w.byte(0x0a);
  w.byte(r.packed);
  for (int k = 0; k < 3; ++k) w.varint(r.c[k]);
  const Volume& v = vols[r.vol];
  const long long bl = 1 + varint_size(v.name_len) + v.name_len;
  w.byte(0x0a);
  w.varint(r.e2);
  w.byte(0x0a);
  w.byte(17);
  const char key[] = "label_volume_name";
  for (int k = 0; k < 17; ++k) w.byte((unsigned char)key[k]);
  w.byte(0x12);
  w.varint(1 + varint_size(bl) + bl);
  w.byte(0x0a);
  w.varint(bl);
  w.byte(0x0a);
  w.varint(v.name_len);
  const unsigned char* name = names + v.name_off;
  for (long long k = 0; k < v.name_len; ++k) w.byte(name[k]);
  w.raw32(masked(~w.crc));
}

}  // namespace cok
}  // namespace ffn
