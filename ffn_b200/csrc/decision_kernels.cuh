// decision_kernels.cuh — decision points of a segmentation (ffn/utils/decision_point.py:27-145) on the device.
// Every empty voxel takes the id of the nearest labelled voxel (smallest id on ties, exact integer distances),
// and every pair of ids that then touch gets the point where they come closest.  HBM-bound passes:
//   init_keys        uint64 label -> compact id by binary search; dust cleared     16 B/voxel (+ kept ids in L2)
//   nid_x            two sweeps per x-line, in place                                16 B/voxel
//   nid_line x2      lower envelope of parabolas per y- / z-line                    16 B/voxel + 16 B/voxel scratch
//   pair_pass x4     7 neighbour offsets over the box, hash table of (a, b)          8 B/voxel per pass (neighbours cached)
// The transform runs on one uint64 key per voxel, key = D * M + L: D the exact squared physical distance to the
// nearest labelled voxel, L its compact id (1..K, in uint64 id order) and M the power of two above K.  The minimum
// key is the lexicographic minimum of (D, id), and key(p) + M * (w (q - p))^2 stays a key, so the exact
// separable distance transform on keys carries the id and breaks ties towards the smallest id.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ffn_b200.h"

namespace ffn {
namespace dpk {

typedef unsigned long long u64;

constexpr u64 kInf = ~0ull;     // no labelled voxel reached
constexpr u64 kEmpty = ~0ull;   // free hash slot
constexpr int kOrderShift = 58; // order index = offset rank << 58 | box-linear voxel index

// Sorted unique ids -> the ids that stay labelled: non-zero and, when dust is cleared, at least `min_size` voxels.
__global__ void flag_kept(const u64* ids, const unsigned* counts, int nruns, long long min_size, unsigned char* flags) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nruns; i += gridDim.x * blockDim.x)
    flags[i] = ids[i] != 0 && (min_size <= 0 || (long long)counts[i] >= min_size);
}

// key = L (distance 0) for a kept label, kInf otherwise; labels of cleared ids are set to 0.
__global__ void init_keys(u64* labels, const u64* kept, int nkept, u64* keys, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const u64 lab = labels[i];
    u64 key = kInf;
    if (lab != 0) {
      int lo = 0, hi = nkept;   // first kept id >= lab
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (kept[mid] < lab) lo = mid + 1; else hi = mid;
      }
      if (lo < nkept && kept[lo] == lab) key = (u64)(lo + 1);
      else labels[i] = 0;
    }
    keys[i] = key;
  }
}

// Along x: the nearest labelled voxel of the same x-line on either side; the smaller key wins.  wx2m = M wx^2.
__global__ void nid_x(u64* keys, int sz, int sy, int sx, u64 wx2m, u64 m) {
  const size_t lines = (size_t)sz * sy;
  for (size_t l = (size_t)blockIdx.x * blockDim.x + threadIdx.x; l < lines; l += (size_t)gridDim.x * blockDim.x) {
    u64* row = keys + l * sx;
    int p = -1;
    u64 lp = 0;
    for (int x = 0; x < sx; ++x) {
      const u64 k = row[x];
      if (k < m) {
        p = x;
        lp = k;
      } else if (p >= 0) {
        const u64 d = (u64)(x - p);
        row[x] = d * d * wx2m + lp;
      }
    }
    p = -1;
    for (int x = sx - 1; x >= 0; --x) {
      const u64 k = row[x];
      if (k < m) {
        p = x;
        lp = k;
      } else if (p >= 0) {
        const u64 d = (u64)(p - x);
        const u64 c = d * d * wx2m + lp;
        row[x] = c < k ? c : k;
      }
    }
  }
}

// Last q at which the parabola of i is still <= that of u (i < u): floor((f_u - f_i + c (u^2 - i^2)) / (2 c (u - i))),
// exact in 128-bit integers and clamped to [-1, len].
__device__ __forceinline__ int sep(int i, int u, u64 fi, u64 fu, u64 c, int len) {
  const __int128 num = (__int128)fu - (__int128)fi + (__int128)c * (__int128)((long long)u * u - (long long)i * i);
  const __int128 den = (__int128)c * (__int128)(2 * (u - i));
  __int128 q = num / den;
  if (num % den != 0 && num < 0) q -= 1;
  return q < -1 ? -1 : (q > len ? len : (int)q);
}

// Later passes (axis = 1: y, axis = 0: z): out(q) = min_p in(p) + c (q - p)^2 with c = M w^2, by the lower envelope
// of parabolas in integer arithmetic (Meijster et al.).  One thread per line; the envelope (s: apex positions, t:
// first q of each apex's region) lives in global scratch laid out [k][line] so neighbouring threads touch
// neighbouring addresses.
__global__ void nid_line(const u64* in, u64* out, int axis, int sz, int sy, int sx, u64 c, int* sbuf, int* tbuf) {
  const int len = axis == 0 ? sz : sy;
  const size_t st = axis == 0 ? (size_t)sy * sx : (size_t)sx;
  const size_t lines = axis == 0 ? (size_t)sy * sx : (size_t)sz * sx;
  for (size_t l = (size_t)blockIdx.x * blockDim.x + threadIdx.x; l < lines; l += (size_t)gridDim.x * blockDim.x) {
    const size_t base = axis == 0 ? l : (l / sx) * (size_t)sy * sx + l % sx;
    int k = -1;
    for (int q = 0; q < len; ++q) {
      const u64 fq = in[base + (size_t)q * st];
      if (fq == kInf) continue;
      while (k >= 0) {
        const int sk = sbuf[(size_t)k * lines + l], tk = tbuf[(size_t)k * lines + l];
        const u64 dk = (u64)(tk > sk ? tk - sk : sk - tk), dq = (u64)(q > tk ? q - tk : tk - q);
        if (in[base + (size_t)sk * st] + c * dk * dk > fq + c * dq * dq) --k;
        else break;
      }
      if (k < 0) {
        k = 0;
        sbuf[l] = q;
        tbuf[l] = 0;
      } else {
        const int sk = sbuf[(size_t)k * lines + l];
        const int w = 1 + sep(sk, q, in[base + (size_t)sk * st], fq, c, len);
        if (w < len) {
          ++k;
          sbuf[(size_t)k * lines + l] = q;
          tbuf[(size_t)k * lines + l] = w;
        }
      }
    }
    if (k < 0) {   // no labelled voxel reaches this line
      for (int q = 0; q < len; ++q) out[base + (size_t)q * st] = kInf;
      continue;
    }
    int sk = sbuf[(size_t)k * lines + l], tk = tbuf[(size_t)k * lines + l];
    u64 fk = in[base + (size_t)sk * st];
    for (int q = len - 1; q >= 0; --q) {
      const u64 d = (u64)(q > sk ? q - sk : sk - q);
      out[base + (size_t)q * st] = fk + c * d * d;
      if (q == tk && k > 0) {
        --k;
        sk = sbuf[(size_t)k * lines + l];
        tk = tbuf[(size_t)k * lines + l];
        fk = in[base + (size_t)sk * st];
      }
    }
  }
}

// ---- pair search ------------------------------------------------------------------------------------------------

struct PairTable {
  u64* key;    // (a << 32 | b), a < b compact ids; kEmpty = free
  u64* dist;   // bits of the minimum dist (non-negative doubles order like their bits)
  u64* cnt;    // rows at the minimum dist
  u64* sum;    // [3][cap] int64 coordinate sums (x, y, z) of those rows
  u64* c2;     // bits of the minimum squared distance to their centroid
  u64* ord;    // minimum order index among the rows at that minimum
  u64 cap;     // power of two
  u64 limit;   // slots that may be claimed before the table counts as full
  u64* used;    // slots reserved
  int* overflow;
};

struct PairGeom {
  int lo[3];     // box start (z, y, x)
  int size[3];   // box extent
  int sy, sx;    // volume extents behind the box
  u64 m;         // M
  int log_m;
  int use_max_distance;
  double max_distance;
};

__device__ __forceinline__ u64 mix64(u64 x) {   // splitmix64 finaliser
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ long long table_slot(const PairTable& t, u64 pk, bool insert) {
  const u64 h = mix64(pk);
  for (u64 p = 0; p < t.cap; ++p) {
    const u64 s = (h + p) & (t.cap - 1);
    const u64 k = *(volatile u64*)&t.key[s];
    if (k == pk) return (long long)s;
    if (k == kEmpty) {
      if (!insert) return -1;
      // Reserve before claiming, so that at most `limit` slots are ever taken and probes stay short; a reservation
      // whose claim loses the race stays counted (the table may then grow once more than needed).
      if (atomicAdd(t.used, 1ull) >= t.limit) {
        *t.overflow = 1;
        return -1;
      }
      const u64 prev = atomicCAS(&t.key[s], kEmpty, pk);
      if (prev == kEmpty || prev == pk) return (long long)s;
    }
  }
  return -1;
}

// Expanded id (0 = none) and edt of a key; beyond max_distance the expansion keeps the original label.
__device__ __forceinline__ unsigned decode(u64 key, const PairGeom& g, double* edt) {
  if (key == kInf) {
    *edt = 0.0;
    return 0;
  }
  const u64 d = key >> g.log_m;
  *edt = __dsqrt_rn((double)d);
  if (d > 0 && g.use_max_distance && *edt > g.max_distance) return 0;
  return (unsigned)(key & (g.m - 1));
}

// One pass over the rows (a-voxel, offset) of the box.  Offsets in itertools.product((0,-1),(0,-1),(0,-1)) order
// are ranks r = 1..7 with (dz, dy, dx) = the bits of r; the b-voxel is the a-voxel + (dz, dy, dx).
//   1: claim the pair's slot, atomicMin of dist          2: count and coordinate sums of the rows at the minimum
//   3: atomicMin of the squared distance to the centroid  4: atomicMin of the order index among the rows still tied
template <int PASS>
__global__ void pair_pass(const u64* keys, PairGeom g, PairTable t) {
  const int bz = g.size[0], by = g.size[1], bx = g.size[2];
  const size_t n = (size_t)bz * by * bx;
  const size_t plane = (size_t)g.sy * g.sx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (PASS == 1 && *(volatile int*)t.overflow) return;   // this table is discarded anyway
    const int x = (int)(i % bx), y = (int)((i / bx) % by), z = (int)(i / ((size_t)bx * by));
    const size_t gi = (size_t)(g.lo[0] + z) * plane + (size_t)(g.lo[1] + y) * g.sx + (g.lo[2] + x);
    double ea;
    const unsigned a = decode(keys[gi], g, &ea);
    if (a == 0) continue;
#pragma unroll 1
    for (int r = 1; r < 8; ++r) {
      const int dz = (r >> 2) & 1, dy = (r >> 1) & 1, dx = r & 1;
      if (z + dz >= bz || y + dy >= by || x + dx >= bx) continue;
      double eb;
      const unsigned b = decode(keys[gi + dz * plane + (size_t)dy * g.sx + dx], g, &eb);
      if (b == 0 || b == a) continue;
      const u64 pk = a < b ? ((u64)a << 32 | b) : ((u64)b << 32 | a);
      const u64 db = (u64)__double_as_longlong(__dmul_rn(__dadd_rn(ea, eb), 0.5));
      const long long s = table_slot(t, pk, PASS == 1);
      if (s < 0) continue;
      if (PASS == 1) {
        if (*(volatile u64*)&t.dist[s] > db) atomicMin(&t.dist[s], db);
        continue;
      }
      if (t.dist[s] != db) continue;
      if (PASS == 2) {
        atomicAdd(&t.cnt[s], 1ull);
        atomicAdd(&t.sum[s], (u64)x);
        atomicAdd(&t.sum[t.cap + s], (u64)y);
        atomicAdd(&t.sum[2 * t.cap + s], (u64)z);
        continue;
      }
      const double cnt = (double)t.cnt[s];
      const double ex = __dsub_rn((double)x, __ddiv_rn((double)(long long)t.sum[s], cnt));
      const double ey = __dsub_rn((double)y, __ddiv_rn((double)(long long)t.sum[t.cap + s], cnt));
      const double ez = __dsub_rn((double)z, __ddiv_rn((double)(long long)t.sum[2 * t.cap + s], cnt));
      const u64 c2 = (u64)__double_as_longlong(
          __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)));
      if (PASS == 3) {
        if (*(volatile u64*)&t.c2[s] > c2) atomicMin(&t.c2[s], c2);
      } else if (t.c2[s] == c2) {
        atomicMin(&t.ord[s], (u64)r << kOrderShift | (u64)i);
      }
    }
  }
}

__global__ void table_init(PairTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.key[s] = kEmpty;
    t.dist[s] = ~0ull;
    t.cnt[s] = 0;
    t.sum[s] = t.sum[t.cap + s] = t.sum[2 * t.cap + s] = 0;
    t.c2[s] = ~0ull;
    t.ord[s] = ~0ull;
  }
}

// One FfnDecisionPoint per occupied slot (unordered): original ids, dist, and the box-relative point of the
// winning row in (x, y, z).
__global__ void emit_pairs(PairTable t, const u64* kept, int by, int bx, FfnDecisionPoint* out, u64* n) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < t.cap; s += (u64)gridDim.x * blockDim.x) {
    const u64 pk = t.key[s];
    if (pk == kEmpty) continue;
    const u64 j = atomicAdd(n, 1ull);
    const u64 i = t.ord[s] & ((1ull << kOrderShift) - 1);
    FfnDecisionPoint p;
    p.id_a = kept[(pk >> 32) - 1];
    p.id_b = kept[(pk & 0xffffffffull) - 1];
    p.dist = __longlong_as_double((long long)t.dist[s]);
    p.point_xyz[0] = (int64_t)(i % bx);
    p.point_xyz[1] = (int64_t)((i / bx) % by);
    p.point_xyz[2] = (int64_t)(i / ((u64)bx * by));
    out[j] = p;
  }
}

}  // namespace dpk
}  // namespace ffn
