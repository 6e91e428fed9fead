// example_kernels.cuh — the kernels of the training example loop (examples.cu): policy resumption, example loading,
// batch cropping and the seed update.  Patches, seeds and labels are float32 [element][z][y][x] of patch extent S.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ffn_b200.h"

namespace exk {

constexpr int kThreads = 256;
constexpr int kMaxWarps = 32;   // the resume kernel runs one warp per element, in one CTA

// One element's generator state.  `off` is the offset of the last yield; fixed resumes at shift k (0: the centre),
// max_pred_moves pops queue[head .. tail) after extending it from the seed at `off`.
struct State {
  int off[3];
  int k, head, tail;
  int active;         // 0 until the first example is loaded
  int pad_;
  long long example;  // index of the element's example in the stream since creation
};

struct Vol {
  const uint8_t* image;
  const long long* labels;
  int ishape[3], lshape[3];
  float offset, scale;
};

struct Args {
  int S[3], F[3], D[3];
  int moves, policy, batch;
  long long SV, FV;                 // voxels of a patch, of a field of view
  int qcap, side;                   // queue entries per element; done cells per axis (2 * moves + 1)
  float pad_logit, centre_logit;
  double seed_thr, label_thr;
  float *seed, *image, *labels;     // [batch][S]
  State* st;
  int* queue;                       // [batch][qcap][3]
  unsigned char* done;              // [batch][side^3]
  const int* shifts;                // [n_shifts][3]
  int n_shifts;
  const Vol* vols;
  const FfnExampleCoord* coords;
  int* used;                        // stream entries taken since the last upload
  int* entry;                       // [batch]: the entry an element loads this step, or -1
  long long* total;                 // examples loaded since creation
  int* error;                       // set when a queue would overflow its bound (never, by construction)
};

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

__device__ __forceinline__ long long at(const Args& a, int z, int y, int x) {
  return ((long long)z * a.S[1] + y) * a.S[2] + x;
}

// numpy's argmax order: the larger value, NaN above every number, the first index among equals.
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

// sorted(..., reverse=True) of (score, (z, y, x)) tuples: the larger score first, then the larger offset tuple.
__device__ __forceinline__ bool before(float s, const int* p, float t, const int* q) {
  if (s != t) return s > t;
  for (int k = 0; k < 3; ++k)
    if (p[k] != q[k]) return p[k] > q[k];
  return false;
}

// Fixed policy (examples.fixed_offsets): the centre, then the shifts in order, each yielded when the seed at it
// passes the threshold.  Returns 1 when exhausted.  One thread.
__device__ int resume_fixed(const Args& a, State& s, const float* seed) {
  const int c[3] = {a.S[0] / 2, a.S[1] / 2, a.S[2] / 2};
  for (int k = s.k; k <= a.n_shifts; ++k) {
    int o[3] = {0, 0, 0};
    if (k > 0)
      for (int d = 0; d < 3; ++d) o[d] = a.shifts[(k - 1) * 3 + d];
    if ((double)seed[at(a, c[0] + o[0], c[1] + o[1], c[2] + o[2])] >= a.seed_thr) {
      for (int d = 0; d < 3; ++d) s.off[d] = o[d];
      s.k = k + 1;
      return 0;
    }
  }
  s.k = a.n_shifts + 1;
  return 1;
}

// max_pred_moves (examples.max_pred_offsets): extend the queue with movement.get_scored_move_offsets of the seed at
// the last yield, sorted in reverse, then pop until an offset inside max_radius, in an unvisited quantised cell,
// valid, and wanted unless it is the centre.  One warp; returns 1 (to every lane) when exhausted.
__device__ int resume_max_pred(const Args& a, State& s, int e, const float* seed, const float* labels, int lane) {
  const int c[3] = {a.S[0] / 2, a.S[1] / 2, a.S[2] / 2};
  int* q = a.queue + (size_t)e * a.qcap * 3;
  float cs[6];
  int cp[6][3];
  int nc = 0;
  for (int ax = 0; ax < 3; ++ax) {
    if (a.D[ax] == 0) continue;
    const int b0 = ax == 0 ? 1 : 0, b1 = ax == 2 ? 1 : 2;   // the face's axes, in C order
    const int n0 = 2 * a.D[b0] + 1, n1 = 2 * a.D[b1] + 1;
    for (int sg = -1; sg <= 1; sg += 2) {
      float bv = 0.f;
      int bi = -1;
      for (int i = lane; i < n0 * n1; i += 32) {
        int p[3];
        p[ax] = sg * a.D[ax];
        p[b0] = i / n1 - a.D[b0];
        p[b1] = i % n1 - a.D[b1];
        const float v = seed[at(a, c[0] + s.off[0] + p[0], c[1] + s.off[1] + p[1], c[2] + s.off[2] + p[2])];
        if (bi < 0 || better(v, i, bv, bi)) bv = v, bi = i;
      }
      for (int m = 16; m; m >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, m);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, m);
        if (oi >= 0 && (bi < 0 || better(ov, oi, bv, bi))) bv = ov, bi = oi;
      }
      if (lane == 0 && !((double)bv < a.seed_thr)) {
        int p[3];
        p[ax] = sg * a.D[ax];
        p[b0] = bi / n1 - a.D[b0];
        p[b1] = bi % n1 - a.D[b1];
        bool dup = false;   // a voxel on an edge can be the maximum of two faces: get_scored_move_offsets' `done`
        for (int j = 0; j < nc; ++j) dup |= cp[j][0] == p[0] && cp[j][1] == p[1] && cp[j][2] == p[2];
        if (!dup) {
          int j = nc++;
          for (; j > 0 && before(bv, p, cs[j - 1], cp[j - 1]); --j) {
            cs[j] = cs[j - 1];
            for (int d = 0; d < 3; ++d) cp[j][d] = cp[j - 1][d];
          }
          cs[j] = bv;
          for (int d = 0; d < 3; ++d) cp[j][d] = p[d];
        }
      }
    }
  }
  int exhausted = 1;
  if (lane == 0) {
    if (s.tail + nc > a.qcap) {
      atomicExch(a.error, 1);
      nc = 0;
    }
    for (int j = 0; j < nc; ++j)
      for (int d = 0; d < 3; ++d) q[(s.tail + j) * 3 + d] = s.off[d] + cp[j][d];
    s.tail += nc;
    while (s.head < s.tail) {
      const int* o = q + s.head++ * 3;
      bool inside = true;
      for (int d = 0; d < 3; ++d) inside &= abs(o[d]) <= a.D[d] * a.moves;
      if (!inside) continue;
      int cell = 0;
      bool centre = true;
      for (int d = 0; d < 3; ++d) {
        const int qd = floor_div(2 * o[d] + a.D[d], 2 * max(a.D[d], 1));
        centre &= qd == 0;
        cell = cell * a.side + qd + a.moves;
      }
      unsigned char* done = a.done + (size_t)e * a.side * a.side * a.side + cell;
      if (*done) continue;
      const long long v = at(a, c[0] + o[0], c[1] + o[1], c[2] + o[2]);
      const bool valid = (double)seed[v] >= a.seed_thr;
      const bool wanted = (double)labels[v] >= a.label_thr;
      if (!valid || (!wanted && !centre)) continue;
      *done = 1;
      for (int d = 0; d < 3; ++d) s.off[d] = o[d];
      exhausted = 0;
      break;
    }
  }
  return __shfl_sync(0xffffffffu, exhausted, 0);
}

// Resumes every element's generator (one warp each), then hands the next stream entries to the exhausted elements
// in element order.
__global__ void __launch_bounds__(kMaxWarps * 32) resume(Args a) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, nw = blockDim.x / 32;
  for (int e = warp; e < a.batch; e += nw) {
    State& s = a.st[e];
    int need = 1;
    if (s.active) {
      const float* seed = a.seed + e * a.SV;
      if (a.policy == FFN_FOV_FIXED) {
        if (lane == 0) need = resume_fixed(a, s, seed);
      } else {
        need = resume_max_pred(a, s, e, seed, a.labels + e * a.SV, lane);
      }
    }
    if (lane == 0) a.entry[e] = need ? 0 : -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int e = 0; e < a.batch; ++e) {
      if (a.entry[e] < 0) continue;
      a.entry[e] = (*a.used)++;
      a.st[e].example = (*a.total)++;
    }
  }
}

// Loads the examples handed out by `resume` (inputs.load_from_numpylike, the object mask of the centre label,
// soften_labels, PermuteAndReflect, offset_and_scale_patches) and starts their generators at the centre, which a
// fresh seed always passes.  grid (blocks, batch).
__global__ void __launch_bounds__(kThreads) load(Args a) {
  const int e = blockIdx.y;
  const int j = a.entry[e];
  if (j < 0) return;
  const FfnExampleCoord cd = a.coords[j];
  const Vol vol = a.vols[cd.volume];
  int start[3];
  for (int d = 0; d < 3; ++d) start[d] = cd.center_xyz[2 - d] - (a.S[d] - 1) / 2;
  if (blockIdx.x == 0) {
    const int cells = a.side * a.side * a.side;
    unsigned char* done = a.done + (size_t)e * cells;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) done[i] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
      State& s = a.st[e];
      s.off[0] = s.off[1] = s.off[2] = 0;
      s.k = 1;
      s.head = s.tail = 0;
      s.active = 1;
      done[(a.moves * a.side + a.moves) * a.side + a.moves] = 1;
    }
  }
  auto lab_at = [&](int z, int y, int x) {
    return vol.labels[((long long)z * vol.lshape[1] + y) * vol.lshape[2] + x];
  };
  const long long centre = lab_at(start[0] + a.S[0] / 2, start[1] + a.S[1] / 2, start[2] + a.S[2] / 2);
  float* seed = a.seed + e * a.SV;
  float* image = a.image + e * a.SV;
  float* labels = a.labels + e * a.SV;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < a.SV; v += (long long)gridDim.x * blockDim.x) {
    int o[3];
    o[2] = (int)(v % a.S[2]);
    o[1] = (int)(v / a.S[2] % a.S[1]);
    o[0] = (int)(v / ((long long)a.S[2] * a.S[1]));
    int src[3];
    for (int d = 0; d < 3; ++d) src[cd.permutation_zyx[d]] = cd.reflect_zyx[d] ? a.S[d] - 1 - o[d] : o[d];
    for (int d = 0; d < 3; ++d) src[d] += start[d];
    const long long l = lab_at(src[0], src[1], src[2]);
    labels[v] = l > 0 && l == centre ? 0.95f : 0.05f;
    const uint8_t u = vol.image[((long long)src[0] * vol.ishape[1] + src[1]) * vol.ishape[2] + src[2]];
    image[v] = __fdiv_rn(__fsub_rn((float)u, vol.offset), vol.scale);
    seed[v] = o[0] == a.S[0] / 2 && o[1] == a.S[1] / 2 && o[2] == a.S[2] / 2 ? a.centre_logit : a.pad_logit;
  }
}

// The field of view of every element at its offset: mask.crop_and_pad of seed, image and labels into [batch][F].
// grid (blocks, batch).
__global__ void __launch_bounds__(kThreads) crop(Args a, float* seed_out, float* image_out, float* labels_out) {
  const int e = blockIdx.y;
  const State& s = a.st[e];
  int base[3];
  for (int d = 0; d < 3; ++d) base[d] = a.S[d] / 2 - a.F[d] / 2 + s.off[d];
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < a.FV; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % a.F[2]), y = (int)(v / a.F[2] % a.F[1]), z = (int)(v / ((long long)a.F[2] * a.F[1]));
    const long long src = e * a.SV + at(a, base[0] + z, base[1] + y, base[2] + x);
    const long long dst = e * a.FV + v;
    seed_out[dst] = a.seed[src];
    image_out[dst] = a.image[src];
    labels_out[dst] = a.labels[src];
  }
}

// BatchExampleIter.update_seeds: the logits [batch][F] into each seed at its offset.  grid (blocks, batch).
__global__ void __launch_bounds__(kThreads) paste(Args a, const float* logits) {
  const int e = blockIdx.y;
  const State& s = a.st[e];
  int base[3];
  for (int d = 0; d < 3; ++d) base[d] = a.S[d] / 2 - a.F[d] / 2 + s.off[d];
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < a.FV; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % a.F[2]), y = (int)(v / a.F[2] % a.F[1]), z = (int)(v / ((long long)a.F[2] * a.F[1]));
    a.seed[e * a.SV + at(a, base[0] + z, base[1] + y, base[2] + x)] = logits[e * a.FV + v];
  }
}

}  // namespace exk
