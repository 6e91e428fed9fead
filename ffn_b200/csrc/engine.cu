// engine.cu — host side of libffn_b200.so: device context, weight packing, canvases, launches,
// and the extern "C" entry points declared in include/ffn_b200.h.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "device_types.cuh"
// the persistent kernel, twice: the product build and one with device cycle counters
#define FFN_KNS plain
#define FFN_PROFILE 0
#include "flood_kernel.cuh"
#undef FFN_KNS
#undef FFN_PROFILE
#define FFN_KNS profiled
#define FFN_PROFILE 1
#include "flood_kernel.cuh"
#undef FFN_KNS
#undef FFN_PROFILE
#include "seed_kernels.cuh"
#include "selftest.cuh"

namespace {

thread_local std::string g_error;

int fail(const std::string& msg) {
  g_error = msg;
  return 1;
}

#define CUDA_OK(expr)                                                                          \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" + \
                  std::to_string(__LINE__) + ")");                                             \
  } while (0)

template <typename T>
int dev_alloc(T** p, size_t n, bool zero = true) {
  CUDA_OK(cudaMalloc(reinterpret_cast<void**>(p), std::max<size_t>(n, 1) * sizeof(T)));
  if (zero) CUDA_OK(cudaMemset(*p, 0, std::max<size_t>(n, 1) * sizeof(T)));
  return 0;
}

}  // namespace

struct FfnEngine {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int sm_count = 0;
  int grid = 0;
  int smem_bytes = 0;
  int compute_mode = FFN_COMPUTE_FP16_TC;
  ffn::Geom g{};
  ffn::Weights w{};
  ffn::Workspace ws{};
  ffn::ChainDev cws[ffn::kMaxChains]{};   // per-chain step workspace (canvas-side pointers stay null here)
  CUtensorMap tmap[ffn::kMaxChains][3]{};
  int use_tmap = 0;
  int max_chains = ffn::kMaxChains;       // chains the multi-seed / batched paths may use (ffn_engine_set_chains)
  ffn::Ctl* d_ctl = nullptr;
  unsigned* d_round_flag = nullptr;
  ffn::CanvasState* d_dummy_state = nullptr;   // [kMaxBufs]
  ffn::Sched* d_dummy_sched = nullptr;
  // predict staging
  float* d_in_seed = nullptr;
  float* d_in_image = nullptr;
  float* d_out = nullptr;
  int predict_cap = 0;
  std::vector<void*> owned;
  double last_kernel_seconds = 0.0;
  bool profiling = false;
  long long launches = 0;
  // Lifetime: canvases hold a raw pointer to their engine.  ffn_engine_destroy with canvases still alive
  // only marks the engine as closing — it stays fully usable through those canvases (reading results after
  // Runner.stop_executor() is the common case) — and the last ffn_canvas_destroy releases it.
  int live_canvases = 0;
  bool closing = false;
};

struct FfnCanvas {
  FfnEngine* eng = nullptr;
  ffn::CanvasDev cv{};
  ffn::ObjDev ob[ffn::kMaxBufs]{};        // object buffers; [0] holds the canvas's own seed array
  int nbufs_alloc = 1;
  float* d_snap = nullptr;                // snapshot seed array (Sched::last_chain), allocated with the extra chains
  std::vector<void*> pools;               // allocations behind object buffers 1.. and the snapshot array
  ffn::CanvasState* d_state = nullptr;    // [kMaxBufs]
  ffn::CanvasState h_state{};             // buffer 0
  ffn::Sched* d_sched = nullptr;
  ffn::Sched h_sched{};
  size_t q_cap = 0, traj_cap = 0;
  long long last_spec[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // last segment_all: early runs started / discarded / their steps / steps executed
  void* d_image = nullptr;
  uint8_t* d_mask = nullptr;
  uint8_t* d_seed_mask = nullptr;
  float* d_pred = nullptr;
  size_t nvox = 0;
  size_t lattice_cells = 0;
  bool resume_pending = false;
};

namespace {

using namespace ffn;

int set_device(const FfnEngine* e) {
  CUDA_OK(cudaSetDevice(e->device));
  return 0;
}

void engine_free(FfnEngine* e) {
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (void* p : e->owned) cudaFree(p);
  cudaFree(e->d_in_seed);
  cudaFree(e->d_in_image);
  cudaFree(e->d_out);
  cudaEventDestroy(e->ev0);
  cudaEventDestroy(e->ev1);
  delete e;
}

Geom make_geom(const FfnModelDesc& m) {
  Geom g{};
  g.fz = m.fov_zyx[0];
  g.fy = m.fov_zyx[1];
  g.fx = m.fov_zyx[2];
  g.mz = g.fz / 2;
  g.my = g.fy / 2;
  g.mx = g.fx / 2;
  g.dz = m.deltas_zyx[0];
  g.dy = m.deltas_zyx[1];
  g.dx = m.deltas_zyx[2];
  g.nconv = 2 * m.depth;
  g.xp = g.fx;                  // no pad column: the dx taps are resolved in the epilogue / by masking
  g.pp = (g.fy + 1) * g.xp;     // one zero line after every z-plane supplies the dy halo
  g.nr = (g.fz - 1) * g.pp + (g.fy - 1) * g.xp + g.fx;
  g.nt = (g.nr + kTileOut - 1) / kTileOut;
  g.halo = g.xp + 1;
  g.guard = ((g.pp + g.halo + 7) / 8) * 8;
  g.rows_alloc = g.guard + g.nt * kTileM + g.guard;
  g.rows_alloc = ((g.rows_alloc + g.pp - 1) / g.pp) * g.pp;   // k-chunk pitch = whole number of z-plane pitches (tensor-map strides)
  g.V = g.fz * g.fy * g.fx;
  g.inv_pp = 1.0f / (float)g.pp;
  g.inv_xp = 1.0f / (float)g.xp;
  return g;
}

// How many chains a launch may use.
int chain_limit(const FfnEngine* e) { return std::max(1, std::min(e->max_chains, (int)kMaxChains)); }

// Launches the persistent kernel once and waits for it.  `c` may be null (predict).
int launch(FfnEngine* e, FfnCanvas* c, int nchains, const Job& job) {
  KParams p{};
  p.g = e->g;
  p.w = e->w;
  p.ws = e->ws;
  if (!e->profiling) p.ws.prof = nullptr;
  if (c) p.cv = c->cv;
  p.nchains = nchains;
  for (int k = 0; k < kMaxChains; ++k) p.ch[k] = e->cws[k];
  for (int b = 0; b < kMaxBufs; ++b) {
    if (c && b < c->nbufs_alloc) p.ob[b] = c->ob[b];
    p.ob[b].st = c ? c->d_state + b : e->d_dummy_state + b;
  }
  p.sched = c ? c->d_sched : e->d_dummy_sched;
  p.ctl = e->d_ctl;
  p.round_flag = e->d_round_flag;
  p.snap = c ? c->d_snap : nullptr;
  std::memcpy(p.tmap, e->tmap, sizeof(p.tmap));
  p.use_tmap = e->use_tmap;
  p.job = job;
  {
    const char* env = std::getenv("FFN_B200_WATCHDOG_S");
    const long long secs = env ? std::atoll(env) : 60;
    p.job.watchdog_ns = (secs > 0 ? secs : 60) * 1000000000ll;
  }
  p.compute_mode = e->compute_mode;
  CUDA_OK(cudaMemsetAsync(e->ws.bar, 0, sizeof(unsigned), cudaStreamPerThread));
  CUDA_OK(cudaMemsetAsync(e->ws.abort_flag, 0, sizeof(int), cudaStreamPerThread));
  CUDA_OK(cudaMemsetAsync(e->d_ctl, 0, sizeof(Ctl), cudaStreamPerThread));
  CUDA_OK(cudaMemsetAsync(e->d_round_flag, 0, sizeof(unsigned), cudaStreamPerThread));
  for (int k = 0; k < kMaxChains; ++k) CUDA_OK(cudaMemsetAsync(e->cws[k].bar, 0, sizeof(unsigned), cudaStreamPerThread));
  void* args[] = {&p};
  CUDA_OK(cudaEventRecord(e->ev0, cudaStreamPerThread));
  CUDA_OK(cudaLaunchCooperativeKernel(e->profiling ? reinterpret_cast<const void*>(profiled::ffn_flood_kernel)
                                                   : reinterpret_cast<const void*>(plain::ffn_flood_kernel), dim3(e->grid),
                                      dim3(kThreads), args, (size_t)e->smem_bytes, cudaStreamPerThread));
  CUDA_OK(cudaEventRecord(e->ev1, cudaStreamPerThread));
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  float ms = 0.f;
  CUDA_OK(cudaEventElapsedTime(&ms, e->ev0, e->ev1));
  e->last_kernel_seconds = ms * 1e-3;
  e->launches++;
  int abort_flag = 0;
  CUDA_OK(cudaMemcpy(&abort_flag, e->ws.abort_flag, sizeof(int), cudaMemcpyDeviceToHost));
  if (abort_flag != 0)
    return fail("device-side wait timed out (abort code " + std::to_string(abort_flag) +
                "): 1 = grid barrier, 2 = mbarrier, 3 = chain barrier, 4 = round flag, 5 = launch exceeded 60 s");
  return 0;
}

int pull_state(FfnCanvas* c) {   // chain 0: the canvas's own flood-fill state
  CUDA_OK(cudaMemcpy(&c->h_state, c->d_state, sizeof(CanvasState), cudaMemcpyDeviceToHost));
  return 0;
}
int push_state(FfnCanvas* c) {
  CUDA_OK(cudaMemcpy(c->d_state, &c->h_state, sizeof(CanvasState), cudaMemcpyHostToDevice));
  return 0;
}

// Seed array, queue, done lattice and trajectory log of one object buffer (buffer 0's seed array is the canvas's own).
int alloc_buf(FfnCanvas* c, int k) {
  ObjDev& ch = c->ob[k];
  if (k > 0) {
    if (dev_alloc(&ch.seed, c->nvox, false)) return 1;
    fill_f32_kernel<<<c->eng->sm_count * 8, 256, 0, cudaStreamPerThread>>>(ch.seed, c->nvox, NAN);
    CUDA_OK(cudaGetLastError());
  }
  if (dev_alloc(&ch.lattice, c->lattice_cells)) return 1;
  if (dev_alloc(&ch.q_score, c->q_cap, false)) return 1;
  if (dev_alloc(&ch.q_pos, c->q_cap * 3, false)) return 1;
  if (dev_alloc(&ch.traj, c->traj_cap * 3, false)) return 1;
  return 0;
}

// Object buffers 1 .. n-1 and the snapshot array, on first use: ONE allocation for the seed arrays and one for the
// small per-object arrays (two dozen separate cudaMalloc calls of 60 MB took 6 - 100 ms of a 2 s segment_all).
int ensure_bufs(FfnCanvas* c, int n) {
  const int first = c->nbufs_alloc;
  const bool need_snap = n > 1 && !c->d_snap;
  if (first >= n && !need_snap) return 0;
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  const int nnew = std::max(n - first, 0);
  const size_t seed_b = up(c->nvox * sizeof(float));
  const size_t lat_b = up(c->lattice_cells * sizeof(*c->ob[0].lattice)), qs_b = up(c->q_cap * sizeof(*c->ob[0].q_score)),
               qp_b = up(c->q_cap * 3 * sizeof(*c->ob[0].q_pos)), tr_b = up(c->traj_cap * 3 * sizeof(*c->ob[0].traj));
  const size_t small_b = lat_b + qs_b + qp_b + tr_b;
  unsigned char *big = nullptr, *small = nullptr;
  const size_t big_total = seed_b * (size_t)(nnew + (need_snap ? 1 : 0));
  if (big_total) {
    CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&big), big_total));
    c->pools.push_back(big);
    fill_f32_kernel<<<c->eng->sm_count * 8, 256, 0, cudaStreamPerThread>>>(reinterpret_cast<float*>(big), big_total / sizeof(float), NAN);
    CUDA_OK(cudaGetLastError());
  }
  if (nnew) {
    CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&small), small_b * (size_t)nnew));
    c->pools.push_back(small);
    CUDA_OK(cudaMemsetAsync(small, 0, small_b * (size_t)nnew, cudaStreamPerThread));
  }
  for (int i = 0; i < nnew; ++i) {
    ObjDev& ob = c->ob[first + i];
    ob.seed = reinterpret_cast<float*>(big + seed_b * (size_t)i);
    unsigned char* q = small + small_b * (size_t)i;
    ob.lattice = reinterpret_cast<decltype(ob.lattice)>(q);
    ob.q_score = reinterpret_cast<decltype(ob.q_score)>(q + lat_b);
    ob.q_pos = reinterpret_cast<decltype(ob.q_pos)>(q + lat_b + qs_b);
    ob.traj = reinterpret_cast<decltype(ob.traj)>(q + lat_b + qs_b + qp_b);
  }
  c->nbufs_alloc = std::max(first, n);
  if (need_snap) {
    c->d_snap = reinterpret_cast<float*>(big + seed_b * (size_t)nnew);
    for (int q = 0; q < 3; ++q) c->h_sched.snap_lo[q] = c->h_sched.snap_hi[q] = 0;
  }
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

int fill_box(FfnCanvas* c, float* arr, const int lo[3], const int hi[3]) {
  const int l[3] = {std::max(lo[0], 0), std::max(lo[1], 0), std::max(lo[2], 0)};
  const int n[3] = {std::min(hi[0], c->cv.sz) - l[0], std::min(hi[1], c->cv.sy) - l[1], std::min(hi[2], c->cv.sx) - l[2]};
  if (n[0] <= 0 || n[1] <= 0 || n[2] <= 0) return 0;
  fill_box_f32_kernel<<<c->eng->sm_count * 4, 256, 0, cudaStreamPerThread>>>(arr, c->cv.sy, c->cv.sx, l[0], l[1], l[2], n[0],
                                                                          n[1], n[2], NAN);
  CUDA_OK(cudaGetLastError());
  return 0;
}

void pack_weights(const Geom& g, const float* const* w, std::vector<__half>& w16, std::vector<__half>& w16x2,
                  std::vector<float>& w32) {
  const int nconv = g.nconv;
  w16.assign(w16_layer_offset_halfs(nconv), __float2half(0.f));
  w16x2.assign(2 * w16_layer_offset_halfs(nconv), __float2half(0.f));
  w32.assign(w32_layer_offset_floats(nconv), 0.f);
  for (int l = 0; l < nconv; ++l) {
    const int cin = l == 0 ? 2 : 32;
    const int nch = l == 0 ? 2 : 4;
    const int cin_pad = l == 0 ? 4 : 32;
    __half* d16 = w16.data() + w16_layer_offset_halfs(l);
    __half* d16hi = w16x2.data() + 2 * w16_layer_offset_halfs(l);
    __half* d16lo = d16hi + (w16_layer_offset_halfs(l + 1) - w16_layer_offset_halfs(l));
    float* d32 = w32.data() + w32_layer_offset_floats(l);
    for (int tap = 0; tap < 27; ++tap)
      for (int ci = 0; ci < cin; ++ci)
        for (int co = 0; co < 32; ++co) {
          const float v = w[l][((size_t)tap * cin + ci) * 32 + co];   // DHWIO: tap = kz*9 + ky*3 + kx
          {
            const int row = tap / 3, n = (tap % 3) * 32 + co;   // tap-row (kz, ky); n stacks kx
            const size_t at = (((size_t)row * nch + ci / 8) * 12 + n / 8) * 64 + (n % 8) * 8 + (ci % 8);
            d16[at] = __float2half_rn(v);
            // split mode: w * 2^kSplitShift = hi + lo (the scaling is exact and keeps lo out of the fp16
            // subnormal range; the epilogue multiplies the accumulators by 2^-kSplitShift)
            const float vs = v * (float)(1 << kSplitShift);
            const __half h = __float2half_rn(vs);
            d16hi[at] = h;
            d16lo[at] = __float2half_rn(vs - __half2float(h));
          }
          d32[((size_t)tap * cin_pad + ci) * 32 + co] = v;
        }
  }
}

int box_copy(FfnCanvas* c, int which, const int32_t lo[3], const int32_t sz[3], void* host, bool to_host) {
  const CanvasDev& cv = c->cv;
  for (int k = 0; k < 3; ++k) {
    const int dim = k == 0 ? cv.sz : k == 1 ? cv.sy : cv.sx;
    if (lo[k] < 0 || sz[k] <= 0 || lo[k] + sz[k] > dim) return fail("box out of canvas bounds");
  }
  size_t esz = 0;
  char* base = nullptr;
  switch (which) {
    case FFN_ARRAY_SEED: esz = 4; base = reinterpret_cast<char*>(c->ob[0].seed); break;
    case FFN_ARRAY_SEGMENTATION: esz = 4; base = reinterpret_cast<char*>(cv.seg); break;
    case FFN_ARRAY_QPROB:
      if (!cv.qprob) return fail("canvas was created without probability maps");
      esz = 1; base = reinterpret_cast<char*>(cv.qprob); break;
    default: return fail("unknown array id");
  }
  cudaMemcpy3DParms prm{};
  cudaPitchedPtr dev = make_cudaPitchedPtr(base, (size_t)cv.sx * esz, (size_t)cv.sx * esz, cv.sy);
  cudaPitchedPtr hst = make_cudaPitchedPtr(host, (size_t)sz[2] * esz, (size_t)sz[2] * esz, sz[1]);
  prm.extent = make_cudaExtent((size_t)sz[2] * esz, sz[1], sz[0]);
  if (to_host) {
    prm.srcPtr = dev;
    prm.srcPos = make_cudaPos((size_t)lo[2] * esz, lo[1], lo[0]);
    prm.dstPtr = hst;
    prm.kind = cudaMemcpyDeviceToHost;
  } else {
    prm.dstPtr = dev;
    prm.dstPos = make_cudaPos((size_t)lo[2] * esz, lo[1], lo[0]);
    prm.srcPtr = hst;
    prm.kind = cudaMemcpyHostToDevice;
  }
  CUDA_OK(cudaMemcpy3D(&prm));
  return 0;
}

}  // namespace

extern "C" {

const char* ffn_last_error(void) { return g_error.c_str(); }

int ffn_engine_create(int device, const FfnModelDesc* model, const float* const* weights_dhwio,
                      const float* const* biases, int compute_mode, FfnEngine** out) {
  if (!model || !weights_dhwio || !biases || !out) return fail("null argument");
  if (model->features != kFeat) return fail("only 32 feature maps are supported");
  if (model->depth < 1 || 2 * model->depth > kMaxConv) return fail("unsupported depth");
  for (int k = 0; k < 3; ++k) {
    if (model->fov_zyx[k] < 3 || model->fov_zyx[k] % 2 == 0) return fail("fov sizes must be odd and >= 3");
    if (model->deltas_zyx[k] < 0 || model->deltas_zyx[k] > model->fov_zyx[k] / 2)
      return fail("deltas must lie in [0, fov // 2]");
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: libffn_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail("bad device index");
  cudaDeviceProp prop{};
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(std::string("device is sm_") + std::to_string(prop.major) + std::to_string(prop.minor) +
                "; this library only contains sm_90a code");
  std::unique_ptr<FfnEngine> e(new FfnEngine());
  e->device = device;
  CUDA_OK(cudaSetDevice(device));
  // Built with --default-stream per-thread: every copy / memset / launch of a host thread goes to that
  // thread's own stream, so engines driven from different host threads run concurrently (SM-partitioned
  // cooperative grids, see ffn_engine_set_grid) while each thread's operations stay ordered.

  CUDA_OK(cudaEventCreate(&e->ev0));
  CUDA_OK(cudaEventCreate(&e->ev1));
  e->sm_count = prop.multiProcessorCount;
  e->compute_mode = compute_mode;
  e->g = make_geom(*model);
  const Geom& g = e->g;
  for (int r = 0; r < g.nt * kTileM; ++r) {   // the device decodes rows with two float multiplies: prove it exact
    const int z = (int)(((float)r + 0.5f) * g.inv_pp);
    const int rem = r - z * g.pp;
    const int y = (int)(((float)rem + 0.5f) * g.inv_xp);
    if (z != r / g.pp || y != rem / g.xp) return fail("float row decode is not exact for this field of view");
  }
  const SmemLayout L = smem_layout(g);
  e->smem_bytes = L.total;
  if ((size_t)L.total > prop.sharedMemPerBlockOptin)
    return fail("field of view too large for the shared-memory operand staging");
  CUDA_OK(cudaFuncSetAttribute(plain::ffn_flood_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  CUDA_OK(cudaFuncSetAttribute(profiled::ffn_flood_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  int per_sm = 0;
  CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, plain::ffn_flood_kernel, kThreads, L.total));
  if (per_sm < 1) return fail("persistent kernel does not fit on an SM");
  e->grid = std::min(e->sm_count, g.nt);
  if ((g.nt + e->grid - 1) / e->grid > kMaxTilesPerCta)
    return fail("field of view needs more than " + std::to_string(kMaxTilesPerCta) + " tiles per SM");

  // weights
  std::vector<__half> w16, w16x2;
  std::vector<float> w32;
  pack_weights(g, weights_dhwio, w16, w16x2, w32);
  __half* d_w16 = nullptr;
  __half* d_w16x2 = nullptr;
  if (dev_alloc(&d_w16x2, w16x2.size())) return 1;
  CUDA_OK(cudaMemcpy(d_w16x2, w16x2.data(), w16x2.size() * sizeof(__half), cudaMemcpyHostToDevice));
  e->w.w16x2 = d_w16x2;
  float *d_w32 = nullptr, *d_bias = nullptr, *d_wlom = nullptr;
  if (dev_alloc(&d_w16, w16.size())) return 1;
  if (dev_alloc(&d_w32, w32.size())) return 1;
  if (dev_alloc(&d_bias, (size_t)g.nconv * 32)) return 1;
  if (dev_alloc(&d_wlom, 32)) return 1;
  CUDA_OK(cudaMemcpy(d_w16, w16.data(), w16.size() * sizeof(__half), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(d_w32, w32.data(), w32.size() * sizeof(float), cudaMemcpyHostToDevice));
  std::vector<float> hb((size_t)g.nconv * 32);
  for (int l = 0; l < g.nconv; ++l) std::memcpy(&hb[(size_t)l * 32], biases[l], 32 * sizeof(float));
  CUDA_OK(cudaMemcpy(d_bias, hb.data(), hb.size() * sizeof(float), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(d_wlom, weights_dhwio[g.nconv], 32 * sizeof(float), cudaMemcpyHostToDevice));
  e->w.w16 = d_w16;
  e->w.w32 = d_w32;
  e->w.bias = d_bias;
  e->w.w_lom = d_wlom;
  e->w.b_lom = biases[g.nconv][0];
  e->owned = {d_w16, d_w16x2, d_w32, d_bias, d_wlom};

  // workspace (all buffers zero-initialised: pad rows / guards must stay zero forever)
  Workspace& ws = e->ws;
  const size_t ra = (size_t)g.rows_alloc;
  if (dev_alloc(&ws.act0_l, 2 * ra * 8)) return 1;
  if (dev_alloc(&ws.act_l[0], 4 * ra * 8)) return 1;
  if (dev_alloc(&ws.act_l[1], 4 * ra * 8)) return 1;
  if (dev_alloc(&ws.act0_f, ra)) return 1;
  if (dev_alloc(&ws.act_f[0], 8 * ra)) return 1;
  if (dev_alloc(&ws.act_f[1], 8 * ra)) return 1;
  if (dev_alloc(&ws.res, 8 * ra)) return 1;
  if (dev_alloc(&ws.bar, 1)) return 1;
  if (dev_alloc(&ws.abort_flag, 1)) return 1;
  if (dev_alloc(&ws.prof, 32 + kTraceEvents * kTraceTiles)) return 1;
  for (void* p : std::vector<void*>{ws.act0_l, ws.act_l[0], ws.act_l[1], ws.act0_f, ws.act_f[0], ws.act_f[1], ws.res,
                                    ws.bar, ws.abort_flag, ws.prof})
    e->owned.push_back(p);
  for (int k = 0; k < kMaxChains; ++k) {   // per-chain step workspace: fp16 operands, raw seed, logits, counters, barrier,
    ChainDev& cw = e->cws[k];              // fp32 residual stream
    if (dev_alloc(&cw.act0_h, 2 * ra * 8)) return 1;
    if (dev_alloc(&cw.act_h[0], 4 * ra * 8)) return 1;
    if (dev_alloc(&cw.act_h[1], 4 * ra * 8)) return 1;
    if (dev_alloc(&cw.seed_raw[0], (size_t)g.nt * kTileM)) return 1;
    if (dev_alloc(&cw.seed_raw[1], (size_t)g.nt * kTileM)) return 1;
    if (dev_alloc(&cw.logits, (size_t)g.nt * kTileM)) return 1;
    if (dev_alloc(&cw.count, 4)) return 1;
    if (dev_alloc(&cw.bar, 1)) return 1;
    if (dev_alloc(&cw.res, (size_t)g.nt * kTileM * kFeat)) return 1;
    for (void* p : std::vector<void*>{cw.act0_h, cw.act_h[0], cw.act_h[1], cw.seed_raw[0], cw.seed_raw[1], cw.logits,
                                      cw.count, cw.bar, cw.res})
      e->owned.push_back(p);
  }
  // Tensor maps for the tile loads (driver entry point fetched at run time: no link-time dependency on libcuda).
  {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn &&
              qres == cudaDriverEntryPointSuccess;
    const int seg_rows = kTileOut + 2 * g.halo;
    for (int k = 0; ok && k < kMaxChains; ++k)
      for (int i = 0; ok && i < 3; ++i) {
        const cuuint32_t nch = i == 0 ? 2 : 4;
        void* base = i == 0 ? (void*)e->cws[k].act0_h : (void*)e->cws[k].act_h[i - 1];
        const cuuint64_t dims[4] = {8, (cuuint64_t)(g.rows_alloc - 2 * g.pp), 3, nch};
        const cuuint64_t strides[3] = {16, (cuuint64_t)g.pp * 16, (cuuint64_t)g.rows_alloc * 16};
        const cuuint32_t box[4] = {8, (cuuint32_t)seg_rows, 3, nch};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        ok = reinterpret_cast<EncodeFn>(fn)(&e->tmap[k][i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
      }
    // The tiled copy moves this layout as 16-byte rows (the k-chunk is the innermost extent), so the twelve 1-D
    // bulk copies per tile are the default; FFN_B200_TMAP=1 selects the tensor-map path.
    const char* env = std::getenv("FFN_B200_TMAP");
    e->use_tmap = (ok && env && std::atoi(env) != 0) ? 1 : 0;
  }
  if (dev_alloc(&e->d_ctl, 1)) return 1;
  if (dev_alloc(&e->d_round_flag, 1)) return 1;
  if (dev_alloc(&e->d_dummy_state, kMaxBufs)) return 1;
  if (dev_alloc(&e->d_dummy_sched, 1)) return 1;
  for (void* p : std::vector<void*>{e->d_ctl, e->d_round_flag, e->d_dummy_state, e->d_dummy_sched}) e->owned.push_back(p);
  *out = e.release();
  return 0;
}

void ffn_engine_destroy(FfnEngine* e) {
  if (!e || e->closing) return;
  if (e->live_canvases > 0) {   // canvases outlive the engine: defer the release to the last of them
    e->closing = true;
    return;
  }
  engine_free(e);
}

int ffn_engine_set_grid(FfnEngine* e, int num_ctas) {
  if (!e) return fail("null engine");
  if (num_ctas <= 0) num_ctas = std::min(e->sm_count, e->g.nt);
  if (num_ctas > e->sm_count || num_ctas > e->g.nt) return fail("grid larger than the SM / tile count");
  if ((e->g.nt + num_ctas - 1) / num_ctas > kMaxTilesPerCta)
    return fail("grid too small: at most " + std::to_string(kMaxTilesPerCta) + " tiles per CTA");
  e->grid = num_ctas;
  return 0;
}

int ffn_engine_set_chains(FfnEngine* e, int max_chains) {
  if (!e) return fail("null engine");
  if (max_chains <= 0) max_chains = kMaxChains;
  if (max_chains > kMaxChains) return fail("at most " + std::to_string(kMaxChains) + " chains");
  e->max_chains = max_chains;
  return 0;
}

int ffn_engine_set_compute_mode(FfnEngine* e, int mode) {
  if (!e) return fail("null engine");
  if (mode != FFN_COMPUTE_FP16_TC && mode != FFN_COMPUTE_FP32 && mode != FFN_COMPUTE_FP16X2_TC)
    return fail("unknown compute mode");
  e->compute_mode = mode;
  return 0;
}

int ffn_engine_info(FfnEngine* e, int64_t info[8]) {
  if (!e || !info) return fail("null argument");
  info[0] = e->sm_count;
  info[1] = e->grid;
  info[2] = e->smem_bytes;
  info[3] = e->g.nt;
  info[4] = e->g.nr;
  info[5] = e->g.V;
  info[6] = e->launches;
  info[7] = (int64_t)(e->last_kernel_seconds * 1e9);
  return 0;
}

int ffn_engine_profile(FfnEngine* e, int64_t out[32], int reset) {
  if (!e) return fail("null argument");
  if (!out) {   // (out == NULL): switch the device-side counters on (reset != 0) or off (reset == 0)
    e->profiling = reset != 0;
    return 0;
  }
  if (set_device(e)) return 1;
  long long h[32];
  CUDA_OK(cudaMemcpy(h, e->ws.prof, sizeof(h), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 32; ++i) out[i] = h[i];
  if (reset) CUDA_OK(cudaMemset(e->ws.prof, 0, sizeof(h)));
  return 0;
}

int ffn_engine_trace(FfnEngine* e, int64_t* out, int64_t n, int reset) {
  if (!e || !out || n < 0 || n > (int64_t)kTraceEvents * kTraceTiles) return fail("bad argument");
  if (set_device(e)) return 1;
  static_assert(sizeof(long long) == sizeof(int64_t), "trace element");
  CUDA_OK(cudaMemcpy(out, e->ws.prof + 32, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (reset) CUDA_OK(cudaMemset(e->ws.prof + 32, 0, sizeof(long long) * kTraceEvents * kTraceTiles));
  return 0;
}

int ffn_predict(FfnEngine* e, const float* seed, const float* image, int batch, float* logits_out) {
  if (!e || !seed || !image || !logits_out || batch < 1) return fail("bad argument");
  if (set_device(e)) return 1;
  const size_t n = (size_t)batch * e->g.V;
  if (batch > e->predict_cap) {
    cudaFree(e->d_in_seed);
    cudaFree(e->d_in_image);
    cudaFree(e->d_out);
    e->d_in_seed = e->d_in_image = e->d_out = nullptr;
    if (dev_alloc(&e->d_in_seed, n, false)) return 1;
    if (dev_alloc(&e->d_in_image, n, false)) return 1;
    if (dev_alloc(&e->d_out, n, false)) return 1;
    e->predict_cap = batch;
  }
  CUDA_OK(cudaMemcpyAsync(e->d_in_seed, seed, n * sizeof(float), cudaMemcpyHostToDevice, cudaStreamPerThread));
  CUDA_OK(cudaMemcpyAsync(e->d_in_image, image, n * sizeof(float), cudaMemcpyHostToDevice, cudaStreamPerThread));
  Job job{};
  job.mode = MODE_PREDICT;
  job.in_seed = e->d_in_seed;
  job.in_image = e->d_in_image;
  job.out_logits = e->d_out;
  job.batch = batch;
  // the patches of a batch are independent: up to chain_limit() of them share one round of the pipeline
  const int nch = e->compute_mode == FFN_COMPUTE_FP16_TC ? std::min(chain_limit(e), batch) : 1;
  if (launch(e, nullptr, nch, job)) return 1;
  CUDA_OK(cudaMemcpy(logits_out, e->d_out, n * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int ffn_canvas_create(FfnEngine* e, const void* image, int image_dtype, const int32_t shape_zyx[3],
                      float image_mean, float image_stddev, const FfnOptions* options,
                      int keep_probability_maps, FfnCanvas** out) {
  if (!e || !image || !shape_zyx || !options || !out) return fail("null argument");
  if (image_dtype != FFN_IMAGE_U8 && image_dtype != FFN_IMAGE_F32) return fail("unknown image dtype");
  if (set_device(e)) return 1;
  const Geom& g = e->g;
  for (int k = 0; k < 3; ++k)
    if (shape_zyx[k] < 1) return fail("bad canvas shape");
  if ((size_t)shape_zyx[0] * shape_zyx[1] * shape_zyx[2] > (size_t)1 << 33) return fail("canvas too large");
  std::unique_ptr<FfnCanvas> c(new FfnCanvas());
  c->eng = e;
  CanvasDev& cv = c->cv;
  cv.sz = shape_zyx[0];
  cv.sy = shape_zyx[1];
  cv.sx = shape_zyx[2];
  c->nvox = (size_t)cv.sz * cv.sy * cv.sx;
  cv.opt = *options;
  {
    // smallest float32 >= the float64 policy threshold: `score < th64` (float64 compare of a
    // float32 score, movement.py:84) <=> `score < th32` in float32.
    float t = (float)options->policy_score_threshold;
    if ((double)t < options->policy_score_threshold) t = std::nextafterf(t, INFINITY);
    cv.policy_th_f32 = t;
  }
  cv.image_is_u8 = image_dtype == FFN_IMAGE_U8;
  cv.mean = image_mean;
  cv.stddev = image_stddev;
  const size_t ibytes = c->nvox * (cv.image_is_u8 ? 1 : 4);
  CUDA_OK(cudaMalloc(&c->d_image, ibytes));
  CUDA_OK(cudaMemcpy(c->d_image, image, ibytes, cudaMemcpyHostToDevice));
  cv.image = c->d_image;
  if (dev_alloc(&c->ob[0].seed, c->nvox, false)) return 1;
  if (dev_alloc(&cv.seg, c->nvox)) return 1;
  if (keep_probability_maps) {
    if (dev_alloc(&cv.qprob, c->nvox)) return 1;
  }
  fill_f32_kernel<<<e->sm_count * 8, 256, 0, cudaStreamPerThread>>>(c->ob[0].seed, c->nvox, NAN);
  CUDA_OK(cudaGetLastError());
  // movement policy storage
  const int del[3] = {std::max(g.dz, 1), std::max(g.dy, 1), std::max(g.dx, 1)};
  const int shp[3] = {cv.sz, cv.sy, cv.sx};
  size_t cells = 1, qcells = 1;
  for (int k = 0; k < 3; ++k) {
    const int n = (shp[k] + del[k] - 1) / del[k];
    cv.lat_off[k] = n + 1;
    cv.lat_dim[k] = 2 * n + 3;
    cells *= (size_t)cv.lat_dim[k];
    qcells *= (size_t)(n + 2);
  }
  c->lattice_cells = cells;
  c->q_cap = std::min<size_t>(6 * qcells + 16, (size_t)1 << 30);
  c->traj_cap = std::min<size_t>(qcells + 16, (size_t)1 << 28);   // one FoV step per lattice cell at most
  cv.q_cap = (int)c->q_cap;
  cv.traj_cap = (int)c->traj_cap;
  if (alloc_buf(c.get(), 0)) return 1;
  if (dev_alloc(&c->d_state, kMaxBufs)) return 1;
  if (dev_alloc(&c->d_sched, 1)) return 1;
  if (dev_alloc(&c->d_pred, (size_t)g.V, false)) return 1;
  std::memset(&c->h_state, 0, sizeof(CanvasState));
  std::memset(&c->h_sched, 0, sizeof(Sched));
  c->h_sched.owner = -1;
  c->h_sched.last_chain = -1;
  for (int k = 0; k < kMaxChains; ++k) c->h_sched.active[k] = kBufsPerChain * k;
  for (int b = 0; b < kMaxBufs; ++b) {
    c->h_sched.bseed[b] = -1;
    c->h_sched.bkind[b] = b == 0 ? 3 : -1;
  }
  CUDA_OK(cudaMemcpy(c->d_sched, &c->h_sched, sizeof(Sched), cudaMemcpyHostToDevice));
  c->h_state.seed_index = -1;
  if (push_state(c.get())) return 1;
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  e->live_canvases++;
  *out = c.release();
  return 0;
}

void ffn_canvas_destroy(FfnCanvas* c) {
  if (!c) return;
  FfnEngine* e = c->eng;
  cudaSetDevice(e->device);
  cudaFree(c->d_image);
  cudaFree(c->ob[0].seed);      // buffer 0 is allocated with the canvas; the others and the snapshot array live in pools
  cudaFree(c->ob[0].lattice);
  cudaFree(c->ob[0].q_score);
  cudaFree(c->ob[0].q_pos);
  cudaFree(c->ob[0].traj);
  for (void* q : c->pools) cudaFree(q);
  cudaFree(c->cv.seg);
  cudaFree(c->cv.qprob);
  cudaFree(c->cv.trace);
  cudaFree(c->d_state);
  cudaFree(c->d_sched);
  cudaFree(c->d_pred);
  cudaFree(c->d_mask);
  cudaFree(c->d_seed_mask);
  delete c;
  if (--e->live_canvases == 0 && e->closing) engine_free(e);
}

int ffn_canvas_set_mask(FfnCanvas* c, int which, const uint8_t* mask) {
  if (!c) return fail("null canvas");
  if (set_device(c->eng)) return 1;
  uint8_t** slot = which == FFN_MASK_MOVEMENT ? &c->d_mask : which == FFN_MASK_SEED ? &c->d_seed_mask : nullptr;
  if (!slot) return fail("unknown mask id");
  if (!mask) {
    cudaFree(*slot);
    *slot = nullptr;
  } else {
    if (!*slot) CUDA_OK(cudaMalloc(reinterpret_cast<void**>(slot), c->nvox));
    CUDA_OK(cudaMemcpy(*slot, mask, c->nvox, cudaMemcpyHostToDevice));
  }
  c->cv.mask = c->d_mask;
  c->cv.seed_mask = c->d_seed_mask;
  return 0;
}

int ffn_canvas_init_seed(FfnCanvas* c, const int32_t pos[3]) {
  if (!c || !pos) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (pos[0] < 0 || pos[1] < 0 || pos[2] < 0 || pos[0] >= c->cv.sz || pos[1] >= c->cv.sy || pos[2] >= c->cv.sx)
    return fail("seed position outside the canvas");
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  // clear only what can be non-NaN (== NumpyArray.clear), then place the seed
  if (fill_box(c, c->ob[0].seed, st.dirty_lo, st.dirty_hi)) return 1;
  CUDA_OK(cudaMemcpyAsync(c->ob[0].seed + ((size_t)pos[0] * c->cv.sy + pos[1]) * c->cv.sx + pos[2],
                          &c->cv.opt.init_activation, sizeof(float), cudaMemcpyHostToDevice, cudaStreamPerThread));
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  for (int k = 0; k < 3; ++k) {
    st.dirty_lo[k] = pos[k];
    st.dirty_hi[k] = pos[k] + 1;
  }
  return push_state(c);
}

int ffn_canvas_segment_at(FfnCanvas* c, const int32_t start[3], int reset, int64_t max_steps, FfnSegStats* out) {
  if (!c || !start || !out) return fail("null argument");
  FfnEngine* e = c->eng;
  if (set_device(e)) return 1;
  if (start[0] < 0 || start[1] < 0 || start[2] < 0 || start[0] >= c->cv.sz || start[1] >= c->cv.sy ||
      start[2] >= c->cv.sx)
    return fail("start position outside the canvas");
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  c->resume_pending = false;   // driving the object by hand consumes a pending checkpoint resume
  st.seg_all = 0;
  const long long steps0 = st.ctr.inference_calls;
  const long long weak0 = st.ctr.seed_got_too_weak;
  if (reset) {
    for (int k = 0; k < 3; ++k) st.start[k] = start[k];
    st.reset_seed = (reset & 2) ? 0 : 1;   // 2: Canvas.reset_seed_per_segment == False (inference.py:486-490)
    st.phase = PH_START_SEGMENT;
    st.popped = 0;
  } else {
    if (st.phase != PH_POP) return fail("no object in flight to resume");
  }
  if (push_state(c)) return 1;
  Job job{};
  job.mode = MODE_SEGMENT;
  double secs = 0;
  for (;;) {
    const long long done = st.ctr.inference_calls - steps0;
    long long chunk = 1 << 15;
    if (max_steps > 0) chunk = std::min<long long>(chunk, max_steps - done);
    job.step_budget = st.ctr.inference_calls + chunk;
    if (launch(e, c, 1, job)) return 1;
    secs += e->last_kernel_seconds;
    if (pull_state(c)) return 1;
    if (st.phase == PH_SEGMENT_DONE) break;
    if (st.phase != PH_POP) return fail("unexpected device phase " + std::to_string(st.phase));
    if (max_steps > 0 && st.ctr.inference_calls - steps0 >= max_steps) break;
  }
  if (st.overflow) return fail("movement queue capacity exceeded");
  out->iters = st.iters;
  for (int k = 0; k < 3; ++k) {
    out->min_pos[k] = st.min_pos[k];
    out->max_pos[k] = st.max_pos[k];
  }
  out->seed_got_too_weak = (int)(st.ctr.seed_got_too_weak - weak0);
  out->queue_len = st.q_tail - st.q_head + (st.popped && st.pop_run ? 1 : 0);
  out->finished = st.phase == PH_SEGMENT_DONE;
  out->reserved = 0;
  st.ctr.device_seconds += secs;
  return push_state(c);
}

int ffn_canvas_segment_all(FfnCanvas* c, const int32_t* seeds, int64_t n_seeds, FfnOrigin* origins_out,
                           int64_t origins_cap, int64_t* n_origins, FfnOverlap* overlaps_out,
                           int64_t overlaps_cap, int64_t* n_overlaps, FfnCounters* counters_out) {
  if (!c || (n_seeds > 0 && !seeds) || !n_origins || !n_overlaps) return fail("null argument");
  FfnEngine* e = c->eng;
  if (set_device(e)) return 1;
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  Sched& sc = c->h_sched;
  // Chains: several objects in flight, committed in seed order (see Sched).  The parity modes and the event
  // trace (Canvas.history) run one object at a time.
  int K = 1;
  if (e->compute_mode == FFN_COMPUTE_FP16_TC && !c->cv.trace) K = chain_limit(e);
  const auto t_enter = std::chrono::steady_clock::now();
  auto since = [&](std::chrono::steady_clock::time_point t) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
  };
  if (ensure_bufs(c, K > 1 ? kBufsPerChain * K : 1)) {
    // not enough device memory for the object buffers of several chains: run one object at a time
    cudaGetLastError();
    K = 1;
  }
  const double ms_bufs = since(t_enter);
  int* d_seeds = nullptr;
  FfnOrigin* d_orig = nullptr;
  FfnOverlap* d_ovl = nullptr;
  int *d_cnt = nullptr, *d_touched = nullptr;
  unsigned char* d_status = nullptr;
  const int ovl_ids = (int)std::min<int64_t>((int64_t)sc.max_id + n_seeds + 2, (int64_t)1 << 30);
  auto cleanup = [&]() {
    cudaFree(d_seeds);
    cudaFree(d_orig);
    cudaFree(d_ovl);
    cudaFree(d_cnt);
    cudaFree(d_touched);
    cudaFree(d_status);
  };
  if (dev_alloc(&d_seeds, (size_t)n_seeds * 3, false) || dev_alloc(&d_orig, (size_t)origins_cap, false) ||
      dev_alloc(&d_ovl, (size_t)overlaps_cap, false) || dev_alloc(&d_cnt, (size_t)ovl_ids) ||
      dev_alloc(&d_touched, (size_t)ovl_ids) || dev_alloc(&d_status, (size_t)n_seeds)) {
    cleanup();
    return 1;
  }
  if (n_seeds && cudaMemcpy(d_seeds, seeds, (size_t)n_seeds * 3 * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) {
    cleanup();
    return fail("seed list copy failed");
  }
  // ---- scheduler and chain states
  const bool resume = c->resume_pending;   // finish the restored in-flight object first (inference.py:538-550)
  c->resume_pending = false;
  sc.commit_idx = 0;
  sc.owner = resume ? 0 : -1;
  sc.nchains = K;
  sc.overflow = 0;
  sc.n_origins = sc.n_overlaps = 0;
  sc.steps_executed = 0;
  sc.spec_runs = sc.spec_discarded = sc.spec_steps_discarded = 0;
  sc.idle_free = sc.idle_wait = 0;
  const unsigned round0 = sc.round;
  sc.all_done = 0;
  sc.ctr = st.ctr;             // cumulative counters of the canvas; the chains count per object from here on
  const bool has_data = st.dirty_hi[0] > st.dirty_lo[0];
  sc.last_chain = has_data ? 0 : -1;   // what Canvas.seed shows right now
  sc.last_in_snap = 0;
  for (int k = 0; k < kMaxChains; ++k) sc.active[k] = kBufsPerChain * k;
  for (int b = 0; b < kMaxBufs; ++b) {
    sc.bseed[b] = -1;
    sc.bround[b] = 0;
    sc.bkind[b] = b >= c->nbufs_alloc || b >= K * kBufsPerChain ? -1 : (b % kBufsPerChain == 0 ? 3 : 0);
  }
  std::vector<CanvasState> hs(kMaxBufs);
  if (cudaMemcpy(hs.data(), c->d_state, sizeof(CanvasState) * kMaxBufs, cudaMemcpyDeviceToHost) != cudaSuccess) {
    cleanup();
    return fail("state copy failed");
  }
  hs[0] = st;
  for (int k = 0; k < kMaxBufs; ++k) {
    CanvasState& h = hs[k];
    h.seg_all = 1;
    h.seed_index = -1;
    h.spec = 0;
    h.popped = 0;
    h.overflow = 0;
    h.ctr = FfnCounters{};
    h.phase = (k == 0 && resume) ? PH_POP : PH_FREE;
    if (!(k == 0 && resume)) h.have_cur = 0;
  }
  if (cudaMemcpy(c->d_state, hs.data(), sizeof(CanvasState) * kMaxBufs, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(c->d_sched, &sc, sizeof(Sched), cudaMemcpyHostToDevice) != cudaSuccess) {
    cleanup();
    return fail("state upload failed");
  }
  Job job{};
  job.mode = MODE_SEGMENT;
  job.seeds = d_seeds;
  job.n_seeds = n_seeds;
  job.origins = d_orig;
  job.origins_cap = origins_cap;
  job.overlaps = d_ovl;
  job.overlaps_cap = overlaps_cap;
  job.ovl_count = d_cnt;
  job.ovl_touched = d_touched;
  job.ovl_ids = ovl_ids;
  job.seed_status = d_status;
  if (const char* dbg = std::getenv("FFN_B200_DEBUG")) job.debug = std::atoi(dbg);
  double secs = 0;
  long long launches = 0;
  int stuck = 0;
  int rc = 0;
  const double ms_setup = since(t_enter);
  for (;;) {
    const long long before_steps = sc.steps_executed, before_idx = sc.commit_idx;
    const unsigned before_round = sc.round;
    job.step_budget = sc.steps_executed + (1 << 15);
    job.round_cap = 2 * (1 << 15) + 8 * n_seeds + 4096;
    if (launch(e, c, K, job)) {
      cleanup();
      return 1;
    }
    secs += e->last_kernel_seconds;
    ++launches;
    if (cudaMemcpy(&sc, c->d_sched, sizeof(Sched), cudaMemcpyDeviceToHost) != cudaSuccess) {
      cleanup();
      return fail("scheduler state copy failed");
    }
    if (sc.all_done) break;
    if ((job.debug & 64) && sc.steps_executed < job.step_budget) {   // a launch ended early without being done: why?
      std::vector<CanvasState> dbg(kMaxBufs);
      cudaMemcpy(dbg.data(), c->d_state, sizeof(CanvasState) * kMaxBufs, cudaMemcpyDeviceToHost);
      std::fprintf(stderr, "[ffn] launch %lld ended early: commit_idx %lld / %lld owner %d round %u active %d %d %d\n", launches,
                   sc.commit_idx, (long long)n_seeds, sc.owner, sc.round, sc.active[0], sc.active[1], sc.active[2]);
      for (int b = 0; b < K * kBufsPerChain; ++b)
        if (sc.bkind[b] > 0)
          std::fprintf(stderr, "   buf %d kind %d seed %lld bround %d | phase %d seed %lld spec %d iters %lld fin_round %d have_cur %d\n", b,
                       sc.bkind[b], sc.bseed[b], sc.bround[b], dbg[b].phase, dbg[b].seed_index, dbg[b].spec, dbg[b].iters,
                       dbg[b].fin_round, dbg[b].have_cur);
    }
    if (sc.overflow & 16) stuck = 3;   // the device watchdog tripped
    (void)before_round;
    if (stuck < 3) stuck = (sc.steps_executed == before_steps && sc.commit_idx == before_idx) ? stuck + 1 : 0;
    if (stuck >= 3) {
      std::vector<CanvasState> dbg(kMaxBufs);
      cudaMemcpy(dbg.data(), c->d_state, sizeof(CanvasState) * kMaxBufs, cudaMemcpyDeviceToHost);
      std::string msg = "segment_all made no progress: device scheduler stalled at seed " + std::to_string(sc.commit_idx) +
                        " of " + std::to_string(n_seeds) + ", owner " + std::to_string(sc.owner) + ", round " +
                        std::to_string(sc.round) + "; buffers (phase/seed/spec/iters/fin_round):";
      for (int k = 0; k < c->nbufs_alloc; ++k)
        msg += " [" + std::to_string(dbg[k].phase) + "/" + std::to_string(dbg[k].seed_index) + "/" + std::to_string(dbg[k].spec) +
               "/" + std::to_string(dbg[k].iters) + "/" + std::to_string(dbg[k].fin_round) + "]";
      rc = fail(msg);
      break;
    }
  }
  const double ms_loop = since(t_enter);
  if (!rc && pull_state(c)) rc = 1;
  // ---- Canvas.seed shows the last object segment_at ran on: bring it into the canvas's own array
  if (!rc && (sc.last_in_snap || sc.last_chain > 0)) {
    const float* src = sc.last_in_snap ? c->d_snap : c->ob[sc.last_chain].seed;
    int lo[3], hi[3];
    CanvasState last{};
    if (!sc.last_in_snap &&
        cudaMemcpy(&last, c->d_state + sc.last_chain, sizeof(CanvasState), cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = fail("state copy failed");
    for (int q = 0; q < 3; ++q) {
      lo[q] = std::max(sc.last_in_snap ? sc.snap_lo[q] : last.dirty_lo[q], 0);
      hi[q] = std::min(sc.last_in_snap ? sc.snap_hi[q] : last.dirty_hi[q], q == 0 ? c->cv.sz : q == 1 ? c->cv.sy : c->cv.sx);
    }
    if (!rc && fill_box(c, c->ob[0].seed, st.dirty_lo, st.dirty_hi)) rc = 1;
    if (!rc && hi[0] > lo[0] && hi[1] > lo[1] && hi[2] > lo[2]) {
      copy_box_f32_kernel<<<e->sm_count * 4, 256, 0, cudaStreamPerThread>>>(c->ob[0].seed, src, c->cv.sy, c->cv.sx, lo[0], lo[1],
                                                                         lo[2], hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]);
      if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(cudaStreamPerThread) != cudaSuccess)
        rc = fail("seed box copy failed");
    }
    for (int q = 0; q < 3; ++q) {
      st.dirty_lo[q] = lo[q];
      st.dirty_hi[q] = hi[q];
    }
  } else if (!rc && sc.last_chain < 0) {
    // no object ran in turn: Canvas.seed is what it was (nothing); early runs on chain 0 leave no trace
    if (fill_box(c, c->ob[0].seed, st.dirty_lo, st.dirty_hi)) rc = 1;
    for (int q = 0; q < 3; ++q) st.dirty_lo[q] = st.dirty_hi[q] = 0;
    cudaStreamSynchronize(cudaStreamPerThread);
  }
  *n_origins = sc.n_origins;
  *n_overlaps = sc.n_overlaps;
  if (!rc && (sc.overflow & 1)) rc = fail("movement queue capacity exceeded");
  if (!rc && (sc.overflow & 8)) rc = fail("trajectory log capacity exceeded");
  if (!rc && origins_out && sc.n_origins)
    if (cudaMemcpy(origins_out, d_orig, (size_t)std::min<long long>(sc.n_origins, origins_cap) * sizeof(FfnOrigin),
                   cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = fail("origins copy failed");
  if (!rc && overlaps_out && sc.n_overlaps)
    if (cudaMemcpy(overlaps_out, d_ovl, (size_t)std::min<long long>(sc.n_overlaps, overlaps_cap) * sizeof(FfnOverlap),
                   cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = fail("overlaps copy failed");
  cleanup();
  if (job.debug & 128)
    std::fprintf(stderr, "[ffn] segment_all host ms: buffers %.2f, setup %.2f, launches %.2f (kernel %.2f), tail %.2f\n", ms_bufs,
                 ms_setup - ms_bufs, ms_loop - ms_setup, secs * 1e3, since(t_enter) - ms_loop);
  st.ctr = sc.ctr;
  st.ctr.max_id = sc.max_id;
  st.ctr.device_seconds += secs;
  st.ctr.kernel_launches += launches;
  st.phase = PH_IDLE;
  st.seg_all = 0;
  st.have_cur = 0;
  c->last_spec[0] = sc.spec_runs;
  c->last_spec[1] = sc.spec_discarded;
  c->last_spec[2] = sc.spec_steps_discarded;
  c->last_spec[3] = sc.steps_executed;
  c->last_spec[4] = (long long)sc.round - (long long)round0;
  c->last_spec[5] = sc.idle_free;
  c->last_spec[6] = sc.idle_wait;
  c->last_spec[7] = K;
  if (counters_out) *counters_out = st.ctr;
  // single-object calls (segment_at, update_at) work on buffer 0 through chain 0
  for (int k = 0; k < kMaxChains; ++k) sc.active[k] = kBufsPerChain * k;
  sc.owner = -1;
  if (cudaMemcpy(c->d_sched, &sc, sizeof(Sched), cudaMemcpyHostToDevice) != cudaSuccess) return fail("scheduler state upload failed");
  if (push_state(c)) return 1;
  return rc;
}

int ffn_canvas_update_at(FfnCanvas* c, const int32_t pos[3], float* pred_out) {
  if (!c || !pos) return fail("null argument");
  FfnEngine* e = c->eng;
  if (set_device(e)) return 1;
  const Geom& g = e->g;
  if (pos[0] - g.mz < 0 || pos[1] - g.my < 0 || pos[2] - g.mx < 0 || pos[0] + g.mz >= c->cv.sz ||
      pos[1] + g.my >= c->cv.sy || pos[2] + g.mx >= c->cv.sx)
    return fail("field of view leaves the canvas");
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  const int saved_phase = st.phase;
  for (int k = 0; k < 3; ++k) st.cur[k] = pos[k];
  st.phase = PH_FORCE_STEP;
  if (push_state(c)) return 1;
  Job job{};
  job.mode = MODE_UPDATE_AT;
  job.pred_out = c->d_pred;
  if (launch(e, c, 1, job)) return 1;
  if (pull_state(c)) return 1;
  st.phase = saved_phase;
  st.ctr.device_seconds += e->last_kernel_seconds;
  if (push_state(c)) return 1;
  if (pred_out) CUDA_OK(cudaMemcpy(pred_out, c->d_pred, (size_t)g.V * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int ffn_canvas_read(FfnCanvas* c, int which, const int32_t lo[3], const int32_t sz[3], void* dst) {
  if (!c || !lo || !sz || !dst) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (which == FFN_ARRAY_IMAGE) {
    // always float32, normalised like runner.py:383-385
    const CanvasDev& cv = c->cv;
    if (lo[0] != 0 || lo[1] != 0 || lo[2] != 0 || sz[0] != cv.sz || sz[1] != cv.sy || sz[2] != cv.sx)
      return fail("image reads must cover the whole canvas");
    if (!cv.image_is_u8) {
      CUDA_OK(cudaMemcpy(dst, cv.image, c->nvox * 4, cudaMemcpyDeviceToHost));
      return 0;
    }
    float* tmp = nullptr;
    if (dev_alloc(&tmp, c->nvox, false)) return 1;
    normalize_u8_kernel<<<c->eng->sm_count * 8, 256, 0, cudaStreamPerThread>>>(
        reinterpret_cast<const uint8_t*>(cv.image), tmp, c->nvox, cv.mean, cv.stddev);
    cudaError_t err = cudaMemcpy(dst, tmp, c->nvox * 4, cudaMemcpyDeviceToHost);
    cudaFree(tmp);
    if (err != cudaSuccess) return fail(cudaGetErrorString(err));
    return 0;
  }
  return box_copy(c, which, lo, sz, dst, true);
}

int ffn_canvas_write(FfnCanvas* c, int which, const int32_t lo[3], const int32_t sz[3], const void* src) {
  if (!c || !lo || !sz || !src) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (which == FFN_ARRAY_IMAGE) return fail("the image is immutable");
  if (box_copy(c, which, lo, sz, const_cast<void*>(src), false)) return 1;
  if (which == FFN_ARRAY_SEED) {
    if (pull_state(c)) return 1;
    CanvasState& st = c->h_state;
    const bool empty = st.dirty_hi[0] <= st.dirty_lo[0];
    for (int k = 0; k < 3; ++k) {
      st.dirty_lo[k] = empty ? lo[k] : std::min(st.dirty_lo[k], lo[k]);
      st.dirty_hi[k] = empty ? lo[k] + sz[k] : std::max(st.dirty_hi[k], lo[k] + sz[k]);
    }
    return push_state(c);
  }
  return 0;
}

int ffn_canvas_policy_state_size(FfnCanvas* c, int64_t* queue_len, int64_t* done_len) {
  if (!c || !queue_len || !done_len) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  // a position popped for the next step but not yet executed (paused launch) is still part of the queue
  *queue_len = c->h_state.q_tail - c->h_state.q_head + ((c->h_state.popped && c->h_state.pop_run) ? 1 : 0);
  std::vector<unsigned> lat(c->lattice_cells);
  CUDA_OK(cudaMemcpy(lat.data(), c->ob[0].lattice, lat.size() * sizeof(unsigned), cudaMemcpyDeviceToHost));
  int64_t n = 0;
  if (c->h_state.epoch)
    for (unsigned v : lat) n += v == c->h_state.epoch;
  *done_len = n;
  return 0;
}

int ffn_canvas_policy_state_get(FfnCanvas* c, double* queue_szyx, int32_t* done_zyx, int32_t start[3]) {
  if (!c || !start) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  const CanvasState& st = c->h_state;
  const int head = st.q_head - ((st.popped && st.pop_run) ? 1 : 0);   // see ffn_canvas_policy_state_size
  const int n = st.q_tail - head;
  if (n > 0 && queue_szyx) {
    std::vector<float> sc(n);
    std::vector<int> ps((size_t)n * 3);
    CUDA_OK(cudaMemcpy(sc.data(), c->ob[0].q_score + head, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(ps.data(), c->ob[0].q_pos + (size_t)head * 3, (size_t)n * 3 * sizeof(int),
                       cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) {
      queue_szyx[4 * i] = sc[i];
      for (int k = 0; k < 3; ++k) queue_szyx[4 * i + 1 + k] = ps[3 * i + k];
    }
  }
  if (done_zyx && st.epoch) {
    std::vector<unsigned> lat(c->lattice_cells);
    CUDA_OK(cudaMemcpy(lat.data(), c->ob[0].lattice, lat.size() * sizeof(unsigned), cudaMemcpyDeviceToHost));
    size_t o = 0;
    const int* d = c->cv.lat_dim;
    for (size_t i = 0; i < lat.size(); ++i)
      if (lat[i] == st.epoch) {
        const int qx = (int)(i % d[2]), qy = (int)((i / d[2]) % d[1]), qz = (int)(i / ((size_t)d[1] * d[2]));
        done_zyx[o++] = qz - c->cv.lat_off[0];
        done_zyx[o++] = qy - c->cv.lat_off[1];
        done_zyx[o++] = qx - c->cv.lat_off[2];
      }
  }
  for (int k = 0; k < 3; ++k) start[k] = st.start[k];
  return 0;
}

int ffn_canvas_policy_state_set(FfnCanvas* c, const double* queue_szyx, int64_t queue_len, const int32_t* done_zyx,
                                int64_t done_len, const int32_t start[3]) {
  if (!c || !start) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (queue_len > c->cv.q_cap) return fail("queue larger than device capacity");
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  st.epoch++;
  st.q_head = 0;
  st.q_tail = (int)queue_len;
  for (int k = 0; k < 3; ++k) st.start[k] = start[k];
  if (queue_len > 0) {
    std::vector<float> sc(queue_len);
    std::vector<int> ps((size_t)queue_len * 3);
    for (int64_t i = 0; i < queue_len; ++i) {
      sc[i] = (float)queue_szyx[4 * i];
      for (int k = 0; k < 3; ++k) ps[3 * i + k] = (int)queue_szyx[4 * i + 1 + k];
    }
    CUDA_OK(cudaMemcpy(c->ob[0].q_score, sc.data(), sc.size() * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(c->ob[0].q_pos, ps.data(), ps.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  const int* d = c->cv.lat_dim;
  for (int64_t i = 0; i < done_len; ++i) {
    const int qz = done_zyx[3 * i] + c->cv.lat_off[0], qy = done_zyx[3 * i + 1] + c->cv.lat_off[1],
              qx = done_zyx[3 * i + 2] + c->cv.lat_off[2];
    if (qz < 0 || qy < 0 || qx < 0 || qz >= d[0] || qy >= d[1] || qx >= d[2]) return fail("done-set entry outside lattice");
    CUDA_OK(cudaMemcpy(c->ob[0].lattice + ((size_t)qz * d[1] + qy) * d[2] + qx, &st.epoch, sizeof(unsigned),
                       cudaMemcpyHostToDevice));
  }
  st.phase = PH_POP;
  st.have_cur = 0;
  st.popped = 0;
  return push_state(c);
}

int ffn_canvas_set_resume(FfnCanvas* c, int64_t iters, const int32_t min_pos[3], const int32_t max_pos[3]) {
  if (!c || !min_pos || !max_pos) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  CanvasState& st = c->h_state;
  st.iters = iters;
  for (int k = 0; k < 3; ++k) {
    st.min_pos[k] = min_pos[k];
    st.max_pos[k] = max_pos[k];
  }
  st.phase = PH_POP;
  st.have_cur = 0;
  st.popped = 0;
  st.seg_t0 = 0;
  c->resume_pending = true;
  return push_state(c);
}

int ffn_canvas_trace(FfnCanvas* c, int64_t capacity, int32_t* events_out, int64_t* n_events) {
  if (!c) return fail("null canvas");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  if (events_out && n_events) {   // fetch what was logged so far
    const int64_t n = std::min<int64_t>(c->h_state.n_trace, c->cv.trace_cap);
    *n_events = c->h_state.n_trace;
    if (n > 0) CUDA_OK(cudaMemcpy(events_out, c->cv.trace, (size_t)n * 4 * sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
  }
  cudaFree(c->cv.trace);
  c->cv.trace = nullptr;
  c->cv.trace_cap = 0;
  if (capacity > 0) {
    if (dev_alloc(&c->cv.trace, (size_t)capacity * 4)) return 1;
    c->cv.trace_cap = (int)capacity;
  }
  c->h_state.n_trace = 0;
  return push_state(c);
}

int ffn_canvas_seed_peaks(FfnCanvas* c, const float voxel_size_zyx[3], const double* noise, int32_t* coords_out,
                          int64_t cap, int64_t* n_out) {
  if (!c || !voxel_size_zyx || !coords_out || !n_out || cap < 1) return fail("bad argument");
  FfnEngine* e = c->eng;
  if (set_device(e)) return 1;
  const CanvasDev& cv = c->cv;
  const size_t n = c->nvox;
  const int blocks = e->sm_count * 16;
  float *a = nullptr, *b = nullptr, *d = nullptr;
  double *d_noise = nullptr, *zbuf = nullptr, *d_w = nullptr;
  int *vbuf = nullptr, *d_coords = nullptr;
  unsigned long long* d_cnt = nullptr;
  auto cleanup = [&]() {
    cudaFree(a); cudaFree(b); cudaFree(d); cudaFree(d_w); cudaFree(d_noise); cudaFree(zbuf); cudaFree(vbuf);
    cudaFree(d_coords); cudaFree(d_cnt);
  };
  const int maxdim = std::max(cv.sz, cv.sy);
  const size_t maxlines = std::max((size_t)cv.sy * cv.sx, (size_t)cv.sz * cv.sx);
  // adaptive threshold: gaussian sigma = 49/6, truncate 4 (seed.py:160-163)
  const double sigma = 49.0 / 6.0;
  const int radius = (int)(4.0 * sigma + 0.5);
  std::vector<double> w(radius + 1);                 // w[0] = centre tap
  {
    double sum = 0;
    for (int k = -radius; k <= radius; ++k) sum += std::exp(-0.5 / (sigma * sigma) * k * k);
    for (int k = 0; k <= radius; ++k) w[k] = std::exp(-0.5 / (sigma * sigma) * k * k) / sum;
  }
  int rc = 0;
  if (dev_alloc(&a, n, false) || dev_alloc(&b, n, false) || dev_alloc(&d, n, false) || dev_alloc(&d_w, w.size(), false) ||
      dev_alloc(&vbuf, (size_t)maxdim * maxlines, false) || dev_alloc(&zbuf, 2 * (size_t)maxdim * maxlines, false) ||
      dev_alloc(&d_coords, (size_t)cap * 3, false) || dev_alloc(&d_cnt, 2) || (noise && dev_alloc(&d_noise, n, false))) {
    cleanup();
    return 1;
  }
  cudaStream_t st = cudaStreamPerThread;
  bool ok = cudaMemcpyAsync(d_w, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice, st) == cudaSuccess;
  if (noise) ok = ok && cudaMemcpyAsync(d_noise, noise, n * sizeof(double), cudaMemcpyHostToDevice, st) == cudaSuccess;
  seedk::sobel_mag<<<blocks, 256, 0, st>>>(cv.image, cv.image_is_u8, cv.mean, cv.stddev, a, cv.sz, cv.sy, cv.sx);
  seedk::gauss_pass<<<blocks, 256, 0, st>>>(a, b, d_w, radius, 0, cv.sz, cv.sy, cv.sx);
  seedk::gauss_pass<<<blocks, 256, 0, st>>>(b, d, d_w, radius, 1, cv.sz, cv.sy, cv.sx);
  seedk::gauss_pass<<<blocks, 256, 0, st>>>(d, b, d_w, radius, 2, cv.sz, cv.sy, cv.sx);
  seedk::edges_kernel<<<blocks, 256, 0, st>>>(a, b, cv.mask, cv.seed_mask, d, n, d_cnt);
  seedk::edt_x<<<blocks, 128, 0, st>>>(d, cv.sz, cv.sy, cv.sx, voxel_size_zyx[2]);
  seedk::edt_line<<<blocks, 128, 0, st>>>(d, 1, cv.sz, cv.sy, cv.sx, voxel_size_zyx[1], vbuf, zbuf);
  seedk::edt_line<<<blocks, 128, 0, st>>>(d, 0, cv.sz, cv.sy, cv.sx, voxel_size_zyx[0], vbuf, zbuf);
  seedk::finish_dt<<<blocks, 256, 0, st>>>(d, cv.seg, cv.mask, cv.seed_mask, n);
  seedk::peaks_kernel<<<blocks, 256, 0, st>>>(d, d_noise, cv.sz, cv.sy, cv.sx, 3, d_coords, (unsigned long long)cap, d_cnt + 1);
  unsigned long long counts[2] = {0, 0};
  ok = ok && cudaGetLastError() == cudaSuccess;
  ok = ok && cudaMemcpyAsync(counts, d_cnt, sizeof(counts), cudaMemcpyDeviceToHost, st) == cudaSuccess;
  ok = ok && cudaStreamSynchronize(st) == cudaSuccess;
  if (!ok) {
    rc = fail(std::string("seed policy kernels failed: ") + cudaGetErrorString(cudaGetLastError()));
  } else {
    *n_out = counts[0] == 0 ? 0 : (int64_t)counts[1];   // everything is an edge: no seeds (seed.py:176-177)
    const int64_t m = std::min<int64_t>(*n_out, cap);
    if (m > 0 && cudaMemcpy(coords_out, d_coords, (size_t)m * 3 * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = fail("seed coordinate copy failed");
  }
  cleanup();
  return rc;
}

int ffn_canvas_set_max_id(FfnCanvas* c, int64_t max_id) {
  if (!c) return fail("null canvas");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  c->h_sched.max_id = (int)max_id;
  c->h_state.ctr.max_id = max_id;
  return push_state(c);
}

int ffn_canvas_get_counters(FfnCanvas* c, FfnCounters* out) {
  if (!c || !out) return fail("null argument");
  if (set_device(c->eng)) return 1;
  if (pull_state(c)) return 1;
  *out = c->h_state.ctr;
  out->max_id = c->h_sched.max_id;
  return 0;
}

int ffn_canvas_spec_stats(FfnCanvas* c, int64_t out[8]) {
  if (!c || !out) return fail("null argument");
  for (int i = 0; i < 8; ++i) out[i] = c->last_spec[i];
  return 0;
}

int ffn_canvas_device_ptr(FfnCanvas* c, int which, void** ptr, int64_t* bytes) {
  if (!c || !ptr || !bytes) return fail("null argument");
  switch (which) {
    case FFN_ARRAY_SEED: *ptr = c->ob[0].seed; *bytes = (int64_t)c->nvox * 4; return 0;
    case FFN_ARRAY_SEGMENTATION: *ptr = c->cv.seg; *bytes = (int64_t)c->nvox * 4; return 0;
    case FFN_ARRAY_QPROB:
      if (!c->cv.qprob) return fail("canvas was created without probability maps");
      *ptr = c->cv.qprob; *bytes = (int64_t)c->nvox; return 0;
    case FFN_ARRAY_IMAGE: *ptr = c->d_image; *bytes = (int64_t)c->nvox * (c->cv.image_is_u8 ? 1 : 4); return 0;
  }
  return fail("unknown array id");
}

int ffn_canvas_add_id_offset(FfnCanvas* c, int32_t offset) {
  if (!c) return fail("null canvas");
  if (set_device(c->eng)) return 1;
  relabel_offset_kernel<<<c->eng->sm_count * 8, 256, 0, cudaStreamPerThread>>>(c->cv.seg, c->nvox, offset);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

int ffn_selftest_umma(int device, int variant, double* out, int n_out) {
  if (!out || n_out < 8) return fail("need >= 8 output slots");
  std::string err;
  if (ffn::selftest::run(device, variant, out, n_out, &err)) return fail(err);
  return 0;
}

}  // extern "C"
