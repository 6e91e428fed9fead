// train.cu — one training step of ConvStack3DFFNModel on the device (ffn_trainer_*): the trainer owns fp32 master
// weights, optimizer slots and the saved state of the forward pass for up to max_batch patches.

#include <cmath>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "device_types.cuh"
#include "host.cuh"
#include "state_blob.cuh"
#include "train_kernels.cuh"

using namespace ffn;
using trk::TGeom;

struct FfnTrainer {
  DevBufs mem;
  int device = 0, sm_count = 0, nconv = 0, max_batch = 0;
  FfnTrainDesc desc{};
  TGeom g{};                               // batch and data_rows are set per call
  int64_t global_step = 0;
  float beta1_power = 0.f, beta2_power = 0.f;
  int nparam = 0;
  std::vector<int> w_off, b_off;           // per conv, then conv_lom
  float *params = nullptr, *grads = nullptr, *slot_a = nullptr, *slot_b = nullptr;
  std::vector<__nv_bfloat16*> wf, wt, x;   // forward / dgrad weight packs, saved operands (per conv)
  std::vector<uint32_t*> mask;             // [i]: ReLU derivative of conv i's input (i = nconv: conv_lom's)
  float *res = nullptr, *gres = nullptr;
  __nv_bfloat16* gout[2] = {nullptr, nullptr};
  float *seed = nullptr, *image = nullptr, *labels = nullptr, *lw = nullptr, *logits = nullptr, *dl = nullptr;
  float *wpart = nullptr, *bpart = nullptr, *hpart = nullptr, *hsum = nullptr;
  double* lpart = nullptr;
  ~FfnTrainer() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
  }
};

namespace {

int cin_of(int l) { return l == 0 ? 2 : 32; }
int kc_of(int l) { return l == 0 ? 2 : 4; }
size_t conv_smem(const TGeom& g, int kc) {
  return (size_t)27 * kc * 512 + (size_t)3 * kc * (trk::kTileRows + 2 * (g.P + 1)) * 16;
}
int data_rows(const TGeom& g, int batch) {
  return (batch * g.Vp + trk::kSplitRows - 1) / trk::kSplitRows * trk::kSplitRows;
}
int head_blocks(const TGeom& g, int batch) { return (batch * g.V + trk::kHeadThreads - 1) / trk::kHeadThreads; }

template <int KC, int KIND>
int launch_conv(FfnTrainer* t, const trk::ConvArgs& a) {
  const size_t smem = conv_smem(t->g, KC);
  const int ntiles = a.g.data_rows / trk::kTileRows;
  trk::conv<KC, KIND><<<std::min(ntiles, 2 * t->sm_count), trk::kConvThreads, smem, cudaStreamPerThread>>>(a);
  CUDA_OK(cudaGetLastError());
  return 0;
}

int launch_reduce(const float* part, int nparts, int ncols, float* out) {
  trk::reduce_partials<<<(ncols + 255) / 256, 256, 0, cudaStreamPerThread>>>(part, nparts, ncols, out);
  CUDA_OK(cudaGetLastError());
  return 0;
}

template <int KC>
int launch_wgrad(FfnTrainer* t, const TGeom& g, int l) {
  trk::wgrad<KC><<<g.data_rows / trk::kSplitRows, trk::kWgradThreads, trk::WgradShape<KC>::kSmem, cudaStreamPerThread>>>(
      t->x[l], t->gout[0], t->wpart, g, cin_of(l));
  CUDA_OK(cudaGetLastError());
  return launch_reduce(t->wpart, g.data_rows / trk::kSplitRows, 27 * cin_of(l) * 32, t->grads + t->w_off[l]);
}

// Forward, loss and backward of the batch in t->seed, t->image, t->labels (and t->lw when use_lw): logits, dlogits,
// the raw gradients of every parameter and the head's loss partial sums (t->lpart, *hb_out of them), on the device.
// Enqueues only; nothing is synchronised.
int run_device(FfnTrainer* t, bool use_lw, int batch, int* hb_out) {
  cudaStream_t st = cudaStreamPerThread;
  TGeom g = t->g;
  g.batch = batch;
  g.data_rows = data_rows(g, batch);
  const size_t nv = (size_t)batch * g.V;
  const int blocks = t->sm_count * 4;
  for (int l = 0; l < t->nconv; ++l)
    trk::pack_weights<<<blocks, 256, 0, st>>>(t->params + t->w_off[l], cin_of(l), kc_of(l), t->wf[l], t->wt[l]);
  trk::stage_input<<<blocks, 256, 0, st>>>(g, t->image, t->seed, t->x[0]);
  CUDA_OK(cudaGetLastError());

  // forward: conv0_a, conv0_b, then (conv_a, conv_b + skip) per residual module
  for (int l = 0; l < t->nconv; ++l) {
    trk::ConvArgs a{};
    a.x = t->x[l];
    a.w = t->wf[l];
    a.bias = t->params + t->b_off[l];
    a.res = t->res;
    a.mask_out = t->mask[l + 1];
    a.out = l + 1 < t->nconv ? t->x[l + 1] : nullptr;
    a.add_res = l >= 3;
    a.g = g;
    const int rc = l == 0 ? launch_conv<2, trk::kFwdA>(t, a) : l % 2 == 0 ? launch_conv<4, trk::kFwdA>(t, a)
                                                                          : launch_conv<4, trk::kFwdB>(t, a);
    if (rc) return 1;
  }

  // loss and conv_lom
  trk::HeadArgs h{};
  h.seed = t->seed;
  h.labels = t->labels;
  h.loss_weights = use_lw ? t->lw : nullptr;
  h.res = t->res;
  h.mask = t->mask[t->nconv];
  h.lom = t->params + t->w_off[t->nconv];
  h.inv_n = 1.0f / (float)nv;
  h.logits = t->logits;
  h.dlogits = t->dl;
  h.gres = t->gres;
  h.gout = t->gout[0];
  h.part = t->hpart;
  h.loss_part = t->lpart;
  h.g = g;
  // The head writes the interior rows; the rows past this batch's patches (up to data_rows, the rows the weight
  // gradient reads) may hold an earlier, larger batch's gradient and must be zero.
  const int tail = g.data_rows - batch * g.Vp;
  CUDA_OK(cudaMemset2DAsync(t->gout[0] + (size_t)(g.guard + batch * g.Vp) * 8, (size_t)g.rows * 16, 0,
                            (size_t)tail * 16, 4, st));
  const int hb = head_blocks(g, batch);
  trk::head<<<hb, trk::kHeadThreads, 0, st>>>(h);
  CUDA_OK(cudaGetLastError());
  if (launch_reduce(t->hpart, hb, trk::kHeadCols, t->hsum)) return 1;
  CUDA_OK(cudaMemcpyAsync(t->grads + t->b_off[t->nconv - 1], t->hsum, 32 * 4, cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t->grads + t->w_off[t->nconv], t->hsum + 32, 33 * 4, cudaMemcpyDeviceToDevice, st));

  // backward: weight gradient of every conv, input gradient of every conv but conv0_a
  const int ntiles = g.data_rows / trk::kTileRows;
  for (int l = t->nconv - 1; l >= 0; --l) {
    if ((l == 0 ? launch_wgrad<2>(t, g, l) : launch_wgrad<4>(t, g, l))) return 1;
    if (l == 0) break;
    trk::ConvArgs a{};
    a.x = t->gout[0];
    a.w = t->wt[l];
    a.res = t->gres;
    a.mask_in = t->mask[l];
    a.out = t->gout[1];
    a.bias_part = t->bpart;
    a.g = g;
    if (l % 2 == 1 ? launch_conv<4, trk::kBwdA>(t, a) : launch_conv<4, trk::kBwdB>(t, a)) return 1;
    if (launch_reduce(t->bpart, ntiles, 32, t->grads + t->b_off[l - 1])) return 1;
    std::swap(t->gout[0], t->gout[1]);
  }
  *hb_out = hb;
  return 0;
}

// run_device on a batch copied from the host, and the loss summed on the host.
int run(FfnTrainer* t, const float* seed, const float* image, const float* labels, const float* loss_weights, int batch,
        double* loss_out) {
  if (!seed || !image || !labels) return fail("null argument");
  if (batch < 1 || batch > t->max_batch)
    return fail("batch " + std::to_string(batch) + " outside [1, " + std::to_string(t->max_batch) + "]");
  CUDA_OK(cudaSetDevice(t->device));
  cudaStream_t st = cudaStreamPerThread;
  const size_t nv = (size_t)batch * t->g.V;
  CUDA_OK(cudaMemcpyAsync(t->seed, seed, nv * 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t->image, image, nv * 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t->labels, labels, nv * 4, cudaMemcpyHostToDevice, st));
  if (loss_weights) CUDA_OK(cudaMemcpyAsync(t->lw, loss_weights, nv * 4, cudaMemcpyHostToDevice, st));
  int hb = 0;
  if (run_device(t, loss_weights != nullptr, batch, &hb)) return 1;
  std::vector<double> lp(hb);
  CUDA_OK(cudaMemcpyAsync(lp.data(), t->lpart, hb * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  double s = 0.0;
  for (double v : lp) s += v;
  if (loss_out) *loss_out = s / (double)nv;
  return 0;
}

// Enqueues the optimizer step at learning_rate on the gradients in t->grads, and advances the global step and Adam's
// beta powers (the host forms Adam's alpha from them, in float32).
int launch_update(FfnTrainer* t, float learning_rate) {
  trk::UpdateArgs u{};
  u.w = t->params;
  u.a = t->slot_a;
  u.b = t->slot_b;
  u.grad = t->grads;
  u.n = t->nparam;
  u.optimizer = t->desc.optimizer;
  u.clip = t->desc.max_gradient_entry_mag;
  u.lr = learning_rate;
  u.momentum = t->desc.momentum;
  u.one_minus_b1 = 1.0f - t->desc.beta1;
  u.one_minus_b2 = 1.0f - t->desc.beta2;
  u.alpha = learning_rate * std::sqrt(1.0f - t->beta2_power) / (1.0f - t->beta1_power);
  u.eps = t->desc.epsilon;
  trk::update<<<t->sm_count * 4, 256, 0, cudaStreamPerThread>>>(u);
  CUDA_OK(cudaGetLastError());
  t->global_step++;
  if (t->desc.optimizer == FFN_OPT_ADAM) {
    t->beta1_power = t->beta1_power * t->desc.beta1;
    t->beta2_power = t->beta2_power * t->desc.beta2;
  }
  return 0;
}

// The loss of one step: the head's partial sums added in the order ffn_trainer_step adds them on the host.
__global__ void sum_loss(const double* part, int n, double nv, double* out) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s = __dadd_rn(s, part[i]);
  *out = __ddiv_rn(s, nv);
}

int copy_params(const FfnTrainer* t, const float* src, float* const* w, float* const* b) {
  for (int l = 0; l <= t->nconv; ++l) {
    const size_t nw = l < t->nconv ? (size_t)27 * cin_of(l) * 32 : 32;
    if (w && w[l]) CUDA_OK(cudaMemcpyAsync(w[l], src + t->w_off[l], nw * 4, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    if (b && b[l])
      CUDA_OK(cudaMemcpyAsync(b[l], src + t->b_off[l], (l < t->nconv ? 32 : 1) * 4, cudaMemcpyDeviceToHost,
                              cudaStreamPerThread));
  }
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

// The trainer's state blob: the header names what the payload's layout depends on; the payload is the step count and
// Adam's beta powers, then params, slot_a and slot_b in the device layout (w_off / b_off).
constexpr uint64_t kStateMagic = 0x31545352544E4646ull;   // "FFNTRST1", little-endian
constexpr uint32_t kStateVersion = 1;

struct Scalars {
  int64_t global_step;
  float beta1_power, beta2_power;
};

blob::Header state_header(const FfnTrainer* t) {
  blob::Header h;
  h.add("depth", t->nconv / 2);
  h.add("optimizer", t->desc.optimizer);
  h.add("nparam", t->nparam);
  return h;
}

std::vector<blob::Section> state_sections(FfnTrainer* t, Scalars* sc) {
  const size_t pb = (size_t)t->nparam * 4;
  return {{sc, sizeof(Scalars), true}, {t->params, pb, false}, {t->slot_a, pb, false}, {t->slot_b, pb, false}};
}

}  // namespace

extern "C" {

int ffn_trainer_create(int device, const FfnModelDesc* model, const float* const* weights_dhwio,
                       const float* const* biases, const FfnTrainDesc* desc, FfnTrainer** out) {
  if (!model || !weights_dhwio || !biases || !desc || !out) return fail("null argument");
  if (check_model(model)) return 1;
  if (desc->optimizer != FFN_OPT_SGD && desc->optimizer != FFN_OPT_MOMENTUM && desc->optimizer != FFN_OPT_ADAM)
    return fail("unknown optimizer (sgd, momentum and adam are supported)");
  if (desc->max_batch < 1) return fail("max_batch must be at least 1");
  TGeom g{};
  g.Z = model->fov_zyx[0];
  g.Y = model->fov_zyx[1];
  g.X = model->fov_zyx[2];
  g.P = g.X + 2;
  g.P2 = (g.Y + 2) * g.P;
  g.Vp = (g.Z + 2) * g.P2;
  g.V = g.Z * g.Y * g.X;
  const int halo = g.P2 + g.P + 1;
  g.guard = (halo + trk::kTileRows) / trk::kTileRows * trk::kTileRows;
  const long long rows = (long long)g.guard * 2 + ((long long)desc->max_batch * g.Vp + trk::kSplitRows) +
                         trk::kKTile + 8;
  if (rows * 32 >= (1ll << 31)) return fail("max_batch x field of view too large for the trainer's row space");
  g.rows = (int)rows;
  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  // the conv kernels' dynamic staging plus their static shared memory (the bias-gradient exchange)
  const std::pair<const void*, int> convs[] = {{(const void*)trk::conv<2, trk::kFwdA>, 2},
                                               {(const void*)trk::conv<4, trk::kFwdA>, 4},
                                               {(const void*)trk::conv<4, trk::kFwdB>, 4},
                                               {(const void*)trk::conv<4, trk::kBwdA>, 4},
                                               {(const void*)trk::conv<4, trk::kBwdB>, 4}};
  size_t conv_static[5];
  for (int i = 0; i < 5; ++i) {
    cudaFuncAttributes attr{};
    CUDA_OK(cudaFuncGetAttributes(&attr, convs[i].first));
    conv_static[i] = attr.sharedSizeBytes;
    if (conv_smem(g, convs[i].second) + attr.sharedSizeBytes > prop.sharedMemPerBlockOptin)
      return fail("field of view too wide for the conv kernel's staging");
  }

  std::unique_ptr<FfnTrainer> t(new FfnTrainer());
  t->device = device;
  t->sm_count = prop.multiProcessorCount;
  t->nconv = 2 * model->depth;
  t->max_batch = desc->max_batch;
  t->desc = *desc;
  t->g = g;
  t->beta1_power = desc->beta1;
  t->beta2_power = desc->beta2;
  for (int l = 0; l <= t->nconv; ++l) {
    t->w_off.push_back(t->nparam);
    t->nparam += l < t->nconv ? 27 * cin_of(l) * 32 : 32;
    t->b_off.push_back(t->nparam);
    t->nparam += l < t->nconv ? 32 : 1;
  }
  std::vector<float> h(t->nparam);
  for (int l = 0; l <= t->nconv; ++l) {
    const int nw = l < t->nconv ? 27 * cin_of(l) * 32 : 32, nb = l < t->nconv ? 32 : 1;
    if (!weights_dhwio[l] || !biases[l]) return fail("null weight or bias array");
    std::copy(weights_dhwio[l], weights_dhwio[l] + nw, h.begin() + t->w_off[l]);
    std::copy(biases[l], biases[l] + nb, h.begin() + t->b_off[l]);
  }
  DevBufs& m = t->mem;
  const size_t R = g.rows;
  if (m.get(&t->params, t->nparam) || m.get(&t->grads, t->nparam, true) || m.get(&t->slot_a, t->nparam, true) ||
      m.get(&t->slot_b, t->nparam, true))
    return 1;
  CUDA_OK(cudaMemcpy(t->params, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  t->wf.assign(t->nconv, nullptr);
  t->wt.assign(t->nconv, nullptr);
  t->x.assign(t->nconv, nullptr);
  t->mask.assign(t->nconv + 1, nullptr);
  for (int l = 0; l < t->nconv; ++l) {
    if (m.get(&t->wf[l], (size_t)27 * kc_of(l) * 256, true) || m.get(&t->x[l], (size_t)kc_of(l) * 8 * R, true) ||
        m.get(&t->mask[l + 1], R, true) || (l > 0 && m.get(&t->wt[l], (size_t)27 * 4 * 256, true)))
      return 1;
  }
  const size_t nv = (size_t)t->max_batch * g.V;
  TGeom gmax = g;
  gmax.batch = t->max_batch;
  gmax.data_rows = data_rows(gmax, t->max_batch);
  const int hb = head_blocks(gmax, t->max_batch);
  if (m.get(&t->res, R * 32, true) || m.get(&t->gres, R * 32, true) || m.get(&t->gout[0], R * 32, true) ||
      m.get(&t->gout[1], R * 32, true) || m.get(&t->seed, nv) || m.get(&t->image, nv) || m.get(&t->labels, nv) ||
      m.get(&t->lw, nv) || m.get(&t->logits, nv) || m.get(&t->dl, nv) ||
      m.get(&t->wpart, (size_t)gmax.data_rows / trk::kSplitRows * 27 * 32 * 32) ||
      m.get(&t->bpart, (size_t)gmax.data_rows / trk::kTileRows * 32) || m.get(&t->hpart, (size_t)hb * trk::kHeadCols) ||
      m.get(&t->hsum, trk::kHeadCols) || m.get(&t->lpart, hb))
    return 1;
  // The dynamic shared-memory cap belongs to the kernel, not to this trainer: it is set to all a block may use, so that
  // creating a trainer of a narrower field of view never lowers it below a wider trainer's launches.
  for (int i = 0; i < 5; ++i)
    CUDA_OK(cudaFuncSetAttribute(convs[i].first, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(prop.sharedMemPerBlockOptin - conv_static[i])));
  CUDA_OK(cudaFuncSetAttribute(trk::wgrad<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, trk::WgradShape<2>::kSmem));
  CUDA_OK(cudaFuncSetAttribute(trk::wgrad<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, trk::WgradShape<4>::kSmem));
  CUDA_OK(cudaDeviceSynchronize());
  *out = t.release();
  return 0;
}

void ffn_trainer_destroy(FfnTrainer* t) { delete t; }

int ffn_trainer_step(FfnTrainer* t, const float* seed, const float* image, const float* labels,
                     const float* loss_weights, int batch, float learning_rate, float* logits_out, double* loss_out) {
  if (!t) return fail("null trainer");
  if (run(t, seed, image, labels, loss_weights, batch, loss_out)) return 1;
  if (launch_update(t, learning_rate)) return 1;
  if (logits_out)
    CUDA_OK(cudaMemcpyAsync(logits_out, t->logits, (size_t)batch * t->g.V * 4, cudaMemcpyDeviceToHost,
                            cudaStreamPerThread));
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

int ffn_trainer_gradients(FfnTrainer* t, const float* seed, const float* image, const float* labels,
                          const float* loss_weights, int batch, float* dlogits_out, float* const* weight_grads,
                          float* const* bias_grads, double* loss_out) {
  if (!t) return fail("null trainer");
  if (run(t, seed, image, labels, loss_weights, batch, loss_out)) return 1;
  if (dlogits_out)
    CUDA_OK(cudaMemcpyAsync(dlogits_out, t->dl, (size_t)batch * t->g.V * 4, cudaMemcpyDeviceToHost, cudaStreamPerThread));
  return copy_params(t, t->grads, weight_grads, bias_grads);
}

int ffn_trainer_train(FfnTrainer* t, FfnExamples* ex, const FfnExampleCoord* coords, int64_t n_coords, int n_steps,
                      const float* learning_rate, double* losses_out, int64_t* n_consumed) {
  if (!t || !ex || !coords || (n_steps > 0 && (!learning_rate || !losses_out))) return fail("null argument");
  if (n_steps < 0) return fail("negative n_steps");
  const int fov[3] = {t->g.Z, t->g.Y, t->g.X};
  if (examples_check_trainer(ex, t->device, fov, t->max_batch)) return 1;
  const int batch = examples_batch(ex);
  if (n_coords < (int64_t)n_steps * batch)
    return fail("a step may take one stream entry per element: pass at least n_steps * batch (" +
                std::to_string((int64_t)n_steps * batch) + ") entries");
  CUDA_OK(cudaSetDevice(t->device));
  cudaStream_t st = cudaStreamPerThread;
  DevBufs tmp;
  double* losses = nullptr;
  if (tmp.get(&losses, n_steps) || examples_upload(ex, coords, (int64_t)n_steps * batch)) return 1;
  const double nv = (double)((size_t)batch * t->g.V);
  for (int i = 0; i < n_steps; ++i) {
    int hb = 0;
    if (examples_advance(ex, t->seed, t->image, t->labels) || run_device(t, false, batch, &hb)) return 1;
    sum_loss<<<1, 1, 0, st>>>(t->lpart, hb, nv, losses + i);
    CUDA_OK(cudaGetLastError());
    if (launch_update(t, learning_rate[i]) || examples_paste(ex, t->logits)) return 1;
  }
  if (n_steps) CUDA_OK(cudaMemcpyAsync(losses_out, losses, n_steps * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return examples_finish(ex, n_consumed);
}

int ffn_trainer_get_weights(FfnTrainer* t, float* const* weights_dhwio, float* const* biases, int64_t* global_step) {
  if (!t) return fail("null trainer");
  CUDA_OK(cudaSetDevice(t->device));
  if (global_step) *global_step = t->global_step;
  return copy_params(t, t->params, weights_dhwio, biases);
}

}  // extern "C"

extern "C" {

int ffn_trainer_get_state(FfnTrainer* t, void* out, int64_t cap, int64_t* n) {
  if (!t) return fail("null trainer");
  CUDA_OK(cudaSetDevice(t->device));
  Scalars sc{t->global_step, t->beta1_power, t->beta2_power};
  return blob::get(kStateMagic, kStateVersion, state_header(t), state_sections(t, &sc), out, cap, n);
}

int ffn_trainer_set_state(FfnTrainer* t, const void* state, int64_t n) {
  if (!t) return fail("null trainer");
  Scalars sc{};
  const std::vector<blob::Section> secs = state_sections(t, &sc);
  const uint8_t* payload = nullptr;
  if (blob::open(state, n, kStateMagic, kStateVersion, state_header(t), secs, "trainer", &payload)) return 1;
  std::memcpy(&sc, payload, sizeof(Scalars));
  if (sc.global_step < 0) return fail("trainer state with a negative global step");
  CUDA_OK(cudaSetDevice(t->device));
  if (blob::put(payload, secs)) return 1;
  t->global_step = sc.global_step;
  t->beta1_power = sc.beta1_power;
  t->beta2_power = sc.beta2_power;
  return 0;
}

}  // extern "C"
