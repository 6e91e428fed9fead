// examples.cu — the training example loop of train.py on the device (ffn_examples_*): per batch element a training
// patch, its seed canvas and the state of its move policy, and the steps that ffn_trainer_train runs between training
// steps (examples_advance, examples_paste).

#include <cmath>
#include <memory>
#include <string>
#include <vector>

#include "example_kernels.cuh"
#include "host.cuh"

using namespace ffn;

struct FfnExamples {
  DevBufs mem;
  int device = 0, n_volumes = 0;
  exk::Args a{};
  std::vector<FfnExampleVolume> vols;   // shapes only (the host pointers are not kept)
  FfnExampleDesc desc{};
  int64_t coords_cap = 0;
  FfnExampleCoord* coords = nullptr;
  float *bseed = nullptr, *bimage = nullptr, *blabels = nullptr, *logits = nullptr;
  int64_t total = 0;                    // examples loaded since creation, as of the last call
  ~FfnExamples() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
  }
};

namespace ffn {

namespace {

int grid_blocks(long long n) { return (int)std::min<long long>((n + exk::kThreads - 1) / exk::kThreads, 128); }

// Every entry must name a volume, crop inside it, and permute and reflect only the axes the description allows.
int check_coords(const FfnExamples* ex, const FfnExampleCoord* coords, int64_t n) {
  const exk::Args& a = ex->a;
  for (int64_t i = 0; i < n; ++i) {
    const FfnExampleCoord& c = coords[i];
    const std::string at = "stream entry " + std::to_string(i) + ": ";
    if (c.volume < 0 || c.volume >= ex->n_volumes) return fail(at + "unknown volume " + std::to_string(c.volume));
    const FfnExampleVolume& v = ex->vols[c.volume];
    int seen = 0;
    for (int d = 0; d < 3; ++d) {
      const long long start = (long long)c.center_xyz[2 - d] - (a.S[d] - 1) / 2;
      if (start < 0 || start + a.S[d] > v.image_shape_zyx[d] || start + a.S[d] > v.label_shape_zyx[d])
        return fail(at + "the crop of centre (" + std::to_string(c.center_xyz[0]) + ", " +
                    std::to_string(c.center_xyz[1]) + ", " + std::to_string(c.center_xyz[2]) +
                    ") leaves volume " + std::to_string(c.volume));
      const int p = c.permutation_zyx[d];
      if (p < 0 || p > 2 || (seen & (1 << p))) return fail(at + "permutation_zyx is not a permutation of (0, 1, 2)");
      seen |= 1 << p;
      if (p != d && !(ex->desc.permutable_zyx[d] && ex->desc.permutable_zyx[p]))
        return fail(at + "permutes an axis that is not permutable");
      if (c.reflect_zyx[d] && !ex->desc.reflectable_zyx[d]) return fail(at + "reflects an axis that is not reflectable");
    }
  }
  return 0;
}

}  // namespace

int examples_check_trainer(const FfnExamples* ex, int device, const int fov_zyx[3], int max_batch) {
  if (ex->device != device) return fail("the examples and the trainer are on different devices");
  for (int d = 0; d < 3; ++d)
    if (ex->a.F[d] != fov_zyx[d]) return fail("the examples' field of view differs from the trainer's");
  if (ex->a.batch > max_batch)
    return fail("examples batch " + std::to_string(ex->a.batch) + " above the trainer's max_batch " +
                std::to_string(max_batch));
  return 0;
}

int examples_batch(const FfnExamples* ex) { return ex->a.batch; }

// Copies the next n stream entries to the device (checked first) and restarts the count of entries taken.
int examples_upload(FfnExamples* ex, const FfnExampleCoord* coords, int64_t n) {
  if (!coords) return fail("null coords");
  if (n >= (1ll << 31)) return fail("too many stream entries in one call");
  if (check_coords(ex, coords, n)) return 1;
  if (n > ex->coords_cap) {
    ex->mem.release(ex->coords);
    ex->coords_cap = 0;
    if (ex->mem.get(&ex->coords, n)) return 1;
    ex->coords_cap = n;
    ex->a.coords = ex->coords;
  }
  cudaStream_t st = cudaStreamPerThread;
  CUDA_OK(cudaMemcpyAsync(ex->coords, coords, n * sizeof(FfnExampleCoord), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(ex->a.used, 0, sizeof(int), st));
  return 0;
}

// One step's batch: resume every generator, load the exhausted elements' next examples, crop [batch][F] into the
// three outputs (device pointers).
int examples_advance(FfnExamples* ex, float* seed, float* image, float* labels) {
  cudaStream_t st = cudaStreamPerThread;
  const exk::Args& a = ex->a;
  exk::resume<<<1, 32 * std::min(a.batch, exk::kMaxWarps), 0, st>>>(a);
  CUDA_OK(cudaGetLastError());
  exk::load<<<dim3(grid_blocks(a.SV), a.batch), exk::kThreads, 0, st>>>(a);
  CUDA_OK(cudaGetLastError());
  exk::crop<<<dim3(grid_blocks(a.FV), a.batch), exk::kThreads, 0, st>>>(a, seed, image, labels);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// Pastes logits [batch][F] (device) into the seeds.
int examples_paste(FfnExamples* ex, const float* logits) {
  exk::paste<<<dim3(grid_blocks(ex->a.FV), ex->a.batch), exk::kThreads, 0, cudaStreamPerThread>>>(ex->a, logits);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// After a synchronisation: the entries taken since the upload, and the overflow check of the queues.
int examples_finish(FfnExamples* ex, int64_t* n_consumed) {
  int used = 0, error = 0;
  long long total = 0;
  CUDA_OK(cudaMemcpy(&used, ex->a.used, sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(&error, ex->a.error, sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(&total, ex->a.total, sizeof(long long), cudaMemcpyDeviceToHost));
  if (error) return fail("a max_pred_moves queue exceeded its bound");
  ex->total = total;
  if (n_consumed) *n_consumed = used;
  return 0;
}

}  // namespace ffn

extern "C" {

int ffn_examples_create(int device, const FfnModelDesc* model, const FfnExampleDesc* desc,
                        const FfnExampleVolume* volumes, int n_volumes, FfnExamples** out) {
  if (!model || !desc || !out || (n_volumes > 0 && !volumes)) return fail("null argument");
  if (check_model(model)) return 1;
  if (n_volumes < 1) return fail("no volumes");
  if (desc->policy != FFN_FOV_FIXED && desc->policy != FFN_FOV_MAX_PRED_MOVES)
    return fail("unknown fov policy (fixed and max_pred_moves are supported)");
  if (desc->fov_moves < 1) return fail("fov_moves must be at least 1");
  if (!(desc->seed_pad > 0.f && desc->seed_pad < 1.f)) return fail("seed_pad must lie in (0, 1)");
  if (!((double)desc->seed_logit_centre >= desc->seed_threshold))
    return fail("the fresh seed's centre fails the threshold: every example would be dropped at its first move "
                "(use a threshold whose logit is at most " + std::to_string(desc->seed_logit_centre) + ")");
  if (desc->batch < 1 || desc->batch > exk::kMaxWarps)
    return fail("batch must lie in [1, " + std::to_string(exk::kMaxWarps) + "]");
  if (desc->policy == FFN_FOV_FIXED && desc->n_shifts > 0 && !desc->shifts_zyx) return fail("null shifts");
  if (desc->n_shifts < 0) return fail("negative n_shifts");

  std::unique_ptr<FfnExamples> ex(new FfnExamples());
  exk::Args& a = ex->a;
  a.policy = desc->policy;
  a.moves = desc->fov_moves + (desc->policy == FFN_FOV_MAX_PRED_MOVES ? 1 : 0);
  a.batch = desc->batch;
  a.SV = a.FV = 1;
  int cells = 1;
  for (int d = 0; d < 3; ++d) {
    a.F[d] = model->fov_zyx[d];
    a.D[d] = model->deltas_zyx[d];
    a.S[d] = a.F[d] + 2 * a.D[d] * a.moves;
    a.SV *= a.S[d];
    a.FV *= a.F[d];
    if (a.D[d] > 0) cells *= 2 * a.moves + 1;
  }
  if (a.SV >= (1ll << 31)) return fail("training patches of 2^31 or more voxels");
  for (int d = 0; d < 3; ++d)
    for (int k = 0; k < 3; ++k)
      if (desc->permutable_zyx[d] && desc->permutable_zyx[k] && a.S[d] != a.S[k])
        return fail("permutable axes must have equal patch extents, got " + std::to_string(a.S[d]) + " and " +
                    std::to_string(a.S[k]));
  if (desc->policy == FFN_FOV_FIXED)
    for (int i = 0; i < desc->n_shifts; ++i)
      for (int d = 0; d < 3; ++d)
        if (std::abs(desc->shifts_zyx[i * 3 + d]) > a.D[d] * a.moves) return fail("a shift leaves the patch");
  // Every yield of max_pred_moves marks a new quantised cell; offsets within max_radius = deltas * moves quantise to
  // [-moves, moves] on axes of nonzero delta and to 0 elsewhere, so an example yields at most `cells` times, and each
  // yield queues at most 6 offsets after the centre.
  a.side = 2 * a.moves + 1;
  a.qcap = 6 * cells + 1;
  a.pad_logit = desc->seed_logit_pad;
  a.centre_logit = desc->seed_logit_centre;
  a.seed_thr = desc->seed_threshold;
  a.label_thr = desc->label_threshold;
  a.n_shifts = desc->policy == FFN_FOV_FIXED ? desc->n_shifts : 0;
  ex->desc = *desc;
  ex->desc.shifts_zyx = nullptr;
  ex->n_volumes = n_volumes;

  cudaDeviceProp prop{};
  if (use_device(device, &prop)) return 1;
  ex->device = device;
  DevBufs& m = ex->mem;
  std::vector<exk::Vol> dv(n_volumes);
  for (int i = 0; i < n_volumes; ++i) {
    const FfnExampleVolume& v = volumes[i];
    if (!v.image || !v.labels) return fail("null volume");
    size_t ni = 1, nl = 1;
    for (int d = 0; d < 3; ++d) {
      if (v.image_shape_zyx[d] < 1 || v.label_shape_zyx[d] < 1) return fail("empty volume");
      ni *= v.image_shape_zyx[d];
      nl *= v.label_shape_zyx[d];
      dv[i].ishape[d] = v.image_shape_zyx[d];
      dv[i].lshape[d] = v.label_shape_zyx[d];
    }
    uint8_t* im = nullptr;
    long long* lb = nullptr;
    if (m.get(&im, ni) || m.get(&lb, nl)) return 1;
    CUDA_OK(cudaMemcpy(im, v.image, ni, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(lb, v.labels, nl * 8, cudaMemcpyHostToDevice));
    dv[i].image = im;
    dv[i].labels = lb;
    dv[i].offset = v.offset;
    dv[i].scale = v.scale;
    ex->vols.push_back(v);
    ex->vols.back().image = nullptr;
    ex->vols.back().labels = nullptr;
  }
  exk::Vol* vd = nullptr;
  int* shifts = nullptr;
  const size_t B = a.batch;
  if (m.get(&vd, n_volumes) || m.get(&shifts, std::max(a.n_shifts, 1) * 3) || m.get(&a.seed, B * a.SV, true) ||
      m.get(&a.image, B * a.SV, true) || m.get(&a.labels, B * a.SV, true) || m.get(&a.st, B, true) ||
      m.get(&a.queue, B * a.qcap * 3, true) || m.get(&a.done, B * a.side * a.side * a.side, true) ||
      m.get(&a.used, 1, true) || m.get(&a.entry, B, true) || m.get(&a.total, 1, true) || m.get(&a.error, 1, true) ||
      m.get(&ex->bseed, B * a.FV) || m.get(&ex->bimage, B * a.FV) || m.get(&ex->blabels, B * a.FV) ||
      m.get(&ex->logits, B * a.FV))
    return 1;
  CUDA_OK(cudaMemcpy(vd, dv.data(), n_volumes * sizeof(exk::Vol), cudaMemcpyHostToDevice));
  if (a.n_shifts) CUDA_OK(cudaMemcpy(shifts, desc->shifts_zyx, a.n_shifts * 3 * sizeof(int), cudaMemcpyHostToDevice));
  a.vols = vd;
  a.shifts = shifts;
  CUDA_OK(cudaDeviceSynchronize());
  *out = ex.release();
  return 0;
}

void ffn_examples_destroy(FfnExamples* ex) { delete ex; }

int ffn_examples_next(FfnExamples* ex, const FfnExampleCoord* coords, int64_t n_coords, float* seed_out,
                      float* image_out, float* labels_out, int32_t* offsets_zyx_out, int64_t* example_out,
                      int64_t* n_consumed) {
  if (!ex) return fail("null examples");
  if (n_coords < ex->a.batch)
    return fail("a step may take one stream entry per element: pass at least batch (" + std::to_string(ex->a.batch) +
                ") entries");
  CUDA_OK(cudaSetDevice(ex->device));
  if (examples_upload(ex, coords, ex->a.batch) || examples_advance(ex, ex->bseed, ex->bimage, ex->blabels)) return 1;
  cudaStream_t st = cudaStreamPerThread;
  const size_t nb = (size_t)ex->a.batch * ex->a.FV * 4;
  if (seed_out) CUDA_OK(cudaMemcpyAsync(seed_out, ex->bseed, nb, cudaMemcpyDeviceToHost, st));
  if (image_out) CUDA_OK(cudaMemcpyAsync(image_out, ex->bimage, nb, cudaMemcpyDeviceToHost, st));
  if (labels_out) CUDA_OK(cudaMemcpyAsync(labels_out, ex->blabels, nb, cudaMemcpyDeviceToHost, st));
  std::vector<exk::State> s(ex->a.batch);
  CUDA_OK(cudaMemcpyAsync(s.data(), ex->a.st, s.size() * sizeof(exk::State), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  for (int e = 0; e < ex->a.batch; ++e) {
    for (int d = 0; d < 3; ++d)
      if (offsets_zyx_out) offsets_zyx_out[e * 3 + d] = s[e].off[d];
    if (example_out) example_out[e] = s[e].example;
  }
  return examples_finish(ex, n_consumed);
}

int ffn_examples_update(FfnExamples* ex, const float* logits) {
  if (!ex || !logits) return fail("null argument");
  CUDA_OK(cudaSetDevice(ex->device));
  CUDA_OK(cudaMemcpyAsync(ex->logits, logits, (size_t)ex->a.batch * ex->a.FV * 4, cudaMemcpyHostToDevice,
                          cudaStreamPerThread));
  if (examples_paste(ex, ex->logits)) return 1;
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

int ffn_examples_read_seeds(FfnExamples* ex, float* out) {
  if (!ex || !out) return fail("null argument");
  CUDA_OK(cudaSetDevice(ex->device));
  CUDA_OK(cudaMemcpyAsync(out, ex->a.seed, (size_t)ex->a.batch * ex->a.SV * 4, cudaMemcpyDeviceToHost,
                          cudaStreamPerThread));
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

}  // extern "C"
