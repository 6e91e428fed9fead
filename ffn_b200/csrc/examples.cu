// examples.cu — the training example loop of train.py on the device (ffn_examples_*): per batch element a training
// patch, its seed canvas and the state of its move policy, and the steps that ffn_trainer_train runs between training
// steps (examples_advance, examples_paste).

#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "example_kernels.cuh"
#include "host.cuh"
#include "state_blob.cuh"

using namespace ffn;

struct FfnExamples {
  DevBufs mem;
  int device = 0, n_volumes = 0;
  exk::Args a{};
  std::vector<FfnExampleVolume> vols;   // shapes only (the host pointers are not kept)
  std::vector<int> shifts;              // the fixed policy's shifts, [n_shifts][3]
  FfnExampleDesc desc{};
  int64_t coords_cap = 0;
  FfnExampleCoord* coords = nullptr;
  float *bseed = nullptr, *bimage = nullptr, *blabels = nullptr, *logits = nullptr;
  int64_t total = 0;                    // examples loaded since creation, as of the last call
  int n_radii = 1;                      // moves are counted at radii 0 .. n_radii - 1
  ~FfnExamples() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
  }
};

namespace ffn {

namespace {

int grid_blocks(long long n) { return (int)std::min<long long>((n + exk::kThreads - 1) / exk::kThreads, 128); }

// Every entry must name a volume, crop inside it, and permute and reflect only the axes the description allows.
// Messages name entry i as `what` i.
int check_coords(const FfnExamples* ex, const FfnExampleCoord* coords, int64_t n, const char* what = "stream entry ") {
  const exk::Args& a = ex->a;
  for (int64_t i = 0; i < n; ++i) {
    const FfnExampleCoord& c = coords[i];
    const std::string at = what + std::to_string(i) + ": ";
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

// The loop's state blob.  The header holds everything the payload's meaning depends on; the payload is the per-element
// device state in the order of state_sections.  Per-step scratch (used, entry, tk_part, tk_arrived, tk_slot, the
// staging buffers and the uploaded coords) is rewritten by every step before it is read, and is not saved.
constexpr uint64_t kStateMagic = 0x31545358454E4646ull;   // "FFNEXST1", little-endian
constexpr uint32_t kStateVersion = 1;

blob::Header state_header(const FfnExamples* ex) {
  const exk::Args& a = ex->a;
  blob::Header h;
  h.add("policy", a.policy);
  h.add3("field of view", a.F);
  h.add3("deltas", a.D);
  h.add("moves", a.moves);
  h.add3("patch extent", a.S);
  h.add("batch", a.batch);
  h.add("qcap", a.qcap);
  h.add("side", a.side);
  h.add("n_radii", ex->n_radii);
  h.add("number of shifts", a.n_shifts);
  for (int i = 0; i < a.n_shifts; ++i) h.add3("shift list", ex->shifts.data() + 3 * i);
  h.add_bits("seed threshold", a.seed_thr);
  h.add_bits("label threshold", a.label_thr);
  h.add_bits("eval threshold", a.eval_thr);
  h.add_bits("pad logit", a.pad_logit);
  h.add_bits("centre logit", a.centre_logit);
  h.add3("permutable axes", ex->desc.permutable_zyx);
  h.add3("reflectable axes", ex->desc.reflectable_zyx);
  h.add("number of volumes", ex->n_volumes);
  for (int i = 0; i < ex->n_volumes; ++i) {
    const FfnExampleVolume& v = ex->vols[i];
    const std::string n = "volume " + std::to_string(i);
    h.add3(n + " image shape", v.image_shape_zyx);
    h.add3(n + " label shape", v.label_shape_zyx);
    h.add_bits(n + " offset", v.offset);
    h.add_bits(n + " scale", v.scale);
  }
  return h;
}

std::vector<blob::Section> state_sections(const FfnExamples* ex) {
  const exk::Args& a = ex->a;
  const size_t B = a.batch, patch = B * a.SV * 4;
  const size_t tk = (exk::kTkMoves + 3 * ex->n_radii) * sizeof(long long);
  const size_t queue = B * a.qcap * 3 * sizeof(int), done = B * a.side * a.side * a.side;
  const size_t ring = exk::kRing * (size_t)exk::plane_floats(a.E) * 4;
  return {{a.st, B * sizeof(exk::State), false},
          {a.ecoord, B * sizeof(FfnExampleCoord), false},
          {a.total, sizeof(long long), false},
          {a.tk, tk, false},
          {a.tk_loss, sizeof(double), false},
          {a.queue, queue, false},
          {a.done, done, false},
          {a.seed, patch, false},
          {a.image, patch, false},
          {a.labels, patch, false},
          {a.ring, ring, false},
          {a.ring_coord, exk::kRing * sizeof(FfnExampleCoord), false}};
}

// The checks of a payload that has passed blob::open: every value a kernel uses as an index or a bound lies in range.
int check_state(const FfnExamples* ex, const uint8_t* payload, const std::vector<blob::Section>& secs) {
  const exk::Args& a = ex->a;
  std::vector<exk::State> st(a.batch);
  std::vector<FfnExampleCoord> ec(a.batch);
  long long total = 0;
  std::vector<long long> tk(secs[3].bytes / sizeof(long long));
  std::memcpy(st.data(), payload + blob::offset(secs, 0), secs[0].bytes);
  std::memcpy(ec.data(), payload + blob::offset(secs, 1), secs[1].bytes);
  std::memcpy(&total, payload + blob::offset(secs, 2), sizeof(long long));
  std::memcpy(tk.data(), payload + blob::offset(secs, 3), secs[3].bytes);
  if (total < 0) return fail("example loop state with a negative example count");
  for (size_t i = 0; i < tk.size(); ++i)
    if (tk[i] < 0) return fail("example loop state with a negative tracker counter");
  const int* queue = reinterpret_cast<const int*>(payload + blob::offset(secs, 5));
  for (int e = 0; e < a.batch; ++e) {
    const exk::State& s = st[e];
    const std::string at = "example loop state, element " + std::to_string(e) + ": ";
    if (s.active != 0 && s.active != 1) return fail(at + "active is neither 0 nor 1");
    // fixed resumes at shift k - 1 (0: the centre); k = n_shifts + 1 once the last shift was yielded or exhausted
    if (s.k < 0 || s.k > a.n_shifts + 1)
      return fail(at + "k = " + std::to_string(s.k) + " outside [0, " + std::to_string(a.n_shifts + 1) + "]");
    if (s.head < 0 || s.head > s.tail || s.tail > a.qcap)
      return fail(at + "queue head " + std::to_string(s.head) + " and tail " + std::to_string(s.tail) +
                  " outside 0 <= head <= tail <= " + std::to_string(a.qcap));
    for (int d = 0; d < 3; ++d)
      if (std::abs(s.off[d]) > a.D[d] * a.moves) return fail(at + "offset outside deltas * moves");
    // a queued offset is a yielded offset plus a face voxel at most deltas away
    for (int j = 0; j < s.tail; ++j)
      for (int d = 0; d < 3; ++d)
        if (std::abs(queue[((size_t)e * a.qcap + j) * 3 + d]) > a.D[d] * (a.moves + 1))
          return fail(at + "queued offset outside deltas * (moves + 1)");
    if (s.active) {
      if (s.example < 0 || s.example >= total) return fail(at + "example index outside the examples loaded");
      const std::string what = "example loop state, the example of element " + std::to_string(e) + ": entry ";
      if (check_coords(ex, &ec[e], 1, what.c_str())) return 1;
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

// One step's batch: resume every generator, track the examples it finished, load the exhausted elements' next examples, crop [batch][F] into the
// three outputs (device pointers).
int examples_advance(FfnExamples* ex, float* seed, float* image, float* labels) {
  cudaStream_t st = cudaStreamPerThread;
  const exk::Args& a = ex->a;
  exk::resume<<<1, 32 * std::min(a.batch, exk::kMaxWarps), 0, st>>>(a);
  CUDA_OK(cudaGetLastError());
  exk::track<<<dim3(a.tk_blocks, a.batch), exk::kThreads, 0, st>>>(a);
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
  if (!std::isfinite(desc->eval_threshold)) return fail("eval_threshold must be finite");

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
  a.eval_thr = desc->eval_threshold;
  a.EV = 1;
  for (int d = 0; d < 3; ++d) {
    a.E[d] = a.F[d] + 2 * a.D[d] * desc->fov_moves;   // train.py's train_eval_size
    a.ecrop[d] = a.S[d] / 2 - a.E[d] / 2;             // mask.crop_and_pad(..., (0, 0, 0), E)
    a.EV *= a.E[d];
  }
  a.tk_blocks = grid_blocks(a.EV);
  // EvalTracker.record_move's radius, int(np.linalg.norm(shift)): the square root of an exact integer, truncated
  std::vector<int> shift_r(std::max(a.n_shifts, 1), 0);
  for (int i = 0; i < a.n_shifts; ++i) {
    const int* o = desc->shifts_zyx + i * 3;
    shift_r[i] = (int)std::sqrt((double)o[0] * o[0] + (double)o[1] * o[1] + (double)o[2] * o[2]);
    ex->n_radii = std::max(ex->n_radii, shift_r[i] + 1);
  }
  ex->desc = *desc;
  ex->desc.shifts_zyx = nullptr;
  if (a.n_shifts) ex->shifts.assign(desc->shifts_zyx, desc->shifts_zyx + a.n_shifts * 3);
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
  int* sr = nullptr;
  if (m.get(&sr, shift_r.size()) || m.get(&a.tk, exk::kTkMoves + 3 * ex->n_radii, true) ||
      m.get(&a.tk_loss, 1, true) || m.get(&a.tk_part, B * a.tk_blocks, true) || m.get(&a.tk_arrived, 2, true) ||
      m.get(&a.tk_slot, B, true) || m.get(&a.ecoord, B, true) || m.get(&a.ring, exk::kRing * exk::plane_floats(a.E), true) ||
      m.get(&a.ring_coord, exk::kRing, true))
    return 1;
  CUDA_OK(cudaMemcpy(sr, shift_r.data(), shift_r.size() * sizeof(int), cudaMemcpyHostToDevice));
  a.shift_r = sr;
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

int ffn_examples_tracker(FfnExamples* ex, FfnTrackerCounts* out, int64_t* moves_by_radius, int n_radii,
                         float* planes, FfnExampleCoord* plane_coords, int32_t* n_planes, int reset) {
  if (!ex) return fail("null examples");
  if (!out || !moves_by_radius || !n_planes) return fail("null argument: counts, moves_by_radius and n_planes are required");
  if (n_radii < ex->n_radii)
    return fail("moves_by_radius holds " + std::to_string(n_radii) + " radii, the shifts need " +
                std::to_string(ex->n_radii));
  if (!planes != !plane_coords) return fail("planes and plane_coords must both be given or both be NULL");
  CUDA_OK(cudaSetDevice(ex->device));
  cudaStream_t st = cudaStreamPerThread;
  const exk::Args& a = ex->a;
  std::vector<long long> tk(exk::kTkMoves + 3 * ex->n_radii);
  double loss = 0.0;
  CUDA_OK(cudaMemcpyAsync(tk.data(), a.tk, tk.size() * sizeof(long long), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(&loss, a.tk_loss, sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  const int n = (int)std::min<long long>(tk[exk::kTkRing], exk::kRing);
  if (planes) {
    const long long pf = exk::plane_floats(a.E);
    for (int i = 0; i < n; ++i) {   // oldest first
      const int slot = (int)((tk[exk::kTkRing] - n + i) % exk::kRing);
      CUDA_OK(cudaMemcpyAsync(planes + i * pf, a.ring + slot * pf, pf * sizeof(float), cudaMemcpyDeviceToHost, st));
      CUDA_OK(cudaMemcpyAsync(plane_coords + i, a.ring_coord + slot, sizeof(FfnExampleCoord), cudaMemcpyDeviceToHost,
                              st));
    }
  }
  if (reset) {
    CUDA_OK(cudaMemsetAsync(a.tk, 0, tk.size() * sizeof(long long), st));
    CUDA_OK(cudaMemsetAsync(a.tk_loss, 0, sizeof(double), st));
  }
  CUDA_OK(cudaStreamSynchronize(st));
  out->steps = tk[exk::kTkSteps];
  out->patches = tk[exk::kTkPatches];
  out->eval_voxels = tk[exk::kTkVoxels];
  for (int k = 0; k < 4; ++k) out->prediction_counts[k] = tk[exk::kTkTP + k];
  out->patch_loss = loss;
  for (int r = 0; r < n_radii; ++r)
    for (int t = 0; t < 3; ++t) moves_by_radius[r * 3 + t] = r < ex->n_radii ? tk[exk::kTkMoves + r * 3 + t] : 0;
  *n_planes = n;
  return 0;
}

int ffn_examples_get_state(FfnExamples* ex, void* out, int64_t cap, int64_t* n) {
  if (!ex) return fail("null examples");
  CUDA_OK(cudaSetDevice(ex->device));
  return blob::get(kStateMagic, kStateVersion, state_header(ex), state_sections(ex), out, cap, n);
}

int ffn_examples_set_state(FfnExamples* ex, const void* state, int64_t n) {
  if (!ex) return fail("null examples");
  const std::vector<blob::Section> secs = state_sections(ex);
  const uint8_t* payload = nullptr;
  if (blob::open(state, n, kStateMagic, kStateVersion, state_header(ex), secs, "example loop", &payload) ||
      check_state(ex, payload, secs))
    return 1;
  CUDA_OK(cudaSetDevice(ex->device));
  if (blob::put(payload, secs)) return 1;
  std::memcpy(&ex->total, payload + blob::offset(secs, 2), sizeof(long long));
  return 0;
}

}  // extern "C"
