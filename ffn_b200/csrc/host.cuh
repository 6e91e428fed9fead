// host.cuh — the host-side idiom of every entry point: errors (fail, CUDA_OK), device selection (use_device), device
// memory (DevBufs), CUB scratch (CubTemp) and the checks of a model description (check_model).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <string>
#include <vector>

#include "device_types.cuh"

namespace ffn {

// Sets the calling thread's last error (ffn_last_error) to msg and returns 1.  Defined in engine.cu.
int fail(const std::string& msg);

#define CUDA_OK(expr)                                                                          \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" + \
                  std::to_string(__LINE__) + ")");                                             \
  } while (0)

// The only owner of device memory: the temporaries of one call, or the buffers an engine or a canvas holds for its
// lifetime.  It frees everything it allocated when it goes away, on every return path.  As a member of an engine or a
// canvas it is destroyed after that object's destructor has made the object's device current.
struct DevBufs {
  std::vector<void*> p;
  DevBufs() = default;
  DevBufs(const DevBufs&) = delete;
  DevBufs& operator=(const DevBufs&) = delete;
  ~DevBufs() { for (void* q : p) cudaFree(q); }
  // *out is set only when the allocation succeeds.
  template <typename T>
  int get(T** out, size_t count, bool zero = false) {
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    void* q = nullptr;
    CUDA_OK(cudaMalloc(&q, bytes));
    p.push_back(q);
    *out = static_cast<T*>(q);
    if (zero) CUDA_OK(cudaMemset(q, 0, bytes));
    return 0;
  }
  // Frees q (null: nothing) and sets it to null.
  template <typename T>
  void release(T*& q) {
    p.erase(std::remove(p.begin(), p.end(), q), p.end());
    cudaFree(q);
    q = nullptr;
  }
};

// One temporary-storage buffer for all CUB calls of one entry point.  Each call is written once, as a callable
// (void* temp, size_t& bytes) -> cudaError_t: alloc() queries every call's size (temp == nullptr) and allocates the
// largest, and run() runs one call against that buffer.  The sizes are queried at the calls' upper bounds on the item
// count; CUB refuses a run that needs more than it is given.
struct CubTemp {
  char* p = nullptr;
  size_t bytes = 0;
  template <typename... F>
  int alloc(DevBufs& bufs, const F&... calls) {
    if ((size_for(calls) || ...)) return 1;
    return bufs.get(&p, bytes);
  }
  template <typename F>
  int size_for(const F& call) {
    size_t b = 0;
    CUDA_OK(call(nullptr, b));
    bytes = std::max(bytes, b);
    return 0;
  }
  template <typename F>
  cudaError_t run(const F& call) const {
    size_t b = bytes;
    return call(p, b);
  }
};

// The library only contains sm_90a code: every entry point that takes a device index accepts an sm_90 device only.
// On success the device is the calling thread's current device and *prop holds its properties.
inline int use_device(int device, cudaDeviceProp* prop) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: libffn_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail("bad device index");
  CUDA_OK(cudaGetDeviceProperties(prop, device));
  if (prop->major != 9 || prop->minor != 0)
    return fail(std::string("device is sm_") + std::to_string(prop->major) + std::to_string(prop->minor) +
                "; this library only contains sm_90a code");
  CUDA_OK(cudaSetDevice(device));
  return 0;
}

// The ConvStack3DFFNModel geometries the library runs, for engines and trainers alike.
inline int check_model(const FfnModelDesc* model) {
  if (model->features != kFeat) return fail("only 32 feature maps are supported");
  if (model->depth < 1 || 2 * model->depth > kMaxConv) return fail("unsupported depth");
  for (int k = 0; k < 3; ++k) {
    if (model->fov_zyx[k] < 3 || model->fov_zyx[k] % 2 == 0) return fail("fov sizes must be odd and >= 3");
    if (model->deltas_zyx[k] < 0 || model->deltas_zyx[k] > model->fov_zyx[k] / 2)
      return fail("deltas must lie in [0, fov // 2]");
  }
  return 0;
}

// The training example loop's steps that ffn_trainer_train runs (defined in examples.cu).  All work is enqueued on
// cudaStreamPerThread; examples_finish reads the call's results after a synchronisation.
int examples_check_trainer(const FfnExamples* ex, int device, const int fov_zyx[3], int max_batch);
int examples_batch(const FfnExamples* ex);
int examples_upload(FfnExamples* ex, const FfnExampleCoord* coords, int64_t n);
int examples_advance(FfnExamples* ex, float* seed, float* image, float* labels);
int examples_paste(FfnExamples* ex, const float* logits);
int examples_finish(FfnExamples* ex, int64_t* n_consumed);

}  // namespace ffn
