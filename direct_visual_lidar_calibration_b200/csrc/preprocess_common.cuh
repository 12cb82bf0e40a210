// preprocess_common.cuh -- the scratch, timing and device plumbing shared by the dataset-building stages
// (preprocess.cu: preprocess_map's point stages; bag_integrate.cu: the bag decoder and static integrator).
#pragma once

#include <cuda_runtime.h>

#include <cfloat>
#include <climits>
#include <vector>

#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {
namespace {

// Device scratch from the process-wide pool; the legacy stream is synchronised before the blocks go back.
class Scratch {
public:
  explicit Scratch(int device) : device_(device) {}
  ~Scratch() {
    cudaStreamSynchronize(cudaStreamLegacy);
    for (void* p : bufs_) MemPool::instance().device_free(device_, p);
  }
  template <class T>
  cudaError_t alloc(size_t count, T** out) {
    void* p = nullptr;
    const cudaError_t e = MemPool::instance().device_alloc(device_, sizeof(T) * (count ? count : 1), &p);
    if (e == cudaSuccess) bufs_.push_back(p);
    *out = static_cast<T*>(p);
    return e;
  }

private:
  int device_;
  std::vector<void*> bufs_;
};

// Stage timing between CUDA events on the legacy stream (only when the caller asks for it).
class StageTimer {
public:
  explicit StageTimer(bool on) : on_(on) {}
  ~StageTimer() {
    for (cudaEvent_t e : ev_) cudaEventDestroy(e);
  }
  cudaError_t mark() {
    if (!on_) return cudaSuccess;
    cudaEvent_t e;
    cudaError_t rc = cudaEventCreate(&e);
    if (rc != cudaSuccess) return rc;
    ev_.push_back(e);
    return cudaEventRecord(e, cudaStreamLegacy);
  }
  // ms between consecutive marks
  cudaError_t read(double* out, int n) {
    if (!on_ || !out) return cudaSuccess;
    cudaError_t rc = cudaEventSynchronize(ev_.back());
    if (rc != cudaSuccess) return rc;
    for (int i = 0; i < n && i + 1 < static_cast<int>(ev_.size()); i++) {
      float ms = 0.0f;
      rc = cudaEventElapsedTime(&ms, ev_[i], ev_[i + 1]);
      if (rc != cudaSuccess) return rc;
      out[i] = ms;
    }
    return cudaSuccess;
  }

private:
  bool on_;
  std::vector<cudaEvent_t> ev_;
};

int prepare_device(int* device) {
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available: this library has no CPU fallback");
    return VLCAL_ERR_NO_DEVICE;
  }
  if (*device < 0) VL_CUDA(cudaGetDevice(device));
  VL_CUDA(cudaSetDevice(*device));
  return VLCAL_OK;
}

unsigned int blocks_for(long long n, int threads) { return static_cast<unsigned int>((n + threads - 1) / threads); }

// static_cast<int>(float) as x86-64 compiles it (cvttss2si): out of int range gives INT_MIN.  cvt.rzi on the GPU
// saturates instead, so the out-of-range case is mapped explicitly.  `f` is already integral (a floorf result).
__host__ __device__ __forceinline__ int float_to_int_x86(float f) {
  return (f >= -2147483648.0f && f < 2147483648.0f) ? static_cast<int>(f) : INT_MIN;
}

__host__ __device__ __forceinline__ bool finite_f(float v) { return fabsf(v) <= FLT_MAX; }

// dst[k] = src[order[k]] for the k < *n_d selected by a compaction
__global__ void __launch_bounds__(256) gather_float4_kernel(const float4* src, const int* order, const int* n_d, float4* dst) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < *n_d) dst[k] = src[order[k]];
}

}  // namespace
}  // namespace vlcal
