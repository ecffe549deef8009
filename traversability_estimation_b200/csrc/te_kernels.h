// te_kernels.h — host-callable launchers of the device code (internal to libte_b200).
#pragma once
#include <cuda_runtime.h>
#include "te_device.cuh"

namespace te {

// A grow-only device allocation: reserve() reallocates (without keeping the contents) only when `bytes` exceeds the capacity.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    else p = nullptr;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

struct ChainOut {
  float* slope;
  float* step;
  float* rough;
  float* trav;
  float* nx;  // may be null
  float* ny;
  float* nz;
};

// te_generic.cu — literal double-precision kernels (any radius / resolution).
void launch_chain_generic(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, int sms, cudaStream_t s);
// zero_next: 128 counter words the kernel zeroes for the next chain call (may be null); pdl: programmatic dependent launch
void launch_fixup(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, const unsigned int* list,
                  const unsigned int* count, unsigned int cap, unsigned int* zero_next, int sms, cudaStream_t s, bool pdl);
void launch_normals(const SlabView& v, const ChainDev& p, const float* elev, float* nx, float* ny, float* nz, int sms, cudaStream_t s);
void launch_slope(long long total, double crit, const float* nz, float* out, int sms, cudaStream_t s);
void launch_step(const SlabView& v, const ChainDev& p, const float* elev, float* out, int sms, cudaStream_t s);
void launch_roughness(const SlabView& v, const ChainDev& p, const float* elev, const float* nx, const float* ny, const float* nz,
                      float* out, int sms, cudaStream_t s);

}  // namespace te
