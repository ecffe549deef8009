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

// te_submap.cu — the read side of a te_map.  A window of te_map_get_submaps that has cells: its block of the map and where its
// layers go.  Columns are numbered flat over (window, layer, column), window by window.
struct SubmapWindow {
  long long col0;  // the window's first column in that numbering
  long long src;   // cell offset of its top-left cell in a source layer: top_col * map rows + top_row
  long long dst;   // float offset of its first layer in `out`
  int rows, cols;
};
struct SubmapGather {
  const float* const* layers;  // device table of the source layers (column-major, default order), in output order
  const SubmapWindow* win;     // device, in column order
  int nwin, map_rows;
  long long ncolumns;          // windows x layers x columns
  float* out;
};
// One k_map_gather_submaps launch for every column of every window (none when there is no column).
void launch_gather_submaps(const SubmapGather& a, int sms, cudaStream_t s);
struct GridGeo;
// valid[q] = getIndex(xy[2q], xy[2q+1]) succeeds and traversability is finite there (device pointers; none launched for n = 0).
void launch_valid_at(const GridGeo& g, const float* trav, int n, const double* xy, unsigned char* valid, cudaStream_t s);

}  // namespace te
