// te_submap.cu — the read side of a te_map: GetGridMap submaps of its resident layers (k_map_gather_submaps) and
// mapHasValidTraversabilityAt for a batch of positions (k_map_valid_at).  Compiled with --fmad=false: k_map_valid_at indexes
// positions with te_grid.cuh's getIndex, which the host and the oracle evaluate without contraction.
#include <algorithm>

#include "te_kernels.h"
#include "te_grid.cuh"

namespace te {
namespace {

constexpr int kGatherWarps = 8;  // warps per block

// One warp per destination column: column j of layer l of window w is the run of w.rows floats starting at cell (top_row,
// top_col + j) of the source layer (column-major, default order), and lands at w.dst + (l * w.cols + j) * w.rows of `out`.
// Columns are numbered flat over (window, layer, column); w.col0 is the first of window w's and a warp finds its window by
// binary search.  16-byte accesses where source and destination agree modulo 16 bytes, 4-byte ones otherwise.
__global__ void __launch_bounds__(kGatherWarps * 32) k_map_gather_submaps(SubmapGather a) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * kGatherWarps;
  for (long long c = (long long)blockIdx.x * kGatherWarps + (threadIdx.x >> 5); c < a.ncolumns; c += nwarps) {
    int lo = 0, hi = a.nwin - 1;  // last window whose first column is <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(&a.win[mid].col0) <= c) lo = mid; else hi = mid - 1;
    }
    const SubmapWindow w = a.win[lo];
    const long long k = c - w.col0;
    const int l = (int)(k / w.cols), j = (int)(k - (long long)l * w.cols);
    const float* __restrict__ src = a.layers[l] + w.src + (size_t)j * a.map_rows;
    float* __restrict__ dst = a.out + w.dst + ((size_t)l * w.cols + j) * w.rows;
    const int n = w.rows;
    int head = n;  // elements copied one by one before the 16-byte body
    if ((((uintptr_t)src ^ (uintptr_t)dst) & 15) == 0) head = min(n, (int)(((16 - ((uintptr_t)src & 15)) & 15) >> 2));
    for (int e = lane; e < head; e += 32) dst[e] = __ldg(src + e);
    if (head < n) {
      const int nv = (n - head) >> 2;
      const float4* __restrict__ s4 = reinterpret_cast<const float4*>(src + head);
      float4* __restrict__ d4 = reinterpret_cast<float4*>(dst + head);
      for (int e = lane; e < nv; e += 32) d4[e] = __ldg(s4 + e);
      for (int e = head + 4 * nv + lane; e < n; e += 32) dst[e] = __ldg(src + e);
    }
  }
}

__global__ void k_map_valid_at(GridGeo g, const float* __restrict__ trav, int n, const double* __restrict__ xy,
                               unsigned char* __restrict__ valid) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  int i, j;
  const bool in = grid_get_index(g, xy[2 * q], xy[2 * q + 1], i, j);
  valid[q] = in && finitef(__ldg(trav + (size_t)j * g.rows + i)) ? 1 : 0;
}

}  // namespace

void launch_gather_submaps(const SubmapGather& a, int sms, cudaStream_t s) {
  if (a.ncolumns <= 0) return;
  const long long blocks = std::min<long long>((a.ncolumns + kGatherWarps - 1) / kGatherWarps, (long long)sms * 16);
  k_map_gather_submaps<<<(unsigned)blocks, kGatherWarps * 32, 0, s>>>(a);
}

void launch_valid_at(const GridGeo& g, const float* trav, int n, const double* xy, unsigned char* valid, cudaStream_t s) {
  if (n <= 0) return;
  k_map_valid_at<<<(n + 255) / 256, 256, 0, s>>>(g, trav, n, xy, valid);
}

}  // namespace te
