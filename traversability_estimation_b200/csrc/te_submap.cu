// te_submap.cu — the read side of a te_map: GetGridMap submaps of its resident layers (k_map_gather_submaps),
// mapHasValidTraversabilityAt for a batch of positions (k_map_valid_at), GridMap::atPosition at points around poses
// (k_map_at_poses), GridMapRosConverter::toOccupancyGrid of its layers (k_map_occupancy) and toPointCloud (k_map_cloud_count,
// k_map_cloud_scatter); and the windows a te_map update cuts out of a larger elevation map (k_map_cut_windows).  Compiled with --fmad=false: k_map_valid_at and k_map_at_poses index positions with te_grid.cuh's getIndex,
// which the host and the oracle evaluate without contraction, k_map_at_poses places points as the polygonal paths do, and
// k_map_cloud_scatter takes x and y from cell_coord as getPosition computes them.
#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "te_kernels.h"
#include "te_grid.cuh"
#include "te_pose.cuh"

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

// n floats from src to dst by one warp: 16-byte accesses where the two agree modulo 16 bytes, 4-byte ones otherwise.
__device__ __forceinline__ void warp_copy_run(float* __restrict__ dst, const float* __restrict__ src, int n, int lane) {
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

// n copies of v at dst by one warp, 16-byte stores from the first 16-byte boundary on.
__device__ __forceinline__ void warp_fill_run(float* __restrict__ dst, float v, int n, int lane) {
  const int head = min(n, (int)(((16 - ((uintptr_t)dst & 15)) & 15) >> 2));
  for (int e = lane; e < head; e += 32) dst[e] = v;
  const int nv = (n - head) >> 2;
  float4* __restrict__ d4 = reinterpret_cast<float4*>(dst + head);
  for (int e = lane; e < nv; e += 32) d4[e] = make_float4(v, v, v, v);
  for (int e = head + 4 * nv + lane; e < n; e += 32) dst[e] = v;
}

// One warp per destination column, numbered flat over (window, layer, column): column j of layer l of window k is the column
// win[k].y + j of its source from source row win[k].x on, read through the window's start index (win[k].z, win[k].w), so at most
// two contiguous runs of the stored column (before and after the row wrap), and NaN 0x7fc00000 (grid_map's unknown cell) for the
// rows and columns the window takes from outside the source.  Integer arithmetic only: the host placed the windows.
__global__ void __launch_bounds__(kGatherWarps * 32) k_map_cut_windows(const __grid_constant__ WindowCut a) {
  const int lane = threadIdx.x & 31;
  const float nan = __uint_as_float(0x7fc00000u);
  const long long per_map = (long long)a.nlayers * a.cols;
  for (long long c = (long long)blockIdx.x * kGatherWarps + (threadIdx.x >> 5); c < a.ncolumns; c += (long long)gridDim.x * kGatherWarps) {
    const int k = (int)(c / per_map);
    const int r = (int)(c - (long long)k * per_map);
    const int l = r / a.cols, j = r - l * a.cols;
    const int4 t = a.win[k];
    const size_t kl = (size_t)k * a.nlayers + l;
    float* __restrict__ dst = a.dst[kl] + (size_t)j * a.rows;
    const float* __restrict__ src = a.src[kl];
    const long long J = (long long)t.y + j;  // the source column
    int i0 = 0, i1 = 0;                      // window rows [i0, i1) lie in the source
    if (J >= 0 && J < a.src_cols) {
      i0 = (int)max(0LL, -(long long)t.x);
      i1 = (int)min((long long)a.rows, (long long)a.src_rows - t.x);
      if (i1 <= i0) i0 = i1 = 0;
    }
    warp_fill_run(dst, nan, i0, lane);
    if (i1 > i0) {
      int sc = (int)J + t.w;
      if (sc >= a.src_cols) sc -= a.src_cols;
      const float* __restrict__ col = src + (size_t)(a.col_of ? __ldg(a.col_of + sc) : sc) * a.src_rows;
      int s0 = t.x + i0 + t.z;  // stored row of window row i0
      if (s0 >= a.src_rows) s0 -= a.src_rows;
      const int n = i1 - i0, n1 = min(n, a.src_rows - s0);
      warp_copy_run(dst + i0, col + s0, n1, lane);
      if (n1 < n) warp_copy_run(dst + i0 + n1, col, n - n1, lane);
    }
    warp_fill_run(dst + i1, nan, a.rows - i1, lane);
  }
}

// Position q on map pos_map[q] of a batch of nmaps maps (pos_map null: map 0); a map outside the batch gives 0.  map_pos: the maps'
// own positions (x, y per map), or null: every map at g's.
__global__ void k_map_valid_at(GridGeo g, const float* __restrict__ trav, int n, const double* __restrict__ xy,
                               const int* __restrict__ pos_map, int nmaps, const double* __restrict__ map_pos,
                               unsigned char* __restrict__ valid) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  if (pos_map) {
    const int m = pos_map[q];
    if (m < 0 || m >= nmaps) { valid[q] = 0; return; }
    trav += (size_t)m * g.rows * g.cols_total;
    if (map_pos) { g.posx = map_pos[2 * m]; g.posy = map_pos[2 * m + 1]; }
  }
  int i, j;
  const bool in = grid_get_index(g, xy[2 * q], xy[2 * q + 1], i, j);
  valid[q] = in && finitef(__ldg(trav + (size_t)j * g.rows + i)) ? 1 : 0;
}

// upper - lower as the reference's host computes it: one IEEE float32 subtraction, round to nearest, never contracted.  Its NaN
// results differ in payload only: the GPU returns its canonical NaN, x86-64's SSE / AVX subtraction (the reference node's, and
// numpy's) returns the first NaN operand quieted, or the default NaN 0xffc00000 for Inf - Inf.  That rule is applied here, so the
// layer is the reference's bit for bit.
__device__ __forceinline__ float range_sub(float u, float l) {
  const float r = __fsub_rn(u, l);
  if (!isnan(r)) return r;
  const unsigned q = isnan(u) ? __float_as_uint(u) : isnan(l) ? __float_as_uint(l) : 0xffc00000u;
  return __uint_as_float(q | 0x00400000u);
}

// uncertainty_range = upper_bound - lower_bound per cell (publishTraversabilityMap).  V cells per thread and access (V = 4: 16-byte).
template <int V>
__global__ void __launch_bounds__(256) k_uncertainty_range(const float* __restrict__ upper, const float* __restrict__ lower,
                                                           float* __restrict__ out, size_t n) {
  const size_t step = (size_t)gridDim.x * blockDim.x * V;
  for (size_t c = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; c < n; c += step) {
    if constexpr (V == 4) {
      const float4 u = __ldg(reinterpret_cast<const float4*>(upper + c)), l = __ldg(reinterpret_cast<const float4*>(lower + c));
      *reinterpret_cast<float4*>(out + c) = make_float4(range_sub(u.x, l.x), range_sub(u.y, l.y), range_sub(u.z, l.z), range_sub(u.w, l.w));
    } else {
      out[c] = range_sub(__ldg(upper + c), __ldg(lower + c));
    }
  }
}

// GridMap::atPosition(layer, position) for every (pose, point) sample: one thread per sample (grid-stride), which places its
// point once, indexes it once on its map, then reads every requested layer at that cell.  Consecutive threads take consecutive
// points of a pose, so the stores of each layer coalesce; the layer reads are scattered 4-byte loads.
__global__ void __launch_bounds__(256) k_map_at_poses(const __grid_constant__ MapAtPoses a) {
  const long long total = (long long)a.nposes * a.npoints;
  const size_t cells = (size_t)a.rows * a.cols;
  const float nan = __uint_as_float(0x7fc00000u);
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < total; s += (long long)gridDim.x * blockDim.x) {
    const int k = (int)s / a.npoints, t = (int)s - k * a.npoints;
    const int m = a.pose_map ? __ldg(a.pose_map + k) : 0;
    GridGeo g{a.rows, a.cols, a.res, a.lenx, a.leny, a.posx, a.posy};
    bool ok = m >= 0 && m < a.nmaps;
    if (ok && a.map_pos) { g.posx = __ldg(a.map_pos + 2 * m); g.posy = __ldg(a.map_pos + 2 * m + 1); }
    const PoseRT T = pose_rt_d(a.poses + 7 * (size_t)k);
    const double2 p = pose_point_d(T, (double)__ldg(a.points + 3 * t), (double)__ldg(a.points + 3 * t + 1),
                                   (double)__ldg(a.points + 3 * t + 2));
    int i = 0, j = 0;
    ok = ok && isfinite(p.x) && isfinite(p.y) && grid_get_index(g, p.x, p.y, i, j);
    const size_t cell = ok ? (size_t)m * cells + (size_t)j * a.rows + i : 0;
    for (int l = 0; l < a.nlayers; ++l) {
      float v = nan;
      if (ok) {
        v = __ldg(a.layer[l] + cell);
        if (l == a.range_l) v = range_sub(v, __ldg(a.lower + cell));
      }
      a.out[(size_t)l * total + s] = v;
    }
    if (a.valid) a.valid[s] = ok ? 1 : 0;
  }
}

// One cell of GridMapRosConverter::toOccupancyGrid: (v - dataMin) / (dataMax - dataMin), NaN -> -1, else 0 + clamp(., 0, 1) * 100
// truncated toward zero, every step one IEEE float32 operation rounded to nearest (den = dataMax - dataMin).  The result's low
// byte is the int8 cell: 0 .. 100, or 0xff (-1).
__device__ __forceinline__ unsigned occupancy_cell(float v, float mn, float den) {
  const float q = __fdiv_rn(__fsub_rn(v, mn), den);
  if (isnan(q)) return 0xffu;
  return (unsigned)__float2int_rz(__fadd_rn(0.0f, __fmul_rn(fminf(fmaxf(0.0f, q), 1.0f), 100.0f)));
}

// toOccupancyGrid of every (layer, map) block of a call: blockIdx.y walks the blocks q = l * nmaps + k, blockIdx.x / threadIdx.x the
// cells of one block.  Block q's grid is its map's column-major layer reversed: out[q * cells + p] is the cell of source index
// cells - 1 - p.  Each thread writes 4-byte words of the block (from its first 4-byte boundary on) from 4 consecutive source cells,
// read as one 16-byte load where that is aligned; up to 3 head and 3 tail bytes per block are written one by one.
__global__ void __launch_bounds__(256) k_map_occupancy(const __grid_constant__ MapOccupancy a) {
  const long long N = a.cells, nblocks = (long long)a.nlayers * a.nmaps;
  for (long long q = blockIdx.y; q < nblocks; q += gridDim.y) {
    const int l = (int)(q / a.nmaps), k = (int)(q - (long long)l * a.nmaps);
    const int m = a.slot ? __ldg(a.slot + k) : k;
    const float* __restrict__ src = a.layer[l] + (size_t)m * N;
    const float* __restrict__ low = l == a.range_l ? a.lower + (size_t)m * N : nullptr;
    const float mn = a.data_min[l], den = __fsub_rn(a.data_max[l], mn);
    unsigned char* __restrict__ dst = a.out + (size_t)q * N;
    const long long head = min(N, (long long)((4u - ((unsigned)(uintptr_t)dst & 3u)) & 3u));
    const long long nw = (N - head) >> 2, tail0 = head + 4 * nw;
    // word u covers output bytes head + 4u .. + 3, i.e. source cells s0 .. s0 + 3 with s0 = N - 4 - head - 4u
    const bool vec = (((uintptr_t)(src + (N - 4 - head)) | (low ? (uintptr_t)(low + (N - 4 - head)) : 0)) & 15u) == 0;
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < nw + 8; u += (long long)gridDim.x * blockDim.x) {
      if (u < nw) {
        const long long s0 = N - 4 - head - 4 * u;
        float4 v;
        if (vec) {
          v = __ldg(reinterpret_cast<const float4*>(src + s0));
          if (low) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(low + s0));
            v = make_float4(__fsub_rn(v.x, w.x), __fsub_rn(v.y, w.y), __fsub_rn(v.z, w.z), __fsub_rn(v.w, w.w));
          }
        } else {
          v = make_float4(__ldg(src + s0), __ldg(src + s0 + 1), __ldg(src + s0 + 2), __ldg(src + s0 + 3));
          if (low)
            v = make_float4(__fsub_rn(v.x, __ldg(low + s0)), __fsub_rn(v.y, __ldg(low + s0 + 1)), __fsub_rn(v.z, __ldg(low + s0 + 2)),
                            __fsub_rn(v.w, __ldg(low + s0 + 3)));
        }
        const unsigned word = occupancy_cell(v.w, mn, den) | occupancy_cell(v.z, mn, den) << 8 | occupancy_cell(v.y, mn, den) << 16 |
                              occupancy_cell(v.x, mn, den) << 24;
        *reinterpret_cast<unsigned*>(dst + head + 4 * u) = word;
      } else {  // u - nw = 0..3: head byte u - nw; 4..7: tail byte u - nw - 4
        const int e = (int)(u - nw);
        const long long p = e < 4 ? (e < head ? e : -1) : (tail0 + e - 4 < N ? tail0 + e - 4 : -1);
        if (p < 0) continue;
        float v = __ldg(src + (N - 1 - p));
        if (low) v = __fsub_rn(v, __ldg(low + (N - 1 - p)));
        dst[p] = (unsigned char)occupancy_cell(v, mn, den);
      }
    }
  }
}

// ---- toPointCloud: count the points of every tile, scan the counts, scatter the records --------------------------------------

constexpr int kCloudThreads = 256;  // a tile is kCloudTile / kCloudThreads chunks of one cell per thread

// A layer at absolute cell d (slot * cells + default-order index): the stored bits, or for uncertainty_range (range) upper - lower
// as te_map_get_layers computes it.
__device__ __forceinline__ float cloud_read(const float* __restrict__ p, bool range, const float* __restrict__ lower, size_t d) {
  const float v = __ldg(p + d);
  return range ? range_sub(v, __ldg(lower + d)) : v;
}

// Map k of the call: its slot, start index and position.
__device__ __forceinline__ CloudMap cloud_map(const MapCloud& a, int k) {
  if (a.maps) return a.maps[k];
  return CloudMap{k, a.sr, a.sc, 0, a.px, a.py};
}

// Buffer cell b (< cells) of map M: its default-order row i and column j.
__device__ __forceinline__ void cloud_cell(const MapCloud& a, const CloudMap& M, unsigned b, int& i, int& j) {
  const unsigned bj = b / (unsigned)a.rows;
  i = (int)(b - bj * (unsigned)a.rows) - M.sr;
  j = (int)bj - M.sc;
  if (i < 0) i += a.rows;
  if (j < 0) j += a.cols;
}

// isValid over the basic layers (when there are any) and getPosition3's check of the point layer at absolute cell d.
__device__ __forceinline__ bool cloud_valid(const MapCloud& a, size_t d) {
  if (!isfinite(cloud_read(a.point, a.basic_range >> 31, a.lower, d))) return false;
  for (int b = 0; b < a.nbasic; ++b)
    if (!isfinite(cloud_read(a.basic[b], (a.basic_range >> b) & 1u, a.lower, d))) return false;
  return true;
}

// One count per tile (grid-stride over the tiles of every map); the entry after the last tile is 0, so that its prefix is the total.
__global__ void __launch_bounds__(kCloudThreads) k_map_cloud_count(const __grid_constant__ MapCloud a) {
  const long long ntiles = (long long)a.nmaps * a.tiles;
  if (blockIdx.x == 0 && threadIdx.x == 0) a.count[ntiles] = 0;
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int k = (int)(t / a.tiles);
    const CloudMap M = cloud_map(a, k);
    const long long b0 = (t - (long long)k * a.tiles) * kCloudTile;
    int n = 0;
    for (int c = 0; c < kCloudTile / kCloudThreads; ++c) {
      const long long b = b0 + c * kCloudThreads + threadIdx.x;
      bool v = false;
      if (b < a.cells) {
        int i, j;
        cloud_cell(a, M, (unsigned)b, i, j);
        v = cloud_valid(a, (size_t)M.slot * a.cells + (size_t)j * a.rows + i);
      }
      n += __syncthreads_count(v);
    }
    if (threadIdx.x == 0) a.count[t] = (unsigned long long)n;
  }
}

// Every tile again: each chunk of kCloudThreads cells ranks its points with a ballot scan, builds their records in shared memory
// (point_step bytes each, in point order) and writes them out as consecutive 4-byte words (single bytes when `out` is not 4-byte
// aligned), so each warp stores one contiguous run.  Points at or past a.capacity are not written.  In device memory it also writes
// the call's offsets.
__global__ void __launch_bounds__(kCloudThreads) k_map_cloud_scatter(const __grid_constant__ MapCloud a) {
  // kCloudThreads records of point_step bytes.  Static, at the largest point_step: dynamic shared memory would make ptxas reserve
  // shared memory for every kernel of this unit.  48 registers allow 5 blocks per SM, and 6 fit in shared memory.
  __shared__ unsigned rec[kCloudThreads * (kCloudMaxFields + 2)];
  __shared__ int wsum[kCloudThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, words = a.point_step >> 2;
  const long long ntiles = (long long)a.nmaps * a.tiles;
  const bool aligned = ((uintptr_t)a.out & 3u) == 0;
  if (a.offsets)
    for (long long k = (long long)blockIdx.x * kCloudThreads + threadIdx.x; k <= a.nmaps; k += (long long)gridDim.x * kCloudThreads)
      a.offsets[k] = (long long)a.first[k * a.tiles];
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int k = (int)(t / a.tiles);
    const CloudMap M = cloud_map(a, k);
    const long long b0 = (t - (long long)k * a.tiles) * kCloudTile;
    long long base = (long long)a.first[t];  // the chunk's first point
    for (int c = 0; c < kCloudTile / kCloudThreads; ++c) {
      const long long b = b0 + c * kCloudThreads + threadIdx.x;
      int i = 0, j = 0;
      size_t d = 0;
      bool v = false;
      if (b < a.cells) {
        cloud_cell(a, M, (unsigned)b, i, j);
        d = (size_t)M.slot * a.cells + (size_t)j * a.rows + i;
        v = cloud_valid(a, d);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, v);
      if (lane == 0) wsum[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < kCloudThreads / 32; ++w) {
        before += w < warp ? wsum[w] : 0;
        total += wsum[w];
      }
      if (v) {
        unsigned* r = rec + (size_t)(before + __popc(bal & ((1u << lane) - 1u))) * words;
        int w = 0;
        for (int e = 0; e < a.nfields; ++e) {
          if (e == a.point_e) {
            r[w++] = __float_as_uint(__double2float_rn(cell_coord(M.px, a.lenx, a.res, i)));
            r[w++] = __float_as_uint(__double2float_rn(cell_coord(M.py, a.leny, a.res, j)));
            r[w++] = __float_as_uint(cloud_read(a.point, a.basic_range >> 31, a.lower, d));
          } else {
            r[w++] = a.field[e] ? __float_as_uint(cloud_read(a.field[e], (a.field_range >> e) & 1u, a.lower, d)) : 0x7fc00000u;
          }
        }
      }
      __syncthreads();
      const long long room = a.capacity - base;
      const int n = (int)max(0LL, min((long long)total, room));
      unsigned char* dst = a.out + base * a.point_step;
      if (aligned) {
        unsigned* d4 = reinterpret_cast<unsigned*>(dst);
        for (int w = threadIdx.x; w < n * words; w += kCloudThreads) d4[w] = rec[w];
      } else {
        const unsigned char* r1 = reinterpret_cast<const unsigned char*>(rec);
        for (int w = threadIdx.x; w < n * a.point_step; w += kCloudThreads) dst[w] = r1[w];
      }
      base += total;
      __syncthreads();  // rec and wsum are rewritten by the next chunk
    }
  }
}

}  // namespace

size_t map_cloud_scan_bytes(long long n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
  return bytes;
}

cudaError_t launch_map_cloud_count(const MapCloud& a, void* tmp, size_t tmp_bytes, int sms, cudaStream_t s) {
  const long long ntiles = (long long)a.nmaps * a.tiles;
  const long long blocks = std::max<long long>(1, std::min<long long>(ntiles, (long long)sms * 16));
  k_map_cloud_count<<<(unsigned)blocks, kCloudThreads, 0, s>>>(a);
  return cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, (const unsigned long long*)a.count, a.first, (int)(ntiles + 1), s);
}

void launch_map_cloud_scatter(const MapCloud& a, int sms, cudaStream_t s) {
  const long long ntiles = (long long)a.nmaps * a.tiles;
  const long long blocks = std::max<long long>(1, std::min<long long>(ntiles, (long long)sms * 16));
  k_map_cloud_scatter<<<(unsigned)blocks, kCloudThreads, 0, s>>>(a);
}

void launch_map_occupancy(const MapOccupancy& a, int sms, cudaStream_t s) {
  const long long nblocks = (long long)a.nlayers * a.nmaps;
  if (nblocks <= 0 || a.cells <= 0) return;
  const long long by = std::min<long long>(nblocks, 65535);
  const long long per_block = (a.cells / 4 + 8 + 255) / 256;  // thread blocks that cover one (layer, map) block at one word each
  const long long bx = std::max<long long>(1, std::min<long long>(per_block, ((long long)sms * 32 + by - 1) / by));
  k_map_occupancy<<<dim3((unsigned)bx, (unsigned)by), 256, 0, s>>>(a);
}

void launch_map_at_poses(const MapAtPoses& a, int sms, cudaStream_t s) {
  const long long total = (long long)a.nposes * a.npoints;
  if (total <= 0) return;
  const long long blocks = std::min<long long>((total + 255) / 256, (long long)sms * 16);
  k_map_at_poses<<<(unsigned)blocks, 256, 0, s>>>(a);
}

void launch_uncertainty_range(const float* upper, const float* lower, float* out, size_t n, int sms, cudaStream_t s) {
  if (n == 0) return;
  const bool vec = n % 4 == 0 && ((reinterpret_cast<uintptr_t>(upper) | reinterpret_cast<uintptr_t>(lower) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0;
  const int V = vec ? 4 : 1;
  const size_t blocks = std::min<size_t>((n / V + 255) / 256, (size_t)sms * 16);
  if (vec) k_uncertainty_range<4><<<(unsigned)blocks, 256, 0, s>>>(upper, lower, out, n);
  else k_uncertainty_range<1><<<(unsigned)blocks, 256, 0, s>>>(upper, lower, out, n);
}

void launch_gather_submaps(const SubmapGather& a, int sms, cudaStream_t s) {
  if (a.ncolumns <= 0) return;
  const long long blocks = std::min<long long>((a.ncolumns + kGatherWarps - 1) / kGatherWarps, (long long)sms * 16);
  k_map_gather_submaps<<<(unsigned)blocks, kGatherWarps * 32, 0, s>>>(a);
}

void launch_cut_windows(const WindowCut& a, int sms, cudaStream_t s) {
  if (a.ncolumns <= 0) return;
  const long long blocks = std::min<long long>((a.ncolumns + kGatherWarps - 1) / kGatherWarps, (long long)sms * 16);
  k_map_cut_windows<<<(unsigned)blocks, kGatherWarps * 32, 0, s>>>(a);
}

void launch_valid_at(const GridGeo& g, const float* trav, int n, const double* xy, const int* pos_map, int nmaps, const double* map_pos,
                     unsigned char* valid, cudaStream_t s) {
  if (n <= 0) return;
  k_map_valid_at<<<(n + 255) / 256, 256, 0, s>>>(g, trav, n, xy, pos_map, nmaps, map_pos, valid);
}

}  // namespace te
