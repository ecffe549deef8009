// te_footprint.cu — TraversabilityMap::traversabilityFootprint(radius, offset) as two kernels.
//
//   k_predicates   isTraversableForFilters (TraversabilityMap.cpp:774-792) for every cell of the slab
//                  and its halo: checkForSlope (:867-893) and checkForStep (:794-865).  Both are pure
//                  functions of the layers (their slope_footprint / step_footprint layers are only
//                  memoisation), so they are evaluated once per cell instead of once per visit.  The
//                  gap walk of checkForStep decides on absolute double positions (submap geometry,
//                  dot products of perpendicular vectors, `norm < max_gap_width`), so this translation
//                  unit is compiled with --fmad=false and replays the reference's operand order.
//   k_sweep        isTraversable(center, radius + offset, ..., radius) (:654-746) for every cell:
//                  walk the SpiralIterator visit order (table built on the host by executing the
//                  iterator's own ring walk) until the first blocked cell.
//
// Layers are column-major float32; the slab/halo conventions are those of te_chain.
#include "te_footprint.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>

namespace te {
namespace {

struct Layers {
  const float* __restrict__ trav;
  const float* __restrict__ slope;
  const float* __restrict__ step;
  const float* __restrict__ elev;
  const float* __restrict__ rough;  // traversability_roughness, only read when verify_rough is set
};

struct FpArgs {
  int rows, cols_total, in_col0, in_ncols, out_col0, out_ncols;
  double res, lenx, leny, posx, posy;
  const double* X;
  const double* Y;
  double rmin, rmax, rmax2, tdefault, maxgap, crit;
  int int_norm;
  int verify_rough;  // checkForRoughness_ (TraversabilityMap.cpp:779)
  int n_spiral;
  const int* spiral;  // di & 0xff | (dj & 0xff) << 8 | edge << 16
  int slope_R, step_R;
  // prefix-sum sweep (k_fp_prepare_p / k_fp_nearest / k_sweep_fast)
  int L;                      // max |column offset| of the certain-in disk
  int nrings;                 // SpiralIterator nRings
  const signed char* halfw;   // [2L+1]: half-width of the certain-in disk per column offset (-1: none)
  const signed char* inner;   // [(nrings+2) x (2L+1)]: half-width of {k^2+l^2 < d^2} intersected with the disk, per ring d
  const int* ring_start;      // [nrings+2]: first index of ring d in `spiral`
  int n_fuzzy;                // offsets lying exactly on the circle: decided per cell on absolute positions
  const int* fuzzy;           // same packing as `spiral`
  const double* P;            // per input-buffer column: rows+1 prefix sums of t' along the row index
  const unsigned* bits;       // per input-buffer column: (rows+31)/32 words of blocked flags
  int words;                  // words per column
  const unsigned char* near;  // per input-buffer cell: distance (rows) to the nearest blocked cell of its column, 255 = none within 31
  signed char halfw_c[64];    // copy of `halfw` in the kernel parameters (constant bank)
  // full-disk sum without a blocked cell in sight (the common case): element offsets into the prefix sums, relative to the
  // centre's own entry P[column j][row i], of the two ends of disk column l (index l + L), and the running cell count
  int off_hi[64], off_lo[64];
  short cntp[65];
  // the same for k_sweep_fast as non-negative BYTE offsets from the prefix entry L columns and L rows before the centre's own
  // (one 32-bit add to a 64-bit base per load instead of a sign-extended 64-bit index computation)
  unsigned off8_hi[64], off8_lo[64];
  // maps of a batch (te_footprint_batched): map m's input buffer, predicate bytes, prefix sums, bit and nearest columns start
  // m * in_ncols columns into theirs, its outputs m * out_ncols columns into theirs.  The sweep kernels take m from blockIdx.z or
  // decode it from their flat index.  Kept last so that the path-check kernels, which do not read it, keep their parameter layout.
  int nmaps;
};

__device__ __forceinline__ float lay(const FpArgs& A, const float* l, int i, int j) {  // caller guarantees (i,j) is in the map
  const int lb = j - A.in_col0;
  if (lb < 0 || lb >= A.in_ncols) return nanf_();
  return __ldg(l + (size_t)lb * A.rows + i);
}

__device__ __forceinline__ bool is_inside_d(const FpArgs& A, double px, double py) {
  return grid_is_inside(A, px, py);
}

__device__ __forceinline__ bool get_index_d(const FpArgs& A, double px, double py, int& i, int& j) {
  return grid_get_index(A, px, py, i, j);
}

__device__ __forceinline__ void bound_position_d(const FpArgs& A, double& px, double& py) {
  grid_bound_position(A, px, py);
}

template <class F>
__device__ __forceinline__ void for_circle_d(const FpArgs& A, int i, int j, double r2, int R, F&& f) {
  const int a0 = max(0, i - R), a1 = min(A.rows - 1, i + R);
  const int b0 = max(0, j - R), b1 = min(A.cols_total - 1, j + R);
  const double cx = A.X[i], cy = A.Y[j];
  for (int a = a0; a <= a1; ++a) {
    const double dx = A.X[a] - cx;
    for (int b = b0; b <= b1; ++b) {
      const double dy = A.Y[b] - cy;
      if (dx * dx + dy * dy <= r2) f(a, b);
    }
  }
}

// TraversabilityMap::checkForSlope, TraversabilityMap.cpp:867-893.
__device__ bool check_slope_d(const FpArgs& A, const Layers& L, int i, int j) {
  if (!(lay(A, L.slope, i, j) == 0.0f)) return true;
  const double windowRadius = 3.0 * A.res;
  const double criticalLength = A.maxgap / 3.0;
  const int nCrit = (int)floor(2 * windowRadius * criticalLength / (A.res * A.res));
  int n = 0;
  for_circle_d(A, i, j, windowRadius * windowRadius, A.slope_R, [&](int a, int b) {
    if (lay(A, L.slope, a, b) == 0.0f) ++n;
  });
  return !(n > nCrit);
}

// TraversabilityMap::checkForRoughness, TraversabilityMap.cpp:895-921 (the slope check on another layer with another count).
__device__ bool check_rough_d(const FpArgs& A, const Layers& L, int i, int j) {
  if (!(lay(A, L.rough, i, j) == 0.0f)) return true;
  const double windowRadius = 3.0 * A.res;
  const double criticalLength = A.maxgap / 3.0;
  const int nCrit = (int)floor(1.5 * windowRadius * criticalLength / (A.res * A.res));
  int n = 0;
  for_circle_d(A, i, j, windowRadius * windowRadius, A.slope_R, [&](int a, int b) {
    if (lay(A, L.rough, a, b) == 0.0f) ++n;
  });
  return !(n > nCrit);
}

// TraversabilityMap::checkForStep, TraversabilityMap.cpp:794-865.
__device__ bool check_step_d(const FpArgs& A, const Layers& L, int i, int j) {
  if (!(lay(A, L.step, i, j) == 0.0f)) return true;
  const double crit = A.crit;
  const double wr = 2.5 * A.res;
  const double cx = A.X[i], cy = A.Y[j];
  const double h0 = (double)lay(A, L.elev, i, j);
  // candidate cells of the 2.5*res circle (at most 21): a bit per box cell, row index outer
  const int R = A.step_R;
  unsigned long long cand = 0ull;
  {
    const int a0 = max(0, i - R), a1 = min(A.rows - 1, i + R);
    const int b0 = max(0, j - R), b1 = min(A.cols_total - 1, j + R);
    for (int a = a0; a <= a1; ++a) {
      const double dx = A.X[a] - cx;
      for (int b = b0; b <= b1; ++b) {
        const double dy = A.Y[b] - cy;
        if (!(dx * dx + dy * dy <= wr * wr)) continue;
        if ((double)lay(A, L.elev, a, b) > crit + h0 && lay(A, L.step, a, b) == 0.0f)
          cand |= 1ull << ((a - (i - R)) * (2 * R + 1) + (b - (j - R)));
      }
    }
  }
  const bool self_only = cand == 0ull;
  if (self_only) cand = 1ull << (R * (2 * R + 1) + R);
  for (int bit = 0; bit < (2 * R + 1) * (2 * R + 1); ++bit) {
    if (!((cand >> bit) & 1ull)) continue;
    const int a = i - R + bit / (2 * R + 1), b = j - R + bit % (2 * R + 1);
    const double sx = A.X[a], sy = A.Y[b];      // subMapPos
    const double tcx = cx - sx, tcy = cy - sy;  // toCenter
    const double half = 0.5 * (2.5 * A.res);
    double tlx = sx + half, tly = sy + half;
    bound_position_d(A, tlx, tly);
    int ti, tj, bi, bj;
    if (!get_index_d(A, tlx, tly, ti, tj)) return false;
    double brx = sx - half, bry = sy - half;
    bound_position_d(A, brx, bry);
    if (!get_index_d(A, brx, bry, bi, bj)) return false;
    const double cornx = A.X[ti] + 0.5 * A.res, corny = A.Y[tj] + 0.5 * A.res;
    const int srows = bi - ti + 1, scols = bj - tj + 1;
    const double slx = (double)srows * A.res, sly = (double)scols * A.res;
    const double spx = cornx - 0.5 * slx, spy = corny - 0.5 * sly;
    const double height = (double)lay(A, L.elev, a, b);
    for (int k = 0; k < srows * scols; ++k) {
      const int si = k % srows, sj = k / srows;
      const int pi = ti + si, pj = tj + sj;
      if (!(lay(A, L.step, pi, pj) == 0.0f && (double)lay(A, L.elev, pi, pj) < height - crit)) continue;
      double px = cell_coord(spx, slx, A.res, si), py = cell_coord(spy, sly, A.res, sj);
      const double vx = px - sx, vy = py - sy;
      if (sqrt(vx * vx + vy * vy) < 0.025) continue;
      if (sqrt(tcx * tcx + tcy * tcy) > 0.025) {
        if (tcx * vx + tcy * vy < 0.0) continue;
      }
      px = sx + vx;
      py = sy + vy;
      for (;;) {
        const double ex = (px - sx) + vx, ey = (py - sy) + vy;
        if (!(sqrt(ex * ex + ey * ey) < A.maxgap && is_inside_d(A, px + vx, py + vy))) break;
        px = px + vx;
        py = py + vy;
      }
      int ei, ej;
      get_index_d(A, px, py, ei, ej);
      // LineIterator (Bresenham) from (a,b) to (ei,ej)
      const int dx = abs(ei - a), dy = abs(ej - b);
      int i1x = (ei >= a) ? 1 : -1, i2x = i1x, i1y = (ej >= b) ? 1 : -1, i2y = i1y;
      int den, num, numAdd, nCells;
      if (dx >= dy) { i1x = 0; i2y = 0; den = dx; num = dx / 2; numAdd = dy; nCells = dx + 1; }
      else { i2x = 0; i1y = 0; den = dy; num = dy / 2; numAdd = dx; nCells = dy + 1; }
      int li = a, lj = b;
      bool gapStart = false, gapEnd = false;
      for (int c = 0; c < nCells; ++c) {
        if (li < 0 || lj < 0 || li >= A.rows || lj >= A.cols_total) break;
        const float ef = lay(A, L.elev, li, lj);
        const double e = (double)ef;
        if (e > height + crit) return false;
        if (e < height - crit || !finitef(ef)) {
          gapStart = true;
        } else if (gapStart) {
          gapEnd = true;
          break;
        }
        num += numAdd;
        if (num >= den) { num -= den; li += i1x; lj += i1y; }
        li += i2x; lj += i2y;
      }
      if (gapStart && !gapEnd) return false;
    }
  }
  return true;
}

// isTraversableForFilters (TraversabilityMap.cpp:774-792) of one cell, with the memoisation-layer values the reference leaves
// behind (NaN where a check did not run on a zero cell).
struct FilterVerdict {
  bool ok;
  float sfp, tfp, rfp;
};
__device__ __forceinline__ FilterVerdict filters_d(const FpArgs& A, const Layers& L, int i, int j) {
  FilterVerdict v{true, nanf_(), nanf_(), nanf_()};
  const bool s_ok = check_slope_d(A, L, i, j);
  bool t_ok = true;
  if (lay(A, L.slope, i, j) == 0.0f) v.sfp = s_ok ? 1.0f : 0.0f;
  if (s_ok) {
    t_ok = check_step_d(A, L, i, j);
    if (lay(A, L.step, i, j) == 0.0f) v.tfp = t_ok ? 1.0f : 0.0f;
  }
  bool r_ok = true;
  if (A.verify_rough && s_ok && t_ok) {  // TraversabilityMap.cpp:779-783: only after slope and step passed
    r_ok = check_rough_d(A, L, i, j);
    if (lay(A, L.rough, i, j) == 0.0f) v.rfp = r_ok ? 1.0f : 0.0f;
  }
  v.ok = s_ok && t_ok && r_ok;
  return v;
}

// SpiralIterator::getCurrentRadius (index-space norm of the offset; Eigen's integer norm when int_norm is set) in metres.
__device__ __forceinline__ double current_radius_d(const FpArgs& A, int di, int dj) {
  const int d2 = di * di + dj * dj;
  const double nr = A.int_norm ? (double)(int)sqrt((double)d2) : sqrt((double)d2);
  return nr * A.res;
}

// isTraversableForFilters for every cell of the input buffer (columns in_col0 .. in_col0+in_ncols), in two steps.  Almost every
// cell passes trivially — checkForSlope / checkForStep / checkForRoughness return true at once unless the cell's own layer
// value is exactly 0 (TraversabilityMap.cpp:869, :796, :897) — so k_pred_classify settles those with two or three coalesced
// loads and collects the others on a work list, which k_pred_heavy walks with one thread per listed cell (the window count,
// the submap / gap walk): the heavy threads are no longer scattered one or two per warp over the whole map.
__global__ void __launch_bounds__(256) k_pred_classify(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp,
                                                       float* step_fp, float* rough_fp, unsigned* __restrict__ list,
                                                       unsigned* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lb = blockIdx.y;
  const bool in = i < A.rows;
  bool heavy = false;
  size_t c = 0;
  if (in) {
    c = ((unsigned)blockIdx.z * A.in_ncols + lb) * (unsigned)A.rows + i;  // cell of the batch, < 2^32: the work list stores it
    heavy = __ldg(L.slope + c) == 0.0f || __ldg(L.step + c) == 0.0f || (A.verify_rough && __ldg(L.rough + c) == 0.0f);
    if (!heavy) {
      blocked[c] = 0;
      const int oj = lb + A.in_col0 - A.out_col0;
      if (oj >= 0 && oj < A.out_ncols) {
        const size_t oc = ((unsigned)blockIdx.z * A.out_ncols + oj) * (unsigned)A.rows + i;
        if (slope_fp) slope_fp[oc] = nanf_();
        if (step_fp) step_fp[oc] = nanf_();
        if (rough_fp) rough_fp[oc] = nanf_();
      }
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, heavy);
  if (m) {
    const int lane = threadIdx.x & 31;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(count, (unsigned)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (heavy) list[base + __popc(m & ((1u << lane) - 1u))] = (unsigned)c;
  }
}

__global__ void __launch_bounds__(128) k_pred_heavy(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp, float* step_fp,
                                                    float* rough_fp, const unsigned* __restrict__ list, const unsigned* __restrict__ count) {
  const unsigned n = *count;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const unsigned c = list[k];
    const int i = (int)(c % (unsigned)A.rows);
    const unsigned col = c / (unsigned)A.rows;            // input-buffer column of the batch
    const unsigned m = col / (unsigned)A.in_ncols;        // its map
    const int j = A.in_col0 + (int)(col - m * (unsigned)A.in_ncols);
    const size_t mc = (size_t)m * A.in_ncols * A.rows;    // the map's first cell: filters_d reads its layers only
    const Layers Lm{L.trav + mc, L.slope + mc, L.step + mc, L.elev + mc, L.rough ? L.rough + mc : nullptr};
    const FilterVerdict v = filters_d(A, Lm, i, j);
    blocked[c] = v.ok ? 0 : 1;
    const int oj = j - A.out_col0;
    if (oj >= 0 && oj < A.out_ncols) {
      const size_t oc = ((size_t)m * A.out_ncols + oj) * A.rows + i;
      if (slope_fp) slope_fp[oc] = v.sfp;
      if (step_fp) step_fp[oc] = v.tfp;
      if (rough_fp) rough_fp[oc] = v.rfp;
    }
  }
}

__global__ void __launch_bounds__(256) k_sweep(FpArgs A, Layers L, const unsigned char* __restrict__ blocked, float* __restrict__ out) {
  const long long total = (long long)A.rows * A.out_ncols * A.nmaps;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % A.rows);
    const unsigned col = (unsigned)(c / A.rows);  // output column of the batch
    const unsigned m = col / (unsigned)A.out_ncols;
    const int j = A.out_col0 + (int)(col - m * (unsigned)A.out_ncols);
    const size_t mc = (size_t)m * A.in_ncols * A.rows;  // the map's first input cell
    const double cx = A.X[i], cy = A.Y[j];
    int n = 0;
    double t = 0.0;
    float result = nanf_();
    bool done = false;
    for (int k = 0; k < A.n_spiral; ++k) {
      const int w = __ldg(A.spiral + k);
      const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
      const int a = i + di, b = j + dj;
      if (a < 0 || b < 0 || a >= A.rows || b >= A.cols_total) continue;
      if (w & 0x10000) {
        const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
        if (!(dx * dx + dy * dy <= A.rmax2)) continue;
      }
      const int lb = b - A.in_col0;
      if (lb < 0 || lb >= A.in_ncols) continue;  // cannot happen with the halo te_footprint demands
      const size_t cc = mc + (size_t)lb * A.rows + a;
      if (blocked[cc]) {
        const int d2 = di * di + dj * dj;
        const double nr = A.int_norm ? (double)(int)sqrt((double)d2) : sqrt((double)d2);
        const double uR = nr * A.res;
        if (A.rmin == 0.0 || uR <= A.rmin) {
          result = 0.0f;
        } else {
          const double factor = ((uR - A.rmin) / (A.rmax - A.rmin) + 1.0) / 2.0;
          t *= factor / (double)n;
          result = (float)t;
        }
        done = true;
        break;
      }
      ++n;
      const float v = __ldg(L.trav + cc);
      t += finitef(v) ? (double)v : A.tdefault;
    }
    if (!done) {
      t /= (double)n;
      result = (float)t;
    }
    out[c] = result;
  }
}

// Distance along the row index from every cell to the nearest blocked cell of its own column (from the packed flags):
// the sweep then needs ONE byte per disk column to know the nearest blocked cell of that column.
__global__ void __launch_bounds__(256) k_fp_nearest(FpArgs A, unsigned char* __restrict__ near) {
  const long long total = (long long)A.rows * A.in_ncols * A.nmaps;  // every column of the batch: they are independent
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % A.rows);
    const unsigned* wcol = A.bits + (size_t)(c / A.rows) * A.words;
    const int r0 = i - 31, w0 = r0 >> 5, sh = r0 & 31;
    const unsigned a0 = (w0 >= 0 && w0 < A.words) ? __ldg(wcol + w0) : 0u;
    const unsigned a1 = (w0 + 1 >= 0 && w0 + 1 < A.words) ? __ldg(wcol + w0 + 1) : 0u;
    const unsigned a2 = (w0 + 2 >= 0 && w0 + 2 < A.words) ? __ldg(wcol + w0 + 2) : 0u;
    const unsigned long long lo = ((unsigned long long)a1 << 32) | a0;
    unsigned long long f = (lo >> sh) | (sh ? ((unsigned long long)a2 << (64 - sh)) : 0ull);  // bit t <-> row r0 + t, centre at bit 31
    f &= ~(1ull << 63);                                                                        // rows i-31 .. i+31
    int kmin = 255;
    const unsigned long long up = f >> 31, dn = f & ((1ull << 31) - 1ull);
    if (up) kmin = __ffsll((long long)up) - 1;
    if (dn) kmin = min(kmin, 31 - (63 - __clzll((long long)dn)));
    near[c] = (unsigned char)kmin;
  }
}

// One warp per input-buffer column: prefix sums of t' = finite(traversability) ? value : default along the row
// index (double; exact for float32 terms, so the order of summation does not matter) and packed blocked flags.
__global__ void __launch_bounds__(256) k_fp_prepare_p(FpArgs A, Layers L, const unsigned char* __restrict__ blocked, double* __restrict__ P,
                                                    unsigned* __restrict__ bits) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int ncols = A.in_ncols * A.nmaps;  // every column of the batch: they are independent
  for (int lb = warp; lb < ncols; lb += nwarps) {
    const float* tcol = L.trav + (size_t)lb * A.rows;
    const unsigned char* bcol = blocked + (size_t)lb * A.rows;
    double* pcol = P + (size_t)lb * (A.rows + 1);
    unsigned* wcol = bits + (size_t)lb * A.words;
    double carry = 0.0;
    if (lane == 0) pcol[0] = 0.0;
    for (int base = 0; base < A.rows; base += 32) {
      const int i = base + lane;
      double v = 0.0;
      bool b = false;
      if (i < A.rows) {
        const float t = __ldg(tcol + i);
        v = finitef(t) ? (double)t : A.tdefault;
        b = bcol[i] != 0;
      }
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const double o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += o;
      }
      if (i < A.rows) pcol[i + 1] = carry + v;
      const unsigned w = __ballot_sync(0xffffffffu, b);
      if (lane == 0) wcol[base >> 5] = w;
      carry += __shfl_sync(0xffffffffu, v, 31);
    }
  }
}

// isTraversable for every cell on prefix sums: the visited set is a lattice disk, so "is anything blocked in it"
// and "sum / count of the visited cells" are 2L+1 column queries instead of ~pi r^2 visits; only when a blocker
// exists is the ring that holds the first one walked in SpiralIterator order.
__global__ void __launch_bounds__(256) k_sweep_fast(FpArgs A, Layers L, const unsigned char* __restrict__ blocked, float* __restrict__ out) {
  const int W = 2 * A.L + 1;
  // one block = 256 consecutive rows of ONE output column (blockIdx.y): a warp's centres share their column, so everything that
  // depends only on the column — which disk columns exist, whether any blocked cell lies near the warp at all — is warp-uniform
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = A.out_col0 + (int)blockIdx.y;
  // map blockIdx.z of the batch: its predicate bytes, prefix sums, bit and nearest columns start mb columns into the batch's
  // (mb + any input-buffer column < 2^31, which run_predicates checks); column b of the map is batch column b - c0
  const int mb = (int)blockIdx.z * A.in_ncols, c0 = A.in_col0 - mb;
  {
    const int lane = threadIdx.x & 31, i0 = i - lane;
    if (i0 >= A.rows) return;  // whole warp beyond the last row
    const bool active = i < A.rows;
    const size_t c = ((unsigned)blockIdx.z * A.out_ncols + blockIdx.y) * (unsigned)A.rows + (active ? i : 0);  // < 2^32
    const double cx = A.X[active ? i : 0], cy = A.Y[j];
    // disk columns that exist in the map and in this slab's buffer.  l_lo is written as a negated minimum: ptxas of CUDA 12.9 for
    // sm_90a fuses max(-L, max(-j, in_col0 - j)) into one three-input VIMNMX3 that reads +L, and the loops bounded by l_hi then ran
    // past it whenever the disk is clipped on the right
    const int l_lo = -min(A.L, min(j, j - A.in_col0)), l_hi = min(A.L, min(A.cols_total - 1 - j, A.in_col0 + A.in_ncols - 1 - j));
    // ---- warp-wide early out: is any cell blocked in the box of rows [i0 - L, i0 + 31 + L] x disk columns?  (packed flags,
    //      a few words per column, shared by the 32 centres)  Mostly not: then no lane has anything to look for.
    bool warp_any;
    {
      const int w0 = max(i0 - A.L, 0) >> 5, w1 = min(i0 + 31 + A.L, A.rows - 1) >> 5;
      unsigned acc = 0;
      for (int l = l_lo + lane; l <= l_hi; l += 32) {  // a lane per disk column, at most four words each
        const unsigned* wc = A.bits + (size_t)(j + l - c0) * A.words;
        for (int w = w0; w <= w1; ++w) acc |= __ldg(wc + w);
      }
      warp_any = __any_sync(0xffffffffu, acc != 0u);
    }
    if (!active) return;
    // ---- nearest blocked cell of the visited set, as a squared index distance ------------------------
    int best = 0x7fffffff;
    if (warp_any) {
      const unsigned char* nr = A.near + (size_t)(j + l_lo - c0) * A.rows + i;
      for (int l = l_lo; l <= l_hi; ++l, nr += A.rows) {
        const int g = (int)__ldg(nr);              // nearest blocked row offset in this column
        const int hw = A.halfw_c[l + A.L];
        if (g <= hw) best = min(best, g * g + l * l);
      }
      for (int q = 0; q < A.n_fuzzy; ++q) {
        const int w = A.fuzzy[q];
        const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
        const int a = i + di, b = j + dj, lb = b - A.in_col0;
        if (a < 0 || b < 0 || a >= A.rows || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
        const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
        if (!(dx * dx + dy * dy <= A.rmax2)) continue;
        if (blocked[(size_t)(mb + lb) * A.rows + a]) best = min(best, di * di + dj * dj);
      }
    }
    // ---- sums over the visited cells before the first blocked one --------------------------------------
    const bool any = best != 0x7fffffff;
    const int dstar = any ? (int)sqrt((double)best) : A.nrings + 1;  // ring of the first blocked cell
    // The first blocked cell in visit order lies in ring dstar: its index-space radius is in [dstar, dstar + 1) (exactly dstar with
    // the integer norm).  Within the inner radius the result is 0 (TraversabilityMap.cpp:694-704) whatever the sums are: most
    // centres near an obstacle end here, without prefix sums or a ring walk.
    if (any && (A.rmin == 0.0 || (A.int_norm ? (double)dstar : (double)(dstar + 1)) * A.res <= A.rmin)) {
      out[c] = 0.0f;
      return;
    }
    const signed char* hwt = any ? (A.inner + (size_t)dstar * W) : A.halfw;
    double t = 0.0, t_b = 0.0;
    int n = 0;
    if (!warp_any && i - A.L >= 0 && i + A.L < A.rows) {
      // nothing blocked near this warp and no clipping along the rows: 2 loads and 2 additions per disk column, offsets from
      // the constant bank
      // biased base: the entry L columns and L rows before the centre's own, so that every table offset is a non-negative byte count
      const char* pb = reinterpret_cast<const char*>(A.P + ((size_t)(j - c0) * ((size_t)A.rows + 1) + i)) -
                       8 * ((ptrdiff_t)A.L * ((ptrdiff_t)A.rows + 1) + A.L);
      auto P8 = [&](unsigned off) { return __ldg(reinterpret_cast<const double*>(pb + off)); };
      int l = l_lo + A.L;
      const int l_end = l_hi + A.L;
      for (; l + 1 <= l_end; l += 2) {
        t += P8(A.off8_hi[l]) - P8(A.off8_lo[l]);
        t_b += P8(A.off8_hi[l + 1]) - P8(A.off8_lo[l + 1]);
      }
      if (l <= l_end) t += P8(A.off8_hi[l]) - P8(A.off8_lo[l]);
      t += t_b;
      n = (int)A.cntp[l_end + 1] - (int)A.cntp[l_lo + A.L];
    } else {
      const double* pc = A.P + (size_t)(j + l_lo - c0) * (A.rows + 1);
      const size_t pstride = (size_t)A.rows + 1;
      if (i - A.L >= 0 && i + A.L < A.rows) {  // no clipping along the rows: two independent accumulators
        int l = l_lo;
        for (; l + 1 <= l_hi; l += 2, pc += 2 * pstride) {
          const int h0 = hwt[l + A.L], h1 = hwt[l + 1 + A.L];
          if (h0 >= 0) { t += pc[i + h0 + 1] - pc[i - h0]; n += 2 * h0 + 1; }
          if (h1 >= 0) { t_b += pc[pstride + i + h1 + 1] - pc[pstride + i - h1]; n += 2 * h1 + 1; }
        }
        if (l <= l_hi) {
          const int h0 = hwt[l + A.L];
          if (h0 >= 0) { t += pc[i + h0 + 1] - pc[i - h0]; n += 2 * h0 + 1; }
        }
      } else {
        for (int l = l_lo; l <= l_hi; ++l, pc += pstride) {
          const int hw = hwt[l + A.L];
          if (hw < 0) continue;
          const int a0 = max(i - hw, 0), a1 = min(i + hw, A.rows - 1);
          t += pc[a1 + 1] - pc[a0];
          n += a1 - a0 + 1;
        }
      }
      t += t_b;
    }
    float result;
    if (!any) {
      for (int q = 0; q < A.n_fuzzy; ++q) {  // on-circle cells belong to the last ring: they are visited last
        const int w = A.fuzzy[q];
        const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
        const int a = i + di, b = j + dj, lb = b - A.in_col0;
        if (a < 0 || b < 0 || a >= A.rows || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
        const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
        if (!(dx * dx + dy * dy <= A.rmax2)) continue;
        const float v = __ldg(L.trav + (size_t)(mb + lb) * A.rows + a);
        t += finitef(v) ? (double)v : A.tdefault;
        ++n;
      }
      t /= (double)n;
      result = (float)t;
    } else {
      // walk ring dstar in visit order up to its first blocked cell
      int di = 0, dj = 0;
      for (int k = A.ring_start[dstar]; k < A.ring_start[dstar + 1]; ++k) {
        const int w = __ldg(A.spiral + k);
        di = (int)(signed char)(w & 0xff);
        dj = (int)(signed char)((w >> 8) & 0xff);
        const int a = i + di, b = j + dj, lb = b - A.in_col0;
        if (a < 0 || b < 0 || a >= A.rows || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
        if (w & 0x10000) {
          const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
          if (!(dx * dx + dy * dy <= A.rmax2)) continue;
        }
        const size_t cc = (size_t)(mb + lb) * A.rows + a;
        if (blocked[cc]) break;
        const float v = __ldg(L.trav + cc);
        t += finitef(v) ? (double)v : A.tdefault;
        ++n;
      }
      const int d2 = di * di + dj * dj;
      const double nr = A.int_norm ? (double)(int)sqrt((double)d2) : sqrt((double)d2);
      const double uR = nr * A.res;
      if (A.rmin == 0.0 || uR <= A.rmin) {
        result = 0.0f;
      } else {
        const double factor = ((uR - A.rmin) / (A.rmax - A.rmin) + 1.0) / 2.0;
        t *= factor / (double)n;
        result = (float)t;
      }
    }
    out[c] = result;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Polygonal footprint sweep: TraversabilityMap::traversabilityFootprint(double footprintYaw), TraversabilityMap.cpp:239-305, with the
// polygon isTraversable (:592-645).  Every cell gets the footprint polygon placed at its centre; the value is 0 when a cell of the
// polygon fails isTraversableForFilters, otherwise the mean of t' over the polygon's cells (traversabilityDefault_ when it covers
// none).  The set of cells inside the polygon is the same offset pattern for every centre EXCEPT for offsets whose cell centre lies
// on (within rounding of) an edge: grid_map::Polygon::isInside decides those on absolute double coordinates, differently from
// centre to centre.  The host classifies the offsets once per polygon (launch_footprint_polygon): certain-in cells become per-column
// runs that are summed from the tile's prefix sums; the few uncertain offsets are decided per centre with the reference's own
// arithmetic — cooperatively when the decision does not depend on the centre's row (an edge parallel to the x axis through cell
// centres: the YAML footprint at 0.02 m has 92 such offsets), 32 offsets per warp pass.  One launch sweeps a list of polygons (the
// footprint at several yaws): a block stages its tile once and sweeps a group of them.
constexpr int PTR = 64, PTC = 16;  // tile of centres: rows x columns
constexpr int PMAXV = 16;          // polygon vertices
constexpr int PB = 130;            // pitch of a staged blocked-count column (uint16)
// Eigen::Quaternion::toRotationMatrix of (cos(yaw/2), 0, 0, sin(yaw/2)), upper-left 2 x 2
struct Rot2 {
  double r00, r01, r10, r11;
};
// One polygon of a sweep: the footprint placed with rotation R, its slices of the call's run and uncertain-offset tables, and its
// output layer (map m's starts m * rows * out_ncols cells into `out`).
struct PolyDesc {
  Rot2 R;
  int run0, nruns;    // runs[run0 .. run0 + nruns)
  int fz0, nfz;       // fz[fz0 .. fz0 + nfz)
  int ncert;          // number of certain cells (sum of the run lengths)
  float* out;
};
struct PolyArgs {
  int Lp;             // reach of the polygon in cells (<= 31), the same at every rotation
  int npts;
  int npoly;          // polygons of the launch
  int group;          // polygons per block: blockIdx.x = g * row_tiles + row tile sweeps polygons g * group .. (g + 1) * group - 1
  int row_tiles;
  const PolyDesc* desc;  // [npoly]
  const int* runs;    // (dj & 0xff) | (lo & 0xff) << 8 | (hi & 0xff) << 16: rows i+lo .. i+hi of column j+dj are certainly inside
  const int* fz;      // (di & 0xff) | (dj & 0xff) << 8 | flags << 16: uncertain offsets, sorted by (dj, di); flag bit 0: the decision
                      // depends on the centre's row; bit 1: same column as the previous entry, next row, neither depends on the row
  // Reduce mode (k_poly_tile<true>; the descriptors' `out` is unused): per centre, the value of the first polygon of the block's
  // group that minimises it (worst), of the first that maximises it (best) and that polygon's index (best_yaw); each null when not
  // wanted.  Group g writes at g * rstride cells (0 without a split; a split leaves the folding to k_poly_combine).
  float* worst;
  float* best;
  int* best_yaw;
  size_t rstride;
  double px[PMAXV], py[PMAXV];
};

// grid_map::Polygon::isInside for the polygon placed at (cx, cy): vertices = R * p + centre in the operand order of Eigen's
// Transform * vector (oracle: teo_footprint_polygon), crossing-number test over (v[i], v[i-1]).
__device__ bool poly_inside_d(const PolyArgs& Q, const Rot2& R, double cx, double cy, double ptx, double pty) {
  int cross = 0;
  const int last = Q.npts - 1;
  double jx = cx + ((R.r00 * Q.px[last] + R.r01 * Q.py[last]) + 0.0);
  double jy = cy + ((R.r10 * Q.px[last] + R.r11 * Q.py[last]) + 0.0);
  for (int k = 0; k < Q.npts; ++k) {
    const double ix = cx + ((R.r00 * Q.px[k] + R.r01 * Q.py[k]) + 0.0);
    const double iy = cy + ((R.r10 * Q.px[k] + R.r11 * Q.py[k]) + 0.0);
    if (((iy > pty) != (jy > pty)) && (ptx < (jx - ix) * (pty - iy) / (jy - iy) + ix)) ++cross;
    jx = ix;
    jy = iy;
  }
  return (cross & 1) != 0;
}

// The tile geometry (PTR x PTC centres, staging origin r0 - Lp, c0 - Lp) is part of the results: a sum over a run is a difference
// of the staged prefix sums, whose float32 rounding depends on where the staged column starts.  kReduce: reduce over the block's
// polygons in registers instead of storing a layer per polygon (PolyArgs::worst / best / best_yaw).
template <bool kReduce>
__global__ void __launch_bounds__(256) k_poly_tile(FpArgs A, PolyArgs Q, const float* __restrict__ trav, const unsigned char* __restrict__ blocked) {
  extern __shared__ double sP[];  // [NC][PS] prefix sums of t'; then [NC][PB] uint16 prefix counts of blocked cells
  const int Lr = Q.Lp, NR = PTR + 2 * Lr, NC = PTC + 2 * Lr, PS = NR + 1;
  unsigned short* sB = reinterpret_cast<unsigned short*>(sP + (size_t)NC * PS);
  // map blockIdx.z of the batch: its input-buffer columns start mb columns into the batch's, its output columns mbo
  const int mb = (int)blockIdx.z * A.in_ncols, mbo = (int)blockIdx.z * A.out_ncols;
  const int tile_r = (int)blockIdx.x % Q.row_tiles, p0 = ((int)blockIdx.x / Q.row_tiles) * Q.group, p1 = min(p0 + Q.group, Q.npoly);
  const int r0 = tile_r * PTR, c0 = A.out_col0 + (int)blockIdx.y * PTC;
  const int rb = r0 - Lr, cb = c0 - Lr;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // ---- phase 1: prefix sums of t' and of the blocked flags, one warp per staged column.  NR <= 4 * 32 (Lp <= 31): a lane takes
  //      four consecutive rows, scans them in registers, the warp scans the lane totals.  Cells outside the map or the slab's
  //      buffer contribute 0, so the sums need no clipping.
  int anyb = 0;
  for (int cc = warp; cc < NC; cc += 8) {
    const int gcol = cb + cc, lb = gcol - A.in_col0;
    const bool col_ok = gcol >= 0 && gcol < A.cols_total && lb >= 0 && lb < A.in_ncols;
    const float* tcol = trav + (size_t)(mb + (col_ok ? lb : 0)) * A.rows;
    const unsigned char* bcol = blocked + (size_t)(mb + (col_ok ? lb : 0)) * A.rows;
    double v[4];
    int cb4[4];
    unsigned bw = 0;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = 4 * lane + m, row = rb + k;
      v[m] = 0.0;
      cb4[m] = 0;
      if (k < NR && col_ok && row >= 0 && row < A.rows) {
        const float t = __ldg(tcol + row);
        v[m] = finitef(t) ? (double)t : A.tdefault;
        cb4[m] = bcol[row] != 0 ? 1 : 0;
        bw |= (unsigned)cb4[m] << (8 * m);
      }
    }
    anyb |= (int)bw;
    v[1] += v[0]; v[2] += v[1]; v[3] += v[2];
    cb4[1] += cb4[0]; cb4[2] += cb4[1]; cb4[3] += cb4[2];
    double tot = v[3];
    int ctot = cb4[3];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const double o = __shfl_up_sync(0xffffffffu, tot, d);
      const int oc = __shfl_up_sync(0xffffffffu, ctot, d);
      if (lane >= d) { tot += o; ctot += oc; }
    }
    double before = __shfl_up_sync(0xffffffffu, tot, 1);
    int cbefore = __shfl_up_sync(0xffffffffu, ctot, 1);
    if (lane == 0) { before = 0.0; cbefore = 0; }
    double* pcol = sP + (size_t)cc * PS;
    unsigned short* ccol = sB + (size_t)cc * PB;
    if (lane == 0) { pcol[0] = 0.0; ccol[0] = 0; }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = 4 * lane + m;
      if (k < NR) { pcol[k + 1] = before + v[m]; ccol[k + 1] = (unsigned short)(cbefore + cb4[m]); }
    }
  }
  const bool tile_any = __syncthreads_or(anyb) != 0;
  // ---- phase 2: a warp is 32 consecutive rows of one column at a time (4 columns per warp), each centre swept for every polygon
  //      of the block's group
  const int i = r0 + (warp & 1) * 32 + lane;
  const int i0 = i - lane;
  if (i0 >= A.rows) return;
  const bool active = i < A.rows;
  const int ic = active ? i : A.rows - 1;
  const double cx = A.X[ic];
  const int k0 = ic - rb;
  for (int q = 0; q < PTC / 4; ++q) {
    const int j = c0 + (warp >> 1) * (PTC / 4) + q;
    if (j >= A.out_col0 + A.out_ncols) break;
    const double cy = A.Y[j];
    // certain cells: per-column runs from the prefix sums (cells outside the map were staged as t' = 0, not blocked)
    const double* pbase = sP + (size_t)(j - cb) * PS + k0;
    const unsigned short* bbase = sB + (size_t)(j - cb) * PB + k0;
    const bool interior = ic - Lr >= 0 && ic + Lr < A.rows && j - Lr >= max(0, A.in_col0) && j + Lr <= min(A.cols_total, A.in_col0 + A.in_ncols) - 1;
    // reduce mode: every value is finite (the callers reject a non-finite traversability_default), so the infinities lose to the
    // first polygon, and strict comparisons keep the earliest polygon of a tie with its own bits (-0.0 and +0.0 included)
    float worst = __int_as_float(0x7f800000), best = __int_as_float(0xff800000);
    int best_y = p0;
    for (int y = p0; y < p1; ++y) {
      const PolyDesc& D = Q.desc[y];
      const Rot2 R = D.R;
      const int* const runs = Q.runs + D.run0;
      const int* const fz = Q.fz + D.fz0;
      const int nruns = D.nruns, nfz = D.nfz;
      double t = 0.0;
      int n = 0, nblk = 0;
      if (interior) {  // no clipping anywhere: the cell count is the table's
        for (int r = 0; r < nruns; ++r) {
          const int w = __ldg(runs + r);
          const int dj = (int)(signed char)(w & 0xff), lo = (int)(signed char)((w >> 8) & 0xff), hi = (int)(signed char)((w >> 16) & 0xff);
          const double* pc = pbase + dj * PS;
          t += pc[hi + 1] - pc[lo];
          if (tile_any) {
            const unsigned short* bc = bbase + dj * PB;
            nblk += (int)bc[hi + 1] - (int)bc[lo];
          }
        }
        n = D.ncert;
      } else {
        for (int r = 0; r < nruns; ++r) {
          const int w = __ldg(runs + r);
          const int dj = (int)(signed char)(w & 0xff), lo = (int)(signed char)((w >> 8) & 0xff), hi = (int)(signed char)((w >> 16) & 0xff);
          const int b = j + dj, lb = b - A.in_col0;
          if (b < 0 || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
          const int a0 = max(ic + lo, 0), a1 = min(ic + hi, A.rows - 1);
          if (a0 > a1) continue;
          const double* pc = pbase + dj * PS;
          t += pc[hi + 1] - pc[lo];
          n += a1 - a0 + 1;
          if (tile_any) {
            const unsigned short* bc = bbase + dj * PB;
            nblk += (int)bc[hi + 1] - (int)bc[lo];
          }
        }
      }
      // uncertain offsets, 32 per pass: lane l decides offset base + l when the decision is the same for every row of the column; the
      // offsets that came out inside and follow each other down a column are then summed as ONE run from the prefix sums
      for (int base = 0; base < nfz; base += 32) {
        const int idx = base + lane;
        int w = 0;
        bool cand = false;
        if (idx < nfz) {
          w = __ldg(fz + idx);
          const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
          if ((w >> 16) & 1) {
            cand = true;  // depends on the row: every lane decides for itself below
          } else {
            const int a = ic + di, b = j + dj;
            // the decision does not depend on the row, so any row's coordinates will do — but they must exist
            const int ar = min(max(a, 0), A.rows - 1), icr = ar - di;
            if (b >= 0 && b < A.cols_total && icr >= 0 && icr < A.rows) cand = poly_inside_d(Q, R, A.X[icr], cy, A.X[ar], A.Y[b]);
          }
        }
        unsigned m = __ballot_sync(0xffffffffu, cand);
        const unsigned ext = m & __ballot_sync(0xffffffffu, ((w >> 17) & 1) != 0);  // inside AND continues its predecessor down the column
        while (m) {
          const int src = __ffs((int)m) - 1;
          const unsigned tail = src == 31 ? 0u : (ext >> (src + 1));
          const int len = __ffs((int)~tail) - 1;  // further entries of the run (0..31 - src)
          m &= ~((len >= 31 ? 0xffffffffu : ((2u << len) - 1u)) << src);
          const int wv = __shfl_sync(0xffffffffu, w, src);
          const int di = (int)(signed char)(wv & 0xff), dj = (int)(signed char)((wv >> 8) & 0xff);
          const int b = j + dj, lb = b - A.in_col0;
          if (b < 0 || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
          const int a0 = ic + di, a1 = a0 + len;
          const int a0c = max(a0, 0), a1c = min(a1, A.rows - 1);
          if (a0c > a1c) continue;
          if (((wv >> 16) & 1) && !poly_inside_d(Q, R, cx, cy, A.X[a0], A.Y[b])) continue;  // row-dependent entries never chain (len == 0)
          const int cc = b - cb;
          const double* pc = sP + (size_t)cc * PS + (a0 - rb);
          t += pc[len + 1] - pc[0];
          n += a1c - a0c + 1;
          if (tile_any) {
            const unsigned short* bc = sB + (size_t)cc * PB + (a0 - rb);
            nblk += (int)bc[len + 1] - (int)bc[0];
          }
        }
      }
      float result;
      if (nblk > 0) result = 0.0f;                       // :297 / :301
      else if (n == 0) result = (float)A.tdefault;       // :625-628
      else result = (float)(t / (double)n);              // :630
      if constexpr (kReduce) {
        if (result < worst) worst = result;
        if (result > best) { best = result; best_y = y; }
      } else {
        if (active) D.out[(size_t)(mbo + j - A.out_col0) * A.rows + i] = result;
      }
    }
    if constexpr (kReduce) {
      if (active) {
        const size_t o = (size_t)(p0 / Q.group) * Q.rstride + (size_t)(mbo + j - A.out_col0) * A.rows + i;
        if (Q.worst) Q.worst[o] = worst;
        if (Q.best) Q.best[o] = best;
        if (Q.best_yaw) Q.best_yaw[o] = best_y;
      }
    }
  }
}

// Reduce mode after a yaw-group split: k_poly_tile left group g's partial reduction at g * n cells of each scratch array (sw: worst,
// sb: best, sk: best_yaw; sb is there when best or best_yaw is wanted).  The groups are runs of consecutive polygons in order, so
// folding them in group order with the same strict comparisons gives the first minimum / maximum over all polygons.
__global__ void k_poly_combine(const float* __restrict__ sw, const float* __restrict__ sb, const int* __restrict__ sk, int ngroups, size_t n,
                               float* worst, float* best, int* best_yaw) {
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    if (worst) {
      float w = sw[c];
      for (int g = 1; g < ngroups; ++g) {
        const float v = sw[(size_t)g * n + c];
        if (v < w) w = v;
      }
      worst[c] = w;
    }
    if (sb) {
      float b = sb[c];
      int k = sk ? sk[c] : 0;
      for (int g = 1; g < ngroups; ++g) {
        const float v = sb[(size_t)g * n + c];
        if (v > b) { b = v; if (sk) k = sk[(size_t)g * n + c]; }
      }
      if (best) best[c] = b;
      if (best_yaw) best_yaw[c] = k;
    }
  }
}

// Is (a, b) one of the cells checkCircularFootprintPath checks on LineD(i0, j0, i1, j1), i.e. its cell c with c % 4 == 0
// (nSkip = 3, TraversabilityMap.cpp:401, :421-425)?  Closed form of the walk: after c steps the minor coordinate has moved
// floor((den / 2 + c * numAdd) / den) cells.
__device__ __forceinline__ bool line_checks_d(int i0, int j0, int i1, int j1, int a, int b) {
  const int dx = abs(i1 - i0), dy = abs(j1 - j0);
  const int sx = (i1 >= i0) ? 1 : -1, sy = (j1 >= j0) ? 1 : -1;
  if (dx >= dy) {
    if (dx == 0) return a == i0 && b == j0;
    const int c = (a - i0) * sx;
    if (c < 0 || c > dx || (c & 3)) return false;
    return b == j0 + sy * (int)(((long long)(dx / 2) + (long long)c * dy) / dx);
  }
  const int c = (b - j0) * sy;
  if (c < 0 || c > dy || (c & 3)) return false;
  return a == i0 + sx * (int)(((long long)(dy / 2) + (long long)c * dx) / dy);
}

// TraversabilityMap::checkInclination (TraversabilityMap.cpp:748-762) on the robot_slope layer; rslope == nullptr: check off.
__device__ bool inclination_ok_d(const FpArgs& A, const float* rslope, double ax, double ay, double bx, double by) {
  if (!rslope) return true;
  int si, sj, ei, ej;
  if (bx == ax && by == ay) {
    if (!is_inside_d(A, ax, ay) || !get_index_d(A, ax, ay, si, sj)) return false;
    return !(lay(A, rslope, si, sj) == 0.0f);
  }
  if (!get_index_d(A, ax, ay, si, sj) || !get_index_d(A, bx, by, ei, ej)) return false;
  LineD line(si, sj, ei, ej);
  for (int c = 0; c < line.n; ++c, line.next()) {
    const float v = lay(A, rslope, line.li, line.lj);
    if (finitef(v) && v == 0.0f) return false;
  }
  return true;
}

// The running, length-weighted mean of the segment means (TraversabilityMap.cpp:440-452); `lengthPath` (an uninitialised local
// in the reference) is the running path length.
__device__ __forceinline__ void add_segment_d(double t, double lx, double ly, int k, double& lengthPath, double& result) {
  const double lengthSegment = sqrt(lx * lx + ly * ly);
  if (k > 1) {
    const double lengthPreviousPath = lengthPath;
    lengthPath += lengthSegment;
    result = (lengthSegment * t + lengthPreviousPath * result) / lengthPath;
  } else {
    lengthPath = lengthSegment;
    result = t;
  }
}

// TraversabilityMap::checkCircularFootprintPath (TraversabilityMap.cpp:345-462) for a batch of paths — one thread per path — on a
// traversability_footprint layer that is valid everywhere: every isTraversable(center, ...) takes the memoised branch
// (:667-673), centres outside the map the default branch (:660-666).  No polygons.
__global__ void __launch_bounds__(128) k_check_paths(FpArgs A, const float* __restrict__ fp, const float* __restrict__ rslope, int npaths, const int* __restrict__ path_begin,
                                                     const double* __restrict__ xy, unsigned char* __restrict__ is_safe,
                                                     double* __restrict__ trav_out) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npaths) return;
  const int b = path_begin[q], n = path_begin[q + 1] - b;
  is_safe[q] = 0;
  trav_out[q] = 0.0;
  if (n <= 0) return;
  auto circle = [&](double cx, double cy, double& t) -> bool {
    int i, j;
    if (!is_inside_d(A, cx, cy) || !get_index_d(A, cx, cy, i, j)) {
      t = A.tdefault;
      return A.tdefault != 0.0;
    }
    t = (double)lay(A, fp, i, j);
    return t != 0.0;
  };
  double result = 0.0, lengthPath = 0.0;
  double sx = 0.0, sy = 0.0, ex = 0.0, ey = 0.0;
  for (int k = 0; k < n; ++k) {
    sx = ex; sy = ey;
    ex = xy[2 * (b + k)]; ey = xy[2 * (b + k) + 1];
    if (n == 1) {
      if (!inclination_ok_d(A, rslope, ex, ey, ex, ey)) return;
      double t;
      if (!circle(ex, ey, t)) return;
      result = t;
    }
    if (n > 1 && k > 0) {
      if (!inclination_ok_d(A, rslope, sx, sy, ex, ey)) return;
      int si, sj, ei, ej;
      if (!get_index_d(A, sx, sy, si, sj) || !get_index_d(A, ex, ey, ei, ej)) return;
      // LineIterator (Bresenham) from the end index to the start index, every fourth cell checked
      LineD line(ei, ej, si, sj);
      int nLine = 0;
      double sum = 0.0;
      for (int c = 0; c < line.n; ++c, line.next()) {
        if ((c & 3) == 0) {
          double t;
          if (!circle(A.X[line.li], A.Y[line.lj], t)) return;
          sum += t;
          ++nLine;
        }
      }
      add_segment_d(sum / (double)nLine, ex - sx, ey - sy, k, lengthPath, result);
    }
  }
  is_safe[q] = 1;
  trav_out[q] = result;
}

// ---------------------------------------------------------------------------------------------------------------------------
// checkCircularFootprintPath as the reference's check_footprint_path service runs it right after computeTraversability: the
// traversability_footprint layer is empty (NaN, TraversabilityMap.cpp:228), so every isTraversable(center, radius + offset, ...)
// takes the branch that walks the SpiralIterator (:679-736) — and stores its result in that layer, which later centres of the
// same path read back through the memoised branch (:673-675).  One warp per path; radius and compute_untraversable_polygon per
// path.  Every path starts from an empty layer.
constexpr int kPathMaxRings = 127;  // the signed-byte packing of the ring table
struct PathArgs {
  const float* rslope;           // robot_slope, nullptr: checkRobotInclination_ off
  int npaths;
  int pose_stride;               // doubles per pose in `poses`: 2 (x y) or 7 (x y z qx qy qz qw)
  const int* path_begin;
  const double* poses;
  const double* radius;          // FootprintPath.radius per path
  const unsigned char* cup;      // FootprintPath.compute_untraversable_polygon per path, nullptr: all 0
  double offset;                 // radiusMax = radius + offset (:348)
  const int* ring_start;         // [kPathMaxRings + 2]: first entry of ring d in `rings`
  const int* rings;              // SpiralIterator visit order of rings 0 .. kPathMaxRings, packed like FpArgs::spiral (no edge bit)
  unsigned char* memo;           // per map cell: isTraversableForFilters 0 = not evaluated yet, 1 = passes, 2 = blocked
  unsigned char* is_safe;
  double* trav_out;
};

// isTraversableForFilters of map cell (a, b) through the per-call memo.  Concurrent writers of a byte store the same value.
__device__ __forceinline__ bool blocked_memo_d(const FpArgs& A, const Layers& L, unsigned char* memo, int a, int b) {
  const size_t c = (size_t)b * A.rows + a;
  unsigned char m = memo[c];
  if (m == 0) {
    const bool heavy = __ldg(L.slope + c) == 0.0f || __ldg(L.step + c) == 0.0f || (A.verify_rough && __ldg(L.rough + c) == 0.0f);
    m = (!heavy || filters_d(A, L, a, b).ok) ? 1 : 2;
    memo[c] = m;
  }
  return m == 2;
}

struct FreshCircle {
  bool ok;      // isTraversable's return value
  double t;     // its `traversability` output
  float cache;  // what it leaves in traversability_footprint at the centre cell
};

// isTraversable(center, rmax, cup, traversability, ..., rmin) on an empty cache, TraversabilityMap.cpp:679-736, by the whole warp:
// the SpiralIterator around index (ci, cj) 32 entries at a time.  Each lane decides map membership (the circle test of the last two
// rings against `center` itself: for a single pose that is the pose, not its cell centre) and isTraversableForFilters; the ballot
// finds the first blocked cell; the double sum is added in visit order, so it is the reference's sum bit for bit.  Warp-uniform.
__device__ FreshCircle fresh_circle_d(const FpArgs& A, const Layers& L, const PathArgs& P, double cx, double cy, int ci, int cj,
                                      double rmin, double rmax, int nr, bool cup) {
  const int lane = threadIdx.x & 31;
  const double r2 = rmax * rmax;
  const int end = __ldg(P.ring_start + nr + 1), edge0 = __ldg(P.ring_start + max(nr - 1, 1));
  double t = 0.0;
  int n = 0;
  for (int base = 0; base < end; base += 32) {
    const int k = base + lane;
    bool member = false, blk = false;
    double v = 0.0;
    int di = 0, dj = 0;
    if (k < end) {
      const int w = __ldg(P.rings + k);
      di = (int)(signed char)(w & 0xff);
      dj = (int)(signed char)((w >> 8) & 0xff);
      const int a = ci + di, b = cj + dj;
      if (a >= 0 && b >= 0 && a < A.rows && b < A.cols_total) {  // SpiralIterator: checkIfIndexInRange
        member = true;
        if (k >= edge0) {                                          // ... and isInside on rings nRings - 1, nRings
          const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
          member = dx * dx + dy * dy <= r2;
        }
      }
      if (member) {
        blk = blocked_memo_d(A, L, P.memo, a, b);
        if (!blk) {
          const float f = __ldg(L.trav + (size_t)b * A.rows + a);
          v = finitef(f) ? (double)f : A.tdefault;                // :719-724
        }
      }
    }
    const unsigned bm = __ballot_sync(0xffffffffu, blk);
    const int first = bm ? __ffs((int)bm) - 1 : 32;
    const unsigned take = __ballot_sync(0xffffffffu, member && !blk) & (first == 32 ? 0xffffffffu : ((1u << first) - 1u));
    n += __popc(take);
#pragma unroll
    for (int l = 0; l < 32; ++l) {
      const double o = __shfl_sync(0xffffffffu, v, l);
      if ((take >> l) & 1u) t += o;
    }
    if (bm) {  // the first blocked cell in visit order (:690-717)
      const double uR = current_radius_d(A, __shfl_sync(0xffffffffu, di, first), __shfl_sync(0xffffffffu, dj, first));
      if (rmin == 0.0 || uR <= rmin) return FreshCircle{false, t, 0.0f};  // :694-704 (cup: later cells change nothing that is read)
      const double factor = ((uR - rmin) / (rmax - rmin) + 1.0) / 2.0;    // :706-708
      t *= factor / (double)n;
      if (!cup) return FreshCircle{false, t, (float)t};                   // :714-717
      t /= (double)n;                                                      // the loop ends (:710); :732-734 divide a second time
      return FreshCircle{true, t, (float)t};
    }
  }
  t /= (double)n;  // :732-734
  return FreshCircle{true, t, (float)t};
}

__device__ __forceinline__ bool lex_less_d(double2 a, double2 b) { return a.x < b.x || (a.x == b.x && a.y < b.y); }

// grid_map::Polygon::monotoneChainConvexHullOfPoints (recalled) of the m > 3 points `sorted` (already in lexicographic order) into
// `hull` (2m entries, the reference's own allocation); returns the vertex count.  One thread.
__device__ int monotone_chain_d(const double2* sorted, int m, double2* hull) {
  auto clockwise = [](double2 o, double2 a, double2 b) {
    const double ux = a.x - o.x, uy = a.y - o.y, wx = b.x - o.x, wy = b.y - o.y;
    return (ux * wy - uy * wx) <= 0;
  };
  int k = 0;
  for (int i = 0; i < m; ++i) {
    while (k >= 2 && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  for (int i = m - 2, t = k + 1; i >= 0; i--) {
    while (k >= t && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  return k - 1;
}

// ---- untraversable polygon (isTraversable with computeUntraversablePolygon, :599-645 and :679-736) -------------------------
// The reference pushes the cell centre of every collected blocked cell and returns monotoneChainConvexHullOfPoints of that list
// (recalled, see monotone_chain_d): 3 points or fewer as given, in visit order; otherwise the sorted monotone chain.  The kernels
// do not keep the list.  A warp records, per map row of the walk, the smallest and largest column index of its collected cells
// (shared atomics), the number of cells and the first three in visit order.  That is exact:
//   - X[a] falls as the row index a grows and Y[b] as the column index b grows, so reading the table by descending row and, within
//     a row, by descending column yields the lexicographic order of std::sort (x, then y) without sorting;
//   - all cells of one row share the double X[a].  Between its two extremes, a row's cells only ever meet the chain as the third
//     point of a vertical triple, whose cross product is exactly 0 (both x differences are 0.0): the point is popped.  Before that
//     the row's second point is tested against the chain from an earlier row, and that cross product is (X[a] - x') times the
//     difference of two column positions: at least res^2 in magnitude, far from rounding for any map whose coordinates stay
//     below res * 2^40, so it never pops.  The chain therefore goes through the same states with the extremes alone, and its
//     stack holds at most one point per row and pass plus two (2 * rows + 2 entries).
// A map row without collected cells has max < min in the table.
constexpr int kFromCircleVertices = 20;    // grid_map::Polygon::fromCircle's default nVertices

struct UntravOut {
  int maxv;     // vertices the caller has room for per path
  int* count;   // per path: vertex count (0: no polygon, -1: not computed); nullptr: polygon not requested
  double* xy;   // per path: maxv (x, y) pairs
};

// The monotone chain of monotone_chain_d over the points of a row table (rows 0 .. nrows-1, row r at map row a0 + r, column
// extremes tmin / tmax), pruned to the row extremes as argued above; `st` receives the hull as (row, column) and has room for
// 2 * nrows + 4 entries.  Returns the vertex count.  One thread.  Used for more than 3 points (or 2 or 3 points hulled twice).
__device__ int table_chain_d(const FpArgs& A, const int* tmin, const int* tmax, int nrows, int a0, int2* st) {
  auto cw = [&](int2 o, int2 p, int2 w) {
    const double ox = A.X[a0 + o.x], oy = A.Y[o.y];
    const double ux = A.X[a0 + p.x] - ox, uy = A.Y[p.y] - oy, wx = A.X[a0 + w.x] - ox, wy = A.Y[w.y] - oy;
    return (ux * wy - uy * wx) <= 0;
  };
  int k = 0;
  for (int r = nrows - 1; r >= 0; --r) {  // lower hull: x ascending = row index descending; y ascending = column descending
    const int lo = tmin[r], hi = tmax[r];
    if (hi < lo) continue;
    for (int e = 0; e < 2 && (e == 0 || lo != hi); ++e) {
      const int2 p = make_int2(r, e ? lo : hi);
      while (k >= 2 && cw(st[k - 2], st[k - 1], p)) k--;
      st[k++] = p;
    }
  }
  const int t = k + 1;
  bool last = true;  // the upper hull starts at the second largest point
  for (int r = 0; r < nrows; ++r) {
    const int lo = tmin[r], hi = tmax[r];
    if (hi < lo) continue;
    for (int e = 0; e < 2 && (e == 0 || lo != hi); ++e) {
      const int2 p = make_int2(r, e ? hi : lo);
      if (last) { last = false; continue; }
      while (k >= t && cw(st[k - 2], st[k - 1], p)) k--;
      st[k++] = p;
    }
  }
  return k - 1;
}

// A warp's polygon scratch in shared memory.
struct UntravScratch {
  int* tmin;
  int* tmax;
  int2* stack;    // 2 * rows + 4 entries; also holds the 20 + 40 points of a fromCircle hull (as double2)
  int2* first;    // the first three collected cells (map row, map column) in visit order
};

// Records the cells whose lanes have `take` set (map row a, map column b; table row a - a0) in visit order = lane order.
__device__ __forceinline__ void collect_cells_d(const UntravScratch& S, bool take, int a, int b, int a0, int& cnt) {
  const int lane = threadIdx.x & 31;
  const unsigned m = __ballot_sync(0xffffffffu, take);
  if (take) {
    const int rank = cnt + __popc(m & ((1u << lane) - 1u));
    if (rank < 3) S.first[rank] = make_int2(a, b);
    atomicMin(S.tmin + (a - a0), b);
    atomicMax(S.tmax + (a - a0), b);
  }
  cnt += __popc(m);
}

__device__ __forceinline__ void clear_table_d(const UntravScratch& S, int nrows) {
  for (int r = threadIdx.x & 31; r < nrows; r += 32) { S.tmin[r] = 0x7fffffff; S.tmax[r] = -0x7fffffff - 1; }
  __syncwarp();
}

// Writes the polygon of `cnt` collected cells, hulled `reps` times (Polygon::convexHull(U, P) = monotone chain of U ++ P, see
// k_check_paths_fresh_poly), to slot q of O.  One thread.
//   reps == 1: monotoneChainConvexHullOfPoints(P): P as given for 3 points or fewer, else the chain.
//   reps >= 2: with 2 or more distinct points, every later hull has more than 3 input points drawn from P's own points, and the
//     chain of a point list depends only on the set of its points (a repeated point is popped by a cross product of exactly 0
//     and pushed again onto the same stack), so it is the chain of P whatever `reps` is.  A single point p grows instead:
//     [p] -> [p, p] -> [p, p, p] -> chain of [p, p, p, p] = [p, p] -> [p, p, p] ...: 2 vertices for even reps, 3 for odd.
__device__ void write_cells_polygon_d(const FpArgs& A, const UntravScratch& S, int nrows, int a0, int cnt, int reps, const UntravOut& O,
                                      int q) {
  int* cout = O.count + q;
  double* xy = O.xy + 2 * (size_t)O.maxv * q;
  if (cnt >= 4 || (cnt >= 2 && reps >= 2)) {
    const int nv = table_chain_d(A, S.tmin, S.tmax, nrows, a0, S.stack);
    *cout = nv;
    for (int v = 0; v < min(nv, O.maxv); ++v) {
      xy[2 * v] = A.X[a0 + S.stack[v].x];
      xy[2 * v + 1] = A.Y[S.stack[v].y];
    }
    return;
  }
  const int nv = (cnt == 1 && reps >= 2) ? 2 + (reps & 1) : cnt;
  *cout = nv;
  for (int v = 0; v < min(nv, O.maxv); ++v) {
    const int2 c = S.first[cnt == 1 ? 0 : v];
    xy[2 * v] = A.X[c.x];
    xy[2 * v + 1] = A.Y[c.y];
  }
}

// isTraversable's spiral walk with computeUntraversablePolygon on an untraversable circle (:687-729): the first blocked cell lies
// within rmin, so the walk goes to the end of the spiral and collects every blocked cell with uR <= rmin (every blocked cell when
// rmin == 0); later blocked cells of the annulus are skipped (:705).  Membership as in fresh_circle_d.  Table row r = map row
// ci - nr + r.  Returns the number of collected cells.  Warp-uniform.
__device__ int spiral_blockers_d(const FpArgs& A, const Layers& L, const PathArgs& P, const UntravScratch& S, double cx, double cy,
                                 int ci, int cj, double rmin, double rmax, int nr) {
  const int lane = threadIdx.x & 31;
  const double r2 = rmax * rmax;
  const int end = __ldg(P.ring_start + nr + 1), edge0 = __ldg(P.ring_start + max(nr - 1, 1));
  clear_table_d(S, 2 * nr + 1);
  int cnt = 0;
  for (int base = 0; base < end; base += 32) {
    const int k = base + lane;
    bool take = false;
    int a = 0, b = 0;
    if (k < end) {
      const int w = __ldg(P.rings + k);
      const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
      a = ci + di;
      b = cj + dj;
      bool member = false;
      if (a >= 0 && b >= 0 && a < A.rows && b < A.cols_total) {
        member = true;
        if (k >= edge0) {
          const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
          member = dx * dx + dy * dy <= r2;
        }
      }
      take = member && blocked_memo_d(A, L, P.memo, a, b) && (rmin == 0.0 || current_radius_d(A, di, dj) <= rmin);
    }
    collect_cells_d(S, take, a, b, ci - nr, cnt);
  }
  __syncwarp();
  return cnt;
}

// grid_map::Polygon::fromCircle(center, radius) (recalled): vertex j = center + Rotation2D(j * 2 * M_PI / 19) * (radius, 0); the
// 20 cosines and sines come from the host's libm (circle_table).  A single pose publishes it as it is; a segment
// hulls it: 20 points, so every later convexHull with it is the same chain (see write_cells_polygon_d).  One thread.
__device__ void write_circle_polygon_d(const double* cs, const double* sn, double cx, double cy, double radius, bool hulled,
                                       double2* pts, const UntravOut& O, int q) {
  const int nc = kFromCircleVertices;
  double2* hull = pts + nc;
  for (int j = 0; j < nc; ++j) {  // insertion sort into lexicographic order (equal points are equal values: order is irrelevant)
    const double2 v = make_double2(cx + cs[j] * radius, cy + sn[j] * radius);
    int i = j;
    while (hulled && i > 0 && lex_less_d(v, pts[i - 1])) { pts[i] = pts[i - 1]; --i; }
    pts[i] = v;
  }
  const int nv = hulled ? monotone_chain_d(pts, nc, hull) : nc;
  const double2* out = hulled ? hull : pts;
  O.count[q] = nv;
  double* xy = O.xy + 2 * (size_t)O.maxv * q;
  for (int v = 0; v < min(nv, O.maxv); ++v) { xy[2 * v] = out[v].x; xy[2 * v + 1] = out[v].y; }
}

struct CircleTable {
  double cs[kFromCircleVertices], sn[kFromCircleVertices];
};

// Per-path footprints and the pose count of a batch.  With fp_begin, path q's footprint is vertices fp_begin[q] .. fp_begin[q+1]-1
// of fp_xyz, as in a whole check_footprint_path request (te_check_footprint_request): none makes the path circular (checked by
// k_check_paths_fresh*), any other count polygonal (checked by k_check_polygon_*).  Without fp_begin every path is circular for
// k_check_paths_fresh* and uses the one footprint of PolyPathArgs for k_check_polygon_*.  Device memory cannot validate the arrays
// on the host, so the kernels do (request_footprint_ok_d, the pose range).
// A batch of maps (te_check_footprint_request_batched): path q is on map path_map[q], whose layers, robot_slope and memo start
// path_map[q] * map_cells cells into theirs.  Each kernel shifts those pointers once it knows its path (map_offset_d), so one map
// and a batch run the same code.
struct RequestArgs {
  const int* fp_begin;   // [npaths + 1], nullptr: no per-path footprints
  const float* fp_xyz;   // 3 floats (x, y, z) per vertex
  int nvertices;         // vertices in fp_xyz
  int maxfp;             // max_footprint_vertices: a longer footprint is not checked
  int nposes;            // < 0: not known, the circular check does not test pose ranges
  double* area_out;      // the area of the circular paths: 0, NaN for a path that is not checked; nullptr: not wanted
  const int* path_map;   // [npaths], nullptr: every path is on map 0
  int nmaps;             // maps of the batch: a path on a map outside 0 .. nmaps-1 is not checked
  long long map_cells;   // rows * cols
};

// The first cell of path q's map in the layers and the memo, or -1 for a map outside the batch.
__device__ __forceinline__ long long map_offset_d(const RequestArgs& R, int q) {
  if (!R.path_map) return 0;
  const int m = R.path_map[q];
  return (m >= 0 && m < R.nmaps) ? m * R.map_cells : -1;
}

// The layers of the map that starts `o` cells in (a null roughness layer stays null).
__device__ __forceinline__ Layers shift_layers_d(const Layers& L, long long o) {
  return Layers{L.trav + o, L.slope + o, L.step + o, L.elev + o, L.rough ? L.rough + o : nullptr};
}

// Whether path q's footprint can be checked: 1..maxfp vertices inside fp_xyz, all finite (host memory rejects the rest).  The
// vertex components are read from `first` in steps of `step` (a warp: lane, 32; one thread: 0, 1).
__device__ __forceinline__ bool request_footprint_ok_d(const RequestArgs& R, int q, int first, int step) {
  const int fb = R.fp_begin[q], nfp = R.fp_begin[q + 1] - fb;
  bool ok = nfp >= 1 && nfp <= R.maxfp && fb >= 0 && (long long)fb + nfp <= R.nvertices;
  for (int c = first; c < 3 * nfp && ok; c += step) ok = isfinite(R.fp_xyz[3 * (size_t)fb + c]);
  return ok;
}

// The body of k_check_paths_fresh; POLY also produces the untraversable polygon (k_check_paths_fresh_poly).  With per-path
// footprints (R.fp_begin) it checks the circular paths of a request and leaves its polygonal paths to k_check_polygon_*.
template <bool POLY>
__device__ __forceinline__ void check_paths_fresh_d(const FpArgs& A, Layers L, PathArgs P, const UntravOut& O, const CircleTable& C,
                                                    const UntravScratch& S, const RequestArgs& R) {
  const int PS = P.pose_stride;  // x and y come first
  const int lane = threadIdx.x & 31;
  const int q = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (q >= P.npaths) return;  // whole warp
  if (R.fp_begin && R.fp_begin[q + 1] != R.fp_begin[q]) return;  // a polygonal path
  const int b = P.path_begin[q], n = P.path_begin[q + 1] - b;
  const double rmin = P.radius[q], rmax = rmin + P.offset;
  const bool cup = P.cup != nullptr && P.cup[q] != 0;
  const double rings = ceil(rmax / A.res);  // SpiralIterator nRings
  const long long mo = map_offset_d(R, q);
  // not checkable here: marked so that no checked result looks alike (with a pose count: also a pose range outside it; written
  // b <= nposes - n, which ptxas compiles to fewer registers in the _poly kernel than a 64-bit b + n, see DESIGN.md)
  if (!(rmin >= 0.0) || !(rings <= (double)kPathMaxRings) || (R.nposes >= 0 && !(b >= 0 && n >= 0 && b <= R.nposes - n)) || mo < 0) {
    if (lane == 0) {
      P.is_safe[q] = 0; P.trav_out[q] = nan("");
      if (R.area_out) R.area_out[q] = nan("");
      if (POLY) O.count[q] = cup ? -1 : 0;
    }
    return;
  }
  L = shift_layers_d(L, mo);  // path q's map
  if (P.rslope) P.rslope += mo;
  P.memo += mo;
  const int nr = (int)rings;
  double result = 0.0, lengthPath = 0.0;
  double sx = 0.0, sy = 0.0, ex = 0.0, ey = 0.0;
  bool ok = n > 0;  // :330-334
  // POLY: the circle that made the path fail and how often its polygon is hulled into the published one
  int fkind = 0;  // 0: nothing published, 1: fromCircle(centre, rmax), 2: hull of the spiral's blocked cells
  double fx = 0.0, fy = 0.0;
  int fi = 0, fj = 0, freps = 1;
  for (int k = 0; k < n && ok; ++k) {
    sx = ex; sy = ey;
    ex = P.poses[PS * (b + k)]; ey = P.poses[PS * (b + k) + 1];
    if (n == 1) {  // :365-387
      if (!inclination_ok_d(A, P.rslope, ex, ey, ex, ey)) { ok = false; break; }
      int i, j;
      if (!is_inside_d(A, ex, ey) || !get_index_d(A, ex, ey, i, j)) {  // :662-667
        result = A.tdefault;
        ok = A.tdefault != 0.0;
        if (POLY && !ok) { fkind = 1; fx = ex; fy = ey; }
      } else {
        const FreshCircle f = fresh_circle_d(A, L, P, ex, ey, i, j, rmin, rmax, nr, cup);
        ok = f.ok;
        result = f.t;
        if (POLY && !ok) { fkind = 2; fx = ex; fy = ey; fi = i; fj = j; }
      }
    }
    if (n > 1 && k > 0) {  // :389-457
      if (!inclination_ok_d(A, P.rslope, sx, sy, ex, ey)) { ok = false; break; }
      int si, sj, ei, ej;
      if (!get_index_d(A, sx, sy, si, sj) || !get_index_d(A, ex, ey, ei, ej)) { ok = false; break; }
      LineD line(ei, ej, si, sj);
      int nLine = 0;
      double sum = 0.0;
      for (int c = 0; c < line.n && ok; ++c, line.next()) {
        if (c & 3) continue;
        const int a = line.li, bb = line.lj;
        const FreshCircle f = fresh_circle_d(A, L, P, A.X[a], A.Y[bb], a, bb, rmin, rmax, nr, cup);
        // A centre an earlier segment of this path checked already holds its float32 result in the layer: the memoised branch
        // (:673-675) reads it back.  Earlier segments (a lane each) are tested in closed form; their poses are inside the map.
        bool seen = false;
        for (int s = 1 + lane; s < k; s += 32) {
          int pi0, pj0, pi1, pj1;
          get_index_d(A, P.poses[PS * (b + s - 1)], P.poses[PS * (b + s - 1) + 1], pi0, pj0);
          get_index_d(A, P.poses[PS * (b + s)], P.poses[PS * (b + s) + 1], pi1, pj1);
          seen = seen || line_checks_d(pi1, pj1, pi0, pj0, a, bb);
        }
        const bool cached = __any_sync(0xffffffffu, seen);
        if (cached) {
          ok = f.cache != 0.0f;
          sum += (double)f.cache;
        } else {
          ok = f.ok;
          sum += f.t;
        }
        // POLY: a cached 0 publishes fromCircle of the cell centre (:673-678), a walked circle the hull of its blocked cells.  The
        // failing circle's polygon is hulled into the path's once for itself and once per later checked cell of the line
        // (:407-412: the && skips isTraversable, the auxiliary polygon stays).
        if (POLY && !ok) { fkind = cached ? 1 : 2; fx = A.X[a]; fy = A.Y[bb]; fi = a; fj = bb; freps = (line.n - 1) / 4 - c / 4 + 1; }
        ++nLine;
      }
      if (!ok) break;  // :414-417, :453-456
      add_segment_d(sum / (double)nLine, ex - sx, ey - sy, k, lengthPath, result);
    }
  }
  if (lane == 0) {
    P.is_safe[q] = ok ? 1 : 0;
    P.trav_out[q] = ok ? result : 0.0;
    if (R.area_out) R.area_out[q] = 0.0;  // TraversabilityResult.area stays 0 for a circular path
  }
  if (POLY) {
    // the last non-empty polygon published for the path: only an untraversable circle has one (inclination failures return first)
    if (!cup || ok || fkind == 0) {
      if (lane == 0) O.count[q] = 0;
    } else if (fkind == 1) {
      if (lane == 0) write_circle_polygon_d(C.cs, C.sn, fx, fy, rmax, n > 1, reinterpret_cast<double2*>(S.stack), O, q);
    } else {
      const int cnt = spiral_blockers_d(A, L, P, S, fx, fy, fi, fj, rmin, rmax, nr);
      if (lane == 0) write_cells_polygon_d(A, S, 2 * nr + 1, fi - nr, cnt, freps, O, q);
    }
  }
}

__global__ void __launch_bounds__(128) k_check_paths_fresh(FpArgs A, Layers L, PathArgs P, RequestArgs R) {
  check_paths_fresh_d<false>(A, L, P, UntravOut{}, CircleTable{}, UntravScratch{}, R);
}

// k_check_paths_fresh that also returns the untraversable polygon of every path (te_check_footprint_paths_fresh2).  Per warp:
// a row table for the 2 * 127 + 1 rows of the largest spiral and the chain stack.  At its 128 registers four blocks fit an SM
// anyway; saying so makes ptxas lay the kernel out about 6 % faster on H100 (DESIGN.md).
constexpr int kFreshTableRows = 2 * kPathMaxRings + 1;
__global__ void __launch_bounds__(128, 4) k_check_paths_fresh_poly(FpArgs A, Layers L, PathArgs P, UntravOut O, CircleTable C,
                                                                RequestArgs R) {
  __shared__ int s_min[4][kFreshTableRows + 1], s_max[4][kFreshTableRows + 1];
  __shared__ int2 s_stack[4][2 * kFreshTableRows + 4];
  __shared__ int2 s_first[4][3];
  static_assert(sizeof(s_stack[0]) >= 3 * kFromCircleVertices * sizeof(double2), "fromCircle points and hull fit the stack");
  const int w = threadIdx.x >> 5;
  check_paths_fresh_d<true>(A, L, P, O, C, UntravScratch{s_min[w], s_max[w], s_stack[w], s_first[w]}, R);
}

// ---------------------------------------------------------------------------------------------------------------------------
// The circular paths of a request on a te_map (launch_map_request_device).  The traversability_footprint cache there persists
// across the paths of a request and across requests, so which isTraversable calls run, and what they read, depends on what
// earlier calls stored.  Every circle the paths could check is a MapKey (one per distinct map, centre, cell, radius and polygon
// flag); k_map_eval_circles_dev evaluates every key on the cache as the request found it, one warp per key, and k_req_replay
// then runs the service loop in order over these records.  A te_map may hold a batch of maps of one geometry (map m's layers,
// cache and memo start m * rows * cols cells into theirs); a key belongs to one of them.
struct MapKey {
  double cx, cy, rmin;  // isTraversable(center, rmin + offset, cup, ..., rmin)
  int ci, cj;           // getIndex(center)
  int cup;              // computeUntraversablePolygon
  int map;              // the map of the batch (0 on a single map)
};
struct MapRecord {
  double t;       // the walk's traversability output (double), or the cached value
  float cache;    // what the walk stores at (ci, cj), or the cached value
  int state;      // 0: walked, traversable; 1: walked, untraversable; 2: the cell was cached when the request began
};

// Key k of the request, by the whole warp w of a block of four: its record (k_map_eval_circles_dev).
__device__ __forceinline__ void map_eval_circle_d(const FpArgs& A, const Layers& L, const PathArgs& P, const MapKey* __restrict__ keys,
                                                  int k, const float* __restrict__ cache, MapRecord* __restrict__ recs) {
  __shared__ Layers s_L[4];
  __shared__ PathArgs s_P[4];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const MapKey K = keys[k];
  MapRecord& R = recs[k];
  // The key's map: its layers, memo and cache start mo cells in.  The walk takes the shifted layer and path arguments from a
  // per-warp copy in shared memory (by reference, as it takes the kernel's own), so no register holds them across the call.
  const long long mo = (long long)K.map * A.rows * A.cols_total;
  const float c0 = __ldg(cache + mo + (size_t)K.cj * A.rows + K.ci);
  if (finitef(c0)) {  // :673-675
    if (lane == 0) { R.t = (double)c0; R.cache = c0; R.state = 2; }
    return;
  }
  if (lane == 0) {
    s_L[w] = shift_layers_d(L, mo);
    s_P[w] = P;
    s_P[w].memo += mo;
  }
  __syncwarp();
  const double rmax = K.rmin + P.offset;
  const int nr = (int)ceil(rmax / A.res);
  const FreshCircle f = fresh_circle_d(A, s_L[w], s_P[w], K.cx, K.cy, K.ci, K.cj, K.rmin, rmax, nr, K.cup != 0);
  if (lane == 0) { R.t = f.t; R.cache = f.cache; R.state = f.ok ? 0 : 1; }
}

// The key count is on the device (*nkeys), so the warps stride over the keys.  The polygons of the failed paths come after the
// replay (k_req_polygons).
__global__ void __launch_bounds__(128, 4) k_map_eval_circles_dev(FpArgs A, Layers L, PathArgs P, const MapKey* __restrict__ keys,
                                                              const unsigned long long* __restrict__ nkeys, const float* __restrict__ cache,
                                                              MapRecord* __restrict__ recs) {
  const long long n = (long long)*nkeys;
  for (long long k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += (gridDim.x * blockDim.x) >> 5)  // whole warps
    map_eval_circle_d(A, L, P, keys, (int)k, cache, recs);
}

// traversabilityFootprint(radius, offset) on a cache: a cached cell takes the memoised branch and keeps its value, every other cell
// gets the sweep's.  `out` (may be null or `cache` itself) receives the cache afterwards.  Block row y merges n cells: `fresh` and
// `out` from y * n on, the cache from slot[y] * n on (slot null: y * n).
__global__ void __launch_bounds__(256) k_map_merge(float* cache, const float* __restrict__ fresh, float* out, size_t n,
                                                   const int* __restrict__ slot) {
  const size_t y = blockIdx.y;
  cache += (slot ? (size_t)slot[y] : y) * n;
  fresh += y * n;
  if (out) out += y * n;
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const float v = finitef(cache[c]) ? cache[c] : fresh[c];
    cache[c] = v;
    if (out) out[c] = v;
  }
}

// Selected maps between their slots of a te_map and packed scratch (launch_map_slots).  PUT: layer l of packed map j goes to
// dst[l] + slot[j] * cells, and the cache / memo slots of the map are emptied (NaN bits 0xffffffff, memo 0: not evaluated).  Not
// PUT: src[l] + slot[j] * cells goes to packed map j of dst[l].  V cells per thread and access (V = 4: 16-byte accesses).
template <bool PUT, int V>
__global__ void __launch_bounds__(256) k_map_slots(MapSlots a) {
  using Vec = typename std::conditional<V == 4, float4, float>::type;
  using Bytes = typename std::conditional<V == 4, unsigned, unsigned char>::type;
  const size_t step = (size_t)gridDim.x * blockDim.x * V;
  for (int j = blockIdx.y; j < a.nsel; j += gridDim.y) {
    const size_t packed = (size_t)j * a.cells, resident = (size_t)a.slot[j] * a.cells;
    const size_t s0 = PUT ? packed : resident, d0 = PUT ? resident : packed;
    for (size_t c = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; c < a.cells; c += step) {
#pragma unroll
      for (int l = 0; l < kMapSlotLayers; ++l)
        if (a.dst[l]) *reinterpret_cast<Vec*>(a.dst[l] + d0 + c) = __ldg(reinterpret_cast<const Vec*>(a.src[l] + s0 + c));
      if (PUT) {
        const float nan = __int_as_float(-1);
        Vec e;
        if constexpr (V == 4) e = make_float4(nan, nan, nan, nan);
        else e = nan;
        *reinterpret_cast<Vec*>(a.cache + resident + c) = e;
        if (a.memo) *reinterpret_cast<Bytes*>(a.memo + resident + c) = 0;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// The work list of the circular paths of a request on a te_map (launch_map_request_device), whichever memory the request came
// from.  It holds one entry per isTraversable call a circular path could make (a single pose; every fourth LineIterator cell of an
// in-map segment) and a "gate" wherever the service loop breaks without a check (a failed checkInclination, a segment with an end
// outside the map).  The list is laid out per map, each map's entries contiguous and in request order (k_req_count ..
// k_req_list); the key entries are deduplicated on their key's bits (k_req_dedup) and every distinct key is walked once on the
// cache as the request found it (k_map_eval_circles_dev); k_req_replay then runs the service loop, one warp per map, and
// k_req_polygons publishes the polygons of the failed paths.
enum : int { kEntKey = 1, kEntOutside = 2, kEntGate = 4, kEntSegEnd = 8, kEntPathEnd = 16 };
struct ReqEntry {
  double cx, cy;  // the centre: a segment cell's centre, a single pose's position
  int q;          // the path
  int flags;      // kEnt*: a key (an in-map centre), a single pose outside the map, or a gate; the last of its segment / path
  int ci, cj;     // getIndex(centre) (kEntKey)
  int seg;        // segment k (1 .. n-1) of the path; 0: a single pose
  int freps;      // a failing segment cell's polygon is hulled into the path's this often (:407-412)
  int map;        // the path's map
  int key;        // k_req_dedup: the canonical entry of a key entry (the first to claim the hash slot)
};
// The failing circle of a replayed path: 0 none, 1 fromCircle(fx, fy), 2 the blocked cells of key `key` (k_req_polygons).
struct ReqFail {
  double fx, fy;
  int fkind, key, freps, pad;
};
constexpr unsigned short kReqNoMap = 0xffff;  // sort key of a pose without entries (maps are 0 .. 65534)
// CUB sorts short arrays with one single-tile kernel and longer ones with several: the sort always runs over at least this many
// keys (the poses, then kReqNoMap), so that a request launches the same kernels whatever its pose count.
constexpr int kReqSortMin = 1 << 16;
struct DevReq {
  int npaths, nposes, nmaps;
  int nsort;                    // keys sorted: max(nposes, kReqSortMin)
  long long map_cells, max_checks;
  const int* path_begin;
  const double* poses;          // 7 doubles per pose
  const double* radius;
  const int* fp_begin;
  const int* path_map;          // nullptr: one map
  const unsigned char* cup;
  const float* rslope;          // robot_slope of map 0, nullptr: no checkInclination
  double offset;
  unsigned char* is_safe;
  double* trav_out;
  double* area_out;
  UntravOut O;                  // O.count nullptr: no polygons
  // workspace (launch_map_request_device)
  unsigned char* status;        // per path: 0 polygonal, 1 replayed, 2 not checked, 3 empty circular path, 4 cut by max_checks
  long long* cnt;               // per pose (+1): entries
  long long* gofs;              // their exclusive scan in request order
  unsigned short* pkey;         // per pose: the sort key (the map, kReqNoMap)
  int* pidx;                    // per pose: its index
  unsigned short* skey;         // sorted
  int* order;                   // poses sorted stably by map
  int* lcnt;                    // entries of the sorted poses (+1)
  int* lofs;                    // their exclusive scan: the list offsets
  int* map_range;               // per map: [first, last) sorted pose index (0, 0: no entries)
  ReqEntry* entries;            // max_checks
  int* kid;                     // per entry: the key id of a canonical key entry
  int* table;                   // hash table of entry index + 1, tmask + 1 slots
  unsigned tmask;
  MapKey* keys;                 // max_checks
  MapRecord* recs;
  ReqFail* fails;               // per path
  unsigned long long* counters; // candidates, keys, stored
  // host memory: a non-finite x or y is checked as the service loop checks it (a single pose outside the map, a segment gate)
  // instead of leaving its path unchecked; only k_req_paths reads it (last, so the other kernels' parameters keep their offsets)
  bool nonfinite_ok;
};

// The path of pose p: the last q with path_begin[q] <= p (k_check_polygon_items' search).
__device__ __forceinline__ int req_path_of_d(const DevReq& D, int p) {
  int lo = 0, hi = D.npaths - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (D.path_begin[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool req_circular_d(const DevReq& D, int q) { return D.fp_begin[q + 1] == D.fp_begin[q]; }

// One thread per path: whether circular path q can be checked (radius, rings, pose range, finite positions unless
// D.nonfinite_ok, map) and every pose of it is found by req_path_of_d.
__global__ void __launch_bounds__(128) k_req_paths(FpArgs A, DevReq D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.npaths) return;
  if (!req_circular_d(D, q)) { D.status[q] = 0; return; }
  const int b = D.path_begin[q], n = D.path_begin[q + 1] - b;
  const double rmin = D.radius[q];
  bool ok = rmin >= 0.0 && ceil((rmin + D.offset) / A.res) <= (double)kPathMaxRings && b >= 0 && n >= 0 && b <= D.nposes - n;
  if (ok && D.path_map) ok = D.path_map[q] >= 0 && D.path_map[q] < D.nmaps;
  for (int k = 0; k < n && ok; ++k)
    ok = (D.nonfinite_ok || (isfinite(D.poses[7 * (size_t)(b + k)]) && isfinite(D.poses[7 * (size_t)(b + k) + 1]))) &&
         req_path_of_d(D, b + k) == q;
  D.status[q] = !ok ? 2 : n == 0 ? 3 : 1;
}

// The entries pose p of a replayed path adds, written to E when E is not null (at most max_checks - off of them).  Returns their
// count.  Request order: a failed inclination's gate first, then the pose's circle (a single pose) or the segment's cells.
__device__ long long req_pose_entries_d(const FpArgs& A, const DevReq& D, int p, ReqEntry* E, long long room) {
  const int q = req_path_of_d(D, p);
  if (D.status[q] != 1) return 0;
  const int b = D.path_begin[q], n = D.path_begin[q + 1] - b, k = p - b;
  // poses before the first path or after the last belong to no path; the search gives them path 0 or npaths - 1
  if (!(k >= 0 && k < n) || (n > 1 && k == 0)) return 0;
  const int m = D.path_map ? D.path_map[q] : 0;
  const float* rslope = D.rslope ? D.rslope + m * D.map_cells : nullptr;
  const double ex = D.poses[7 * (size_t)p], ey = D.poses[7 * (size_t)p + 1];
  const double sx = n > 1 ? D.poses[7 * (size_t)(p - 1)] : ex, sy = n > 1 ? D.poses[7 * (size_t)(p - 1) + 1] : ey;
  const int last = (p == b + n - 1) ? kEntPathEnd : 0;
  long long c = 0;
  auto put = [&](double cx, double cy, int flags, int ci, int cj, int freps) {
    if (E && c < room) E[c] = ReqEntry{cx, cy, q, flags, ci, cj, n > 1 ? k : 0, freps, m, -1};
    ++c;
  };
  // the candidates count a check's circles whatever checkInclination says: the gate goes in front of them
  if (rslope && !inclination_ok_d(A, rslope, sx, sy, ex, ey)) put(ex, ey, kEntGate, 0, 0, 1);
  if (n == 1) {
    int i, j;
    if (get_index_d(A, ex, ey, i, j)) put(ex, ey, kEntKey | last, i, j, 1);
    else put(ex, ey, kEntOutside | last, 0, 0, 1);
    return c;
  }
  int si, sj, ei, ej;
  if (!get_index_d(A, sx, sy, si, sj) || !get_index_d(A, ex, ey, ei, ej)) {
    put(ex, ey, kEntGate | last, 0, 0, 1);
    return c;
  }
  LineD line(ei, ej, si, sj);
  const int nchk = (line.n + 3) / 4;
  if (!E) return c + nchk;
  for (int cc = 0; cc < line.n && c < room; ++cc, line.next()) {
    if (cc & 3) continue;
    const int flags = kEntKey | (cc / 4 == nchk - 1 ? kEntSegEnd | last : 0);
    put(A.X[line.li], A.Y[line.lj], flags, line.li, line.lj, (line.n - 1) / 4 - cc / 4 + 1);
  }
  return c;
}

// 1. Count: one thread per pose index (and one more for the scan's total).
__global__ void __launch_bounds__(128) k_req_count(FpArgs A, DevReq D) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > D.nposes) return;
  D.cnt[p] = p < D.nposes ? req_pose_entries_d(A, D, p, nullptr, 0) : 0;
}

// One thread per path after the scan: the capacity cut (a replayed or empty circular path whose entries end past max_checks, and
// so every later one), and the outputs of every circular path the replay does not answer.
__global__ void __launch_bounds__(128) k_req_cut(DevReq D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.npaths) return;
  int s = D.status[q];
  if ((s == 1 || s == 3) && D.gofs[D.path_begin[q + 1]] > D.max_checks) D.status[q] = s = 4;
  if (s == 0 || s == 1) return;
  const bool cup = D.cup != nullptr && D.cup[q] != 0;
  const bool checked = s == 3;  // an empty path: ok = n > 0 is false (:330-334)
  D.is_safe[q] = 0;
  D.trav_out[q] = checked ? 0.0 : nan("");
  D.area_out[q] = checked ? 0.0 : nan("");
  if (D.O.count) D.O.count[q] = (checked || !cup) ? 0 : -1;
}

// One thread per pose: the sort key (the pose's map, kReqNoMap without entries) and the pose index.
__global__ void __launch_bounds__(128) k_req_keys(DevReq D) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= D.nsort) return;
  bool has = p < D.nposes && D.cnt[p] > 0;  // the padding sorts last
  int m = 0;
  if (has) {
    const int q = req_path_of_d(D, p);
    has = D.status[q] == 1;
    m = D.path_map ? D.path_map[q] : 0;
  }
  D.pkey[p] = has ? (unsigned short)m : kReqNoMap;
  D.pidx[p] = p;
}

// One thread per sorted pose index (and one more): its entry count, and the first / last sorted index of each map.
__global__ void __launch_bounds__(128) k_req_sorted(DevReq D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > D.nposes) return;
  const unsigned short m = i < D.nposes ? D.skey[i] : kReqNoMap;
  D.lcnt[i] = m != kReqNoMap ? (int)D.cnt[D.order[i]] : 0;
  if (m == kReqNoMap) return;
  if (i == 0 || D.skey[i - 1] != m) D.map_range[2 * m] = i;
  if (i == D.nposes - 1 || D.skey[i + 1] != m) D.map_range[2 * m + 1] = i + 1;
}

// 2. List: one thread per sorted pose index writes its entries at its offset.
__global__ void __launch_bounds__(128) k_req_list(FpArgs A, DevReq D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nposes || D.skey[i] == kReqNoMap) return;
  const int off = D.lofs[i];
  req_pose_entries_d(A, D, D.order[i], D.entries + off, D.max_checks - off);
}

__device__ __forceinline__ unsigned long long dbits_d(double d) { return (unsigned long long)__double_as_longlong(d); }

// The identity of a key entry's isTraversable call: map, centre, cell, radius and polygon flag, bit for bit.
__device__ __forceinline__ bool req_same_key_d(const DevReq& D, const ReqEntry& a, const ReqEntry& b) {
  const bool ca = D.cup && D.cup[a.q], cb = D.cup && D.cup[b.q];
  return a.map == b.map && dbits_d(a.cx) == dbits_d(b.cx) && dbits_d(a.cy) == dbits_d(b.cy) && a.ci == b.ci && a.cj == b.cj &&
         dbits_d(D.radius[a.q]) == dbits_d(D.radius[b.q]) && ca == cb;
}

// 3. Dedup: the threads stride over the entries.  A key entry claims its key's slot of an open-addressing table (linear probing); the entry that
// claims it is the key's canonical entry and allocates the key's id and MapKey, every other entry with that key records the
// canonical entry.  Which entry wins a slot varies from run to run; the key and its record do not.
__device__ __forceinline__ void req_dedup_entry_d(const DevReq& D, int e) {
  const ReqEntry E = D.entries[e];
  if (!(E.flags & kEntKey)) return;
  const bool cup = D.cup && D.cup[E.q];
  const double rmin = D.radius[E.q];
  unsigned long long h = dbits_d(E.cx) * 0x9E3779B97F4A7C15ULL;
  h = (h ^ (h >> 29)) + dbits_d(E.cy) * 0xBF58476D1CE4E5B9ULL;
  h = (h ^ (h >> 31)) + dbits_d(rmin) * 0x94D049BB133111EBULL;
  h ^= ((unsigned long long)(unsigned)E.ci << 33) ^ ((unsigned long long)(unsigned)E.cj << 1) ^ (unsigned long long)cup;
  h += (unsigned long long)(unsigned)E.map * 0xD6E8FEB86659FD93ULL;
  unsigned slot = (unsigned)(h ^ (h >> 32)) & D.tmask;
  int canon = -1;
  for (;;) {
    int s = D.table[slot];
    if (s == 0) {
      s = atomicCAS(D.table + slot, 0, e + 1);
      if (s == 0) { canon = e; break; }
    }
    if (req_same_key_d(D, D.entries[s - 1], E)) { canon = s - 1; break; }
    slot = (slot + 1) & D.tmask;
  }
  D.entries[e].key = canon;
  atomicAdd(D.counters + 0, 1ULL);  // candidates
  if (canon == e) {
    const int id = (int)atomicAdd(D.counters + 1, 1ULL);  // distinct keys
    D.kid[e] = id;
    D.keys[id] = MapKey{E.cx, E.cy, rmin, E.ci, E.cj, cup ? 1 : 0, E.map};
  }
}

__global__ void __launch_bounds__(256) k_req_dedup(DevReq D) {
  const int total = D.lofs[D.nposes];
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) req_dedup_entry_d(D, e);
}

// 5. Replay: the service loop of one map, one warp per map, over the map's entries in request order, 32 at a time.  Why this is
// the sequential loop (one check after the other, as the reference runs it) exactly:
//   - Which value a check reads depends only on the checks before it in its map: in the sequential loop a cell holds a value this
//     request stored iff an executed earlier check of the request walked it, and then that walk's float.  The live cache holds
//     exactly those: a cell the request stored, or one cached when it began, is finite (the walks store finite values); an empty
//     cell was empty when the request began, so its key's record is a walk.
//   - Within a window every lane assumes that all lanes before it run.  Among lanes of one cell only the first can find the cell
//     empty and walk; every later one reads the first one's float (the live value, or the float its record stores).  So under
//     that assumption each lane's value and verdict are the sequential loop's.
//   - The assumption holds up to and including the first failing lane f: no lane before it fails, and entries of one path are
//     consecutive, so the sequential loop runs lanes 0 .. f in this order.  They commit: first touches store their float, and one
//     lane folds the values in visit order, so sums, add_segment_d and the verdicts are the sequential loop's bit for bit.
//   - The sequential loop then skips the rest of f's path (the `break`s); the next window starts at the first entry of a later
//     path.  Lanes after f that belong to later paths are evaluated again there: their assumption included dropped lanes, which
//     store nothing.
//   - Gates fail without a polygon, as the loop's `break`.  Maps share nothing, so their warps run independently.
__global__ void __launch_bounds__(128) k_req_replay(FpArgs A, DevReq D, float* cache) {
  __shared__ double s_t[4][32];
  __shared__ int s_v[4][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (m >= D.nmaps) return;  // whole warp
  const int lo = D.map_range[2 * m], hi = D.map_range[2 * m + 1];
  if (lo >= hi) return;  // a map without circular paths
  int e0 = D.lofs[lo];
  const int e1 = D.lofs[hi];
  float* const mc = cache + m * D.map_cells;
  // lane 0: the path being folded
  int cur = -1, dead = -1, nLine = 0;
  bool ok = false;
  double result = 0.0, lengthPath = 0.0, sum = 0.0;
  ReqFail F{};
  unsigned long long stored = 0;
  while (e0 < e1) {
    const int e = e0 + lane;
    const bool have = e < e1;
    ReqEntry E{};
    if (have) E = D.entries[e];
    // the dropped rest of a failed path is a prefix of the window
    const unsigned dmask = __ballot_sync(0xffffffffu, have && E.q == dead);
    if (dmask & 1u) {
      e0 += (~dmask) ? __ffs((int)~dmask) - 1 : 32;
      continue;
    }
    const bool key = have && (E.flags & kEntKey);
    const unsigned long long cell = key ? (unsigned long long)E.cj * A.rows + E.ci : ~0ULL - lane;
    const int leader = __ffs((int)__match_any_sync(0xffffffffu, cell)) - 1;
    float live = 0.0f, rcache = 0.0f;
    MapRecord R{};
    if (key) {
      live = mc[cell];
      R = D.recs[D.kid[E.key]];
      rcache = R.cache;
    }
    const float lead_cache = __shfl_sync(0xffffffffu, rcache, leader);
    const bool walk = key && leader == lane && !finitef(live);
    double t = 0.0;
    bool lok = true;
    int fk = 0;  // the lane's polygon kind if it fails
    if (key) {
      if (walk) { t = R.t; lok = R.state == 0; fk = 2; }  // :679-736
      else {                                              // :673-678
        const float v = finitef(live) ? live : lead_cache;
        t = (double)v; lok = v != 0.0f; fk = 1;
      }
    } else if (have && (E.flags & kEntOutside)) {         // :662-667
      t = A.tdefault; lok = A.tdefault != 0.0; fk = 1;
    } else if (have) {                                    // a gate
      lok = false;
    }
    const unsigned fails = __ballot_sync(0xffffffffu, have && !lok);
    const int f = fails ? __ffs((int)fails) - 1 : 32;
    const int nhave = __popc(__ballot_sync(0xffffffffu, have));
    const int ncommit = min(f + 1, nhave);
    const bool commit_walk = walk && lane < ncommit;
    if (commit_walk) mc[cell] = R.cache;
    stored += __popc(__ballot_sync(0xffffffffu, commit_walk));
    s_t[w][lane] = t;
    s_v[w][lane] = (lok ? 1 : 0) | (fk << 1);
    __syncwarp();
    if (lane == 0) {
      for (int l = 0; l < ncommit; ++l) {
        const ReqEntry G = D.entries[e0 + l];
        const double tl = s_t[w][l];
        const bool okl = s_v[w][l] & 1;
        if (G.q != cur) {  // a new path: :345-362
          cur = G.q; ok = true; result = 0.0; lengthPath = 0.0; sum = 0.0; nLine = 0;
          F = ReqFail{0.0, 0.0, 0, -1, 1, 0};
        }
        if (G.flags & kEntGate) {
          ok = false;  // :365-367, :389-396: break without a polygon
        } else if (G.seg == 0) {  // :365-387
          result = tl;
          ok = okl;
        } else {  // :398-452
          sum += tl;
          ++nLine;
          if (!okl) {
            ok = false;
            F.freps = G.freps;
          } else if (G.flags & kEntSegEnd) {
            const int b = D.path_begin[G.q];
            const double* pe = D.poses + 7 * (size_t)(b + G.seg);
            const double* ps = pe - 7;
            add_segment_d(sum / (double)nLine, pe[0] - ps[0], pe[1] - ps[1], G.seg, lengthPath, result);
            sum = 0.0;
            nLine = 0;
          }
        }
        if (!okl && !(G.flags & kEntGate)) {
          F.fkind = s_v[w][l] >> 1; F.fx = G.cx; F.fy = G.cy;
          F.key = F.fkind == 2 ? D.kid[G.key] : -1;
        }
        if (!ok || (G.flags & kEntPathEnd)) {  // the path's answer (:458-461)
          const int q = G.q;
          D.is_safe[q] = ok ? 1 : 0;
          D.trav_out[q] = ok ? result : 0.0;
          D.area_out[q] = 0.0;
          const bool cup = D.cup != nullptr && D.cup[q] != 0;
          if (!cup || ok || F.fkind == 0) F.fkind = 0;
          if (D.O.count && F.fkind == 0) D.O.count[q] = 0;
          D.fails[q] = F;
          if (!ok) dead = q;
          cur = -1;
        }
      }
    }
    dead = __shfl_sync(0xffffffffu, dead, 0);
    e0 += (f < nhave) ? f + 1 : nhave;
    __syncwarp();
  }
  if (lane == 0 && stored) atomicAdd(D.counters + 2, stored);
}

// 6. Polygons: one warp per path; a path the replay did not leave a failing circle to publish exits at once.  The pair
// k_check_paths_fresh_poly calls: fromCircle, or spiral_blockers_d on the failing key and write_cells_polygon_d with its freps.
__global__ void __launch_bounds__(128, 4) k_req_polygons(FpArgs A, Layers L, PathArgs P, DevReq D, CircleTable C) {
  __shared__ int s_min[4][kFreshTableRows + 1], s_max[4][kFreshTableRows + 1];
  __shared__ int2 s_stack[4][2 * kFreshTableRows + 4];
  __shared__ int2 s_first[4][3];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (q >= D.npaths || D.status[q] != 1) return;  // whole warp
  const ReqFail F = D.fails[q];
  if (F.fkind == 0) return;
  const double rmax = D.radius[q] + D.offset;
  const UntravScratch S{s_min[w], s_max[w], s_stack[w], s_first[w]};
  if (F.fkind == 1) {
    const int n = D.path_begin[q + 1] - D.path_begin[q];
    if (lane == 0) write_circle_polygon_d(C.cs, C.sn, F.fx, F.fy, rmax, n > 1, reinterpret_cast<double2*>(S.stack), D.O, q);
    return;
  }
  const MapKey K = D.keys[F.key];
  const long long mo = (long long)K.map * D.map_cells;
  L = shift_layers_d(L, mo);
  P.memo += mo;
  const int nr = (int)ceil(rmax / A.res);
  const int cnt = spiral_blockers_d(A, L, P, S, K.cx, K.cy, K.ci, K.cj, K.rmin, rmax, nr);
  if (lane == 0) write_cells_polygon_d(A, S, 2 * nr + 1, K.ci - nr, cnt, F.freps, D.O, q);
}

// ---------------------------------------------------------------------------------------------------------------------------
// TraversabilityMap::checkPolygonalFootprintPath (TraversabilityMap.cpp:464-584) for a batch of paths that share one footprint
// polygon.  A work item is one polygon the reference evaluates: the footprint at the pose of a single-pose path, or the convex hull
// of segment (k-1, k) of a longer path.  Items are independent (the polygonal check keeps no traversability_footprint cache), so
// k_check_polygon_items runs one warp per pose index and k_check_polygon_combine folds the items of a path in order (:569-579).
struct PolyItem {
  int q;             // path of the item; -1: the pose is not an item
  int flag;          // 0: unsafe (checkInclination or isTraversable failed), 1: traversable, 2: not checkable
  double mean;       // isTraversable's `traversability`
  double hull_area;  // getArea of the checked polygon (the hull, or polygon2 for a single pose)
  double poly1_area; // getArea of the (possibly augmented) polygon1 list
};

struct PolyPathArgs {
  const float* rslope;           // robot_slope, nullptr: checkRobotInclination_ off
  int npaths, nposes, nfp;
  int mcap;                      // hull input points one warp's shared memory holds (2 * mcap + mcap double2)
  const int* path_begin;
  const double* poses;           // 7 per pose: x y z qx qy qz qw
  const unsigned char* cons;     // FootprintPath.conservative per path, nullptr: all 0
  unsigned char* memo;           // per map cell isTraversableForFilters memo (see blocked_memo_d)
  PolyItem* items;               // [nposes]
  unsigned char* is_safe;
  double* trav_out;
  double* area_out;
  float fx[kPolyMaxVerts], fy[kPolyMaxVerts], fz[kPolyMaxVerts];  // footprint vertices (geometry_msgs/Point32)
};

// Translation * Quaternion of a pose: Eigen::QuaternionBase::toRotationMatrix of the quaternion as given (not normalised), rows 0
// and 1 (the z of a transformed vertex is dropped, :505-507).
struct PoseRT {
  double tx, ty, r00, r01, r02, r10, r11, r12;
};
__device__ __forceinline__ PoseRT pose_rt_d(const double* p) {
  const double qx = p[3], qy = p[4], qz = p[5], qw = p[6];
  const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  PoseRT T;
  T.tx = p[0]; T.ty = p[1];
  T.r00 = 1.0 - (tyy + tzz); T.r01 = txy - twz; T.r02 = txz + twy;
  T.r10 = txy + twz; T.r11 = 1.0 - (txx + tzz); T.r12 = tyz - twx;
  return T;
}

// `toPosition * orientation * positionToVertex` (:496-500) for footprint vertex v, in the operand order of Eigen's Transform * vector.
// The vertex comes from the path's own footprint `fxyz` in global memory, or without one from the kernel parameters.
__device__ __forceinline__ double2 footprint_vertex_d(const PolyPathArgs& P, const float* fxyz, const PoseRT& T, int v) {
  double vx, vy, vz;
  if (fxyz) {
    vx = (double)fxyz[3 * v]; vy = (double)fxyz[3 * v + 1]; vz = (double)fxyz[3 * v + 2];
  } else {
    vx = (double)P.fx[v]; vy = (double)P.fy[v]; vz = (double)P.fz[v];
  }
  return make_double2(((T.r00 * vx + T.r01 * vy) + T.r02 * vz) + T.tx, ((T.r10 * vx + T.r11 * vy) + T.r12 * vz) + T.ty);
}

// grid_map::Polygon::getArea (recalled, see the oracle): the shoelace sum in vertex order, one thread.
__device__ double polygon_area_d(const double2* v, int n) {
  double area = 0.0;
  int j = n - 1;
  for (int i = 0; i < n; i++) {
    area += (v[j].x + v[i].x) * (v[j].y - v[i].y);
    j = i;
  }
  return fabs(area / 2.0);
}

// grid_map::Polygon::isInside (crossing-number test over (v[i], v[i-1]), as poly_inside_d) on a vertex list in shared memory.
__device__ __forceinline__ bool polygon_inside_d(const double2* v, int n, double px, double py) {
  int cross = 0;
  for (int i = 0, j = n - 1; i < n; j = i++) {
    if (((v[i].y > py) != (v[j].y > py)) && (px < (v[j].x - v[i].x) * (py - v[i].y) / (v[j].y - v[i].y) + v[i].x)) ++cross;
  }
  return (cross & 1) != 0;
}

// The untraversable polygons of the polygonal path check (k_check_polygon_items_poly / k_check_polygon_combine_poly).
struct PolyUntravArgs {
  const unsigned char* cup;  // FootprintPath.compute_untraversable_polygon per path, nullptr: all 0
  int* item_count;           // [nposes]: the item's vertex count (-1: its bounding box spans more than kUntravRows rows)
  double* item_xy;           // [nposes][maxv] (x, y)
  UntravOut out;             // per path
};

// Dynamic shared memory of one warp of k_check_polygon_items: sA, sB (3 mcap points); with the polygon also its UntravScratch.
__host__ __device__ inline size_t poly_warp_smem(int mcap, bool poly) {
  size_t s = sizeof(double2) * 3 * (size_t)mcap;
  if (poly) s += sizeof(int2) * (2 * kUntravRows + 4 + 4) + sizeof(int) * 2 * kUntravRows;
  return s;
}

// One warp per pose index p.  Shared memory per warp: sA (2 mcap points: the hull input polygon1 ++ polygon2, then the hull) and
// sB (mcap points: a conservative path's earlier polygon2, then the sorted hull input).  POLY: with compute_untraversable_polygon
// set for the item's path, the walk goes on past blocked cells and collects them (:602-608, :634-638).  With per-path footprints
// (R.fp_begin) each polygonal path uses its own, and the poses of circular paths are no items.
template <bool POLY>
__device__ __forceinline__ void check_polygon_item_d(const FpArgs& A, Layers L, const PolyPathArgs& P, const PolyUntravArgs& U,
                                                     const RequestArgs& R) {
  extern __shared__ double2 sPoly[];
  const int lane = threadIdx.x & 31;
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (p >= P.nposes) return;  // whole warp
  double2* sA = POLY ? reinterpret_cast<double2*>(reinterpret_cast<char*>(sPoly) + (threadIdx.x >> 5) * poly_warp_smem(P.mcap, true))
                     : sPoly + (size_t)(threadIdx.x >> 5) * 3 * P.mcap;
  double2* sB = sA + 2 * P.mcap;
  UntravScratch S{};
  if (POLY) {
    S.stack = reinterpret_cast<int2*>(sB + P.mcap);
    S.first = S.stack + 2 * kUntravRows + 4;
    S.tmin = reinterpret_cast<int*>(S.first + 4);
    S.tmax = S.tmin + kUntravRows;
  }
  PolyItem it{-1, 2, 0.0, 0.0, 0.0};
  // the path of pose p: the last q with path_begin[q] <= p
  int lo = 0, hi = P.npaths - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.path_begin[mid] <= p) lo = mid; else hi = mid - 1;
  }
  const int q = lo, b = P.path_begin[q], e = P.path_begin[q + 1], n = e - b, k = p - b;
  if (R.fp_begin && R.fp_begin[q + 1] == R.fp_begin[q]) return;  // a pose of a circular path
  const long long mo = map_offset_d(R, q);
  if (!(b >= 0 && b <= p && p < e && e <= P.nposes && (n == 1 || k >= 1)) || mo < 0) {
    if (lane == 0) P.items[p] = it;
    return;
  }
  L = shift_layers_d(L, mo);  // path q's map
  const float* const rslope = P.rslope ? P.rslope + mo : nullptr;
  unsigned char* const memo = P.memo + mo;
  it.q = q;
  const bool cup = POLY && U.cup != nullptr && U.cup[q] != 0;
  int ncollected = 0;  // POLY: blocked cells collected by the walk
  bool hit = false;    // POLY: the walk stopped at a blocked cell without collecting
  int nr_walk = 0, si_walk = 0;
  int nfp = P.nfp;
  const float* fxyz = nullptr;  // the path's own footprint
  if (R.fp_begin) {
    if (!__all_sync(0xffffffffu, request_footprint_ok_d(R, q, lane, 32))) {
      if (lane == 0) P.items[p] = it;  // flag 2
      return;
    }
    const int fb = R.fp_begin[q];
    nfp = R.fp_begin[q + 1] - fb;
    fxyz = R.fp_xyz + 3 * (size_t)fb;
  }
  const bool cons = n > 1 && P.cons != nullptr && P.cons[q] != 0;
  const int m = n == 1 ? nfp : cons ? 2 * nfp * (k + 1) : 2 * nfp;  // points of polygon1 ++ polygon2
  bool finite = true;
  for (int s = (cons ? 0 : max(k - 1, 0)) + lane; s <= k; s += 32)
    for (int c = 0; c < 7; ++c) finite = finite && isfinite(P.poses[7 * (size_t)(b + s) + c]);
  if (!__all_sync(0xffffffffu, finite) || m > P.mcap || (cons && nfp * (k + 1) > kPolyConsCap)) {
    if (lane == 0) P.items[p] = it;  // flag 2
    return;
  }
  const double* pk = P.poses + 7 * (size_t)(b + k);
  const double ex = pk[0], ey = pk[1];
  const double sx = n == 1 ? ex : pk[-7], sy = n == 1 ? ey : pk[-6];
  const int h = m / 2;  // polygon1 = sA[0, h), polygon2 = sA[h, m) for n > 1
  if (n == 1) {  // polygon2 of the pose
    const PoseRT T = pose_rt_d(pk);
    if (lane < nfp) sA[lane] = footprint_vertex_d(P, fxyz, T, lane);
  } else if (!cons) {  // polygon1 = T_{k-1}(footprint), polygon2 = T_k(footprint)
    const PoseRT T = pose_rt_d(lane < nfp ? pk - 7 : pk);
    if (lane < 2 * nfp) sA[lane] = footprint_vertex_d(P, fxyz, T, lane < nfp ? lane : lane - nfp);
  } else {
    // polygon2 of pose k-1 by footprint slot s = 0..k-1 (list order: slot k-1 first): slot s holds T_s(footprint) plus the
    // start-to-end vectors d_{s+1}, ..., d_{k-1} added in that order (:510-520).  Entry i is always lane i % 32's.
    for (int j = 0; j < k; ++j) {
      const double* pj = P.poses + 7 * (size_t)(b + j);
      const PoseRT T = pose_rt_d(pj);
      const double dx = j > 0 ? pj[0] - pj[-7] : 0.0, dy = j > 0 ? pj[1] - pj[-6] : 0.0;
      for (int i = lane; i < nfp * (j + 1); i += 32) {
        if (i >= nfp * j) sB[i] = footprint_vertex_d(P, fxyz, T, i - nfp * j);
        else sB[i] = make_double2(sB[i].x + dx, sB[i].y + dy);
      }
    }
    __syncwarp();
    // polygon1 = polygon2(k-1) ++ (T_k(footprint) - d_k); polygon2 = T_k(footprint) ++ (polygon2(k-1) + d_k)
    const PoseRT T = pose_rt_d(pk);
    const double dx = ex - sx, dy = ey - sy;
    const int ns = nfp * k;
    for (int l = lane; l < h; l += 32) {
      if (l < ns) {
        const double2 w = sB[(k - 1 - l / nfp) * nfp + l % nfp];
        sA[l] = w;
        sA[h + nfp + l] = make_double2(w.x + dx, w.y + dy);
      } else {
        const double2 w = footprint_vertex_d(P, fxyz, T, l - ns);
        sA[l] = make_double2(w.x - dx, w.y - dy);
        sA[h + l - ns] = w;
      }
    }
  }
  __syncwarp();
  if (lane == 0 && n > 1 && k > 1) it.poly1_area = polygon_area_d(sA, h);
  int nh = m;  // Polygon(points) as given: a single pose's polygon2, or a hull input of at most 3 points
  if (n > 1 && m > 3) {
    // lexicographic order by rank (ties between equal points by position; they change no later result)
    for (int i = lane; i < m; i += 32) {
      const double2 a = sA[i];
      int r = 0;
      for (int j = 0; j < m; ++j) {
        const double2 c = sA[j];
        r += (lex_less_d(c, a) || (c.x == a.x && c.y == a.y && j < i)) ? 1 : 0;
      }
      sB[r] = a;
    }
    __syncwarp();
    if (lane == 0) nh = monotone_chain_d(sB, m, sA);
    nh = __shfl_sync(0xffffffffu, nh, 0);
    __syncwarp();
  }
  if (lane == 0) it.hull_area = polygon_area_d(sA, nh);
  // checkInclination (:524-526, :550-554), then isTraversable(polygon) (:592-645)
  bool ok = inclination_ok_d(A, rslope, sx, sy, ex, ey);
  double t = 0.0;
  if (ok) {
    double tlx = sA[0].x, tly = sA[0].y, brx = tlx, bry = tly;  // PolygonIterator::findSubmapParameters
    for (int i = 1; i < nh; ++i) {
      const double2 w = sA[i];
      tlx = fmax(tlx, w.x); tly = fmax(tly, w.y);
      brx = fmin(brx, w.x); bry = fmin(bry, w.y);
    }
    bound_position_d(A, tlx, tly);
    bound_position_d(A, brx, bry);
    int si, sj, ei, ej;
    get_index_d(A, tlx, tly, si, sj);
    get_index_d(A, brx, bry, ei, ej);
    const int nr = ei - si + 1, nc = ej - sj + 1;
    const long long total = (nr > 0 && nc > 0) ? (long long)nr * nc : 0;
    unsigned cnt = 0;
    // POLY: collect the blocked cells (table row = map row - si) unless the bounding box has more rows than the table
    const bool collect = POLY && cup && nr <= kUntravRows;
    if (POLY && collect) { clear_table_d(S, nr); nr_walk = nr; si_walk = si; }
    for (long long base = 0; base < total; base += 32) {  // SubmapIterator order, 32 cells per pass; the sum in visit order
      const long long c = base + lane;
      bool member = false, blk = false;
      double v = 0.0;
      int a = 0, bb = 0;
      if (c < total) {
        a = si + (int)(c / nc);
        bb = sj + (int)(c % nc);
        if (a >= 0 && bb >= 0 && a < A.rows && bb < A.cols_total && polygon_inside_d(sA, nh, A.X[a], A.Y[bb])) {
          member = true;
          blk = blocked_memo_d(A, L, memo, a, bb);
          if (!blk) {
            const float f = __ldg(L.trav + (size_t)bb * A.rows + a);
            v = finitef(f) ? (double)f : A.tdefault;  // :613-619
          }
        }
      }
      if (POLY && collect) {
        collect_cells_d(S, blk, a, bb, si, ncollected);
        if (ncollected > 0) { ok = false; continue; }  // no sum is read after the first blocked cell
      }
      if (__any_sync(0xffffffffu, blk)) { ok = false; if (POLY) hit = true; break; }  // :602-611
      const unsigned take = __ballot_sync(0xffffffffu, member);
      cnt += __popc(take);
#pragma unroll
      for (int l = 0; l < 32; ++l) {
        const double o = __shfl_sync(0xffffffffu, v, l);
        if ((take >> l) & 1u) t += o;
      }
    }
    if (ok) {
      if (cnt == 0) {  // :623-628
        t = A.tdefault;
        ok = A.tdefault != 0.0;
      } else {
        t /= (double)cnt;  // :630
      }
    }
  }
  if (lane == 0) {
    it.flag = ok ? 1 : 0;
    it.mean = t;
    P.items[p] = it;
  }
  if (POLY && cup) {
    // isTraversable's polygon (:634-642): empty when traversable or when nothing was collected (checkInclination failed first, or
    // no cell centre is inside and traversability_default is 0); 3 cells or fewer in visit order; else the chain
    __syncwarp();
    if (lane == 0) {
      const UntravOut O{U.out.maxv, U.item_count, U.item_xy};
      if (hit) *(O.count + p) = -1;  // more bounding-box rows than the table holds
      else write_cells_polygon_d(A, S, nr_walk, si_walk, ncollected, 1, O, p);
    }
  }
}

__global__ void __launch_bounds__(128) k_check_polygon_items(FpArgs A, Layers L, PolyPathArgs P, RequestArgs R) {
  check_polygon_item_d<false>(A, L, P, PolyUntravArgs{}, R);
}

__global__ void __launch_bounds__(128) k_check_polygon_items_poly(FpArgs A, Layers L, PolyPathArgs P, PolyUntravArgs U, RequestArgs R) {
  check_polygon_item_d<true>(A, L, P, U, R);
}

// One thread per path: the area-weighted combination of the segment results in path order (:522-579).  An unsafe path reports 0;
// a path the items could not check (bad range, non-finite pose, conservative list past the cap) is_safe 0 and NaN.  POLY: the
// polygon of the item that failed (the reference publishes every segment's polygon and returns after the first failing one,
// :555-567; traversable segments publish nothing); -1 for a path the items could not check.  With per-path footprints (R.fp_begin)
// the polygonal paths only; a footprint that cannot be checked makes its path not checkable.
template <bool POLY>
__device__ __forceinline__ void check_polygon_combine_d(const PolyPathArgs& P, const PolyUntravArgs& U, const RequestArgs& R) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= P.npaths) return;
  int nfp = P.nfp;  // the path's footprint vertices
  bool fp_ok = true;
  if (R.fp_begin) {
    if (R.fp_begin[q + 1] == R.fp_begin[q]) return;  // a circular path: k_check_paths_fresh* writes its outputs
    fp_ok = request_footprint_ok_d(R, q, 0, 1);
    nfp = R.fp_begin[q + 1] - R.fp_begin[q];
  }
  int failed = -1;  // POLY: pose index of the failing item
  const int b = P.path_begin[q], e = P.path_begin[q + 1], n = e - b;
  bool checkable = fp_ok && b >= 0 && e >= b && e <= P.nposes && map_offset_d(R, q) >= 0;  // an empty path on no map too
  unsigned char safe = 0;
  double trav = 0.0, area = 0.0;
  if (checkable && n > 0) {
    const bool cons = n > 1 && P.cons != nullptr && P.cons[q] != 0;
    if (cons && (long long)nfp * n > kPolyConsCap) checkable = false;
    for (long long c = 7LL * b; c < 7LL * e && checkable; ++c) checkable = isfinite(P.poses[c]);
    const int k0 = n == 1 ? 0 : 1;
    for (int k = k0; k < n && checkable; ++k) checkable = P.items[b + k].q == q && P.items[b + k].flag != 2;
    if (checkable) {
      bool ok = true;
      for (int k = k0; k < n && ok; ++k) {
        const PolyItem it = P.items[b + k];
        ok = it.flag == 1;
        if (!ok) { if (POLY) failed = b + k; break; }  // :536-538, :564-567
        if (n == 1 || k == 1) {  // :541-542, :576-578
          area = it.hull_area;
          trav = it.mean;
        } else {  // :570-575
          const double areaPrevious = area;
          const double areaPolygon = it.hull_area - it.poly1_area;
          area += areaPolygon;
          trav = (areaPolygon * it.mean + areaPrevious * trav) / area;
        }
      }
      if (ok) safe = 1;
      else trav = area = 0.0;
    }
  }
  if (!checkable) trav = area = nan("");
  P.is_safe[q] = safe;
  P.trav_out[q] = trav;
  P.area_out[q] = area;
  if (POLY) {
    const bool cup = U.cup != nullptr && U.cup[q] != 0;
    const int nv = !cup ? 0 : !checkable ? -1 : failed >= 0 ? U.item_count[failed] : 0;
    U.out.count[q] = nv;
    const double* src = U.item_xy + 2 * (size_t)U.out.maxv * (failed >= 0 ? failed : 0);
    double* dst = U.out.xy + 2 * (size_t)U.out.maxv * q;
    for (int v = 0; v < 2 * min(nv, U.out.maxv); ++v) dst[v] = src[v];
  }
}

__global__ void __launch_bounds__(128) k_check_polygon_combine(PolyPathArgs P, RequestArgs R) {
  check_polygon_combine_d<false>(P, PolyUntravArgs{}, R);
}

__global__ void __launch_bounds__(128) k_check_polygon_combine_poly(PolyPathArgs P, PolyUntravArgs U, RequestArgs R) {
  check_polygon_combine_d<true>(P, U, R);
}

inline int signum(int v) { return (0 < v) - (v < 0); }

// grid_map::SpiralIterator::generateRing, executed literally (SURVEY.md A.3): rings 0 .. nRings in visit order, packed
// di & 0xff | (dj & 0xff) << 8; ring_start[d] = first entry of ring d, ring_start[nRings + 1] = number of entries.
std::vector<int> spiral_rings(int nRings, std::vector<int>& ring_start) {
  std::vector<int> s;
  ring_start.assign(nRings + 2, 0);
  s.push_back(0);
  for (int d = 1; d <= nRings; ++d) {
    ring_start[d] = (int)s.size();
    std::vector<std::pair<int, int>> ring;
    int px = d, py = 0;
    do {
      ring.emplace_back(px, py);
      const int nx = -signum(py), ny = signum(px);
      if (nx != 0 && (unsigned)std::sqrt((double)((px + nx) * (px + nx) + py * py)) == (unsigned)d) px += nx;
      else if (ny != 0 && (unsigned)std::sqrt((double)(px * px + (py + ny) * (py + ny))) == (unsigned)d) py += ny;
      else { px += nx; py += ny; }
    } while (px != d || py != 0);
    for (auto it = ring.rbegin(); it != ring.rend(); ++it) s.push_back((it->first & 0xff) | ((it->second & 0xff) << 8));
  }
  ring_start[nRings + 1] = (int)s.size();
  return s;
}

// The visit order of SpiralIterator(radius) with the edge bit on the rings that apply the circle test (nRings - 1, nRings).
std::vector<int> build_spiral(double radius, double res) {
  const int nRings = (int)std::ceil(radius / res);
  std::vector<int> ring_start;
  std::vector<int> s = spiral_rings(nRings, ring_start);
  for (int d = std::max(nRings - 1, 1); d <= nRings; ++d)
    for (int k = ring_start[d]; k < ring_start[d + 1]; ++k) s[k] |= 0x10000;
  return s;
}

}  // namespace

void FootprintState::release() {
  for (DevBuf* b : {&spiral, &block, &tables, &prefix, &list, &poly, &reduce, &rings, &memo, &items, &upoly, &devreq}) b->release();
  req_counters = nullptr;
  tables_valid = false;
  valid = false;
}

namespace {
// The geometry part of the kernel arguments.
FpArgs geometry_args(const SlabView& v, const te_geometry* g) {
  FpArgs a{};
  a.rows = v.rows; a.cols_total = v.cols_total; a.in_col0 = v.in_col0; a.in_ncols = v.in_ncols;
  a.out_col0 = v.out_col0; a.out_ncols = v.out_ncols;
  a.res = g->resolution; a.lenx = g->length_x; a.leny = g->length_y; a.posx = g->position_x; a.posy = g->position_y;
  a.X = v.X; a.Y = v.Y;
  return a;
}
}  // namespace

void launch_check_paths(const SlabView& v, const te_geometry* g, double traversability_default, const float* footprint, const float* robot_slope, int npaths,
                        const int* path_begin, const double* xy, unsigned char* is_safe, double* trav, cudaStream_t s) {
  FpArgs a = geometry_args(v, g);
  a.tdefault = traversability_default;
  k_check_paths<<<(npaths + 127) / 128, 128, 0, s>>>(a, footprint, robot_slope, npaths, path_begin, xy, is_safe, trav);
}

int footprint_halo(const te_geometry* g, const te_footprint_params* p) {
  const double res = g->resolution;
  const int spiral = (int)std::ceil((p->radius + p->offset) / res);
  // predicates of a visited cell: slope window 3 cells; step: 2.5-cell circle + 3x3 submap + gap walk
  const int walk = (int)std::ceil(p->max_gap_width / res) + 1;
  return spiral + std::max(4, 3 + 1 + walk);
}

namespace {
// The geometry and isTraversableForFilters parameters of the kernel arguments.
FpArgs filter_args(const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* rough) {
  FpArgs a = geometry_args(v, g);
  a.tdefault = p->traversability_default;
  a.maxgap = p->max_gap_width; a.crit = p->critical_step_height; a.int_norm = p->radius_is_integer_norm;
  a.verify_rough = (p->verify_roughness != 0 && rough != nullptr) ? 1 : 0;
  a.slope_R = (int)std::floor(3.0 * g->resolution / g->resolution) + 1;
  a.step_R = (int)std::floor(2.5 * g->resolution / g->resolution) + 1;
  return a;
}

// The per-call isTraversableForFilters memo of the path checks (blocked_memo_d): one byte per map cell of each of `nmaps` maps,
// cleared on `s`.
int reset_filter_memo(FootprintState& st, const SlabView& v, int nmaps, cudaStream_t s) {
  const size_t ncell = (size_t)v.rows * v.cols_total * nmaps;
  if (st.memo.reserve(ncell) != cudaSuccess) { st.why = "allocating the predicate memo failed"; return TE_ERR_CUDA; }
  if (cudaMemsetAsync(st.memo.p, 0, ncell, s) != cudaSuccess) { st.why = "cudaMemsetAsync(predicate memo) failed"; return TE_ERR_CUDA; }
  return 0;
}

// The ring table of the fresh path checks, rings 0 .. kPathMaxRings, uploaded once per context: the visit order inside a ring does
// not depend on the radius.
int ensure_ring_table(FootprintState& st, cudaStream_t s) {
  if (st.rings.p) return 0;
  std::vector<int> ring_start;
  const std::vector<int> sp = spiral_rings(kPathMaxRings, ring_start);
  std::vector<int> table(ring_start);
  table.insert(table.end(), sp.begin(), sp.end());
  if (st.rings.reserve(sizeof(int) * table.size()) != cudaSuccess) { st.why = "allocating the ring table failed"; return TE_ERR_CUDA; }
  if (cudaMemcpyAsync(st.rings.p, table.data(), sizeof(int) * table.size(), cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess) {
    st.rings.release();
    st.why = "ring table upload failed";
    return TE_ERR_CUDA;
  }
  return 0;
}

// The path arguments every circular kernel takes: the ring table (after ensure_ring_table) and the memo.
PathArgs path_args(const FootprintState& st, const te_footprint_params* p, const float* robot_slope) {
  PathArgs P{};
  P.rslope = robot_slope;
  P.offset = p->offset;
  P.ring_start = (const int*)st.rings.p;
  P.rings = P.ring_start + kPathMaxRings + 2;
  P.memo = (unsigned char*)st.memo.p;
  return P;
}

CircleTable circle_table() {
  CircleTable C{};
  for (int j = 0; j < kFromCircleVertices; ++j) {  // Polygon::fromCircle: theta = j * 2 * M_PI / (nVertices - 1)
    volatile double theta = j * 2 * M_PI / (kFromCircleVertices - 1);  // volatile: libm at run time, never a folded constant
    C.cs[j] = std::cos(theta);
    C.sn[j] = std::sin(theta);
  }
  return C;
}

// The item kernel (one warp per pose index, skipped without poses) and then the combine kernel of a polygonal check.  Four warps
// per block while their shared memory stays small (below 48 KB, or 100 KB with the polygon tables); one warp per block for long
// conservative paths.  `extra` are the arguments both kernels take after the PolyPathArgs.
template <class KItems, class KCombine, class... Extra>
int launch_polygon_kernels(FootprintState& st, KItems items, KCombine combine, const char* items_name, bool poly, const FpArgs& a,
                           const Layers& L, const PolyPathArgs& P, cudaStream_t s, int* launches, const Extra&... extra) {
  if (P.nposes > 0) {
    const size_t per_warp = poly_warp_smem(P.mcap, poly);
    const int wpb = per_warp * 4 <= (poly ? 100 : 48) * 1024 ? 4 : 1;
    const size_t smem = per_warp * wpb;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(items, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      st.why = std::string("cudaFuncSetAttribute(") + items_name + ") failed";
      return TE_ERR_CUDA;
    }
    const long long blocks = ((long long)P.nposes + wpb - 1) / wpb;
    items<<<(unsigned)blocks, 32 * wpb, smem, s>>>(a, L, P, extra...);
    ++*launches;
  }
  combine<<<(unsigned)((P.npaths + 127) / 128), 128, 0, s>>>(P, extra...);
  ++*launches;
  return 0;
}
}  // namespace

int launch_path_checks(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const PathChecks& r,
                       bool circular, bool clear_memo, cudaStream_t s, int* launches) {
  *launches = 0;
  const bool circles = circular && (r.footprint_begin || !r.footprint);
  const bool polygons = r.footprint_begin || r.footprint;
  const int maxfp = r.footprint_begin ? r.max_footprint_vertices : r.nfp;
  if (polygons && (maxfp < 0 || maxfp > kPolyMaxVerts || r.max_points < 2 || r.max_points > 2 * kPolyConsCap)) {
    st.why = "bad footprint size";
    return TE_ERR_BAD_ARG;
  }
  if (circles)
    if (int rc = ensure_ring_table(st, s)) return rc;
  if (clear_memo)  // one memo for both kinds of path: it depends on the layers only
    if (int rc = reset_filter_memo(st, v, r.nmaps, s)) return rc;
  const FpArgs a = filter_args(v, g, p, r.rough);
  const Layers L{r.trav, r.slope, r.step, r.elev, r.rough};
  const RequestArgs R{r.footprint_begin, r.footprint_xyz, r.nvertices, r.max_footprint_vertices, r.nposes, r.area_out,
                      r.path_map, r.nmaps, (long long)v.rows * v.cols_total};
  if (circles) {
    PathArgs C = path_args(st, p, r.robot_slope);
    C.npaths = r.npaths; C.pose_stride = r.pose_stride; C.path_begin = r.path_begin; C.poses = r.poses; C.radius = r.radius;
    C.cup = r.cup; C.is_safe = r.is_safe; C.trav_out = r.trav_out;
    const unsigned blocks = (unsigned)((32LL * r.npaths + 127) / 128);
    if (!r.ucount) k_check_paths_fresh<<<blocks, 128, 0, s>>>(a, L, C, R);
    else k_check_paths_fresh_poly<<<blocks, 128, 0, s>>>(a, L, C, UntravOut{r.max_vertices, r.ucount, r.uxy}, circle_table(), R);
    ++*launches;
  }
  if (!polygons) return 0;
  // the polygonal paths: per pose index one item record and, with polygons, a count and max_vertices points copied to the paths
  // by the combine kernel
  const size_t nitems = (size_t)std::max(r.nposes, 1);
  if (st.items.reserve(sizeof(PolyItem) * nitems) != cudaSuccess) { st.why = "allocating the polygon items failed"; return TE_ERR_CUDA; }
  PolyPathArgs P{};
  P.rslope = r.robot_slope; P.npaths = r.npaths; P.nposes = r.nposes; P.nfp = r.nfp; P.mcap = r.max_points;
  P.path_begin = r.path_begin; P.poses = r.poses; P.cons = r.conservative;
  P.memo = (unsigned char*)st.memo.p;
  P.items = (PolyItem*)st.items.p;
  P.is_safe = r.is_safe; P.trav_out = r.trav_out; P.area_out = r.area_out;
  for (int k = 0; r.footprint && k < r.nfp; ++k) {
    P.fx[k] = r.footprint[3 * k]; P.fy[k] = r.footprint[3 * k + 1]; P.fz[k] = r.footprint[3 * k + 2];
  }
  if (!r.ucount) return launch_polygon_kernels(st, k_check_polygon_items, k_check_polygon_combine, "k_check_polygon_items", false, a, L, P, s,
                                               launches, R);
  const size_t cbytes = (sizeof(int) * nitems + 15) / 16 * 16;
  if (st.upoly.reserve(cbytes + sizeof(double2) * nitems * (size_t)std::max(r.max_vertices, 1)) != cudaSuccess) {
    st.why = "allocating the untraversable polygons failed";
    return TE_ERR_CUDA;
  }
  const PolyUntravArgs U{r.cup, (int*)st.upoly.p, (double*)((char*)st.upoly.p + cbytes), UntravOut{r.max_vertices, r.ucount, r.uxy}};
  return launch_polygon_kernels(st, k_check_polygon_items_poly, k_check_polygon_combine_poly, "k_check_polygon_items_poly", true, a, L, P, s,
                                launches, U, R);
}

namespace {
size_t align16(size_t b) { return (b + 15) / 16 * 16; }
}  // namespace

int launch_map_request_device(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p,
                              const float* trav, const float* slope, const float* step, const float* rough, const float* elev,
                              const float* robot_slope, float* cache, int nmaps, const int* path_map, int npaths, int nposes,
                              const int* path_begin, const double* poses, const double* radius, const int* footprint_begin,
                              const unsigned char* cup, unsigned char* is_safe, double* trav_out, double* area_out, int max_vertices,
                              int* ucount, double* uxy, long long max_checks, bool nonfinite_ok, int sms, cudaStream_t s,
                              int* launches) {
  *launches = 0;
  if (nmaps < 1 || (!path_map && nmaps != 1)) { st.why = "a batch of maps needs a map per path"; return TE_ERR_BAD_ARG; }
  if (int rc = ensure_ring_table(st, s)) return rc;
  // the workspace: per path, per pose, per map, per entry (max_checks), the hash table and CUB's scratch
  const size_t np1 = (size_t)nposes + 1, nc = (size_t)std::max(max_checks, 1LL);
  const int nsort = std::max(nposes, kReqSortMin);
  unsigned tslots = 32;
  while (tslots < 2 * nc) tslots *= 2;
  size_t cub_scan1 = 0, cub_sort = 0, cub_scan2 = 0;
  if (cub::DeviceScan::ExclusiveSum(nullptr, cub_scan1, (const long long*)nullptr, (long long*)nullptr, (int)np1, s) != cudaSuccess ||
      cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (const unsigned short*)nullptr, (unsigned short*)nullptr, (const int*)nullptr,
                                      (int*)nullptr, nsort, 0, 16, s) != cudaSuccess ||
      cub::DeviceScan::ExclusiveSum(nullptr, cub_scan2, (const int*)nullptr, (int*)nullptr, (int)np1, s) != cudaSuccess) {
    st.why = "sizing the scan / sort scratch failed";
    return TE_ERR_CUDA;
  }
  const size_t cub_bytes = std::max(cub_scan1, std::max(cub_sort, cub_scan2));
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = align16(off + bytes); return o; };
  const size_t o_counters = take(4 * sizeof(unsigned long long)), o_range = take(2 * sizeof(int) * (size_t)nmaps);
  const size_t o_status = take((size_t)npaths), o_fails = take(sizeof(ReqFail) * (size_t)npaths);
  const size_t o_cnt = take(sizeof(long long) * np1), o_gofs = take(sizeof(long long) * np1);
  const size_t o_pkey = take(sizeof(unsigned short) * nsort), o_skey = take(sizeof(unsigned short) * nsort);
  const size_t o_pidx = take(sizeof(int) * nsort), o_order = take(sizeof(int) * nsort);
  const size_t o_lcnt = take(sizeof(int) * np1), o_lofs = take(sizeof(int) * np1);
  const size_t o_entries = take(sizeof(ReqEntry) * nc), o_kid = take(sizeof(int) * nc), o_keys = take(sizeof(MapKey) * nc);
  const size_t o_recs = take(sizeof(MapRecord) * nc), o_table = take(sizeof(int) * (size_t)tslots), o_cub = take(cub_bytes);
  if (st.devreq.reserve(off) != cudaSuccess) { st.why = "allocating the device request workspace failed"; return TE_ERR_CUDA; }
  char* base = (char*)st.devreq.p;
  DevReq D{};
  D.npaths = npaths; D.nposes = nposes; D.nmaps = nmaps; D.nsort = nsort;
  D.map_cells = (long long)g->rows * g->cols; D.max_checks = max_checks;
  D.path_begin = path_begin; D.poses = poses; D.radius = radius; D.fp_begin = footprint_begin; D.path_map = path_map; D.cup = cup;
  D.rslope = robot_slope; D.offset = p->offset;
  D.is_safe = is_safe; D.trav_out = trav_out; D.area_out = area_out; D.O = UntravOut{max_vertices, ucount, uxy};
  D.status = (unsigned char*)(base + o_status); D.fails = (ReqFail*)(base + o_fails);
  D.cnt = (long long*)(base + o_cnt); D.gofs = (long long*)(base + o_gofs);
  D.pkey = (unsigned short*)(base + o_pkey); D.skey = (unsigned short*)(base + o_skey);
  D.pidx = (int*)(base + o_pidx); D.order = (int*)(base + o_order); D.lcnt = (int*)(base + o_lcnt); D.lofs = (int*)(base + o_lofs);
  D.map_range = (int*)(base + o_range); D.entries = (ReqEntry*)(base + o_entries); D.kid = (int*)(base + o_kid);
  D.table = (int*)(base + o_table); D.tmask = tslots - 1; D.keys = (MapKey*)(base + o_keys); D.recs = (MapRecord*)(base + o_recs);
  D.counters = (unsigned long long*)(base + o_counters);
  D.nonfinite_ok = nonfinite_ok;
  st.req_counters = D.counters;
  void* tmp = base + o_cub;
  if (cudaMemsetAsync(base + o_counters, 0, o_status - o_counters, s) != cudaSuccess ||  // counters and map ranges
      cudaMemsetAsync(D.table, 0, sizeof(int) * (size_t)tslots, s) != cudaSuccess) {
    st.why = "clearing the device request workspace failed";
    return TE_ERR_CUDA;
  }
  const FpArgs a = filter_args(v, g, p, rough);
  const Layers L{trav, slope, step, elev, rough};
  const PathArgs P = path_args(st, p, robot_slope);
  auto blocks = [](long long n, int per) { return (unsigned)std::max((n + per - 1) / per, 1LL); };
  size_t b1 = cub_bytes, b2 = cub_bytes, b3 = cub_bytes;
  k_req_paths<<<blocks(npaths, 128), 128, 0, s>>>(a, D);
  k_req_count<<<blocks(nposes + 1, 128), 128, 0, s>>>(a, D);
  cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, b1, (const long long*)D.cnt, D.gofs, (int)np1, s);
  k_req_cut<<<blocks(npaths, 128), 128, 0, s>>>(D);
  k_req_keys<<<blocks(nsort, 128), 128, 0, s>>>(D);
  if (e == cudaSuccess)
    e = cub::DeviceRadixSort::SortPairs(tmp, b2, (const unsigned short*)D.pkey, D.skey, (const int*)D.pidx, D.order, nsort, 0, 16, s);
  k_req_sorted<<<blocks(nposes + 1, 128), 128, 0, s>>>(D);
  if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp, b3, (const int*)D.lcnt, D.lofs, (int)np1, s);
  k_req_list<<<blocks(nposes, 128), 128, 0, s>>>(a, D);
  k_req_dedup<<<(unsigned)std::min<long long>(blocks((long long)nc, 256), 8LL * sms), 256, 0, s>>>(D);
  k_map_eval_circles_dev<<<(unsigned)std::min<long long>(blocks((long long)nc, 4), 16LL * sms), 128, 0, s>>>(
      a, L, P, D.keys, D.counters + 1, cache, D.recs);
  k_req_replay<<<blocks(nmaps, 4), 128, 0, s>>>(a, D, cache);
  *launches = 12;  // nine kernels and three CUB calls, each counted as one launch (a CUB call runs two or more kernels)
  if (ucount) {
    k_req_polygons<<<blocks(npaths, 4), 128, 0, s>>>(a, L, P, D, circle_table());
    ++*launches;
  }
  if (e != cudaSuccess) { st.why = std::string("scan / sort failed: ") + cudaGetErrorString(e); return TE_ERR_CUDA; }
  return 0;
}

int launch_map_merge(const float* fresh, float* cache, float* out, size_t n, const int* slot, int nsel, int sms, cudaStream_t s) {
  const long long per_map = std::max<long long>((long long)sms * 8 / nsel, 1);
  const long long blocks = std::min<long long>((long long)((n + 255) / 256), per_map);
  k_map_merge<<<dim3((unsigned)std::max(blocks, 1LL), (unsigned)nsel), 256, 0, s>>>(cache, fresh, out, n, slot);
  return 0;
}

void launch_map_slots(const MapSlots& a, bool put, int sms, cudaStream_t s) {
  // 16-byte accesses when every map slot and every layer starts on a 16-byte boundary
  bool vec = a.cells % 4 == 0 && (reinterpret_cast<uintptr_t>(a.cache) & 15u) == 0;
  for (int l = 0; l < kMapSlotLayers; ++l)
    vec = vec && ((reinterpret_cast<uintptr_t>(a.src[l]) | reinterpret_cast<uintptr_t>(a.dst[l])) & 15u) == 0;
  const int V = vec ? 4 : 1;
  const long long per_map = std::max<long long>((long long)sms * 8 / a.nsel, 1);
  const long long bx = std::max(std::min<long long>((long long)((a.cells / V + 255) / 256), per_map), 1LL);
  const dim3 grid((unsigned)bx, (unsigned)std::min(a.nsel, 65535));
  if (put) {
    if (vec) k_map_slots<true, 4><<<grid, 256, 0, s>>>(a);
    else k_map_slots<true, 1><<<grid, 256, 0, s>>>(a);
  } else {
    if (vec) k_map_slots<false, 4><<<grid, 256, 0, s>>>(a);
    else k_map_slots<false, 1><<<grid, 256, 0, s>>>(a);
  }
}

// isTraversableForFilters for every cell of the slab + halo of each of the nmaps maps into st.block (k_pred_classify +
// k_pred_heavy); fills the geometry / parameter part of the kernel arguments.  Shared by the circular and the polygonal sweep.
int run_predicates(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                   const float* slope, const float* step, const float* rough, const float* elev, float* slope_fp, float* step_fp,
                   float* rough_fp, int sms, cudaStream_t s, FpArgs* out_args) {
  const double rmax = p->radius + p->offset;
  if (nmaps < 1 || nmaps > 65535) { st.why = "number of maps outside 1 .. 65535"; return TE_ERR_UNSUPPORTED; }
  const size_t ncell_in = (size_t)v.rows * v.in_ncols * nmaps;
  if (ncell_in >= ((size_t)1 << 32)) { st.why = "slab or batch of 2^32 or more cells"; return TE_ERR_UNSUPPORTED; }
  if ((size_t)v.in_ncols * nmaps >= ((size_t)1 << 31)) { st.why = "batch of 2^31 or more columns"; return TE_ERR_UNSUPPORTED; }
  if (st.block.reserve(ncell_in) != cudaSuccess) { st.why = "allocating the predicate bytes failed"; return TE_ERR_CUDA; }
  FpArgs a = filter_args(v, g, p, rough);
  a.rmin = p->radius; a.rmax = rmax; a.rmax2 = rmax * rmax;
  a.n_spiral = st.n_spiral; a.spiral = (const int*)st.spiral.p;
  a.nmaps = nmaps;
  const Layers L{trav, slope, step, elev, rough};
  const long long t1 = (long long)ncell_in;
  const int g1 = (int)std::min<long long>((t1 + 127) / 128, (long long)sms * 16);
  {
    if (st.list.reserve(sizeof(unsigned) * (ncell_in + 1)) != cudaSuccess) { st.why = "allocating the predicate work list failed"; return TE_ERR_CUDA; }
    unsigned* cnt = (unsigned*)st.list.p;          // word 0: list length; entries follow
    unsigned* lst = cnt + 1;
    cudaMemsetAsync(cnt, 0, sizeof(unsigned), s);
    const dim3 gc((unsigned)((v.rows + 255) / 256), (unsigned)v.in_ncols, (unsigned)nmaps);
    k_pred_classify<<<gc, 256, 0, s>>>(a, L, (unsigned char*)st.block.p, slope_fp, step_fp, rough_fp, lst, cnt);
    k_pred_heavy<<<std::max(g1, 1), 128, 0, s>>>(a, L, (unsigned char*)st.block.p, slope_fp, step_fp, rough_fp, lst, cnt);
  }
  *out_args = a;
  return 0;
}

int launch_footprint(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                     const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                     float* step_fp, float* rough_fp, int sms, cudaStream_t s, int* launches) {
  const double rmax = p->radius + p->offset;
  if (std::ceil(rmax / g->resolution) > 120.0) { st.why = "footprint radius exceeds 120 cells"; return TE_ERR_UNSUPPORTED; }
  if (!st.valid || std::memcmp(&st.key_geo, g, sizeof(*g)) != 0 || std::memcmp(&st.key_par, p, sizeof(*p)) != 0) {
    const std::vector<int> sp = build_spiral(rmax, g->resolution);
    if (st.spiral.reserve(sp.size() * sizeof(int)) != cudaSuccess) { st.why = "allocating the spiral table failed"; return TE_ERR_CUDA; }
    if (cudaMemcpyAsync(st.spiral.p, sp.data(), sp.size() * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess) { st.why = "spiral table upload failed"; return TE_ERR_CUDA; }
    st.n_spiral = (int)sp.size();
    st.key_geo = *g;
    st.key_par = *p;
    st.valid = true;
    st.tables_valid = false;
  }
  FpArgs a{};
  if (int rc = run_predicates(st, v, g, p, nmaps, trav, slope, step, rough, elev, slope_fp, step_fp, rough_fp, sms, s, &a)) return rc;
  const size_t ncols_in = (size_t)v.in_ncols * nmaps, ncell_in = (size_t)v.rows * ncols_in;  // input-buffer columns / cells of the batch
  const Layers L{trav, slope, step, elev, rough};
  const long long t1 = (long long)ncell_in, t2 = (long long)v.rows * v.out_ncols * nmaps;
  const int g2 = (int)std::min<long long>((t2 + 255) / 256, (long long)sms * 8);
  const int Lmax = (int)std::floor(rmax / g->resolution + 1e-9);
  const bool fast = Lmax <= 31 && v.out_ncols <= 65535 && std::getenv("TE_FOOTPRINT_BRUTE") == nullptr;
  if (!fast) {
    k_sweep<<<std::max(g2, 1), 256, 0, s>>>(a, L, (const unsigned char*)st.block.p, out);
    if (launches) *launches = 3;
    return 0;
  }
  // ---- prefix-sum sweep: tables (cached with the spiral) + per-call prefix/bit arrays -----------------
  if (!st.tables_valid) {
    const double res = g->resolution, r2 = rmax * rmax, tol = 1e-9 * r2 + 1e-300;
    const int nR = (int)std::ceil(rmax / res), Wd = 2 * Lmax + 1;
    std::vector<signed char> halfw(Wd, -1), inner((size_t)(nR + 2) * Wd, -1);
    std::vector<int> fuzzy, ring_start(nR + 2, 0);
    for (int l = -Lmax; l <= Lmax; ++l)
      for (int k = -Lmax - 1; k <= Lmax + 1; ++k) {
        const double d2 = (double)(k * k + l * l) * res * res;
        if (d2 < r2 - tol) halfw[l + Lmax] = (signed char)std::max<int>(halfw[l + Lmax], std::abs(k));
        else if (std::fabs(d2 - r2) <= tol && k >= -Lmax && k <= Lmax) fuzzy.push_back((k & 0xff) | ((l & 0xff) << 8) | 0x10000);
      }
    for (int d = 0; d <= nR + 1; ++d)
      for (int l = -Lmax; l <= Lmax; ++l) {
        int u = -1;
        for (int k = 0; k <= halfw[l + Lmax]; ++k)
          if (k * k + l * l < d * d) u = k;
        inner[(size_t)d * Wd + l + Lmax] = (signed char)u;
      }
    {  // ring boundaries of the spiral table: ring d = entries with floor(|offset|) == d, in table order
      const std::vector<int> sp = build_spiral(rmax, res);
      int idx = 0;
      for (int d = 0; d <= nR; ++d) {
        ring_start[d] = idx;
        while (idx < (int)sp.size()) {
          const int di = (int)(signed char)(sp[idx] & 0xff), dj = (int)(signed char)((sp[idx] >> 8) & 0xff);
          if ((int)std::sqrt((double)(di * di + dj * dj)) != d) break;
          ++idx;
        }
      }
      ring_start[nR + 1] = idx;
    }
    const size_t bytes = halfw.size() + inner.size() + 4 * (fuzzy.size() + 1) + 4 * ring_start.size() + 64;
    if (st.tables.reserve(bytes) != cudaSuccess) { st.why = "allocating the footprint tables failed"; return TE_ERR_CUDA; }
    char* base = (char*)st.tables.p;
    size_t off = 0;
    auto put = [&](const void* src, size_t n, size_t align) {
      off = (off + align - 1) / align * align;
      cudaMemcpyAsync(base + off, src, n, cudaMemcpyHostToDevice, s);
      const size_t at = off;
      off += n;
      return at;
    };
    st.off_ring = put(ring_start.data(), 4 * ring_start.size(), 4);
    st.off_fuzzy = put(fuzzy.empty() ? (const void*)ring_start.data() : (const void*)fuzzy.data(), 4 * std::max<size_t>(fuzzy.size(), 1), 4);
    st.off_halfw = put(halfw.data(), halfw.size(), 1);
    st.off_inner = put(inner.data(), inner.size(), 1);
    if (cudaStreamSynchronize(s) != cudaSuccess) { st.why = "footprint table upload failed"; return TE_ERR_CUDA; }
    std::memset(st.h_halfw, -1, sizeof(st.h_halfw));
    std::memcpy(st.h_halfw, halfw.data(), std::min(halfw.size(), sizeof(st.h_halfw)));
    st.n_fuzzy = (int)fuzzy.size();
    st.L = Lmax;
    st.nrings = nR;
    st.tables_valid = true;
  }
  const int words = (v.rows + 31) / 32;
  const size_t pbytes = sizeof(double) * (size_t)(v.rows + 1) * ncols_in;
  const size_t wbytes = (sizeof(unsigned) * (size_t)words * ncols_in + 15) / 16 * 16;
  const size_t gbytes = ncell_in;
  if (st.prefix.reserve(pbytes + wbytes + gbytes) != cudaSuccess) { st.why = "allocating the footprint prefix sums failed"; return TE_ERR_CUDA; }
  char* const prefix = (char*)st.prefix.p;
  const char* const tables = (const char*)st.tables.p;
  a.L = st.L; a.nrings = st.nrings; a.n_fuzzy = st.n_fuzzy; a.words = words;
  a.ring_start = (const int*)(tables + st.off_ring);
  a.fuzzy = (const int*)(tables + st.off_fuzzy);
  a.halfw = (const signed char*)(tables + st.off_halfw);
  a.inner = (const signed char*)(tables + st.off_inner);
  a.P = (const double*)prefix;
  a.bits = (const unsigned*)(prefix + pbytes);
  a.near = (const unsigned char*)prefix + pbytes + wbytes;
  std::memcpy(a.halfw_c, st.h_halfw, sizeof(a.halfw_c));
  {
    const int pstride = v.rows + 1;  // pitch of a prefix-sum column
    a.cntp[0] = 0;
    for (int k = 0; k < 64; ++k) {
      const int l = k - st.L, h = (k <= 2 * st.L) ? (int)st.h_halfw[k] : -1;
      a.off_hi[k] = h >= 0 ? l * pstride + h + 1 : 0;
      a.off_lo[k] = h >= 0 ? l * pstride - h : 0;   // a column outside the disk contributes P[0] - P[0]
      const long long bias = (long long)st.L * pstride + st.L;
      a.off8_hi[k] = (unsigned)(8 * (bias + a.off_hi[k]));
      a.off8_lo[k] = (unsigned)(8 * (bias + a.off_lo[k]));
      a.cntp[k + 1] = (short)(a.cntp[k] + (h >= 0 ? 2 * h + 1 : 0));
    }
  }
  const int g3 = (int)std::min<long long>((long long)sms * 8, ((long long)ncols_in + 7) / 8);
  const int g1b = (int)std::min<long long>((t1 + 255) / 256, (long long)sms * 8);
  k_fp_prepare_p<<<std::max(g3, 1), 256, 0, s>>>(a, L, (const unsigned char*)st.block.p, (double*)prefix, (unsigned*)(prefix + pbytes));
  k_fp_nearest<<<std::max(g1b, 1), 256, 0, s>>>(a, (unsigned char*)prefix + pbytes + wbytes);
  const dim3 gs((unsigned)((v.rows + 255) / 256), (unsigned)v.out_ncols, (unsigned)nmaps);
  k_sweep_fast<<<gs, 256, 0, s>>>(a, L, (const unsigned char*)st.block.p, out);
  if (launches) *launches = 5;
  return 0;
}

int polygon_reach(const te_geometry* g, int npts, const double* pts_xy) {
  double r = 0.0;
  for (int k = 0; k < npts; ++k) r = std::max(r, std::hypot(pts_xy[2 * k], pts_xy[2 * k + 1]));
  return (int)std::ceil(r / g->resolution) + 1;
}

int footprint_polygon_halo(const te_geometry* g, const te_footprint_params* p, int npts, const double* pts_xy) {
  const int walk = (int)std::ceil(p->max_gap_width / g->resolution) + 1;
  return polygon_reach(g, npts, pts_xy) + std::max(4, 3 + 1 + walk);
}

namespace {
// Offsets (di, dj) of the cells inside the polygon placed at a cell centre, relative to that centre: certain-in cells as runs per
// column offset, cells within `tol` of a comparison of grid_map::Polygon::isInside as the uncertain list.
struct PolyTables {
  std::vector<int> runs, fz;
};
bool classify_polygon(double res, int Lp, int npts, const double* px, const double* py, const double R[4], PolyTables* out, std::string* why) {
  std::vector<double> vx(npts), vy(npts);
  for (int k = 0; k < npts; ++k) {
    vx[k] = (R[0] * px[k] + R[1] * py[k]) + 0.0;
    vy[k] = (R[2] * px[k] + R[3] * py[k]) + 0.0;
  }
  const double tol = 1e-7 * res;  // rounding moves a comparison by ~1e-13 m at most; anything closer than this is decided per centre
  out->runs.clear();
  out->fz.clear();
  for (int dj = -Lp; dj <= Lp; ++dj) {
    int run_lo = 0;
    bool in_run = false;
    for (int di = -Lp; di <= Lp + 1; ++di) {
      bool inside = false, fuzzy = false, row_dep = false;
      if (di <= Lp) {
        // cell centre relative to the polygon's centre: X decreases with the row index, Y with the column index
        const double ptx = -res * (double)di, pty = -res * (double)dj;
        int cross = 0;
        for (int i = 0, j = npts - 1; i < npts; j = i++) {
          // equal y (bitwise; per centre both get the same centre coordinate added): (v[i].y > pt.y) == (v[j].y > pt.y) always
          if (vy[i] == vy[j]) continue;
          const bool ui = std::fabs(vy[i] - pty) < tol, uj = std::fabs(vy[j] - pty) < tol;
          if (ui || uj) fuzzy = true;  // (v.y > pt.y) may fall either way: depends on the column pair only
          const bool ci = vy[i] > pty, cj = vy[j] > pty;
          if ((ci != cj) || ui || uj) {
            const double thr = (vx[j] - vx[i]) * (pty - vy[i]) / (vy[j] - vy[i]) + vx[i];
            // the x comparison involves the centre's row; so does a threshold that is a quotient of two rounding-sized numbers
            if (std::fabs(ptx - thr) < tol || std::fabs(vy[j] - vy[i]) < 1e3 * tol) { fuzzy = true; row_dep = true; }
            if ((ci != cj) && ptx < thr) ++cross;
          }
        }
        inside = (cross & 1) != 0;
      }
      if (fuzzy) {
        if (out->fz.size() >= 4096) { *why = "footprint polygon has more than 4096 cells on its outline"; return false; }
        int chain = 0;
        if (!row_dep && !out->fz.empty()) {
          const int pw = out->fz.back();
          if ((int)(signed char)((pw >> 8) & 0xff) == dj && (int)(signed char)(pw & 0xff) == di - 1 && ((pw >> 16) & 1) == 0) chain = 1;
        }
        out->fz.push_back((di & 0xff) | ((dj & 0xff) << 8) | ((row_dep ? 1 : 0) << 16) | (chain << 17));
        inside = false;
      }
      if (inside && !in_run) { in_run = true; run_lo = di; }
      if (!inside && in_run) {
        in_run = false;
        out->runs.push_back((dj & 0xff) | ((run_lo & 0xff) << 8) | (((di - 1) & 0xff) << 16));
      }
    }
  }
  return true;
}

// Eigen::Quaternion::toRotationMatrix of AngleAxisd(yaw, UnitZ) = (w, 0, 0, z) = (cos(yaw/2), 0, 0, sin(yaw/2)), upper-left 2 x 2,
// in Eigen's operation order.  Yaw 0 gives w = 1, z = 0 exactly: the identity that traversability_x uses.
Rot2 yaw_rotation(double yaw) {
  const double w = std::cos(0.5 * yaw), z = std::sin(0.5 * yaw);
  const double tz = 2.0 * z, twz = tz * w, tzz = tz * z;
  return Rot2{1.0 - (0.0 + tzz), 0.0 - twz, 0.0 + twz, 1.0 - (0.0 + tzz)};
}

// Yaw groups of a k_poly_tile launch: a block sweeps a group of consecutive polygons of its tile.  Tiles alone fill an H100 from
// 4 * sms of them (at the largest reach two blocks are resident per SM: two waves); fewer tiles split the polygons into as many
// groups as bring the launch to 4 * sms blocks, at most one per polygon.  A group restages its tile, so larger groups save
// staging; which block sweeps a layer never changes its bits.
int polygon_groups(long long tiles, int npoly, int sms) {
  const long long want = std::max(1LL, (4LL * sms + tiles - 1) / tiles);
  return (int)std::min<long long>(npoly, want);
}
}  // namespace

// traversabilityFootprint(yaw) for every layer of `polys`: predicates once, the polygon tables of every rotation in one upload,
// then one k_poly_tile launch for all of them (and, in reduce mode with yaw groups, one k_poly_combine).
int launch_footprint_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int npts,
                             const double* pts_xy, int npoly, const PolygonLayer* polys, const PolygonReduce* reduce, const float* trav,
                             const float* slope, const float* step, const float* rough, const float* elev, int nmaps, int sms,
                             cudaStream_t s, int* launches) {
  if (npts < 3 || npts > PMAXV) { st.why = "footprint polygon needs 3 to 16 vertices"; return TE_ERR_UNSUPPORTED; }
  if (npoly < 1) { st.why = "no polygon layer to sweep"; return TE_ERR_UNSUPPORTED; }
  if (reduce && !reduce->worst && !reduce->best && !reduce->best_yaw) { st.why = "no reduction output"; return TE_ERR_UNSUPPORTED; }
  const int Lp = polygon_reach(g, npts, pts_xy);
  if (Lp > 31) { st.why = "footprint polygon reaches further than 31 cells from its centre"; return TE_ERR_UNSUPPORTED; }
  PolyArgs q{};
  q.Lp = Lp; q.npts = npts; q.npoly = npoly;
  for (int k = 0; k < npts; ++k) { q.px[k] = pts_xy[2 * k]; q.py[k] = pts_xy[2 * k + 1]; }
  // the call's table: npoly descriptors, then the runs of every polygon, then their uncertain offsets
  std::vector<PolyDesc> desc(npoly);
  std::vector<int> runs, fz;
  {
    PolyTables tb;
    for (int k = 0; k < npoly; ++k) {
      PolyDesc& d = desc[k];
      d.R = yaw_rotation(polys[k].yaw);
      const double R[4] = {d.R.r00, d.R.r01, d.R.r10, d.R.r11};
      if (!classify_polygon(g->resolution, Lp, npts, q.px, q.py, R, &tb, &st.why)) return TE_ERR_UNSUPPORTED;
      d.run0 = (int)runs.size(); d.nruns = (int)tb.runs.size();
      d.fz0 = (int)fz.size(); d.nfz = (int)tb.fz.size();
      d.ncert = 0;
      for (int rw : tb.runs) d.ncert += (int)(signed char)((rw >> 16) & 0xff) - (int)(signed char)((rw >> 8) & 0xff) + 1;
      d.out = polys[k].out;
      runs.insert(runs.end(), tb.runs.begin(), tb.runs.end());
      fz.insert(fz.end(), tb.fz.begin(), tb.fz.end());
    }
  }
  const size_t dbytes = sizeof(PolyDesc) * desc.size(), bytes = dbytes + sizeof(int) * (runs.size() + fz.size());
  std::vector<char> blob(bytes);
  std::memcpy(blob.data(), desc.data(), dbytes);
  if (!runs.empty()) std::memcpy(blob.data() + dbytes, runs.data(), sizeof(int) * runs.size());
  if (!fz.empty()) std::memcpy(blob.data() + dbytes + sizeof(int) * runs.size(), fz.data(), sizeof(int) * fz.size());
  FpArgs a{};
  if (int rc = run_predicates(st, v, g, p, nmaps, trav, slope, step, rough, elev, nullptr, nullptr, nullptr, sms, s, &a)) return rc;
  if (st.poly.p && st.poly.cap < bytes) cudaStreamSynchronize(s);  // kernels of an earlier call may still read the old tables
  if (st.poly.reserve(bytes) != cudaSuccess) { st.why = "allocating the polygon tables failed"; return TE_ERR_CUDA; }
  if (cudaMemcpyAsync(st.poly.p, blob.data(), bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) { st.why = "polygon table upload failed"; return TE_ERR_CUDA; }
  q.desc = (const PolyDesc*)st.poly.p;
  q.runs = (const int*)((const char*)st.poly.p + dbytes);
  q.fz = q.runs + runs.size();
  const size_t smem = sizeof(double) * (size_t)(PTC + 2 * Lp) * (PTR + 2 * Lp + 1) + (size_t)(PTC + 2 * Lp) * (PB * 2);
  if (!st.poly_attr) {
    const size_t smax = sizeof(double) * (size_t)(PTC + 62) * (PTR + 63) + (size_t)(PTC + 62) * (PB * 2);
    if (cudaFuncSetAttribute(k_poly_tile<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess) {
      st.why = "cudaFuncSetAttribute(max dynamic shared memory) failed"; return TE_ERR_CUDA;
    }
    st.poly_attr = true;
  }
  q.row_tiles = (v.rows + PTR - 1) / PTR;
  const int col_tiles = (v.out_ncols + PTC - 1) / PTC;
  const int ngroups = polygon_groups((long long)q.row_tiles * col_tiles * nmaps, npoly, sms);
  q.group = (npoly + ngroups - 1) / ngroups;
  const int nsplit = (npoly + q.group - 1) / q.group;  // groups actually launched
  const int nblocks_x = q.row_tiles * nsplit;
  const dim3 grid((unsigned)nblocks_x, (unsigned)col_tiles, (unsigned)nmaps);
  if (!reduce) {
    k_poly_tile<false><<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
    if (launches) *launches = 3;
    return 0;
  }
  // Reduce mode.  Without a split the sweep writes the outputs.  With one, each group writes its partial results to st.reduce:
  // the split only happens below 4 * sms tiles, so that is under (4 * sms + tiles) * PTR * PTC cells per array.
  const size_t n = (size_t)nmaps * v.out_ncols * v.rows;
  if (nsplit == 1) {
    q.worst = reduce->worst; q.best = reduce->best; q.best_yaw = reduce->best_yaw;
    k_poly_tile<true><<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
    if (launches) *launches = 3;
    return 0;
  }
  const bool want_best = reduce->best || reduce->best_yaw;
  const size_t per = (size_t)nsplit * n, sbytes = sizeof(float) * per * ((reduce->worst ? 1 : 0) + (want_best ? 1 : 0) + (reduce->best_yaw ? 1 : 0));
  if (st.reduce.p && st.reduce.cap < sbytes) cudaStreamSynchronize(s);  // kernels of an earlier call may still use the old scratch
  if (st.reduce.reserve(sbytes) != cudaSuccess) { st.why = "allocating the reduction scratch failed"; return TE_ERR_CUDA; }
  float* next = (float*)st.reduce.p;
  if (reduce->worst) { q.worst = next; next += per; }
  if (want_best) { q.best = next; next += per; }
  if (reduce->best_yaw) q.best_yaw = (int*)next;
  q.rstride = n;
  k_poly_tile<true><<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
  const int cblocks = (int)std::min<size_t>((n + 255) / 256, (size_t)sms * 8);
  k_poly_combine<<<cblocks, 256, 0, s>>>(q.worst, q.best, q.best_yaw, nsplit, n, reduce->worst, reduce->best, reduce->best_yaw);
  if (launches) *launches = 4;
  return 0;
}

}  // namespace te
