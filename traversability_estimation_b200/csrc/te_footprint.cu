// te_footprint.cu — TraversabilityMap::traversabilityFootprint(radius, offset): the circular footprint sweep, and the predicate
// pass that the polygonal sweep (te_footprint_polygon.cu) shares.
//
//   k_pred_classify, k_pred_heavy   isTraversableForFilters (TraversabilityMap.cpp:774-792) for every cell of the slab and its
//                  halo: checkForSlope (:867-893) and checkForStep (:794-865).  Both are pure functions of the layers (their
//                  slope_footprint / step_footprint layers are only memoisation), so they are evaluated once per cell instead of
//                  once per visit.  The gap walk of checkForStep decides on absolute double positions (submap geometry, dot
//                  products of perpendicular vectors, `norm < max_gap_width`), so this translation unit is compiled with
//                  --fmad=false and replays the reference's operand order.
//   k_sweep        isTraversable(center, radius + offset, ..., radius) (:654-746) for every cell: walk the SpiralIterator
//                  visit order (table built on the host by executing the iterator's own ring walk) until the first blocked cell.
//   k_fp_prepare_p, k_fp_nearest, k_sweep_fast   the same on per-column prefix sums of the traversability and packed blocked
//                  flags: the visited set is a lattice disk, walked ring by ring only where a blocked cell lies in it.
//
// Layers are column-major float32; the slab/halo conventions are those of te_chain.
#include "te_fp_device.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace te {
namespace {

// isTraversableForFilters for every cell of the input buffer (columns in_col0 .. in_col0+in_ncols), in two steps.  Almost every
// cell passes trivially — checkForSlope / checkForStep / checkForRoughness return true at once unless the cell's own layer
// value is exactly 0 (TraversabilityMap.cpp:869, :796, :897) — so k_pred_classify settles those with two or three coalesced
// loads and collects the others on a work list, which k_pred_heavy walks with one thread per listed cell (the window count,
// the submap / gap walk): the heavy threads are no longer scattered one or two per warp over the whole map.
// CODES (a te_map sweep, SweepRecord): each cell's recorded-layer code (te_fp_device.cuh) also goes to codes[c], 0 for a cell no
// check runs on.
template <bool CODES>
__device__ __forceinline__ void pred_classify_d(const FpArgs& A, const Layers& L, unsigned char* __restrict__ blocked, float* slope_fp,
                                                float* step_fp, float* rough_fp, unsigned* __restrict__ list, unsigned* __restrict__ count,
                                                unsigned char* __restrict__ codes) {
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
      if constexpr (CODES) codes[c] = 0;
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

__global__ void __launch_bounds__(256) k_pred_classify(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp,
                                                       float* step_fp, float* rough_fp, unsigned* __restrict__ list,
                                                       unsigned* __restrict__ count) {
  pred_classify_d<false>(A, L, blocked, slope_fp, step_fp, rough_fp, list, count, nullptr);
}

__global__ void __launch_bounds__(256) k_pred_classify_codes(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp,
                                                             float* step_fp, float* rough_fp, unsigned* __restrict__ list,
                                                             unsigned* __restrict__ count, unsigned char* __restrict__ codes) {
  pred_classify_d<true>(A, L, blocked, slope_fp, step_fp, rough_fp, list, count, codes);
}

// AT: the maps sit at their own positions (FpArgs::pos); the shared-position instantiation reads A as it always did.
template <bool AT, bool CODES>
__device__ __forceinline__ void pred_heavy_d(const FpArgs& A, const Layers& L, unsigned char* __restrict__ blocked, float* slope_fp,
                                             float* step_fp, float* rough_fp, const unsigned* __restrict__ list,
                                             const unsigned* __restrict__ count, unsigned char* __restrict__ codes) {
  const unsigned n = *count;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const unsigned c = list[k];
    const int i = (int)(c % (unsigned)A.rows);
    const unsigned col = c / (unsigned)A.rows;            // input-buffer column of the batch
    const unsigned m = col / (unsigned)A.in_ncols;        // its map
    const int j = A.in_col0 + (int)(col - m * (unsigned)A.in_ncols);
    const size_t mc = (size_t)m * A.in_ncols * A.rows;    // the map's first cell: filters_d reads its layers only
    const Layers Lm{L.trav + mc, L.slope + mc, L.step + mc, L.elev + mc, L.rough ? L.rough + mc : nullptr};
    FilterVerdict v;
    if constexpr (AT) v = filters_d(map_args_d(A, m), Lm, i, j);
    else v = filters_d(A, Lm, i, j);
    blocked[c] = v.ok ? 0 : 1;
    if constexpr (CODES) codes[c] = (unsigned char)verdict_code_d(v);
    const int oj = j - A.out_col0;
    if (oj >= 0 && oj < A.out_ncols) {
      const size_t oc = ((size_t)m * A.out_ncols + oj) * A.rows + i;
      if (slope_fp) slope_fp[oc] = v.sfp;
      if (step_fp) step_fp[oc] = v.tfp;
      if (rough_fp) rough_fp[oc] = v.rfp;
    }
  }
}

template <bool AT>
__global__ void __launch_bounds__(128) k_pred_heavy(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp, float* step_fp,
                                                    float* rough_fp, const unsigned* __restrict__ list, const unsigned* __restrict__ count) {
  pred_heavy_d<AT, false>(A, L, blocked, slope_fp, step_fp, rough_fp, list, count, nullptr);
}

template <bool AT>
__global__ void __launch_bounds__(128) k_pred_heavy_codes(FpArgs A, Layers L, unsigned char* __restrict__ blocked, float* slope_fp,
                                                          float* step_fp, float* rough_fp, const unsigned* __restrict__ list,
                                                          const unsigned* __restrict__ count, unsigned char* __restrict__ codes) {
  pred_heavy_d<AT, true>(A, L, blocked, slope_fp, step_fp, rough_fp, list, count, codes);
}

// The recorded layers of a te_map sweep (SweepRecord).  Every empty centre walks its spiral, and the spiral starts at the centre, so
// k_plane_centres records each empty cell's own code (codes, from the predicates).  A walk reaches only empty cells, whose codes
// that records, and cached cells.  A cached cell got its value from a walk centred on it, which recorded it, so this is the whole
// record unless the map's bytes were reset while its cache stayed (a change of the memo key, SweepRecord::walk): only then does
// k_plane_walks walk every empty centre of the map (one warp each, record_circle_d) to reach the cached cells.
__global__ void __launch_bounds__(256) k_plane_centres(const unsigned char* __restrict__ codes, const float* __restrict__ cache,
                                                       const int* __restrict__ slot, unsigned char* plane, size_t cells, int nmaps) {
  const size_t total = cells * nmaps;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (size_t)gridDim.x * blockDim.x) {
    const size_t m = x / cells, r = (slot ? (size_t)slot[m] : m) * cells + (x - m * cells);
    if (finitef(__ldg(cache + r))) continue;
    if (const unsigned char code = __ldg(codes + x)) plane[r] |= code;
  }
}

template <bool AT>
__global__ void __launch_bounds__(128) k_plane_walks(FpArgs A0, Layers L, PathArgs P, const float* __restrict__ cache,
                                                     const int* __restrict__ slot, unsigned char* plane, const int* __restrict__ flags) {
  const unsigned m = blockIdx.y;  // block row m: map m of the launch
  if (!flags[m]) return;
  const size_t cells = (size_t)A0.rows * A0.cols_total, r0 = (slot ? (size_t)slot[m] : m) * cells;
  FpArgs Am;
  if constexpr (AT) Am = map_args_d(A0, m);
  const FpArgs& A = AT ? Am : A0;
  const Layers Lm = shift_layers_d(L, (long long)(m * cells));
  for (size_t c = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < cells; c += ((size_t)gridDim.x * blockDim.x) >> 5) {
    if (finitef(__ldg(cache + r0 + c))) continue;  // whole warp
    const int i = (int)(c % A.rows), j = (int)(c / A.rows);
    record_circle_d(A, Lm, P, plane + r0, nullptr, A.X[i], A.Y[j], i, j, A.rmin, A.rmax, (int)ceil(A.rmax / A.res), false);
  }
}

template <bool AT>
__global__ void __launch_bounds__(256) k_sweep(FpArgs A, Layers L, const unsigned char* __restrict__ blocked, float* __restrict__ out) {
  const long long total = (long long)A.rows * A.out_ncols * A.nmaps;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % A.rows);
    const unsigned col = (unsigned)(c / A.rows);  // output column of the batch
    const unsigned m = col / (unsigned)A.out_ncols;
    const int j = A.out_col0 + (int)(col - m * (unsigned)A.out_ncols);
    const size_t mc = (size_t)m * A.in_ncols * A.rows;  // the map's first input cell
    const double* const X = AT ? A.X + (size_t)m * A.xs : A.X;  // the map's coordinate tables
    const double* const Y = AT ? A.Y + (size_t)m * A.ys : A.Y;
    const double cx = X[i], cy = Y[j];
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
        const double dx = X[a] - cx, dy = Y[b] - cy;
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
// index (double; exact for float32 terms, so the order of summation does not matter) and packed blocked flags.  Only for a finite
// default (launch_footprint); a default far outside the layer's range, such as 1e6, loses the low bits of the terms after it.
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
template <bool AT>
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
    const double* const X = AT ? A.X + (size_t)blockIdx.z * A.xs : A.X;  // the map's coordinate tables
    const double* const Y = AT ? A.Y + (size_t)blockIdx.z * A.ys : A.Y;
    const double cx = X[active ? i : 0], cy = Y[j];
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
        const double dx = X[a] - cx, dy = Y[b] - cy;
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
        const double dx = X[a] - cx, dy = Y[b] - cy;
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
          const double dx = X[a] - cx, dy = Y[b] - cy;
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
  for (DevBuf* b : {&spiral, &block, &tables, &prefix, &list, &poly, &reduce, &rings, &memo, &items, &upoly, &codes, &devreq}) b->release();
  req_counters = nullptr;
  tables_valid = false;
  valid = false;
}

// The geometry part of the kernel arguments.
FpArgs geometry_args(const SlabView& v, const te_geometry* g) {
  FpArgs a{};
  a.rows = v.rows; a.cols_total = v.cols_total; a.in_col0 = v.in_col0; a.in_ncols = v.in_ncols;
  a.out_col0 = v.out_col0; a.out_ncols = v.out_ncols;
  a.res = g->resolution; a.lenx = g->length_x; a.leny = g->length_y; a.posx = g->position_x; a.posy = g->position_y;
  a.X = v.X; a.Y = v.Y;
  a.xs = v.xs; a.ys = v.ys; a.pos = v.pos;
  return a;
}

bool footprint_reach_ok(double resolution, const te_footprint_params* p) {
  return !(std::ceil((p->radius + p->offset) / resolution) > 120.0);
}

int footprint_halo(const te_geometry* g, const te_footprint_params* p) {
  const double res = g->resolution;
  const int spiral = (int)std::ceil((p->radius + p->offset) / res);
  // predicates of a visited cell: slope window 3 cells; step: 2.5-cell circle + 3x3 submap + gap walk
  const int walk = (int)std::ceil(p->max_gap_width / res) + 1;
  return spiral + std::max(4, 3 + 1 + walk);
}

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

// isTraversableForFilters for every cell of the slab + halo of each of the nmaps maps into st.block (k_pred_classify +
// k_pred_heavy); fills the geometry / parameter part of the kernel arguments.  Shared by the circular and the polygonal sweep.
int run_predicates(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                   const float* slope, const float* step, const float* rough, const float* elev, float* slope_fp, float* step_fp,
                   float* rough_fp, int sms, cudaStream_t s, FpArgs* out_args, unsigned char* codes) {
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
    unsigned char* const blk = (unsigned char*)st.block.p;
    if (!codes) {
      k_pred_classify<<<gc, 256, 0, s>>>(a, L, blk, slope_fp, step_fp, rough_fp, lst, cnt);
      (a.pos ? k_pred_heavy<true> : k_pred_heavy<false>)<<<std::max(g1, 1), 128, 0, s>>>(a, L, blk, slope_fp, step_fp, rough_fp, lst, cnt);
    } else {
      k_pred_classify_codes<<<gc, 256, 0, s>>>(a, L, blk, slope_fp, step_fp, rough_fp, lst, cnt, codes);
      (a.pos ? k_pred_heavy_codes<true> : k_pred_heavy_codes<false>)<<<std::max(g1, 1), 128, 0, s>>>(a, L, blk, slope_fp, step_fp,
                                                                                                     rough_fp, lst, cnt, codes);
    }
  }
  *out_args = a;
  return 0;
}

int launch_footprint(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                     const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                     float* step_fp, float* rough_fp, int sms, cudaStream_t s, int* launches, const SweepRecord* rec) {
  const double rmax = p->radius + p->offset;
  if (!footprint_reach_ok(g->resolution, p)) { st.why = "footprint radius exceeds 120 cells"; return TE_ERR_UNSUPPORTED; }
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
  unsigned char* codes = nullptr;
  const size_t cells = (size_t)v.rows * v.cols_total;
  if (rec) {
    if (v.in_col0 != 0 || v.in_ncols != v.cols_total) { st.why = "a recorded sweep takes whole maps"; return TE_ERR_BAD_ARG; }
    if (st.codes.reserve(cells * nmaps + sizeof(int) * (size_t)nmaps + 16) != cudaSuccess) {
      st.why = "allocating the recorded-layer codes failed";
      return TE_ERR_CUDA;
    }
    codes = (unsigned char*)st.codes.p;
  }
  if (int rc = run_predicates(st, v, g, p, nmaps, trav, slope, step, rough, elev, slope_fp, step_fp, rough_fp, sms, s, &a, codes)) return rc;
  const Layers L{trav, slope, step, elev, rough};
  int nrec = 0;  // the recording's launches
  if (rec) {
    const long long gp = std::min<long long>(((long long)(cells * nmaps) + 255) / 256, (long long)sms * 8);
    k_plane_centres<<<(unsigned)std::max(gp, 1LL), 256, 0, s>>>(codes, rec->cache, rec->slot, rec->plane, cells, nmaps);
    nrec = 1;
    if (rec->walk) {
      if (int rc = ensure_ring_table(st, s)) return rc;
      const std::vector<int> flags(rec->walk, rec->walk + nmaps);
      int* dflags = (int*)(codes + (cells * nmaps + 15) / 16 * 16);
      // pageable source: consumed before cudaMemcpyAsync returns, ordered after the kernels queued before on the stream
      if (cudaMemcpyAsync(dflags, flags.data(), sizeof(int) * (size_t)nmaps, cudaMemcpyHostToDevice, s) != cudaSuccess) {
        st.why = "uploading the maps to walk failed";
        return TE_ERR_CUDA;
      }
      const PathArgs P = path_args(st, p, nullptr);
      const dim3 gw((unsigned)std::max(sms * 16 / nmaps, 1), (unsigned)nmaps);
      (a.pos ? k_plane_walks<true> : k_plane_walks<false>)<<<gw, 128, 0, s>>>(a, L, P, rec->cache, rec->slot, rec->plane, dflags);
      nrec = 2;
    }
  }
  const size_t ncols_in = (size_t)v.in_ncols * nmaps, ncell_in = (size_t)v.rows * ncols_in;  // input-buffer columns / cells of the batch
  const long long t1 = (long long)ncell_in, t2 = (long long)v.rows * v.out_ncols * nmaps;
  const int g2 = (int)std::min<long long>((t2 + 255) / 256, (long long)sms * 8);
  // The tables classify lattice offsets (k, l) by d2 = (k^2 + l^2) res^2 against r2 = rmax^2; the reference tests the same cell with
  // dx * dx + dy * dy <= r2 on absolute cell centres, dx = X[a] - X[i] (likewise dy).  Each centre is (B + res * (-idx)) rounded,
  // B = (position + offset) rounded once per map and so common to both, and res * (-idx) is below 2M in magnitude: dx is
  // -k res + e with |e| <= 2 ulp(M) (two products and two sums, half an ulp each), M the largest |coordinate| the call touches.
  // Then dx^2 + dy^2 = d2 + 2 res (|k| + |l|) * 2 ulp(M) at most = d2 + 4 sqrt(2) r ulp(M) near the circle, plus relative roundings
  // of a few 2^-53 that 1e-9 r2 covers.  tol = max(1e-9 r2, 8 r ulp(M)): an offset closer than that to the circle goes to the
  // uncertain list and is decided per centre on absolute doubles.  Near the origin 1e-9 r2 is the larger one, so the tables are
  // what they always were; far out (a UTM or LV95 map) more offsets become uncertain.  Lmax, the largest |offset| that can be
  // inside, widens with the same bound.
  const double res = g->resolution, r2 = rmax * rmax, cu = coord_ulp(v.coord_max + rmax);
  const double tol_far = 8.0 * rmax * cu, tol = std::max(1e-9 * r2, tol_far) + 1e-300;
  const int Lmax = lattice_reach(rmax, res, cu);
  // The prefix sums hold the default of every invalid cell of a column: a NaN or infinite default would make every disk below the
  // column's first invalid cell non-finite, where the reference adds it only for the invalid cells it visits.  k_sweep adds in
  // visit order, so it takes that case.
  const bool fast = Lmax <= 31 && v.out_ncols <= 65535 && std::isfinite(p->traversability_default) &&
                    std::getenv("TE_FOOTPRINT_BRUTE") == nullptr;
  if (!fast) {
    (a.pos ? k_sweep<true> : k_sweep<false>)<<<std::max(g2, 1), 256, 0, s>>>(a, L, (const unsigned char*)st.block.p, out);
    if (launches) *launches = 3 + nrec;
    return 0;
  }
  // ---- prefix-sum sweep: tables (cached with the spiral) + per-call prefix/bit arrays -----------------
  if (!st.tables_valid || st.tables_ulp != cu) {  // maps of an _at entry move M: the tables follow the tolerance
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
    st.tables_ulp = cu;
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
  (a.pos ? k_sweep_fast<true> : k_sweep_fast<false>)<<<gs, 256, 0, s>>>(a, L, (const unsigned char*)st.block.p, out);
  if (launches) *launches = 5 + nrec;
  return 0;
}

}  // namespace te
