// te_fp_device.cuh — what more than one footprint unit compiles (te_footprint.cu, te_footprint_polygon.cu, te_paths.cu,
// te_map_request.cu); te_capi.cu sees te_footprint.h only.
//
//   - the kernel argument structs, and the host helpers that fill them, each defined in the unit named at its declaration;
//   - isTraversableForFilters on the chain layers (checkForSlope, checkForStep, checkForRoughness) and SpiralIterator's radius;
//   - the circle walk that the stateless path checks (te_paths.cu, an empty traversability_footprint cache per path) and the te_map
//     replay (te_map_request.cu, one cache across paths and requests) share: checkInclination, the running path mean, the
//     isTraversableForFilters memo, isTraversable on an empty cache and the untraversable polygon of a circle.
//
// The argument structs are in namespace te because the host helpers pass them from unit to unit.  The device code is in an
// anonymous namespace: each unit compiles its own copy of what it calls, and each kernel is defined in one unit.
#pragma once
#include <vector>

#include "te_footprint.h"

namespace te {

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
  // maps at their own positions (SlabView::xs / ys / pos): map m's coordinate tables start m * xs entries into X and m * ys into Y,
  // its position is pos[2m], pos[2m + 1]; xs = ys = 0 and pos null: every map at (posx, posy)
  int xs, ys;
  const double* pos;
  // maps with parameters of their own (PathChecks::map_params): map m reads mp[m] instead of tdefault, maxgap, crit, int_norm,
  // verify_rough and the walk's offset (map_params_d, map_walk_offset_d); null: every map reads the fields above
  const FpMapParams* mp;
};

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

constexpr int kFromCircleVertices = 20;    // grid_map::Polygon::fromCircle's default nVertices
// cos / sin of fromCircle's vertex angles, from the host's libm (circle_table)
struct CircleTable {
  double cs[kFromCircleVertices], sn[kFromCircleVertices];
};

// ---- host helpers of more than one unit ----------------------------------------------------------------------------------
// te_footprint.cu: the geometry part of the kernel arguments, and the geometry and isTraversableForFilters parameters.
FpArgs geometry_args(const SlabView& v, const te_geometry* g);
FpArgs filter_args(const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* rough);
// te_footprint.cu: isTraversableForFilters for every cell of the slab + halo of each of the nmaps maps into st.block (and, with
// `codes`, each cell's recorded-layer code into codes).
int run_predicates(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                   const float* slope, const float* step, const float* rough, const float* elev, float* slope_fp, float* step_fp,
                   float* rough_fp, int sms, cudaStream_t s, FpArgs* out_args, unsigned char* codes = nullptr);
// te_paths.cu: SpiralIterator's rings, the ring table of the circle walk, the path arguments and the fromCircle table.
std::vector<int> spiral_rings(int nRings, std::vector<int>& ring_start);
int ensure_ring_table(FootprintState& st, cudaStream_t s);
PathArgs path_args(const FootprintState& st, const te_footprint_params* p, const float* robot_slope);
CircleTable circle_table();

namespace {

__device__ __forceinline__ float lay(const FpArgs& A, const float* l, int i, int j) {  // caller guarantees (i,j) is in the map
  const int lb = j - A.in_col0;
  if (lb < 0 || lb >= A.in_ncols) return nanf_();
  return __ldg(l + (size_t)lb * A.rows + i);
}

// The arguments of map m of a batch whose maps sit at their own positions: its coordinate tables and position.
__device__ __forceinline__ FpArgs map_args_d(const FpArgs& A, unsigned m) {
  FpArgs a = A;
  a.X += (size_t)m * A.xs;
  a.Y += (size_t)m * A.ys;
  a.posx = A.pos[2 * (size_t)m];
  a.posy = A.pos[2 * (size_t)m + 1];
  return a;
}

// Map m's own parameters (A.mp) over those of the call, for a batch whose maps have parameters of their own.
__device__ __forceinline__ void map_params_d(FpArgs& A, unsigned m) {
  const FpMapParams q = A.mp[m];
  A.tdefault = q.tdefault;
  A.maxgap = q.maxgap;
  A.crit = q.crit;
  A.int_norm = q.int_norm;
  A.verify_rough = q.verify_rough;
}

// The arguments of path or key map m: its tables and position when the maps sit at their own (AT), its parameters when the maps
// have their own (EACH: A.mp is set).  Kernels instantiate EACH apart so that the one-parameter-set case keeps its parameters in
// the constant bank, and its registers.
template <bool AT, bool EACH>
__device__ __forceinline__ FpArgs map_view_d(const FpArgs& A0, unsigned m) {
  FpArgs a = AT ? map_args_d(A0, m) : A0;
  if constexpr (EACH) map_params_d(a, m);
  return a;
}

// radiusMax - radius of map m's circle walks: its own offset when the maps have their own parameters (EACH), else the call's.
template <bool EACH>
__device__ __forceinline__ double map_walk_offset_d(const FpArgs& A, double offset, unsigned m) {
  if constexpr (EACH) return A.mp[m].offset;
  return offset;
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

// ---- the slope_footprint / step_footprint / roughness_footprint layers a te_map records ----------------------------------
// One byte per cell: two bits per layer (bits 0-1 slope_footprint, 2-3 step_footprint, 4-5 roughness_footprint), each
// 0 = NaN (not written), 1 = 0.0f, 2 = 1.0f.  A visit of the reference writes a cell's FilterVerdict fields, which depend on the
// cell, the layers and the isTraversableForFilters parameters only, so a record is the byte OR the verdict's code.
__device__ __forceinline__ unsigned fp_field_code_d(float v) { return v == 0.0f ? 1u : v == 1.0f ? 2u : 0u; }
__device__ __forceinline__ unsigned verdict_code_d(const FilterVerdict& v) {
  return fp_field_code_d(v.sfp) | fp_field_code_d(v.tfp) << 2 | fp_field_code_d(v.rfp) << 4;
}
// isTraversableForFilters fails at a cell iff one of its checks wrote 0 (a check fails only on a cell whose own layer is 0).
__device__ __forceinline__ bool code_blocked_d(unsigned code) { return (code & 0x15u & ~(code >> 1)) != 0; }

// The code map cell (a, b) holds once the reference visits it: what `plane` recorded, or the verdict's.  A plane byte with a
// slope or step field was written by a visit under the plane's parameters, so it is complete; a byte without one (nothing
// recorded, or roughness_footprint alone after te_map_clear_footprint) takes the verdict.  A cell the isTraversableForFilters
// memo (may be null) holds as passing passed every check that ran: each writes 1 where its layer is 0, so the verdict needs no
// evaluation.  0 for a cell no check runs on.
__device__ __forceinline__ unsigned visit_code_d(const FpArgs& A, const Layers& L, const unsigned char* plane, const unsigned char* memo,
                                                 int a, int b) {
  const size_t c = (size_t)b * A.rows + a;
  const bool zs = __ldg(L.slope + c) == 0.0f, zt = __ldg(L.step + c) == 0.0f, zr = A.verify_rough && __ldg(L.rough + c) == 0.0f;
  if (!(zs || zt || zr)) return 0u;
  const unsigned code = plane[c];
  if (code & 0x0fu) return code;
  if (memo && memo[c] == 1) return code | (zs ? 2u : 0u) | (zt ? 8u : 0u) | (zr ? 32u : 0u);
  return code | verdict_code_d(filters_d(A, L, a, b));
}

// SpiralIterator::getCurrentRadius (index-space norm of the offset; Eigen's integer norm when int_norm is set) in metres.
__device__ __forceinline__ double current_radius_d(const FpArgs& A, int di, int dj) {
  const int d2 = di * di + dj * dj;
  const double nr = A.int_norm ? (double)(int)sqrt((double)d2) : sqrt((double)d2);
  return nr * A.res;
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

// Records in `plane` the cells at which isTraversable(center, rmax, cup, ..., rmin) on an empty cache calls
// isTraversableForFilters (TraversabilityMap.cpp:687-729), by the whole warp: the spiral with fresh_circle_d's membership, up to and
// including the first blocked cell.  With cup the loop does not return there (:714): it goes on past blocked cells within rmin and
// ends after the first blocked cell beyond rmin met while the circle is still traversable (:705-711).  `memo`: visit_code_d's.
// Warp-uniform.
__device__ void record_circle_d(const FpArgs& A, const Layers& L, const PathArgs& P, unsigned char* plane, const unsigned char* memo,
                                double cx, double cy, int ci, int cj, double rmin, double rmax, int nr, bool cup) {
  const int lane = threadIdx.x & 31;
  const double r2 = rmax * rmax;
  const int end = __ldg(P.ring_start + nr + 1), edge0 = __ldg(P.ring_start + max(nr - 1, 1));
  bool untrav = false;  // cup: a blocked cell within rmin has made the circle untraversable
  for (int base = 0; base < end; base += 32) {
    const int k = base + lane;
    bool member = false, within = true;
    unsigned code = 0u;
    int a = 0, b = 0;
    if (k < end) {
      const int w = __ldg(P.rings + k);
      const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
      a = ci + di;
      b = cj + dj;
      if (a >= 0 && b >= 0 && a < A.rows && b < A.cols_total) {
        member = true;
        if (k >= edge0) {
          const double dx = A.X[a] - cx, dy = A.Y[b] - cy;
          member = dx * dx + dy * dy <= r2;
        }
      }
      if (member) {
        code = visit_code_d(A, L, plane, memo, a, b);
        within = rmin == 0.0 || current_radius_d(A, di, dj) <= rmin;
      }
    }
    const bool blk = member && code_blocked_d(code);
    const unsigned bw = __ballot_sync(0xffffffffu, blk && within), bb = __ballot_sync(0xffffffffu, blk && !within);
    int last = 32;  // the last lane the walk visits
    if (!cup) {
      if (bw | bb) last = __ffs((int)(bw | bb)) - 1;
    } else if (!untrav && bb) {
      const int f = __ffs((int)bb) - 1;
      if (!(bw & ((1u << f) - 1u))) last = f;
    }
    if (code && lane <= last) plane[(size_t)b * A.rows + a] = (unsigned char)code;
    if (last < 32) return;
    untrav = untrav || bw != 0u;
  }
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

// Per-warp row table rows of the polygon kernels: the 2 * 127 + 1 rows of the largest spiral.
constexpr int kFreshTableRows = 2 * kPathMaxRings + 1;

// The layers of the map that starts `o` cells in (a null roughness layer stays null).
__device__ __forceinline__ Layers shift_layers_d(const Layers& L, long long o) {
  return Layers{L.trav + o, L.slope + o, L.step + o, L.elev + o, L.rough ? L.rough + o : nullptr};
}

}  // namespace
}  // namespace te
