// te_paths.cu — the stateless footprint path checks: TraversabilityMap::checkCircularFootprintPath on a complete
// traversability_footprint layer (k_check_paths) or on an empty one per path (k_check_paths_fresh, _poly), and
// checkPolygonalFootprintPath (k_check_polygon_items, k_check_polygon_combine, _poly), alone or mixed in one request
// (launch_path_checks).  A te_map's circular paths share one cache instead and run in te_map_request.cu; both walk the circle
// with fresh_circle_d (te_fp_device.cuh).  Compiled with --fmad=false: the checks replay the reference's double arithmetic.
#include "te_fp_device.cuh"
#include "te_pose.cuh"

#include <algorithm>
#include <cmath>

namespace te {
namespace {

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

// Footprint vertex v placed at the pose T (te_pose.cuh).  The vertex comes from the path's own footprint `fxyz` in global memory, or
// without one from the kernel parameters.
__device__ __forceinline__ double2 footprint_vertex_d(const PolyPathArgs& P, const float* fxyz, const PoseRT& T, int v) {
  double vx, vy, vz;
  if (fxyz) {
    vx = (double)fxyz[3 * v]; vy = (double)fxyz[3 * v + 1]; vz = (double)fxyz[3 * v + 2];
  } else {
    vx = (double)P.fx[v]; vy = (double)P.fy[v]; vz = (double)P.fz[v];
  }
  return pose_point_d(T, vx, vy, vz);
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
// (R.fp_begin) each polygonal path uses its own, and the poses of circular paths are no items.  AT: the maps sit at their own
// positions (FpArgs::pos), and the item takes its path's map's tables and position.  Maps with parameters of their own
// (FpArgs::mp): the item takes its path's map's.
// REC (k_check_polygon_items_rec, after the items and combine kernels): no outputs; an item the path loop reaches (every earlier
// item of its checkable path traversable, its own checkInclination passed) records in `plane` the cells its isTraversable visits:
// the PolygonIterator prefix up to and including the first blocked cell, or the whole polygon with compute_untraversable_polygon
// (:601-611).
template <bool POLY, bool AT, bool EACH, bool REC = false>
__device__ __forceinline__ void check_polygon_item_d(const FpArgs& A0, Layers L, const PolyPathArgs& P, const PolyUntravArgs& U,
                                                     const RequestArgs& R, unsigned char* plane = nullptr) {
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
    if (lane == 0 && !REC) P.items[p] = it;
    return;
  }
  if constexpr (REC) {  // the path loop reaches item k: its path is checkable and items k0 .. k-1 are traversable
    bool reach = true;
    for (int j = (n == 1 ? 0 : 1) + lane; j < n; j += 32) {
      const PolyItem o = P.items[b + j];
      reach = reach && o.q == q && o.flag != 2 && (j >= k || o.flag == 1);
    }
    if (!__all_sync(0xffffffffu, reach)) return;
    plane += mo;
  }
  L = shift_layers_d(L, mo);  // path q's map
  FpArgs Am;
  if constexpr (AT || EACH) Am = map_view_d<AT, EACH>(A0, R.path_map ? R.path_map[q] : 0);
  const FpArgs& A = AT || EACH ? Am : A0;
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
      if (lane == 0 && !REC) P.items[p] = it;  // flag 2
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
    if (lane == 0 && !REC) P.items[p] = it;  // flag 2
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
    if constexpr (REC) {
      const bool all = U.cup != nullptr && U.cup[q] != 0;
      for (long long base = 0; base < total; base += 32) {
        const long long c = base + lane;
        unsigned code = 0u;
        int a = 0, bb = 0;
        if (c < total) {
          a = si + (int)(c / nc);
          bb = sj + (int)(c % nc);
          if (a >= 0 && bb >= 0 && a < A.rows && bb < A.cols_total && polygon_inside_d(sA, nh, A.X[a], A.Y[bb]))
            code = visit_code_d(A, L, plane, memo, a, bb);
        }
        const unsigned bm = all ? 0u : __ballot_sync(0xffffffffu, code_blocked_d(code));
        if (code && (!bm || lane < __ffs((int)bm))) plane[(size_t)bb * A.rows + a] = (unsigned char)code;
        if (bm) break;
      }
      return;
    }
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
  if constexpr (REC) return;
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

template <bool AT, bool EACH>
__global__ void __launch_bounds__(128) k_check_polygon_items(FpArgs A, Layers L, PolyPathArgs P, RequestArgs R) {
  check_polygon_item_d<false, AT, EACH>(A, L, P, PolyUntravArgs{}, R);
}

template <bool AT, bool EACH>
__global__ void __launch_bounds__(128) k_check_polygon_items_rec(FpArgs A, Layers L, PolyPathArgs P, PolyUntravArgs U, RequestArgs R,
                                                                 unsigned char* plane) {
  check_polygon_item_d<false, AT, EACH, true>(A, L, P, U, R, plane);
}

template <bool AT, bool EACH>
__global__ void __launch_bounds__(128) k_check_polygon_items_poly(FpArgs A, Layers L, PolyPathArgs P, PolyUntravArgs U, RequestArgs R) {
  check_polygon_item_d<true, AT, EACH>(A, L, P, U, R);
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

}  // namespace

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

void launch_check_paths(const SlabView& v, const te_geometry* g, double traversability_default, const float* footprint, const float* robot_slope, int npaths,
                        const int* path_begin, const double* xy, unsigned char* is_safe, double* trav, cudaStream_t s) {
  FpArgs a = geometry_args(v, g);
  a.tdefault = traversability_default;
  k_check_paths<<<(npaths + 127) / 128, 128, 0, s>>>(a, footprint, robot_slope, npaths, path_begin, xy, is_safe, trav);
}

namespace {
// The per-call isTraversableForFilters memo of the path checks (blocked_memo_d): one byte per map cell of each of `nmaps` maps,
// cleared on `s`.
int reset_filter_memo(FootprintState& st, const SlabView& v, int nmaps, cudaStream_t s) {
  const size_t ncell = (size_t)v.rows * v.cols_total * nmaps;
  if (st.memo.reserve(ncell) != cudaSuccess) { st.why = "allocating the predicate memo failed"; return TE_ERR_CUDA; }
  if (cudaMemsetAsync(st.memo.p, 0, ncell, s) != cudaSuccess) { st.why = "cudaMemsetAsync(predicate memo) failed"; return TE_ERR_CUDA; }
  return 0;
}
}  // namespace

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

namespace {
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
  FpArgs a = filter_args(v, g, p, r.rough);
  a.mp = r.map_params;  // a te_map batch whose maps have parameters of their own: read by the polygonal items only
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
  // maps at their own positions (a te_map): the instantiations that read each path's map's tables; maps with parameters of their
  // own: those that read each path's map's
  const bool at = a.pos != nullptr, each = a.mp != nullptr;
  int rc = 0;
  if (!r.ucount) {
    rc = launch_polygon_kernels(st,
                                at ? (each ? k_check_polygon_items<true, true> : k_check_polygon_items<true, false>)
                                   : (each ? k_check_polygon_items<false, true> : k_check_polygon_items<false, false>),
                                k_check_polygon_combine, "k_check_polygon_items", false, a, L, P, s, launches, R);
  } else {
    const size_t cbytes = (sizeof(int) * nitems + 15) / 16 * 16;
    if (st.upoly.reserve(cbytes + sizeof(double2) * nitems * (size_t)std::max(r.max_vertices, 1)) != cudaSuccess) {
      st.why = "allocating the untraversable polygons failed";
      return TE_ERR_CUDA;
    }
    const PolyUntravArgs U{r.cup, (int*)st.upoly.p, (double*)((char*)st.upoly.p + cbytes), UntravOut{r.max_vertices, r.ucount, r.uxy}};
    rc = launch_polygon_kernels(st,
                                at ? (each ? k_check_polygon_items_poly<true, true> : k_check_polygon_items_poly<true, false>)
                                   : (each ? k_check_polygon_items_poly<false, true> : k_check_polygon_items_poly<false, false>),
                                k_check_polygon_combine_poly, "k_check_polygon_items_poly", true, a, L, P, s, launches, U, R);
  }
  if (rc || !r.plane || P.nposes <= 0) return rc;
  // a te_map's recorded layers: the items the path loop reaches walk their polygons again, reading the items of the first pass
  const auto rec = at ? (each ? k_check_polygon_items_rec<true, true> : k_check_polygon_items_rec<true, false>)
                      : (each ? k_check_polygon_items_rec<false, true> : k_check_polygon_items_rec<false, false>);
  const size_t per_warp = poly_warp_smem(P.mcap, false);
  const int wpb = per_warp * 4 <= 48 * 1024 ? 4 : 1;
  if (per_warp * wpb > 48 * 1024 &&
      cudaFuncSetAttribute(rec, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(per_warp * wpb)) != cudaSuccess) {
    st.why = "cudaFuncSetAttribute(k_check_polygon_items_rec) failed";
    return TE_ERR_CUDA;
  }
  const PolyUntravArgs U{r.cup, nullptr, nullptr, UntravOut{}};
  rec<<<(unsigned)(((long long)P.nposes + wpb - 1) / wpb), 32 * wpb, per_warp * wpb, s>>>(a, L, P, U, R, r.plane);
  ++*launches;
  return 0;
}

}  // namespace te
