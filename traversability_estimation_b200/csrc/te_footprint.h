// te_footprint.h — host interface of the footprint sweep (te_footprint.cu).
#pragma once
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include "../../include/te_b200.h"
#include "te_device.cuh"
#include "te_grid.cuh"
#include "te_kernels.h"

namespace te {

struct FootprintState {
  std::string why;
  bool valid = false;
  te_geometry key_geo{};
  te_footprint_params key_par{};
  DevBuf spiral;  // packed (di,dj) of the SpiralIterator visit order
  int n_spiral = 0;
  DevBuf block;   // per-cell predicate bytes for the slab + halo
  // prefix-sum sweep: half-width / ring tables (depend on radius and resolution) and per-call prefix sums + bit columns
  DevBuf tables;
  bool tables_valid = false;
  size_t off_ring = 0, off_fuzzy = 0, off_halfw = 0, off_inner = 0;
  int n_fuzzy = 0, L = 0, nrings = 0;
  signed char h_halfw[64] = {0};
  DevBuf prefix;  // per input-buffer column: prefix sums of t', packed blocked flags, nearest-blocked bytes (k_sweep_fast)
  DevBuf list;    // work list of the cells whose predicates need the window / gap-walk code (word 0: length)
  DevBuf poly;    // polygon sweep: per-polygon descriptors, then the run / uncertain-offset tables of every polygon of the call
  bool poly_attr = false;
  DevBuf reduce;  // polygon sweep in reduce mode with yaw groups: every group's partial worst / best / best_yaw of every cell
  DevBuf rings;   // fresh path checks: ring starts + SpiralIterator visit order of rings 0..127 (built once)
  DevBuf memo;    // fresh and polygonal path checks: per-cell isTraversableForFilters memo of one call
  DevBuf items;   // polygonal path checks: one result record per pose index
  DevBuf upoly;   // polygonal path checks with untraversable polygons: per pose index a vertex count and max_vertices points
  DevBuf mapbuf;  // map requests: circle keys, inclination segments, their records and hulls; then the cache cells to store
  void invalidate() { valid = false; tables_valid = false; }
  void release();
};

int footprint_halo(const te_geometry* g, const te_footprint_params* p);

// The sweeps run on `nmaps` (1 .. 65535) maps of the slab's shape stored back to back: map m's layers start m * rows * in_ncols
// cells into every input, its outputs m * rows * out_ncols cells into every output.  The tables are built once per call.
int launch_footprint(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                     const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                     float* step_fp, float* rough_fp, int sms, cudaStream_t s, int* launches);

// TraversabilityMap::traversabilityFootprint(double footprintYaw) (TraversabilityMap.cpp:239-305): the footprint polygon placed at
// every cell centre, rotated by `yaw` (yaw 0: the unrotated traversability_x), into `out` (device; map m's layer starts
// m * rows * out_ncols cells into it).  One call sweeps a list of such layers: the predicates run once, then ONE k_poly_tile launch
// sweeps every layer; each layer equals, bit for bit, what a call with that layer alone gives.
struct PolygonLayer {
  double yaw;
  float* out;
};
// Reduce mode: instead of one layer per polygon, per cell the value of the first polygon that minimises it (worst), of the first
// that maximises it (best) and that polygon's index in `polys` (best_yaw); each null when not wanted, not all three.  Device
// pointers laid out as a layer; the polygons' `out` is unused.  Needs a finite traversability_default.  The reduction runs in the
// sweep; when the launch splits the polygons into yaw groups, the groups' partial results go to st.reduce and one more kernel
// folds them.
struct PolygonReduce {
  float* worst;
  float* best;
  int* best_yaw;
};
int footprint_polygon_halo(const te_geometry* g, const te_footprint_params* p, int npts, const double* pts_xy);
int launch_footprint_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int npts,
                             const double* pts_xy, int npoly, const PolygonLayer* polys, const PolygonReduce* reduce, const float* trav,
                             const float* slope, const float* step, const float* rough, const float* elev, int nmaps, int sms,
                             cudaStream_t s, int* launches);

// TraversabilityMap::checkCircularFootprintPath for a batch of paths on a complete traversability_footprint layer (device pointers).
void launch_check_paths(const SlabView& v, const te_geometry* g, double traversability_default, const float* footprint, const float* robot_slope, int npaths,
                        const int* path_begin, const double* xy, unsigned char* is_safe, double* trav, cudaStream_t s);

// Checks of footprint paths on the chain layers with an empty traversability_footprint cache per path: circular paths as
// TraversabilityMap::checkCircularFootprintPath (te_check_footprint_paths_fresh2), polygonal paths as checkPolygonalFootprintPath
// (te_check_footprint_paths_polygon2), or both mixed in one request (te_check_footprint_request).  Whole map; device pointers
// except `footprint`.
constexpr int kPolyMaxVerts = 16;   // footprint vertices
constexpr int kPolyConsCap = 1024;  // vertices of a conservative path's polygon2 (nfp * poses up to the segment)
// An item of a polygonal path whose bounding box spans more than kUntravRows map rows cannot build its untraversable polygon
// (shared-memory row table): its path gets count -1.
constexpr int kUntravRows = 1024;
struct PathChecks {
  const float *trav, *slope, *step, *rough, *elev;  // isTraversableForFilters' layers; rough null unless verify_roughness
  const float* robot_slope;                          // null: no checkRobotInclination
  // A batch of maps of one geometry (te_check_footprint_request_batched): map m's cells start m * rows * cols cells into every
  // layer and into the memo (nmaps maps' worth, cleared once), and path q is on map path_map[q] (device memory; null: every path
  // is on map 0).  A path on a map outside 0 .. nmaps-1 is not checked.
  int nmaps;
  const int* path_map;
  int npaths;
  int nposes;                     // poses in `poses`; < 0: not known (circular paths then need no pose range check)
  const int* path_begin;          // [npaths + 1]
  const double* poses;            // pose_stride doubles per pose: x y, or x y z qx qy qz qw (polygonal paths need 7)
  int pose_stride;
  const double* radius;           // per path; read for circular paths only
  // Per-path footprints: path q has vertices footprint_begin[q] .. footprint_begin[q+1]-1 of footprint_xyz (3 floats each), none
  // for a circular path, 1..max_footprint_vertices for a polygonal one.  Without footprint_begin every path is circular, unless
  // `footprint` (HOST memory, nfp x 3 floats) is the one footprint all paths share.
  const int* footprint_begin;
  const float* footprint_xyz;
  int nvertices, max_footprint_vertices;
  int nfp;
  const float* footprint;
  const unsigned char* conservative;  // per path, may be null
  const unsigned char* cup;           // compute_untraversable_polygon per path, may be null
  // Hull input points of one polygonal item (polygon1 ++ polygon2): 2 * nfp without conservative paths, 2 * nfp * (poses of the
  // longest conservative path) otherwise, for the largest footprint.
  int max_points;
  unsigned char* is_safe;
  double* trav_out;
  double* area_out;                   // may be null when every path is circular
  int max_vertices;
  int* ucount;                        // null: no untraversable polygons; else per path a vertex count and max_vertices points in uxy
  double* uxy;
};
// Asynchronous on `s`.  Launches one kernel for the circular paths (when `r` can have any and `circular` is set; a te_map checks
// them on its cache instead), then for the polygonal paths an items kernel when there are poses and a combine kernel, whatever the
// footprints.  `clear_memo`: start from an empty isTraversableForFilters memo (st.memo); otherwise the caller keeps st.memo valid
// for these layers (a te_map).
int launch_path_checks(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const PathChecks& r,
                       bool circular, bool clear_memo, cudaStream_t s, int* launches);

// A request on a te_map (te_map_check_footprint_request): its polygonal paths run launch_path_checks on the memo the map keeps.
// Its circular paths: launch_map_circles reads and fills the traversability_footprint cache `cache` (device, NaN = empty) in the
// reference's order; every path array and output is in HOST memory, hX / hY are the host copies of the cell-centre tables, and
// the call returns synchronised.
struct MapRequestStats {
  long long candidates = 0;  // isTraversable calls the circular paths could make
  long long keys = 0;        // distinct circles among them (what k_map_eval_circles evaluates)
  long long stored = 0;      // cache cells the request stored
};
int launch_map_circles(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                       const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                       float* cache, const double* hX, const double* hY, int npaths, const int* path_begin, const double* poses,
                       const double* radius, const int* footprint_begin, const unsigned char* cup, unsigned char* is_safe,
                       double* trav_out, double* area_out, int max_vertices, int* ucount, double* uxy, cudaStream_t s, int* launches,
                       MapRequestStats* stats);
// traversabilityFootprint(radius, offset) on a cache: cache = finite(cache) ? cache : fresh over n cells; `out` (device, may be
// null) receives the result too.
int launch_map_merge(const float* fresh, float* cache, float* out, size_t n, int sms, cudaStream_t s);

}  // namespace te
