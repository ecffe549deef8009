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
  DevBuf poly[2];  // run / uncertain-offset tables of the unrotated and the rotated footprint polygon
  bool poly_attr = false;
  DevBuf rings;   // fresh path checks: ring starts + SpiralIterator visit order of rings 0..127 (built once)
  DevBuf memo;    // fresh and polygonal path checks: per-cell isTraversableForFilters memo of one call
  DevBuf items;   // polygonal path checks: one result record per pose index
  DevBuf upoly;   // polygonal path checks with untraversable polygons: per pose index a vertex count and max_vertices points
  DevBuf mapbuf;  // map requests: circle keys, inclination segments, their records and hulls; then the cache cells to store
  void invalidate() { valid = false; tables_valid = false; }
  void release();
};

int footprint_halo(const te_geometry* g, const te_footprint_params* p);

int launch_footprint(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                     const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                     float* step_fp, float* rough_fp, int sms, cudaStream_t s, int* launches);

// TraversabilityMap::traversabilityFootprint(double footprintYaw) (TraversabilityMap.cpp:239-305): layers traversability_x / _rot.
int footprint_polygon_halo(const te_geometry* g, const te_footprint_params* p, int npts, const double* pts_xy);
int launch_footprint_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int npts,
                             const double* pts_xy, double yaw, const float* trav, const float* slope, const float* step,
                             const float* rough, const float* elev, float* out_x, float* out_rot, int sms, cudaStream_t s, int* launches);

// TraversabilityMap::checkCircularFootprintPath for a batch of paths on a complete traversability_footprint layer (device pointers).
void launch_check_paths(const SlabView& v, const te_geometry* g, double traversability_default, const float* footprint, const float* robot_slope, int npaths,
                        const int* path_begin, const double* xy, unsigned char* is_safe, double* trav, cudaStream_t s);

// The same on the chain layers with an empty traversability_footprint cache per path (te_check_footprint_paths_fresh); whole map,
// device pointers, radius / compute_untraversable_polygon per path.  Asynchronous on `s`.  `ucount` != nullptr: also the
// untraversable polygon of every path (vertex count, up to `max_vertices` points in `uxy`; te_check_footprint_paths_fresh2).
int launch_check_paths_fresh(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                             const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                             int npaths, const int* path_begin, const double* xy, const double* radius, const unsigned char* cup,
                             unsigned char* is_safe, double* trav_out, int max_vertices, int* ucount, double* uxy, cudaStream_t s);

// TraversabilityMap::checkPolygonalFootprintPath for a batch of paths sharing one footprint (te_check_footprint_paths_polygon);
// whole map, device pointers except `footprint_xyz` (host, nfp x 3 floats).  `max_points` bounds the hull input of one item
// (polygon1 ++ polygon2): 2 * nfp without conservative paths, 2 * nfp * (poses of the longest conservative path) otherwise.
constexpr int kPolyMaxVerts = 16;   // footprint vertices
constexpr int kPolyConsCap = 1024;  // vertices of a conservative path's polygon2 (nfp * poses up to the segment)
// `ucount` != nullptr: also the untraversable polygon of every path with cup[q] set (te_check_footprint_paths_polygon2); an item
// whose bounding box spans more than kUntravRows map rows cannot build it (shared-memory row table): its path gets count -1.
constexpr int kUntravRows = 1024;
int launch_check_paths_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                               const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                               int nfp, const float* footprint_xyz, int npaths, int nposes, const int* path_begin, const double* poses,
                               const unsigned char* conservative, int max_points, unsigned char* is_safe, double* trav_out,
                               double* area_out, const unsigned char* cup, int max_vertices, int* ucount, double* uxy,
                               cudaStream_t s, int* launches);

// A whole check_footprint_path request (te_check_footprint_request): the two checks above on one predicate memo, each path with its
// own footprint (footprint_begin / footprint_xyz, device pointers): none is circular (radius[q]), 1..max_footprint_vertices vertices
// polygonal.  Poses are 7 doubles for both kinds.  `max_points` bounds the hull input of a polygonal item as in
// launch_check_paths_polygon, for the largest footprint.  Three launches (two without poses), whatever the footprints.
int launch_check_request(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                         const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                         int npaths, int nposes, const int* path_begin, const double* poses, const double* radius, int nvertices,
                         const int* footprint_begin, const float* footprint_xyz, int max_footprint_vertices,
                         const unsigned char* conservative, const unsigned char* cup, int max_points, unsigned char* is_safe,
                         double* trav_out, double* area_out, int max_vertices, int* ucount, double* uxy, cudaStream_t s,
                         int* launches);

// A request on a te_map (te_map_check_footprint_request).  Its polygonal paths: the polygonal half of launch_check_request on the
// memo in st.memo, which the caller keeps (device pointers).  Its circular paths: launch_map_circles reads and fills the
// traversability_footprint cache `cache` (device, NaN = empty) in the reference's order; every path array and output is in HOST
// memory, hX / hY are the host copies of the cell-centre tables, and the call returns synchronised.
int launch_map_polygons(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const float* trav,
                        const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                        int npaths, int nposes, const int* path_begin, const double* poses, int nvertices, const int* footprint_begin,
                        const float* footprint_xyz, int max_footprint_vertices, const unsigned char* conservative,
                        const unsigned char* cup, int max_points, unsigned char* is_safe, double* trav_out, double* area_out,
                        int max_vertices, int* ucount, double* uxy, cudaStream_t s, int* launches);
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
