// te_footprint.h — host interface of the footprint sweeps (te_footprint.cu, te_footprint_polygon.cu), the footprint path checks
// (te_paths.cu) and the te_map footprint cache (te_map_request.cu).
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
  double tables_ulp = 0.0;  // coord_ulp of the coordinates the tables' tolerance was sized for
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
  DevBuf codes;   // te_map sweeps: the predicates' recorded-layer code of every cell, then one flag per map (SweepRecord)
  DevBuf devreq;  // map requests: the work list, its keys and records, the hash table and the scan / sort scratch
  const unsigned long long* req_counters = nullptr;  // in devreq: candidates, keys, stored of the last map request
  void invalidate() { valid = false; tables_valid = false; }
  void release();
};

int footprint_halo(const te_geometry* g, const te_footprint_params* p);
// Whether launch_footprint takes p's circle at this resolution: radius + offset within 120 cells (TE_ERR_UNSUPPORTED otherwise).
bool footprint_reach_ok(double resolution, const te_footprint_params* p);

// The parameters a request reads per map when the maps of a te_map batch have robots of their own (te_map_check_footprint_request
// _each / _device_each): the circle walk's offset and traversability_default, SpiralIterator's radius flag and the
// isTraversableForFilters parameters, each as filter_args / path_args take it from a te_footprint_params.  A device table of one
// entry per map (FpArgs::mp); the radius is a path's own, so it is not here.
struct FpMapParams {
  double offset, tdefault, maxgap, crit;
  int int_norm, verify_rough;
};

// The sweeps run on `nmaps` (1 .. 65535) maps of the slab's shape stored back to back: map m's layers start m * rows * in_ncols
// cells into every input, its outputs m * rows * out_ncols cells into every output.  The tables are built once per call.
// rec (a te_map, null otherwise): the sweep also records in rec->plane the cells at which traversabilityFootprint(radius, offset)
// calls isTraversableForFilters on the cache rec->cache as the sweep found it: the spiral prefix of every empty centre.  Map k of the
// launch is map slot[k] (slot: device, nmaps entries; null: k) of the plane and the cache, whole maps of v.rows * v.cols_total cells.
// The empty centres alone are the record while every cached cell of a map is recorded; walk (HOST, nmaps entries; null: none)
// marks the maps where that need not hold, whose empty centres then walk their spirals (one launch more, and a host synchronisation
// the first time a state walks).
struct SweepRecord {
  unsigned char* plane;
  const float* cache;
  const int* slot;
  const unsigned char* walk;
};
int launch_footprint(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int nmaps, const float* trav,
                     const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                     float* step_fp, float* rough_fp, int sms, cudaStream_t s, int* launches, const SweepRecord* rec = nullptr);

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
// Per-map polygons (te_map_footprint_polygon_keep): map k of the launch sweeps two layers, polys[0] (yaw 0: traversability_x) and
// polys[poly_of[k]] (its own yaw: traversability_rot), each into its polygon's `out` at map slot[k] instead of k.  poly_of: a
// host array of nmaps entries in 1 .. npoly-1; slot: a device table of nmaps map slots, or null (slot k is k).  Maps at their own
// positions (v.pos) read their own coordinate tables.  One sweep launch whatever the maps, yaws and positions; each layer equals,
// bit for bit, what a call with that map and yaw alone gives.  No reduction.
struct PolygonMaps {
  const int* poly_of;
  const int* slot;
};
int footprint_polygon_halo(const te_geometry* g, const te_footprint_params* p, int npts, const double* pts_xy);
int launch_footprint_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int npts,
                             const double* pts_xy, int npoly, const PolygonLayer* polys, const PolygonReduce* reduce,
                             const PolygonMaps* maps, const float* trav, const float* slope, const float* step, const float* rough,
                             const float* elev, int nmaps, int sms, cudaStream_t s, int* launches);

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
  // A te_map batch whose maps have parameters of their own: device table of nmaps entries; null: the call's one parameter set
  // for every map.  Read by launch_map_request_device and by launch_path_checks' polygonal kernels.
  const FpMapParams* map_params;
  // A te_map's recorded slope_footprint / step_footprint / roughness_footprint (te_fp_device.cuh: one byte per cell of every map,
  // like the memo), or null.  Set: the request also records the cells at which the service loop calls isTraversableForFilters
  // (launch_map_request_device: the walks the replay commits; launch_path_checks: the polygonal items the path loop reaches).
  unsigned char* plane;
};
// Asynchronous on `s`.  Launches one kernel for the circular paths (when `r` can have any and `circular` is set; a te_map checks
// them on its cache instead), then for the polygonal paths an items kernel when there are poses and a combine kernel, whatever the
// footprints.  `clear_memo`: start from an empty isTraversableForFilters memo (st.memo); otherwise the caller keeps st.memo valid
// for these layers (a te_map).
int launch_path_checks(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, const PathChecks& r,
                       bool circular, bool clear_memo, cudaStream_t s, int* launches);

// A request on a te_map (te_map_check_footprint_request(_batched, _device)): its polygonal paths run launch_path_checks on the
// memo the map keeps.  Its circular paths: launch_map_request_device reads and fills the traversability_footprint cache `cache`
// (device, NaN = empty) in the reference's order.  It takes the layers, the map batch, the path arrays and the outputs from `r`,
// every array in DEVICE memory (a host request stages them; poses of 7 doubles, footprint_begin set), and is asynchronous on `s`,
// without a host synchronisation.  A batch of r.nmaps maps: the layers, robot_slope, the cache and the memo hold map m from
// m * rows * cols cells on, and path q is on map r.path_map[q] (path_map null: one map).  A path the kernels cannot check
// (radius, rings, pose range, non-finite position unless `nonfinite_ok`, map outside the batch), and every circular path from
// the first whose work-list entries end past `max_checks` on, gets is_safe 0, NaN traversability and area and count -1 where its
// polygon was requested, and reads and stores nothing.  `nonfinite_ok` (host memory, where the request was validated): a
// non-finite x or y is answered as the service loop answers it, a single pose there as outside the map and a segment with such an
// end as a failed check without a polygon.  The workspace (st.devreq) is sized from npaths, nposes, nmaps and max_checks; the
// request's counters stay on the device at st.req_counters.  Launches: 12 (nine kernels, three CUB calls counted as one each),
// and one more with polygons (r.ucount), whatever the paths and maps.  Every call clears a hash table of 2 * max_checks slots
// (rounded up to a power of two; 8 bytes per entry of max_checks).
struct MapRequestStats {
  long long candidates = 0;  // isTraversable calls the circular paths could make
  long long keys = 0;        // distinct circles among them (what k_map_eval_circles_dev evaluates)
  long long stored = 0;      // cache cells the request stored
};
int launch_map_request_device(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p,
                              const PathChecks& r, float* cache, long long max_checks, bool nonfinite_ok, int sms, cudaStream_t s,
                              int* launches);
// traversabilityFootprint(radius, offset) on a cache: cache = finite(cache) ? cache : fresh over nsel blocks of n cells; `out`
// (device, may be null) receives the result too.  Block j of `fresh` and `out` starts at j * n, its cache block at slot[j] * n
// (slot: a device table of nsel map slots; null: j * n, the whole batch as nsel = 1 block of every cell).  One launch.
int launch_map_merge(const float* fresh, float* cache, float* out, size_t n, const int* slot, int nsel, int sms, cudaStream_t s);

// Selected maps of a te_map (te_map_chain_maps, te_map_set_layers_maps, te_map_footprint_maps, te_map_carry_layers): packed map j
// is at j * cells in scratch, its resident copy at slot[j] * cells in the te_map's layers, cache and memo.  Up to kMapSlotLayers
// layers move in one launch; a layer with a null dst is skipped.  put: packed src -> resident dst, the maps' cache slots become
// NaN (empty; cache may be null) and their memo slots 0 (memo may be null), and their slots of every non-null fill layer take the
// bits fill_bits; otherwise resident src -> packed dst (cache, memo and fill unused).  A null slot table is the identity (slot[j]
// = j: every map of the te_map when nsel = nmaps).  Grid-stride over maps and cells, 16-byte accesses when cells % 4 == 0 and
// every pointer is 16-byte aligned.  One launch, whatever nsel and the layers.
constexpr int kMapSlotLayers = 8;
struct MapSlots {
  const float* src[kMapSlotLayers];
  float* dst[kMapSlotLayers];
  float* fill[kMapSlotLayers];
  unsigned fill_bits;
  float* cache;
  unsigned char* memo;
  const int* slot;  // device, nsel entries, or null
  int nsel;
  size_t cells;     // per map
};
void launch_map_slots(const MapSlots& a, bool put, int sms, cudaStream_t s);

// A te_map's recorded slope_footprint / step_footprint / roughness_footprint bytes (te_fp_device.cuh), n cells: clear the first two
// (te_map_clear_footprint), or decode layer `field` (0, 1, 2 in that order) into floats.  One launch each.
void launch_plane_clear(unsigned char* plane, size_t n, int sms, cudaStream_t s);
void launch_plane_decode(const unsigned char* plane, int field, float* out, size_t n, int sms, cudaStream_t s);

}  // namespace te
