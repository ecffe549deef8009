/*
 * te_b200.h — C ABI of the H100-native (sm_90a) traversability filter chain and footprint sweep.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  Each entry point
 * names the reference interface it replaces (path:line relative to the reference repository
 * leggedrobotics/traversability_estimation).  The reference-side binding a maintainer would add
 * (the filters::FilterBase<grid_map::GridMap> plugin shells) is in
 * traversability_estimation_b200/plugin/ and described in INTEGRATION.md.
 *
 * Layers are float32, column-major exactly like grid_map::Matrix (Eigen::MatrixXf):
 * value(i, j) = data[j * rows + i]; NaN/Inf = invalid cell (GridMap::isValid == std::isfinite).
 *
 * Every function returns TE_OK (0) or a negative te_status; it never throws.  The message of the
 * last failure on the calling thread is available from te_last_error().  There is NO CPU fallback:
 * without a CUDA device every compute entry point fails with TE_ERR_CUDA.
 */
#ifndef TE_B200_H
#define TE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TE_B200_ABI_VERSION 1

typedef enum te_status {
  TE_OK = 0,
  TE_ERR_BAD_ARG = -1,       /* null pointer, non-positive size, invalid parameter value */
  TE_ERR_MISSING_LAYER = -2, /* a required input layer pointer is null (reference: GridMap::at throws) */
  TE_ERR_CUDA = -3,          /* CUDA runtime/driver failure, or no device */
  TE_ERR_UNSUPPORTED = -4,   /* e.g. non-zero circular-buffer start index */
  TE_ERR_NCCL = -5           /* reserved (the halo exchange of this library is peer-mapped, see te_halo_pull) */
} te_status;

/* Where the layer pointers passed to a call live. */
typedef enum te_memory { TE_MEM_HOST = 0, TE_MEM_DEVICE = 1 } te_memory;

/* grid_map::GridMap geometry, doubles exactly as the container holds them; needed bit-for-bit
 * because CircleIterator decides window membership on absolute double positions.
 * (grid_map_core GridMap::getSize/getResolution/getLength/getPosition/getStartIndex) */
typedef struct te_geometry {
  int32_t rows, cols;
  double resolution;
  double length_x, length_y;
  double position_x, position_y;
  int32_t start_row, start_col; /* grid_map circular-buffer start index (GridMap::getStartIndex): cell (i, j) is stored at buffer
                                   index ((i + start_row) % rows, (j + start_col) % cols).  te_chain, te_footprint(2) and
                                   te_footprint_polygon with TE_MEM_HOST on a whole map (no slab) take and return layers in
                                   that order (the copies to and from the device unwrap / re-wrap); everything else wants 0
                                   (TE_ERR_UNSUPPORTED otherwise: convertToDefaultStartIndex) */
} te_geometry;

/* Column slab of a larger map (multi-GPU tiling, one slab per rank).  Inputs cover columns
 * [col_begin - halo_left, col_begin + col_count + halo_right) of the global map; outputs cover
 * [col_begin, col_begin + col_count).  Columns outside the global map need not exist.
 * Pass NULL for "the whole map". */
typedef struct te_slab {
  int32_t col_begin, col_count;
  int32_t halo_left, halo_right;
} te_slab;

enum { TE_NORMALS_FIXTURE = 0, TE_NORMALS_RAW_MOMENT = 1 };

/* Parameters of the YAML chain (traversability_estimation/config/robot_filter_parameter.yaml:2-37);
 * names follow the filters' own parameter names. */
typedef struct te_chain_params {
  double normals_radius;          /* NormalVectorsFilter `radius` (:8) */
  int32_t normals_algorithm;      /* TE_NORMALS_* */
  int32_t normals_positive_axis;  /* `normal_vector_positive_axis` 0=x 1=y 2=z (:9) */
  double slope_critical;          /* SlopeFilter `critical_value` (:14), SlopeFilter.cpp:36-46 */
  double step_critical;           /* StepFilter `critical_value` (:18), StepFilter.cpp:40-50 */
  double step_first_radius;       /* `first_window_radius` (:19) */
  double step_second_radius;      /* `second_window_radius` (:20) */
  int32_t step_critical_cells;    /* `critical_cell_number` (:21) */
  int32_t reserved0;
  double roughness_critical;      /* RoughnessFilter `critical_value` (:26), RoughnessFilter.cpp:38-48 */
  double roughness_radius;        /* `estimation_radius` (:27) */
  float fuse_weight;              /* MathExpressionFilter (:29-33): weight*((slope+step)+roughness) in float32 */
  int32_t reserved1;
} te_chain_params;

/* TraversabilityMap::traversabilityFootprint(radius, offset) and the members it reads. */
typedef struct te_footprint_params {
  double radius;                  /* = radiusMin; TraversabilityMap.cpp:313 */
  double offset;                  /* radiusMax = radius + offset */
  double traversability_default;  /* traversabilityDefault_ (robot_footprint_parameter.yaml:8) */
  double max_gap_width;           /* maxGapWidth_ (robot.yaml:10) */
  double critical_step_height;    /* criticalStepHeight_ (TraversabilityMap.cpp:117-126) */
  int32_t radius_is_integer_norm; /* SpiralIterator::getCurrentRadius via Eigen integer norm (1) or exact (0) */
  int32_t verify_roughness;       /* checkForRoughness_ (robot_footprint_parameter.yaml:9 `verify_roughness_footprint`):
                                     isTraversableForFilters also runs checkForRoughness (TraversabilityMap.cpp:779-783, 895-921);
                                     needs the traversability_roughness layer, i.e. te_footprint2 */
} te_footprint_params;

/* Which implementation te_chain uses. AUTO picks the fused stencil when the window shapes have a
 * specialised instantiation, else the generic kernel; both compute the same layers. */
typedef enum te_kernel { TE_KERNEL_AUTO = 0, TE_KERNEL_GENERIC = 1, TE_KERNEL_FUSED = 2 } te_kernel;

typedef struct te_ctx te_ctx;

/* Lifetime: one context per plugin instance / per rank.  Owns a non-blocking CUDA stream, the
 * per-geometry position tables and staging buffers.  Thread-safe: one in-flight call per context. */
int te_create(te_ctx** out, int device);
int te_destroy(te_ctx* ctx);
const char* te_last_error(void);
int te_abi_version(void);

/* Page-locked host memory for layers handed to TE_MEM_HOST calls (cudaHostAlloc): pageable layers work too, but their
 * transfers are staged by the driver at roughly half the PCIe rate.  The plugin shells keep their cached layers here. */
int te_host_alloc(void** out, size_t bytes);
int te_host_free(void* p);

/* Run subsequent calls on an external stream (cudaStream_t passed as void*; NULL restores the
 * context's own stream).  Device-memory calls are asynchronous on that stream; te_synchronize waits. */
int te_set_stream(te_ctx* ctx, void* cuda_stream);
int te_synchronize(te_ctx* ctx);
int te_set_kernel(te_ctx* ctx, int te_kernel_choice);
/* Counters since creation: kernels launched, cells that took the certified slow path in the fused kernel. */
int te_get_stats(te_ctx* ctx, int64_t* kernel_launches, int64_t* slow_path_cells);

/* Device-side timing of the kernels this context launches (CUDA events on the launching stream).
 * te_get_timing waits for the stream, returns the accumulated milliseconds of the main chain kernel
 * and of the fix-up kernel and the number of timed launches, then resets the accumulators. */
int te_enable_timing(te_ctx* ctx, int on);
int te_get_timing(te_ctx* ctx, double* main_ms, double* fixup_ms, int64_t* samples);
/* Work-list counters of the last fused launch: [0] cells the fp32 stencil could not certify (tier 2,
 * fp64 on centred coordinates); [1] work-list entries reserved for them (warp-private chunks, padding included);
 * [2] non-zero if a work list overflowed (cannot happen: the lists are sized for every cell of the launch);
 * [4] cells tier 2 passed on to the literal kernel (tier 3); [3] reserved (0). */
int te_get_flag_counters(te_ctx* ctx, uint32_t out[5]);
/* Why tier 2 passed cells of the last fused launch on to the literal kernel: reasons[r] = cells escalated for reason r
 * (1 degenerate / 2 rank-deficient / 3 small eigen-gap full window, 4 no convergence / 5 rank / 6 conditioning of a partial
 * window, 7 null eigenvector, 8 n_z == 0, 9 n_z on a float32 rounding boundary); valid_cells[n] = escalated cells whose
 * normals window held n valid cells.  Diagnostics only; no reference counterpart. */
int te_get_escalation_stats(te_ctx* ctx, uint32_t reasons[16], uint32_t valid_cells[26]);
/* The fix-up work list of the last fused launch: tier = 2 the cells the fp32 stencil flagged for the fp64 fix-up, tier = 3 the
 * cells tier 2 passed on to the literal kernel.  *count receives the number of entries and out[0 .. min(*count, capacity))
 * the entries themselves, in list order (chunk padding dropped); out may be null when capacity is 0.  An entry is the cell's
 * index in the launch (map index * rows * out_cols + column * rows + row) | do_n << 30 | do_s << 31, where do_n asks for the
 * normals part (slope, roughness, normals) and do_s for the step part; tier-3 entries carry do_n only.  Only the LAST launch
 * is reported: a host-memory te_chain that pipelines column chunks reports its last chunk.  Diagnostics only; no reference
 * counterpart. */
int te_get_fixup_cells(te_ctx* ctx, int tier, uint32_t capacity, uint32_t* out, uint32_t* count);
/* Work decomposition the fused kernel uses for `nmaps` maps of rows x out_ncols output cells on a GPU with `sms`
 * multiprocessors (host arithmetic only, needs no GPU; no reference counterpart — the reference iterates cell by cell).
 * Units are (level, map, column segment, 60-row strip), popped from a queue in that order; a level is a run of columns cut
 * into segments of one length.  out[0] = strips per map, out[1] = levels, then per level {first unit, first column,
 * segment length, segments per map}, then the total number of units: 2 + 4*levels + 1 values (levels <= 4, so 19). */
int te_fused_plan(int rows, int out_ncols, int nmaps, int sms, int32_t out[19]);

/* filters::SlopeFilter<grid_map::GridMap>::update — traversability_estimation_filters/src/SlopeFilter.cpp:59-89.
 * in: surface_normal_z, out: the `map_type` layer. */
int te_slope(te_ctx* ctx, const te_geometry* g, double critical_value, const float* surface_normal_z,
             float* out, int memory);

/* grid_map::NormalVectorsFilter::update (area method) — third-party, configured at
 * robot_filter_parameter.yaml:3-9.  out: surface_normal_{x,y,z}. */
int te_normals(te_ctx* ctx, const te_geometry* g, const te_chain_params* p, const float* elevation,
               float* nx, float* ny, float* nz, int memory);

/* filters::StepFilter<grid_map::GridMap>::update — StepFilter.cpp:102-182 (both passes; the
 * temporary step_height layer never leaves the device). */
int te_step(te_ctx* ctx, const te_geometry* g, const te_chain_params* p, const float* elevation,
            float* out, int memory);

/* filters::RoughnessFilter<grid_map::GridMap>::update — RoughnessFilter.cpp:73-132. */
int te_roughness(te_ctx* ctx, const te_geometry* g, const te_chain_params* p, const float* elevation,
                 const float* nx, const float* ny, const float* nz, float* out, int memory);

/* The whole chain filters::FilterChain<grid_map::GridMap>::update runs at TraversabilityMap.cpp:214:
 * normals -> slope, step, roughness -> weighted sum; normals are deleted unless pointers are given
 * (DeletionFilter, robot_filter_parameter.yaml:34-37).  `slab` NULL = whole map. */
int te_chain(te_ctx* ctx, const te_geometry* g, const te_slab* slab, const te_chain_params* p,
             const float* elevation, float* slope, float* step, float* roughness, float* traversability,
             float* nx_or_null, float* ny_or_null, float* nz_or_null, int memory);

/* nmaps independent maps of identical geometry, stored back to back (map m at offset m*rows*cols). */
int te_chain_batched(te_ctx* ctx, const te_geometry* g, const te_chain_params* p, int32_t nmaps,
                     const float* elevation, float* slope, float* step, float* roughness,
                     float* traversability, int memory);

/* TraversabilityMap::traversabilityFootprint(const double& radius, const double& offset) —
 * traversability_estimation/src/TraversabilityMap.cpp:307-318 with isTraversable (:654-746),
 * isTraversableForFilters (:774-792), checkForStep (:794-865), checkForSlope (:867-893).
 * out: traversability_footprint; slope_footprint/step_footprint memoisation layers optional.
 * traversability_default may be NaN or infinite: a cell whose disk visits an invalid traversability cell before its first blocked
 * one then gets NaN / that infinity (0 when the blocked cell lies within the radius), every other cell what a finite default
 * gives.  Such a default takes the visit-by-visit sweep, about 50 times slower than the prefix-sum sweep at the YAML footprint. */
int te_footprint(te_ctx* ctx, const te_geometry* g, const te_slab* slab, const te_footprint_params* p,
                 const float* traversability, const float* slope, const float* step, const float* elevation,
                 float* traversability_footprint, float* slope_footprint_or_null, float* step_footprint_or_null,
                 int memory);

/* te_footprint with the traversability_roughness layer: when p->verify_roughness is set, a visited cell is also blocked by
 * checkForRoughness (TraversabilityMap.cpp:895-921: more than floor(1.5 * 3 res * max_gap_width / 3 / res^2) cells of zero
 * roughness traversability within 3 res).  `roughness` may be NULL when the flag is clear; roughness_footprint receives the
 * memoisation layer the reference keeps (optional). */
int te_footprint2(te_ctx* ctx, const te_geometry* g, const te_slab* slab, const te_footprint_params* p,
                  const float* traversability, const float* slope, const float* step, const float* roughness_or_null,
                  const float* elevation, float* traversability_footprint, float* slope_footprint_or_null,
                  float* step_footprint_or_null, float* roughness_footprint_or_null, int memory);

/* TraversabilityMap::traversabilityFootprint(double footprintYaw), TraversabilityMap.cpp:239-305 — what the reference's
 * `traversability_footprint` service runs (TraversabilityEstimation.cpp:272-276): every cell gets the footprint polygon
 * (footprint/footprint_polygon, robot_footprint_parameter.yaml:3; `polygon_xy` = npts vertices (x, y) in the footprint frame,
 * 3..16) placed at its centre, unrotated -> layer traversability_x, rotated by footprint_yaw about z -> traversability_rot.  Each
 * value is isTraversable(polygon, traversability) (:592-645): 0 when a cell inside the polygon (grid_map::PolygonIterator) fails
 * isTraversableForFilters, else the mean of the traversability layer over those cells (traversability_default for invalid
 * cells, and when the polygon covers no cell).  Uses p->traversability_default, max_gap_width, critical_step_height,
 * verify_roughness (radius / offset are ignored).  Slab halo: te_footprint's predicate halo + the polygon's reach.
 * traversability_default may be NaN or infinite: a polygon that holds an invalid cell and no blocked one then gives that default,
 * as the reference's sum does, every other cell what a finite default gives; the same holds for the batched, list-of-yaws and
 * te_map polygon sweeps (not for the reductions over yaws, which refuse such a default).
 * TE_ERR_UNSUPPORTED for a polygon that reaches further than 31 cells from its centre. */
int te_footprint_polygon(te_ctx* ctx, const te_geometry* g, const te_slab* slab, const te_footprint_params* p, int32_t npts,
                         const double* polygon_xy, double footprint_yaw, const float* traversability, const float* slope,
                         const float* step, const float* roughness_or_null, const float* elevation, float* traversability_x,
                         float* traversability_rot, int memory);

/* TraversabilityMap::traversabilityFootprint(const double& radius, const double& offset) — TraversabilityMap.cpp:307-318, as
 * te_footprint2 — for nmaps independent whole maps of identical geometry in one call (multi-robot and MPC roll-out batches; the
 * layout of te_chain_batched: map m at offset m*rows*cols in every layer, input and output).  Map m's outputs equal, bit for bit,
 * what te_footprint2 returns for that map alone; a map never reads the cells of another.  1 <= nmaps <= 65535 (TE_ERR_BAD_ARG
 * below 1), nmaps*rows*cols < 2^32 and nmaps*cols < 2^31 (TE_ERR_UNSUPPORTED otherwise); a circular-buffer start index is
 * TE_ERR_UNSUPPORTED.  TE_MEM_HOST stages the nmaps*cols columns of every layer; TE_MEM_DEVICE is asynchronous on the context
 * stream. */
int te_footprint_batched(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, int32_t nmaps,
                         const float* traversability, const float* slope, const float* step, const float* roughness_or_null,
                         const float* elevation, float* traversability_footprint, float* slope_footprint_or_null,
                         float* step_footprint_or_null, float* roughness_footprint_or_null, int memory);

/* TraversabilityMap::traversabilityFootprint(double footprintYaw) — TraversabilityMap.cpp:239-305, as te_footprint_polygon — for
 * nmaps whole maps in the layout and with the limits of te_footprint_batched: map m's traversability_x / traversability_rot equal,
 * bit for bit, what te_footprint_polygon returns for that map alone. */
int te_footprint_polygon_batched(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                                 const double* polygon_xy, double footprint_yaw, const float* traversability, const float* slope,
                                 const float* step, const float* roughness_or_null, const float* elevation, float* traversability_x,
                                 float* traversability_rot, int memory);

/* traversabilityFootprint(footprintYaw) at a whole list of yaws in one call: the cost of a non-circular robot at every heading a
 * lattice / hybrid-A* planner or a sampling MPC plans over.  Layer k of map m is at offset (k*nmaps + m)*rows*cols of
 * traversability_yaws (column-major as every layer) and equals, bit for bit, the traversability_rot that
 * te_footprint_polygon(..., footprint_yaw = yaws[k], ...) returns for map m alone; a yaw of exactly 0.0 therefore also equals its
 * traversability_x.  The layers take the layout and limits of te_footprint_polygon_batched: nmaps whole maps back to back,
 * 1 <= nmaps <= 65535 (nmaps = 1: a single map), the same cell and column bounds, and a circular-buffer start index is
 * TE_ERR_UNSUPPORTED.  polygon_xy (3..16 vertices) and yaws are HOST arrays in both memory modes: the host classifies the
 * polygon's cells once per yaw.  Parameters from p: exactly what te_footprint_polygon uses.  1 <= nyaws <= 1024: below 1
 * TE_ERR_BAD_ARG, above 1024 TE_ERR_UNSUPPORTED (the cap bounds the host classification and table upload per call; 1024 headings
 * are 0.35 degrees apart).  TE_ERR_BAD_ARG for a non-finite yaw and a null yaws or output; TE_ERR_UNSUPPORTED for a polygon that
 * reaches further than 31 cells from its centre; TE_ERR_MISSING_LAYER for verify_roughness without roughness_or_null.  The
 * predicates run once and one kernel sweeps every yaw.  TE_MEM_HOST stages the nyaws*nmaps*cols output columns; TE_MEM_DEVICE is
 * asynchronous on the context stream. */
int te_footprint_polygon_yaws(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                              const double* polygon_xy, int32_t nyaws, const double* yaws, const float* traversability,
                              const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                              float* traversability_yaws, int memory);

/* Per-cell reductions of te_footprint_polygon_yaws over its yaws, without the stack: the worst heading (can the robot turn on the
 * spot here? 0 as soon as any heading is blocked) and the best heading with its index (a hybrid-A* heuristic, a heading-free cost
 * map).  With v_k the value te_footprint_polygon_yaws writes for yaws[k] at a cell of map m:
 *   worst[m, cell] = v_j for the first j that minimises v_k over k;
 *   best[m, cell] = v_k and best_yaw[m, cell] = k (int32) for the first k that maximises v_k.
 * Comparisons are IEEE; a tie goes to the lower heading index, whose value bits are returned (-0.0 and +0.0 are not reordered).
 * Each output is one layer per map, map m at offset m*rows*cols, or NULL when not wanted.  The reduction runs inside the sweep:
 * device memory holds three layers, not nyaws.  Arguments, layout, limits and errors are those of te_footprint_polygon_yaws, plus
 * TE_ERR_BAD_ARG when all three outputs are NULL or p->traversability_default is not finite (with a finite default every v_k is
 * finite).  TE_MEM_HOST stages only the requested outputs; TE_MEM_DEVICE is asynchronous on the context stream. */
int te_footprint_polygon_yaws_reduce(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                                     const double* polygon_xy, int32_t nyaws, const double* yaws, const float* traversability,
                                     const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                     float* worst_or_null, float* best_or_null, int32_t* best_yaw_or_null, int memory);

/* TraversabilityMap::checkFootprintPath for circular footprints — checkCircularFootprintPath, TraversabilityMap.cpp:345-462 —
 * for a BATCH of paths in one launch (one thread per path: the service callback of the reference checks one path per call;
 * planners and MPC roll-outs ask for hundreds).  It is evaluated on a complete traversability_footprint layer, i.e. the output
 * of te_footprint(radius, offset) for the radius of the paths: every isTraversable(center, radius + offset, ...) of the reference
 * then takes its memoised branch (:667-673: traversability = layer value, traversable iff value != 0), a centre outside the map the
 * default branch (:660-666).  Path q is the poses poses_xy[2*path_begin[q] .. 2*path_begin[q+1]) (x, y in the map frame); for a
 * path of one pose the circle at the pose is checked (:365-390), otherwise every fourth cell (nSkip = 3, :401) of the grid line
 * between consecutive poses, and the segment means are combined weighted by segment length (:437-449).  Outputs per path:
 * TraversabilityResult.is_safe and .traversability (0 when unsafe); .area is 0 for circular footprints.  Not covered:
 * the untraversable polygon, publishing.  Poses of a multi-pose path must lie inside the map
 * (the reference does not check getIndex's return value there): such a path is reported unsafe. */
int te_check_footprint_paths(te_ctx* ctx, const te_geometry* g, const float* traversability_footprint,
                             double traversability_default, int32_t npaths, const int32_t* path_begin, const double* poses_xy,
                             uint8_t* is_safe, double* traversability, int memory);

/* te_check_footprint_paths with checkRobotInclination_ set (TraversabilityMap.cpp:359-363, :386-390): before the circles of a
 * pose / segment are looked at, TraversabilityMap::checkInclination (:748-762) reads the `robot_slope` layer (robotSlopeType_,
 * config/robot.yaml:1; column-major like every layer) — at the pose for a single pose, along LineIterator(start, end) otherwise,
 * skipping invalid cells — and the path is unsafe as soon as a cell is exactly 0.0.  robot_slope_or_null == NULL is the call above.
 * A single pose outside the map (the reference's atPosition throws) is reported unsafe. */
int te_check_footprint_paths2(te_ctx* ctx, const te_geometry* g, const float* traversability_footprint,
                              const float* robot_slope_or_null, double traversability_default, int32_t npaths,
                              const int32_t* path_begin, const double* poses_xy, uint8_t* is_safe, double* traversability, int memory);

/* checkCircularFootprintPath (TraversabilityMap.cpp:345-462) as the reference's check_footprint_path service answers it on a
 * freshly computed map (TraversabilityEstimation.cpp:278-295): computeTraversability leaves traversability_footprint empty (NaN,
 * TraversabilityMap.cpp:225-228), so every isTraversable(center, radius + offset, ...) walks the SpiralIterator over the chain
 * layers (:679-736) instead of reading a swept layer.  That branch differs from te_check_footprint_paths2:
 *   - a blocked cell between radius and radius + offset (the first one in visit order) makes the circle untraversable (:714-717);
 *   - a circle's mean reaches the path sum in double, not rounded to float32 (:733);
 *   - a single pose is evaluated at the pose itself: the circle test of the outer two rings is against the pose position;
 *   - compute_untraversable_polygon[q] != 0 (FootprintPath.compute_untraversable_polygon; NULL = all 0) keeps the walk going: a
 *     first blocker in that annulus leaves the circle traversable with its mean divided by the cell count twice (:707, :733);
 *   - a centre that an earlier segment of the same path checked reads the float32 value the first check stored (:673-675):
 *     traversable iff it is != 0.
 * Cache across paths: every path is answered as the first check after computeTraversability, on an empty cache; within a path
 * the cache is reproduced exactly.  The reference keeps the cache across the paths of a request and across requests until the
 * next map update; te_map_check_footprint_request on a te_map (below) answers as it does.
 * Layers: the chain outputs traversability, traversability_slope, traversability_step (traversability_roughness when
 * p->verify_roughness is set) and elevation; robot_slope_or_null switches checkRobotInclination_ on, as in
 * te_check_footprint_paths2.  From `p` only offset (radiusMax = radius + offset; the reference hard-codes 0.15, :348),
 * traversability_default, max_gap_width, critical_step_height, radius_is_integer_norm and verify_roughness are used; p->radius
 * is ignored — radius[q] is FootprintPath.radius of path q.  Paths, outputs and conventions (empty path, poses outside the map,
 * lengthPath) as te_check_footprint_paths2.  Whole maps only.
 * Errors: TE_ERR_MISSING_LAYER for a missing layer; TE_ERR_BAD_ARG for null or negative arguments and, in TE_MEM_HOST, a radius
 * that is NaN or negative; TE_ERR_UNSUPPORTED in TE_MEM_HOST when ceil((radius + offset) / resolution) exceeds 127 rings, and
 * in TE_MEM_DEVICE for a non-zero start index.  TE_MEM_DEVICE is asynchronous on the context stream and cannot read the radii:
 * a path with such a radius gets is_safe = 0 and traversability = NaN (a checked path never yields NaN).  TE_MEM_HOST takes a
 * circular-buffer start index (the layers are unwrapped on upload; poses are map-frame positions and need no change). */
int te_check_footprint_paths_fresh(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, const float* traversability,
                                   const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                   const float* robot_slope_or_null, int32_t npaths, const int32_t* path_begin, const double* poses_xy,
                                   const double* radius, const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe,
                                   double* traversability_out, int memory);

/* checkPolygonalFootprintPath (TraversabilityMap.cpp:464-584), the half of the check_footprint_path service that runs when
 * FootprintPath.footprint has vertices (checkFootprintPath :320-343), for a batch of paths on the chain layers.  Per pose k of a
 * path the footprint is placed with the pose's full 3-D orientation: vertex = R(q_k) * v + t_k, x and y kept (:488-508), R being
 * Eigen's Quaternion::toRotationMatrix of (qx, qy, qz, qw) AS GIVEN (not normalised), v the float32 vertex widened to double.  A
 * single-pose path checks that polygon (:522-543); a longer path checks the convex hull of consecutive footprints per segment
 * (:545-579) and combines the segment means weighted by hull area: area += getArea(hull) - getArea(polygon1).  With
 * conservative[q] set (FootprintPath.conservative; NULL = all 0) each footprint also gets the previous one shifted forward and vice
 * versa (:510-520); the lists accumulate along the path, and getArea is taken of the concatenated (non-simple) polygon1 list, as
 * the reference does.  isTraversable(polygon) (:592-645): PolygonIterator over the hull's bounding box bound to the map, unsafe at
 * the first cell failing isTraversableForFilters, else the mean of traversability (traversability_default for invalid cells; the
 * default when no cell centre is inside, traversable iff it is != 0).  robot_slope_or_null switches checkRobotInclination_ on
 * (checkInclination, :748-762) as in te_check_footprint_paths2.
 * RECALLED, not in the reference checkout: grid_map 1.6.x Polygon::convexHull (monotone chain of polygon1 ++ polygon2, lexicographic
 * sort, cross <= 0 pops; 3 points or fewer kept as given), Polygon::getArea (shoelace from j = n-1, abs(area / 2.0)),
 * Polygon::isInside, PolygonIterator, and Eigen's toRotationMatrix operand order (oracle/README.md).
 * Arguments: footprint_xyz = nfootprint (1..16) vertices x, y, z as float32 (geometry_msgs/Point32), a HOST array in both modes,
 * shared by every path; poses = 7 doubles per pose, x y z qx qy qz qw (geometry_msgs/Pose order); path q = poses
 * path_begin[q] .. path_begin[q+1]-1, nposes = path_begin[npaths].  From `p` only traversability_default, max_gap_width,
 * critical_step_height and verify_roughness are used.  compute_untraversable_polygon is not an argument: in isTraversable it only
 * changes the published polygon, never is_safe, traversability or area.  Outputs: TraversabilityResult.is_safe, .traversability,
 * .area.  Poses outside the map are legal (PolygonIterator bounds the hull to the map); with robot_slope a pose outside the map
 * makes the path unsafe.  An empty path is unsafe with 0.
 * Deviation: an unsafe path reports 0 in traversability and area; the reference returns early (:536-538, :564-567) and leaves the
 * values of earlier segments in its result.  A footprint of zero area (1 or 2 vertices, collinear) can give a combined area of 0
 * and traversability 0/0 = NaN, as in the reference.
 * Limits: a conservative path may not need more than 1024 vertices in polygon2 (nfootprint * poses <= 1024).  Whole maps only.
 * Errors: TE_ERR_MISSING_LAYER for a missing layer; TE_ERR_BAD_ARG for null pointers, a negative count, nfootprint outside 1..16,
 * a non-finite footprint vertex, and in TE_MEM_HOST for nposes != path_begin[npaths], a decreasing path_begin or a non-finite
 * pose; TE_ERR_UNSUPPORTED in TE_MEM_HOST for a conservative path past the vertex cap, and in TE_MEM_DEVICE for a non-zero start
 * index.  TE_MEM_DEVICE is asynchronous on the context stream and cannot read the paths: a path it cannot check (non-finite
 * pose, past the conservative cap, a range outside 0..nposes) gets is_safe = 0 and NaN in traversability and area.  A conservative
 * flag array in TE_MEM_DEVICE sizes the kernel's shared memory for the cap (slower); TE_MEM_HOST sizes it from the paths and
 * takes a circular-buffer start index (the layers are unwrapped on upload). */
int te_check_footprint_paths_polygon(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, const float* traversability,
                                     const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                     const float* robot_slope_or_null, int32_t nfootprint, const float* footprint_xyz, int32_t npaths,
                                     int32_t nposes, const int32_t* path_begin, const double* poses,
                                     const uint8_t* conservative_or_null, uint8_t* is_safe, double* traversability_out,
                                     double* area_out, int memory);

/* The untraversable polygon of the two path checks above: what the check_footprint_path service publishes on its
 * untraversable_polygon topic for a path with compute_untraversable_polygon set (it always checks with publishPolygons = true,
 * TraversabilityEstimation.cpp:290).  te_check_footprint_paths_fresh2 / _polygon2 take the arguments of te_check_footprint_paths_fresh
 * / _polygon plus the polygon outputs, and compute is_safe, traversability and area exactly as those do; with
 * untraversable_count_or_null == NULL (and untraversable_xy_or_null == NULL) each IS its predecessor.
 * Output per path q: the LAST NON-EMPTY polygon the service publishes for the path (publishUntraversablePolygon skips empty ones,
 * :934), or none.  untraversable_count[q] = its vertex count (0: none; always 0 when compute_untraversable_polygon[q] is 0), and
 * untraversable_xy[2 * max_vertices * q ...] = its first min(count, max_vertices) (x, y) vertices in the reference's order (the rest
 * of the slot is unspecified).  A count above max_vertices means the polygon was cut to that prefix: call again with more room.  The z of the published polygon
 * (computeMeanHeightFromPoses, TraversabilityMap.hpp:311) is left to the caller.
 *   Circular paths (checkCircularFootprintPath :345-462, isTraversable :654-746): a circle whose spiral walk finds a first blocked
 *   cell within radius walks on to the end of the spiral and collects every blocked cell with getCurrentRadius() <= radius (every
 *   blocked cell for radius 0); the polygon is monotoneChainConvexHullOfPoints of their cell centres: 3 points or fewer as visited,
 *   more as the convex hull from the lexicographically smallest vertex, counter-clockwise.  A single pose outside the map with
 *   traversability_default 0, and a centre an earlier segment of the path cached as 0, give Polygon::fromCircle(centre,
 *   radius + offset).  A single pose publishes its circle's polygon; a longer path publishes, for its failing segment,
 *   convexHull(path polygon, failing circle's polygon) taken once per checked line cell from the failing one on (:407-412), which
 *   is that polygon's hull except for 1 to 3 collected cells: 2 or 3 cells give their hull; 1 cell gives the point 2 times for an
 *   even number of hulls and 3 times for an odd one.  checkInclination failures publish nothing.
 *   Polygonal paths (checkPolygonalFootprintPath :464-584, isTraversable(polygon) :592-645): compute_untraversable_polygon_or_null
 *   (FootprintPath.compute_untraversable_polygon per path; NULL = all 0) lets the PolygonIterator walk go on past blocked cells; the
 *   polygon is monotoneChainConvexHullOfPoints of all blocked cell centres of the failing segment (or single pose).
 * RECALLED, not in the reference checkout (grid_map 1.6.x): Polygon::fromCircle(center, radius, nVertices = 20): vertex j =
 * center + Rotation2D(j * 2 * M_PI / 19) * (radius, 0), so the last vertex repeats the first up to the rounding of sin(2 pi); the
 * cosines and sines come from the host's libm.  Polygon::convexHull(P1, P2) = monotoneChainConvexHullOfPoints(P1 ++ P2).
 * Bound: a polygonal segment's (or pose's) footprint hull may span at most 1024 map rows when its polygon is requested.  Circular
 * paths have no bound beyond the 127-ring radius limit.
 * Errors, beyond those of the predecessors: TE_ERR_BAD_ARG for max_vertices < 0, a count pointer without an xy pointer while
 * max_vertices > 0, and an xy pointer without a count pointer; TE_ERR_UNSUPPORTED in TE_MEM_HOST when a requested polygonal
 * polygon passes the 1024-row bound (the other outputs are written).  TE_MEM_DEVICE cannot read the paths: a path whose polygon
 * was requested but could not be computed (past the bound, or a path the check marks with NaN) gets count -1; its is_safe,
 * traversability and area are those of the predecessor.  TE_MEM_HOST accepts a circular-buffer start index as the
 * predecessors do. */
int te_check_footprint_paths_fresh2(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, const float* traversability,
                                    const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                    const float* robot_slope_or_null, int32_t npaths, const int32_t* path_begin, const double* poses_xy,
                                    const double* radius, const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe,
                                    double* traversability_out, int32_t max_vertices, int32_t* untraversable_count_or_null,
                                    double* untraversable_xy_or_null, int memory);
int te_check_footprint_paths_polygon2(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, const float* traversability,
                                      const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                      const float* robot_slope_or_null, int32_t nfootprint, const float* footprint_xyz, int32_t npaths,
                                      int32_t nposes, const int32_t* path_begin, const double* poses,
                                      const uint8_t* conservative_or_null, uint8_t* is_safe, double* traversability_out,
                                      double* area_out, const uint8_t* compute_untraversable_polygon_or_null, int32_t max_vertices,
                                      int32_t* untraversable_count_or_null, double* untraversable_xy_or_null, int memory);

/* A whole CheckFootprintPath request (TraversabilityEstimation.cpp:278-295) in one call: FootprintPath[] with circular and
 * polygonal paths mixed, each with its own footprint, results in request order.  Every circular path sees an empty
 * traversability_footprint cache; for the reference node's answers over a sequence of requests use te_map_check_footprint_request.  Path q is circular when its footprint has no
 * vertices (checkFootprintPath, TraversabilityMap.cpp:320-343: any non-empty polygon takes the polygonal branch) and gets, bit for
 * bit, what te_check_footprint_paths_fresh2 gives for it alone with radius[q] and compute_untraversable_polygon[q]; its area is 0,
 * as in the reference's result.  Otherwise it gets what te_check_footprint_paths_polygon2 gives for it alone with its own
 * footprint, conservative[q] and compute_untraversable_polygon[q]; radius[q] is then ignored, as FootprintPath.radius is.
 * Everything those two entries document carries over per kind of path: layers and `p`, empty paths, poses outside the map,
 * robot_slope, the empty traversability_footprint cache per path, the deviation that an unsafe path reports 0, the 127-ring,
 * conservative-cap and 1024-row limits, the untraversable polygon outputs (max_vertices, count, xy slots) and, in TE_MEM_HOST, a
 * circular-buffer start index.  New here:
 *   - poses = 7 doubles per pose (x y z qx qy qz qw) for both kinds; a circular path reads x and y only.  Path q = poses
 *     path_begin[q] .. path_begin[q+1]-1, nposes = path_begin[npaths];
 *   - footprint_xyz = nvertices vertices x, y, z as float32; path q's footprint = vertices footprint_begin[q] ..
 *     footprint_begin[q+1]-1 (0: circular, 1..16: polygonal).  Unlike te_check_footprint_paths_polygon2's footprint these arrays
 *     follow `memory`;
 *   - max_footprint_vertices (0..16) bounds every footprint and sizes the polygonal kernel's shared memory;
 *   - one call uploads the layers once (TE_MEM_HOST) and clears one isTraversableForFilters memo, which both kinds of path share
 *     (it depends on the layers only, so sharing it changes no result).
 * Errors: those of the two entries, applied to each kind of path (TE_ERR_BAD_ARG for p->offset < 0 always); TE_ERR_BAD_ARG for
 * max_footprint_vertices outside 0..16, null or negative arguments (footprint_xyz may be null when nvertices is 0), and in
 * TE_MEM_HOST for a footprint_begin that does not start at 0, decreases or does not end at nvertices, a footprint with more
 * vertices than max_footprint_vertices, and a non-finite vertex.  TE_MEM_DEVICE is asynchronous on the context stream and
 * cannot read the paths: a path whose footprint cannot be checked (over max_footprint_vertices, outside the vertex array, a
 * non-finite vertex), or that its own entry could not check, gets is_safe = 0, NaN in traversability and area, and count -1
 * where its polygon was requested; the other paths are unaffected. */
int te_check_footprint_request(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, const float* traversability,
                               const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                               const float* robot_slope_or_null, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                               const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                               const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative_or_null,
                               const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe, double* traversability_out,
                               double* area_out, int32_t max_vertices, int32_t* untraversable_count_or_null,
                               double* untraversable_xy_or_null, int memory);

/* te_check_footprint_request for the paths of a whole batch of maps in one call (multi-robot and MPC roll-out batches, after
 * te_chain_batched).  Layers: nmaps whole maps of geometry g in the layout of te_chain_batched / te_footprint_batched, map m at
 * offset m*rows*cols in every layer, robot_slope included.  Path q is on map path_map[q] (0..nmaps-1; any order, and a map may have
 * no paths); poses are map-frame positions, the same for every map.  The other arguments and outputs are those of
 * te_check_footprint_request, and path q gets, bit for bit, what te_check_footprint_request returns for it on map path_map[q]
 * alone (is_safe, traversability, area and the untraversable polygon).  Each map has its own isTraversableForFilters memo; a path
 * never reads the cells of another map.  Errors: those of te_check_footprint_request, per path, plus TE_ERR_BAD_ARG for nmaps < 1,
 * a null path_map and, in TE_MEM_HOST, a path_map entry outside 0..nmaps-1; TE_ERR_UNSUPPORTED for a circular-buffer start index
 * and for nmaps*cols >= 2^31.  TE_MEM_HOST stages the nmaps*cols columns of every layer once; TE_MEM_DEVICE is asynchronous on the
 * context stream and cannot read path_map: a path on a map outside the batch gets is_safe = 0, NaN in traversability and area,
 * and count -1 where its polygon was requested; the other paths are unaffected.  The launches are those of one
 * te_check_footprint_request, whatever nmaps. */
int te_check_footprint_request_batched(te_ctx* ctx, const te_geometry* g, const te_footprint_params* p, int32_t nmaps,
                                       const float* traversability, const float* slope, const float* step,
                                       const float* roughness_or_null, const float* elevation, const float* robot_slope_or_null,
                                       const int32_t* path_map, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                       const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                       const float* footprint_xyz, int32_t max_footprint_vertices,
                                       const uint8_t* conservative_or_null, const uint8_t* compute_untraversable_polygon_or_null,
                                       uint8_t* is_safe, double* traversability_out, double* area_out, int32_t max_vertices,
                                       int32_t* untraversable_count_or_null, double* untraversable_xy_or_null, int memory);

/* ---- te_map: a traversability map that stays on the device between calls -------------------------------------------------------
 * The reference keeps its layers, the traversability_footprint cache and the isTraversableForFilters memo in one TraversabilityMap;
 * computeTraversability (TraversabilityMap.cpp:202-237) resets them and nothing else does (resetTraversabilityFootprintLayers,
 * :195-200, has no caller).  So the answers of its check_footprint_path service depend on the checks before them: a circle
 * whose first blocked cell lies between radius and radius + offset is untraversable the first time (:714-717) but stores a
 * positive value (:708) that every later check of that cell reads back as traversable (:673-675).  A te_map holds that state on
 * the device, so a node that keeps one te_map answers as the reference node does, and uploads its layers once per map update
 * instead of once per call.  The stateless entries above keep answering every call on an empty cache.
 *
 * A te_map belongs to one te_ctx: it runs on that context's stream under its lock and must be destroyed before the context.  It
 * owns, on the device, the layers traversability, traversability_slope, traversability_step, traversability_roughness (optional),
 * elevation, robot_slope (optional), the elevation map's carried layers (optional, te_map_carry_layers below) and
 * traversability_x / traversability_rot (optional, te_map_footprint_polygon_keep); the
 * traversability_footprint cache (float32, NaN = empty); and the isTraversableForFilters
 * memo, which is kept until the layers or one of max_gap_width, critical_step_height and verify_roughness change.  Whole maps only.
 * Host layers may carry a circular-buffer start index: they are unwrapped on upload and outputs are re-wrapped to the start index
 * of the last te_map_chain / te_map_set_layers.  Every entry but te_map_create / te_map_destroy fails with TE_ERR_BAD_ARG before
 * layers were set.  Host-memory entries return synchronised; device-memory ones are asynchronous on the context stream.
 *
 * Batches.  te_map_chain_batched / te_map_set_layers_batched give a te_map nmaps >= 1 maps of one geometry (a robot each, say),
 * in the layout of te_chain_batched: map m at offset m*rows*cols in every layer, the cache and the memo.  Each map has its own
 * cache and memo, and for each map m everything a call returns or stores is, bit for bit, what a separate single-map te_map
 * holding map m returns or stores for the same calls restricted to map m (for a request: that map's paths, in their relative
 * request order).  A path never reads or writes another map's cells, cache or memo.  Limits as te_footprint_batched: nmaps
 * 1..65535 (TE_ERR_BAD_ARG below 1, TE_ERR_UNSUPPORTED above), nmaps*rows*cols < 2^32 and nmaps*cols < 2^31 (TE_ERR_UNSUPPORTED);
 * a circular-buffer start index in g is TE_ERR_UNSUPPORTED for every _batched entry (the _wrapped entries below take one per
 * map).  On a batch te_map_footprint, the polygon
 * entries, te_map_get_layers, te_map_get_footprint and te_map_clear_footprint work on every map, their outputs holding the maps
 * back to back per layer; te_map_check_footprint_request, te_map_get_submaps and te_map_valid_at need a map index and fail with
 * TE_ERR_BAD_ARG on a te_map of more than one map (use their _batched entries).  The single-map entries on a te_map of one map
 * are unchanged, start indices included.  The maps of a batch may also sit at their own positions (te_map_chain_batched_at and the
 * other _at entries below): the rule above then holds with a single-map te_map holding map m at map m's position. */
typedef struct te_map te_map;
int te_map_create(te_ctx* ctx, te_map** out);
int te_map_destroy(te_map* map);

/* computeTraversability (:202-237): te_chain on `elevation` into the map's layers, each optionally copied out (NULL: kept on the
 * device only).  Empties the cache and the memo and leaves the map without robot_slope and carried layers (te_map_carry_layers
 * adds them). */
int te_map_chain(te_map* map, const te_geometry* g, const te_chain_params* p, const float* elevation, float* slope_or_null,
                 float* step_or_null, float* roughness_or_null, float* traversability_or_null, int memory);

/* setTraversabilityMap: the layers as given (a map received or loaded from a bag).  Empties the cache and the memo.
 * TE_ERR_MISSING_LAYER for a missing required layer. */
int te_map_set_layers(te_map* map, const te_geometry* g, const float* traversability, const float* slope, const float* step,
                      const float* roughness_or_null, const float* elevation, const float* robot_slope_or_null, int memory);

/* computeTraversability for every map of a batch: te_chain_batched on nmaps elevation maps (layout and limits above) into the
 * te_map's layers, each optionally copied out for every map.  Empties every cache and memo and leaves the batch without
 * robot_slope, as te_map_chain does; te_map_chain is its nmaps = 1 case. */
int te_map_chain_batched(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elevation,
                         float* slope_or_null, float* step_or_null, float* roughness_or_null, float* traversability_or_null, int memory);

/* setTraversabilityMap for every map of a batch: every layer holds nmaps maps back to back.  Empties every cache and memo; the only
 * way to give a batch robot_slope.  te_map_set_layers is its nmaps = 1 case. */
int te_map_set_layers_batched(te_map* map, const te_geometry* g, int32_t nmaps, const float* traversability, const float* slope,
                              const float* step, const float* roughness_or_null, const float* elevation,
                              const float* robot_slope_or_null, int memory);

/* Updates of some maps of a batch: te_map_chain_maps, te_map_set_layers_maps and te_map_footprint_maps act on the maps
 * map_index[0..nsel) only, as the single-map entry would on a te_map holding that map alone, and leave every bit of the other maps'
 * layers, caches and memos as it was.  So a batch keeps modelling one reference node per map when the maps are updated
 * independently (a robot receives a new elevation map, a simulated environment resets its terrain).  Rules:
 *   - map_index is a HOST array in both memory modes, read before the call returns (pageable or page-locked, the caller may reuse
 *     it at once); nsel is 1..nmaps and the entries are distinct and in 0..nmaps-1, in any order.  Layer arguments and outputs
 *     hold the nsel maps back to back in map_index order.
 *   - g must equal the batch's geometry bit for bit (TE_ERR_BAD_ARG otherwise).  A start index, in g or on the te_map's layers, is
 *     TE_ERR_UNSUPPORTED, as for every _batched entry (use te_map_chain there, or the _wrapped entries below, whose start indices
 *     these entries accept).  A te_map without layers is TE_ERR_BAD_ARG.
 *   - Every map of a batch holds the same layers, so the optional layers stay those the batch holds: te_map_chain_maps, which gives
 *     a map roughness and no robot_slope as te_map_chain does, is TE_ERR_UNSUPPORTED on a batch that holds robot_slope or lacks
 *     roughness; te_map_set_layers_maps must be given exactly the batch's optional layers (TE_ERR_MISSING_LAYER for a missing one,
 *     TE_ERR_BAD_ARG for an extra one).
 *   - Every argument error is found before anything is written: the te_map is then unchanged.
 *   - The selected maps' caches are emptied and their memo bytes cleared; the memo of the other maps and its parameter key stay.
 * The selected maps move through scratch the te_map keeps, grown to the largest nsel seen and released by te_map_destroy, in bytes
 * per cell of the selected maps: te_map_chain_maps 20 in host memory, 16 in device memory (the elevation is read in place);
 * te_map_set_layers_maps 4 per layer given in host memory, none in device memory; te_map_footprint_maps 4 per layer the sweep
 * reads (16, or 20 with verify_roughness) plus 4 for the sweep's values, a buffer te_map_footprint shares (it holds the whole
 * batch once te_map_footprint has run).  Plus 4 bytes per selected map for the slot table.  Launches: those of te_chain_batched
 * (te_map_chain_maps) or te_footprint_batched (te_map_footprint_maps) on nsel maps, plus one kernel that puts the maps in place
 * (te_map_set_layers_maps: that kernel alone) or, for the sweep, one that gathers them and the merge into the caches; none per
 * selected map. */

/* computeTraversability for the maps map_index[0..nsel) of a batch: te_chain_batched on nsel elevation maps (back to back in
 * map_index order) into those maps' layers; each output optionally copied out, nsel maps back to back in map_index order. */
int te_map_chain_maps(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                      const float* elevation, float* slope_or_null, float* step_or_null, float* roughness_or_null,
                      float* traversability_or_null, int memory);

/* setTraversabilityMap for those maps only: every layer holds nsel maps back to back in map_index order. */
int te_map_set_layers_maps(te_map* map, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* traversability,
                           const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                           const float* robot_slope_or_null, int memory);

/* Maps at their own positions (a fleet, simulated environments with their own origins, robot-centric submaps around each robot).
 * The four entries below take the arguments of the entry of the same name plus position_xy, a HOST array of one (x, y) pair per map
 * the call updates (nmaps pairs, or nsel in map_index order), read before the call returns: map m then sits at that position
 * instead of g's, with g's rows, cols, resolution and length.  position_xy NULL puts every map it updates at g's position: the
 * entry of the same name is that case.  Everything a te_map entry returns or stores for a map (layers, cache, memo, request outputs
 * and untraversable polygons, te_map_request_stats, submaps and their te_submap_info, te_map_valid_at_batched, the footprint sweeps
 * and their reductions) is then, bit for bit, what a single-map te_map
 * holding that map at its position returns or stores.  Rules:
 *   - A non-finite position is TE_ERR_BAD_ARG, found before anything is written (the te_map is then unchanged).
 *   - The _maps_at entries move only the selected maps; they check g against the batch bit for bit except for position_x /
 *     position_y, as the _maps entries check all of it.  Every other rule of the _maps entries applies.
 *   - te_map_chain_image(_maps) puts the maps it updates at g's position; te_map_carry_layers does not move a map.
 *   - Requests (te_map_check_footprint_request_batched, _device) take each path's centres, getIndex and checkInclination from its
 *     map's position, in the work list, the dedup keys (the map is part of a key), the walks, the replay and the polygonal paths.
 *     The polygon entries (te_map_footprint_polygon(_yaws, _yaws_reduce)) classify the polygon's offsets per position: on maps at
 *     several positions they sweep one map at a time (one sweep per map, outputs in the batch layout).
 *     te_map_footprint_polygon_keep sweeps maps at several positions in one launch, each on its own tables.
 *   - Memory: when the maps of a call do not all sit at one position the te_map keeps per-map tables on the device, 8 bytes per
 *     row and per column of every map of the call (cell-centre coordinates) plus 16 per map (the position), and for a chain call
 *     1 byte more per row and column (the fused kernel's on-circle masks); they are rebuilt when the positions change.
 * The kernels read a map's tables through a per-map stride that is 0 when every map sits at one position, so that case reads what
 * it reads without positions. */
int te_map_chain_batched_at(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elevation,
                            float* slope_or_null, float* step_or_null, float* roughness_or_null, float* traversability_or_null, int memory,
                            const double* position_xy);
int te_map_set_layers_batched_at(te_map* map, const te_geometry* g, int32_t nmaps, const float* traversability, const float* slope,
                                 const float* step, const float* roughness_or_null, const float* elevation,
                                 const float* robot_slope_or_null, int memory, const double* position_xy);
int te_map_chain_maps_at(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                         const float* elevation, float* slope_or_null, float* step_or_null, float* roughness_or_null,
                         float* traversability_or_null, int memory, const double* position_xy);
int te_map_set_layers_maps_at(te_map* map, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* traversability,
                              const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                              const float* robot_slope_or_null, int memory, const double* position_xy);
/* Where the maps sit: position_xy[2m], position_xy[2m + 1] for map m (nmaps pairs).  TE_ERR_BAD_ARG before layers were set. */
int te_map_positions(te_map* map, double* position_xy);

/* Maps in their own circular-buffer order (robot-centric maps moved with GridMap::move, each published with its own outer / inner
 * start index).  The four entries below take the arguments of the _at entry of the same stem plus start_index, a HOST array of one
 * (start_row, start_col) pair per map the call updates (nmaps pairs, or nsel in map_index order), read before the call returns.
 * Each map's block of every layer argument is in the buffer order of its pair: cell (i, j) of the map is stored at
 * ((j + start_col) % cols) * rows + (i + start_row) % rows of the block, in both memory modes.  start_index NULL means (0, 0) for
 * every map, and the entry is then its _at entry bit for bit.  Rules:
 *   - g's start_row / start_col must be 0 (the array is the only source of the index) and every pair must lie in 0 .. rows-1,
 *     0 .. cols-1: TE_ERR_BAD_ARG otherwise, found before anything is written.  Every other rule of the _at entry applies.
 *   - The te_map keeps each map's start index until that map is reloaded: a whole-batch _wrapped call sets every map's, a _wrapped
 *     selection the selected maps'; te_map_chain_maps(_at), te_map_set_layers_maps(_at), te_map_chain_image_maps and a
 *     te_map_chain_windows selection give the maps they load (0, 0), and the other whole-batch entries give every map (0, 0).
 *   - While a map has a start index, these HOST outputs hold its block in that buffer order: the chain outputs of these entries,
 *     te_map_get_layers (uncertainty_range included), te_map_get_footprint, te_map_footprint(_maps),
 *     te_map_footprint_polygon(_yaws, _yaws_reduce) (best_yaw included) and te_map_footprint_polygon_keep; te_map_carry_layers takes
 *     its block in that order in both memory modes.  DEVICE outputs stay in default order.  Everything that depends on positions
 *     (requests, submaps, te_map_valid_at_batched, te_map_at_poses) is unaffected, as in grid_map.
 *   - The selection entries (_maps, te_map_footprint_maps, te_map_carry_layers and te_map_footprint_polygon_keep with map_index)
 *     work on such a te_map; a te_map whose start index came in g (te_map_chain / te_map_set_layers) keeps refusing them.
 *   - The moves run on the GPU: one k_map_cut_windows launch puts every map and layer of an input call in default order (device
 *     inputs are read in place; host inputs take one copy per layer into scratch the te_map keeps first), and one re-wraps every
 *     map's block of the host outputs into that scratch before one copy back per output array.  So a whole-batch _wrapped update
 *     costs the launches of its _at entry plus one, whatever nmaps, and one more when it also returns host outputs.  Scratch: 4 bytes
 *     per cell of every layer moved, grown to the largest call and released by te_map_destroy. */
int te_map_chain_batched_wrapped(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elevation,
                                 float* slope_or_null, float* step_or_null, float* roughness_or_null, float* traversability_or_null,
                                 int memory, const double* position_xy_or_null, const int32_t* start_index);
int te_map_set_layers_batched_wrapped(te_map* map, const te_geometry* g, int32_t nmaps, const float* traversability, const float* slope,
                                      const float* step, const float* roughness_or_null, const float* elevation,
                                      const float* robot_slope_or_null, int memory, const double* position_xy_or_null,
                                      const int32_t* start_index);
int te_map_chain_maps_wrapped(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                              const float* elevation, float* slope_or_null, float* step_or_null, float* roughness_or_null,
                              float* traversability_or_null, int memory, const double* position_xy_or_null, const int32_t* start_index);
int te_map_set_layers_maps_wrapped(te_map* map, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* traversability,
                                   const float* slope, const float* step, const float* roughness_or_null, const float* elevation,
                                   const float* robot_slope_or_null, int memory, const double* position_xy_or_null,
                                   const int32_t* start_index);
/* Each map's start index: start_index[2m], start_index[2m + 1] for map m (nmaps pairs; a single map whose start index came in g
 * reports g's).  TE_ERR_BAD_ARG before layers were set. */
int te_map_start_indices(te_map* map, int32_t* start_index);

/* ---- Elevation images: the reference node's image topic (TraversabilityEstimation::imageCallback) ------------------------------
 * The node turns a grayscale height image into the elevation layer (GridMapRosConverter::initializeFromImage on the first image,
 * then addLayerFromImage(image, "elevation", map, min_height, max_height)) and runs computeTraversability on it.  The entries
 * below do the same: the per-pixel arithmetic runs on the GPU, on the image's own 1 or 2 bytes per cell, and the rest is
 * te_map_chain(_batched/_maps).  The node keeps the sensor_msgs header, encoding string and byte order: it passes an encoding
 * code and, for an is_bigendian mono16 image, swaps the bytes itself (pixels are read in host byte order).
 *
 * Encodings.  Mono only: TE_IMAGE_MONO8 (mono8, 8UC1) and TE_IMAGE_MONO16 (mono16, 16UC1), elevation(i, j) = lower + (upper -
 * lower) * ((float)pixel(i, j) / maxv) with lower = (float)min_height, upper = (float)max_height and maxv = 255 or 65535, every
 * operation float32 and IEEE-rounded, as GridMapCvConverter::addLayerFromImage does it.  So pixel 0 gives lower, and the top
 * pixel gives lower + (upper - lower) * 1.0f, which need not equal upper.  min_height and max_height are not checked: a reversed,
 * equal or overflowing pair gives the bits the reference's formula gives.  The colour encodings are TE_ERR_UNSUPPORTED: the
 * reference first greys them with OpenCV's cvtColor, whose fixed-point coefficients depend on the OpenCV version and build, so no
 * result here could be pinned to the reference's. */
enum {
  TE_IMAGE_MONO8 = 0,
  TE_IMAGE_MONO16 = 1,
  /* TE_ERR_UNSUPPORTED (see above) */
  TE_IMAGE_RGB8 = 2, TE_IMAGE_BGR8 = 3, TE_IMAGE_RGBA8 = 4, TE_IMAGE_BGRA8 = 5,
  TE_IMAGE_RGB16 = 6, TE_IMAGE_BGR16 = 7, TE_IMAGE_RGBA16 = 8, TE_IMAGE_BGRA16 = 9
};

/* initializeFromImage(image, resolution, map, position): GridMap::setGeometry(Length(resolution * height, resolution * width),
 * resolution, position), i.e. rows = (int)round(resolution * height / resolution), cols likewise with width, length = size *
 * resolution, the position as given and start index 0.  Host arithmetic, no GPU needed.  TE_ERR_BAD_ARG (out untouched) for a
 * null out, height or width < 1, a resolution that is not finite and > 0, and a position that is not finite. */
int te_image_geometry(int32_t height, int32_t width, double resolution, double position_x, double position_y, te_geometry* out);

/* imageCallback's addLayerFromImage followed by computeTraversability, for nmaps images (nmaps = 1: a single map): te_map_chain
 * (nmaps = 1) or te_map_chain_batched on the elevation the images give, with the same outputs, limits, cache and memo reset and
 * no robot_slope afterwards; te_map_get_layers(TE_LAYER_ELEVATION) returns that elevation.
 *   - Images are row-major, as sensor_msgs/Image: g->rows x g->cols pixels, image row i being map row i (so the layer, column-major,
 *     is the image transposed); row i of image m starts at images + m * image_stride_bytes + i * row_stride_bytes.
 *     image_stride_bytes is ignored for nmaps = 1.  The images are in `memory`.
 *   - TE_ERR_UNSUPPORTED for a start index in g (an image map has none) and a colour encoding; TE_ERR_BAD_ARG for an unknown
 *     encoding, row_stride_bytes < cols * bytes per pixel, image_stride_bytes < rows * row_stride_bytes (nmaps > 1) and, for
 *     mono16, an odd images address or stride (checked in both memory modes); TE_ERR_MISSING_LAYER for null images.  Every
 *     argument error is found before anything is written: the te_map is then unchanged.
 *   - Host memory stages the image bytes only (1 or 2 per cell, not 4) and returns synchronised; device memory reads the images
 *     in place and is asynchronous on the context stream.  Scratch the te_map keeps, grown to the largest call and released by
 *     te_map_destroy: 1 or 2 bytes per cell of the nmaps maps in host memory (the staged images), none in device memory.
 *   - Launches: those of te_map_chain(_batched) plus one conversion kernel, whatever nmaps. */
int te_map_chain_image(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nmaps, int32_t encoding,
                       const void* images, int64_t row_stride_bytes, int64_t image_stride_bytes, double min_height, double max_height,
                       float* slope_or_null, float* step_or_null, float* roughness_or_null, float* traversability_or_null, int memory);

/* The same for the maps map_index[0..nsel) of a batch only: te_map_chain_maps on the elevation the nsel images give (image k goes
 * to map map_index[k]), under the rules of the _maps entries above and the image rules of te_map_chain_image.  Scratch: that of
 * te_map_chain_maps in host memory (20 bytes per selected cell) plus the staged images (1 or 2), and 20 in device memory (the
 * converted elevation is packed before it is put in place).  Launches: those of te_map_chain_maps plus one. */
int te_map_chain_image_maps(te_map* map, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                            int32_t encoding, const void* images, int64_t row_stride_bytes, int64_t image_stride_bytes,
                            double min_height, double max_height, float* slope_or_null, float* step_or_null,
                            float* roughness_or_null, float* traversability_or_null, int memory);

/* traversabilityFootprint(radius, offset) (:307-318) on the cache: a cached cell keeps its value (the memoised branch, :673-675),
 * every other cell gets te_footprint2's value for `p`; traversability_footprint_or_null receives the cache afterwards.  The
 * prefix-sum sweep may differ from the visit-by-visit one in the last float32 bit of a few cells (DESIGN.md §4.3); those values
 * then stay in the cache.  Errors as te_footprint2 (TE_ERR_MISSING_LAYER: verify_roughness without a roughness layer).  On a
 * batch: every map's cache, te_footprint_batched's sweep, nmaps layers out. */
int te_map_footprint(te_map* map, const te_footprint_params* p, float* traversability_footprint_or_null, int memory);

/* traversabilityFootprint(radius, offset) on the caches of the maps map_index[0..nsel) only (rules above te_map_chain_maps): each
 * selected cache becomes what te_map_footprint gives that map; the output holds the nsel caches afterwards in map_index order. */
int te_map_footprint_maps(te_map* map, const te_footprint_params* p, int32_t nsel, const int32_t* map_index,
                          float* traversability_footprint_or_null, int memory);

/* traversabilityFootprint(yaw) (:239-305): te_footprint_polygon on the map's layers.  Reads and changes no cache.  On a batch:
 * te_footprint_polygon_batched's outputs (and te_footprint_polygon_yaws(_reduce)'s for the two entries below: layer k of map m at
 * (k*nmaps + m)*rows*cols). */
int te_map_footprint_polygon(te_map* map, const te_footprint_params* p, int32_t npts, const double* polygon_xy, double footprint_yaw,
                             float* traversability_x, float* traversability_rot, int memory);

/* te_footprint_polygon_yaws on the map's layers: layer k (at k*rows*cols) is the traversability_rot of yaws[k].  Yaws, limits and
 * errors as te_footprint_polygon_yaws; the map's start index is fine.  Reads and changes no cache.  In host memory every layer is
 * re-wrapped to the map's start index, as te_map's other outputs; in device memory the layers are in the map's default (unwrapped)
 * order, as te_map_footprint_polygon's. */
int te_map_footprint_polygon_yaws(te_map* map, const te_footprint_params* p, int32_t npts, const double* polygon_xy, int32_t nyaws,
                                  const double* yaws, float* traversability_yaws, int memory);

/* te_footprint_polygon_yaws_reduce on the map's layers: one layer each, NULL when not wanted.  Outputs, errors and memory order as
 * te_map_footprint_polygon_yaws (best_yaw is re-wrapped as the float layers are).  Reads and changes no cache. */
int te_map_footprint_polygon_yaws_reduce(te_map* map, const te_footprint_params* p, int32_t npts, const double* polygon_xy,
                                         int32_t nyaws, const double* yaws, float* worst_or_null, float* best_or_null,
                                         int32_t* best_yaw_or_null, int memory);

/* The reference's traversability_footprint service (TraversabilityEstimation.cpp:272-276, TraversabilityMap::traversabilityFootprint
 * (footprintYaw), :239-305) kept on the map: traversability_x and traversability_rot become layers the te_map holds
 * (TE_LAYER_TRAVERSABILITY_X / _ROT), published by te_map_get_layers and served by te_map_get_submaps(_batched), as the reference
 * adds them to the map it publishes and cuts submaps from.
 *   - Swept maps: nsel = 0 with map_index_or_null NULL sweeps every map; otherwise the maps map_index[0..nsel), under the rules of
 *     the _maps entries above (a host array of distinct indices, outputs back to back in map_index order, TE_ERR_UNSUPPORTED for a
 *     start index).
 *   - footprint_yaw is a HOST array: nyaws = 1 gives every swept map that yaw, nyaws = the number of swept maps gives map k the
 *     k-th (in map_index order for a selection); any other count is TE_ERR_BAD_ARG.  Yaws are taken as te_map_footprint_polygon
 *     takes its yaw.  More than 1024 distinct yaws (compared by bits) is TE_ERR_UNSUPPORTED.
 *   - Each swept map then holds, bit for bit, the traversability_x / traversability_rot that te_map_footprint_polygon(p,
 *     polygon, its yaw) returns on a single-map te_map holding that map at its position.  Maps not swept keep their two layers
 *     bit for bit; a map never swept holds NaN with bits 0xffffffff (the first call gives the two layers to every map of the
 *     batch, as every map of a batch holds the same layers).  The cache, the memo and every other layer are left alone.
 *   - traversability_x_or_null / traversability_rot_or_null receive copies of the swept maps' new layers: in host memory
 *     re-wrapped to a single map's start index, and the call returns synchronised; in device memory in default order, and the
 *     call is asynchronous on the context stream.
 *   - Errors as te_map_footprint_polygon (TE_ERR_BAD_ARG for a map without layers, a polygon without 3..16 finite vertices and a
 *     non-finite yaw; TE_ERR_UNSUPPORTED for a polygon that reaches further than 31 cells; TE_ERR_MISSING_LAYER for
 *     verify_roughness without roughness), plus those of the selection and the yaws above and TE_ERR_BAD_ARG for an unknown
 *     memory mode.  Every argument error is found before anything is written: the te_map is then unchanged.
 *   - Lifetime, as each new map of the reference replaces the old one wholesale: te_map_chain(_batched, _batched_at),
 *     te_map_set_layers(_batched, _batched_at) and te_map_chain_image drop both layers (TE_ERR_MISSING_LAYER until the next
 *     call here); te_map_chain_maps(_at), te_map_set_layers_maps(_at) and te_map_chain_image_maps keep the batch's layers and fill
 *     the selected maps' with 0xffffffff, as for carried layers; every other entry leaves them as they are (te_map_clear_footprint
 *     too: resetTraversabilityFootprintLayers does not clear them).
 *   - Memory: 8 bytes per cell and map, resident from the first call until te_map_destroy; a selection uses the _maps scratch as
 *     te_map_footprint_maps does (plus 8 bytes per selected cell for host outputs).  Launches, whatever the maps, yaws and
 *     positions: the two predicate kernels and one sweep, plus for a selection the kernel that gathers its layers and, with
 *     outputs, the one that gathers those. */
int te_map_footprint_polygon_keep(te_map* map, const te_footprint_params* p, int32_t nsel, const int32_t* map_index_or_null,
                                  int32_t npts, const double* polygon_xy, int32_t nyaws, const double* footprint_yaw,
                                  float* traversability_x_or_null, float* traversability_rot_or_null, int memory);

/* A CheckFootprintPath request on the map, as the reference service loop answers it (TraversabilityEstimation.cpp:278-295, with
 * publishPolygons = true).  Arguments, outputs, conventions, limits and errors are those of te_check_footprint_request, with the
 * layers and the memory mode taken from the map: every array is in HOST memory (requests come from a ROS message); the call
 * validates the request, stages it to the device, runs the kernels of te_map_check_footprint_request_device with a work list
 * sized so that no path is cut, and returns synchronised.  One more limit: TE_ERR_UNSUPPORTED when the circular paths could make
 * more than 2^30 circle checks (see max_checks there; the work list would need over 100 GB).  Launches: those of
 * te_map_check_footprint_request_device, without the circular paths' when the request has none.  Planners whose requests live
 * on the device use te_map_check_footprint_request_device.  Paths run in request order.  A circular path's isTraversable calls
 * (:654-746) read and fill the cache exactly as the reference's do: a centre outside the map gives the default and stores
 * nothing; a cached cell (a finite value, isValid) gives its float32 value and is traversable iff it is != 0 (with
 * compute_untraversable_polygon, a cached 0 publishes Polygon::fromCircle); any other cell walks the spiral with this check's
 * radius, offset and flag, returns the double mean to the path sum and stores (float) of what the reference stores.  A walk can
 * store a NaN or an infinity (an invalid cell under a non-finite traversability_default, an infinite ring factor at offset 0):
 * the cell is then not cached, and the next check there walks again with its own radius and flag.  Checks after the first failure of a segment, and the
 * checks of a segment or pose whose checkInclination fails, do not run and store nothing.  Polygonal paths neither read nor
 * change the cache. */
int te_map_check_footprint_request(te_map* map, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                   const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                   const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative_or_null,
                                   const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe, double* traversability_out,
                                   double* area_out, int32_t max_vertices, int32_t* untraversable_count_or_null,
                                   double* untraversable_xy_or_null);

/* te_map_check_footprint_request on a batch: path q is on map path_map[q] (a host array, like every other request array; an
 * entry outside 0..nmaps-1 is TE_ERR_BAD_ARG, as is a null path_map).  Paths run in request order, each on its own map's layers,
 * cache and memo, so a map's answers and cache equal those of a single-map te_map given that map's paths in the same order; maps
 * may interleave and may have no paths.  The launches are those of one te_map_check_footprint_request, whatever nmaps. */
int te_map_check_footprint_request_batched(te_map* map, const te_footprint_params* p, const int32_t* path_map, int32_t npaths,
                                           int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius,
                                           int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                           int32_t max_footprint_vertices, const uint8_t* conservative_or_null,
                                           const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe,
                                           double* traversability_out, double* area_out, int32_t max_vertices,
                                           int32_t* untraversable_count_or_null, double* untraversable_xy_or_null);

/* te_map_check_footprint_request(_batched) with every array in DEVICE memory, for planners whose paths are made on the GPU: the
 * call is asynchronous on the context stream (te_set_stream), makes no host synchronisation and reads no request array on the
 * host, so it can be captured in a CUDA graph.  path_map_or_null: path q is on map path_map[q]; NULL only on a te_map of one map.
 * The host entries stage their arrays and run this same implementation, so for a valid request every output, the cache
 * afterwards and te_map_request_stats are, bit for bit, what the host entry returns and leaves for the same request on the same
 * map state.  Paths run in request order, each on its own map's layers, cache and
 * memo; a start index on the map's layers changes nothing (poses are map-frame positions, the layers are resident unwrapped).
 * Device-memory conventions, as te_check_footprint_request's: a path the library cannot check (a negative or NaN radius, more
 * than 127 rings, a non-finite x or y, a pose range outside 0..nposes, a map outside 0..nmaps-1, a bad footprint) gets is_safe
 * = 0, NaN traversability and area, and count -1 where its polygon was requested; it reads and stores nothing, so the other
 * paths and the cache equal a host request without it.
 * max_checks sizes the device work list of circle checks: one entry per isTraversable call a circular path could make (every
 * fourth LineIterator cell of an in-map segment, every single pose), plus one per check the host loop skips (a failed
 * checkInclination, a segment with an end outside the map), in request order.  When the request needs more, the first circular
 * path whose entries do not fit and every circular path after it get the convention above and store nothing; everything before
 * them is exact, so outputs and cache equal a host request of the paths that fit.  Polygonal paths do not use the list and are
 * always answered; max_checks = 0 answers only them.  The workspace is reserved from npaths, nposes, the maps and max_checks
 * (about 120 bytes per entry): a call with the same or smaller sizes allocates nothing.  Every call clears a hash table of
 * 2 * max_checks slots (8 bytes per entry), so a generous max_checks costs that memset on each call.  te_map_request_stats after a device
 * request synchronises the context stream and returns the counters the request left on the device (candidates, distinct keys,
 * stored cells; those of the host entry for the same request).
 * Errors, returned synchronously as by the host entry: TE_ERR_BAD_ARG for a map without layers, a NULL path_map on a batch, null
 * pointers, negative counts, max_footprint_vertices outside 0..16, max_vertices / polygon pointer mismatches, p->offset < 0 and
 * max_checks < 0; TE_ERR_UNSUPPORTED for max_checks > 2^30; TE_ERR_MISSING_LAYER for verify_roughness without a roughness layer.
 * Launches: the same kernels whatever npaths, nposes and the maps; te_get_stats counts 12 (13 with polygons, plus the polygonal
 * paths' 1-2), each of the three CUB scan / sort calls as one. */
int te_map_check_footprint_request_device(te_map* map, const te_footprint_params* p, const int32_t* path_map_or_null,
                                          int32_t npaths, int32_t nposes, const int32_t* path_begin, const double* poses,
                                          const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                          const float* footprint_xyz, int32_t max_footprint_vertices,
                                          const uint8_t* conservative_or_null, const uint8_t* compute_untraversable_polygon_or_null,
                                          uint8_t* is_safe, double* traversability_out, double* area_out, int32_t max_vertices,
                                          int32_t* untraversable_count_or_null, double* untraversable_xy_or_null, int64_t max_checks);

/* Maps with robots of their own (a mixed fleet, simulated environments with randomised robots): the three entries below take the
 * arguments of the entry they stand for with `params` instead of `p`, a HOST array of nmaps parameter sets indexed by map (not by
 * path, and for a selection still by map index), read before the call returns.  Map m's paths and sweep read params[m], as a
 * reference node reads its own robot's traversability_default, max_gap_width, critical_step_height, verify_roughness_footprint,
 * circular_footprint_offset and radius.
 *   - Per map: everything a call returns or stores for map m (request outputs and untraversable polygons, the cache, the memo,
 *     map m's share of te_map_request_stats) is, bit for bit, what the entry it stands for returns or stores on a single-map
 *     te_map holding map m at its position, given params[m].  With every params[m] equal (the radius aside for the requests,
 *     which take it per path), each entry is that entry given params[0], launches included.
 *   - The memo is kept per map: each map's bytes are cleared when its own max_gap_width, critical_step_height or verify_roughness
 *     differ from those its memo was filled under, and kept otherwise.  The single-parameter entries apply the same rule with p for
 *     every map.
 *   - Errors: every rule of the entry applies to each map's params[m] (TE_ERR_BAD_ARG for offset < 0 and, for the sweep, radius
 *     < 0; for the sweep TE_ERR_UNSUPPORTED for radius + offset over 120 cells; TE_ERR_MISSING_LAYER for verify_roughness without a roughness layer), over every map for a request and over the swept
 *     maps for the sweep; a null params is TE_ERR_BAD_ARG.  Every error is found on the host, before anything is written: the
 *     te_map is then unchanged.
 * Requests: the kernels of the entry they stand for, whatever nmaps and the parameters: a path's circle walks, dedup keys (the map
 * is part of every key, so two maps never share a walk), replay, polygons and polygonal items read its map's parameters from a
 * per-map table the te_map keeps on the device (40 bytes per map, uploaded only when its bytes change, so a call with unchanged
 * parameters makes no host synchronisation and can be captured in a CUDA graph).  When every map's entry is the same there is no
 * table. */
int te_map_check_footprint_request_each(te_map* map, const te_footprint_params* params, const int32_t* path_map, int32_t npaths,
                                        int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius,
                                        int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                        int32_t max_footprint_vertices, const uint8_t* conservative_or_null,
                                        const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe,
                                        double* traversability_out, double* area_out, int32_t max_vertices,
                                        int32_t* untraversable_count_or_null, double* untraversable_xy_or_null);
int te_map_check_footprint_request_device_each(te_map* map, const te_footprint_params* params, const int32_t* path_map_or_null,
                                               int32_t npaths, int32_t nposes, const int32_t* path_begin, const double* poses,
                                               const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                               const float* footprint_xyz, int32_t max_footprint_vertices,
                                               const uint8_t* conservative_or_null,
                                               const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe,
                                               double* traversability_out, double* area_out, int32_t max_vertices,
                                               int32_t* untraversable_count_or_null, double* untraversable_xy_or_null,
                                               int64_t max_checks);
/* traversabilityFootprint(radius, offset) on the caches of every map (nsel = 0, map_index_or_null NULL: te_map_footprint) or of the
 * maps map_index[0..nsel) (te_map_footprint_maps, whose rules apply), map m with params[m]; the output holds the swept caches
 * afterwards as that entry's does.  The swept maps are grouped by bitwise-identical params entries and each group is swept as one
 * te_map_footprint_maps selection: the sweep's per-radius tables stay kernel parameters.  Launches: those of te_map_footprint_maps
 * (without output) once per distinct parameter set, plus, with an output and more than one set, the gather of the swept caches
 * that te_map_get_footprint (a whole batch) or te_map_footprint_maps (a selection) makes for its output.  One set is the entry it
 * stands for, launches included; a te_map whose start index came in g holds one map, so it always has one set.  Each set
 * other than the previous sweep's rebuilds the sweep's tables on the host, as
 * te_map_footprint does when its parameters change.  Unknown memory modes are TE_ERR_BAD_ARG. */
int te_map_footprint_each(te_map* map, const te_footprint_params* params, int32_t nsel, const int32_t* map_index_or_null,
                          float* traversability_footprint_or_null, int memory);

/* The cache as publishTraversabilityMap publishes its traversability_footprint layer (in host memory: in the map's buffer
 * order; device memory needs a map without a start index), and resetTraversabilityFootprintLayers (:195-200).  On a batch: every
 * map's cache, back to back. */
int te_map_get_footprint(te_map* map, float* traversability_footprint, int memory);
/* The isTraversableForFilters memo the requests keep, one byte per cell of every map (maps back to back, each column-major in
 * default order, whatever its start index): 0 not evaluated since the memo was last cleared for that map, 1 passes, 2 blocked.
 * Host memory, returns synchronised.  No reference counterpart: it lets a caller see which maps' memo a call kept. */
int te_map_get_memo(te_map* map, uint8_t* memo);
/* resetTraversabilityFootprintLayers (:195-200): every map's cache empty, slope_footprint and step_footprint NaN (see te_layer);
 * roughness_footprint and the memo stay. */
int te_map_clear_footprint(te_map* map);

/* Counters of the last te_map_check_footprint_request(_batched): out[0] isTraversable calls its circular paths could make, out[1]
 * distinct circles among them (each is walked once on the device), out[2] cache stores the request made (its walks that ran);
 * totals over every map of a batch.  While every walk stores a finite value out[2] <= out[1]; a walk that stores a NaN or an
 * infinity leaves its cell uncached, so a later check there walks and stores again, and out[2] can exceed out[1].  No reference
 * counterpart. */
int te_map_request_stats(te_map* map, int64_t out[3]);

/* ---- The read side of a te_map: the layers the reference node publishes and serves ----------------------------------------
 * The layers, as bits of a mask; an output that holds several has them back to back in this order. */
typedef enum te_layer {
  TE_LAYER_TRAVERSABILITY = 1 << 0,
  TE_LAYER_SLOPE = 1 << 1,      /* traversability_slope */
  TE_LAYER_STEP = 1 << 2,       /* traversability_step */
  TE_LAYER_ROUGHNESS = 1 << 3,  /* traversability_roughness: te_map_chain, or te_map_set_layers with one */
  TE_LAYER_ELEVATION = 1 << 4,
  TE_LAYER_ROBOT_SLOPE = 1 << 5,  /* te_map_set_layers with one */
  TE_LAYER_FOOTPRINT = 1 << 6,  /* traversability_footprint: the cache (NaN = empty) */
  TE_LAYER_ALL = 0x7f,
  /* 1 << 7 is unassigned.  The elevation map's own layers, which the reference's filter chain carries into the traversability
   * map unchanged (mapOut = mapIn): te_map_carry_layers gives them.  The node asks the elevation mapping's submap service for
   * elevation plus upper_bound / lower_bound, or with a raw map for the variances and time (TraversabilityEstimation.cpp:60-69,
   * 264), and setElevationMap refuses a map without them (TraversabilityMap.cpp:145-150). */
  TE_LAYER_UPPER_BOUND = 1 << 8,
  TE_LAYER_LOWER_BOUND = 1 << 9,
  TE_LAYER_VARIANCE = 1 << 10,
  TE_LAYER_HORIZONTAL_VARIANCE_X = 1 << 11,
  TE_LAYER_HORIZONTAL_VARIANCE_Y = 1 << 12,
  TE_LAYER_HORIZONTAL_VARIANCE_XY = 1 << 13,
  TE_LAYER_TIME = 1 << 14,
  TE_LAYER_CARRIED = 0x7f00,  /* the seven bits above */
  /* upper_bound - lower_bound, derived when read: publishTraversabilityMap adds it to the copy it publishes
   * (TraversabilityMap.cpp:178-180).  te_map_get_layers only. */
  TE_LAYER_UNCERTAINTY_RANGE = 1 << 15,
  /* The traversability_footprint service's layers (TraversabilityMap.cpp:239-305): te_map_footprint_polygon_keep gives them. */
  TE_LAYER_TRAVERSABILITY_X = 1 << 16,
  TE_LAYER_TRAVERSABILITY_ROT = 1 << 17,
  /* 1 << 18 .. 1 << 20 are unassigned.  The layers isTraversableForFilters memoises its checks in (checkForSlope :867-893,
   * checkForStep :794-865, checkForRoughness :895-921): computeTraversability adds them all NaN (:225-228), and a check writes
   * 0.0 or 1.0 at a cell it visits whose own input layer (traversability_slope, _step, _roughness) is exactly 0.  The step check
   * runs only after the slope check passed, the roughness check only after both and with verify_roughness.  A te_map holds, per
   * map, what a reference node with that map's footprint parameters (its memo key, te_map_get_memo) holds after the same calls:
   *   - te_map_chain*, te_map_set_layers*, te_map_chain_image*, te_map_chain_submap / _windows and the _maps updates reset the
   *     selected maps' layers to NaN, as they empty the cache;
   *   - a request (te_map_check_footprint_request, _batched, _each, _device, _device_each) records every cell at which the
   *     service loop calls isTraversableForFilters, in order: a circle's walk only where the centre's traversability_footprint is
   *     not valid when the loop reaches it (:673), its spiral up to and including the first blocked cell (with
   *     compute_untraversable_polygon on to where the loop ends, :687-729); a polygonal item the path loop reaches, its
   *     PolygonIterator cells up to the first blocked one, or every one with compute_untraversable_polygon (:600-611).  Cells the
   *     request's kernels evaluate but the loop never reaches stay NaN;
   *   - te_map_footprint, _maps and _each (traversabilityFootprint(radius, offset), :307-318) record the spiral prefix of every
   *     centre whose cache cell is empty; on an empty cache that is every cell, with the values te_footprint2 returns in
   *     slope_fp / step_fp / rough_fp;
   *   - a change of a map's memo key (max_gap_width, critical_step_height, verify_roughness) by a request or a sweep resets that
   *     map's layers to NaN first;
   *   - te_map_clear_footprint (resetTraversabilityFootprintLayers, :195-200) resets slope_footprint and step_footprint and keeps
   *     roughness_footprint.
   * DIFFERENCE: the polygon sweeps (te_map_footprint_polygon, _yaws, _yaws_reduce, _keep) record nothing; the reference's
   * traversabilityFootprint(yaw) writes these layers at the cells its polygons visit (:601).
   * Served wherever TE_LAYER_FOOTPRINT is (te_map_get_layers, te_map_get_submaps(_batched), te_map_at_poses,
   * te_map_get_occupancy, te_map_get_point_cloud fields), NaN as the quiet NaN 0x7fc00000 of the reference's layers.  Every
   * te_map serves roughness_footprint (NaN where nothing wrote it); the reference's map has that layer only when
   * verify_roughness_footprint is set. */
  TE_LAYER_SLOPE_FOOTPRINT = 1 << 21,
  TE_LAYER_STEP_FOOTPRINT = 1 << 22,
  TE_LAYER_ROUGHNESS_FOOTPRINT = 1 << 23,
  TE_LAYER_FOOTPRINT_MEMO = 0xe00000  /* the three bits above */
} te_layer;

/* mapOut = mapIn for the layers the chain does not make: the carried layers of `layer_mask` (TE_LAYER_CARRIED bits) and
 * robot_slope (TE_LAYER_ROBOT_SLOPE) into the te_map, next to the layers te_map_chain / te_map_set_layers gave it.  A node that
 * initialises from a grid map with robot_slope (initializeTraversabilityMapFromGridMap, TraversabilityEstimation.cpp:331-362:
 * the layer survives computeTraversability, and checkInclination reads it, TraversabilityMap.cpp:748-762) calls te_map_chain and
 * then this, instead of copying the chain's outputs out and back through te_map_set_layers.  The image and init paths add
 * missing bounds as 0.0 (TraversabilityEstimation.cpp:159-161, 340-345): a NULL layer pointer does that.
 *   - layers: a HOST array of one pointer per set bit of layer_mask, in bit order; each is in `memory` or NULL (the layer is then
 *     filled with 0.0f on the device, as GridMap::add(layer, 0.0)).
 *   - nsel = 0 with map_index NULL: every map, each layer holding the nmaps maps back to back.  Host layers may carry the map's
 *     circular-buffer start index (unwrapped on upload, as te_map_set_layers); device layers are in default order.  Otherwise the
 *     maps map_index[0..nsel) only, under the rules of the _maps entries above (a host map_index of distinct entries, layers nsel
 *     maps back to back in map_index order, no start index), and only layers the batch already holds: every map of a batch
 *     holds the same layers, so a new layer is given to every map at once.
 *   - Leaves the cache and the memo as they are: no carried layer feeds isTraversableForFilters, and robot_slope only gates the
 *     later path checks (checkInclination).
 *   - Lifetime, as the reference's map is replaced wholesale by each new one: te_map_chain(_batched), te_map_set_layers(_batched)
 *     and te_map_chain_image drop every carried layer (as they drop robot_slope); te_map_chain_maps, te_map_set_layers_maps and
 *     te_map_chain_image_maps keep the batch's carried layers and fill the selected maps' with NaN (robot_slope keeps the rules
 *     of those entries).
 *   - Errors: TE_ERR_BAD_ARG for a map without layers, an empty mask or any other bit (the chain's layers, the cache,
 *     uncertainty_range, 1 << 7, unknown bits), a null layers array, an unknown memory mode, a bad selection and a layer the
 *     batch does not hold given to a selection; TE_ERR_UNSUPPORTED for a selection on a map with a start index.  Every argument
 *     error is found before anything is written: the te_map is then unchanged.
 *   - Memory: a resident buffer of 4 bytes per cell and map per carried layer, allocated on first use and released by
 *     te_map_destroy.  A selection in host memory stages its layers in the _maps scratch (4 bytes per given layer and selected
 *     cell).  Launches: one kernel that puts a selection in place and fills its NULL layers, or for every map one fill kernel
 *     when a pointer is NULL (none otherwise).  Host memory returns synchronised; device memory is asynchronous. */
int te_map_carry_layers(te_map* map, int32_t nsel, const int32_t* map_index_or_null, uint32_t layer_mask, const float* layers[],
                        int memory);

/* One window of GridMap::getSubmap(position, length, isSuccess) (TraversabilityEstimation.cpp:305, getSubmapInformation; SURVEY.md
 * A.1, recalled from grid_map 1.6.x).  The submap is the block [top_row, top_row + rows) x [top_col, top_col + cols) of the map in
 * default (unwrapped) order, with start index 0: a circular-buffer start index changes no field.  requested_row / requested_col
 * is the requested position's index in the submap (indexInSubmap).  A failed window (success 0: isSuccess false, e.g. a position
 * outside the map) has every field 0 but offset, as getSubmap returns an empty map.  offset: floats before the window's layers in
 * te_map_get_submaps's output (te_submap_geometry: with one layer per window); a failed window takes no space. */
typedef struct te_submap_info {
  int32_t success;
  int32_t rows, cols;
  int32_t top_row, top_col;
  int32_t requested_row, requested_col;
  int32_t reserved;
  double length_x, length_y;
  double position_x, position_y;
  int64_t offset;
} te_submap_info;

/* The submap geometry of n windows (position_xy, length_xy: n (x, y) pairs each) on the map `g`.  Host arithmetic, no GPU needed.
 * TE_ERR_BAD_ARG for a negative or non-finite length or position (the reference does not check them: a negative length makes
 * blocks of negative size), before any record is written. */
int te_submap_geometry(const te_geometry* g, int32_t n, const double* position_xy, const double* length_xy, te_submap_info* info);

/* ---- Updates from a larger elevation map: the reference node's main update path --------------------------------------------
 * updateTraversability (TraversabilityEstimation.cpp:202-222) asks elevation mapping for getSubmap(robot position, mapLength_) with
 * the layers of elevationMapLayers_ (elevation plus upper_bound / lower_bound, or the variances and time for a raw map,
 * TraversabilityMap.cpp:64-76), and setElevationMap (:135-154) hands that submap to computeTraversability (mapOut = mapIn).  The two
 * entries below cut the windows out of the larger map on the GPU and chain them, in one call.
 *   - src: the elevation map, with any circular-buffer start index (elevation mapping's moves).  src_mask: TE_LAYER_ELEVATION
 *     (required) and any of TE_LAYER_CARRIED; src_layers: a HOST array of one pointer per set bit, in bit order, each a whole map
 *     of src's size in its buffer order, in `memory`.  robot_slope is not a source layer: elevationMapLayers_ never holds it.
 *   - Device memory reads the source in place and is asynchronous on the context stream.  Host memory stages only the source
 *     columns the windows touch (one copy per contiguous run of stored columns and layer, through the context's staging buffers)
 *     and returns synchronised.  Neither can be captured in a CUDA graph: the chain synchronises for its escalation counters.
 *   - Errors, every argument error found before anything is written (the te_map is then unchanged): TE_ERR_BAD_ARG for a bad src
 *     geometry or start index, a src_mask without elevation or with other bits, a null src_layers, an unknown memory mode, a
 *     non-finite position, a non-finite or negative length, and a window whose indices on the source do not fit in int32;
 *     TE_ERR_MISSING_LAYER for a NULL layer the mask names; those of the chain parameters.
 *   - Launches: those of the chain entry the call stands for (below), plus one k_map_cut_windows, whatever the windows and layers:
 *     the carried layers are cut straight into their place. */

/* getSubmap(position, length) on src, then te_map_chain on the submap's elevation and te_map_carry_layers on its other layers: the
 * te_map becomes one map of the submap's geometry (start index 0) and holds, bit for bit, the layers, cache, memo, requests,
 * submaps and te_map_get_layers that te_map_chain(g_sub, elevation) followed by te_map_carry_layers(its carried layers) give, g_sub
 * and the layers being getSubmap's (te_submap_geometry: bounding at the edges, so clipped there).  info receives te_submap_geometry's
 * record.  When getSubmap's isSuccess is false (info->success = 0) the call returns TE_ERR_BAD_ARG and leaves the te_map as it was,
 * as the reference node skips the update when its submap request fails. */
int te_map_chain_submap(te_map* map, const te_geometry* src, uint32_t src_mask, const float* src_layers[], double position_x,
                        double position_y, double length_x, double length_y, const te_chain_params* p, te_submap_info* info, int memory);

/* One window of src per map of a batch, in one call: a fleet of robot-centric maps cut out of one shared map (a GPU elevation
 * mapper, a global map, a simulator's terrain).  map_index_or_null NULL reloads the whole batch with nmaps maps, under the rules of
 * te_map_chain_batched_at; otherwise the nmaps maps map_index[0..nmaps) are updated under the rules of te_map_chain_maps_at (distinct
 * host indices, g checked against the batch except for its position, the robot_slope / roughness refusal, the traversability_x /
 * _rot fill) and every other map keeps its layers, cache and memo.  position_xy: a HOST array of the requested (robot) positions,
 * one (x, y) pair per map updated.
 *   - Window rule.  A batch has one size (rows n, cols m of g), while getSubmap's size moves by a cell with the position, so a
 *     window is getSubmap's top-left with the batch's size.  g->resolution must equal src's bit for bit (TE_ERR_BAD_ARG): cells are
 *     copied, not resampled.  The top-left corner (x + 0.5 g->length_x, y + 0.5 g->length_y) is indexed with getIndex's
 *     expressions, floored and not checked against the source: (ti, tj), which may be negative or past the source.  Map cell (i, j)
 *     is source cell (ti + i, tj + j), NaN 0x7fc00000 (the unknown cell) outside the source.  The map's position is getSubmap's at
 *     that size: getPosition(ti, tj) + 0.5 res - 0.5 (n res), likewise in y (te_map_positions returns it).  For a window at least
 *     one cell inside the source on every side, where te_submap_geometry(src, (x, y), g's length) has size (n, m), top-left,
 *     position and cells are getSubmap's, bit for bit.
 *   - Carried layers as te_map_carry_layers gives them: a whole-batch reload holds exactly those of src_mask; a selection may give
 *     only layers the batch holds (TE_ERR_BAD_ARG otherwise), and the batch's other carried layers of the selected maps are filled
 *     with NaN as te_map_chain_maps_at fills them.
 *   - For every map, everything the te_map returns or stores equals, bit for bit, what te_map_chain_batched_at /
 *     te_map_chain_maps_at at the window positions, followed by te_map_carry_layers, give on the cut layers.
 *   - Launches: those of te_map_chain_batched_at / te_map_chain_maps_at on the same maps and positions plus one (on a selection of a
 *     batch that holds more than eight carried and traversability_x / _rot layers, one fill launch fewer when the given layers bring
 *     the fill under nine).  A selection uses the scratch of te_map_chain_maps (16 bytes per selected cell) plus the cut elevation
 *     (4); the window table is 8 bytes per window and layer plus 8 per window, and 4 per source column in host memory. */
int te_map_chain_windows(te_map* map, const te_geometry* g, const te_geometry* src, uint32_t src_mask, const float* src_layers[],
                         int32_t nmaps, const int32_t* map_index_or_null, const double* position_xy, const te_chain_params* p, int memory);

/* publishTraversabilityMap (TraversabilityMap.cpp:172-186): the layers of `layer_mask` (te_layer bits), each rows x cols, back to
 * back in bit order (on a batch: per layer the nmaps maps back to back, nmaps*rows*cols floats a layer).  In host memory each is re-wrapped to the map's start index, as te_map's other outputs, and the call returns
 * synchronised; in device memory they are in the map's default (unwrapped) order, asynchronously.  TE_ERR_MISSING_LAYER for a
 * layer the map does not hold (roughness after te_map_set_layers without it, robot_slope after te_map_chain, a carried layer
 * te_map_carry_layers did not give since the last whole-map update, traversability_x / _rot before te_map_footprint_polygon_keep);
 * TE_ERR_BAD_ARG for an empty mask or unknown bits.
 * TE_LAYER_UNCERTAINTY_RANGE is upper_bound - lower_bound, one IEEE float32 subtraction per cell computed on the device
 * (TraversabilityMap.cpp:178-180), with NaN results carrying the payload an x86-64 host's subtraction gives them (the first NaN
 * operand, quieted; 0xffc00000 for Inf - Inf), so bit for bit what the reference publishes there.  It needs both bounds
 * (TE_ERR_MISSING_LAYER otherwise).  In host memory it goes through a staging buffer of 4 bytes per cell of every map. */
int te_map_get_layers(te_map* map, uint32_t layer_mask, float* out, int memory);

/* The get_traversability_map service (TraversabilityEstimation.cpp:297-316) for nwin windows in one call: info[k] as
 * te_submap_geometry gives it, and window k's layers of `layer_mask` from out + info[k].offset on, in bit order, each
 * rows_k x cols_k column-major with start index 0, as getSubmap returns them.  position_xy, length_xy and info are host arrays;
 * `out` is in `memory` (host: returns synchronised; device: asynchronous on the context stream).  When the windows take more
 * than out_capacity floats the call fills info, writes nothing else and returns TE_ERR_BAD_ARG: the total is the last record's
 * offset plus its layers, so the caller can call again with more room.  One kernel launch for all windows and layers (none when
 * every window fails).  Layer errors as te_map_get_layers, except that TE_LAYER_UNCERTAINTY_RANGE is TE_ERR_BAD_ARG: the
 * service cuts its submaps from the traversability map itself (TraversabilityEstimation.cpp:303-313), which has no such layer.
 * Window errors as te_submap_geometry. */
int te_map_get_submaps(te_map* map, int32_t nwin, const double* position_xy, const double* length_xy, uint32_t layer_mask,
                       te_submap_info* info, float* out, int64_t out_capacity, int memory);

/* te_map_get_submaps on a batch: window k is taken from map win_map[k] (a host array; an entry outside 0..nmaps-1 is
 * TE_ERR_BAD_ARG).  Output layout, te_submap_info and the capacity protocol are those of te_map_get_submaps. */
int te_map_get_submaps_batched(te_map* map, int32_t nwin, const int32_t* win_map, const double* position_xy, const double* length_xy,
                               uint32_t layer_mask, te_submap_info* info, float* out, int64_t out_capacity, int memory);

/* mapHasValidTraversabilityAt (TraversabilityMap.cpp:971-983) for n positions (xy: n (x, y) pairs): valid[q] = 1 when getIndex
 * finds the position in the map and traversability is finite there, else 0.  xy and valid are in `memory`; device memory is
 * asynchronous on the context stream. */
int te_map_valid_at(te_map* map, int32_t n, const double* xy, uint8_t* valid, int memory);

/* te_map_valid_at on a batch: position q is on map pos_map[q]; pos_map, xy and valid are in `memory`.  In host memory a map
 * outside 0..nmaps-1 is TE_ERR_BAD_ARG; in device memory (not read on the host) that position gets 0. */
int te_map_valid_at_batched(te_map* map, int32_t n, const int32_t* pos_map, const double* xy, uint8_t* valid, int memory);

/* GridMap::atPosition(layer, position), as checkInclination reads robot_slope (TraversabilityMap.cpp:751), at npoints robot-frame
 * points around each of nposes poses, for every layer of `layer_mask`, in one kernel launch.
 *   - poses: 7 doubles per pose, x y z qx qy qz qw (geometry_msgs/Pose order).  points_xyz: 3 floats per point, x y z
 *     (geometry_msgs/Point32 order).  Point t of pose k lies at `toPosition * orientation * point`, computed as
 *     checkPolygonalFootprintPath places a footprint vertex (:488-507): the quaternion as given, not normalised, and the z of the
 *     result dropped.  The single point (0, 0, 0) gives the pose's (x, y) exactly, so that is plain atPosition at a list of
 *     positions.
 *   - pose k is on map pose_map[k], at that map's own position (te_map_positions); pose_map may be NULL on a te_map of one map.
 *     Positions are map-frame: a start index changes nothing, as in grid_map, since the layers are resident unwrapped.
 *   - layer_mask: any te_layer bits the map holds, TE_LAYER_FOOTPRINT (the cache, NaN where empty), the carried layers,
 *     TE_LAYER_TRAVERSABILITY_X / _ROT and TE_LAYER_UNCERTAINTY_RANGE (upper_bound - lower_bound at the cell, bit for bit as
 *     te_map_get_layers computes it) included.
 *   - out: per layer in bit order nposes * npoints floats, pose-major: layer l of point t of pose k at out[(l * nposes + k) *
 *     npoints + t].  A valid point (its pose's map in the batch, x and y finite, getIndex finds the cell) gets the cell's float32
 *     bits exactly, NaN payloads included; any other point, where atPosition would throw, gets NaN 0x7fc00000.
 *     valid_or_null[k * npoints + t] is 1 for a valid point and 0 otherwise.
 * Every array is in `memory`.  Host memory returns synchronised.  Device memory is asynchronous on the context stream: no host
 * synchronisation and no argument array read on the host, so the call can be captured in a CUDA graph.  nposes = 0 launches
 * nothing.  Errors, all found before anything is written: TE_ERR_BAD_ARG for a map without layers, an empty mask or unknown bits,
 * null poses / points_xyz / out, nposes < 0, npoints < 1, an unknown memory mode, a NULL pose_map on a batch and, in host memory
 * only, a pose_map entry outside 0..nmaps-1 (in device memory that pose's points are invalid, as in te_map_valid_at_batched);
 * TE_ERR_MISSING_LAYER as te_map_get_layers; TE_ERR_UNSUPPORTED for nposes * npoints >= 2^31. */
int te_map_at_poses(te_map* map, const int32_t* pose_map_or_null, int32_t nposes, const double* poses, int32_t npoints,
                    const float* points_xyz, uint32_t layer_mask, float* out, uint8_t* valid_or_null, int memory);

/* ---- Occupancy grids (GridMapRosConverter::toOccupancyGrid), as grid_map_visualization publishes a traversability map -------
 * visualization.launch with config/visualization/traversability.yaml publishes traversability, traversability_slope,
 * traversability_step and traversability_roughness as nav_msgs/OccupancyGrid, each with data_min 1.0 and data_max 0.0 (SURVEY.md
 * A.7).  The entries below give the grids' data and MapMetaData; headers, stamps and frame ids stay the caller's. */

/* nav_msgs/MapMetaData of a grid (its map_load_time is the caller's). */
typedef struct te_occupancy_info {
  int32_t width, height;      /* getSize(): rows, cols */
  float resolution;           /* (float)resolution */
  int32_t reserved;
  double origin_x, origin_y;  /* getPosition() - 0.5 * getLength(), per axis in double; z 0, orientation identity */
} te_occupancy_info;

/* The MapMetaData of n grids of maps of geometry g: record k at position (position_xy[2k], position_xy[2k + 1]), or, with
 * position_xy_or_null NULL, n records at g's position (te_map_positions gives a batch's positions).  g's start index changes
 * nothing.  Host arithmetic, no GPU needed.  TE_ERR_BAD_ARG for a null or bad geometry, n < 0, a null out (n > 0) and a non-finite
 * position, before any record is written. */
int te_occupancy_grid_info(const te_geometry* g, int32_t n, const double* position_xy_or_null, te_occupancy_info* out);

/* toOccupancyGrid of every layer of layer_mask for the maps of the call, in one kernel launch.
 *   - Maps: nsel 0 with map_index_or_null NULL is every map of the batch; otherwise the maps map_index[0..nsel), a HOST array of
 *     distinct indices in 0..nmaps-1 in any order, read before the call returns, as for the _maps entries.  Start indices never
 *     matter, so every te_map takes a selection, one whose start index came in g included.
 *   - Layers: any bits te_map_get_layers accepts, with its TE_ERR_MISSING_LAYER rules: the carried layers, robot_slope, the
 *     traversability_footprint cache (NaN where empty), traversability_x / _rot, and TE_LAYER_UNCERTAINTY_RANGE (upper_bound -
 *     lower_bound, one IEEE float32 subtraction per cell; its NaN payload does not matter, NaN gives -1).
 *   - Ranges: data_min and data_max are HOST arrays of one float per set bit, in bit order: each layer has its own range.
 *   - Cells: value = (v - data_min) / (data_max - data_min), each step one IEEE float32 operation rounded to nearest; NaN gives -1,
 *     anything else 0 + min(max(0, value), 1) * 100, truncated toward zero.  So data_max == data_min gives 0 or 100 (+-Inf clamped),
 *     or -1 where v equals data_min; a NaN or Inf bound is not checked and gives the formula's result.
 *   - Output: per layer in bit order, the call's maps back to back in call order, rows*cols bytes each: map block k of layer l
 *     starts at byte (l * n + k) * rows * cols, n the maps of the call.  A block is the map's grid: cell (i, j) of the map in
 *     default (unwrapped) order at byte rows*cols - 1 - (j*rows + i), whatever its start index (unlike te_map_get_layers, whose
 *     host output is re-wrapped).  Reshaped (cols, rows) in C order it is OccupancyGrid.data as (height, width).
 *   - Memory: host memory writes the grids into staging and copies them back once; the call returns synchronised.  Device
 *     memory is asynchronous on the context stream, with no host synchronisation and no allocation once the scratch exists.  A
 *     whole-batch device call passes everything to the kernel by value, so it can be captured in a CUDA graph; a selection
 *     uploads its slot table as the _maps entries do, and is not promised to be capturable.
 *   - Errors, every one found before anything is written (out is then untouched): TE_ERR_BAD_ARG for a map without layers, an
 *     empty mask or unknown bits, a null data_min, data_max or out, an unknown memory mode and a bad selection;
 *     TE_ERR_MISSING_LAYER as te_map_get_layers. */
int te_map_get_occupancy(te_map* map, int32_t nsel, const int32_t* map_index_or_null, uint32_t layer_mask, const float* data_min,
                         const float* data_max, int8_t* out, int memory);

/* ---- Point clouds (GridMapRosConverter::toPointCloud), as grid_map_visualization publishes a traversability map -------------
 * visualization.launch with config/visualization/traversability.yaml publishes traversability_cloud, type point_cloud with layer
 * elevation: PointCloudVisualization::visualize calls toPointCloud(map, "elevation", cloud), which passes every layer of the map in
 * message order (SURVEY.md A.8, recalled from grid_map_ros 1.6.x).  The entry below gives the clouds' PointCloud2.data and widths;
 * the header, stamp and frame id stay the caller's.
 *
 * The field layout, one rule: one float32 field per entry of `fields`, 4 bytes each at consecutive offsets, the entry equal to
 * point_layer replaced by three fields x, y, z; point_step = 4 * the number of fields; height 1, is_dense false, width = the map's
 * points, row_step = width * point_step.
 *
 * toPointCloud for the maps of the call, in a fixed number of launches (te_get_stats counts 3: a count kernel, one cub scan, a
 * scatter kernel), whatever the maps, fields, start indices and points.
 *   - Maps: nsel 0 with map_index_or_null NULL is every map of the batch; otherwise the maps map_index[0..nsel), a HOST array of
 *     distinct indices in 0..nmaps-1 in any order, read before the call returns.  Every te_map takes a selection, one whose start
 *     index came in g included: each map is read in its own buffer order and at its own position.
 *   - fields: a HOST array of nfields (1..32) entries in the published map's layer order.  Each is one te_layer bit that
 *     te_map_get_layers accepts (the carried layers, robot_slope, TE_LAYER_FOOTPRINT (the cache, NaN where empty),
 *     traversability_x / _rot, TE_LAYER_UNCERTAINTY_RANGE with te_map_get_layers' NaN-payload rule, TE_LAYER_SLOPE_FOOTPRINT /
 *     _STEP_FOOTPRINT / _ROUGHNESS_FOOTPRINT as the te_map recorded them), at most once, or 0: a field holding NaN 0x7fc00000 at
 *     every point, as the reference publishes a layer nothing wrote (computeTraversability's add(), TraversabilityMap.cpp:225-228).
 *   - point_layer: one te_layer bit the map holds.  It decides which cells are points; it need not be in `fields`, and then the
 *     records have no x, y, z, as in the reference.
 *   - basic_mask: the map's basic layers as te_layer bits (0: none, as in the reference's bags).
 *   - Points: the cells of each map in its buffer order (linear index k: buffer cell (k % rows, k / rows) under the map's start
 *     index, as GridMapIterator walks it), keeping those where the point layer and, when basic_mask is not 0, every basic layer
 *     is finite (getPosition3, isValid).  x, y: (float) of getPosition of the cell, on its unwrapped index at its map's position
 *     (te_grid.cuh's cell_coord), rounded to nearest; z and every other field: the float32 bits as stored, NaN payloads and -0.0
 *     included.  This order holds in both memory modes.
 *   - Output: offsets, nsel + 1 (or nmaps + 1) int64 in `memory`: offsets[0] = 0, map k of the call has width offsets[k + 1] -
 *     offsets[k] and its blob starts at byte point_step * offsets[k] of `data`; the blobs are back to back in call order.
 *   - Capacity, in points: host memory, when the clouds hold more than capacity_points the call fills offsets, writes nothing to
 *     data and returns TE_ERR_BAD_ARG (capacity 0 with a NULL data is a sizing query); device memory, offsets are always complete
 *     and points at or past capacity_points are not written, so the call reads nothing back.
 *   - Memory: host memory computes the offsets on the device and copies them back once, then writes the records into staging and
 *     copies back total * point_step bytes; the call returns synchronised.  Device memory is asynchronous on the context stream,
 *     with no host synchronisation and no allocation once the scratch exists (16 bytes per tile of 1024 cells plus the scan's).
 *     A whole-batch device call passes its arguments by value (maps at several positions or start indices read a per-map table
 *     uploaded when it changes), so it can be captured in a CUDA graph; a selection uploads its table as the _maps entries do.
 *   - Errors, every one found before anything is written: TE_ERR_BAD_ARG for a map without layers, nfields outside 1..32, a null
 *     fields or offsets, a null data with capacity_points > 0, a negative capacity_points, an entry that is neither 0 nor one known
 *     bit or that repeats one, a point_layer that is not one known bit, unknown bits in basic_mask, an unknown memory mode and a
 *     bad selection; TE_ERR_MISSING_LAYER as te_map_get_layers for the field, point and basic layers. */
int te_map_get_point_cloud(te_map* map, int32_t nsel, const int32_t* map_index_or_null, int32_t nfields, const uint32_t* fields,
                           uint32_t point_layer, uint32_t basic_mask, void* data, int64_t capacity_points, int64_t* offsets,
                           int memory);

/* ---- Multi-GPU: one map tiled into column slabs, one process (rank) per GPU (SURVEY.md §8e) -------------------------------
 * The chain and the footprint sweep are stencils of fixed radius, so the only exchange step is a one-shot copy of the
 * neighbours' boundary columns of the INPUT layer(s) into this rank's halo.  The reference has no counterpart (it is a
 * single-process CPU node; TraversabilityMap.cpp:202-237 runs the chain on one whole map); these entry points are what a
 * sharded caller of te_chain / te_footprint needs around the `te_slab` argument:
 *   1. every rank exports its slab buffer (te_ipc_export) and a "layer ready" event (te_event_create_ipc), ships the two
 *      handles (TE_IPC_HANDLE_BYTES and 64 bytes) to its neighbours over any channel (MPI, a socket, torch.distributed), and opens theirs
 *      (te_ipc_open / te_event_open_ipc) — once;
 *   2. per map: te_event_record(ready) after the rank's producer wrote its owned columns; te_halo_pull() then waits for the
 *      neighbours' ready events on the context stream and copies their boundary columns straight out of their buffers over
 *      NVLink (peer-mapped cudaMemcpyAsync, no staging, no collective); te_chain(..., slab, ..., TE_MEM_DEVICE) follows on the
 *      same stream.  Outputs stay sharded.
 * A cross-process event wait sees the most recent te_event_record that the RECORDING process had issued when the waiting
 * process called te_halo_pull; callers that rewrite a layer per frame order the two host-side (a message after the record)
 * and must not overwrite boundary columns a neighbour may still be pulling (double-buffer, or wait for the neighbour's own
 * event recorded after its pull). */
#define TE_IPC_HANDLE_BYTES 80 /* CUDA IPC handle of the containing allocation + offset of the pointer inside it */
int te_ipc_export(const void* device_ptr, void* handle_TE_IPC_HANDLE_BYTES);
int te_ipc_open(const void* handle_TE_IPC_HANDLE_BYTES, void** device_ptr_out);
int te_ipc_close(void* device_ptr);
/* Interprocess events (cudaEventInterprocess | cudaEventDisableTiming). */
int te_event_create_ipc(te_ctx* ctx, void** event_out, void* handle_64_bytes_out);
int te_event_open_ipc(const void* handle_64_bytes, void** event_out);
int te_event_record(te_ctx* ctx, void* event);   /* on the context stream */
int te_event_destroy(void* event);

/* A neighbour's slab buffer as mapped into this process: `layer` holds the global columns
 * [slab.col_begin - slab.halo_left, slab.col_begin + slab.col_count + slab.halo_right) of a rows x cols layer. */
typedef struct te_halo_peer {
  const float* layer;   /* te_ipc_open()ed pointer (or a plain device pointer of a peer-accessible GPU in this process) */
  te_slab slab;         /* the neighbour's slab */
  void* ready_event;    /* te_event_open_ipc()ed event, or NULL: no wait */
} te_halo_peer;

/* Fill this rank's halo columns of `layer` (a buffer laid out like the te_chain input for `slab`) from the neighbours' OWNED
 * columns, asynchronously on the context stream.  The exchange is one hop: TE_ERR_BAD_ARG if a neighbour owns fewer columns
 * than the halo needs.  Pass NULL for a side without a neighbour (map edge). */
int te_halo_pull(te_ctx* ctx, const te_geometry* g, const te_slab* slab, float* layer,
                 const te_halo_peer* left_or_null, const te_halo_peer* right_or_null);

#ifdef __cplusplus
}
#endif
#endif
