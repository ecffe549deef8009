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
 * out: traversability_footprint; slope_footprint/step_footprint memoisation layers optional. */
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
 * elevation and robot_slope (optional); the traversability_footprint cache (float32, NaN = empty); and the isTraversableForFilters
 * memo, which is kept until the layers or one of max_gap_width, critical_step_height and verify_roughness change.  Whole maps only.
 * Host layers may carry a circular-buffer start index: they are unwrapped on upload and outputs are re-wrapped to the start index
 * of the last te_map_chain / te_map_set_layers.  Every entry but te_map_create / te_map_destroy fails with TE_ERR_BAD_ARG before
 * layers were set.  Host-memory entries return synchronised; device-memory ones are asynchronous on the context stream. */
typedef struct te_map te_map;
int te_map_create(te_ctx* ctx, te_map** out);
int te_map_destroy(te_map* map);

/* computeTraversability (:202-237): te_chain on `elevation` into the map's layers, each optionally copied out (NULL: kept on the
 * device only).  Empties the cache and the memo and leaves the map without robot_slope. */
int te_map_chain(te_map* map, const te_geometry* g, const te_chain_params* p, const float* elevation, float* slope_or_null,
                 float* step_or_null, float* roughness_or_null, float* traversability_or_null, int memory);

/* setTraversabilityMap: the layers as given (a map received or loaded from a bag).  Empties the cache and the memo.
 * TE_ERR_MISSING_LAYER for a missing required layer. */
int te_map_set_layers(te_map* map, const te_geometry* g, const float* traversability, const float* slope, const float* step,
                      const float* roughness_or_null, const float* elevation, const float* robot_slope_or_null, int memory);

/* traversabilityFootprint(radius, offset) (:307-318) on the cache: a cached cell keeps its value (the memoised branch, :673-675),
 * every other cell gets te_footprint2's value for `p`; traversability_footprint_or_null receives the cache afterwards.  The
 * prefix-sum sweep may differ from the visit-by-visit one in the last float32 bit of a few cells (DESIGN.md §4.3); those values
 * then stay in the cache.  Errors as te_footprint2 (TE_ERR_MISSING_LAYER: verify_roughness without a roughness layer). */
int te_map_footprint(te_map* map, const te_footprint_params* p, float* traversability_footprint_or_null, int memory);

/* traversabilityFootprint(yaw) (:239-305): te_footprint_polygon on the map's layers.  Reads and changes no cache. */
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

/* A CheckFootprintPath request on the map, as the reference service loop answers it (TraversabilityEstimation.cpp:278-295, with
 * publishPolygons = true).  Arguments, outputs, conventions, limits and errors are those of te_check_footprint_request, with the
 * layers and the memory mode taken from the map: every array is in HOST memory (requests come from a ROS message, and which checks
 * run depends on values earlier checks cached, which the host resolves); the call returns synchronised.  Planners whose requests
 * live on the device use te_check_footprint_request.  Paths run in request order.  A circular path's isTraversable calls
 * (:654-746) read and fill the cache exactly as the reference's do: a centre outside the map gives the default and stores
 * nothing; a cached cell gives its float32 value and is traversable iff it is != 0 (with compute_untraversable_polygon, a cached 0
 * publishes Polygon::fromCircle); any other cell walks the spiral with this check's radius, offset and flag, returns the double
 * mean to the path sum and stores (float) of what the reference stores.  Checks after the first failure of a segment, and the
 * checks of a segment or pose whose checkInclination fails, do not run and store nothing.  Polygonal paths neither read nor
 * change the cache. */
int te_map_check_footprint_request(te_map* map, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                   const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                   const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative_or_null,
                                   const uint8_t* compute_untraversable_polygon_or_null, uint8_t* is_safe, double* traversability_out,
                                   double* area_out, int32_t max_vertices, int32_t* untraversable_count_or_null,
                                   double* untraversable_xy_or_null);

/* The cache as publishTraversabilityMap publishes its traversability_footprint layer (in host memory: in the map's buffer
 * order; device memory needs a map without a start index), and resetTraversabilityFootprintLayers (:195-200). */
int te_map_get_footprint(te_map* map, float* traversability_footprint, int memory);
int te_map_clear_footprint(te_map* map);

/* Counters of the last te_map_check_footprint_request: out[0] isTraversable calls its circular paths could make, out[1] distinct
 * circles among them (each is walked once on the device), out[2] cache cells the request stored.  No reference counterpart. */
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
  TE_LAYER_ALL = 0x7f
} te_layer;

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

/* publishTraversabilityMap (TraversabilityMap.cpp:172-186): the layers of `layer_mask` (te_layer bits), each rows x cols, back to
 * back in bit order.  In host memory each is re-wrapped to the map's start index, as te_map's other outputs, and the call returns
 * synchronised; in device memory they are in the map's default (unwrapped) order, asynchronously.  TE_ERR_MISSING_LAYER for a
 * layer the map does not hold (roughness after te_map_set_layers without it, robot_slope after te_map_chain); TE_ERR_BAD_ARG
 * for an empty mask or unknown bits. */
int te_map_get_layers(te_map* map, uint32_t layer_mask, float* out, int memory);

/* The get_traversability_map service (TraversabilityEstimation.cpp:297-316) for nwin windows in one call: info[k] as
 * te_submap_geometry gives it, and window k's layers of `layer_mask` from out + info[k].offset on, in bit order, each
 * rows_k x cols_k column-major with start index 0, as getSubmap returns them.  position_xy, length_xy and info are host arrays;
 * `out` is in `memory` (host: returns synchronised; device: asynchronous on the context stream).  When the windows take more
 * than out_capacity floats the call fills info, writes nothing else and returns TE_ERR_BAD_ARG: the total is the last record's
 * offset plus its layers, so the caller can call again with more room.  One kernel launch for all windows and layers (none when
 * every window fails).  Layer errors as te_map_get_layers; window errors as te_submap_geometry. */
int te_map_get_submaps(te_map* map, int32_t nwin, const double* position_xy, const double* length_xy, uint32_t layer_mask,
                       te_submap_info* info, float* out, int64_t out_capacity, int memory);

/* mapHasValidTraversabilityAt (TraversabilityMap.cpp:971-983) for n positions (xy: n (x, y) pairs): valid[q] = 1 when getIndex
 * finds the position in the map and traversability is finite there, else 0.  xy and valid are in `memory`; device memory is
 * asynchronous on the context stream. */
int te_map_valid_at(te_map* map, int32_t n, const double* xy, uint8_t* valid, int memory);

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
