// te_capi_host.h — what the two host units of the C API share (te_capi.cu: the context and the stateless entries; te_map.cu:
// the resident te_map).  Declarations only: every definition is in te_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/te_b200.h"
#include "te_kernels.h"
#include "te_fused.h"
#include "te_footprint.h"

struct te_ctx {
  int device = 0;
  int sms = 132;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  int kernel_choice = TE_KERNEL_AUTO;
  int64_t launches = 0;
  int64_t slow_cells = 0;

  te_geometry geo{};
  bool have_geo = false;
  te::DevBuf dX, dY;
  std::vector<double> hX, hY;

  te::DevBuf stage[20];          // TE_MEM_HOST staging (handed out in order by Staging; te_check_footprint_request_batched takes 19)
  te::DevBuf worklist, worklist3, counter;  // fused-kernel fix-up lists (tier 2, tier 3) and their counters
  // The counters are two 512-byte blocks used alternately: the last kernel of a chain call (k_fixup_cells) zeroes the block of the
  // NEXT call, so a call needs no cudaMemsetAsync of its own (one stream operation and one launch gap less per map).
  int counter_phase = 0;    // block of the most recent fused launch (what the statistics entry points read)
  int counter_clean = -1;   // block known to be zero on the stream (-1: none)
  cudaStream_t counter_stream = nullptr;  // the stream whose order that knowledge belongs to
  te::FusedState fused;      // tensor maps / tables of the fused stencil
  te::FootprintState fp;

  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;  // te_chain(TE_MEM_HOST) pipeline
  bool timing = false;
  struct Ev3 { cudaEvent_t a, b, c; };
  std::vector<Ev3> events;   // timing events, created once and reused (te_get_timing rewinds events_used)
  size_t events_used = 0;
};

namespace te {
namespace host {

// Records the message te_last_error returns (one per thread, whichever unit raised it) and returns code.
int fail(int code, const char* fmt, ...);

#define TE_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess) return fail(TE_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

// Holds the context's lock and its device for the duration of an entry.
struct Guard {
  te_ctx* c;
  int prev = -1;
  bool ok = false;
  explicit Guard(te_ctx* ctx);
  ~Guard();
};

#define TE_ENTER(ctx)                                                   \
  if (!(ctx)) return fail(TE_ERR_BAD_ARG, "context is null");           \
  Guard guard__(ctx);                                                   \
  if (!guard__.ok) return fail(TE_ERR_CUDA, "cudaSetDevice(%d) failed", (ctx)->device)

// Checks the launches just enqueued and counts them (te_get_stats).
int launch_check(te_ctx* c, const char* what, int n = 1);

int check_geometry(const te_geometry* g, bool allow_start_index = false);
// Same validation as the filters' configure(): SlopeFilter.cpp:41, StepFilter.cpp:45,58,71,84, RoughnessFilter.cpp:43,55.
int check_params(const te_chain_params* p);
// Validates the geometry of an entry that honours a circular-buffer start index where `supported` (whole maps in host memory:
// the staging copies unwrap and re-wrap the layers) and returns it with the start index cleared.  The kernels always see the
// default order: positions depend on the unwrapped index only.
int unwrap_geometry(const te_geometry* g, bool supported, te_geometry* out);
// The context's coordinate tables for g, rebuilt (after the kernels queued before) when g changes.
int ensure_geometry(te_ctx* c, const te_geometry* g);

// Columns [c0, c0 + n) between a device buffer in default order (column c at dev + c * rows) and a host layer.  With a start
// index (sr, sc) != (0, 0) the host layer is a whole map of `cols` columns stored as a grid_map circular buffer: cell (i, j) of
// the map lives at stored[((j + sc) % cols) * rows + (i + sr) % rows] (GridMap::getIndex... / convertToDefaultStartIndex,
// SURVEY.md A.1) and moves in up to four 2-D copies.  Otherwise the host layer is in default order too: one plain copy.  This
// is what lets the TE_MEM_HOST entries take the message / GridMap buffers of a moving (robot-centric) map as they are, without
// an unwrapped host copy (SURVEY.md §8f-1).  upload_cols and download_cols are the only code that knows this layout.
// Cells are `elem` bytes (float32 layers: 4; image bytes, whose "columns" are image rows: 1 or 2).  The host columns lie
// `host_pitch` bytes apart (0: packed, elem * rows; a padded pitch needs start index 0); the device columns are packed.
cudaError_t upload_cols(void* dev, const void* host, int rows, int cols, int sr, int sc, int c0, int n, cudaStream_t s,
                        size_t elem = sizeof(float), size_t host_pitch = 0);
cudaError_t download_cols(float* host, const float* dev, int rows, int cols, int sr, int sc, int c0, int n, cudaStream_t s);

// The staging of one call.  In host memory it hands out the context's staging buffers in order, uploads the inputs on the
// context stream and records the outputs; finish() copies those back and returns once they are on the host.  In device memory
// every pointer passes through and finish() enqueues nothing.  Host layers are `rows` x ncols in default order or, with the start
// index of `g`, whole maps in circular-buffer order (upload_cols).  The first failure is kept in `rc`: later steps do nothing.
struct Staging {
  te_ctx* c;
  bool host;
  int rows, cols, sr, sc;
  int rc = TE_OK;
  int used = 0;
  // ncols > 0: nlayers layers of that many columns back to back (4-byte cells: float32, or int32 copied as they are)
  struct Out { void* host; const void* dev; size_t bytes; int ncols, nlayers; };
  Out outs[sizeof(te_ctx::stage) / sizeof(te::DevBuf)];
  int nout = 0;

  Staging(te_ctx* ctx, bool host_memory, const te_geometry* g);
  void check(cudaError_t e, const char* what);
  // The next staging buffer, at least `bytes` long (grow-only: once every slot has reached its largest size, nothing is allocated).
  void* slot(size_t bytes);
  size_t layer_bytes(int ncols) const;
  // An input layer of `ncols` columns; null stays null.
  const float* in_layer(const float* h, int ncols);
  // An input array of `n` elements; null stays null.
  template <class T>
  const T* in(const T* h, size_t n);
  // `nlayers` output layers of `ncols` columns in one staging buffer / an output array of `n` elements; null stays null.
  template <class T>
  T* out_layer(T* h, int ncols, int nlayers = 1);
  template <class T>
  T* out(T* h, size_t n);
  void* record(void* h, size_t bytes, int ncols, int nlayers);
  int finish();
};

// The coordinate tables of a launch over maps at their own positions (device, built by map_tables): map k of the launch has X at
// X + k * rows, Y at Y + k * cols and its position at pos[2k], pos[2k + 1]; masks: its fused mask tables (chain launches).
struct PosTables {
  const double* X;
  const double* Y;
  const double* pos;
  double coord_max;  // the largest |cell-centre coordinate| over the maps
  te::MapMasks masks;
};

te::SlabView make_view(te_ctx* c, const te_geometry* g, const te_slab& s);
// v on the per-map tables t (t null: v as it is).
te::SlabView view_at(te::SlabView v, const te_geometry* g, const PosTables* t);

// te_chain, te_chain_batched and the te_map chain launches (device memory, tab: maps at their own positions).
int chain_common(te_ctx* c, const te_geometry* g_in, const te_slab* slab, const te_chain_params* p, int nmaps, const float* elev,
                 float* slope, float* step, float* rough, float* trav, float* nx, float* ny, float* nz, int memory,
                 const PosTables* tab = nullptr);

// Output of a polygon footprint entry: `count` layers of the call's maps back to back from `out`, layer k rotated by yaws[k].
struct PolygonOutputs {
  float* out;
  int count;
  const double* yaws;
};

// te_footprint_polygon (one map or slab), te_footprint_polygon_batched (nmaps whole maps), te_footprint_polygon_yaws(_reduce) (nmaps
// whole maps, a list of yaws) and the te_map polygon entries: every layer of `outs` from one sweep or, with `reduce` (HOST or
// device pointers as `memory` says), the reductions over the yaws of its one output, whose `out` is then unused.  `start_index_ok`:
// in host memory the staging takes a circular-buffer map (whole single maps).  `resident`: the layers are a te_map's, on the device
// in default order, swept with the map's own state; they are never staged, and a start index is then fine in either memory (device
// outputs are in default order).
int footprint_polygon_common(te_ctx* c, te::FootprintState* resident, const te_geometry* g_in, const te_slab* slab,
                             const te_footprint_params* p, int nmaps, int32_t npts, const double* pts_xy, const float* trav,
                             const float* slope, const float* step, const float* rough, const float* elev, int nouts,
                             const PolygonOutputs* outs, const te::PolygonReduce* reduce, int memory, bool start_index_ok);

// The batch of a footprint entry: nmaps whole maps of one geometry back to back (te_footprint_batched, te_footprint_polygon_batched),
// or one map or slab (nmaps = 1).  nmaps is a grid dimension of the sweep kernels, and their predicate work list stores 32-bit cell
// indices of the batch.
int check_footprint_batch(const te_geometry* g, int nmaps);
// The list of yaws of the yaws entries (the cap bounds the host classification and the table upload of one call).
int check_yaws(int32_t nyaws, const double* yaws);
int check_reduce_outputs(const te::PolygonReduce& r);
// The untraversable-polygon outputs of te_check_footprint_paths_fresh2 / _polygon2: both null (no polygon), or counts with room
// for max_vertices >= 0 points per path (xy may be null only when max_vertices is 0).
int check_polygon_outputs(int32_t max_vertices, const int32_t* ucount, const double* uxy);
// The host-side validation of a te_check_footprint_request request (paths, footprints, radii, conservative caps, finite poses and
// vertices); sets *mp to the hull input bound of a polygonal item.  per_map: p holds one parameter set per map and path q uses
// that of its map, p[path_map[q]] (path_map null: p[0]).
int check_request_host(const te_geometry* g, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                       const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                       const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative, int* mp_out,
                       bool per_map = false, const int32_t* path_map = nullptr);
// Stages the path arrays of `r` and points `r` at the device copies (host memory; null stays null).
void stage_paths(Staging& st, te::PathChecks& r);

}  // namespace host
}  // namespace te
