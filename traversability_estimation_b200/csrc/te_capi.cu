// te_capi.cu — the extern "C" boundary of libte_b200 (see include/te_b200.h).
// Host-side responsibilities only: argument validation with the reference's conventions, the
// per-geometry position tables, host<->device staging for TE_MEM_HOST callers, kernel selection.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/te_b200.h"
#include "te_kernels.h"
#include "te_fused.h"
#include "te_footprint.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define TE_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess) return fail(TE_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

using te::DevBuf;
using te::cell_coord;

// Largest index offset that can satisfy the circle test.  A cell at offset R + 1 lies (R + 1) * res from the centre up to a few
// ulps of the absolute coordinates (~1e-14 m); it can pass `d^2 <= r^2` only if radius / res is within rounding of R + 1, and
// only then is the guard cell scanned (the literal kernels test every candidate with the reference's own arithmetic anyway).
inline int reach_generous(double radius, double res) {
  const double q = radius / res;
  const int R = (int)std::floor(q);
  return (q - (double)R > 1.0 - 1e-6) ? R + 1 : R;
}
// Dependency radius in cells (what a slab halo must provide).
inline int reach_true(double radius, double res) { return (int)std::floor(radius / res + 1e-9); }

}  // namespace

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
  DevBuf dX, dY;
  std::vector<double> hX, hY;

  DevBuf stage[20];          // TE_MEM_HOST staging (handed out in order by Staging; te_check_footprint_request_batched takes 19)
  DevBuf worklist, worklist3, counter;  // fused-kernel fix-up lists (tier 2, tier 3) and their counters
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

namespace {

int check_geometry(const te_geometry* g, bool allow_start_index = false) {
  if (!g) return fail(TE_ERR_BAD_ARG, "geometry is null");
  if (g->rows <= 0 || g->cols <= 0) return fail(TE_ERR_BAD_ARG, "map size must be positive (rows=%d cols=%d)", g->rows, g->cols);
  if (!(g->resolution > 0.0) || !std::isfinite(g->resolution)) return fail(TE_ERR_BAD_ARG, "resolution must be positive");
  if (g->start_row != 0 || g->start_col != 0) {
    if (!allow_start_index)
      return fail(TE_ERR_UNSUPPORTED, "circular-buffer start index (%d,%d) != (0,0): call convertToDefaultStartIndex() first",
                  g->start_row, g->start_col);
    if (g->start_row < 0 || g->start_row >= g->rows || g->start_col < 0 || g->start_col >= g->cols)
      return fail(TE_ERR_BAD_ARG, "circular-buffer start index (%d,%d) outside the map", g->start_row, g->start_col);
  }
  if ((long long)g->rows * g->cols > 0x7fffffffLL * 2) return fail(TE_ERR_UNSUPPORTED, "map has more than 2^32 cells");
  return TE_OK;
}

// Same validation as the filters' configure(): SlopeFilter.cpp:41, StepFilter.cpp:45,58,71,84,
// RoughnessFilter.cpp:43,55.
int check_params(const te_chain_params* p) {
  if (!p) return fail(TE_ERR_BAD_ARG, "chain parameters are null");
  if (!(p->normals_radius >= 0.0)) return fail(TE_ERR_BAD_ARG, "normals radius must be >= 0");
  if (p->normals_algorithm != TE_NORMALS_FIXTURE && p->normals_algorithm != TE_NORMALS_RAW_MOMENT)
    return fail(TE_ERR_BAD_ARG, "unknown normals algorithm %d", p->normals_algorithm);
  if (p->normals_positive_axis < 0 || p->normals_positive_axis > 2) return fail(TE_ERR_BAD_ARG, "positive axis must be 0, 1 or 2");
  if (p->slope_critical > M_PI_2 || p->slope_critical < 0.0 || std::isnan(p->slope_critical))
    return fail(TE_ERR_BAD_ARG, "Critical slope must be in the interval [0, PI/2]");
  if (!(p->step_critical >= 0.0)) return fail(TE_ERR_BAD_ARG, "Critical step height must be greater than zero");
  if (!(p->step_first_radius >= 0.0) || !(p->step_second_radius >= 0.0))
    return fail(TE_ERR_BAD_ARG, "step window radii must be greater than zero");
  if (p->step_critical_cells <= 0) return fail(TE_ERR_BAD_ARG, "Number of critical cells must be greater than zero");
  if (!(p->roughness_critical >= 0.0)) return fail(TE_ERR_BAD_ARG, "Critical roughness must be greater than zero");
  if (!(p->roughness_radius >= 0.0)) return fail(TE_ERR_BAD_ARG, "Roughness estimation radius must be greater than zero");
  return TE_OK;
}

int ensure_geometry(te_ctx* c, const te_geometry* g) {
  if (c->have_geo && std::memcmp(&c->geo, g, sizeof(te_geometry)) == 0) return TE_OK;
  c->hX.resize(g->rows);
  c->hY.resize(g->cols);
  for (int i = 0; i < g->rows; ++i) c->hX[i] = cell_coord(g->position_x, g->length_x, g->resolution, i);
  for (int j = 0; j < g->cols; ++j) c->hY[j] = cell_coord(g->position_y, g->length_y, g->resolution, j);
  TE_CUDA(c->dX.reserve(sizeof(double) * g->rows));
  TE_CUDA(c->dY.reserve(sizeof(double) * g->cols));
  // The tables may still be in use by kernels queued on the stream: order the overwrite after them.
  TE_CUDA(cudaMemcpyAsync(c->dX.p, c->hX.data(), sizeof(double) * g->rows, cudaMemcpyHostToDevice, c->stream));
  TE_CUDA(cudaMemcpyAsync(c->dY.p, c->hY.data(), sizeof(double) * g->cols, cudaMemcpyHostToDevice, c->stream));
  TE_CUDA(cudaStreamSynchronize(c->stream));  // hX/hY are reused
  c->geo = *g;
  c->have_geo = true;
  c->fused.invalidate();
  c->fp.invalidate();
  return TE_OK;
}

te::ChainDev make_chain_dev(const te_geometry* g, const te_chain_params* p) {
  te::ChainDev d{};
  const double res = g->resolution;
  d.rn = p->normals_radius; d.rn2 = d.rn * d.rn; d.Rn = reach_generous(d.rn, res);
  d.alg = p->normals_algorithm; d.axis = p->normals_positive_axis;
  d.slope_crit = p->slope_critical;
  d.step_crit = p->step_critical;
  d.r1 = p->step_first_radius; d.r1sq = d.r1 * d.r1; d.R1 = reach_generous(d.r1, res);
  d.r2 = p->step_second_radius; d.r2sq = d.r2 * d.r2; d.R2 = reach_generous(d.r2, res);
  d.ncrit = p->step_critical_cells;
  d.rough_crit = p->roughness_critical;
  d.rr = p->roughness_radius; d.rr2 = d.rr * d.rr; d.Rr = reach_generous(d.rr, res);
  d.fuse_w = p->fuse_weight;
  return d;
}

int chain_halo(const te_geometry* g, const te_chain_params* p) {
  const double res = g->resolution;
  const int hn = reach_true(p->normals_radius, res), hr = reach_true(p->roughness_radius, res);
  const int hs = reach_true(p->step_first_radius, res) + reach_true(p->step_second_radius, res);
  return std::max(hn, std::max(hr, hs));
}

int resolve_slab(const te_geometry* g, const te_slab* s, int need_halo, te_slab* out) {
  if (!s) {
    *out = te_slab{0, g->cols, 0, 0};
    return TE_OK;
  }
  if (s->col_begin < 0 || s->col_count <= 0 || s->col_begin + s->col_count > g->cols)
    return fail(TE_ERR_BAD_ARG, "slab columns [%d,%d) outside map of %d columns", s->col_begin, s->col_begin + s->col_count, g->cols);
  if (s->halo_left < 0 || s->halo_right < 0 || s->halo_left > s->col_begin || s->halo_right > g->cols - (s->col_begin + s->col_count))
    return fail(TE_ERR_BAD_ARG, "slab halo (%d,%d) reaches outside the map", s->halo_left, s->halo_right);
  const int need_l = std::min(need_halo, s->col_begin);
  const int need_r = std::min(need_halo, g->cols - (s->col_begin + s->col_count));
  if (s->halo_left < need_l || s->halo_right < need_r)
    return fail(TE_ERR_BAD_ARG, "slab halo (%d,%d) smaller than the dependency radius %d of these parameters", s->halo_left,
                s->halo_right, need_halo);
  *out = *s;
  return TE_OK;
}

te::SlabView make_view(te_ctx* c, const te_geometry* g, const te_slab& s) {
  te::SlabView v{};
  v.rows = g->rows;
  v.cols_total = g->cols;
  v.in_col0 = s.col_begin - s.halo_left;
  v.in_ncols = s.halo_left + s.col_count + s.halo_right;
  v.out_col0 = s.col_begin;
  v.out_ncols = s.col_count;
  v.X = (const double*)c->dX.p;
  v.Y = (const double*)c->dY.p;
  v.res = g->resolution;
  v.coord_max = std::max(std::fabs(g->position_x) + 0.5 * g->length_x, std::fabs(g->position_y) + 0.5 * g->length_y);
  return v;
}

struct Guard {
  te_ctx* c;
  int prev = -1;
  bool ok = false;
  explicit Guard(te_ctx* ctx) : c(ctx) {
    c->mu.lock();
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    ok = cudaSetDevice(c->device) == cudaSuccess;
  }
  ~Guard() {
    if (prev >= 0 && prev != c->device) cudaSetDevice(prev);
    c->mu.unlock();
  }
};

#define TE_ENTER(ctx)                                                   \
  if (!(ctx)) return fail(TE_ERR_BAD_ARG, "context is null");           \
  Guard guard__(ctx);                                                   \
  if (!guard__.ok) return fail(TE_ERR_CUDA, "cudaSetDevice(%d) failed", (ctx)->device)

// Checks the launches just enqueued and counts them (te_get_stats).
int launch_check(te_ctx* c, const char* what, int n = 1) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TE_ERR_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  c->launches += n;
  return TE_OK;
}

// Validates the geometry of an entry that honours a circular-buffer start index where `supported` (whole maps in host memory:
// the staging copies unwrap and re-wrap the layers) and returns it with the start index cleared.  The kernels always see the
// default order: positions depend on the unwrapped index only.
int unwrap_geometry(const te_geometry* g, bool supported, te_geometry* out) {
  if (int rc = check_geometry(g, true)) return rc;
  if ((g->start_row != 0 || g->start_col != 0) && !supported)
    return fail(TE_ERR_UNSUPPORTED, "circular-buffer start index (%d,%d) != (0,0) is supported for whole maps in host memory only",
                g->start_row, g->start_col);
  *out = *g;
  out->start_row = out->start_col = 0;
  return TE_OK;
}

// The layers isTraversableForFilters reads, in the order every footprint entry reports them.
int check_filter_layers(const te_footprint_params* p, const float* trav, const float* slope, const float* step, const float* elev,
                        const float* rough) {
  if (!trav) return fail(TE_ERR_MISSING_LAYER, "layer traversability is missing");
  if (!slope) return fail(TE_ERR_MISSING_LAYER, "layer traversability_slope is missing");
  if (!step) return fail(TE_ERR_MISSING_LAYER, "layer traversability_step is missing");
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (p->verify_roughness && !rough) return fail(TE_ERR_MISSING_LAYER, "layer traversability_roughness is missing (verify_roughness is set)");
  return TE_OK;
}

// Columns [c0, c0 + n) between a device buffer in default order (column c at dev + c * rows) and a host layer.  With a start
// index (sr, sc) != (0, 0) the host layer is a whole map of `cols` columns stored as a grid_map circular buffer: cell (i, j) of
// the map lives at stored[((j + sc) % cols) * rows + (i + sr) % rows] (GridMap::getIndex... / convertToDefaultStartIndex,
// SURVEY.md A.1) and moves in up to four 2-D copies.  Otherwise the host layer is in default order too: one plain copy.  This
// is what lets the TE_MEM_HOST entries take the message / GridMap buffers of a moving (robot-centric) map as they are, without
// an unwrapped host copy (SURVEY.md §8f-1).  upload_cols and download_cols are the only code that knows this layout.
template <class F>
cudaError_t for_wrapped_pieces(int rows, int cols, int sr, int sc, int c0, int n, F&& copy) {
  for (int done = 0; done < n;) {
    const int c = c0 + done, js = (c + sc) % cols;  // stored column of map column c
    const int m = std::min(n - done, cols - js);     // columns until the stored index wraps
    const size_t d = (size_t)c * rows, h = (size_t)js * rows;
    // rows [0, rows - sr) of the map are stored rows [sr, rows); rows [rows - sr, rows) are stored rows [0, sr)
    cudaError_t e = copy(d, h + sr, rows - sr, m);
    if (e == cudaSuccess && sr > 0) e = copy(d + (rows - sr), h, sr, m);
    if (e != cudaSuccess) return e;
    done += m;
  }
  return cudaSuccess;
}

cudaError_t upload_cols(float* dev, const float* host, int rows, int cols, int sr, int sc, int c0, int n, cudaStream_t s) {
  const size_t pitch = sizeof(float) * (size_t)rows;
  if (sr == 0 && sc == 0) return cudaMemcpyAsync(dev + (size_t)c0 * rows, host + (size_t)c0 * rows, pitch * n, cudaMemcpyHostToDevice, s);
  return for_wrapped_pieces(rows, cols, sr, sc, c0, n, [&](size_t d, size_t h, int r, int m) {
    return cudaMemcpy2DAsync(dev + d, pitch, host + h, pitch, sizeof(float) * r, m, cudaMemcpyHostToDevice, s);
  });
}

cudaError_t download_cols(float* host, const float* dev, int rows, int cols, int sr, int sc, int c0, int n, cudaStream_t s) {
  const size_t pitch = sizeof(float) * (size_t)rows;
  if (sr == 0 && sc == 0) return cudaMemcpyAsync(host + (size_t)c0 * rows, dev + (size_t)c0 * rows, pitch * n, cudaMemcpyDeviceToHost, s);
  return for_wrapped_pieces(rows, cols, sr, sc, c0, n, [&](size_t d, size_t h, int r, int m) {
    return cudaMemcpy2DAsync(host + h, pitch, dev + d, pitch, sizeof(float) * r, m, cudaMemcpyDeviceToHost, s);
  });
}

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
  Out outs[sizeof(te_ctx::stage) / sizeof(DevBuf)];
  int nout = 0;

  Staging(te_ctx* ctx, bool host_memory, const te_geometry* g)
      : c(ctx), host(host_memory), rows(g->rows), cols(g->cols), sr(g->start_row), sc(g->start_col) {}

  void check(cudaError_t e, const char* what) {
    if (rc == TE_OK && e != cudaSuccess) rc = fail(TE_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
  }
  // The next staging buffer, at least `bytes` long (grow-only: once every slot has reached its largest size, nothing is allocated).
  void* slot(size_t bytes) {
    if (rc != TE_OK) return nullptr;
    if (used == (int)(sizeof(outs) / sizeof(outs[0]))) {
      rc = fail(TE_ERR_CUDA, "out of staging buffers");
      return nullptr;
    }
    DevBuf& b = c->stage[used++];
    check(b.reserve(std::max<size_t>(bytes, 1)), "staging allocation");
    return rc == TE_OK ? b.p : nullptr;
  }
  size_t layer_bytes(int ncols) const { return sizeof(float) * (size_t)rows * ncols; }
  // An input layer of `ncols` columns; null stays null.
  const float* in_layer(const float* h, int ncols) {
    if (!host || !h) return h;
    float* d = (float*)slot(layer_bytes(ncols));
    if (d) check(upload_cols(d, h, rows, cols, sr, sc, 0, ncols, c->stream), "layer upload");
    return d;
  }
  // An input array of `n` elements; null stays null.
  template <class T>
  const T* in(const T* h, size_t n) {
    if (!host || !h) return h;
    T* d = (T*)slot(sizeof(T) * n);
    if (d && n) check(cudaMemcpyAsync(d, h, sizeof(T) * n, cudaMemcpyHostToDevice, c->stream), "upload");
    return d;
  }
  // `nlayers` output layers of `ncols` columns in one staging buffer / an output array of `n` elements; null stays null.
  template <class T>
  T* out_layer(T* h, int ncols, int nlayers = 1) {
    static_assert(sizeof(T) == sizeof(float), "layers have 4-byte cells");
    return (T*)record(h, layer_bytes(ncols) * nlayers, ncols, nlayers);
  }
  template <class T>
  T* out(T* h, size_t n) { return (T*)record(h, sizeof(T) * n, 0, 0); }
  void* record(void* h, size_t bytes, int ncols, int nlayers) {
    if (!host || !h) return h;
    void* d = slot(bytes);
    if (d) outs[nout++] = Out{h, d, bytes, ncols, nlayers};
    return d;
  }
  int finish() {
    if (!host || rc != TE_OK) return rc;
    for (int k = 0; k < nout; ++k) {
      const Out& o = outs[k];
      if (!o.ncols) {
        check(cudaMemcpyAsync(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost, c->stream), "download");
      } else if (sr == 0 && sc == 0) {  // default order: the layers are one run of columns
        check(download_cols((float*)o.host, (const float*)o.dev, rows, cols, 0, 0, 0, o.ncols * o.nlayers, c->stream), "download");
      } else {  // a start index wraps the columns of one map: re-wrap each layer on its own
        for (int l = 0; l < o.nlayers; ++l) {
          const size_t off = (size_t)l * rows * o.ncols;
          check(download_cols((float*)o.host + off, (const float*)o.dev + off, rows, cols, sr, sc, 0, o.ncols, c->stream), "download");
        }
      }
    }
    check(cudaStreamSynchronize(c->stream), "cudaStreamSynchronize");
    return rc;
  }
};

// The next triple of timing events; the pool grows on demand and is reused after te_get_timing.
int next_timing_slot(te_ctx* c, te_ctx::Ev3** out) {
  if (c->events_used == c->events.size()) {
    te_ctx::Ev3 ev{};
    TE_CUDA(cudaEventCreate(&ev.a)); TE_CUDA(cudaEventCreate(&ev.b)); TE_CUDA(cudaEventCreate(&ev.c));
    c->events.push_back(ev);
  }
  *out = &c->events[c->events_used];
  return TE_OK;
}

// Device-memory chain on one slab: picks the kernel.
int run_chain_device(te_ctx* c, const te_geometry* g, const te::SlabView& v, const te_chain_params* p, const float* elev,
                     const te::ChainOut& o, int nmaps) {
  const te::ChainDev d = make_chain_dev(g, p);
  bool use_fused = false;
  if (c->kernel_choice != TE_KERNEL_GENERIC) {
    use_fused = te::fused_eligible(c->fused, c->hX, c->hY, g, p, c->stream);
    if (!use_fused && c->kernel_choice == TE_KERNEL_FUSED)
      return fail(TE_ERR_UNSUPPORTED, "fused stencil has no instantiation for these window shapes: %s", c->fused.why.c_str());
    if (use_fused) {
      if (const char* why = te::fused_launch_obstacle(v, nmaps, elev, o)) {
        if (c->kernel_choice == TE_KERNEL_FUSED) return fail(TE_ERR_UNSUPPORTED, "fused stencil cannot run this launch: %s", why);
        use_fused = false;  // TE_KERNEL_AUTO: the generic kernel computes the same layers
      }
    }
  }
  const size_t in_stride = (size_t)g->rows * v.in_ncols, out_stride = (size_t)g->rows * v.out_ncols;
  if (use_fused) {
    // The work lists hold every cell of the launch (plus chunk padding), so they cannot overflow: a degenerate map (exact planes,
    // holes everywhere) sends all of its cells down the certified slow path instead of returning uncertified fp32 values.
    const size_t cells = out_stride * (size_t)nmaps;
    const size_t cap = te::fused_list_capacity(cells, c->sms);
    if (cap >= ((size_t)1 << 32)) return fail(TE_ERR_UNSUPPORTED, "launch of %zu cells exceeds the work-list index range", cells);
    TE_CUDA(c->worklist.reserve(sizeof(unsigned) * cap));
    TE_CUDA(c->worklist3.reserve(sizeof(unsigned) * cells));
    {
      const void* before = c->counter.p;
      TE_CUDA(c->counter.reserve(sizeof(unsigned) * 256));
      if (c->counter.p != before) c->counter_clean = -1;
    }
    {  // one launch covers every map of the batch
      const te::ChainOut& om = o;
      const int phase = c->counter_phase ^ 1;
      unsigned* const cnt = (unsigned*)c->counter.p + 128 * phase;
      unsigned* const cnt_next = (unsigned*)c->counter.p + 128 * (phase ^ 1);
      if (c->counter_stream != c->stream) c->counter_clean = -1;  // zeroed in another stream's order: not ordered before this launch
      c->counter_stream = c->stream;
      if (c->counter_clean != phase) TE_CUDA(cudaMemsetAsync(cnt, 0, sizeof(unsigned) * 128, c->stream));
      c->counter_clean = -1;
      c->counter_phase = phase;
      te_ctx::Ev3* ev = nullptr;
      if (c->timing) {
        if (int rc = next_timing_slot(c, &ev)) return rc;
        TE_CUDA(cudaEventRecord(ev->a, c->stream));
      }
      int rc = te::launch_chain_fused(c->fused, v, d, nmaps, elev, om, (unsigned*)c->worklist.p, cnt, (unsigned)cap, c->sms, c->stream);
      if (rc != 0) return fail(TE_ERR_CUDA, "fused chain launch failed: %s", c->fused.why.c_str());
      if (int r2 = launch_check(c, "k_chain_fused")) return r2;
      if (c->timing) TE_CUDA(cudaEventRecord(ev->b, c->stream));
      te::FixupArgs fa;
      te::make_fixup_args(c->fused, v, d, &fa);
      // tiers 2 and 3 are programmatic dependent launches unless events are recorded in between (timing): their grids are set
      // up while the predecessor drains and wait on griddepcontrol.wait before they read the lists
      te::launch_fixup_t2(fa, elev, om, (const unsigned*)c->worklist.p, cnt, (unsigned)cap, (unsigned*)c->worklist3.p, cnt + 4,
                          (unsigned)cells, c->sms, c->stream, !c->timing);
      if (int r2 = launch_check(c, "k_fixup_t2")) return r2;
      te::launch_fixup(v, d, elev, om, (const unsigned*)c->worklist3.p, cnt + 4, (unsigned)cells, cnt_next, c->sms, c->stream, true);
      if (int r2 = launch_check(c, "k_fixup_cells")) return r2;
      c->counter_clean = phase ^ 1;  // k_fixup_cells zeroes the other block
      if (c->timing) {
        TE_CUDA(cudaEventRecord(ev->c, c->stream));
        ++c->events_used;
      }
    }
  } else {
    for (int m = 0; m < nmaps; ++m) {
      te::ChainOut om = o;
      om.slope += m * out_stride; om.step += m * out_stride; om.rough += m * out_stride; om.trav += m * out_stride;
      if (om.nx) om.nx += m * out_stride;
      if (om.ny) om.ny += m * out_stride;
      if (om.nz) om.nz += m * out_stride;
      te_ctx::Ev3* ev = nullptr;
      if (c->timing) {
        if (int rc = next_timing_slot(c, &ev)) return rc;
        TE_CUDA(cudaEventRecord(ev->a, c->stream));
      }
      te::launch_chain_generic(v, d, elev + m * in_stride, om, c->sms, c->stream);
      if (int r2 = launch_check(c, "k_chain_generic")) return r2;
      if (c->timing) {
        TE_CUDA(cudaEventRecord(ev->b, c->stream));
        TE_CUDA(cudaEventRecord(ev->c, c->stream));
        ++c->events_used;
      }
    }
  }
  return TE_OK;
}

}  // namespace

extern "C" {

int te_abi_version(void) { return TE_B200_ABI_VERSION; }

const char* te_last_error(void) { return g_last_error.c_str(); }

int te_create(te_ctx** out, int device) {
  if (!out) return fail(TE_ERR_BAD_ARG, "out pointer is null");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0)
    return fail(TE_ERR_CUDA, "no CUDA device available (%s); libte_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(TE_ERR_BAD_ARG, "device %d out of range [0,%d)", device, n);
  int prev = 0;
  cudaGetDevice(&prev);
  TE_CUDA(cudaSetDevice(device));
  te_ctx* c = new te_ctx();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sms = prop.multiProcessorCount;
  e = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete c;
    cudaSetDevice(prev);
    return fail(TE_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e));
  }
  c->stream = c->own_stream;
  cudaSetDevice(prev);
  *out = c;
  return TE_OK;
}

int te_destroy(te_ctx* c) {
  if (!c) return TE_OK;
  {
    Guard g(c);
    if (g.ok) {
      cudaStreamSynchronize(c->stream);
      c->dX.release();
      c->dY.release();
      for (auto& b : c->stage) b.release();
      c->worklist.release();
      c->worklist3.release();
      c->counter.release();
      c->fused.release();
      c->fp.release();
      for (auto& e : c->events) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); cudaEventDestroy(e.c); }
      if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
      if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
      if (c->own_stream) cudaStreamDestroy(c->own_stream);
    }
  }
  delete c;
  return TE_OK;
}

int te_host_alloc(void** out, size_t bytes) {
  if (!out) return fail(TE_ERR_BAD_ARG, "out pointer is null");
  *out = nullptr;
  TE_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return TE_OK;
}

int te_host_free(void* p) {
  if (!p) return TE_OK;
  TE_CUDA(cudaFreeHost(p));
  return TE_OK;
}

int te_set_stream(te_ctx* c, void* s) {
  TE_ENTER(c);
  c->stream = s ? (cudaStream_t)s : c->own_stream;
  return TE_OK;
}

int te_synchronize(te_ctx* c) {
  TE_ENTER(c);
  TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

int te_set_kernel(te_ctx* c, int choice) {
  TE_ENTER(c);
  if (choice < TE_KERNEL_AUTO || choice > TE_KERNEL_FUSED) return fail(TE_ERR_BAD_ARG, "unknown kernel choice %d", choice);
  c->kernel_choice = choice;
  return TE_OK;
}

int te_get_stats(te_ctx* c, int64_t* launches, int64_t* slow) {
  TE_ENTER(c);
  if (launches) *launches = c->launches;
  if (slow) {
    // the fix-up counter of the last fused launch (device word 0); cumulative host tally otherwise
    unsigned last[4] = {0, 0, 0, 0};
    if (c->counter.p) {
      TE_CUDA(cudaStreamSynchronize(c->stream));
      TE_CUDA(cudaMemcpy(last, (unsigned*)c->counter.p + 128 * c->counter_phase, sizeof(last), cudaMemcpyDeviceToHost));
    }
    *slow = (int64_t)last[1];  // cells flagged (word 0 counts reserved list entries, chunk padding included)
  }
  return TE_OK;
}

int te_enable_timing(te_ctx* c, int on) {
  TE_ENTER(c);
  c->timing = on != 0;
  return TE_OK;
}

int te_get_timing(te_ctx* c, double* main_ms, double* fixup_ms, int64_t* samples) {
  TE_ENTER(c);
  TE_CUDA(cudaStreamSynchronize(c->stream));
  double m = 0.0, f = 0.0;
  for (size_t k = 0; k < c->events_used; ++k) {
    const auto& e = c->events[k];
    float t1 = 0.f, t2 = 0.f;
    TE_CUDA(cudaEventElapsedTime(&t1, e.a, e.b));
    TE_CUDA(cudaEventElapsedTime(&t2, e.b, e.c));
    m += t1;
    f += t2;
  }
  if (main_ms) *main_ms = m;
  if (fixup_ms) *fixup_ms = f;
  if (samples) *samples = (int64_t)c->events_used;
  c->events_used = 0;
  return TE_OK;
}

int te_fused_plan(int rows, int out_ncols, int nmaps, int sms, int32_t out[19]) {
  if (rows <= 0 || out_ncols <= 0 || nmaps <= 0 || sms <= 0 || !out) return TE_ERR_BAD_ARG;
  int tmp[19];
  te::fused_plan(rows, out_ncols, nmaps, sms, tmp);
  for (int i = 0; i < 19; ++i) out[i] = tmp[i];
  return TE_OK;
}

int te_get_flag_counters(te_ctx* c, uint32_t out[5]) {
  TE_ENTER(c);
  if (!out) return fail(TE_ERR_BAD_ARG, "null argument");
  for (int k = 0; k < 5; ++k) out[k] = 0;
  if (c->counter.p) {
    unsigned raw[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    TE_CUDA(cudaStreamSynchronize(c->stream));
    TE_CUDA(cudaMemcpy(raw, (unsigned*)c->counter.p + 128 * c->counter_phase, sizeof(raw), cudaMemcpyDeviceToHost));
    out[0] = raw[1];            // cells flagged by the fp32 stencil
    out[1] = raw[0];            // list entries reserved (warp-private chunks, padding included)
    out[2] = raw[2] | raw[5];   // a work list overflowed (never: the lists hold every cell of the launch)
    out[4] = raw[4];            // cells tier 2 passed on to the literal kernel
  }
  return TE_OK;
}

int te_get_escalation_stats(te_ctx* c, uint32_t reasons[16], uint32_t valid_cells[26]) {
  TE_ENTER(c);
  if (!reasons || !valid_cells) return fail(TE_ERR_BAD_ARG, "null argument");
  unsigned raw[64];
  std::memset(raw, 0, sizeof(raw));
  if (c->counter.p) {
    TE_CUDA(cudaStreamSynchronize(c->stream));
    TE_CUDA(cudaMemcpy(raw, (unsigned*)c->counter.p + 128 * c->counter_phase, sizeof(raw), cudaMemcpyDeviceToHost));
  }
  for (int k = 0; k < 16; ++k) reasons[k] = raw[8 + k];
  for (int k = 0; k < 26; ++k) valid_cells[k] = raw[24 + k];
  return TE_OK;
}

int te_slope(te_ctx* c, const te_geometry* g, double crit, const float* nz, float* out, int memory) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (crit > M_PI_2 || crit < 0.0 || std::isnan(crit)) return fail(TE_ERR_BAD_ARG, "Critical slope must be in the interval [0, PI/2]");
  if (!nz) return fail(TE_ERR_MISSING_LAYER, "layer surface_normal_z is missing");
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  Staging st(c, memory == TE_MEM_HOST, g);
  const float* din = st.in_layer(nz, g->cols);
  float* dout = st.out_layer(out, g->cols);
  if (st.rc) return st.rc;
  te::launch_slope((long long)g->rows * g->cols, crit, din, dout, c->sms, c->stream);
  if (int rc = launch_check(c, "k_slope")) return rc;
  return st.finish();
}

int te_normals(te_ctx* c, const te_geometry* g, const te_chain_params* p, const float* elev, float* nx, float* ny, float* nz, int memory) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (int rc = check_params(p)) return rc;
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (!nx || !ny || !nz) return fail(TE_ERR_BAD_ARG, "output layer is null");
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g);
  const float* din = st.in_layer(elev, g->cols);
  float* o[3] = {st.out_layer(nx, g->cols), st.out_layer(ny, g->cols), st.out_layer(nz, g->cols)};
  if (st.rc) return st.rc;
  te_slab s{0, g->cols, 0, 0};
  te::launch_normals(make_view(c, g, s), make_chain_dev(g, p), din, o[0], o[1], o[2], c->sms, c->stream);
  if (int rc = launch_check(c, "k_normals")) return rc;
  return st.finish();
}

int te_step(te_ctx* c, const te_geometry* g, const te_chain_params* p, const float* elev, float* out, int memory) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (int rc = check_params(p)) return rc;
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g);
  const float* din = st.in_layer(elev, g->cols);
  float* dout = st.out_layer(out, g->cols);
  if (st.rc) return st.rc;
  te_slab s{0, g->cols, 0, 0};
  te::launch_step(make_view(c, g, s), make_chain_dev(g, p), din, dout, c->sms, c->stream);
  if (int rc = launch_check(c, "k_step")) return rc;
  return st.finish();
}

int te_roughness(te_ctx* c, const te_geometry* g, const te_chain_params* p, const float* elev, const float* nx, const float* ny,
                 const float* nz, float* out, int memory) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (int rc = check_params(p)) return rc;
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (!nx || !ny || !nz) return fail(TE_ERR_MISSING_LAYER, "layer surface_normal_{x,y,z} is missing");
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g);
  const float* in[4] = {st.in_layer(elev, g->cols), st.in_layer(nx, g->cols), st.in_layer(ny, g->cols), st.in_layer(nz, g->cols)};
  float* dout = st.out_layer(out, g->cols);
  if (st.rc) return st.rc;
  te_slab s{0, g->cols, 0, 0};
  te::launch_roughness(make_view(c, g, s), make_chain_dev(g, p), in[0], in[1], in[2], in[3], dout, c->sms, c->stream);
  if (int rc = launch_check(c, "k_roughness")) return rc;
  return st.finish();
}

// Host-memory chain on a large map: column chunks flow H2D -> kernels -> D2H on three streams so that the two PCIe
// directions and the compute overlap (the transfers dominate: 20 B/cell over PCIe against 20 B/cell over HBM).
static int chain_host_pipelined(te_ctx* c, Staging& st, const te_geometry* g, const te_slab& s, const te_chain_params* p, const float* elev,
                                float* const host_out[7]) {
  const int rows = g->rows, need = chain_halo(g, p);
  const int in_cols = s.halo_left + s.col_count + s.halo_right;
  float* const din = (float*)st.slot(st.layer_bytes(in_cols));
  float* dev_out[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  for (int k = 0; k < 7; ++k)
    if (host_out[k]) dev_out[k] = (float*)st.slot(st.layer_bytes(s.col_count));
  if (st.rc) return st.rc;
  if (!c->s_h2d) TE_CUDA(cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking));
  if (!c->s_d2h) TE_CUDA(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
  const int nchunk = std::min(16, std::max(2, s.col_count / 512));
  const int chunk = (s.col_count + nchunk - 1) / nchunk;
  // events and the drain of the three streams are released on every exit path
  struct Pipeline {
    te_ctx* c;
    std::vector<cudaEvent_t> ev;
    cudaError_t make(cudaEvent_t* out) {
      cudaError_t e = cudaEventCreateWithFlags(out, cudaEventDisableTiming);
      if (e == cudaSuccess) ev.push_back(*out);
      return e;
    }
    ~Pipeline() {
      cudaStreamSynchronize(c->s_h2d);
      cudaStreamSynchronize(c->stream);
      cudaStreamSynchronize(c->s_d2h);
      for (cudaEvent_t e : ev) cudaEventDestroy(e);
    }
  } pipe{c, {}};
  std::vector<cudaEvent_t> up(nchunk), done(nchunk);
  for (int k = 0; k < nchunk; ++k) {
    TE_CUDA(pipe.make(&up[k]));
    TE_CUDA(pipe.make(&done[k]));
  }
  cudaEvent_t start;
  TE_CUDA(pipe.make(&start));
  TE_CUDA(cudaEventRecord(start, c->stream));  // order after whatever the caller queued on the context stream
  TE_CUDA(cudaStreamWaitEvent(c->s_h2d, start, 0));
  TE_CUDA(cudaStreamWaitEvent(c->s_d2h, start, 0));
  te::SlabView v = make_view(c, g, s);
  int uploaded = 0;  // input-buffer columns already queued for upload
  int rc = TE_OK;
  for (int k = 0; k < nchunk && rc == TE_OK; ++k) {
    const int off = k * chunk, cnt = std::min(chunk, s.col_count - off);
    if (cnt <= 0) break;
    // chunk k reads input-buffer columns [halo_left + off - need, halo_left + off + cnt + need)
    const int upto = std::min(in_cols, s.halo_left + off + cnt + need);
    if (upto > uploaded) {
      cudaError_t e = upload_cols(din, elev, rows, st.cols, st.sr, st.sc, uploaded, upto - uploaded, c->s_h2d);
      if (e != cudaSuccess) { rc = fail(TE_ERR_CUDA, "H2D chunk copy failed: %s", cudaGetErrorString(e)); break; }
      uploaded = upto;
    }
    cudaEventRecord(up[k], c->s_h2d);
    cudaStreamWaitEvent(c->stream, up[k], 0);
    te::SlabView vk = v;
    vk.out_col0 = s.col_begin + off;
    vk.out_ncols = cnt;
    te::ChainOut ok{dev_out[0] + (size_t)off * rows, dev_out[1] + (size_t)off * rows, dev_out[2] + (size_t)off * rows,
                    dev_out[3] + (size_t)off * rows, dev_out[4] ? dev_out[4] + (size_t)off * rows : nullptr,
                    dev_out[5] ? dev_out[5] + (size_t)off * rows : nullptr, dev_out[6] ? dev_out[6] + (size_t)off * rows : nullptr};
    rc = run_chain_device(c, g, vk, p, din, ok, 1);
    if (rc != TE_OK) break;
    cudaEventRecord(done[k], c->stream);
    cudaStreamWaitEvent(c->s_d2h, done[k], 0);
    for (int l = 0; l < 7; ++l)
      if (host_out[l]) {
        cudaError_t e = download_cols(host_out[l], dev_out[l], rows, st.cols, st.sr, st.sc, off, cnt, c->s_d2h);
        if (e != cudaSuccess) { rc = fail(TE_ERR_CUDA, "D2H chunk copy failed: %s", cudaGetErrorString(e)); break; }
      }
  }
  cudaStreamSynchronize(c->s_h2d);
  cudaStreamSynchronize(c->stream);
  cudaError_t e = cudaStreamSynchronize(c->s_d2h);
  if (rc == TE_OK && e != cudaSuccess) rc = fail(TE_ERR_CUDA, "pipelined chain failed: %s", cudaGetErrorString(e));
  return rc;
}

static int chain_common(te_ctx* c, const te_geometry* g_in, const te_slab* slab, const te_chain_params* p, int nmaps, const float* elev,
                        float* slope, float* step, float* rough, float* trav, float* nx, float* ny, float* nz, int memory) {
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST && slab == nullptr && nmaps == 1, &g0)) return rc;
  const te_geometry* g = &g0;
  if (int rc = check_params(p)) return rc;
  if (nmaps <= 0) return fail(TE_ERR_BAD_ARG, "number of maps must be positive");
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (!slope || !step || !rough || !trav) return fail(TE_ERR_BAD_ARG, "output layer is null");
  te_slab s;
  if (int rc = resolve_slab(g, slab, chain_halo(g, p), &s)) return rc;
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g_in);
  float* host_out[7] = {slope, step, rough, trav, nx, ny, nz};
  if (memory == TE_MEM_HOST && nmaps == 1 && s.col_count >= 1024 && (size_t)g->rows * s.col_count >= ((size_t)1 << 22))
    return chain_host_pipelined(c, st, g, s, p, elev, host_out);
  const float* din = st.in_layer(elev, (s.halo_left + s.col_count + s.halo_right) * nmaps);
  float* o[7];
  for (int k = 0; k < 7; ++k) o[k] = st.out_layer(host_out[k], s.col_count * nmaps);
  if (st.rc) return st.rc;
  if (int rc = run_chain_device(c, g, make_view(c, g, s), p, din, te::ChainOut{o[0], o[1], o[2], o[3], o[4], o[5], o[6]}, nmaps)) return rc;
  return st.finish();
}

int te_chain(te_ctx* c, const te_geometry* g, const te_slab* slab, const te_chain_params* p, const float* elev, float* slope,
             float* step, float* rough, float* trav, float* nx, float* ny, float* nz, int memory) {
  TE_ENTER(c);
  return chain_common(c, g, slab, p, 1, elev, slope, step, rough, trav, nx, ny, nz, memory);
}

int te_chain_batched(te_ctx* c, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elev, float* slope,
                     float* step, float* rough, float* trav, int memory) {
  TE_ENTER(c);
  return chain_common(c, g, nullptr, p, nmaps, elev, slope, step, rough, trav, nullptr, nullptr, nullptr, memory);
}

// The batch of a footprint entry: nmaps whole maps of one geometry back to back (te_footprint_batched, te_footprint_polygon_batched),
// or one map or slab (nmaps = 1).  nmaps is a grid dimension of the sweep kernels, and their predicate work list stores 32-bit cell
// indices of the batch.
static int check_footprint_batch(const te_geometry* g, int nmaps) {
  if (nmaps <= 0) return fail(TE_ERR_BAD_ARG, "number of maps must be positive");
  if (nmaps > 65535) return fail(TE_ERR_UNSUPPORTED, "batch of %d maps: at most 65535", nmaps);
  if ((unsigned long long)nmaps * g->rows * g->cols >= (1ULL << 32)) return fail(TE_ERR_UNSUPPORTED, "batch of 2^32 or more cells");
  if ((unsigned long long)nmaps * g->cols >= (1ULL << 31)) return fail(TE_ERR_UNSUPPORTED, "batch of 2^31 or more columns");
  return TE_OK;
}

// te_footprint2 (one map or slab) and te_footprint_batched (nmaps whole maps).
static int footprint_common(te_ctx* c, const te_geometry* g_in, const te_slab* slab, const te_footprint_params* p, int nmaps,
                            const float* trav, const float* slope, const float* step, const float* rough, const float* elev, float* out,
                            float* slope_fp, float* step_fp, float* rough_fp, int memory) {
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST && slab == nullptr && nmaps == 1, &g0)) return rc;
  const te_geometry* g = &g0;
  if (!p) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (!(p->radius >= 0.0) || !(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint radius/offset must be >= 0");
  if (int rc = check_footprint_batch(g, nmaps)) return rc;
  if (int rc = check_filter_layers(p, trav, slope, step, elev, rough)) return rc;
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  const bool use_rough = p->verify_roughness != 0;
  te_slab s;
  if (int rc = resolve_slab(g, slab, te::footprint_halo(g, p), &s)) return rc;
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g_in);
  const int in_cols = (s.halo_left + s.col_count + s.halo_right) * nmaps, out_cols = s.col_count * nmaps;
  const float* in[5] = {st.in_layer(trav, in_cols), st.in_layer(slope, in_cols), st.in_layer(step, in_cols), st.in_layer(elev, in_cols),
                        st.in_layer(use_rough ? rough : nullptr, in_cols)};
  float* o[4] = {st.out_layer(out, out_cols), st.out_layer(slope_fp, out_cols), st.out_layer(step_fp, out_cols),
                 st.out_layer(use_rough ? rough_fp : nullptr, out_cols)};
  if (st.rc) return st.rc;
  int nl = 0;
  int rc = te::launch_footprint(c->fp, make_view(c, g, s), g, p, nmaps, in[0], in[1], in[2], in[4], in[3], o[0], o[1], o[2], o[3], c->sms,
                                c->stream, &nl);
  if (rc != 0) return fail(rc, "footprint sweep failed: %s", c->fp.why.c_str());
  if (int r2 = launch_check(c, "footprint", nl)) return r2;
  return st.finish();
}

int te_footprint2(te_ctx* c, const te_geometry* g, const te_slab* slab, const te_footprint_params* p, const float* trav,
                  const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                  float* step_fp, float* rough_fp, int memory) {
  TE_ENTER(c);
  return footprint_common(c, g, slab, p, 1, trav, slope, step, rough, elev, out, slope_fp, step_fp, rough_fp, memory);
}

int te_footprint_batched(te_ctx* c, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, const float* trav,
                         const float* slope, const float* step, const float* rough, const float* elev, float* out, float* slope_fp,
                         float* step_fp, float* rough_fp, int memory) {
  TE_ENTER(c);
  return footprint_common(c, g, nullptr, p, nmaps, trav, slope, step, rough, elev, out, slope_fp, step_fp, rough_fp, memory);
}

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
static int footprint_polygon_common(te_ctx* c, te::FootprintState* resident, const te_geometry* g_in, const te_slab* slab,
                                    const te_footprint_params* p, int nmaps, int32_t npts, const double* pts_xy, const float* trav,
                                    const float* slope, const float* step, const float* rough, const float* elev, int nouts,
                                    const PolygonOutputs* outs, const te::PolygonReduce* reduce, int memory, bool start_index_ok) {
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, resident || (memory == TE_MEM_HOST && start_index_ok), &g0)) return rc;
  const te_geometry* g = &g0;
  if (!p) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (npts < 3 || npts > 16 || !pts_xy) return fail(TE_ERR_BAD_ARG, "footprint polygon needs 3 to 16 vertices");
  for (int k = 0; k < nouts; ++k)
    for (int y = 0; y < outs[k].count; ++y)
      if (!std::isfinite(outs[k].yaws[y])) return fail(TE_ERR_BAD_ARG, "footprint yaw is not finite");
  for (int k = 0; k < 2 * npts; ++k)
    if (!std::isfinite(pts_xy[k])) return fail(TE_ERR_BAD_ARG, "footprint polygon vertex is not finite");
  // with a finite default every value is finite, so the reductions need no NaN rule
  if (reduce && !std::isfinite(p->traversability_default)) return fail(TE_ERR_BAD_ARG, "traversability_default is not finite (reductions over yaws)");
  if (int rc = check_footprint_batch(g, nmaps)) return rc;
  if (int rc = check_filter_layers(p, trav, slope, step, elev, rough)) return rc;
  for (int k = 0; k < nouts; ++k)
    if (!outs[k].out && !reduce) return fail(TE_ERR_BAD_ARG, "output layer is null");
  const bool use_rough = p->verify_roughness != 0;
  te_slab s;
  if (int rc = resolve_slab(g, slab, te::footprint_polygon_halo(g, p, npts, pts_xy), &s)) return rc;
  if (int rc = ensure_geometry(c, g)) return rc;
  Staging st(c, memory == TE_MEM_HOST, g_in);
  const int in_cols = (s.halo_left + s.col_count + s.halo_right) * nmaps, out_cols = s.col_count * nmaps;
  const float* in[5] = {trav, slope, step, elev, use_rough ? rough : nullptr};
  if (!resident)
    for (const float*& l : in) l = st.in_layer(l, in_cols);
  std::vector<te::PolygonLayer> layers;
  for (int k = 0; k < nouts; ++k) {
    if ((long long)outs[k].count * out_cols >= (1LL << 31)) return fail(TE_ERR_UNSUPPORTED, "output of 2^31 or more columns");
    float* const o = reduce ? nullptr : st.out_layer(outs[k].out, out_cols, outs[k].count);  // one staging buffer for all layers
    for (int y = 0; y < outs[k].count; ++y)
      layers.push_back(te::PolygonLayer{outs[k].yaws[y], o ? o + (size_t)y * out_cols * g->rows : nullptr});
  }
  te::PolygonReduce red{};
  if (reduce) red = {st.out_layer(reduce->worst, out_cols), st.out_layer(reduce->best, out_cols), st.out_layer(reduce->best_yaw, out_cols)};
  if (st.rc) return st.rc;
  te::FootprintState& fp = resident ? *resident : c->fp;
  int nl = 0;
  int rc = te::launch_footprint_polygon(fp, make_view(c, g, s), g, p, npts, pts_xy, (int)layers.size(), layers.data(), reduce ? &red : nullptr,
                                        in[0], in[1], in[2], in[4], in[3], nmaps, c->sms, c->stream, &nl);
  if (rc != 0) return fail(rc, "polygon footprint sweep failed: %s", fp.why.c_str());
  if (int r2 = launch_check(c, "polygon footprint", nl)) return r2;
  return st.finish();
}

// traversability_x is the footprint at yaw 0: the rotation of yaw 0 is the identity, exactly (te::launch_footprint_polygon).
static int footprint_polygon_pair(te_ctx* c, const te_geometry* g, const te_slab* slab, const te_footprint_params* p, int nmaps,
                                  int32_t npts, const double* pts_xy, double yaw, const float* trav, const float* slope, const float* step,
                                  const float* rough, const float* elev, float* out_x, float* out_rot, int memory) {
  static const double identity = 0.0;
  const PolygonOutputs outs[2] = {{out_x, 1, &identity}, {out_rot, 1, &yaw}};
  return footprint_polygon_common(c, nullptr, g, slab, p, nmaps, npts, pts_xy, trav, slope, step, rough, elev, 2, outs, nullptr, memory,
                                  slab == nullptr && nmaps == 1);
}

int te_footprint_polygon(te_ctx* c, const te_geometry* g, const te_slab* slab, const te_footprint_params* p, int32_t npts,
                         const double* pts_xy, double yaw, const float* trav, const float* slope, const float* step, const float* rough,
                         const float* elev, float* out_x, float* out_rot, int memory) {
  TE_ENTER(c);
  return footprint_polygon_pair(c, g, slab, p, 1, npts, pts_xy, yaw, trav, slope, step, rough, elev, out_x, out_rot, memory);
}

int te_footprint_polygon_batched(te_ctx* c, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                                 const double* pts_xy, double yaw, const float* trav, const float* slope, const float* step,
                                 const float* rough, const float* elev, float* out_x, float* out_rot, int memory) {
  TE_ENTER(c);
  return footprint_polygon_pair(c, g, nullptr, p, nmaps, npts, pts_xy, yaw, trav, slope, step, rough, elev, out_x, out_rot, memory);
}

// The list of yaws of the yaws entries (the cap bounds the host classification and the table upload of one call).
static int check_yaws(int32_t nyaws, const double* yaws) {
  if (nyaws < 1 || !yaws) return fail(TE_ERR_BAD_ARG, "footprint yaws: need 1 or more");
  if (nyaws > 1024) return fail(TE_ERR_UNSUPPORTED, "%d footprint yaws: at most 1024 per call", nyaws);
  return TE_OK;
}

static int check_reduce_outputs(const te::PolygonReduce& r) {
  if (!r.worst && !r.best && !r.best_yaw) return fail(TE_ERR_BAD_ARG, "no output: worst, best and best_yaw are all null");
  return TE_OK;
}

int te_footprint_polygon_yaws(te_ctx* c, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                              const double* pts_xy, int32_t nyaws, const double* yaws, const float* trav, const float* slope,
                              const float* step, const float* rough, const float* elev, float* out, int memory) {
  TE_ENTER(c);
  if (int rc = check_yaws(nyaws, yaws)) return rc;
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  const PolygonOutputs outs[1] = {{out, nyaws, yaws}};
  return footprint_polygon_common(c, nullptr, g, nullptr, p, nmaps, npts, pts_xy, trav, slope, step, rough, elev, 1, outs, nullptr, memory,
                                  false);
}

int te_footprint_polygon_yaws_reduce(te_ctx* c, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, int32_t npts,
                                     const double* pts_xy, int32_t nyaws, const double* yaws, const float* trav, const float* slope,
                                     const float* step, const float* rough, const float* elev, float* worst, float* best,
                                     int32_t* best_yaw, int memory) {
  TE_ENTER(c);
  if (int rc = check_yaws(nyaws, yaws)) return rc;
  const te::PolygonReduce red{worst, best, best_yaw};
  if (int rc = check_reduce_outputs(red)) return rc;
  const PolygonOutputs outs[1] = {{nullptr, nyaws, yaws}};
  return footprint_polygon_common(c, nullptr, g, nullptr, p, nmaps, npts, pts_xy, trav, slope, step, rough, elev, 1, outs, &red, memory,
                                  false);
}

int te_footprint(te_ctx* c, const te_geometry* g, const te_slab* slab, const te_footprint_params* p, const float* trav,
                 const float* slope, const float* step, const float* elev, float* out, float* slope_fp, float* step_fp, int memory) {
  if (p && p->verify_roughness) return fail(TE_ERR_MISSING_LAYER, "verify_roughness is set: call te_footprint2 with the traversability_roughness layer");
  return te_footprint2(c, g, slab, p, trav, slope, step, nullptr, elev, out, slope_fp, step_fp, nullptr, memory);
}

// The untraversable-polygon outputs of te_check_footprint_paths_fresh2 / _polygon2: both null (no polygon), or counts with room
// for max_vertices >= 0 points per path (xy may be null only when max_vertices is 0).
static int check_polygon_outputs(int32_t max_vertices, const int32_t* ucount, const double* uxy) {
  if (max_vertices < 0) return fail(TE_ERR_BAD_ARG, "max_vertices must be >= 0, got %d", max_vertices);
  if (ucount && !uxy && max_vertices > 0) return fail(TE_ERR_BAD_ARG, "untraversable_count given without untraversable_xy");
  if (!ucount && uxy) return fail(TE_ERR_BAD_ARG, "untraversable_xy given without untraversable_count");
  return TE_OK;
}

// The radius of circular path q in host memory: the fresh check walks rings 0 .. 127 of the spiral.
static int check_circular_radius(const te_geometry* g, const te_footprint_params* p, int32_t q, double radius) {
  if (!(radius >= 0.0)) return fail(TE_ERR_BAD_ARG, "radius of path %d is negative or NaN", q);
  if (!(std::ceil((radius + p->offset) / g->resolution) <= 127.0))
    return fail(TE_ERR_UNSUPPORTED, "radius of path %d + offset spans more than 127 cells", q);
  return TE_OK;
}

int te_check_footprint_paths(te_ctx* c, const te_geometry* g, const float* footprint, double traversability_default, int32_t npaths,
                             const int32_t* path_begin, const double* poses_xy, uint8_t* is_safe, double* traversability, int memory) {
  return te_check_footprint_paths2(c, g, footprint, nullptr, traversability_default, npaths, path_begin, poses_xy, is_safe, traversability, memory);
}

int te_check_footprint_paths2(te_ctx* c, const te_geometry* g, const float* footprint, const float* robot_slope, double traversability_default,
                              int32_t npaths, const int32_t* path_begin, const double* poses_xy, uint8_t* is_safe, double* traversability,
                              int memory) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (!footprint) return fail(TE_ERR_MISSING_LAYER, "layer traversability_footprint is missing");
  if (npaths < 0 || !path_begin || !poses_xy || !is_safe || !traversability) return fail(TE_ERR_BAD_ARG, "null argument or negative path count");
  if (npaths == 0) return TE_OK;
  if (int rc = ensure_geometry(c, g)) return rc;
  const bool host = memory != TE_MEM_DEVICE;
  int32_t nposes = 0;
  if (host) {  // path_begin is readable here, so the pose count is known
    nposes = path_begin[npaths];
    if (nposes < 0) return fail(TE_ERR_BAD_ARG, "path_begin must be non-decreasing");
  }
  Staging st(c, host, g);
  const float* dfp = st.in_layer(footprint, g->cols);
  const float* drs = st.in_layer(robot_slope, g->cols);
  const int32_t* dpb = st.in(path_begin, (size_t)npaths + 1);
  const double* dxy = st.in(poses_xy, 2 * (size_t)nposes);
  uint8_t* dsafe = st.out(is_safe, (size_t)npaths);
  double* dtrav = st.out(traversability, (size_t)npaths);
  if (st.rc) return st.rc;
  const te_slab s{0, g->cols, 0, 0};
  te::launch_check_paths(make_view(c, g, s), g, traversability_default, dfp, drs, npaths, dpb, dxy, dsafe, dtrav, c->stream);
  if (int rc = launch_check(c, "k_check_paths")) return rc;
  return st.finish();
}

int te_check_footprint_paths_fresh(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, const float* trav, const float* slope,
                                   const float* step, const float* rough, const float* elev, const float* robot_slope, int32_t npaths,
                                   const int32_t* path_begin, const double* poses_xy, const double* radius, const uint8_t* cup,
                                   uint8_t* is_safe, double* traversability, int memory) {
  return te_check_footprint_paths_fresh2(c, g_in, p, trav, slope, step, rough, elev, robot_slope, npaths, path_begin, poses_xy, radius, cup,
                                         is_safe, traversability, 0, nullptr, nullptr, memory);
}

// Stages the path arrays of `r` and points `r` at the device copies (host memory; null stays null).
static void stage_paths(Staging& st, te::PathChecks& r) {
  const size_t np = (size_t)r.npaths;
  r.path_map = st.in(r.path_map, np);
  r.path_begin = st.in(r.path_begin, np + 1);
  r.poses = st.in(r.poses, (size_t)r.pose_stride * r.nposes);
  r.radius = st.in(r.radius, np);
  r.footprint_begin = st.in(r.footprint_begin, np + 1);
  r.footprint_xyz = st.in(r.footprint_xyz, 3 * (size_t)r.nvertices);
  r.conservative = st.in(r.conservative, np);
  r.cup = st.in(r.cup, np);
  r.is_safe = st.out(r.is_safe, np);
  r.trav_out = st.out(r.trav_out, np);
  r.area_out = st.out(r.area_out, np);
  r.ucount = st.out(r.ucount, np);
  r.uxy = st.out(r.uxy, 2 * (size_t)r.max_vertices * np);
}

// The body of te_check_footprint_paths_fresh2, te_check_footprint_paths_polygon2, te_check_footprint_request and
// te_check_footprint_request_batched once the entry has put its arguments into `r` (the caller's pointers): the checks they share,
// then in host memory `host_checks(g, r)` (the entry's validation of the path arrays; it sets r.nposes where the entry has none,
// and r.max_points), the staging of r.nmaps maps, the launches and the download.  Device memory reads nothing back: a path that
// cannot be checked gets is_safe 0 and NaN (te_b200.h).  A batch (r.path_map) takes maps in default order only.
static int run_path_checks(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, te::PathChecks r, int memory, const char* what,
                           const std::function<int(const te_geometry*, te::PathChecks&)>& host_checks) {
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, memory != TE_MEM_DEVICE && !r.path_map, &g0)) return rc;
  const te_geometry* g = &g0;
  if (r.nmaps < 1) return fail(TE_ERR_BAD_ARG, "number of maps must be positive");
  if ((long long)r.nmaps * g->cols >= (1LL << 31)) return fail(TE_ERR_UNSUPPORTED, "batch of 2^31 or more columns");
  if (!p) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  const bool circular = r.footprint_begin || !r.footprint, polygonal = r.footprint_begin || r.footprint;
  if (circular && !(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint offset must be >= 0");
  if (int rc = check_filter_layers(p, r.trav, r.slope, r.step, r.elev, r.rough)) return rc;
  if (r.npaths < 0 || !r.path_begin || !r.poses || (circular && !r.radius) || !r.is_safe || !r.trav_out ||
      (polygonal && (r.nposes < 0 || !r.area_out)))
    return fail(TE_ERR_BAD_ARG, "null argument or negative count");
  if (int rc = check_polygon_outputs(r.max_vertices, r.ucount, r.uxy)) return rc;
  if (r.npaths == 0) return TE_OK;
  if (int rc = ensure_geometry(c, g)) return rc;
  const bool host = memory != TE_MEM_DEVICE;
  if (host)
    if (int rc = host_checks(g, r)) return rc;
  int32_t* const ucount = r.ucount;
  Staging st(c, host, g_in);
  const int ncols = g->cols * r.nmaps;
  r.trav = st.in_layer(r.trav, ncols);
  r.slope = st.in_layer(r.slope, ncols);
  r.step = st.in_layer(r.step, ncols);
  r.elev = st.in_layer(r.elev, ncols);
  r.rough = st.in_layer(p->verify_roughness ? r.rough : nullptr, ncols);
  r.robot_slope = st.in_layer(r.robot_slope, ncols);
  stage_paths(st, r);
  if (st.rc) return st.rc;
  const te_slab s{0, g->cols, 0, 0};
  int nl = 0;
  int rc = te::launch_path_checks(c->fp, make_view(c, g, s), g, p, r, true, true, c->stream, &nl);
  if (rc != 0) return fail(rc, "%s failed: %s", what, c->fp.why.c_str());
  if (int r2 = launch_check(c, what, nl)) return r2;
  if (int r2 = st.finish()) return r2;
  if (host && ucount)  // the row bound of a polygonal path's polygon table (kUntravRows) is only known once the hulls are
    for (int32_t q = 0; q < r.npaths; ++q)
      if (ucount[q] < 0)
        return fail(TE_ERR_UNSUPPORTED, "the untraversable polygon of path %d spans more than %d map rows", q, te::kUntravRows);
  return TE_OK;
}

int te_check_footprint_paths_fresh2(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, const float* trav, const float* slope,
                                    const float* step, const float* rough, const float* elev, const float* robot_slope, int32_t npaths,
                                    const int32_t* path_begin, const double* poses_xy, const double* radius, const uint8_t* cup,
                                    uint8_t* is_safe, double* traversability, int32_t max_vertices, int32_t* ucount, double* uxy,
                                    int memory) {
  TE_ENTER(c);
  te::PathChecks r{};
  r.trav = trav; r.slope = slope; r.step = step; r.rough = rough; r.elev = elev; r.robot_slope = robot_slope; r.nmaps = 1;
  r.npaths = npaths; r.nposes = -1; r.path_begin = path_begin; r.poses = poses_xy; r.pose_stride = 2; r.radius = radius; r.cup = cup;
  r.is_safe = is_safe; r.trav_out = traversability; r.max_vertices = max_vertices; r.ucount = ucount; r.uxy = uxy;
  return run_path_checks(c, g_in, p, r, memory, "fresh path check", [&](const te_geometry* g, te::PathChecks& h) -> int {
    if (path_begin[0] < 0) return fail(TE_ERR_BAD_ARG, "path_begin[0] must be >= 0");
    for (int32_t q = 0; q < npaths; ++q) {
      if (path_begin[q + 1] < path_begin[q]) return fail(TE_ERR_BAD_ARG, "path_begin must be non-decreasing");
      if (int rc = check_circular_radius(g, p, q, radius[q])) return rc;
    }
    h.nposes = path_begin[npaths];
    return TE_OK;
  });
}

int te_check_footprint_paths_polygon(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, const float* trav, const float* slope,
                                     const float* step, const float* rough, const float* elev, const float* robot_slope, int32_t nfootprint,
                                     const float* footprint_xyz, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                     const double* poses, const uint8_t* conservative, uint8_t* is_safe, double* traversability,
                                     double* area, int memory) {
  return te_check_footprint_paths_polygon2(c, g_in, p, trav, slope, step, rough, elev, robot_slope, nfootprint, footprint_xyz, npaths, nposes,
                                           path_begin, poses, conservative, is_safe, traversability, area, nullptr, 0, nullptr, nullptr,
                                           memory);
}

int te_check_footprint_paths_polygon2(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, const float* trav, const float* slope,
                                      const float* step, const float* rough, const float* elev, const float* robot_slope, int32_t nfootprint,
                                      const float* footprint_xyz, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                      const double* poses, const uint8_t* conservative, uint8_t* is_safe, double* traversability,
                                      double* area, const uint8_t* cup, int32_t max_vertices, int32_t* ucount, double* uxy, int memory) {
  TE_ENTER(c);
  if (!footprint_xyz) return fail(TE_ERR_BAD_ARG, "null argument or negative count");
  if (nfootprint < 1 || nfootprint > te::kPolyMaxVerts) return fail(TE_ERR_BAD_ARG, "footprint needs 1..%d vertices, got %d", te::kPolyMaxVerts, nfootprint);
  for (int k = 0; k < 3 * nfootprint; ++k)
    if (!std::isfinite(footprint_xyz[k])) return fail(TE_ERR_BAD_ARG, "footprint vertex %d is not finite", k / 3);
  te::PathChecks r{};
  r.trav = trav; r.slope = slope; r.step = step; r.rough = rough; r.elev = elev; r.robot_slope = robot_slope; r.nmaps = 1;
  r.npaths = npaths; r.nposes = nposes; r.path_begin = path_begin; r.poses = poses; r.pose_stride = 7;
  r.nfp = nfootprint; r.footprint = footprint_xyz; r.conservative = conservative; r.cup = ucount ? cup : nullptr;
  // the hull input bound of one item; host memory sizes it from the paths
  r.max_points = conservative ? 2 * te::kPolyConsCap : 2 * nfootprint;
  r.is_safe = is_safe; r.trav_out = traversability; r.area_out = area; r.max_vertices = max_vertices; r.ucount = ucount; r.uxy = uxy;
  return run_path_checks(c, g_in, p, r, memory, "polygonal path check", [&](const te_geometry*, te::PathChecks& h) -> int {
    if (path_begin[0] < 0) return fail(TE_ERR_BAD_ARG, "path_begin[0] must be >= 0");
    if (path_begin[npaths] != nposes) return fail(TE_ERR_BAD_ARG, "path_begin[npaths] = %d != nposes = %d", path_begin[npaths], nposes);
    h.max_points = 2 * nfootprint;
    for (int32_t q = 0; q < npaths; ++q) {
      const int32_t n = path_begin[q + 1] - path_begin[q];
      if (n < 0) return fail(TE_ERR_BAD_ARG, "path_begin must be non-decreasing");
      if (conservative && conservative[q] && n > 1) {
        if ((long long)nfootprint * n > te::kPolyConsCap)
          return fail(TE_ERR_UNSUPPORTED, "conservative path %d needs %lld polygon vertices, more than %d", q, (long long)nfootprint * n,
                      te::kPolyConsCap);
        h.max_points = std::max(h.max_points, 2 * nfootprint * n);
      }
    }
    for (size_t k = 0; k < 7 * (size_t)nposes; ++k)
      if (!std::isfinite(poses[k])) return fail(TE_ERR_BAD_ARG, "pose %zu is not finite", k / 7);
    return TE_OK;
  });
}

// The host-side validation of a te_check_footprint_request request (paths, footprints, radii, conservative caps, finite poses and
// vertices); sets *mp to the hull input bound of a polygonal item.
static int check_request_host(const te_geometry* g, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                              const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                              const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative, int* mp_out) {
  if (path_begin[0] < 0) return fail(TE_ERR_BAD_ARG, "path_begin[0] must be >= 0");
  if (path_begin[npaths] != nposes) return fail(TE_ERR_BAD_ARG, "path_begin[npaths] = %d != nposes = %d", path_begin[npaths], nposes);
  if (footprint_begin[0] != 0) return fail(TE_ERR_BAD_ARG, "footprint_begin[0] must be 0, got %d", footprint_begin[0]);
  if (footprint_begin[npaths] != nvertices)
    return fail(TE_ERR_BAD_ARG, "footprint_begin[npaths] = %d != nvertices = %d", footprint_begin[npaths], nvertices);
  for (int32_t q = 0; q < npaths; ++q) {
    if (path_begin[q + 1] < path_begin[q]) return fail(TE_ERR_BAD_ARG, "path_begin must be non-decreasing");
    if (footprint_begin[q + 1] < footprint_begin[q]) return fail(TE_ERR_BAD_ARG, "footprint_begin must be non-decreasing");
  }
  int mp = 2;
  for (int32_t q = 0; q < npaths; ++q) {
    const int32_t n = path_begin[q + 1] - path_begin[q], nfp = footprint_begin[q + 1] - footprint_begin[q];
    if (nfp == 0) {  // circular: te_check_footprint_paths_fresh2
      if (int rc = check_circular_radius(g, p, q, radius[q])) return rc;
      continue;
    }
    // polygonal: te_check_footprint_paths_polygon2
    if (nfp > max_footprint_vertices)
      return fail(TE_ERR_BAD_ARG, "footprint of path %d has %d vertices, more than max_footprint_vertices = %d", q, nfp,
                  max_footprint_vertices);
    mp = std::max(mp, 2 * nfp);
    if (conservative && conservative[q] && n > 1) {
      if ((long long)nfp * n > te::kPolyConsCap)
        return fail(TE_ERR_UNSUPPORTED, "conservative path %d needs %lld polygon vertices, more than %d", q, (long long)nfp * n,
                    te::kPolyConsCap);
      mp = std::max(mp, 2 * nfp * n);
    }
    for (size_t k = 7 * (size_t)path_begin[q]; k < 7 * (size_t)path_begin[q + 1]; ++k)
      if (!std::isfinite(poses[k])) return fail(TE_ERR_BAD_ARG, "pose %zu is not finite", k / 7);
  }
  for (int k = 0; k < 3 * nvertices; ++k)
    if (!std::isfinite(footprint_xyz[k])) return fail(TE_ERR_BAD_ARG, "footprint vertex %d is not finite", k / 3);
  *mp_out = mp;
  return TE_OK;
}

// te_check_footprint_request (one map, path_map null) and te_check_footprint_request_batched (nmaps maps, path q on path_map[q]).
static int footprint_request_common(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, int32_t nmaps, const float* trav,
                                    const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                                    const int32_t* path_map, int32_t npaths, int32_t nposes, const int32_t* path_begin, const double* poses,
                                    const double* radius, int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                    int32_t max_footprint_vertices, const uint8_t* conservative, const uint8_t* cup, uint8_t* is_safe,
                                    double* traversability, double* area, int32_t max_vertices, int32_t* ucount, double* uxy,
                                    int memory) {
  if (nvertices < 0 || !footprint_begin || (nvertices > 0 && !footprint_xyz)) return fail(TE_ERR_BAD_ARG, "null argument or negative count");
  if (max_footprint_vertices < 0 || max_footprint_vertices > te::kPolyMaxVerts)
    return fail(TE_ERR_BAD_ARG, "max_footprint_vertices must be 0..%d, got %d", te::kPolyMaxVerts, max_footprint_vertices);
  // The hull input bound of a polygonal item: as te_check_footprint_paths_polygon2 for the largest footprint; host memory sizes it
  // from the paths.
  te::PathChecks r{};
  r.trav = trav; r.slope = slope; r.step = step; r.rough = rough; r.elev = elev; r.robot_slope = robot_slope;
  r.nmaps = nmaps; r.path_map = path_map;
  r.npaths = npaths; r.nposes = nposes; r.path_begin = path_begin; r.poses = poses; r.pose_stride = 7; r.radius = radius;
  r.footprint_begin = footprint_begin; r.footprint_xyz = footprint_xyz; r.nvertices = nvertices;
  r.max_footprint_vertices = max_footprint_vertices; r.conservative = conservative; r.cup = cup;
  r.max_points = conservative && max_footprint_vertices > 0 ? 2 * te::kPolyConsCap : 2 * std::max(max_footprint_vertices, 1);
  r.is_safe = is_safe; r.trav_out = traversability; r.area_out = area; r.max_vertices = max_vertices; r.ucount = ucount; r.uxy = uxy;
  return run_path_checks(c, g_in, p, r, memory, "footprint path request", [&](const te_geometry* g, te::PathChecks& h) {
    for (int32_t q = 0; path_map && q < npaths; ++q)
      if (path_map[q] < 0 || path_map[q] >= nmaps)
        return fail(TE_ERR_BAD_ARG, "path_map[%d] = %d is outside 0..%d", q, path_map[q], nmaps - 1);
    return check_request_host(g, p, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin, footprint_xyz,
                              max_footprint_vertices, conservative, &h.max_points);
  });
}

int te_check_footprint_request(te_ctx* c, const te_geometry* g_in, const te_footprint_params* p, const float* trav, const float* slope,
                               const float* step, const float* rough, const float* elev, const float* robot_slope, int32_t npaths,
                               int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius, int32_t nvertices,
                               const int32_t* footprint_begin, const float* footprint_xyz, int32_t max_footprint_vertices,
                               const uint8_t* conservative, const uint8_t* cup, uint8_t* is_safe, double* traversability, double* area,
                               int32_t max_vertices, int32_t* ucount, double* uxy, int memory) {
  TE_ENTER(c);
  return footprint_request_common(c, g_in, p, 1, trav, slope, step, rough, elev, robot_slope, nullptr, npaths, nposes, path_begin, poses,
                                  radius, nvertices, footprint_begin, footprint_xyz, max_footprint_vertices, conservative, cup, is_safe,
                                  traversability, area, max_vertices, ucount, uxy, memory);
}

int te_check_footprint_request_batched(te_ctx* c, const te_geometry* g, const te_footprint_params* p, int32_t nmaps, const float* trav,
                                       const float* slope, const float* step, const float* rough, const float* elev,
                                       const float* robot_slope, const int32_t* path_map, int32_t npaths, int32_t nposes,
                                       const int32_t* path_begin, const double* poses, const double* radius, int32_t nvertices,
                                       const int32_t* footprint_begin, const float* footprint_xyz, int32_t max_footprint_vertices,
                                       const uint8_t* conservative, const uint8_t* cup, uint8_t* is_safe, double* traversability,
                                       double* area, int32_t max_vertices, int32_t* ucount, double* uxy, int memory) {
  TE_ENTER(c);
  if (!path_map) return fail(TE_ERR_BAD_ARG, "path_map is null");
  return footprint_request_common(c, g, p, nmaps, trav, slope, step, rough, elev, robot_slope, path_map, npaths, nposes, path_begin, poses,
                                  radius, nvertices, footprint_begin, footprint_xyz, max_footprint_vertices, conservative, cup, is_safe,
                                  traversability, area, max_vertices, ucount, uxy, memory);
}

// ---- te_map: the layers, the traversability_footprint cache and the isTraversableForFilters memo, resident on the device -------
struct te_map {
  te_ctx* ctx = nullptr;
  bool have_layers = false;
  te_geometry geo_in{};  // as the layers came (host memory: with their circular-buffer start index)
  te_geometry geo{};     // the same with the start index cleared: the device layers are in default order
  DevBuf trav, slope, step, rough, elev, rslope, cache, fresh;
  DevBuf gather;  // te_map_get_submaps: the source-layer table, then the windows (te::SubmapWindow)
  bool have_rough = false, have_rslope = false;
  te::FootprintState fp;  // the map's own scratch; fp.memo is the resident memo
  bool memo_valid = false;
  double memo_gap = 0.0, memo_crit = 0.0;
  int memo_rough = 0;
  te::MapRequestStats last{};
};

namespace {

size_t map_cells(const te_map* m) { return (size_t)m->geo.rows * m->geo.cols; }

int map_ready(const te_map* m) {
  if (!m->have_layers) return fail(TE_ERR_BAD_ARG, "the map has no layers yet: call te_map_chain or te_map_set_layers first");
  return TE_OK;
}

// New layers: the geometry, an empty cache and a memo to be rebuilt.
int map_reset(te_map* m, const te_geometry* g_in, const te_geometry* g) {
  te_ctx* c = m->ctx;
  const size_t bytes = sizeof(float) * (size_t)g->rows * g->cols;
  for (DevBuf* b : {&m->trav, &m->slope, &m->step, &m->elev, &m->cache}) TE_CUDA(b->reserve(bytes));
  TE_CUDA(cudaMemsetAsync(m->cache.p, 0xff, bytes, c->stream));  // all-ones bits: NaN, the empty cache of computeTraversability (:225-228)
  m->geo_in = *g_in;
  m->geo = *g;
  m->memo_valid = false;
  m->have_layers = false;
  return TE_OK;
}

// One layer into the map: host layers are unwrapped from their start index; device layers are copied.
int map_put_layer(te_map* m, DevBuf& dst, const float* src, int memory) {
  te_ctx* c = m->ctx;
  const te_geometry& g = m->geo_in;
  TE_CUDA(dst.reserve(sizeof(float) * map_cells(m)));
  if (memory == TE_MEM_HOST) TE_CUDA(upload_cols((float*)dst.p, src, g.rows, g.cols, g.start_row, g.start_col, 0, g.cols, c->stream));
  else TE_CUDA(cudaMemcpyAsync(dst.p, src, sizeof(float) * map_cells(m), cudaMemcpyDeviceToDevice, c->stream));
  return TE_OK;
}

// A map layer out: host layers are re-wrapped to the map's start index (the caller synchronises); device layers are copied.
int map_get_layer(te_map* m, float* dst, const void* src, int memory) {
  te_ctx* c = m->ctx;
  const te_geometry& g = m->geo_in;
  if (memory == TE_MEM_HOST) TE_CUDA(download_cols(dst, (const float*)src, g.rows, g.cols, g.start_row, g.start_col, 0, g.cols, c->stream));
  else TE_CUDA(cudaMemcpyAsync(dst, src, sizeof(float) * map_cells(m), cudaMemcpyDeviceToDevice, c->stream));
  return TE_OK;
}

// The resident isTraversableForFilters memo for these parameters: kept while the layers and max_gap_width, critical_step_height
// and verify_roughness (all that checkForStep / checkForSlope / checkForRoughness read) stay the same, cleared otherwise.
int map_memo(te_map* m, const te_footprint_params* p) {
  const int rough = p->verify_roughness != 0;
  if (m->memo_valid && m->memo_gap == p->max_gap_width && m->memo_crit == p->critical_step_height && m->memo_rough == rough) return TE_OK;
  TE_CUDA(m->fp.memo.reserve(map_cells(m)));
  TE_CUDA(cudaMemsetAsync(m->fp.memo.p, 0, map_cells(m), m->ctx->stream));
  m->memo_valid = true;
  m->memo_gap = p->max_gap_width;
  m->memo_crit = p->critical_step_height;
  m->memo_rough = rough;
  return TE_OK;
}

int map_footprint_params(const te_map* m, const te_footprint_params* p) {
  if (!p) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (p->verify_roughness && !m->have_rough)
    return fail(TE_ERR_MISSING_LAYER, "layer traversability_roughness is missing (verify_roughness is set)");
  return TE_OK;
}

// The map's layers of `mask`, in te_layer bit order (the order of every output that holds several).
int map_layers(const te_map* m, uint32_t mask, const float* out[7], int* n) {
  if (mask == 0 || (mask & ~(uint32_t)TE_LAYER_ALL)) return fail(TE_ERR_BAD_ARG, "layer mask 0x%x: need a non-empty subset of 0x%x", mask, TE_LAYER_ALL);
  static const char* const names[7] = {"traversability", "traversability_slope", "traversability_step", "traversability_roughness",
                                       "elevation", "robot_slope", "traversability_footprint"};
  const DevBuf* const src[7] = {&m->trav, &m->slope, &m->step, m->have_rough ? &m->rough : nullptr, &m->elev,
                                m->have_rslope ? &m->rslope : nullptr, &m->cache};
  *n = 0;
  for (int b = 0; b < 7; ++b) {
    if (!((mask >> b) & 1u)) continue;
    if (!src[b]) return fail(TE_ERR_MISSING_LAYER, "layer %s is missing: the map does not hold it", names[b]);
    out[(*n)++] = (const float*)src[b]->p;
  }
  return TE_OK;
}

#define TE_MAP_ENTER(map)                                   \
  if (!(map)) return fail(TE_ERR_BAD_ARG, "map is null");   \
  te_ctx* c = (map)->ctx;                                   \
  TE_ENTER(c)

}  // namespace

int te_map_create(te_ctx* c, te_map** out) {
  if (!out) return fail(TE_ERR_BAD_ARG, "out pointer is null");
  *out = nullptr;
  TE_ENTER(c);
  te_map* m = new te_map();
  m->ctx = c;
  *out = m;
  return TE_OK;
}

int te_map_destroy(te_map* m) {
  if (!m) return TE_OK;
  {
    Guard g(m->ctx);
    if (g.ok) {
      cudaStreamSynchronize(m->ctx->stream);
      for (DevBuf* b : {&m->trav, &m->slope, &m->step, &m->rough, &m->elev, &m->rslope, &m->cache, &m->fresh, &m->gather}) b->release();
      m->fp.release();
    }
  }
  delete m;
  return TE_OK;
}

int te_map_chain(te_map* m, const te_geometry* g_in, const te_chain_params* p, const float* elev, float* slope, float* step, float* rough,
                 float* trav, int memory) {
  TE_MAP_ENTER(m);
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST, &g0)) return rc;
  if (int rc = check_params(p)) return rc;
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (int rc = map_reset(m, g_in, &g0)) return rc;
  TE_CUDA(m->rough.reserve(sizeof(float) * map_cells(m)));
  if (int rc = map_put_layer(m, m->elev, elev, memory)) return rc;
  if (int rc = chain_common(c, &g0, nullptr, p, 1, (const float*)m->elev.p, (float*)m->slope.p, (float*)m->step.p, (float*)m->rough.p,
                            (float*)m->trav.p, nullptr, nullptr, nullptr, TE_MEM_DEVICE))
    return rc;
  m->have_rough = true;
  m->have_rslope = false;  // computeTraversability leaves robot_slope to a later setTraversabilityMap
  m->have_layers = true;
  const std::pair<float*, DevBuf*> outs[4] = {{slope, &m->slope}, {step, &m->step}, {rough, &m->rough}, {trav, &m->trav}};
  for (const auto& o : outs)
    if (o.first)
      if (int rc = map_get_layer(m, o.first, o.second->p, memory)) return rc;
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

int te_map_set_layers(te_map* m, const te_geometry* g_in, const float* trav, const float* slope, const float* step, const float* rough,
                      const float* elev, const float* robot_slope, int memory) {
  TE_MAP_ENTER(m);
  te_geometry g0;
  if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST, &g0)) return rc;
  if (!trav) return fail(TE_ERR_MISSING_LAYER, "layer traversability is missing");
  if (!slope) return fail(TE_ERR_MISSING_LAYER, "layer traversability_slope is missing");
  if (!step) return fail(TE_ERR_MISSING_LAYER, "layer traversability_step is missing");
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (int rc = map_reset(m, g_in, &g0)) return rc;
  if (int rc = map_put_layer(m, m->trav, trav, memory)) return rc;
  if (int rc = map_put_layer(m, m->slope, slope, memory)) return rc;
  if (int rc = map_put_layer(m, m->step, step, memory)) return rc;
  if (int rc = map_put_layer(m, m->elev, elev, memory)) return rc;
  if (rough)
    if (int rc = map_put_layer(m, m->rough, rough, memory)) return rc;
  if (robot_slope)
    if (int rc = map_put_layer(m, m->rslope, robot_slope, memory)) return rc;
  m->have_rough = rough != nullptr;
  m->have_rslope = robot_slope != nullptr;
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));  // the caller may reuse its layers on return
  m->have_layers = true;
  return TE_OK;
}

int te_map_footprint(te_map* m, const te_footprint_params* p, float* out, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  if (!(p->radius >= 0.0) || !(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint radius/offset must be >= 0");
  const te_geometry* g = &m->geo;
  if (int rc = ensure_geometry(c, g)) return rc;
  TE_CUDA(m->fresh.reserve(sizeof(float) * map_cells(m)));
  const te_slab s{0, g->cols, 0, 0};
  const float* rough = p->verify_roughness ? (const float*)m->rough.p : nullptr;
  int nl = 0;
  int rc = te::launch_footprint(m->fp, make_view(c, g, s), g, p, 1, (const float*)m->trav.p, (const float*)m->slope.p, (const float*)m->step.p,
                                rough, (const float*)m->elev.p, (float*)m->fresh.p, nullptr, nullptr, nullptr, c->sms, c->stream, &nl);
  if (rc != 0) return fail(rc, "footprint sweep failed: %s", m->fp.why.c_str());
  te::launch_map_merge((const float*)m->fresh.p, (float*)m->cache.p, (out && memory == TE_MEM_DEVICE) ? out : nullptr, map_cells(m), c->sms,
                       c->stream);
  if (int r2 = launch_check(c, "map footprint", nl + 1)) return r2;
  if (out && memory == TE_MEM_HOST) {
    if (int r2 = map_get_layer(m, out, m->cache.p, memory)) return r2;
    TE_CUDA(cudaStreamSynchronize(c->stream));
  }
  return TE_OK;
}

// The te_map polygon entries: footprint_polygon_common on the map's resident layers with the map's own state.  They neither read
// nor change the traversability_footprint cache or the memo.
static int map_footprint_polygon(te_map* m, const te_footprint_params* p, int32_t npts, const double* pts_xy, int nouts,
                                 const PolygonOutputs* outs, const te::PolygonReduce* reduce, int memory) {
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  return footprint_polygon_common(m->ctx, &m->fp, &m->geo_in, nullptr, p, 1, npts, pts_xy, (const float*)m->trav.p, (const float*)m->slope.p,
                                  (const float*)m->step.p, m->have_rough ? (const float*)m->rough.p : nullptr, (const float*)m->elev.p,
                                  nouts, outs, reduce, memory, true);
}

int te_map_footprint_polygon(te_map* m, const te_footprint_params* p, int32_t npts, const double* pts_xy, double yaw, float* out_x,
                             float* out_rot, int memory) {
  TE_MAP_ENTER(m);
  static const double identity = 0.0;  // traversability_x: yaw 0, the identity
  const PolygonOutputs outs[2] = {{out_x, 1, &identity}, {out_rot, 1, &yaw}};
  return map_footprint_polygon(m, p, npts, pts_xy, 2, outs, nullptr, memory);
}

int te_map_footprint_polygon_yaws(te_map* m, const te_footprint_params* p, int32_t npts, const double* pts_xy, int32_t nyaws,
                                  const double* yaws, float* out, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = check_yaws(nyaws, yaws)) return rc;
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  const PolygonOutputs outs[1] = {{out, nyaws, yaws}};
  return map_footprint_polygon(m, p, npts, pts_xy, 1, outs, nullptr, memory);
}

int te_map_footprint_polygon_yaws_reduce(te_map* m, const te_footprint_params* p, int32_t npts, const double* pts_xy, int32_t nyaws,
                                         const double* yaws, float* worst, float* best, int32_t* best_yaw, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = check_yaws(nyaws, yaws)) return rc;
  const te::PolygonReduce red{worst, best, best_yaw};
  if (int rc = check_reduce_outputs(red)) return rc;
  const PolygonOutputs outs[1] = {{nullptr, nyaws, yaws}};
  return map_footprint_polygon(m, p, npts, pts_xy, 1, outs, &red, memory);
}

int te_map_check_footprint_request(te_map* m, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                   const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                   const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative,
                                   const uint8_t* cup, uint8_t* is_safe, double* traversability, double* area, int32_t max_vertices,
                                   int32_t* ucount, double* uxy) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  if (!(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint offset must be >= 0");
  if (npaths < 0 || nposes < 0 || nvertices < 0 || !path_begin || !poses || !radius || !footprint_begin ||
      (nvertices > 0 && !footprint_xyz) || !is_safe || !traversability || !area)
    return fail(TE_ERR_BAD_ARG, "null argument or negative count");
  if (max_footprint_vertices < 0 || max_footprint_vertices > te::kPolyMaxVerts)
    return fail(TE_ERR_BAD_ARG, "max_footprint_vertices must be 0..%d, got %d", te::kPolyMaxVerts, max_footprint_vertices);
  if (int rc = check_polygon_outputs(max_vertices, ucount, uxy)) return rc;
  m->last = te::MapRequestStats{};
  if (npaths == 0) return TE_OK;
  const te_geometry* g = &m->geo;
  int mp = 2;
  if (int rc = check_request_host(g, p, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin, footprint_xyz,
                                  max_footprint_vertices, conservative, &mp))
    return rc;
  if (int rc = ensure_geometry(c, g)) return rc;
  if (int rc = map_memo(m, p)) return rc;
  const te::SlabView v = make_view(c, g, te_slab{0, g->cols, 0, 0});
  const float* rough = p->verify_roughness ? (const float*)m->rough.p : nullptr;
  const float* rslope = m->have_rslope ? (const float*)m->rslope.p : nullptr;
  int nl = 0;
  if (nvertices > 0) {  // the polygonal paths (TraversabilityMap.cpp:464-584) read the memo and leave the cache alone
    te::PathChecks r{};
    r.trav = (const float*)m->trav.p; r.slope = (const float*)m->slope.p; r.step = (const float*)m->step.p; r.rough = rough;
    r.elev = (const float*)m->elev.p; r.robot_slope = rslope; r.nmaps = 1;
    r.npaths = npaths; r.nposes = nposes; r.path_begin = path_begin; r.poses = poses; r.pose_stride = 7;
    r.footprint_begin = footprint_begin; r.footprint_xyz = footprint_xyz; r.nvertices = nvertices;
    r.max_footprint_vertices = max_footprint_vertices; r.conservative = conservative; r.cup = cup; r.max_points = mp;
    r.is_safe = is_safe; r.trav_out = traversability; r.area_out = area; r.max_vertices = max_vertices; r.ucount = ucount; r.uxy = uxy;
    Staging st(c, true, g);
    stage_paths(st, r);
    if (st.rc) return st.rc;
    int rc = te::launch_path_checks(m->fp, v, g, p, r, false, false, c->stream, &nl);
    if (rc != 0) return fail(rc, "map request (polygonal paths) failed: %s", m->fp.why.c_str());
    if (int r2 = launch_check(c, "map request (polygonal paths)", nl)) return r2;
    if (int r2 = st.finish()) return r2;
  }
  // the circular paths (TraversabilityMap.cpp:345-462) in request order on the cache; they write their own outputs on the host
  int rc = te::launch_map_circles(m->fp, v, g, p, (const float*)m->trav.p, (const float*)m->slope.p, (const float*)m->step.p, rough,
                                  (const float*)m->elev.p, rslope, (float*)m->cache.p, c->hX.data(), c->hY.data(), npaths, path_begin,
                                  poses, radius, footprint_begin, cup, is_safe, traversability, area, max_vertices, ucount, uxy, c->stream,
                                  &nl, &m->last);
  if (rc != 0) return fail(rc, "map request (circular paths) failed: %s", m->fp.why.c_str());
  if (int r2 = launch_check(c, "map request (circular paths)", nl)) return r2;
  if (ucount)  // the row bound of a polygonal path's polygon table (kUntravRows) is only known once the hulls are
    for (int32_t q = 0; q < npaths; ++q)
      if (ucount[q] < 0)
        return fail(TE_ERR_UNSUPPORTED, "the untraversable polygon of path %d spans more than %d map rows", q, te::kUntravRows);
  return TE_OK;
}

int te_map_get_footprint(te_map* m, float* dst, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!dst) return fail(TE_ERR_BAD_ARG, "output layer is null");
  if (memory != TE_MEM_HOST && (m->geo_in.start_row != 0 || m->geo_in.start_col != 0))
    return fail(TE_ERR_UNSUPPORTED, "the map's layers came with a circular-buffer start index: read its cache into host memory");
  if (int rc = map_get_layer(m, dst, m->cache.p, memory)) return rc;
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

int te_map_clear_footprint(te_map* m) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  TE_CUDA(cudaMemsetAsync(m->cache.p, 0xff, sizeof(float) * map_cells(m), c->stream));
  return TE_OK;
}

int te_map_request_stats(te_map* m, int64_t out[3]) {
  TE_MAP_ENTER(m);
  if (!out) return fail(TE_ERR_BAD_ARG, "null argument");
  out[0] = m->last.candidates;
  out[1] = m->last.keys;
  out[2] = m->last.stored;
  return TE_OK;
}

// ---- The read side: GetGridMap submaps, the published layers and mapHasValidTraversabilityAt -----------------------------------
namespace {

// te_submap_geometry's records of `n` windows on the map `g` (its start index changes nothing: te::grid_submap), with offsets for
// `nlayers` layers per window; *total receives the floats they take.  Every window is checked before any record is written.
int submap_windows(const te_geometry* g, int32_t n, const double* pos, const double* len, int nlayers, te_submap_info* info,
                   int64_t* total) {
  if (n < 0) return fail(TE_ERR_BAD_ARG, "negative window count");
  if (n > 0 && (!pos || !len || !info)) return fail(TE_ERR_BAD_ARG, "null argument");
  for (int32_t k = 0; k < n; ++k) {  // the reference does not validate these; a negative length would make negative-sized blocks
    if (!std::isfinite(pos[2 * k]) || !std::isfinite(pos[2 * k + 1])) return fail(TE_ERR_BAD_ARG, "window %d: position is not finite", k);
    if (!(len[2 * k] >= 0.0 && len[2 * k + 1] >= 0.0) || !std::isfinite(len[2 * k]) || !std::isfinite(len[2 * k + 1]))
      return fail(TE_ERR_BAD_ARG, "window %d: length must be finite and >= 0", k);
  }
  const te::GridGeo A{g->rows, g->cols, g->resolution, g->length_x, g->length_y, g->position_x, g->position_y};
  int64_t off = 0;
  for (int32_t k = 0; k < n; ++k) {
    te_submap_info r{};
    te::SubmapGeo s{};
    if (te::grid_submap(A, pos[2 * k], pos[2 * k + 1], len[2 * k], len[2 * k + 1], s)) {
      r.success = 1;
      r.rows = s.rows; r.cols = s.cols; r.top_row = s.top_row; r.top_col = s.top_col;
      r.requested_row = s.req_row; r.requested_col = s.req_col;
      r.length_x = s.lenx; r.length_y = s.leny; r.position_x = s.posx; r.position_y = s.posy;
    }
    r.offset = off;
    off += (int64_t)nlayers * r.rows * r.cols;
    info[k] = r;
  }
  if (total) *total = off;
  return TE_OK;
}

}  // namespace

int te_submap_geometry(const te_geometry* g, int32_t n, const double* position_xy, const double* length_xy, te_submap_info* info) {
  if (int rc = check_geometry(g, true)) return rc;
  return submap_windows(g, n, position_xy, length_xy, 1, info, nullptr);
}

int te_map_get_layers(te_map* m, uint32_t layer_mask, float* out, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  const float* src[7];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, src, &nl)) return rc;
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  for (int k = 0; k < nl; ++k)
    if (int rc = map_get_layer(m, out + (size_t)k * map_cells(m), src[k], memory)) return rc;
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

int te_map_get_submaps(te_map* m, int32_t nwin, const double* position_xy, const double* length_xy, uint32_t layer_mask,
                       te_submap_info* info, float* out, int64_t out_capacity, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  const float* src[7];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, src, &nl)) return rc;
  int64_t total = 0;
  if (int rc = submap_windows(&m->geo, nwin, position_xy, length_xy, nl, info, &total)) return rc;
  if (out_capacity < total)
    return fail(TE_ERR_BAD_ARG, "the submaps take %lld floats but out holds %lld: call again with more room", (long long)total,
                (long long)out_capacity);
  if (total == 0) return TE_OK;
  if (!out) return fail(TE_ERR_BAD_ARG, "output is null");
  // the table k_map_gather_submaps reads: the source layers in its first two records, then the windows that have cells
  static_assert(sizeof(const float*) * 7 <= 2 * sizeof(te::SubmapWindow), "layer table");
  std::vector<te::SubmapWindow> table(2);
  std::memcpy((void*)table.data(), src, sizeof(const float*) * nl);
  long long columns = 0;
  for (int32_t k = 0; k < nwin; ++k) {
    const te_submap_info& r = info[k];
    if (!r.success) continue;
    table.push_back(te::SubmapWindow{columns, (long long)r.top_col * m->geo.rows + r.top_row, r.offset, r.rows, r.cols});
    columns += (long long)nl * r.cols;
  }
  const size_t bytes = sizeof(te::SubmapWindow) * table.size();
  if (m->gather.p && m->gather.cap < bytes) TE_CUDA(cudaStreamSynchronize(c->stream));  // an earlier gather may still read it
  TE_CUDA(m->gather.reserve(bytes));
  TE_CUDA(cudaMemcpyAsync(m->gather.p, table.data(), bytes, cudaMemcpyHostToDevice, c->stream));
  Staging st(c, memory == TE_MEM_HOST, &m->geo);  // host memory: gather into staging, then one copy of the packed floats
  float* dout = st.out(out, (size_t)total);
  if (st.rc) return st.rc;
  const te::SubmapGather a{(const float* const*)m->gather.p, (const te::SubmapWindow*)m->gather.p + 2, (int)table.size() - 2,
                           m->geo.rows, columns, dout};
  te::launch_gather_submaps(a, c->sms, c->stream);
  if (int rc = launch_check(c, "k_map_gather_submaps")) return rc;
  return st.finish();
}

int te_map_valid_at(te_map* m, int32_t n, const double* xy, uint8_t* valid, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (n < 0) return fail(TE_ERR_BAD_ARG, "negative position count");
  if (n == 0) return TE_OK;
  if (!xy || !valid) return fail(TE_ERR_BAD_ARG, "null argument");
  Staging st(c, memory == TE_MEM_HOST, &m->geo);
  const double* dxy = st.in(xy, 2 * (size_t)n);
  uint8_t* dvalid = st.out(valid, (size_t)n);
  if (st.rc) return st.rc;
  const te_geometry& g = m->geo;
  te::launch_valid_at(te::GridGeo{g.rows, g.cols, g.resolution, g.length_x, g.length_y, g.position_x, g.position_y},
                      (const float*)m->trav.p, n, dxy, dvalid, c->stream);
  if (int rc = launch_check(c, "k_map_valid_at")) return rc;
  return st.finish();
}

// A te IPC handle is the CUDA handle of the ALLOCATION that contains the pointer (cudaIpcGetMemHandle always describes the whole
// allocation; sub-allocating pools such as torch's caching allocator hand out interior pointers) plus the offset into it.
struct TeIpcHandle {
  cudaIpcMemHandle_t mem;
  uint64_t offset;
  uint64_t reserved;
};
static_assert(sizeof(TeIpcHandle) == TE_IPC_HANDLE_BYTES, "te IPC handle layout");

namespace {
std::mutex g_ipc_mu;
std::map<void*, void*> g_ipc_opened;  // pointer handed out by te_ipc_open -> base of the mapping to close
}  // namespace

int te_ipc_export(const void* device_ptr, void* handle) {
  if (!device_ptr || !handle) return fail(TE_ERR_BAD_ARG, "null argument");
  typedef CUresult (*PFN_range)(CUdeviceptr*, size_t*, CUdeviceptr);
  static PFN_range range = nullptr;
  if (!range) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return fail(TE_ERR_CUDA, "cuMemGetAddressRange entry point unavailable");
    range = reinterpret_cast<PFN_range>(p);
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, (CUdeviceptr)device_ptr) != CUDA_SUCCESS) return fail(TE_ERR_CUDA, "cuMemGetAddressRange failed (not a device allocation?)");
  TeIpcHandle h{};
  TE_CUDA(cudaIpcGetMemHandle(&h.mem, reinterpret_cast<void*>(base)));
  h.offset = (uint64_t)((CUdeviceptr)device_ptr - base);
  std::memcpy(handle, &h, sizeof(h));
  return TE_OK;
}

int te_ipc_open(const void* handle, void** out) {
  if (!handle || !out) return fail(TE_ERR_BAD_ARG, "null argument");
  TeIpcHandle h;
  std::memcpy(&h, handle, sizeof(h));
  void* base = nullptr;
  TE_CUDA(cudaIpcOpenMemHandle(&base, h.mem, cudaIpcMemLazyEnablePeerAccess));
  *out = (char*)base + h.offset;
  std::lock_guard<std::mutex> lock(g_ipc_mu);
  g_ipc_opened[*out] = base;
  return TE_OK;
}

int te_ipc_close(void* p) {
  if (!p) return TE_OK;
  void* base = p;
  {
    std::lock_guard<std::mutex> lock(g_ipc_mu);
    auto it = g_ipc_opened.find(p);
    if (it != g_ipc_opened.end()) { base = it->second; g_ipc_opened.erase(it); }
  }
  TE_CUDA(cudaIpcCloseMemHandle(base));
  return TE_OK;
}

int te_event_create_ipc(te_ctx* c, void** event_out, void* handle) {
  TE_ENTER(c);
  if (!event_out || !handle) return fail(TE_ERR_BAD_ARG, "null argument");
  cudaEvent_t ev;
  TE_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming | cudaEventInterprocess));
  cudaIpcEventHandle_t h;
  cudaError_t e = cudaIpcGetEventHandle(&h, ev);
  if (e != cudaSuccess) {
    cudaEventDestroy(ev);
    return fail(TE_ERR_CUDA, "cudaIpcGetEventHandle failed: %s", cudaGetErrorString(e));
  }
  static_assert(sizeof(h) == 64, "cudaIpcEventHandle_t is 64 bytes");
  std::memcpy(handle, &h, sizeof(h));
  *event_out = (void*)ev;
  return TE_OK;
}

int te_event_open_ipc(const void* handle, void** event_out) {
  if (!handle || !event_out) return fail(TE_ERR_BAD_ARG, "null argument");
  cudaIpcEventHandle_t h;
  std::memcpy(&h, handle, sizeof(h));
  cudaEvent_t ev;
  TE_CUDA(cudaIpcOpenEventHandle(&ev, h));
  *event_out = (void*)ev;
  return TE_OK;
}

int te_event_record(te_ctx* c, void* event) {
  TE_ENTER(c);
  if (!event) return fail(TE_ERR_BAD_ARG, "event is null");
  TE_CUDA(cudaEventRecord((cudaEvent_t)event, c->stream));
  return TE_OK;
}

int te_event_destroy(void* event) {
  if (!event) return TE_OK;
  TE_CUDA(cudaEventDestroy((cudaEvent_t)event));
  return TE_OK;
}

int te_halo_pull(te_ctx* c, const te_geometry* g, const te_slab* slab, float* layer, const te_halo_peer* left,
                 const te_halo_peer* right) {
  TE_ENTER(c);
  if (int rc = check_geometry(g)) return rc;
  if (!slab || !layer) return fail(TE_ERR_BAD_ARG, "null argument");
  te_slab s;
  if (int rc = resolve_slab(g, slab, 0, &s)) return rc;
  const size_t col_bytes = sizeof(float) * (size_t)g->rows;
  // Global columns [first, first + count) into this rank's buffer, from the OWNED columns of `p`.
  auto pull = [&](const te_halo_peer* p, int first, int count, const char* side) -> int {
    if (count <= 0) return TE_OK;
    if (!p || !p->layer) return fail(TE_ERR_BAD_ARG, "slab has a %s halo of %d columns but no %s neighbour was given", side, count, side);
    const te_slab& q = p->slab;
    if (q.col_begin < 0 || q.col_count <= 0 || q.halo_left < 0 || q.halo_right < 0 || q.col_begin + q.col_count > g->cols)
      return fail(TE_ERR_BAD_ARG, "%s neighbour's slab is malformed", side);
    if (first < q.col_begin || first + count > q.col_begin + q.col_count)
      return fail(TE_ERR_BAD_ARG, "%s halo columns [%d,%d) are not owned by the %s neighbour [%d,%d): the exchange is one hop", side,
                  first, first + count, side, q.col_begin, q.col_begin + q.col_count);
    if (p->ready_event) TE_CUDA(cudaStreamWaitEvent(c->stream, (cudaEvent_t)p->ready_event, 0));
    const char* src = (const char*)p->layer + col_bytes * (size_t)(first - (q.col_begin - q.halo_left));
    char* dst = (char*)layer + col_bytes * (size_t)(first - (s.col_begin - s.halo_left));
    TE_CUDA(cudaMemcpyAsync(dst, src, col_bytes * (size_t)count, cudaMemcpyDefault, c->stream));
    return TE_OK;
  };
  if (int rc = pull(left, s.col_begin - s.halo_left, s.halo_left, "left")) return rc;
  if (int rc = pull(right, s.col_begin + s.col_count, s.halo_right, "right")) return rc;
  return TE_OK;
}

}  // extern "C"
