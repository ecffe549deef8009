// te_map.cu — the te_map entries of the C ABI (include/te_b200.h): a batch of maps whose layers, traversability_footprint cache
// and isTraversableForFilters memo stay on the device between calls, and the stateless geometry entries its callers use.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <algorithm>
#include <limits>
#include <map>
#include <vector>

#include "te_capi_host.h"

using namespace te::host;
using te::DevBuf;
using te::cell_coord;

namespace {

constexpr int kLayerBits = 24;  // te_layer bits 0 .. 23 (1 << 7, 1 << 18 .. 1 << 20 unassigned)
const char* const kLayerNames[kLayerBits] = {"traversability", "traversability_slope", "traversability_step", "traversability_roughness",
                                             "elevation", "robot_slope", "traversability_footprint", nullptr, "upper_bound", "lower_bound",
                                             "variance", "horizontal_variance_x", "horizontal_variance_y", "horizontal_variance_xy",
                                             "time", "uncertainty_range", "traversability_x", "traversability_rot", nullptr, nullptr,
                                             nullptr, "slope_footprint", "step_footprint", "roughness_footprint"};
constexpr int kFootprintMemoBit = 21;  // TE_LAYER_SLOPE_FOOTPRINT: field 0 of the recorded bytes (te_fp_device.cuh)
// The layers every map holds once it has any (te_map_chain, te_map_set_layers), the cache included.
constexpr uint32_t kLayersAlways = TE_LAYER_TRAVERSABILITY | TE_LAYER_SLOPE | TE_LAYER_STEP | TE_LAYER_ELEVATION | TE_LAYER_FOOTPRINT;

}  // namespace

// A te_map holds nmaps maps of one geometry in the layout of te_chain_batched: map m starts m * rows * cols cells into every layer,
// the cache and the memo.  The single-map entries are the nmaps = 1 case of the same bodies.
struct te_map {
  te_ctx* ctx = nullptr;
  bool have_layers = false;
  int nmaps = 1;
  te_geometry geo_in{};  // as the layers came (host memory: with their circular-buffer start index)
  te_geometry geo{};     // the same with the start index cleared: the device layers are in default order
  // The resident layers, indexed by te_layer bit: layer[b] holds bit b's layer of every map while `held` has bit b.  Bit 6,
  // traversability_footprint, is the cache; uncertainty_range (bit 15) is derived from the bounds and never held.  Bits 21 .. 23
  // (slope_footprint, step_footprint, roughness_footprint) are never held either: layer[b] receives them decoded from `plane`
  // when they are read.
  DevBuf layer[kLayerBits];
  uint32_t held = 0;
  DevBuf fresh;  // te_map_footprint(_maps): the sweep before its merge into the cache
  DevBuf gather;  // te_map_get_submaps: the source-layer table, then the windows (te::SubmapWindow)
  // The _maps entries: the selected maps' layers packed back to back (grown to the largest selection) and their slot table
  DevBuf sel[te::kMapSlotLayers], slots;
  DevBuf image;  // te_map_chain_image(_maps) in host memory: the staged image bytes, packed
  DevBuf cut;    // the window table of k_map_cut_windows (te_map_chain_submap / _windows, and the moves of `start` below)
  DevBuf wrap;   // maps in their buffer order on the device: host inputs before they are unwrapped, host outputs once re-wrapped
  te::FootprintState fp;  // the map's own scratch; fp.memo is the resident memo
  // memo_valid: fp.memo holds every map's bytes, each map's evaluated under the parameters of its key (map_memo)
  bool memo_valid = false;
  struct MemoKey {
    double gap, crit;
    int rough;
  };
  std::vector<MemoKey> memo_key;
  // The recorded slope_footprint / step_footprint / roughness_footprint (te_fp_device.cuh: one byte per cell of every map), valid
  // while plane_valid, map k's recorded under the parameters plane_key[k] (map_plane); not valid: NaN everywhere.
  DevBuf plane;
  bool plane_valid = false;
  std::vector<MemoKey> plane_key;
  // plane_covers[k]: every cached cell of map k is recorded (its value came from a walk centred on it, which recorded it).  Only a
  // reset of the map's bytes on a memo-key change that keeps its cache breaks it, until the cache is emptied (map_footprint then
  // walks the map's empty centres).
  std::vector<char> plane_covers;
  // The per-map parameter table of the last request whose maps have parameters of their own (map_param_table), with what it holds
  std::vector<te::FpMapParams> par_key;
  DevBuf par_tab;
  te::MapRequestStats last{};
  bool last_device = false;  // the last request ran in device memory: its counters are on the device (fp.req_counters)
  // Where each map sits: pos[2m], pos[2m + 1] (te_map_positions).  geo's position for every map unless an _at entry put maps
  // elsewhere.  spread: the maps do not all sit at one position, so the kernels read per-map tables (map_tables).
  std::vector<double> pos;
  bool spread = false;
  // Each map's circular-buffer start index (start[2m], start[2m + 1]: te_map_start_indices), as the _wrapped entries gave it; (0, 0)
  // for maps the other entries loaded.  The device layers stay in default order; host inputs of a map with a start index are
  // unwrapped and its host outputs re-wrapped by k_map_cut_windows (a single map whose start index came in g, geo_in, keeps the
  // staging copies of upload_cols / download_cols instead, and all zeros here).
  std::vector<int32_t> start;
  // Per-map device tables (map_tables), cached with what they were built from: tab_all for every map in index order, tab_launch
  // for a chain launch (with the fused mask tables) or a selection.
  struct PosTab {
    std::vector<double> key;
    double coord_max = 0.0;
    size_t mask_off = 0;
    DevBuf buf;
  } tab_all, tab_launch;
  // te_map_get_point_cloud: the tile counts, their prefix sums and the scan's scratch; and the per-map tables (te::CloudMap) of a
  // whole batch and of a selection, each uploaded only when it changes, so that a captured whole-batch call keeps reading its own.
  DevBuf cloud;
  struct CloudTab {
    std::vector<te::CloudMap> key;
    DevBuf buf;
  } cloud_all, cloud_sel;
};

namespace {

size_t map_cells(const te_map* m) { return (size_t)m->geo.rows * m->geo.cols; }
// The resident layer of te_layer bit `bit` (a one-bit mask).
float* lay(const te_map* m, uint32_t bit) { return (float*)m->layer[__builtin_ctz(bit)].p; }
size_t batch_cells(const te_map* m) { return map_cells(m) * m->nmaps; }  // every map of the te_map

// The maps a _maps entry updates: n distinct indices of the batch, a host array.  The whole-batch entries pass none.
struct MapSel {
  int32_t n;
  const int32_t* idx;
};

// Validates n (x, y) map positions of an _at entry (null: none given).  Writes nothing.
int check_positions(const double* xy, int n) {
  if (!xy) return TE_OK;
  for (int k = 0; k < 2 * n; ++k)
    if (!std::isfinite(xy[k])) return fail(TE_ERR_BAD_ARG, "position_xy[%d] (map %d's %c) is not finite", k, k / 2, k % 2 ? 'y' : 'x');
  return TE_OK;
}

// The positions of n maps of a launch: position_xy as given, or (x, y) for every map when it is null.
std::vector<double> launch_positions(const double* xy, int n, double x, double y) {
  std::vector<double> v(2 * (size_t)n);
  for (int k = 0; k < n; ++k) {
    v[2 * k] = xy ? xy[2 * k] : x;
    v[2 * k + 1] = xy ? xy[2 * k + 1] : y;
  }
  return v;
}

// Whether every one of the n positions xy is (x, y), bit for bit.
bool all_at(const double* xy, int n, double x, double y) {
  for (int k = 0; k < n; ++k)
    if (std::memcmp(xy + 2 * k, &x, sizeof(double)) != 0 || std::memcmp(xy + 2 * k + 1, &y, sizeof(double)) != 0) return false;
  return true;
}

// The geometry the kernels see when every map of the te_map sits at one position: the te_map's, at that position.  False when the
// maps are spread over several positions (the per-map tables then apply).
bool map_geometry(const te_map* m, te_geometry* g) {
  if (m->spread) return false;
  *g = m->geo;
  if (!m->pos.empty()) { g->position_x = m->pos[0]; g->position_y = m->pos[1]; }
  return true;
}
// The same with the start index of the layers as they came (geo_in).
te_geometry map_geometry_in(const te_map* m) {
  te_geometry g = m->geo_in;
  if (!m->pos.empty()) { g.position_x = m->pos[0]; g.position_y = m->pos[1]; }
  return g;
}

// Device tables of n maps of geometry g at the positions xy (2n doubles, launch order): the cell-centre coordinates (X: n * rows,
// Y: n * cols, as getPositionFromIndex gives them at each map's position) and the positions, plus for a chain launch (p set) the
// fused mask tables of every map.  Cached in t while the geometry, the positions and the step radii stay the same; a rebuild is
// ordered after the kernels that may still read the old tables.
int map_tables(te_ctx* c, te_map::PosTab& t, const te_geometry& g, const double* xy, int n, const te_chain_params* p, PosTables* out) {
  const double none = std::numeric_limits<double>::quiet_NaN();
  std::vector<double> key = {(double)g.rows, (double)g.cols, g.resolution, g.length_x, g.length_y,
                             p ? p->step_first_radius : none, p ? p->step_second_radius : none};
  key.insert(key.end(), xy, xy + 2 * (size_t)n);
  const size_t R = g.rows, C = g.cols;
  const size_t dbytes = sizeof(double) * ((R + C) * n + 2 * (size_t)n);
  if (!t.buf.p || t.key.size() != key.size() || std::memcmp(t.key.data(), key.data(), sizeof(double) * key.size()) != 0) {
    std::vector<double> h((R + C) * n + 2 * (size_t)n);
    double cmax = 0.0;
    for (int k = 0; k < n; ++k) {
      const double px = xy[2 * k], py = xy[2 * k + 1];
      for (size_t i = 0; i < R; ++i) h[k * R + i] = cell_coord(px, g.length_x, g.resolution, (int)i);
      for (size_t j = 0; j < C; ++j) h[R * n + k * C + j] = cell_coord(py, g.length_y, g.resolution, (int)j);
      h[(R + C) * n + 2 * k] = px;
      h[(R + C) * n + 2 * k + 1] = py;
      cmax = std::max(cmax, std::max(std::fabs(px) + 0.5 * g.length_x, std::fabs(py) + 0.5 * g.length_y));
    }
    std::vector<unsigned char> mk;
    if (p) {
      mk.resize((R + C) * n);
      for (int k = 0; k < n; ++k) {
        te::fused_mask_bits(p, h.data() + k * R, (int)R, mk.data() + k * R);
        te::fused_mask_bits(p, h.data() + R * n + k * C, (int)C, mk.data() + R * n + k * C);
      }
    }
    const size_t bytes = dbytes + mk.size();
    if (t.buf.p && t.buf.cap < bytes) TE_CUDA(cudaStreamSynchronize(c->stream));  // earlier kernels may still read the tables
    TE_CUDA(t.buf.reserve(bytes));
    // pageable sources: consumed before cudaMemcpyAsync returns, ordered after the kernels queued before on the stream
    TE_CUDA(cudaMemcpyAsync(t.buf.p, h.data(), dbytes, cudaMemcpyHostToDevice, c->stream));
    if (!mk.empty()) TE_CUDA(cudaMemcpyAsync((char*)t.buf.p + dbytes, mk.data(), mk.size(), cudaMemcpyHostToDevice, c->stream));
    t.key = std::move(key);
    t.coord_max = cmax;
    t.mask_off = dbytes;
  }
  const double* base = (const double*)t.buf.p;
  out->X = base;
  out->Y = base + R * n;
  out->pos = base + (R + C) * n;
  out->coord_max = t.coord_max;
  const unsigned char* mk = p ? (const unsigned char*)t.buf.p + t.mask_off : nullptr;
  out->masks = te::MapMasks{mk, mk ? mk + R * n : nullptr, (unsigned)R, (unsigned)C};
  return TE_OK;
}

// The tables of the maps s.idx[0..s.n) (idx null: every map, in index order) at their positions.
int map_tables_of(te_map* m, const MapSel& s, PosTables* out) {
  if (!s.idx) return map_tables(m->ctx, m->tab_all, m->geo, m->pos.data(), m->nmaps, nullptr, out);
  std::vector<double> xy(2 * (size_t)s.n);
  for (int k = 0; k < s.n; ++k) { xy[2 * k] = m->pos[2 * s.idx[k]]; xy[2 * k + 1] = m->pos[2 * s.idx[k] + 1]; }
  return map_tables(m->ctx, m->tab_launch, m->geo, xy.data(), s.n, nullptr, out);
}

// Records where the maps of an update now sit: every map (idx null) or the maps idx[0..n) at the launch positions xy.
void map_place(te_map* m, const int32_t* idx, int n, const std::vector<double>& xy) {
  if (!idx) {
    m->pos = xy;
  } else {
    for (int k = 0; k < n; ++k) { m->pos[2 * idx[k]] = xy[2 * k]; m->pos[2 * idx[k] + 1] = xy[2 * k + 1]; }
  }
  m->spread = !all_at(m->pos.data(), m->nmaps, m->pos[0], m->pos[1]);
}

int map_ready(const te_map* m) {
  if (!m->have_layers) return fail(TE_ERR_BAD_ARG, "the map has no layers yet: call te_map_chain or te_map_set_layers first");
  return TE_OK;
}

// The entries that address one map of a te_map by position take a map index on a batch (the `_batched` entry).
int map_single(const te_map* m, const char* batched) {
  if (m->nmaps > 1) return fail(TE_ERR_BAD_ARG, "the te_map holds %d maps: call %s with a map index", m->nmaps, batched);
  return TE_OK;
}

// A host array of map indices of a batched entry: every entry in 0 .. nmaps-1.
int check_map_indices(const te_map* m, const int32_t* idx, int32_t n, const char* what) {
  if (n > 0 && !idx) return fail(TE_ERR_BAD_ARG, "%s is null", what);
  for (int32_t k = 0; k < n; ++k)
    if (idx[k] < 0 || idx[k] >= m->nmaps) return fail(TE_ERR_BAD_ARG, "%s[%d] = %d is outside 0..%d", what, k, idx[k], m->nmaps - 1);
  return TE_OK;
}

// New layers for nmaps maps of geometry g: the geometry, an empty cache and a memo to be rebuilt.  Checks the batch limits of the
// stateless batched entries (a start index on a batch is TE_ERR_UNSUPPORTED: unwrap_geometry).
int map_reset(te_map* m, const te_geometry* g_in, const te_geometry* g, int nmaps) {
  te_ctx* c = m->ctx;
  if (int rc = check_footprint_batch(g, nmaps)) return rc;
  const size_t bytes = sizeof(float) * (size_t)g->rows * g->cols * nmaps;
  for (int b = 0; b < kLayerBits; ++b)
    if ((kLayersAlways >> b) & 1u) TE_CUDA(m->layer[b].reserve(bytes));
  TE_CUDA(cudaMemsetAsync(lay(m, TE_LAYER_FOOTPRINT), 0xff, bytes, c->stream));  // all-ones bits: NaN, the empty cache of computeTraversability (:225-228)
  m->geo_in = *g_in;
  m->geo = *g;
  m->nmaps = nmaps;
  m->start.assign(2 * (size_t)nmaps, 0);  // a _wrapped entry sets the maps' start indices once their layers are in
  m->memo_valid = false;
  m->plane_valid = false;
  m->have_layers = false;
  m->held = kLayersAlways;  // a new map replaces the old one wholesale, its elevation map's layers included
  return TE_OK;
}

// The resident isTraversableForFilters memo for these parameters (p[0] for every map, or with `each` p[k] for map k): a map's bytes
// are kept while the layers and its max_gap_width, critical_step_height and verify_roughness (all that checkForStep /
// checkForSlope / checkForRoughness read) stay the same, and cleared otherwise, one memset per run of neighbouring maps to clear.
// One byte per cell of every map.
int map_memo(te_map* m, const te_footprint_params* p, bool each) {
  auto key = [&](int k) {
    const te_footprint_params& q = p[each ? k : 0];
    return te_map::MemoKey{q.max_gap_width, q.critical_step_height, q.verify_roughness != 0};
  };
  auto same = [](const te_map::MemoKey& a, const te_map::MemoKey& b) { return a.gap == b.gap && a.crit == b.crit && a.rough == b.rough; };
  const size_t cells = map_cells(m);
  if (!m->memo_valid) {
    TE_CUDA(m->fp.memo.reserve(batch_cells(m)));
    m->memo_key.assign(m->nmaps, key(0));
  }
  for (int k = 0; k < m->nmaps;) {
    if (m->memo_valid && same(m->memo_key[k], key(k))) { ++k; continue; }
    int e = k;
    for (; e < m->nmaps && !(m->memo_valid && same(m->memo_key[e], key(e))); ++e) m->memo_key[e] = key(e);
    TE_CUDA(cudaMemsetAsync((unsigned char*)m->fp.memo.p + k * cells, 0, (e - k) * cells, m->ctx->stream));
    k = e;
  }
  m->memo_valid = true;
  return TE_OK;
}

// The recorded layers, reserved for the whole batch and all NaN (under no parameters) when first needed.
int map_plane_ready(te_map* m) {
  if (m->plane_valid) return TE_OK;
  TE_CUDA(m->plane.reserve(batch_cells(m)));
  TE_CUDA(cudaMemsetAsync(m->plane.p, 0, batch_cells(m), m->ctx->stream));
  const double none = std::numeric_limits<double>::quiet_NaN();
  m->plane_key.assign(m->nmaps, te_map::MemoKey{none, none, -1});
  m->plane_covers.assign(m->nmaps, 1);  // the caches are empty: no request or sweep since the layers came
  m->plane_valid = true;
  return TE_OK;
}

// The recorded layers for a request or a sweep on the maps `sel` (null: every map) under these parameters (p[0] for every map, or
// with `each` p[k] for map k): a map keeps its bytes while its memo key (map_memo) stays, and is reset to NaN otherwise.
int map_plane(te_map* m, const te_footprint_params* p, bool each, const MapSel* sel) {
  auto key = [&](int k) {
    const te_footprint_params& q = p[each ? k : 0];
    return te_map::MemoKey{q.max_gap_width, q.critical_step_height, q.verify_roughness != 0};
  };
  const size_t cells = map_cells(m);
  if (int rc = map_plane_ready(m)) return rc;
  const int n = sel ? sel->n : m->nmaps;
  for (int j = 0; j < n; ++j) {
    const int k = sel ? sel->idx[j] : j;
    const te_map::MemoKey a = m->plane_key[k], b = key(k);
    if (a.gap == b.gap && a.crit == b.crit && a.rough == b.rough) continue;
    if (a.rough >= 0) m->plane_covers[k] = 0;  // recorded under other parameters: the cache, which stays, is no longer covered
    m->plane_key[k] = b;
    TE_CUDA(cudaMemsetAsync((unsigned char*)m->plane.p + k * cells, 0, cells, m->ctx->stream));
  }
  return TE_OK;
}

// The per-map parameter table of a request whose maps have parameters of their own (params: one per map): *out is its device copy,
// uploaded only when its bytes change (ordered after the kernels that may still read the old table; a table that grows first
// waits for them), or null when every map's entry is the same, the request then being one of params[0].  The radius is not in
// the table: a request takes it per path.
int map_param_table(te_map* m, const te_footprint_params* params, const te::FpMapParams** out) {
  std::vector<te::FpMapParams> h(m->nmaps);
  for (int k = 0; k < m->nmaps; ++k) {
    const te_footprint_params& q = params[k];
    h[k] = te::FpMapParams{q.offset, q.traversability_default, q.max_gap_width, q.critical_step_height, q.radius_is_integer_norm,
                           q.verify_roughness != 0 ? 1 : 0};
  }
  *out = nullptr;
  bool uniform = true;
  for (int k = 1; k < m->nmaps && uniform; ++k) uniform = std::memcmp(&h[k], &h[0], sizeof(h[0])) == 0;
  if (uniform) return TE_OK;
  const size_t bytes = sizeof(te::FpMapParams) * h.size();
  if (m->par_key.size() != h.size() || std::memcmp(m->par_key.data(), h.data(), bytes) != 0) {
    if (m->par_tab.p && m->par_tab.cap < bytes) TE_CUDA(cudaStreamSynchronize(m->ctx->stream));
    TE_CUDA(m->par_tab.reserve(bytes));
    // pageable source: consumed before cudaMemcpyAsync returns, ordered after the kernels queued before on the stream
    TE_CUDA(cudaMemcpyAsync(m->par_tab.p, h.data(), bytes, cudaMemcpyHostToDevice, m->ctx->stream));
    m->par_key = std::move(h);
  }
  *out = (const te::FpMapParams*)m->par_tab.p;
  return TE_OK;
}

int map_footprint_params(const te_map* m, const te_footprint_params* p) {
  if (!p) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (p->verify_roughness && !(m->held & TE_LAYER_ROUGHNESS))
    return fail(TE_ERR_MISSING_LAYER, "layer traversability_roughness is missing (verify_roughness is set)");
  return TE_OK;
}

// The resident buffer of te_layer bit b when the map holds that layer, else null (uncertainty_range is derived: null).
DevBuf* map_layer_buf(te_map* m, int b) { return ((m->held >> b) & 1u) ? &m->layer[b] : nullptr; }

// The map's layers of `mask`, in te_layer bit order (the order of every output that holds several).  with_range: the mask may
// ask for TE_LAYER_UNCERTAINTY_RANGE (te_map_get_layers), whose entry is then null: the caller derives it from the bounds.
int map_layers(te_map* m, uint32_t mask, bool with_range, const float* out[kLayerBits], int* n) {
  if (!with_range && (mask & TE_LAYER_UNCERTAINTY_RANGE))
    return fail(TE_ERR_BAD_ARG, "layer uncertainty_range is published with the map, not held by it: submaps have no such layer");
  const uint32_t known = TE_LAYER_ALL | TE_LAYER_CARRIED | TE_LAYER_TRAVERSABILITY_X | TE_LAYER_TRAVERSABILITY_ROT |
                         TE_LAYER_FOOTPRINT_MEMO | (with_range ? (uint32_t)TE_LAYER_UNCERTAINTY_RANGE : 0u);
  if (mask == 0 || (mask & ~known)) return fail(TE_ERR_BAD_ARG, "layer mask 0x%x: need a non-empty subset of 0x%x", mask, known);
  *n = 0;
  for (int b = 0; b < kLayerBits; ++b) {
    if (!((mask >> b) & 1u)) continue;
    if (b == 15) {
      if ((m->held & (TE_LAYER_UPPER_BOUND | TE_LAYER_LOWER_BOUND)) != (TE_LAYER_UPPER_BOUND | TE_LAYER_LOWER_BOUND))
        return fail(TE_ERR_MISSING_LAYER, "layer uncertainty_range needs upper_bound and lower_bound: the map does not hold both");
      out[(*n)++] = nullptr;
      continue;
    }
    if ((TE_LAYER_FOOTPRINT_MEMO >> b) & 1u) {  // decoded from the recorded bytes into layer[b]
      const size_t n_cells = batch_cells(m);
      TE_CUDA(m->layer[b].reserve(sizeof(float) * n_cells));
      if (int rc = map_plane_ready(m)) return rc;
      te::launch_plane_decode((const unsigned char*)m->plane.p, b - kFootprintMemoBit, (float*)m->layer[b].p, n_cells, m->ctx->sms,
                              m->ctx->stream);
      if (int rc = launch_check(m->ctx, "k_plane_decode")) return rc;
      out[(*n)++] = (const float*)m->layer[b].p;
      continue;
    }
    const DevBuf* src = map_layer_buf(m, b);
    if (!src) return fail(TE_ERR_MISSING_LAYER, "layer %s is missing: the map does not hold it", kLayerNames[b]);
    out[(*n)++] = (const float*)src->p;
  }
  return TE_OK;
}

int check_selection(const te_map* m, const MapSel& s);

// Validates a selection on a te_map that has layers and, when the entry takes one (with_geometry), g against the batch's
// geometry; any_position: except its position (the _at entries).  Writes nothing.
int map_select(const te_map* m, bool with_geometry, const te_geometry* g, const MapSel& s, bool any_position = false) {
  if (int rc = map_ready(m)) return rc;
  if (with_geometry) {
    if (int rc = check_geometry(g, true)) return rc;
    if (g->start_row != 0 || g->start_col != 0)
      return fail(TE_ERR_UNSUPPORTED, "circular-buffer start index (%d,%d) != (0,0) is unsupported for the _maps entries", g->start_row,
                  g->start_col);
  }
  if (m->geo_in.start_row != 0 || m->geo_in.start_col != 0)
    return fail(TE_ERR_UNSUPPORTED, "the te_map's layers came with a circular-buffer start index: use te_map_chain / te_map_set_layers");
  if (with_geometry) {
    te_geometry gc = *g;
    if (any_position) { gc.position_x = m->geo.position_x; gc.position_y = m->geo.position_y; }
    if (std::memcmp(&gc, &m->geo, sizeof(te_geometry)) != 0)
      return fail(TE_ERR_BAD_ARG, "the geometry differs from the te_map's: reload the whole batch to change it");
  }
  return check_selection(m, s);
}

// Validates the selection s on a te_map: 1..nmaps distinct indices of the batch.  Writes nothing.
int check_selection(const te_map* m, const MapSel& s) {
  if (s.n < 1 || s.n > m->nmaps) return fail(TE_ERR_BAD_ARG, "nsel = %d: need 1..%d", s.n, m->nmaps);
  if (!s.idx) return fail(TE_ERR_BAD_ARG, "map_index is null");
  std::vector<char> seen(m->nmaps, 0);
  for (int32_t k = 0; k < s.n; ++k) {
    const int32_t v = s.idx[k];
    if (v < 0 || v >= m->nmaps) return fail(TE_ERR_BAD_ARG, "map_index[%d] = %d is outside 0..%d", k, v, m->nmaps - 1);
    if (seen[v]++) return fail(TE_ERR_BAD_ARG, "map_index[%d] = %d is selected twice", k, v);
  }
  return TE_OK;
}

// Scratch for the packed layers m->sel[l] of the selection with bit l of `layers` set, and its slot table on the device.  A buffer
// that grows first waits for the kernels that may still read it.  The slot table is uploaded from a copy of map_index made here,
// so the caller may reuse its array as soon as the call returns, whatever kind of host memory it is: a copy from pageable memory
// has read its source when cudaMemcpyAsync returns, one from page-locked memory only when the stream reaches it.
int map_stage_selection(te_map* m, const MapSel& s, unsigned layers) {
  te_ctx* c = m->ctx;
  const size_t bytes = sizeof(float) * map_cells(m) * s.n, tbytes = sizeof(int32_t) * s.n;
  bool grow = m->slots.p && m->slots.cap < tbytes;
  for (int l = 0; l < te::kMapSlotLayers; ++l) grow = grow || (((layers >> l) & 1u) && m->sel[l].p && m->sel[l].cap < bytes);
  if (grow) TE_CUDA(cudaStreamSynchronize(c->stream));
  for (int l = 0; l < te::kMapSlotLayers; ++l)
    if ((layers >> l) & 1u) TE_CUDA(m->sel[l].reserve(bytes));
  TE_CUDA(m->slots.reserve(tbytes));
  const std::vector<int32_t> idx(s.idx, s.idx + s.n);  // pageable: consumed before cudaMemcpyAsync returns
  TE_CUDA(cudaMemcpyAsync(m->slots.p, idx.data(), tbytes, cudaMemcpyHostToDevice, c->stream));
  return TE_OK;
}

// The packed layers src (each null or nsel maps back to back; src[k] is the layer of the k-th bit of `bits`) into the selected maps'
// resident layers, in one launch that also empties those maps' caches, fills their carried and polygon layers with NaN (the new
// maps come without them, but every map of a batch holds the same layers) and, when the memo is live, clears their memo bytes.
// The te_map-wide memo key stays.  A batch that holds more than kMapSlotLayers such layers fills the rest in a second launch.
// keep: carried layer bits whose slots of the selected maps the caller has already written (te_map_chain_windows): those are not
// filled.
int map_put_selected(te_map* m, const MapSel& s, uint32_t bits, const float* const src[te::kMapSlotLayers], uint32_t keep = 0) {
  te_ctx* c = m->ctx;
  te::MapSlots a{};
  std::vector<float*> fill;
  for (int b = 0, k = 0; b < kLayerBits; ++b) {
    if ((bits >> b) & 1u) {
      a.src[k] = src[k];
      a.dst[k] = src[k] ? (float*)m->layer[b].p : nullptr;
      ++k;
    }
    if (((m->held & ~keep & (TE_LAYER_CARRIED | TE_LAYER_TRAVERSABILITY_X | TE_LAYER_TRAVERSABILITY_ROT)) >> b) & 1u)
      fill.push_back((float*)m->layer[b].p);
  }
  const int nf = std::min((int)fill.size(), te::kMapSlotLayers);
  std::copy(fill.begin(), fill.begin() + nf, a.fill);
  a.fill_bits = 0xffffffffu;
  a.cache = lay(m, TE_LAYER_FOOTPRINT);
  a.memo = m->memo_valid ? (unsigned char*)m->fp.memo.p : nullptr;  // reserved for the whole batch while valid (map_memo)
  for (int j = 0; m->plane_valid && j < s.n; ++j) {  // the recorded layers of the new maps: NaN, over an empty cache
    TE_CUDA(cudaMemsetAsync((unsigned char*)m->plane.p + s.idx[j] * map_cells(m), 0, map_cells(m), c->stream));
    m->plane_covers[s.idx[j]] = 1;
  }
  a.slot = (const int*)m->slots.p;
  a.nsel = s.n;
  a.cells = map_cells(m);
  te::launch_map_slots(a, true, c->sms, c->stream);
  if (nf == (int)fill.size()) return launch_check(c, "k_map_slots (put)");
  te::MapSlots f{};
  std::copy(fill.begin() + nf, fill.end(), f.fill);
  f.fill_bits = a.fill_bits;
  f.slot = a.slot;
  f.nsel = a.nsel;
  f.cells = a.cells;
  te::launch_map_slots(f, true, c->sms, c->stream);
  return launch_check(c, "k_map_slots (put)", 2);
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
      for (DevBuf* b : {&m->fresh, &m->gather, &m->slots, &m->image, &m->cut, &m->wrap, &m->par_tab, &m->plane}) b->release();
      for (DevBuf& b : m->layer) b.release();
      for (DevBuf& b : m->sel) b.release();
      m->tab_all.buf.release();
      m->tab_launch.buf.release();
      m->cloud.release();
      m->cloud_all.buf.release();
      m->cloud_sel.buf.release();
      m->fp.release();
    }
  }
  delete m;
  return TE_OK;
}

namespace {

// te_map_chain_image(_maps)'s images, as the caller passed them.
struct ImageIn {
  int32_t encoding;
  const void* px;
  int64_t row_stride, image_stride;
  double min_height, max_height;
};

// te_map_chain_submap / te_map_chain_windows' source: a larger elevation map (any start index) with the layers of `mask`
// (elevation and carried layers, in bit order, in `memory`), and where each window of the call starts in it, in launch order.
struct CutIn {
  const te_geometry* src;
  uint32_t mask;
  int nlayers;
  const float* layers[te::kCutMaxLayers];
  int memory;
  std::vector<int2> top;
};

// Where map_chain's elevation comes from: a float32 layer, images that k_image_to_layer turns into one, or windows that
// k_map_cut_windows cuts out of a larger map together with its carried layers.
struct ElevSource {
  const float* layer;
  const ImageIn* image;
  const CutIn* cut;
};

// Validates nmaps images of geometry g and returns their bytes per pixel.  Writes nothing.
int check_image(const ImageIn& im, const te_geometry& g, int nmaps, int* bpp) {
  if (im.encoding >= TE_IMAGE_RGB8 && im.encoding <= TE_IMAGE_BGRA16)
    return fail(TE_ERR_UNSUPPORTED, "colour image encoding %d: only mono8 and mono16 images are taken (the reference greys colour "
                "images with OpenCV's cvtColor, whose coefficients depend on the OpenCV version and build)", im.encoding);
  if (im.encoding != TE_IMAGE_MONO8 && im.encoding != TE_IMAGE_MONO16) return fail(TE_ERR_BAD_ARG, "unknown image encoding %d", im.encoding);
  if (!im.px) return fail(TE_ERR_MISSING_LAYER, "the images that give layer elevation are missing");
  const int b = im.encoding == TE_IMAGE_MONO16 ? 2 : 1;
  if (im.row_stride < (int64_t)g.cols * b)
    return fail(TE_ERR_BAD_ARG, "row_stride_bytes = %lld is less than a row of %d pixels of %d bytes", (long long)im.row_stride, g.cols, b);
  if (nmaps > 1 && (im.row_stride > INT64_MAX / g.rows || im.image_stride < im.row_stride * g.rows))
    return fail(TE_ERR_BAD_ARG, "image_stride_bytes = %lld is less than %d rows of %lld bytes", (long long)im.image_stride, g.rows,
                (long long)im.row_stride);
  if (b == 2 && (((uintptr_t)im.px | (uint64_t)im.row_stride | (uint64_t)(nmaps > 1 ? im.image_stride : 0)) & 1))
    return fail(TE_ERR_BAD_ARG, "mono16 images need an even address, row_stride_bytes and image_stride_bytes");
  *bpp = b;
  return TE_OK;
}

// addLayerFromImage: nmaps images of geometry g into the float32 elevation `out` (nmaps maps back to back), one launch.  In host
// memory only the image bytes are staged, packed in m->image; device images are read in place.
int map_convert_image(te_map* m, const te_geometry& g, const ImageIn& im, int bpp, int nmaps, int memory, float* out) {
  te_ctx* c = m->ctx;
  te::ImageToLayer a{im.px, im.row_stride, im.image_stride, g.rows, g.cols, nmaps, bpp, (float)im.min_height, 0.0f, out};
  a.diff = (float)im.max_height - a.lower;  // float32 operands and result: mapValueDifference
  if (memory == TE_MEM_HOST) {  // the image rows are the columns of the staged bytes
    const size_t row = (size_t)bpp * g.cols, image = row * g.rows;
    TE_CUDA(m->image.reserve(image * nmaps));
    char* dst = (char*)m->image.p;
    if (nmaps == 1 || (im.image_stride == im.row_stride * g.rows && (int64_t)g.rows * nmaps <= INT32_MAX)) {
      TE_CUDA(upload_cols(dst, im.px, g.cols, g.rows * nmaps, 0, 0, 0, g.rows * nmaps, c->stream, bpp, im.row_stride));
    } else {
      for (int k = 0; k < nmaps; ++k)
        TE_CUDA(upload_cols(dst + k * image, (const char*)im.px + k * im.image_stride, g.cols, g.rows, 0, 0, 0, g.rows, c->stream, bpp,
                            im.row_stride));
    }
    a.px = dst;
    a.row_stride = (long long)row;
    a.image_stride = (long long)image;
  }
  te::launch_image_to_layer(a, c->stream);
  return launch_check(c, "k_image_to_layer");
}

// One k_map_cut_windows launch (te_kernels.h WindowCut) of the windows `win`, nl layers each, from sources of src_rows x src_cols
// cells: its table goes to m->cut (the windows, the source pointers, the destination pointers, then col_of).  A table that grows
// first waits for the launches that may still read it.
int map_launch_cut(te_map* m, const std::vector<int4>& win, const std::vector<const float*>& src, const std::vector<float*>& dst,
                   const std::vector<int>& col_of, int nl, int rows, int cols, int src_rows, int src_cols) {
  te_ctx* c = m->ctx;
  const int n = (int)win.size();
  const size_t wbytes = sizeof(int4) * n, pbytes = sizeof(float*) * src.size(), cbytes = sizeof(int) * col_of.size();
  std::vector<char> h(wbytes + 2 * pbytes + cbytes);
  std::memcpy(h.data(), win.data(), wbytes);
  std::memcpy(h.data() + wbytes, src.data(), pbytes);
  std::memcpy(h.data() + wbytes + pbytes, dst.data(), pbytes);
  if (cbytes) std::memcpy(h.data() + wbytes + 2 * pbytes, col_of.data(), cbytes);
  if (m->cut.p && m->cut.cap < h.size()) TE_CUDA(cudaStreamSynchronize(c->stream));  // an earlier launch may still read it
  TE_CUDA(m->cut.reserve(h.size()));
  // pageable source: consumed before cudaMemcpyAsync returns, ordered after the kernels queued before on the stream
  TE_CUDA(cudaMemcpyAsync(m->cut.p, h.data(), h.size(), cudaMemcpyHostToDevice, c->stream));
  const char* t = (const char*)m->cut.p;
  te::WindowCut a{};
  a.win = (const int4*)t;
  a.src = (const float* const*)(t + wbytes);
  a.dst = (float* const*)(t + wbytes + pbytes);
  a.col_of = cbytes ? (const int*)(t + wbytes + 2 * pbytes) : nullptr;
  a.nlayers = nl;
  a.nmaps = n;
  a.rows = rows;
  a.cols = cols;
  a.src_rows = src_rows;
  a.src_cols = src_cols;
  a.ncolumns = (long long)n * nl * cols;
  te::launch_cut_windows(a, c->sms, c->stream);
  return launch_check(c, "k_map_cut_windows");
}

// One map's layer of the te_map's geometry moved whole: from src, read through the start index (sr, sc), to dst (device pointers).
struct MapBlock {
  const float* src;
  float* dst;
  int32_t sr, sc;
};

// Every block in one k_map_cut_windows launch (none for no block).
int map_move_blocks(te_map* m, const std::vector<MapBlock>& b) {
  if (b.empty()) return TE_OK;
  std::vector<int4> win(b.size());
  std::vector<const float*> src(b.size());
  std::vector<float*> dst(b.size());
  for (size_t k = 0; k < b.size(); ++k) {
    win[k] = int4{0, 0, b[k].sr, b[k].sc};
    src[k] = b[k].src;
    dst[k] = b[k].dst;
  }
  const int rows = m->geo.rows, cols = m->geo.cols;
  return map_launch_cut(m, win, src, dst, {}, 1, rows, cols, rows, cols);
}

// Whether any of the n (start_row, start_col) pairs st is not (0, 0) (st null: none).
bool any_start(const int32_t* st, int n) {
  if (!st) return false;
  for (int k = 0; k < 2 * n; ++k)
    if (st[k] != 0) return true;
  return false;
}

// The start indices of the maps s->idx[0..s->n) (s null: every map), pairs in that order.
std::vector<int32_t> map_starts(const te_map* m, const MapSel* s) {
  if (!s) return m->start;
  std::vector<int32_t> st(2 * (size_t)s->n);
  for (int k = 0; k < s->n; ++k) { st[2 * k] = m->start[2 * s->idx[k]]; st[2 * k + 1] = m->start[2 * s->idx[k] + 1]; }
  return st;
}

// Validates the start_index of a _wrapped entry: n pairs inside a map of rows x cols (null: none).  Writes nothing.
int check_start_indices(const int32_t* st, int n, int rows, int cols) {
  if (!st) return TE_OK;
  for (int k = 0; k < n; ++k)
    if (st[2 * k] < 0 || st[2 * k] >= rows || st[2 * k + 1] < 0 || st[2 * k + 1] >= cols)
      return fail(TE_ERR_BAD_ARG, "start_index[%d] = (%d, %d) is outside the map of %d x %d cells", k, st[2 * k], st[2 * k + 1], rows, cols);
  return TE_OK;
}

// Records the start indices of an update's maps: every map (idx null) or the maps idx[0..n), from the pairs st in call order
// (null: (0, 0)).
void map_set_starts(te_map* m, const int32_t* idx, int n, const int32_t* st) {
  for (int k = 0; k < n; ++k) {
    const int t = idx ? idx[k] : k;
    m->start[2 * t] = st ? st[2 * k] : 0;
    m->start[2 * t + 1] = st ? st[2 * k + 1] : 0;
  }
}

// m->wrap, at least `bytes` long; growing it first waits for the launches that may still read it.
int map_wrap_reserve(te_map* m, size_t bytes) {
  if (m->wrap.p && m->wrap.cap < bytes) TE_CUDA(cudaStreamSynchronize(m->ctx->stream));
  TE_CUDA(m->wrap.reserve(bytes));
  return TE_OK;
}

// The one way caller layers come into a te_map.  in[k], the layer of the k-th bit of `bits`, is null or holds the call's maps back
// to back in `memory`, map k of the call in the buffer order of the start index st[2k], st[2k + 1] (st null: (0, 0)).  A whole
// batch (sel null) lands in its resident layers, reserved for the batch; a host layer is read through geo_in's start index (a
// single map's, upload_cols).  A selection lands in the scratch m->sel[k], or is read in place when it is device memory with no
// start index; its scratch, with the buffers of `scratch`, and its slot table are staged first (map_stage_selection).  Every
// layer that needs unwrapping moves in one k_map_cut_windows launch, host layers after one copy each into m->wrap.  dev[k]
// receives layer k's device pointer, default order, the call's maps back to back (null where in[k] is).
int map_in(te_map* m, const MapSel* sel, uint32_t bits, const float* const in[], const int32_t* st, int memory, unsigned scratch,
           const float* dev[]) {
  te_ctx* c = m->ctx;
  const int n = sel ? sel->n : m->nmaps;
  const size_t cells = map_cells(m), lcells = cells * n;
  const bool wrapped = any_start(st, n), staged = memory == TE_MEM_HOST || wrapped;
  const int nl = __builtin_popcount(bits);
  if (sel) {
    for (int k = 0; k < nl; ++k)
      if (in[k] && staged) scratch |= 1u << k;
    if (int rc = map_stage_selection(m, *sel, scratch)) return rc;
  }
  std::vector<const float*> win;
  std::vector<float*> wto;
  for (int b = 0, k = 0; b < kLayerBits; ++b) {
    if (!((bits >> b) & 1u)) continue;
    const float* src = in[k];
    float* to = sel ? (float*)m->sel[k].p : nullptr;
    if (src && !sel) {
      TE_CUDA(m->layer[b].reserve(sizeof(float) * lcells));
      to = (float*)m->layer[b].p;
    }
    if (src && wrapped) {
      win.push_back(src);
      wto.push_back(to);
    } else if (src && !sel && memory == TE_MEM_HOST) {
      const te_geometry& g = m->geo_in;
      TE_CUDA(upload_cols(to, src, g.rows, g.cols, g.start_row, g.start_col, 0, g.cols * n, c->stream));
    } else if (src && (!sel || memory == TE_MEM_HOST)) {
      TE_CUDA(cudaMemcpyAsync(to, src, sizeof(float) * lcells, sel ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
    }
    dev[k++] = !src ? nullptr : staged || !sel ? to : src;
  }
  if (win.empty()) return TE_OK;
  if (memory == TE_MEM_HOST) {
    if (int rc = map_wrap_reserve(m, sizeof(float) * lcells * win.size())) return rc;
    for (size_t l = 0; l < win.size(); ++l) {
      float* d = (float*)m->wrap.p + l * lcells;
      TE_CUDA(cudaMemcpyAsync(d, win[l], sizeof(float) * lcells, cudaMemcpyHostToDevice, c->stream));
      win[l] = d;
    }
  }
  std::vector<MapBlock> blocks;
  for (size_t l = 0; l < win.size(); ++l)
    for (int k = 0; k < n; ++k) blocks.push_back(MapBlock{win[l] + k * cells, wto[l] + k * cells, st[2 * k], st[2 * k + 1]});
  return map_move_blocks(m, blocks);
}

// Host outputs in buffer order: block b's src is a map in default order on the device, its dst the HOST array that takes it in the
// buffer order of the block's start index.  One launch re-wraps every block into m->wrap, then one copy per run of blocks that
// are contiguous on the host brings them back.  The caller synchronises.
int map_wrap_out(te_map* m, const std::vector<MapBlock>& b) {
  if (b.empty()) return TE_OK;
  const size_t cells = map_cells(m);
  const int rows = m->geo.rows, cols = m->geo.cols;
  if (int rc = map_wrap_reserve(m, sizeof(float) * cells * b.size())) return rc;
  float* const w = (float*)m->wrap.p;
  std::vector<MapBlock> d(b.size());
  for (size_t k = 0; k < b.size(); ++k)
    d[k] = MapBlock{b[k].src, w + k * cells, (rows - b[k].sr) % rows, (cols - b[k].sc) % cols};
  if (int rc = map_move_blocks(m, d)) return rc;
  for (size_t k = 0; k < b.size();) {
    size_t e = k + 1;
    while (e < b.size() && b[e].dst == b[e - 1].dst + cells) ++e;
    TE_CUDA(cudaMemcpyAsync(b[k].dst, w + k * cells, sizeof(float) * cells * (e - k), cudaMemcpyDeviceToHost, m->ctx->stream));
    k = e;
  }
  return TE_OK;
}

// The one way a te_map's layers go out to the caller.  src[l] holds the call's maps back to back or, `resident`, each map in its
// slot (map k of a selection at sel->idx[k]); out[l] (null: not wanted) takes the call's maps back to back in `memory`.  Host
// outputs of maps with a start index of their own come back in buffer order (map_wrap_out).  Otherwise a whole batch is copied
// (in host memory through geo_in's start index, a single map's: download_cols), a packed selection is copied, and a resident
// selection is gathered by one k_map_slots launch, straight into device outputs and into the caller's staged m->sel[0 .. nl)
// before a copy to host ones.  Host memory returns synchronised.
int map_out(te_map* m, const MapSel* sel, int nl, const float* const src[], bool resident, float* const out[], int memory) {
  te_ctx* c = m->ctx;
  const bool host = memory == TE_MEM_HOST;
  const int n = sel ? sel->n : m->nmaps;
  const size_t cells = map_cells(m);
  const std::vector<int32_t> st = map_starts(m, sel);
  std::vector<const float*> from(src, src + nl);
  if (host && any_start(st.data(), n)) {
    std::vector<MapBlock> b;
    for (int l = 0; l < nl; ++l)
      if (out[l])
        for (int k = 0; k < n; ++k)
          b.push_back(MapBlock{src[l] + (size_t)(sel && resident ? sel->idx[k] : k) * cells, out[l] + k * cells, st[2 * k], st[2 * k + 1]});
    if (int rc = map_wrap_out(m, b)) return rc;
    from.assign(nl, nullptr);
  } else if (sel && resident && std::any_of(out, out + nl, [](float* o) { return o != nullptr; })) {
    te::MapSlots a{};
    for (int l = 0; l < nl; ++l) {
      a.src[l] = out[l] ? src[l] : nullptr;
      a.dst[l] = !out[l] ? nullptr : host ? (float*)m->sel[l].p : out[l];
      from[l] = host ? a.dst[l] : nullptr;
    }
    a.slot = (const int*)m->slots.p;
    a.nsel = n;
    a.cells = cells;
    te::launch_map_slots(a, false, c->sms, c->stream);
    if (int rc = launch_check(c, "k_map_slots (get)")) return rc;
  }
  const te_geometry& g = m->geo_in;
  for (int l = 0; l < nl; ++l) {
    if (!out[l] || !from[l]) continue;
    if (host && !sel) TE_CUDA(download_cols(out[l], from[l], g.rows, g.cols, g.start_row, g.start_col, 0, g.cols * n, c->stream));
    else TE_CUDA(cudaMemcpyAsync(out[l], from[l], sizeof(float) * cells * n, host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  }
  if (host) TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

// The windows of `cut` into the maps of a chain launch of geometry m->geo, in one launch: the elevation of map k of the launch to
// elev + k * cells (the te_map's layer on a whole-batch update, the selection's packed scratch otherwise), each carried layer
// straight to its resident slot (map k, or sel->idx[k]).  Device sources are read in place; host sources stage only the source
// columns the windows touch, one copy per contiguous run of stored columns and layer, and the kernel finds them through a
// column table.
int map_cut(te_map* m, const CutIn& cut, const MapSel* sel, float* elev) {
  te_ctx* c = m->ctx;
  const te_geometry& s = *cut.src;
  const int n = (int)cut.top.size(), nl = cut.nlayers, rows = m->geo.rows, cols = m->geo.cols;
  const size_t cells = map_cells(m);
  std::vector<float*> dst((size_t)n * nl);
  int l = 0;
  for (int b = 0; b < kLayerBits; ++b) {
    if (!((cut.mask >> b) & 1u)) continue;
    float* base = elev;
    if (b != 4) {
      DevBuf& buf = m->layer[b];
      if (!sel) TE_CUDA(buf.reserve(sizeof(float) * batch_cells(m)));
      base = (float*)buf.p;
    }
    for (int k = 0; k < n; ++k) dst[(size_t)k * nl + l] = base + (size_t)(b != 4 && sel ? sel->idx[k] : k) * cells;
    ++l;
  }
  const float* srcl[te::kCutMaxLayers];
  std::vector<int> col_of;
  for (int k = 0; k < nl; ++k) srcl[k] = cut.layers[k];
  if (cut.memory == TE_MEM_HOST) {
    std::vector<char> touched(s.cols, 0);
    for (const int2& t : cut.top)
      for (long long J = std::max(0LL, (long long)t.y); J < std::min((long long)s.cols, (long long)t.y + cols); ++J)
        touched[(J + s.start_col) % s.cols] = 1;
    col_of.assign(s.cols, -1);
    int nst = 0;
    for (int j = 0; j < s.cols; ++j)
      if (touched[j]) col_of[j] = nst++;
    Staging st(c, true, &s);
    float* staged = (float*)st.slot(sizeof(float) * s.rows * (size_t)nst * nl);
    if (st.rc) return st.rc;
    for (int j = 0; j < s.cols;) {  // runs of touched stored columns
      if (!touched[j]) { ++j; continue; }
      int e = j;
      while (e < s.cols && touched[e]) ++e;
      for (int k = 0; k < nl; ++k)
        TE_CUDA(cudaMemcpyAsync(staged + ((size_t)k * nst + col_of[j]) * s.rows, cut.layers[k] + (size_t)j * s.rows,
                                sizeof(float) * s.rows * (size_t)(e - j), cudaMemcpyHostToDevice, c->stream));
      j = e;
    }
    for (int k = 0; k < nl; ++k) srcl[k] = staged + (size_t)k * nst * s.rows;
  }
  std::vector<int4> win(n);
  std::vector<const float*> src((size_t)n * nl);
  for (int k = 0; k < n; ++k) {
    win[k] = int4{cut.top[k].x, cut.top[k].y, s.start_row, s.start_col};
    for (int l2 = 0; l2 < nl; ++l2) src[(size_t)k * nl + l2] = srcl[l2];
  }
  return map_launch_cut(m, win, src, dst, col_of, nl, rows, cols, s.rows, s.cols);
}

// te_map_chain (nmaps = 1), te_map_chain_batched and, with a selection, te_map_chain_maps, from an elevation layer, from images
// (te_map_chain_image(_maps)) or from windows of a larger map (te_map_chain_submap / _windows): the selected maps' layers are
// chained into scratch (the elevation staged there in host memory, read in place in device memory; images converted and windows
// cut there in both) and k_map_slots puts them in place.  Windows also carry the source's carried layers: on a whole batch they
// replace the batch's, on a selection they go straight to the selected maps' slots and only the batch's other carried layers are
// filled with NaN.
// at: an _at entry, whose maps go to position_xy (null: g's position) and whose g may differ from the batch's in its position.
// start_index (the _wrapped entries): the start index of each map of the call (null: (0, 0)), which its elevation comes in and
// its host outputs go back in.
int map_chain(te_map* m, const te_geometry* g_in, const te_chain_params* p, int nmaps, const ElevSource& src, float* slope, float* step,
              float* rough, float* trav, int memory, const MapSel* sel = nullptr, bool at = false, const double* position_xy = nullptr,
              const int32_t* start_index = nullptr) {
  te_ctx* c = m->ctx;
  te_geometry g0;
  if (src.image && g_in && (g_in->start_row != 0 || g_in->start_col != 0))
    return fail(TE_ERR_UNSUPPORTED, "circular-buffer start index (%d,%d) != (0,0): an image map has none", g_in->start_row, g_in->start_col);
  if (sel) {
    if (int rc = map_select(m, true, g_in, *sel, at)) return rc;
    g0 = m->geo;
    nmaps = sel->n;
  } else if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST && nmaps == 1 && !src.cut, &g0)) {
    return rc;
  }
  if (int rc = check_params(p)) return rc;
  if (nmaps > 0) {
    if (int rc = check_positions(position_xy, nmaps)) return rc;
    if (int rc = check_start_indices(start_index, nmaps, g0.rows, g0.cols)) return rc;
  }
  if (!src.layer && !src.image && !src.cut) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  if (sel && src.cut)
    if (const uint32_t extra = src.cut->mask & TE_LAYER_CARRIED & ~m->held)
      return fail(TE_ERR_BAD_ARG, "layer %s is given to some maps but the batch does not hold it: every map of a batch holds the same "
                  "layers, so give it to every map (map_index NULL)", kLayerNames[__builtin_ctz(extra)]);
  if (sel && (m->held & (TE_LAYER_ROUGHNESS | TE_LAYER_ROBOT_SLOPE)) != TE_LAYER_ROUGHNESS)
    return fail(TE_ERR_UNSUPPORTED, "the batch %s, and te_map_chain_maps gives a map roughness and no robot_slope: every map of a batch holds "
                "the same layers, so use te_map_set_layers_maps or reload the whole batch",
                m->held & TE_LAYER_ROBOT_SLOPE ? "holds robot_slope" : "has no roughness");
  int bpp = 0;
  if (src.image)
    if (int rc = check_image(*src.image, g0, nmaps, &bpp)) return rc;
  if (!sel) {
    if (int rc = map_reset(m, g_in, &g0, nmaps)) return rc;
    TE_CUDA(m->layer[3].reserve(sizeof(float) * batch_cells(m)));
  }
  // where the chain reads and writes: elevation, slope, step, roughness, traversability (sel[0]: the staged, unwrapped,
  // converted or cut elevation)
  DevBuf* const lay[5] = {sel ? &m->sel[0] : &m->layer[4], sel ? &m->sel[1] : &m->layer[1], sel ? &m->sel[2] : &m->layer[2],
                          sel ? &m->sel[3] : &m->layer[3], sel ? &m->sel[4] : &m->layer[0]};
  const float* din = nullptr;
  if (int rc = map_in(m, sel, TE_LAYER_ELEVATION, &src.layer, start_index, memory, src.layer ? 0x1eu : 0x1fu, &din)) return rc;
  if (src.image) {
    if (int rc = map_convert_image(m, g0, *src.image, bpp, nmaps, memory, (float*)lay[0]->p)) return rc;
    din = (const float*)lay[0]->p;
  }
  if (src.cut) {
    if (int rc = map_cut(m, *src.cut, sel, (float*)lay[0]->p)) return rc;
    din = (const float*)lay[0]->p;
    if (!sel) m->held |= src.cut->mask & TE_LAYER_CARRIED;
  }
  // where the launch's maps go; maps away from g0's position take per-map tables
  const std::vector<double> at_xy = launch_positions(position_xy, nmaps, g_in->position_x, g_in->position_y);
  PosTables tab{};
  const bool spread = !all_at(at_xy.data(), nmaps, g0.position_x, g0.position_y);
  if (spread)
    if (int rc = map_tables(c, m->tab_launch, g0, at_xy.data(), nmaps, p, &tab)) return rc;
  if (int rc = chain_common(c, &g0, nullptr, p, nmaps, din, (float*)lay[1]->p, (float*)lay[2]->p, (float*)lay[3]->p, (float*)lay[4]->p,
                            nullptr, nullptr, nullptr, TE_MEM_DEVICE, spread ? &tab : nullptr))
    return rc;
  map_place(m, sel ? sel->idx : nullptr, nmaps, at_xy);
  map_set_starts(m, sel ? sel->idx : nullptr, nmaps, start_index);
  if (sel) {
    const float* const src_l[te::kMapSlotLayers] = {(const float*)lay[4]->p, (const float*)lay[1]->p, (const float*)lay[2]->p,
                                                    (const float*)lay[3]->p, din};
    const uint32_t chained = TE_LAYER_TRAVERSABILITY | TE_LAYER_SLOPE | TE_LAYER_STEP | TE_LAYER_ROUGHNESS | TE_LAYER_ELEVATION;
    if (int rc = map_put_selected(m, *sel, chained, src_l, src.cut ? src.cut->mask & TE_LAYER_CARRIED : 0u)) return rc;
  } else {
    m->held |= TE_LAYER_ROUGHNESS;  // computeTraversability leaves robot_slope to a later setTraversabilityMap
    m->have_layers = true;
  }
  // the launch's maps are back to back in lay[] on a whole batch and on a selection
  float* const out[4] = {slope, step, rough, trav};
  const float* const dev[4] = {(const float*)lay[1]->p, (const float*)lay[2]->p, (const float*)lay[3]->p, (const float*)lay[4]->p};
  return map_out(m, sel, 4, dev, false, out, memory);
}

// te_map_set_layers (nmaps = 1), te_map_set_layers_batched and, with a selection, te_map_set_layers_maps: the selected maps'
// layers (staged in host memory, read in place in device memory) go to their slots in one k_map_slots launch.  The optional
// layers must then be those the batch holds.
int map_set_layers(te_map* m, const te_geometry* g_in, int nmaps, const float* trav, const float* slope, const float* step,
                   const float* rough, const float* elev, const float* robot_slope, int memory, const MapSel* sel = nullptr,
                   bool at = false, const double* position_xy = nullptr, const int32_t* start_index = nullptr) {
  te_ctx* c = m->ctx;
  te_geometry g0;
  if (sel) {
    if (int rc = map_select(m, true, g_in, *sel, at)) return rc;
    nmaps = sel->n;
    g0 = m->geo;
  } else if (int rc = unwrap_geometry(g_in, memory == TE_MEM_HOST && nmaps == 1, &g0)) {
    return rc;
  }
  if (nmaps > 0) {
    if (int rc = check_positions(position_xy, nmaps)) return rc;
    if (int rc = check_start_indices(start_index, nmaps, g0.rows, g0.cols)) return rc;
  }
  const std::vector<double> at_xy = launch_positions(position_xy, std::max(nmaps, 0), g_in->position_x, g_in->position_y);
  if (!trav) return fail(TE_ERR_MISSING_LAYER, "layer traversability is missing");
  if (!slope) return fail(TE_ERR_MISSING_LAYER, "layer traversability_slope is missing");
  if (!step) return fail(TE_ERR_MISSING_LAYER, "layer traversability_step is missing");
  if (!elev) return fail(TE_ERR_MISSING_LAYER, "layer elevation is missing");
  const uint32_t given = (rough ? TE_LAYER_ROUGHNESS : 0u) | (robot_slope ? TE_LAYER_ROBOT_SLOPE : 0u);
  for (const uint32_t b : {(uint32_t)TE_LAYER_ROUGHNESS, (uint32_t)TE_LAYER_ROBOT_SLOPE}) {
    if (!sel || !((m->held ^ given) & b)) continue;
    if (m->held & b)
      return fail(TE_ERR_MISSING_LAYER, "layer %s is missing: the batch holds it, so every map needs it", kLayerNames[__builtin_ctz(b)]);
    return fail(TE_ERR_BAD_ARG, "layer %s is given but the batch does not hold it: reload the whole batch to add it",
                kLayerNames[__builtin_ctz(b)]);
  }
  if (!sel)
    if (int rc = map_reset(m, g_in, &g0, nmaps)) return rc;
  // bits 0 .. 5: the layers of te_map_set_layers in bit order
  const float* const in[6] = {trav, slope, step, rough, elev, robot_slope};
  const float* dev[6];
  if (int rc = map_in(m, sel, 0x3fu, in, start_index, memory, 0u, dev)) return rc;
  if (sel) {
    if (int rc = map_put_selected(m, *sel, 0x3fu, dev)) return rc;
  } else {
    m->held |= given;
  }
  map_place(m, sel ? sel->idx : nullptr, nmaps, at_xy);
  map_set_starts(m, sel ? sel->idx : nullptr, nmaps, start_index);
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));  // the caller may reuse its layers on return
  m->have_layers = true;
  return TE_OK;
}

}  // namespace

int te_map_chain(te_map* m, const te_geometry* g_in, const te_chain_params* p, const float* elev, float* slope, float* step, float* rough,
                 float* trav, int memory) {
  TE_MAP_ENTER(m);
  return map_chain(m, g_in, p, 1, ElevSource{elev, nullptr}, slope, step, rough, trav, memory);
}

int te_map_chain_batched(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elev, float* slope,
                         float* step, float* rough, float* trav, int memory) {
  TE_MAP_ENTER(m);
  return map_chain(m, g, p, nmaps, ElevSource{elev, nullptr}, slope, step, rough, trav, memory);
}

int te_map_set_layers(te_map* m, const te_geometry* g_in, const float* trav, const float* slope, const float* step, const float* rough,
                      const float* elev, const float* robot_slope, int memory) {
  TE_MAP_ENTER(m);
  return map_set_layers(m, g_in, 1, trav, slope, step, rough, elev, robot_slope, memory);
}

int te_map_set_layers_batched(te_map* m, const te_geometry* g, int32_t nmaps, const float* trav, const float* slope, const float* step,
                              const float* rough, const float* elev, const float* robot_slope, int memory) {
  TE_MAP_ENTER(m);
  return map_set_layers(m, g, nmaps, trav, slope, step, rough, elev, robot_slope, memory);
}

int te_map_chain_maps(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index, const float* elev,
                      float* slope, float* step, float* rough, float* trav, int memory) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  return map_chain(m, g, p, nsel, ElevSource{elev, nullptr}, slope, step, rough, trav, memory, &sel);
}

int te_map_chain_batched_at(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elev, float* slope,
                            float* step, float* rough, float* trav, int memory, const double* position_xy) {
  TE_MAP_ENTER(m);
  return map_chain(m, g, p, nmaps, ElevSource{elev, nullptr}, slope, step, rough, trav, memory, nullptr, true, position_xy);
}

int te_map_set_layers_batched_at(te_map* m, const te_geometry* g, int32_t nmaps, const float* trav, const float* slope, const float* step,
                                 const float* rough, const float* elev, const float* robot_slope, int memory, const double* position_xy) {
  TE_MAP_ENTER(m);
  return map_set_layers(m, g, nmaps, trav, slope, step, rough, elev, robot_slope, memory, nullptr, true, position_xy);
}

int te_map_chain_maps_at(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                         const float* elev, float* slope, float* step, float* rough, float* trav, int memory, const double* position_xy) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  return map_chain(m, g, p, nsel, ElevSource{elev, nullptr}, slope, step, rough, trav, memory, &sel, true, position_xy);
}

int te_map_set_layers_maps_at(te_map* m, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* trav,
                              const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                              int memory, const double* position_xy) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  return map_set_layers(m, g, nsel, trav, slope, step, rough, elev, robot_slope, memory, &sel, true, position_xy);
}

int te_map_positions(te_map* m, double* position_xy) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!position_xy) return fail(TE_ERR_BAD_ARG, "position_xy is null");
  std::memcpy(position_xy, m->pos.data(), sizeof(double) * m->pos.size());
  return TE_OK;
}

namespace {

// The _wrapped entries take the start index in their own array only.
int check_wrapped_geometry(const te_geometry* g) {
  if (g && (g->start_row != 0 || g->start_col != 0))
    return fail(TE_ERR_BAD_ARG, "g has start index (%d,%d): the _wrapped entries take each map's start index in start_index, and g's "
                "must be (0,0)", g->start_row, g->start_col);
  return TE_OK;
}

}  // namespace

int te_map_chain_batched_wrapped(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nmaps, const float* elev, float* slope,
                                 float* step, float* rough, float* trav, int memory, const double* position_xy, const int32_t* start_index) {
  TE_MAP_ENTER(m);
  if (int rc = check_wrapped_geometry(g)) return rc;
  return map_chain(m, g, p, nmaps, ElevSource{elev, nullptr}, slope, step, rough, trav, memory, nullptr, true, position_xy, start_index);
}

int te_map_set_layers_batched_wrapped(te_map* m, const te_geometry* g, int32_t nmaps, const float* trav, const float* slope, const float* step,
                                      const float* rough, const float* elev, const float* robot_slope, int memory, const double* position_xy,
                                      const int32_t* start_index) {
  TE_MAP_ENTER(m);
  if (int rc = check_wrapped_geometry(g)) return rc;
  return map_set_layers(m, g, nmaps, trav, slope, step, rough, elev, robot_slope, memory, nullptr, true, position_xy, start_index);
}

int te_map_chain_maps_wrapped(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                              const float* elev, float* slope, float* step, float* rough, float* trav, int memory, const double* position_xy,
                              const int32_t* start_index) {
  TE_MAP_ENTER(m);
  if (int rc = check_wrapped_geometry(g)) return rc;
  const MapSel sel{nsel, map_index};
  return map_chain(m, g, p, nsel, ElevSource{elev, nullptr}, slope, step, rough, trav, memory, &sel, true, position_xy, start_index);
}

int te_map_set_layers_maps_wrapped(te_map* m, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* trav,
                                   const float* slope, const float* step, const float* rough, const float* elev, const float* robot_slope,
                                   int memory, const double* position_xy, const int32_t* start_index) {
  TE_MAP_ENTER(m);
  if (int rc = check_wrapped_geometry(g)) return rc;
  const MapSel sel{nsel, map_index};
  return map_set_layers(m, g, nsel, trav, slope, step, rough, elev, robot_slope, memory, &sel, true, position_xy, start_index);
}

int te_map_start_indices(te_map* m, int32_t* start_index) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!start_index) return fail(TE_ERR_BAD_ARG, "start_index is null");
  if (m->geo_in.start_row != 0 || m->geo_in.start_col != 0) {  // a single map whose start index came in g
    start_index[0] = m->geo_in.start_row;
    start_index[1] = m->geo_in.start_col;
    return TE_OK;
  }
  std::memcpy(start_index, m->start.data(), sizeof(int32_t) * m->start.size());
  return TE_OK;
}

int te_image_geometry(int32_t height, int32_t width, double resolution, double position_x, double position_y, te_geometry* out) {
  if (!out) return fail(TE_ERR_BAD_ARG, "out is null");
  if (height < 1 || width < 1) return fail(TE_ERR_BAD_ARG, "image size %d x %d: need at least 1 x 1", height, width);
  if (!(resolution > 0.0) || !std::isfinite(resolution)) return fail(TE_ERR_BAD_ARG, "resolution must be finite and positive");
  if (!std::isfinite(position_x) || !std::isfinite(position_y)) return fail(TE_ERR_BAD_ARG, "position must be finite");
  // initializeFromImage: setGeometry(Length(resolution * height, resolution * width), resolution, position)
  const double length_x = resolution * height, length_y = resolution * width;
  if (!std::isfinite(length_x) || !std::isfinite(length_y)) return fail(TE_ERR_BAD_ARG, "resolution * image size is not finite");
  te_geometry g{};
  g.rows = (int)std::round(length_x / resolution);  // setGeometry: size = round(length / resolution), length = size * resolution
  g.cols = (int)std::round(length_y / resolution);
  g.resolution = resolution;
  g.length_x = g.rows * resolution;
  g.length_y = g.cols * resolution;
  g.position_x = position_x;
  g.position_y = position_y;
  *out = g;
  return TE_OK;
}

int te_map_chain_image(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nmaps, int32_t encoding, const void* images,
                       int64_t row_stride_bytes, int64_t image_stride_bytes, double min_height, double max_height, float* slope,
                       float* step, float* rough, float* trav, int memory) {
  TE_MAP_ENTER(m);
  const ImageIn im{encoding, images, row_stride_bytes, image_stride_bytes, min_height, max_height};
  return map_chain(m, g, p, nmaps, ElevSource{nullptr, &im}, slope, step, rough, trav, memory);
}

int te_map_chain_image_maps(te_map* m, const te_geometry* g, const te_chain_params* p, int32_t nsel, const int32_t* map_index,
                            int32_t encoding, const void* images, int64_t row_stride_bytes, int64_t image_stride_bytes, double min_height,
                            double max_height, float* slope, float* step, float* rough, float* trav, int memory) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  const ImageIn im{encoding, images, row_stride_bytes, image_stride_bytes, min_height, max_height};
  return map_chain(m, g, p, nsel, ElevSource{nullptr, &im}, slope, step, rough, trav, memory, &sel);
}

int te_map_set_layers_maps(te_map* m, const te_geometry* g, int32_t nsel, const int32_t* map_index, const float* trav, const float* slope,
                           const float* step, const float* rough, const float* elev, const float* robot_slope, int memory) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  return map_set_layers(m, g, nsel, trav, slope, step, rough, elev, robot_slope, memory, &sel);
}

// mapOut = mapIn for robot_slope and the carried layers.  Every map: given layers are copied in (map_in), and one k_map_slots
// launch with the identity slot table fills the NULL ones with 0.0f.  A selection: given layers (staged in host memory, read in
// place in device memory) go to their slots and the NULL ones are filled, in one k_map_slots launch.  Neither touches the cache
// or the memo.
int te_map_carry_layers(te_map* m, int32_t nsel, const int32_t* map_index, uint32_t layer_mask, const float* layers[], int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  const uint32_t allowed = (uint32_t)TE_LAYER_ROBOT_SLOPE | (uint32_t)TE_LAYER_CARRIED;
  if (layer_mask == 0 || (layer_mask & ~allowed))
    return fail(TE_ERR_BAD_ARG, "layer mask 0x%x: te_map_carry_layers takes a non-empty subset of 0x%x (robot_slope and the elevation "
                "map's layers)", layer_mask, allowed);
  if (!layers) return fail(TE_ERR_BAD_ARG, "layers is null");
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  const bool whole = nsel == 0 && !map_index;
  const MapSel sel{nsel, map_index};
  if (!whole) {
    if (int rc = map_select(m, false, nullptr, sel)) return rc;
    if (const uint32_t extra = layer_mask & ~m->held)
      return fail(TE_ERR_BAD_ARG, "layer %s is given to some maps but the batch does not hold it: every map of a batch holds the same "
                  "layers, so give it to every map (nsel = 0, map_index NULL)", kLayerNames[__builtin_ctz(extra)]);
  }
  // maps with a start index of their own (the _wrapped entries) take their layers in that buffer order
  const std::vector<int32_t> starts = map_starts(m, whole ? nullptr : &sel);
  if (whole)  // the NULL layers too: they are filled
    for (int b = 0; b < kLayerBits; ++b)
      if ((layer_mask >> b) & 1u) TE_CUDA(m->layer[b].reserve(sizeof(float) * batch_cells(m)));
  const float* dev[te::kMapSlotLayers];
  if (int rc = map_in(m, whole ? nullptr : &sel, layer_mask, layers, starts.data(), memory, 0u, dev)) return rc;
  // a selection's layers go to their slots; the NULL ones are filled
  te::MapSlots a{};
  a.nsel = whole ? m->nmaps : sel.n;
  a.cells = map_cells(m);
  a.fill_bits = 0u;  // GridMap::add(layer, 0.0)
  a.slot = whole ? nullptr : (const int*)m->slots.p;
  bool launch = !whole;
  for (int b = 0, k = 0; b < kLayerBits; ++b) {
    if (!((layer_mask >> b) & 1u)) continue;
    if (dev[k] && !whole) {
      a.src[k] = dev[k];
      a.dst[k] = (float*)m->layer[b].p;
    } else if (!dev[k]) {
      a.fill[k] = (float*)m->layer[b].p;
      launch = true;
    }
    ++k;
  }
  if (launch) {
    te::launch_map_slots(a, true, c->sms, c->stream);
    if (int rc = launch_check(c, "k_map_slots (carry)")) return rc;
  }
  if (whole) m->held |= layer_mask;
  if (memory == TE_MEM_HOST) TE_CUDA(cudaStreamSynchronize(c->stream));  // the caller may reuse its layers on return
  return TE_OK;
}

// The resident layers a footprint sweep reads into in[]: te_layer bits 0 .. 4 (trav, slope, step, rough when verify_roughness,
// elev).  A selection's are gathered into m->sel[0 .. 4] by one k_map_slots launch, which the caller counts.
int map_sweep_inputs(te_map* m, const te_footprint_params* p, const MapSel* sel, const float* in[5]) {
  unsigned gathered = 0;
  for (int b = 0; b < 5; ++b) {
    in[b] = b == 3 && !p->verify_roughness ? nullptr : (const float*)m->layer[b].p;
    if (in[b]) gathered |= 1u << b;
  }
  if (!sel) return TE_OK;
  if (int rc = map_stage_selection(m, *sel, gathered)) return rc;
  te::MapSlots a{};
  for (int l = 0; l < 5; ++l) {
    a.src[l] = in[l];
    a.dst[l] = in[l] ? (float*)m->sel[l].p : nullptr;
    in[l] = a.dst[l];
  }
  a.slot = (const int*)m->slots.p;
  a.nsel = sel->n;
  a.cells = map_cells(m);
  te::launch_map_slots(a, false, m->ctx->sms, m->ctx->stream);
  return TE_OK;
}

// te_map_footprint (sel null: every map, swept in place) and te_map_footprint_maps (the selected maps' input layers gathered
// into scratch by one k_map_slots launch, swept as a batch of nsel maps and merged into their cache slots).  A map's sweep reads
// only its own cells, so each selected map gets the values a whole-batch sweep gives it.
static int map_footprint(te_map* m, const te_footprint_params* p, const MapSel* sel, float* out, int memory) {
  te_ctx* c = m->ctx;
  if (int rc = sel ? map_select(m, false, nullptr, *sel) : map_ready(m)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  if (!(p->radius >= 0.0) || !(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint radius/offset must be >= 0");
  te_geometry gm;
  PosTables tab{};
  const bool spread = !map_geometry(m, &gm);  // the maps at several positions: their own tables
  if (spread) gm = m->geo;
  const te_geometry* g = &gm;
  if (int rc = ensure_geometry(c, g)) return rc;
  const int n = sel ? sel->n : m->nmaps;
  if (spread)
    if (int rc = map_tables_of(m, MapSel{n, sel ? sel->idx : nullptr}, &tab)) return rc;
  TE_CUDA(m->fresh.reserve(sizeof(float) * map_cells(m) * n));
  const te_slab s{0, g->cols, 0, 0};
  const float* in[5];
  if (int rc = map_sweep_inputs(m, p, sel, in)) return rc;
  const int fixed = sel ? 2 : 1;  // k_map_merge, and k_map_slots for a selection
  // the sweep's own limit, found before the recorded layers change
  if (!te::footprint_reach_ok(g->resolution, p)) return fail(TE_ERR_UNSUPPORTED, "footprint radius + offset spans more than 120 cells");
  if (int rc = map_plane(m, p, false, sel)) return rc;
  std::vector<unsigned char> walk(n);
  bool any_walk = false;
  for (int k = 0; k < n; ++k) any_walk |= (walk[k] = m->plane_covers[sel ? sel->idx[k] : k] ? 0 : 1) != 0;
  const te::SweepRecord rec{(unsigned char*)m->plane.p, lay(m, TE_LAYER_FOOTPRINT), sel ? (const int*)m->slots.p : nullptr,
                            any_walk ? walk.data() : nullptr};
  int nl = 0;
  int rc = te::launch_footprint(m->fp, view_at(make_view(c, g, s), g, spread ? &tab : nullptr), g, p, n, in[0], in[1], in[2], in[3], in[4],
                                (float*)m->fresh.p, nullptr, nullptr, nullptr, c->sms, c->stream, &nl, &rec);
  if (rc != 0) return fail(rc, "footprint sweep failed: %s", m->fp.why.c_str());
  // host memory: the whole cache is read back from its resident layer, a selection's from packed scratch (its trav slot)
  float* const dout = !out ? nullptr : memory == TE_MEM_DEVICE ? out : sel ? (float*)m->sel[0].p : nullptr;
  te::launch_map_merge((const float*)m->fresh.p, lay(m, TE_LAYER_FOOTPRINT), dout, sel ? map_cells(m) : batch_cells(m),
                       sel ? (const int*)m->slots.p : nullptr, sel ? n : 1, c->sms, c->stream);
  if (int r2 = launch_check(c, "map footprint", nl + fixed)) return r2;
  if (!out || memory != TE_MEM_HOST) return TE_OK;
  const float* const from = sel ? dout : lay(m, TE_LAYER_FOOTPRINT);  // the swept maps back to back
  return map_out(m, sel, 1, &from, false, &out, memory);
}

int te_map_footprint(te_map* m, const te_footprint_params* p, float* out, int memory) {
  TE_MAP_ENTER(m);
  return map_footprint(m, p, nullptr, out, memory);
}

int te_map_footprint_maps(te_map* m, const te_footprint_params* p, int32_t nsel, const int32_t* map_index, float* out, int memory) {
  TE_MAP_ENTER(m);
  const MapSel sel{nsel, map_index};
  return map_footprint(m, p, &sel, out, memory);
}

// te_map_footprint(_maps) with map k's parameters params[k]: the swept maps grouped by bitwise-identical parameters, in order of
// first appearance, each group swept as a te_map_footprint_maps selection (the sweep's per-radius tables stay kernel parameters).
// One group is the entry it stands for, output included; several gather the swept caches afterwards with map_out.
int te_map_footprint_each(te_map* m, const te_footprint_params* params, int32_t nsel, const int32_t* map_index, float* out, int memory) {
  TE_MAP_ENTER(m);
  const bool whole = nsel == 0 && !map_index;
  const MapSel sel{nsel, map_index};
  if (int rc = whole ? map_ready(m) : map_select(m, false, nullptr, sel)) return rc;
  if (!params) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  const int n = whole ? m->nmaps : sel.n;
  std::vector<std::vector<int32_t>> groups;
  std::map<std::vector<unsigned char>, size_t> group_of;
  for (int k = 0; k < n; ++k) {
    const int32_t mi = whole ? k : map_index[k];
    const te_footprint_params* p = params + mi;
    if (int rc = map_footprint_params(m, p)) return rc;
    if (!(p->radius >= 0.0) || !(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint radius/offset of map %d must be >= 0", mi);
    // the sweep's own limit, found here so that no group is swept before a later one fails
    if (!te::footprint_reach_ok(m->geo.resolution, p))
      return fail(TE_ERR_UNSUPPORTED, "footprint radius + offset of map %d spans more than 120 cells", mi);
    const unsigned char* b = (const unsigned char*)p;
    const auto it = group_of.emplace(std::vector<unsigned char>(b, b + sizeof(*p)), groups.size());
    if (it.second) groups.emplace_back();
    groups[it.first->second].push_back(mi);
  }
  if (groups.size() == 1) return map_footprint(m, params + groups[0][0], whole ? nullptr : &sel, out, memory);
  for (const std::vector<int32_t>& gi : groups) {
    const MapSel gs{(int32_t)gi.size(), gi.data()};
    if (int rc = map_footprint(m, params + gi[0], &gs, nullptr, memory)) return rc;
  }
  if (!out) return TE_OK;
  // the caller's selection back in m->slots (and its host staging in m->sel[0]) for map_out's gather
  if (!whole)
    if (int rc = map_stage_selection(m, sel, memory == TE_MEM_HOST ? 1u : 0u)) return rc;
  const float* const from = lay(m, TE_LAYER_FOOTPRINT);
  return map_out(m, whole ? nullptr : &sel, 1, &from, !whole, &out, memory);
}

// The te_map polygon entries: footprint_polygon_common on the map's resident layers with the map's own state.  They neither read
// nor change the traversability_footprint cache or the memo.
static int map_footprint_polygon(te_map* m, const te_footprint_params* p, int32_t npts, const double* pts_xy, int nouts,
                                 const PolygonOutputs* outs, const te::PolygonReduce* reduce, int memory) {
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  if (memory == TE_MEM_HOST && any_start(m->start.data(), m->nmaps)) {
    // maps with start indices of their own: the sweep writes device staging in default order, then map_out re-wraps every map's
    // block of every output layer (best_yaw moves as 4-byte cells like the float layers)
    Staging st(m->ctx, true, &m->geo);
    const size_t bc = batch_cells(m);
    std::vector<const float*> src;
    std::vector<float*> dst;
    auto stage = [&](float* host, int count) -> float* {
      if (!host) return nullptr;
      float* d = (float*)st.slot(sizeof(float) * bc * count);
      for (int y = 0; d && y < count; ++y) {
        src.push_back(d + y * bc);
        dst.push_back(host + y * bc);
      }
      return d;
    };
    std::vector<PolygonOutputs> dev(outs, outs + nouts);
    for (PolygonOutputs& o : dev) o.out = stage(o.out, o.count);
    te::PolygonReduce red{};
    if (reduce) red = te::PolygonReduce{stage(reduce->worst, 1), stage(reduce->best, 1), (int32_t*)stage((float*)reduce->best_yaw, 1)};
    if (st.rc) return st.rc;
    if (int rc = map_footprint_polygon(m, p, npts, pts_xy, nouts, dev.data(), reduce ? &red : nullptr, TE_MEM_DEVICE)) return rc;
    return map_out(m, nullptr, (int)src.size(), src.data(), false, dst.data(), TE_MEM_HOST);
  }
  const float* in[5];  // trav, slope, step, rough, elev
  if (int rc = map_sweep_inputs(m, p, nullptr, in)) return rc;
  if (m->spread) {
    // Maps at several positions: the sweep classifies the polygon's offsets against absolute positions on the host, so each map
    // is swept on its own geometry (one sweep per map, every output in the batch's layout).  Map m's layers and its layer of
    // each output start m * rows * cols floats in; layer y of a list of yaws is at (y * nmaps + m) * rows * cols.
    const size_t cells = map_cells(m);
    for (int mi = 0; mi < m->nmaps; ++mi) {
      te_geometry g = m->geo;
      g.position_x = m->pos[2 * mi];
      g.position_y = m->pos[2 * mi + 1];
      std::vector<PolygonOutputs> om;
      for (int k = 0; k < nouts; ++k)
        for (int y = 0; y < outs[k].count; ++y)
          om.push_back(PolygonOutputs{outs[k].out ? outs[k].out + (y * (size_t)m->nmaps + mi) * cells : nullptr, 1, outs[k].yaws + y});
      te::PolygonReduce rm{};
      if (reduce)
        rm = te::PolygonReduce{reduce->worst ? reduce->worst + mi * cells : nullptr, reduce->best ? reduce->best + mi * cells : nullptr,
                               reduce->best_yaw ? reduce->best_yaw + mi * cells : nullptr};
      // the reductions run over the yaws of one output: keep it one output of every yaw
      const PolygonOutputs one{nullptr, reduce ? outs[0].count : 0, reduce ? outs[0].yaws : nullptr};
      const size_t o = mi * cells;
      if (int rc = footprint_polygon_common(m->ctx, &m->fp, &g, nullptr, p, 1, npts, pts_xy, in[0] + o, in[1] + o, in[2] + o,
                                            in[3] ? in[3] + o : nullptr, in[4] + o, reduce ? 1 : (int)om.size(), reduce ? &one : om.data(),
                                            reduce ? &rm : nullptr, memory, true))
        return rc;
    }
    return TE_OK;
  }
  const te_geometry g = map_geometry_in(m);
  return footprint_polygon_common(m->ctx, &m->fp, &g, nullptr, p, m->nmaps, npts, pts_xy, in[0], in[1], in[2], in[3], in[4], nouts, outs,
                                  reduce, memory, true);
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

// traversabilityFootprint(footprintYaw) kept on the map: every map (whole) or the maps sel.idx[0..sel.n) of the batch, each at its
// own yaw, swept by one k_poly_tile_maps launch on the resident layers (a selection's gathered into the _maps scratch by one
// k_map_slots launch) straight into the map slots of the resident traversability_x / traversability_rot.  The outputs are copies
// of the swept maps' layers: a whole batch's read back as te_map_get_layers does, a selection's gathered by one more k_map_slots
// launch.
int te_map_footprint_polygon_keep(te_map* m, const te_footprint_params* p, int32_t nsel, const int32_t* map_index, int32_t npts,
                                  const double* pts_xy, int32_t nyaws, const double* yaws, float* out_x, float* out_rot, int memory) {
  TE_MAP_ENTER(m);
  const bool whole = nsel == 0 && !map_index;
  const MapSel sel{nsel, map_index};
  if (int rc = whole ? map_ready(m) : map_select(m, false, nullptr, sel)) return rc;
  if (int rc = map_footprint_params(m, p)) return rc;
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  if (npts < 3 || npts > 16 || !pts_xy) return fail(TE_ERR_BAD_ARG, "footprint polygon needs 3 to 16 vertices");
  for (int k = 0; k < 2 * npts; ++k)
    if (!std::isfinite(pts_xy[k])) return fail(TE_ERR_BAD_ARG, "footprint polygon vertex is not finite");
  const int n = whole ? m->nmaps : sel.n;
  if (!yaws) return fail(TE_ERR_BAD_ARG, "footprint_yaw is null");
  if (nyaws != 1 && nyaws != n) return fail(TE_ERR_BAD_ARG, "%d footprint yaws for %d maps: need 1, or one per swept map", nyaws, n);
  // polygon 0: the identity (traversability_x); polygon 1 + k: the k-th distinct yaw, by bits (traversability_rot)
  std::vector<te::PolygonLayer> polys(1, te::PolygonLayer{0.0, nullptr});
  std::vector<int> poly_of(n);
  std::map<uint64_t, int> index;
  for (int k = 0; k < n; ++k) {
    const double y = yaws[nyaws == 1 ? 0 : k];
    if (!std::isfinite(y)) return fail(TE_ERR_BAD_ARG, "footprint yaw %d is not finite", nyaws == 1 ? 0 : k);
    uint64_t bits;
    std::memcpy(&bits, &y, sizeof bits);
    const auto it = index.emplace(bits, (int)polys.size());
    if (it.second) {
      if (polys.size() > 1024) return fail(TE_ERR_UNSUPPORTED, "more than 1024 distinct footprint yaws: at most 1024 per call");
      polys.push_back(te::PolygonLayer{y, nullptr});
    }
    poly_of[k] = it.first->second;
  }
  te_geometry gm;
  PosTables tab{};
  const bool spread = !map_geometry(m, &gm);  // the maps at several positions: their own tables
  if (spread) gm = m->geo;
  const te_geometry* g = &gm;
  if (int rc = ensure_geometry(c, g)) return rc;
  if (spread)
    if (int rc = map_tables_of(m, MapSel{n, whole ? nullptr : sel.idx}, &tab)) return rc;
  const float* in[5];
  if (int rc = map_sweep_inputs(m, p, whole ? nullptr : &sel, in)) return rc;
  const int fixed = whole ? 0 : 1;  // the selection's k_map_slots
  // the first sweep gives every map of the batch the two layers: the maps it does not sweep hold NaN (0xffffffff)
  const uint32_t kept = TE_LAYER_TRAVERSABILITY_X | TE_LAYER_TRAVERSABILITY_ROT;
  const size_t lbytes = sizeof(float) * batch_cells(m);
  for (const uint32_t b : {(uint32_t)TE_LAYER_TRAVERSABILITY_X, (uint32_t)TE_LAYER_TRAVERSABILITY_ROT}) {
    TE_CUDA(m->layer[__builtin_ctz(b)].reserve(lbytes));
    if (!(m->held & kept) && !whole) TE_CUDA(cudaMemsetAsync(lay(m, b), 0xff, lbytes, c->stream));
  }
  polys[0].out = lay(m, TE_LAYER_TRAVERSABILITY_X);
  for (size_t k = 1; k < polys.size(); ++k) polys[k].out = lay(m, TE_LAYER_TRAVERSABILITY_ROT);
  const te::PolygonMaps pm{poly_of.data(), whole ? nullptr : (const int*)m->slots.p};
  const te_slab s{0, g->cols, 0, 0};
  int nl = 0;
  int rc = te::launch_footprint_polygon(m->fp, view_at(make_view(c, g, s), g, spread ? &tab : nullptr), g, p, npts, pts_xy, (int)polys.size(),
                                        polys.data(), nullptr, &pm, in[0], in[1], in[2], in[3], in[4], n, c->sms, c->stream, &nl);
  if (rc != 0) return fail(rc, "polygon footprint sweep failed: %s", m->fp.why.c_str());
  if (int r2 = launch_check(c, "map polygon footprint", nl + fixed)) return r2;
  m->held |= kept;
  // a selection's host outputs are gathered into sel[0 .. 1], free again once the sweep has read them
  float* const outs[2] = {out_x, out_rot};
  const float* const src[2] = {lay(m, TE_LAYER_TRAVERSABILITY_X), lay(m, TE_LAYER_TRAVERSABILITY_ROT)};
  return map_out(m, whole ? nullptr : &sel, 2, src, true, outs, memory);
}

// The work-list entries launch_map_request_device needs at most for the circular paths of a validated host request: the count of
// req_pose_entries_d with every checkInclination gate counted when the map has robot_slope, so that no path is cut.  It walks no
// line.  *circles: whether the request has a circular path.
// map_pos: the maps' own positions (x, y per map; path q on map path_map[q], or map 0), or null: every map at g's.
static long long map_request_checks(const te_geometry* g, bool rslope, int32_t npaths, const int32_t* path_begin, const double* poses,
                                    const int32_t* footprint_begin, bool* circles, const int32_t* path_map = nullptr,
                                    const double* map_pos = nullptr) {
  te::GridGeo G{g->rows, g->cols, g->resolution, g->length_x, g->length_y, g->position_x, g->position_y};
  long long total = 0;
  *circles = false;
  for (int32_t q = 0; q < npaths; ++q) {
    if (footprint_begin[q + 1] != footprint_begin[q]) continue;  // polygonal
    *circles = true;
    if (map_pos) {
      const int32_t mq = path_map ? path_map[q] : 0;
      G.posx = map_pos[2 * mq];
      G.posy = map_pos[2 * mq + 1];
    }
    const int32_t b = path_begin[q], n = path_begin[q + 1] - b;
    for (int32_t k = n == 1 ? 0 : 1; k < n; ++k) {  // pose 0 of a longer path adds nothing
      const double* e = poses + 7 * (size_t)(b + k);
      int si, sj, ei, ej;
      if (n > 1 && te::grid_get_index(G, e[-7], e[-6], si, sj) && te::grid_get_index(G, e[0], e[1], ei, ej))
        total += (te::LineD(ei, ej, si, sj).n + 3) / 4;  // every fourth LineIterator cell
      else
        total += 1;  // a single pose, or a segment's gate
      if (rslope) total += 1;
    }
  }
  return total;
}

// te_map_check_footprint_request(_batched, _each) in host memory (path_map null: a single map; else checked by the entry) and
// te_map_check_footprint_request_device(_each).  Host memory validates the paths, sizes max_checks so that no path is cut and
// stages the arrays; then both run the same launches, and host memory downloads the outputs.  each: one parameter set per map
// (the _each entries, p null); otherwise p for every map.
static int map_request(te_map* m, const te_footprint_params* p, const te_footprint_params* each, const int32_t* path_map,
                       int32_t npaths, int32_t nposes,
                       const int32_t* path_begin, const double* poses, const double* radius, int32_t nvertices,
                       const int32_t* footprint_begin, const float* footprint_xyz, int32_t max_footprint_vertices,
                       const uint8_t* conservative, const uint8_t* cup, uint8_t* is_safe, double* traversability, double* area,
                       int32_t max_vertices, int32_t* ucount, double* uxy, long long max_checks, int memory) {
  te_ctx* c = m->ctx;
  const bool host = memory == TE_MEM_HOST;
  if (each) {
    for (int k = 0; k < m->nmaps; ++k) {
      if (int rc = map_footprint_params(m, each + k)) return rc;
      if (!(each[k].offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint offset of map %d must be >= 0", k);
    }
  } else {
    if (int rc = map_footprint_params(m, p)) return rc;
    if (!(p->offset >= 0.0)) return fail(TE_ERR_BAD_ARG, "footprint offset must be >= 0");
  }
  if (npaths < 0 || nposes < 0 || nvertices < 0 || !path_begin || !poses || !radius || !footprint_begin ||
      (nvertices > 0 && !footprint_xyz) || !is_safe || !traversability || !area)
    return fail(TE_ERR_BAD_ARG, "null argument or negative count");
  if (max_footprint_vertices < 0 || max_footprint_vertices > te::kPolyMaxVerts)
    return fail(TE_ERR_BAD_ARG, "max_footprint_vertices must be 0..%d, got %d", te::kPolyMaxVerts, max_footprint_vertices);
  if (int rc = check_polygon_outputs(max_vertices, ucount, uxy)) return rc;
  if (!host) {
    if (max_checks < 0) return fail(TE_ERR_BAD_ARG, "max_checks must be >= 0, got %lld", max_checks);
    if (max_checks > (1LL << 30)) return fail(TE_ERR_UNSUPPORTED, "max_checks above 2^30");
  }
  m->last = te::MapRequestStats{};
  m->last_device = false;
  if (npaths == 0) return TE_OK;
  te_geometry gm;
  const bool spread = !map_geometry(m, &gm);  // the maps at several positions: the kernels read each map's tables
  if (spread) gm = m->geo;
  const te_geometry* g = &gm;
  // the hull input bound of a polygonal item: as te_check_footprint_request; host memory sizes it from the paths
  int mp = conservative && max_footprint_vertices > 0 ? 2 * te::kPolyConsCap : 2 * std::max(max_footprint_vertices, 1);
  bool circles = true;  // device memory cannot tell: the circular kernels run and find none
  if (host) {
    if (int rc = check_request_host(g, each ? each : p, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin,
                                    footprint_xyz, max_footprint_vertices, conservative, &mp, each != nullptr, path_map))
      return rc;
    max_checks = map_request_checks(g, m->held & TE_LAYER_ROBOT_SLOPE, npaths, path_begin, poses, footprint_begin, &circles, path_map,
                                    spread ? m->pos.data() : nullptr);
    if (max_checks > (1LL << 30))
      return fail(TE_ERR_UNSUPPORTED, "the circular paths need %lld circle checks, more than 2^30", max_checks);
  }
  if (int rc = ensure_geometry(c, g)) return rc;
  if (int rc = map_memo(m, each ? each : p, each != nullptr)) return rc;
  if (int rc = map_plane(m, each ? each : p, each != nullptr, nullptr)) return rc;
  // maps with parameters of their own: the kernels read each map's from a table (none when they are all one set, p = each[0]);
  // what does not vary per map comes from each[0], and the roughness layer is read when any map verifies roughness
  const te::FpMapParams* table = nullptr;
  te_footprint_params base{};
  if (each) {
    if (int rc = map_param_table(m, each, &table)) return rc;
    base = each[0];
    for (int k = 0; table && k < m->nmaps; ++k) base.verify_roughness |= each[k].verify_roughness != 0;
    p = &base;
  }
  PosTables tab{};
  if (spread)
    if (int rc = map_tables_of(m, MapSel{m->nmaps, nullptr}, &tab)) return rc;
  const te::SlabView v = view_at(make_view(c, g, te_slab{0, g->cols, 0, 0}), g, spread ? &tab : nullptr);
  const float* in[5];  // trav, slope, step, rough, elev
  if (int rc = map_sweep_inputs(m, p, nullptr, in)) return rc;
  te::PathChecks r{};
  r.trav = in[0]; r.slope = in[1]; r.step = in[2]; r.rough = in[3]; r.elev = in[4];
  r.robot_slope = m->held & TE_LAYER_ROBOT_SLOPE ? lay(m, TE_LAYER_ROBOT_SLOPE) : nullptr; r.nmaps = m->nmaps; r.path_map = path_map;
  r.npaths = npaths; r.nposes = nposes; r.path_begin = path_begin; r.poses = poses; r.pose_stride = 7; r.radius = radius;
  r.footprint_begin = footprint_begin; r.footprint_xyz = footprint_xyz; r.nvertices = nvertices;
  r.max_footprint_vertices = max_footprint_vertices; r.conservative = conservative; r.cup = cup; r.max_points = mp;
  r.is_safe = is_safe; r.trav_out = traversability; r.area_out = area; r.max_vertices = max_vertices; r.ucount = ucount; r.uxy = uxy;
  r.map_params = table;
  r.plane = (unsigned char*)m->plane.p;
  Staging st(c, host, g);
  stage_paths(st, r);
  if (st.rc) return st.rc;
  int nl = 0;
  if (nvertices > 0) {  // the polygonal paths (TraversabilityMap.cpp:464-584) read the memo and leave the cache alone
    int rc = te::launch_path_checks(m->fp, v, g, p, r, false, false, c->stream, &nl);
    if (rc != 0) return fail(rc, "map request (polygonal paths) failed: %s", m->fp.why.c_str());
    if (int r2 = launch_check(c, "map request (polygonal paths)", nl)) return r2;
  }
  if (circles) {  // the circular paths (TraversabilityMap.cpp:345-462) in request order on the cache
    int rc = te::launch_map_request_device(m->fp, v, g, p, r, lay(m, TE_LAYER_FOOTPRINT), max_checks, host, c->sms, c->stream, &nl);
    if (rc != 0) return fail(rc, "map request (circular paths) failed: %s", m->fp.why.c_str());
    if (int r2 = launch_check(c, "map request (circular paths)", nl)) return r2;
    m->last_device = true;
  }
  if (int rc = st.finish()) return rc;
  if (host && ucount)  // the row bound of a polygonal path's polygon table (kUntravRows) is only known once the hulls are
    for (int32_t q = 0; q < npaths; ++q)
      if (ucount[q] < 0)
        return fail(TE_ERR_UNSUPPORTED, "the untraversable polygon of path %d spans more than %d map rows", q, te::kUntravRows);
  return TE_OK;
}

int te_map_check_footprint_request(te_map* m, const te_footprint_params* p, int32_t npaths, int32_t nposes, const int32_t* path_begin,
                                   const double* poses, const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                   const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative,
                                   const uint8_t* cup, uint8_t* is_safe, double* traversability, double* area, int32_t max_vertices,
                                   int32_t* ucount, double* uxy) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_single(m, "te_map_check_footprint_request_batched")) return rc;
  return map_request(m, p, nullptr, nullptr, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin, footprint_xyz,
                     max_footprint_vertices, conservative, cup, is_safe, traversability, area, max_vertices, ucount, uxy, 0,
                     TE_MEM_HOST);
}

int te_map_check_footprint_request_batched(te_map* m, const te_footprint_params* p, const int32_t* path_map, int32_t npaths,
                                           int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius,
                                           int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                           int32_t max_footprint_vertices, const uint8_t* conservative, const uint8_t* cup,
                                           uint8_t* is_safe, double* traversability, double* area, int32_t max_vertices, int32_t* ucount,
                                           double* uxy) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!path_map) return fail(TE_ERR_BAD_ARG, "path_map is null");
  if (int rc = check_map_indices(m, path_map, std::max(npaths, 0), "path_map")) return rc;
  return map_request(m, p, nullptr, path_map, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin, footprint_xyz,
                     max_footprint_vertices, conservative, cup, is_safe, traversability, area, max_vertices, ucount, uxy, 0,
                     TE_MEM_HOST);
}

int te_map_check_footprint_request_device(te_map* m, const te_footprint_params* p, const int32_t* path_map, int32_t npaths,
                                          int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius,
                                          int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                          int32_t max_footprint_vertices, const uint8_t* conservative, const uint8_t* cup,
                                          uint8_t* is_safe, double* traversability, double* area, int32_t max_vertices, int32_t* ucount,
                                          double* uxy, int64_t max_checks) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!path_map && m->nmaps > 1) return fail(TE_ERR_BAD_ARG, "path_map is null on a te_map of %d maps", m->nmaps);
  return map_request(m, p, nullptr, path_map, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin, footprint_xyz,
                     max_footprint_vertices, conservative, cup, is_safe, traversability, area, max_vertices, ucount, uxy,
                     (long long)max_checks, TE_MEM_DEVICE);
}

int te_map_check_footprint_request_each(te_map* m, const te_footprint_params* params, const int32_t* path_map, int32_t npaths,
                                        int32_t nposes, const int32_t* path_begin, const double* poses, const double* radius,
                                        int32_t nvertices, const int32_t* footprint_begin, const float* footprint_xyz,
                                        int32_t max_footprint_vertices, const uint8_t* conservative, const uint8_t* cup,
                                        uint8_t* is_safe, double* traversability, double* area, int32_t max_vertices, int32_t* ucount,
                                        double* uxy) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!params) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (!path_map) return fail(TE_ERR_BAD_ARG, "path_map is null");
  if (int rc = check_map_indices(m, path_map, std::max(npaths, 0), "path_map")) return rc;
  return map_request(m, nullptr, params, path_map, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin,
                     footprint_xyz, max_footprint_vertices, conservative, cup, is_safe, traversability, area, max_vertices, ucount,
                     uxy, 0, TE_MEM_HOST);
}

int te_map_check_footprint_request_device_each(te_map* m, const te_footprint_params* params, const int32_t* path_map,
                                               int32_t npaths, int32_t nposes, const int32_t* path_begin, const double* poses,
                                               const double* radius, int32_t nvertices, const int32_t* footprint_begin,
                                               const float* footprint_xyz, int32_t max_footprint_vertices, const uint8_t* conservative,
                                               const uint8_t* cup, uint8_t* is_safe, double* traversability, double* area,
                                               int32_t max_vertices, int32_t* ucount, double* uxy, int64_t max_checks) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!params) return fail(TE_ERR_BAD_ARG, "footprint parameters are null");
  if (!path_map && m->nmaps > 1) return fail(TE_ERR_BAD_ARG, "path_map is null on a te_map of %d maps", m->nmaps);
  return map_request(m, nullptr, params, path_map, npaths, nposes, path_begin, poses, radius, nvertices, footprint_begin,
                     footprint_xyz, max_footprint_vertices, conservative, cup, is_safe, traversability, area, max_vertices, ucount,
                     uxy, (long long)max_checks, TE_MEM_DEVICE);
}

int te_map_get_footprint(te_map* m, float* dst, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!dst) return fail(TE_ERR_BAD_ARG, "output layer is null");
  if (memory != TE_MEM_HOST && (m->geo_in.start_row != 0 || m->geo_in.start_col != 0))
    return fail(TE_ERR_UNSUPPORTED, "the map's layers came with a circular-buffer start index: read its cache into host memory");
  const float* const from = lay(m, TE_LAYER_FOOTPRINT);
  return map_out(m, nullptr, 1, &from, false, &dst, memory);
}

int te_map_get_memo(te_map* m, uint8_t* dst) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!dst) return fail(TE_ERR_BAD_ARG, "output is null");
  if (!m->memo_valid) {  // no request since the layers came: nothing evaluated
    std::memset(dst, 0, batch_cells(m));
    return TE_OK;
  }
  TE_CUDA(cudaMemcpyAsync(dst, m->fp.memo.p, batch_cells(m), cudaMemcpyDeviceToHost, c->stream));
  TE_CUDA(cudaStreamSynchronize(c->stream));
  return TE_OK;
}

int te_map_clear_footprint(te_map* m) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  TE_CUDA(cudaMemsetAsync(lay(m, TE_LAYER_FOOTPRINT), 0xff, sizeof(float) * batch_cells(m), c->stream));
  if (m->plane_valid) {
    m->plane_covers.assign(m->nmaps, 1);  // every cache is empty
    te::launch_plane_clear((unsigned char*)m->plane.p, batch_cells(m), c->sms, c->stream);
    return launch_check(c, "k_plane_clear");
  }
  return TE_OK;
}

int te_map_request_stats(te_map* m, int64_t out[3]) {
  TE_MAP_ENTER(m);
  if (!out) return fail(TE_ERR_BAD_ARG, "null argument");
  if (m->last_device) {  // the counters a device request left on the device
    unsigned long long dev[3];
    TE_CUDA(cudaStreamSynchronize(c->stream));
    TE_CUDA(cudaMemcpy(dev, m->fp.req_counters, sizeof(dev), cudaMemcpyDeviceToHost));
    m->last = te::MapRequestStats{(long long)dev[0], (long long)dev[1], (long long)dev[2]};
    m->last_device = false;
  }
  out[0] = m->last.candidates;
  out[1] = m->last.keys;
  out[2] = m->last.stored;
  return TE_OK;
}

// ---- The read side: GetGridMap submaps, the published layers and mapHasValidTraversabilityAt -----------------------------------
namespace {

// te_submap_geometry's records of `n` windows on the map `g` (its start index changes nothing: te::grid_submap), with offsets for
// `nlayers` layers per window; *total receives the floats they take.  Every window is checked before any record is written.
// map_pos: the position of window k's map is map_pos[2 * win_map[k]], map_pos[... + 1] (null: g's for every window).
int submap_windows(const te_geometry* g, int32_t n, const double* pos, const double* len, int nlayers, te_submap_info* info,
                   int64_t* total, const int32_t* win_map = nullptr, const double* map_pos = nullptr) {
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
    te::GridGeo Ak = A;
    if (map_pos) {
      const int32_t mk = win_map ? win_map[k] : 0;
      Ak.posx = map_pos[2 * mk];
      Ak.posy = map_pos[2 * mk + 1];
    }
    if (te::grid_submap(Ak, pos[2 * k], pos[2 * k + 1], len[2 * k], len[2 * k + 1], s)) {
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

// ---- The update from a larger elevation map: requestElevationMap's getSubmap, then setElevationMap and computeTraversability ----
namespace {

// Validates the source of te_map_chain_submap / _windows into `out` (windows still empty).  Writes nothing.
int cut_source(const te_geometry* src, uint32_t mask, const float* layers[], int memory, CutIn* out) {
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  if (int rc = check_geometry(src, true)) return rc;
  const uint32_t allowed = (uint32_t)TE_LAYER_ELEVATION | (uint32_t)TE_LAYER_CARRIED;
  if (!(mask & TE_LAYER_ELEVATION) || (mask & ~allowed))
    return fail(TE_ERR_BAD_ARG, "source mask 0x%x: need elevation (0x%x) and any of the elevation map's carried layers (0x%x)", mask,
                (unsigned)TE_LAYER_ELEVATION, (unsigned)TE_LAYER_CARRIED);
  if (!layers) return fail(TE_ERR_BAD_ARG, "layers is null");
  out->src = src;
  out->mask = mask;
  out->memory = memory;
  out->nlayers = 0;
  for (int b = 0; b < kLayerBits; ++b) {
    if (!((mask >> b) & 1u)) continue;
    const float* l = layers[out->nlayers];
    if (!l) return fail(TE_ERR_MISSING_LAYER, "layer %s is missing: the source mask names it", kLayerNames[b]);
    out->layers[out->nlayers++] = l;
  }
  return TE_OK;
}

}  // namespace

int te_map_chain_submap(te_map* m, const te_geometry* src, uint32_t src_mask, const float* src_layers[], double position_x,
                        double position_y, double length_x, double length_y, const te_chain_params* p, te_submap_info* info,
                        int memory) {
  TE_MAP_ENTER(m);
  CutIn cut;
  if (int rc = cut_source(src, src_mask, src_layers, memory, &cut)) return rc;
  if (int rc = check_params(p)) return rc;
  if (!info) return fail(TE_ERR_BAD_ARG, "info is null");
  const double pos[2] = {position_x, position_y}, len[2] = {length_x, length_y};
  te_submap_info r{};
  if (int rc = submap_windows(src, 1, pos, len, 1, &r, nullptr)) return rc;
  *info = r;
  if (!r.success)
    return fail(TE_ERR_BAD_ARG, "getSubmap((%g, %g), (%g, %g)) fails on the source map: the te_map is left as it was", position_x,
                position_y, length_x, length_y);
  const te_geometry g{r.rows, r.cols, src->resolution, r.length_x, r.length_y, r.position_x, r.position_y, 0, 0};
  cut.top.push_back(int2{r.top_row, r.top_col});
  return map_chain(m, &g, p, 1, ElevSource{nullptr, nullptr, &cut}, nullptr, nullptr, nullptr, nullptr, memory);
}

int te_map_chain_windows(te_map* m, const te_geometry* g, const te_geometry* src, uint32_t src_mask, const float* src_layers[],
                         int32_t nmaps, const int32_t* map_index, const double* position_xy, const te_chain_params* p, int memory) {
  TE_MAP_ENTER(m);
  CutIn cut;
  if (int rc = cut_source(src, src_mask, src_layers, memory, &cut)) return rc;
  if (int rc = check_geometry(g, true)) return rc;
  if (std::memcmp(&g->resolution, &src->resolution, sizeof(double)) != 0)
    return fail(TE_ERR_BAD_ARG, "resolution %.17g differs from the source's %.17g: windows copy cells, they do not resample", g->resolution,
                src->resolution);
  if (nmaps < 1) return fail(TE_ERR_BAD_ARG, "number of maps must be positive");
  if (!position_xy) return fail(TE_ERR_BAD_ARG, "position_xy is null");
  if (int rc = check_positions(position_xy, nmaps)) return rc;
  // getSubmap's top-left index with the batch's size: floored, so that it may lie outside the source, and within int32
  const te::GridGeo A{src->rows, src->cols, src->resolution, src->length_x, src->length_y, src->position_x, src->position_y};
  std::vector<double> at(2 * (size_t)nmaps);
  cut.top.resize(nmaps);
  for (int32_t k = 0; k < nmaps; ++k) {
    double ti, tj;
    te::grid_window_top(A, position_xy[2 * k] + 0.5 * g->length_x, position_xy[2 * k + 1] + 0.5 * g->length_y, ti, tj);
    if (!(ti >= (double)INT32_MIN && ti + (g->rows - 1) <= (double)INT32_MAX && tj >= (double)INT32_MIN &&
          tj + (g->cols - 1) <= (double)INT32_MAX))
      return fail(TE_ERR_BAD_ARG, "window %d at (%g, %g): its cells' indices on the source do not fit in int32", k, position_xy[2 * k],
                  position_xy[2 * k + 1]);
    cut.top[k] = int2{(int)ti, (int)tj};
    te::grid_window_position(A, (int)ti, (int)tj, g->rows, g->cols, at[2 * k], at[2 * k + 1]);
  }
  if (!map_index) return map_chain(m, g, p, nmaps, ElevSource{nullptr, nullptr, &cut}, nullptr, nullptr, nullptr, nullptr, memory, nullptr,
                                   true, at.data());
  const MapSel sel{nmaps, map_index};
  return map_chain(m, g, p, nmaps, ElevSource{nullptr, nullptr, &cut}, nullptr, nullptr, nullptr, nullptr, memory, &sel, true, at.data());
}

int te_map_get_layers(te_map* m, uint32_t layer_mask, float* out, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  const float* src[kLayerBits];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, true, src, &nl)) return rc;
  if (!out) return fail(TE_ERR_BAD_ARG, "output layer is null");
  // uncertainty_range (a null entry) is computed straight into a device output; in host memory into staging, then copied back
  // with the other layers
  Staging st(c, true, &m->geo);
  float* outs[kLayerBits];
  for (int k = 0; k < nl; ++k) {  // per layer every map, back to back
    outs[k] = out + (size_t)k * batch_cells(m);
    if (src[k]) continue;
    float* d = memory == TE_MEM_HOST ? (float*)st.slot(sizeof(float) * batch_cells(m)) : outs[k];
    if (st.rc) return st.rc;
    te::launch_uncertainty_range(lay(m, TE_LAYER_UPPER_BOUND), lay(m, TE_LAYER_LOWER_BOUND), d, batch_cells(m), c->sms, c->stream);
    if (int rc = launch_check(c, "k_uncertainty_range")) return rc;
    src[k] = d;
    if (memory != TE_MEM_HOST) outs[k] = nullptr;  // already there
  }
  return map_out(m, nullptr, nl, src, false, outs, memory);
}

// te_map_get_submaps (win_map null: map 0) and te_map_get_submaps_batched (window k on map win_map[k], checked by the entry): only
// the source offset of a window's record depends on its map.
static int map_submaps(te_map* m, int32_t nwin, const int32_t* win_map, const double* position_xy, const double* length_xy,
                       uint32_t layer_mask, te_submap_info* info, float* out, int64_t out_capacity, int memory) {
  te_ctx* c = m->ctx;
  const float* src[kLayerBits];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, false, src, &nl)) return rc;
  int64_t total = 0;
  if (int rc = submap_windows(&m->geo, nwin, position_xy, length_xy, nl, info, &total, win_map, m->pos.data())) return rc;
  if (out_capacity < total)
    return fail(TE_ERR_BAD_ARG, "the submaps take %lld floats but out holds %lld: call again with more room", (long long)total,
                (long long)out_capacity);
  if (total == 0) return TE_OK;
  if (!out) return fail(TE_ERR_BAD_ARG, "output is null");
  // the table k_map_gather_submaps reads: the source layers in its first kHead records, then the windows that have cells
  constexpr int kHead = 6;
  static_assert(sizeof(const float*) * (kLayerBits - 2) <= kHead * sizeof(te::SubmapWindow), "layer table");  // not 1 << 7, range
  std::vector<te::SubmapWindow> table(kHead);
  std::memcpy((void*)table.data(), src, sizeof(const float*) * nl);
  long long columns = 0;
  for (int32_t k = 0; k < nwin; ++k) {
    const te_submap_info& r = info[k];
    if (!r.success) continue;
    const long long map0 = win_map ? (long long)win_map[k] * (long long)map_cells(m) : 0;
    table.push_back(te::SubmapWindow{columns, map0 + (long long)r.top_col * m->geo.rows + r.top_row, r.offset, r.rows, r.cols});
    columns += (long long)nl * r.cols;
  }
  const size_t bytes = sizeof(te::SubmapWindow) * table.size();
  if (m->gather.p && m->gather.cap < bytes) TE_CUDA(cudaStreamSynchronize(c->stream));  // an earlier gather may still read it
  TE_CUDA(m->gather.reserve(bytes));
  TE_CUDA(cudaMemcpyAsync(m->gather.p, table.data(), bytes, cudaMemcpyHostToDevice, c->stream));
  Staging st(c, memory == TE_MEM_HOST, &m->geo);  // host memory: gather into staging, then one copy of the packed floats
  float* dout = st.out(out, (size_t)total);
  if (st.rc) return st.rc;
  const te::SubmapGather a{(const float* const*)m->gather.p, (const te::SubmapWindow*)m->gather.p + kHead, (int)table.size() - kHead,
                           m->geo.rows, columns, dout};
  te::launch_gather_submaps(a, c->sms, c->stream);
  if (int rc = launch_check(c, "k_map_gather_submaps")) return rc;
  return st.finish();
}

int te_map_get_submaps(te_map* m, int32_t nwin, const double* position_xy, const double* length_xy, uint32_t layer_mask,
                       te_submap_info* info, float* out, int64_t out_capacity, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_single(m, "te_map_get_submaps_batched")) return rc;
  return map_submaps(m, nwin, nullptr, position_xy, length_xy, layer_mask, info, out, out_capacity, memory);
}

int te_map_get_submaps_batched(te_map* m, int32_t nwin, const int32_t* win_map, const double* position_xy, const double* length_xy,
                               uint32_t layer_mask, te_submap_info* info, float* out, int64_t out_capacity, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = check_map_indices(m, win_map, std::max(nwin, 0), "win_map")) return rc;
  return map_submaps(m, nwin, win_map, position_xy, length_xy, layer_mask, info, out, out_capacity, memory);
}

// te_map_valid_at (pos_map null: map 0) and te_map_valid_at_batched (position q on map pos_map[q], in `memory`).
static int map_valid_at(te_map* m, int32_t n, const int32_t* pos_map, const double* xy, uint8_t* valid, int memory) {
  te_ctx* c = m->ctx;
  if (n < 0) return fail(TE_ERR_BAD_ARG, "negative position count");
  if (n == 0) return TE_OK;
  if (!xy || !valid) return fail(TE_ERR_BAD_ARG, "null argument");
  Staging st(c, memory == TE_MEM_HOST, &m->geo);
  const double* dxy = st.in(xy, 2 * (size_t)n);
  const int32_t* dmap = st.in(pos_map, (size_t)n);
  uint8_t* dvalid = st.out(valid, (size_t)n);
  if (st.rc) return st.rc;
  te_geometry g;
  PosTables tab{};
  const bool spread = !map_geometry(m, &g);  // the maps at several positions: the kernel takes each map's
  if (spread) {
    g = m->geo;
    if (int rc = map_tables_of(m, MapSel{m->nmaps, nullptr}, &tab)) return rc;
  }
  te::launch_valid_at(te::GridGeo{g.rows, g.cols, g.resolution, g.length_x, g.length_y, g.position_x, g.position_y},
                      lay(m, TE_LAYER_TRAVERSABILITY), n, dxy, dmap, m->nmaps, spread ? tab.pos : nullptr, dvalid, c->stream);
  if (int rc = launch_check(c, "k_map_valid_at")) return rc;
  return st.finish();
}

int te_map_valid_at(te_map* m, int32_t n, const double* xy, uint8_t* valid, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (int rc = map_single(m, "te_map_valid_at_batched")) return rc;
  return map_valid_at(m, n, nullptr, xy, valid, memory);
}

int te_map_valid_at_batched(te_map* m, int32_t n, const int32_t* pos_map, const double* xy, uint8_t* valid, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (n > 0 && !pos_map) return fail(TE_ERR_BAD_ARG, "pos_map is null");
  if (memory == TE_MEM_HOST)  // device memory cannot be read here: the kernel gives 0 for a map outside the batch
    if (int rc = check_map_indices(m, pos_map, std::max(n, 0), "pos_map")) return rc;
  return map_valid_at(m, n, pos_map, xy, valid, memory);
}

int te_map_at_poses(te_map* m, const int32_t* pose_map, int32_t nposes, const double* poses, int32_t npoints, const float* points_xyz,
                    uint32_t layer_mask, float* out, uint8_t* valid, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (!poses || !points_xyz || !out) return fail(TE_ERR_BAD_ARG, "poses, points_xyz or out is null");
  if (nposes < 0) return fail(TE_ERR_BAD_ARG, "negative pose count");
  if (npoints < 1) return fail(TE_ERR_BAD_ARG, "need at least one point, got %d", npoints);
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  if (!pose_map && m->nmaps > 1) return fail(TE_ERR_BAD_ARG, "pose_map is null on a te_map of %d maps", m->nmaps);
  // device memory cannot be read here: the kernel gives NaN and valid 0 for a map outside the batch
  if (pose_map && memory == TE_MEM_HOST)
    if (int rc = check_map_indices(m, pose_map, nposes, "pose_map")) return rc;
  const float* src[kLayerBits];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, true, src, &nl)) return rc;
  const long long total = (long long)nposes * npoints;
  if (total >= (1LL << 31)) return fail(TE_ERR_UNSUPPORTED, "%d poses x %d points: 2^31 samples or more", nposes, npoints);
  if (total == 0) return TE_OK;
  te::MapAtPoses a{};
  a.range_l = -1;
  for (int l = 0; l < nl; ++l) {
    if (src[l]) {
      a.layer[l] = src[l];
    } else {  // uncertainty_range: upper_bound - lower_bound at the cell, as te_map_get_layers computes it
      a.layer[l] = lay(m, TE_LAYER_UPPER_BOUND);
      a.lower = lay(m, TE_LAYER_LOWER_BOUND);
      a.range_l = l;
    }
  }
  a.nlayers = nl;
  Staging st(c, memory == TE_MEM_HOST, &m->geo);
  a.poses = st.in(poses, 7 * (size_t)nposes);
  a.pose_map = st.in(pose_map, (size_t)nposes);
  a.points = st.in(points_xyz, 3 * (size_t)npoints);
  a.out = st.out(out, (size_t)nl * total);
  a.valid = st.out(valid, (size_t)total);
  if (st.rc) return st.rc;
  te_geometry g;
  PosTables tab{};
  if (!map_geometry(m, &g)) {  // the maps at several positions: the kernel takes each map's
    g = m->geo;
    if (int rc = map_tables_of(m, MapSel{m->nmaps, nullptr}, &tab)) return rc;
    a.map_pos = tab.pos;
  }
  a.rows = g.rows; a.cols = g.cols; a.nmaps = m->nmaps; a.nposes = nposes; a.npoints = npoints;
  a.res = g.resolution; a.lenx = g.length_x; a.leny = g.length_y; a.posx = g.position_x; a.posy = g.position_y;
  te::launch_map_at_poses(a, c->sms, c->stream);
  if (int rc = launch_check(c, "k_map_at_poses")) return rc;
  return st.finish();  // host memory: returns synchronised
}

int te_occupancy_grid_info(const te_geometry* g, int32_t n, const double* position_xy, te_occupancy_info* out) {
  if (int rc = check_geometry(g, true)) return rc;
  if (n < 0) return fail(TE_ERR_BAD_ARG, "negative record count");
  if (n == 0) return TE_OK;
  if (!out) return fail(TE_ERR_BAD_ARG, "out is null");
  if (position_xy) {
    if (int rc = check_positions(position_xy, n)) return rc;
  } else if (!std::isfinite(g->position_x) || !std::isfinite(g->position_y)) {
    return fail(TE_ERR_BAD_ARG, "the geometry's position is not finite");
  }
  for (int32_t k = 0; k < n; ++k) {  // MapMetaData: origin = getPosition() - 0.5 * getLength(), per axis in double
    const double px = position_xy ? position_xy[2 * k] : g->position_x, py = position_xy ? position_xy[2 * k + 1] : g->position_y;
    out[k] = te_occupancy_info{g->rows, g->cols, (float)g->resolution, 0, px - 0.5 * g->length_x, py - 0.5 * g->length_y};
  }
  return TE_OK;
}

int te_map_get_occupancy(te_map* m, int32_t nsel, const int32_t* map_index, uint32_t layer_mask, const float* data_min,
                         const float* data_max, int8_t* out, int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  const float* src[kLayerBits];
  int nl = 0;
  if (int rc = map_layers(m, layer_mask, true, src, &nl)) return rc;
  if (!data_min || !data_max || !out) return fail(TE_ERR_BAD_ARG, "data_min, data_max or out is null");
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  const bool whole = nsel == 0 && !map_index;
  // the grids never depend on a start index (toOccupancyGrid walks the unwrapped index), so any te_map takes a selection
  if (!whole)
    if (int rc = check_selection(m, MapSel{nsel, map_index})) return rc;
  te::MapOccupancy a{};
  a.range_l = -1;
  for (int l = 0; l < nl; ++l) {
    if (src[l]) {
      a.layer[l] = src[l];
    } else {  // uncertainty_range: upper_bound - lower_bound per cell, as te_map_get_layers computes it
      a.layer[l] = lay(m, TE_LAYER_UPPER_BOUND);
      a.lower = lay(m, TE_LAYER_LOWER_BOUND);
      a.range_l = l;
    }
    a.data_min[l] = data_min[l];
    a.data_max[l] = data_max[l];
  }
  a.nlayers = nl;
  a.nmaps = whole ? m->nmaps : nsel;
  a.cells = (long long)map_cells(m);
  if (!whole) {  // the slot table of the _maps entries
    if (int rc = map_stage_selection(m, MapSel{nsel, map_index}, 0)) return rc;
    a.slot = (const int*)m->slots.p;
  }
  Staging st(c, memory == TE_MEM_HOST, &m->geo);  // host memory: the grids into staging, then one copy back
  a.out = (unsigned char*)st.out(out, (size_t)nl * a.nmaps * a.cells);
  if (st.rc) return st.rc;
  te::launch_map_occupancy(a, c->sms, c->stream);
  if (int rc = launch_check(c, "k_map_occupancy")) return rc;
  return st.finish();  // host memory: returns synchronised
}

namespace {

// The device copy of a call's per-map table t, uploaded only when it differs from what the buffer holds; growing it first waits for
// the launches that may still read it.
int cloud_table(te_map* m, te_map::CloudTab& t, const std::vector<te::CloudMap>& v, const te::CloudMap** out) {
  const size_t bytes = sizeof(te::CloudMap) * v.size();
  if (t.key.size() != v.size() || std::memcmp(t.key.data(), v.data(), bytes) != 0) {
    if (t.buf.p && t.buf.cap < bytes) TE_CUDA(cudaStreamSynchronize(m->ctx->stream));
    TE_CUDA(t.buf.reserve(bytes));
    t.key = v;  // pageable: consumed before cudaMemcpyAsync returns
    TE_CUDA(cudaMemcpyAsync(t.buf.p, t.key.data(), bytes, cudaMemcpyHostToDevice, m->ctx->stream));
  }
  *out = (const te::CloudMap*)t.buf.p;
  return TE_OK;
}

}  // namespace

int te_map_get_point_cloud(te_map* m, int32_t nsel, const int32_t* map_index, int32_t nfields, const uint32_t* fields,
                           uint32_t point_layer, uint32_t basic_mask, void* data, int64_t capacity_points, int64_t* offsets,
                           int memory) {
  TE_MAP_ENTER(m);
  if (int rc = map_ready(m)) return rc;
  if (nfields < 1 || nfields > te::kCloudMaxFields) return fail(TE_ERR_BAD_ARG, "nfields = %d: need 1..%d", nfields, te::kCloudMaxFields);
  if (!fields || !offsets) return fail(TE_ERR_BAD_ARG, "fields or offsets is null");
  if (capacity_points < 0) return fail(TE_ERR_BAD_ARG, "negative capacity_points");
  if (!data && capacity_points > 0) return fail(TE_ERR_BAD_ARG, "data is null with capacity_points %lld", (long long)capacity_points);
  const uint32_t known = TE_LAYER_ALL | TE_LAYER_CARRIED | TE_LAYER_UNCERTAINTY_RANGE | TE_LAYER_TRAVERSABILITY_X | TE_LAYER_TRAVERSABILITY_ROT |
                         TE_LAYER_FOOTPRINT_MEMO;
  const auto one_bit = [&](uint32_t b) { return b != 0 && (b & (b - 1)) == 0 && (b & known) != 0; };
  uint32_t given = 0;
  for (int e = 0; e < nfields; ++e) {
    const uint32_t f = fields[e];
    if (f == 0) continue;
    if (!one_bit(f)) return fail(TE_ERR_BAD_ARG, "fields[%d] = 0x%x: need 0 (a NaN field) or one te_layer bit", e, f);
    if (given & f) return fail(TE_ERR_BAD_ARG, "fields[%d] = 0x%x appears twice", e, f);
    given |= f;
  }
  if (!one_bit(point_layer)) return fail(TE_ERR_BAD_ARG, "point_layer 0x%x: need one te_layer bit", point_layer);
  if (basic_mask & ~known) return fail(TE_ERR_BAD_ARG, "basic_mask 0x%x has bits outside 0x%x", basic_mask, known);
  if (memory != TE_MEM_HOST && memory != TE_MEM_DEVICE) return fail(TE_ERR_BAD_ARG, "unknown memory mode %d", memory);
  const bool whole = nsel == 0 && !map_index;
  if (!whole)
    if (int rc = check_selection(m, MapSel{nsel, map_index})) return rc;
  const float* held_src[kLayerBits];
  int nl = 0;
  if (int rc = map_layers(m, given | point_layer | basic_mask, true, held_src, &nl)) return rc;  // TE_ERR_MISSING_LAYER

  // uncertainty_range reads upper_bound and subtracts lower_bound
  const auto src = [&](uint32_t bit) { return bit == TE_LAYER_UNCERTAINTY_RANGE ? lay(m, TE_LAYER_UPPER_BOUND) : lay(m, bit); };
  te::MapCloud a{};
  a.point_e = -1;
  for (int e = 0; e < nfields; ++e) {
    if (fields[e] == point_layer) a.point_e = e;
    else if (fields[e]) a.field[e] = src(fields[e]);
    if (fields[e] == TE_LAYER_UNCERTAINTY_RANGE) a.field_range |= 1u << e;
  }
  a.nfields = nfields;
  a.point = src(point_layer);
  if (point_layer == TE_LAYER_UNCERTAINTY_RANGE) a.basic_range |= 1u << 31;
  for (int b = 0; b < kLayerBits; ++b) {
    if (!((basic_mask >> b) & 1u)) continue;
    if (b == 15) a.basic_range |= 1u << a.nbasic;
    a.basic[a.nbasic++] = src(1u << b);
  }
  if (((given | point_layer | basic_mask) & TE_LAYER_UNCERTAINTY_RANGE)) a.lower = lay(m, TE_LAYER_LOWER_BOUND);
  a.point_step = 4 * (nfields + (a.point_e >= 0 ? 2 : 0));

  // each map's slot, start index (a single map's may have come in g) and position
  const int n = whole ? m->nmaps : nsel;
  const te_geometry& g = m->geo;
  std::vector<te::CloudMap> maps(n);
  for (int k = 0; k < n; ++k) {
    const int s = whole ? k : map_index[k];
    const bool in_g = m->geo_in.start_row != 0 || m->geo_in.start_col != 0;
    const bool at = !m->pos.empty();
    maps[k] = te::CloudMap{s, in_g ? m->geo_in.start_row : m->start[2 * s], in_g ? m->geo_in.start_col : m->start[2 * s + 1], 0,
                           at ? m->pos[2 * s] : g.position_x, at ? m->pos[2 * s + 1] : g.position_y};
  }
  bool uniform = whole;  // a whole batch with one start index and position takes them by value
  for (int k = 1; k < n && uniform; ++k)
    uniform = maps[k].sr == maps[0].sr && maps[k].sc == maps[0].sc && std::memcmp(&maps[k].px, &maps[0].px, 2 * sizeof(double)) == 0;
  if (uniform) {
    a.sr = maps[0].sr; a.sc = maps[0].sc; a.px = maps[0].px; a.py = maps[0].py;
  } else if (int rc = cloud_table(m, whole ? m->cloud_all : m->cloud_sel, maps, &a.maps)) {
    return rc;
  }
  a.rows = g.rows; a.cols = g.cols; a.nmaps = n; a.cells = (long long)map_cells(m);
  a.lenx = g.length_x; a.leny = g.length_y; a.res = g.resolution;
  a.tiles = (int)((a.cells + te::kCloudTile - 1) / te::kCloudTile);

  // scratch: the counts, their prefix sums, the scan's temporary storage
  const long long nt = (long long)n * a.tiles + 1;
  const size_t cbytes = (sizeof(unsigned long long) * nt + 255) / 256 * 256, tmp_bytes = te::map_cloud_scan_bytes(nt);
  if (m->cloud.p && m->cloud.cap < 2 * cbytes + tmp_bytes) TE_CUDA(cudaStreamSynchronize(c->stream));
  TE_CUDA(m->cloud.reserve(2 * cbytes + tmp_bytes));
  a.count = (unsigned long long*)m->cloud.p;
  a.first = (unsigned long long*)((char*)m->cloud.p + cbytes);
  TE_CUDA(te::launch_map_cloud_count(a, (char*)m->cloud.p + 2 * cbytes, tmp_bytes, c->sms, c->stream));
  if (int rc = launch_check(c, "k_map_cloud_count, DeviceScan", 2)) return rc;
  // offsets[k] = the first point of map k's first tile; offsets[n] = the total (the entry after the last tile).  Host memory
  // copies them back before the scatter; in device memory the scatter kernel writes them.
  const bool host = memory == TE_MEM_HOST;
  a.capacity = capacity_points;
  a.out = (unsigned char*)data;
  a.offsets = host ? nullptr : (long long*)offsets;
  Staging st(c, host, &g);  // host memory: the records into staging, then one copy of total * point_step bytes
  if (host) {
    TE_CUDA(cudaMemcpy2DAsync(offsets, sizeof(int64_t), a.first, sizeof(int64_t) * a.tiles, sizeof(int64_t), n + 1,
                              cudaMemcpyDeviceToHost, c->stream));
    TE_CUDA(cudaStreamSynchronize(c->stream));
    if (offsets[n] > capacity_points)
      return fail(TE_ERR_BAD_ARG, "the clouds hold %lld points but data has room for %lld: call again with more room",
                  (long long)offsets[n], (long long)capacity_points);
    a.capacity = offsets[n];
    a.out = st.out((uint8_t*)data, (size_t)offsets[n] * a.point_step);
    if (st.rc) return st.rc;
  }
  te::launch_map_cloud_scatter(a, c->sms, c->stream);
  if (int rc = launch_check(c, "k_map_cloud_scatter")) return rc;
  return st.finish();  // host memory: returns synchronised
}
