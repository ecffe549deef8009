/*
 * map_oracle.cpp — CPU ORACLE of te_map (test infrastructure, NOT product code).
 *
 * A sequential restatement of the reference's check_footprint_path service loop (TraversabilityEstimation.cpp:278-295, with
 * publishPolygons = true) on a TraversabilityMap whose traversability_footprint layer persists: the caller passes the cache in and
 * gets it back (float32, NaN = empty), and the paths of a request run one after another in request order.  Circular paths restate
 * checkCircularFootprintPath (traversability_estimation/src/TraversabilityMap.cpp:345-462) with isTraversable(center, ...) :654-746
 * as untraversable_oracle.cpp does, with its per-path std::map cache replaced by the persistent layer.  Polygonal paths keep no
 * cache: each one is teo_check_polygonal_paths2 on its own.  teo_map_footprint restates traversabilityFootprint(radius, offset)
 * (:307-318) on the layer: a cell whose value is finite takes the memoised branch and keeps it, every other cell walks its spiral.
 *
 * PARITY UNPINNED like the rest of the footprint oracle.  Literal IEEE double; build with -ffp-contract=off.
 */
#include "untraversable_oracle.cpp"

namespace {

// isTraversable(center, radiusMax, cup, traversability, untraversablePolygon, radiusMin), :654-746, on the layer `cache`.
bool is_traversable(const Map& m, const teo_footprint_params& p, const std::vector<unsigned char>& blocked, const SpiralOffsets& sp,
                    float* cache, V2 center, double radiusMax, bool cup, double& t, std::vector<V2>& untraversablePolygon,
                    double radiusMin) {
  bool circleIsTraversable = true;
  std::vector<V2> untraversablePositions;
  untraversablePolygon.clear();                                              // :659
  if (!is_inside(m, center)) {                                               // :662-667
    t = p.traversability_default;
    circleIsTraversable = p.traversability_default != 0.0;
    if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
    return circleIsTraversable;
  }
  int ci, cj;
  get_index(m, center, ci, cj);
  const size_t indexCenter = (size_t)cj * m.rows + ci;
  if (std::isfinite(cache[indexCenter])) {                                   // :673-678
    t = cache[indexCenter];
    circleIsTraversable = t != 0.0;
    if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
    return circleIsTraversable;
  }
  int nCells = 0;
  t = 0.0;
  bool traversableRadiusBiggerMinRadius = false;
  const double r2 = radiusMax * radiusMax;
  for (size_t k = 0; k < sp.di.size() && !traversableRadiusBiggerMinRadius; ++k) {  // :687-688
    const int a = ci + sp.di[k], c = cj + sp.dj[k];
    if (a < 0 || c < 0 || a >= m.rows || c >= m.cols) continue;
    if (sp.edge[k]) {
      const double dx = m.X[a] - center.x, dy = m.Y[c] - center.y;
      if (!(dx * dx + dy * dy <= r2)) continue;
    }
    const size_t cell = (size_t)c * m.rows + a;
    if (blocked[cell]) {                                                     // :689-690
      const int ddi = sp.di[k], ddj = sp.dj[k];
      const double untraversableRadius = p.radius_is_integer_norm ? (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res
                                                                  : std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
      if (radiusMin == 0.0 || untraversableRadius <= radiusMin) {            // :694-704
        cache[indexCenter] = 0.0f;
        circleIsTraversable = false;
        untraversablePositions.push_back(V2{m.X[a], m.Y[c]});
      } else if (circleIsTraversable) {                                      // :705-711
        const double factor = ((untraversableRadius - radiusMin) / (radiusMax - radiusMin) + 1.0) / 2.0;
        t *= factor / nCells;
        cache[indexCenter] = static_cast<float>(t);
        circleIsTraversable = true;
        traversableRadiusBiggerMinRadius = true;
      }
      if (!cup) return false;                                                // :714-717
    } else {
      nCells++;
      const float v = m.trav[cell];
      t += std::isfinite(v) ? (double)v : p.traversability_default;
    }
  }
  if (cup && !circleIsTraversable) untraversablePolygon = monotone_chain(untraversablePositions);  // :728-730
  if (circleIsTraversable) {                                                 // :732-735
    t /= nCells;
    cache[indexCenter] = static_cast<float>(t);
  }
  return circleIsTraversable;
}

Map make_map(const teo_geometry* g, const float* trav, const float* slope, const float* step, const float* elev) {
  Map m{g->rows, g->cols, g->resolution, {g->length_x, g->length_y}, {g->position_x, g->position_y}, trav, slope, step, elev, {}, {}};
  m.X.resize(m.rows);
  m.Y.resize(m.cols);
  for (int i = 0; i < m.rows; ++i) m.X[i] = cell_coord(m.pos.x, m.len.x, m.res, i);
  for (int j = 0; j < m.cols; ++j) m.Y[j] = cell_coord(m.pos.y, m.len.y, m.res, j);
  return m;
}

}  // namespace

// One request; poses are 7 doubles per pose, path q's footprint is footprint_xyz rows footprint_begin[q] .. footprint_begin[q+1]-1
// (none: circular).  `cache` (rows x cols, column-major) is read and updated.
extern "C" int teo_map_check_request(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                     const float* step, const float* rough, const float* elev, const float* robot_slope, int npaths,
                                     const int32_t* path_begin, const double* poses, const double* radius, const int32_t* footprint_begin,
                                     const float* footprint_xyz, const uint8_t* conservative_or_null, const uint8_t* cup_or_null,
                                     float* cache, uint8_t* is_safe, double* traversability, double* area, int max_vertices,
                                     int32_t* count, double* xy) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || npaths < 0 ||
      !path_begin || !poses || !radius || !footprint_begin || !cache || !is_safe || !traversability || !area || max_vertices < 0 ||
      !count || (max_vertices > 0 && !xy))
    return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = make_map(g, trav, slope, step, elev);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, 1);
  const double offset = p->offset;

  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], arraySize = path_begin[q + 1] - b;
    const int nfp = footprint_begin[q + 1] - footprint_begin[q];
    if (nfp > 0) {  // checkPolygonalFootprintPath: no cache
      const int32_t pb[2] = {0, arraySize};
      const uint8_t cons = conservative_or_null ? conservative_or_null[q] : 0, cup = cup_or_null ? cup_or_null[q] : 0;
      if (teo_check_polygonal_paths2(g, p, trav, slope, step, rough, elev, robot_slope, nfp, footprint_xyz + 3 * (size_t)footprint_begin[q],
                                     1, pb, poses + 7 * (size_t)b, &cons, is_safe + q, traversability + q, area + q, &cup, max_vertices,
                                     count + q, xy + 2 * (size_t)max_vertices * q))
        return 1;
      continue;
    }
    area[q] = 0.0;
    is_safe[q] = 0;
    traversability[q] = 0.0;
    std::vector<V2> published;
    auto publishUntraversablePolygon = [&](const std::vector<V2>& poly) {   // :928-938
      if (!poly.empty()) published = poly;
    };
    const double pathRadius = radius[q];
    const bool computeUntraversablePolygon = cup_or_null && cup_or_null[q];
    const SpiralOffsets sp = spiral_offsets(pathRadius + offset, m.res);
    auto checkInclination = [&](V2 start, V2 end) -> bool {                 // :748-762
      if (!robot_slope) return true;
      if (end.x == start.x && end.y == start.y) {
        int i, j;
        if (!is_inside(m, start) || !get_index(m, start, i, j)) return false;
        return !(robot_slope[(size_t)j * m.rows + i] == 0.0f);
      }
      int si, sj, ei, ej;
      if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) return false;
      bool ok = true;
      for_line(si, sj, ei, ej, [&](int a, int c) {
        const float v = robot_slope[(size_t)c * m.rows + a];
        if (!std::isfinite(v)) return true;
        if (v == 0.0f) { ok = false; return false; }
        return true;
      });
      return ok;
    };
    double result = 0.0, lengthPath = 0.0;
    bool safe = arraySize > 0;
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    std::vector<V2> untraversablePolygon;
    for (int i = 0; i < arraySize && safe; i++) {
      start = end;
      end = V2{poses[7 * (size_t)(b + i)], poses[7 * (size_t)(b + i) + 1]};
      if (arraySize == 1) {
        if (!checkInclination(end, end)) { safe = false; break; }
        double t;
        const bool ok = is_traversable(m, *p, blocked, sp, cache, end, pathRadius + offset, computeUntraversablePolygon, t,
                                       untraversablePolygon, pathRadius);
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);
        if (!ok) { safe = false; break; }
        result = t;
      }
      if (arraySize > 1 && i > 0) {
        if (!checkInclination(start, end)) { safe = false; break; }
        double traversabilityTemp = 0.0, traversabilitySum = 0.0;
        int nLine = 0;
        int si, sj, ei, ej;
        if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) { safe = false; break; }
        std::vector<V2> auxiliaryUntraversablePolygon;
        bool pathIsTraversable = true;
        int visit = 0;
        for_line(ei, ej, si, sj, [&](int a, int c) {
          if ((visit++ & 3) != 0) return true;
          const V2 center{m.X[a], m.Y[c]};
          pathIsTraversable = pathIsTraversable && is_traversable(m, *p, blocked, sp, cache, center, pathRadius + offset,
                                                                  computeUntraversablePolygon, traversabilityTemp,
                                                                  auxiliaryUntraversablePolygon, pathRadius);
          if (computeUntraversablePolygon && !auxiliaryUntraversablePolygon.empty())
            untraversablePolygon = convex_hull(untraversablePolygon, auxiliaryUntraversablePolygon);
          traversabilitySum += traversabilityTemp;
          nLine++;
          return true;
        });
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);
        if (pathIsTraversable) {
          const double t = traversabilitySum / (double)nLine;
          const double lengthSegment = std::sqrt((end.x - start.x) * (end.x - start.x) + (end.y - start.y) * (end.y - start.y));
          if (i > 1) {
            const double lengthPreviousPath = lengthPath;
            lengthPath += lengthSegment;
            result = (lengthSegment * t + lengthPreviousPath * result) / lengthPath;
          } else {
            lengthPath = lengthSegment;
            result = t;
          }
        } else {
          safe = false;
        }
      }
    }
    count[q] = (int32_t)published.size();
    for (int v = 0; v < (int)published.size() && v < max_vertices; ++v) {
      xy[2 * ((size_t)max_vertices * q + v)] = published[v].x;
      xy[2 * ((size_t)max_vertices * q + v) + 1] = published[v].y;
    }
    if (!safe) continue;
    is_safe[q] = 1;
    traversability[q] = result;
  }
  return 0;
}

// traversabilityFootprint(radius, offset) (:307-318) on `cache`: every cell's isTraversable(centre, radius + offset, ..., radius).
extern "C" int teo_map_footprint(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                 const float* step, const float* rough, const float* elev, float* cache) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !p || !trav || !slope || !step || !elev || !cache) return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = make_map(g, trav, slope, step, elev);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, 1);
  const SpiralOffsets sp = spiral_offsets(p->radius + p->offset, m.res);
  std::vector<V2> none;
  for (int j = 0; j < m.cols; ++j)
    for (int i = 0; i < m.rows; ++i) {
      double t;
      is_traversable(m, *p, blocked, sp, cache, V2{m.X[i], m.Y[j]}, p->radius + p->offset, false, t, none, p->radius);
    }
  return 0;
}
