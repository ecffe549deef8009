/*
 * memo_layers_oracle.cpp — CPU ORACLE of the slope_footprint / step_footprint / roughness_footprint layers a te_map records (test
 * infrastructure, NOT product code).
 *
 * The reference's checkForSlope / checkForStep / checkForRoughness (TraversabilityMap.cpp:794-921) write 0 or 1 into these layers
 * at a cell they visit whose own input layer is exactly 0, and isTraversableForFilters (:774-792) runs the step check only after
 * the slope check passed and the roughness check only after both.  What a check writes is a function of the cell and the layers,
 * so this oracle keeps the values compute_blocked gives for every cell and copies them into the three layers at every cell the
 * reference visits, in the reference's order and with its early returns:
 *   - teo_memo_request: one check_footprint_path request on a persistent traversability_footprint layer, paths one after another
 *     (TraversabilityEstimation.cpp:278-295): checkCircularFootprintPath (circular_footprint_path of the footprint oracle) with
 *     isTraversable(center, ...) :654-746, and checkPolygonalFootprintPath :464-584 with isTraversable(polygon, ...) :592-645;
 *   - teo_memo_sweep: traversabilityFootprint(radius, offset) :307-318 on that layer.
 * The request restates the walks of paths_oracle.cpp (included: its geometry helpers and polygon pieces) with the visits added.
 * Build with -ffp-contract=off.
 */
#include "paths_oracle.cpp"

namespace {

struct Recorder {
  const float* s;  // per cell: what each check writes when it visits the cell (NaN: nothing)
  const float* t;
  const float* r;
  float* so;       // the three layers
  float* to;
  float* ro;
  void visit(size_t c) const {
    if (!std::isnan(s[c])) so[c] = s[c];
    if (!std::isnan(t[c])) to[c] = t[c];
    if (!std::isnan(r[c])) ro[c] = r[c];
  }
};

struct RecChecker {
  const Map& m;
  const teo_footprint_params& p;
  const std::vector<unsigned char>& blocked;
  const float* robot_slope;
  const Recorder& rec;

  // isTraversable(center, radiusMax, cup, traversability, untraversablePolygon, radiusMin), :654-746, on `cache`.
  bool circle_traversable(float* cache, const SpiralOffsets& sp, V2 center, double radiusMax, bool cup, double& t,
                          Polygon& untraversablePolygon, double radiusMin) const {
    bool circleIsTraversable = true;
    Polygon untraversablePositions;
    untraversablePolygon.clear();
    if (!is_inside(m, center)) {                                                       // :662-667
      t = p.traversability_default;
      circleIsTraversable = p.traversability_default != 0.0;
      if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
      return circleIsTraversable;
    }
    int ci, cj;
    get_index(m, center, ci, cj);
    const size_t indexCenter = (size_t)cj * m.rows + ci;
    if (std::isfinite(cache[indexCenter])) {                                           // :673-678
      t = cache[indexCenter];
      circleIsTraversable = t != 0.0;
      if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
      return circleIsTraversable;
    }
    int nCells = 0;
    t = 0.0;
    bool traversableRadiusBiggerMinRadius = false;
    const double r2 = radiusMax * radiusMax;
    for (size_t k = 0; k < sp.di.size() && !traversableRadiusBiggerMinRadius; ++k) {   // :687-688
      const int a = ci + sp.di[k], c = cj + sp.dj[k];
      if (a < 0 || c < 0 || a >= m.rows || c >= m.cols) continue;
      if (sp.edge[k]) {
        const double dx = m.X[a] - center.x, dy = m.Y[c] - center.y;
        if (!(dx * dx + dy * dy <= r2)) continue;
      }
      const size_t cell = (size_t)c * m.rows + a;
      rec.visit(cell);                                                                 // :689 isTraversableForFilters
      if (blocked[cell]) {
        const int ddi = sp.di[k], ddj = sp.dj[k];
        const double untraversableRadius = p.radius_is_integer_norm
            ? (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res
            : std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
        if (radiusMin == 0.0 || untraversableRadius <= radiusMin) {                    // :694-704
          cache[indexCenter] = 0.0f;
          circleIsTraversable = false;
          untraversablePositions.push_back(V2{m.X[a], m.Y[c]});
        } else if (circleIsTraversable) {                                              // :705-711
          const double factor = ((untraversableRadius - radiusMin) / (radiusMax - radiusMin) + 1.0) / 2.0;
          t *= factor / nCells;
          cache[indexCenter] = static_cast<float>(t);
          circleIsTraversable = true;
          traversableRadiusBiggerMinRadius = true;
        }
        if (!cup) return false;                                                        // :714-717
      } else {
        nCells++;
        const float v = m.trav[cell];
        t += std::isfinite(v) ? (double)v : p.traversability_default;
      }
    }
    if (cup && !circleIsTraversable) untraversablePolygon = monotone_chain(untraversablePositions);
    if (circleIsTraversable) {
      t /= nCells;
      cache[indexCenter] = static_cast<float>(t);
    }
    return circleIsTraversable;
  }

  // The cells isTraversable(polygon, cup, ...) visits, :592-645 (PolygonIterator as in paths_oracle.cpp).  Returns its verdict.
  bool polygon_traversable(const Polygon& poly, bool cup) const {
    unsigned nCells = 0;
    bool pathIsTraversable = true;
    V2 topLeft = poly.empty() ? V2{0.0, 0.0} : poly[0], bottomRight = topLeft;
    for (const V2& q : poly) {
      topLeft = V2{std::max(topLeft.x, q.x), std::max(topLeft.y, q.y)};
      bottomRight = V2{std::min(bottomRight.x, q.x), std::min(bottomRight.y, q.y)};
    }
    bound_position(m, topLeft);
    bound_position(m, bottomRight);
    int si, sj, ei, ej;
    get_index(m, topLeft, si, sj);
    get_index(m, bottomRight, ei, ej);
    for (int a = si; a <= ei; ++a)
      for (int b = sj; b <= ej; ++b) {
        if (a < 0 || b < 0 || a >= m.rows || b >= m.cols) continue;
        if (!polygon_is_inside(poly, V2{m.X[a], m.Y[b]})) continue;
        const size_t c = (size_t)b * m.rows + a;
        rec.visit(c);                                                                  // :601
        if (blocked[c]) {
          pathIsTraversable = false;
          if (!cup) return false;
        } else {
          nCells++;
        }
      }
    if (pathIsTraversable && nCells == 0) pathIsTraversable = p.traversability_default != 0.0;  // :623-628
    return pathIsTraversable;
  }

  // checkPolygonalFootprintPath, :464-584: the polygons it checks, in order, until one fails.
  void polygonal_path(const double* poses, int arraySize, int nfp, const float* footprint_xyz, bool conservative, bool cup) const {
    Polygon polygon1, polygon2;
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    for (int i = 0; i < arraySize; i++) {
      polygon1 = polygon2;
      start = end;
      polygon2.clear();
      const double* pose = poses + 7 * (size_t)i;
      end = V2{pose[0], pose[1]};
      for (int v = 0; v < nfp; ++v) polygon2.push_back(transform(pose, footprint_xyz + 3 * v));
      if (conservative && i > 0) {
        const V2 startToEnd = end - start;
        const Polygon vertices1 = polygon1, vertices2 = polygon2;
        for (const V2& vertex : vertices1) polygon2.push_back(vertex + startToEnd);
        for (const V2& vertex : vertices2) polygon1.push_back(vertex - startToEnd);
      }
      if (arraySize == 1) {
        if (!check_inclination(m, robot_slope, end, end)) return;
        if (!polygon_traversable(polygon2, cup)) return;
      }
      if (arraySize > 1 && i > 0) {
        if (!check_inclination(m, robot_slope, start, end)) return;
        if (!polygon_traversable(convex_hull(polygon1, polygon2), cup)) return;
      }
    }
  }
};

struct Oracle {
  Map m;
  std::vector<unsigned char> blocked;
  std::vector<float> s, t, r;
  Recorder rec;
  Oracle(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope, const float* step,
         const float* rough, const float* elev, float* so, float* to, float* ro)
      : m(map_of(g, trav, slope, step, elev)) {
    const size_t n = (size_t)m.rows * m.cols;
    s.resize(n); t.resize(n); r.resize(n);
    compute_blocked(m, *p, rough, blocked, s.data(), t.data(), r.data(), 1);
    rec = Recorder{s.data(), t.data(), r.data(), so, to, ro};
  }
};

}  // namespace

// One request (arguments as teo_check_request, cache required) that records its visits into slope_fp / step_fp / rough_fp.
extern "C" int teo_memo_request(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                const float* step, const float* rough, const float* elev, const float* robot_slope, int npaths,
                                const int32_t* path_begin, const double* poses, const double* radius, const int32_t* footprint_begin,
                                const float* footprint_xyz, const uint8_t* conservative_or_null, const uint8_t* cup_or_null,
                                float* cache, float* slope_fp, float* step_fp, float* rough_fp) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !p || !trav || !slope || !step || !elev || npaths < 0 || !path_begin || !poses ||
      !radius || !footprint_begin || !cache || !slope_fp || !step_fp || !rough_fp)
    return 1;
  if (p->verify_roughness && !rough) return 1;
  const Oracle o(g, p, trav, slope, step, rough, elev, slope_fp, step_fp, rough_fp);
  const RecChecker check{o.m, *p, o.blocked, robot_slope, o.rec};
  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], n = path_begin[q + 1] - b;
    const int f = footprint_begin[q], nfp = footprint_begin[q + 1] - f;
    const bool cup = cup_or_null && cup_or_null[q];
    if (nfp > 0) {
      check.polygonal_path(poses + 7 * (size_t)b, n, nfp, footprint_xyz + 3 * (size_t)f, conservative_or_null && conservative_or_null[q],
                           cup);
      continue;
    }
    const double pathRadius = radius[q], radiusMax = pathRadius + p->offset;
    const SpiralOffsets sp = spiral_offsets(radiusMax, o.m.res);
    double t = 0.0;
    circular_footprint_path(o.m, robot_slope, poses + 7 * (size_t)b, 7, n, cup, t, convex_hull,
                            [&](V2 center, double& tc, Polygon& up) {
                              return check.circle_traversable(cache, sp, center, radiusMax, cup, tc, up, pathRadius);
                            },
                            [](const Polygon&) {});
  }
  return 0;
}

// traversabilityFootprint(radius, offset) on `cache`, recording its visits.
extern "C" int teo_memo_sweep(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                              const float* step, const float* rough, const float* elev, float* cache, float* slope_fp, float* step_fp,
                              float* rough_fp) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !p || !trav || !slope || !step || !elev || !cache || !slope_fp || !step_fp || !rough_fp)
    return 1;
  if (p->verify_roughness && !rough) return 1;
  const Oracle o(g, p, trav, slope, step, rough, elev, slope_fp, step_fp, rough_fp);
  const RecChecker check{o.m, *p, o.blocked, nullptr, o.rec};
  const SpiralOffsets sp = spiral_offsets(p->radius + p->offset, o.m.res);
  Polygon none;
  for (int j = 0; j < o.m.cols; ++j)
    for (int i = 0; i < o.m.rows; ++i) {
      double t;
      check.circle_traversable(cache, sp, V2{o.m.X[i], o.m.Y[j]}, p->radius + p->offset, false, t, none, p->radius);
    }
  return 0;
}
