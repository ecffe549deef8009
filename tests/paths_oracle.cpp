/*
 * paths_oracle.cpp — CPU ORACLE of the footprint path checks (test infrastructure, NOT product code): te_check_footprint_paths_fresh2,
 * te_check_footprint_paths_polygon2, te_check_footprint_request and te_map.
 *
 * Restates the reference's check_footprint_path service loop (TraversabilityEstimation.cpp:278-295, publishPolygons = true) for one
 * request: checkCircularFootprintPath (traversability_estimation/src/TraversabilityMap.cpp:345-462, circular_footprint_path of the
 * footprint oracle) with isTraversable(center, ...) :654-746, and checkPolygonalFootprintPath (:464-584) with isTraversable(polygon,
 * ...) :592-645, each with computeUntraversablePolygon as the path asks.  Per path it reports is_safe, traversability, area and the
 * untraversable polygon the service publishes: the last non-empty one publishUntraversablePolygon receives (:928-938 skips empty
 * ones), or none.
 *
 * isTraversable(center) reads and writes the traversability_footprint layer through a cache:
 *   - none given: the map is freshly computed (computeTraversability, :202-237, leaves the layer NaN, :228) and every path starts
 *     from it; a sparse overlay holds the cells the path writes.  Paths are independent and run in parallel.
 *   - a layer given (float32, rows x cols, column-major, NaN = empty): it persists across paths and calls, as in a running service;
 *     paths run one after another in request order.  teo_map_footprint restates traversabilityFootprint(radius, offset) (:307-318)
 *     on it.
 * isTraversableForFilters (:774-792), LineIterator, SpiralIterator, PolygonIterator and checkInclination come from the footprint
 * oracle, whose translation unit is compiled into this one.
 *
 * RECALLED from grid_map 1.6.x (grid_map is not part of the reference checkout; like SURVEY.md Appendix A):
 *   Polygon::convexHull(P1, P2)  = monotoneChainConvexHullOfPoints(P1.vertices ++ P2.vertices)
 *   monotoneChainConvexHullOfPoints(points): size <= 3 -> Polygon(points) as given; otherwise std::sort lexicographically
 *     (x, then y, operator<), lower hull i = 0..m-1, upper hull i = m-2..0 with t = k+1, pop while k >= 2 (resp. >= t) and
 *     cross(A - O, B - O) <= 0 (cross(u, w) = u.x*w.y - u.y*w.x); the result is the first k-1 points.
 *   Polygon::fromCircle(center, radius, nVertices = 20): for j = 0 .. nVertices-1, theta = j * 2 * M_PI / (nVertices - 1),
 *     vertex = center + Eigen::Rotation2D<double>(theta).toRotationMatrix() * (radius, 0.0).
 *   Polygon::getArea() = |sum_i (v[j].x + v[i].x) * (v[j].y - v[i].y)| / 2, j = i-1 cyclic starting at j = n-1, abs(area / 2.0).
 *   Eigen::Quaternion::toRotationMatrix (oracle/README.md), applied to the quaternion as given (not normalised).
 *
 * Deviation noted (also in include/te_b200.h): an unsafe path reports 0 in traversability and area; the reference returns early
 * and leaves the values of earlier segments in its result.
 * PARITY UNPINNED like the rest of the footprint oracle.  All geometry is literal IEEE double in the operand order written (build
 * with -ffp-contract=off).
 */
#include "../oracle/te_oracle_footprint.cpp"

#include <map>

namespace {

// ---- grid_map::Polygon pieces (recalled) -----------------------------------------------------------------------------------

// Eigen::QuaternionBase::toRotationMatrix, rows 0 and 1 (the z component of a vertex is dropped afterwards), and
// `toPosition * orientation * positionToVertex` (:496-500): Translation * Quaternion -> Isometry, applied to the vertex.
// q = x y z qx qy qz qw.
V2 transform(const double* q, const float* v) {
  const double qx = q[3], qy = q[4], qz = q[5], qw = q[6];
  const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const double R[2][3] = {{1.0 - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1.0 - (txx + tzz), tyz - twx}};
  const double vx = (double)v[0], vy = (double)v[1], vz = (double)v[2];
  return V2{((R[0][0] * vx + R[0][1] * vy) + R[0][2] * vz) + q[0], ((R[1][0] * vx + R[1][1] * vy) + R[1][2] * vz) + q[1]};
}

double polygon_area(const Polygon& v) {                                                // Polygon::getArea
  double area = 0.0;
  int j = (int)v.size() - 1;
  for (int i = 0; i < (int)v.size(); i++) {
    area += (v[j].x + v[i].x) * (v[j].y - v[i].y);
    j = i;
  }
  return std::abs(area / 2.0);
}

Polygon monotone_chain(const Polygon& points) {                                        // Polygon::monotoneChainConvexHullOfPoints
  if (points.size() <= 3) return points;
  Polygon hull(2 * points.size());
  Polygon sorted(points);
  std::sort(sorted.begin(), sorted.end(), [](const V2& a, const V2& b) { return a.x < b.x || (a.x == b.x && a.y < b.y); });
  auto clockwise = [](V2 o, V2 a, V2 b) {
    const V2 u = a - o, w = b - o;
    return (u.x * w.y - u.y * w.x) <= 0;
  };
  int k = 0;
  for (int i = 0; i < (int)sorted.size(); ++i) {                                       // lower hull
    while (k >= 2 && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  for (int i = (int)sorted.size() - 2, t = k + 1; i >= 0; i--) {                       // upper hull
    while (k >= t && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  hull.resize(k - 1);
  return hull;
}

Polygon convex_hull(const Polygon& p1, const Polygon& p2) {                            // Polygon::convexHull
  Polygon both(p1);
  both.insert(both.end(), p2.begin(), p2.end());
  return monotone_chain(both);
}

Polygon from_circle(V2 center, double radius) {                                        // Polygon::fromCircle
  const int nVertices = 20;
  Polygon polygon;
  for (int j = 0; j < nVertices; j++) {
    volatile double theta = j * 2 * M_PI / (nVertices - 1);  // volatile: libm at run time, as the library computes its table
    const double c = std::cos(theta), s = std::sin(theta);
    const V2 centerToVertex{c * radius + (-s) * 0.0, s * radius + c * 0.0};  // Rotation2D(theta).toRotationMatrix() * (radius, 0)
    polygon.push_back(center + centerToVertex);
  }
  return polygon;
}

// publishUntraversablePolygon (:928-938) skips empty polygons: the path reports the last non-empty one.
void publish(Polygon& published, const Polygon& polygon) {
  if (!polygon.empty()) published = polygon;
}

// ---- the traversability_footprint layer --------------------------------------------------------------------------------------

struct FreshCache {  // the cells one path writes on a freshly computed map; all others are NaN
  std::map<size_t, float> cells;
  float get(size_t c) const {
    const auto it = cells.find(c);
    return it == cells.end() ? kNaNf : it->second;
  }
  void set(size_t c, float v) { cells[c] = v; }
};

struct LayerCache {  // the caller's persistent layer
  float* layer;
  float get(size_t c) const { return layer[c]; }
  void set(size_t c, float v) { layer[c] = v; }
};

struct Checker {
  const Map& m;
  const teo_footprint_params& p;
  const std::vector<unsigned char>& blocked;  // isTraversableForFilters (:774-792) of every cell
  const float* robot_slope;

  // isTraversable(center, radiusMax, computeUntraversablePolygon, traversability, untraversablePolygon, radiusMin), :654-746.
  template <class Cache>
  bool circle_traversable(Cache& cache, const SpiralOffsets& sp, V2 center, double radiusMax, bool cup, double& t,
                          Polygon& untraversablePolygon, double radiusMin) const {
    bool circleIsTraversable = true;
    Polygon untraversablePositions;
    untraversablePolygon.clear();                                                      // :659
    if (!is_inside(m, center)) {                                                       // :662-667
      t = p.traversability_default;
      circleIsTraversable = p.traversability_default != 0.0;
      if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
      return circleIsTraversable;
    }
    int ci, cj;
    get_index(m, center, ci, cj);                                                      // :671-672
    const size_t indexCenter = (size_t)cj * m.rows + ci;
    if (std::isfinite(cache.get(indexCenter))) {                                       // :673-678
      t = cache.get(indexCenter);
      circleIsTraversable = t != 0.0;
      if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
      return circleIsTraversable;
    }
    int nCells = 0;                                                                    // :681-682
    t = 0.0;
    bool traversableRadiusBiggerMinRadius = false;
    const double r2 = radiusMax * radiusMax;
    for (size_t k = 0; k < sp.di.size() && !traversableRadiusBiggerMinRadius; ++k) {   // :687-688
      const int a = ci + sp.di[k], c = cj + sp.dj[k];
      if (a < 0 || c < 0 || a >= m.rows || c >= m.cols) continue;                      // SpiralIterator: checkIfIndexInRange
      if (sp.edge[k]) {                                                                // ... isInside on the last two rings, against `center`
        const double dx = m.X[a] - center.x, dy = m.Y[c] - center.y;
        if (!(dx * dx + dy * dy <= r2)) continue;
      }
      const size_t cell = (size_t)c * m.rows + a;
      if (blocked[cell]) {                                                             // :689-690
        const int ddi = sp.di[k], ddj = sp.dj[k];
        const double untraversableRadius = p.radius_is_integer_norm                    // :691 getCurrentRadius()
            ? (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res
            : std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
        if (radiusMin == 0.0 || untraversableRadius <= radiusMin) {                    // :694-704
          cache.set(indexCenter, 0.0f);
          circleIsTraversable = false;
          untraversablePositions.push_back(V2{m.X[a], m.Y[c]});
        } else if (circleIsTraversable) {                                              // :705-711
          const double factor = ((untraversableRadius - radiusMin) / (radiusMax - radiusMin) + 1.0) / 2.0;
          t *= factor / nCells;
          cache.set(indexCenter, static_cast<float>(t));
          circleIsTraversable = true;
          traversableRadiusBiggerMinRadius = true;
        }
        if (!cup) return false;                                                        // :714-717
      } else {
        nCells++;                                                                      // :719
        const float v = m.trav[cell];
        t += std::isfinite(v) ? (double)v : p.traversability_default;                  // :720-724
      }
    }
    if (cup && !circleIsTraversable) untraversablePolygon = monotone_chain(untraversablePositions);  // :728-730
    if (circleIsTraversable) {                                                         // :732-735
      t /= nCells;
      cache.set(indexCenter, static_cast<float>(t));
    }
    return circleIsTraversable;                                                        // :745
  }

  // isTraversable(polygon, computeUntraversablePolygon, traversability, untraversablePolygon), :592-645.  PolygonIterator as in
  // teo_footprint_polygon.
  bool polygon_traversable(const Polygon& poly, bool cup, double& traversability, Polygon& untraversablePolygon) const {
    unsigned nCells = 0;                                                               // :594
    traversability = 0.0;                                                              // :595
    bool pathIsTraversable = true;                                                     // :596
    Polygon untraversablePositions;                                                    // :597
    V2 topLeft = poly.empty() ? V2{0.0, 0.0} : poly[0], bottomRight = topLeft;         // PolygonIterator::findSubmapParameters
    for (const V2& q : poly) {
      topLeft = V2{std::max(topLeft.x, q.x), std::max(topLeft.y, q.y)};
      bottomRight = V2{std::min(bottomRight.x, q.x), std::min(bottomRight.y, q.y)};
    }
    bound_position(m, topLeft);
    bound_position(m, bottomRight);
    int si, sj, ei, ej;
    get_index(m, topLeft, si, sj);
    get_index(m, bottomRight, ei, ej);
    for (int a = si; a <= ei; ++a)                                                     // :600 SubmapIterator order
      for (int b = sj; b <= ej; ++b) {
        if (a < 0 || b < 0 || a >= m.rows || b >= m.cols) continue;
        if (!polygon_is_inside(poly, V2{m.X[a], m.Y[b]})) continue;                    // PolygonIterator::isInside
        const size_t c = (size_t)b * m.rows + a;
        if (blocked[c]) {                                                              // :601-611
          pathIsTraversable = false;
          if (!cup) return false;
          untraversablePositions.push_back(V2{m.X[a], m.Y[b]});                        // getPosition
        } else {
          nCells++;                                                                    // :613
          const float v = m.trav[c];
          traversability += std::isfinite(v) ? (double)v : p.traversability_default;   // :614-618
        }
      }
    if (pathIsTraversable) {                                                           // :623-632
      if (nCells == 0) {
        traversability = p.traversability_default;
        pathIsTraversable = p.traversability_default != 0.0;
      } else {
        traversability /= nCells;
      }
    }
    if (cup) {                                                                         // :634-642
      if (pathIsTraversable) untraversablePolygon.clear();
      else untraversablePolygon = monotone_chain(untraversablePositions);
    }
    return pathIsTraversable;
  }

  // checkPolygonalFootprintPath, :464-584, for one path of n poses (7 doubles each) and a footprint of nfp vertices (3 floats each).
  // Returns is_safe; traversability and area are result.traversability and result.area when safe.
  bool polygonal_path(const double* poses, int arraySize, int nfp, const float* footprint_xyz, bool conservative, bool cup,
                      Polygon& published, double& resultTraversability, double& resultArea) const {
    if (arraySize <= 0) return false;                                                  // :330-334
    double traversability = 0.0;                                                       // :471
    Polygon polygon, polygon1, polygon2, untraversablePolygon;                         // :473-476
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    for (int i = 0; i < arraySize; i++) {                                              // :480
      polygon1 = polygon2;                                                             // :481
      start = end;                                                                     // :482
      polygon2.clear();                                                                // :483
      const double* pose = poses + 7 * (size_t)i;                                      // :488-494 (x y z qx qy qz qw)
      end = V2{pose[0], pose[1]};                                                      // :495-496
      for (int v = 0; v < nfp; ++v) polygon2.push_back(transform(pose, footprint_xyz + 3 * v));  // :498-508
      if (conservative && i > 0) {                                                     // :510-520
        const V2 startToEnd = end - start;
        const Polygon vertices1 = polygon1, vertices2 = polygon2;
        for (const V2& vertex : vertices1) polygon2.push_back(vertex + startToEnd);
        for (const V2& vertex : vertices2) polygon1.push_back(vertex - startToEnd);
      }
      if (arraySize == 1) {                                                            // :522
        polygon = polygon2;
        if (!check_inclination(m, robot_slope, end, end)) return false;                // :524-526
        const bool ok = polygon_traversable(polygon, cup, traversability, untraversablePolygon);  // :527
        if (cup) publish(published, untraversablePolygon);                             // :529-534
        if (!ok) return false;                                                         // :536-539
        resultTraversability = traversability;                                         // :541
        resultArea = polygon_area(polygon);                                            // :542
      }
      if (arraySize > 1 && i > 0) {                                                    // :545
        polygon = convex_hull(polygon1, polygon2);                                     // :546
        if (!check_inclination(m, robot_slope, start, end)) return false;              // :550-554
        const bool ok = polygon_traversable(polygon, cup, traversability, untraversablePolygon);  // :555
        if (cup) publish(published, untraversablePolygon);                             // :557-562
        if (!ok) return false;                                                         // :564-567
        if (i > 1) {                                                                   // :570-575
          const double areaPrevious = resultArea;
          const double areaPolygon = polygon_area(polygon) - polygon_area(polygon1);
          resultArea += areaPolygon;
          resultTraversability = (areaPolygon * traversability + areaPrevious * resultTraversability) / resultArea;
        } else {                                                                       // :576-578
          resultArea = polygon_area(polygon);
          resultTraversability = traversability;
        }
      }
    }
    return true;                                                                       // :582
  }
};

}  // namespace

// One CheckFootprintPath request.  Path q has poses path_begin[q] .. path_begin[q+1]-1 (7 doubles each: x y z qx qy qz qw; a
// circular path reads x and y only) and the footprint rows footprint_begin[q] .. footprint_begin[q+1]-1 of footprint_xyz (none:
// circular, with radius[q]).  cache_or_null: see the header.  Outputs per path: is_safe, traversability, area (0 for circular
// paths), count = the vertex count of the published untraversable polygon, xy[2 * max_vertices * q ...] its first
// min(count, max_vertices) vertices.
extern "C" int teo_check_request(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                 const float* step, const float* rough, const float* elev, const float* robot_slope, int npaths,
                                 const int32_t* path_begin, const double* poses, const double* radius, const int32_t* footprint_begin,
                                 const float* footprint_xyz, const uint8_t* conservative_or_null, const uint8_t* cup_or_null,
                                 float* cache_or_null, uint8_t* is_safe, double* traversability, double* area, int max_vertices,
                                 int32_t* count, double* xy) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || npaths < 0 ||
      !path_begin || !poses || !radius || !footprint_begin || !is_safe || !traversability || !area || max_vertices < 0 || !count ||
      (max_vertices > 0 && !xy))
    return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = map_of(g, trav, slope, step, elev);
  const int nt = thread_count(0);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, nt);
  std::map<double, SpiralOffsets> spirals;
  for (int q = 0; q < npaths; ++q)
    if (footprint_begin[q + 1] == footprint_begin[q] && !spirals.count(radius[q]))
      spirals[radius[q]] = spiral_offsets(radius[q] + p->offset, m.res);
  const Checker check{m, *p, blocked, robot_slope};

  auto path = [&](int q, auto& cache) {
    const int b = path_begin[q], n = path_begin[q + 1] - b;
    const int f = footprint_begin[q], nfp = footprint_begin[q + 1] - f;
    const bool cup = cup_or_null && cup_or_null[q];                                    // :351, :467
    Polygon published;
    double t = 0.0, a = 0.0;
    bool safe;
    if (nfp > 0) {
      const bool conservative = conservative_or_null && conservative_or_null[q];
      safe = check.polygonal_path(poses + 7 * (size_t)b, n, nfp, footprint_xyz + 3 * (size_t)f, conservative, cup, published, t, a);
    } else {
      const double pathRadius = radius[q], radiusMax = pathRadius + p->offset;         // :347-348
      const SpiralOffsets& sp = spirals.at(pathRadius);
      auto isTraversable = [&](V2 center, double& tc, Polygon& untraversablePolygon) {
        return check.circle_traversable(cache, sp, center, radiusMax, cup, tc, untraversablePolygon, pathRadius);
      };
      safe = circular_footprint_path(m, robot_slope, poses + 7 * (size_t)b, 7, n, cup, t, convex_hull, isTraversable,
                                     [&](const Polygon& polygon) { publish(published, polygon); });
    }
    is_safe[q] = safe;
    traversability[q] = safe ? t : 0.0;
    area[q] = safe ? a : 0.0;
    count[q] = (int32_t)published.size();
    for (int v = 0; v < (int)published.size() && v < max_vertices; ++v) {
      xy[2 * ((size_t)max_vertices * q + v)] = published[v].x;
      xy[2 * ((size_t)max_vertices * q + v) + 1] = published[v].y;
    }
  };
  if (cache_or_null) {
    LayerCache cache{cache_or_null};
    for (int q = 0; q < npaths; ++q) path(q, cache);
  } else {
#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
    for (int q = 0; q < npaths; ++q) {
      FreshCache cache;
      path(q, cache);
    }
  }
  return 0;
}

// traversabilityFootprint(radius, offset) (:307-318) on `cache`: every cell's isTraversable(centre, radius + offset, ..., radius).
// A cell whose value is finite takes the memoised branch and keeps it; every other cell walks its spiral.
extern "C" int teo_map_footprint(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                 const float* step, const float* rough, const float* elev, float* cache) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !p || !trav || !slope || !step || !elev || !cache) return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = map_of(g, trav, slope, step, elev);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, 1);
  const SpiralOffsets sp = spiral_offsets(p->radius + p->offset, m.res);
  const Checker check{m, *p, blocked, nullptr};
  LayerCache layer{cache};
  Polygon none;
  for (int j = 0; j < m.cols; ++j)
    for (int i = 0; i < m.rows; ++i) {
      double t;
      check.circle_traversable(layer, sp, V2{m.X[i], m.Y[j]}, p->radius + p->offset, false, t, none, p->radius);
    }
  return 0;
}
