/*
 * untraversable_oracle.cpp — CPU ORACLE of the untraversable polygons of te_check_footprint_paths_fresh2 and
 * te_check_footprint_paths_polygon2 (test infrastructure, NOT product code).
 *
 * Restates, for publishPolygons = true (TraversabilityEstimation.cpp:290), what the check_footprint_path service publishes on its
 * untraversable_polygon topic: checkCircularFootprintPath (traversability_estimation/src/TraversabilityMap.cpp:345-462) with
 * isTraversable(center, ...) :654-746, and checkPolygonalFootprintPath (:464-584) with isTraversable(polygon, ...) :592-645, each
 * with computeUntraversablePolygon as the path asks.  is_safe, traversability and area are restated too (they must equal those of
 * paths_fresh_oracle.cpp / polygon_paths_oracle.cpp).  It compiles polygon_paths_oracle.cpp (and through it the footprint oracle)
 * into this translation unit and reuses their grid_map pieces, monotone chain and filters.
 *
 * PARITY UNPINNED like the rest of the footprint oracle.  All geometry is literal IEEE double in the operand order written (build
 * with -ffp-contract=off).
 */
#include "polygon_paths_oracle.cpp"

#include <algorithm>
#include <map>

// ---------------------------------------------------------------------------------------------------------------------------
// teo_check_circular_paths_fresh2: the same check, plus the untraversable polygon the service publishes per path (publishPolygons =
// true, TraversabilityEstimation.cpp:290): the last non-empty polygon publishUntraversablePolygon receives (:928-938 skips empty
// ones), or none.  count[q] = its vertex count, xy[2 * max_vertices * q ...] its first min(count, max_vertices) vertices.
//
// RECALLED from grid_map 1.6.x (grid_map is not part of the reference checkout):
//   Polygon::fromCircle(center, radius, nVertices = 20): for j = 0 .. nVertices-1, theta = j * 2 * M_PI / (nVertices - 1),
//     vertex = center + Eigen::Rotation2D<double>(theta).toRotationMatrix() * (radius, 0.0).
//   Polygon::convexHull(P1, P2) = monotoneChainConvexHullOfPoints(P1.vertices ++ P2.vertices).
//   monotoneChainConvexHullOfPoints: monotone_chain of polygon_paths_oracle.cpp (3 points or fewer returned as given).
namespace {

std::vector<V2> convex_hull(const std::vector<V2>& p1, const std::vector<V2>& p2) {
  std::vector<V2> both(p1);
  both.insert(both.end(), p2.begin(), p2.end());
  return monotone_chain(both);
}

std::vector<V2> from_circle(V2 center, double radius) {
  const int nVertices = 20;
  std::vector<V2> polygon;
  for (int j = 0; j < nVertices; j++) {
    volatile double theta = j * 2 * M_PI / (nVertices - 1);  // volatile: libm at run time, as the library computes its table
    const double c = std::cos(theta), s = std::sin(theta);
    const V2 centerToVertex{c * radius + (-s) * 0.0, s * radius + c * 0.0};  // Rotation2D(theta).toRotationMatrix() * (radius, 0)
    polygon.push_back(center + centerToVertex);
  }
  return polygon;
}

}  // namespace

extern "C" int teo_check_circular_paths_fresh2(const teo_geometry* g, const teo_footprint_params* p, const float* trav,
                                               const float* slope, const float* step, const float* rough, const float* elev,
                                               const float* robot_slope, int npaths, const int32_t* path_begin, const double* poses_xy,
                                               const double* radius, const uint8_t* cup_or_null, uint8_t* is_safe, double* traversability,
                                               int max_vertices, int32_t* count, double* xy) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || npaths < 0 ||
      !path_begin || !poses_xy || !radius || !is_safe || !traversability || max_vertices < 0 || !count || (max_vertices > 0 && !xy))
    return 1;
  if (p->verify_roughness && !rough) return 1;
  Map m{g->rows, g->cols, g->resolution, {g->length_x, g->length_y}, {g->position_x, g->position_y}, trav, slope, step, elev, {}, {}};
  m.X.resize(m.rows);
  m.Y.resize(m.cols);
  for (int i = 0; i < m.rows; ++i) m.X[i] = cell_coord(m.pos.x, m.len.x, m.res, i);
  for (int j = 0; j < m.cols; ++j) m.Y[j] = cell_coord(m.pos.y, m.len.y, m.res, j);
  int nt = 1;
#ifdef _OPENMP
  nt = omp_get_max_threads();
#endif
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, nt);
  const double offset = p->offset;
  std::map<double, SpiralOffsets> spirals;
  for (int q = 0; q < npaths; ++q)
    if (!spirals.count(radius[q])) spirals[radius[q]] = spiral_offsets(radius[q] + offset, m.res);

#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], arraySize = path_begin[q + 1] - b;
    is_safe[q] = 0;
    traversability[q] = 0.0;
    std::vector<V2> published;                                               // the last non-empty polygon published
    auto publishUntraversablePolygon = [&](const std::vector<V2>& poly) {   // :928-938
      if (!poly.empty()) published = poly;
    };
    auto finish = [&]() {
      count[q] = (int32_t)published.size();
      for (int v = 0; v < (int)published.size() && v < max_vertices; ++v) {
        xy[2 * ((size_t)max_vertices * q + v)] = published[v].x;
        xy[2 * ((size_t)max_vertices * q + v) + 1] = published[v].y;
      }
    };
    if (arraySize <= 0) { finish(); continue; }
    const double pathRadius = radius[q];
    const bool computeUntraversablePolygon = cup_or_null && cup_or_null[q];
    const SpiralOffsets& sp = spirals.at(pathRadius);
    std::map<size_t, float> cache;

    // isTraversable(center, radiusMax, computeUntraversablePolygon, traversability, untraversablePolygon, radiusMin), :654-746
    auto isTraversable = [&](V2 center, double radiusMax, bool cup, double& t, std::vector<V2>& untraversablePolygon,
                             double radiusMin) -> bool {
      bool circleIsTraversable = true;
      std::vector<V2> untraversablePositions;
      untraversablePolygon.clear();                                          // :659
      if (!is_inside(m, center)) {                                           // :662-667
        t = p->traversability_default;
        circleIsTraversable = p->traversability_default != 0.0;
        if (cup && !circleIsTraversable) untraversablePolygon = from_circle(center, radiusMax);
        return circleIsTraversable;
      }
      int ci, cj;
      get_index(m, center, ci, cj);
      const size_t indexCenter = (size_t)cj * m.rows + ci;
      auto it = cache.find(indexCenter);
      if (it != cache.end() && std::isfinite(it->second)) {                  // :673-678
        t = it->second;
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
        if (blocked[cell]) {                                                 // :689-690
          const int ddi = sp.di[k], ddj = sp.dj[k];
          const double untraversableRadius = p->radius_is_integer_norm
              ? (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res
              : std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
          if (radiusMin == 0.0) {                                            // :694-699
            cache[indexCenter] = 0.0f;
            circleIsTraversable = false;
            untraversablePositions.push_back(V2{m.X[a], m.Y[c]});
          } else {
            if (untraversableRadius <= radiusMin) {                          // :700-704
              cache[indexCenter] = 0.0f;
              circleIsTraversable = false;
              untraversablePositions.push_back(V2{m.X[a], m.Y[c]});
            } else if (circleIsTraversable) {                                // :705-711
              const double factor = ((untraversableRadius - radiusMin) / (radiusMax - radiusMin) + 1.0) / 2.0;
              t *= factor / nCells;
              cache[indexCenter] = static_cast<float>(t);
              circleIsTraversable = true;
              traversableRadiusBiggerMinRadius = true;
            }
          }
          if (!cup) return false;                                            // :714-717
        } else {
          nCells++;
          const float v = trav[cell];
          t += std::isfinite(v) ? (double)v : p->traversability_default;
        }
      }
      if (cup && !circleIsTraversable) untraversablePolygon = monotone_chain(untraversablePositions);  // :728-730
      if (circleIsTraversable) {                                             // :732-735
        t /= nCells;
        cache[indexCenter] = static_cast<float>(t);
      }
      return circleIsTraversable;
    };

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
    bool safe = true;
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    std::vector<V2> untraversablePolygon;                                    // :358
    for (int i = 0; i < arraySize && safe; i++) {                            // :360
      start = end;
      end = V2{poses_xy[2 * (b + i)], poses_xy[2 * (b + i) + 1]};
      if (arraySize == 1) {                                                  // :365
        if (!checkInclination(end, end)) { safe = false; break; }            // :366-370 (returns before publishing)
        double t;
        const bool pathIsTraversable = isTraversable(end, pathRadius + offset, computeUntraversablePolygon, t, untraversablePolygon,
                                                     pathRadius);            // :371-372
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);  // :373-380
        if (!pathIsTraversable) { safe = false; break; }                     // :381-384
        result = t;
      }
      if (arraySize > 1 && i > 0) {                                          // :389
        if (!checkInclination(start, end)) { safe = false; break; }
        double traversabilityTemp = 0.0, traversabilitySum = 0.0;
        int nLine = 0;
        int si, sj, ei, ej;
        if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) { safe = false; break; }
        std::vector<V2> auxiliaryUntraversablePolygon;                       // :402
        bool pathIsTraversable = true;
        int visit = 0;
        for_line(ei, ej, si, sj, [&](int a, int c) {                         // :404
          if ((visit++ & 3) != 0) return true;
          const V2 center{m.X[a], m.Y[c]};
          pathIsTraversable = pathIsTraversable && isTraversable(center, pathRadius + offset, computeUntraversablePolygon,
                                                                 traversabilityTemp, auxiliaryUntraversablePolygon, pathRadius);
          if (computeUntraversablePolygon && !auxiliaryUntraversablePolygon.empty())      // :410-412, publishPolygons = true
            untraversablePolygon = convex_hull(untraversablePolygon, auxiliaryUntraversablePolygon);
          traversabilitySum += traversabilityTemp;
          nLine++;
          return true;
        });
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);  // :428-438
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
    finish();
    if (!safe) continue;
    is_safe[q] = 1;
    traversability[q] = result;
  }
  return 0;
}
// ---------------------------------------------------------------------------------------------------------------------------
// teo_check_polygonal_paths2: the same check, plus the untraversable polygon the service publishes per path (publishPolygons =
// true): isTraversable(polygon, computeUntraversablePolygon, ...) :592-645 with the flag of the path, published after every checked
// segment (or the single pose) unless checkInclination returned first (:524-534, :550-561); the last non-empty one is reported
// (publishUntraversablePolygon skips empty polygons, :928-938).  count[q] = its vertex count, xy[2 * max_vertices * q ...] its first
// min(count, max_vertices) vertices.
namespace {

bool polygon_traversable_cup(const Map& m, const teo_footprint_params& p, const std::vector<unsigned char>& blocked,
                             const std::vector<V2>& poly, bool computeUntraversablePolygon, double& traversability,
                             std::vector<V2>& untraversablePolygon) {
  unsigned nCells = 0;                                                              // :594
  traversability = 0.0;                                                             // :595
  bool pathIsTraversable = true;                                                    // :596
  std::vector<V2> untraversablePositions;                                           // :597
  V2 topLeft = poly.empty() ? V2{0.0, 0.0} : poly[0], bottomRight = topLeft;        // PolygonIterator::findSubmapParameters
  for (const V2& q : poly) {
    topLeft = V2{std::max(topLeft.x, q.x), std::max(topLeft.y, q.y)};
    bottomRight = V2{std::min(bottomRight.x, q.x), std::min(bottomRight.y, q.y)};
  }
  bound_position(m, topLeft);
  bound_position(m, bottomRight);
  int si, sj, ei, ej;
  get_index(m, topLeft, si, sj);
  get_index(m, bottomRight, ei, ej);
  for (int a = si; a <= ei; ++a)                                                    // :601 SubmapIterator order
    for (int b = sj; b <= ej; ++b) {
      if (a < 0 || b < 0 || a >= m.rows || b >= m.cols) continue;
      if (!polygon_is_inside(poly, V2{m.X[a], m.Y[b]})) continue;                   // PolygonIterator::isInside
      const size_t c = (size_t)b * m.rows + a;
      if (blocked[c]) {                                                             // :602-611
        pathIsTraversable = false;
        if (computeUntraversablePolygon) {
          untraversablePositions.push_back(V2{m.X[a], m.Y[b]});                     // getPosition
        } else {
          return false;
        }
      } else {
        nCells++;                                                                   // :613
        const float v = m.trav[c];
        traversability += std::isfinite(v) ? (double)v : p.traversability_default;  // :614-618
      }
    }
  if (pathIsTraversable) {                                                          // :622-632
    if (nCells == 0) {
      traversability = p.traversability_default;
      pathIsTraversable = p.traversability_default != 0.0;
    } else {
      traversability /= nCells;
    }
  }
  if (computeUntraversablePolygon) {                                                // :634-642
    if (pathIsTraversable) untraversablePolygon.clear();
    else untraversablePolygon = monotone_chain(untraversablePositions);
  }
  return pathIsTraversable;
}

}  // namespace

extern "C" int teo_check_polygonal_paths2(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                          const float* step, const float* rough, const float* elev, const float* robot_slope,
                                          int nfootprint, const float* footprint_xyz, int npaths, const int32_t* path_begin,
                                          const double* poses, const uint8_t* conservative_or_null, uint8_t* is_safe,
                                          double* traversability_out, double* area_out, const uint8_t* cup_or_null, int max_vertices,
                                          int32_t* count, double* xy) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || nfootprint < 1 ||
      !footprint_xyz || npaths < 0 || !path_begin || !poses || !is_safe || !traversability_out || !area_out || max_vertices < 0 ||
      !count || (max_vertices > 0 && !xy))
    return 1;
  if (p->verify_roughness && !rough) return 1;
  Map m{g->rows, g->cols, g->resolution, {g->length_x, g->length_y}, {g->position_x, g->position_y}, trav, slope, step, elev, {}, {}};
  m.X.resize(m.rows);
  m.Y.resize(m.cols);
  for (int i = 0; i < m.rows; ++i) m.X[i] = cell_coord(m.pos.x, m.len.x, m.res, i);
  for (int j = 0; j < m.cols; ++j) m.Y[j] = cell_coord(m.pos.y, m.len.y, m.res, j);
  int nt = 1;
#ifdef _OPENMP
  nt = omp_get_max_threads();
#endif
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, nt);

  auto checkInclination = [&](V2 start, V2 end) -> bool {                          // :748-762
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

#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], arraySize = path_begin[q + 1] - b;
    const bool conservative = conservative_or_null && conservative_or_null[q];
    const bool computeUntraversablePolygon = cup_or_null && cup_or_null[q];       // :467
    is_safe[q] = 0;
    traversability_out[q] = 0.0;
    area_out[q] = 0.0;
    std::vector<V2> published;
    auto publishUntraversablePolygon = [&](const std::vector<V2>& poly) {          // :928-938
      if (!poly.empty()) published = poly;
    };
    double traversability = 0.0;
    double resultTraversability = 0.0, resultArea = 0.0;
    std::vector<V2> polygon, polygon1, polygon2, untraversablePolygon;             // :473-476
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    bool safe = arraySize > 0;                                                     // :330-334
    for (int i = 0; i < arraySize && safe; i++) {
      polygon1 = polygon2;
      start = end;
      polygon2.clear();
      const double* pp = poses + 7 * (size_t)(b + i);
      const Pose7 pose{pp[0], pp[1], pp[2], pp[3], pp[4], pp[5], pp[6]};
      end = V2{pose.x, pose.y};
      for (int v = 0; v < nfootprint; ++v) polygon2.push_back(transform(pose, footprint_xyz + 3 * v));
      if (conservative && i > 0) {
        const V2 startToEnd = end - start;
        const std::vector<V2> vertices1 = polygon1, vertices2 = polygon2;
        for (const V2& vertex : vertices1) polygon2.push_back(vertex + startToEnd);
        for (const V2& vertex : vertices2) polygon1.push_back(vertex - startToEnd);
      }
      if (arraySize == 1) {                                                        // :522
        polygon = polygon2;
        if (!checkInclination(end, end)) { safe = false; break; }                  // :524-526
        const bool ok = polygon_traversable_cup(m, *p, blocked, polygon, computeUntraversablePolygon, traversability,
                                                untraversablePolygon);                 // :527
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);  // :529-534
        if (!ok) { safe = false; break; }
        resultTraversability = traversability;
        resultArea = polygon_area(polygon);
      }
      if (arraySize > 1 && i > 0) {                                                // :545
        std::vector<V2> both(polygon1);
        both.insert(both.end(), polygon2.begin(), polygon2.end());
        polygon = monotone_chain(both);
        if (!checkInclination(start, end)) { safe = false; break; }                // :550-554
        const bool ok = polygon_traversable_cup(m, *p, blocked, polygon, computeUntraversablePolygon, traversability,
                                                untraversablePolygon);                 // :555
        if (computeUntraversablePolygon) publishUntraversablePolygon(untraversablePolygon);  // :557-562
        if (!ok) { safe = false; break; }
        if (i > 1) {
          const double areaPrevious = resultArea;
          const double areaPolygon = polygon_area(polygon) - polygon_area(polygon1);
          resultArea += areaPolygon;
          resultTraversability = (areaPolygon * traversability + areaPrevious * resultTraversability) / resultArea;
        } else {
          resultArea = polygon_area(polygon);
          resultTraversability = traversability;
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
    traversability_out[q] = resultTraversability;
    area_out[q] = resultArea;
  }
  return 0;
}
