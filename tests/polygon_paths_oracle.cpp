/*
 * polygon_paths_oracle.cpp — CPU ORACLE of te_check_footprint_paths_polygon (test infrastructure, NOT product code).
 *
 * Restates TraversabilityMap::checkPolygonalFootprintPath, traversability_estimation/src/TraversabilityMap.cpp:464-584, and
 * isTraversable(polygon, ...) :592-645, line by line, for a batch of paths that share one footprint polygon.  isTraversableForFilters
 * (:774-792) is the footprint oracle's compute_blocked; PolygonIterator uses its bound_position, get_index and polygon_is_inside;
 * checkInclination (:748-762) is restated as in the circular path oracles.  That translation unit is compiled into this one.
 *
 * RECALLED from grid_map 1.6.x (grid_map is not part of the reference checkout; like SURVEY.md Appendix A):
 *   Polygon::convexHull(P1, P2)  = monotoneChainConvexHullOfPoints(P1.vertices ++ P2.vertices)
 *   monotoneChainConvexHullOfPoints(points): size <= 3 -> Polygon(points) as given; otherwise std::sort lexicographically
 *     (x, then y, operator<), lower hull i = 0..m-1, upper hull i = m-2..0 with t = k+1, pop while k >= 2 (resp. >= t) and
 *     cross(A - O, B - O) <= 0 (cross(u, w) = u.x*w.y - u.y*w.x); the result is the first k-1 points.
 *   Polygon::getArea() = |sum_i (v[j].x + v[i].x) * (v[j].y - v[i].y)| / 2, j = i-1 cyclic starting at j = n-1, abs(area / 2.0).
 *   Eigen::Quaternion::toRotationMatrix (oracle/README.md), applied to the quaternion as given (not normalised).
 *
 * Deviation noted (also in include/te_b200.h): an unsafe path reports 0 in traversability and area; the reference returns early
 * (:536-538, :564-567) and leaves the values of earlier segments in its result.
 * PARITY UNPINNED like the rest of the footprint oracle.  All geometry is literal IEEE double in the operand order written (build
 * with -ffp-contract=off).
 */
#include "../oracle/te_oracle_footprint.cpp"

namespace {

struct Pose7 {
  double x, y, z, qx, qy, qz, qw;
};

// Eigen::QuaternionBase::toRotationMatrix (recalled), rows 0 and 1: the z component of a vertex is dropped afterwards.
void rotation_rows(const Pose7& q, double R[2][3]) {
  const double tx = 2.0 * q.qx, ty = 2.0 * q.qy, tz = 2.0 * q.qz;
  const double twx = tx * q.qw, twy = ty * q.qw, twz = tz * q.qw;
  const double txx = tx * q.qx, txy = ty * q.qx, txz = tz * q.qx;
  const double tyy = ty * q.qy, tyz = tz * q.qy, tzz = tz * q.qz;
  R[0][0] = 1.0 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz;         R[1][1] = 1.0 - (txx + tzz); R[1][2] = tyz - twx;
}

// `toPosition * orientation * positionToVertex` (:496-500): Translation * Quaternion -> Isometry, applied to the point.
V2 transform(const Pose7& q, const float* v) {
  double R[2][3];
  rotation_rows(q, R);
  const double vx = (double)v[0], vy = (double)v[1], vz = (double)v[2];
  return V2{((R[0][0] * vx + R[0][1] * vy) + R[0][2] * vz) + q.x, ((R[1][0] * vx + R[1][1] * vy) + R[1][2] * vz) + q.y};
}

// grid_map::Polygon::getArea (recalled).
double polygon_area(const std::vector<V2>& v) {
  double area = 0.0;
  int j = (int)v.size() - 1;
  for (int i = 0; i < (int)v.size(); i++) {
    area += (v[j].x + v[i].x) * (v[j].y - v[i].y);
    j = i;
  }
  return std::abs(area / 2.0);
}

// grid_map::Polygon::monotoneChainConvexHullOfPoints (recalled).
std::vector<V2> monotone_chain(const std::vector<V2>& points) {
  if (points.size() <= 3) return points;
  std::vector<V2> hull(2 * points.size());
  std::vector<V2> sorted(points);
  std::sort(sorted.begin(), sorted.end(), [](const V2& a, const V2& b) { return a.x < b.x || (a.x == b.x && a.y < b.y); });
  auto clockwise = [](V2 o, V2 a, V2 b) {
    const V2 u = a - o, w = b - o;
    return (u.x * w.y - u.y * w.x) <= 0;
  };
  int k = 0;
  for (int i = 0; i < (int)sorted.size(); ++i) {                                   // lower hull
    while (k >= 2 && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  for (int i = (int)sorted.size() - 2, t = k + 1; i >= 0; i--) {                   // upper hull
    while (k >= t && clockwise(hull[k - 2], hull[k - 1], sorted[i])) k--;
    hull[k++] = sorted[i];
  }
  hull.resize(k - 1);
  return hull;
}

// TraversabilityMap::isTraversable(polygon, computeUntraversablePolygon, traversability, ...), :592-645.  The flag only changes the
// untraversable polygon (published, not returned), so it is left out.  PolygonIterator as in teo_footprint_polygon.
bool polygon_traversable(const Map& m, const teo_footprint_params& p, const std::vector<unsigned char>& blocked,
                         const std::vector<V2>& poly, double& traversability) {
  unsigned nCells = 0;                                                              // :594
  traversability = 0.0;                                                             // :595
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
      if (blocked[c]) return false;                                                 // :602-611
      nCells++;                                                                     // :613
      const float v = m.trav[c];
      traversability += std::isfinite(v) ? (double)v : p.traversability_default;    // :614-618
    }
  if (nCells == 0) {                                                                // :623-628
    traversability = p.traversability_default;
    return p.traversability_default != 0.0;
  }
  traversability /= nCells;                                                         // :630
  return true;
}

}  // namespace

extern "C" int teo_check_polygonal_paths(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope,
                                         const float* step, const float* rough, const float* elev, const float* robot_slope,
                                         int nfootprint, const float* footprint_xyz, int npaths, const int32_t* path_begin,
                                         const double* poses, const uint8_t* conservative_or_null, uint8_t* is_safe,
                                         double* traversability_out, double* area_out) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || nfootprint < 1 ||
      !footprint_xyz || npaths < 0 || !path_begin || !poses || !is_safe || !traversability_out || !area_out)
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
  std::vector<unsigned char> blocked;  // isTraversableForFilters (:774-792): a pure function of the layers
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, nt);

  auto checkInclination = [&](V2 start, V2 end) -> bool {                          // :748-762
    if (!robot_slope) return true;                                                 // checkRobotInclination_ off
    if (end.x == start.x && end.y == start.y) {                                    // :750
      int i, j;
      if (!is_inside(m, start) || !get_index(m, start, i, j)) return false;        // atPosition would throw
      return !(robot_slope[(size_t)j * m.rows + i] == 0.0f);                       // :751
    }
    int si, sj, ei, ej;
    if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) return false;
    bool ok = true;
    for_line(si, sj, ei, ej, [&](int a, int c) {                                   // :756
      const float v = robot_slope[(size_t)c * m.rows + a];
      if (!std::isfinite(v)) return true;                                          // :757
      if (v == 0.0f) { ok = false; return false; }                                 // :758
      return true;
    });
    return ok;
  };

#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], arraySize = path_begin[q + 1] - b;
    const bool conservative = conservative_or_null && conservative_or_null[q];
    is_safe[q] = 0;                                                                // :468
    traversability_out[q] = 0.0;                                                   // :469
    area_out[q] = 0.0;                                                             // :470
    if (arraySize <= 0) continue;                                                  // :330-334
    double traversability = 0.0;                                                   // :471
    double resultTraversability = 0.0, resultArea = 0.0;
    std::vector<V2> polygon, polygon1, polygon2;                                   // :475
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    bool safe = true;
    for (int i = 0; i < arraySize && safe; i++) {                                  // :480
      polygon1 = polygon2;                                                         // :481
      start = end;                                                                 // :482
      polygon2.clear();                                                            // :483
      const double* pp = poses + 7 * (size_t)(b + i);
      const Pose7 pose{pp[0], pp[1], pp[2], pp[3], pp[4], pp[5], pp[6]};           // :488-494 (x y z qx qy qz qw)
      end = V2{pose.x, pose.y};                                                    // :495-496
      for (int v = 0; v < nfootprint; ++v) polygon2.push_back(transform(pose, footprint_xyz + 3 * v));  // :498-508
      if (conservative && i > 0) {                                                 // :510-520
        const V2 startToEnd = end - start;
        const std::vector<V2> vertices1 = polygon1, vertices2 = polygon2;
        for (const V2& vertex : vertices1) polygon2.push_back(vertex + startToEnd);
        for (const V2& vertex : vertices2) polygon1.push_back(vertex - startToEnd);
      }
      if (arraySize == 1) {                                                        // :522
        polygon = polygon2;
        if (!checkInclination(end, end)) { safe = false; break; }                  // :524-526
        if (!polygon_traversable(m, *p, blocked, polygon, traversability)) { safe = false; break; }  // :527, :536-539
        resultTraversability = traversability;                                     // :541
        resultArea = polygon_area(polygon);                                        // :542
      }
      if (arraySize > 1 && i > 0) {                                                // :545
        std::vector<V2> both(polygon1);                                            // :546 convexHull(polygon1, polygon2)
        both.insert(both.end(), polygon2.begin(), polygon2.end());
        polygon = monotone_chain(both);
        if (!checkInclination(start, end)) { safe = false; break; }                // :550-554
        if (!polygon_traversable(m, *p, blocked, polygon, traversability)) { safe = false; break; }  // :555, :564-567
        if (i > 1) {                                                               // :570-575
          const double areaPrevious = resultArea;
          const double areaPolygon = polygon_area(polygon) - polygon_area(polygon1);
          resultArea += areaPolygon;
          resultTraversability = (areaPolygon * traversability + areaPrevious * resultTraversability) / resultArea;
        } else {                                                                   // :576-578
          resultArea = polygon_area(polygon);
          resultTraversability = traversability;
        }
      }
    }
    if (!safe) continue;
    is_safe[q] = 1;                                                                // :582
    traversability_out[q] = resultTraversability;
    area_out[q] = resultArea;
  }
  return 0;
}
