/*
 * paths_fresh_oracle.cpp — CPU ORACLE of te_check_footprint_paths_fresh (test infrastructure, NOT product code).
 *
 * Restates TraversabilityMap::checkCircularFootprintPath, traversability_estimation/src/TraversabilityMap.cpp:345-462, as the
 * check_footprint_path service runs it (publishPolygons = true, TraversabilityEstimation.cpp:278-295) right after
 * computeTraversability (:202-237), which leaves the traversability_footprint layer empty (NaN, :228).  isTraversable
 * (:654-746) then walks the SpiralIterator over the chain layers at arbitrary centre positions and stores its result in that
 * layer; this restatement keeps a real per-path cache (cell -> float) and reads it through the memoised branch (:673-675).
 * Every path starts from an empty cache.
 *
 * It reuses the circular-sweep oracle's grid_map pieces (getIndex, isInside, LineIterator, the SpiralIterator visit order) and
 * its isTraversableForFilters (compute_blocked) by compiling that translation unit into this one.
 *
 * PARITY UNPINNED like the rest of the footprint oracle (same author; no reference data exercises these lines).
 * All geometry is literal IEEE double in the operand order written (build with -ffp-contract=off).
 */
#include "../oracle/te_oracle_footprint.cpp"

#include <map>

extern "C" int teo_check_circular_paths_fresh(const teo_geometry* g, const teo_footprint_params* p, const float* trav,
                                              const float* slope, const float* step, const float* rough, const float* elev,
                                              const float* robot_slope, int npaths, const int32_t* path_begin, const double* poses_xy,
                                              const double* radius, const uint8_t* cup_or_null, uint8_t* is_safe, double* traversability) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || npaths < 0 ||
      !path_begin || !poses_xy || !radius || !is_safe || !traversability)
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
  const double offset = p->offset;  // :348 (0.15 in the reference)
  std::map<double, SpiralOffsets> spirals;
  for (int q = 0; q < npaths; ++q)
    if (!spirals.count(radius[q])) spirals[radius[q]] = spiral_offsets(radius[q] + offset, m.res);

#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int q = 0; q < npaths; ++q) {
    const int b = path_begin[q], arraySize = path_begin[q + 1] - b;
    is_safe[q] = 0;                                                          // :352-353
    traversability[q] = 0.0;
    if (arraySize <= 0) continue;                                            // :330-334
    const double pathRadius = radius[q];                                     // :347
    const bool computeUntraversablePolygon = cup_or_null && cup_or_null[q];  // :351
    const SpiralOffsets& sp = spirals.at(pathRadius);
    std::map<size_t, float> cache;  // traversability_footprint cells written during this path (all others NaN)

    // isTraversable(center, radiusMax, computeUntraversablePolygon, traversability, ..., radiusMin), :654-746
    auto isTraversable = [&](V2 center, double radiusMax, bool cup, double& t, double radiusMin) -> bool {
      bool circleIsTraversable = true;
      if (!is_inside(m, center)) {                                           // :662-667
        t = p->traversability_default;
        return p->traversability_default != 0.0;
      }
      int ci, cj;
      get_index(m, center, ci, cj);                                          // :671-672
      const size_t indexCenter = (size_t)cj * m.rows + ci;
      auto it = cache.find(indexCenter);
      if (it != cache.end() && std::isfinite(it->second)) {                  // :673-675
        t = it->second;
        return t != 0.0;
      }
      int nCells = 0;                                                        // :681-682
      t = 0.0;
      bool traversableRadiusBiggerMinRadius = false;
      const double r2 = radiusMax * radiusMax;
      for (size_t k = 0; k < sp.di.size() && !traversableRadiusBiggerMinRadius; ++k) {  // :687-688
        const int a = ci + sp.di[k], c = cj + sp.dj[k];
        if (a < 0 || c < 0 || a >= m.rows || c >= m.cols) continue;          // SpiralIterator: checkIfIndexInRange
        if (sp.edge[k]) {                                                    // ... isInside on the last two rings, against `center`
          const double dx = m.X[a] - center.x, dy = m.Y[c] - center.y;
          if (!(dx * dx + dy * dy <= r2)) continue;
        }
        const size_t cell = (size_t)c * m.rows + a;
        if (blocked[cell]) {                                                 // :689-690
          const int ddi = sp.di[k], ddj = sp.dj[k];
          const double untraversableRadius = p->radius_is_integer_norm       // :691 getCurrentRadius()
              ? (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res
              : std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
          if (radiusMin == 0.0) {                                            // :694-698
            cache[indexCenter] = 0.0f;
            circleIsTraversable = false;
          } else {
            if (untraversableRadius <= radiusMin) {                          // :700-704
              cache[indexCenter] = 0.0f;
              circleIsTraversable = false;
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
          nCells++;                                                          // :719
          const float v = trav[cell];
          t += std::isfinite(v) ? (double)v : p->traversability_default;     // :720-724
        }
      }
      if (circleIsTraversable) {                                             // :732-735
        t /= nCells;
        cache[indexCenter] = static_cast<float>(t);
      }
      return circleIsTraversable;                                            // :745
    };

    auto checkInclination = [&](V2 start, V2 end) -> bool {                 // :748-762
      if (!robot_slope) return true;                                         // checkRobotInclination_ off
      if (end.x == start.x && end.y == start.y) {                            // :750
        int i, j;
        if (!is_inside(m, start) || !get_index(m, start, i, j)) return false;  // atPosition would throw
        return !(robot_slope[(size_t)j * m.rows + i] == 0.0f);               // :751
      }
      int si, sj, ei, ej;
      if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) return false;
      bool ok = true;
      for_line(si, sj, ei, ej, [&](int a, int c) {                           // :756
        const float v = robot_slope[(size_t)c * m.rows + a];
        if (!std::isfinite(v)) return true;                                  // :757
        if (v == 0.0f) { ok = false; return false; }                         // :758
        return true;
      });
      return ok;
    };

    double result = 0.0, lengthPath = 0.0;  // result.traversability; lengthPath (:443, uninitialised there): the running length
    bool safe = true;
    V2 start{0.0, 0.0}, end{0.0, 0.0};
    for (int i = 0; i < arraySize && safe; i++) {                            // :360
      start = end;                                                           // :361
      end = V2{poses_xy[2 * (b + i)], poses_xy[2 * (b + i) + 1]};            // :362-363
      if (arraySize == 1) {                                                  // :365
        if (!checkInclination(end, end)) { safe = false; break; }            // :366-370
        double t;
        if (!isTraversable(end, pathRadius + offset, computeUntraversablePolygon, t, pathRadius)) { safe = false; break; }  // :371-385
        result = t;                                                          // :386
      }
      if (arraySize > 1 && i > 0) {                                          // :389
        if (!checkInclination(start, end)) { safe = false; break; }          // :390-394
        double traversabilityTemp = 0.0, traversabilitySum = 0.0;            // :395
        int nLine = 0;
        int si, sj, ei, ej;
        if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) { safe = false; break; }  // poses must lie in the map
        bool pathIsTraversable = true;
        int visit = 0;
        for_line(ei, ej, si, sj, [&](int a, int c) {                         // :404 LineIterator(endIndex, startIndex)
          if ((visit++ & 3) != 0) return true;                               // :421-425: nSkip = 3 cells skipped after a check
          const V2 center{m.X[a], m.Y[c]};                                   // :406
          pathIsTraversable = pathIsTraversable &&
                              isTraversable(center, pathRadius + offset, computeUntraversablePolygon, traversabilityTemp, pathRadius);  // :407-408
          // :414-417 never returns early with publishPolygons; the && above skips every later isTraversable instead
          traversabilitySum += traversabilityTemp;                           // :419
          nLine++;                                                           // :420
          return true;
        });
        if (pathIsTraversable) {                                             // :441-452
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
          safe = false;                                                      // :453-456
        }
      }
    }
    if (!safe) continue;
    is_safe[q] = 1;                                                          // :460
    traversability[q] = result;
  }
  return 0;
}
