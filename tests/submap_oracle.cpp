/*
 * submap_oracle.cpp — CPU ORACLE of GridMap::getSubmap's geometry (test infrastructure, NOT product code): te_submap_geometry,
 * te_map_get_submaps and te_map_valid_at are checked against it.
 *
 * Restates grid_map::getSubmapInformation as GridMap::getSubmap(position, length, isSuccess) calls it for the get_traversability_map
 * service (TraversabilityEstimation.cpp:297-316), with the grid_map pieces of the footprint oracle, whose translation unit is
 * compiled into this one: boundPositionToRange (bound_position), getIndexFromPosition (get_index) and the cell-centre table
 * (getPositionFromIndex).  checkForStep (oracle/te_oracle_footprint.cpp, check_step) restates the same steps inline for its
 * 2.5 * res windows.
 *
 * RECALLED from grid_map 1.6.x (grid_map is not part of the reference checkout; like SURVEY.md Appendix A.1):
 *   topLeft = position - halfTransform * length, halfTransform = 0.5 * diag(-1, -1); bound; getIndex (fail: isSuccess false)
 *   bottomRight = position + halfTransform * length; bound; getIndex (fail: isSuccess false)
 *   topLeftCorner = getPosition(topLeftIndex) - halfTransform * (res, res)
 *   size = bottomRightIndex - topLeftIndex + 1; length = size * res; position = topLeftCorner - 0.5 * length
 *   indexInSubmap = getIndexFromPosition(position requested, submap length, submap position, res, size) (fail: isSuccess false)
 * A failed window is all zeros, as getSubmap returns an empty GridMap.
 */
#include "../oracle/te_oracle_footprint.cpp"

extern "C" {

/* One record per window, 11 doubles: success, rows, cols, top_row, top_col, requested_row, requested_col, length_x, length_y,
 * position_x, position_y. */
int teo_submap_geometry(const teo_geometry* g, int n, const double* position_xy, const double* length_xy, double* out) {
  const Map m = map_of(g, nullptr, nullptr, nullptr, nullptr);
  for (int k = 0; k < n; ++k) {
    double* r = out + 11 * k;
    for (int f = 0; f < 11; ++f) r[f] = 0.0;
    const V2 pos{position_xy[2 * k], position_xy[2 * k + 1]};
    const V2 len{length_xy[2 * k], length_xy[2 * k + 1]};
    V2 tl{pos.x + 0.5 * len.x, pos.y + 0.5 * len.y};
    bound_position(m, tl);
    int ti, tj, bi, bj;
    if (!get_index(m, tl, ti, tj)) continue;
    V2 br{pos.x - 0.5 * len.x, pos.y - 0.5 * len.y};
    bound_position(m, br);
    if (!get_index(m, br, bi, bj)) continue;
    const V2 topLeftCorner{m.X[ti] + 0.5 * m.res, m.Y[tj] + 0.5 * m.res};
    const int srows = bi - ti + 1, scols = bj - tj + 1;
    const V2 subLength{(double)srows * m.res, (double)scols * m.res};
    const V2 subPosition{topLeftCorner.x - 0.5 * subLength.x, topLeftCorner.y - 0.5 * subLength.y};
    Map sub = m;
    sub.rows = srows;
    sub.cols = scols;
    sub.len = subLength;
    sub.pos = subPosition;
    int ri, rj;
    if (!get_index(sub, pos, ri, rj)) continue;
    const double rec[11] = {1.0, (double)srows, (double)scols, (double)ti, (double)tj, (double)ri, (double)rj,
                            subLength.x, subLength.y, subPosition.x, subPosition.y};
    for (int f = 0; f < 11; ++f) r[f] = rec[f];
  }
  return 0;
}

/* mapHasValidTraversabilityAt (TraversabilityMap.cpp:971-983): getIndex, then std::isfinite of traversability there. */
int teo_valid_at(const teo_geometry* g, const float* traversability, int n, const double* xy, uint8_t* valid) {
  const Map m = map_of(g, traversability, nullptr, nullptr, nullptr);
  for (int q = 0; q < n; ++q) {
    int i, j;
    valid[q] = get_index(m, V2{xy[2 * q], xy[2 * q + 1]}, i, j) && std::isfinite(m.at(m.trav, i, j)) ? 1 : 0;
  }
  return 0;
}

}  // extern "C"
