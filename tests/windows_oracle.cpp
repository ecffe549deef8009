/*
 * windows_oracle.cpp — CPU ORACLE of the windows te_map_chain_windows and te_map_chain_submap cut out of a larger elevation map
 * (test infrastructure, NOT product code).
 *
 * Restates the window rule on the grid_map pieces of the footprint oracle, whose translation unit is compiled into this one, as
 * submap_oracle.cpp does: the cell-centre arithmetic (cell_coord, getPositionFromIndex) and getIndexFromPosition's expressions
 * (get_index), here with floor instead of truncation and without the inside test, so that a window's top-left index may be
 * negative or past the map.
 *   top-left = (x + 0.5 * length_x, y + 0.5 * length_y); (ti, tj) = floor(-((top-left - 0.5 * map length) - map position) / res)
 *   window position = getPosition(ti, tj) + 0.5 * res - 0.5 * (size * res), getSubmap's expressions at a fixed size
 *   cell (i, j) = map cell (ti + i, tj + j), stored at ((ti + i + start_row) % rows, (tj + j + start_col) % cols) of the
 *                 circular buffer; NaN (std::numeric_limits<float>::quiet_NaN(), grid_map's unknown cell) outside the map
 */
#include "../oracle/te_oracle_footprint.cpp"

extern "C" {

/* The top-left index and position of n windows of rows x cols cells at the positions xy on the map g: top[2k], top[2k + 1] and
 * pos[2k], pos[2k + 1].  length_x / length_y: the windows' length (the batch's geometry). */
int teo_window_geometry(const teo_geometry* g, int n, int rows, int cols, double length_x, double length_y, const double* xy,
                        int64_t* top, double* pos) {
  const Map m = map_of(g, nullptr, nullptr, nullptr, nullptr);
  for (int k = 0; k < n; ++k) {
    const V2 tl{xy[2 * k] + 0.5 * length_x, xy[2 * k + 1] + 0.5 * length_y};
    const double vx = ((tl.x - 0.5 * m.len.x) - m.pos.x) / m.res;
    const double vy = ((tl.y - 0.5 * m.len.y) - m.pos.y) / m.res;
    const int64_t ti = (int64_t)std::floor(-vx), tj = (int64_t)std::floor(-vy);
    top[2 * k] = ti;
    top[2 * k + 1] = tj;
    pos[2 * k] = (cell_coord(m.pos.x, m.len.x, m.res, (int)ti) + 0.5 * m.res) - 0.5 * ((double)rows * m.res);
    pos[2 * k + 1] = (cell_coord(m.pos.y, m.len.y, m.res, (int)tj) + 0.5 * m.res) - 0.5 * ((double)cols * m.res);
  }
  return 0;
}

/* The rows x cols cells from map cell (ti, tj) of `layer`, a map of src_rows x src_cols cells stored column-major as a circular
 * buffer with start index (start_row, start_col), into out (column-major): NaN where the window leaves the map. */
int teo_cut(int src_rows, int src_cols, int start_row, int start_col, const float* layer, int64_t ti, int64_t tj, int rows, int cols,
            float* out) {
  for (int j = 0; j < cols; ++j)
    for (int i = 0; i < rows; ++i) {
      const int64_t a = ti + i, b = tj + j;
      float v = kNaNf;
      if (a >= 0 && a < src_rows && b >= 0 && b < src_cols)
        v = layer[(size_t)((b + start_col) % src_cols) * src_rows + (size_t)((a + start_row) % src_rows)];
      out[(size_t)j * rows + i] = v;
    }
  return 0;
}

}  // extern "C"
