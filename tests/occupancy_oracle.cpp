/*
 * occupancy_oracle.cpp — CPU ORACLE of GridMapRosConverter::toOccupancyGrid (grid_map_ros 1.6.x, SURVEY.md A.7; test
 * infrastructure, NOT product code): te_map_get_occupancy and te_occupancy_grid_info are checked against it.
 *
 * The loop is restated as grid_map writes it: a GridMapIterator walks the layer's storage (column-major buffer order, linear index
 * k at buffer index (k % rows, k / rows)), reads the cell there (map.at(layer, *iterator)), and places the value at
 * data[nCells - index - 1] with index = getLinearIndexFromIndex(iterator.getUnwrappedIndex(), size, false) = j * rows + i, the
 * unwrapped index being the buffer index minus the start index, modulo the size.  The cell arithmetic is float32 in the operand
 * order written, with std::min / std::max / std::isnan, and the float -> int8_t assignment of the message's data vector.
 * Build with -ffp-contract=off -fno-fast-math.
 */
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>

extern "C" {

/* One layer (rows x cols, column-major in the buffer order of start index (start_row, start_col)) into out (rows * cols bytes,
 * OccupancyGrid.data). */
int teo_occupancy_grid(int rows, int cols, int start_row, int start_col, const float* layer, float dataMin, float dataMax,
                       int8_t* out) {
  if (rows <= 0 || cols <= 0 || start_row < 0 || start_row >= rows || start_col < 0 || start_col >= cols) return -1;
  const float cellMin = 0;
  const float cellMax = 100;
  const float cellRange = cellMax - cellMin;
  const size_t nCells = (size_t)rows * cols;
  for (size_t k = 0; k < nCells; ++k) {  // GridMapIterator: the linear index over the storage
    const int bi = (int)(k % (size_t)rows), bj = (int)(k / (size_t)rows);
    float value = (layer[k] - dataMin) / (dataMax - dataMin);
    if (std::isnan(value))
      value = -1;
    else
      value = cellMin + std::min(std::max(0.0f, value), 1.0f) * cellRange;
    const int i = (bi - start_row + rows) % rows, j = (bj - start_col + cols) % cols;  // getUnwrappedIndex
    const size_t index = (size_t)j * rows + i;  // getLinearIndexFromIndex(..., false): column-major
    out[nCells - index - 1] = (int8_t)value;
  }
  return 0;
}

/* MapMetaData of toOccupancyGrid: resolution (float), width = rows, height = cols, origin = position - 0.5 * length. */
int teo_occupancy_info(int rows, int cols, double resolution, double length_x, double length_y, double position_x,
                       double position_y, int32_t* size, float* res, double* origin) {
  size[0] = rows;
  size[1] = cols;
  *res = (float)resolution;
  origin[0] = position_x - 0.5 * length_x;
  origin[1] = position_y - 0.5 * length_y;
  return 0;
}

}  // extern "C"
