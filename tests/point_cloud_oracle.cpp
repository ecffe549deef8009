/*
 * point_cloud_oracle.cpp — CPU ORACLE of GridMapRosConverter::toPointCloud(map, layers, pointLayer, cloud) (grid_map_ros 1.6.x,
 * SURVEY.md A.8; test infrastructure, NOT product code): te_map_get_point_cloud is checked against it.
 *
 * The loop is restated as grid_map writes it.  A GridMapIterator walks the storage: linear index k at buffer index (k % rows,
 * k / rows), the start index not unwrapped.  A cell is skipped when the map has basic layers and one of them is not finite there
 * (isValid(index)), or when the point layer is not finite there (getPosition3 returns false).  Otherwise each field of the record
 * is filled: x and y are (float) of getPosition(index), z is the point layer's value, every other field is at(layer, index).
 * getPosition is restated here from SURVEY.md A.1: the buffer index is unwrapped (index minus start index, wrapped into [0, size)),
 * then position = (mapPosition + (0.5 length - 0.5 resolution)) + resolution * (-unwrapped) per axis, in double.
 * Fields are copied as 4-byte words, so NaN payloads and -0.0 survive.  Build with -ffp-contract=off -fno-fast-math.
 */
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace {

// GridMap::getPosition (getPositionFromIndex) along one axis: buffer index b of a map of n cells with start index s.
double position_of(int b, int n, int s, double map_pos, double length, double res) {
  const int u = ((b - s) % n + n) % n;  // getIndexFromBufferIndex
  const double offset = 0.5 * length - 0.5 * res;
  return (map_pos + offset) + res * (-(double)u);
}

uint32_t bits(float v) {
  uint32_t u;
  std::memcpy(&u, &v, 4);
  return u;
}

}  // namespace

extern "C" {

/* One map: nfields fields (field[e], rows x cols column-major in the buffer order of start index (start_row, start_col), or
 * null for a NaN 0x7fc00000 field), the entry point_e (-1: none) expanding to x, y, z; `point` the point layer (whether or not it
 * is a field) and basic[0..nbasic) the basic layers.  Writes the records as 4-byte words to out (room for rows * cols records)
 * and returns the number of points, or -1 for bad arguments. */
long long teo_point_cloud(int rows, int cols, int start_row, int start_col, double resolution, double length_x, double length_y,
                          double position_x, double position_y, int nfields, const float* const* field, int point_e,
                          const float* point, int nbasic, const float* const* basic, uint32_t* out) {
  if (rows <= 0 || cols <= 0 || start_row < 0 || start_row >= rows || start_col < 0 || start_col >= cols || !point) return -1;
  const bool hasBasicLayers = nbasic > 0;
  const size_t nCells = (size_t)rows * cols;
  long long n = 0;
  uint32_t* r = out;
  for (size_t k = 0; k < nCells; ++k) {  // GridMapIterator
    const int i = (int)(k % (size_t)rows), j = (int)(k / (size_t)rows);
    if (hasBasicLayers) {
      bool valid = true;
      for (int b = 0; b < nbasic; ++b) valid = valid && std::isfinite(basic[b][k]);
      if (!valid) continue;
    }
    const float value = point[k];
    if (!std::isfinite(value)) continue;  // getPosition3
    const double px = position_of(i, rows, start_row, position_x, length_x, resolution);
    const double py = position_of(j, cols, start_col, position_y, length_y, resolution);
    for (int e = 0; e < nfields; ++e) {
      if (e == point_e) {
        *r++ = bits((float)px);
        *r++ = bits((float)py);
        *r++ = bits((float)(double)value);
      } else {
        *r++ = field[e] ? bits(field[e][k]) : 0x7fc00000u;
      }
    }
    ++n;
  }
  return n;
}

}  // extern "C"
