// te_grid.cuh — the grid_map index arithmetic that the host and the kernels must agree on bit for bit: cell centres, isInside,
// getIndex and the LineIterator walk.  The map request (te_map_check_footprint_request) enumerates on the host the circles the
// kernels then walk, so both sides compile this one definition (the literal translation units build with --fmad=false; the host
// compiler targets x86-64 without FMA, so neither side contracts a*b+c).
#pragma once
#include <cstdlib>

namespace te {

// grid_map::getPositionFromIndex operand order (SURVEY.md A.1).
__host__ __device__ __forceinline__ double cell_coord(double map_pos, double length, double res, int idx) {
  const double offset = 0.5 * length - 0.5 * res;
  return (map_pos + offset) + res * (-(double)idx);
}

// GridMap::isInside and GridMap::getIndex on a map in the default start index: the index (i, j) and whether the position lies in
// the map.  G is any geometry with the members rows, cols_total, res, lenx, leny, posx and posy (the kernels' FpArgs, the host's
// GridGeo); reading them in place keeps the kernels' code as it was.
template <class G>
__host__ __device__ __forceinline__ bool grid_is_inside(const G& A, double px, double py) {
  const double tx = -((px - A.posx) - 0.5 * A.lenx);
  const double ty = -((py - A.posy) - 0.5 * A.leny);
  return tx >= 0.0 && ty >= 0.0 && tx < A.lenx && ty < A.leny;
}

template <class G>
__host__ __device__ __forceinline__ bool grid_get_index(const G& A, double px, double py, int& i, int& j) {
  const double vx = ((px - 0.5 * A.lenx) - A.posx) / A.res;
  const double vy = ((py - 0.5 * A.leny) - A.posy) / A.res;
  i = (int)(-vx);
  j = (int)(-vy);
  return grid_is_inside(A, px, py) && i >= 0 && j >= 0 && i < A.rows && j < A.cols_total;
}

struct GridGeo {
  int rows, cols_total;
  double res, lenx, leny, posx, posy;
};

// grid_map::LineIterator (Bresenham) from index (i0, j0) to (i1, j1): `n` cells, (li, lj) the current one.
struct LineD {
  int li, lj, i1x, i2x, i1y, i2y, den, num, numAdd, n;
  __host__ __device__ __forceinline__ LineD(int i0, int j0, int i1, int j1) {
    const int dx = abs(i1 - i0), dy = abs(j1 - j0);
    i1x = (i1 >= i0) ? 1 : -1; i2x = i1x; i1y = (j1 >= j0) ? 1 : -1; i2y = i1y;
    if (dx >= dy) { i1x = 0; i2y = 0; den = dx; num = dx / 2; numAdd = dy; n = dx + 1; }
    else { i2x = 0; i1y = 0; den = dy; num = dy / 2; numAdd = dx; n = dy + 1; }
    li = i0; lj = j0;
  }
  __host__ __device__ __forceinline__ void next() {
    num += numAdd;
    if (num >= den) { num -= den; li += i1x; lj += i1y; }
    li += i2x; lj += i2y;
  }
};

}  // namespace te
