// te_grid.cuh — the grid_map index arithmetic that the host and the kernels must agree on bit for bit: cell centres, isInside,
// getIndex, boundPositionToRange, getSubmap's geometry and the LineIterator walk.  The map request (te_map_check_footprint_request)
// enumerates on the host the circles the kernels then walk, so both sides compile this one definition (the literal translation units build with --fmad=false; the host
// compiler targets x86-64 without FMA, so neither side contracts a*b+c).
#pragma once
#include <cmath>
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

// grid_map::boundPositionToRange (SURVEY.md A.2): a position moved into the map by a few ulps where it lies on or beyond an edge.
template <class G>
__host__ __device__ __forceinline__ void grid_bound_position(const G& A, double& px, double& py) {
  double sx = (px - A.posx) + 0.5 * A.lenx, sy = (py - A.posy) + 0.5 * A.leny;
  double ex = 10.0 * 2.220446049250313e-16, ey = ex;
  if (fabs(px) > 1.0) ex *= fabs(px);
  if (fabs(py) > 1.0) ey *= fabs(py);
  if (sx <= 0.0) sx = ex; else if (sx >= A.lenx) sx = A.lenx - ex;
  if (sy <= 0.0) sy = ey; else if (sy >= A.leny) sy = A.leny - ey;
  px = (sx + A.posx) - 0.5 * A.lenx;
  py = (sy + A.posy) - 0.5 * A.leny;
}

// GridMap::getSubmap(position, length, isSuccess) -> getSubmapInformation (SURVEY.md A.1): the corners position ± length / 2 are
// bound to the map and indexed; the submap is the block of cells between them, its length is its size times the resolution, its
// position puts its top-left corner on the top-left cell's corner, and the requested position is indexed in the submap.
//
// A circular-buffer start index changes none of this.  grid_map indexes the corners in buffer order and maps them back with
// getIndexFromBufferIndex, so the size is a difference of unwrapped indices; the top-left corner's position comes from
// getPositionFromIndex, which unwraps; and the submap is copied out with start index 0 (getBufferRegionsForSubmap).  So on layers
// in default order (a te_map's) the submap is the plain block [top_row, top_row + rows) x [top_col, top_col + cols).
struct SubmapGeo {
  int top_row, top_col, rows, cols;  // block of the map in default order
  int req_row, req_col;              // indexInSubmap
  double lenx, leny, posx, posy;     // the submap's length and position
};

// False where getSubmap's isSuccess is false; `s` is then left as it was.
template <class G>
__host__ __device__ __forceinline__ bool grid_submap(const G& A, double px, double py, double lx, double ly, SubmapGeo& s) {
  double tlx = px + 0.5 * lx, tly = py + 0.5 * ly;
  grid_bound_position(A, tlx, tly);
  int ti, tj, bi, bj;
  if (!grid_get_index(A, tlx, tly, ti, tj)) return false;
  double brx = px - 0.5 * lx, bry = py - 0.5 * ly;
  grid_bound_position(A, brx, bry);
  if (!grid_get_index(A, brx, bry, bi, bj)) return false;
  const double cornx = cell_coord(A.posx, A.lenx, A.res, ti) + 0.5 * A.res, corny = cell_coord(A.posy, A.leny, A.res, tj) + 0.5 * A.res;
  const int rows = bi - ti + 1, cols = bj - tj + 1;
  const double slx = (double)rows * A.res, sly = (double)cols * A.res;
  const GridGeo sub{rows, cols, A.res, slx, sly, cornx - 0.5 * slx, corny - 0.5 * sly};
  int ri, rj;
  if (!grid_get_index(sub, px, py, ri, rj)) return false;
  s = SubmapGeo{ti, tj, rows, cols, ri, rj, sub.lenx, sub.leny, sub.posx, sub.posy};
  return true;
}

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
