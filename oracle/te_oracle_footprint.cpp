/*
 * te_oracle_footprint.cpp — CPU ORACLE of the circular footprint sweep (test infrastructure, NOT product code).
 *
 * Restates TraversabilityMap::traversabilityFootprint(radius, offset)
 *   traversability_estimation/src/TraversabilityMap.cpp:307-318
 * and everything it reaches: isTraversable(center, radiusMax, ..., radiusMin) :654-746,
 * isTraversableForFilters :774-792, checkForStep :794-865, checkForSlope :867-893, checkForRoughness :895-921, together with the
 * grid_map_core pieces those lines call (SpiralIterator, CircleIterator, LineIterator, getSubmap,
 * getIndex, isInside — SURVEY.md Appendix A.1-A.3, recalled from ros-noetic-grid-map 1.6.x).
 *
 * PARITY UNPINNED: the reference's fixture holds NaN in all three footprint layers, so nothing in
 * the reference pins this code; the decisions taken are listed in oracle/README.md.
 * All geometry is literal IEEE double in the operand order written (build with -ffp-contract=off).
 */
#include "te_oracle.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

constexpr float kNaNf = std::numeric_limits<float>::quiet_NaN();

struct V2 {
  double x, y;
};
inline V2 operator+(V2 a, V2 b) { return {a.x + b.x, a.y + b.y}; }
inline V2 operator-(V2 a, V2 b) { return {a.x - b.x, a.y - b.y}; }
inline double norm(V2 a) { return std::sqrt(a.x * a.x + a.y * a.y); }
inline double dot(V2 a, V2 b) { return a.x * b.x + a.y * b.y; }

struct Map {
  int rows, cols;
  double res;
  V2 len, pos;
  const float* trav;
  const float* slope;
  const float* step;
  const float* elev;
  std::vector<double> X, Y;
  float at(const float* l, int i, int j) const { return l[(size_t)j * rows + i]; }
};

inline double cell_coord(double map_pos, double length, double res, int idx) {
  const double offset = 0.5 * length - 0.5 * res;
  return (map_pos + offset) + res * (-(double)idx);
}

// OpenMP threads: nthreads > 0 as given, otherwise all.
int thread_count(int nthreads) {
#ifdef _OPENMP
  return nthreads > 0 ? nthreads : omp_get_max_threads();
#else
  return (void)nthreads, 1;
#endif
}

// The map and its cell-centre tables X (rows) and Y (columns), grid_map::getPosition.
Map map_of(const teo_geometry* g, const float* trav, const float* slope, const float* step, const float* elev) {
  Map m{g->rows, g->cols, g->resolution, {g->length_x, g->length_y}, {g->position_x, g->position_y}, trav, slope, step, elev, {}, {}};
  m.X.resize(m.rows);
  m.Y.resize(m.cols);
  for (int i = 0; i < m.rows; ++i) m.X[i] = cell_coord(m.pos.x, m.len.x, m.res, i);
  for (int j = 0; j < m.cols; ++j) m.Y[j] = cell_coord(m.pos.y, m.len.y, m.res, j);
  return m;
}

// grid_map::checkIfPositionWithinMap (A.1): half-open box test in the flipped frame.
inline bool is_inside(const Map& m, V2 p) {
  const double tx = -((p.x - m.pos.x) - 0.5 * m.len.x);
  const double ty = -((p.y - m.pos.y) - 0.5 * m.len.y);
  return tx >= 0.0 && ty >= 0.0 && tx < m.len.x && ty < m.len.y;
}

// grid_map::getIndexFromPosition (A.1): truncation of -(position - 0.5*length - mapPosition)/resolution.
inline bool get_index(const Map& m, V2 p, int& i, int& j) {
  const double vx = ((p.x - 0.5 * m.len.x) - m.pos.x) / m.res;
  const double vy = ((p.y - 0.5 * m.len.y) - m.pos.y) / m.res;
  i = (int)(-vx);
  j = (int)(-vy);
  return is_inside(m, p) && i >= 0 && j >= 0 && i < m.rows && j < m.cols;
}

// grid_map::boundPositionToRange (A.2).
inline void bound_position(const Map& m, V2& p) {
  double sh[2] = {(p.x - m.pos.x) + 0.5 * m.len.x, (p.y - m.pos.y) + 0.5 * m.len.y};
  const double pp[2] = {p.x, p.y};
  const double ln[2] = {m.len.x, m.len.y};
  for (int k = 0; k < 2; ++k) {
    double eps = 10.0 * std::numeric_limits<double>::epsilon();
    if (std::fabs(pp[k]) > 1.0) eps *= std::fabs(pp[k]);
    if (sh[k] <= 0.0) { sh[k] = eps; continue; }
    if (sh[k] >= ln[k]) { sh[k] = ln[k] - eps; continue; }
  }
  p.x = (sh[0] + m.pos.x) - 0.5 * m.len.x;
  p.y = (sh[1] + m.pos.y) - 0.5 * m.len.y;
}

template <class F>
inline void for_circle(const Map& m, int i, int j, double radius, F&& f) {
  const int R = (int)std::floor(radius / m.res) + 1;
  const double r2 = radius * radius;
  const int a0 = std::max(0, i - R), a1 = std::min(m.rows - 1, i + R);
  const int b0 = std::max(0, j - R), b1 = std::min(m.cols - 1, j + R);
  for (int a = a0; a <= a1; ++a) {
    const double dx = m.X[a] - m.X[i];
    for (int b = b0; b <= b1; ++b) {
      const double dy = m.Y[b] - m.Y[j];
      if (dx * dx + dy * dy <= r2) f(a, b);
    }
  }
}

// TraversabilityMap::checkForSlope, TraversabilityMap.cpp:867-893 (memoisation removed: pure function).
bool check_slope(const Map& m, const teo_footprint_params& p, int i, int j) {
  if (!(m.at(m.slope, i, j) == 0.0)) return true;                                    // :869
  const double windowRadius = 3.0 * m.res;                                            // :871
  const double criticalLength = p.max_gap_width / 3.0;                                // :872
  const int nSlopesCritical = (int)std::floor(2 * windowRadius * criticalLength / std::pow(m.res, 2));  // :873
  int nSlopes = 0;
  bool ok = true;
  for_circle(m, i, j, windowRadius, [&](int a, int b) {
    if (m.at(m.slope, a, b) == 0.0) ++nSlopes;                                        // :881
    if (nSlopes > nSlopesCritical) ok = false;                                        // :882-885
  });
  return ok;
}

// TraversabilityMap::checkForRoughness, TraversabilityMap.cpp:895-921 (memoisation removed: pure function of the layer).
bool check_roughness(const Map& m, const teo_footprint_params& p, const float* rough, int i, int j) {
  if (!((double)rough[(size_t)j * m.rows + i] == 0.0)) return true;                   // :897
  const double windowRadius = 3.0 * m.res;                                            // :899
  const double criticalLength = p.max_gap_width / 3.0;                                // :900
  const int nRoughnessCritical = (int)std::floor(1.5 * windowRadius * criticalLength / std::pow(m.res, 2));  // :901
  int nRoughness = 0;
  bool ok = true;
  for_circle(m, i, j, windowRadius, [&](int a, int b) {
    if ((double)rough[(size_t)b * m.rows + a] == 0.0) ++nRoughness;                   // :909
    if (nRoughness > nRoughnessCritical) ok = false;                                  // :910-913
  });
  return ok;
}

// grid_map::LineIterator (Bresenham, A.1 family): cells from (i0,j0) to (i1,j1) inclusive.
template <class F>
inline void for_line(int i0, int j0, int i1, int j1, F&& f) {
  const int dx = std::abs(i1 - i0), dy = std::abs(j1 - j0);
  int inc1x = (i1 >= i0) ? 1 : -1, inc2x = inc1x;
  int inc1y = (j1 >= j0) ? 1 : -1, inc2y = inc1y;
  int den, num, numAdd, nCells;
  if (dx >= dy) { inc1x = 0; inc2y = 0; den = dx; num = dx / 2; numAdd = dy; nCells = dx + 1; }
  else { inc2x = 0; inc1y = 0; den = dy; num = dy / 2; numAdd = dx; nCells = dy + 1; }
  int i = i0, j = j0;
  for (int c = 0; c < nCells; ++c) {
    if (!f(i, j)) return;
    num += numAdd;
    if (num >= den) { num -= den; i += inc1x; j += inc1y; }
    i += inc2x; j += inc2y;
  }
}

// TraversabilityMap::checkInclination, TraversabilityMap.cpp:748-762, on the layer robotSlopeType_ names (robot.yaml:1); NULL is
// checkRobotInclination_ off.  A single pose outside the map makes atPosition throw: reported unsafe here.  Invalid (NaN) cells
// compare unequal to 0 and pass (:757).
bool check_inclination(const Map& m, const float* robot_slope, V2 start, V2 end) {
  if (!robot_slope) return true;
  int si, sj, ei, ej;
  if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) return false;       // poses must lie in the map
  if (end.x == start.x && end.y == start.y) return !(robot_slope[(size_t)sj * m.rows + si] == 0.0f);  // :750-751
  bool ok = true;
  for_line(si, sj, ei, ej, [&](int a, int c) { return ok = !(robot_slope[(size_t)c * m.rows + a] == 0.0f); });  // :756-758
  return ok;
}

using Polygon = std::vector<V2>;

// TraversabilityMap::checkCircularFootprintPath, TraversabilityMap.cpp:345-462 (publishPolygons = true) for one path, pose k at
// xy[stride * k].  isTraversable(center, t, polygon) is isTraversable(center, radius + offset, cup, t, polygon, radius) :654-746;
// with `cup` set, `hull` is Polygon::convexHull and publish is publishUntraversablePolygon.  Returns is_safe, with
// result.traversability in `result`.  Deviation noted: `lengthPath` (:443) is uninitialised there; the running length is used.
template <class IsTraversable, class Publish>
bool circular_footprint_path(const Map& m, const float* robot_slope, const double* xy, int stride, int arraySize, bool cup, double& result,
                             Polygon (*hull)(const Polygon&, const Polygon&), IsTraversable&& isTraversable, Publish&& publish) {
  if (arraySize <= 0) return false;                                                   // :330-334
  double lengthPath = 0.0;
  V2 start{0.0, 0.0}, end{0.0, 0.0};
  Polygon untraversablePolygon;                                                       // :357
  for (int i = 0; i < arraySize; i++) {                                               // :360
    start = end;                                                                      // :361
    end = V2{xy[(size_t)stride * i], xy[(size_t)stride * i + 1]};                     // :362-363
    if (arraySize == 1) {                                                             // :365
      if (!check_inclination(m, robot_slope, end, end)) return false;                 // :366-370 (returns before publishing)
      const bool pathIsTraversable = isTraversable(end, result, untraversablePolygon);  // :371-372, :386
      if (cup) publish(untraversablePolygon);                                         // :373-381
      if (!pathIsTraversable) return false;                                           // :382-385
    }
    if (arraySize > 1 && i > 0) {                                                     // :389
      if (!check_inclination(m, robot_slope, start, end)) return false;               // :390-394
      int si, sj, ei, ej;
      if (!get_index(m, start, si, sj) || !get_index(m, end, ei, ej)) return false;   // poses must lie in the map
      double traversabilityTemp = 0.0, traversabilitySum = 0.0;                       // :395
      int nLine = 0, visit = 0;
      Polygon auxiliaryUntraversablePolygon;                                          // :402
      bool pathIsTraversable = true;
      for_line(ei, ej, si, sj, [&](int a, int c) {                                    // :404 LineIterator(endIndex, startIndex)
        if ((visit++ & 3) != 0) return true;                                          // :421-425: nSkip = 3 cells skipped after a check
        const V2 center{m.X[a], m.Y[c]};                                              // :406
        pathIsTraversable = pathIsTraversable && isTraversable(center, traversabilityTemp, auxiliaryUntraversablePolygon);  // :407-408
        if (cup && !auxiliaryUntraversablePolygon.empty())                            // :410-412
          untraversablePolygon = hull(untraversablePolygon, auxiliaryUntraversablePolygon);
        // :414-417 never returns early with publishPolygons; the && above skips every later isTraversable instead
        traversabilitySum += traversabilityTemp;                                      // :419
        nLine++;                                                                      // :420
        return true;
      });
      if (cup) publish(untraversablePolygon);                                         // :429-439
      if (!pathIsTraversable) return false;                                           // :453-456
      const double t = traversabilitySum / (double)nLine;                             // :442
      const double lengthSegment = std::sqrt((end.x - start.x) * (end.x - start.x) + (end.y - start.y) * (end.y - start.y));  // :444
      if (i > 1) {                                                                    // :445-448
        const double lengthPreviousPath = lengthPath;
        lengthPath += lengthSegment;
        result = (lengthSegment * t + lengthPreviousPath * result) / lengthPath;
      } else {                                                                        // :449-452
        lengthPath = lengthSegment;
        result = t;
      }
    }
  }
  return true;                                                                        // :460
}

// TraversabilityMap::checkForStep, TraversabilityMap.cpp:794-865 (memoisation removed).
bool check_step(const Map& m, const teo_footprint_params& p, int i, int j) {
  if (!(m.at(m.step, i, j) == 0.0)) return true;                                      // :796
  const double crit = p.critical_step_height;
  const double windowRadiusStep = 2.5 * m.res;                                        // :798
  const V2 center{m.X[i], m.Y[j]};
  double height = (double)m.at(m.elev, i, j);                                         // :803
  std::vector<std::pair<int, int>> indices;
  for_circle(m, i, j, windowRadiusStep, [&](int a, int b) {
    if ((double)m.at(m.elev, a, b) > crit + height && m.at(m.step, a, b) == 0.0) indices.emplace_back(a, b);  // :806-808
  });
  if (indices.empty()) indices.emplace_back(i, j);                                    // :810
  for (const auto& idx : indices) {
    const int a = idx.first, b = idx.second;
    const V2 subLen{2.5 * m.res, 2.5 * m.res};                                       // :812
    const V2 subMapPos{m.X[a], m.Y[b]};                                               // :815
    const V2 toCenter = center - subMapPos;                                           // :816
    // GridMap::getSubmap -> getSubmapInformation (A.1)
    V2 tl{subMapPos.x + 0.5 * subLen.x, subMapPos.y + 0.5 * subLen.y};
    bound_position(m, tl);
    int ti, tj, bi, bj;
    if (!get_index(m, tl, ti, tj)) return false;                                      // :818-822 (isSuccess false)
    V2 br{subMapPos.x - 0.5 * subLen.x, subMapPos.y - 0.5 * subLen.y};
    bound_position(m, br);
    if (!get_index(m, br, bi, bj)) return false;
    const V2 topLeftCorner{m.X[ti] + 0.5 * m.res, m.Y[tj] + 0.5 * m.res};
    const int srows = bi - ti + 1, scols = bj - tj + 1;
    const V2 subLength{(double)srows * m.res, (double)scols * m.res};
    const V2 subPosition{topLeftCorner.x - 0.5 * subLength.x, topLeftCorner.y - 0.5 * subLength.y};
    height = (double)m.at(m.elev, a, b);                                              // :823
    for (int k = 0; k < srows * scols; ++k) {                                         // GridMapIterator over the submap (:824)
      const int si = k % srows, sj = k / srows;
      const int pi = ti + si, pj = tj + sj;
      if (!(m.at(m.step, pi, pj) == 0.0 && (double)m.at(m.elev, pi, pj) < height - crit)) continue;  // :825
      V2 pos{cell_coord(subPosition.x, subLength.x, m.res, si), cell_coord(subPosition.y, subLength.y, m.res, sj)};  // :827
      const V2 vec = pos - subMapPos;                                                 // :828
      if (norm(vec) < 0.025) continue;                                                // :829
      if (norm(toCenter) > 0.025) {                                                   // :830
        if (dot(toCenter, vec) < 0.0) continue;                                       // :831
      }
      pos = subMapPos + vec;                                                          // :833
      while (norm((pos - subMapPos) + vec) < p.max_gap_width && is_inside(m, pos + vec)) pos = pos + vec;  // :834
      int ei, ej;
      get_index(m, pos, ei, ej);                                                      // :835-836
      bool gapStart = false, gapEnd = false, fail = false;
      for_line(a, b, ei, ej, [&](int li, int lj) {                                    // :839
        if (li < 0 || lj < 0 || li >= m.rows || lj >= m.cols) return false;
        const double e = (double)m.at(m.elev, li, lj);
        if (e > height + crit) { fail = true; return false; }                         // :840-843
        if (e < height - crit || !std::isfinite(m.at(m.elev, li, lj))) {              // :844-846
          gapStart = true;
        } else if (gapStart) {
          gapEnd = true;                                                              // :847-850
          return false;
        }
        return true;
      });
      if (fail) return false;
      if (gapStart && !gapEnd) return false;                                          // :852-855
    }
  }
  return true;                                                                        // :858
}

// grid_map::SpiralIterator visit order (A.3): ring 0 = centre; ring d generated by the walk that starts
// at offset (d,0); rings are consumed back to front.  `edge` marks the rings that apply the circle test.
struct SpiralOffsets {
  std::vector<int> di, dj;
  std::vector<unsigned char> edge;
};

inline int signum(int v) { return (0 < v) - (v < 0); }

SpiralOffsets spiral_offsets(double radius, double res) {
  SpiralOffsets s;
  const int nRings = (int)std::ceil(radius / res);
  s.di.push_back(0); s.dj.push_back(0); s.edge.push_back(0);
  for (int d = 1; d <= nRings; ++d) {
    std::vector<std::pair<int, int>> ring;
    int px = d, py = 0;
    do {
      ring.emplace_back(px, py);
      const int nx = -signum(py), ny = signum(px);
      if (nx != 0 && (unsigned)std::sqrt((double)((px + nx) * (px + nx) + py * py)) == (unsigned)d) px += nx;
      else if (ny != 0 && (unsigned)std::sqrt((double)(px * px + (py + ny) * (py + ny))) == (unsigned)d) py += ny;
      else { px += nx; py += ny; }
    } while (px != d || py != 0);
    for (auto it = ring.rbegin(); it != ring.rend(); ++it) {
      s.di.push_back(it->first);
      s.dj.push_back(it->second);
      s.edge.push_back((d == nRings || d == nRings - 1) ? 1 : 0);
    }
  }
  return s;
}

// isTraversableForFilters (TraversabilityMap.cpp:774-792) is a pure function of the layers: evaluated once per cell.
void compute_blocked(const Map& m, const teo_footprint_params& prm, const float* rough, std::vector<unsigned char>& blocked,
                     float* slope_fp, float* step_fp, float* rough_fp, int nt) {
  const teo_footprint_params* p = &prm;
  const size_t n = (size_t)m.rows * m.cols;
  blocked.assign(n, 0);
#pragma omp parallel for schedule(dynamic, 8) num_threads(nt)
  for (int j = 0; j < m.cols; ++j)
    for (int i = 0; i < m.rows; ++i) {
      const size_t c = (size_t)j * m.rows + i;
      const bool s_ok = check_slope(m, *p, i, j);
      bool t_ok = true;
      if (slope_fp) slope_fp[c] = (m.at(m.slope, i, j) == 0.0) ? (s_ok ? 1.0f : 0.0f) : kNaNf;  // :887,:883
      if (step_fp) step_fp[c] = kNaNf;
      if (s_ok) {                                                                      // short-circuit of :777-778
        t_ok = check_step(m, *p, i, j);
        if (step_fp && m.at(m.step, i, j) == 0.0) step_fp[c] = t_ok ? 1.0f : 0.0f;     // :859,:842,:854
      }
      bool r_ok = true;
      if (rough_fp) rough_fp[c] = kNaNf;
      if (s_ok && t_ok && p->verify_roughness) {                                       // :779-783: only after slope and step passed
        r_ok = check_roughness(m, *p, rough, i, j);
        if (rough_fp && (double)rough[c] == 0.0) rough_fp[c] = r_ok ? 1.0f : 0.0f;     // :915,:911
      }
      blocked[c] = !(s_ok && t_ok && r_ok);
    }
}

}  // namespace

extern "C" {

int teo_spiral_offsets(double radius, double resolution, int32_t* di, int32_t* dj, int cap) {
  if (!(radius >= 0.0) || !(resolution > 0.0)) return -1;
  const SpiralOffsets s = spiral_offsets(radius, resolution);
  // far from the border the circle test reduces to the exact lattice test (no position rounding)
  int n = 0;
  const double r2 = radius * radius;
  for (size_t k = 0; k < s.di.size(); ++k) {
    if (s.edge[k]) {
      const double dx = resolution * (double)s.di[k], dy = resolution * (double)s.dj[k];
      if (!(dx * dx + dy * dy <= r2)) continue;
    }
    if (n < cap) { di[n] = s.di[k]; dj[n] = s.dj[k]; }
    ++n;
  }
  return n;
}

int teo_footprint(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope, const float* step,
                  const float* elev, float* out, float* slope_fp, float* step_fp, int nthreads) {
  return teo_footprint2(g, p, trav, slope, step, nullptr, elev, out, slope_fp, step_fp, nullptr, nthreads);
}

int teo_footprint2(const teo_geometry* g, const teo_footprint_params* p, const float* trav, const float* slope, const float* step,
                   const float* rough, const float* elev, float* out, float* slope_fp, float* step_fp, float* rough_fp, int nthreads) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || !trav || !slope || !step || !elev || !out) return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = map_of(g, trav, slope, step, elev);
  const int nt = thread_count(nthreads);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, slope_fp, step_fp, rough_fp, nt);

  const double radiusMin = p->radius;                         // :313  isTraversable(center, radius + offset, traversability, radius)
  const double radiusMax = p->radius + p->offset;
  const SpiralOffsets sp = spiral_offsets(radiusMax, m.res);
  const double r2 = radiusMax * radiusMax;
#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int j = 0; j < m.cols; ++j)
    for (int i = 0; i < m.rows; ++i) {
      // isTraversable(center = getPosition(cell), radiusMax, false, ..., radiusMin), :654-746, branch :679-736
      const double cx = m.X[i], cy = m.Y[j];
      int nCells = 0;
      double t = 0.0;
      float result = kNaNf;
      bool done = false;
      for (size_t k = 0; k < sp.di.size() && !done; ++k) {
        const int a = i + sp.di[k], b = j + sp.dj[k];
        if (a < 0 || b < 0 || a >= m.rows || b >= m.cols) continue;                    // checkIfIndexInRange
        if (sp.edge[k]) {                                                              // SpiralIterator::isInside on the last two rings
          const double dx = m.X[a] - cx, dy = m.Y[b] - cy;
          if (!(dx * dx + dy * dy <= r2)) continue;
        }
        const size_t c = (size_t)b * m.rows + a;
        if (blocked[c]) {                                                              // :690
          double uR;                                                                   // :691 getCurrentRadius()
          const int ddi = sp.di[k], ddj = sp.dj[k];
          if (p->radius_is_integer_norm) uR = (double)(int)std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
          else uR = std::sqrt((double)(ddi * ddi + ddj * ddj)) * m.res;
          if (radiusMin == 0.0) {
            result = 0.0f;                                                             // :695
          } else if (uR <= radiusMin) {
            result = 0.0f;                                                             // :701
          } else {
            const double factor = ((uR - radiusMin) / (radiusMax - radiusMin) + 1.0) / 2.0;  // :706
            t *= factor / nCells;                                                      // :707
            result = (float)t;                                                         // :708
          }
          done = true;                                                                 // :714-717
        } else {
          ++nCells;                                                                    // :719
          const float v = trav[c];
          t += std::isfinite(v) ? (double)v : p->traversability_default;               // :720-724
        }
      }
      if (!done) {
        t /= nCells;                                                                   // :733
        result = (float)t;                                                             // :734
      }
      out[(size_t)j * m.rows + i] = result;
    }
  return 0;
}

// grid_map::Polygon::isInside (grid_map_core Polygon.cpp, recalled): crossing-number test on the vertex list.
static bool polygon_is_inside(const std::vector<V2>& v, V2 pt) {
  int cross = 0;
  for (size_t i = 0, j = v.size() - 1; i < v.size(); j = i++) {
    if (((v[i].y > pt.y) != (v[j].y > pt.y)) &&
        (pt.x < (v[j].x - v[i].x) * (pt.y - v[i].y) / (v[j].y - v[i].y) + v[i].x))
      ++cross;
  }
  return (cross % 2) != 0;
}

// TraversabilityMap::traversabilityFootprint(double footprintYaw), TraversabilityMap.cpp:239-305: every cell gets the footprint
// polygon (footprint/footprint_polygon, robot_footprint_parameter.yaml:3) placed at its centre, unrotated -> traversability_x and
// rotated by footprintYaw about z -> traversability_rot, each evaluated by isTraversable(polygon, traversability) :592-645:
// grid_map::PolygonIterator (bounding box of the vertices bound to the map — findSubmapParameters —, cells in SubmapIterator
// order, Polygon::isInside on the cell centre) -> 0.0 as soon as a cell fails isTraversableForFilters (:601-611), otherwise the
// mean of the traversability layer with traversabilityDefault_ for invalid cells (:612-619,:630), traversabilityDefault_ when the
// polygon covers no cell (:625-628).  Vertices: `toPosition * orientation * positionToVertex` (:277-278) = Eigen
// Translation * Quaternion -> Isometry transform (rotation MATRIX of the quaternion, Quaternion::toRotationMatrix) applied to the
// point, restated in that operand order; the quaternion of kindr::AngleAxisD(yaw, 0, 0, 1) * identity is (cos(yaw/2), 0, 0, sin(yaw/2)).
// PARITY UNPINNED like the rest of this file (PolygonIterator / Polygon recalled from grid_map 1.6.x, no reference data).
int teo_footprint_polygon(const teo_geometry* g, const teo_footprint_params* p, int npts, const double* pts_xy, double yaw,
                          const float* trav, const float* slope, const float* step, const float* rough, const float* elev,
                          float* out_x, float* out_rot, int nthreads) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0) || !p || npts < 3 || !pts_xy || !trav || !slope || !step || !elev ||
      !out_x || !out_rot)
    return 1;
  if (p->verify_roughness && !rough) return 1;
  const Map m = map_of(g, trav, slope, step, elev);
  const int nt = thread_count(nthreads);
  std::vector<unsigned char> blocked;
  compute_blocked(m, *p, rough, blocked, nullptr, nullptr, nullptr, nt);
  // rotation matrices (Eigen::Quaternion::toRotationMatrix with x = y = 0)
  double R[2][2][2];
  for (int which = 0; which < 2; ++which) {
    const double w = which ? std::cos(0.5 * yaw) : 1.0, z = which ? std::sin(0.5 * yaw) : 0.0;
    const double tz = 2.0 * z, twz = tz * w, tzz = tz * z;
    R[which][0][0] = 1.0 - (0.0 + tzz); R[which][0][1] = 0.0 - twz;
    R[which][1][0] = 0.0 + twz;         R[which][1][1] = 1.0 - (0.0 + tzz);
  }
#pragma omp parallel for schedule(dynamic, 4) num_threads(nt)
  for (int j = 0; j < m.cols; ++j) {
    std::vector<V2> poly(npts);
    for (int i = 0; i < m.rows; ++i) {
      const V2 pos{m.X[i], m.Y[j]};                                                   // :266 getPosition(*iterator, position)
      for (int which = 0; which < 2; ++which) {
        for (int k = 0; k < npts; ++k) {                                              // :273-290
          const double px = pts_xy[2 * k], py = pts_xy[2 * k + 1];
          const double rx = (R[which][0][0] * px + R[which][0][1] * py) + 0.0;        // linear() * v (the z column is zero)
          const double ry = (R[which][1][0] * px + R[which][1][1] * py) + 0.0;
          poly[k] = V2{pos.x + rx, pos.y + ry};                                       // + translation()
        }
        // PolygonIterator::findSubmapParameters
        V2 topLeft = poly[0], bottomRight = poly[0];
        for (const V2& q : poly) {
          topLeft = V2{std::max(topLeft.x, q.x), std::max(topLeft.y, q.y)};
          bottomRight = V2{std::min(bottomRight.x, q.x), std::min(bottomRight.y, q.y)};
        }
        bound_position(m, topLeft);
        bound_position(m, bottomRight);
        int si, sj, ei, ej;
        get_index(m, topLeft, si, sj);
        get_index(m, bottomRight, ei, ej);
        unsigned nCells = 0;
        double t = 0.0;
        bool ok = true;
        for (int a = si; a <= ei && ok; ++a)                                          // SubmapIterator: column index fastest
          for (int b = sj; b <= ej; ++b) {
            if (a < 0 || b < 0 || a >= m.rows || b >= m.cols) continue;
            if (!polygon_is_inside(poly, V2{m.X[a], m.Y[b]})) continue;               // PolygonIterator::isInside
            const size_t c = (size_t)b * m.rows + a;
            if (blocked[c]) { ok = false; break; }                                    // :601-611 (computeUntraversablePolygon false)
            ++nCells;                                                                 // :613
            const float v = trav[c];
            t += std::isfinite(v) ? (double)v : p->traversability_default;            // :614-618
          }
        float result;
        if (!ok) {
          result = 0.0f;                                                              // :297 / :301
        } else if (nCells == 0) {
          result = (float)p->traversability_default;                                  // :625-628 (0.0 either way when the default is 0)
        } else {
          result = (float)(t / nCells);                                               // :630, stored to a float layer :295,:299
        }
        (which ? out_rot : out_x)[(size_t)j * m.rows + i] = result;
      }
    }
  }
  return 0;
}

// circular_footprint_path for a batch of paths on a traversability_footprint layer that is valid everywhere (after
// traversabilityFootprint(radius, offset), :307-318): every isTraversable(center, ...) takes the memoised branch :673-678; centres
// outside the map take :662-667 (traversability = default).  checkRobotInclination_ (:366, :390) is off, no polygons.
int teo_check_circular_paths(const teo_geometry* g, const float* footprint, double traversability_default, int npaths,
                             const int32_t* path_begin, const double* poses_xy, uint8_t* is_safe, double* traversability) {
  return teo_check_circular_paths2(g, footprint, nullptr, traversability_default, npaths, path_begin, poses_xy, is_safe, traversability);
}

// The same with checkRobotInclination_ set: `robot_slope` is check_inclination's layer, NULL switches the check off.
int teo_check_circular_paths2(const teo_geometry* g, const float* footprint, const float* robot_slope, double traversability_default,
                              int npaths, const int32_t* path_begin, const double* poses_xy, uint8_t* is_safe, double* traversability) {
  if (!g || g->rows <= 0 || g->cols <= 0 || !footprint || npaths < 0 || !path_begin || !poses_xy || !is_safe || !traversability) return 1;
  const Map m = map_of(g, nullptr, nullptr, nullptr, nullptr);
  auto memoised = [&](V2 c, double& t, Polygon&) -> bool {                  // isTraversable(center, ...) on the memoised layer
    int i, j;
    if (!is_inside(m, c) || !get_index(m, c, i, j)) {                       // :662-667
      t = traversability_default;
      return traversability_default != 0.0;
    }
    t = (double)footprint[(size_t)j * m.rows + i];                          // :674
    return t != 0.0;                                                         // :675
  };
  for (int q = 0; q < npaths; ++q) {
    double result = 0.0;
    const bool ok = circular_footprint_path(m, robot_slope, poses_xy + 2 * (size_t)path_begin[q], 2, path_begin[q + 1] - path_begin[q],
                                            false, result, nullptr, memoised, [](const Polygon&) {});
    is_safe[q] = ok;                                                         // :352-353, :460
    traversability[q] = ok ? result : 0.0;
  }
  return 0;
}

}  // extern "C"
