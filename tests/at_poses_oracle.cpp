/*
 * at_poses_oracle.cpp — CPU ORACLE of GridMap::atPosition at robot-frame points around poses (test infrastructure, NOT product
 * code): te_map_at_poses is checked against it.
 *
 * Point t of pose k (poses: 7 doubles x y z qx qy qz qw; points: 3 floats x y z) is placed as checkPolygonalFootprintPath places a
 * footprint vertex (TraversabilityMap.cpp:488-507; the transform of paths_oracle.cpp): `toPosition * orientation * point`, the
 * Eigen Translation * Quaternion transform with Quaternion::toRotationMatrix of the quaternion as given (not normalised), rows 0
 * and 1, in the operand order of Transform * vector.  The position is then indexed with getIndexFromPosition (get_index of the
 * footprint oracle, whose translation unit is compiled into this one).  atPosition throws where the index is not found; the
 * library's convention there is NaN 0x7fc00000 and valid 0.
 * All geometry is literal IEEE double in the operand order written (build with -ffp-contract=off).
 */
#include "../oracle/te_oracle_footprint.cpp"

#include <cstring>

extern "C" {

/* One layer (rows x cols, column-major) at npoints points around each of nposes poses: out[k * npoints + t] is the value of the
 * cell getIndex finds and valid 1, or, where the position is not finite or getIndex fails, NaN 0x7fc00000 and valid 0. */
int teo_at_poses(const teo_geometry* g, const float* layer, int nposes, const double* poses, int npoints, const float* points,
                 float* out, uint8_t* valid) {
  const Map m = map_of(g, layer, nullptr, nullptr, nullptr);
  const uint32_t nan_bits = 0x7fc00000u;
  float nan;
  std::memcpy(&nan, &nan_bits, sizeof nan);
  for (int k = 0; k < nposes; ++k) {
    const double* q = poses + 7 * (size_t)k;
    const double qx = q[3], qy = q[4], qz = q[5], qw = q[6];
    const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
    const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
    const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
    const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
    const double R[2][3] = {{1.0 - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1.0 - (txx + tzz), tyz - twx}};
    for (int t = 0; t < npoints; ++t) {
      const float* v = points + 3 * (size_t)t;
      const double vx = (double)v[0], vy = (double)v[1], vz = (double)v[2];
      const V2 p{((R[0][0] * vx + R[0][1] * vy) + R[0][2] * vz) + q[0], ((R[1][0] * vx + R[1][1] * vy) + R[1][2] * vz) + q[1]};
      int i, j;
      const bool ok = std::isfinite(p.x) && std::isfinite(p.y) && get_index(m, p, i, j);
      const size_t s = (size_t)k * npoints + t;
      out[s] = ok ? m.at(layer, i, j) : nan;
      valid[s] = ok ? 1 : 0;
    }
  }
  return 0;
}

}  // extern "C"
