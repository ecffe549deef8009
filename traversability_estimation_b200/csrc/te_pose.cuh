// te_pose.cuh — a geometry_msgs/Pose applied to a robot-frame point as checkPolygonalFootprintPath places a footprint vertex
// (TraversabilityMap.cpp:488-507): `toPosition * orientation * point`, the Eigen Translation * Quaternion transform, with the z of
// the result dropped.  The polygonal path checks (te_paths.cu) and te_map_at_poses (te_submap.cu) both place points with it; both
// translation units build with --fmad=false, so neither contracts a*b+c.
#pragma once

namespace te {

// Translation * Quaternion of a pose: Eigen::QuaternionBase::toRotationMatrix of the quaternion as given (not normalised), rows 0
// and 1 (the z of a transformed vertex is dropped, :505-507).
struct PoseRT {
  double tx, ty, r00, r01, r02, r10, r11, r12;
};
// p: 7 doubles, x y z qx qy qz qw.
__device__ __forceinline__ PoseRT pose_rt_d(const double* p) {
  const double qx = p[3], qy = p[4], qz = p[5], qw = p[6];
  const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  PoseRT T;
  T.tx = p[0]; T.ty = p[1];
  T.r00 = 1.0 - (tyy + tzz); T.r01 = txy - twz; T.r02 = txz + twy;
  T.r10 = txy + twz; T.r11 = 1.0 - (txx + tzz); T.r12 = tyz - twx;
  return T;
}

// `toPosition * orientation * positionToVertex` (:496-500) for the point (vx, vy, vz), in the operand order of Eigen's
// Transform * vector: its x and y.
__device__ __forceinline__ double2 pose_point_d(const PoseRT& T, double vx, double vy, double vz) {
  return make_double2(((T.r00 * vx + T.r01 * vy) + T.r02 * vz) + T.tx, ((T.r10 * vx + T.r11 * vy) + T.r12 * vz) + T.ty);
}

}  // namespace te
