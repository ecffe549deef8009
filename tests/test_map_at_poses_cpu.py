"""The CPU restatement of te_map_at_poses (tests/at_poses_oracle.cpp, teo_at_poses) on hand-worked cases: the pose transform of the
polygonal paths followed by getIndex.  The map is 8 x 8 cells of 0.5 m centred on the origin, so row i's centre is 1.75 - 0.5 i
(and column j's likewise), and cell (i, j) holds 100 i + j."""
import numpy as np
from scipy.spatial.transform import Rotation

import at_poses_oracle as so

N, RES = 8, 0.5
LAYER = np.asfortranarray(100.0 * np.arange(N)[:, None] + np.arange(N)[None, :], dtype=np.float32)


def _geo(oracle):
    return oracle.Geometry.make(N, N, RES)


def _cell(x, y):
    """getIndex by hand: truncation of (2 - x) / 0.5 and (2 - y) / 0.5 (no case here lies on a cell edge)."""
    return int((2.0 - x) / RES), int((2.0 - y) / RES)


def _one(oracle, pose, point):
    v, ok = so.at_poses(_geo(oracle), LAYER, [pose], [point])
    return float(v[0, 0]), int(ok[0, 0])


def test_identity_pose_origin_point(oracle):
    v, ok = _one(oracle, (0.3, -0.6, 5.0, 0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.0))
    i, j = _cell(0.3, -0.6)
    assert (i, j) == (3, 5) and ok == 1 and v == LAYER[i, j]


def test_yaw_moves_a_unit_offset(oracle):
    # 90 degrees about z: (1, 0, 0) goes to (0, 1); from (0.1, 0.1) the point lands at (0.1, 1.1)
    s = np.sqrt(0.5)
    v, ok = _one(oracle, (0.1, 0.1, 0.0, 0.0, 0.0, s, s), (1.0, 0.0, 0.0))
    assert ok == 1 and v == LAYER[_cell(0.1, 1.1)]
    # 180 degrees, (qx, qy, qz, qw) = (0, 0, 1, 0): exactly (x, y) -> (-x, -y)
    v, ok = _one(oracle, (0.25, 0.25, 0.0, 0.0, 0.0, 1.0, 0.0), (1.0, 0.5, 0.0))
    assert ok == 1 and v == LAYER[_cell(-0.75, -0.25)] == LAYER[5, 4]


def test_tilt_moves_x_and_y_by_z(oracle):
    # a unit quaternion tilting 60 degrees about (1, -1, 0): the point's z moves both x and y
    q = Rotation.from_rotvec(np.deg2rad(60.0) * np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)).as_quat()   # x y z w
    point = np.array([0.2, -0.1, 0.9], np.float32)
    p = Rotation.from_quat(q).apply(point.astype(np.float64)) + [0.3, 0.2, 0.0]
    flat = Rotation.from_quat(q).apply(point.astype(np.float64) * [1, 1, 0]) + [0.3, 0.2, 0.0]
    assert _cell(p[0], p[1]) != _cell(flat[0], flat[1])              # without z the cell differs in both indices
    assert all(a != b for a, b in zip(_cell(p[0], p[1]), _cell(flat[0], flat[1])))
    v, ok = _one(oracle, (0.3, 0.2, 0.0, *q), point)
    assert ok == 1 and v == LAYER[_cell(p[0], p[1])]


def test_non_normalised_quaternion_is_used_as_given(oracle):
    # (qx, qy, qz, qw) = (1, 1, 0, 1): toRotationMatrix rows (-1, 2, 2) and (2, -1, -2), so (0, 0, z) goes to (2z, -2z)
    z = np.float32(0.3)
    v, ok = _one(oracle, (0.0, 0.0, 0.0, 1.0, 1.0, 0.0, 1.0), (0.0, 0.0, z))
    i, j = _cell(2.0 * float(z), -2.0 * float(z))
    assert (i, j) == (2, 5) and ok == 1 and v == LAYER[i, j]
    # normalised, the same quaternion would put the point elsewhere
    qn = np.array([1.0, 1.0, 0.0, 1.0]) / np.sqrt(3.0)
    vn, _ = _one(oracle, (0.0, 0.0, 0.0, *qn), (0.0, 0.0, z))
    assert vn != v


def test_off_map_and_non_finite_points_are_invalid(oracle):
    poses = [(2.5, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0), (np.nan, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.0, 0.0, 0.0, np.inf, 1.0)]
    v, ok = so.at_poses(_geo(oracle), LAYER, poses, [(0.0, 0.0, 0.0)])
    assert not ok.any()
    assert (v.view(np.uint32) == 0x7fc00000).all()
    # grid_map's half-open box: the edge x = 2 lies in row 0, the edge x = -2 outside, just inside it row 7
    poses = [(2.0, 0.1, 0, 0, 0, 0, 1), (-2.0, 0.1, 0, 0, 0, 0, 1), (-1.999, 0.1, 0, 0, 0, 0, 1)]
    v, ok = so.at_poses(_geo(oracle), LAYER, poses, [(0, 0, 0)])
    assert ok[:, 0].tolist() == [1, 0, 1] and v[0, 0] == LAYER[0, 3] and v[2, 0] == LAYER[7, 3]
