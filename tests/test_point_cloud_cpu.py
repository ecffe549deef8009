"""The CPU restatement of GridMapRosConverter::toPointCloud (tests/point_cloud_oracle.cpp) against an independent numpy
restatement, the Python field layout of the clouds, and the cloud of the reference's published map (the fixture bag)."""
import numpy as np
import pytest

import point_cloud_oracle as pco


def _random_map(rng, rows, cols, names, special=0.1):
    """Layers with NaN (several payloads), +-Inf, -0.0 and ordinary values."""
    out = {}
    for n in names:
        a = rng.normal(0.0, 2.0, (rows, cols)).astype(np.float32)
        r = rng.random((rows, cols))
        a[r < special] = np.nan
        a[(r >= special) & (r < 1.3 * special)] = np.inf
        a[(r >= 1.3 * special) & (r < 1.6 * special)] = -np.inf
        a[(r >= 1.6 * special) & (r < 1.8 * special)] = -0.0
        nan_payload = rng.random((rows, cols)) < 0.3 * special
        a.view(np.uint32)[nan_payload] = 0xffc01234
        out[n] = np.asfortranarray(a)
    return out


CASES = [  # rows, cols, start, basic, point in fields
    (7, 5, (0, 0), (), True), (7, 5, (3, 4), (), True), (1, 1, (0, 0), (), True), (1, 9, (0, 6), ("b0",), True),
    (9, 1, (8, 0), ("b0", "b1"), False), (33, 17, (32, 16), ("b0",), True), (64, 3, (13, 1), (), False), (2, 2, (1, 1), ("b1",), True)]


@pytest.mark.parametrize("rows,cols,start,basic,with_point", CASES)
def test_oracle_equals_numpy(rows, cols, start, basic, with_point):
    rng = np.random.default_rng(rows * 100 + cols)
    lay = _random_map(rng, rows, cols, ["p", "f0", "f1", "b0", "b1"])
    fields = ["f0", "nanfield", "p", "f1"] if with_point else ["f1", "nanfield", "f0"]
    kw = dict(resolution=0.07, length=(rows * 0.07, cols * 0.07), position=(12.5, -3.25), basic=basic, nan_layers=("nanfield",),
              start=start)
    got, n = pco.point_cloud(lay, fields, "p", **kw)
    want, nw = pco.point_cloud_numpy(lay, fields, "p", **kw)
    assert n == nw and np.array_equal(got, want)
    valid = np.isfinite(lay["p"])
    for b in basic:
        valid &= np.isfinite(lay[b])
    assert n == int(valid.sum())
    assert len(got) == n * 4 * (len(fields) + 2 * with_point)


def test_start_index_moves_points_not_values():
    rng = np.random.default_rng(4)
    rows, cols = 11, 6
    U = _random_map(rng, rows, cols, ["p", "f"])             # default order
    kw = dict(resolution=0.1, length=(1.1, 0.6), position=(0.0, 0.0))
    plain, n = pco.point_cloud(U, ["p", "f"], "p", **kw)
    s = (4, 2)
    B = {k: np.roll(v, s, axis=(0, 1)) for k, v in U.items()}  # the same map in the buffer order of start index s
    moved, m = pco.point_cloud(B, ["p", "f"], "p", start=s, **kw)
    assert n == m
    dt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("f", "<u4")]
    a, b = np.sort(plain.view(dt), order=["x", "y"]), np.sort(moved.view(dt), order=["x", "y"])
    assert a.tobytes() == b.tobytes()                         # the same points ...
    assert plain.tobytes() != moved.tobytes()                 # ... in buffer order


def test_field_layout(te):
    layout, step = te.capi.point_cloud_fields(pco.PUBLISHED, "elevation")
    names = [n for n, _ in layout]
    assert names == ["upper_bound", "lower_bound", "uncertainty_range", "x", "y", "z", "traversability_slope", "traversability_step",
                     "traversability_roughness", "traversability", "step_footprint", "slope_footprint", "traversability_footprint"]
    assert [o for _, o in layout] == list(range(0, 52, 4)) and step == 52
    layout, step = te.capi.point_cloud_fields(["traversability", "step_footprint"], "elevation")  # point layer not a field
    assert layout == [("traversability", 0), ("step_footprint", 4)] and step == 8
    dt = te.capi.point_cloud_dtype(*te.capi.point_cloud_fields(["a", "elevation"], "elevation"))
    assert dt.itemsize == 16 and dt.names == ("a", "x", "y", "z") and dt.fields["y"][1] == 8


def test_fixture_bag_cloud(tmp_path):
    msg = pco.fixture_bag(tmp_path)
    assert msg.layers == pco.PUBLISHED and msg.basic_layers == []
    assert (msg.outer_start_index, msg.inner_start_index) == (0, 0)
    kw = dict(resolution=msg.resolution, length=(msg.length_x, msg.length_y), position=msg.pose[:2],
              nan_layers=(), basic=msg.basic_layers)
    data, n = pco.point_cloud(msg.data, msg.layers, "elevation", **kw)
    assert n == 13300 and len(data) == 13300 * 52
    want, _ = pco.point_cloud_numpy(msg.data, msg.layers, "elevation", **kw)
    assert np.array_equal(data, want)
    rec = data.view(np.float32).reshape(n, 13)
    # cell (0, 0) is the +x, +y corner: position + 0.5 length - 0.5 resolution; cell (99, 132) the other
    assert rec[0, 3] == np.float32(1.5 - 0.015) and rec[0, 4] == np.float32(1.995 - 0.015)
    assert abs(rec[-1, 3] - (-1.485)) < 1e-6 and abs(rec[-1, 4] - (-1.98)) < 1e-6
    assert rec[1, 3] == np.float32(1.485 - 0.03) and rec[100, 4] == np.float32(1.98 - 0.03)  # row, then column
    assert np.array_equal(rec[:, 5].view(np.uint32), msg.data["elevation"].reshape(-1, order="F").view(np.uint32))
    assert (rec[:, 10:].view(np.uint32) == 0x7fc00000).all()  # the memo and footprint layers of a fresh map
