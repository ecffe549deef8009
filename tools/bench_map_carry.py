"""Carrying the elevation map's layers through a te_map update, and publishing them, against the host round trips a node needs
without te_map_carry_layers.

Two workloads: one map of 8192² cells and a batch of 256 maps of 512² (synth.terrain "mixed" at 0.02 m, one seed per map).
Every host buffer is page-locked; the host-memory entries return synchronised, so each case is timed with the host clock around
its calls, median of --reps after --warmup, the cases alternating.
  - init: initialising from a grid map with robot_slope (initializeTraversabilityMapFromGridMap).  "carry" is te_map_chain(_batched)
    without outputs plus te_map_carry_layers(robot_slope); "round trip" is te_map_chain(_batched) with its four outputs copied to
    the host plus te_map_set_layers(_batched) of those four, the elevation and robot_slope.
  - publish: the layers publishTraversabilityMap sends with bounds (traversability, elevation, upper_bound, lower_bound and
    uncertainty_range).  "device range" is one te_map_get_layers of all five; "numpy range" is te_map_get_layers of the four held
    layers plus numpy's upper - lower into a page-locked buffer.
Then, once per workload, the results are checked bit for bit: the layers and the cache of the carry map equal those of the round
trip map, and the device uncertainty_range equals numpy's.  One JSON line per case and one per check, with the GPU and its power
limit.

    python tools/bench_map_carry.py [--reps 5] [--warmup 1] [--only 8192|batch]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_map_update import gpu_info  # noqa: E402

RES = 0.02
PUBLISH = ["traversability", "elevation", "upper_bound", "lower_bound"]


def run(te, torch, ctx, L, nmaps, size, args, gpu, power):
    g = te.Geometry.make(size, size, RES)
    p = te.ChainParams.yaml_defaults(0)
    cells = nmaps * size * size
    label = f"{size}x{size}" if nmaps == 1 else f"{nmaps}x{size}x{size}"

    def pinned(n=1):   # n layers of every map, each map column-major
        return torch.empty((n, cells), dtype=torch.float32, pin_memory=True).numpy()

    elev = pinned()[0]
    for k in range(nmaps):
        elev[k * size * size:(k + 1) * size * size] = synth_terrain(size, 7000 + k)
    rng = np.random.default_rng(1)
    rs, up, lo = pinned()[0], pinned()[0], pinned()[0]
    rs[:] = rng.uniform(0.0, 0.6, cells).astype(np.float32)
    rs[rng.random(cells) < 0.001] = 0.0
    lo[:] = elev - rng.uniform(0.0, 0.1, cells).astype(np.float32)
    up[:] = elev + rng.uniform(0.0, 0.1, cells).astype(np.float32)
    outs = pinned(4)
    lay = {"slope": outs[0], "step": outs[1], "roughness": outs[2], "traversability": outs[3]}

    def check(code):
        if code != 0:
            raise RuntimeError(L.te_last_error().decode())

    def chain(m, with_outputs):
        o = [lay[k].ctypes.data if with_outputs else None for k in ("slope", "step", "roughness", "traversability")]
        if nmaps == 1:
            check(L.te_map_chain(m._h, C.byref(g), C.byref(p), elev.ctypes.data, *o, te.MEM_HOST))
        else:
            check(L.te_map_chain_batched(m._h, C.byref(g), C.byref(p), nmaps, elev.ctypes.data, *o, te.MEM_HOST))

    carry_m, trip_m = ctx.map(), ctx.map()
    rs_ptr = (C.c_void_p * 1)(rs.ctypes.data)
    bounds = (C.c_void_p * 2)(up.ctypes.data, lo.ctypes.data)

    def init_carry():
        chain(carry_m, False)
        check(L.te_map_carry_layers(carry_m._h, 0, None, te.capi.layer_mask(["robot_slope"]), rs_ptr, te.MEM_HOST))

    def init_round_trip():
        chain(trip_m, True)
        args_ = [lay["traversability"].ctypes.data, lay["slope"].ctypes.data, lay["step"].ctypes.data, lay["roughness"].ctypes.data,
                 elev.ctypes.data, rs.ctypes.data]
        if nmaps == 1:
            check(L.te_map_set_layers(trip_m._h, C.byref(g), *args_, te.MEM_HOST))
        else:
            check(L.te_map_set_layers_batched(trip_m._h, C.byref(g), nmaps, *args_, te.MEM_HOST))

    pub_dev, pub_np = pinned(5), pinned(5)
    mask_all = te.capi.layer_mask(PUBLISH + ["uncertainty_range"])
    mask_held = te.capi.layer_mask(PUBLISH)

    def publish_device():
        check(L.te_map_get_layers(carry_m._h, mask_all, pub_dev.ctypes.data, te.MEM_HOST))

    def publish_numpy():
        check(L.te_map_get_layers(carry_m._h, mask_held, pub_np.ctypes.data, te.MEM_HOST))
        np.subtract(pub_np[2], pub_np[3], out=pub_np[4])   # bit order: traversability, elevation, upper, lower

    def restore_bounds():   # te_map_chain drops the carried layers: put the bounds the publish cases read back, untimed
        check(L.te_map_carry_layers(carry_m._h, 0, None, te.capi.layer_mask(["upper_bound", "lower_bound"]), bounds, te.MEM_HOST))

    cases = {"init carry": init_carry, "init round trip": init_round_trip, "publish device range": publish_device,
             "publish numpy range": publish_numpy}
    launches = {}
    for name, fn in cases.items():
        l0 = ctx.stats()[0]
        fn()
        launches[name] = ctx.stats()[0] - l0
        for _ in range(args.warmup):
            fn()
        if name == "init carry":
            restore_bounds()
    times = {name: [] for name in cases}
    with np.errstate(invalid="ignore", over="ignore"):
        for _ in range(args.reps):
            for name, fn in cases.items():
                t0 = time.perf_counter()
                fn()
                ctx.synchronize()
                times[name].append(1e3 * (time.perf_counter() - t0))
                if name == "init carry":
                    restore_bounds()
    pcie = {"init carry": 4 * cells * 2, "init round trip": 4 * cells * (1 + 4 + 6),
            "publish device range": 4 * cells * 5, "publish numpy range": 4 * cells * 4}
    for name, t in times.items():
        print(json.dumps({"case": name, "maps": nmaps, "size": label, "median_ms": round(float(np.median(t)), 3),
                          "range_ms": [round(min(t), 3), round(max(t), 3)], "pcie_mb": round(pcie[name] / 1e6, 1),
                          "launches": launches[name], "gpu": gpu, "power_limit_w": power}), flush=True)

    # bit-for-bit checks: the carry map against the round-trip map, the device range against numpy's
    init_carry()
    init_round_trip()
    names = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation", "robot_slope",
             "traversability_footprint"]
    same_layers = True
    a, b = pinned()[0], pinned()[0]
    for name in names:
        mask = te.capi.layer_mask([name])
        check(L.te_map_get_layers(carry_m._h, mask, a.ctypes.data, te.MEM_HOST))
        check(L.te_map_get_layers(trip_m._h, mask, b.ctypes.data, te.MEM_HOST))
        same_layers &= bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
    restore_bounds()
    publish_device()
    with np.errstate(invalid="ignore", over="ignore"):
        want = up - lo
    same_range = bool(np.array_equal(pub_dev[4].view(np.uint32), want.view(np.uint32)))
    print(json.dumps({"check": "bit for bit", "size": label, "carry_equals_round_trip": same_layers,
                      "device_range_equals_numpy": same_range, "gpu": gpu, "power_limit_w": power}), flush=True)
    carry_m.close()
    trip_m.close()
    return same_layers and same_range


def synth_terrain(size, seed):
    import synth
    return synth.terrain(size, size, RES, seed, "mixed").astype(np.float32).T.reshape(-1)   # column-major


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", choices=["8192", "batch"], default=None)
    args = ap.parse_args()
    import torch
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_carry needs a CUDA device")
    gpu, power = gpu_info(torch)
    ctx = te.Context(0)
    L = te.load_library()
    ok = True
    for nmaps, size, key in ((1, 8192, "8192"), (256, 512, "batch")):
        if args.only in (None, key):
            ok &= run(te, torch, ctx, L, nmaps, size, args, gpu, power)
    ctx.close()
    if not ok:
        raise SystemExit("results differ bit for bit")


if __name__ == "__main__":
    main()
