"""traversability_x / traversability_rot kept on a te_map (te_map_footprint_polygon_keep) against the calls a node makes without it.

(a) A fleet: 256 maps of 512² cells (synth.terrain "mixed" at 0.02 m, 32 terrains cycled over the maps), map m at its own
    position (a 40 m grid, off the cell lattice), map m's footprint yaw the (m % 4)-th of four.  Cases:
      - keep:  one te_map_footprint_polygon_keep call on the batched te_map (te_map_chain_batched_at), every map at its yaw;
      - loop:  te_map_footprint_polygon on each of 256 single-map te_maps holding the same maps at the same positions, at the
               map's yaw, device outputs;
      - batch: today's te_map_footprint_polygon on the batched te_map at one yaw, device outputs (on maps at several positions it
               sweeps one map at a time).
(b) One 8192² map: te_map_footprint_polygon_keep against te_map_footprint_polygon with device outputs (the cost of storing the
    layers).
The YAML footprint (robot_footprint_parameter.yaml:3), parameters from robot.yaml.  Device memory, the library on torch's stream,
CUDA events around whole calls, median of --reps after --warmup, cases alternating.  Every kept layer is checked bit for bit
against the loop's (a) or the stateless call's (b); the batch case's traversability_x and, for the maps at its yaw,
traversability_rot likewise.  One JSON line per case, one per check, with the GPU and its power limit.

    python tools/bench_map_polygon.py [--maps 256] [--size 512] [--big 8192] [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_footprint_yaws import gpu_info  # noqa: E402

RES = 0.02
POLY = np.array([[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]], np.float64)
YAWS = np.array([0.0, 0.7854, 1.5708, -2.3562])


def time_cases(torch, stream, ctx, cases, reps, warmup):
    """Median ms per case of CUDA events around each call, the cases alternating in order and reverse order."""
    ms = {k: [] for k in cases}
    for rep in range(warmup + reps):
        for k in (list(cases) if rep % 2 == 0 else list(cases)[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            cases[k]()
            b.record(stream)
            b.synchronize()
            if rep >= warmup:
                ms[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--big", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_polygon needs a CUDA device")
    gpu, power = gpu_info(torch)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    L = ctx._L
    p = te.ChainParams.yaml_defaults(0)
    ft = te.FootprintParams.yaml_defaults()
    pts = np.ascontiguousarray(POLY)
    dev = lambda n: torch.empty(n, dtype=torch.float32, device="cuda")  # noqa: E731
    bad = 0

    def polygon(m, yaw, ox, orot):
        m._check(L.te_map_footprint_polygon(m._h, C.byref(ft), len(pts), pts.ctypes.data, float(yaw), ox.data_ptr(), orot.data_ptr(),
                                            te.MEM_DEVICE))

    def keep(m, yaws):
        ys = np.ascontiguousarray(yaws, dtype=np.float64)
        m._check(L.te_map_footprint_polygon_keep(m._h, C.byref(ft), 0, None, len(pts), pts.ctypes.data, len(ys), ys.ctypes.data,
                                                 None, None, te.MEM_DEVICE))

    def kept(m, n, cells):
        out = dev(2 * n * cells)
        m.get_layers(te.capi.POLYGON_LAYERS, out=out, memory=te.MEM_DEVICE)
        torch.cuda.synchronize()
        return out[:n * cells], out[n * cells:]

    def same(a, b):
        return bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))

    # ---- (a) the fleet ----
    n, size = args.maps, args.size
    cells = size * size
    g = te.Geometry.make(size, size, RES)
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    terrains = [synth.terrain(size, size, RES, 7000 + k, "mixed").astype(np.float32) for k in range(min(n, 32))]
    z = np.stack([terrains[k % len(terrains)] for k in range(n)])
    yaws = YAWS[np.arange(n) % len(YAWS)]
    batch = ctx.map()
    batch.chain_batched(g, p, n, z, positions=pos)
    loop = []
    for k in range(n):
        m = ctx.map()
        m.chain(te.Geometry.make(size, size, RES, tuple(pos[k])), p, z[k])
        loop.append(m)
    lx, lr = dev(n * cells), dev(n * cells)
    bx, br = dev(n * cells), dev(n * cells)
    cases = {
        "keep": lambda: keep(batch, yaws),
        "loop": lambda: [polygon(loop[k], yaws[k], lx[k * cells:(k + 1) * cells], lr[k * cells:(k + 1) * cells]) for k in range(n)],
        "batch": lambda: polygon(batch, YAWS[1], bx, br),
    }
    launches = {}
    for k, f in cases.items():
        n0 = ctx.stats()[0]
        f()
        launches[k] = ctx.stats()[0] - n0
    t = time_cases(torch, stream, ctx, cases, args.reps, args.warmup)
    for k in cases:
        print(json.dumps({"bench": "map_polygon", "workload": f"{n} x {size}^2 at {n} positions, {len(YAWS)} yaws", "case": k,
                          "ms": round(t[k], 3), "speedup_of_keep": round(t[k] / t["keep"], 2), "launches": int(launches[k]),
                          "gpu": gpu, "power_limit_w": power}))
    kx, kr = kept(batch, n, cells)
    at1 = np.nonzero(yaws == YAWS[1])[0]
    ok = same(kx, lx) and same(kr, lr) and same(kx, bx) and all(same(kr[k * cells:(k + 1) * cells], br[k * cells:(k + 1) * cells])
                                                               for k in at1)
    bad += not ok
    print(json.dumps({"bench": "map_polygon", "check": "(a) keep == loop (and batch at its yaw), bit for bit", "ok": ok}))
    for m in [batch] + loop:
        m.close()
    del lx, lr, bx, br, kx, kr
    torch.cuda.empty_cache()

    # ---- (b) one large map ----
    if args.big:
        size = args.big
        cells = size * size
        m = ctx.map()
        m.chain(te.Geometry.make(size, size, RES), p, synth.terrain(size, size, RES, 8100, "mixed").astype(np.float32))
        ox, orot = dev(cells), dev(cells)
        cases = {"keep": lambda: keep(m, [YAWS[1]]), "polygon": lambda: polygon(m, YAWS[1], ox, orot)}
        t = time_cases(torch, stream, ctx, cases, args.reps, args.warmup)
        for k in cases:
            print(json.dumps({"bench": "map_polygon", "workload": f"1 x {size}^2", "case": k, "ms": round(t[k], 3),
                              "keep_over_polygon": round(t["keep"] / t["polygon"], 3), "gpu": gpu, "power_limit_w": power}))
        kx, kr = kept(m, 1, cells)
        ok = same(kx, ox) and same(kr, orot)
        bad += not ok
        print(json.dumps({"bench": "map_polygon", "check": "(b) keep == te_map_footprint_polygon, bit for bit", "ok": ok}))
        m.close()
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
