"""A fleet of maps at their own positions: one batched te_map (te_map_chain_batched_at) against a loop over single-map te_maps.

256 maps of 512² cells (synth.terrain "mixed" at 0.02 m, one seed per map), map m centred at its own position (a 40 m grid of
robots, off the cell lattice so that positions are not whole cells apart).  One frame of a node serving every robot:
  - chain: computeTraversability of every map (elevation uploaded from page-locked host memory, no outputs);
  - footprint: traversabilityFootprint(radius, offset) on every map's cache (te_map_footprint, no output);
  - submaps: one 2 m x 2 m GetGridMap window of traversability around every robot (te_map_get_submaps(_batched), host memory).
"batch" runs each step once on the batch; "loop" runs it once per map on 256 single-map te_maps.  Host clock around each step,
ended by a synchronise, median of --reps after --warmup, the two cases alternating.  Then the batch's layers, caches and submaps
are checked bit for bit against the loop's.  One JSON line per case and step, and one for the check, with the GPU and its power
limit.  Footprint path requests are not timed in this frame yet.

    python tools/bench_map_positions.py [--maps 256] [--size 512] [--reps 5] [--warmup 1]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    from traversability_estimation_b200.capi import MEM_HOST

    gpu, power = gpu_info(torch)
    n, size = args.maps, args.size
    g = te.Geometry.make(size, size, RES)
    p = te.ChainParams.yaml_defaults(0)
    ft = te.FootprintParams.yaml_defaults()
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    gs = [te.Geometry.make(size, size, RES, position=tuple(c)) for c in pos]
    # page-locked, in the library's layout (map after map, each column-major): neither case copies on the host
    zb = torch.empty((n, size, size), dtype=torch.float32, pin_memory=True).numpy()
    for k in range(n):
        zb[k] = synth.terrain(size, size, RES, 9000 + k, "mixed").T
    zc = [zb[k].T for k in range(n)]
    ctx = te.Context(0)
    batch = ctx.map()
    batch._g, batch._n = g, n
    loop = [ctx.map() for _ in range(n)]
    win = pos.copy()
    ln = np.full((n, 2), 2.0)
    wmap = np.arange(n, dtype=np.int32)

    steps = {
        "chain": (lambda: batch._check(batch._L.te_map_chain_batched_at(batch._h, C.byref(g), C.byref(p), n, zb.ctypes.data, None, None,
                                                                        None, None, MEM_HOST, pos.ctypes.data)),
                  lambda: [loop[k].chain(gs[k], p, zc[k]) for k in range(n)]),
        "footprint": (lambda: batch._check(batch._L.te_map_footprint(batch._h, C.byref(ft), None, MEM_HOST)),
                      lambda: [loop[k]._check(loop[k]._L.te_map_footprint(loop[k]._h, C.byref(ft), None, MEM_HOST))
                               for k in range(n)]),
        "submaps": (lambda: batch.get_submaps_batched(wmap, win, ln, ["traversability"]),
                    lambda: [loop[k].get_submaps(win[k:k + 1], ln[k:k + 1], ["traversability"]) for k in range(n)]),
    }
    times = {(s, c): [] for s in steps for c in ("batch", "loop")}
    for rep in range(args.warmup + args.reps):
        for s, (fb, fl) in steps.items():
            for c, f in (("batch", fb), ("loop", fl)) if rep % 2 == 0 else (("loop", fl), ("batch", fb)):
                ctx.synchronize()
                t0 = time.perf_counter()
                f()
                ctx.synchronize()
                if rep >= args.warmup:
                    times[(s, c)].append(time.perf_counter() - t0)
    for s in steps:
        tb, tl = float(np.median(times[(s, "batch")])), float(np.median(times[(s, "loop")]))
        for c, t in (("batch", tb), ("loop", tl)):
            print(json.dumps({"bench": "map_positions", "step": s, "case": c, "maps": n, "size": size, "ms": round(1e3 * t, 3),
                              "speedup_vs_loop": round(tl / tb, 2) if c == "batch" else 1.0, "gpu": gpu, "power_limit": power}))
    # bit for bit: layers, caches and submaps of the batch against the loop's
    names = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation",
             "traversability_footprint"]
    hb = batch.get_layers(names)
    bad = 0
    sb = batch.get_submaps_batched(wmap, win, ln, ["traversability"])
    for k in range(n):
        hl = loop[k].get_layers(names)
        bad += sum(not np.array_equal(hb[x][k].view(np.uint32), hl[x].view(np.uint32)) for x in names)
        (_, sl), = loop[k].get_submaps(win[k:k + 1], ln[k:k + 1], ["traversability"])
        bad += not np.array_equal(sb[k][1]["traversability"].view(np.uint32), sl["traversability"].view(np.uint32))
    print(json.dumps({"bench": "map_positions", "check": "batch == loop, bit for bit", "mismatches": int(bad)}))
    for m in [batch] + loop:
        m.close()
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
