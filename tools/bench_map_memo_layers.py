"""What recording slope_footprint / step_footprint / roughness_footprint costs the te_map requests and sweep, and what reading
them costs.

256 maps of 512² (synth.terrain "mixed" at 0.02 m, one seed per map, layers from te_map_chain_batched), 16 planner-like paths per
map (2-8 poses 0.1-0.5 m apart, every other path circular with radius 0.3, the others the YAML rectangle at a random yaw), the YAML
footprint parameters, on empty caches (te_map_clear_footprint before each call, not timed).  Cases, host clock around each call
(which ends synchronised; the device entry is followed by a synchronise), median of --reps after --warmup, cases alternating:
  - request: te_map_check_footprint_request_batched, host memory;
  - device: te_map_check_footprint_request_device, every request array already on the device;
  - footprint: te_map_footprint on the whole batch, no output;
  - footprint_after_request: the same sweep on the caches the host request left (the request not timed), the node's
    request-then-sweep sequence;
  - get_layers_8192: te_map_get_layers of the three layers of one 8192² map, after a sweep, into a device tensor (--big 0 skips
    it, as a run on a library without these layers must).
One JSON line per case with the GPU, its power limit and its SM clock limit, and one with the crc32 of every output and cache, so
that a run on the library before the change (TE_B200_LIBRARY=<its libte_b200.so>) can be checked against a run after it: the
recording must change neither.

    python tools/bench_map_memo_layers.py [--maps 256] [--size 512] [--paths-per-map 16] [--reps 10] [--warmup 2] [--big 8192]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_map_each import RES, YAML, gpu_info, request  # noqa: E402

MEMO_LAYERS = ["slope_footprint", "step_footprint", "roughness_footprint"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--paths-per-map", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--big", type=int, default=8192)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    name, power, clock = gpu_info(torch)
    lib = os.environ.get("TE_B200_LIBRARY", "in-tree")
    nmaps, n, per_map = args.maps, args.size, args.paths_per_map
    g = te.Geometry.make(n, n, RES)
    ctx = te.Context(0)
    b = ctx.map()
    b.chain_batched(g, te.ChainParams.yaml_defaults(0), nmaps, np.stack([synth.terrain(n, n, RES, 5000 + k, "mixed") for k in range(nmaps)]))
    pm, begin, poses, radius, fbeg, fxyz = request(np.random.default_rng(7), nmaps, per_map, n)
    fp = te.FootprintParams.yaml_defaults()
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    npaths = len(radius)
    D = dict(path_begin=dev(begin, np.int32), poses=dev(poses, np.float64), radius=dev(radius, np.float64),
             footprint_begin=dev(fbeg, np.int32), footprint_xyz=dev(fxyz, np.float32))
    out = dict(is_safe=torch.zeros(npaths, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"),
               area_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"))
    dpm = dev(pm, np.int32)
    mfv = len(YAML)

    def host_request():
        return b.check_footprint_request_batched(fp, pm, begin, poses, radius, fbeg, fxyz, max_footprint_vertices=mfv)

    def device_request():
        b.check_footprint_request_device(fp, D["path_begin"], D["poses"], D["radius"], D["footprint_begin"], D["footprint_xyz"],
                                         max_checks=1 << 21, path_map=dpm, max_footprint_vertices=mfv, **out)
        torch.cuda.synchronize()

    def sweep():
        b._check(b._L.te_map_footprint(b._h, te.capi.C.byref(fp), None, 0))

    def emit(row):
        print(json.dumps(dict(row, gpu=name, power_limit_w=power, sm_clock_max_mhz=clock, library=lib)), flush=True)

    # the outputs each case leaves, as crc32s
    crc = lambda *arrs: "%08x" % zlib.crc32(b"".join(np.ascontiguousarray(a).tobytes() for a in arrs))  # noqa: E731
    sums = {}
    b.clear_footprint()
    sums["request"] = crc(*host_request(), b.get_footprint(), b.get_memo(), np.asarray(b.request_stats()))
    b.clear_footprint()
    device_request()
    sums["device"] = crc(*(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out")), b.get_footprint(), b.get_memo(),
                         np.asarray(b.request_stats()))
    b.clear_footprint()
    sweep()
    sums["footprint"] = crc(b.get_footprint())

    b.clear_footprint()
    host_request()
    sweep()
    sums["footprint_after_request"] = crc(b.get_footprint())

    cases = {"request": host_request, "device": device_request, "footprint": sweep, "footprint_after_request": sweep}
    before = {"footprint_after_request": host_request}   # untimed, after the clear
    ts = {k: [] for k in cases}
    for rep in range(args.warmup + args.reps):
        for k in (list(cases) if rep % 2 == 0 else list(reversed(list(cases)))):
            b.clear_footprint()
            if k in before:
                before[k]()
            ctx.synchronize()
            t = time.perf_counter()
            cases[k]()
            ctx.synchronize()
            if rep >= args.warmup:
                ts[k].append((time.perf_counter() - t) * 1e3)
    for k in cases:
        emit({"bench": "map_memo_layers", "case": k, "maps": nmaps, "size": f"{n}x{n}", "paths": npaths,
              "ms": round(float(np.median(ts[k])), 3)})
    b.close()

    if args.big > 0:
        gb = te.Geometry.make(args.big, args.big, RES)
        m = ctx.map()
        z = np.asfortranarray(synth.terrain(args.big, args.big, RES, 6000, "mixed"), dtype=np.float32)
        m.chain(gb, te.ChainParams.yaml_defaults(0), z)
        m.footprint(fp)
        dst = torch.empty(3 * args.big * args.big, dtype=torch.float32, device="cuda")
        tl = []
        for rep in range(args.warmup + args.reps):
            ctx.synchronize()
            t = time.perf_counter()
            m.get_layers(MEMO_LAYERS, out=dst, memory=1)
            ctx.synchronize()
            if rep >= args.warmup:
                tl.append((time.perf_counter() - t) * 1e3)
        emit({"bench": "map_memo_layers", "case": "get_layers_8192", "size": f"{args.big}x{args.big}", "ms": round(float(np.median(tl)), 3)})
        m.close()
    print(json.dumps({"bench": "map_memo_layers", "library": lib, "output_crc32": sums}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
