"""A fleet whose robots differ: every map of a batched te_map with its own footprint parameters (te_map_check_footprint_request_each,
te_map_check_footprint_request_device_each, te_map_footprint_each) against today's workaround, one te_map per parameter set.

256 maps of 512² (synth.terrain "mixed" at 0.02 m, one seed per map, layers from te_map_chain_batched), 16 planner-like paths per
map (2-8 poses 0.1-0.5 m apart, every other path circular with radius 0.3, the others the YAML rectangle at a random yaw), on
empty caches (cleared before each call, not timed).  Two parameter mixes: 4 robot types spread over the batch (map m is type
m % 4) and 256 distinct sets (every map its own offset and traversability_default).  Cases, host clock around each call (which
ends synchronised; the device entry is followed by a synchronise and the copy of its outputs to the host), median of --reps after --warmup, cases alternating:
  - each: one te_map_check_footprint_request_each call on the batch, host memory;
  - device_each: one te_map_check_footprint_request_device_each call, every request array already on the device;
  - workaround: one te_map per parameter set holding its maps, each asked for its maps' paths with
    te_map_check_footprint_request_batched, in turn;
  - uniform: te_map_check_footprint_request_batched with one parameter set for every map, and _each with that set repeated
    (no per-map table then), for the cost of the entry itself on the uniform case.
Then the sweep: te_map_footprint_each with the 4 types against 4 te_map_footprint_maps calls on the same maps, no output.  Every
case's outputs and caches are checked bit for bit against the workaround's (the sweep's against the 4 calls').  One JSON line per
case with launches per call, the GPU, its power limit and its SM clock limit.

    python tools/bench_map_each.py [--maps 256] [--size 512] [--paths-per-map 16] [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_paths import planner_paths  # noqa: E402

RES = 0.02
YAML = [(0.45, 0.30, 0.0), (0.45, -0.30, 0.0), (-0.45, -0.30, 0.0), (-0.45, 0.30, 0.0)]
LAYERS = ("traversability", "traversability_slope", "traversability_step", "elevation", "traversability_roughness")
# the four robot types of a mixed fleet: (offset, traversability_default, max_gap_width, critical_step_height, verify_roughness)
TYPES = [(0.15, 0.5, 0.3, 0.12, 0), (0.0, 0.0, 0.1, 0.05, 0), (0.3, 1.0, 0.5, 0.25, 1), (0.05, 0.3, 0.2, 0.08, 0)]


def gpu_info(torch):
    """The GPU's name, power limit (W) and SM clock limit (MHz), read in the same run as the measurement."""
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power, clock = (float(v) for v in out.splitlines()[0].split(","))
    except Exception:
        power = clock = None
    return name, power, clock


def params_of(te, offset, tdefault, gap, crit, rough):
    p = te.FootprintParams.yaml_defaults()
    p.offset, p.traversability_default, p.max_gap_width, p.critical_step_height, p.verify_roughness = offset, tdefault, gap, crit, rough
    return p


def request(rng, nmaps, per_map, n):
    """path_map, begin, poses (7 wide), radius, footprint_begin, footprint_xyz of per_map planner paths per map, map by map."""
    fy = np.asarray(YAML, np.float32)
    begin, poses, fbeg, fxyz = [0], [], [0], []
    for _ in range(nmaps):
        b, xy = planner_paths(rng, n, per_map, RES)
        yaw = rng.uniform(0, 2 * np.pi, len(xy))
        z = np.zeros(len(xy))
        poses.append(np.stack([xy[:, 0], xy[:, 1], z, z, z, np.sin(yaw / 2), np.cos(yaw / 2)], axis=1))
        begin.extend((b[1:] + begin[-1]).tolist())
        for q in range(per_map):
            if q % 2 == 0:
                fxyz.append(fy)
            fbeg.append(fbeg[-1] + (len(fy) if q % 2 == 0 else 0))
    return (np.repeat(np.arange(nmaps, dtype=np.int32), per_map), np.asarray(begin, np.int32), np.concatenate(poses),
            np.full(nmaps * per_map, 0.3), np.asarray(fbeg, np.int32), np.concatenate(fxyz))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--paths-per-map", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    name, power, clock = gpu_info(torch)
    nmaps, n, per_map = args.maps, args.size, args.paths_per_map
    g = te.Geometry.make(n, n, RES)
    ctx = te.Context(0)
    b = ctx.map()
    b.chain_batched(g, te.ChainParams.yaml_defaults(0), nmaps, np.stack([synth.terrain(n, n, RES, 5000 + k, "mixed") for k in range(nmaps)]))
    L = b.get_layers(list(LAYERS))
    pm, begin, poses, radius, fbeg, fxyz = request(np.random.default_rng(7), nmaps, per_map, n)
    mixes = {"4_types": [params_of(te, *TYPES[m % 4]) for m in range(nmaps)],
             f"{nmaps}_sets": [params_of(te, 0.01 * (m % 31), 0.25 + 0.5 * m / nmaps, 0.3, 0.12, 0) for m in range(nmaps)]}
    arrays = {k: (te.FootprintParams * nmaps)(*v) for k, v in mixes.items()}   # built once, as a node keeps its fleet's table
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    npaths = len(radius)
    D = dict(path_begin=dev(begin, np.int32), poses=dev(poses, np.float64), radius=dev(radius, np.float64),
             footprint_begin=dev(fbeg, np.int32), footprint_xyz=dev(fxyz, np.float32))
    out = dict(is_safe=torch.zeros(npaths, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"),
               area_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"))
    dpm = dev(pm, np.int32)
    max_checks = 1 << 21
    mfv = len(YAML)
    bad = 0

    def host_each(m, params, path_map, sel):
        r = (begin, poses, radius, fbeg, fxyz) if sel is None else sel
        return m.check_footprint_request_each(params, path_map, *r, max_footprint_vertices=mfv)

    def device_each(params):
        b.check_footprint_request_device(None, D["path_begin"], D["poses"], D["radius"], D["footprint_begin"], D["footprint_xyz"],
                                         max_checks=max_checks, path_map=dpm, max_footprint_vertices=mfv, params=params, **out)
        torch.cuda.synchronize()
        return tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out"))

    def emit(row):
        print(json.dumps(dict(row, gpu=name, power_limit_w=power, sm_clock_max_mhz=clock, maps=nmaps, size=f"{n}x{n}",
                              paths=npaths, poses=int(begin[-1]))), flush=True)

    def timed(cases, clears):
        """Median host-clock ms of each case over the reps, cases alternating, every case on emptied caches."""
        ts = {k: [] for k in cases}
        for rep in range(args.warmup + args.reps):
            order = list(cases) if rep % 2 == 0 else list(reversed(list(cases)))
            for k in order:
                for c in clears[k]:
                    c.clear_footprint()
                ctx.synchronize()
                t = time.perf_counter()
                cases[k]()
                ctx.synchronize()
                if rep >= args.warmup:
                    ts[k].append((time.perf_counter() - t) * 1e3)
        return {k: float(np.median(v)) for k, v in ts.items()}

    def launches(fn):
        a = ctx.stats()[0]
        fn()
        return ctx.stats()[0] - a

    for mix, params in mixes.items():
        # the workaround: one te_map per distinct parameter set, holding that set's maps
        groups = {}
        for m, p in enumerate(params):
            groups.setdefault(bytes(p), []).append(m)
        maps, parts = [], []
        for key, members in groups.items():
            w = ctx.map()
            idx = np.asarray(members)
            w.set_layers_batched(g, len(idx), *(L[k][idx] for k in LAYERS[:4]), roughness=L[LAYERS[4]][idx])
            sel = np.nonzero(np.isin(pm, idx))[0]
            local = np.searchsorted(idx, pm[sel]).astype(np.int32)
            nb = np.concatenate([[0], np.cumsum(begin[sel + 1] - begin[sel])]).astype(np.int32)
            nf = np.concatenate([[0], np.cumsum(fbeg[sel + 1] - fbeg[sel])]).astype(np.int32)
            ps = np.concatenate([poses[begin[q]:begin[q + 1]] for q in sel])
            fx = np.concatenate([fxyz[fbeg[q]:fbeg[q + 1]] for q in sel])
            maps.append((w, params[members[0]], idx))
            parts.append((sel, local, (nb, ps, radius[sel], nf, fx)))

        def workaround():
            res = [np.zeros(npaths, np.uint8), np.zeros(npaths), np.zeros(npaths)]
            for (w, p, _), (sel, local, r) in zip(maps, parts):
                for o, v in zip(res, w.check_footprint_request_batched(p, local, *r, max_footprint_vertices=mfv)):
                    o[sel] = v
            return tuple(res)

        # bit for bit: outputs and caches of the _each entries against the workaround's
        for m, _, _ in maps:
            m.clear_footprint()
        b.clear_footprint()
        want = workaround()
        got = host_each(b, params, pm, None)
        bad += sum(not np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, want))
        cb = b.get_footprint()
        for w, _, idx in maps:
            bad += int(not np.array_equal(cb[idx].view(np.uint32), w.get_footprint().reshape(cb[idx].shape).view(np.uint32)))
        b.clear_footprint()
        got = device_each(params)
        bad += sum(not np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, want))
        bad += int(not np.array_equal(b.get_footprint().view(np.uint32), cb.view(np.uint32)))
        ws = [w for w, _, _ in maps]
        arr = arrays[mix]
        cases = {"each": lambda: host_each(b, arr, pm, None), "device_each": lambda: device_each(arr), "workaround": workaround}
        counts = {}
        for k, f in cases.items():
            for c in ([b] if k != "workaround" else ws):
                c.clear_footprint()
            counts[k] = launches(f)
        t = timed(cases, {"each": [b], "device_each": [b], "workaround": ws})
        for k in cases:
            emit({"bench": "map_each", "mix": mix, "parameter_sets": len(groups), "case": k, "ms": round(t[k], 3),
                  "launches": counts[k], "speedup_vs_workaround": round(t["workaround"] / t[k], 2)})
        for w in ws:
            w.close()

    # the uniform case: the batched entry and _each with one set repeated
    p0 = mixes["4_types"][0]
    uni = (te.FootprintParams * nmaps)(*([p0] * nmaps))
    cases = {"batched": lambda: b.check_footprint_request_batched(p0, pm, begin, poses, radius, fbeg, fxyz, max_footprint_vertices=mfv),
             "each_uniform": lambda: host_each(b, uni, pm, None)}
    counts = {}
    for k, f in cases.items():
        b.clear_footprint()
        counts[k] = launches(f)
    t = timed(cases, {"batched": [b], "each_uniform": [b]})
    for k in cases:
        emit({"bench": "map_each", "mix": "uniform", "parameter_sets": 1, "case": k, "ms": round(t[k], 3), "launches": counts[k]})

    # the sweep: te_map_footprint_each with 4 types against 4 te_map_footprint_maps calls
    params = mixes["4_types"]
    arr = (te.FootprintParams * nmaps)(*params)
    sels = [np.arange(k, nmaps, 4, dtype=np.int32) for k in range(4)]

    def sweep_each():
        b._check(b._L.te_map_footprint_each(b._h, arr, 0, None, None, 0))

    def sweep_maps():
        for k, s in enumerate(sels):
            b._check(b._L.te_map_footprint_maps(b._h, C.byref(params[k]), len(s), s.ctypes.data, None, 0))

    b.clear_footprint()
    sweep_maps()
    ref = b.get_footprint()
    b.clear_footprint()
    sweep_each()
    bad += int(not np.array_equal(b.get_footprint().view(np.uint32), ref.view(np.uint32)))
    cases = {"footprint_each": sweep_each, "footprint_maps_x4": sweep_maps}
    counts = {}
    for k, f in cases.items():
        b.clear_footprint()
        counts[k] = launches(f)
    t = timed(cases, {k: [b] for k in cases})
    for k in cases:
        emit({"bench": "map_each", "mix": "4_types", "parameter_sets": 4, "case": k, "ms": round(t[k], 3), "launches": counts[k]})
    print(json.dumps({"bench": "map_each", "check": "each == workaround, bit for bit", "mismatches": int(bad)}), flush=True)
    b.close()
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
