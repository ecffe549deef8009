"""Circular footprint path checks on a 4096^2 map: the fresh-cache entry against the sweep + memoised check.

  (a) te_check_footprint_paths_fresh (TE_MEM_DEVICE): the paths straight from the chain layers;
  (b) te_footprint(0.3, 0.15) over the whole map, then te_check_footprint_paths2 (TE_MEM_DEVICE) on the swept layer.

The two answer different questions (see include/te_b200.h): (a) is what the reference's service returns on a freshly computed
map, (b) what it returns once the footprint layer has been swept.  Paths are planner-like: 2-8 poses 0.1-0.5 m apart, radius
0.3 m.  Batches of 1, 100 and 1000 paths are timed with CUDA events after warm-up; the result is one JSON line per batch size,
with the GPU name and its power limit.

    python tools/bench_paths.py [--size 4096] [--reps 20]

--footprint polygon times te_check_footprint_paths_polygon (TE_MEM_DEVICE) instead, with the YAML footprint polygon
(robot_footprint_parameter.yaml:3) and planner-like paths with a random yaw per pose, conservative off and on, and the CPU oracle
of the same call (tests/paths_oracle.cpp, all host threads, one run; it includes the oracle's whole-map
isTraversableForFilters pass, which the GPU evaluates only where a polygon looks).

--untraversable times te_check_footprint_paths_fresh2 (radius 0.3 m) and te_check_footprint_paths_polygon2 (YAML footprint) in
TE_MEM_DEVICE with compute_untraversable_polygon off and on for every path (room for 256 vertices per path), next to the CPU
oracle of the same calls (tests/paths_oracle.cpp; all host threads, one run).

--request times te_check_footprint_request against the calls a node makes without it: te_check_footprint_paths_fresh on the
circular paths and te_check_footprint_paths_polygon once per distinct footprint.  Every other path is circular (radius 0.3 m,
offset 0.15 m), the rest polygonal over 1 or 4 distinct footprints, with a random yaw per pose.  Both in TE_MEM_DEVICE (CUDA
events; the split calls write one output set each and nothing is scattered back) and in TE_MEM_HOST (host clock around the
call, which ends in a synchronise; the split calls upload the layers once per call).  Outputs of the two are compared bit for bit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def planner_paths(rng, n, npaths, res):
    half = 0.45 * n * res
    begin, poses = [0], []
    for _ in range(npaths):
        k = int(rng.integers(2, 9))
        p = [rng.uniform(-half, half, size=2)]
        for _ in range(k - 1):
            ang, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(ang), np.sin(ang)]))
        poses.extend(np.asarray(p).tolist())
        begin.append(len(poses))
    return np.asarray(begin, np.int32), np.asarray(poses, np.float64).reshape(-1, 2)


def gpu_info(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--footprint", choices=("circle", "polygon"), default="circle")
    ap.add_argument("--untraversable", action="store_true")
    ap.add_argument("--request", action="store_true")
    ap.add_argument("--map", action="store_true")
    args = ap.parse_args()
    if args.map:
        return main_map(args)
    if args.request:
        return main_request(args)
    if args.untraversable:
        return main_untraversable(args)
    if args.footprint == "polygon":
        return main_polygon(args)
    import torch
    import synth
    import traversability_estimation_b200 as te

    n, res = args.size, 0.02
    g = te.Geometry.make(n, n, res)
    fp = te.FootprintParams.yaml_defaults()            # radius 0.3, offset 0.15 (robot_footprint_parameter.yaml)
    ctx = te.Context(0)
    z = synth.terrain(n, n, res, 4096, "mixed")
    layers = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).T)).cuda()  # noqa: E731
    trav, slope, step, elev = (dev(a) for a in (layers["traversability"], layers["slope"], layers["step"], z))
    swept = torch.empty_like(trav)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    L = te.load_library()
    L.te_check_footprint_paths2.argtypes = [C.c_void_p, C.POINTER(te.Geometry), C.c_void_p, C.c_void_p, C.c_double, C.c_int32] + \
        [C.c_void_p] * 4 + [C.c_int]
    name, power = gpu_info(torch)
    rng = np.random.default_rng(1)
    for batch in (1, 100, 1000):
        begin, poses = planner_paths(rng, n, batch, res)
        db = torch.from_numpy(begin).cuda()
        dp = torch.from_numpy(poses).cuda()
        dr = torch.full((batch,), 0.3, dtype=torch.float64, device="cuda")
        safe_a = torch.empty(batch, dtype=torch.uint8, device="cuda")
        t_a = torch.empty(batch, dtype=torch.float64, device="cuda")
        safe_b, t_b = torch.empty_like(safe_a), torch.empty_like(t_a)
        torch.cuda.synchronize()

        def run_a():
            ctx.check_footprint_paths_fresh(g, fp, trav, slope, step, elev, db, dp, dr, memory=te.MEM_DEVICE, is_safe=safe_a,
                                            traversability_out=t_a)

        def run_b():
            ctx.footprint(g, fp, trav, slope, step, elev, swept, te.MEM_DEVICE)
            rc = L.te_check_footprint_paths2(ctx._h, C.byref(g), swept.data_ptr(), None, fp.traversability_default, batch,
                                             db.data_ptr(), dp.data_ptr(), safe_b.data_ptr(), t_b.data_ptr(), te.MEM_DEVICE)
            assert rc == 0, rc

        res_ms = {}
        for key, fn in (("fresh", run_a), ("sweep_then_check", run_b)):
            for _ in range(args.warmup):
                fn()
            stream.synchronize()
            ts = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            res_ms[key] = {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts))}
        stream.synchronize()
        differ = int((safe_a != safe_b).sum().item())
        print(json.dumps({"gpu": name, "power_limit_w": power, "map": f"{n}x{n}", "resolution": res, "radius": 0.3,
                          "offset": fp.offset, "paths": batch, "poses": int(begin[-1]), **res_ms,
                          "safe_fresh": int(safe_a.sum().item()), "safe_swept": int(safe_b.sum().item()), "is_safe_differs": differ}),
              flush=True)
    ctx.set_stream(None)
    ctx.close()


YAML_FOOTPRINT = [(0.45, 0.30, 0.0), (0.45, -0.30, 0.0), (-0.45, -0.30, 0.0), (-0.45, 0.30, 0.0)]  # robot_footprint_parameter.yaml:3


def main_polygon(args):
    import time
    import torch
    import synth
    import traversability_estimation_b200 as te
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import paths_oracle as po
    from oracle import binding as ob

    n, res = args.size, 0.02
    g, og = te.Geometry.make(n, n, res), ob.Geometry.make(n, n, res)
    fp, ofp = te.FootprintParams.yaml_defaults(), ob.FootprintParams.yaml_defaults()
    fxyz = np.asarray(YAML_FOOTPRINT, np.float32)
    ctx = te.Context(0)
    z = synth.terrain(n, n, res, 4096, "mixed")
    layers = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    oracle_layers = dict(traversability=layers["traversability"], slope=layers["slope"], step=layers["step"], elevation=z)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).T)).cuda()  # noqa: E731
    trav, slope, step, elev = (dev(a) for a in (layers["traversability"], layers["slope"], layers["step"], z))
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = gpu_info(torch)
    rng = np.random.default_rng(1)
    for batch in (1, 100, 1000):
        begin, xy = planner_paths(rng, n, batch, res)
        yaw = rng.uniform(0, 2 * np.pi, len(xy))
        poses = np.stack([xy[:, 0], xy[:, 1], np.zeros(len(xy)), np.zeros(len(xy)), np.zeros(len(xy)), np.sin(yaw / 2),
                          np.cos(yaw / 2)], axis=1)
        db, dp = torch.from_numpy(begin).cuda(), torch.from_numpy(poses).cuda()
        for conservative in (0, 1):
            cons = np.full(batch, conservative, np.uint8)
            dc = torch.from_numpy(cons).cuda()
            safe = torch.empty(batch, dtype=torch.uint8, device="cuda")
            tout = torch.empty(batch, dtype=torch.float64, device="cuda")
            aout = torch.empty(batch, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()

            def run():
                ctx.check_footprint_paths_polygon(g, fp, trav, slope, step, elev, fxyz, db, dp, conservative=dc if conservative else None,
                                                  memory=te.MEM_DEVICE, is_safe=safe, traversability_out=tout, area_out=aout)

            for _ in range(args.warmup):
                run()
            stream.synchronize()
            ts = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run()
                e1.record(stream)
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            t0 = time.perf_counter()
            want = po.check_request(og, ofp, oracle_layers, begin, poses, footprint_xyz=fxyz,
                                    conservative=cons if conservative else None)[:3]
            cpu_ms = (time.perf_counter() - t0) * 1e3
            got = (safe.cpu().numpy(), tout.cpu().numpy(), aout.cpu().numpy())
            same = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, want))
            print(json.dumps({"gpu": name, "power_limit_w": power, "map": f"{n}x{n}", "resolution": res, "footprint": "yaml_polygon",
                              "paths": batch, "poses": int(begin[-1]), "conservative": conservative,
                              "gpu_median_ms": float(np.median(ts)), "gpu_min_ms": float(np.min(ts)),
                              "cpu_oracle_ms": cpu_ms, "cpu_threads": os.cpu_count(), "safe": int(got[0].sum()),
                              "matches_oracle": bool(same)}), flush=True)
    ctx.set_stream(None)
    ctx.close()


def main_untraversable(args):
    import time
    import torch
    import synth
    import traversability_estimation_b200 as te
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import paths_oracle as po
    from oracle import binding as ob

    n, res, cap = args.size, 0.02, 256
    g, og = te.Geometry.make(n, n, res), ob.Geometry.make(n, n, res)
    fp, ofp = te.FootprintParams.yaml_defaults(), ob.FootprintParams.yaml_defaults()
    fxyz = np.asarray(YAML_FOOTPRINT, np.float32)
    ctx = te.Context(0)
    z = synth.terrain(n, n, res, 4096, "mixed")
    layers = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    oracle_layers = dict(traversability=layers["traversability"], slope=layers["slope"], step=layers["step"], elevation=z)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).T)).cuda()  # noqa: E731
    trav, slope, step, elev = (dev(a) for a in (layers["traversability"], layers["slope"], layers["step"], z))
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = gpu_info(torch)
    rng = np.random.default_rng(1)

    def timed(run):
        for _ in range(args.warmup):
            run()
        stream.synchronize()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            run()
            e1.record(stream)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts)), float(np.min(ts))

    for batch in (1, 100, 1000):
        begin, xy = planner_paths(rng, n, batch, res)
        yaw = rng.uniform(0, 2 * np.pi, len(xy))
        poses = np.stack([xy[:, 0], xy[:, 1], np.zeros(len(xy)), np.zeros(len(xy)), np.zeros(len(xy)), np.sin(yaw / 2),
                          np.cos(yaw / 2)], axis=1)
        db, dxy, dp = (torch.from_numpy(a).cuda() for a in (begin, xy, poses))
        dr = torch.full((batch,), 0.3, dtype=torch.float64, device="cuda")
        safe = torch.empty(batch, dtype=torch.uint8, device="cuda")
        tout = torch.empty(batch, dtype=torch.float64, device="cuda")
        aout = torch.empty(batch, dtype=torch.float64, device="cuda")
        cnt = torch.empty(batch, dtype=torch.int32, device="cuda")
        uxy = torch.empty((batch, cap, 2), dtype=torch.float64, device="cuda")
        for cup_on in (0, 1):
            cup = np.full(batch, cup_on, np.uint8)
            dcup = torch.from_numpy(cup).cuda()
            torch.cuda.synchronize()
            kw = dict(memory=te.MEM_DEVICE, is_safe=safe, traversability_out=tout, untraversable_capacity=cap, untraversable_count=cnt,
                      untraversable_xy=uxy)
            for kind in ("circle", "polygon"):
                if kind == "circle":
                    def run():
                        ctx.check_footprint_paths_fresh(g, fp, trav, slope, step, elev, db, dxy, dr, compute_untraversable_polygon=dcup,
                                                        **kw)
                else:
                    def run():
                        ctx.check_footprint_paths_polygon(g, fp, trav, slope, step, elev, fxyz, db, dp, compute_untraversable_polygon=dcup,
                                                          area_out=aout, **kw)
                med, mn = timed(run)
                t0 = time.perf_counter()
                if kind == "circle":
                    want = po.check_request(og, ofp, oracle_layers, begin, xy, 0.3, cup=cup, capacity=cap)
                else:
                    want = po.check_request(og, ofp, oracle_layers, begin, poses, footprint_xyz=fxyz, cup=cup, capacity=cap)
                want_counts = want[3]
                cpu_ms = (time.perf_counter() - t0) * 1e3
                got = cnt.cpu().numpy()
                print(json.dumps({"gpu": name, "power_limit_w": power, "map": f"{n}x{n}", "resolution": res, "footprint": kind,
                                  "paths": batch, "poses": int(begin[-1]), "compute_untraversable_polygon": cup_on,
                                  "gpu_median_ms": med, "gpu_min_ms": mn, "cpu_oracle_ms": cpu_ms, "cpu_threads": os.cpu_count(),
                                  "safe": int(safe.sum().item()), "polygons": int((got > 0).sum()),
                                  "counts_match_oracle": bool(np.array_equal(got, want_counts))}), flush=True)
    ctx.set_stream(None)
    ctx.close()


def request_footprints(k):
    """k distinct footprints (1 or 4): the YAML rectangle, then a smaller rectangle, a hexagon and an octagon."""
    ring = lambda m, r: [(r * np.cos(2 * np.pi * i / m), r * np.sin(2 * np.pi * i / m), 0.0) for i in range(m)]  # noqa: E731
    fps = [YAML_FOOTPRINT, [(0.35, 0.25, 0.0), (0.35, -0.25, 0.0), (-0.35, -0.25, 0.0), (-0.35, 0.25, 0.0)], ring(6, 0.4), ring(8, 0.45)]
    return [np.asarray(f, np.float32) for f in fps[:k]]


def main_request(args):
    import time
    import torch
    import synth
    import traversability_estimation_b200 as te

    n, res = args.size, 0.02
    g = te.Geometry.make(n, n, res)
    fp = te.FootprintParams.yaml_defaults()            # offset 0.15
    ctx = te.Context(0)
    z = synth.terrain(n, n, res, 4096, "mixed")
    layers = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    host = {k: np.asfortranarray(a, np.float32) for k, a in (("trav", layers["traversability"]), ("slope", layers["slope"]),
                                                             ("step", layers["step"]), ("elev", z))}
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731
    dl = {k: dev(a) for k, a in host.items()}
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = gpu_info(torch)
    rng = np.random.default_rng(1)

    def timed(run, device):
        for _ in range(args.warmup):
            run()
        stream.synchronize()
        ts = []
        for _ in range(args.reps):
            if device:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run()
                e1.record(stream)
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            else:   # host memory: every call ends in a synchronise of the context stream
                t0 = time.perf_counter()
                run()
                ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), float(np.min(ts))

    for batch in (1, 100, 1000):
        begin, xy = planner_paths(rng, n, batch, res)
        yaw = rng.uniform(0, 2 * np.pi, len(xy))
        poses = np.stack([xy[:, 0], xy[:, 1], np.zeros(len(xy)), np.zeros(len(xy)), np.zeros(len(xy)), np.sin(yaw / 2),
                          np.cos(yaw / 2)], axis=1)
        for nfps in (1, 4):
            fps = request_footprints(nfps)
            kind = np.where(np.arange(batch) % 2 == 1, -1, (np.arange(batch) // 2) % nfps)   # odd paths circular
            fbeg = np.concatenate([[0], np.cumsum([0 if k < 0 else len(fps[k]) for k in kind])]).astype(np.int32)
            fxyz = np.concatenate([fps[k] for k in kind if k >= 0] + [np.zeros((0, 3), np.float32)])
            radius = np.full(batch, 0.3)
            groups = []   # (path indices, path_begin, poses) of the calls a node makes today: circular first, then per footprint
            for k in range(-1, nfps):
                idx = np.nonzero(kind == k)[0]
                if len(idx):
                    b = np.concatenate([[0], np.cumsum(begin[idx + 1] - begin[idx])]).astype(np.int32)
                    groups.append((k, idx, b, np.concatenate([poses[begin[q]:begin[q + 1]] for q in idx])))
            row = {"gpu": name, "power_limit_w": power, "map": f"{n}x{n}", "resolution": res, "paths": batch,
                   "poses": int(begin[-1]), "circular": int((kind < 0).sum()), "distinct_footprints": nfps, "calls_split": len(groups)}

            # host memory: numpy in, numpy out
            def req_host():
                return ctx.check_footprint_request(g, fp, host["trav"], host["slope"], host["step"], host["elev"], begin, poses,
                                                   radius, fbeg, fxyz)

            def split_host():
                out = [np.zeros(batch, np.uint8), np.zeros(batch), np.zeros(batch)]
                for k, idx, b, p in groups:
                    if k < 0:
                        r = ctx.check_footprint_paths_fresh(g, fp, host["trav"], host["slope"], host["step"], host["elev"], b,
                                                            p[:, :2].copy(), radius[idx])
                        r = (r[0], r[1], np.zeros(len(idx)))
                    else:
                        r = ctx.check_footprint_paths_polygon(g, fp, host["trav"], host["slope"], host["step"], host["elev"], fps[k], b, p)
                    for o, v in zip(out, r):
                        o[idx] = v
                return out

            got, want = req_host(), split_host()
            row["identical"] = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, want))
            row["host_request_ms"], row["host_request_min_ms"] = timed(req_host, False)
            row["host_split_ms"], row["host_split_min_ms"] = timed(split_host, False)

            # device memory: tensors in, preallocated tensors out; the split writes one output set per call (no scatter timed)
            d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
            db, dp, dr, dfb, dfx = d(begin), d(poses), d(radius), d(fbeg), d(fxyz)
            outs = lambda m: dict(is_safe=torch.empty(m, dtype=torch.uint8, device="cuda"),  # noqa: E731
                                  traversability_out=torch.empty(m, dtype=torch.float64, device="cuda"))
            rout = dict(outs(batch), area_out=torch.empty(batch, dtype=torch.float64, device="cuda"))
            dgroups = []
            for k, idx, b, p in groups:
                o = outs(len(idx))
                if k >= 0:
                    o["area_out"] = torch.empty(len(idx), dtype=torch.float64, device="cuda")
                dgroups.append((k, d(b), d(p[:, :2]) if k < 0 else d(p), d(radius[idx]), o))
            mfv = max([len(f) for f in fps])
            torch.cuda.synchronize()

            def req_dev():
                ctx.check_footprint_request(g, fp, dl["trav"], dl["slope"], dl["step"], dl["elev"], db, dp, dr, dfb, dfx,
                                            max_footprint_vertices=mfv, memory=te.MEM_DEVICE, **rout)

            def split_dev():
                for k, b, p, r, o in dgroups:
                    if k < 0:
                        ctx.check_footprint_paths_fresh(g, fp, dl["trav"], dl["slope"], dl["step"], dl["elev"], b, p, r,
                                                        memory=te.MEM_DEVICE, **o)
                    else:
                        ctx.check_footprint_paths_polygon(g, fp, dl["trav"], dl["slope"], dl["step"], dl["elev"], fps[k], b, p,
                                                          memory=te.MEM_DEVICE, **o)

            row["device_request_ms"], row["device_request_min_ms"] = timed(req_dev, True)
            row["device_split_ms"], row["device_split_min_ms"] = timed(split_dev, True)
            stream.synchronize()
            dev_got = [rout[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out")]
            row["device_identical"] = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(dev_got, want))
            print(json.dumps(row), flush=True)
    ctx.set_stream(None)
    ctx.close()


def main_map(args):
    """te_map_check_footprint_request against te_check_footprint_request, both in host memory, on planner-like batches with every
    other path circular (radius 0.3) and the YAML footprint on the others.  `map_cleared_ms`: the map request on an empty cache
    (te_map_clear_footprint before each call, not timed); `map_repeat_ms`: the same request again on the cache it left.  The
    device time is the sum of the map request's kernels (torch.profiler, CUDA activities) per call."""
    import time
    import torch
    import synth
    import traversability_estimation_b200 as te

    n, res = args.size, 0.02
    g = te.Geometry.make(n, n, res)
    fp = te.FootprintParams.yaml_defaults()
    ctx = te.Context(0)
    z = synth.terrain(n, n, res, 4096, "mixed")
    layers = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    host = {k: np.asfortranarray(a, np.float32) for k, a in (("trav", layers["traversability"]), ("slope", layers["slope"]),
                                                             ("step", layers["step"]), ("elev", z))}
    m = ctx.map()
    t0 = time.perf_counter()
    m.set_layers(g, host["trav"], host["slope"], host["step"], host["elev"])
    set_ms = (time.perf_counter() - t0) * 1e3
    name, power = gpu_info(torch)
    rng = np.random.default_rng(1)

    def timed(run, before=None):
        for _ in range(args.warmup):
            if before:
                before()
            run()
        ts = []
        for _ in range(args.reps):
            if before:
                before()
            t = time.perf_counter()
            run()
            ts.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ts)), float(np.min(ts))

    for batch in (1, 100, 1000):
        begin, xy = planner_paths(rng, n, batch, res)
        yaw = rng.uniform(0, 2 * np.pi, len(xy))
        poses = np.stack([xy[:, 0], xy[:, 1], np.zeros(len(xy)), np.zeros(len(xy)), np.zeros(len(xy)), np.sin(yaw / 2),
                          np.cos(yaw / 2)], axis=1)
        fps = request_footprints(1)
        kind = np.where(np.arange(batch) % 2 == 1, -1, 0)
        fbeg = np.concatenate([[0], np.cumsum([0 if k < 0 else len(fps[0]) for k in kind])]).astype(np.int32)
        fxyz = np.concatenate([fps[0] for k in kind if k >= 0] + [np.zeros((0, 3), np.float32)])
        radius = np.full(batch, 0.3)

        def stateless():
            return ctx.check_footprint_request(g, fp, host["trav"], host["slope"], host["step"], host["elev"], begin, poses, radius,
                                               fbeg, fxyz)

        def on_map():
            return m.check_footprint_request(fp, begin, poses, radius, fbeg, fxyz)

        m.clear_footprint()
        first = on_map()
        cand, keys, stored = m.request_stats()
        row = {"gpu": name, "power_limit_w": power, "map": f"{n}x{n}", "resolution": res, "paths": batch, "poses": int(begin[-1]),
               "circular": int((kind < 0).sum()), "candidate_checks": cand, "distinct_keys": keys, "cells_stored": stored,
               "set_layers_ms": round(set_ms, 2)}
        want = stateless()
        # equal unless paths of the batch check the same cells: the map then answers as the reference does, the stateless entry
        # on an empty cache per path
        row["equal_to_stateless"] = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(first, want))
        row["stateless_ms"], row["stateless_min_ms"] = timed(stateless)
        row["map_cleared_ms"], row["map_cleared_min_ms"] = timed(on_map, m.clear_footprint)
        row["map_repeat_ms"], row["map_repeat_min_ms"] = timed(on_map)
        for label, before in (("cleared", m.clear_footprint), ("repeat", None)):
            reps = 5
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    if before:
                        before()
                    on_map()
            ev = [e for e in prof.key_averages() if "k_map_" in e.key or "k_check_polygon" in e.key]
            row[f"map_{label}_kernels_ms"] = round(sum(e.self_device_time_total for e in ev) / 1e3 / reps, 4)
        print(json.dumps(row), flush=True)
    m.close()
    ctx.close()


if __name__ == "__main__":
    main()
