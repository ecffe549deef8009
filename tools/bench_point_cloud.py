"""Point clouds of a te_map (te_map_get_point_cloud, GridMapRosConverter::toPointCloud) against the path a node has without it:
te_map_get_layers, then the compaction of the cells with a finite elevation and the interleaving of their fields into PointCloud2
records on the host (numpy) or in torch.

The published traversability map's 13 fields (upper_bound, lower_bound, uncertainty_range, x, y, z, traversability_slope, _step,
_roughness, traversability, step_footprint, slope_footprint, traversability_footprint; the two memo layers as NaN fields, point
layer elevation) on (a) one 8192² map (synth.terrain "mixed" at 0.02 m with ~1 % NaN holes, chained), (b) a fleet of 256 maps of
512² at 256 positions, chained in one batch, and (c) one selected map of that fleet (today's path reads back the whole batch: there
is no per-map read).
  - host memory: page-locked outputs; te_map_get_point_cloud (with room, so no sizing call) against te_map_get_layers + numpy; a
    host clock around whole calls, which return synchronised.
  - device memory: the library on torch's stream; te_map_get_point_cloud against te_map_get_layers + a torch boolean-mask gather
    and interleave; CUDA events.
Cases alternate; medians of --reps after --warmup.  The kernels' time (k_map_cloud_count, the cub scan, k_map_cloud_scatter) comes
from a separate torch.profiler run, the bytes/s from the byte model below.  Every cloud is checked, byte for byte, against the numpy
path.  One JSON line per case and per check, with the GPU and its power limit.

    python tools/bench_point_cloud.py [--maps 256] [--size 512] [--big 8192] [--reps 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_footprint_yaws import gpu_info  # noqa: E402
from bench_map_polygon import time_cases  # noqa: E402

RES = 0.02
PUBLISHED = ["upper_bound", "lower_bound", "uncertainty_range", "elevation", "traversability_slope", "traversability_step",
             "traversability_roughness", "traversability", "step_footprint", "slope_footprint", "traversability_footprint"]
NAN = ("step_footprint", "slope_footprint")
POINT = "elevation"
# the layers today's path reads back: every held field and the point layer, in te_layer bit order
READ = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation",
        "traversability_footprint", "upper_bound", "lower_bound", "uncertainty_range"]


def model_bytes(cells, points, fields, nbasic=0):
    """The kernels' byte model (DESIGN.md §4.8): per cell 4 B of the point layer and of each basic layer, read twice (count and
    scatter); per point 4 B of each held field other than the point layer (8 for uncertainty_range, 0 for a NaN field) read and
    point_step bytes written."""
    per_point = sum(0 if f in NAN or f == POINT else 8 if f == "uncertainty_range" else 4 for f in fields)
    step = 4 * (len(fields) + 2)
    return cells * 8 * (1 + nbasic) + points * (per_point + step)


def numpy_clouds(lay, rows, cols, g, pos, maps):
    """lay: name -> (nmaps, cols * rows) float32 (te_map_get_layers' host output, start index 0); the clouds of `maps`, back to back."""
    out = []
    i = np.arange(rows * cols) % rows
    j = np.arange(rows * cols) // rows
    for m in maps:
        k = np.nonzero(np.isfinite(lay[POINT][m]))[0]
        x = ((pos[m, 0] + (0.5 * g.length_x - 0.5 * g.resolution)) + g.resolution * (-i[k].astype(np.float64))).astype(np.float32)
        y = ((pos[m, 1] + (0.5 * g.length_y - 0.5 * g.resolution)) + g.resolution * (-j[k].astype(np.float64))).astype(np.float32)
        cols_ = []
        for f in PUBLISHED:
            if f == POINT:
                cols_ += [x.view(np.uint32), y.view(np.uint32), lay[f][m][k].view(np.uint32)]
            elif f in NAN:
                cols_.append(np.full(len(k), 0x7fc00000, np.uint32))
            else:
                cols_.append(lay[f][m][k].view(np.uint32))
        out.append(np.stack(cols_, axis=1).reshape(-1))
    return np.concatenate(out).view(np.uint8)


def torch_clouds(torch, lay, rows, cols, g, pos, maps):
    """The same in torch: one boolean mask over the maps of the call, one gather per field, one interleave."""
    sel = torch.as_tensor(maps, device="cuda")
    ok = torch.isfinite(lay[POINT][sel])
    N = rows * cols
    c = torch.arange(N, device="cuda")
    i, j = (c % rows).double(), (c // rows).double()
    p = torch.as_tensor(pos, device="cuda")[sel]
    x = ((p[:, :1] + (0.5 * g.length_x - 0.5 * g.resolution)) + g.resolution * (-i)[None]).float()
    y = ((p[:, 1:] + (0.5 * g.length_y - 0.5 * g.resolution)) + g.resolution * (-j)[None]).float()
    nan = torch.tensor(float("nan"), device="cuda")
    cols_ = []
    for f in PUBLISHED:
        if f == POINT:
            cols_ += [x[ok], y[ok], lay[f][sel][ok]]
        elif f in NAN:
            cols_.append(nan.expand(int(ok.sum())))
        else:
            cols_.append(lay[f][sel][ok])
    return torch.stack(cols_, dim=1).reshape(-1).view(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--big", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_point_cloud needs a CUDA device")
    gpu, power = gpu_info(torch)
    L = te.load_library()
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    p = te.ChainParams.yaml_defaults(0)
    fields = np.array([0 if f in NAN else 1 << te.capi.LAYER_BITS[f] for f in PUBLISHED], np.uint32)
    point = 1 << te.capi.LAYER_BITS[POINT]
    read_mask = te.capi.layer_mask(READ)
    order = te.capi.layer_order(read_mask)
    step = 4 * (len(PUBLISHED) + 2)
    bad = 0

    def emit(rec):
        rec.update(gpu=gpu, power_limit_w=power)
        print(json.dumps(rec), flush=True)

    def check(label, ok):
        nonlocal bad
        bad += not ok
        print(json.dumps({"bench": "point_cloud", "check": label, "ok": bool(ok)}), flush=True)

    def run(label, m, g, nmaps, sel):
        """sel None: every map; otherwise one selected map index."""
        rows, cols = g.rows, g.cols
        N = rows * cols
        maps = list(range(nmaps)) if sel is None else [sel]
        n = len(maps)
        idx = None if sel is None else np.array([sel], np.int32)
        nsel, iaddr = (0, None) if idx is None else (1, idx.ctypes.data)
        pos = m.positions()
        offs = np.zeros(n + 1, np.int64)
        # the clouds' size, for page-locked and device outputs of exactly that many points
        rc = L.te_map_get_point_cloud(m._h, nsel, iaddr, len(fields), fields.ctypes.data, point, 0, None, 0, offs.ctypes.data, te.MEM_HOST)
        total = int(offs[-1])
        assert rc in (0, -1) and offs[0] == 0 and total > 0
        h_cloud = torch.empty(total * step, dtype=torch.uint8, pin_memory=True).numpy()
        h_lay = torch.empty(len(order) * nmaps * N, dtype=torch.float32, pin_memory=True).numpy()
        d_cloud = torch.empty(total * step, dtype=torch.uint8, device="cuda")
        d_offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        d_lay = torch.empty(len(order) * nmaps * N, dtype=torch.float32, device="cuda")
        res = {}

        def cloud(out, o, memory):
            ctx._check(L.te_map_get_point_cloud(m._h, nsel, iaddr, len(fields), fields.ctypes.data, point, 0, te.capi._addr(out), total,
                                                te.capi._addr(o), memory))

        def today_host():
            ctx._check(L.te_map_get_layers(m._h, read_mask, h_lay.ctypes.data, te.MEM_HOST))
            lay = {f: h_lay.reshape(len(order), nmaps, N)[k] for k, f in enumerate(order)}
            res["host"] = numpy_clouds(lay, rows, cols, g, pos, maps)

        def today_device():
            ctx._check(L.te_map_get_layers(m._h, read_mask, d_lay.data_ptr(), te.MEM_DEVICE))
            lay = {f: d_lay.view(len(order), nmaps, N)[k] for k, f in enumerate(order)}
            res["device"] = torch_clouds(torch, lay, rows, cols, g, pos, maps)

        hcases = {"point_cloud host": lambda: cloud(h_cloud, offs, te.MEM_HOST), "get_layers+numpy host": today_host}
        hms = {k: [] for k in hcases}
        for rep in range(args.warmup + args.reps):
            for k in (list(hcases) if rep % 2 == 0 else list(hcases)[::-1]):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                hcases[k]()
                dt = (time.perf_counter() - t0) * 1e3
                if rep >= args.warmup:
                    hms[k].append(dt)
        hms = {k: float(np.median(v)) for k, v in hms.items()}
        dcases = {"point_cloud device": lambda: cloud(d_cloud, d_offs, te.MEM_DEVICE), "get_layers+torch device": today_device}
        dms = time_cases(torch, stream, ctx, dcases, 2 * args.reps, args.warmup)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                dcases["point_cloud device"]()
            torch.cuda.synchronize()
        names = ("k_map_cloud_count", "k_map_cloud_scatter", "DeviceScan")
        kern = {nm: [e for e in prof.key_averages() if nm in e.key] for nm in names}
        per_call = {nm: sum(e.device_time_total for e in v) / args.reps / 1e3 for nm, v in kern.items()}
        kernel_ms = sum(per_call.values())
        nbytes = model_bytes(n * N, total, PUBLISHED)
        workload = f"{label}: {len(PUBLISHED)} layers, {total} points"
        pcie = {"point_cloud host": total * step + 8 * (n + 1) + (0 if idx is None else 4 * n), "get_layers+numpy host": 4 * len(order) * nmaps * N,
                "point_cloud device": 0 if idx is None else 4 * n, "get_layers+torch device": 0}
        for k, v in list(hms.items()) + list(dms.items()):
            base = hms["point_cloud host"] if "host" in k else dms["point_cloud device"]
            rec = {"bench": "point_cloud", "workload": workload, "case": k, "ms": round(v, 4), "pcie_bytes": int(pcie[k]),
                   "speedup_of_point_cloud": round(v / base, 2)}
            if k == "point_cloud device":
                rec.update(kernel_ms=round(kernel_ms, 4), **{f"{nm}_ms": round(t, 4) for nm, t in per_call.items()},
                           model_bytes=int(nbytes), model_bytes_per_cell=round(nbytes / (n * N), 1),
                           achieved_gb_s=round(nbytes / (kernel_ms * 1e-3) / 1e9, 1))
            emit(rec)
        # byte-for-byte checks against the numpy path
        cloud(h_cloud, offs, te.MEM_HOST)
        today_host()
        want = res["host"]
        check(f"{label}: host cloud == get_layers + numpy", np.array_equal(h_cloud, want))
        cloud(d_cloud, d_offs, te.MEM_DEVICE)
        today_device()
        torch.cuda.synchronize()
        check(f"{label}: device cloud == get_layers + numpy", np.array_equal(d_cloud.cpu().numpy(), want))
        check(f"{label}: device offsets == host offsets", np.array_equal(d_offs.cpu().numpy(), offs))
        check(f"{label}: get_layers + torch == get_layers + numpy", np.array_equal(res["device"].cpu().numpy(), want))
        check(f"{label}: holes dropped", total < n * N)

    def holes(z, seed):
        z = z.astype(np.float32)
        z[np.random.default_rng(seed).random(z.shape) < 0.01] = np.nan
        return z

    def carry_bounds(m):
        e = m.get_layers(["elevation"])["elevation"]
        m.carry_layers(["upper_bound", "lower_bound"], [e + np.float32(0.05), e - np.float32(0.05)])

    # ---- (a) one large map ----
    if args.big:
        size = args.big
        g = te.Geometry.make(size, size, RES)
        m = ctx.map()
        m.chain(g, p, holes(synth.terrain(size, size, RES, 8100, "mixed"), 1))
        carry_bounds(m)
        run(f"(a) 1 x {size}^2", m, g, 1, None)
        m.close()
        torch.cuda.empty_cache()

    # ---- (b), (c) the fleet ----
    n, size = args.maps, args.size
    g = te.Geometry.make(size, size, RES)
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    terrains = [holes(synth.terrain(size, size, RES, 7000 + k, "mixed"), 2 + k) for k in range(min(n, 32))]
    batch = ctx.map()
    batch.chain_batched(g, p, n, np.stack([terrains[k % len(terrains)] for k in range(n)]), positions=pos)
    carry_bounds(batch)
    run(f"(b) {n} x {size}^2 at {n} positions", batch, g, n, None)
    run(f"(c) map {n // 2 + 1} of {n} x {size}^2", batch, g, n, n // 2 + 1)
    batch.close()
    ctx.set_stream(None)
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
