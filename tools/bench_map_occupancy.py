"""Occupancy grids of a te_map's layers (te_map_get_occupancy, GridMapRosConverter::toOccupancyGrid) against the path a node has
without it: te_map_get_layers, then the same float32 conversion and reversed cell order on the host (numpy) or in torch.

The four grids of config/visualization/traversability.yaml (traversability, _slope, _step, _roughness; data_min 1, data_max 0) on
(a) one 8192² map (synth.terrain "mixed" at 0.02 m, chained), (b) a fleet of 256 maps of 512² at 256 positions, chained in one
batch, and (c) one selected map of that fleet (today's path reads back the whole batch: there is no per-map read).
  - host memory: page-locked outputs; te_map_get_occupancy against te_map_get_layers + numpy; host clock around whole calls, which
    return synchronised.
  - device memory: the library on torch's stream; te_map_get_occupancy against te_map_get_layers + torch; CUDA events.
Cases alternate; medians of --reps after --warmup.  k_map_occupancy's time comes from a separate torch.profiler run, its bytes/s
from the byte model below.  Every grid is checked, byte for byte, against the numpy conversion of te_map_get_layers' output.  One
JSON line per case and per check, with the GPU and its power limit.

    python tools/bench_map_occupancy.py [--maps 256] [--size 512] [--big 8192] [--reps 5] [--warmup 2]
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
YAML = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness"]
LO, HI = 1.0, 0.0


def model_bytes(cells, nlayers):
    """The kernel's byte model (DESIGN.md §4.7): per cell and layer 4 bytes read (8 for uncertainty_range, not used here) and 1
    written."""
    return cells * nlayers * (4 + 1)


def numpy_grids(layers):
    """layers: float32 (nl, n, cols * rows) column-major blocks -> int8 grids of the same shape (toOccupancyGrid, float32 steps)."""
    f = np.float32
    with np.errstate(all="ignore"):
        q = (layers - f(LO)) / (f(HI) - f(LO))
        nan = np.isnan(q)
        r = f(0) + np.minimum(np.maximum(f(0), np.where(nan, f(0), q)), f(1)) * f(100)
        g = np.where(nan, np.int8(-1), r.astype(np.int8))
    return g[..., ::-1]


def torch_grids(torch, layers):
    """The same in torch: one elementwise op per kernel (nothing contracted), then the reversed cell order."""
    q = (layers - LO) / (HI - LO)
    nan = torch.isnan(q)
    r = 0.0 + torch.clamp(torch.nan_to_num(q, 0.0), 0.0, 1.0) * 100.0
    return torch.where(nan, torch.tensor(-1, dtype=torch.int8, device=layers.device), r.to(torch.int8)).flip(-1)


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
        raise SystemExit("bench_map_occupancy needs a CUDA device")
    gpu, power = gpu_info(torch)
    L = te.load_library()
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    p = te.ChainParams.yaml_defaults(0)
    mask = te.capi.layer_mask(YAML)
    nl = len(YAML)
    lo, hi = np.full(nl, LO, np.float32), np.full(nl, HI, np.float32)
    bad = 0

    def emit(rec):
        rec.update(gpu=gpu, power_limit_w=power)
        print(json.dumps(rec), flush=True)

    def check(label, ok):
        nonlocal bad
        bad += not ok
        print(json.dumps({"bench": "map_occupancy", "check": label, "ok": bool(ok)}), flush=True)

    def run(label, m, g, nmaps, sel):
        """sel None: every map; otherwise one selected map index."""
        rows, cols = g.rows, g.cols
        n = nmaps if sel is None else 1
        N = rows * cols
        idx = None if sel is None else np.array([sel], np.int32)
        nsel, iaddr = (0, None) if idx is None else (1, idx.ctypes.data)
        h_occ = torch.empty(nl * n * N, dtype=torch.int8, pin_memory=True).numpy()
        h_lay = torch.empty(nl * nmaps * N, dtype=torch.float32, pin_memory=True).numpy()
        d_occ = torch.empty(nl * n * N, dtype=torch.int8, device="cuda")
        d_lay = torch.empty(nl * nmaps * N, dtype=torch.float32, device="cuda")
        res = {}

        def occ(out, memory):
            ctx._check(L.te_map_get_occupancy(m._h, nsel, iaddr, mask, lo.ctypes.data, hi.ctypes.data, te.capi._addr(out), memory))

        def today_host():
            ctx._check(L.te_map_get_layers(m._h, mask, h_lay.ctypes.data, te.MEM_HOST))
            lay = h_lay.reshape(nl, nmaps, N)
            res["host"] = numpy_grids(lay if sel is None else lay[:, sel:sel + 1])

        def today_device():
            ctx._check(L.te_map_get_layers(m._h, mask, d_lay.data_ptr(), te.MEM_DEVICE))
            lay = d_lay.view(nl, nmaps, N)
            res["device"] = torch_grids(torch, lay if sel is None else lay[:, sel:sel + 1])

        # host memory: host clock around calls that return synchronised
        hcases = {"occupancy host": lambda: occ(h_occ, te.MEM_HOST), "get_layers+numpy host": today_host}
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
        # device memory: CUDA events on the shared stream
        dcases = {"occupancy device": lambda: occ(d_occ, te.MEM_DEVICE), "get_layers+torch device": today_device}
        dms = time_cases(torch, stream, ctx, dcases, 2 * args.reps, args.warmup)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                dcases["occupancy device"]()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "k_map_occupancy" in e.key]
        count = sum(e.count for e in kern)
        kernel_ms = sum(e.device_time_total for e in kern) / max(count, 1) / 1e3
        nbytes = model_bytes(n * N, nl)
        workload = f"{label}: {nl} layers"
        pcie = {"occupancy host": nl * n * N + (0 if idx is None else 4), "get_layers+numpy host": 4 * nl * nmaps * N,
                "occupancy device": 0 if idx is None else 4, "get_layers+torch device": 0}
        for k, v in list(hms.items()) + list(dms.items()):
            base = hms["occupancy host"] if "host" in k else dms["occupancy device"]
            rec = {"bench": "map_occupancy", "workload": workload, "case": k, "ms": round(v, 4), "pcie_bytes": pcie[k],
                   "speedup_of_occupancy": round(v / base, 2)}
            if k == "occupancy device":
                rec.update(kernel_ms=round(kernel_ms, 4), kernel_launches=count, model_bytes=int(nbytes),
                           achieved_gb_s=round(nbytes / (kernel_ms * 1e-3) / 1e9, 1))
            emit(rec)
        # bit-for-bit checks against the numpy conversion of te_map_get_layers' output
        occ(h_occ, te.MEM_HOST)
        today_host()
        want = res["host"].reshape(-1)
        check(f"{label}: host occupancy == get_layers + numpy", np.array_equal(h_occ, want))
        occ(d_occ, te.MEM_DEVICE)
        today_device()
        torch.cuda.synchronize()
        check(f"{label}: device occupancy == get_layers + numpy", np.array_equal(d_occ.cpu().numpy(), want))
        check(f"{label}: get_layers + torch == get_layers + numpy", np.array_equal(res["device"].reshape(-1).cpu().numpy(), want))
        check(f"{label}: grids span -1 .. 100", len(np.unique(want)) > 50)

    # ---- (a) one large map ----
    if args.big:
        size = args.big
        g = te.Geometry.make(size, size, RES)
        m = ctx.map()
        m.chain(g, p, synth.terrain(size, size, RES, 8100, "mixed").astype(np.float32))
        run(f"(a) 1 x {size}^2", m, g, 1, None)
        m.close()
        torch.cuda.empty_cache()

    # ---- (b), (c) the fleet ----
    n, size = args.maps, args.size
    g = te.Geometry.make(size, size, RES)
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    terrains = [synth.terrain(size, size, RES, 7000 + k, "mixed").astype(np.float32) for k in range(min(n, 32))]
    batch = ctx.map()
    batch.chain_batched(g, p, n, np.stack([terrains[k % len(terrains)] for k in range(n)]), positions=pos)
    run(f"(b) {n} x {size}^2 at {n} positions", batch, g, n, None)
    run(f"(c) map {n // 2 + 1} of {n} x {size}^2", batch, g, n, n // 2 + 1)
    batch.close()
    ctx.set_stream(None)
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
