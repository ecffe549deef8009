"""Updating some maps of a batched te_map: te_map_chain_maps / te_map_footprint_maps against reloading or sweeping the whole batch.

A te_map holds a batch of nmaps maps of size x size cells at 0.02 m (synth.terrain "mixed", one seed per map), loaded with
te_map_chain_batched.  Timed in host memory from pinned buffers, host clock around each call and a synchronisation of the
context stream (the sweeps without an output return before their kernels end), median of --reps after --warmup, the cases
alternating:
  - te_map_chain_maps for 1, 16 and nmaps maps (a fixed permutation's first maps; no outputs, the layers stay resident), against
    te_map_chain_batched of the whole batch (what a server without te_map_chain_maps does when one map changes);
  - te_map_footprint_maps of 1 map against te_map_footprint on the batch (radius 0.3 m, offset 0.15 m; no outputs).
Then the results are checked bit for bit against the whole-batch path: after te_map_chain_maps of 16 maps on a batch, every layer
of every map and the outputs of the call equal a second te_map loaded with te_map_chain_batched on the same elevations; the
footprint_maps output of one map equals that map's layer of te_map_footprint on the whole batch.  One JSON line per case, and one
with the checks, with the GPU and its power limit.

    python tools/bench_map_update.py [--maps 256] [--size 512] [--reps 10] [--warmup 2]
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

RES = 0.02
LAYERS = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"]


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
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_update needs a CUDA device")
    gpu, power = gpu_info(torch)
    n, rc = args.maps, args.size
    g = te.Geometry.make(rc, rc, RES)
    p, fp = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    ctx = te.Context(0)
    L = te.load_library()

    def pinned(nm):   # nm maps back to back, each column-major (the library's host layout)
        return torch.empty((nm, rc, rc), dtype=torch.float32, pin_memory=True).numpy()

    old, new = pinned(n), pinned(n)
    for k in range(n):
        old[k] = synth.terrain(rc, rc, RES, 1000 + k, "mixed").T
        new[k] = synth.terrain(rc, rc, RES, 5000 + k, "mixed").T
    perm = np.random.default_rng(0).permutation(n).astype(np.int32)
    sels = [s for s in (1, 16, n) if s <= n]
    packed = {s: pinned(s) for s in sels}   # the selected maps' new elevations, in selection order
    for s in sels:
        packed[s][:] = new[perm[:s]]

    def check(code):
        if code != 0:
            raise RuntimeError(L.te_last_error().decode())

    b = ctx.map()
    b.chain_batched(g, p, n, old.transpose(0, 2, 1))
    cases = {f"chain_maps {s}": (lambda s=s: L.te_map_chain_maps(b._h, C.byref(g), C.byref(p), s, perm[:s].ctypes.data,
                                                                 packed[s].ctypes.data, None, None, None, None, te.MEM_HOST))
             for s in sels}
    cases[f"chain_batched {n}"] = lambda: L.te_map_chain_batched(b._h, C.byref(g), C.byref(p), n, old.ctypes.data, None, None, None,
                                                                 None, te.MEM_HOST)
    cases["footprint_maps 1"] = lambda: L.te_map_footprint_maps(b._h, C.byref(fp), 1, perm[:1].ctypes.data, None, te.MEM_HOST)
    cases[f"footprint {n}"] = lambda: L.te_map_footprint(b._h, C.byref(fp), None, te.MEM_HOST)
    launches = {}
    for name, fn in cases.items():
        l0 = ctx.stats()[0]
        check(fn())
        launches[name] = ctx.stats()[0] - l0
        for _ in range(args.warmup):
            check(fn())
    ctx.synchronize()
    times = {name: [] for name in cases}
    for _ in range(args.reps):
        for name, fn in cases.items():
            t0 = time.perf_counter()
            check(fn())
            ctx.synchronize()   # a sweep without an output returns before its kernels finish
            times[name].append(1e3 * (time.perf_counter() - t0))
    whole = float(np.median(times[f"chain_batched {n}"]))
    sweep = float(np.median(times[f"footprint {n}"]))
    for name, t in times.items():
        sel = int(name.split()[-1])
        ref = whole if name.startswith("chain") else sweep
        print(json.dumps({"case": name, "maps": n, "size": f"{rc}x{rc}", "median_ms": round(float(np.median(t)), 3),
                          "range_ms": [round(min(t), 3), round(max(t), 3)], "share_of_whole_batch": round(float(np.median(t)) / ref, 4),
                          "elevation_upload_mb": round(sel * rc * rc * 4 / 1e6, 1) if name.startswith("chain") else 0.0,
                          "launches": launches[name], "gpu": gpu, "power_limit_w": power}), flush=True)

    # bit-for-bit checks against the whole-batch path
    s = 16 if n >= 16 else n
    sel = perm[:s]
    mixed = pinned(n)
    mixed[:] = old
    mixed[sel] = new[sel]
    check(L.te_map_chain_batched(b._h, C.byref(g), C.byref(p), n, old.ctypes.data, None, None, None, None, te.MEM_HOST))
    outs = {k: pinned(s) for k in ("slope", "step", "roughness", "traversability")}
    check(L.te_map_chain_maps(b._h, C.byref(g), C.byref(p), s, sel.ctypes.data, packed[s].ctypes.data if s in packed else None,
                              *(outs[k].ctypes.data for k in ("slope", "step", "roughness", "traversability")), te.MEM_HOST))
    w = ctx.map()
    w.chain_batched(g, p, n, mixed.transpose(0, 2, 1))
    same_layers, same_outputs = True, True
    for name in LAYERS:
        lb = torch.empty(n * rc * rc, dtype=torch.float32, device="cuda")
        lw = torch.empty_like(lb)
        b.get_layers([name], out=lb, memory=te.MEM_DEVICE)
        w.get_layers([name], out=lw, memory=te.MEM_DEVICE)
        ctx.synchronize()
        same_layers &= bool(torch.equal(lb.view(torch.int32), lw.view(torch.int32)))
        key = {"traversability": "traversability", "traversability_slope": "slope", "traversability_step": "step",
               "traversability_roughness": "roughness"}.get(name)
        if key:
            want = lw.view(n, rc, rc)[torch.from_numpy(sel.astype(np.int64)).cuda()].cpu()
            same_outputs &= bool(torch.equal(torch.from_numpy(outs[key]).view(torch.int32), want.view(torch.int32)))
        del lb, lw
    j = int(perm[0])
    one = pinned(1)
    allc = pinned(n)
    check(L.te_map_footprint_maps(b._h, C.byref(fp), 1, perm[:1].ctypes.data, one.ctypes.data, te.MEM_HOST))
    check(L.te_map_footprint(w._h, C.byref(fp), allc.ctypes.data, te.MEM_HOST))
    same_sweep = bool(np.array_equal(one[0].view(np.uint32), allc[j].view(np.uint32)))
    print(json.dumps({"check": "bit-for-bit against the whole-batch path", "chain_maps_maps": s, "layers_equal": same_layers,
                      "outputs_equal": same_outputs, "footprint_maps_equal": same_sweep, "gpu": gpu, "power_limit_w": power}), flush=True)
    w.close()
    b.close()
    ctx.close()
    if not (same_layers and same_outputs and same_sweep):
        raise SystemExit("outputs differ from the whole-batch path")


if __name__ == "__main__":
    main()
