"""A fleet of robot-centric maps, each in its own circular-buffer order: one batched te_map that takes them as they are
(te_map_chain_batched_wrapped) against unwrapping them around te_map_chain_batched_at and against a loop over single-map te_maps.

256 maps of 512² cells (synth.terrain "mixed" at 0.02 m, one seed per map) at 256 positions (a 40 m grid off the cell lattice),
map m in the buffer order of a random start index (seeded), with upper_bound / lower_bound carried.  One frame of a node serving
every robot: the chain, the bounds carried, and the published layers read back to host memory in each map's buffer order
(traversability, _slope, _step, _roughness, elevation, upper_bound, lower_bound, uncertainty_range).
  - wrapped: te_map_chain_batched_wrapped + te_map_carry_layers + te_map_get_layers (one unwrap per input call, one re-wrap);
  - roll: the maps unwrapped on the host (np.roll) or, for device inputs, on the device (torch.roll), te_map_chain_batched_at +
    te_map_carry_layers + te_map_get_layers, then every output re-wrapped with np.roll;
  - loop: 256 single-map te_maps, each with its start index in g (te_map_chain + te_map_carry_layers + te_map_get_layers).
Inputs from page-locked host memory (--memory host) or device memory (--memory device).  Host clock around each frame, ended by a
synchronise, median of --reps after --warmup, the cases alternating.  Then a separate torch.profiler run of one wrapped frame
gives the time of its k_map_cut_windows launches, their bytes (8 per cell and layer moved) and their TB/s.  The wrapped frame's
outputs are checked bit for bit against the loop's.  One JSON line per case, one for the gather, one for the check, with the GPU
and its power limit.

    python tools/bench_map_wrapped.py [--maps 256] [--size 512] [--memory host|device] [--reps 5] [--warmup 1] [--seed 0]
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
BOUNDS = ["upper_bound", "lower_bound"]
PUBLISHED = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"] + BOUNDS + \
    ["uncertainty_range"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--memory", choices=("host", "device"), default="host")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    from traversability_estimation_b200.capi import MEM_DEVICE, MEM_HOST, layer_mask

    gpu, power = gpu_info(torch)
    n, size, dev = args.maps, args.size, args.memory == "device"
    g = te.Geometry.make(size, size, RES)
    p = te.ChainParams.yaml_defaults(0)
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    rng = np.random.default_rng(args.seed)
    st = np.stack([rng.integers(0, size, n), rng.integers(0, size, n)], axis=1).astype(np.int32)
    # each map's layers in its buffer order, stored as the library reads them (map after map, each column-major), page-locked
    lay = {k: torch.empty((n, size, size), dtype=torch.float32, pin_memory=True).numpy() for k in ("elevation",) + tuple(BOUNDS)}
    for m in range(n):
        z = synth.terrain(size, size, RES, 9000 + m, "mixed")
        for k, a in (("elevation", z), ("upper_bound", z + 0.05), ("lower_bound", z - 0.05)):
            lay[k][m] = np.roll(a.astype(np.float32), tuple(st[m]), axis=(0, 1)).T
    dlay = {k: torch.from_numpy(v).cuda() for k, v in lay.items()} if dev else None
    mem = MEM_DEVICE if dev else MEM_HOST
    src = dlay if dev else lay
    addr = (lambda a: a.data_ptr()) if dev else (lambda a: a.ctypes.data)  # noqa: E731
    ctx = te.Context(0)
    wrapped, rolled = ctx.map(), ctx.map()
    loop = [ctx.map() for _ in range(n)]
    gs = []
    for m in range(n):
        gm = te.Geometry.make(size, size, RES, position=tuple(pos[m]))
        gm.start_row, gm.start_col = int(st[m, 0]), int(st[m, 1])
        gs.append(gm)
    out = {c: np.empty((len(PUBLISHED), n, size, size), np.float32) for c in ("wrapped", "roll")}
    out_loop = np.empty((len(PUBLISHED), n, size, size), np.float32)

    def frame_wrapped():
        ctx._order_after_torch(mem)
        wrapped._check(wrapped._L.te_map_chain_batched_wrapped(wrapped._h, C.byref(g), C.byref(p), n, addr(src["elevation"]), None, None,
                                                               None, None, mem, pos.ctypes.data, st.ctypes.data))
        wrapped._g, wrapped._n = g, n
        ptrs = (C.c_void_p * 2)(*(addr(src[k]) for k in BOUNDS))
        wrapped._check(wrapped._L.te_map_carry_layers(wrapped._h, 0, None, layer_mask(BOUNDS), ptrs, mem))
        wrapped._check(wrapped._L.te_map_get_layers(wrapped._h, layer_mask(PUBLISHED), out["wrapped"].ctypes.data, MEM_HOST))

    def frame_roll():
        if dev:   # unwrap on the device, one torch.roll per map and layer
            un = {k: torch.stack([torch.roll(v[m], (-int(st[m, 1]), -int(st[m, 0])), dims=(0, 1)) for m in range(n)]) for k, v in dlay.items()}
            ctx._order_after_torch(MEM_DEVICE)
        else:     # unwrap on the host
            un = {k: np.stack([np.roll(v[m], (-int(st[m, 1]), -int(st[m, 0])), axis=(0, 1)) for m in range(n)]) for k, v in lay.items()}
        a = (lambda t: t.data_ptr()) if dev else (lambda t: t.ctypes.data)  # noqa: E731
        rolled._check(rolled._L.te_map_chain_batched_at(rolled._h, C.byref(g), C.byref(p), n, a(un["elevation"]), None, None, None, None,
                                                        mem, pos.ctypes.data))
        rolled._g, rolled._n = g, n
        ptrs = (C.c_void_p * 2)(*(a(un[k]) for k in BOUNDS))
        rolled._check(rolled._L.te_map_carry_layers(rolled._h, 0, None, layer_mask(BOUNDS), ptrs, mem))
        o = out["roll"]
        rolled._check(rolled._L.te_map_get_layers(rolled._h, layer_mask(PUBLISHED), o.ctypes.data, MEM_HOST))
        for k in range(len(PUBLISHED)):   # re-wrap every output on the host (column-major maps: rows are the last axis)
            for m in range(n):
                o[k, m] = np.roll(o[k, m], (int(st[m, 1]), int(st[m, 0])), axis=(0, 1))

    def frame_loop():
        for m in range(n):
            s = loop[m]
            s._check(s._L.te_map_chain(s._h, C.byref(gs[m]), C.byref(p), lay["elevation"][m].ctypes.data, None, None, None, None, MEM_HOST))
            s._g, s._n = gs[m], 1
            ptrs = (C.c_void_p * 2)(*(lay[k][m].ctypes.data for k in BOUNDS))
            s._check(s._L.te_map_carry_layers(s._h, 0, None, layer_mask(BOUNDS), ptrs, MEM_HOST))
            o = np.empty((len(PUBLISHED), size, size), np.float32)
            s._check(s._L.te_map_get_layers(s._h, layer_mask(PUBLISHED), o.ctypes.data, MEM_HOST))
            out_loop[:, m] = o

    cases = {"wrapped": frame_wrapped, "roll": frame_roll, "loop": frame_loop}
    times = {c: [] for c in cases}
    order = list(cases)
    for rep in range(args.warmup + args.reps):
        for c in order if rep % 2 == 0 else order[::-1]:
            ctx.synchronize()
            t0 = time.perf_counter()
            cases[c]()
            ctx.synchronize()
            if rep >= args.warmup:
                times[c].append(time.perf_counter() - t0)
    tw = float(np.median(times["wrapped"]))
    for c in cases:
        t = float(np.median(times[c]))
        print(json.dumps({"bench": "map_wrapped", "case": c, "memory": args.memory, "maps": n, "size": size, "ms": round(1e3 * t, 3),
                          "wrapped_speedup": round(t / tw, 2), "gpu": gpu, "power_limit": power}))
    # the gather's own time: one wrapped frame under torch.profiler
    from torch.profiler import ProfilerActivity, profile
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        frame_wrapped()
        ctx.synchronize()
    ev = [e for e in prof.events() if "k_map_cut_windows" in e.name]
    us = sum(e.device_time for e in ev) if ev else 0.0
    moved = 1 + len(BOUNDS) + len(PUBLISHED)   # layers moved per frame: elevation, the bounds, every published layer
    nbytes = 8 * moved * n * size * size
    print(json.dumps({"bench": "map_wrapped", "kernel": "k_map_cut_windows", "memory": args.memory, "launches": len(ev),
                      "us": round(us, 1), "bytes": nbytes, "TB/s": round(nbytes / (us * 1e-6) / 1e12, 3) if us else None, "gpu": gpu,
                      "power_limit": power}))
    bad = int(sum(not np.array_equal(out["wrapped"][k].view(np.uint32), out_loop[k].view(np.uint32)) for k in range(len(PUBLISHED))))
    bad_roll = int(sum(not np.array_equal(out["roll"][k].view(np.uint32), out_loop[k].view(np.uint32)) for k in range(len(PUBLISHED))))
    print(json.dumps({"bench": "map_wrapped", "check": "wrapped == loop, bit for bit", "mismatched_layers": bad,
                      "roll_mismatched_layers": bad_roll}))
    for m in [wrapped, rolled] + loop:
        m.close()
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
