"""Footprint sweeps of a batch of maps: one te_footprint_batched / te_footprint_polygon_batched call against a loop of per-map
te_footprint2 / te_footprint_polygon calls, both in TE_MEM_DEVICE.

Input: nmaps maps of size x size cells at 0.02 m (synth.terrain "mixed", 1 % NaN holes, one seed per map), put through
te_chain_batched once; the sweeps read its layers.  Three sweeps, as BASELINE.json config 4's multi-robot / MPC-roll-out batches
would ask for them:
  - circular, radius 0.3 m, offset 0.15 m (robot_footprint_parameter.yaml);
  - circular, offset 0;
  - polygonal, the YAML footprint (0.9 x 0.6 m) at yaw 0.7854 (traversability_x and traversability_rot).
Each is timed with CUDA events around the whole batch (the batched call, or the loop of nmaps calls), median of --reps after
--warmup, the two alternating.  The context runs on torch's stream, so the loop waits for nothing but its own calls; its time
includes what the host spends per call (ctypes, argument checks, the polygon's host-side tables), which the host clock around
the enqueue (`*_enqueue_ms`) shows: where it is close to the event time, the GPU waited for the host.  Printed per batch size and
sweep, one JSON line: both medians, the kernel launches of one batch (te_get_stats), whether the two outputs are identical bit for
bit, and the GPU with its power limit.

    python tools/bench_footprint_batched.py [--maps 256 16] [--size 512] [--reps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
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
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]   # robot_footprint_parameter.yaml:3
YAW = 0.7854


def gpu_info(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def timed(torch, stream, fn, reps_ms, enqueue_ms):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    t0 = time.perf_counter()
    fn()
    enqueue_ms.append(1e3 * (time.perf_counter() - t0))
    b.record(stream)
    b.synchronize()
    reps_ms.append(a.elapsed_time(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, nargs="+", default=[256, 16])
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_footprint_batched needs a CUDA device")
    gpu, power = gpu_info(torch)
    n_rc = args.size
    g = te.Geometry.make(n_rc, n_rc, RES)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    for nmaps in args.maps:
        z = torch.from_numpy(np.stack([np.ascontiguousarray(synth.terrain(n_rc, n_rc, RES, 1000 + k, "mixed").T)
                                       for k in range(nmaps)])).cuda()
        slope, step, rough, trav = (torch.empty_like(z) for _ in range(4))
        ctx.chain_batched(g, te.ChainParams.yaml_defaults(0), nmaps, z, slope, step, rough, trav, te.MEM_DEVICE)
        for sweep in ("circle offset 0.15", "circle offset 0", "polygon yaw 0.7854"):
            fp = te.FootprintParams.yaml_defaults()
            if sweep == "circle offset 0":
                fp.offset = 0.0
            nout = 2 if sweep.startswith("polygon") else 1
            ob = [torch.empty_like(z) for _ in range(nout)]
            ol = [torch.empty_like(z) for _ in range(nout)]
            if nout == 1:
                def batched():
                    ctx.footprint_batched(g, fp, nmaps, trav, slope, step, z, ob[0], te.MEM_DEVICE)

                def loop():
                    for k in range(nmaps):
                        ctx.footprint(g, fp, trav[k], slope[k], step[k], z[k], ol[0][k], te.MEM_DEVICE)
            else:
                def batched():
                    ctx.footprint_polygon_batched(g, fp, nmaps, POLY, YAW, trav, slope, step, z, ob[0], ob[1], te.MEM_DEVICE)

                def loop():
                    for k in range(nmaps):
                        ctx.footprint_polygon(g, fp, POLY, YAW, trav[k], slope[k], step[k], z[k], ol[0][k], ol[1][k], te.MEM_DEVICE)
            launches = {}
            for name, fn in (("batched", batched), ("loop", loop)):
                l0 = ctx.stats()[0]
                fn()
                torch.cuda.synchronize()
                launches[name] = ctx.stats()[0] - l0
            for _ in range(args.warmup):
                batched()
                loop()
            torch.cuda.synchronize()
            tb, tl, hb, hl = [], [], [], []
            for _ in range(args.reps):
                timed(torch, stream, batched, tb, hb)
                timed(torch, stream, loop, tl, hl)
            same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(ob, ol))
            mb, ml = float(np.median(tb)), float(np.median(tl))
            print(json.dumps({"maps": nmaps, "size": f"{n_rc}x{n_rc}", "sweep": sweep,
                              "batched_ms": round(mb, 4), "loop_ms": round(ml, 4), "speedup": round(ml / mb, 3),
                              "batched_ms_range": [round(min(tb), 4), round(max(tb), 4)],
                              "loop_ms_range": [round(min(tl), 4), round(max(tl), 4)],
                              "batched_enqueue_ms": round(float(np.median(hb)), 4), "loop_enqueue_ms": round(float(np.median(hl)), 4),
                              "launches_batched": launches["batched"], "launches_loop": launches["loop"],
                              "bit_identical": bool(same), "gpu": gpu, "power_limit_w": power}), flush=True)
        del z, slope, step, rough, trav
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
