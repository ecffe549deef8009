"""Polygonal footprint sweep at a list of headings: one te_footprint_polygon_yaws call against a loop of per-heading calls, both in
TE_MEM_DEVICE on one stream.

Input: synth.terrain ("mixed", 1 % NaN holes) at 0.02 m, put through te_chain (one map) or te_chain_batched (a batch) once; the
sweeps read its layers.  Footprint: the YAML rectangle (robot_footprint_parameter.yaml:3, 0.9 x 0.6 m); nyaws headings evenly
spaced over [0, 2 pi), as a lattice / hybrid-A* planner's heading bins.  Workloads:
  - one 4096 x 4096 map with nyaws = 2, 8, 16, 36, 72 (--yaws);
  - 256 maps of 512 x 512 with nyaws = 8 (--batch-maps, --batch-yaws).
The loop keeps traversability_rot of one te_footprint_polygon call per heading (te_footprint_polygon_batched for the batch: one
call per heading over all maps).  Each is timed with CUDA events around the whole call or loop, median of --reps after --warmup,
the two alternating.  Printed per workload, one JSON line: both medians and ranges, the host clock around the enqueue, the kernel
launches of one call and of one loop (te_get_stats), whether every stacked layer equals the loop's bit for bit, the achieved
bytes/s of the stacked call and its share of the H100 SXM data-sheet 3.35 TB/s, and the GPU with its power limit.

Byte model (the least the sweep must move): the four input layers it reads (traversability, slope, step, elevation: 16 B per
cell, once) plus the float32 output (4 B per cell and heading).  The predicate bytes, the staged tiles and the halo re-reads are
not counted.

--profile adds one torch.profiler run of one stacked call and one loop per workload, after the timing, and prints their kernel
time per kernel name (a separate run: tracing slows the host).

--reduce compares, instead, the per-cell reductions over the headings that a planner keeps (worst heading, best heading and its
index): one te_footprint_polygon_yaws_reduce call against one te_footprint_polygon_yaws call followed by torch amin / amax /
argmax over the stack.  Both run in TE_MEM_DEVICE (torch on the GPU) and in TE_MEM_HOST (numpy outputs; the stack's reduction
then runs in torch on the host, where such a caller has it), the two variants alternating; --host-reps sets the host repetitions.
Workloads: 4096 x 4096 with nyaws = 16, 36, 72 (--yaws defaults to these) and 256 maps of 512 x 512 with nyaws = 8.  Each JSON
line also gives whether the two agree bit for bit, the output bytes each variant allocates on the device and moves to the host,
and the byte model of the reduce call: the same 16 B of input per cell plus 12 B of output (worst, best, best_yaw).

    python tools/bench_footprint_yaws.py [--yaws 2 8 16 36 72] [--size 4096] [--batch-maps 256] [--batch-size 512] [--batch-yaws 8]
                                         [--reps 20] [--warmup 3] [--profile] [--reduce [--host-reps 3]]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import re
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
HBM_BYTES_PER_S = 3.35e12                                              # H100 SXM data sheet
IN_BYTES_PER_CELL, OUT_BYTES_PER_CELL_YAW = 16, 4
REDUCE_OUT_BYTES_PER_CELL = 12                                         # worst, best (float32) and best_yaw (int32)


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


def kernel_times(torch, fn):
    """Kernel and copy time in ms per name of one run of fn (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = e.self_device_time_total / 1e3
        if t > 0:
            m = re.search(r"\bk_\w+", e.key)
            key = m.group(0) if m else e.key[:60]
            out[key] = out.get(key, 0.0) + t
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def layers(torch, te, ctx, nmaps, size):
    """Geometry and the device layers (z, slope, step, trav) of nmaps terrain maps, each (nmaps, cols, rows)."""
    import synth
    g = te.Geometry.make(size, size, RES)
    z = torch.from_numpy(np.stack([np.ascontiguousarray(synth.terrain(size, size, RES, 1000 + k, "mixed").T)
                                   for k in range(nmaps)])).cuda()
    slope, step, rough, trav = (torch.empty_like(z) for _ in range(4))
    if nmaps == 1:
        ctx.chain(g, te.ChainParams.yaml_defaults(0), z[0], slope[0], step[0], rough[0], trav[0], te.MEM_DEVICE)
    else:
        ctx.chain_batched(g, te.ChainParams.yaml_defaults(0), nmaps, z, slope, step, rough, trav, te.MEM_DEVICE)
    return g, z, slope, step, trav


def run(args, torch, te, ctx, stream, gpu, power, nmaps, size, yaw_counts):
    g, z, slope, step, trav = layers(torch, te, ctx, nmaps, size)
    fp = te.FootprintParams.yaml_defaults()
    scratch_x = torch.empty_like(z)
    for nyaws in yaw_counts:
        yaws = [2.0 * math.pi * k / nyaws for k in range(nyaws)]
        stacked_out = torch.empty((nyaws,) + tuple(z.shape), dtype=torch.float32, device="cuda")
        loop_out = torch.empty_like(stacked_out)

        def stacked():
            ctx.footprint_polygon_yaws(g, fp, nmaps, POLY, yaws, trav, slope, step, z, stacked_out, te.MEM_DEVICE)

        if nmaps == 1:
            def loop():
                for k, yaw in enumerate(yaws):
                    ctx.footprint_polygon(g, fp, POLY, yaw, trav[0], slope[0], step[0], z[0], scratch_x[0], loop_out[k, 0], te.MEM_DEVICE)
        else:
            def loop():
                for k, yaw in enumerate(yaws):
                    ctx.footprint_polygon_batched(g, fp, nmaps, POLY, yaw, trav, slope, step, z, scratch_x, loop_out[k], te.MEM_DEVICE)
        launches = {}
        for name, fn in (("stacked", stacked), ("loop", loop)):
            l0 = ctx.stats()[0]
            fn()
            torch.cuda.synchronize()
            launches[name] = ctx.stats()[0] - l0
        for _ in range(args.warmup):
            stacked()
            loop()
        torch.cuda.synchronize()
        ts, tl, hs, hl = [], [], [], []
        for _ in range(args.reps):
            timed(torch, stream, stacked, ts, hs)
            timed(torch, stream, loop, tl, hl)
        same = torch.equal(stacked_out.view(torch.int32), loop_out.view(torch.int32))
        ms, ml = float(np.median(ts)), float(np.median(tl))
        cells = nmaps * size * size
        nbytes = cells * (IN_BYTES_PER_CELL + OUT_BYTES_PER_CELL_YAW * nyaws)
        rec = {"maps": nmaps, "size": f"{size}x{size}", "nyaws": nyaws,
               "stacked_ms": round(ms, 4), "loop_ms": round(ml, 4), "speedup": round(ml / ms, 3),
               "stacked_ms_range": [round(min(ts), 4), round(max(ts), 4)], "loop_ms_range": [round(min(tl), 4), round(max(tl), 4)],
               "stacked_enqueue_ms": round(float(np.median(hs)), 4), "loop_enqueue_ms": round(float(np.median(hl)), 4),
               "launches_stacked": launches["stacked"], "launches_loop": launches["loop"], "bit_identical": bool(same),
               "model_bytes": nbytes, "stacked_GBps": round(nbytes / (ms * 1e-3) / 1e9, 1),
               "stacked_share_of_3.35TBps": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 4), "gpu": gpu, "power_limit_w": power}
        print(json.dumps(rec), flush=True)
        if args.profile:
            print(json.dumps({"maps": nmaps, "size": f"{size}x{size}", "nyaws": nyaws, "profile_stacked_ms": kernel_times(torch, stacked),
                              "profile_loop_ms": kernel_times(torch, loop)}), flush=True)
        del stacked_out, loop_out
        torch.cuda.empty_cache()


def run_reduce(args, torch, te, ctx, stream, gpu, power, nmaps, size, yaw_counts):
    """--reduce: one reduce call against the stacked call plus torch amin / amax / argmax, in device and in host memory."""
    g, z, slope, step, trav = layers(torch, te, ctx, nmaps, size)
    fp = te.FootprintParams.yaml_defaults()
    cells = nmaps * size * size
    host_in = [t.cpu().numpy() for t in (trav, slope, step, z)]
    for nyaws in yaw_counts:
        yaws = [2.0 * math.pi * k / nyaws for k in range(nyaws)]
        for memory in ("device", "host"):
            if memory == "device":
                mem, lay = te.MEM_DEVICE, (trav, slope, step, z)
                red = (torch.empty_like(z), torch.empty_like(z), torch.empty(z.shape, dtype=torch.int32, device="cuda"))
                stack = torch.empty((nyaws,) + tuple(z.shape), dtype=torch.float32, device="cuda")
                reps = args.reps
            else:
                mem, lay = te.MEM_HOST, host_in
                red = (np.empty(z.shape, np.float32), np.empty(z.shape, np.float32), np.empty(z.shape, np.int32))
                stack = np.empty((nyaws,) + tuple(z.shape), np.float32)
                reps = args.host_reps
            got = {}

            def reduce_call():
                ctx.footprint_polygon_yaws_reduce(g, fp, nmaps, POLY, yaws, *lay, *red, mem)

            def stacked_call():
                ctx.footprint_polygon_yaws(g, fp, nmaps, POLY, yaws, *lay, stack, mem)
                s = stack if memory == "device" else torch.from_numpy(stack)
                got["stacked"] = (s.amin(0), s.amax(0), s.argmax(0))

            launches = {}
            for name, fn in (("reduce", reduce_call), ("stacked", stacked_call)):
                l0 = ctx.stats()[0]
                fn()
                torch.cuda.synchronize()
                launches[name] = ctx.stats()[0] - l0
            for _ in range(args.warmup if memory == "device" else 0):
                reduce_call()
                stacked_call()
            torch.cuda.synchronize()
            tr, tsk, hr, hs = [], [], [], []
            for _ in range(reps):
                timed(torch, stream, reduce_call, tr, hr)
                timed(torch, stream, stacked_call, tsk, hs)
            mine = [torch.as_tensor(x).cpu() for x in red]
            ref = [x.cpu() for x in got["stacked"]]
            same = (torch.equal(mine[0].view(torch.int32), ref[0].view(torch.int32)) and
                    torch.equal(mine[1].view(torch.int32), ref[1].view(torch.int32)) and torch.equal(mine[2].long(), ref[2]))
            mr, ms = float(np.median(tr)), float(np.median(tsk))
            nbytes = cells * (IN_BYTES_PER_CELL + REDUCE_OUT_BYTES_PER_CELL)
            stack_bytes = cells * OUT_BYTES_PER_CELL_YAW * nyaws
            rec = {"mode": "reduce", "memory": memory, "maps": nmaps, "size": f"{size}x{size}", "nyaws": nyaws, "reps": reps,
                   "reduce_ms": round(mr, 4), "stacked_ms": round(ms, 4), "speedup": round(ms / mr, 3),
                   "reduce_ms_range": [round(min(tr), 4), round(max(tr), 4)], "stacked_ms_range": [round(min(tsk), 4), round(max(tsk), 4)],
                   "reduce_enqueue_ms": round(float(np.median(hr)), 4), "stacked_enqueue_ms": round(float(np.median(hs)), 4),
                   "launches_reduce": launches["reduce"], "launches_stacked": launches["stacked"], "bit_identical": bool(same),
                   # output bytes on the device (the library's staging buffers in host memory) and, in host memory, over PCIe
                   "reduce_out_bytes": cells * REDUCE_OUT_BYTES_PER_CELL, "stacked_out_bytes": stack_bytes,
                   "reduce_d2h_bytes": cells * REDUCE_OUT_BYTES_PER_CELL if memory == "host" else 0,
                   "stacked_d2h_bytes": stack_bytes if memory == "host" else 0,
                   "model_bytes": nbytes, "reduce_GBps": round(nbytes / (mr * 1e-3) / 1e9, 1),
                   "reduce_share_of_3.35TBps": round(nbytes / (mr * 1e-3) / HBM_BYTES_PER_S, 4), "gpu": gpu, "power_limit_w": power}
            print(json.dumps(rec), flush=True)
            del stack, red, got
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--yaws", type=int, nargs="*", default=None)
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--batch-maps", type=int, default=256)
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--batch-yaws", type=int, nargs="*", default=[8])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--reduce", action="store_true")
    ap.add_argument("--host-reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_footprint_yaws needs a CUDA device")
    gpu, power = gpu_info(torch)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    bench = run_reduce if args.reduce else run
    yaws = args.yaws if args.yaws is not None else ([16, 36, 72] if args.reduce else [2, 8, 16, 36, 72])
    if yaws:
        bench(args, torch, te, ctx, stream, gpu, power, 1, args.size, yaws)
    if args.batch_maps and args.batch_yaws:
        bench(args, torch, te, ctx, stream, gpu, power, args.batch_maps, args.batch_size, args.batch_yaws)
    ctx.close()


if __name__ == "__main__":
    main()
