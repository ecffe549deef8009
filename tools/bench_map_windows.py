"""A te_map computed from windows of a larger elevation map (te_map_chain_windows, te_map_chain_submap) against the composition a
user writes without them.

(a) A fleet: one 8192² fused elevation map (elevation, upper_bound, lower_bound; synth.terrain "mixed" plus noise) with a
    circular-buffer start index, cut into 256 maps of 512² at 0.02 m, and separately, the same layers read at 0.03 m, into 256 maps
    of 134² (the reference's 4 m map at 0.03 m), at 256 robot positions spread over the map and a little past its edges.  Device memory: one te_map_chain_windows call against a torch
    gather of the windows with the same float64 arithmetic (asserted to give the same bits), te_map_chain_batched_at and
    te_map_carry_layers.  CUDA events on torch's stream around whole calls, median of --reps after --warmup, cases alternating.
    k_map_cut_windows' time comes from a separate torch.profiler run, and its bytes moved (every window cell written, every cell
    inside the source read, 4 bytes per layer) over that time give its achieved TB/s.
(b) The node: one 4 m window of that map at 0.03 m in host memory (pageable numpy layers in buffer order): te_map_chain_submap against
    te_submap_geometry, numpy slicing with the start index, te_map_chain and te_map_carry_layers.  Host clock, median of --reps.
Both paths of every case are checked to leave the same layers and positions, bit for bit.  One JSON line per case and per check,
with the GPU and its power limit.

    python tools/bench_map_windows.py [--size 8192] [--maps 256] [--reps 10] [--warmup 3]
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

from bench_footprint_yaws import gpu_info  # noqa: E402
from bench_map_polygon import time_cases  # noqa: E402

NAMES = ("elevation", "upper_bound", "lower_bound")


def window_tops(g, src, xy):
    """te_map_chain_windows' window rule in numpy float64 (te_grid.cuh grid_window_top / grid_window_position, same operand order):
    top-left indices (n, 2) int64 and map positions (n, 2)."""
    tl = xy + 0.5 * np.array([g.length_x, g.length_y])
    v = ((tl - 0.5 * np.array([src.length_x, src.length_y])) - np.array([src.position_x, src.position_y])) / src.resolution
    top = np.floor(-v).astype(np.int64)
    off = 0.5 * np.array([src.length_x, src.length_y]) - 0.5 * src.resolution
    corner = ((np.array([src.position_x, src.position_y]) + off) + src.resolution * (-top.astype(np.float64))) + 0.5 * src.resolution
    return top, corner - 0.5 * (np.array([g.rows, g.cols], np.float64) * src.resolution)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_windows needs a CUDA device")
    gpu, power = gpu_info(torch)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    L = te.load_library()
    p = te.ChainParams.yaml_defaults(0)
    N = args.size
    start = (N // 3, (2 * N) // 5)

    def source(res):
        g = te.Geometry.make(N, N, res, (3.7, -1.9))
        g.start_row, g.start_col = start
        return g
    rng = np.random.default_rng(5)
    unwrapped = {"elevation": synth.terrain(N, N, 0.02, 3, "mixed").astype(np.float32)}
    unwrapped["upper_bound"] = unwrapped["elevation"] + rng.uniform(0, 0.1, (N, N)).astype(np.float32)
    unwrapped["lower_bound"] = unwrapped["elevation"] - rng.uniform(0, 0.1, (N, N)).astype(np.float32)
    stored = {n: np.asfortranarray(np.roll(a, start, axis=(0, 1))) for n, a in unwrapped.items()}
    del unwrapped
    dev = {n: torch.from_numpy(np.ascontiguousarray(a.T)).cuda() for n, a in stored.items()}   # (cols, rows): column-major
    bad = 0

    def held(m, nmaps, g):
        out = torch.empty(len(NAMES) + 4, nmaps * g.rows * g.cols, dtype=torch.float32, device="cuda")
        L.te_map_get_layers(m._h, 0x0f | te.capi.layer_mask(NAMES), out.data_ptr(), te.MEM_DEVICE)
        return out

    def fleet(rows, res):
        nonlocal bad
        src = source(res)
        g = te.Geometry.make(rows, rows, res)
        half = 0.5 * N * res
        xy = np.stack([src.position_x + rng.uniform(-1.05 * half, 1.05 * half, args.maps),
                       src.position_y + rng.uniform(-1.05 * half, 1.05 * half, args.maps)], axis=1)
        top, at = window_tops(g, src, xy)
        at = np.ascontiguousarray(at)
        top_t = torch.from_numpy(top).cuda()
        ar = torch.arange(rows, device="cuda")
        ri, ci = top_t[:, 0:1] + ar, top_t[:, 1:2] + ar                      # (maps, rows) source rows / columns
        vr, vc = (ri >= 0) & (ri < N), (ci >= 0) & (ci < N)
        sr, sc = (ri + start[0]) % N, (ci + start[1]) % N
        nan = torch.tensor([0x7fc00000], dtype=torch.int32, device="cuda").view(torch.float32)
        cut = {n: torch.empty(args.maps * rows * rows, dtype=torch.float32, device="cuda") for n in NAMES}

        def gather():
            ok = vc[:, :, None] & vr[:, None, :]                           # (maps, cols, rows): column-major windows
            for n in NAMES:
                v = dev[n][sc[:, :, None], sr[:, None, :]]
                cut[n].copy_(torch.where(ok, v, nan).reshape(-1))

        m_new, m_old = ctx.map(), ctx.map()
        lay = {n: dev[n].reshape(-1) for n in NAMES}

        def new():
            m_new.chain_windows(g, src, lay, xy, p, memory=te.MEM_DEVICE)

        def old():
            gather()
            rc = L.te_map_chain_batched_at(m_old._h, C.byref(g), C.byref(p), args.maps, cut["elevation"].data_ptr(), None, None, None,
                                           None, te.MEM_DEVICE, at.ctypes.data)
            assert rc == 0, L.te_last_error()
            m_old.carry_layers(NAMES[1:], [cut[n] for n in NAMES[1:]], memory=te.MEM_DEVICE)

        cases = {"chain_windows": new, "gather+chain_batched_at+carry": old}
        ms = time_cases(torch, stream, ctx, cases, args.reps, args.warmup)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                new()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "k_map_cut_windows" in e.key]
        count = sum(e.count for e in kern)
        kernel_ms = sum(e.device_time_total for e in kern) / max(count, 1) / 1e3
        inside = int(((vr.sum(1) * vc.sum(1))).sum())
        nbytes = 4 * len(NAMES) * (args.maps * rows * rows + inside)
        workload = f"fleet: {args.maps} x {rows}^2 at {res} m from {N}^2, {len(NAMES)} layers, start index {start}"
        for k in cases:
            rec = {"bench": "map_windows", "workload": workload, "case": k, "ms": round(ms[k], 3),
                   "speedup_of_chain_windows": round(ms[k] / ms["chain_windows"], 3), "gpu": gpu, "power_limit_w": power}
            if k == "chain_windows":
                rec.update(cut_kernel_ms=round(kernel_ms, 4), cut_launches=count, cut_bytes=nbytes,
                           cut_tb_s=round(nbytes / (kernel_ms * 1e-3) / 1e12, 3))
            print(json.dumps(rec))
        new()
        old()
        torch.cuda.synchronize()
        a, b = held(m_new, args.maps, g), held(m_old, args.maps, g)
        same = bool(torch.equal(a.view(torch.int32), b.view(torch.int32))) and np.array_equal(m_new.positions(), at)
        same_cut = bool(torch.equal(a[4].view(torch.int32), cut["elevation"].view(torch.int32)))
        torch.cuda.synchronize()
        bad += not (same and same_cut)
        print(json.dumps({"bench": "map_windows", "check": f"{workload}: chain_windows == gather + chain_batched_at + carry, "
                          "layers and positions bit for bit; torch gather == k_map_cut_windows", "ok": same and same_cut,
                          "windows_fully_inside": int(((vr.all(1)) & (vc.all(1))).sum())}))
        m_new.close()
        m_old.close()
        del cut, a, b
        torch.cuda.empty_cache()

    fleet(512, 0.02)
    fleet(134, 0.03)

    # (b) the node's update from host memory
    host = {n: stored[n] for n in NAMES}
    src = source(0.03)
    pos, length = (src.position_x + 11.3, src.position_y - 27.9), (4.0, 4.0)
    m_new, m_old = ctx.map(), ctx.map()

    def node_new():
        info = m_new.chain_submap(src, host, pos, length, p)
        assert info.success == 1

    def node_old():
        info = te.capi.submap_geometry(src, [pos], [length])[0]
        r, c = int(info["rows"]), int(info["cols"])
        ri = (int(info["top_row"]) + np.arange(r) + start[0]) % N
        ci = (int(info["top_col"]) + np.arange(c) + start[1]) % N
        win = {n: host[n][np.ix_(ri, ci)] for n in NAMES}
        gs = te.Geometry(r, c, src.resolution, info["length_x"], info["length_y"], info["position_x"], info["position_y"], 0, 0)
        m_old.chain(gs, p, win["elevation"])
        m_old.carry_layers(NAMES[1:], [win[n] for n in NAMES[1:]])

    cases = {"chain_submap": node_new, "numpy+chain+carry": node_old}
    t = {k: [] for k in cases}
    for rep in range(args.warmup + args.reps):
        for k in (list(cases) if rep % 2 == 0 else list(cases)[::-1]):
            a = time.perf_counter()
            cases[k]()
            if rep >= args.warmup:
                t[k].append((time.perf_counter() - a) * 1e3)
    ms = {k: float(np.median(v)) for k, v in t.items()}
    info = te.capi.submap_geometry(src, [pos], [length])[0]
    workload = f"node: one {length[0]} m window ({int(info['rows'])} x {int(info['cols'])}) of {N}^2 from host memory"
    for k in cases:
        print(json.dumps({"bench": "map_windows", "workload": workload, "case": k, "ms": round(ms[k], 3),
                          "speedup_of_chain_submap": round(ms[k] / ms["chain_submap"], 3), "gpu": gpu, "power_limit_w": power}))
    names = list(te.capi.LAYERS[:5]) + list(NAMES[1:])
    ga, gb = m_new.get_layers(names), m_old.get_layers(names)
    same = all(np.array_equal(ga[n].view(np.uint32), gb[n].view(np.uint32)) for n in names) and \
        np.array_equal(m_new.positions(), m_old.positions())
    bad += not same
    print(json.dumps({"bench": "map_windows", "check": f"{workload}: chain_submap == numpy + chain + carry, bit for bit", "ok": same}))
    m_new.close()
    m_old.close()
    ctx.close()
    if bad:
        raise SystemExit(f"{bad} checks failed")


if __name__ == "__main__":
    main()
