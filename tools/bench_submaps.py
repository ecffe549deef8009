"""The read side of a te_map: what a node pays per map update to serve its map from the device.

(a) Node-like update at --size² cells of 0.02 m (synth.terrain "mixed"), elevation in pinned host memory.  Today's path is
    te_map_chain with its four chain layers copied out to pinned host layers (the node keeps a host GridMap beside the te_map to
    answer getSubmap).  The new path is te_map_chain with no host outputs plus one te_map_get_submaps call in host memory for
    1 / 16 / 256 windows of 4 m x 4 m around random centres, every layer the map holds after te_map_chain (traversability,
    traversability_slope, traversability_step, traversability_roughness, elevation, traversability_footprint).  Both return
    synchronised, so each update is timed with the host clock; medians of --reps, the two paths alternating, with the bytes
    each moves over PCIe.
(b) The device-memory gather alone: one te_map_get_submaps call against a loop of one cudaMemcpy2DAsync per (window, layer) on
    the same stream, CUDA events, both outputs compared bit for bit.  Achieved bandwidth counts every gathered float read once
    and written once, against a device-to-device copy of 1 GiB measured the same way (torch copy_).
Prints one JSON line per measurement with the GPU and its power limit.

    python tools/bench_submaps.py [--size 8192] [--windows 1 16 256] [--reps 10] [--warmup 2]
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

from bench_footprint_batched import gpu_info  # noqa: E402

RES = 0.02
WINDOW = 4.0
HELD = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation",
        "traversability_footprint"]


def cudart():
    """The CUDA runtime torch loads (for cudaMemcpy2DAsync), else the toolkit's."""
    cands = []
    try:
        import nvidia.cuda_runtime as cr
        cands += [os.path.join(p, "lib", "libcudart.so.12") for p in cr.__path__]
    except ImportError:
        pass
    cands += ["/usr/local/cuda/lib64/libcudart.so.12", "libcudart.so.12"]
    for c in cands:
        try:
            return C.CDLL(c)
        except OSError:
            continue
    raise SystemExit("bench_submaps needs libcudart.so.12 for the cudaMemcpy2DAsync baseline")


def windows(rng, n, g):
    """n 4 m x 4 m windows whose centres keep them inside the map."""
    half = np.array([g.length_x, g.length_y]) / 2 - WINDOW
    pos = np.array([g.position_x, g.position_y]) + rng.uniform(-1, 1, (n, 2)) * half
    return pos, np.full((n, 2), WINDOW)


def median_ms(xs):
    return round(float(np.median(xs)), 4), [round(float(min(xs)), 4), round(float(max(xs)), 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--windows", type=int, nargs="+", default=[1, 16, 256])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_submaps needs a CUDA device")
    gpu, power = gpu_info(torch)
    n = args.size
    g = te.Geometry.make(n, n, RES)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # the library's calls, torch's copies and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    m = ctx.map()
    m._g = g   # the map's geometry, for the Python view's layer shapes (te_map_chain is called through the C ABI below)
    L = ctx._L
    p = te.ChainParams.yaml_defaults(0)
    elev = torch.from_numpy(np.ascontiguousarray(synth.terrain(n, n, RES, 7, "mixed").T)).pin_memory()
    outs = [torch.empty((n, n), dtype=torch.float32).pin_memory() for _ in range(4)]
    chain = L.te_map_chain
    get = L.te_map_get_submaps
    mask = te.capi.layer_mask(HELD)
    cell_bytes = 4 * n * n
    rng = np.random.default_rng(3)

    def check(rc):
        if rc != 0:
            raise te.TEError(rc, L.te_last_error().decode())

    def old():
        check(chain(m._h, C.byref(g), C.byref(p), elev.data_ptr(), *(o.data_ptr() for o in outs), te.MEM_HOST))

    # (a) node-like update
    for nw in args.windows:
        pos, ln = windows(rng, nw, g)
        geo = te.capi.submap_geometry(g, pos, ln)
        total = len(HELD) * int((geo["rows"].astype(np.int64) * geo["cols"]).sum())
        host = torch.empty(total, dtype=torch.float32).pin_memory()
        info = np.zeros(nw, dtype=te.capi.SUBMAP_INFO_DTYPE)

        def new():
            check(chain(m._h, C.byref(g), C.byref(p), elev.data_ptr(), None, None, None, None, te.MEM_HOST))
            check(get(m._h, nw, pos.ctypes.data, ln.ctypes.data, mask, info.ctypes.data, host.data_ptr(), total, te.MEM_HOST))

        for _ in range(args.warmup):
            old()
            new()
        t_old, t_new = [], []
        for _ in range(args.reps):
            for fn, ts in ((old, t_old), (new, t_new)):
                t0 = time.perf_counter()
                fn()
                ts.append(1e3 * (time.perf_counter() - t0))
        mo, ro = median_ms(t_old)
        mn, rn = median_ms(t_new)
        print(json.dumps({"part": "a", "size": f"{n}x{n}", "windows": nw, "layers": len(HELD),
                          "old_ms": mo, "old_range": ro, "new_ms": mn, "new_range": rn, "speedup": round(mo / mn, 3),
                          "old_pcie_mb": round((cell_bytes + 4 * cell_bytes) / 1e6, 1),
                          "new_pcie_mb": round((cell_bytes + 4 * total) / 1e6, 2), "gpu": gpu, "power_limit_w": power}),
              flush=True)

    # (b) device-memory gather against one cudaMemcpy2DAsync per (window, layer); the map holds the layers of the last update
    rt = cudart()
    rt.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
    src = torch.empty((len(HELD), n, n), dtype=torch.float32, device="cuda")    # the resident layers, default order
    lay = m.get_layers(HELD, out=src, memory=te.MEM_DEVICE)
    base = [lay[k].data_ptr() for k in HELD]
    big = torch.empty(1 << 28, dtype=torch.float32, device="cuda")
    big2 = torch.empty_like(big)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        ev[0].record(stream)
        fn()
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    for _ in range(args.warmup):
        big2.copy_(big)
    copy_ms = float(np.median([timed(lambda: big2.copy_(big)) for _ in range(args.reps)]))
    copy_gbs = 2 * big.numel() * 4 / copy_ms / 1e6
    for nw in args.windows:
        pos, ln = windows(rng, nw, g)
        geo = te.capi.submap_geometry(g, pos, ln)
        total = len(HELD) * int((geo["rows"].astype(np.int64) * geo["cols"]).sum())
        out_k = torch.empty(total, dtype=torch.float32, device="cuda")
        out_l = torch.empty(total, dtype=torch.float32, device="cuda")
        info = np.zeros(nw, dtype=te.capi.SUBMAP_INFO_DTYPE)
        copies = []
        for w in range(nw):
            r0, c0, nr, nc, off = (int(geo[f][w]) for f in ("top_row", "top_col", "rows", "cols", "offset"))
            for k in range(len(HELD)):
                dst = out_l.data_ptr() + 4 * (len(HELD) * off + k * nr * nc)
                copies.append((dst, 4 * nr, base[k] + 4 * (c0 * n + r0), 4 * n, 4 * nr, nc))

        def kernel():
            check(get(m._h, nw, pos.ctypes.data, ln.ctypes.data, mask, info.ctypes.data, out_k.data_ptr(), total, te.MEM_DEVICE))

        def loop():
            for c in copies:
                e = rt.cudaMemcpy2DAsync(*c, 3, C.c_void_p(stream.cuda_stream))   # cudaMemcpyDeviceToDevice
                if e != 0:
                    raise RuntimeError(f"cudaMemcpy2DAsync failed: {e}")

        l0 = ctx.stats()[0]
        kernel()
        launches = ctx.stats()[0] - l0
        for _ in range(args.warmup):
            kernel()
            loop()
        t_k, t_l = [], []
        for _ in range(args.reps):
            t_k.append(timed(kernel))
            t_l.append(timed(loop))
        same = torch.equal(out_k.view(torch.int32), out_l.view(torch.int32))
        mk, rk = median_ms(t_k)
        ml, rl = median_ms(t_l)
        print(json.dumps({"part": "b", "size": f"{n}x{n}", "windows": nw, "layers": len(HELD), "mb_gathered": round(4 * total / 1e6, 2),
                          "kernel_ms": mk, "kernel_range": rk, "memcpy2d_loop_ms": ml, "memcpy2d_range": rl,
                          "memcpy2d_calls": len(copies), "kernel_launches": launches,
                          "kernel_gbs": round(2 * 4 * total / mk / 1e6, 1), "memcpy2d_gbs": round(2 * 4 * total / ml / 1e6, 1),
                          "d2d_copy_gbs": round(copy_gbs, 1), "bit_identical": bool(same), "gpu": gpu, "power_limit_w": power}),
              flush=True)
    m.close()
    ctx.close()


if __name__ == "__main__":
    main()
