"""Elevation images (te_map_chain_image) against converting them on the host and calling te_map_chain(_batched).

Workloads: one 8192² mono16 image, and 256 mono16 images of 512² (te_map_chain_image with nmaps = 256), at 0.02 m, pixels from
synth.terrain "mixed" scaled to 0..65535 (NaN cells at 0).  Timed with the host clock around each call (host-memory calls return
synchronised; the device call is followed by a synchronisation of the context stream), median of --reps after --warmup, the
cases alternating:
  - image: te_map_chain_image on the page-locked host image (uploads 2 B per cell);
  - numpy+chain: the same addLayerFromImage arithmetic in numpy float32 into a page-locked column-major buffer, then
    te_map_chain(_batched) in host memory (uploads 4 B per cell); the numpy part is also reported alone;
  - device: te_map_chain_image on the image already in device memory.
No outputs are copied back (the layers stay resident), so every case runs the same chain.  Then the conversion kernel alone:
k_image_to_layer's device time summed with torch.profiler over --reps device calls, in a separate pass, against its (2 + 4)
bytes per cell, as bytes/s and as a share of the HBM peak (MEASURED_PEAKS.json's hbm_gbs when the file is there, else the
H100 SXM data sheet's 3.35 TB/s, which is named as such).  Checks that the elevation te_map_chain_image leaves equals the numpy
conversion bit for bit.  One JSON line per workload, with the GPU and its power limit.

    python tools/bench_image.py [--reps 10] [--warmup 2]
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

RES, LO, HI = 0.02, -1.5, 2.5
DATASHEET_HBM_GBS = 3350.0


def gpu_info(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(path))["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs"
    except Exception:
        return DATASHEET_HBM_GBS, "H100 SXM data sheet (not measured)"


def numpy_convert(img, out):
    """addLayerFromImage in numpy float32 (each operation rounded to float32, as the reference): (n, rows, cols) uint16 into the
    (n, cols, rows) float32 buffer `out`, i.e. per map column-major."""
    lo, hi = np.float32(LO), np.float32(HI)
    np.add(lo, (hi - lo) * (img.transpose(0, 2, 1).astype(np.float32) / np.float32(65535.0)), out=out)


def median_ms(ts):
    return float(np.median(ts) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_image.py needs a CUDA device")
    gpu, power = gpu_info(torch)
    peak, peak_src = hbm_peak()
    L = te.load_library()
    ctx = te.Context(0)
    p = te.ChainParams.yaml_defaults(0)

    for nmaps, size in ((1, 8192), (256, 512)):
        rows = cols = size
        cells = nmaps * rows * cols
        z = [synth.terrain(rows, cols, RES, seed=40 + k, preset="mixed") for k in range(min(nmaps, 8))]
        img_t = torch.empty((nmaps, rows, cols), dtype=torch.int16, pin_memory=True)
        img = img_t.numpy().view(np.uint16)
        for k in range(nmaps):
            zk = z[k % len(z)]
            lo, hi = np.nanmin(zk), np.nanmax(zk)
            img[k] = np.nan_to_num((zk - lo) / (hi - lo) * 65535.0, nan=0.0).astype(np.uint16)
        elev_t = torch.empty((nmaps, cols, rows), dtype=torch.float32, pin_memory=True)
        elev = elev_t.numpy()
        dev_img = img_t.cuda()
        torch.cuda.synchronize()
        g = te.image_geometry(rows, cols, RES)
        m = ctx.map()
        rs, ims = cols * 2, rows * cols * 2

        def image():
            ctx._check(L.te_map_chain_image(m._h, C.byref(g), C.byref(p), nmaps, te.IMAGE_MONO16, img.ctypes.data, rs, ims, LO, HI,
                                            None, None, None, None, te.MEM_HOST))

        def device():
            ctx._check(L.te_map_chain_image(m._h, C.byref(g), C.byref(p), nmaps, te.IMAGE_MONO16, dev_img.data_ptr(), rs, ims, LO, HI,
                                            None, None, None, None, te.MEM_DEVICE))
            ctx.synchronize()

        def convert():
            numpy_convert(img, elev)

        def chain():
            if nmaps == 1:
                ctx._check(L.te_map_chain(m._h, C.byref(g), C.byref(p), elev.ctypes.data, None, None, None, None, te.MEM_HOST))
            else:
                ctx._check(L.te_map_chain_batched(m._h, C.byref(g), C.byref(p), nmaps, elev.ctypes.data, None, None, None, None,
                                                  te.MEM_HOST))

        times = {"image": [], "numpy+chain": [], "numpy": [], "device": []}
        for r in range(args.warmup + args.reps):
            t0 = time.perf_counter(); image(); t1 = time.perf_counter()
            convert(); t2 = time.perf_counter(); chain(); t3 = time.perf_counter()
            device(); t4 = time.perf_counter()
            if r >= args.warmup:
                times["image"].append(t1 - t0)
                times["numpy"].append(t2 - t1)
                times["numpy+chain"].append(t3 - t1)
                times["device"].append(t4 - t3)

        image()
        m._g, m._n = g, nmaps
        got = m.get_layers(["elevation"])["elevation"]
        got = got[None] if nmaps == 1 else got
        same = bool(np.array_equal(np.ascontiguousarray(got.transpose(0, 2, 1)).view(np.uint32), elev.view(np.uint32)))

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                device()
        kern = [e for e in prof.events() if e.device_type.name == "CUDA" and "k_image_to_layer" in e.name]
        kern_us = sum(e.device_time for e in kern) / max(len(kern), 1)
        nbytes = cells * (2 + 4)
        gbs = nbytes / (kern_us * 1e-6) / 1e9 if kern_us else None
        print(json.dumps({
            "workload": f"{nmaps} x {size}^2 mono16", "cells": cells,
            **{f"{k}_ms": round(median_ms(v), 3) for k, v in times.items()},
            "upload_bytes_image": cells * 2, "upload_bytes_float": cells * 4,
            "k_image_to_layer_us": round(kern_us, 2), "k_image_to_layer_launches": len(kern), "k_image_to_layer_bytes": nbytes,
            "k_image_to_layer_gbs": round(gbs, 1) if gbs else None,
            "share_of_hbm_peak": round(gbs / peak, 3) if gbs else None, "hbm_peak_gbs": peak, "hbm_peak_source": peak_src,
            "elevation_bit_identical": same, "gpu": gpu, "power_limit_w": power}), flush=True)
        m.close()
        del dev_img
    ctx.close()


if __name__ == "__main__":
    main()
