"""Layers at robot-frame points around poses (te_map_at_poses) against the path a user has without it: te_map_get_layers in device
memory, then the same float64 pose transform and getIndex arithmetic in torch and an advanced-index gather.

(a) A fleet: 256 maps of 512² cells (synth.terrain "mixed" at 0.02 m, 32 terrains cycled over the maps) at 256 positions (a 40 m
    grid, off the cell lattice), every cache filled by te_map_footprint; 16 poses per map (4 096 poses, yawed and tilted, a few
    off the map) and a 17 x 11 pattern of points at 0.1 m (187 points, a height scan around a legged robot); elevation,
    traversability and traversability_footprint.
(b) One 8192² map, 100 000 single-point poses ((0, 0, 0): atPosition at a list of positions), traversability.
Device memory, the library on torch's stream, CUDA events around whole calls, median of --reps after --warmup, cases alternating.
The two paths are checked to agree bit for bit, values and validity.  Kernel times come from a separate torch.profiler run, and
achieved bytes/s from the byte model of DESIGN.md §4.3 over the kernel time.  One JSON line per case and per check, with the GPU
and its power limit.

    python tools/bench_map_at_poses.py [--maps 256] [--size 512] [--big 8192] [--reps 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_footprint_yaws import gpu_info  # noqa: E402
from bench_map_polygon import time_cases  # noqa: E402

RES = 0.02


def model_bytes(nposes, npoints, nlayers, batched):
    """DESIGN.md §4.3: per pose its 56-byte pose (and a 4-byte map index on a batch), per point 12 bytes, per sample one 32-byte
    sector read and 4 bytes written per layer and 1 byte of valid."""
    return nposes * (56 + (4 if batched else 0)) + npoints * 12 + nposes * npoints * (nlayers * (32 + 4) + 1)


def poses_around(rng, centers, half):
    """One pose per centre within 1.05 * half of it: yaw-only quaternions for most, tilted unit ones for every fourth."""
    n = len(centers)
    xy = centers + rng.uniform(-1.05 * half, 1.05 * half, (n, 2))
    yaw = rng.uniform(0, 2 * np.pi, n)
    q = np.stack([np.zeros(n), np.zeros(n), np.sin(yaw / 2), np.cos(yaw / 2)], axis=1)
    tilt = rng.normal(size=(n, 4))
    q[::4] = (tilt / np.linalg.norm(tilt, axis=1, keepdims=True))[::4]
    return np.concatenate([xy, rng.uniform(-0.5, 0.5, (n, 1)), q], axis=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=256)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--big", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import synth
    import traversability_estimation_b200 as te

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_at_poses needs a CUDA device")
    gpu, power = gpu_info(torch)
    ctx = te.Context(0)
    stream = torch.cuda.Stream()   # torch's work, the library's calls and the events share one stream
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    p = te.ChainParams.yaml_defaults(0)
    nan_bits = torch.tensor([0x7fc00000], dtype=torch.int32, device="cuda").view(torch.float32)
    bad = 0

    def today(m, g, nmaps, pos_t, names, poses, pts, pose_map, layers):
        """te_map_get_layers into `layers`, then the transform, getIndex and a gather in torch (float64, one op per kernel, so
        nothing is contracted)."""
        m.get_layers(names, out=layers, memory=te.MEM_DEVICE)
        x, y, qx, qy, qz, qw = (poses[:, k:k + 1] for k in (0, 1, 3, 4, 5, 6))
        tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
        twx, twy, twz = tx * qw, ty * qw, tz * qw
        txx, txy, txz = tx * qx, ty * qx, tz * qx
        tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
        vx, vy, vz = (pts[:, k].double()[None, :] for k in range(3))
        px = (((1.0 - (tyy + tzz)) * vx + (txy - twz) * vy) + (txz + twy) * vz) + x
        py = (((txy + twz) * vx + (1.0 - (txx + tzz)) * vy) + (tyz - twx) * vz) + y
        mp = pose_map.long()[:, None] if pose_map is not None else torch.zeros_like(x, dtype=torch.long)
        mx, my = pos_t[mp, 0], pos_t[mp, 1]
        i = (-(((px - 0.5 * g.length_x) - mx) / g.resolution)).nan_to_num(0.0).to(torch.int64)
        j = (-(((py - 0.5 * g.length_y) - my) / g.resolution)).nan_to_num(0.0).to(torch.int64)
        sx, sy = -((px - mx) - 0.5 * g.length_x), -((py - my) - 0.5 * g.length_y)
        ok = (sx >= 0) & (sy >= 0) & (sx < g.length_x) & (sy < g.length_y) & (i >= 0) & (j >= 0) & (i < g.rows) & (j < g.cols)
        cell = torch.where(ok, (mp * g.cols + j) * g.rows + i, 0)
        vals = layers.view(len(names), nmaps * g.rows * g.cols)[:, cell]
        return torch.where(ok[None], vals, nan_bits), ok

    def run(label, m, g, nmaps, positions, names, poses_np, pts_np, pose_map_np):
        nonlocal bad
        poses = torch.from_numpy(poses_np).cuda()
        pts = torch.from_numpy(pts_np).cuda()
        pose_map = None if pose_map_np is None else torch.from_numpy(pose_map_np).cuda()
        pos_t = torch.from_numpy(np.ascontiguousarray(positions, np.float64)).cuda()
        n, t, nl = len(poses_np), len(pts_np), len(names)
        out = torch.empty(nl * n * t, dtype=torch.float32, device="cuda")
        valid = torch.empty(n * t, dtype=torch.uint8, device="cuda")
        layers = torch.empty(nl * nmaps * g.rows * g.cols, dtype=torch.float32, device="cuda")
        res = {}
        cases = {
            "at_poses": lambda: m.at_poses(poses, pts, names, pose_map=pose_map, out=out, valid=valid, memory=te.MEM_DEVICE),
            "get_layers+torch": lambda: res.__setitem__("t", today(m, g, nmaps, pos_t, names, poses, pts, pose_map, layers)),
        }
        ms = time_cases(torch, stream, ctx, cases, args.reps, args.warmup)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                cases["at_poses"]()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "k_map_at_poses" in e.key]
        count = sum(e.count for e in kern)
        kernel_ms = sum(e.device_time_total for e in kern) / max(count, 1) / 1e3
        nbytes = model_bytes(n, t, nl, pose_map_np is not None)
        workload = f"{label}: {n} poses x {t} points, {nl} layers"
        for k in cases:
            rec = {"bench": "map_at_poses", "workload": workload, "case": k, "ms": round(ms[k], 4),
                   "speedup_of_at_poses": round(ms[k] / ms["at_poses"], 2), "gpu": gpu, "power_limit_w": power}
            if k == "at_poses":
                rec.update(kernel_ms=round(kernel_ms, 4), kernel_launches=count, model_bytes=int(nbytes),
                           achieved_gb_s=round(nbytes / (kernel_ms * 1e-3) / 1e9, 1))
            print(json.dumps(rec))
        cases["at_poses"]()
        cases["get_layers+torch"]()
        torch.cuda.synchronize()
        vals, ok = res["t"]
        same = bool(torch.equal(out.view(torch.int32), vals.reshape(-1).view(torch.int32))) and \
            bool(torch.equal(valid.bool(), ok.reshape(-1)))
        bad += not same
        print(json.dumps({"bench": "map_at_poses", "check": f"{label}: at_poses == get_layers + torch, bit for bit", "ok": same,
                          "valid_fraction": round(float(valid.float().mean()), 3)}))

    rng = np.random.default_rng(17)
    # ---- (a) the fleet ----
    n, size = args.maps, args.size
    g = te.Geometry.make(size, size, RES)
    side = int(np.ceil(np.sqrt(n)))
    pos = np.array([(40.0 * (k % side) + 0.0137 * k, 40.0 * (k // side) - 0.0071 * k) for k in range(n)], np.float64)
    terrains = [synth.terrain(size, size, RES, 7000 + k, "mixed").astype(np.float32) for k in range(min(n, 32))]
    batch = ctx.map()
    batch.chain_batched(g, p, n, np.stack([terrains[k % len(terrains)] for k in range(n)]), positions=pos)
    batch.footprint(te.FootprintParams.yaml_defaults())
    pose_map = np.repeat(np.arange(n, dtype=np.int32), 16)
    poses = poses_around(rng, pos[pose_map], 0.5 * size * RES)
    ax, ay = np.meshgrid(0.1 * (np.arange(17) - 8), 0.1 * (np.arange(11) - 5), indexing="ij")
    pattern = np.stack([ax.ravel(), ay.ravel(), np.zeros(ax.size)], axis=1).astype(np.float32)
    run(f"(a) {n} x {size}^2 at {n} positions", batch, g, n, pos, ["traversability", "elevation", "traversability_footprint"], poses,
        pattern, pose_map)
    batch.close()
    torch.cuda.empty_cache()

    # ---- (b) one large map ----
    if args.big:
        size = args.big
        g = te.Geometry.make(size, size, RES)
        m = ctx.map()
        m.chain(g, p, synth.terrain(size, size, RES, 8100, "mixed").astype(np.float32))
        poses = poses_around(rng, np.zeros((100_000, 2)), 0.5 * size * RES)
        run(f"(b) 1 x {size}^2", m, g, 1, np.zeros((1, 2)), ["traversability"], poses, np.zeros((1, 3), np.float32), None)
        m.close()
    ctx.set_stream(None)
    ctx.close()
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
