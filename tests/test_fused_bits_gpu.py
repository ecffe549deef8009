"""Bit identity of the fused chain kernel: the CRC32 of every output layer of k_chain_fused, on the 8192^2 bench map and on
2048^2 maps (with and without the surface normal outputs, and at 0.03 m where the other window shape is instantiated), must
stay what the build these values were recorded from computed.  Changes to the instruction stream of the kernel (constants,
selects, min/max grouping, build switches) are meant to leave every bit of every layer unchanged.

Recorded on an H100 80GB HBM3, identical from the build before the per-step instruction cuts and the build after them;
`python tests/test_fused_bits_gpu.py` prints the table for the library it loads."""
import zlib

import pytest

pytestmark = pytest.mark.gpu

LAYERS = ("slope", "step", "roughness", "traversability")
NORMALS = ("nx", "ny", "nz")

# name: (cells per side, resolution, bench terrain seed, normals outputs)
CASES = {
    "8192": (8192, 0.02, 3, False),
    "2048": (2048, 0.02, 3, False),
    "2048_normals": (2048, 0.02, 3, True),
    "2048_res003": (2048, 0.03, 5, False),
    "2048_res003_normals": (2048, 0.03, 5, True),
}

EXPECTED = {
    '2048': {'slope': 0x4565e026, 'step': 0x3859bf1d, 'roughness': 0x2e190a4e, 'traversability': 0x9b3b3d16},
    '2048_normals': {'slope': 0x4565e026, 'step': 0x3859bf1d, 'roughness': 0x2e190a4e, 'traversability': 0x9b3b3d16, 'nx': 0xc7c904b3, 'ny': 0xb93ad3cb, 'nz': 0xbbb8fe2f},
    '2048_res003': {'slope': 0xe3b366fa, 'step': 0xca3e7110, 'roughness': 0x4a31721b, 'traversability': 0xe50973c4},
    '2048_res003_normals': {'slope': 0xe3b366fa, 'step': 0xca3e7110, 'roughness': 0x4a31721b, 'traversability': 0xe50973c4, 'nx': 0x9f850fba, 'ny': 0x1893418b, 'nz': 0xe9752c2e},
    '8192': {'slope': 0xcb719ff9, 'step': 0xad36fe7b, 'roughness': 0xab037a1d, 'traversability': 0xce82e1ae},
}


def fused_crcs(te, ctx, n, res, seed, normals):
    import torch
    import bench
    z = bench.terrain_torch(torch, n, 0, n, n, seed, 0.01, torch.device("cuda"))  # (cols, rows): column-major map
    torch.cuda.synchronize()  # the context runs on its own stream: the input must be complete
    g, p = te.Geometry.make(n, n, res), te.ChainParams.yaml_defaults(0)
    names = LAYERS + (NORMALS if normals else ())
    outs = {k: torch.empty((n, n), dtype=torch.float32, device="cuda") for k in names}
    ctx.set_stream(None)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        ctx.chain(g, p, z, *(outs[k] for k in LAYERS), te.MEM_DEVICE,
                  **({k: outs[k] for k in NORMALS} if normals else {}))
        ctx.synchronize()
        launches, _ = ctx.stats()
        assert launches > 0
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
    return {k: zlib.crc32(outs[k].cpu().numpy().tobytes()) for k in names}


@pytest.mark.parametrize("case", sorted(CASES))
def test_fused_outputs_are_bit_identical(te, ctx, case):
    got = fused_crcs(te, ctx, *CASES[case])
    assert got == EXPECTED[case], {k: (f"{got[k]:#010x}", f"{EXPECTED[case].get(k, 0):#010x}") for k in got if got[k] != EXPECTED[case].get(k)}


if __name__ == "__main__":
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "tools")):
        sys.path.insert(0, p)
    import traversability_estimation_b200 as te_mod
    c = te_mod.Context(0)
    print("EXPECTED = {")
    for name in sorted(CASES):
        crc = fused_crcs(te_mod, c, *CASES[name])
        print(f"    {name!r}: {{" + ", ".join(f"{k!r}: {v:#010x}" for k, v in crc.items()) + "},")
    print("}")
    c.close()
