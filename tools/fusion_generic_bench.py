"""Per-call timing of affine fusion's generic tile kernel (csrc/fuse.cu), the path bench.py does not time: what the TMA
kernels do not take (winner fusion types, nearest neighbour, float32 sources, the blend LUT) and the view-sharded
partial sums of multi-GPU fusion (bs_fuse_accumulate over two halves of the views, then bs_fuse_finish).

Seeded scene: --tiles views of --tile voxels (x, y, z; default 6 of 512 x 512 x 256) cut with 10 % overlap from one
smooth random field, on a 3-wide grid with sub-pixel jitter.  Their union is split into --block cubes (default 256^3)
and every block is one call with the views that overlap it, output on the device.  Each case is timed with CUDA
events over all its blocks.

Every --lib (default: the library of this tree) is one build of libbsgpu.so, e.g. a parent commit's and a change's.
The libraries fuse from the same device buffers on the same stream; one untimed pass checks that every library writes
byte-identical blocks to the first one's, then the libraries take turns, --repeats rounds per case.  Prints the card,
its power limit and, per case and library, the median ms per call, the spread of the rounds and Mvoxels/s as one JSON
line.

    python tools/fusion_generic_bench.py [--lib A.so --lib B.so] [--tiles 6] [--tile 512,512,256] [--block 256]
                                         [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bsgpu  # noqa: E402
from bsgpu import fusion as bf  # noqa: E402

nat = bsgpu.native

# name: (fusion type, interpolation, source dtype, blend LUT size, output dtype, accumulate)
CASES = {
    "MAX_INTENSITY": ("MAX_INTENSITY", 1, "u16", 0, nat.DTYPE_U16, False),
    "nearest_neighbour": ("AVG_BLEND", 0, "u16", 0, nat.DTYPE_F32, False),
    "float32_sources": ("AVG_BLEND", 1, "f32", 0, nat.DTYPE_F32, False),
    "blend_lut": ("AVG_BLEND", 1, "u16", 100, nat.DTYPE_F32, False),
    "accumulate": ("AVG_BLEND", 1, "u16", 0, nat.DTYPE_F32, True),
}


def make_scene(n, size, seed, dev):
    """uint16 and float32 device tiles (the same values) and their registrations."""
    import torch
    import torch.nn.functional as F
    g = torch.Generator(device=dev).manual_seed(seed)
    rng = np.random.default_rng(seed)
    sx, sy, sz = size
    cols = min(n, 3)
    rows = (n + cols - 1) // cols
    step = (int(sx * 0.9), int(sy * 0.9))
    W, H = step[0] * (cols - 1) + sx, step[1] * (rows - 1) + sy
    coarse = torch.rand((1, 1, sz // 8 + 1, H // 8 + 1, W // 8 + 1), generator=g, device=dev) * 2500.0 + 500.0
    field = F.interpolate(coarse, size=(sz, H, W), mode="trilinear", align_corners=False)[0, 0]
    u16, f32, models = [], [], []
    for i in range(n):
        x0, y0 = (i % cols) * step[0], (i // cols) * step[1]
        t = field[:, y0:y0 + sy, x0:x0 + sx] + torch.randn((sz, sy, sx), generator=g, device=dev) * 40.0
        t = t.clamp(0.0, 60000.0).round()
        u16.append(t.to(torch.int32).to(torch.uint16).contiguous())
        f32.append(t.contiguous())
        models.append(np.hstack([np.eye(3), (np.array([x0, y0, 0.0]) + rng.uniform(-2, 2, 3))[:, None]]))
    del field, coarse
    return u16, f32, models, (W, H, sz)


def library_context(path, stream):
    """A context of the libbsgpu.so at ``path`` (each path is loaded once, next to any other)."""
    nat._lib = None
    nat.LIB_PATH = os.path.abspath(path)
    return nat.Context(0, stream=stream.cuda_stream)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None)
    ap.add_argument("--tiles", type=int, default=6)
    ap.add_argument("--tile", default="512,512,256")
    ap.add_argument("--block", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    import torch
    libs = a.lib or [nat.LIB_PATH]
    dev = torch.device("cuda", 0)
    # the contexts launch on this stream too (not the legacy default stream, which they would replace by their own)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    size = tuple(int(v) for v in a.tile.split(","))
    u16, f32, models, extent = make_scene(a.tiles, size, a.seed, dev)
    torch.cuda.synchronize()
    regs = dict(enumerate(models))
    dims = {i: size for i in regs}
    blocks = [(off, sz) for off, sz, _ in bf.grid_create(extent, (a.block,) * 3)]
    vids = [bf.find_overlapping_views(dims, regs, off, tuple(off[d] + sz[d] - 1 for d in range(3))) for off, sz in blocks]
    block_vox = sum(int(np.prod(sz)) for _, sz in blocks)

    ctxs = [library_context(p, stream) for p in libs]
    handles = [{"u16": [c.volume_wrap(t, size, nat.DTYPE_U16) for t in u16],
                "f32": [c.volume_wrap(t, size, nat.DTYPE_F32) for t in f32]} for c in ctxs]
    nmax = max(int(np.prod(sz)) for _, sz in blocks)
    outs = [torch.empty(nmax * 4, dtype=torch.uint8, device=dev) for _ in ctxs]
    swi = torch.empty(nmax, dtype=torch.float32, device=dev)
    sw = torch.empty(nmax, dtype=torch.float32, device=dev)

    def calls(li, case):
        """one closure per block: the call a user makes for it, output into outs[li]"""
        ft, interp, src, lut, out_dt, acc = CASES[case]
        c = ctxs[li]
        p = c.fuse_params(ft, interp, out_dt, lut, 0.0, 4000.0)
        res = []
        for (off, sz), vs in zip(blocks, vids):
            gv = [dict(src_to_world=models[v], vol_handle=handles[li][src][v], blend_border=bf.adjust_blending(models[v])[0],
                       blend_range=bf.adjust_blending(models[v])[1]) for v in vs]
            nv = int(np.prod(sz))
            out = outs[li][:nv * (4 if out_dt == nat.DTYPE_F32 else 2)]
            if acc:
                h = (len(gv) + 1) // 2
                va, vb = c.make_views(gv[:h]), c.make_views(gv[h:])

                def f(c=c, va=va, vb=vb, off=off, sz=sz, p=p, nv=nv, out=out):
                    swi[:nv].zero_()
                    sw[:nv].zero_()
                    c.fuse_accumulate(va, off, sz, p, swi, sw)
                    c.fuse_accumulate(vb, off, sz, p, swi, sw)
                    c.fuse_finish(swi, sw, nv, p, out)
            else:
                views = c.make_views(gv)

                def f(c=c, views=views, off=off, sz=sz, p=p, out=out):
                    c.fuse_block(views, off, sz, p, out=out)
            res.append((f, out))
        return res

    result = {"card_power_limit": card, "tiles": a.tiles, "tile_xyz": size, "blocks": len(blocks),
              "block_voxels": block_vox, "libs": libs, "cases": {}}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for case in CASES:
        per_lib = [calls(li, case) for li in range(len(ctxs))]
        # untimed pass (also the warm-up): every block of every library against the first library's
        mismatches = 0
        for b in range(len(blocks)):
            ref = None
            for li, cl in enumerate(per_lib):
                f, out = cl[b]
                f()
                if ref is None:
                    ref = out.clone()
                elif not torch.equal(ref, out):
                    mismatches += 1
        times = [[] for _ in ctxs]
        for r in range(a.repeats):
            order = list(range(len(ctxs)))
            if r % 2:
                order.reverse()
            for li in order:
                start.record(stream)
                for f, _ in per_lib[li]:
                    f()
                end.record(stream)
                end.synchronize()
                times[li].append(start.elapsed_time(end) / len(blocks))
        result["cases"][case] = {
            "byte_equal": mismatches == 0, "mismatched_blocks": mismatches,
            "ms_per_call": [round(float(np.median(t)), 3) for t in times],
            "spread_ms": [[round(min(t), 3), round(max(t), 3)] for t in times],
            "mvoxels_s": [round(block_vox / (float(np.median(t)) * len(blocks) / 1000.0) / 1e6, 1) for t in times]}
        print(case, json.dumps(result["cases"][case]), file=sys.stderr, flush=True)
    for c in ctxs:
        c.close()
    print(json.dumps(result), flush=True)
    if not all(v["byte_equal"] for v in result["cases"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
