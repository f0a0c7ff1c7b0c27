"""Intensity-correction benchmark: two 2048 x 2048 x 256 uint16 views at 10 % overlap in x, match-intensities at its
defaults (8,8,8 coefficients, render scale 0.25, 1000 iterations), then the coefficient application and the fusion of
the overlap with and without corrected sources.  Prints one JSON line with the card and its power limit.

    python tools/intensity_bench.py [--size 2048,2048,256] [--overlap 0.1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bsgpu  # noqa: E402
from bsgpu import intensity as bint  # noqa: E402

HBM_TBS = 3.35


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def view(nx, ny, nz, gain, seed):
    z = np.arange(nz, dtype=np.float32)[:, None, None]
    y = np.arange(ny, dtype=np.float32)[None, :, None]
    rng = np.random.default_rng(seed)
    out = np.empty((nz, ny, nx), np.uint16)
    for z0 in range(0, nz, 16):
        zz = z[z0:z0 + 16]
        x = np.arange(nx, dtype=np.float32)[None, None, :] + seed * 0.0
        I = 600 + 250 * np.sin((x + gain[1]) / 41.0) * np.cos(y / 57.0) + 2 * zz
        out[z0:z0 + 16] = np.clip(gain[0] * I + rng.normal(0, 3, I.shape), 0, 65535).astype(np.uint16)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="2048,2048,256")
    ap.add_argument("--overlap", type=float, default=0.1)
    args = ap.parse_args()
    nx, ny, nz = (int(v) for v in args.size.split(","))
    shift = int(round(nx * (1 - args.overlap)))
    A = view(nx, ny, nz, (1.0, 0.0), 1)
    B = view(nx, ny, nz, (1.2, float(shift)), 2)
    regA = np.eye(3, 4)
    regB = np.eye(3, 4)
    regB[0, 3] = shift
    n = (8, 8, 8)
    res = dict(card=card(), size=[nx, ny, nz], overlap=args.overlap)
    with bsgpu.Context(0) as ctx:
        ha, hb = ctx.volume_upload(A), ctx.volume_upload(B)
        va = bint.device_view(ha, regA, np.eye(3, 4), (nx, ny, nz), n)
        vb = bint.device_view(hb, regB, np.eye(3, 4), (nx, ny, nz), n)
        lo = np.maximum(bint.view_bounds((nx, ny, nz), regA)[0], bint.view_bounds((nx, ny, nz), regB)[0])
        hi = np.minimum(bint.view_bounds((nx, ny, nz), regA)[1], bint.view_bounds((nx, ny, nz), regB)[1])
        rmin, rmax = bint.render_range(lo, hi, 0.25)
        kw = (0.25, rmin, rmax, 1.0, float("nan"), 1000, 1000, 5.1, 0.1, 10, 3.0)
        bint.match_pair(ctx, va, vb, *kw)                                   # warm-up
        ctx.profile_enable(True)
        ctx.profile_reset()
        t0 = time.perf_counter()
        cells, counts = bint.match_pair(ctx, va, vb, *kw)
        ctx.synchronize()
        res["match_pair_s"] = time.perf_counter() - t0
        res["intensity_render_ms"] = ctx.profile_get("intensity_render")[0]
        res["intensity_ransac_ms"] = ctx.profile_get("intensity_ransac")[0]
        res.update(counts)
        # the host part of match_pair: filter + acceptance of every eligible bucket
        h, keys, offs, cnts, vals = ctx.intensity_candidates(va, vb, *kw[:5])
        a, b, c = ctx.intensity_ransac(h, len(keys), 1000, 1000, 5.1)
        ctx.intensity_candidates_free(h)
        t0 = time.perf_counter()
        for k in np.nonzero(c > 0)[0]:
            v = vals[offs[k]:offs[k] + cnts[k]]
            bint.filter_accept(v[:, 0], v[:, 1], a[k], b[k], 5.1, 3.0, 0.1, 10)
        res["host_filter_s"] = time.perf_counter() - t0
        res["residuals"] = int(sum(int(cnts[k]) * 1000 for k in range(len(keys)) if c[k] >= 0))
        # application: 2 B in + 4 B out per voxel
        ca = np.full((8, 8, 8), 1.1)
        cb = np.full((8, 8, 8), -3.0)
        hc = ctx.intensity_apply(hb, (nx, ny, nz), np.eye(3, 4), ca, cb)
        ctx.volume_free(hc)
        ctx.profile_reset()
        reps = 5
        for _ in range(reps):
            hc = ctx.intensity_apply(hb, (nx, ny, nz), np.eye(3, 4), ca, cb)
            ctx.volume_free(hc)
        ms = ctx.profile_get("intensity_apply")[0] / reps
        res["intensity_apply_ms"] = ms
        res["intensity_apply_GBs"] = 6.0 * nx * ny * nz / (ms * 1e6)
        res["intensity_apply_share_of_hbm"] = res["intensity_apply_GBs"] / (HBM_TBS * 1e3)
        # fusion of the overlap slab from raw uint16 and from corrected float32 sources
        hca = ctx.intensity_apply(ha, (nx, ny, nz), np.eye(3, 4), np.ones((8, 8, 8)), np.zeros((8, 8, 8)))
        hcb = ctx.intensity_apply(hb, (nx, ny, nz), np.eye(3, 4), ca, cb)
        blocks = [((shift - 64 + 256 * i, 256 * j, 0), (256, 256, 128)) for i in range(2) for j in range(8)]
        for name, hs in (("fuse_raw_ms", (ha, hb)), ("fuse_corrected_ms", (hca, hcb))):
            views = [dict(src_to_world=r, vol_handle=h, blend_border=(0, 0, 0), blend_range=(40, 40, 40))
                     for r, h in zip((regA, regB), hs)]
            ctx.fuse_blocks(views, [m for m, _ in blocks], [s for _, s in blocks])
            ctx.profile_reset()
            ctx.fuse_blocks(views, [m for m, _ in blocks], [s for _, s in blocks])
            res[name] = ctx.profile_get("fuse")[0]
        for h in (ha, hb, hca, hcb):
            ctx.volume_free(h)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
