"""Measure `nonrigid-fusion` on a seeded 2 x 4 grid of 512x512x256 uint16 tiles with 15 % overlap, each tile warped by
its own smooth non-affine field and registered by its grid translation only, with about 3000 bead correspondences per
overlapping pair (seeded, generated here).

Prints one JSON line: the device time and launch count of the profile tags "mls_grid" and "nonrigid_fuse", the
control-point x point evaluations per second of k_mls_grid, fused Gvoxel/s of k_nonrigid_fuse, the end-to-end command
time (N5 source reads, uploads, zstd output included), the card name and power limit read in the same run, and,
labelled as a CPU figure, the float64 oracle on one bounded super-block.  The dataset goes to a temporary directory.

``--intensity``: instead, write seeded 8x8x8-cell intensity coefficients for every tile and run the command without and
with them (`intensity_n5_path`), alternating, ``--repeats`` times each after one warm-up run of each.  Reports the
seconds end to end of every run, then one profiled run of each with the device time and launch count of
"intensity_apply" next to "mls_grid" and "nonrigid_fuse", and the card name and power limit.

    python tools/nonrigid_bench.py [--tiles 4x2] [--size 512x512x256] [--beads 3000] [--intensity [--repeats 3]]
                                   [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return q


def pattern(w):
    """The world intensity field: a few smooth sinusoids plus a bead-like lattice modulation (float32)."""
    x, y, z = w[..., 0], w[..., 1], w[..., 2]
    return (1000.0 + 300.0 * np.sin(0.11 * x) * np.sin(0.13 * y) + 200.0 * np.cos(0.17 * z + 0.05 * x)
            + 150.0 * np.sin(0.31 * x + 0.23 * y) * np.cos(0.29 * z)).astype(np.float32)


def psi(w, k):
    """Tile k's warp (world px) at world points (..., 3): a smooth field of about 1.5 px."""
    ph = 0.7 * k
    return np.stack([1.5 * np.sin(2 * np.pi * w[..., 2] / 180.0 + ph) * np.cos(2 * np.pi * w[..., 1] / 400.0),
                     1.2 * np.cos(2 * np.pi * w[..., 0] / 350.0 + ph), 0.6 * np.sin(2 * np.pi * w[..., 1] / 300.0 + ph)],
                    axis=-1)


def make_dataset(tmp, tiles_xy, size, n_beads, seed=5):
    from bsgpu import n5 as bn5, spimdata
    from tests.test_nonrigid_cpu import write_correspondences, write_points
    nx, ny = tiles_xy
    step = [int(round(size[d] * 0.85)) for d in range(2)]
    specs = []
    for j in range(ny):
        for i in range(nx):
            specs.append(dict(setup=len(specs), size_xyz=size, translation_xyz=(i * step[0], j * step[1], 0)))
    xml = os.path.join(tmp, "dataset.xml")
    spimdata.write_dataset_xml(xml, "dataset.n5", specs)
    src = bn5.N5Store(os.path.join(tmp, "dataset.n5"), create=True)
    zz, yy, xx = np.meshgrid(np.arange(size[2]), np.arange(size[1]), np.arange(size[0]), indexing="ij")
    for k, s in enumerate(specs):
        img = np.empty(size[::-1], np.uint16)
        for z0 in range(0, size[2], 32):
            sl = slice(z0, z0 + 32)
            w = np.stack([xx[sl], yy[sl], zz[sl]], axis=-1).astype(np.float32) + np.asarray(s["translation_xyz"], np.float32)
            w = w + psi(w, k).astype(np.float32)
            img[sl] = np.clip(np.rint(pattern(w)), 0, 65535)
        bn5.write_bdv_setup(src, s["setup"], 0, img, block_size=(128, 128, 64))
    # beads at true world points in every overlap (neighbours and diagonals); local = solve l + t + psi(l + t) = p
    rng = np.random.default_rng(seed)
    pts = {k: [] for k in range(len(specs))}
    rows = {k: [] for k in range(len(specs))}
    boxes = [(np.asarray(s["translation_xyz"], float), np.asarray(s["translation_xyz"], float) + np.asarray(size) - 1) for s in specs]
    for a in range(len(specs)):
        for b in range(a + 1, len(specs)):
            lo, hi = np.maximum(boxes[a][0], boxes[b][0]) + 3, np.minimum(boxes[a][1], boxes[b][1]) - 3
            if np.any(hi <= lo):
                continue
            p = rng.uniform(lo, hi, (n_beads, 3))
            loc = {}
            for k in (a, b):
                t = boxes[k][0]
                l = p - t
                for _ in range(8):
                    l = p - t - psi(l + t, k)
                loc[k] = l
            ia, ib = len(pts[a]), len(pts[b])
            pts[a].extend(loc[a])
            pts[b].extend(loc[b])
            rows[a] += [(ia + i, (0, b), "beads", ib + i) for i in range(n_beads)]
            rows[b] += [(ib + i, (0, a), "beads", ia + i) for i in range(n_beads)]
    ips = bn5.N5Store(os.path.join(tmp, "interestpoints.n5"), create=True)
    for k in range(len(specs)):
        write_points(ips, (0, k), "beads", np.asarray(pts[k]).reshape(-1, 3))
        write_correspondences(ips, (0, k), "beads", rows[k])
    return xml, sum(len(v) for v in pts.values())


def intensity_runs(ctx, xml, tmp, repeats, res, seed=9):
    """nonrigid-fusion without and with seeded coefficients (a in [0.8, 1.2], b in [-20, 20] per cell), alternating."""
    import shutil
    from bsgpu import commands, intensity as bint, spimdata
    views = spimdata.SpimData2.load(xml).view_ids()
    rng = np.random.default_rng(seed)
    co = {v: (rng.uniform(0.8, 1.2, (8, 8, 8)), rng.uniform(-20.0, 20.0, (8, 8, 8))) for v in views}
    cpath = os.path.join(tmp, "coeff.n5")
    bint.write_coefficients(cpath, "N5", "", "intensity", co)
    modes = {"plain": {}, "intensity": dict(intensity_n5_path=cpath)}

    def run(mode):
        out = os.path.join(tmp, f"{mode}.n5")
        t0 = time.perf_counter()
        blocks = commands.nonrigid_fusion(xml, ctx, out, "fused/s0", ["beads"], data_type="UINT16", min_intensity=0.0,
                                          max_intensity=2000.0, **modes[mode])
        ctx.synchronize()
        s = time.perf_counter() - t0
        shutil.rmtree(out)
        return s, len(blocks)

    for mode in modes:                                   # first calls: module load, allocations
        run(mode)
    secs = {mode: [] for mode in modes}
    for _ in range(repeats):
        for mode in modes:
            s, n = run(mode)
            secs[mode].append(round(s, 2))
            res[f"{mode}_blocks_written"] = n
    for mode in modes:
        res[f"{mode}_command_s"] = secs[mode]
        res[f"{mode}_command_s_median"] = float(np.median(secs[mode]))
        ctx.profile_enable(True)
        ctx.profile_reset()
        run(mode)
        for tag in ("mls_grid", "nonrigid_fuse", "intensity_apply"):
            ms, n = ctx.profile_get(tag)
            res[f"{mode}_{tag}_ms"], res[f"{mode}_{tag}_launches"] = round(ms, 2), n
        ctx.profile_enable(False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", default="4x2")
    ap.add_argument("--size", default="512x512x256")
    ap.add_argument("--beads", type=int, default=3000)
    ap.add_argument("--intensity", action="store_true")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tiles = tuple(int(v) for v in a.tiles.split("x"))
    size = tuple(int(v) for v in a.size.split("x"))
    import bsgpu
    from bsgpu import commands, native
    from oracle import nonrigid_oracle as no
    res = dict(card=card(), tiles=a.tiles, size=a.size, beads_per_pair=a.beads)
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        xml, n_points = make_dataset(tmp, tiles, size, a.beads)
        res["dataset_s"] = round(time.perf_counter() - t0, 1)
        res["points_total"] = n_points
        if a.intensity:
            with bsgpu.Context(0) as ctx:
                intensity_runs(ctx, xml, tmp, a.repeats, res)
            emit(res, a.out)
            return
        with bsgpu.Context(0) as ctx:
            evals = [0]
            voxels = [0]
            fuse, dbg = ctx.nonrigid_fuse_blocks, ctx.nonrigid_debug_grid

            def counted_fuse(views, mins, sizes, *args, **kw):
                npts = sum(len(v["target_world_xyz"]) for v in views)
                for s in sizes:
                    evals[0] += int(np.prod(no.grid_dims(s))) * npts
                    voxels[0] += int(np.prod(s))
                return fuse(views, mins, sizes, *args, **kw)

            def counted_dbg(view, mn, sz, *args, **kw):
                evals[0] += int(np.prod(no.grid_dims(sz))) * len(view["target_world_xyz"])
                return dbg(view, mn, sz, *args, **kw)

            ctx.nonrigid_fuse_blocks, ctx.nonrigid_debug_grid = counted_fuse, counted_dbg
            run = lambda out: commands.nonrigid_fusion(xml, ctx, os.path.join(tmp, out), "fused/s0", ["beads"],
                                                       data_type="UINT16", min_intensity=0.0, max_intensity=2000.0)
            run("warm.n5")                                 # first call: module load, allocations
            evals[0] = voxels[0] = 0
            ctx.profile_enable(True)
            ctx.profile_reset()
            t0 = time.perf_counter()
            blocks = run("fused.n5")
            ctx.synchronize()
            res["command_s"] = round(time.perf_counter() - t0, 2)
            res["blocks_written"] = len(blocks)
            for tag in ("mls_grid", "nonrigid_fuse"):
                ms, n = ctx.profile_get(tag)
                res[f"{tag}_ms"], res[f"{tag}_launches"] = round(ms, 2), n
            res["cp_point_evals"] = evals[0]
            res["cp_point_evals_per_s"] = evals[0] / (res["mls_grid_ms"] * 1e-3)
            res["fused_voxels"] = voxels[0]
            res["fused_gvoxel_per_s"] = voxels[0] / (res["nonrigid_fuse_ms"] * 1e-3) / 1e9
            ctx.profile_enable(False)
        # CPU arm: the float64 oracle on one bounded super-block of the first overlap, two views, 3000 points each
        from tests.test_nonrigid_cpu import translation
        rng = np.random.default_rng(1)
        step = int(round(size[0] * 0.85))
        views = []
        for k, t in enumerate(((0.0, 0.0, 0.0), (float(step), 0.0, 0.0))):
            img = rng.integers(900, 1100, (64, 128, size[0])).astype(np.uint16)
            l = rng.uniform((step - t[0], 0, 0), (size[0] - 1 - t[0], 127, 63), (3000, 3))
            views.append(dict(img=img, src_to_world=translation(t), targets=l + t + rng.normal(0, 1, l.shape), locals=l))
        bsz = (64, 64, 32)
        t0 = time.perf_counter()
        no.fuse_block(views, (step, 32, 16), bsz)
        cpu_s = time.perf_counter() - t0
        res["cpu_oracle_block"] = "x".join(str(v) for v in bsz)
        res["cpu_oracle_s"] = round(cpu_s, 2)
        res["cpu_oracle_mvoxel_per_s"] = round(float(np.prod(bsz)) / cpu_s / 1e6, 4)
    emit(res, a.out)


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
