"""Measure `detect-interestpoints` on one seeded 1024x1024x256 uint16 bead view (the per-tile shape of BASELINE
configs[3]) at -dsxy 2 with --medianFilter off / 5 / 10 / 20.

Prints one JSON line: per-stage device time from the bs_profile tags (downsample, median, dog_load / dog_blur /
dog_extrema, sample), end-to-end seconds per view (N5 read + upload included), the median stage's Mvoxel/s next to its
operations model, the card name and power limit read in the same run, and, labelled as a CPU figure,
scipy.ndimage.median_filter (single thread) on a few of the same slices.  The dataset goes to a temporary directory.

    python tools/ip_detect_bench.py [--size 1024x1024x256] [--radii 0,5,10,20] [--reps 3] [--out result.json]
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

STAGES = ("downsample", "median", "dog_load", "dog_blur", "dog_extrema", "sample")


def bead_view(size_xyz, seed=11, n_beads=4000):
    from scipy.ndimage import gaussian_filter
    nx, ny, nz = size_xyz
    rng = np.random.default_rng(seed)
    img = np.zeros((nz, ny, nx), np.float32)
    img[rng.integers(0, nz, n_beads), rng.integers(0, ny, n_beads), rng.integers(0, nx, n_beads)] = 4.0e5
    img = gaussian_filter(img, (1.5, 2.5, 2.5), output=np.float32)
    yy = np.linspace(0.0, 1.0, ny, dtype=np.float32)[None, :, None]
    img += 100.0 + 60.0 * yy                                   # a background slope for the median to take out
    img += rng.normal(0.0, 4.0, img.shape).astype(np.float32)
    return np.clip(np.rint(img), 0, 65535).astype(np.uint16)


def fkeys(a):
    u = a.astype(np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def bisection_passes(slice_f32, radius):
    """Counting passes k_median_divide runs per voxel on this slice: the bits below the common prefix of the footprint's
    minimum and maximum key (0 when they are equal)."""
    from scipy.ndimage import maximum_filter, minimum_filter
    from oracle import ip_oracle as io
    fp = io.imagej_footprint(radius)
    k = fkeys(slice_f32)
    lo = minimum_filter(k, footprint=fp, mode="reflect")
    hi = maximum_filter(k, footprint=fp, mode="reflect")
    x = (lo ^ hi).astype(np.uint64)
    bits = np.zeros(x.shape, np.int64)
    while np.any(x):
        bits += x > 0
        x >>= np.uint64(1)
    return float(bits.mean())


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="1024x1024x256")
    ap.add_argument("--radii", default="0,5,10,20")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-slices", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bsgpu
    from bsgpu import commands, n5 as bn5, spimdata
    from oracle import ip_oracle as io
    size = tuple(int(v) for v in a.size.split("x"))
    radii = [int(r) for r in a.radii.split(",")]
    result = {"workload": f"one {a.size} uint16 bead view, -dsxy 2 -dsz 1, sigma 1.8, threshold 0.008, blockSize 512,512,128"}
    result["card"], result["nvidia_smi"] = card()
    with tempfile.TemporaryDirectory() as tmp:
        vol = bead_view(size)
        st = bn5.N5Store(os.path.join(tmp, "dataset.n5"), create=True)
        bn5.write_bdv_setup(st, 0, 0, vol, (256, 256, 64))
        xml = spimdata.write_dataset_xml(os.path.join(tmp, "dataset.xml"), "dataset.n5",
                                         [dict(setup=0, size_xyz=size, tile=0, translation_xyz=(0, 0, 0))])
        ds_img = io.downsample_float(vol, (2, 2, 1))
        dvox = ds_img.size
        rows = []
        with bsgpu.Context(0) as ctx:
            for r in radii:
                kw = dict(sigma=1.8, threshold=0.008, min_intensity=0.0, max_intensity=2048.0 if not r else 20.0,
                          downsample_xy=2, median_filter=r or None, store_intensities=True, dry_run=True)
                commands.detect_interestpoints(xml, ctx, "bench", **kw)           # warm-up (modules, allocations)
                e2e, prof, npts = [], {s: 0.0 for s in STAGES}, 0
                for _ in range(a.reps):
                    ctx.profile_enable(True)
                    ctx.profile_reset()
                    t0 = time.perf_counter()
                    res = commands.detect_interestpoints(xml, ctx, "bench", **kw)
                    ctx.synchronize()
                    e2e.append(time.perf_counter() - t0)
                    for s in STAGES:
                        prof[s] += ctx.profile_get(s)[0] / a.reps
                    ctx.profile_enable(False)
                    npts = len(res[(0, 0)][0])
                row = {"median_radius": r, "points": npts, "e2e_s_per_view": [round(v, 3) for v in e2e],
                       "device_ms": {s: round(v, 3) for s, v in prof.items()}}
                if r:
                    n = int(io.imagej_footprint(r).sum())
                    passes = float(np.mean([bisection_passes(ds_img[z], r) for z in (0, ds_img.shape[0] // 2)]))
                    ms = prof["median"]
                    reads = dvox * n * (1 + passes)
                    row["median"] = {"mvoxel_per_s": round(dvox / ms / 1e3, 1), "footprint_points": n,
                                     "mean_counting_passes": round(passes, 2),
                                     "shared_key_reads_per_voxel": round(n * (1 + passes)),
                                     "shared_key_reads_per_s": f"{reads / ms * 1e3:.3e}"}
                    from scipy.ndimage import median_filter
                    fp = io.imagej_footprint(r)
                    t0 = time.perf_counter()
                    for z in range(a.cpu_slices):
                        median_filter(ds_img[z], footprint=fp, mode="reflect")
                    dt = time.perf_counter() - t0
                    row["cpu_scipy_median_filter"] = {
                        "mvoxel_per_s": round(a.cpu_slices * ds_img[0].size / dt / 1e6, 3), "threads": 1,
                        "sample": f"scipy.ndimage.median_filter on {a.cpu_slices} of the {ds_img.shape[0]} downsampled slices"}
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    result["runs"] = rows
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
