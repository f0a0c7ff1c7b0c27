"""estimate-bounding-box throughput: a seeded 2 x 2-tile dataset of 1024 x 1024 x 256 uint16 views (10 % overlap,
BDV-N5, raw 128 x 128 x 64 blocks) with a bright ellipsoid covering part of the field and scattered beads, estimated at
--downsampling 1, 2 and 4 with the default --minObjectSize 25 and --background 5.  Prints one JSON line: the card and its
power limit (read in the same run), and per downsampling the end-to-end seconds, the device time of every stage
(profile tags `fuse_plan` + `fuse`, `min_filter`, `min_max`, `threshold_bbox`), the host time spent reading and
uploading the source volumes, and the min filter's rate at 8 B per voxel per pass against the data sheet's 3.35 TB/s.

    python tools/bbox_bench.py [--tile 1024,1024,256] [--repeats 2] [--workdir /tmp]

Everything it writes goes to a temporary directory under --workdir, removed at the end."""
import argparse
import json
import math
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bsgpu  # noqa: E402
from bsgpu import commands, n5 as bn5, spimdata  # noqa: E402

HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes / s
MF_MAX_R = 64               # largest radius of one bs_min_filter pass (csrc/bbox.cu)


def make_dataset(root, tile, overlap=0.1, n_beads=3000, seed=5):
    """2 x 2 tiles cut from one seeded world: background 100 + N(0, 5), +800 inside an ellipsoid over the middle of the
    field, Gaussian beads (sigma 1.5, peak 2000) scattered everywhere.  Generated on the device, tile by tile."""
    import torch
    step = int(round(tile[0] * (1.0 - overlap)))
    world = (step + tile[0], step + tile[1], tile[2])
    rng = np.random.default_rng(seed)
    beads = rng.uniform((0, 0, 0), world, (n_beads, 3))
    centre = np.array(world) * np.array([0.55, 0.45, 0.5])
    radii = np.array(world) * np.array([0.3, 0.25, 0.35])
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    g = torch.Generator(device="cuda")
    for j in range(2):
        for i in range(2):
            s = 2 * j + i
            off = (step * i, step * j, 0)
            g.manual_seed(seed * 100 + s)
            z, y, x = (torch.arange(tile[d], device="cuda", dtype=torch.float32) + off[d] for d in (2, 1, 0))
            v = 100.0 + 5.0 * torch.randn((tile[2], tile[1], tile[0]), generator=g, device="cuda")
            inside = (((x[None, None, :] - centre[0]) / radii[0]) ** 2 + ((y[None, :, None] - centre[1]) / radii[1]) ** 2
                      + ((z[:, None, None] - centre[2]) / radii[2]) ** 2) <= 1.0
            v += 800.0 * inside
            for b in beads:
                lo = [int(math.floor(b[d] - off[d])) - 4 for d in range(3)]
                if any(lo[d] + 9 <= 0 or lo[d] >= tile[d] for d in range(3)):
                    continue
                a = [max(lo[d], 0) for d in range(3)]
                e = [min(lo[d] + 9, tile[d]) for d in range(3)]
                dz, dy, dx = (torch.arange(a[d], e[d], device="cuda", dtype=torch.float32) + off[d] - float(b[d])
                              for d in (2, 1, 0))
                v[a[2]:e[2], a[1]:e[1], a[0]:e[0]] += 2000.0 * torch.exp(
                    -(dz[:, None, None] ** 2 + dy[None, :, None] ** 2 + dx[None, None, :] ** 2) / (2 * 1.5 ** 2))
            host = torch.clamp(torch.round(v), 0, 65535).to(torch.int32).cpu().numpy().astype(np.uint16)
            bn5.write_bdv_setup(store, s, 0, host, (128, 128, 64))
            tiles.append(dict(setup=s, size_xyz=tile, tile=s, translation_xyz=off))
            del v, inside, host
    return spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)


class Timer:
    def __init__(self):
        self.t = {}

    def wrap(self, obj, name, key):
        f = getattr(obj, name)

        def w(*a, **k):
            t0 = time.perf_counter()
            try:
                return f(*a, **k)
            finally:
                self.t[key] = self.t.get(key, 0.0) + time.perf_counter() - t0
        setattr(obj, name, w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tile", default="1024,1024,256")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    tile = tuple(int(v) for v in a.tile.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    tmp = tempfile.mkdtemp(prefix="bbox_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        xml = make_dataset(tmp, tile)
        t_make = time.perf_counter() - t0
        print(f"dataset ready in {t_make:.1f} s", flush=True)
        ctx = bsgpu.Context(0)
        commands.estimate_bounding_box(xml, ctx, "warm", downsampling=4, dry_run=True)      # module load, first launches
        T = Timer()
        T.wrap(bn5.N5Store, "read_region", "read")
        T.wrap(bn5.N5Store, "read_volume", "read")
        T.wrap(ctx, "volume_upload", "upload")
        tags = ("fuse_plan", "fuse", "min_filter", "min_max", "threshold_bbox")
        runs = []
        for ds in (1, 2, 4):
            for rep in range(a.repeats):
                T.t.clear()
                ctx.profile_enable(True)
                ctx.profile_reset()
                t0 = time.perf_counter()
                res = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=ds, dry_run=True)
                wall = time.perf_counter() - t0
                prof = {tag: ctx.profile_get(tag) for tag in tags}
                ctx.profile_enable(False)
                vox = int(np.prod(res["dims"]))
                passes = 3 * max(1, -(-res["radius"] // MF_MAX_R))
                mf_s = prof["min_filter"][0] / 1e3
                mf_rate = 8.0 * vox * passes / mf_s if mf_s > 0 else float("nan")
                runs.append(dict(downsampling=ds, repeat=rep, dims=res["dims"], radius=res["radius"],
                                 box=[res["min"], res["max"]], count=res["count"], wall_s=round(wall, 3),
                                 device_ms={tag: round(ms, 3) for tag, (ms, _) in prof.items()},
                                 launches={tag: n for tag, (_, n) in prof.items()},
                                 host_s=dict(read=round(T.t.get("read", 0.0), 3), upload=round(T.t.get("upload", 0.0), 3)),
                                 min_filter_GB_per_s=round(mf_rate / 1e9, 1),
                                 min_filter_share_of_hbm_peak=round(mf_rate / HBM_PEAK, 3)))
                print(f"ds {ds} #{rep}: {wall:.2f} s, min_filter {prof['min_filter'][0]:.2f} ms", flush=True)
        ctx.close()
        print(json.dumps(dict(card=card, tile_xyz=list(tile), views=4, overlap=0.1, input_setup_s=round(t_make, 1),
                              runs=runs)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
