"""extract-psfs throughput: two seeded 2048 x 2048 x 400 uint16 views (BDV-N5, raw 128 x 128 x 64 blocks) of 50 000
detections each, numbered in the order detect-interestpoints writes them (1024 x 1024 x 128 full-resolution blocks,
z-blocks outermost) or, with --order intensity, in an order that does not follow space (as --maxSpots numbers them),
extracted with the default 19 x 19 x 25 box and --allPoints.  Prints one JSON line: the card and its power
limit (read in the same run), and per repeat the end-to-end seconds, the device time of the `psf` kernel, the host time
spent reading the s0 windows and uploading them, and the number of windows.

    python tools/psf_bench.py [--view 2048,2048,400] [--points 50000] [--order blocks|intensity] [--repeats 2]
                              [--workdir /tmp]

Everything it writes goes to a temporary directory under --workdir, removed at the end."""
import argparse
import json
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


def make_dataset(root, view, n_points, order, seed=7):
    """Two views of background 100 + N(0, 5) (generated on the device, the same pixels for both) and n_points uniform
    detections per view, in detect-interestpoints block order or in random (intensity-like) order."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    host = np.empty(view[::-1], dtype=np.uint16)
    for z0 in range(0, view[2], 50):
        z1 = min(z0 + 50, view[2])
        v = 100.0 + 5.0 * torch.randn((z1 - z0, view[1], view[0]), generator=g, device="cuda")
        host[z0:z1] = torch.clamp(torch.round(v), 0, 65535).to(torch.int32).cpu().numpy().astype(np.uint16)
        del v
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    for s in range(2):
        bn5.write_bdv_setup(store, s, 0, host, (128, 128, 64))
        tiles.append(dict(setup=s, size_xyz=view, tile=s, translation_xyz=(s * view[0], 0, 0)))
    del host
    xml = spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)
    data = spimdata.SpimData2.load(xml)
    ips = bn5.N5Store(os.path.join(root, "interestpoints.n5"), create=True)
    rng = np.random.default_rng(seed)
    for s in range(2):
        loc = rng.uniform((0, 0, 0), view, (n_points, 3))
        if order == "blocks":
            loc = loc[np.lexsort((loc[:, 0] // 1024, loc[:, 1] // 1024, loc[:, 2] // 128))]
        group = f"tpId_0_viewSetupId_{s}/beads"
        commands._write_view_points(ips, group, np.arange(n_points), loc)
        data.set_interest_points("beads", "bench", {(0, s): group})
    data.save(xml, backup=False)
    return xml


class Timer:
    def __init__(self):
        self.t, self.n = {}, {}

    def wrap(self, obj, name, key):
        f = getattr(obj, name)

        def w(*a, **k):
            t0 = time.perf_counter()
            try:
                return f(*a, **k)
            finally:
                self.t[key] = self.t.get(key, 0.0) + time.perf_counter() - t0
                self.n[key] = self.n.get(key, 0) + 1
        setattr(obj, name, w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--view", default="2048,2048,400")
    ap.add_argument("--points", type=int, default=50000)
    ap.add_argument("--order", choices=("blocks", "intensity"), default="blocks")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    view = tuple(int(v) for v in a.view.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    tmp = tempfile.mkdtemp(prefix="psf_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        xml = make_dataset(tmp, view, a.points, a.order)
        t_make = time.perf_counter() - t0
        print(f"dataset ready in {t_make:.1f} s", flush=True)
        ctx = bsgpu.Context(0)
        commands.extract_psfs(xml, ctx, "beads", all_points=True, view_selection=dict(vi=["0,0"]),
                              dry_run=True)                                      # module load, first launches
        T = Timer()
        T.wrap(bn5.N5Store, "read_region", "read")
        T.wrap(ctx, "volume_upload", "upload")
        runs = []
        for rep in range(a.repeats):
            T.t.clear()
            T.n.clear()
            ctx.profile_enable(True)
            ctx.profile_reset()
            t0 = time.perf_counter()
            res = commands.extract_psfs(xml, ctx, "beads", all_points=True, dry_run=True)
            wall = time.perf_counter() - t0
            ms, launches = ctx.profile_get("psf")
            ctx.profile_enable(False)
            runs.append(dict(repeat=rep, wall_s=round(wall, 3), psf_kernel_ms=round(ms, 3), psf_launches=launches,
                             read_s=round(T.t.get("read", 0.0), 3), upload_s=round(T.t.get("upload", 0.0), 3),
                             windows=T.n.get("upload", 0), points=[n for _, n in res.values()]))
            print(f"#{rep}: {wall:.2f} s, psf {ms:.2f} ms in {launches} launches, read {T.t.get('read', 0):.2f} s, "
                  f"upload {T.t.get('upload', 0):.2f} s", flush=True)
        ctx.close()
        print(json.dumps(dict(card=card, view_xyz=list(view), views=2, points_per_view=a.points, order=a.order,
                              psf_size=[19, 19, 25], input_setup_s=round(t_make, 1), runs=runs)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
