"""resave throughput: N seeded views (default 8 of 2048 x 2048 x 256 uint16) in a BDV-N5 container, re-saved to OME-ZARR
with the default pyramid (propose_mipmaps) and zstd level 3.  Prints the card, its power limit, GB/s of s0 end to end,
and where the time went: read + decode, upload, the `downsample` kernel (profile tag), download, the split of each
downloaded level into storage chunks, compress + write.

    python tools/resave_bench.py [--views 8] [--size 2048,2048,256] [--workdir /tmp]

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
from bsgpu import zarr as bz  # noqa: E402


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


def make_input(root, views, size):
    """Seeded uint16 views in raw N5 blocks: one smooth-plus-noise 64-plane slab (a coarse random field upsampled 16x,
    plus Gaussian noise), shifted by a per-view, per-slab offset so that no two slabs are equal."""
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    sx, sy, sz = size
    rng = np.random.default_rng(100)
    coarse = rng.uniform(500, 3000, (4, sy // 16 + 1, sx // 16 + 1)).astype(np.float32)
    base = np.repeat(np.repeat(np.repeat(coarse, 16, 0), 16, 1), 16, 2)[:64, :sy, :sx]
    base += rng.standard_normal(base.shape, dtype=np.float32) * 40.0
    base = np.clip(base, 0, 60000).astype(np.uint16)
    for s in range(views):
        store.set_attributes(f"setup{s}", {"downsamplingFactors": [[1, 1, 1]], "dataType": "uint16"})
        store.create_dataset(bn5.bdv_dataset(s, 0, 0), size, (128, 128, 64), np.uint16, "raw")
        for z0 in range(0, sz, 64):
            slab = base[:min(64, sz - z0)] + np.uint16(37 * s + z0 // 64)
            store.save_block(bn5.bdv_dataset(s, 0, 0), slab, (0, 0, z0 // 64))
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(s * sx * 0.9, 0, 0)))
        print(f"input view {s} written", flush=True)
    return spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", default="2048,2048,256")
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    size = tuple(int(v) for v in a.size.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    root = tempfile.mkdtemp(prefix="resave_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        xml = make_input(root, a.views, size)
        t_make = time.perf_counter() - t0
        ctx = bsgpu.Context(0)
        T = Timer()
        # read + decode of the source and of stored levels; compress + write of every chunk
        for cls in (bn5.N5Store, bz.ZarrStore):
            T.wrap(cls, "read_region", "read_decode")
        T.wrap(bz.ZarrStore, "write_chunk", "compress_write")
        T.wrap(bz.ZarrStore, "save_block", "split_compress_write")
        T.wrap(ctx, "volume_upload", "upload")
        T.wrap(ctx, "volume_download", "download")
        ctx.profile_enable(True)
        ctx.profile_reset()
        xo = os.path.join(root, "out", "dataset.xml")
        os.makedirs(os.path.dirname(xo))
        print(f"input ready in {t_make:.1f} s; resaving", flush=True)
        t0 = time.perf_counter()
        plan = commands.resave(xml, ctx, xml_out=xo)
        ctx.synchronize()
        wall = time.perf_counter() - t0
        ds_ms, ds_n = ctx.profile_get("downsample")
        ctx.profile_enable(False)
        s0_bytes = a.views * size[0] * size[1] * size[2] * 2

        ctx.close()
        out = dict(card=card, views=a.views, size_xyz=list(size), downsamplings=[list(s) for s in plan["downsamplings"]],
                   compute_blocks=plan["compute_blocks"], input_setup_s=round(t_make, 2), wall_s=round(wall, 2),
                   s0_GB=round(s0_bytes / 1e9, 3), GB_per_s=round(s0_bytes / 1e9 / wall, 3),
                   split_s=dict(read_decode=round(T.t.get("read_decode", 0.0), 2), upload=round(T.t.get("upload", 0.0), 2),
                                downsample_kernel=round(ds_ms / 1e3, 3), downsample_launches=ds_n,
                                download=round(T.t.get("download", 0.0), 2),
                                split_chunks=round(T.t.get("split_compress_write", 0.0) - T.t.get("compress_write", 0.0), 2),
                                compress_write=round(T.t.get("compress_write", 0.0), 2)))
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
