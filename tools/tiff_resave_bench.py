"""resave from TIFF: does host TIFF reading bound it?  N seeded views (default 2 of 2048 x 2048 x 256 uint16) are
written three ways -- uncompressed TIFF, Deflate TIFF (zlib level 1, 64-row strips) and raw N5 (128 x 128 x 64
blocks) -- and each is re-saved to OME-ZARR with the default pyramid (propose_mipmaps) and zstd level 3, the three
sources alternating for --rounds rounds.  Prints the card, its power limit, and per run GB/s of s0 end to end and the
split: read + decode of the source (TIFF or N5), read + decode of the stored levels read back for the pyramid,
upload, the `downsample` kernel (profile tag), and compress + write.

    python tools/tiff_resave_bench.py [--views 2] [--size 2048,2048,256] [--rounds 2] [--workdir /tmp]

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
from bsgpu import commands, n5 as bn5, spimdata, tiff as btiff  # noqa: E402
from bsgpu import zarr as bz  # noqa: E402
from tests.tiff_files import write_tiff  # noqa: E402


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


def make_inputs(root, views, size):
    """The same seeded views (a coarse random field upsampled 16x plus Gaussian noise, shifted per view and per
    64-plane slab) as raw N5, uncompressed TIFF and Deflate TIFF datasets.  Returns {source: xml}."""
    sx, sy, sz = size
    rng = np.random.default_rng(100)
    coarse = rng.uniform(500, 3000, (4, sy // 16 + 1, sx // 16 + 1)).astype(np.float32)
    base = np.repeat(np.repeat(np.repeat(coarse, 16, 0), 16, 1), 16, 2)[:64, :sy, :sx]
    base += rng.standard_normal(base.shape, dtype=np.float32) * 40.0
    base = np.clip(base, 0, 60000).astype(np.uint16)
    tiles = [dict(setup=s, size_xyz=size, tile=s, translation_xyz=(s * sx * 0.9, 0, 0)) for s in range(views)]
    xmls = {}
    for name in ("n5", "tiff_raw", "tiff_deflate"):
        os.makedirs(os.path.join(root, name))
        xmls[name] = spimdata.write_dataset_xml(os.path.join(root, name, "dataset.xml"), "dataset.n5", tiles)
    store = bn5.N5Store(os.path.join(root, "n5", "dataset.n5"), create=True)
    maps = {"tiff_raw": {}, "tiff_deflate": {}}
    for s in range(views):
        vol = np.concatenate([base[:min(64, sz - z0)] + np.uint16(37 * s + z0 // 64) for z0 in range(0, sz, 64)])
        bn5.write_bdv_setup(store, s, 0, vol, (128, 128, 64), compression="raw")
        maps["tiff_raw"][(0, s)] = (write_tiff(os.path.join(root, "tiff_raw", f"tile{s}.tif"), list(vol), big=True), 0, 0)
        maps["tiff_deflate"][(0, s)] = (write_tiff(os.path.join(root, "tiff_deflate", f"tile{s}.tif"), list(vol),
                                                   big=True, compression=8, rows_per_strip=64, level=1), 0, 0)
        print(f"input view {s} written", flush=True)
    for name, m in maps.items():
        d = spimdata.SpimData2.load(xmls[name])
        d.set_file_map_loader(m)
        d.save(xmls[name], backup=False)
    return xmls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=2)
    ap.add_argument("--size", default="2048,2048,256")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    size = tuple(int(v) for v in a.size.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    root = tempfile.mkdtemp(prefix="tiff_resave_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        xmls = make_inputs(root, a.views, size)
        t_make = time.perf_counter() - t0
        ctx = bsgpu.Context(0)
        T = Timer()
        T.wrap(btiff.Series, "read_region", "read_decode_source")
        T.wrap(bn5.N5Store, "read_region", "read_decode_n5")          # the N5 source
        T.wrap(bz.ZarrStore, "read_region", "read_decode_levels")     # stored levels read back for the pyramid
        T.wrap(commands._Sink, "save", "compress_write")              # every block or chunk resave writes
        T.wrap(commands._Sink, "save_chunk", "compress_write")
        T.wrap(ctx, "volume_upload", "upload")
        s0_bytes = a.views * size[0] * size[1] * size[2] * 2
        print(f"inputs ready in {t_make:.1f} s", flush=True)
        runs = []
        for r in range(a.rounds):
            for name, xml in xmls.items():
                T.t.clear()
                xo = os.path.join(root, f"out_{name}_{r}", "dataset.xml")
                os.makedirs(os.path.dirname(xo))
                ctx.profile_enable(True)
                ctx.profile_reset()
                t0 = time.perf_counter()
                commands.resave(xml, ctx, xml_out=xo)
                ctx.synchronize()
                wall = time.perf_counter() - t0
                ds_ms, ds_n = ctx.profile_get("downsample")
                ctx.profile_enable(False)
                src = T.t.get("read_decode_n5" if name == "n5" else "read_decode_source", 0.0)
                runs.append(dict(source=name, round=r, wall_s=round(wall, 2), GB_per_s=round(s0_bytes / 1e9 / wall, 3),
                                 split_s=dict(read_decode_source=round(src, 2),
                                              read_decode_levels=round(T.t.get("read_decode_levels", 0.0), 2),
                                              upload=round(T.t.get("upload", 0.0), 2),
                                              downsample_kernel=round(ds_ms / 1e3, 3), downsample_launches=ds_n,
                                              compress_write=round(T.t.get("compress_write", 0.0), 2))))
                print(json.dumps(runs[-1]), flush=True)
                shutil.rmtree(os.path.dirname(xo))
        ctx.close()
        print(json.dumps(dict(card=card, views=a.views, size_xyz=list(size), s0_GB=round(s0_bytes / 1e9, 3),
                              input_setup_s=round(t_make, 2), runs=runs)))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
