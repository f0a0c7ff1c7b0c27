"""downsample throughput: a seeded 2048 x 2048 x 256 uint16 N5 dataset s0 (128^3 zstd blocks, what nonrigid-fusion
writes by default) and `-ds "2,2,1; 2,2,1; 2,2,2"` into s1 .. s3, once with the default --blockScale 1,1,1 (every level
re-read from the container) and once with 4,4,2 (s2 and s3 derived from each resident s1 block).  Prints one JSON line:
the card and its power limit, end-to-end seconds and GB/s of s0 per run, and where the time went: read + decode,
upload, the `downsample` kernel (profile tag), download, compress + write.

    python tools/downsample_bench.py [--size 2048,2048,256] [--workdir /tmp]

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
from bsgpu import commands, n5 as bn5  # noqa: E402

STEPS = "2,2,1; 2,2,1; 2,2,2"
OUT = ["s1", "s2", "s3"]
BLOCK = (128, 128, 128)


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


def make_input(root, size):
    """Seeded uint16 s0: a coarse random field upsampled 16x plus Gaussian noise, one 128-plane slab shifted per slab."""
    store = bn5.N5Store(root, create=True)
    sx, sy, sz = size
    rng = np.random.default_rng(100)
    coarse = rng.uniform(500, 3000, (8, sy // 16 + 1, sx // 16 + 1)).astype(np.float32)
    base = np.repeat(np.repeat(np.repeat(coarse, 16, 0), 16, 1), 16, 2)[:BLOCK[2], :sy, :sx]
    base += rng.standard_normal(base.shape, dtype=np.float32) * 40.0
    base = np.clip(base, 0, 60000).astype(np.uint16)
    store.create_dataset("s0", size, BLOCK, np.uint16, "zstd")
    for z0 in range(0, sz, BLOCK[2]):
        store.save_block("s0", base[:min(BLOCK[2], sz - z0)] + np.uint16(z0 // BLOCK[2]), (0, 0, z0 // BLOCK[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="2048,2048,256")
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    size = tuple(int(v) for v in a.size.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    tmp = tempfile.mkdtemp(prefix="downsample_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        src = os.path.join(tmp, "in.n5")
        make_input(src, size)
        t_make = time.perf_counter() - t0
        print(f"input ready in {t_make:.1f} s", flush=True)
        ctx = bsgpu.Context(0)
        # warm-up: module load and the kernel at every step shape, on a small copy
        warm = os.path.join(tmp, "warm.n5")
        bn5.N5Store(warm, create=True).write_volume("s0", np.ones((64, 256, 256), np.uint16), BLOCK, "zstd")
        commands.downsample(warm, ctx, "s0", OUT, STEPS)
        T = Timer()
        T.wrap(bn5.N5Store, "read_region", "read_decode")
        T.wrap(bn5.N5Store, "write_block", "compress_write")
        T.wrap(ctx, "volume_upload", "upload")
        T.wrap(ctx, "volume_download", "download")
        s0_bytes = size[0] * size[1] * size[2] * 2
        runs = []
        for scale in ((1, 1, 1), (4, 4, 2)):
            root = os.path.join(tmp, "run.n5")
            shutil.rmtree(root, ignore_errors=True)
            shutil.copytree(src, root)
            T.t.clear()
            ctx.profile_enable(True)
            ctx.profile_reset()
            t0 = time.perf_counter()
            commands.downsample(root, ctx, "s0", OUT, STEPS, block_scale=scale)
            ctx.synchronize()
            wall = time.perf_counter() - t0
            ds_ms, ds_n = ctx.profile_get("downsample")
            ctx.profile_enable(False)
            runs.append(dict(block_scale=list(scale), wall_s=round(wall, 2), GB_per_s=round(s0_bytes / 1e9 / wall, 3),
                             split_s=dict(read_decode=round(T.t.get("read_decode", 0.0), 2),
                                          upload=round(T.t.get("upload", 0.0), 2),
                                          downsample_kernel=round(ds_ms / 1e3, 3), downsample_launches=ds_n,
                                          download=round(T.t.get("download", 0.0), 2),
                                          compress_write=round(T.t.get("compress_write", 0.0), 2))))
            print(f"block_scale {scale}: {wall:.2f} s", flush=True)
        ctx.close()
        print(json.dumps(dict(card=card, size_xyz=list(size), block_size=list(BLOCK), downsampling=STEPS,
                              input_setup_s=round(t_make, 2), s0_GB=round(s0_bytes / 1e9, 3), runs=runs)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
