"""What split-images costs affine-fusion: a seeded 2-tile 2048 x 2048 x 256 uint16 BDV-N5 dataset (tiles 1792 px apart
in x, raw 128^3 blocks) fused with AVG_BLEND into a uint16 N5 container, once as it is and once split to 512,512,256
with 32 px overlap (50 sub-views read through the split loader).  Sub-views re-read their overlaps and the blocks
around every cut, so the split run reads more.  Prints one JSON line: the card and its power limit, and per run the
end-to-end seconds of affine_fusion, the bytes of decoded N5 blocks it read, and the device time of the fusion kernels
(profile tag `fuse`).

    python tools/split_bench.py [--size 2048,2048,256] [--fusion AVG_BLEND] [--workdir /tmp]

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

BLOCK = (128, 128, 128)


def make_input(root, size, stride):
    """Two seeded uint16 tiles of ``size``: a coarse random field upsampled 16x plus noise, one 128-plane slab per
    block row, offset per slab; tile 1 sits ``stride`` px to the right of tile 0."""
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    sx, sy, sz = size
    tiles = []
    for s in range(2):
        rng = np.random.default_rng(200 + s)
        coarse = rng.uniform(500, 3000, (8, sy // 16 + 1, sx // 16 + 1)).astype(np.float32)
        base = np.repeat(np.repeat(np.repeat(coarse, 16, 0), 16, 1), 16, 2)[:BLOCK[2], :sy, :sx]
        base += rng.standard_normal(base.shape, dtype=np.float32) * 40.0
        base = np.clip(base, 0, 60000).astype(np.uint16)
        bn5.set_bdv_attributes(store, s, 0, [(1, 1, 1)], np.uint16)
        ds = bn5.bdv_dataset(s, 0, 0)
        store.create_dataset(ds, size, BLOCK, np.uint16, "raw")
        for z0 in range(0, sz, BLOCK[2]):
            store.save_block(ds, base[:min(BLOCK[2], sz - z0)] + np.uint16(z0 // BLOCK[2]), (0, 0, z0 // BLOCK[2]))
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(stride * s, 0, 0)))
    return spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="2048,2048,256")
    ap.add_argument("--fusion", default="AVG_BLEND")
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    size = tuple(int(v) for v in a.size.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    tmp = tempfile.mkdtemp(prefix="split_bench_", dir=a.workdir)
    try:
        t0 = time.perf_counter()
        xml = make_input(tmp, size, size[0] - 256)
        split = os.path.join(tmp, "split.xml")
        plan = commands.split_images(xml, (512, 512, 256), (32, 32, 32), xml_out=split)
        t_make = time.perf_counter() - t0
        print(f"input ready in {t_make:.1f} s", flush=True)
        ctx = bsgpu.Context(0)
        read = [0]
        orig = bn5.N5Store.read_block

        def counted(self, path, grid_pos):
            b = orig(self, path, grid_pos)
            if b is not None and "dataset.n5" in self.root:
                read[0] += b.nbytes
            return b
        bn5.N5Store.read_block = counted
        runs = []
        # the first pass warms module loads and kernel shapes; the second is reported
        for rep in range(2):
            for name, x in (("unsplit", xml), ("split", split)):
                out = os.path.join(tmp, f"{name}.n5")
                shutil.rmtree(out, ignore_errors=True)
                commands.create_fusion_container(x, out, block_size=BLOCK, dtype="uint16", min_intensity=0.0,
                                                 max_intensity=65535.0, compression="raw")
                read[0] = 0
                ctx.profile_enable(True)
                ctx.profile_reset()
                t0 = time.perf_counter()
                commands.affine_fusion(out, ctx, a.fusion)
                ctx.synchronize()
                wall = time.perf_counter() - t0
                fuse_ms, fuse_n = ctx.profile_get("fuse")
                ctx.profile_enable(False)
                if rep:
                    runs.append(dict(project=name, views=2 if name == "unsplit" else len(plan["views"]),
                                     wall_s=round(wall, 2), read_GB=round(read[0] / 1e9, 3),
                                     fuse_kernel_s=round(fuse_ms / 1e3, 3), fuse_launches=fuse_n))
                print(f"{name} (pass {rep}): {wall:.2f} s, {read[0] / 1e9:.2f} GB read", flush=True)
        ctx.close()
        u, s = runs
        print(json.dumps(dict(card=card, size_xyz=list(size), fusion=a.fusion, split_size=list(plan["size"]),
                              split_overlap=list(plan["overlap"]), input_setup_s=round(t_make, 2), runs=runs,
                              read_ratio=round(s["read_GB"] / u["read_GB"], 3),
                              wall_ratio=round(s["wall_s"] / u["wall_s"], 3))))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
