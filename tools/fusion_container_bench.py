"""affine-fusion into a plain N5 container and into a BDV/N5 project (`create-fusion-container --bdv -xo`): the same
seeded dataset (default 4 uint16 views of 512 x 512 x 128 in a row, 10 % overlap), the same uint16 AVG_BLEND fusion and
two-level pyramid, raw blocks so that the time is the device and the file system, not a codec.  The two layouts run
alternately, --repeats times each, after one warm-up fusion; the output checks that both hold the same voxels.  Prints
the card, its power limit and the command-level seconds of every run as one JSON line.

    python tools/fusion_container_bench.py [--views 4] [--size 512,512,128] [--repeats 3] [--workdir /tmp]

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
from bsgpu import commands, n5 as bn5, spimdata, viewsource  # noqa: E402


def make_input(root, views, size):
    """Seeded uint16 views: a coarse random field upsampled 8x plus Gaussian noise, one field shifted along x so that
    neighbouring views share their overlap."""
    rng = np.random.default_rng(7)
    sx, sy, sz = size
    step = int(sx * 0.9)
    width = step * (views - 1) + sx
    coarse = rng.uniform(500, 3000, (sz // 8 + 1, sy // 8 + 1, width // 8 + 1)).astype(np.float32)
    field = np.repeat(np.repeat(np.repeat(coarse, 8, 0), 8, 1), 8, 2)[:sz, :sy, :width]
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    for s in range(views):
        vol = field[:, :, s * step:s * step + sx] + rng.standard_normal((sz, sy, sx), dtype=np.float32) * 40.0
        bn5.write_bdv_setup(store, s, 0, np.clip(vol, 0, 60000).astype(np.uint16), (128, 128, 64))
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(s * step, 0, 0)))
    return spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--size", default="512,512,128")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workdir", default=tempfile.gettempdir())
    a = ap.parse_args()
    size = tuple(int(v) for v in a.size.split(","))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    root = tempfile.mkdtemp(prefix="fusion_container_bench_", dir=a.workdir)
    try:
        xml = make_input(root, a.views, size)
        kw = dict(storage="N5", block_size=(128, 128, 64), dtype="uint16", min_intensity=0.0, max_intensity=4000.0,
                  downsamplings=[(2, 2, 1), (2, 2, 2)], compression="raw")
        ctx = bsgpu.Context(0)
        outs = {}

        def run(name, i):
            out, xo = os.path.join(root, f"{name}{i}.n5"), os.path.join(root, f"{name}{i}.xml")
            commands.create_fusion_container(xml, out, bdv=name == "bdv", xml_out=xo if name == "bdv" else None, **kw)
            t0 = time.perf_counter()
            commands.affine_fusion(out, ctx, "AVG_BLEND")
            ctx.synchronize()
            dt = time.perf_counter() - t0
            outs[name] = (out, xo)
            return dt

        run("plain", "_warmup")
        times = {"plain": [], "bdv": []}
        for i in range(a.repeats):
            for name in ("plain", "bdv"):
                times[name].append(round(run(name, i), 3))
        ctx.close()
        plain = bn5.N5Store(outs["plain"][0])
        src = viewsource.open_views(spimdata.SpimData2.load(outs["bdv"][1]))
        same = all(np.array_equal(plain.read_volume(f"ch0tp0/s{l}"), src.read_volume((0, 0), l)) for l in range(3))
        dims = bn5.read_fusion_container(outs["plain"][0])[1]["mr_infos"][0][0]["dimensions"]
        print(json.dumps(dict(card=card, views=a.views, size_xyz=list(size), fused_xyz=dims, repeats=a.repeats,
                              plain_n5_s=times["plain"], bdv_n5_s=times["bdv"], identical_voxels=same)))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
