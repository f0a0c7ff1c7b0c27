"""Measure `match-interestpoints` (PRECISE_TRANSLATION, defaults n = 3, r = 1) on two seeded views of 50 000 beads
each that overlap by 30 % (generated here, written to a temporary directory).

Prints one JSON line: the device time and launch count of the profile tags "knn" and "desc_match" with the FP64 rate
of the descriptor search against the 34 TFLOP/s data-sheet figure (operations counted by desc_match_flops), the host
RANSAC time, the end-to-end command seconds, the card name and power limit read in the same run, and, labelled as a
CPU figure, the float64 oracle's search on 2 000 points.

    python tools/match_bench.py [--beads 50000] [--out result.json]
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

FP64_PEAK = 34e12          # H100 SXM data sheet, FP64 (non-tensor)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return q


def desc_match_flops(na, nb, n=3, k=4):
    """FP64 operations of the exhaustive search: per (a, b) k^2 squared distances (3 sub + 3 mul + 2 add), then per
    subset pair n - 1 adds and one compare; C(k, n)^2 subset pairs."""
    from math import comb
    return float(na) * nb * (8 * k * k + comb(k, n) ** 2 * n)


def make_views(n_beads, seed=1):
    """Two views (world = view A's frame): B sees the beads with x in the last 30 % of A's range, shifted."""
    rng = np.random.default_rng(seed)
    size = np.array([2000.0, 2000.0, 400.0])
    a = rng.uniform(0, 1, (n_beads, 3)) * size
    shift = np.array([0.7 * size[0], 0.0, 0.0])
    keep = a[:, 0] >= shift[0]
    b = np.vstack([a[keep] - shift + rng.normal(0, 0.3, (int(keep.sum()), 3)),
                   rng.uniform(0, 1, (n_beads - int(keep.sum()), 3)) * size])
    return a, b, shift, size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beads", type=int, default=50000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bsgpu
    from bsgpu import commands, matching as bm, n5 as bn5, spimdata
    from oracle import match_oracle as mo
    from tests.test_match_cpu import write_points

    a, b, shift, size = make_views(args.beads)
    out = dict(card=card(), beads_per_view=args.beads)
    with bsgpu.Context(0) as ctx:
        # warm-up of both instantiations, then the timed kernels
        h = ctx.descriptors_build(a[:2000])
        ctx.descriptors_match(h, h)
        ctx.descriptors_free(h)
        ctx.profile_enable(True)
        ctx.profile_reset()
        ha, hb = ctx.descriptors_build(a), ctx.descriptors_build(b)
        t0 = time.perf_counter()
        best_b, best, second = ctx.descriptors_match(ha, hb)
        out["desc_match_wall_s"] = time.perf_counter() - t0
        ctx.descriptors_free(ha)
        ctx.descriptors_free(hb)
        for tag in ("knn", "desc_match"):
            ms, n = ctx.profile_get(tag)
            out[f"{tag}_ms"], out[f"{tag}_launches"] = ms, n
        ctx.profile_enable(False)
        fl = desc_match_flops(len(a), len(b))
        out["desc_match_fp64_tflops"] = fl / (out["desc_match_ms"] * 1e-3) / 1e12
        out["desc_match_share_of_34_tflops"] = out["desc_match_fp64_tflops"] * 1e12 / FP64_PEAK
        cand = bm.ratio_test(best_b, best, second, 3.0)
        t0 = time.perf_counter()
        inl, _ = bm.ransac(a[cand], b[best_b[cand]] + shift, bm.Model())
        out["ransac_ms"], out["candidates"], out["inliers"] = (time.perf_counter() - t0) * 1e3, len(cand), len(inl)

        with tempfile.TemporaryDirectory() as tmp:
            dims = tuple(int(v) for v in size)
            spimdata.write_dataset_xml(os.path.join(tmp, "dataset.xml"), "dataset.n5", [
                dict(setup=0, size_xyz=dims, tile=0, translation_xyz=(0, 0, 0)),
                dict(setup=1, size_xyz=dims, tile=1, translation_xyz=tuple(shift))])
            store = bn5.N5Store(os.path.join(tmp, "interestpoints.n5"), create=True)
            write_points(store, (0, 0), "beads", a)
            write_points(store, (0, 1), "beads", b)
            t0 = time.perf_counter()
            res = commands.match_interestpoints(os.path.join(tmp, "dataset.xml"), ctx, ["beads"], "PRECISE_TRANSLATION")
            out["command_s"] = time.perf_counter() - t0
            out["command_correspondences"] = int(sum(len(v) for v in res.values()))

    n_cpu = 2000
    t0 = time.perf_counter()
    mo.match(a[:n_cpu], b[:n_cpu])
    cpu_s = time.perf_counter() - t0
    out["cpu_oracle_2000_s"] = cpu_s
    out["cpu_oracle_pairs_per_s"] = n_cpu * n_cpu / cpu_s
    out["gpu_pairs_per_s"] = len(a) * len(b) / (out["desc_match_ms"] * 1e-3)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
