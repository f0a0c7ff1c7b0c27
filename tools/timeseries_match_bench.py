"""Measure `match-interestpoints -rtp ALL_TO_ALL_WITH_RANGE` (PRECISE_TRANSLATION, defaults n = 3, r = 1, 10 000
RANSAC iterations) on a seeded time-lapse: T timepoints x V views in a row (30 % overlap in x), one cloud of beads that
drifts by a few px and under a degree about z from timepoint to timepoint, the same nominal registrations at every
timepoint (generated here, written to a temporary directory).

Prints one JSON line: the task count (same-time and cross-time), the device time and launch count of the profile tags
"knn" and "desc_match", the host RANSAC time (every `matching.ransac` call of the command, timed around the call), the
end-to-end command seconds, the correspondences written, and the card name and power limit read in the same run.  The
command runs once, with the kernel profile on; the host RANSAC dominates it, so the profile's events do not matter.

    python tools/timeseries_match_bench.py [--timepoints 4] [--views 2] [--range 1] [--beads 2000] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def write_scene(root, timepoints, views, beads_per_view, seed=1, tile=(600.0, 600.0, 150.0), overlap=0.3):
    """Beads uniform in the row of views (about ``beads_per_view`` per view), moved at every timepoint by a rigid drift
    (up to 3 px per axis, up to 0.5 degrees about z), each view's beads + 0.3 px of noise written to interestpoints.n5;
    the XML holds the grid translations at every timepoint.  Returns the XML path."""
    from bsgpu import n5 as bn5, spimdata
    from tests.test_match_cpu import compose, rot_z, write_points
    from tests.test_timeseries_cpu import repeat_timepoint
    rng = np.random.default_rng(seed)
    step = tile[0] * (1 - overlap)
    extent = np.array([step * (views - 1) + tile[0], tile[1], tile[2]])
    n = int(round(beads_per_view * extent[0] / tile[0]))
    beads = rng.uniform(0, 1, (n, 3)) * extent
    store = bn5.N5Store(os.path.join(root, "interestpoints.n5"), create=True)
    for t in range(timepoints):
        D = compose(np.hstack([np.eye(3), rng.uniform(-3, 3, (3, 1))]), rot_z(rng.uniform(-0.5, 0.5), extent / 2))
        moved = beads @ D[:, :3].T + D[:, 3]
        for s in range(views):
            loc = moved - (s * step, 0.0, 0.0)
            loc = loc[np.all((loc >= 0) & (loc <= np.array(tile) - 1), axis=1)]
            write_points(store, (t, s), "beads", loc + rng.normal(0, 0.3, loc.shape))
    xml = os.path.join(root, "dataset.xml")
    size = tuple(int(v) for v in tile)
    spimdata.write_dataset_xml(xml, "dataset.n5", [dict(setup=s, size_xyz=size, tile=s, translation_xyz=(s * step, 0, 0))
                                                   for s in range(views)])
    repeat_timepoint(xml, timepoints)
    return xml


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timepoints", type=int, default=4)
    ap.add_argument("--views", type=int, default=2)
    ap.add_argument("--range", type=int, default=1)
    ap.add_argument("--beads", type=int, default=2000, help="beads per view")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bsgpu
    from bsgpu import commands, matching as bm
    from match_bench import card

    out = dict(card=card(), timepoints=args.timepoints, views=args.views, range_tp=args.range,
               beads_per_view=args.beads)
    ransac = bm.ransac
    spent = []

    def timed_ransac(*a, **k):
        t0 = time.perf_counter()
        try:
            return ransac(*a, **k)
        finally:
            spent.append(time.perf_counter() - t0)

    with tempfile.TemporaryDirectory() as tmp, bsgpu.Context(0) as ctx:
        xml = write_scene(tmp, args.timepoints, args.views, args.beads)
        # warm-up of the (3, 4) instantiations outside the timed run
        h = ctx.descriptors_build(np.random.default_rng(0).uniform(0, 100, (2000, 3)))
        ctx.descriptors_match(h, h)
        ctx.descriptors_free(h)
        ctx.profile_enable(True)
        ctx.profile_reset()
        bm.ransac = timed_ransac
        try:
            t0 = time.perf_counter()
            res = commands.match_interestpoints(xml, ctx, ["beads"], "PRECISE_TRANSLATION",
                                                registration_tp="ALL_TO_ALL_WITH_RANGE", range_tp=args.range)
            out["command_s"] = time.perf_counter() - t0
        finally:
            bm.ransac = ransac
        for tag in ("knn", "desc_match"):
            ms, n = ctx.profile_get(tag)
            out[f"{tag}_ms"], out[f"{tag}_launches"] = ms, n
        ctx.profile_enable(False)
    out["tasks"] = len(res)
    out["cross_time_tasks"] = sum(a[0] != b[0] for a, _, b, _ in res)
    out["ransac_calls"], out["ransac_s"] = len(spent), float(sum(spent))
    out["ransac_share_of_command"] = out["ransac_s"] / out["command_s"]
    out["correspondences"] = int(sum(len(v) for v in res.values()))
    out["cross_time_correspondences"] = int(sum(len(v) for (a, _, b, _), v in res.items() if a[0] != b[0]))
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
