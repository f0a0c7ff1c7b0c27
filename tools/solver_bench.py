"""Solver relaxation on the device (bs_solve_tiles) at two problem shapes, with the float64 oracle as a CPU arm.

  stitching: a 16 x 16 x 4 tile grid (1024 tiles, 2688 links x 8 box corners), TRANSLATION; ONE_ROUND_SIMPLE, and
             ONE_ROUND_ITERATIVE with one inconsistent link planted (two rounds)
  ip:        128 views on an 8 x 8 x 2 grid, ~1 M correspondences over 288 links, AFFINE regularized by RIGID (0.1)

Per workload: wall ms of the call, kernel ms of the persistent solve ("solve" profile tag), iterations, us per iteration,
the bytes one iteration must read (the distance pass: p, q and w of every match, 56 B per match) and the achieved rate
against the H100's 3.35 TB/s.  The CPU arm is the oracle's time per iteration over a few iterations of the same
problem.  The card's name and power limit are read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bsgpu  # noqa: E402
from bsgpu import matching as bm, solver as bsv  # noqa: E402
from oracle import solver_oracle as so  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def grid_problem(dims, spacing, matches_per_link, noise, seed, affine=False, bogus=False):
    rng = np.random.default_rng(seed)
    idx = {}
    for z in range(dims[2]):
        for y in range(dims[1]):
            for x in range(dims[0]):
                idx[(x, y, z)] = len(idx)
    pos = np.array([[spacing[0] * x, spacing[1] * y, spacing[2] * z] for (x, y, z) in idx]) + 1e4
    links = [(idx[k], idx[(k[0] + dx, k[1] + dy, k[2] + dz)]) for k in idx for dx, dy, dz in ((1, 0, 0), (0, 1, 0), (0, 0, 1))
             if (k[0] + dx, k[1] + dy, k[2] + dz) in idx]
    n = len(pos)
    shift = rng.normal(0, 2.0, (n, 3))
    lin = np.tile(np.eye(3), (n, 1, 1)) + (0.002 * rng.normal(size=(n, 3, 3)) if affine else 0.0)
    ta, tb, p, q = [], [], [], []
    for a, b in links:
        m = matches_per_link() if callable(matches_per_link) else matches_per_link
        c = (pos[a] + pos[b]) / 2 + rng.uniform(-0.4, 0.4, (m, 3)) * spacing
        for t, lst in ((a, p), (b, q)):
            Li = np.linalg.inv(lin[t])
            lst.append((c - pos[t] - shift[t]) @ Li.T + pos[t] + rng.normal(0, noise, (m, 3)))
        ta.append(np.full(m, a))
        tb.append(np.full(m, b))
    if bogus:
        m = 8
        c = (pos[0] + pos[n - 1]) / 2 + rng.uniform(-0.4, 0.4, (m, 3)) * spacing
        ta.append(np.full(m, 0))
        tb.append(np.full(m, n - 1))
        p.append(c)
        q.append(c + (150.0, -170.0, 90.0))
    prob = bsv.build_problem(n, *(np.concatenate(x) for x in (ta, tb, p, q)), np.ones(sum(len(x) for x in ta)))
    prob.fixed = np.zeros(n, np.int32)
    prob.fixed[0] = 1
    return prob


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in out.split(",")]
        return name, plim
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def run(ctx, label, prob, model, method, cpu_iters):
    ctx.profile_enable(True)
    ctx.profile_reset()
    t0 = time.perf_counter()
    M, removed, st = bsv.solve(ctx, prob, model, method, max_error=5.0, max_iterations=10000, max_plateau_width=200)
    wall = (time.perf_counter() - t0) * 1e3
    ms, launches = ctx.profile_get("solve")
    ctx.profile_enable(False)
    n_matches = len(prob.w)
    iters = st["iterations"]
    # the last round's kernel carries `iters` iterations; earlier rounds are in the same tag
    per_iter_us = ms * 1e3 / max(1, iters) if launches == 1 else float("nan")
    bytes_iter = 56 * n_matches
    row = dict(workload=label, method=method, tiles=prob.n_tiles, links=len(prob.links), matches=n_matches, rounds=st["rounds"],
               removed=len(removed), iterations=iters, wall_ms=round(wall, 2), kernel_ms=round(ms, 3), kernel_launches=launches,
               blocks=st["blocks"], models_in_shared=st["models_in_shared"], skipped_fits=st["skipped_fits"])
    if launches == 1:
        row.update(us_per_iteration=round(per_iter_us, 3), bytes_per_iteration=bytes_iter,
                   achieved_GBps=round(bytes_iter / (per_iter_us * 1e-6) / 1e9, 1),
                   fraction_of_hbm=round(bytes_iter / (per_iter_us * 1e-6) / HBM_BYTES_PER_S, 4))
    if cpu_iters:
        _, off, order = bsv.colouring(prob.n_tiles, prob.links)
        M0 = bsv.prealign(prob, model)
        t0 = time.perf_counter()
        so.solve_tiles(off, order, prob.fixed, prob.links, prob.match_offsets, prob.p, prob.q, prob.w, M0,
                       transformation=model.tm, regularization=model.rm, lam=model.lam, max_iterations=cpu_iters,
                       max_plateau_width=10 ** 6)
        row["cpu_oracle_us_per_iteration"] = round((time.perf_counter() - t0) * 1e6 / cpu_iters, 1)
        row["cpu_oracle_iterations_timed"] = cpu_iters
    return row


def main():
    name, plim = card()
    print(json.dumps(dict(card=name, power_limit=plim)))
    with bsgpu.Context(0) as ctx:
        warm = grid_problem((3, 3, 1), (100.0, 100.0, 60.0), 8, 0.3, 1)
        bsv.solve(ctx, warm, bm.Model("TRANSLATION", "NONE"), max_plateau_width=10)
        st = grid_problem((16, 16, 4), (400.0, 400.0, 200.0), 8, 0.3, 2)
        st_bogus = grid_problem((16, 16, 4), (400.0, 400.0, 200.0), 8, 0.3, 2, bogus=True)
        rng = np.random.default_rng(3)
        ip = grid_problem((8, 8, 2), (400.0, 400.0, 200.0), lambda: int(rng.integers(3000, 4000)), 0.5, 4, affine=True)
        rows = [run(ctx, "stitching", st, bm.Model("TRANSLATION", "NONE"), "ONE_ROUND_SIMPLE", 3),
                run(ctx, "stitching", st_bogus, bm.Model("TRANSLATION", "NONE"), "ONE_ROUND_ITERATIVE", 0),
                run(ctx, "ip", ip, bm.Model("AFFINE", "RIGID", 0.1), "ONE_ROUND_SIMPLE", 3)]
    for r in rows:
        r.update(card=name, power_limit=plim)
        print(json.dumps(r))


if __name__ == "__main__":
    main()
