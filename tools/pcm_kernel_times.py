"""Device time per phase-correlation pair of every profiled kernel tag at the benchmark's shape (512^3 uint16 crops,
padded to 540^3), with bench.py's parameters: CUDA events around each launch (bs_launch_scope), averaged over
--reps profiled batches of --pairs pairs after one warm-up batch.  Prints one JSON line per setting:
{"tags": {tag: ms per pair}, "sum_ms": ..., "env": {BS_FFT_* settings}}.  The dispatch switches are read at each
launch, so --sweep VAR=a,b,... measures every value of VAR in turn on the same workload (e.g.
--sweep BS_FFT_XY_FUSE=0,1 compares the kernels each chain launches, --sweep BS_FFT_XY_KX=70,74,78 the role split of
the fused forward kernel).

--probe reads the role probe of k_fft_xy_col540, which only a library built with `make EXTRA=-DPCM_XY_PROBE` has:
after each fused launch the library prints, summed over the CTAs of each role, thread 0's time in plane hand-off
waits and the rest of its time (busy).  The setting's line then gains "roles": per role the busy and wait time per
CTA and launch in us, and its tile rate while busy (x: line pairs, y: columns, per us per SM).  The probe
synchronises after every fused launch, so take the tags' times from a build without it."""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import bsgpu  # noqa: E402
from bsgpu import synthetic  # noqa: E402

TAGS = ("fft_x_r2c", "fft_y", "fft_xy", "fft_z_xpower", "fft_y_inv", "fft_x_c2r", "peaks", "select", "pearson")

ap = argparse.ArgumentParser(description=__doc__)
ap.add_argument("--pairs", type=int, default=16)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--sweep", default=None, help="VAR=a,b,...: one measurement per value of the environment variable")
ap.add_argument("--probe", action="store_true", help="report the fused kernel's role probe (a -DPCM_XY_PROBE build)")
args = ap.parse_args()


def probe_lines(fn):
    """Run fn() with file descriptor 2 captured; return the library's probe lines as dicts."""
    with tempfile.TemporaryFile() as tmp:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read().decode()
    return [json.loads(l.split(" ", 1)[1]) for l in text.splitlines() if l.startswith("pcm_xy_probe ")]


def roles(lines):
    if not lines:
        return None
    kx, ctas = lines[0]["kx"], lines[0]["ctas"]
    tot = {k: sum(l[k] for l in lines) for k in ("x_busy_us", "x_wait_us", "y_busy_us", "y_wait_us")}
    per = {"x": (kx, "line_pairs"), "y": (ctas - kx, "y_columns")}
    out = {}
    for r, (n, unit) in per.items():
        busy, wait = tot[r + "_busy_us"], tot[r + "_wait_us"]
        out[r] = {"ctas": n, "busy_us": round(busy / n / len(lines), 1), "wait_us": round(wait / n / len(lines), 1),
                  "rate": round(sum(l[unit] for l in lines) / busy, 3) if busy else None}
    return out


if args.sweep:
    var, vals = args.sweep.split("=", 1)
    settings = [(var, v) for v in vals.split(",")]
else:
    settings = [(None, None)]

n = 512
ctx = bsgpu.Context(0)
imgs1, imgs2, _ = synthetic.make_pcm_workload(args.pairs, n=n, device=torch.device("cuda", 0), seed=42)
torch.cuda.synchronize()
params = ctx.pcm_params(peaks_to_check=5, do_subpixel=True, min_overlap_frac=0.25, extension=(10, 10, 10))
dims = [(n, n, n)] * args.pairs
for var, val in settings:
    if var:
        os.environ[var] = val
    ctx.pcm_batch(imgs1, imgs2, params, dims, bsgpu.native.DTYPE_U16)
    ctx.profile_reset()
    ctx.profile_enable(True)

    def reps():
        for _ in range(args.reps):
            ctx.pcm_batch(imgs1, imgs2, params, dims, bsgpu.native.DTYPE_U16)

    lines = probe_lines(reps) if args.probe else reps()
    ctx.profile_enable(False)
    npairs = args.pairs * args.reps
    tags = {}
    for tag in TAGS:
        ms, cnt = ctx.profile_get(tag)
        if cnt:
            tags[tag] = round(ms / npairs, 4)
    env = {k: v for k, v in sorted(os.environ.items()) if k.startswith("BS_FFT_")}
    res = {"tags": tags, "sum_ms": round(sum(tags.values()), 4), "env": env}
    if args.probe:
        res["roles"] = roles(lines)
    print(json.dumps(res), flush=True)
ctx.close()
