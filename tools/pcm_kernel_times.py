"""Device time per phase-correlation pair of every profiled kernel tag at the benchmark's shape (512^3 uint16 crops,
padded to 540^3), with bench.py's parameters: CUDA events around each launch (bs_launch_scope), averaged over
--reps profiled batches of --pairs pairs after one warm-up batch.  Prints one JSON line per setting:
{"tags": {tag: ms per pair}, "sum_ms": ..., "env": {BS_FFT_* settings}}.  The dispatch switches are read at each
launch, so --sweep VAR=a,b,... measures every value of VAR in turn on the same workload (e.g.
--sweep BS_FFT_XY_FUSE=0,1 compares the kernels each chain launches)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import bsgpu  # noqa: E402
from bsgpu import synthetic  # noqa: E402

TAGS = ("fft_x_r2c", "fft_y", "fft_xy", "fft_z_xpower", "fft_y_inv", "fft_x_c2r", "peaks", "select", "pearson")

ap = argparse.ArgumentParser(description=__doc__)
ap.add_argument("--pairs", type=int, default=16)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--sweep", default=None, help="VAR=a,b,...: one measurement per value of the environment variable")
args = ap.parse_args()
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
    for _ in range(args.reps):
        ctx.pcm_batch(imgs1, imgs2, params, dims, bsgpu.native.DTYPE_U16)
    ctx.profile_enable(False)
    npairs = args.pairs * args.reps
    tags = {}
    for tag in TAGS:
        ms, cnt = ctx.profile_get(tag)
        if cnt:
            tags[tag] = round(ms / npairs, 4)
    env = {k: v for k, v in sorted(os.environ.items()) if k.startswith("BS_FFT_")}
    print(json.dumps({"tags": tags, "sum_ms": round(sum(tags.values()), 4), "env": env}), flush=True)
ctx.close()
