"""estimate-bounding-box (mvrecon BoundingBoxMinFilterThreshold, recalled; PARITY_GAPS B2-B5) in numpy / scipy, float64
where it matters: the downsampled grid, the threshold, the box minimum filter and the mapping of the kept voxels back
to world coordinates.  Also a brute-force box minimum for the tests."""
import math

import numpy as np
from scipy import ndimage


def grid(lo, hi, ds):
    """B2: (g_min, dims) of the downsampled grid over the world box [lo, hi]; voxel i is world point ds (g_min + i)."""
    g_min = np.array([math.floor(int(v) / ds) for v in lo], dtype=np.int64)
    g_max = np.array([math.ceil(int(v) / ds) for v in hi], dtype=np.int64)
    return g_min, g_max - g_min + 1


def threshold(mn, mx, background):
    """B3: t = mn + (mx - mn) background / 100 in float64."""
    return float(mn) + (float(mx) - float(mn)) * float(background) / 100.0


def radius(size, ds):
    """B4: max(1, floor(size / ds + 0.5))."""
    return max(1, int(math.floor(size / ds + 0.5)))


def min_filter(vol, r):
    """B4: minimum over the box |q - p|_inf <= r per axis (r int or (rx, ry, rz)), clipped to the volume, NaN ignored
    (fmin).  scipy's minimum_filter with `nearest` extension gives the clipped box minimum; NaNs are replaced by +inf
    first and restored where the whole box was NaN."""
    rx, ry, rz = (r, r, r) if np.isscalar(r) else r
    v = np.asarray(vol, dtype=np.float32)
    nan = np.isnan(v)
    size = (2 * rz + 1, 2 * ry + 1, 2 * rx + 1)
    out = ndimage.minimum_filter(np.where(nan, np.float32(np.inf), v), size=size, mode="nearest")
    if nan.any():
        all_nan = ndimage.minimum_filter(nan.astype(np.uint8), size=size, mode="nearest").astype(bool)
        out[all_nan] = np.nan
    return out


def brute_min_filter(vol, r):
    """The box minimum voxel by voxel (np.fmin over the clipped box): the definition min_filter is checked against."""
    rx, ry, rz = (r, r, r) if np.isscalar(r) else r
    v = np.asarray(vol, dtype=np.float32)
    nz, ny, nx = v.shape
    out = np.empty_like(v)
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                box = v[max(z - rz, 0):z + rz + 1, max(y - ry, 0):y + ry + 1, max(x - rx, 0):x + rx + 1]
                out[z, y, x] = np.fmin.reduce(box, axis=None)
    return out


def threshold_bbox(vol, t):
    """(min_xyz, max_xyz, count) of the voxels > t compared in float64; (-1,) * 3 twice and 0 when there are none."""
    keep = np.asarray(vol, dtype=np.float64) > float(t)
    n = int(keep.sum())
    if n == 0:
        return (-1, -1, -1), (-1, -1, -1), 0
    idx = np.argwhere(keep)                     # [z, y, x]
    return tuple(int(v) for v in idx.min(axis=0)[::-1]), tuple(int(v) for v in idx.max(axis=0)[::-1]), n


def world_box(i_min, i_max, g_min, ds, lo, hi):
    """B5: world min ds (g_min + i_min - 1), max ds (g_min + i_max + 1) (one downsampled voxel of margin on each side),
    intersected with [lo, hi]."""
    g = np.asarray(g_min, dtype=np.int64)
    wmin = ds * (g + np.asarray(i_min, dtype=np.int64) - 1)
    wmax = ds * (g + np.asarray(i_max, dtype=np.int64) + 1)
    return np.maximum(wmin, np.asarray(lo, dtype=np.int64)), np.minimum(wmax, np.asarray(hi, dtype=np.int64))


def estimate(fused, lo, hi, ds, background=5.0, size=25):
    """B3-B5 on a fused downsampled volume [z, y, x] over the grid of (lo, hi, ds).  Returns dict(min, max, threshold,
    min_max, radius, count), min / max None when no voxel passes."""
    g_min, dims = grid(lo, hi, ds)
    assert tuple(fused.shape[::-1]) == tuple(int(v) for v in dims)
    v = np.asarray(fused, dtype=np.float32)
    mn, mx = float(np.nanmin(v)), float(np.nanmax(v))
    t = threshold(mn, mx, background)
    r = radius(size, ds)
    i_min, i_max, n = threshold_bbox(min_filter(v, r), t)
    out = dict(threshold=t, min_max=(mn, mx), radius=r, count=n, min=None, max=None)
    if n:
        wmin, wmax = world_box(i_min, i_max, g_min, ds, lo, hi)
        out.update(min=[int(x) for x in wmin], max=[int(x) for x in wmax])
    return out
