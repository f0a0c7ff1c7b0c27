"""CPU restatement of the per-view steps `detect-interestpoints` runs around the DoG
(src/main/java/net/preibisch/bigstitcher/spark/SparkInterestPointDetection.java:532-609, openAndDownsample :991-1111,
detection/LazyBackgroundSubtract.java:74-140).

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.  Recalled choices (ImageJ's kernel shape, the
LazyDownsample2x arithmetic, the NLinear sampling) are named here and listed in PARITY_GAPS.md.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.ndimage import median_filter

from oracle import dog_oracle


def imagej_footprint(radius: int) -> np.ndarray:
    """RankFilters.makeLineRadii for an integer radius: r2 = r*r + 1, kRadius = floor(sqrt(r2 + 1e-10)), row dy spans
    |dx| <= floor(sqrt(r2 - dy^2 + 1e-10)).  Boolean [2k+1, 2k+1] footprint (an odd number of points)."""
    r2 = int(radius) * int(radius) + 1
    k = int(math.sqrt(r2 + 1e-10))
    fp = np.zeros((2 * k + 1, 2 * k + 1), dtype=bool)
    for dy in range(-k, k + 1):
        h = int(math.sqrt(r2 - dy * dy + 1e-10))
        fp[dy + k, k - h:k + h + 1] = True
    return fp


def median_divide(vol: np.ndarray, radius: int) -> np.ndarray:
    """LazyBackgroundSubtract: per z-slice, the median m of the ImageJ footprint over the mirror-double extension
    (scipy mode 'reflect': d c b a | a b c d), then v / m where m > 0, else 0 -- all float32.  vol: [z, y, x]."""
    fp = imagej_footprint(radius)
    v = vol.astype(np.float32)
    out = np.zeros_like(v)
    for z in range(v.shape[0]):
        m = median_filter(v[z], footprint=fp, mode="reflect")
        np.divide(v[z], m, out=out[z], where=m > 0)
    return out


def downsample_float(vol: np.ndarray, factors_xyz) -> np.ndarray:
    """LazyDownsample2x chain to float32: every x halving, then every y, then every z; a step is
    out[i] = 0.5f * (in[2i] + in[2i+1]) with floor(d / 2) output elements."""
    a = vol.astype(np.float32)
    half = np.float32(0.5)
    for axis_xyz, f in enumerate(factors_xyz):
        ax = 2 - axis_xyz
        while f > 1:
            n = a.shape[ax] // 2
            lo = np.take(a, np.arange(0, 2 * n, 2), axis=ax)
            hi = np.take(a, np.arange(1, 2 * n, 2), axis=ax)
            a = (half * (lo + hi)).astype(np.float32)
            f //= 2
    return a


def sample_nlinear(vol: np.ndarray, loc_xyz) -> np.ndarray:
    """n-linear interpolation in float64 on the border extension of vol [z, y, x] at (n, 3) points {x, y, z}."""
    v = vol.astype(np.float64)
    loc = np.asarray(loc_xyz, dtype=np.float64).reshape(-1, 3)
    dims = v.shape[::-1]
    out = np.zeros(len(loc))
    for i, p in enumerate(loc):
        b = np.floor(p)
        t = p - b
        acc = 0.0
        for code in range(8):
            w = 1.0
            idx = []
            for d in range(3):
                bit = (code >> d) & 1
                w *= t[d] if bit else 1.0 - t[d]
                idx.append(int(min(max(b[d] + bit, 0), dims[d] - 1)))
            acc += w * v[idx[2], idx[1], idx[0]]
        out[i] = acc
    return out


def level_transform(mipmap_transform, remaining_xyz) -> np.ndarray:
    """mipmapTransform[level] o scale(remaining downsampling), no extra shift (J/SparkInterestPointDetection.java:
    1067-1081): downsampled pixel -> full-resolution view pixel, 3x4."""
    M = np.vstack([np.asarray(mipmap_transform, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
    S = np.diag([float(v) for v in remaining_xyz] + [1.0])
    return (M @ S)[:3]


def detect_interestpoints_reference(level_vol, remaining_xyz, mipmap_transform, sigma, threshold, min_intensity,
                                    max_intensity, find_max=True, find_min=False, localization=True, median_radius=None,
                                    max_spots=0):
    """The whole per-view pipeline on one mipmap level volume [z, y, x]: float downsampling, optional median division,
    DoG over every voxel but the outermost layer, intensities from the pre-median image, the brightest ``max_spots``
    (stable sort, descending), and the transform to full-resolution pixels.
    Returns dict(loc (n, 3) full-resolution, voxel (n, 3) downsampled, intensities float32 (n,) in float64 rounded to
    float32, downsampled (n, 3) locations)."""
    img = downsample_float(level_vol, remaining_xyz)
    det = median_divide(img, median_radius) if median_radius else img
    dims = img.shape[::-1]
    if min(dims) < 3:
        pts = []
    else:
        pts = dog_oracle.detect(det, (1, 1, 1), tuple(d - 2 for d in dims), sigma, threshold, min_intensity,
                                max_intensity, find_max, find_min, localization)
    loc = np.array([p[0] for p in pts], dtype=np.float64).reshape(-1, 3)
    vox = np.array([p[2] for p in pts], dtype=np.int64).reshape(-1, 3)
    inten = sample_nlinear(img, loc).astype(np.float32)
    if max_spots and max_spots > 0:
        if len(loc) > max_spots:
            order = sorted(range(len(loc)), key=lambda i: -float(inten[i]))[:max_spots]
            loc, vox, inten = loc[order], vox[order], inten[order]
    T = level_transform(mipmap_transform, remaining_xyz)
    full = loc @ T[:, :3].T + T[:, 3]
    return dict(loc=full, voxel=vox, intensities=inten, downsampled=loc)
