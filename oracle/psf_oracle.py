"""CPU restatement of `extract-psfs` (mvrecon PSFExtraction, recalled): the bead average around interest points.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.

Every sample is the n-linear interpolation of ``ip_oracle.sample_nlinear`` (border extension, corners in the same
order, x toggling fastest, the same double weights), with the float32 roundings PARITY_GAPS #37 pins: each corner term
is (float)(v w) and the eight terms are summed in float.  ``ip_oracle.sample_nlinear`` sums in float64 instead, so it
is the bound check (tests/test_psf_cpu.py), and this module spells the float steps so that the device sums can be
compared bit for bit.  The PSF voxel sum is accumulated in float64, point by point in the order given, exactly as
``bs_psf_accumulate`` does.
"""
from __future__ import annotations

import numpy as np

POINTS_PER_CHUNK = 64


def offsets(psf_size_xyz) -> np.ndarray:
    """(sz * sy * sx, 3) float64 {x, y, z} offsets in [-h, h], x fastest (the PSF voxel order)."""
    sx, sy, sz = (int(v) for v in psf_size_xyz)
    z, y, x = np.mgrid[0:sz, 0:sy, 0:sx]
    return np.stack([x.ravel() - (sx - 1) // 2, y.ravel() - (sy - 1) // 2, z.ravel() - (sz - 1) // 2], 1).astype(np.float64)


def sample(vol: np.ndarray, loc_xyz) -> np.ndarray:
    """float32 n-linear samples (PARITY_GAPS #37) of vol [z, y, x] at (..., 3) points {x, y, z}, border extension."""
    loc = np.asarray(loc_xyz, dtype=np.float64)
    b = np.floor(loc)
    t = loc - b
    b = b.astype(np.int64)
    dims = vol.shape[::-1]
    acc = np.zeros(loc.shape[:-1], dtype=np.float32)
    for code in range(8):                                    # x toggles fastest
        w = np.ones(loc.shape[:-1])
        idx = []
        for d in range(3):
            bit = (code >> d) & 1
            w = w * (t[..., d] if bit else 1.0 - t[..., d])
            idx.append(np.clip(b[..., d] + bit, 0, dims[d] - 1))
        v = vol[idx[2], idx[1], idx[0]].astype(np.float32).astype(np.float64)
        acc = acc + (v * w).astype(np.float32)               # float32 + float32, rounded once
    return acc


def accumulate(vol: np.ndarray, points_xyz, psf_size_xyz, sum=None) -> np.ndarray:
    """``sum`` (float64 [sz, sy, sx], zeros when None) plus the samples of the PSF box around every point of the FULL
    view ``vol`` [z, y, x], added point by point in the order given."""
    s = [int(v) for v in psf_size_xyz]
    out = np.zeros(s[::-1], dtype=np.float64) if sum is None else np.array(sum, dtype=np.float64)
    flat = out.reshape(-1)
    pts = np.asarray(points_xyz, dtype=np.float64).reshape(-1, 3)
    o = offsets(s)
    for c in range(0, len(pts), POINTS_PER_CHUNK):
        p = pts[c:c + POINTS_PER_CHUNK]
        samples = sample(vol, p[:, None, :] + o[None, :, :])  # (chunk, voxels): p + o in float64, as on the device
        for row in samples:
            flat += row.astype(np.float64)
    return out


def extract(vol: np.ndarray, points_xyz, psf_size_xyz) -> np.ndarray:
    """The PSF of one view: the float64 sum over the points divided by their count, as float32 [sz, sy, sx]; not
    normalised.  At least one point."""
    pts = np.asarray(points_xyz, dtype=np.float64).reshape(-1, 3)
    return (accumulate(vol, pts, psf_size_xyz) / len(pts)).astype(np.float32)
