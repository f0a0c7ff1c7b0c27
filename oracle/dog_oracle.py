"""CPU restatement of the reference's Difference-of-Gaussian interest-point detection for one block.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg, never by the
product.  PARITY UNPINNED: the arithmetic lives in net.preibisch:multiview-reconstruction 8.0.0
(DoGImgLib2.computeDoG / computeSigmas, imglib2 Gauss3, LocalExtrema, quadratic localisation), which is not under
/root/reference; this follows the call site src/main/java/net/preibisch/bigstitcher/spark/
SparkInterestPointDetection.java:469-566 (parameters :476-503, block + 1 px halo :397-424) and the published algorithm
as recalled (every recalled constant is named below and listed in PARITY_GAPS.md).
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import correlate1d

STEPS_PER_OCTAVE = 4          # DoGImgLib2 / DifferenceOfGaussian.computeK(4): k = 2^(1/4)
IMAGE_SIGMA = 0.5             # DifferenceOfGUI.defaultImageSigma*
INITIAL_THRESHOLD_DIV = 3.0   # candidates at |DoG| >= threshold / 3, kept after localisation at |value| >= threshold


def compute_sigmas(sigma: float):
    """DoGImgLib2.computeSigmas: the two blur sigmas (relative to the image's own 0.5) and 1 / (k - 1)."""
    k = 2.0 ** (1.0 / STEPS_PER_OCTAVE)
    s1, s2 = sigma, sigma * k
    return np.sqrt(s1 * s1 - IMAGE_SIGMA ** 2), np.sqrt(s2 * s2 - IMAGE_SIGMA ** 2), 1.0 / (k - 1.0)


def gauss_kernel(sigma: float) -> np.ndarray:
    """Gauss3: truncated, normalised; half kernel SIZE max(2, int(3 sigma + 0.5) + 1) (radius = size - 1)."""
    size = max(2, int(3.0 * sigma + 0.5) + 1)
    r = size - 1
    x = np.arange(-r, r + 1, dtype=np.float64)
    k = np.exp(-0.5 * (x / sigma) ** 2)
    return (k / k.sum()).astype(np.float32)


def dog_volume(img: np.ndarray, sigma: float, min_intensity: float, max_intensity: float) -> np.ndarray:
    """(G_sa * I' - G_sb * I') / (k - 1) on the whole [z,y,x] image, I' = (I - min) / (max - min), float32,
    Views.extendMirrorDouble borders (scipy mode 'reflect': d c b a | a b c d | d c b a)."""
    sa, sb, kinv = compute_sigmas(sigma)
    f = ((img.astype(np.float32) - np.float32(min_intensity)) * np.float32(1.0 / (max_intensity - min_intensity))).astype(np.float32)
    a, b = f, f
    for axis in (2, 1, 0):          # x, y, z
        a = correlate1d(a, gauss_kernel(sa), axis=axis, mode="reflect", output=np.float32)
        b = correlate1d(b, gauss_kernel(sb), axis=axis, mode="reflect", output=np.float32)
    return ((a - b) * np.float32(kinv)).astype(np.float32)


def _load(img, min_intensity, max_intensity):
    """I' as k_dog_load forms it: (float(v) - float(min)) * float(1 / (max - min)), all float32."""
    return ((img.astype(np.float32) - np.float32(min_intensity)) * np.float32(1.0 / (max_intensity - min_intensity))).astype(np.float32)


def _correlate_valid(x, k, axis):
    """out[i] = sum_t k[t] * x[i + t] along ``axis`` in float64 (no border handling: x already carries the halo)."""
    n = x.shape[axis] - len(k) + 1
    out = np.zeros(x.shape[:axis] + (n,) + x.shape[axis + 1:])
    sl = [slice(None)] * x.ndim
    for t, kt in enumerate(np.asarray(k, dtype=np.float64)):
        sl[axis] = slice(t, t + n)
        out += kt * x[tuple(sl)]
    return out


def dog_reference(img, interval_min_xyz, interval_size_xyz, sigma, min_intensity, max_intensity,
                  drop_outer_tap_axis=None, pad_mode="symmetric"):
    """Float64 reference of the DoG box the extremum stage reads: (G_sa * I' - G_sb * I') * float(1 / (k - 1)) over
    [interval_min - 1, interval_min + interval_size + 1) per axis, [z, y, x], with I' in float32 as the device loads it
    and the float32 taps of gauss_kernel, correlated in float64 on the mirror-double extension of the image
    (np.pad mode 'symmetric' == Views.extendMirrorDouble, also where the extension exceeds the image).
    Returns (dog, G_sa * |I'|, G_sb * |I'|), all float64 of shape (size + 2)[::-1]; the last two set the error bar.
    ``drop_outer_tap_axis`` (0 = x, 1 = y, 2 = z) zeroes the outermost taps of both kernels on that axis and
    ``pad_mode`` changes the border fold: wrong references, used to show that a test's bar can tell them apart."""
    sa, sb, kinv = compute_sigmas(sigma)
    ka, kb = gauss_kernel(sa), gauss_kernel(sb)
    ra, rb = len(ka) // 2, len(kb) // 2
    f = _load(img, min_intensity, max_intensity).astype(np.float64)
    lo = [int(interval_min_xyz[d]) - 1 - rb for d in range(3)]
    hi = [int(interval_min_xyz[d]) + int(interval_size_xyz[d]) + 1 + rb for d in range(3)]
    dims = img.shape[::-1]
    widths = [(max(0, -lo[d]), max(0, hi[d] - dims[d])) for d in (2, 1, 0)]
    ext = np.pad(f, widths, mode=pad_mode)
    box = ext[tuple(slice(lo[d] + widths[2 - d][0], hi[d] + widths[2 - d][0]) for d in (2, 1, 0))]

    def blur(x, k, r):
        x = x[tuple(slice(rb - r, x.shape[a] - (rb - r)) for a in range(3))]
        for d in (0, 1, 2):         # x, y, z
            kk = np.array(k, dtype=np.float64)
            if d == drop_outer_tap_axis:
                kk[0] = kk[-1] = 0.0
            x = _correlate_valid(x, kk, 2 - d)
        return x

    ga, gb = blur(box, ka, ra), blur(box, kb, rb)
    dog = (ga - gb) * float(np.float32(kinv))
    return dog, blur(np.abs(box), ka, ra), blur(np.abs(box), kb, rb)


def extrema(dog_box, interval_min_xyz, threshold=0.008, find_max=True, find_min=False, localization=True):
    """The extremum and localisation stage on a DoG box [z, y, x] covering [interval_min - 1, interval_min + size + 1)
    per axis (float32 values): detections of the interval's voxels, sorted by (z, y, x), as
    [(loc_xyz, value, voxel_xyz, is_max)].  Candidates at |DoG| >= float32(threshold / 3) (float32 compare), kept at
    |value| >= threshold in double (PARITY_GAPS #26)."""
    x0, y0, z0 = (int(v) for v in interval_min_xyz)
    thr0 = np.float32(threshold / INITIAL_THRESHOLD_DIV if localization else threshold)
    out = []
    c = dog_box[1:-1, 1:-1, 1:-1]
    cand = np.zeros(c.shape, bool)
    if find_max:
        cand |= c >= thr0
    if find_min:
        cand |= -c >= thr0
    for (kz, ky, kx) in np.argwhere(cand):
        nb = dog_box[kz:kz + 3, ky:ky + 3, kx:kx + 3].astype(np.float64)
        v = float(np.float32(nb[1, 1, 1]))
        others = np.delete(nb.ravel(), 13)
        is_max = find_max and v >= thr0 and not np.any(others > v)
        is_min = find_min and -v >= thr0 and not np.any(others < v)
        if not (is_max or is_min):
            continue
        d = np.zeros(3)
        val = v
        if localization:
            g = np.array([0.5 * (nb[1, 1, 2] - nb[1, 1, 0]), 0.5 * (nb[1, 2, 1] - nb[1, 0, 1]), 0.5 * (nb[2, 1, 1] - nb[0, 1, 1])])
            H = np.empty((3, 3))
            H[0, 0] = nb[1, 1, 2] - 2 * v + nb[1, 1, 0]
            H[1, 1] = nb[1, 2, 1] - 2 * v + nb[1, 0, 1]
            H[2, 2] = nb[2, 1, 1] - 2 * v + nb[0, 1, 1]
            H[0, 1] = H[1, 0] = 0.25 * (nb[1, 2, 2] - nb[1, 2, 0] - nb[1, 0, 2] + nb[1, 0, 0])
            H[0, 2] = H[2, 0] = 0.25 * (nb[2, 1, 2] - nb[2, 1, 0] - nb[0, 1, 2] + nb[0, 1, 0])
            H[1, 2] = H[2, 1] = 0.25 * (nb[2, 2, 1] - nb[2, 0, 1] - nb[0, 2, 1] + nb[0, 0, 1])
            det = np.linalg.det(H)
            if abs(det) >= 1e-30 and np.isfinite(det):
                d = np.clip(-np.linalg.solve(H, g), -0.5, 0.5)
                val = v + 0.5 * float(g @ d)
            if abs(val) < threshold:
                continue
        elif abs(v) < threshold:
            continue
        x, y, z = x0 + int(kx), y0 + int(ky), z0 + int(kz)
        out.append(((x + d[0], y + d[1], z + d[2]), val, (x, y, z), bool(is_max)))
    out.sort(key=lambda p: (p[2][2], p[2][1], p[2][0]))
    return out


def detect(img: np.ndarray, interval_min_xyz, interval_size_xyz, sigma=1.8, threshold=0.008, min_intensity=0.0,
           max_intensity=65535.0, find_max=True, find_min=False, localization=True):
    """Detections inside the block, sorted by (z, y, x): [(loc_xyz, value, voxel_xyz, is_max)].  The DoG is evaluated
    on the (virtually infinite, mirror-extended) image, so a block's result does not depend on the block grid."""
    # neighbours of border voxels come from the mirror extension of the IMAGE, not of the DoG: recompute the 1-px rim
    ext = np.pad(img, 1 + 64, mode="symmetric")
    pad = dog_volume(ext, sigma, min_intensity, max_intensity)[64:-64, 64:-64, 64:-64]
    x0, y0, z0 = (int(v) for v in interval_min_xyz)
    nx, ny, nz = (int(v) for v in interval_size_xyz)
    return extrema(pad[z0:z0 + nz + 2, y0:y0 + ny + 2, x0:x0 + nx + 2], interval_min_xyz, threshold, find_max, find_min,
                   localization)
