"""CPU oracle for intensity correction: pair candidates, the RANSAC hypothesis stream, the filter / acceptance, the
coefficient solve and the coefficient application.

TEST INFRASTRUCTURE ONLY: never imported by the product.  Rendering and application repeat the device's float32
operation order (include/bsgpu.h, bs_intensity_pair_candidates / bs_intensity_apply): numpy float32 arithmetic is
IEEE round-to-nearest without contraction, like the __f*_rn intrinsics of csrc/intensity.cu.  Arrays are [z, y, x].

candidates_reference and apply_reference state the same two operations plainly in float64, with no float32 operation
order (the content_weights_reference convention of fusion_oracle.py): a misunderstanding that the bit-level oracle
shares with the device (the cell formula, the centre convention of the coefficient field) shows up against them.
"""
from __future__ import annotations

import numpy as np

SEED = 0x2545F4914F6CDD1D
_M64 = (1 << 64) - 1
F = np.float32


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def draw(key: int, h: int, n: int):
    """The two candidate indices of hypothesis h of bucket ``key`` with n candidates."""
    base = SEED ^ ((key << 32) & _M64)
    i = splitmix64(base ^ (2 * h)) % n
    j = splitmix64(base ^ (2 * h + 1)) % (n - 1)
    return i, j + (j >= i)


def cell_index(p, n, d):
    """clamp(floor(p n / d), 0, n - 1) per axis (float64)."""
    return np.clip(np.floor(np.asarray(p, np.float64) * n / d), 0, n - 1).astype(np.int64)


def _affine(m, x, y, z):
    m = np.asarray(m, np.float64).reshape(3, 4)
    return [((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3] for r in range(3)]


def sample(vol, q):
    """n-linear float32 sample with border extension on both sides at float32 coordinates q = (qx, qy, qz)."""
    dz, dy, dx = vol.shape
    v = vol.astype(F) if vol.dtype != F else vol
    f = [np.floor(c) for c in q]
    r = [(q[k] - f[k]).astype(F) for k in range(3)]
    i = [f[k].astype(np.int64) for k in range(3)]
    lo = [np.clip(i[k], 0, d - 1) for k, d in enumerate((dx, dy, dz))]
    hi = [np.clip(i[k] + 1, 0, d - 1) for k, d in enumerate((dx, dy, dz))]

    def at(x, y, z):
        return v[z, y, x]
    lerp = lambda a, b, t: (a + t * (b - a)).astype(F)
    c00 = lerp(at(lo[0], lo[1], lo[2]), at(hi[0], lo[1], lo[2]), r[0])
    c01 = lerp(at(lo[0], hi[1], lo[2]), at(hi[0], hi[1], lo[2]), r[0])
    c10 = lerp(at(lo[0], lo[1], hi[2]), at(hi[0], lo[1], hi[2]), r[0])
    c11 = lerp(at(lo[0], hi[1], hi[2]), at(hi[0], hi[1], hi[2]), r[0])
    return lerp(lerp(c00, c01, r[1]), lerp(c10, c11, r[1]), r[2])


def candidates(level_a, view_a, level_b, view_b, render_scale, render_min, render_max, min_threshold=1.0,
               max_threshold=float("nan")):
    """Buckets (keys, offsets, counts) and float32 values (n, 2) of one pair, as bs_intensity_pair_candidates.
    ``view_*``: dicts(world_to_px, px_to_level, full_dims, n_cells)."""
    rng = [np.arange(render_min[k], render_max[k] + 1, dtype=np.int64) for k in range(3)]
    rz, ry, rx = np.meshgrid(rng[2], rng[1], rng[0], indexing="ij")
    w = [r.ravel().astype(np.float64) / render_scale for r in (rx, ry, rz)]
    keep = np.ones(w[0].shape, bool)
    vals, cells = [], []
    for vol, v in ((level_a, view_a), (level_b, view_b)):
        p = _affine(v["world_to_px"], *w)
        fd = np.asarray(v["full_dims"], np.float64)
        for k in range(3):
            keep &= (p[k] >= 0.0) & (p[k] <= fd[k] - 1.0)
        q = [c.astype(F) for c in _affine(v["px_to_level"], *p)]
        val = sample(vol, q)
        keep &= val.astype(np.float64) >= min_threshold
        if not np.isnan(max_threshold):
            keep &= val.astype(np.float64) <= max_threshold
        n = np.asarray(v["n_cells"], np.int64)
        c = [cell_index(p[k], n[k], fd[k]) for k in range(3)]
        cells.append(c[0] + n[0] * (c[1] + n[1] * c[2]))
        vals.append(val)
    nb = int(np.prod(view_b["n_cells"]))
    key = cells[0] * nb + cells[1]
    idx = np.nonzero(keep)[0]
    order = idx[np.argsort(key[idx], kind="stable")]
    keys, counts = np.unique(key[order], return_counts=True)
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    return keys.astype(np.int64), offsets, counts.astype(np.int64), np.stack([vals[0][order], vals[1][order]], axis=1)


def sample_reference(vol, q):
    """float64 n-linear sample with border extension at float64 positions q = (qx, qy, qz), and the largest |corner|
    that entered each sample."""
    v = np.asarray(vol, np.float64)
    dims = v.shape[::-1]
    f = [np.floor(np.asarray(c, np.float64)) for c in q]
    t = [np.asarray(q[k], np.float64) - f[k] for k in range(3)]
    i = [f[k].astype(np.int64) for k in range(3)]
    out = np.zeros(np.shape(t[0]))
    cmax = np.zeros(np.shape(t[0]))
    for corner in range(8):
        o = [(corner >> k) & 1 for k in range(3)]
        w = np.ones(np.shape(t[0]))
        idx = []
        for k in range(3):
            w = w * (t[k] if o[k] else 1.0 - t[k])
            idx.append(np.clip(i[k] + o[k], 0, dims[k] - 1))
        c = v[idx[2], idx[1], idx[0]]
        out += w * c
        cmax = np.maximum(cmax, np.abs(c))
    return out, cmax


def candidates_reference(level_a, view_a, level_b, view_b, render_scale, render_min, render_max, min_threshold=1.0,
                         max_threshold=float("nan"), corners=False):
    """candidates() in float64: for every render point r the world position r / s, both full-resolution positions
    p = world_to_px w, the inside test 0 <= p <= d - 1, the values (sample_reference at px_to_level p, border
    extension), the thresholds v >= min and v <= max (max NaN: none) on those values, the cells clamp(floor(p n / d), 0, n - 1) and
    the key cellA x cells(B) + cellB.  Same (keys, offsets, counts, values (n, 2) float64) layout; ``corners`` also
    returns the largest |corner| of each value (n, 2)."""
    rng = [np.arange(render_min[k], render_max[k] + 1, dtype=np.int64) for k in range(3)]
    rz, ry, rx = np.meshgrid(rng[2], rng[1], rng[0], indexing="ij")
    w = np.stack([r.ravel() for r in (rx, ry, rz)]).astype(np.float64) / float(render_scale)
    keep = np.ones(w.shape[1], bool)
    vals, cmaxs, cells = [], [], []
    for vol, v in ((level_a, view_a), (level_b, view_b)):
        m = np.asarray(v["world_to_px"], np.float64).reshape(3, 4)
        p = m[:, :3] @ w + m[:, 3:]
        fd = np.asarray(v["full_dims"], np.float64)[:, None]
        keep &= np.all((p >= 0.0) & (p <= fd - 1.0), axis=0)
        ml = np.asarray(v["px_to_level"], np.float64).reshape(3, 4)
        val, cmax = sample_reference(vol, ml[:, :3] @ p + ml[:, 3:])
        keep &= val >= min_threshold
        if not np.isnan(max_threshold):
            keep &= val <= max_threshold
        n = np.asarray(v["n_cells"], np.int64)[:, None]
        c = np.clip(np.floor(p * n / fd), 0, n - 1).astype(np.int64)
        cells.append(c[0] + n[0] * (c[1] + n[1] * c[2]))
        vals.append(val)
        cmaxs.append(cmax)
    key = cells[0] * int(np.prod(view_b["n_cells"])) + cells[1]
    idx = np.nonzero(keep)[0]
    order = idx[np.argsort(key[idx], kind="stable")]
    keys, counts = np.unique(key[order], return_counts=True)
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    out = (keys.astype(np.int64), offsets, counts.astype(np.int64), np.stack([vals[0][order], vals[1][order]], axis=1))
    return out + (np.stack([cmaxs[0][order], cmaxs[1][order]], axis=1),) if corners else out


def ransac_bucket(values, key, num_iterations=1000, max_epsilon=5.1):
    """(a, b, count) of the best hypothesis of one bucket; (nan, nan, 0) when every hypothesis is skipped."""
    x, y = values[:, 0].astype(np.float64), values[:, 1].astype(np.float64)
    n = len(x)
    best = (np.nan, np.nan, 0)
    best_cnt = -1
    for h in range(num_iterations):
        i, j = draw(int(key), h, n)
        if x[i] == x[j]:
            continue
        a = (y[j] - y[i]) / (x[j] - x[i])
        b = y[i] - a * x[i]
        cnt = int(np.count_nonzero(np.abs((a * x + b) - y) < max_epsilon))
        if cnt > best_cnt:
            best, best_cnt = (a, b, cnt), cnt
    return best


def fit_affine1d(x, y, w=None):
    """Weighted least-squares y = a x + b; None when singular."""
    w = np.ones_like(x) if w is None else w
    sw = w.sum()
    xm, ym = (w * x).sum() / sw, (w * y).sum() / sw
    sxx = (w * (x - xm) ** 2).sum()
    if not sxx > 0:
        return None
    a = (w * (x - xm) * (y - ym)).sum() / sxx
    return a, ym - a * xm


def filter_accept(x, y, a, b, max_epsilon, max_trust, min_inlier_ratio, min_num_inliers):
    """Inliers of (a, b), then the mpicbg filter loop; the accepted inlier mask or None."""
    inl = np.abs((a * x + b) - y) < max_epsilon
    need = max(min_num_inliers, 2)
    if inl.sum() < need or inl.sum() < min_inlier_ratio * len(x):
        return None
    while True:
        n0 = int(inl.sum())
        m = fit_affine1d(x[inl], y[inl])
        if m is None:
            return None
        r = np.abs(m[0] * x + m[1] - y)
        med = np.median(r[inl])
        inl = inl & (r <= max_trust * med)
        if inl.sum() >= n0:
            break
    if inl.sum() < need or inl.sum() < min_inlier_ratio * len(x):
        return None
    return inl


def apply(vol, window_min, level_to_full, full_dims, ca, cb):
    """float32 a(q) v + b(q) (the operation order of bs_intensity_apply)."""
    z, y, x = np.meshgrid(*[np.arange(s) for s in vol.shape], indexing="ij")
    l = [(F(window_min[0]) + x.astype(F)).astype(F), (F(window_min[1]) + y.astype(F)).astype(F),
         (F(window_min[2]) + z.astype(F)).astype(F)]
    m = np.asarray(level_to_full, np.float64).reshape(3, 4).astype(F)
    n = ca.shape[::-1]
    lo, hi, t = [], [], []
    for r in range(3):
        q = (((m[r, 0] * l[0]).astype(F) + (m[r, 1] * l[1]).astype(F)).astype(F) + (m[r, 2] * l[2]).astype(F)).astype(F)
        q = (q + m[r, 3]).astype(F)
        sc = F(n[r] / full_dims[r])
        u = (((q + F(0.5)).astype(F) * sc).astype(F) - F(0.5)).astype(F)
        u = np.minimum(np.maximum(u, F(0)), F(n[r] - 1))
        f = np.floor(u)
        lo.append(f.astype(np.int64))
        hi.append(np.minimum(f.astype(np.int64) + 1, n[r] - 1))
        t.append((u - f).astype(F))
    lerp = lambda a, b, s: (a + (s * (b - a)).astype(F)).astype(F)
    out = []
    for g in (ca.astype(F), cb.astype(F)):
        c00 = lerp(g[lo[2], lo[1], lo[0]], g[lo[2], lo[1], hi[0]], t[0])
        c01 = lerp(g[lo[2], hi[1], lo[0]], g[lo[2], hi[1], hi[0]], t[0])
        c10 = lerp(g[hi[2], lo[1], lo[0]], g[hi[2], lo[1], hi[0]], t[0])
        c11 = lerp(g[hi[2], hi[1], lo[0]], g[hi[2], hi[1], hi[0]], t[0])
        out.append(lerp(lerp(c00, c01, t[1]), lerp(c10, c11, t[1]), t[2]))
    return ((out[0] * vol.astype(F)).astype(F) + out[1]).astype(F)


def apply_reference(vol, window_min, level_to_full, full_dims, ca, cb, parts=False):
    """apply() in float64: at every voxel l = window_min + index of the (window of the) level volume, the
    full-resolution position q = level_to_full l; a(q) and b(q) are the n-linear interpolation of the cell values
    placed at the cell centres (c + 0.5) d / n - 0.5, held constant beyond the first and last centre of each axis
    (PARITY_GAPS I9); the result is a v + b.  ``parts`` also returns a(q) and b(q)."""
    z, y, x = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in vol.shape], indexing="ij")
    l = np.stack([x + window_min[0], y + window_min[1], z + window_min[2]])
    m = np.asarray(level_to_full, np.float64).reshape(3, 4)
    q = np.einsum("rk,k...->r...", m[:, :3], l) + m[:, 3].reshape(3, 1, 1, 1)
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    n = ca.shape[::-1]
    # cell c's centre sits at (c + 0.5) d / n - 0.5, so q is at fractional cell position (q + 0.5) n / d - 0.5
    u = [np.clip((q[r] + 0.5) * n[r] / float(full_dims[r]) - 0.5, 0.0, n[r] - 1.0) for r in range(3)]
    a, _ = sample_reference(ca, u)
    b, _ = sample_reference(cb, u)
    out = a * np.asarray(vol, np.float64) + b
    return (out, a, b) if parts else out
