"""Intensity correction: the host side of `match-intensities`, `solve-intensities` and the coefficient input of
`affine-fusion --intensityN5Path` and `nonrigid-fusion --intensityN5Path`.

  match-intensities   J/SparkIntensityMatching.java:84-190 (IntensityCorrection.matchRansac per view pair)
  solve-intensities   J/IntensitySolver.java:50-123      (IntensityCorrection.solve, writeCoefficients)

The device renders every pair's overlap and draws the RANSAC hypotheses (csrc/intensity.cu); the host keeps the best
hypothesis per bucket, refines it with the mpicbg filter loop, and solves the coefficients with a vectorised float64
Gauss-Seidel relaxation.  Choices recalled from upstream are listed in PARITY_GAPS.md (rows I1-I9).

Coefficients of a view are a grid of n = (nx, ny, nz) cells over its full-resolution pixels; cell c maps intensity v
to a_c v + b_c.  Stored per view as a float64 dataset `{group}/setup{s}/timepoint{t}/{dataset}`: N5 dimensions
[nx, ny, nz, 2] (x fastest; index 0 of the last axis is a, 1 is b), Zarr shape (2, nz, ny, nx).
"""
from __future__ import annotations

import json
import os
import warnings

import numpy as np

from . import fusion as bf
from . import n5 as bn5
from . import solver as bsolver
from . import zarr as bzarr

#: InterpolatedAffineModel1D<InterpolatedAffineModel1D<AffineModel1D, TranslationModel1D>, IdentityModel> lambdas
LAMBDA_TRANSLATION = 0.01
LAMBDA_IDENTITY = 0.01
#: identityConnect between 6-neighbour cells of one view: matches at intensities 0 and 1 with this weight
IDENTITY_WEIGHT = 0.1
#: TileConfiguration.optimize(maxAllowedError, maxIterations, maxPlateauwidth = maxIterations)
SOLVE_MAX_ERROR = 0.01

COEFFICIENTS_SIZE_KEY = "coefficientsSize"


# ------------------------------------------------------------------------------------------------ pairs and geometry
def view_bounds(dims_xyz, reg):
    """IntensityCorrection.getBounds: the real world interval of the transformed pixel box [0, d - 1]."""
    M = np.asarray(reg, dtype=np.float64).reshape(3, 4)
    c = np.array([[x, y, z] for x in (0, dims_xyz[0] - 1) for y in (0, dims_xyz[1] - 1) for z in (0, dims_xyz[2] - 1)],
                 dtype=np.float64)
    w = c @ M[:, :3].T + M[:, 3]
    return w.min(axis=0), w.max(axis=0)


def pairs(view_ids, bounds):
    """Every selected i < j whose bounds intersect, across timepoints (J/SparkIntensityMatching.java:137-161)."""
    out = []
    for i, a in enumerate(view_ids):
        for b in view_ids[i + 1:]:
            lo = np.maximum(bounds[a][0], bounds[b][0])
            hi = np.minimum(bounds[a][1], bounds[b][1])
            if np.all(lo <= hi):
                out.append((a, b))
    return out


def render_range(lo, hi, render_scale):
    """The render grid of an intersection: integers r with ceil(lo s) <= r <= floor(hi s)."""
    s = float(render_scale)
    return (np.ceil(np.asarray(lo) * s).astype(np.int64), np.floor(np.asarray(hi) * s).astype(np.int64))


def _h(m):
    return np.vstack([np.asarray(m, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])


def inverse(m):
    return np.linalg.inv(_h(m))[:3]


# ------------------------------------------------------------------------------------------------ bucket acceptance
def fit_affine1d(x, y):
    """Least-squares AffineModel1D y = a x + b over the points; None when singular (all x equal)."""
    xm, ym = x.mean(), y.mean()
    dx = x - xm
    sxx = float(dx @ dx)
    if not sxx > 0.0:
        return None
    a = float(dx @ (y - ym)) / sxx
    return a, float(ym - a * xm)


def filter_accept(x, y, a, b, max_epsilon, max_trust, min_inlier_ratio, min_num_inliers):
    """The device hypothesis's inliers recomputed in float64, then mpicbg's filter loop (fit the inliers, drop those
    whose residual exceeds max_trust x the median residual, until nothing is dropped).  Accepted when the inliers are
    >= max(min_num_inliers, 2) and >= min_inlier_ratio x n before and after filtering; returns the inlier mask or None
    (a singular fit rejects the bucket)."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    need = max(int(min_num_inliers), 2)

    def enough(m):
        k = int(m.sum())
        return k >= need and k >= min_inlier_ratio * len(x)
    inl = np.abs((a * x + b) - y) < max_epsilon
    if not enough(inl):
        return None
    while True:
        n0 = int(inl.sum())
        m = fit_affine1d(x[inl], y[inl])
        if m is None:
            return None
        r = np.abs(m[0] * x + m[1] - y)
        inl = inl & (r <= max_trust * np.median(r[inl]))
        if int(inl.sum()) >= n0:
            break
    return inl if enough(inl) else None


# ------------------------------------------------------------------------------------------------ matches I/O
def _pair_group(a, b):
    return f"tp{a[0]}_setup{a[1]}-tp{b[0]}_setup{b[1]}"


class MatchesIO:
    """Pairwise coefficient matches under one N5 container (ViewPairCoefficientMatchesIO's role): the root attribute
    `coefficientsSize`, and per view pair a group `tp{t}_setup{s}-tp{t}_setup{s}` with attribute `cells`
    ([[cellA, cellB, offset, count], ...]) and the float32 list dataset `values` of the accepted inlier pairs (vA, vB)
    of every cell pair, in that order.  A pair without accepted cells has no group."""

    def __init__(self, path, create=False):
        self.store = bn5.N5Store(path, create=create)

    def write_coefficients_size(self, size):
        self.store.set_attributes("", {COEFFICIENTS_SIZE_KEY: [int(v) for v in size]})

    def read_coefficients_size(self):
        return [int(v) for v in self.store.get_attributes("")[COEFFICIENTS_SIZE_KEY]]

    def write(self, a, b, cells):
        """cells: [(cellA, cellB, values (k, 2) float32)]"""
        if not cells:
            return
        g = _pair_group(a, b)
        rows, vals, off = [], [], 0
        for ca, cb, v in cells:
            rows.append([int(ca), int(cb), off, len(v)])
            vals.append(np.asarray(v, np.float32))
            off += len(v)
        self.store.write_list(f"{g}/values", np.concatenate(vals), 1 << 16)
        self.store.set_attributes(g, {"cells": rows})

    def read(self, a, b):
        """[(cellA, cellB, values)] or None when the pair has no matches."""
        g = _pair_group(a, b)
        rows = self.store.get_attributes(g).get("cells")
        if rows is None:
            return None
        vals = self.store.read_list(f"{g}/values")
        return [(r[0], r[1], vals[r[2]:r[2] + r[3]]) for r in rows]


# ------------------------------------------------------------------------------------------------ match one pair
def match_pair(ctx, view_a, view_b, render_scale, render_min, render_max, min_threshold,
               max_threshold, min_num_candidates, num_iterations, max_epsilon, min_inlier_ratio, min_num_inliers,
               max_trust, chunk_points=0):
    """Candidates and RANSAC on the device, filter and acceptance on the host.  ``view_*``: dicts for
    Context.intensity_candidates (vol_handle = the resident level volume).  Returns [(cellA, cellB, inliers (k, 2))]
    and the timing-free counters (buckets, eligible, accepted)."""
    h, keys, offs, cnts, vals = ctx.intensity_candidates(view_a, view_b, render_scale, render_min, render_max,
                                                         min_threshold, max_threshold, chunk_points)
    try:
        a, b, cnt = ctx.intensity_ransac(h, len(keys), min_num_candidates, num_iterations, max_epsilon)
    finally:
        ctx.intensity_candidates_free(h)
    nb = int(np.prod(view_b["n_cells"]))
    out = []
    for k in range(len(keys)):
        if cnt[k] <= 0:
            continue
        v = vals[offs[k]:offs[k] + cnts[k]]
        inl = filter_accept(v[:, 0], v[:, 1], a[k], b[k], max_epsilon, max_trust, min_inlier_ratio, min_num_inliers)
        if inl is not None:
            out.append((int(keys[k]) // nb, int(keys[k]) % nb, v[inl]))
    return out, dict(buckets=len(keys), eligible=int((cnt >= 0).sum()), accepted=len(out))


def render_level(reg, render_scale, factors, mts):
    """best_mipmap_level for the render transform (scale(s) . registration)."""
    S = np.diag([float(render_scale)] * 3 + [1.0])
    return bf.best_mipmap_level((S @ _h(reg))[:3], factors, mts)


def device_view(handle, reg, mt, full_dims, n_cells):
    return dict(vol_handle=handle, world_to_px=inverse(reg), px_to_level=inverse(mt), full_dims=tuple(int(d) for d in full_dims),
                n_cells=tuple(int(n) for n in n_cells))


# ------------------------------------------------------------------------------------------------ solve
def cell_neighbours(n):
    """6-neighbour pairs (c, c') with c < c' of an x-fastest cell grid."""
    nx, ny, nz = n
    idx = np.arange(nx * ny * nz).reshape(nz, ny, nx)
    return np.concatenate([np.stack([idx[:, :, :-1].ravel(), idx[:, :, 1:].ravel()], 1),
                           np.stack([idx[:, :-1, :].ravel(), idx[:, 1:, :].ravel()], 1),
                           np.stack([idx[:-1, :, :].ravel(), idx[1:, :, :].ravel()], 1)]).astype(np.int64)


def build_links(views, n_cells, matches):
    """Tiles t = view index * cells + cell; links (t1, t2) each reduced once to the moments of its matches
    (sum w, w x, w y, w x^2, w x y, w y^2; x on t1's side, y on t2's).  ``matches``: {(viewA, viewB): [(cellA, cellB,
    values (k, 2))]}."""
    nc = int(np.prod(n_cells))
    vi = {v: i for i, v in enumerate(views)}
    t1, t2, mom = [], [], []
    for (va, vb), cells in matches.items():
        for ca, cb, v in cells:
            x, y = v[:, 0].astype(np.float64), v[:, 1].astype(np.float64)
            t1.append(vi[va] * nc + ca)
            t2.append(vi[vb] * nc + cb)
            mom.append([len(x), x.sum(), y.sum(), x @ x, x @ y, y @ y])
    nb = cell_neighbours(n_cells)
    w = IDENTITY_WEIGHT                  # points (0, 0) and (1, 1)
    ident = [2 * w, w, w, w, w, w]
    for i in range(len(views)):
        t1.extend((i * nc + nb[:, 0]).tolist())
        t2.extend((i * nc + nb[:, 1]).tolist())
        mom.extend([ident] * len(nb))
    return np.asarray(t1, np.int64), np.asarray(t2, np.int64), np.asarray(mom, np.float64).reshape(-1, 6)


def solve(views, n_cells, matches, max_iterations=1000):
    """{view: (a, b)} with a, b float64 [nz, ny, nx].  One 1-D tile per (view, cell), model
    (1 - l2) ((1 - l1) affine + l1 translation) + l2 identity fitted to the partners' current models, colour by colour
    (greedy colouring: tiles of one colour share no link), solver.proceed on the mean tile error as the stopping rule.
    Views without any match keep identity coefficients."""
    nc = int(np.prod(n_cells))
    T = len(views) * nc
    t1, t2, mom = build_links(views, n_cells, matches)
    A, B = np.ones(T), np.zeros(T)
    if T and len(t1):
        links = np.stack([t1, t2], 1)
        col, offsets, order = bsolver.colouring(T, links)
        W, Sx, Sy, Sxx, Sxy, Syy = mom.T
        errors = []
        for _ in range(int(max_iterations)):
            for c in range(len(offsets) - 1):
                tiles = order[offsets[c]:offsets[c + 1]]
                sel = np.zeros(T, bool)
                sel[tiles] = True
                acc = np.zeros((T, 5))         # sum w, own, own^2, target, own * target
                for own_t, oth_t, so, soo, sp, sop in ((t1, t2, Sx, Sxx, Sy, Sxy), (t2, t1, Sy, Syy, Sx, Sxy)):
                    m = sel[own_t]
                    au, bu = A[oth_t[m]], B[oth_t[m]]
                    contrib = np.stack([W[m], so[m], soo[m], au * sp[m] + bu * W[m], au * sop[m] + bu * so[m]], 1)
                    np.add.at(acc, own_t[m], contrib)
                w, sx, sxx, st, sxt = acc[tiles].T
                den = w * sxx - sx * sx
                ok = (w > 0) & (den > 1e-12 * np.maximum(w * sxx, 1e-300))
                a1 = np.where(ok, (w * sxt - sx * st) / np.where(ok, den, 1.0), 1.0)
                b1 = np.where(ok, (st - a1 * sx) / np.where(w > 0, w, 1.0), 0.0)
                b2 = np.where(w > 0, (st - sx) / np.where(w > 0, w, 1.0), 0.0)
                a = (1 - LAMBDA_IDENTITY) * ((1 - LAMBDA_TRANSLATION) * a1 + LAMBDA_TRANSLATION) + LAMBDA_IDENTITY
                b = (1 - LAMBDA_IDENTITY) * ((1 - LAMBDA_TRANSLATION) * b1 + LAMBDA_TRANSLATION * b2)
                A[tiles[ok]], B[tiles[ok]] = a[ok], b[ok]
            # per link the weighted RMS distance |M1(x) - M2(y)|, from the moments
            a1, b1, a2, b2 = A[t1], B[t1], A[t2], B[t2]
            d2 = (a1 * a1 * Sxx + a2 * a2 * Syy + b1 * b1 * W + b2 * b2 * W - 2 * a1 * a2 * Sxy + 2 * a1 * b1 * Sx
                  - 2 * a1 * b2 * Sx - 2 * a2 * b1 * Sy + 2 * a2 * b2 * Sy - 2 * b1 * b2 * W)
            te_num, te_w = np.zeros(T), np.zeros(T)
            for t in (t1, t2):
                np.add.at(te_num, t, np.maximum(d2, 0.0))
                np.add.at(te_w, t, W)
            linked = te_w > 0
            errors.append(float(np.mean(np.sqrt(te_num[linked] / te_w[linked]))))
            if not bsolver.proceed(errors, SOLVE_MAX_ERROR, int(max_iterations)):
                break
    shape = tuple(int(n) for n in n_cells)[::-1]
    matched = {v for pair in matches for v in pair if matches[pair]}
    out = {}
    for i, v in enumerate(views):
        if v in matched:
            out[v] = (A[i * nc:(i + 1) * nc].reshape(shape).copy(), B[i * nc:(i + 1) * nc].reshape(shape).copy())
        else:
            out[v] = (np.ones(shape), np.zeros(shape))
    return out


# ------------------------------------------------------------------------------------------------ coefficients I/O
def guess_storage(path, storage=None):
    """`-s` or the path's ending (J/IntensitySolver.java:58-73); HDF5 is not supported."""
    if storage is None:
        p = path.rstrip("/").lower()
        storage = "ZARR" if p.endswith(".zarr") else "N5" if p.endswith(".n5") else \
            "HDF5" if p.endswith((".h5", ".hdf5")) else None
        if storage is None:
            raise ValueError(f"unable to guess the storage format of {path!r}: pass storage='N5' or 'ZARR'")
    storage = storage.upper()
    if storage == "HDF5":
        raise NotImplementedError("HDF5 coefficient storage")
    if storage not in ("N5", "ZARR"):
        raise ValueError(f"unknown storage {storage!r}")
    return storage


def coefficient_dataset(group, view, dataset):
    """`{group}/setup{s}/timepoint{t}/{dataset}` (J/IntensitySolver.java:47)."""
    return "/".join(p for p in (group.strip("/"), f"setup{view[1]}", f"timepoint{view[0]}", dataset) if p)


def write_coefficients(path, storage, group, dataset, coefficients):
    """coefficients: {view: (a, b)} float64 [nz, ny, nx] each."""
    for v, (a, b) in coefficients.items():
        ds = coefficient_dataset(group, v, dataset)
        nz, ny, nx = a.shape
        if storage == "N5":
            st = bn5.N5Store(path, create=True)
            st.create_dataset(ds, [nx, ny, nz, 2], [nx, ny, nz, 2], np.float64)
            st.write_block(ds, (0, 0, 0, 0), np.ascontiguousarray(np.stack([a, b]), dtype=np.float64))
        else:
            bzarr.ZarrStore(path, create=True)
            d = os.path.join(path, ds)
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, ".zarray"), "w") as f:
                json.dump({"zarr_format": 2, "shape": [2, nz, ny, nx], "chunks": [2, nz, ny, nx], "dtype": "<f8",
                           "compressor": None, "fill_value": 0, "order": "C", "filters": None,
                           "dimension_separator": "/"}, f)
            os.makedirs(os.path.join(d, "0", "0", "0"), exist_ok=True)
            with open(os.path.join(d, "0", "0", "0", "0"), "wb") as f:
                f.write(np.ascontiguousarray(np.stack([a, b]), dtype="<f8").tobytes())


def read_coefficients(path, storage, group, dataset, view):
    """(a, b) float64 [nz, ny, nx] of one view, or None when the view has no dataset."""
    ds = coefficient_dataset(group, view, dataset)
    if not os.path.isdir(path):
        return None
    if storage == "N5":
        st = bn5.N5Store(path)
        if "dimensions" not in st.get_attributes(ds):
            return None
        blk = st.read_block(ds, (0, 0, 0, 0))
        return blk[0].copy(), blk[1].copy()
    meta_p = os.path.join(path, ds, ".zarray")
    if not os.path.exists(meta_p):
        return None
    with open(meta_p) as f:
        m = json.load(f)
    _, nz, ny, nx = m["shape"]
    with open(os.path.join(path, ds, "0", "0", "0", "0"), "rb") as f:
        arr = np.frombuffer(f.read(), dtype=np.dtype(m["dtype"])).astype(np.float64).reshape(2, nz, ny, nx)
    return arr[0].copy(), arr[1].copy()


def view_coefficients(path, storage, group, dataset, views):
    """{view: (a, b)} of every view in ``views``, read before anything is fused (`--intensityN5Path`, with
    `--intensityN5Storage` / `--intensityN5Group` / `--intensityN5Dataset`).  ``storage`` None: guessed from the path
    (guess_storage, HDF5 raises NotImplementedError).  A view without a coefficient dataset raises ValueError."""
    storage = guess_storage(path, storage)
    out = {}
    for v in views:
        c = read_coefficients(path, storage, group, dataset, v)
        if c is None:
            raise ValueError(f"no intensity coefficients for view (timepoint {v[0]}, setup {v[1]}) in {path} "
                             f"({coefficient_dataset(group, v, dataset)})")
        out[v] = c
    return out


def check_coefficients_size(stored, wanted):
    """A --numCoefficients that differs from the stored one warns and continues (J/IntensitySolver.java:95-98)."""
    if list(stored) != list(wanted):
        warnings.warn("numCoefficients stored with matches is different from specified numCoefficients argument!")
        return False
    return True

