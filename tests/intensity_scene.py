"""Planted intensity scenes and an oracle-backed context for the intensity-correction tests (plain module, no tests)."""
import numpy as np

from bsgpu import n5 as bn5, spimdata
from oracle import intensity_oracle as io
from tests import synth
from tests.fake_ctx import FakeContext


def gain(shape_zyx, lo, hi, axis):
    """A smooth ramp from lo to hi along one axis (0 z, 1 y, 2 x) of a [z, y, x] tile."""
    n = shape_zyx[axis]
    r = np.linspace(lo, hi, n)
    sh = [1, 1, 1]
    sh[axis] = n
    return np.broadcast_to(r.reshape(sh), shape_zyx)


def planted_dataset(tmp_path, tile=(96, 96, 24), overlap=32, gains=True, seed=3):
    """2 x 2 tiles (x, y) of one seeded smooth volume; view v is stored as round(g_v(p) I + o_v) with a different
    smooth gain ramp in [0.7, 1.3] per view (``gains``) or as round(I).  Returns (xml, {setup: raw float tile})."""
    tx, ty, tz = tile
    nom = (tx - overlap, ty - overlap)
    G = synth.field((tz + 8, ty + nom[1] + 8, tx + nom[0] + 8), seed=seed, sigma=3.0, mean=800.0, std=250.0)
    ramps = [(0.7, 1.1, 2, 10.0), (1.3, 0.9, 1, -5.0), (0.9, 1.25, 2, 0.0), (1.2, 0.75, 1, 8.0)]
    tiles, raw = [], {}
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    for s, (gx, gy) in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
        I = G[4:4 + tz, 4 + gy * nom[1]:4 + gy * nom[1] + ty, 4 + gx * nom[0]:4 + gx * nom[0] + tx].astype(np.float64)
        raw[s] = I
        if gains:
            lo, hi, ax, off = ramps[s]
            I = gain(I.shape, lo, hi, ax) * I + off
        vol = np.clip(np.rint(I), 0, 65535).astype(np.uint16)
        bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 32))
        tiles.append(dict(setup=s, size_xyz=tile, tile=s, translation_xyz=(gx * nom[0], gy * nom[1], 0)))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    return xml, raw


class IntensityFakeContext(FakeContext):
    """FakeContext plus the intensity entry points, computed by oracle/intensity_oracle.py."""

    def __init__(self):
        super().__init__()
        self.cands = {}

    def intensity_candidates(self, view_a, view_b, render_scale, render_min, render_max, min_threshold=1.0,
                             max_threshold=float("nan"), chunk_points=0):
        keys, offs, cnts, vals = io.candidates(self.vols[view_a["vol_handle"]], view_a, self.vols[view_b["vol_handle"]],
                                               view_b, render_scale, render_min, render_max, min_threshold, max_threshold)
        h = self.next
        self.next += 1
        self.cands[h] = (keys, offs, cnts, vals)
        return h, keys, offs, cnts, vals

    def intensity_candidates_free(self, h):
        del self.cands[h]

    def intensity_ransac(self, h, n_buckets, min_num_candidates=1000, num_iterations=1000, max_epsilon=5.1):
        keys, offs, cnts, vals = self.cands[h]
        a, b, c = np.full(n_buckets, np.nan), np.full(n_buckets, np.nan), np.full(n_buckets, -1, np.int32)
        for k in range(n_buckets):
            if cnts[k] >= max(2, min_num_candidates):
                a[k], b[k], c[k] = io.ransac_bucket(vals[offs[k]:offs[k] + cnts[k]], int(keys[k]), num_iterations, max_epsilon)
        return a, b, c

    def intensity_apply(self, h, full_dims_xyz, level_to_full, coeff_a, coeff_b, window_min_xyz=(0, 0, 0)):
        return self.volume_upload(io.apply(self.vols[h], window_min_xyz, level_to_full, full_dims_xyz, coeff_a, coeff_b))


def overlap_disagreement(views, regs, dims, pairs, render_scale=0.5):
    """Median |A - B| over the render points of every overlap: ``views`` {v: [z, y, x] float array}."""
    from bsgpu import intensity as bint
    d = []
    ident = np.eye(3, 4)
    for a, b in pairs:
        ba, bb = bint.view_bounds(dims[a], regs[a]), bint.view_bounds(dims[b], regs[b])
        rmin, rmax = bint.render_range(np.maximum(ba[0], bb[0]), np.minimum(ba[1], bb[1]), render_scale)
        va = dict(world_to_px=bint.inverse(regs[a]), px_to_level=ident, full_dims=dims[a], n_cells=(1, 1, 1))
        vb = dict(world_to_px=bint.inverse(regs[b]), px_to_level=ident, full_dims=dims[b], n_cells=(1, 1, 1))
        _, _, _, vals = io.candidates(views[a].astype(np.float32), va, views[b].astype(np.float32), vb, render_scale,
                                      rmin, rmax, -np.inf)
        d.append(np.abs(vals[:, 0].astype(np.float64) - vals[:, 1]))
    return float(np.median(np.concatenate(d)))


# ------------------------------------------------------------------------------------------------ kernel-test scenes
# Scenes for the candidate, RANSAC and apply kernels whose float64 geometry is exact (integer translations, power-of-two
# scales, render scale 1 or a power of two): on them the keys and the kept set of the float64 reference equal the
# device's exactly, and only the values carry a tolerance (candidate_value_bound).
U = 2.0 ** -24          # unit roundoff of float32 round-to-nearest

#: the command default --numCoefficients 8,8,8 on 128 x 128 x 64 views, B half a cell away on every axis: ~3 400
#: buckets out of 512 x 512 keys, so every k_compact thread scans 256 keys
DEFAULT_GRID = dict(dims=(128, 128, 64), n_cells=(8, 8, 8), shift=(8, 8, 4))
#: ~23 000 buckets: k_scatter's cursors (8 B per bucket) need ~180 KB and k_seg_count's counters ~90 KB of shared
#: memory, both above the 48 KB a kernel gets without opting in
WIDE_SLOTS = dict(dims=(128, 128, 48), n_cells=(16, 16, 24), shift=(4, 4, 0))
#: ~31 800 buckets: 8 B each exceeds the 227 KB of shared memory one CTA may opt into (BS_ERR_UNSUPPORTED)
TOO_MANY_SLOTS = dict(dims=(128, 128, 16), n_cells=(32, 32, 8), shift=(2, 2, 0))


def translation(t):
    m = np.eye(3, 4)
    m[:, 3] = t
    return m


def shifted_grid_scene(dims, n_cells, shift, seed=0):
    """Two views of ``dims`` (x, y, z) on one voxel grid, B translated by the integer ``shift``: A uint16, B float32
    with B(p) = 1.5 A(p + shift) + 7 + integer noise, so each bucket holds a noisy line.  Returns (A, B, view_a,
    view_b, render_min, render_max) with views as bint.device_view (vol_handle 0).  The render range is the overlap
    grown by one plane below in x: those points lie outside B, and the render plane is not a multiple of 32 points."""
    from bsgpu import intensity as bint
    rng = np.random.default_rng(seed)
    dx, dy, dz = dims
    sx, sy, sz = shift
    G = rng.integers(1, 1000, (dz + sz, dy + sy, dx + sx))
    A = G[:dz, :dy, :dx].astype(np.uint16)
    B = (1.5 * G[sz:, sy:, sx:] + 7 + rng.integers(-2, 3, (dz, dy, dx))).astype(np.float32)
    va = bint.device_view(0, np.eye(3, 4), np.eye(3, 4), dims, n_cells)
    vb = bint.device_view(0, translation(shift), np.eye(3, 4), dims, n_cells)
    rmin = np.array([sx - 1, sy, sz])
    rmax = np.array([dx - 1, dy - 1, dz - 1])
    return A, B, va, vb, rmin, rmax


def integer_scene(seed=11):
    """uint8 on both sides, with values on the thresholds and points on the edges the kernels switch on.

    A: full resolution 64 x 48 x 16 seen through its 2x level (32 x 24 x 8, mipmap transform 2 l + 0.5), registered
    with a 90 degree rotation about z (world = (47 - py, px, pz)); B: level 0, 40 x 64 x 16, translated by (20, 0, 0).
    At render scale 1 every point is an integer p, so A is sampled at quarter positions and every float32 lerp of
    uint8 data is exact.  Both volumes are 2x2x2-blocky draws from {0, 1, 2, 3, 100, 199, 200, 201, 255}: block
    interiors sample to exact integers, so values hit min_threshold 1 and max_threshold 200 exactly.  The overlap
    reaches p = d - 1 (A's x, B's y), and cell borders p n / d in {16, 32, 48} (A x, B y), 12, 24 (A y), 20 (B x)
    and 8 (z) are integers that render points hit."""
    from bsgpu import intensity as bint, zarr as bzarr
    rng = np.random.default_rng(seed)
    lv = np.array([0, 1, 2, 3, 100, 199, 200, 201, 255], np.uint8)

    def blocky(shape_zyx):
        small = lv[rng.integers(0, len(lv), tuple(s // 2 for s in shape_zyx))]
        return small.repeat(2, 0).repeat(2, 1).repeat(2, 2)
    LA = blocky((8, 24, 32))
    B = blocky((16, 64, 40))
    regA = np.array([[0, -1, 0, 47], [1, 0, 0, 0], [0, 0, 1, 0]], np.float64)
    mtA = np.asarray(bzarr.mipmap_transform_default((2, 2, 2)), np.float64)
    va = bint.device_view(0, regA, mtA, (64, 48, 16), (4, 4, 2))
    vb = bint.device_view(0, translation((20, 0, 0)), np.eye(3, 4), (40, 64, 16), (2, 4, 2))
    return LA, B, va, vb, np.array([20, 0, 0]), np.array([47, 63, 15])


def candidate_value_bound(cmax):
    """|float32 n-linear sample - float64 sample| <= 16 u max|corner| (PARITY_GAPS row 37): three levels of
    lerps a0 + t (a1 - a0), each adding at most 3 roundings of at most max|corner|, plus the float32 rounding of the
    sample position, whose effect is bounded by the same corner spread."""
    return 16 * U * cmax


def apply_bound(vol, window_min, level_to_full, full_dims, ca, cb):
    """Bound on |bs_intensity_apply - apply_reference| per voxel, first order in u = 2^-24 (float32 rounding):
      q_r     level_to_full rounded to float32 (1 u) then 3 products and 3 sums: |dq| <= 7 u S_r,
              S_r = sum_k |m_rk l_k| + |m_r3|;
      u_r     (q + 0.5) sc - 0.5 with sc = float32(n / d) (1 u) and 3 roundings:
              |du| <= (n / d) (|dq| + 4 u (|q| + 0.5)) + u (n + 1); clamp, floor and t = u - floor(u) are exact;
      a, b    the n-linear field moves by at most G_r |du_r| (G_r: the largest step between neighbouring cells along r),
              and 7 lerps in 3 levels add at most 3 u max|cell| per level: 9 u max|cell|;
      a v + b 2 roundings: 2 u (|a v| + |b|).
    |out - ref| <= |v| (9 u A + sum G^a du) + 9 u B + sum G^b du + 2 u (|a v| + |b|), with A, B = max |cell|."""
    vol = np.asarray(vol, np.float64)
    z, y, x = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in vol.shape], indexing="ij")
    l = np.stack([x + window_min[0], y + window_min[1], z + window_min[2]])
    m = np.asarray(level_to_full, np.float64).reshape(3, 4)
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    n = ca.shape[::-1]
    ga, gb = np.zeros(np.shape(x)), np.zeros(np.shape(x))
    for r in range(3):
        S = sum(np.abs(m[r, k] * l[k]) for k in range(3)) + abs(m[r, 3])
        q = sum(m[r, k] * l[k] for k in range(3)) + m[r, 3]
        du = n[r] / full_dims[r] * (7 * U * S + 4 * U * (np.abs(q) + 0.5)) + U * (n[r] + 1)
        ax = 2 - r
        step = lambda c: float(np.abs(np.diff(c, axis=ax)).max()) if c.shape[ax] > 1 else 0.0
        ga += step(ca) * du
        gb += step(cb) * du
    out, a, b = io.apply_reference(vol, window_min, level_to_full, full_dims, ca, cb, parts=True)
    return (np.abs(vol) * (9 * U * np.abs(ca).max() + ga) + 9 * U * np.abs(cb).max() + gb
            + 2 * U * (np.abs(a * vol) + np.abs(b)))


def apply_case(x, level, dtype, seed=0):
    """One bs_intensity_apply case: a window of y 7 and z 5 voxels and the given x at the far corner of a level
    volume, its level transform (0 identity, 1 anisotropic (2, 2, 1), 2 4x), a in [0, 3] and b in [-40, -1].  The
    cell grid has 1 cell along one axis and one cell per full-resolution pixel along another, by dtype.  Returns
    (vol, window_min, level_to_full, full_dims, ca, cb)."""
    from bsgpu import zarr as bzarr
    rng = np.random.default_rng(seed)
    f = [(1, 1, 1), (2, 2, 1), (4, 4, 4)][level]
    wdims = (x, 7, 5)
    wmin = (3, 4, 2)
    full = tuple((wmin[k] + wdims[k]) * f[k] for k in range(3))
    mt = np.asarray(bzarr.mipmap_transform_default(f), np.float64)
    n = {np.uint8: (1, full[1], 3), np.uint16: (full[0], 1, 2), np.float32: (5, 3, full[2])}[dtype]
    hi = {np.uint8: 256, np.uint16: 65536, np.float32: 1000}[dtype]
    vol = (rng.random(wdims[::-1]) * hi).astype(dtype)
    ca = rng.uniform(0.0, 3.0, n[::-1])
    cb = rng.uniform(-40.0, -1.0, n[::-1])
    return vol, wmin, mt, full, ca, cb


# ------------------------------------------------------------------------------------------------ RANSAC buckets
def pair_counts(x, y, eps):
    """Inlier count |a x + b - y| < eps of the line through every pair (p, q), p < q, x_p != x_q, with (a, b)
    computed as the device does (float64): {(p, q): count}."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    out = {}
    for p in range(len(x)):
        q = np.arange(p + 1, len(x))
        q = q[x[q] != x[p]]
        a = (y[q] - y[p]) / (x[q] - x[p])
        b = y[p] - a * x[p]
        c = (np.abs((a[:, None] * x[None, :] + b[:, None]) - y[None, :]) < eps).sum(axis=1)
        out.update({(p, int(k)): int(v) for k, v in zip(q, c)})
    return out


def later_round_bucket(n=64, h_special=1024, eps=1e-3, seed=0):
    """float32 (x, y) of one bucket (key 0) whose only collinear triple within eps is three special candidates on
    y = 2 x + 3, at the two indices hypothesis ``h_special`` draws and a third that no earlier hypothesis pairs with
    either: every hypothesis h < h_special counts 2 inliers, and the first to count 3 is h_special.  The noise is
    redrawn (seed + 1, ...) until pair_counts shows no other triple."""
    i, j = io.draw(0, h_special, n)
    earlier = {frozenset(io.draw(0, h, n)) for h in range(h_special)}
    assert frozenset((i, j)) not in earlier
    k = next(k for k in range(n) if k not in (i, j) and not {frozenset((i, k)), frozenset((j, k))} & earlier)
    special = {frozenset((i, j)), frozenset((i, k)), frozenset((j, k))}
    for s in range(seed, seed + 100):
        rng = np.random.default_rng(s)
        x = rng.uniform(0.0, 1000.0, n).astype(np.float32)
        y = rng.uniform(0.0, 1000.0, n).astype(np.float32)
        x[[i, j, k]] = (100.0, 200.0, 300.0)
        y[[i, j, k]] = (203.0, 403.0, 603.0)
        c = pair_counts(x, y, eps)
        if all(v == (3 if frozenset(pq) in special else 2) for pq, v in c.items()):
            return x, y
    raise AssertionError("no noise draw without a collinear triple")
