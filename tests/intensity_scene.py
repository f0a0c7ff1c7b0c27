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
