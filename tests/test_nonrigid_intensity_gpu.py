"""nonrigid-fusion --intensityN5Path on the device: identity coefficients change no bit, corrected blocks against an
oracle (intensity_oracle.apply on every full view, then nonrigid_oracle.fuse_block), and the planted-gain chain
match-intensities -> solve-intensities -> nonrigid-fusion against affine-fusion with the same coefficients."""
import os

import numpy as np
import pytest

from bsgpu import commands, intensity as bint, n5 as bn5, spimdata, zarr as bzarr
from oracle import intensity_oracle as io
from tests.intensity_scene import planted_dataset
from tests.test_nonrigid_cpu import write_correspondences, write_points
from tests.test_nonrigid_gpu import _close, _dataset, _faces, _oracle_volume
from tests.test_nonrigid_intensity_cpu import seeded_coefficients

pytestmark = pytest.mark.gpu

DIMS = (104, 340, 20)          # the box of _dataset's three views


def oracle_corrected_volume(xml, tiles, ips, coeffs, out_dtype, mn, mx):
    """The reference for corrected non-rigid blocks: every full view corrected by intensity_oracle.apply (window 0,
    identity level transform: s0 is full resolution), then the non-rigid oracle on the corrected float32 views."""
    corrected = [dict(t, img=io.apply(t["img"], (0, 0, 0), np.eye(3, 4), t["size_xyz"], *coeffs[(0, t["setup"])]))
                 for t in tiles]
    return _oracle_volume(xml, corrected, ips, DIMS, (0, 0, 0), (64, 64, 16), out_dtype, mn, mx)


def _read(out, storage="N5"):
    return (bn5.N5Store(out) if storage == "N5" else bzarr.ZarrStore(out)).read_volume("fused/s0")


@pytest.mark.parametrize("dtype", ["UINT16", "FLOAT32"])
def test_identity_coefficients_change_no_bit(ctx, tmp_path, dtype):
    xml, tiles, _ = _dataset(tmp_path)
    ident = {(0, t["setup"]): (np.ones((2, 2, 3)), np.zeros((2, 2, 3))) for t in tiles}
    bint.write_coefficients(str(tmp_path / "id.n5"), "N5", "", "intensity", ident)
    outs = []
    for name, kw in (("a.n5", {}), ("b.n5", dict(intensity_n5_path=str(tmp_path / "id.n5")))):
        out = str(tmp_path / name)
        commands.nonrigid_fusion(xml, ctx, out, "fused/s0", ["beads"], block_size=(32, 32, 16), data_type=dtype,
                                 min_intensity=500.0, max_intensity=1600.0, **kw)
        outs.append(_read(out))
    assert np.array_equal(outs[0], outs[1]) and outs[0].any()


@pytest.mark.parametrize("storage, dtype", [("N5", "FLOAT32"), ("ZARR", "UINT16")])
def test_corrected_blocks_match_the_oracle(ctx, tmp_path, monkeypatch, storage, dtype):
    xml, tiles, ips = _dataset(tmp_path)
    co = seeded_coefficients([(0, t["setup"]) for t in tiles])
    cpath = str(tmp_path / "coeff.zarr")
    bint.write_coefficients(cpath, "ZARR", "", "intensity", co)
    origins = []
    apply = ctx.intensity_apply

    def recorded(h, full, mt, a, b, window_min_xyz=(0, 0, 0)):
        origins.append(tuple(int(v) for v in window_min_xyz))
        return apply(h, full, mt, a, b, window_min_xyz)
    monkeypatch.setattr(ctx, "intensity_apply", recorded)
    out = str(tmp_path / ("fused.n5" if storage == "N5" else "fused.zarr"))
    # one super-block per call: every chunk stages its own windows, most of them away from the view's origin
    commands.nonrigid_fusion(xml, ctx, out, "fused/s0", ["beads"], storage=storage, block_size=(32, 32, 16),
                             data_type=dtype, min_intensity=500.0, max_intensity=1600.0, blocks_per_call=1,
                             intensity_n5_path=cpath)
    assert sum(o != (0, 0, 0) for o in origins) >= 4, origins
    np_dt = np.float32 if dtype == "FLOAT32" else np.uint16
    want, _ = oracle_corrected_volume(xml, tiles, ips, co, np_dt, 500.0, 1600.0)
    got = _read(out, storage)
    data = spimdata.SpimData2.load(xml)
    faces = _faces([(data.model(*v), tuple(data.setups[v[1]].size)) for v in data.view_ids()], (0, 0, 0), DIMS)
    _close(got, want, faces=faces)
    # the coefficients matter: the uncorrected oracle is far from the result
    plain, _ = _oracle_volume(xml, tiles, ips, DIMS, (0, 0, 0), (64, 64, 16), np_dt, 500.0, 1600.0)
    assert np.abs(got.astype(np.float64) - plain).max() > 20.0


# ------------------------------------------------------------------------------------------ the planted-gain chain
def _lattice_correspondences(xml, step=12):
    """Beads on a lattice in every pairwise overlap, each at its exact local position in both views (the
    registrations are correct), label "beads"."""
    data = spimdata.SpimData2.load(xml)
    views = data.view_ids()
    regs = {v: data.model(*v) for v in views}
    boxes = {v: bint.view_bounds(data.setups[v[1]].size, regs[v]) for v in views}
    pts = {v: [] for v in views}
    rows = {v: [] for v in views}
    for i, a in enumerate(views):
        for b in views[i + 1:]:
            lo = np.maximum(boxes[a][0], boxes[b][0]) + 2
            hi = np.minimum(boxes[a][1], boxes[b][1]) - 2
            if np.any(hi < lo):
                continue
            p = np.stack(np.meshgrid(*[np.arange(lo[d], hi[d] + 1e-9, step) for d in range(3)], indexing="ij"),
                         -1).reshape(-1, 3)
            ia, ib = len(pts[a]), len(pts[b])
            for v in (a, b):
                inv = bint.inverse(regs[v])
                pts[v].extend(p @ inv[:, :3].T + inv[:, 3])
            rows[a] += [(ia + k, b, "beads", ib + k) for k in range(len(p))]
            rows[b] += [(ib + k, a, "beads", ia + k) for k in range(len(p))]
    ips = bn5.N5Store(os.path.join(os.path.dirname(xml), "interestpoints.n5"), create=True)
    for v in views:
        write_points(ips, v, "beads", np.asarray(pts[v]).reshape(-1, 3))
        write_correspondences(ips, v, "beads", rows[v])
    return data, views, regs


def _per_view_disagreement(ctx, tmp_path, xml, views, name, **kw):
    """Every view non-rigidly fused on its own (float32), then the median |A - B| over the voxels two of them both
    cover with non-zero weight."""
    fused = {}
    for v in views:
        out = str(tmp_path / f"{name}_{v[1]}.n5")
        commands.nonrigid_fusion(xml, ctx, out, "s0", ["beads"], block_size=(64, 64, 32),
                                 view_selection=dict(tile_ids=[v[1]]), **kw)
        st = bn5.N5Store(out)
        fused[v] = (np.asarray(st.get_attributes("s0")["offset"]), st.read_volume("s0"))
    d = []
    for i, a in enumerate(views):
        for b in views[i + 1:]:
            (oa, A), (ob, B) = fused[a], fused[b]
            lo = np.maximum(oa, ob)
            hi = np.minimum(oa + A.shape[::-1], ob + B.shape[::-1])
            if np.any(hi <= lo):
                continue
            sa = A[lo[2] - oa[2]:hi[2] - oa[2], lo[1] - oa[1]:hi[1] - oa[1], lo[0] - oa[0]:hi[0] - oa[0]]
            sb = B[lo[2] - ob[2]:hi[2] - ob[2], lo[1] - ob[1]:hi[1] - ob[1], lo[0] - ob[0]:hi[0] - ob[0]]
            m = (sa > 0) & (sb > 0)
            d.append(np.abs(sa[m].astype(np.float64) - sb[m]))
    return float(np.median(np.concatenate(d)))


def test_planted_chain_matches_affine_fusion(ctx, tmp_path):
    xml, _ = planted_dataset(tmp_path, tile=(128, 128, 32), overlap=32)
    data, views, regs = _lattice_correspondences(xml)
    m = str(tmp_path / "matches.n5")
    got = commands.match_intensities(xml, ctx, m, num_coefficients=(4, 4, 2), render_scale=0.5)
    assert sum(len(c) for c in got.values()) >= 8
    cpath = str(tmp_path / "coeff.n5")
    commands.solve_intensities(xml, cpath, m, num_coefficients=(4, 4, 2))

    out = str(tmp_path / "nonrigid.n5")
    commands.nonrigid_fusion(xml, ctx, out, "s0", ["beads"], block_size=(64, 64, 32), intensity_n5_path=cpath)
    nr = bn5.N5Store(out)
    aff_out = str(tmp_path / "affine.n5")
    commands.create_fusion_container(xml, aff_out, block_size=(64, 64, 32))
    s0 = commands.affine_fusion(aff_out, ctx, intensity_n5_path=cpath)[0]
    af = bn5.N5Store(aff_out).read_volume(s0)
    got = nr.read_volume("s0")
    assert got.shape == af.shape == (32, 224, 224) and nr.get_attributes("s0")["offset"] == [0, 0, 0]
    assert (af != 0).mean() > 0.5
    faces = _faces([(regs[v], tuple(data.setups[v[1]].size)) for v in views], (0, 0, 0), got.shape[::-1])
    _close(got, af, faces=faces)

    before = _per_view_disagreement(ctx, tmp_path, xml, views, "plain")
    after = _per_view_disagreement(ctx, tmp_path, xml, views, "corrected", intensity_n5_path=cpath)
    assert after < 0.5 * before, (before, after)
