"""Intensity correction on the H100: candidates, chunking, RANSAC and the coefficient application against
oracle/intensity_oracle.py, identity coefficients through affine-fusion, and the planted chain end to end."""
import numpy as np
import pytest

import bsgpu
from bsgpu import commands, intensity as bint, n5 as bn5, spimdata
from oracle import intensity_oracle as io
from tests.intensity_scene import overlap_disagreement, planted_dataset

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    with bsgpu.Context(0) as c:
        yield c


def _pair(seed=4):
    """Two integer-valued views of different dtypes, one rotated, and a 2x level for B."""
    rng = np.random.default_rng(seed)
    A = rng.integers(0, 400, (20, 40, 48)).astype(np.uint16)
    B = rng.integers(0, 400, (24, 36, 52)).astype(np.float32)
    th = np.deg2rad(7.0)
    regA = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float64)
    regB = np.array([[np.cos(th), -np.sin(th), 0, 20.3], [np.sin(th), np.cos(th), 0, 3.1], [0, 0, 1, -1.7]])
    mtB = np.array([[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 1, 0]], np.float64)   # level 1 of a view 2x in x, y
    fullB = (104, 72, 24)
    return A, B, regA, regB, mtB, fullB


def _views(ctx, A, B, regA, regB, mtB, fullB, n=(3, 2, 2)):
    ha, hb = ctx.volume_upload(A), ctx.volume_upload(B)
    va = bint.device_view(ha, regA, np.eye(3, 4), A.shape[::-1], n)
    vb = bint.device_view(hb, regB, mtB, fullB, (2, 3, 1))
    return ha, hb, va, vb


def test_candidates_equal_the_oracle_and_do_not_depend_on_chunking(ctx):
    A, B, regA, regB, mtB, fullB = _pair()
    ha, hb, va, vb = _views(ctx, A, B, regA, regB, mtB, fullB)
    try:
        lo = np.maximum(bint.view_bounds(A.shape[::-1], regA)[0], bint.view_bounds(fullB, regB)[0])
        hi = np.minimum(bint.view_bounds(A.shape[::-1], regA)[1], bint.view_bounds(fullB, regB)[1])
        rmin, rmax = bint.render_range(lo, hi, 0.75)
        want = io.candidates(A, va, B, vb, 0.75, rmin, rmax, 20.5, 380.5)
        runs = []
        for chunk in (0, 977, 5000):
            h, *got = ctx.intensity_candidates(va, vb, 0.75, rmin, rmax, 20.5, 380.5, chunk_points=chunk)
            ctx.intensity_candidates_free(h)
            runs.append(got)
        for got in runs:
            for g, w in zip(got, want):
                assert g.shape == w.shape and np.array_equal(g, w)
        assert len(want[0]) >= 6 and len(want[3]) > 1000
        # RANSAC (a, b, count) per bucket
        h, keys, offs, cnts, vals = ctx.intensity_candidates(va, vb, 0.75, rmin, rmax, 20.5, 380.5)
        try:
            a, b, c = ctx.intensity_ransac(h, len(keys), min_num_candidates=50, num_iterations=300, max_epsilon=40.0)
        finally:
            ctx.intensity_candidates_free(h)
        checked = 0
        for k in range(len(keys)):
            if cnts[k] < 50:
                assert c[k] == -1
                continue
            wa, wb, wc = io.ransac_bucket(vals[offs[k]:offs[k] + cnts[k]], int(keys[k]), 300, 40.0)
            assert (a[k], b[k], c[k]) == (wa, wb, wc)
            checked += 1
        assert checked >= 3
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("level", [0, 1])
def test_apply_within_2_ulp_of_the_oracle(ctx, dtype, level):
    rng = np.random.default_rng(5)
    vol = (rng.random((14, 30, 37)) * 250).astype(dtype)
    mt = np.eye(3, 4) if level == 0 else np.array([[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 2, 0.5]])
    full = (90, 70, 40)
    wmin = (5, 3, 2)
    ca = rng.uniform(0.6, 1.4, (3, 4, 5))
    cb = rng.uniform(-20, 20, (3, 4, 5))
    h = ctx.volume_upload(vol)
    try:
        hc = ctx.intensity_apply(h, full, mt, ca, cb, wmin)
        got = ctx.volume_download(hc)
        ctx.volume_free(hc)
    finally:
        ctx.volume_free(h)
    want = io.apply(vol, wmin, mt, full, ca, cb)
    ulp = np.spacing(np.abs(want).astype(np.float32))
    assert got.dtype == np.float32 and np.all(np.abs(got - want) <= 2 * ulp)


@pytest.mark.parametrize("out_dtype", ["float32", "uint16"])
def test_identity_coefficients_fuse_bit_identically(ctx, tmp_path, out_dtype):
    # x size 44 (not a multiple of 8): the plain path stages whole views too, so both runs fuse with the same kernel
    xml, _ = planted_dataset(tmp_path, tile=(44, 40, 12), overlap=12)
    data = spimdata.SpimData2.load(xml)
    ident = {v: (np.ones((1, 2, 2)), np.zeros((1, 2, 2))) for v in data.view_ids()}   # 2 x 2 x 1 cells
    bint.write_coefficients(str(tmp_path / "id.n5"), "N5", "", "intensity", ident)
    outs = []
    for name, kw in (("a.n5", {}), ("b.n5", dict(intensity_n5_path=str(tmp_path / "id.n5")))):
        out = str(tmp_path / name)
        commands.create_fusion_container(xml, out, block_size=(32, 32, 16), dtype=out_dtype, min_intensity=0.0,
                                         max_intensity=2000.0)
        s0 = commands.affine_fusion(out, ctx, **kw)[0]
        outs.append(bn5.N5Store(out).read_volume(s0))
    assert np.array_equal(outs[0], outs[1]) and outs[0].any()


def test_planted_chain_end_to_end(ctx, tmp_path):
    xml, _ = planted_dataset(tmp_path, tile=(128, 128, 32), overlap=32)
    m = str(tmp_path / "matches.n5")
    got = commands.match_intensities(xml, ctx, m, num_coefficients=(4, 4, 2), render_scale=0.5)
    assert sum(len(c) for c in got.values()) >= 8
    co = commands.solve_intensities(xml, str(tmp_path / "coeff.n5"), m, num_coefficients=(4, 4, 2))
    data = spimdata.SpimData2.load(xml)
    views = data.view_ids()
    regs = {v: data.model(*v) for v in views}
    dims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in views}
    store = bn5.N5Store(str(tmp_path / "dataset.n5"))
    stored, corrected = {}, {}
    for v in views:
        stored[v] = store.read_volume(bn5.bdv_dataset(v[1], v[0], 0))
        h = ctx.volume_upload(stored[v])
        hc = ctx.intensity_apply(h, dims[v], np.eye(3, 4), *co[v])
        corrected[v] = ctx.volume_download(hc)
        ctx.volume_free(hc)
        ctx.volume_free(h)
    prs = bint.pairs(views, {v: bint.view_bounds(dims[v], regs[v]) for v in views})
    before = overlap_disagreement(stored, regs, dims, prs)
    after = overlap_disagreement(corrected, regs, dims, prs)
    assert after <= 0.25 * before, (before, after)
    out = str(tmp_path / "fused.n5")
    commands.create_fusion_container(xml, out, block_size=(64, 64, 32))
    s0 = commands.affine_fusion(out, ctx, intensity_n5_path=str(tmp_path / "coeff.n5"))[0]
    assert np.isfinite(bn5.N5Store(out).read_volume(s0)).all()


def test_no_planted_gain_gives_identity_coefficients(ctx, tmp_path):
    xml, _ = planted_dataset(tmp_path, tile=(128, 128, 32), overlap=32, gains=False)
    m = str(tmp_path / "matches.n5")
    got = commands.match_intensities(xml, ctx, m, num_coefficients=(4, 4, 2), render_scale=0.5)
    assert sum(len(c) for c in got.values()) > 0
    co = commands.solve_intensities(xml, str(tmp_path / "coeff.zarr"), m, num_coefficients=(4, 4, 2))
    for a, b in co.values():
        assert np.abs(a - 1.0).max() < 1e-9 and np.abs(b).max() < 1e-9
