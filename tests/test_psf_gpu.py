"""extract-psfs on the device: bs_psf_accumulate bit-identical to oracle/psf_oracle.py for uint8, uint16 and float32
windows, its argument errors, and the chain detect-interestpoints -> match-interestpoints -> extract-psfs on planted
beads."""
import ctypes as C

import numpy as np
import pytest

import bsgpu
from oracle import psf_oracle as po

pytestmark = pytest.mark.gpu

SIZE = (19, 19, 25)
DTYPES = {"u8": (np.uint8, 255), "u16": (np.uint16, 65535), "f32": (np.float32, None)}


def _volume(shape, kind, seed):
    dt, top = DTYPES[kind]
    rng = np.random.default_rng(seed)
    if top is None:
        return rng.normal(300.0, 900.0, shape).astype(np.float32)
    return rng.integers(0, top + 1, shape).astype(dt)


def _face_points(full, rng, n=60):
    """Points within h of every face (and beyond it), plus interior and integer ones."""
    full = np.asarray(full, dtype=np.float64)
    h = (np.array(SIZE) - 1) / 2
    pts = [rng.uniform(-1.0, full) for _ in range(n)]
    for d in range(3):
        for side in (0, 1):
            p = rng.uniform(0, full)
            p[d] = rng.uniform(0, h[d]) if side == 0 else full[d] - 1 - rng.uniform(0, h[d])
            pts.append(p)
    pts += [np.zeros(3), full - 1, np.floor(full / 2), np.array([-0.5, full[1] - 0.25, 3.75])]
    return np.array(pts)


@pytest.mark.parametrize("kind", sorted(DTYPES))
def test_whole_view_with_points_at_every_face_is_bit_identical(ctx, kind):
    vol = _volume((30, 41, 37), kind, 1)
    full = vol.shape[::-1]
    pts = _face_points(full, np.random.default_rng(2))
    h = ctx.volume_upload(vol)
    try:
        got = ctx.psf_accumulate(h, (0, 0, 0), full, pts, SIZE)
        one = ctx.psf_accumulate(h, (0, 0, 0), full, pts[:1], SIZE)
        none = ctx.psf_accumulate(h, (0, 0, 0), full, pts[:0], SIZE, np.full(SIZE[::-1], 7.5))
        split = ctx.psf_accumulate(h, (0, 0, 0), full, pts[:23], SIZE)
        ctx.psf_accumulate(h, (0, 0, 0), full, pts[23:], SIZE, split)
    finally:
        ctx.volume_free(h)
    assert np.array_equal(got, po.accumulate(vol, pts, SIZE))
    assert np.array_equal(one, po.accumulate(vol, pts[:1], SIZE))
    assert np.array_equal(none, np.full(SIZE[::-1], 7.5))
    assert np.array_equal(split, got)


@pytest.mark.parametrize("kind", sorted(DTYPES))
def test_window_away_from_the_origin_is_bit_identical(ctx, kind):
    from bsgpu import commands
    vol = _volume((60, 90, 80), kind, 3)
    full = vol.shape[::-1]
    rng = np.random.default_rng(4)
    pts = np.column_stack([rng.uniform(25, 55, 300), rng.uniform(30, 60, 300), rng.uniform(20, 40, 300)])
    pts[:3] = [(25.0, 30.0, 20.0), (54.99, 59.5, 39.75), (40.5, 45.0, 30.0)]
    (start, stop, wmin, wsize), = commands.psf_slabs(pts, SIZE, full, 1 << 30)
    assert (start, stop) == (0, len(pts)) and np.all(wmin > 0) and np.all(wmin + wsize < full)
    win = np.ascontiguousarray(vol[wmin[2]:wmin[2] + wsize[2], wmin[1]:wmin[1] + wsize[1], wmin[0]:wmin[0] + wsize[0]])
    h = ctx.volume_upload(win)
    try:
        got = ctx.psf_accumulate(h, wmin, full, pts, SIZE)
    finally:
        ctx.volume_free(h)
    assert np.array_equal(got, po.accumulate(vol, pts, SIZE))


def test_argument_errors_leave_the_context_working(ctx):
    lib = bsgpu.load_library()
    vol = _volume((10, 12, 14), "u16", 5)
    full = vol.shape[::-1]
    pts = np.array([[5.5, 6.0, 4.25]])
    h = ctx.volume_upload(vol)
    try:
        for size in ((4, 5, 5), (5, 2, 5), (5, 5, 8)):
            with pytest.raises(bsgpu.BsError):
                ctx.psf_accumulate(h, (0, 0, 0), full, pts, size)
        for wmin, fd in (((-1, 0, 0), full), ((1, 0, 0), full), ((0, 0, 0), (14, 12, 9))):
            with pytest.raises(bsgpu.BsError):
                ctx.psf_accumulate(h, wmin, fd, pts, (5, 5, 5))
        with pytest.raises(bsgpu.BsError):
            ctx.psf_accumulate(h + 12345, (0, 0, 0), full, pts, (5, 5, 5))
        s = np.zeros((5, 5, 5))
        dbl = C.POINTER(C.c_double)
        for n, size in ((-1, (5, 5, 5)), (1, (5, 5, 0)), (1, (-3, 5, 5)), (1, (5, -1, 5))):   # BS_ERR_ARG = -1
            rc = lib.bs_psf_accumulate(ctx.h, h, (C.c_longlong * 3)(0, 0, 0), (C.c_longlong * 3)(*full),
                                       pts.ctypes.data_as(dbl), n, (C.c_int * 3)(*size), s.ctypes.data_as(dbl))
            assert rc == -1, (n, size)
        assert np.all(s == 0)
        got = ctx.psf_accumulate(h, (0, 0, 0), full, pts, (5, 5, 5))
    finally:
        ctx.volume_free(h)
    assert np.array_equal(got, po.accumulate(vol, pts, (5, 5, 5)))


def _moments(psf, sigma):
    """sigma {x, y, z} of the PSF above its background (the median of the voxels beyond 4 sigma), over the box of
    3 sigma around the centre."""
    o = po.offsets(psf.shape[::-1]).reshape(psf.shape + (3,))
    r = np.sqrt(sum((o[..., d] / sigma[d]) ** 2 for d in range(3)))
    m = psf.astype(np.float64) - np.median(psf[r > 4])
    inner = np.all([np.abs(o[..., d]) <= round(3 * sigma[d]) for d in range(3)], axis=0)
    w = np.where(inner, m, 0.0)
    return np.array([np.sqrt((w * o[..., d] ** 2).sum() / w.sum()) for d in range(3)])


def test_chain_detect_match_extract(ctx, tmp_path):
    from bsgpu import commands, n5 as bn5, spimdata
    from bsgpu.commands import _InterestPoints, _psf_points
    from tests.test_interestpoints_gpu import _beads
    sigma = (2.0, 2.0, 2.5)
    rng = np.random.default_rng(11)
    gx, gy = np.meshgrid(np.arange(14.0, 195.0, 24.0), np.arange(14.0, 147.0, 24.0))   # jittered grid, >= 16 px apart
    world = np.column_stack([gx.ravel() + rng.uniform(-4, 4, gx.size), gy.ravel() + rng.uniform(-4, 4, gx.size),
                             rng.uniform(14, 34, gx.size)])
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles, vols = [], {}
    for s, t in enumerate((0.0, 64.0)):                     # the tiles overlap by 80 px in x
        local = world - (t, 0, 0)
        inside = local[(local[:, 0] > -8) & (local[:, 0] < 152)]
        vols[(0, s)] = _beads((48, 160, 144), [tuple(p) for p in inside], 20 + s, sigma_xy=sigma[0], sigma_z=sigma[2])
        bn5.write_bdv_setup(store, s, 0, vols[(0, s)], (64, 64, 16))
        tiles.append(dict(setup=s, size_xyz=(144, 160, 48), tile=s, translation_xyz=(t + (1.5 if s else 0.0), 0, 0)))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    commands.detect_interestpoints(xml, ctx, "beads", sigma=2.0, threshold=0.01, min_intensity=0.0,
                                   max_intensity=1000.0, downsample_xy=1, block_size=(64, 64, 24))
    res = commands.match_interestpoints(xml, ctx, ["beads"], "PRECISE_TRANSLATION", ransac_min_num_inliers=8,
                                        transformation_model="TRANSLATION", regularization_model="NONE")
    assert len(res) == 1 and all(len(p) >= 8 for p in res.values()), {k: len(v) for k, v in res.items()}
    got = commands.extract_psfs(xml, ctx, "beads")
    data = spimdata.SpimData2.load(xml)
    assert data.point_spread_functions() == {(0, 0): "psf_t0_vs0.tif", (0, 1): "psf_t0_vs1.tif"}
    views = data.view_ids()
    ips = _InterestPoints(bn5.N5Store(str(tmp_path / "interestpoints.n5")), views, ["beads"],
                          {v: data.model(*v) for v in views}, tables=True)
    for v in views:
        _, loc = _psf_points(ips, v, "beads", False)
        psf, n = got[v]
        assert n == len(loc) >= 8
        assert np.array_equal(psf, po.extract(vols[v], loc, SIZE))
        assert np.unravel_index(psf.argmax(), psf.shape) == tuple((s - 1) // 2 for s in SIZE[::-1])
        meas = _moments(psf, sigma)
        o = po.offsets(SIZE).reshape(SIZE[::-1] + (3,))
        ideal = 1000.0 * np.exp(-sum(o[..., d] ** 2 / (2 * sigma[d] ** 2) for d in range(3)))
        want = _moments(ideal, sigma)                      # the same truncated box on the planted Gaussian
        assert np.all(np.abs(meas / want - 1) <= 0.10), (meas, want)
