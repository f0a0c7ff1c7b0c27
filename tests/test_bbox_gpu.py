"""estimate-bounding-box on the device: bs_min_filter, bs_volume_min_max and bs_threshold_bbox against the oracle, the
command's device fusion against the fusion oracle, and the chain estimate -> create-fusion-container -b ->
affine-fusion."""
import numpy as np
import pytest

import bsgpu
from bsgpu import commands, fusion, n5 as bn5, spimdata
from oracle import bbox_oracle as bo
from oracle import fusion_oracle as fo
from tests import test_fusion_gpu
from tests.test_bbox_cpu import BEADS, bbox_scene

pytestmark = pytest.mark.gpu

SHAPE = (37, 45, 70)            # [z, y, x]: no axis a multiple of the kernels' 128 / 64 / 32 tiles


def _volume(seed, shape=SHAPE, nans=0):
    rng = np.random.default_rng(seed)
    v = rng.normal(0.0, 100.0, shape).astype(np.float32)
    for _ in range(nans):
        v[tuple(int(rng.integers(0, s)) for s in shape)] = np.nan
    return v


@pytest.mark.parametrize("r", [1, 3, 6, 17, 100, (0, 2, 5), (70, 1, 40)])
def test_min_filter_is_bit_identical_to_the_oracle(ctx, r):
    v = _volume(11, nans=5)
    h = ctx.volume_upload(v)
    try:
        g = ctx.min_filter(h, (r,) * 3 if np.isscalar(r) else r)
        got = ctx.volume_download(g)
        ctx.volume_free(g)
    finally:
        ctx.volume_free(h)
    want = bo.min_filter(v, r)
    assert got.tobytes() == want.tobytes()


def test_min_filter_on_thin_and_all_nan_volumes(ctx):
    for v in (_volume(3, (1, 9, 300)), _volume(4, (130, 1, 1))):
        h = ctx.volume_upload(v)
        g = ctx.min_filter(h, (3, 3, 3))
        assert ctx.volume_download(g).tobytes() == bo.min_filter(v, 3).tobytes()
        for x in (g, h):
            ctx.volume_free(x)
    v = np.full((3, 4, 5), np.nan, np.float32)       # a box of NaNs only gives NaN (the payload is not specified)
    v[2, 3, 4] = 7.0
    h = ctx.volume_upload(v)
    g = ctx.min_filter(h, (1, 1, 1))
    got, want = ctx.volume_download(g), bo.min_filter(v, 1)
    for x in (g, h):
        ctx.volume_free(x)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(want).any()
    assert got[~np.isnan(got)].tobytes() == want[~np.isnan(want)].tobytes()


def test_min_max_and_threshold_bbox_match_numpy(ctx):
    v = _volume(7, nans=3)
    h = ctx.volume_upload(v)
    try:
        mn, mx = ctx.volume_min_max(h)
        assert (mn, mx) == (float(np.nanmin(v)), float(np.nanmax(v)))
        for t in (mn, 0.0, 250.0, float(v[5, 6, 7]), float(np.nextafter(np.float32(mx), np.float32(0))), mx, np.inf):
            assert ctx.threshold_bbox(h, t) == bo.threshold_bbox(v, t), t
        assert ctx.threshold_bbox(h, mx) == ((-1, -1, -1), (-1, -1, -1), 0)
    finally:
        ctx.volume_free(h)
    h = ctx.volume_upload(np.full((2, 3, 4), np.nan, np.float32))
    assert all(np.isnan(x) for x in ctx.volume_min_max(h))
    ctx.volume_free(h)


def test_bad_arguments_raise_and_the_context_stays_usable(ctx):
    v = _volume(5)
    h = ctx.volume_upload(v)
    hu = ctx.volume_upload(np.ones((4, 5, 6), np.uint16))
    try:
        for call in (lambda: ctx.min_filter(h, (1, -1, 1)), lambda: ctx.min_filter(hu, (1, 1, 1)),
                     lambda: ctx.min_filter(987654321, (1, 1, 1)), lambda: ctx.volume_min_max(hu),
                     lambda: ctx.volume_min_max(987654321), lambda: ctx.threshold_bbox(hu, 0.0),
                     lambda: ctx.threshold_bbox(987654321, 0.0)):
            with pytest.raises(bsgpu.BsError) as e:
                call()
            assert e.value.code == -1
        g = ctx.min_filter(h, (2, 2, 2))
        assert ctx.volume_download(g).tobytes() == bo.min_filter(v, 2).tobytes()
        ctx.volume_free(g)
    finally:
        ctx.volume_free(h)
        ctx.volume_free(hu)


def test_command_fusion_and_box_match_the_oracles(ctx, tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    ds, size = 2, 8
    d = spimdata.SpimData2.load(xml)
    src = commands.bvs.open_views(d)
    lo, hi = (b.astype(np.int64) for b in commands.views_bounding_box(d, d.view_ids()))
    g_min, dims = commands.bounding_box_grid(lo, hi, ds)
    h, buf = ctx.volume_empty(dims)
    try:
        commands.fuse_downsampled(ctx, d, src, d.view_ids(), ds, g_min, dims, buf)
        got = ctx.volume_download(h)
    finally:
        ctx.volume_free(h)
    regs = fusion.adjust_all_transforms({v: d.model(*v) for v in d.view_ids()}, downsampling=float(ds))
    views = []
    for v in d.view_ids():
        border, rng = fusion.adjust_blending(regs[v])
        views.append(fo.View(src.read_volume(v, 0), regs[v], border, rng))
    bmin, bsize = tuple(int(x) for x in g_min), tuple(int(x) for x in dims)
    want = fo.fuse_block(views, bmin, bsize, fo.AVG_BLEND)
    test_fusion_gpu._run.last = (views, bmin, bsize)
    test_fusion_gpu._assert_close(got, want)

    res = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=ds, discarded_object_size=size)
    exp = bo.estimate(got, lo, hi, ds, 5.0, size)
    assert {k: res[k] for k in exp} == exp
    assert res["dims"] == [int(x) for x in dims] and res["count"] > 0
    for b in BEADS:
        assert not all(res["min"][k] <= b[k] <= res["max"][k] for k in range(3)), b
    assert [b.tolist() for b in spimdata.SpimData2.load(xml).bounding_boxes()["auto"]] == [res["min"], res["max"]]


def test_estimate_then_fuse_the_box_on_the_device(ctx, tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    full = str(tmp_path / "full.n5")
    commands.create_fusion_container(xml, full, block_size=(32, 32, 16))
    commands.affine_fusion(full, ctx)
    res = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=2, discarded_object_size=8)
    box = str(tmp_path / "box.n5")
    commands.create_fusion_container(xml, box, bounding_box="auto", block_size=(32, 32, 16))
    commands.affine_fusion(box, ctx)
    f = bn5.N5Store(full).read_volume("ch0tp0/s0")
    b = bn5.N5Store(box).read_volume("ch0tp0/s0")
    (x0, y0, z0), (x1, y1, z1) = res["min"], res["max"]
    assert b.shape == (z1 - z0 + 1, y1 - y0 + 1, x1 - x0 + 1)
    # the full box starts at world 0.  The box's blocks are anchored at its own minimum, so the float coordinate of a
    # voxel may round differently in the last bit than in the full fusion (bit-identical when the box is on the
    # full fusion's block grid, tests/test_fusion_container_gpu.py)
    np.testing.assert_allclose(b, f[z0:z1 + 1, y0:y1 + 1, x0:x1 + 1], rtol=1e-6, atol=0)
    assert b.min() > 500.0
