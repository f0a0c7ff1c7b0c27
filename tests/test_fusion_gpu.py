"""GPU parity tests, hot path 2: libbsgpu fusion (through the C ABI) against
oracle/fusion_oracle.py.  Bar: float32 voxels within 1e-4 relative (north_star); integer
outputs within 1 grey level where the float result sits on a rounding boundary."""
import numpy as np
import pytest

import bsgpu
from oracle import fusion_oracle as fo
from tests import synth

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _scene(seed=0, n=3, shape=(40, 48, 56), dtype=np.uint16, rot=0.0, jitter=True):
    """n overlapping tiles along x (and a little y/z) cut from one field."""
    rng = np.random.default_rng(seed)
    G = synth.field((shape[0] + 40, shape[1] + 40, shape[2] * n + 40), seed=seed, sigma=1.5)
    views = []
    for i in range(n):
        off = np.array([i * (shape[2] - 14), 3 * i, 2 * i], dtype=np.float64)  # xyz
        vol = synth.tile_from(G, (int(off[2]), int(off[1]), int(off[0])), shape, seed * 10 + i, noise=5.0, dtype=dtype)
        t = off + (rng.uniform(-2, 2, 3) if jitter else 0.0)
        M = synth.translation(t)
        if rot:
            R = synth.rot_z(rot, center_xyz=(shape[2] / 2, shape[1] / 2, 0))
            M = (np.vstack([M, [0, 0, 0, 1]]) @ np.vstack([R, [0, 0, 0, 1]]))[:3]
        views.append((vol, M))
    return views


def _run(ctx, views, bmin, bsize, fusion_type, out_dtype="float32", interpolation=1, lut=0,
         min_i=0.0, max_i=65535.0, contents=None, content_sigmas=(2.0, 4.0)):
    import bsgpu
    nat = bsgpu.native
    handles = [ctx.volume_upload(v) for v, _ in views]
    chandles = [0] * len(views)
    ov = []
    gv = []
    for i, (vol, M) in enumerate(views):
        border, rng = fo.adjust_blending(M)
        c = None
        if fusion_type in (fo.AVG_CONTENT, fo.AVG_BLEND_CONTENT):
            chandles[i] = ctx.content_weights(handles[i], *content_sigmas)
            c = fo.content_weights(vol, *content_sigmas)
        ov.append(fo.View(vol, M, border, rng, c))
        gv.append(dict(src_to_world=M, vol_handle=handles[i], content_handle=chandles[i],
                       blend_border=border, blend_range=rng))
    od = {"float32": nat.DTYPE_F32, "uint16": nat.DTYPE_U16, "uint8": nat.DTYPE_U8}[out_dtype]
    p = ctx.fuse_params(fusion_type, interpolation, od, lut, min_i, max_i)
    got = ctx.fuse_block(gv, bmin, bsize, p)
    want = fo.fuse_block(ov, bmin, bsize, fusion_type, interpolation, out_dtype, min_i, max_i, lut)
    for h in handles + [c for c in chandles if c]:
        ctx.volume_free(h)
    _run.last = (ov, bmin, bsize)
    return got, want


def _near_view_face(idx_zyx, tol=2e-3):
    """True when the output voxel maps to within ``tol`` px of a face of some view: the only
    place where the (discontinuous) inside / dist==0 tests may legitimately flip between two
    correct float evaluations of the same affine."""
    ov, bmin, bsize = _run.last
    w = np.array([bmin[0] + idx_zyx[2], bmin[1] + idx_zyx[1], bmin[2] + idx_zyx[0]], dtype=np.float64)
    for v in ov:
        inv = fo.invert_affine(v.src_to_world)
        s = inv[:, :3] @ w + inv[:, 3]
        dims = np.array(v.img.shape[::-1], dtype=np.float64)
        if np.all(s > -1 - tol) and np.all(s < dims + tol) and \
                (np.any(np.abs(s) < tol) or np.any(np.abs(s - (dims - 1)) < tol)):
            return True
    return False


def _assert_close(got, want, rtol=RTOL):
    assert got.shape == want.shape and got.dtype == want.dtype
    if got.dtype == np.float32:
        # relative to the voxel's own value, floored at a quarter of the image's typical intensity: the n-linear
        # interpolation error scales with the local gradient (a 3e-5 px coordinate rounding times ~150 grey
        # levels per px), not with the value, so "1e-4 relative" is only meaningful for voxels that are not
        # close to zero (synthetic fields clip their 3-sigma tail at 0; real camera data has an offset)
        nz = np.abs(want[want != 0])
        floor = 0.25 * float(nz.mean()) if nz.size else 1.0
        denom = np.maximum(np.abs(want), max(floor, 1.0))
        err = np.abs(got - want) / denom
        bad = np.argwhere(err > rtol)
        assert len(bad) <= 1e-3 * got.size + 2, f"{len(bad)} voxels beyond rtol, max {err.max()}"
        for idx in bad:
            # (a) on a face the inside / dist == 0 tests may flip; (b) within ~1.5 px of a face of EVERY
            # contributing view the blending weights are 1e-6..1e-3 and sum(w I) / sum(w) amplifies the
            # 3e-5 px float rounding of the source coordinate (2 dw/w = 2 * 3e-5 / dist): bounded at 3e-3 there
            e = err[tuple(idx)]
            assert _near_view_face(tuple(idx)) or (e < 3e-3 and _near_view_face(tuple(idx), tol=1.5)), \
                f"rel err {e} at {tuple(idx)} away from any view face"
    else:
        d = np.abs(got.astype(np.int64) - want.astype(np.int64))
        # one grey level at most, and only where the float result sits within ~1e-7 rel of a rounding
        # boundary (with a converter gain of 65 levels per unit that is < 2 % of the voxels)
        assert d.max() <= 1 and (d > 0).mean() < 2e-2


@pytest.mark.parametrize("ft", [fo.AVG, fo.AVG_BLEND, fo.MAX_INTENSITY, fo.LOWEST_VIEWID_WINS,
                                fo.HIGHEST_VIEWID_WINS, fo.CLOSEST_PIXEL_WINS])
def test_fusion_types_translation(ctx, ft):
    views = _scene(seed=1)
    got, want = _run(ctx, views, (-3, -2, -1), (150, 60, 47), ft)
    _assert_close(got, want)
    assert np.count_nonzero(want) > 0.5 * want.size


def test_avg_blend_rotated_views(ctx):
    views = _scene(seed=2, rot=0.5)
    got, want = _run(ctx, views, (0, 0, 0), (140, 50, 40), fo.AVG_BLEND)
    _assert_close(got, want)


def test_avg_blend_anisotropic_scale(ctx):
    views = _scene(seed=3, n=2)
    S = np.diag([1.0, 1.0, 2.5, 1.0])
    views = [(v, (S @ np.vstack([M, [0, 0, 0, 1]]))[:3]) for v, M in views]
    got, want = _run(ctx, views, (0, 0, 0), (100, 50, 100), fo.AVG_BLEND)
    _assert_close(got, want)


@pytest.mark.parametrize("ft", [fo.AVG_CONTENT, fo.AVG_BLEND_CONTENT])
@pytest.mark.parametrize("sigmas", [(2.0, 4.0), (20.0, 40.0)])      # small, and upstream's defaults (north_star bar 1e-4)
def test_content_based(ctx, ft, sigmas):
    views = _scene(seed=4, n=2)
    got, want = _run(ctx, views, (0, 0, 0), (100, 50, 40), ft, content_sigmas=sigmas)
    _assert_close(got, want)


def test_content_weight_volume(ctx):
    vol = synth.tile_from(synth.field((40, 44, 52), seed=5), (0, 0, 0), (40, 44, 52), 5)
    h = ctx.volume_upload(vol)
    c = ctx.content_weights(h, 2.0, 4.0)
    got = ctx.volume_download(c, vol.shape[::-1])
    want = fo.content_weights(vol, 2.0, 4.0)
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max()
    ctx.volume_free(h)
    ctx.volume_free(c)


def test_blend_lut_mode(ctx):
    views = _scene(seed=6)
    got, want = _run(ctx, views, (0, 0, 0), (150, 50, 40), fo.AVG_BLEND, lut=30)
    _assert_close(got, want)


def test_nearest_neighbour(ctx):
    views = _scene(seed=7, jitter=False)
    got, want = _run(ctx, views, (0, 0, 0), (120, 50, 40), fo.AVG_BLEND, interpolation=0)
    _assert_close(got, want)


@pytest.mark.parametrize("out_dtype,mn,mx", [("uint16", 0.0, 65535.0), ("uint8", 200.0, 1800.0), ("uint16", 500.0, 1500.0)])
def test_integer_outputs(ctx, out_dtype, mn, mx):
    views = _scene(seed=8)
    got, want = _run(ctx, views, (0, 0, 0), (150, 50, 40), fo.AVG_BLEND, out_dtype=out_dtype, min_i=mn, max_i=mx)
    _assert_close(got, want)


def test_float_and_u8_sources(ctx):
    views = _scene(seed=9, dtype=np.float32)
    got, want = _run(ctx, views, (0, 0, 0), (150, 50, 40), fo.AVG_BLEND)
    _assert_close(got, want)
    v8 = [((v / 8).astype(np.uint8), M) for v, M in _scene(seed=9)]
    got, want = _run(ctx, v8, (0, 0, 0), (150, 50, 40), fo.AVG)
    _assert_close(got, want)


def test_single_view_identity_is_input(ctx):
    vol = synth.tile_from(synth.field((32, 40, 48), seed=10), (0, 0, 0), (32, 40, 48), 10)
    got, want = _run(ctx, [(vol, synth.translation((0, 0, 0)))], (0, 0, 0), (48, 40, 32), fo.AVG)
    assert np.array_equal(got, vol.astype(np.float32))
    _assert_close(got, want)


def test_block_seam_invariance(ctx):
    """Fusing 4 sub-blocks must be bit-identical to fusing the whole block at once."""
    import bsgpu
    views = _scene(seed=11)
    handles = [ctx.volume_upload(v) for v, _ in views]
    gv = []
    for (vol, M), h in zip(views, handles):
        border, rng = fo.adjust_blending(M)
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    whole = ctx.fuse_block(gv, (0, 0, 0), (128, 48, 40))
    parts = np.zeros_like(whole)
    for ox in (0, 64):
        for oy in (0, 24):
            parts[:, oy:oy + 24, ox:ox + 64] = ctx.fuse_block(gv, (ox, oy, 0), (64, 24, 40))
    assert np.array_equal(whole, parts)
    for h in handles:
        ctx.volume_free(h)


def test_empty_views_and_outside_block(ctx):
    views = _scene(seed=12, n=1)
    got, want = _run(ctx, views, (5000, 5000, 5000), (33, 17, 9), fo.AVG_BLEND)
    assert not got.any() and not want.any()
    out = ctx.fuse_block([], (0, 0, 0), (16, 8, 4))
    assert out.shape == (4, 8, 16) and not out.any()


def test_many_views_chunked_culling(ctx):
    """> 256 views exercises the chunked per-CTA culling."""
    vol = synth.tile_from(synth.field((16, 16, 16), seed=13), (0, 0, 0), (16, 16, 16), 13)
    views = [(vol, synth.translation((10 * (i % 20), 10 * ((i // 20) % 15), 0))) for i in range(300)]
    got, want = _run(ctx, views, (0, 0, 0), (210, 160, 16), fo.AVG_BLEND)
    _assert_close(got, want)


def test_view_sharded_accumulate_equals_gather(ctx):
    """SURVEY 8e scatter mode: partial sums over view subsets, summed, then finished ==
    single-pass fusion up to float re-association."""
    import torch
    views = _scene(seed=14)
    handles = [ctx.volume_upload(v) for v, _ in views]
    gv = []
    for (vol, M), h in zip(views, handles):
        border, rng = fo.adjust_blending(M)
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    bmin, bsz = (0, 0, 0), (150, 50, 40)
    p = ctx.fuse_params(fo.AVG_BLEND)
    whole = ctx.fuse_block(gv, bmin, bsz, p)
    n = 150 * 50 * 40
    swi = torch.zeros(n, dtype=torch.float32, device="cuda")
    sw = torch.zeros(n, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.fuse_accumulate(gv[:1], bmin, bsz, p, swi, sw)
    ctx.fuse_accumulate(gv[1:], bmin, bsz, p, swi, sw)
    out = np.empty((40, 50, 150), np.float32)
    ctx.fuse_finish(swi, sw, n, p, out)
    _assert_close(out, whole, rtol=1e-5)
    for h in handles:
        ctx.volume_free(h)


def test_bad_arguments(ctx):
    import bsgpu
    with pytest.raises(bsgpu.BsError):
        ctx.fuse_block([dict(src_to_world=np.eye(3, 4), vol_handle=987654)], (0, 0, 0), (4, 4, 4))
    vol = np.zeros((4, 4, 4), np.uint16)
    h = ctx.volume_upload(vol)
    with pytest.raises(bsgpu.BsError):
        ctx.fuse_block([dict(src_to_world=np.zeros((3, 4)), vol_handle=h)], (0, 0, 0), (4, 4, 4))
    with pytest.raises(bsgpu.BsError):
        ctx.fuse_block([dict(src_to_world=np.eye(3, 4), vol_handle=h)], (0, 0, 0), (4, 4, 4),
                       ctx.fuse_params(fusion_type=99))
    ctx.volume_free(h)


@pytest.mark.parametrize("dtype", [np.uint16, np.float32, np.uint8])
@pytest.mark.parametrize("factors", [(2, 2, 1), (2, 2, 2), (1, 1, 2)])
def test_device_pyramid_step_bit_exact(ctx, dtype, factors):
    rng = np.random.default_rng(3)
    vol = (rng.random((21, 34, 45)) * 250).astype(dtype)
    h = ctx.volume_upload(vol)
    h2 = ctx.downsample(h, factors)
    want = fo.downsample2x(vol, factors)
    got = ctx.volume_download(h2, want.shape[::-1], dtype)
    assert np.array_equal(got, want)
    ctx.volume_free(h)
    ctx.volume_free(h2)


# ---- the code paths bench.py runs (BASELINE configs[2]): big tiles, so that whole output tiles lie on the
# blending plateau / strictly inside one view (single-view fast path), next to multi-view blend zones.
def _run_c(ctx, views, bmin, bsize, fusion_type=fo.AVG_BLEND):
    """GPU block vs the C/OpenMP oracle (oracle/c_fusion, itself checked against the numpy oracle)."""
    from oracle import c_fusion
    handles = [ctx.volume_upload(v) for v, _ in views]
    ov, gv = [], []
    for (vol, M), h in zip(views, handles):
        border, rng = fo.adjust_blending(M)
        ov.append(fo.View(vol, M, border, rng, None))
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    got = ctx.fuse_block(gv, bmin, bsize, ctx.fuse_params(fusion_type))
    want = c_fusion.fuse_block(ov, bmin, bsize, fusion_type)
    for h in handles:
        ctx.volume_free(h)
    _run.last = (ov, bmin, bsize)
    return got, want


def _sparse_tile(shape_zyx, region_zyx, seed):
    """uint16 tile that is zero except for a smooth random sub-region (keeps 576^3 tiles cheap)."""
    from scipy.ndimage import gaussian_filter
    vol = np.zeros(shape_zyx, np.uint16)
    sl = tuple(slice(max(0, a), min(s, b)) for (a, b), s in zip(region_zyx, shape_zyx))
    shp = tuple(s.stop - s.start for s in sl)
    rng = np.random.default_rng(seed)
    g = gaussian_filter(rng.standard_normal(shp).astype(np.float32), 1.5)
    vol[sl] = np.clip(np.rint(g / g.std() * 300 + 2000), 0, 65535).astype(np.uint16)   # > 6 sigma above 0: the relative bar is meaningful
    return vol


@pytest.mark.parametrize("rot", [0.0, 0.5])
def test_large_tiles_all_fast_paths(ctx, rot):
    shape = (160, 168, 176)
    views = _scene(seed=21, n=2, shape=shape, rot=rot)
    got, want = _run_c(ctx, views, (-4, -3, -2), (344, 180, 168))
    _assert_close(got, want)
    assert np.count_nonzero(want) > 0.7 * want.size


@pytest.mark.parametrize("rot", [0.0, 0.5])
def test_config3_superblock_576_tiles(ctx, rot):
    """One real BASELINE configs[2] task: a 256x256x128 super-block at the junction of eight 576^3 tiles
    (stride 491, jitter in [-2,2]^3), float32 AVG_BLEND, against the C oracle at 1e-4."""
    tile, stride = 576, 491
    bmin, bsize = (384, 384, 448), (256, 256, 128)
    rng = np.random.default_rng(7)
    a = np.deg2rad(rot)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    views = []
    for k in range(2):
        for j in range(2):
            for i in range(2):
                t = stride * np.array([i, j, k], dtype=np.float64) + rng.uniform(-2, 2, 3)
                c = np.array([tile / 2, tile / 2, 0.0])
                M = np.hstack([R, (t + c - R @ c)[:, None]])
                # source region the block can touch (+ margin), in this tile's pixel coordinates
                lo = np.array(bmin) - t - 12
                hi = np.array(bmin) + np.array(bsize) - t + 12
                region = [(int(lo[d]), int(hi[d])) for d in (2, 1, 0)]
                views.append((_sparse_tile((tile,) * 3, region, 100 + 4 * k + 2 * j + i), M))
    got, want = _run_c(ctx, views, bmin, bsize)
    _assert_close(got, want)
    assert np.count_nonzero(want) > 0.9 * want.size


def test_windowed_views_equal_full_views(ctx):
    """Block-wise source staging (SURVEY a11): uploading only the sub-interval of each view that the block touches
    (full_dims / window_min) gives bit-identical voxels to fusing from the whole views."""
    shape = (96, 104, 176)
    views = _scene(seed=31, n=2, shape=shape)
    bmin, bsize = (150, 10, 20), (90, 80, 50)
    full_h = [ctx.volume_upload(v) for v, _ in views]
    gv_full, gv_win, win_h = [], [], []
    for (vol, M), h in zip(views, full_h):
        border, rng = fo.adjust_blending(M)
        gv_full.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
        inv = fo.invert_affine(M)
        lo = inv[:, :3] @ np.array(bmin, float) + inv[:, 3]
        hi = inv[:, :3] @ (np.array(bmin, float) + np.array(bsize) - 1) + inv[:, 3]
        dims = np.array(vol.shape[::-1])
        w0 = np.clip(np.floor(np.minimum(lo, hi)).astype(int) - 1, 0, dims - 1)
        w1 = np.clip(np.floor(np.maximum(lo, hi)).astype(int) + 2, 0, dims - 1)
        w0[0] &= ~7                                          # keep the window's x size / offset TMA friendly
        w1[0] = min(dims[0] - 1, (w1[0] | 7))
        sub = np.ascontiguousarray(vol[w0[2]:w1[2] + 1, w0[1]:w1[1] + 1, w0[0]:w1[0] + 1])
        assert sub.shape[2] % 8 == 0
        hw = ctx.volume_upload(sub)
        win_h.append(hw)
        gv_win.append(dict(src_to_world=M, vol_handle=hw, blend_border=border, blend_range=rng,
                           full_dims=tuple(int(d) for d in dims), window_min=tuple(int(v) for v in w0)))
    a = ctx.fuse_block(gv_full, bmin, bsize)
    b = ctx.fuse_block(gv_win, bmin, bsize)
    assert np.count_nonzero(a) > 0.5 * a.size
    assert np.array_equal(a, b)
    # the same through the rotated (general) kernel
    R = synth.rot_z(0.4, center_xyz=(80, 50, 0))
    for g in gv_full + gv_win:
        g["src_to_world"] = (np.vstack([R, [0, 0, 0, 1]]) @ np.vstack([g["src_to_world"], [0, 0, 0, 1]]))[:3]
    # (windows were sized for the unrotated block footprint; shrink the block so they still cover it)
    a = ctx.fuse_block(gv_full, (160, 20, 24), (60, 50, 40))
    b = ctx.fuse_block(gv_win, (160, 20, 24), (60, 50, 40))
    assert np.array_equal(a, b)
    for h in full_h + win_h:
        ctx.volume_free(h)


def test_fuse_blocks_list_equals_single_calls(ctx):
    views = _scene(seed=32, n=3, shape=(48, 64, 72))
    handles = [ctx.volume_upload(v) for v, _ in views]
    gv = []
    for (vol, M), h in zip(views, handles):
        border, rng = fo.adjust_blending(M)
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    mins = [(0, 0, 0), (64, 0, 0), (0, 32, 8), (100, 20, 30), (5000, 0, 0)]
    sizes = [(64, 32, 24), (70, 40, 17), (33, 31, 9), (64, 16, 8), (16, 16, 8)]
    many = ctx.fuse_blocks(gv, mins, sizes)
    for mn, sz, got in zip(mins, sizes, many):
        assert np.array_equal(got, ctx.fuse_block(gv, mn, sz))
    assert not many[-1].any()
    for h in handles:
        ctx.volume_free(h)


def test_oblique_rotation_uses_the_fully_general_kernel(ctx):
    """A rotation about x couples y and z: no translation and no xy-affine structure, every voxel samples 8 taps."""
    views = _scene(seed=33, n=2, shape=(72, 80, 96))
    R = synth.rot_x(0.7, center_xyz=(0, 40, 36))
    views = [(v, (np.vstack([R, [0, 0, 0, 1]]) @ np.vstack([M, [0, 0, 0, 1]]))[:3]) for v, M in views]
    got, want = _run_c(ctx, views, (-3, -2, -1), (190, 84, 76))
    _assert_close(got, want)
    assert np.count_nonzero(want) > 0.6 * want.size


def test_xy_affine_path_equals_generic_path(ctx):
    """Rotation about z + xy scale: the z-marching xy-affine tiles and the per-voxel generic tiles agree to rounding."""
    views = _scene(seed=34, n=3, shape=(72, 80, 96), rot=0.5)
    S = np.diag([1.01, 0.99, 1.0, 1.0])
    views = [(v, (S @ np.vstack([M, [0, 0, 0, 1]]))[:3]) for v, M in views]
    # xy-affine tiles run only when EVERY view of the call is xy-affine: a uint16 view (x size a multiple of 8, so
    # the call stays on the TMA kernels) rotated about x and placed far outside the block is culled from every tile
    # but sends the whole call to the per-voxel tiles
    far = synth.translation((5000.0, 5000.0, 5000.0))
    far = (np.vstack([far, [0, 0, 0, 1]]) @ np.vstack([synth.rot_x(0.7, center_xyz=(0, 8, 8)), [0, 0, 0, 1]]))[:3]
    handles = [ctx.volume_upload(v) for v, _ in views] + [ctx.volume_upload(np.ones((16, 16, 16), np.uint16))]
    gv = []
    for M, h in zip([M for _, M in views] + [far], handles):
        border, rng = fo.adjust_blending(M)
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    a = ctx.fuse_block(gv[:-1], (0, 0, 0), (250, 80, 72))
    b = ctx.fuse_block(gv, (0, 0, 0), (250, 80, 72))
    assert np.count_nonzero(a) > 0.6 * a.size
    err = np.abs(a - b) / np.maximum(np.abs(b), 250.0)
    assert err.max() < 2e-5
    for h in handles:
        ctx.volume_free(h)


@pytest.mark.parametrize("out_dtype", ["float32", "uint16", "uint8"])
@pytest.mark.parametrize("ft,rot", [("AVG_BLEND", 0.0), ("AVG_BLEND", 0.4), ("MAX_INTENSITY", 0.0)])
def test_big_endian_output_is_the_byte_swapped_block(ctx, out_dtype, ft, rot):
    """bs_fuse_params.out_big_endian: the block leaves the device as an N5 payload (translation kernel, general
    kernel and the generic tile kernel + swap pass), odd sizes so the scalar and the paired stores both run."""
    views = _scene(seed=35, n=3, shape=(40, 48, 56), rot=rot)
    handles = [ctx.volume_upload(v) for v, _ in views]
    gv = []
    for (vol, M), h in zip(views, handles):
        border, rng = fo.adjust_blending(M)
        gv.append(dict(src_to_world=M, vol_handle=h, blend_border=border, blend_range=rng))
    dt = {"float32": bsgpu.native.DTYPE_F32, "uint16": bsgpu.native.DTYPE_U16, "uint8": bsgpu.native.DTYPE_U8}[out_dtype]
    mins, sizes = [(1, 0, 0), (40, 3, 2)], [(71, 33, 17), (64, 16, 8)]
    le = ctx.fuse_blocks(gv, mins, sizes, ctx.fuse_params(ft, 1, dt, 0, 0.0, 4000.0))
    be = ctx.fuse_blocks(gv, mins, sizes, ctx.fuse_params(ft, 1, dt, 0, 0.0, 4000.0, out_big_endian=True))
    for a, b in zip(le, be):
        assert a.any()
        assert b.dtype.byteorder in (">", "|") and np.array_equal(a, b.astype(a.dtype))
        assert a.tobytes() == b.byteswap().tobytes()
    for h in handles:
        ctx.volume_free(h)


@pytest.mark.parametrize("out_dtype", ["uint8", "uint16", "float32"])
def test_masks_mode_matches_oracle(ctx, out_dtype):
    """bs_mask_blocks (--masks): bit-identical to the oracle, geometry only (no volumes), rotated and scaled views,
    mask offset, big-endian payloads, more views than one kernel-parameter group."""
    dt = {"float32": bsgpu.native.DTYPE_F32, "uint16": bsgpu.native.DTYPE_U16, "uint8": bsgpu.native.DTYPE_U8}[out_dtype]
    geom = [(synth.translation((2.0, 0.0, 0.0)), (40, 30, 20)),
            (np.vstack([synth.rot_z(7.0, center_xyz=(20, 15, 0)), [0, 0, 0, 1]]) @ np.vstack([synth.translation((35.25, 4.5, 3.0)), [0, 0, 0, 1]]), (40, 30, 20)),
            (np.diag([1.0, 1.0, 2.5, 1.0]) @ np.vstack([synth.translation((10.0, 28.0, 1.0)), [0, 0, 0, 1]]), (30, 20, 8))]
    geom = [(np.asarray(M)[:3], d) for M, d in geom]
    views = [dict(src_to_world=M, vol_handle=0, full_dims=d) for M, d in geom]
    mins, sizes = [(-3, -2, -1), (30, 10, 5)], [(90, 60, 30), (33, 17, 9)]
    for off in ((0.0, 0.0, 0.0), (1.5, 0.0, -0.5)):
        got = ctx.mask_blocks(views, mins, sizes, off, dt)
        be = ctx.mask_blocks(views, mins, sizes, off, dt, out_big_endian=True)
        for mn, sz, g, b in zip(mins, sizes, got, be):
            want = fo.mask_block(geom, mn, sz, off, out_dtype)
            assert np.array_equal(g, want) and np.count_nonzero(want) > 0
            assert sz != sizes[0] or np.count_nonzero(want) < want.size       # the big block has uncovered voxels
            assert np.array_equal(b.astype(g.dtype), g)
    many = [dict(src_to_world=synth.translation((3.0 * i, 0.0, 0.0)), vol_handle=0, full_dims=(2, 4, 4)) for i in range(70)]
    g = ctx.mask_blocks(many, [(0, 0, 0)], [(220, 4, 4)], (0, 0, 0), dt)[0]
    want = fo.mask_block([(v["src_to_world"], v["full_dims"]) for v in many], (0, 0, 0), (220, 4, 4), (0, 0, 0), out_dtype)
    assert np.array_equal(g, want) and g[0, 0, 208] > 0 and g[0, 0, 209] == 0
    # dims from a resident volume when full_dims is not given
    h = ctx.volume_upload(np.zeros((6, 10, 20), np.uint16))
    g = ctx.mask_blocks([dict(src_to_world=synth.translation((2.0, 0.0, 0.0)), vol_handle=h)], [(0, 0, 0)], [(30, 12, 8)], (0, 0, 0), dt)[0]
    assert np.array_equal(g, fo.mask_block([(synth.translation((2.0, 0.0, 0.0)), (20, 10, 6))], (0, 0, 0), (30, 12, 8), (0, 0, 0), out_dtype))
    ctx.volume_free(h)
    with pytest.raises(bsgpu.BsError):
        ctx.mask_blocks([dict(src_to_world=synth.translation((0, 0, 0)), vol_handle=0)], [(0, 0, 0)], [(4, 4, 4)])
