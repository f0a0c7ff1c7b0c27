"""Intensity-correction kernels on the H100 at the sizes and edges they switch on: every device result against the
bit-level oracle (oracle/intensity_oracle.py, the device's float32 operation order) and against its float64
reference (candidates_reference / apply_reference) within the bound written next to it.

  candidates  k_compact with 256 keys per thread (the default 8 x 8 x 8 cells), k_seg_count / k_scatter with dynamic
              shared memory above 48 KB, z-chunking, thresholds hit exactly, empty outputs and the two rejections;
  RANSAC      several candidate tiles, hypothesis rounds after the first, the strict inlier test, the tie rule, skipped
              hypotheses, the min_num_candidates boundary, and every bucket of the large grids;
  apply       x across one and several 256-thread blocks, 1 cell and 1 cell per pixel, 2x / 4x levels, u8 / u16 / f32;
  fusion      affine_fusion --intensityN5Path on a view fused from its 2x level with non-identity coefficients."""
import numpy as np
import pytest

import bsgpu
from bsgpu import commands, fusion as bf, intensity as bint, n5 as bn5, spimdata, zarr as bzarr
from oracle import fusion_oracle as fo
from oracle import intensity_oracle as io
from tests import synth
from tests import test_fusion_gpu as tfg
from tests.intensity_scene import (DEFAULT_GRID, TOO_MANY_SLOTS, WIDE_SLOTS, apply_bound, apply_case,
                                   candidate_value_bound, integer_scene, later_round_bucket, shifted_grid_scene)

pytestmark = pytest.mark.gpu

NAN = float("nan")


# ------------------------------------------------------------------------------------------------ candidates
def _upload(ctx, A, B, va, vb):
    ha, hb = ctx.volume_upload(A), ctx.volume_upload(B)
    return ha, hb, dict(va, vol_handle=ha), dict(vb, vol_handle=hb)


def _candidates(ctx, va, vb, rmin, rmax, tmin=1.0, tmax=NAN, chunk=0):
    h, *got = ctx.intensity_candidates(va, vb, 1.0, rmin, rmax, tmin, tmax, chunk_points=chunk)
    ctx.intensity_candidates_free(h)
    return got


def _assert_candidates(got, want, ref):
    """Bit-identical to the oracle; the same keys, offsets and counts as the float64 reference (exact geometry), and
    values within 16 u max|corner| of it (candidate_value_bound, PARITY_GAPS row 37)."""
    for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(g, w)
    keys, offs, cnts, vals, cmax = ref
    for g, w in zip(got[:3], (keys, offs, cnts)):
        assert np.array_equal(g, w)
    assert np.all(np.abs(got[3] - vals) <= candidate_value_bound(cmax))


_GRIDS = {"default_grid": DEFAULT_GRID, "wide_slots": WIDE_SLOTS}


@pytest.fixture(scope="module", params=sorted(_GRIDS))
def grid(request):
    """A large exact-geometry scene with its oracle and float64 reference outputs (computed once per module)."""
    A, B, va, vb, rmin, rmax = shifted_grid_scene(**_GRIDS[request.param])
    want = io.candidates(A, va, B, vb, 1.0, rmin, rmax)
    ref = io.candidates_reference(A, va, B, vb, 1.0, rmin, rmax, corners=True)
    return request.param, (A, B, va, vb, rmin, rmax), want, ref


def test_candidates_at_large_cell_grids_and_every_chunking(ctx, grid):
    """default_grid: 3 375 buckets of 262 144 keys (k_compact scans 256 keys per thread).  wide_slots: 23 064
    buckets, so k_scatter needs 184 KB and k_seg_count 92 KB of dynamic shared memory.  Chunks of 0 (one chunk),
    plane - 1 and plane (one plane each) and 3 planes + 777 points write the same bytes; the render plane (121 x 120
    and 125 x 124 points) is a multiple of neither 32 nor 4096."""
    name, (A, B, va, vb, rmin, rmax), want, ref = grid
    assert len(want[0]) == {"default_grid": 3375, "wide_slots": 23064}[name]
    plane = int((rmax[0] - rmin[0] + 1) * (rmax[1] - rmin[1] + 1))
    assert plane % 32 and plane % 4096
    ha, hb, va, vb = _upload(ctx, A, B, va, vb)
    try:
        runs = [_candidates(ctx, va, vb, rmin, rmax, chunk=c) for c in (0, plane - 1, plane, 3 * plane + 777)]
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    for got in runs:
        _assert_candidates(got, want, ref)


def test_ransac_over_every_bucket_of_a_large_grid(ctx, grid):
    """Every eligible bucket: the returned count is the float64 recount of |a x + b - y| < eps for the returned
    (a, b).  A deterministic sample of 50 buckets (the first, the last and every k-th) equals the replayed stream of
    ransac_bucket exactly."""
    name, (A, B, va, vb, rmin, rmax), want, _ = grid
    keys, offs, cnts, vals = want
    min_n = {"default_grid": 100, "wide_slots": 20}[name]
    ha, hb, va, vb = _upload(ctx, A, B, va, vb)
    try:
        h, *_ = ctx.intensity_candidates(va, vb, 1.0, rmin, rmax)
        try:
            a, b, c = ctx.intensity_ransac(h, len(keys), min_num_candidates=min_n, num_iterations=1000, max_epsilon=5.1)
        finally:
            ctx.intensity_candidates_free(h)
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    ok = cnts >= min_n
    assert ok.all() and np.all(c >= 2)
    seg = np.repeat(np.arange(len(keys)), cnts)
    x, y = vals[:, 0].astype(np.float64), vals[:, 1].astype(np.float64)
    inl = np.abs((a[seg] * x + b[seg]) - y) < 5.1
    assert np.array_equal(np.bincount(seg, weights=inl, minlength=len(keys)).astype(np.int64), c)
    assert c.mean() > 0.5 * cnts.mean()                        # each bucket is a noisy line: RANSAC finds it
    for k in np.unique(np.r_[0, len(keys) - 1, np.linspace(0, len(keys) - 1, 48).astype(int)]):
        wa, wb, wc = io.ransac_bucket(vals[offs[k]:offs[k] + cnts[k]], int(keys[k]), 1000, 5.1)
        assert (a[k], b[k], c[k]) == (wa, wb, wc)


@pytest.mark.parametrize("tmax", [200.0, NAN])
@pytest.mark.parametrize("chunk", [0, 64 * 28 + 5])
def test_integer_scene_thresholds_and_edges(ctx, tmax, chunk):
    """uint8 on both sides, A through its 2x level with a 90 degree rotation (integer_scene): values exactly at
    min_threshold 1 (and at max_threshold 200) are kept, points on p = d - 1 are inside, points on cell borders fall
    in the upper cell.  The float32 samples are exact here, so the values equal the float64 reference.  Chunk 1797:
    the 64 x 28 plane plus 5 points, one plane per chunk."""
    LA, B, va, vb, rmin, rmax = integer_scene()
    want = io.candidates(LA, va, B, vb, 1.0, rmin, rmax, 1.0, tmax)
    ref = io.candidates_reference(LA, va, B, vb, 1.0, rmin, rmax, 1.0, tmax, corners=True)
    ha, hb, dva, dvb = _upload(ctx, LA, B, va, vb)
    try:
        got = _candidates(ctx, dva, dvb, rmin, rmax, 1.0, tmax, chunk)
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    _assert_candidates(got, want, ref)
    assert np.array_equal(got[3], ref[3]) and (got[3] == 1.0).any()


def test_empty_outputs(ctx):
    """An empty render range gives 0 buckets and a valid handle, whose RANSAC returns empty arrays; a non-empty range
    where no point passes the thresholds gives 0 buckets too."""
    LA, B, va, vb, rmin, rmax = integer_scene()
    ha, hb, va, vb = _upload(ctx, LA, B, va, vb)
    try:
        h, keys, offs, cnts, vals = ctx.intensity_candidates(va, vb, 1.0, rmin, (rmax[0], rmin[1] - 1, rmax[2]))
        assert len(keys) == len(offs) == len(cnts) == len(vals) == 0
        a, b, c = ctx.intensity_ransac(h, 0, min_num_candidates=0)
        assert len(a) == len(b) == len(c) == 0
        ctx.intensity_candidates_free(h)
        keys, offs, cnts, vals = _candidates(ctx, va, vb, rmin, rmax, 256.0)
        assert len(keys) == len(vals) == 0
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)


def _assert_integer_scene_on_device(ctx):
    LA, B, va, vb, rmin, rmax = integer_scene()
    ha, hb, dva, dvb = _upload(ctx, LA, B, va, vb)
    try:
        got = _candidates(ctx, dva, dvb, rmin, rmax)
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    for g, w in zip(got, io.candidates(LA, va, B, vb, 1.0, rmin, rmax)):
        assert np.array_equal(g, w)


def test_rejections_leave_the_context_usable(ctx):
    """cells(A) x cells(B) above 2^26 is BS_ERR_ARG; more buckets than one CTA's shared memory holds (31 752 x 8 B) is
    BS_ERR_UNSUPPORTED.  The next call after each still equals the oracle."""
    vol = np.ones((9, 32, 32), np.uint8)
    h = ctx.volume_upload(vol)
    try:
        v = bint.device_view(h, np.eye(3, 4), np.eye(3, 4), (32, 32, 9), (32, 32, 9))
        with pytest.raises(bsgpu.BsError) as e:
            ctx.intensity_candidates(v, v, 1.0, (0, 0, 0), (31, 31, 8))
        assert e.value.code == -1
    finally:
        ctx.volume_free(h)
    _assert_integer_scene_on_device(ctx)
    A, B, va, vb, rmin, rmax = shifted_grid_scene(**TOO_MANY_SLOTS)
    ha, hb, va, vb = _upload(ctx, A, B, va, vb)
    try:
        with pytest.raises(bsgpu.BsError) as e:
            ctx.intensity_candidates(va, vb, 1.0, rmin, rmax)
        assert e.value.code == -4
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    _assert_integer_scene_on_device(ctx)


# ------------------------------------------------------------------------------------------------ RANSAC
def _bucket(ctx, x, y):
    """Resident candidates of one bucket (key 0) holding (x_i, y_i) in order: views of n_cells (1, 1, 1) over
    1 x 1 x n float32 volumes, identity geometry, render scale 1, no threshold."""
    n = len(x)
    A = np.asarray(x, np.float32).reshape(1, 1, n)
    B = np.asarray(y, np.float32).reshape(1, 1, n)
    ha, hb = ctx.volume_upload(A), ctx.volume_upload(B)
    try:
        va, vb = (bint.device_view(hh, np.eye(3, 4), np.eye(3, 4), (n, 1, 1), (1, 1, 1)) for hh in (ha, hb))
        h, keys, offs, cnts, vals = ctx.intensity_candidates(va, vb, 1.0, (0, 0, 0), (n - 1, 0, 0), -np.inf)
    finally:
        ctx.volume_free(ha)
        ctx.volume_free(hb)
    assert keys.tolist() == [0] and np.array_equal(vals, np.stack([A.ravel(), B.ravel()], 1))
    return h, vals


def _ransac(ctx, x, y, min_num_candidates=2, num_iterations=1000, max_epsilon=5.1):
    h, vals = _bucket(ctx, x, y)
    try:
        a, b, c = ctx.intensity_ransac(h, 1, min_num_candidates, num_iterations, max_epsilon)
    finally:
        ctx.intensity_candidates_free(h)
    got = (a[0], b[0], int(c[0]))
    if c[0] >= 0:
        want = io.ransac_bucket(vals, 0, num_iterations, max_epsilon)
        assert got[2] == want[2] and np.array_equal(got[:2], want[:2], equal_nan=True)
    return got


def _line(x, y, h):
    """(a, b) of hypothesis h of bucket 0, as the device computes it (float64)."""
    i, j = io.draw(0, h, len(x))
    xi, yi, xj, yj = (float(np.float32(v)) for v in (x[i], y[i], x[j], y[j]))
    a = (yj - yi) / (xj - xi)
    return a, yi - a * xi


@pytest.mark.parametrize("n", [5000, 2048 * 3 + 17])
def test_ransac_reads_every_tile(ctx, n):
    """An exactly linear bucket (y = 2 x + 3, distinct x) of more than one 2048-candidate tile: every candidate is an
    inlier of every hypothesis, so all tie and the winner is h = 0 with exactly its line."""
    x = np.random.default_rng(n).permutation(n).astype(np.float32)
    y = 2 * x + 3
    a, b, c = _ransac(ctx, x, y)
    assert c == n and (a, b) == _line(x, y, 0) == (2.0, 3.0)


def test_ransac_ties_go_to_the_lowest_unskipped_hypothesis(ctx):
    """Every hypothesis counts all n (eps far above the jitter), each with a different line; h = 0 and h = 1 are
    skipped (equal x), so the winner is h = 2 and (a, b) is exactly its line."""
    n = 300
    rng = np.random.default_rng(7)
    x = rng.permutation(n).astype(np.float32)
    for h in (0, 1):
        i, j = io.draw(0, h, n)
        x[j] = x[i]
    assert [x[io.draw(0, h, n)[0]] == x[io.draw(0, h, n)[1]] for h in (0, 1, 2)] == [True, True, False]
    y = (2 * x + 3 + rng.uniform(-0.01, 0.01, n)).astype(np.float32)
    a, b, c = _ransac(ctx, x, y, max_epsilon=1e9)
    assert c == n and (a, b) == _line(x, y, 2) and (a, b) != _line(x, y, 999)


@pytest.mark.parametrize("iters", [1, 1023, 1024, 1025, 2049])
def test_ransac_hypothesis_rounds_after_the_first(ctx, iters):
    """later_round_bucket: the only three collinear candidates are first drawn together by h = 1024, the first
    hypothesis of the second round of 256 threads x 4.  Only runs that reach h = 1024 count 3."""
    x, y = later_round_bucket()
    a, b, c = _ransac(ctx, x, y, num_iterations=iters, max_epsilon=1e-3)
    if iters > 1024:
        assert (a, b, c) == (2.0, 3.0, 3)
    else:
        assert c == 2 and (a, b) == _line(x, y, 0)


def test_ransac_inlier_test_is_strict(ctx):
    """Integer data, y = x on 89 candidates and y = x + 4 on 11 (x 45..55): at eps 4.0 the shifted residuals (exactly 4)
    are not inliers, at the next double above 4 they are.  Lines through one shifted and one plain candidate reach
    at most ~60, so y = x wins at 4.0."""
    x = np.arange(100, dtype=np.float32)
    y = x + np.where((x >= 45) & (x <= 55), 4.0, 0.0).astype(np.float32)
    p = np.random.default_rng(3).permutation(100)
    x, y = x[p], y[p]
    assert _ransac(ctx, x, y, max_epsilon=4.0) == (1.0, 0.0, 89)
    a, b, c = _ransac(ctx, x, y, max_epsilon=float(np.nextafter(4.0, np.inf)))
    assert c == 100 and (a, b) in ((1.0, 0.0), (1.0, 4.0))


def test_ransac_skipped_hypotheses(ctx):
    a, b, c = _ransac(ctx, np.full(10, 5.0), np.arange(10.0))
    assert np.isnan(a) and np.isnan(b) and c == 0
    assert _ransac(ctx, [1.0, 3.0], [2.0, 8.0]) == (3.0, -1.0, 2)


def test_ransac_min_num_candidates_boundary(ctx):
    x = np.arange(7, dtype=np.float32)
    assert _ransac(ctx, x, 2 * x + 1, min_num_candidates=7)[2] == 7
    assert _ransac(ctx, x, 2 * x + 1, min_num_candidates=8)[2] == -1
    for m in (0, 1):
        a, b, c = _ransac(ctx, [4.0], [9.0], min_num_candidates=m)
        assert c == -1 and np.isnan(a) and np.isnan(b)


# ------------------------------------------------------------------------------------------------ apply
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("x", [1, 255, 256, 257, 600])
def test_apply_kernel(ctx, x, level, dtype):
    """apply_case: a window at the far corner of an identity / (2, 2, 1) / 4x level, 1 cell on one axis and one per
    full-resolution pixel on another, a in [0, 3], b < 0.  Within 2 ulp of the oracle, and within apply_bound (its
    float32 operation count over |a v| + |b|, plus the coordinate rounding times the coefficient slope) of the float64
    reference."""
    vol, wmin, mt, full, ca, cb = apply_case(x, level, dtype, seed=x + 10 * level)
    h = ctx.volume_upload(vol)
    try:
        hc = ctx.intensity_apply(h, full, mt, ca, cb, wmin)
        got = ctx.volume_download(hc)
        ctx.volume_free(hc)
    finally:
        ctx.volume_free(h)
    want = io.apply(vol, wmin, mt, full, ca, cb)
    assert got.dtype == np.float32 and got.shape == vol.shape
    assert np.all(np.abs(got - want) <= 2 * np.spacing(np.abs(want).astype(np.float32)))
    ref = io.apply_reference(vol, wmin, mt, full, ca, cb)
    assert np.all(np.abs(got - ref) <= apply_bound(vol, wmin, mt, full, ca, cb))


def test_apply_rejects_a_grid_axis_of_65536(ctx):
    h = ctx.volume_upload(np.ones((1, 65536, 1), np.uint8))
    try:
        with pytest.raises(bsgpu.BsError) as e:
            ctx.intensity_apply(h, (1, 65536, 1), np.eye(3, 4), np.ones((1, 1, 1)), np.zeros((1, 1, 1)))
        assert e.value.code == -4
    finally:
        ctx.volume_free(h)
    vol, wmin, mt, full, ca, cb = apply_case(257, 1, np.uint16)
    h = ctx.volume_upload(vol)
    try:
        hc = ctx.intensity_apply(h, full, mt, ca, cb, wmin)
        got = ctx.volume_download(hc)
        ctx.volume_free(hc)
    finally:
        ctx.volume_free(h)
    want = io.apply(vol, wmin, mt, full, ca, cb)
    assert np.all(np.abs(got - want) <= 2 * np.spacing(np.abs(want).astype(np.float32)))


# ------------------------------------------------------------------------------------------------ fusion
FULL = {0: (64, 48, 24), 1: (96, 64, 32)}
MT1 = np.array([[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 2, 0.5]], np.float64)   # level 1 -> full resolution


def _two_level_dataset(tmp_path):
    """View 0: 64 x 48 x 24 at the origin, level 0 only.  View 1: 96 x 64 x 32 registered as world = 0.5 (p + (80, 8,
    4)), its N5 setup carrying a 2x level, so fusion reads it from level 1 (unit world step).  Coefficient ramps over
    4 x 3 x 2 and 3 x 4 x 2 cells.  Returns (xml, coefficient path, {view: level volume}, {view: registration})."""
    G = synth.field((40, 60, 100), seed=21, sigma=2.0, mean=800.0, std=200.0)
    lvl = {0: np.clip(np.rint(G[:24, :48, :64]), 0, 65535).astype(np.uint16),
           1: np.clip(np.rint(G[2:18, 4:36, 40:88] * 1.1 + 30), 0, 65535).astype(np.uint16)}
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    bn5.write_bdv_setup(store, 0, 0, lvl[0], (64, 64, 32))
    s0 = np.repeat(np.repeat(np.repeat(lvl[1], 2, 0), 2, 1), 2, 2)
    bn5.write_bdv_setup(store, 1, 0, s0, (64, 64, 32), downsampling_factors=((1, 1, 1), (2, 2, 2)))
    store.write_volume(bn5.bdv_dataset(1, 0, 1), lvl[1], (64, 64, 32), "raw")
    tiles = [dict(setup=0, size_xyz=FULL[0], tile=0, translation_xyz=(0, 0, 0)),
             dict(setup=1, size_xyz=FULL[1], tile=1, translation_xyz=(80, 8, 4))]
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    data = spimdata.SpimData2.load(xml)
    data.add_registration((0, 1), "scale", np.diag([0.5, 0.5, 0.5, 1.0])[:3])
    data.save(xml)
    regs = {v: spimdata.SpimData2.load(xml).model(0, v) for v in (0, 1)}
    g = lambda shape, lo, hi, axis: np.broadcast_to(np.linspace(lo, hi, shape[axis]).reshape(
        [shape[axis] if k == axis else 1 for k in range(3)]), shape).copy()
    co = {(0, 0): (g((2, 3, 4), 0.6, 1.4, 2) + g((2, 3, 4), 0.0, 0.3, 0), g((2, 3, 4), -30.0, 20.0, 1)),
          (0, 1): (g((2, 4, 3), 1.5, 0.8, 1), g((2, 4, 3), 25.0, -40.0, 2) + g((2, 4, 3), 0.0, 10.0, 0))}
    cpath = str(tmp_path / "coeff.n5")
    bint.write_coefficients(cpath, "N5", "", "intensity", co)
    return xml, cpath, lvl, regs, co


def _expected_fusion(lvl, regs, co, mts, bb_min, size, ft, apply_mts=None):
    """fuse_block over the level volumes corrected by apply_reference; ``apply_mts`` (default ``mts``): the
    level-to-full transforms handed to the correction."""
    views = []
    for v in (0, 1):
        ca, cb = co[(0, v)]
        img = io.apply_reference(lvl[v], (0, 0, 0), (apply_mts or mts)[v], FULL[v], ca, cb).astype(np.float32)
        m = (np.vstack([regs[v], [0, 0, 0, 1]]) @ np.vstack([mts[v], [0, 0, 0, 1]]))[:3]
        border, rng = fo.adjust_blending(m)
        content = fo.content_weights(img) if ft == fo.AVG_BLEND_CONTENT else None
        views.append(fo.View(img, m, border, rng, content))
    return views, fo.fuse_block(views, bb_min, size, ft)


@pytest.mark.parametrize("ft", ["AVG_BLEND", "AVG_BLEND_CONTENT"])
def test_fusion_applies_the_coefficients_at_the_fused_level(ctx, tmp_path, ft):
    """affine_fusion(..., intensity_n5_path=) against fuse_block over the level volumes corrected by apply_reference
    with the mipmap transform written here (content weights from the corrected volumes), within the fusion tolerance
    (test_fusion_gpu._assert_close, PARITY_GAPS row 29).  Correcting view 1 with the level-0 transform instead gives
    an expected block far outside that tolerance, so the test sees which transform reaches bs_intensity_apply."""
    xml, cpath, lvl, regs, co = _two_level_dataset(tmp_path)
    factors = [(1, 1, 1), (2, 2, 2)]
    assert bf.best_mipmap_level(regs[1], factors, [bzarr.mipmap_transform_default(f) for f in factors]) == 1
    out = str(tmp_path / "fused.n5")
    commands.create_fusion_container(xml, out, block_size=(32, 32, 16))
    s0 = commands.affine_fusion(out, ctx, fusion_type=ft, intensity_n5_path=cpath)[0]
    got = bn5.N5Store(out).read_volume(s0)
    meta = bn5.read_fusion_container(out)[1]
    bb_min = tuple(int(v) for v in meta["bb_min"])
    size = got.shape[::-1]
    fid = getattr(fo, ft)
    views, want = _expected_fusion(lvl, regs, co, {0: np.eye(3, 4), 1: MT1}, bb_min, size, fid)
    tfg._run.last = (views, bb_min, size)
    tfg._assert_close(got, want)
    _, wrong = _expected_fusion(lvl, regs, co, {0: np.eye(3, 4), 1: MT1}, bb_min, size, fid,
                                apply_mts={0: np.eye(3, 4), 1: np.eye(3, 4)})
    nz = np.abs(wrong[wrong != 0])
    err = np.abs(got - wrong) / np.maximum(np.abs(wrong), max(0.25 * float(nz.mean()), 1.0))
    assert (err > tfg.RTOL).sum() > 100 * (1e-3 * got.size + 2) and err.max() > 100 * tfg.RTOL
