"""detect-interestpoints on the device: bs_median_divide and bs_downsample_float bit-identical to the oracle,
bs_sample_nlinear within its float32 bound, and the command end to end against oracle/ip_oracle.py on a bead
dataset written as SpimData2 XML + BDV-N5."""
import numpy as np
import pytest

from oracle import ip_oracle as io

pytestmark = pytest.mark.gpu


def _roundtrip(ctx, fn, vol, *args):
    h = ctx.volume_upload(vol)
    try:
        o = fn(h, *args)
        try:
            return ctx.volume_download(o)
        finally:
            ctx.volume_free(o)
    finally:
        ctx.volume_free(h)


def _u16(shape, seed, lo=0, hi=4000):
    return np.random.default_rng(seed).integers(lo, hi, shape).astype(np.uint16)


def _u8_ties(shape, seed):
    return np.random.default_rng(seed).integers(0, 4, shape).astype(np.uint8)


def _f32_signed(shape, seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(0.5, 1.0, shape).astype(np.float32)
    v[rng.random(shape) < 0.1] = 0.0
    v[-1] = 3.25                                     # a constant slice
    return v


MEDIAN_CASES = [
    # (name, volume factory, radius)
    ("u16_37x29x3", lambda: _u16((3, 29, 37), 1), 1),
    ("u16_37x29x3", lambda: _u16((3, 29, 37), 2), 2),
    ("u16_70x45x2", lambda: _u16((2, 45, 70), 3), 3),
    ("u16_70x45x2", lambda: _u16((2, 45, 70), 4), 10),
    ("u16_83x41x1", lambda: _u16((1, 41, 83), 5), 25),
    ("u8_ties_45x33x2", lambda: _u8_ties((2, 33, 45), 6), 1),
    ("u8_ties_45x33x2", lambda: _u8_ties((2, 33, 45), 7), 10),
    ("u8_ties_45x33x2", lambda: _u8_ties((2, 33, 45), 8), 25),
    ("f32_signed_39x27x3", lambda: _f32_signed((3, 27, 39), 9), 2),
    ("f32_signed_39x27x3", lambda: _f32_signed((3, 27, 39), 10), 10),
    ("f32_signed_39x27x3", lambda: _f32_signed((3, 27, 39), 11), 25),
    ("u16_slice_smaller_than_r_5x3x2", lambda: _u16((2, 3, 5), 12), 10),
    ("f32_slice_smaller_than_r_1x2x1", lambda: _f32_signed((1, 2, 1), 13), 25),
    ("u16_1x1x4", lambda: _u16((4, 1, 1), 14), 3),
]


@pytest.mark.parametrize("name,make,radius", MEDIAN_CASES, ids=[f"{c[0]}_r{c[2]}" for c in MEDIAN_CASES])
def test_median_divide_bit_identical(ctx, name, make, radius):
    vol = make()
    got = _roundtrip(ctx, ctx.median_divide, vol, radius)
    want = io.median_divide(vol, radius)
    assert got.dtype == np.float32 and got.shape == vol.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
        (name, radius, int((got.view(np.uint32) != want.view(np.uint32)).sum()))


def test_median_radius_limit_then_context_still_works(ctx):
    import bsgpu
    vol = _u16((2, 20, 24), 15)
    h = ctx.volume_upload(vol)
    try:
        with pytest.raises(bsgpu.BsError):
            ctx.median_divide(h, bsgpu.native.MEDIAN_MAX_RADIUS + 1)
        with pytest.raises(bsgpu.BsError):
            ctx.median_divide(h, 0)
        o = ctx.median_divide(h, bsgpu.native.MEDIAN_MAX_RADIUS)
        got = ctx.volume_download(o)
        ctx.volume_free(o)
    finally:
        ctx.volume_free(h)
    assert np.array_equal(got.view(np.uint32), io.median_divide(vol, bsgpu.native.MEDIAN_MAX_RADIUS).view(np.uint32))


def _f32_order_sensitive(shape, seed):
    """Values spanning many binades with 24 significant bits, so pair averages round and a different order of the
    x / y / z steps gives different bits."""
    rng = np.random.default_rng(seed)
    m = rng.integers(1 << 23, 1 << 24, shape).astype(np.float64)
    e = rng.integers(-30, 10, shape)
    s = np.where(rng.random(shape) < 0.3, -1.0, 1.0)
    return (s * np.ldexp(m, e)).astype(np.float32)


@pytest.mark.parametrize("factors", [(1, 1, 1), (2, 2, 1), (4, 4, 2), (8, 8, 1)])
@pytest.mark.parametrize("kind", ["u16", "u8", "f32"])
def test_downsample_float_bit_identical(ctx, factors, kind):
    shape = (9, 35, 67)
    vol = {"u16": lambda: _u16(shape, 20, 0, 65535), "u8": lambda: _u8_ties(shape, 21),
           "f32": lambda: _f32_order_sensitive(shape, 22)}[kind]()
    got = _roundtrip(ctx, ctx.downsample_float, vol, factors)
    want = io.downsample_float(vol, factors)
    assert got.shape == want.shape == tuple(shape[a] // factors[2 - a] for a in range(3))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if kind == "f32" and factors == (4, 4, 2):
        # the oracle's order is the one that matters: averaging z first gives other bits on this input
        zfirst = io.downsample_float(io.downsample_float(vol, (1, 1, 2)), (4, 4, 1))
        assert not np.array_equal(zfirst.view(np.uint32), want.view(np.uint32))


def test_downsample_float_rejects_bad_factors(ctx):
    import bsgpu
    h = ctx.volume_upload(_u16((4, 8, 8), 23))
    try:
        for f in ((3, 1, 1), (256, 1, 1), (16, 1, 1), (0, 1, 1)):
            with pytest.raises(bsgpu.BsError):
                ctx.downsample_float(h, f)
    finally:
        ctx.volume_free(h)


# float32 n-linear bound: 8 corner terms each rounded to float32 and 7 float32 additions of partial sums, all bounded by
# max |corner|: |got - exact| <= 16 * 2^-24 * max |corner|
NLINEAR_BOUND_ULPS = 16 * 2.0 ** -24


@pytest.mark.parametrize("kind", ["u16", "f32"])
def test_sample_nlinear_within_bound(ctx, kind):
    shape = (7, 11, 13)
    vol = _u16(shape, 30, 0, 65535) if kind == "u16" else _f32_signed(shape, 31)
    dims = np.array(shape[::-1], dtype=np.float64)
    rng = np.random.default_rng(32)
    pts = [rng.uniform(-1.0, dims) for _ in range(400)]                       # inside and up to 1 px outside
    pts += [np.array(c, dtype=np.float64) * (dims - 1) for c in np.ndindex(2, 2, 2)]   # corners
    pts += [np.array([dims[0] - 1, 3.5, 2.25]), np.array([0.0, dims[1] - 1, 4.75]), np.array([6.5, 0.0, dims[2] - 1]),
            np.array([dims[0] - 0.25, dims[1] - 0.5, dims[2] - 0.75]), np.array([-0.999, -0.5, -1.0])]
    loc = np.array(pts)
    h = ctx.volume_upload(vol)
    try:
        got = ctx.sample_nlinear(h, loc)
        ints = np.array([[x, y, z] for z in range(shape[0]) for y in range(shape[1]) for x in range(shape[2])], np.float64)
        exact = ctx.sample_nlinear(h, ints)
    finally:
        ctx.volume_free(h)
    want = io.sample_nlinear(vol, loc)
    v64 = vol.astype(np.float64)
    for p, g, w in zip(loc, got, want):
        b = np.floor(p).astype(np.int64)
        corner = max(abs(v64[min(max(b[2] + k, 0), shape[0] - 1), min(max(b[1] + j, 0), shape[1] - 1),
                             min(max(b[0] + i, 0), shape[2] - 1)]) for i in (0, 1) for j in (0, 1) for k in (0, 1))
        assert abs(float(g) - w) <= NLINEAR_BOUND_ULPS * corner, (p, g, w)
    assert np.array_equal(exact, vol.astype(np.float32).ravel())              # integer points: the voxel exactly


# ------------------------------------------------------------------------------------------------ command end to end
def _beads(shape_zyx, centres_xyz, seed, sigma_xy=6.0, sigma_z=1.8, amp=1000.0, bg=100.0, noise=2.0):
    z, y, x = np.mgrid[0:shape_zyx[0], 0:shape_zyx[1], 0:shape_zyx[2]].astype(np.float64)
    img = np.full(shape_zyx, bg) + np.random.default_rng(seed).normal(0.0, noise, shape_zyx)
    for cx, cy, cz in centres_xyz:
        img += amp * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * sigma_xy ** 2) - (z - cz) ** 2 / (2 * sigma_z ** 2))
    return np.clip(np.rint(img), 0, 65535).astype(np.uint16)


BEADS0 = [(30.3, 25.6, 8.2), (90.7, 30.2, 12.6), (60.1, 70.4, 15.3), (100.4, 75.8, 7.7)]
BEADS1 = [(25.2, 20.7, 6.4), (70.6, 55.3, 11.1)]
KW = dict(sigma=1.8, threshold=0.01, min_intensity=0.0, max_intensity=1000.0)


@pytest.fixture(scope="module")
def bead_dataset(tmp_path_factory):
    from bsgpu import n5 as bn5, spimdata
    from oracle import fusion_oracle as fo
    root = tmp_path_factory.mktemp("ip")
    v0 = _beads((24, 96, 128), BEADS0, 1)
    v1 = _beads((20, 80, 96), BEADS1, 2)
    v2 = np.full((8, 40, 40), 100, np.uint16)                                  # nothing to detect
    store = bn5.N5Store(str(root / "dataset.n5"), create=True)
    bn5.write_bdv_setup(store, 0, 0, v0, (64, 64, 16), downsampling_factors=((1, 1, 1), (2, 2, 1)))
    store.write_volume(bn5.bdv_dataset(0, 0, 1), fo.downsample2x(v0, (2, 2, 1)), (64, 64, 16))
    bn5.write_bdv_setup(store, 1, 0, v1, (64, 64, 16))
    bn5.write_bdv_setup(store, 2, 0, v2, (64, 64, 16))
    xml = spimdata.write_dataset_xml(str(root / "dataset.xml"), "dataset.n5", [
        dict(setup=0, size_xyz=(128, 96, 24), tile=0, translation_xyz=(0, 0, 0)),
        dict(setup=1, size_xyz=(96, 80, 20), tile=1, translation_xyz=(100, 0, 0)),
        dict(setup=2, size_xyz=(40, 40, 8), tile=2, translation_xyz=(0, 100, 0))])
    return dict(root=root, xml=xml, store=store, vols={(0, 0): v0, (0, 1): v1, (0, 2): v2})


def _oracle(ds, view, median=None, max_spots=0, **kw):
    from bsgpu import n5 as bn5
    if view == (0, 0):
        lvl_vol, remaining, mt = ds["store"].read_volume(bn5.bdv_dataset(0, 0, 1)), (2, 2, 1), \
            [[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 1, 0]]
    else:
        lvl_vol, remaining, mt = ds["vols"][view], (4, 4, 1), np.eye(4)[:3]
    return io.detect_interestpoints_reference(lvl_vol, remaining, mt, median_radius=median, max_spots=max_spots,
                                              **{**KW, **kw})


def _stored(ds, view, label):
    from bsgpu import n5 as bn5
    st = bn5.N5Store(str(ds["root"] / "interestpoints.n5"))
    g = f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}"
    return st, g, st.read_list(g + "/interestpoints/loc"), st.read_list(g + "/interestpoints/id")


def test_detect_interestpoints_end_to_end(ctx, bead_dataset):
    from bsgpu import commands, spimdata
    ds = bead_dataset
    res = commands.detect_interestpoints(ds["xml"], ctx, "beads", downsample_xy=4, block_size=(8, 8, 6),
                                         store_intensities=True, **KW)
    assert sorted(res) == [(0, 0), (0, 1), (0, 2)]
    for view, beads, total, level_f in (((0, 0), BEADS0, 4, 2), ((0, 1), BEADS1, 4, 1)):
        want = _oracle(ds, view)
        st, g, loc, ids = _stored(ds, view, "beads")
        assert len(loc) == len(want["loc"]) >= len(beads)
        assert np.array_equal(ids.ravel(), np.arange(len(loc), dtype=np.uint64))
        # same detections: the stored (grid-order) list is a permutation of the oracle's whole-view list
        order = np.lexsort(loc.T[::-1])
        worder = np.lexsort(want["loc"].T[::-1])
        assert np.allclose(loc[order], want["loc"][worder], atol=1e-3 * total, rtol=0)
        assert len({tuple(np.rint(p / 1e-3)) for p in loc}) == len(loc)                   # no duplicates
        # planted centres come back in full-resolution pixels; the reference's transform adds no half-pixel shift for
        # the additional downsampling, so a bead at c is reported at c - (F - f) / 2 in x and y (PARITY_GAPS)
        bias = np.array([(total - level_f) / 2, (total - level_f) / 2, 0.0])
        for c in beads:
            assert np.min(np.linalg.norm(loc - (np.array(c) - bias), axis=1)) < 1.0, (view, c)
        inten = st.read_list(g + "/intensities")
        assert inten.dtype == np.float32 and inten.shape == (len(loc), 1)
        assert np.allclose(inten[order, 0], want["intensities"][worder], rtol=1e-5)
    st, g, loc, ids = _stored(ds, (0, 2), "beads")
    assert loc.shape[0] == 0 and ids.shape[0] == 0 and st.dataset_attributes(g + "/intensities")["dimensions"] == [0]
    ips = spimdata.SpimData2.load(ds["xml"]).interest_points()
    assert all(ips[v]["beads"]["path"] == f"tpId_0_viewSetupId_{v[1]}/beads" for v in ((0, 0), (0, 1), (0, 2)))
    assert ips[(0, 0)]["beads"]["params"] == ("DOG (Spark) s=1.8 t=0.01 overlappingOnly=false min=false max=true "
                                              "downsampleXY=4 downsampleZ=1 minIntensity=0.0 maxIntensity=1000.0")


def test_block_grid_union_equals_whole_view(ctx, bead_dataset):
    from bsgpu import commands
    vol = bead_dataset["vols"][(0, 1)]
    h = ctx.volume_upload(vol)
    try:
        f = ctx.downsample_float(h, (2, 2, 1))
        dims, _ = ctx.volume_info(f)
        kw = dict(sigma=1.8, threshold=0.004, max_intensity=1000.0)
        whole = ctx.dog_detect(f, (1, 1, 1), tuple(d - 2 for d in dims), **kw)
        parts = [p for mn, sz in commands.interestpoint_blocks(dims, (7, 9, 4)) for p in ctx.dog_detect(f, mn, sz, **kw)]
        ctx.volume_free(f)
    finally:
        ctx.volume_free(h)
    key = lambda p: (p[2][2], p[2][1], p[2][0])   # noqa: E731
    assert len(parts) == len({p[2] for p in parts})
    assert sorted(parts, key=key) == sorted(whole, key=key) and len(whole) >= 2


def test_median_filter_run_matches_oracle(ctx, bead_dataset):
    from bsgpu import commands
    ds = bead_dataset
    kw = dict(KW, max_intensity=12.0)
    commands.detect_interestpoints(ds["xml"], ctx, "median", downsample_xy=4, block_size=(16, 16, 8), median_filter=10,
                                   **kw)
    for view in ((0, 0), (0, 1)):
        want = _oracle(ds, view, median=10, **kw)
        _, _, loc, _ = _stored(ds, view, "median")
        assert len(loc) == len(want["loc"]) >= 1
        assert np.allclose(loc[np.lexsort(loc.T[::-1])], want["loc"][np.lexsort(want["loc"].T[::-1])], atol=4e-3, rtol=0)


def test_max_spots_labels_and_sharding(ctx, bead_dataset):
    from bsgpu import commands, spimdata
    ds = bead_dataset
    first = _stored(ds, (0, 0), "beads")[2] if (ds["root"] / "interestpoints.n5").exists() else None
    # max_spots: the 3 brightest of view 0, in the order of the stable descending sort
    commands.detect_interestpoints(ds["xml"], ctx, "top", downsample_xy=4, block_size=(8, 8, 6), max_spots=3,
                                   store_intensities=True, **KW)
    want = _oracle(ds, (0, 0), max_spots=3)
    st, g, loc, ids = _stored(ds, (0, 0), "top")
    assert np.allclose(loc, want["loc"], atol=4e-3, rtol=0) and np.array_equal(ids.ravel(), np.arange(3))
    inten = st.read_list(g + "/intensities").ravel()
    assert np.all(np.diff(inten) <= 0)
    # a second label leaves the first untouched; re-running the first replaces it
    if first is not None:
        assert np.array_equal(_stored(ds, (0, 0), "beads")[2], first)
    commands.detect_interestpoints(ds["xml"], ctx, "top", downsample_xy=4, block_size=(8, 8, 6), max_spots=2, **KW)
    st, g, loc, _ = _stored(ds, (0, 0), "top")
    assert len(loc) == 2 and not (ds["root"] / "interestpoints.n5" / g / "intensities").exists()
    labels = spimdata.SpimData2.load(ds["xml"]).interest_points()[(0, 0)]
    assert "top" in labels and (first is None or "beads" in labels)
    # shard (0, 2) + (1, 2) merged by a list-gathering stub == shard (0, 1)
    run = dict(downsample_xy=4, block_size=(8, 8, 6), dry_run=True, **KW)
    one = commands.detect_interestpoints(ds["xml"], ctx, "s", **run)
    rank1 = {}
    commands.detect_interestpoints(ds["xml"], ctx, "s", shard=(1, 2), allgather=lambda o: [rank1.setdefault(1, o)], **run)
    two = commands.detect_interestpoints(ds["xml"], ctx, "s", shard=(0, 2), allgather=lambda o: [o, rank1[1]], **run)
    assert list(two) == list(one) and set(rank1[1]) == {(0, 1)}
    for v in one:
        assert np.array_equal(two[v][0], one[v][0])
