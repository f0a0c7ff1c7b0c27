"""extract-psfs on the CPU: the oracle (oracle/psf_oracle.py) against analytic beads and the float64 interpolator, and the
command end to end through an oracle-backed context: point choice, runs of points, TIFF and XML output, errors and
sharding."""
import os
import shutil
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata, tiff
from oracle import ip_oracle as io
from oracle import psf_oracle as po
from tests.fake_ctx import FakeContext

SIZE = (7, 7, 9)
SIGMA = (1.5, 1.5, 2.0)


class PsfFakeContext(FakeContext):
    """FakeContext plus bs_psf_accumulate, computed by the oracle on the window placed in an otherwise empty view."""

    def __init__(self, free_bytes=1 << 40):
        super().__init__()
        self.free_bytes = free_bytes
        self.windows = []

    def memory_free(self):
        return self.free_bytes

    def psf_accumulate(self, h, window_min, full_dims, points, psf_size, sum=None):
        win = self.vols[h]
        assert all(s % 2 == 1 and s >= 1 for s in psf_size)
        w = [int(v) for v in window_min]
        assert all(w[d] >= 0 and w[d] + win.shape[2 - d] <= full_dims[d] for d in range(3))
        self.windows.append((tuple(w), win.shape[::-1], len(points)))
        full = np.zeros(tuple(int(v) for v in full_dims)[::-1], dtype=win.dtype)
        full[w[2]:w[2] + win.shape[0], w[1]:w[1] + win.shape[1], w[0]:w[0] + win.shape[2]] = win
        out = po.accumulate(full, points, psf_size, sum)
        if sum is not None:
            sum[...] = out
            return sum
        return out


def gaussian(shape_zyx, centres_xyz, amp=1000.0, sigma=SIGMA, bg=0.0):
    z, y, x = np.mgrid[0:shape_zyx[0], 0:shape_zyx[1], 0:shape_zyx[2]].astype(np.float64)
    v = np.full(shape_zyx, bg)
    for cx, cy, cz in centres_xyz:
        v += amp * np.exp(-(x - cx) ** 2 / (2 * sigma[0] ** 2) - (y - cy) ** 2 / (2 * sigma[1] ** 2)
                          - (z - cz) ** 2 / (2 * sigma[2] ** 2))
    return v


def write_points(root, data, view, label, loc, partners=()):
    """Points ``loc`` (ids 0..n-1) of ``view`` and one correspondence row per id in ``partners`` (to view (0, 99))."""
    store = bn5.N5Store(os.path.join(root, "interestpoints.n5"), create=True)
    group = f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}"
    commands._write_view_points(store, group, np.arange(len(loc)), np.asarray(loc, dtype=np.float64))
    store.write_correspondences(group, [(int(i), (0, 99), label, int(i)) for i in partners])
    data.set_interest_points(label, "test", {tuple(view): group})


def psf_scene(root, dtype=np.uint16, seed=1):
    """Three views (48 x 40 x 24) of scattered Gaussian beads on a background, BDV-N5; points 'beads' in views 0 and 1
    (some of them with correspondences), view 2 without points.  Returns (xml, {view: volume}, {view: (loc, partners)})."""
    os.makedirs(root, exist_ok=True)
    rng = np.random.default_rng(seed)
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    vols, tiles, pts = {}, [], {}
    for s in range(3):
        loc = np.column_stack([rng.uniform(-1.0, 48.5, 14), rng.uniform(-1.0, 40.5, 14), rng.uniform(-1.0, 24.5, 14)])
        loc[:3] = [(0.2, 0.0, 23.7), (47.9, 39.5, 0.3), (24.0, 20.0, 12.0)]          # at faces and on a voxel
        v = gaussian((24, 40, 48), loc, bg=100.0) + rng.normal(0.0, 3.0, (24, 40, 48))
        v = np.clip(np.rint(v), 0, 255 if dtype == np.uint8 else 65535).astype(dtype) if dtype != np.float32 \
            else v.astype(np.float32)
        bn5.write_bdv_setup(store, s, 0, v, (16, 16, 8))
        tiles.append(dict(setup=s, size_xyz=(48, 40, 24), tile=s, translation_xyz=(50 * s, 0, 0)))
        vols[(0, s)] = v
        pts[(0, s)] = (loc, sorted(rng.choice(14, 8, replace=False).tolist()))
    xml = spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)
    data = spimdata.SpimData2.load(xml)
    for v in ((0, 0), (0, 1)):
        write_points(root, data, v, "beads", *pts[v])
    data.save(xml, backup=False)
    return xml, vols, pts


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _entries(xml):
    return [(p.get("timepoint"), p.get("setup"), p.findtext("file"))
            for p in ET.parse(xml).getroot().findall("PointSpreadFunctions/PointSpreadFunction")]


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_sample_is_the_float64_interpolator_within_the_nlinear_bound():
    rng = np.random.default_rng(3)
    vol = rng.uniform(-500.0, 60000.0, (6, 9, 11)).astype(np.float32)
    loc = np.column_stack([rng.uniform(-2, 13, 500), rng.uniform(-2, 11, 500), rng.uniform(-2, 8, 500)])
    got, want = po.sample(vol, loc), io.sample_nlinear(vol, loc)
    assert got.dtype == np.float32
    assert np.all(np.abs(got - want) <= 16 * 2.0 ** -24 * np.abs(vol).max())
    ints = np.array([[x, y, z] for z in range(6) for y in range(9) for x in range(11)], np.float64)
    assert np.array_equal(po.sample(vol, ints), vol.ravel())


def test_single_bead_at_a_voxel_gives_the_gaussian_samples_exactly(tmp_path):
    vol = gaussian((24, 40, 48), [(20, 17, 11)]).astype(np.float32)
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    bn5.write_bdv_setup(store, 0, 0, vol, (16, 16, 8))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5",
                                     [dict(setup=0, size_xyz=(48, 40, 24), tile=0, translation_xyz=(0, 0, 0))])
    data = spimdata.SpimData2.load(xml)
    write_points(str(tmp_path), data, (0, 0), "beads", [(20.0, 17.0, 11.0)])
    data.save(xml)
    res = commands.extract_psfs(xml, PsfFakeContext(), "beads", SIZE, all_points=True, dry_run=True)
    psf, n = res[(0, 0)]
    assert n == 1 and psf.dtype == np.float32 and psf.shape == SIZE[::-1]
    assert np.array_equal(psf, vol[11 - 4:11 + 5, 17 - 3:17 + 4, 20 - 3:20 + 4])


def test_sub_pixel_beads_average_to_the_gaussian_within_the_nlinear_bound():
    rng = np.random.default_rng(4)
    cen = np.column_stack([rng.uniform(10, 70, 40), rng.uniform(10, 70, 40), rng.uniform(10, 30, 40)])
    o = po.offsets(SIZE)
    want = 1000.0 * np.exp(-(o[:, 0] ** 2 + o[:, 1] ** 2) / (2 * SIGMA[0] ** 2) - o[:, 2] ** 2 / (2 * SIGMA[2] ** 2))
    got = np.zeros(len(o))
    for c in cen:                                            # one bead per volume: no neighbours in the box
        vol = gaussian((40, 80, 80), [c]).astype(np.float32)
        got += po.extract(vol, [c], SIZE).reshape(-1)
    got /= len(cen)
    bound = 1000.0 * sum(1.0 / (8.0 * s * s) for s in SIGMA)   # |f''| h^2 / 8 per axis, h = 1
    err = np.abs(got - want)
    assert err.max() <= bound, (err.max(), bound)
    assert got.argmax() == len(o) // 2


def test_oracle_accumulate_is_sequential_in_float64():
    rng = np.random.default_rng(5)
    vol = rng.uniform(0, 1000, (10, 12, 14)).astype(np.float32)
    pts = np.column_stack([rng.uniform(0, 14, 9), rng.uniform(0, 12, 9), rng.uniform(0, 10, 9)])
    o = po.offsets((3, 5, 3))
    want = np.zeros(len(o))
    for p in pts:
        want += po.sample(vol, p + o).astype(np.float64)
    got = po.accumulate(vol, pts[:4], (3, 5, 3))
    got = po.accumulate(vol, pts[4:], (3, 5, 3), got)
    assert np.array_equal(got.reshape(-1), want)


# ------------------------------------------------------------------------------------------------ the command
def test_corresponding_points_by_default_and_every_point_with_all_points(tmp_path):
    xml, vols, pts = psf_scene(str(tmp_path))
    ctx = PsfFakeContext()
    for all_points in (False, True):
        res = commands.extract_psfs(xml, ctx, "beads", SIZE, all_points=all_points, view_selection=dict(vi=["0,0", "0,1"]),
                                    dry_run=True)
        for v in ((0, 0), (0, 1)):
            loc, partners = pts[v]
            ids = list(range(len(loc))) if all_points else partners
            assert res[v][1] == len(ids)
            assert np.array_equal(res[v][0], po.extract(vols[v], loc[ids], SIZE))


def test_the_sum_does_not_depend_on_the_runs_of_points(tmp_path, monkeypatch):
    xml, vols, pts = psf_scene(str(tmp_path))
    sel = dict(vi=["0,0", "0,1"])
    one = PsfFakeContext()
    whole = commands.extract_psfs(xml, one, "beads", SIZE, all_points=True, view_selection=sel, dry_run=True)
    assert len(one.windows) == 2
    # about one point's window per run, the runs taken as they are even where they overlap
    monkeypatch.setattr(commands, "psf_slabs", lambda loc, s, full, _: commands.psf_runs(loc, s, full, 2 * 11 * 11 * 13))
    many = PsfFakeContext()
    split = commands.extract_psfs(xml, many, "beads", SIZE, all_points=True, view_selection=sel, dry_run=True)
    assert len(many.windows) > 10
    for v in whole:
        assert np.array_equal(whole[v][0], split[v][0])


def _check_plan(plan, loc, full, max_voxels=None):
    """The plan covers the points in order, each window lies in the view and holds every tap of its points."""
    assert plan[0][0] == 0 and plan[-1][1] == len(loc)
    assert all(a[1] == b[0] for a, b in zip(plan, plan[1:]))
    o = po.offsets(SIZE)
    for start, stop, wmin, wsize in plan:
        assert np.all(wmin >= 0) and np.all(wmin + wsize <= full)
        if max_voxels is not None:
            assert np.prod(wsize) <= max_voxels
        taps = np.floor(loc[start:stop, None, :] + o[None]).reshape(-1, 3)
        for bit in (0, 1):
            t = np.clip(taps + bit, 0, np.array(full) - 1)
            assert np.all(t >= wmin) and np.all(t < wmin + wsize)


def _scattered(rng, n, full):
    return np.column_stack([rng.uniform(-3, full[d] + 3, n) for d in range(3)])


def test_runs_follow_the_point_order_and_windows_hold_every_tap():
    rng = np.random.default_rng(6)
    full = (60, 50, 40)
    loc = _scattered(rng, 200, full)
    loc = loc[np.argsort(loc[:, 2])]
    runs = commands.psf_runs(loc, SIZE, full, 60 * 50 * 14)
    assert len(runs) > 2
    _check_plan(runs, loc, full, 60 * 50 * 14)
    _check_plan(commands.psf_slabs(loc, SIZE, full, 60 * 50 * 14), loc, full)


@pytest.mark.parametrize("budget", [1, 11 * 11 * 13, 40 * 40 * 20, 1 << 30])
def test_shuffled_ids_read_the_view_at_most_once(budget):
    """Ids in intensity order (detect-interestpoints --maxSpots) do not follow space: the plan still reads no more
    than the box of all taps, and that box lies in the view."""
    rng = np.random.default_rng(7)
    full = (200, 180, 60)
    loc = _scattered(rng, 2000, full)                       # uniform positions, so the id order is spatially random
    plan = commands.psf_slabs(loc, SIZE, full, budget)
    _check_plan(plan, loc, full)
    assert sum(int(np.prod(p[3])) for p in plan) <= np.prod(full)
    if budget == 40 * 40 * 20:                              # runs this size overlap: read the box of all taps once
        assert sum(int(np.prod(r[3])) for r in commands.psf_runs(loc, SIZE, full, budget)) > 2 * np.prod(full)
        assert len(plan) == 1


def test_clustered_ids_keep_their_runs():
    """Points that do follow space (two clusters one after the other) are read in two small windows, not the box of
    both."""
    rng = np.random.default_rng(8)
    full = (400, 400, 100)
    loc = np.vstack([rng.uniform((10, 10, 10), (50, 50, 30), (100, 3)), rng.uniform((340, 340, 60), (390, 390, 90), (100, 3))])
    plan = commands.psf_slabs(loc, SIZE, full, 80 * 80 * 50)
    assert [(p[0], p[1]) for p in plan] == [(0, 100), (100, 200)]
    _check_plan(plan, loc, full, 80 * 80 * 50)


@pytest.mark.parametrize("budget", [11 * 11 * 13, 20 * 20 * 12])
def test_command_reads_each_view_at_most_once(tmp_path, monkeypatch, budget):
    xml, vols, pts = psf_scene(str(tmp_path))              # ids in random spatial order
    sel = dict(vi=["0,0", "0,1"])
    monkeypatch.setattr(commands, "PSF_SLAB_BYTES", 2 * budget)
    ctx = PsfFakeContext()
    res = commands.extract_psfs(xml, ctx, "beads", SIZE, all_points=True, view_selection=sel, dry_run=True)
    assert sum(n for _, _, n in ctx.windows) == 28
    assert sum(int(np.prod(w[1])) for w in ctx.windows) <= 2 * 48 * 40 * 24
    for v in res:
        assert np.array_equal(res[v][0], po.extract(vols[v], pts[v][0], SIZE))


def test_tiff_and_xml_round_trip_keep_other_views_and_replace_their_own(tmp_path):
    xml, vols, pts = psf_scene(str(tmp_path))
    data = spimdata.SpimData2.load(xml)
    data.set_point_spread_functions({(0, 2): "psf_t0_vs2.tif"})                      # an entry of another view
    data.save(xml, backup=False)
    ctx = PsfFakeContext()
    res = commands.extract_psfs(xml, ctx, "beads", SIZE, view_selection=dict(vi=["0,0"]))
    assert _entries(xml) == [("0", "0", "psf_t0_vs0.tif"), ("0", "2", "psf_t0_vs2.tif")]
    assert _entries(xml + "~1") == [("0", "2", "psf_t0_vs2.tif")]
    tf = tiff.TiffFile(str(tmp_path / "psfs" / "psf_t0_vs0.tif"))
    try:
        assert tf.pages[0].description.startswith(b"ImageJ=") and b"slices=9" in tf.pages[0].description
        assert all(p.offsets[0] % 2 == 0 for p in tf.pages)
        assert np.array_equal(tf.series()[0].read_volume(), res[(0, 0)][0])
    finally:
        tf.close()
    before = _bytes(xml)
    res = commands.extract_psfs(xml, ctx, "beads", SIZE, all_points=True, view_selection=dict(vi=["0,0", "0,1"]))
    assert _bytes(xml + "~1") == before
    assert _entries(xml) == [("0", "0", "psf_t0_vs0.tif"), ("0", "1", "psf_t0_vs1.tif"), ("0", "2", "psf_t0_vs2.tif")]
    assert spimdata.SpimData2.load(xml).point_spread_functions()[(0, 1)] == "psf_t0_vs1.tif"
    for v in ((0, 0), (0, 1)):
        tf = tiff.TiffFile(str(tmp_path / "psfs" / commands.psf_file_name(v)))
        try:
            assert np.array_equal(tf.series()[0].read_volume(), res[v][0])
        finally:
            tf.close()


def test_xml_out_and_dry_run(tmp_path):
    xml, vols, pts = psf_scene(str(tmp_path / "a"))
    before = _bytes(xml)
    res = commands.extract_psfs(xml, PsfFakeContext(), "beads", SIZE, view_selection=dict(vi=["0,1"]), dry_run=True)
    assert set(res) == {(0, 1)} and _bytes(xml) == before
    assert not os.path.exists(tmp_path / "a" / "psfs") and not os.path.exists(xml + "~1")
    out = str(tmp_path / "a" / "out.xml")
    commands.extract_psfs(xml, PsfFakeContext(), "beads", SIZE, view_selection=dict(vi=["0,1"]), xml_out=out)
    assert _bytes(xml) == before and _entries(out) == [("0", "1", "psf_t0_vs1.tif")]
    assert os.path.exists(tmp_path / "a" / "psfs" / "psf_t0_vs1.tif")


@pytest.mark.parametrize("kw, match", [
    (dict(psf_size=(19, 19, 24)), "odd"), (dict(psf_size=(19, 19)), "odd"), (dict(psf_size=(0, 1, 1)), "odd"),
    (dict(psf_size=(-1, 1, 1)), "odd"), (dict(psf_size=(3, 3, 2.5)), "odd"), (dict(psf_size=(True, 1, 1)), "odd"),
    (dict(label="nuclei"), "no view has"), (dict(view_selection=dict(vi=["0,0", "0,2"])), r"\[\(0, 2\)\]"),
    (dict(view_selection=dict(vi=["0,0", "0,1"]), empty=(0, 1)), r"\[\(0, 1\)\] have no corresponding"),
])
def test_errors_write_nothing(tmp_path, kw, match):
    xml, vols, pts = psf_scene(str(tmp_path))
    kw = dict(kw)
    empty = kw.pop("empty", None)
    if empty is not None:                                   # points, but none of them corresponds
        data = spimdata.SpimData2.load(xml)
        write_points(str(tmp_path), data, empty, "beads", pts[empty][0], ())
        data.save(xml, backup=False)
    before = _bytes(xml)
    args = dict(label="beads", psf_size=SIZE)
    args.update(kw)
    ctx = PsfFakeContext()
    with pytest.raises(ValueError, match=match):
        commands.extract_psfs(xml, ctx, **args)
    assert _bytes(xml) == before and not os.path.exists(xml + "~1")
    assert not os.path.exists(tmp_path / "psfs") and ctx.windows == []


def test_a_window_the_device_cannot_hold_raises_memory_error(tmp_path):
    xml, vols, pts = psf_scene(str(tmp_path))
    before = _bytes(xml)
    ctx = PsfFakeContext(free_bytes=1000)
    with pytest.raises(MemoryError, match="extract-psfs"):
        commands.extract_psfs(xml, ctx, "beads", SIZE, view_selection=dict(vi=["0,0"]))
    assert _bytes(xml) == before and not os.path.exists(tmp_path / "psfs") and ctx.windows == []


def test_two_ranks_write_what_one_writes(tmp_path):
    xml1, _, _ = psf_scene(str(tmp_path / "one"))
    shutil.copytree(tmp_path / "one", tmp_path / "two")
    xml2 = str(tmp_path / "two" / "dataset.xml")
    run = dict(label="beads", psf_size=SIZE, all_points=True, view_selection=dict(vi=["0,0", "0,1"]))
    one = commands.extract_psfs(xml1, PsfFakeContext(), **run)
    rank1 = {}
    part = commands.extract_psfs(xml2, PsfFakeContext(), shard=(1, 2), allgather=lambda o: [rank1.setdefault(1, o)], **run)
    assert set(part) == {(0, 1)} and not os.path.exists(tmp_path / "two" / "psfs")
    two = commands.extract_psfs(xml2, PsfFakeContext(), shard=(0, 2), allgather=lambda o: [o, rank1[1]], **run)
    assert set(one) == set(two) == {(0, 0), (0, 1)}
    for v in one:
        name = commands.psf_file_name(v)
        assert _bytes(tmp_path / "one" / "psfs" / name) == _bytes(tmp_path / "two" / "psfs" / name)
    assert _entries(xml1) == _entries(xml2)


@pytest.mark.parametrize("nz", [1, 9, 10, 25, 100])
def test_tiff_ifds_and_strips_start_on_word_boundaries(tmp_path, nz):
    import struct
    vol = np.random.default_rng(nz).normal(size=(nz, 3, 5)).astype(np.float32)
    path = str(tmp_path / "s.tif")
    tiff.write_float32_stack(path, vol)
    raw = _bytes(path)
    off = struct.unpack("<I", raw[4:8])[0]
    while off:
        assert off % 2 == 0
        n = struct.unpack("<H", raw[off:off + 2])[0]
        off = struct.unpack("<I", raw[off + 2 + 12 * n:off + 6 + 12 * n])[0]
    tf = tiff.TiffFile(path)
    try:
        assert all(p.offsets[0] % 2 == 0 for p in tf.pages)
        assert np.array_equal(tf.series()[0].read_volume(), vol)
    finally:
        tf.close()
