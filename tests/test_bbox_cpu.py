"""estimate-bounding-box on the CPU: the oracle (box minimum, threshold, grid mapping) and the command end to end through
an oracle-backed context, including the chain estimate -> create-fusion-container -b -> affine-fusion."""
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata
from oracle import bbox_oracle as bo
from tests.fake_ctx import FakeContext
from tests.test_fusion_container_cpu import _root_attrs

OBJECT = ((30, 20, 8), (80, 70, 32))                       # world min / max (inclusive) of the bright object
BEADS = [(100, 100, 20), (12, 102, 10), (102, 14, 28), (14, 10, 20)]   # beads away from the object (x, y, z)


class BboxFakeContext(FakeContext):
    """FakeContext plus the estimate-bounding-box entries, computed by the oracle."""

    def __init__(self, free_bytes=1 << 40):
        super().__init__()
        self.free_bytes = free_bytes

    def memory_free(self):
        return self.free_bytes

    def volume_empty(self, dims_xyz):
        h = self.volume_upload(np.zeros(tuple(int(v) for v in dims_xyz)[::-1], dtype=np.float32))
        return h, self.vols[h]

    def min_filter(self, h, radius_xyz):
        return self.volume_upload(bo.min_filter(self.vols[h], tuple(int(v) for v in radius_xyz)))

    def volume_min_max(self, h):
        v = self.vols[h]
        return float(np.nanmin(v)), float(np.nanmax(v))

    def threshold_bbox(self, h, t):
        return bo.threshold_bbox(self.vols[h], t)


def bbox_scene(root, tile=(64, 64, 40), step=56, seed=3):
    """2 x 2 uint16 tiles (overlap 8 px) cut from one world volume: background ~100 with noise, a bright object over
    OBJECT, crossing all four tiles, and Gaussian beads (sigma 1, peak ~3000) at BEADS.  BDV-N5 dataset.  Returns
    (xml path, world volume [z, y, x] float64)."""
    os.makedirs(root, exist_ok=True)
    rng = np.random.default_rng(seed)
    shape = (tile[2], step + tile[1], step + tile[0])
    world = 100.0 + rng.normal(0.0, 3.0, shape)
    (x0, y0, z0), (x1, y1, z1) = OBJECT
    world[z0:z1 + 1, y0:y1 + 1, x0:x1 + 1] += 900.0
    zz, yy, xx = np.mgrid[0:shape[0], 0:shape[1], 0:shape[2]]
    for (bx, by, bz) in BEADS:
        world += 3000.0 * np.exp(-((xx - bx) ** 2 + (yy - by) ** 2 + (zz - bz) ** 2) / 2.0)
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    for j in range(2):
        for i in range(2):
            s = 2 * j + i
            v = world[:, step * j:step * j + tile[1], step * i:step * i + tile[0]]
            bn5.write_bdv_setup(store, s, 0, np.clip(np.rint(v), 0, 65535).astype(np.uint16), (32, 32, 16))
            tiles.append(dict(setup=s, size_xyz=tile, tile=s, translation_xyz=(step * i, step * j, 0)))
    return spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles), world


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _definitions(xml, name):
    return [b for b in ET.parse(xml).getroot().findall("BoundingBoxes/BoundingBoxDefinition") if b.get("name") == name]


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("shape,r", [((5, 7, 9), 1), ((6, 5, 11), 2), ((4, 6, 5), 20), ((1, 6, 8), 2),
                                     ((7, 1, 6), (1, 3, 2)), ((9, 8, 1), (0, 1, 4))])
def test_oracle_min_filter_equals_brute_force(shape, r):
    rng = np.random.default_rng(sum(shape))
    v = rng.normal(0.0, 100.0, shape).astype(np.float32)
    np.testing.assert_array_equal(bo.min_filter(v, r), bo.brute_min_filter(v, r))


def test_oracle_min_filter_ignores_nan():
    rng = np.random.default_rng(1)
    v = rng.uniform(0.0, 1.0, (6, 7, 8)).astype(np.float32)
    v[3, 2, 4] = np.nan
    v[0, 0, 0:2] = np.nan
    got = bo.min_filter(v, 1)
    np.testing.assert_array_equal(got, bo.brute_min_filter(v, 1))
    assert not np.isnan(got).any()
    w = np.full((3, 3, 3), np.nan, np.float32)
    w[2, 2, 2] = 5.0
    got = bo.min_filter(w, 1)
    np.testing.assert_array_equal(got, bo.brute_min_filter(w, 1))
    assert np.isnan(got[0, 0, 0]) and got[1, 1, 1] == 5.0          # a box of NaNs only stays NaN


def test_bead_vanishes_and_object_survives():
    v = np.full((30, 30, 30), 10.0, np.float32)
    v[4:7, 4:7, 4:7] = 1000.0                                     # a 3-voxel bead
    v[10:25, 12:27, 8:23] = 500.0                                 # a 15-voxel object
    f = bo.min_filter(v, 2)
    assert f[4:7, 4:7, 4:7].max() == 10.0
    assert f[12:23, 14:25, 10:21].min() == 500.0 and f[17, 19, 15] == 500.0
    mn, mx, n = bo.threshold_bbox(f, 100.0)
    assert (mn, mx, n) == ((10, 14, 12), (20, 24, 22), 11 ** 3)


def test_voxel_exactly_at_the_threshold_is_excluded():
    v = np.zeros((4, 5, 6), np.float32)
    v[1, 2, 3] = 100.0
    v[2, 3, 4] = 50.0
    t = bo.threshold(0.0, 100.0, 50.0)
    assert t == 50.0
    assert bo.threshold_bbox(v, t) == ((3, 2, 1), (3, 2, 1), 1)
    assert bo.threshold_bbox(v, np.nextafter(50.0, 0.0)) == ((3, 2, 1), (4, 3, 2), 2)
    assert bo.threshold_bbox(v, 100.0) == ((-1, -1, -1), (-1, -1, -1), 0)


def test_grid_and_world_mapping_by_hand():
    lo, hi, ds = (-9, 3, 0), (30, 17, 7), 4
    g_min, dims = commands.bounding_box_grid(lo, hi, ds)
    # floor(-9 / 4) = -3, floor(3 / 4) = 0, floor(0 / 4) = 0; ceil(30 / 4) = 8, ceil(17 / 4) = 5, ceil(7 / 4) = 2
    assert g_min.tolist() == [-3, 0, 0] and dims.tolist() == [12, 6, 3]
    og, od = bo.grid(lo, hi, ds)
    assert og.tolist() == g_min.tolist() and od.tolist() == dims.tolist()
    # kept voxels x 0..5, y 2..5, z 0..2: world 4 (g_min + i - 1) .. 4 (g_min + i + 1), then clipped to [lo, hi]
    wmin, wmax = bo.world_box((0, 2, 0), (5, 5, 2), g_min, ds, lo, hi)
    assert wmin.tolist() == [-9, 4, 0]          # -16 clipped to -9; 4 (0 + 2 - 1) = 4; -4 clipped to 0
    assert wmax.tolist() == [12, 17, 7]         # 4 (-3 + 5 + 1) = 12; 24 clipped to 17; 12 clipped to 7
    assert bo.radius(25, 4) == 6 and bo.radius(2, 4) == 1 and bo.radius(0, 1) == 1 and bo.radius(10, 4) == 3


# ------------------------------------------------------------------------------------------------ the command
def test_views_bounding_box_is_the_box_create_fusion_container_fuses(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    d = spimdata.SpimData2.load(xml)
    lo, hi = commands.views_bounding_box(d, d.view_ids())
    assert lo.tolist() == [0, 0, 0] and hi.tolist() == [119, 119, 39]
    commands.create_fusion_container(xml, str(tmp_path / "f.n5"), block_size=(32, 32, 16))
    a = _root_attrs(str(tmp_path / "f.n5"))
    assert (a["Boundingbox_min"], a["Boundingbox_max"]) == ([0, 0, 0], [119, 119, 39])


def test_command_finds_the_object_and_drops_the_beads(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    ctx = BboxFakeContext()
    ds, size = 2, 8
    res = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=ds, discarded_object_size=size)
    r = res["radius"]
    assert r == 4 and res["dims"] == [61, 61, 21]
    lo, hi = np.array(res["min"]), np.array(res["max"])
    # the min filter erodes the object by r downsampled voxels, the margin adds one back on each side
    omin, omax = np.array(OBJECT[0]), np.array(OBJECT[1])
    assert np.all(lo >= omin - ds) and np.all(hi <= omax + ds), res
    assert np.all(lo <= omin + (r + 1) * ds) and np.all(hi >= omax - (r + 1) * ds), res
    for b in BEADS:
        assert not np.all((np.array(b) >= lo) & (np.array(b) <= hi)), b
    # the command's result is the oracle's B3-B5 on the same fused grid
    d = spimdata.SpimData2.load(xml)
    vlo, vhi = (b.astype(np.int64) for b in commands.views_bounding_box(d, d.view_ids()))
    g_min, dims = commands.bounding_box_grid(vlo, vhi, ds)
    h, fused = ctx.volume_empty(dims)
    commands.fuse_downsampled(ctx, d, commands.bvs.open_views(d), d.view_ids(), ds, g_min, dims, fused)
    want = bo.estimate(fused, vlo, vhi, ds, 5.0, size)
    assert {k: res[k] for k in want} == want
    assert res["count"] > 0 and res["min_max"][1] > 2500.0
    assert [b.tolist() for b in spimdata.SpimData2.load(xml).bounding_boxes()["auto"]] == [res["min"], res["max"]]


def test_second_run_replaces_the_definition_and_keeps_a_backup(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    d = spimdata.SpimData2.load(xml)
    d.set_bounding_box("other", (1, 2, 3), (4, 5, 6))
    d.save(xml, backup=False)
    ctx = BboxFakeContext()
    before = _bytes(xml)
    a = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=2, discarded_object_size=8)
    assert _bytes(xml + "~1") == before
    b = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=4, discarded_object_size=8, background_intensity=10)
    assert len(_definitions(xml, "auto")) == 1 and len(_definitions(xml, "other")) == 1
    boxes = spimdata.SpimData2.load(xml).bounding_boxes()
    assert [v.tolist() for v in boxes["auto"]] == [b["min"], b["max"]]
    assert [v.tolist() for v in boxes["other"]] == [[1, 2, 3], [4, 5, 6]]
    assert a["dims"] != b["dims"]


def test_dry_run_leaves_the_xml_unchanged(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    before = _bytes(xml)
    res = commands.estimate_bounding_box(xml, BboxFakeContext(), "auto", downsampling=2, discarded_object_size=8,
                                         dry_run=True)
    assert res["count"] > 0
    assert _bytes(xml) == before and not os.path.exists(xml + "~1")


@pytest.mark.parametrize("kw,match", [
    (dict(name=""), "name"),
    (dict(downsampling=0), "downsampling"),
    (dict(downsampling=1.5), "downsampling"),
    (dict(background_intensity=-1.0), "background"),
    (dict(background_intensity=100.5), "background"),
    (dict(discarded_object_size=-1), "minObjectSize"),
    (dict(view_selection=dict(vi=["5,5"])), "No views"),
    (dict(background_intensity=100.0), "threshold"),       # nothing is strictly above the maximum
])
def test_errors_leave_the_xml_unchanged(tmp_path, kw, match):
    xml, _ = bbox_scene(str(tmp_path))
    before = _bytes(xml)
    args = dict(name="auto", downsampling=4, discarded_object_size=8)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        commands.estimate_bounding_box(xml, BboxFakeContext(), args.pop("name"), **args)
    assert _bytes(xml) == before and not os.path.exists(xml + "~1")


def test_a_grid_the_device_cannot_hold_raises_memory_error(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    before = _bytes(xml)
    # ds 1: 120 x 120 x 40 voxels, 12 bytes each, plus four 64 x 64 x 40 float32 sources
    need = 12 * 120 * 120 * 40 + 4 * 4 * 64 * 64 * 40
    with pytest.raises(MemoryError, match="larger --downsampling"):
        commands.estimate_bounding_box(xml, BboxFakeContext(free_bytes=need - 1), "auto", downsampling=1)
    commands.estimate_bounding_box(xml, BboxFakeContext(free_bytes=need), "auto", downsampling=1,
                                   discarded_object_size=8, dry_run=True)
    assert _bytes(xml) == before


def test_estimate_then_fuse_the_box(tmp_path):
    xml, _ = bbox_scene(str(tmp_path))
    ctx = BboxFakeContext()
    res = commands.estimate_bounding_box(xml, ctx, "auto", downsampling=2, discarded_object_size=8)
    out = str(tmp_path / "box.n5")
    commands.create_fusion_container(xml, out, bounding_box="auto", block_size=(32, 32, 16))
    commands.affine_fusion(out, ctx)
    size = [res["max"][d] - res["min"][d] + 1 for d in range(3)]
    got = bn5.N5Store(out).read_volume("ch0tp0/s0")
    assert got.shape == tuple(size[::-1])
    assert got.min() > 500.0           # the eroded object with one voxel of margin lies inside the bright object
