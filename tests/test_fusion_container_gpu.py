"""Named bounding boxes and BigStitcher-project containers on the device: a box on the super-block grid of the full
extent fuses to exactly the matching sub-array at every level, an unaligned box meets the fusion oracle's bar, the
BDV/N5 and BDV/OME-ZARR projects hold the same bits as the plain containers, and a fused BDV/N5 project feeds
detect-interestpoints."""
import os

import numpy as np
import pytest

from bsgpu import commands, fusion, n5 as bn5, spimdata, viewsource
from bsgpu import zarr as bz
from oracle import fusion_oracle as fo
from tests import test_fusion_gpu
from tests.test_fusion_container_cpu import _root_attrs, scene

pytestmark = pytest.mark.gpu

STEPS = [(2, 2, 1), (2, 2, 2)]
KW = dict(block_size=(64, 32, 16), min_intensity=0.0, max_intensity=3000.0, downsamplings=STEPS)


def _levels(out, c=0, t=0):
    """Every level of volume (c, t) of a plain N5 or OME-ZARR fusion container."""
    a = _root_attrs(out)
    if a["FusionFormat"] == "N5":
        st = bn5.N5Store(out)
        return [st.read_volume(lv["dataset"]) for lv in a["MultiResolutionInfos"][c + t * a["NumChannels"]]]
    st = bz.ZarrStore(out)
    return [st.read_volume(lv["dataset"], c, t) for lv in a["MultiResolutionInfos"][0]]


def _with_box(xml, name, lo, hi):
    d = spimdata.SpimData2.load(xml)
    d.set_bounding_box(name, lo, hi)
    d.save(xml)


@pytest.mark.parametrize("dtype", ["uint16", "float32"])
def test_aligned_box_is_the_sub_array_of_the_full_fusion(ctx, tmp_path, dtype):
    xml, _ = scene(str(tmp_path), nc=1, nt=1, size=(200, 150, 48), step=150)
    full = str(tmp_path / "full.n5")
    commands.create_fusion_container(xml, full, dtype=dtype, **KW)
    lo = np.array(_root_attrs(full)["Boundingbox_min"])
    compute = (128, 64, 16)                      # block_size x the default block scale (2, 2, 1)
    off = np.array([compute[0], compute[1], compute[2]])
    size = np.array([150, 70, 25])
    _with_box(xml, "aligned", lo + off, lo + off + size - 1)
    box = str(tmp_path / "box.n5")
    commands.create_fusion_container(xml, box, dtype=dtype, bounding_box="aligned", **KW)
    for out in (full, box):
        commands.affine_fusion(out, ctx, "AVG_BLEND")
    f, b = _levels(full), _levels(box)
    absd = [(1, 1, 1), (2, 2, 1), (4, 4, 2)]
    for l, (fl, bl) in enumerate(zip(f, b)):
        o = off // absd[l]
        assert bl.shape == tuple((size // absd[l])[::-1])
        assert np.array_equal(bl, fl[o[2]:o[2] + bl.shape[0], o[1]:o[1] + bl.shape[1], o[0]:o[0] + bl.shape[2]]), l
    assert b[0].max() > 0


def test_unaligned_box_meets_the_fusion_oracle(ctx, tmp_path):
    xml, vols = scene(str(tmp_path), nc=1, nt=1, size=(200, 150, 48), step=150)
    lo, size = np.array([37, 21, 5]), np.array([230, 100, 30])
    _with_box(xml, "b", lo, lo + size - 1)
    out = str(tmp_path / "box.zarr")
    commands.create_fusion_container(xml, out, dtype="float32", bounding_box="b", block_size=(64, 32, 16))
    commands.affine_fusion(out, ctx, "AVG_BLEND")
    got = bz.ZarrStore(out).read_volume("0")
    d = spimdata.SpimData2.load(xml)
    views = []
    for v in d.view_ids():
        M = d.model(*v)
        border, rng = fusion.adjust_blending(M)
        views.append(fo.View(vols[v], M, border, rng))
    want = fo.fuse_block(views, tuple(int(x) for x in lo), tuple(int(x) for x in size), fo.AVG_BLEND)
    test_fusion_gpu._run.last = (views, tuple(int(x) for x in lo), tuple(int(x) for x in size))
    test_fusion_gpu._assert_close(got, want)
    assert np.count_nonzero(want) > 0.9 * want.size


def test_bdv_projects_hold_the_plain_containers_bits(ctx, tmp_path):
    xml, _ = scene(str(tmp_path), nc=2, nt=2, size=(160, 96, 32), step=120)
    for storage in ("N5", "ZARR"):
        plain, bdv, xo = (str(tmp_path / n) for n in (f"plain_{storage}", f"bdv_{storage}", f"bdv_{storage}.xml"))
        commands.create_fusion_container(xml, plain, storage=storage, dtype="uint16", **KW)
        commands.create_fusion_container(xml, bdv, storage=storage, dtype="uint16", bdv=True, xml_out=xo, **KW)
        for out in (plain, bdv):
            commands.affine_fusion(out, ctx, "AVG_BLEND")
        src = viewsource.open_views(spimdata.SpimData2.load(xo))
        for c in range(2):
            for t in range(2):
                want = _levels(plain, c, t)
                assert len(src.mipmap_info((t, c))[0]) == len(want) == 3
                for l, w in enumerate(want):
                    assert np.array_equal(src.read_volume((t, c), l), w), (storage, c, t, l)
                assert want[0].max() > 0
        assert not np.array_equal(_levels(plain, 0, 0)[0], _levels(plain, 1, 1)[0])


def test_fused_bdv_n5_project_feeds_detect_interestpoints(ctx, tmp_path):
    from tests.test_interestpoints_gpu import _beads
    rng = np.random.default_rng(11)
    world = []
    while len(world) < 30:                              # beads at least 10 px apart, away from the volume's faces
        p = np.array([rng.uniform(8, 184), rng.uniform(8, 88), rng.uniform(5, 19)])
        if all(np.linalg.norm(p - q) >= 10 for q in world):
            world.append(p)
    world = np.array(world)
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles = []
    for s, tx in enumerate((0, 64)):
        vol = _beads((24, 96, 128), [tuple(p) for p in world - (tx, 0, 0)], 1 + s, sigma_xy=1.6, sigma_z=1.6)
        bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 16))
        tiles.append(dict(setup=s, size_xyz=(128, 96, 24), tile=s, translation_xyz=(tx, 0, 0)))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    _with_box(xml, "embryo", (4, 2, 1), (187, 93, 22))
    out, xo = str(tmp_path / "fused.n5"), str(tmp_path / "fused" / "dataset-fused.xml")
    commands.create_fusion_container(xml, out, storage="N5", bounding_box="embryo", bdv=True, xml_out=xo,
                                     dtype="uint16", block_size=(64, 32, 8), downsamplings=[(2, 2, 1)])
    commands.affine_fusion(out, ctx, "AVG_BLEND")
    res = commands.detect_interestpoints(xo, ctx, "beads", sigma=1.6, threshold=0.01, min_intensity=0.0,
                                         max_intensity=1000.0, downsample_xy=1, block_size=(64, 64, 24))
    loc = res[(0, 0)][0]
    want = world - (4, 2, 1)                            # the fused frame starts at the box minimum
    dist = np.array([np.min(np.linalg.norm(loc - p, axis=1)) for p in want])
    assert np.all(dist < 0.5), (dist.max(), want[np.argmax(dist)])
    assert len(loc) >= len(want)
    assert os.path.isdir(tmp_path / "fused" / "interestpoints.n5")
    assert spimdata.SpimData2.load(xo).interest_points()[(0, 0)]["beads"]["path"] == "tpId_0_viewSetupId_0/beads"
