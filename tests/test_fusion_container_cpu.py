"""create-fusion-container's named bounding boxes (-b), channel / timepoint counts (-ch / -tp) and BigStitcher-project
output (--bdv -xo), and affine-fusion filling those containers, on the CPU through the oracle-backed fake context."""
import copy
import json
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata, viewsource
from bsgpu import zarr as bz
from tests import synth
from tests.fake_ctx import FakeContext


def scene(root, nc=2, nt=2, size=(40, 36, 20), step=28, seed=7, dtype=np.uint16):
    """Two tiles along x for each of ``nc`` channels and ``nt`` timepoints, cut from one field (each channel and
    timepoint scaled differently), as a BDV-N5 dataset.  Returns (xml path, {(tp, setup): [z, y, x] volume})."""
    os.makedirs(root, exist_ok=True)
    G = synth.field((size[2] + 8, size[1] + 8, step + size[0] + 8), seed=seed, sigma=1.0)
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles, vols = [], {}
    for tile in range(2):
        for ch in range(nc):
            s = tile * nc + ch
            tiles.append(dict(setup=s, size_xyz=size, tile=tile, channel=ch, translation_xyz=(step * tile, 0, 0)))
            for t in range(nt):
                v = synth.tile_from(G * (1.0 + 0.3 * ch + 0.1 * t), (2, 3, 2 + step * tile), size[::-1],
                                    100 * t + s, noise=5.0, dtype=dtype)
                bn5.write_bdv_setup(store, s, t, v, (16, 16, 8))
                vols[(t, s)] = v
    xml = spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)
    tree = ET.parse(xml)
    vrs = tree.getroot().find("ViewRegistrations")
    first = list(vrs)
    for t in range(1, nt):
        for vr in first:
            c = copy.deepcopy(vr)
            c.set("timepoint", str(t))
            vrs.append(c)
    tree.getroot().find("SequenceDescription/Timepoints/integerpattern").text = "0" if nt == 1 else f"0-{nt - 1}"
    tree.write(xml, encoding="UTF-8", xml_declaration=True)
    return xml, vols


def _metadata_files(root):
    """{relative path: bytes} of every attributes.json / .zattrs / .zarray / .zgroup under a container."""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f in ("attributes.json", ".zattrs", ".zarray", ".zgroup"):
                p = os.path.join(dp, f)
                out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def _root_attrs(path):
    name = ".zattrs" if os.path.exists(os.path.join(path, ".zgroup")) else "attributes.json"
    return json.load(open(os.path.join(path, name)))["Bigstitcher-Spark"]


# ------------------------------------------------------------------------------------------------ bounding boxes
def test_bounding_boxes_round_trip_unknown_and_duplicated_names(tmp_path):
    xml, _ = scene(str(tmp_path), nc=1, nt=1)
    d = spimdata.SpimData2.load(xml)
    assert d.bounding_boxes() == {}
    d.set_bounding_box("embryo", (3, -4, 2), (30, 20, 15))
    d.set_bounding_box("small", (0, 0, 0), (7, 7, 7))
    d.set_bounding_box("embryo", (5, 6, 1), (25, 26, 11))          # the later definition of a name wins
    d.save(xml)
    e = spimdata.SpimData2.load(xml)
    boxes = e.bounding_boxes()
    assert sorted(boxes) == ["embryo", "small"]
    assert [b.dtype for b in boxes["embryo"]] == [np.int64, np.int64]
    assert [b.tolist() for b in boxes["embryo"]] == [[5, 6, 1], [25, 26, 11]]
    assert [b.tolist() for b in boxes["small"]] == [[0, 0, 0], [7, 7, 7]]
    defs = e.root.findall("BoundingBoxes/BoundingBoxDefinition")
    assert [(b.get("name"), b.findtext("min"), b.findtext("max")) for b in defs][0] == ("embryo", "3 -4 2", "30 20 15")
    out = str(tmp_path / "fused.n5")
    with pytest.raises(ValueError, match="Bounding box 'nothere' not present in XML."):
        commands.create_fusion_container(xml, out, bounding_box="nothere")
    assert not os.path.exists(out)
    commands.create_fusion_container(xml, out, bounding_box="embryo", block_size=(16, 16, 8))
    a = _root_attrs(out)
    assert (a["Boundingbox_min"], a["Boundingbox_max"]) == ([5, 6, 1], [25, 26, 11])
    assert bn5.N5Store(out).dataset_attributes("ch0tp0/s0")["dimensions"] == [21, 21, 11]


@pytest.mark.parametrize("storage", ["N5", "ZARR"])
def test_named_box_with_and_without_anisotropy(tmp_path, storage):
    xml, _ = scene(str(tmp_path), nc=1, nt=1)
    d = spimdata.SpimData2.load(xml)
    d.set_bounding_box("b", (-2, 1, -3), (20, 30, 12))
    d.save(xml)
    plain = str(tmp_path / "plain")
    commands.create_fusion_container(xml, plain, storage=storage, bounding_box="b", block_size=(16, 16, 8))
    a = _root_attrs(plain)
    assert (a["Boundingbox_min"], a["Boundingbox_max"], a["PreserveAnisotropy"]) == ([-2, 1, -3], [20, 30, 12], False)
    assert "AnisotropyFactor" not in a
    # af = 2.5: z from floor(-3 / 2.5) = floor(-1.2) = -2 to ceil(12 / 2.5) = ceil(4.8) = 5; x and y untouched
    aniso = str(tmp_path / "aniso")
    commands.create_fusion_container(xml, aniso, storage=storage, bounding_box="b", preserve_anisotropy=True,
                                     anisotropy_factor=2.5, block_size=(16, 16, 8))
    a = _root_attrs(aniso)
    assert (a["Boundingbox_min"], a["Boundingbox_max"]) == ([-2, 1, -2], [20, 30, 5])
    assert a["PreserveAnisotropy"] is True and a["AnisotropyFactor"] == 2.5
    dims = a["MultiResolutionInfos"][0][0]["dimensions"][:3]
    assert dims == [23, 30, 8]
    with pytest.raises(ValueError, match="anisotropy_factor"):
        commands.create_fusion_container(xml, str(tmp_path / "nan"), storage=storage, bounding_box="b",
                                         preserve_anisotropy=True)


def test_bdv_without_xml_out_is_an_error(tmp_path):
    xml, _ = scene(str(tmp_path), nc=1, nt=1)
    for storage in ("N5", "ZARR"):
        out = str(tmp_path / f"fused_{storage}")
        with pytest.raises(ValueError, match="-xo"):
            commands.create_fusion_container(xml, out, storage=storage, bdv=True)
        assert not os.path.exists(out)


@pytest.mark.parametrize("storage", ["N5", "ZARR"])
def test_channel_and_timepoint_counts(tmp_path, storage):
    xml, vols = scene(str(tmp_path), nc=1, nt=1)
    out = str(tmp_path / "fused")
    commands.create_fusion_container(xml, out, storage=storage, block_size=(16, 16, 8), num_channels=2,
                                     num_timepoints=3)
    a = _root_attrs(out)
    assert (a["NumChannels"], a["NumTimepoints"]) == (2, 3)
    if storage == "N5":
        assert [lv[0]["dataset"] for lv in a["MultiResolutionInfos"]] == [
            f"ch{c}tp{t}/s0" for t in range(3) for c in range(2)]
    else:
        assert len(a["MultiResolutionInfos"]) == 1
        assert bz.ZarrStore(out).array_meta("0")["shape"][:2] == [3, 2]
    ctx = FakeContext()
    # the XML has one channel and one timepoint: the caller has to name the container volume
    for kw in ({}, dict(channel=1), dict(timepoint=2)):
        with pytest.raises(ValueError, match="give channel and timepoint"):
            commands.affine_fusion(out, ctx, **kw)
    with pytest.raises(ValueError, match="outside the container"):
        commands.affine_fusion(out, ctx, channel=2, timepoint=0)
    commands.affine_fusion(out, ctx, channel=1, timepoint=2)
    if storage == "N5":
        st = bn5.N5Store(out)
        got = {(c, t): st.read_volume(f"ch{c}tp{t}/s0") for c in range(2) for t in range(3)}
    else:
        st = bz.ZarrStore(out)
        got = {(c, t): st.read_volume("0", c, t) for c in range(2) for t in range(3)}
    # every view of the XML went into volume (1, 2); the others stay empty
    assert got[(1, 2)].max() > 0 and got[(1, 2)].shape == (20, 36, 68)
    assert all(not v.any() for k, v in got.items() if k != (1, 2))
    ref = str(tmp_path / "ref")
    commands.create_fusion_container(xml, ref, storage=storage, block_size=(16, 16, 8))
    commands.affine_fusion(ref, ctx)
    want = bn5.N5Store(ref).read_volume("ch0tp0/s0") if storage == "N5" else bz.ZarrStore(ref).read_volume("0")
    assert np.array_equal(got[(1, 2)], want)


# ------------------------------------------------------------------------------------------------ BDV layouts
def test_bdv_n5_layout_and_project_xml(tmp_path):
    xml, _ = scene(str(tmp_path), nc=2, nt=2)
    out, xo = str(tmp_path / "fused.n5"), str(tmp_path / "proj" / "fused.xml")
    commands.create_fusion_container(xml, out, block_size=(16, 16, 8), dtype="uint8", bdv=True, xml_out=xo,
                                     downsamplings=[(2, 2, 1), (2, 2, 2)])
    st = bn5.N5Store(out)
    a = _root_attrs(out)
    assert a["FusionFormat"] == "BDV/N5" and a["OutputXML"] == xo and a["InputXML"] == os.path.abspath(xml)
    mr = a["MultiResolutionInfos"]
    # volume (c, t) is entry c + t * NumChannels
    assert [lv[0]["dataset"] for lv in mr] == ["setup0/timepoint0/s0", "setup1/timepoint0/s0",
                                               "setup0/timepoint1/s0", "setup1/timepoint1/s0"]
    assert [l["dataset"] for l in mr[3]] == [f"setup1/timepoint1/s{l}" for l in range(3)]
    for c in range(2):
        assert st.get_attributes(f"setup{c}") == {"downsamplingFactors": [[1, 1, 1], [2, 2, 1], [4, 4, 2]],
                                                  "dataType": "uint8"}
        for t in range(2):
            assert st.get_attributes(f"setup{c}/timepoint{t}") == {"resolution": [1.0, 1.0, 1.0], "multiScale": True}
            dims = [st.dataset_attributes(f"setup{c}/timepoint{t}/s{l}")["dimensions"] for l in range(3)]
            assert dims == [[68, 36, 20], [34, 18, 20], [17, 9, 10]]
    assert not os.path.exists(os.path.join(out, "ch0tp0"))
    p = spimdata.SpimData2.load(xo)
    assert p.image_loader() == ("bdv.n5", out)
    assert p.root.findtext("SequenceDescription/ImageLoader/n5") == "../fused.n5"
    assert sorted(p.setups) == [0, 1] and p.timepoints == [0, 1] and p.view_ids() == [(t, c) for t in (0, 1) for c in (0, 1)]
    assert all(p.setups[c].size == (68, 36, 20) and p.setups[c].attributes == dict(illumination=0, channel=c, tile=0, angle=0)
               for c in range(2))
    assert p.channels_ordered() == [0, 1] and np.array_equal(p.model(1, 1), np.eye(4)[:3])
    assert p.registrations[(1, 1)][0][0] == "calibration"
    vs = p.root.find("SequenceDescription/ViewSetups/ViewSetup")
    assert (vs.findtext("name"), vs.findtext("voxelSize/unit"), vs.findtext("voxelSize/size")) == (
        "setup 0", "micrometer", "1.0 1.0 1.0")
    src = viewsource.open_views(p)
    assert src.mipmap_info((1, 0))[0] == [(1, 1, 1), (2, 2, 1), (4, 4, 2)] and src.level_dims((1, 1), 2) == (17, 9, 10)
    # anisotropy: voxel size and calibration (1, 1, af)
    xa = str(tmp_path / "aniso.xml")
    commands.create_fusion_container(xml, str(tmp_path / "aniso.n5"), block_size=(16, 16, 8), bdv=True, xml_out=xa,
                                     preserve_anisotropy=True, anisotropy_factor=2.0)
    pa = spimdata.SpimData2.load(xa)
    assert np.array_equal(pa.model(0, 0), np.diag([1.0, 1.0, 2.0, 1.0])[:3])
    assert pa.root.findtext("SequenceDescription/ViewSetups/ViewSetup/voxelSize/size") == "1.0 1.0 2.0"
    assert pa.setups[0].size == (68, 36, 11)          # z: 0 .. ceil(19 / 2)


def test_bdv_zarr_loader_xml(tmp_path):
    xml, _ = scene(str(tmp_path), nc=2, nt=2)
    out, xo = str(tmp_path / "fused.zarr"), str(tmp_path / "fused.xml")
    commands.create_fusion_container(xml, out, block_size=(16, 16, 8), bdv=True, xml_out=xo, downsamplings=[(2, 2, 1)])
    a = _root_attrs(out)
    assert a["FusionFormat"] == "BDV/OME-ZARR" and a["OutputXML"] == xo
    p = spimdata.SpimData2.load(xo)
    assert p.image_loader() == ("bdv.multimg.zarr", out)
    assert p.zarr_groups() == {(t, c): ("", c, t) for c in range(2) for t in range(2)}
    zg = p.root.findall("SequenceDescription/ImageLoader/zgroups/zgroup")
    assert [(g.get("setup"), g.get("tp"), g.get("path"), g.get("indicies")) for g in zg] == [
        ("0", "0", "", "[0, 0]"), ("1", "0", "", "[1, 0]"), ("0", "1", "", "[0, 1]"), ("1", "1", "", "[1, 1]")]
    src = viewsource.open_views(p)
    assert src.mipmap_info((1, 1))[0] == [(1, 1, 1), (2, 2, 1)] and src.level_dims((0, 1), 1) == (34, 18, 20)
    # the arrays are those of the plain container
    plain = str(tmp_path / "plain.zarr")
    commands.create_fusion_container(xml, plain, block_size=(16, 16, 8), downsamplings=[(2, 2, 1)])
    assert {k: v for k, v in _metadata_files(out).items() if k != ".zattrs"} == \
        {k: v for k, v in _metadata_files(plain).items() if k != ".zattrs"}


# ------------------------------------------------------------------------------------------------ defaults unchanged
@pytest.mark.parametrize("storage", ["N5", "ZARR"])
def test_defaults_write_the_same_metadata_bytes(tmp_path, storage):
    xml, _ = scene(str(tmp_path), nc=2, nt=2)
    kw = dict(storage=storage, block_size=(16, 16, 8), dtype="uint16", downsamplings=[(2, 2, 1)])
    base = str(tmp_path / "base")
    commands.create_fusion_container(xml, base, **kw)
    # the new options at their defaults, the XML's own counts, and a named box equal to the box of all views
    lo, hi = [_root_attrs(base)[k] for k in ("Boundingbox_min", "Boundingbox_max")]
    d = spimdata.SpimData2.load(xml)
    d.set_bounding_box("all", lo, hi)
    d.save(xml)
    for i, extra in enumerate((dict(bounding_box=None, bdv=False, xml_out=None, num_channels=None, num_timepoints=None),
                               dict(num_channels=2, num_timepoints=2), dict(bounding_box="all"))):
        other = str(tmp_path / f"other{i}")
        commands.create_fusion_container(xml, other, **kw, **extra)
        assert _metadata_files(other) == _metadata_files(base)
    assert len(_metadata_files(base)) >= (3 if storage == "ZARR" else 9)


def test_affine_fusion_writes_the_same_voxels_into_every_layout(tmp_path):
    xml, _ = scene(str(tmp_path), nc=2, nt=2)
    ctx = FakeContext()
    kw = dict(block_size=(16, 16, 8), dtype="uint16", min_intensity=0.0, max_intensity=3000.0,
              downsamplings=[(2, 2, 1), (2, 2, 2)])
    got = {}
    for name, storage, bdv in (("n5", "N5", False), ("bdv_n5", "N5", True), ("zarr", "ZARR", False),
                               ("bdv_zarr", "ZARR", True)):
        out, xo = str(tmp_path / name), str(tmp_path / f"{name}.xml")
        commands.create_fusion_container(xml, out, storage=storage, bdv=bdv, xml_out=xo if bdv else None, **kw)
        commands.affine_fusion(out, ctx, "AVG_BLEND", block_scale=(2, 2, 1))
        if bdv:       # read back through the project XML
            src = viewsource.open_views(spimdata.SpimData2.load(xo))
            got[name] = {(c, t, l): src.read_volume((t, c), l) for c in range(2) for t in range(2) for l in range(3)}
        else:
            meta = (bn5.read_fusion_container if storage == "N5" else bz.read_fusion_container_zarr)(out)[1]
            st = bn5.N5Store(out) if storage == "N5" else bz.ZarrStore(out)
            got[name] = {(c, t, l): (st.read_volume(meta["mr_infos"][c + 2 * t][l]["dataset"]) if storage == "N5"
                                     else st.read_volume(str(l), c, t))
                         for c in range(2) for t in range(2) for l in range(3)}
    assert not ctx.vols
    for k, v in got["n5"].items():
        assert v.dtype == np.uint16 and v.max() > 0
        for name in ("bdv_n5", "zarr", "bdv_zarr"):
            assert np.array_equal(got[name][k], v), (name, k)
    # every (channel, timepoint) volume holds its own views
    assert not np.array_equal(got["n5"][(0, 0, 0)], got["n5"][(1, 0, 0)])
    assert not np.array_equal(got["n5"][(0, 0, 0)], got["n5"][(0, 1, 0)])


def test_readme_example_named_box_bdv_n5_multires(tmp_path):
    """`create-fusion-container -x dataset.xml -o fused.n5 -xo dataset-fused.xml -s N5 -b embryo --bdv --multiRes -d
    UINT8` followed by `affine-fusion -o fused.n5`, on a dataset large enough for a two-level pyramid."""
    xml, vols = scene(str(tmp_path), nc=1, nt=1, size=(150, 140, 16), step=100)
    d = spimdata.SpimData2.load(xml)
    d.set_bounding_box("embryo", (20, 4, 2), (229, 135, 13))
    d.save(xml)
    out, xo = str(tmp_path / "fused.n5"), str(tmp_path / "dataset-fused.xml")
    commands.create_fusion_container(xml, out, storage="N5", bounding_box="embryo", bdv=True, xml_out=xo,
                                     multi_res=True, dtype="uint8", max_intensity=3000.0, block_size=(64, 64, 8))
    commands.affine_fusion(out, FakeContext())
    p = spimdata.SpimData2.load(xo)
    src = viewsource.open_views(p)
    factors = src.mipmap_info((0, 0))[0]
    assert factors == [(1, 1, 1), (2, 2, 1)] and p.setups[0].size == (210, 132, 12)
    s0 = src.read_volume((0, 0), 0)
    assert s0.dtype == np.uint8 and s0.shape == (12, 132, 210) and s0.max() > 0
    assert src.read_volume((0, 0), 1).shape == (12, 66, 105)
    # the same box out of a fusion of every view
    full = str(tmp_path / "full.n5")
    commands.create_fusion_container(xml, full, storage="N5", dtype="uint8", max_intensity=3000.0, block_size=(64, 64, 8))
    commands.affine_fusion(full, FakeContext(), block_scale=(1, 1, 1))
    lo = _root_attrs(full)["Boundingbox_min"]
    f0 = bn5.N5Store(full).read_volume("ch0tp0/s0")
    o = [20 - lo[0], 4 - lo[1], 2 - lo[2]]
    assert np.array_equal(s0, f0[o[2]:o[2] + 12, o[1]:o[1] + 132, o[0]:o[0] + 210])
