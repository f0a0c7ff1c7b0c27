"""TIFF datasets (`spimreconstruction.filemap2`) on the CPU: the reader against Pillow-written files and against files
assembled byte by byte (both byte orders, BigTIFF, tiles, Deflate + Predictor 2, the ImageJ and OME-TIFF layouts),
region reads and what they touch, the refusals, the loader XML and its frame rule, and resave / affine-fusion giving
the same bytes from a TIFF dataset as from the N5 twin.  Driven through the oracle-backed fake context."""
import io
import os
import shutil

import numpy as np
import pytest
from PIL import Image

from bsgpu import commands, spimdata, tiff, viewsource
from bsgpu import zarr as bz
from tests import synth
from tests.fake_ctx import FakeContext
from tests.tiff_files import imagej_description, twin_datasets, write_tiff


def _vol(shape, dtype, seed):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype) == np.float32:
        return (rng.standard_normal(shape) * 1e3).astype(np.float32)
    return rng.integers(0, np.iinfo(dtype).max, shape, endpoint=True).astype(dtype)


def _series(path, i=0):
    return tiff.TiffFile(str(path)).series()[i]


# ------------------------------------------------------------------------------------------------ against Pillow
@pytest.mark.parametrize("compression", [None, "tiff_deflate", "tiff_adobe_deflate", "packbits"])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("strip_size", [None, 700])
def test_pillow_multipage_files(tmp_path, compression, dtype, strip_size):
    vol = _vol((5, 37, 53), dtype, 1)
    vol[:, :10, :10] = vol[0, 0, 0]                           # runs PackBits can repeat
    ims = [Image.fromarray(p) for p in vol]
    kw = {} if compression is None else dict(compression=compression)
    if strip_size:
        kw["strip_size"] = strip_size
    ims[0].save(tmp_path / "p.tif", save_all=True, append_images=ims[1:], **kw)
    tf = tiff.TiffFile(str(tmp_path / "p.tif"))
    if strip_size and compression:
        assert len(tf.pages[0].offsets) > 1                   # more than one strip per plane
    s = tf.series()[0]
    got = s.read_volume()
    assert s.dims == (53, 37, 5) and got.dtype == vol.dtype and np.array_equal(got, vol)
    assert got.tobytes() == vol.tobytes()


# ------------------------------------------------------------------------------------------------ hand-assembled
def test_big_endian_strips(tmp_path):
    vol = _vol((4, 11, 13), np.uint16, 2)
    p = write_tiff(tmp_path / "be.tif", list(vol), order=">", rows_per_strip=3)
    assert open(p, "rb").read(4) == b"MM\x00\x2a"
    tf = tiff.TiffFile(p)
    assert tf.order == ">" and len(tf.pages[0].offsets) == 4
    assert np.array_equal(tf.series()[0].read_volume(), vol)
    f = write_tiff(tmp_path / "bef.tif", list(_vol((2, 9, 7), np.float32, 3)), order=">", compression=8)
    assert np.array_equal(_series(f).read_volume(), _vol((2, 9, 7), np.float32, 3))


@pytest.mark.parametrize("order", ["<", ">"])
def test_bigtiff(tmp_path, order):
    vol = _vol((3, 17, 19), np.uint16, 4)
    p = write_tiff(tmp_path / "b.tif", list(vol), order=order, big=True, rows_per_strip=5, compression=32946)
    head = open(p, "rb").read(8)
    assert head[2:4] == (b"\x2b\x00" if order == "<" else b"\x00\x2b")
    tf = tiff.TiffFile(p)
    assert tf.big and np.array_equal(tf.series()[0].read_volume(), vol)


@pytest.mark.parametrize("compression", [1, 8])
def test_tiles_with_partial_edge_tiles(tmp_path, compression):
    vol = _vol((3, 29, 37), np.uint16, 5)
    p = write_tiff(tmp_path / "t.tif", list(vol), tile=(16, 16), compression=compression)
    tf = tiff.TiffFile(p)
    assert tf.pages[0].tile == (16, 16) and len(tf.pages[0].offsets) == 6
    s = tf.series()[0]
    assert np.array_equal(s.read_volume(), vol)
    assert np.array_equal(s.read_region((14, 15, 1), (20, 14, 2)), vol[1:3, 15:29, 14:34])


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_deflate_with_horizontal_predictor(tmp_path, dtype):
    vol = _vol((3, 13, 21), dtype, 6)
    vol[0, :, 0] = np.iinfo(dtype).max                        # differences that wrap
    vol[0, :, 1] = 0
    for order in "<>":
        p = write_tiff(tmp_path / f"pr{order == '<'}.tif", list(vol), order=order, compression=8, predictor=2,
                       rows_per_strip=4)
        tf = tiff.TiffFile(p)
        assert tf.pages[0].predictor == 2
        assert np.array_equal(tf.series()[0].read_volume(), vol)


def _hyperstack(c, z, t, shape=(7, 9), dtype=np.uint16):
    """Planes with known values: plane (c, z, t) is 1000 c + 100 z + 10 t plus the pixel's (y + x) % 7."""
    yy, xx = np.mgrid[0:shape[0], 0:shape[1]]
    return {(ci, zi, ti): (1000 * ci + 100 * zi + 10 * ti + (yy + xx) % 7).astype(dtype)
            for ci in range(c) for zi in range(z) for ti in range(t)}


def test_imagej_hyperstack(tmp_path):
    planes = _hyperstack(2, 3, 2)
    order = [planes[(c, z, t)] for t in range(2) for z in range(3) for c in range(2)]      # czt, channel fastest
    p = write_tiff(tmp_path / "ij.tif", order, description=imagej_description(2, 3, 2))
    s = _series(p)
    assert (s.channels, s.slices, s.frames, s.dims) == (2, 3, 2, (9, 7, 3))
    for c in range(2):
        for t in range(2):
            assert np.array_equal(s.read_volume(c, t), np.stack([planes[(c, z, t)] for z in range(3)]))


def test_imagej_single_ifd_contiguous_planes(tmp_path):
    planes = _hyperstack(2, 3, 2)
    order = [planes[(c, z, t)] for t in range(2) for z in range(3) for c in range(2)]
    p = write_tiff(tmp_path / "ijc.tif", order, description=imagej_description(2, 3, 2), contiguous=True,
                   rows_per_strip=2, order=">")
    tf = tiff.TiffFile(p)
    assert len(tf.pages) == 1
    s = tf.series()[0]
    for c in range(2):
        for t in range(2):
            assert np.array_equal(s.read_volume(c, t), np.stack([planes[(c, z, t)] for z in range(3)]))
    assert np.array_equal(s.read_region((2, 3, 1), (4, 2, 1), 1, 1)[0], planes[(1, 1, 1)][3:5, 2:6])


OME_TWO_SERIES = """<?xml version="1.0" encoding="UTF-8"?>
<OME xmlns="http://www.openmicroscopy.org/Schemas/OME/2016-06" UUID="urn:uuid:1">
  <Image ID="Image:0" Name="tile0"><Pixels ID="Pixels:0" DimensionOrder="XYCZT" Type="uint16" SizeX="9" SizeY="7"
    SizeZ="3" SizeC="2" SizeT="1"><TiffData IFD="0" PlaneCount="6"/></Pixels></Image>
  <Image ID="Image:1" Name="tile1"><Pixels ID="Pixels:1" DimensionOrder="XYCZT" Type="uint16" SizeX="9" SizeY="7"
    SizeZ="3" SizeC="2" SizeT="1">{tiffdata}</Pixels></Image>
</OME>"""


@pytest.mark.parametrize("tiffdata", [
    '<TiffData IFD="6" PlaneCount="6"/>',
    # one element per plane, in a shuffled order
    "".join(f'<TiffData IFD="{6 + 2 * z + c}" FirstZ="{z}" FirstC="{c}" PlaneCount="1"/>'
            for z, c in ((2, 1), (0, 0), (1, 1), (0, 1), (2, 0), (1, 0))),
    "",                                                       # implicit: the IFDs after series 0
])
def test_ome_tiff_two_series_xyczt(tmp_path, tiffdata):
    a, b = _hyperstack(2, 3, 1), _hyperstack(2, 3, 1)
    b = {k: v + 5 for k, v in b.items()}
    order = [a[(c, z, 0)] for z in range(3) for c in range(2)] + [b[(c, z, 0)] for z in range(3) for c in range(2)]
    p = write_tiff(tmp_path / "x.ome.tif", order, description=OME_TWO_SERIES.format(tiffdata=tiffdata))
    ss = tiff.TiffFile(p).series()
    assert len(ss) == 2
    for s, planes in zip(ss, (a, b)):
        assert (s.channels, s.slices, s.frames) == (2, 3, 1)
        for c in range(2):
            assert np.array_equal(s.read_volume(c, 0), np.stack([planes[(c, z, 0)] for z in range(3)]))


def test_ome_tiff_first_coordinates(tmp_path):
    """XYZCT (z fastest), planes placed by FirstC / FirstT."""
    planes = _hyperstack(2, 2, 2)
    xml = ('<OME xmlns="http://www.openmicroscopy.org/Schemas/OME/2016-06"><Image ID="Image:0"><Pixels '
           'DimensionOrder="XYZCT" Type="uint16" SizeX="9" SizeY="7" SizeZ="2" SizeC="2" SizeT="2">'
           '<TiffData IFD="4" FirstT="1" PlaneCount="4"/><TiffData IFD="0" FirstC="0" PlaneCount="2"/>'
           '<TiffData IFD="2" FirstC="1" PlaneCount="2"/></Pixels></Image></OME>')
    order = [planes[(c, z, t)] for t in range(2) for c in range(2) for z in range(2)]
    s = _series(write_tiff(tmp_path / "f.ome.tif", order, description=xml))
    for c in range(2):
        for t in range(2):
            assert np.array_equal(s.read_volume(c, t), np.stack([planes[(c, z, t)] for z in range(2)]))


# ------------------------------------------------------------------------------------------------ regions
def test_regions_equal_zero_padded_slices(tmp_path):
    vol = _vol((9, 23, 31), np.uint16, 7)
    rng = np.random.default_rng(8)
    for name, kw in (("raw", dict(rows_per_strip=4)), ("tiles", dict(tile=(16, 16), compression=8)),
                     ("deflate", dict(rows_per_strip=5, compression=8, predictor=2)), ("one", {})):
        s = _series(write_tiff(tmp_path / f"{name}.tif", list(vol), **kw))
        full = s.read_volume()
        pad = np.zeros((9 + 120, 23 + 120, 31 + 120), np.uint16)
        pad[60:-60, 60:-60, 60:-60] = full
        for _ in range(40):
            mn = rng.integers(-15, 35, 3)
            sz = rng.integers(1, 20, 3)
            got = s.read_region(mn, sz)
            want = pad[60 + mn[2]:60 + mn[2] + sz[2], 60 + mn[1]:60 + mn[1] + sz[1], 60 + mn[0]:60 + mn[0] + sz[0]]
            assert got.shape == tuple(sz[::-1]) and np.array_equal(got, want), (name, mn, sz)
        assert not s.read_region((40, 0, 0), (3, 3, 3)).any()         # wholly outside
        assert not s.read_region((0, 0, -5), (3, 3, 5)).any()


class CountingFile(io.RawIOBase):
    """A file object that records the byte range of every read."""

    def __init__(self, path):
        self.f = open(path, "rb")
        self.reads = []

    def seek(self, off, whence=0):
        return self.f.seek(off, whence)

    def tell(self):
        return self.f.tell()

    def read(self, n=-1):
        pos = self.f.tell()
        b = self.f.read(n)
        self.reads.append((pos, len(b)))
        return b

    def readinto(self, buf):
        pos = self.f.tell()
        n = self.f.readinto(buf)
        self.reads.append((pos, n))
        return n

    def readable(self):
        return True

    def close(self):
        self.f.close()


def test_one_plane_region_reads_only_that_planes_strips(tmp_path):
    vol = _vol((64, 40, 50), np.uint16, 9)
    p = write_tiff(tmp_path / "s.tif", list(vol), rows_per_strip=8)
    fh = CountingFile(p)
    tf = tiff.TiffFile(p, fh=fh)
    page = tf.pages[37]
    fh.reads.clear()
    got = tf.series()[0].read_region((5, 9, 37), (30, 20, 1))
    assert np.array_equal(got[0], vol[37, 9:29, 5:35])
    # rows 9..28 lie in strips 1..3 of plane 37, which were written back to back: one read of exactly those rows
    row = 50 * 2
    assert fh.reads == [(int(page.offsets[1]) + 1 * row, 20 * row)]
    lo, hi = int(page.offsets[0]), int(page.offsets[-1] + page.counts[-1])
    assert all(lo <= a and a + n <= hi for a, n in fh.reads)
    fh.reads.clear()
    tf.series()[0].read_region((0, 0, 10), (50, 40, 2))           # two whole planes: one read each
    assert [n for _, n in fh.reads] == [40 * row, 40 * row]
    # compressed strips: only the strips the rows lie in are read
    q = write_tiff(tmp_path / "c.tif", list(vol), rows_per_strip=8, compression=8)
    fh = CountingFile(q)
    tf = tiff.TiffFile(q, fh=fh)
    page = tf.pages[3]
    fh.reads.clear()
    assert np.array_equal(tf.series()[0].read_region((0, 17, 3), (50, 5, 1))[0], vol[3, 17:22])
    assert fh.reads == [(int(page.offsets[2]), int(page.counts[2]))]


# ------------------------------------------------------------------------------------------------ refusals
def test_unsupported_files_raise(tmp_path):
    v16 = _vol((2, 5, 6), np.uint16, 10)
    cases = [
        (dict(compression=5), "LZW"),
        (dict(samples_per_pixel=3), "RGB"),
        (dict(), "sample type int16"),
    ]
    for i, (kw, msg) in enumerate(cases):
        planes = list(v16.astype(np.int16)) if "int16" in msg else list(v16)
        p = write_tiff(tmp_path / f"e{i}.tif", planes, **kw)
        with pytest.raises(NotImplementedError, match=msg) as e:
            tiff.TiffFile(p)
        assert p in str(e.value)
    p = write_tiff(tmp_path / "fp.tif", list(_vol((2, 5, 6), np.float32, 11)), compression=8, predictor=2)
    with pytest.raises(NotImplementedError, match="Predictor 2 .* float32") as e:
        tiff.TiffFile(p)
    assert p in str(e.value)
    xml = ('<OME xmlns="http://www.openmicroscopy.org/Schemas/OME/2016-06"><Image ID="Image:0"><Pixels '
           'DimensionOrder="XYZCT" Type="uint16" SizeX="6" SizeY="5" SizeZ="4" SizeC="1" SizeT="1">'
           '<TiffData IFD="0" PlaneCount="2"><UUID FileName="m.ome.tif">urn:uuid:1</UUID></TiffData>'
           '<TiffData IFD="0" FirstZ="2" PlaneCount="2"><UUID FileName="other.ome.tif">urn:uuid:2</UUID></TiffData>'
           '</Pixels></Image></OME>')
    p = write_tiff(tmp_path / "m.ome.tif", list(v16), description=xml)
    with pytest.raises(NotImplementedError, match="multi-file OME-TIFF .*other.ome.tif") as e:
        tiff.TiffFile(p).series()
    assert p in str(e.value)
    with pytest.raises(FileNotFoundError, match="missing.tif"):
        tiff.TiffFile(str(tmp_path / "missing.tif"))


def _tiff_dataset(tmp_path, vols, translations=None, **kw):
    return twin_datasets(str(tmp_path), vols, translations or {s: (30.0 * s, 0, 0) for s in vols}, **kw)


def test_loader_refusals_and_missing_files(tmp_path):
    vols = {0: _vol((4, 6, 8), np.uint16, 12), 1: _vol((4, 6, 8), np.uint16, 13)}
    _, xt = _tiff_dataset(tmp_path, vols)
    d = spimdata.SpimData2.load(xt)
    il = d.root.find("SequenceDescription/ImageLoader")
    z = spimdata.ET.SubElement(il, "ZGrouped")
    z.text = "true"
    with pytest.raises(NotImplementedError, match="ZGrouped"):
        viewsource.open_views(d)
    il.remove(z)
    os.remove(tmp_path / "tif" / "raw" / "tile1.tif")
    src = viewsource.open_views(d)
    assert np.array_equal(src.read_volume((0, 0)), vols[0])
    with pytest.raises(FileNotFoundError, match="tile1.tif"):
        src.read_region((0, 1), 0, (0, 0, 0), (2, 2, 2))
    with pytest.raises(ValueError, match="only level 0"):
        src.level_dims((0, 0), 1)
    # a split loader wrapping a TIFF loader is still not read
    d.root.find("SequenceDescription").remove(il)
    outer = spimdata.ET.SubElement(d.root.find("SequenceDescription"), "ImageLoader", format=spimdata.SPLIT_LOADER)
    outer.append(il)
    with pytest.raises(NotImplementedError, match="ImageLoader format spimreconstruction.filemap2"):
        viewsource.open_views(d)


def test_split_images_refuses_a_tiff_dataset_and_writes_nothing(tmp_path):
    vols = {0: _vol((8, 20, 24), np.uint16, 14)}
    _, xt = _tiff_dataset(tmp_path, vols)
    before = {os.path.join(dp, f): open(os.path.join(dp, f), "rb").read()
              for dp, _, fs in os.walk(tmp_path / "tif") for f in fs}
    for xo in (None, str(tmp_path / "tif" / "split.xml")):
        with pytest.raises(NotImplementedError, match="resave it to N5 or OME-ZARR first"):
            commands.split_images(xt, "16,16,8", "4,4,4", xml_out=xo, fake_interest_points=True)
    after = {os.path.join(dp, f): open(os.path.join(dp, f), "rb").read()
             for dp, _, fs in os.walk(tmp_path / "tif") for f in fs}
    assert after == before
    assert not os.path.exists(xt + "~1") and not os.path.exists(tmp_path / "tif" / "interestpoints.n5")


# ------------------------------------------------------------------------------------------------ XML
def test_file_map_loader_round_trip(tmp_path):
    vols = {0: _vol((3, 5, 7), np.uint16, 15), 1: _vol((3, 5, 7), np.uint16, 16)}
    _, xt = _tiff_dataset(tmp_path, vols)
    elsewhere = write_tiff(tmp_path / "abs.tif", list(vols[1]))
    d = spimdata.SpimData2.load(xt)
    assert d.image_loader() == (spimdata.FILEMAP_LOADER, None)
    raw = str(tmp_path / "tif" / "raw")
    assert d.file_mappings() == {(0, 0): (os.path.join(raw, "tile0.tif"), 0, 0),
                                 (0, 1): (os.path.join(raw, "tile1.tif"), 0, 0)}
    il = d.root.find("SequenceDescription/ImageLoader")
    m = il.find("files").findall("FileMapping")[1]
    assert (m.get("view_setup"), m.get("timepoint"), m.get("series"), m.get("channel")) == ("1", "0", "0", "0")
    assert m.find("file").get("type") == "relative" and m.find("file").text == "raw/tile1.tif"
    assert [c.tag for c in d.root.find("SequenceDescription")][0] == "ImageLoader"
    # absolute paths are read as they are
    m.find("file").set("type", "absolute")
    m.find("file").text = elsewhere
    assert d.file_mappings()[(0, 1)] == (elsewhere, 0, 0)
    assert np.array_equal(viewsource.open_views(d).read_volume((0, 1)), vols[1])
    # written next to another XML: the paths are re-based, then read back from a moved BasePath
    d.set_file_map_loader({(0, 0): (os.path.join(raw, "tile0.tif"), 2, 1), (0, 1): (elsewhere, 0, 0)},
                          xml_path=str(tmp_path / "o" / "x.xml"))
    os.makedirs(tmp_path / "o")
    d.save(str(tmp_path / "o" / "x.xml"))
    e = spimdata.SpimData2.load(str(tmp_path / "o" / "x.xml"))
    assert [f.text for f in e.root.iter("file")] == ["../tif/raw/tile0.tif", "../abs.tif"]
    assert e.file_mappings() == {(0, 0): (os.path.join(raw, "tile0.tif"), 2, 1), (0, 1): (elsewhere, 0, 0)}
    e.root.find("BasePath").text = "sub/x"               # "../tif/raw/tile0.tif" from o/sub/x
    os.makedirs(tmp_path / "o" / "sub" / "tif" / "raw")
    moved = str(tmp_path / "o" / "sub" / "tif" / "raw" / "tile0.tif")
    shutil.copy(os.path.join(raw, "tile0.tif"), moved)
    assert e.file_mappings()[(0, 0)] == (moved, 2, 1)
    e.set_file_map_loader({(0, 0): (moved, 0, 0)})
    assert viewsource.open_views(e).read_volume((0, 0)).tobytes() == vols[0].tobytes()


def test_frame_rule(tmp_path):
    """A file of more than one frame is read at the frame of the view's timepoint id, one of one frame at frame 0."""
    planes = _hyperstack(2, 3, 3)
    p3 = write_tiff(tmp_path / "t3.tif", [planes[(c, z, t)] for t in range(3) for z in range(3) for c in range(2)],
                    description=imagej_description(2, 3, 3))
    p1 = write_tiff(tmp_path / "t1.tif", [planes[(0, z, 0)] for z in range(3)])
    tiles = [dict(setup=s, size_xyz=(9, 7, 3), tile=s, translation_xyz=(0, 0, 0)) for s in range(3)]
    xml = spimdata.write_dataset_xml(str(tmp_path / "d.xml"), "unused", tiles)
    d = spimdata.SpimData2.load(xml)
    # three timepoints: copy the registrations of timepoint 0
    vrs = d.root.find("ViewRegistrations")
    for vr in list(vrs):
        for tp in (1, 2):
            c = spimdata.copy.deepcopy(vr)
            c.set("timepoint", str(tp))
            vrs.append(c)
    maps = {}
    for tp in range(3):
        maps[(tp, 0)] = (p3, 0, 0)
        maps[(tp, 1)] = (p3, 0, 1)
        maps[(tp, 2)] = (p1, 0, 0)
    d.set_file_map_loader(maps, xml)
    d.save(xml, backup=False)
    src = viewsource.open_views(spimdata.SpimData2.load(xml))
    for tp in range(3):
        for setup, c in ((0, 0), (1, 1)):
            assert np.array_equal(src.read_volume((tp, setup)), np.stack([planes[(c, z, tp)] for z in range(3)]))
        assert np.array_equal(src.read_volume((tp, 2)), np.stack([planes[(0, z, 0)] for z in range(3)]))
    assert src.mipmap_info((1, 0))[0] == [(1, 1, 1)] and src.level_dims((1, 0), 0) == (9, 7, 3)
    bad = viewsource.TiffViews({(3, 0): (p3, 0, 0), (0, 0): (p3, 0, 2), (0, 1): (p3, 1, 0)})
    with pytest.raises(ValueError, match="frame 3"):
        bad.read_volume((3, 0))
    with pytest.raises(ValueError, match="channel 2"):
        bad.read_volume((0, 0))
    with pytest.raises(ValueError, match="not series 1"):
        bad.read_volume((0, 1))


# ------------------------------------------------------------------------------------------------ end to end
def _files(root):
    return {os.path.relpath(os.path.join(dp, f), root): open(os.path.join(dp, f), "rb").read()
            for dp, _, fs in os.walk(root) for f in fs}


def test_resave_and_affine_fusion_equal_the_n5_twin(tmp_path):
    G = synth.field((40, 60, 120), seed=3, sigma=1.0)
    vols = {s: synth.tile_from(G, (2, 3, 30 * s + 2), (24, 40, 48), 20 + s, noise=5.0) for s in range(2)}
    xn, xt = _tiff_dataset(tmp_path, vols, compression=8, rows_per_strip=7)
    ctx = FakeContext()
    kw = dict(block_size=(16, 16, 8), block_scale=(2, 2, 1), downsampling=[(1, 1, 1), (2, 2, 1), (4, 4, 2)])
    out = {}
    for name, x in (("n", xn), ("t", xt)):
        for n5 in (False, True):
            d = tmp_path / f"{name}{int(n5)}"
            os.makedirs(d)
            commands.resave(x, ctx, xml_out=str(d / "dataset.xml"), n5=n5, **kw)
            out[(name, n5)] = _files(str(d / ("dataset.n5" if n5 else "dataset.ome.zarr")))
            e = spimdata.SpimData2.load(str(d / "dataset.xml"))
            assert e.image_loader()[0] == ("bdv.n5" if n5 else "bdv.multimg.zarr")
            assert e.root.find(f".//ImageLoader[@format='{spimdata.FILEMAP_LOADER}']") is None
            assert e.root.find(".//FileMapping") is None
    for n5 in (False, True):
        assert len(out[("t", n5)]) > 10 and out[("t", n5)] == out[("n", n5)]
    fused = {}
    for name, x in (("n", xn), ("t", xt)):
        f = str(tmp_path / f"fused_{name}.zarr")
        commands.create_fusion_container(x, f, block_size=(16, 16, 16), dtype="uint16", min_intensity=0.0,
                                         max_intensity=4000.0, downsamplings=[(2, 2, 1)])
        commands.affine_fusion(f, ctx, "AVG_BLEND")
        fused[name] = {k: v for k, v in _files(f).items() if not k.endswith(".zattrs")}
        st = bz.ZarrStore(f)
        assert st.read_volume("0").max() > 0
    assert fused["t"] == fused["n"] and len(fused["n"]) > 4


def test_resave_refuses_an_output_holding_the_tiff_files(tmp_path):
    vols = {0: _vol((4, 6, 8), np.uint16, 17)}
    _, xt = _tiff_dataset(tmp_path, vols)
    with pytest.raises(ValueError, match="overlaps the input container .*tile0.tif"):
        commands.resave(xt, FakeContext(), out_path=str(tmp_path / "tif" / "raw"), downsampling=[(1, 1, 1)])
    # the default output next to the XML is fine: the files are not inside it
    commands.resave(xt, FakeContext(), downsampling=[(1, 1, 1)])
    assert np.array_equal(viewsource.open_views(spimdata.SpimData2.load(xt)).read_volume((0, 0)), vols[0])
