"""`resave` and the `bdv.multimg.zarr` input on the CPU: the loader XML, the general Zarr reader, the OME-NGFF
mipmap factors, N5 <-> OME-ZARR round trips with every pyramid level checked against a numpy restatement of the
half-pixel chain, the planning errors, and stitching / affine-fusion giving the same answers on either container.
Driven through the oracle-backed fake context."""
import gzip
import json
import os
import zlib

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata, viewsource
from bsgpu import zarr as bz
from bsgpu import zstd as bzstd
from tests import synth
from tests.fake_ctx import FakeContext


def half_pixel_chain(vol, steps):
    """Every level of the pyramid by absolute factors ``steps``: one 2x average per doubled axis, x then y then z,
    out[i] = (in[2i] + in[2i+1] + 1) >> 1 for integers, 0.5 (a + b) for float32, floor(d / 2) voxels."""
    levels, cur = [vol], vol
    for a, b in zip(steps, steps[1:]):
        for ax, d in ((2, 0), (1, 1), (0, 2)):
            if b[d] == a[d]:
                continue
            n = cur.shape[ax] // 2
            lo = np.take(cur, np.arange(0, 2 * n, 2), axis=ax)
            hi = np.take(cur, np.arange(1, 2 * n, 2), axis=ax)
            if cur.dtype == np.float32:
                cur = (np.float32(0.5) * (lo + hi)).astype(np.float32)
            else:
                cur = ((lo.astype(np.uint32) + hi.astype(np.uint32) + 1) >> 1).astype(vol.dtype)
        levels.append(cur)
    return levels


def _dataset(tmp_path, sizes=((45, 37, 23), (40, 33, 21)), dtype=np.uint16):
    G = synth.field((40, 60, 120), seed=3, sigma=1.0)
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles, vols = [], {}
    for s, size in enumerate(sizes):
        x0 = 30 * s
        vols[s] = synth.tile_from(G, (2, 3, x0 + 2), size[::-1], 20 + s, noise=5.0, dtype=dtype)
        bn5.write_bdv_setup(store, s, 0, vols[s], (16, 16, 8), compression="zstd" if s else "raw")
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(x0, 0, 0)))
    return spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles), vols


# ------------------------------------------------------------------------------------------------ loader XML
def test_zarr_loader_xml_round_trip(tmp_path):
    xml, _ = _dataset(tmp_path)
    d = spimdata.SpimData2.load(xml)
    groups = {(0, 0): ("s0-t0.zarr", 0, 0), (0, 1): ("s1-t0.zarr", 2, 1)}
    d.set_image_loader("bdv.multimg.zarr", str(tmp_path / "sub" / "dataset.ome.zarr"), xml, groups)
    d.save(xml)
    assert os.path.exists(xml + "~1")
    e = spimdata.SpimData2.load(xml)
    fmt, path = e.image_loader()
    assert fmt == "bdv.multimg.zarr" and path == str(tmp_path / "sub" / "dataset.ome.zarr")
    assert e.zarr_groups() == groups
    il = e.root.find("SequenceDescription/ImageLoader")
    assert il.find("zarr").get("type") == "relative" and il.find("zarr").text == "sub/dataset.ome.zarr"
    g = il.find("zgroups").findall("zgroup")[1]
    assert (g.get("setup"), g.get("tp"), g.get("path"), g.get("indicies")) == ("1", "0", "s1-t0.zarr", "[2, 1]")
    assert [c.tag for c in e.root.find("SequenceDescription")][0] == "ImageLoader"
    # absolute container paths read as they are; other loaders still raise the same error
    il.find("zarr").set("type", "absolute")
    il.find("zarr").text = "/elsewhere/x.ome.zarr"
    assert e.image_loader()[1] == "/elsewhere/x.ome.zarr"
    il.set("format", "bdv.hdf5")
    with pytest.raises(NotImplementedError, match="ImageLoader format bdv.hdf5"):
        viewsource.open_views(e)
    d.set_image_loader("bdv.n5", str(tmp_path / "dataset.n5"), xml)
    assert d.image_loader() == ("bdv.n5", str(tmp_path / "dataset.n5")) and d.zarr_groups() == {}


# ------------------------------------------------------------------------------------------------ Zarr reader
def _hand_array(root, path, arr_tczyx, chunks, dtype, sep, compressor, fill=0, skip=()):
    os.makedirs(os.path.join(root, path), exist_ok=True)
    meta = {"zarr_format": 2, "shape": list(arr_tczyx.shape), "chunks": list(chunks), "dtype": dtype,
            "compressor": compressor, "fill_value": fill, "order": "C", "filters": None}
    if sep is not None:
        meta["dimension_separator"] = sep
    with open(os.path.join(root, path, ".zarray"), "w") as f:
        json.dump(meta, f)
    grid = [-(-s // c) for s, c in zip(arr_tczyx.shape, chunks)]
    for idx in np.ndindex(*grid):
        if idx in skip:
            continue
        full = np.zeros(chunks, dtype=np.dtype(dtype))
        sl = tuple(slice(i * c, (i + 1) * c) for i, c in zip(idx, chunks))
        part = arr_tczyx[sl]
        full[tuple(slice(0, n) for n in part.shape)] = part
        raw = full.tobytes()
        cid = compressor["id"] if compressor else None
        payload = {None: raw, "gzip": gzip.compress(raw) if cid == "gzip" else None,
                   "zlib": zlib.compress(raw) if cid == "zlib" else None,
                   "zstd": bzstd.compress(raw) if cid == "zstd" else None}[cid]
        key = (sep or ".").join(str(i) for i in idx)
        p = os.path.join(root, path, *key.split("/"))
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(payload)


@pytest.mark.parametrize("dtype", ["<u2", ">u2", "|u1", ">f4", "<f4"])
@pytest.mark.parametrize("sep", ["/", ".", None])
@pytest.mark.parametrize("codec", [None, "gzip", "zlib", "zstd"])
def test_zarr_reader_hand_built_arrays(tmp_path, dtype, sep, codec):
    rng = np.random.default_rng(1)
    arr = (rng.uniform(0, 250, (2, 3, 11, 9, 13))).astype(np.dtype(dtype))
    root = str(tmp_path / "a.zarr")
    comp = {"id": codec, "level": 1} if codec else None
    _hand_array(root, "g/0", arr, (1, 1, 4, 4, 5), dtype, sep, comp, fill=7, skip={(1, 2, 2, 2, 2)})
    st = bz.ZarrStore(root)
    want = arr.astype(np.dtype(dtype).newbyteorder("="))
    want[1, 2, 8:, 8:, 10:] = 7                                    # the missing chunk reads as fill_value
    got = st.read_volume("g/0", c=2, t=1)
    assert got.dtype == want.dtype and got.dtype.isnative
    assert np.array_equal(got, want[1, 2])
    assert np.array_equal(st.read_volume("g/0", c=1, t=0), want[0, 1])
    assert np.array_equal(st.read_region("g/0", (3, 2, 1), (9, 6, 9), c=2, t=1), want[1, 2, 1:10, 2:8, 3:12])


def test_zarr_reader_rejects_unknown_codecs(tmp_path):
    arr = np.arange(2 * 3 * 4, dtype=np.uint16).reshape(1, 1, 2, 3, 4)
    root = str(tmp_path / "b.zarr")
    _hand_array(root, "0", arr, (1, 1, 2, 3, 4), "<u2", "/", None)
    with open(os.path.join(root, "0", ".zarray")) as f:
        meta = json.load(f)
    meta["compressor"] = {"id": "blosc", "cname": "lz4", "clevel": 5, "shuffle": 1}
    with open(os.path.join(root, "0", ".zarray"), "w") as f:
        json.dump(meta, f)
    with pytest.raises(NotImplementedError, match="blosc"):
        bz.ZarrStore(root).read_volume("0")


def _multiscale(root, scales, shapes):
    st = bz.ZarrStore(root, create=True)
    for i, shp in enumerate(shapes):
        st.create_array(f"v/{i}", (1, 1) + tuple(shp[::-1]), (1, 1, 4, 4, 4), "uint16")
    st.set_attributes("v", {"multiscales": [{"version": "0.4", "axes": [{"name": n} for n in "tczyx"], "datasets": [
        {"path": str(i), "coordinateTransformations": [{"type": "scale", "scale": [1.0, 1.0] + list(s[::-1])}]}
        for i, s in enumerate(scales)]}]})
    return st


def test_multiscale_factors_from_scales(tmp_path):
    st = _multiscale(str(tmp_path / "m.zarr"), [(0.5, 0.5, 2.0), (1.0, 1.0, 2.0), (2.0, 2.0, 4.0)],
                     [(45, 37, 23), (22, 18, 23), (12, 9, 11)])
    lv = bz.read_multiscales(st, "v")
    assert [l["factors"] for l in lv] == [(1, 1, 1), (2, 2, 1), (4, 4, 2)]
    assert [l["dims"] for l in lv] == [(45, 37, 23), (22, 18, 23), (12, 9, 11)]
    with pytest.raises(ValueError, match="not integers"):
        bz.read_multiscales(_multiscale(str(tmp_path / "n.zarr"), [(1, 1, 1), (1.5, 2, 1)], [(45, 37, 23), (30, 18, 23)]), "v")
    with pytest.raises(ValueError, match="do not match"):
        bz.read_multiscales(_multiscale(str(tmp_path / "o.zarr"), [(1, 1, 1), (2, 2, 1)], [(45, 37, 23), (20, 18, 23)]), "v")


# ------------------------------------------------------------------------------------------------ resave
STEPS = [(1, 1, 1), (2, 2, 1), (4, 4, 2), (8, 8, 2)]


def _levels_of(xml, view):
    src = viewsource.open_views(spimdata.SpimData2.load(xml))
    factors, mts = src.mipmap_info(view)
    return src, factors, mts, [src.read_volume(view, l) for l in range(len(factors))]


@pytest.mark.parametrize("block_scale", [(4, 4, 4), (1, 2, 1)])      # resident pyramid / levels from the stored ones
def test_resave_n5_zarr_n5_every_level_bitwise(tmp_path, block_scale):
    xml, vols = _dataset(tmp_path)
    ctx = FakeContext()
    os.makedirs(tmp_path / "z")
    os.makedirs(tmp_path / "n")
    xz, xn = str(tmp_path / "z" / "dataset.xml"), str(tmp_path / "n" / "dataset.xml")
    plan = commands.resave(xml, ctx, xml_out=xz, block_size=(8, 8, 4), block_scale=block_scale, downsampling=STEPS)
    assert plan["out_path"] == str(tmp_path / "z" / "dataset.ome.zarr")
    commands.resave(xz, ctx, xml_out=xn, n5=True, block_size=(16, 8, 8), block_scale=(2, 2, 2), downsampling=STEPS,
                    compression="gzip")
    assert spimdata.SpimData2.load(xz).image_loader() == ("bdv.multimg.zarr", str(tmp_path / "z" / "dataset.ome.zarr"))
    assert spimdata.SpimData2.load(xn).image_loader() == ("bdv.n5", str(tmp_path / "n" / "dataset.n5"))
    for s, vol in vols.items():
        want = half_pixel_chain(vol, STEPS)
        for x in (xz, xn):
            src, factors, mts, got = _levels_of(x, (0, s))
            assert factors == STEPS
            assert np.allclose(mts[2], [[4, 0, 0, 1.5], [0, 4, 0, 1.5], [0, 0, 2, 0.5]])
            for g, w in zip(got, want):
                assert g.dtype == w.dtype and np.array_equal(g, w)
    zst = bz.ZarrStore(str(tmp_path / "z" / "dataset.ome.zarr"))
    m = zst.array_meta("s1-t0.zarr/2")
    assert m["shape"] == [1, 1, 10, 8, 10] and m["chunks"] == [1, 1, 4, 8, 8] and m["compressor"]["id"] == "zstd"
    ms = zst.get_attributes("s1-t0.zarr")["multiscales"][0]
    assert ms["datasets"][3]["coordinateTransformations"][0]["scale"] == [1.0, 1.0, 2.0, 8.0, 8.0]
    assert ms["datasets"][3]["coordinateTransformations"][1]["translation"] == [0.0, 0.0, 0.5, 3.5, 3.5]
    nst = bn5.N5Store(str(tmp_path / "n" / "dataset.n5"))
    assert nst.get_attributes("setup1")["downsamplingFactors"] == [list(f) for f in STEPS]
    assert nst.dataset_attributes("setup1/timepoint0/s3")["dimensions"] == [5, 4, 10]


def test_resave_float32_and_uint8_views(tmp_path):
    for dt in (np.float32, np.uint8):
        d = tmp_path / np.dtype(dt).name
        os.makedirs(d)
        xml, vols = _dataset(d, sizes=((19, 17, 9),), dtype=dt)
        commands.resave(xml, FakeContext(), xml_out=str(d / "z.xml"), block_size=(8, 8, 4), block_scale=(2, 2, 2),
                        downsampling="1,1,1; 2,2,2; 4,4,2", compression="raw")
        got = _levels_of(str(d / "z.xml"), (0, 0))[3]
        for g, w in zip(got, half_pixel_chain(vols[0], [(1, 1, 1), (2, 2, 2), (4, 4, 2)])):
            assert g.dtype == w.dtype and np.array_equal(g, w)


@pytest.mark.parametrize("block_scale", [(8, 8, 2), (1, 1, 1)])      # resident pyramid / levels from the stored ones
def test_resave_sharded_ranks_write_the_same_container(tmp_path, block_scale):
    import threading
    xml, vols = _dataset(tmp_path)
    xo = str(tmp_path / "w.xml")
    bar = threading.Barrier(2)
    errors = []

    def rank(r):
        try:
            commands.resave(xml, FakeContext(), xml_out=xo, shard=(r, 2), block_size=(8, 8, 4), block_scale=block_scale,
                            downsampling=STEPS, barrier=lambda: bar.wait(timeout=60))
        except Exception as e:          # noqa: BLE001 -- reported below
            errors.append(e)
            bar.abort()

    ts = [threading.Thread(target=rank, args=(r,)) for r in (0, 1)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for s, vol in vols.items():
        for g, w in zip(_levels_of(xo, (0, s))[3], half_pixel_chain(vol, STEPS)):
            assert np.array_equal(g, w)


def test_resave_retries_failed_blocks(tmp_path):
    from bsgpu import native
    xml, vols = _dataset(tmp_path)

    class Flaky(FakeContext):
        n = 0

        def downsample(self, h, f):
            Flaky.n += 1
            if Flaky.n % 3 == 0:
                raise native.BsError(5, "transient")
            return super().downsample(h, f)

    commands.resave(xml, Flaky(), xml_out=str(tmp_path / "r.xml"), block_size=(8, 8, 4), block_scale=(2, 2, 1),
                    downsampling=STEPS[:2])
    for s, vol in vols.items():
        for g, w in zip(_levels_of(str(tmp_path / "r.xml"), (0, s))[3], half_pixel_chain(vol, STEPS[:2])):
            assert np.array_equal(g, w)

    class Broken(FakeContext):
        def volume_upload(self, vol):
            raise native.BsError(5, "down")

    with pytest.raises(RuntimeError, match="still failing after 2 attempts"):
        commands.resave(xml, Broken(), xml_out=str(tmp_path / "b.xml"), retries=2, downsampling=STEPS[:1])


def test_resave_planning_errors_dry_run_and_defaults(tmp_path):
    xml, _ = _dataset(tmp_path)
    ctx = FakeContext()
    for bad, msg in (("2,2,1; 4,4,1", "full resolution"), ("1,1,1; 4,4,1", "not 1x or 2x"),
                     ("1,1,1; 2,2,1; 2,1,1", "not 1x or 2x"), ("1,1", "triples")):
        with pytest.raises(ValueError, match=msg):
            commands.resave(xml, ctx, downsampling=bad)
    with pytest.raises(NotImplementedError, match="Blosc"):
        commands.resave(xml, ctx, compression="Blosc")
    before = sorted(os.listdir(tmp_path))
    xml_text = open(xml).read()
    p = commands.resave(xml, ctx, dry_run=True)
    assert sorted(os.listdir(tmp_path)) == before and open(xml).read() == xml_text and ctx.vols == {}
    assert p["out_path"] == str(tmp_path / "dataset.ome.zarr") and p["xml_out"] == xml
    assert p["downsamplings"] == [(1, 1, 1)]                 # 45 x 37 x 23: nothing over 256 px
    assert p["compute_blocks"] == 2                           # 128 x 128 x 64 x (16, 16, 1): one block per view
    q = commands.resave(xml, ctx, xml_out=str(tmp_path / "o" / "x.xml"), n5=True, dry_run=True)
    assert q["out_path"] == str(tmp_path / "o" / "dataset.n5") and not os.path.exists(tmp_path / "o")
    assert commands.resave(xml, ctx, dry_run=True, block_size=(16, 16, 8), block_scale=(1, 1, 1))["compute_blocks"] == 54
    # the default output is written next to the (input) XML, which then points at it
    commands.resave(xml, ctx, block_size=(16, 16, 8))
    assert os.path.isdir(tmp_path / "dataset.ome.zarr") and os.path.exists(xml + "~1")
    assert spimdata.SpimData2.load(xml).image_loader()[0] == "bdv.multimg.zarr"


def test_resave_refuses_to_overwrite_its_input(tmp_path):
    xml, vols = _dataset(tmp_path)
    ctx = FakeContext()
    n5_attrs = open(tmp_path / "dataset.n5" / "setup0" / "timepoint0" / "s0" / "attributes.json").read()
    xml_text = open(xml).read()
    for kw in (dict(n5=True),                                            # dataset.n5 next to its own XML
               dict(out_path=str(tmp_path / "dataset.n5" / "inner.ome.zarr")),
               dict(out_path=str(tmp_path))):
        with pytest.raises(ValueError, match="overlaps the input container"):
            commands.resave(xml, ctx, downsampling=STEPS[:2], **kw)
    assert open(tmp_path / "dataset.n5" / "setup0" / "timepoint0" / "s0" / "attributes.json").read() == n5_attrs
    assert open(xml).read() == xml_text and not os.path.exists(tmp_path / "dataset.n5" / "inner.ome.zarr")
    assert np.array_equal(_levels_of(xml, (0, 0))[3][0], vols[0])
    # an OME-ZARR dataset re-saved with the defaults would land on its own container
    os.makedirs(tmp_path / "z")
    xz = str(tmp_path / "z" / "dataset.xml")
    commands.resave(xml, ctx, xml_out=xz, block_size=(8, 8, 4), downsampling=STEPS[:2])
    with pytest.raises(ValueError, match="overlaps the input container"):
        commands.resave(xz, ctx, downsampling=STEPS[:2])
    assert np.array_equal(_levels_of(xz, (0, 1))[3][0], vols[1])


def test_resave_rank0_creates_the_container_before_the_others_start(tmp_path):
    xml, _ = _dataset(tmp_path)
    kw = dict(xml_out=str(tmp_path / "o" / "x.xml"), block_size=(8, 8, 4), downsampling=STEPS)
    with pytest.raises(ValueError, match="needs barrier"):
        commands.resave(xml, FakeContext(), shard=(1, 2), **kw)

    class Stop(Exception):
        pass

    def barrier():
        raise Stop

    with pytest.raises(Stop):                        # rank 1 waits before touching the output
        commands.resave(xml, FakeContext(), shard=(1, 2), barrier=barrier, **kw)
    assert not os.path.exists(tmp_path / "o")
    with pytest.raises(Stop):                        # rank 0 has created every dataset when it first waits
        commands.resave(xml, FakeContext(), shard=(0, 2), barrier=barrier, **kw)
    st = bz.ZarrStore(str(tmp_path / "o" / "dataset.ome.zarr"))
    assert [st.array_meta(f"s{s}-t0.zarr/{l}")["shape"][2:] for s in (0, 1) for l in (0, 3)] == [
        [23, 37, 45], [11, 4, 5], [21, 33, 40], [10, 4, 5]]


def test_resave_checks_every_view_before_writing(tmp_path):
    xml, _ = _dataset(tmp_path)
    bn5.write_bdv_setup(bn5.N5Store(str(tmp_path / "dataset.n5")), 1, 0, np.zeros((21, 33, 40), np.uint32), (16, 16, 8))
    with pytest.raises(NotImplementedError, match="uint32 view"):
        commands.resave(xml, FakeContext(), xml_out=str(tmp_path / "o" / "x.xml"))
    assert not os.path.exists(tmp_path / "o")
    xml2, _ = _dataset(tmp_path / "b", sizes=((45, 37, 23), (40, 33, 3)))
    with pytest.raises(ValueError, match="too small"):
        commands.resave(xml2, FakeContext(), xml_out=str(tmp_path / "b" / "o" / "x.xml"),
                        downsampling="1,1,1; 2,2,2; 4,4,4")
    assert not os.path.exists(tmp_path / "b" / "o")


def test_propose_mipmaps():
    assert commands.propose_mipmaps((2048, 2048, 256)) == [(1, 1, 1), (2, 2, 2), (4, 4, 4), (8, 8, 8)]
    assert commands.propose_mipmaps((2048, 1024, 200), (0.4, 0.4, 2.0)) == [
        (1, 1, 1), (2, 2, 1), (4, 4, 1), (8, 8, 2)]
    assert commands.propose_mipmaps((256, 100, 7)) == [(1, 1, 1)]


# ------------------------------------------------------------------------------------------------ same answers
def test_stitching_and_affine_fusion_agree_on_n5_and_zarr(tmp_path):
    xml, _ = _dataset(tmp_path, sizes=((48, 40, 24), (48, 40, 24)))
    ctx = FakeContext()
    os.makedirs(tmp_path / "z")
    os.makedirs(tmp_path / "n")
    xz, xn = str(tmp_path / "z" / "dataset.xml"), str(tmp_path / "n" / "dataset.xml")
    kw = dict(block_size=(16, 16, 8), block_scale=(2, 2, 1), downsampling=[(1, 1, 1), (2, 2, 1)])
    commands.resave(xml, ctx, xml_out=xz, **kw)
    commands.resave(xz, ctx, xml_out=xn, n5=True, **kw)
    res = {}
    for name, x in (("z", xz), ("n", xn)):
        raw = commands.stitching(x, ctx, downsampling=(1, 1, 1))
        res[name] = [(r.pair, r.shift_int if hasattr(r, "shift_int") else None, np.asarray(r.transform).tolist(), r.r)
                     for r in raw if r is not None]
        out = str(tmp_path / f"fused_{name}.zarr")
        commands.create_fusion_container(x, out, block_size=(16, 16, 16), dtype="uint16", min_intensity=0.0,
                                         max_intensity=4000.0, downsamplings=[(2, 2, 1)])
        commands.affine_fusion(out, ctx, "AVG_BLEND")
    assert res["z"] == res["n"] and len(res["z"]) == 1
    sz, sn = bz.ZarrStore(str(tmp_path / "fused_z.zarr")), bz.ZarrStore(str(tmp_path / "fused_n.zarr"))
    for lvl in ("0", "1"):
        m = sz.array_meta(lvl)
        for idx in np.ndindex(*[-(-s // c) for s, c in zip(m["shape"], m["chunks"])]):
            assert open(sz._chunk_path(lvl, idx), "rb").read() == open(sn._chunk_path(lvl, idx), "rb").read()
