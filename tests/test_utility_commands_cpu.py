"""The utility commands without a GPU: downsample through the oracle-backed context (every level the chained
fo.downsample2x of the level above, metadata, zero blocks, N5 / Zarr layouts, world-2 sharding), clear-interestpoints,
clear-registrations and transform-points."""
import os
import socket
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata
from bsgpu import zarr as bz
from oracle import fusion_oracle as fo
from tests.fake_ctx import FakeContext
from tests.test_match_cpu import RUN, MatchFakeContext, planted_scene, read_rows

STEPS = "2,2,1; 2,2,2; 1,2,2"
OUT = ["s1", "s2", "s3"]


def _volume(dims_xyz, dtype, seed=0):
    rng = np.random.default_rng(seed)
    shape = tuple(dims_xyz)[::-1]
    if dtype == "float32":
        return rng.normal(100.0, 40.0, shape).astype(np.float32)
    top = np.iinfo(dtype).max
    return rng.integers(0, top + 1, shape, dtype=np.int64).astype(dtype)


def _write_input(root, layout, vol, bs, name="s0", compression="zstd"):
    """``vol`` as dataset ``name``: layout "n5" (3-D dataset), "zarr3" ((z, y, x) array) or "zarr5" ((1, 1, z, y, x))."""
    dims = list(vol.shape[::-1])
    if layout == "n5":
        st = bn5.N5Store(root, create=True)
        st.create_dataset(name, dims, bs, vol.dtype, compression)
        st.save_block(name, vol, (0, 0, 0))
        return st
    st = bz.ZarrStore(root, create=True)
    lead = [1, 1] if layout == "zarr5" else []
    st.create_array(name, lead + dims[::-1], lead + list(bs)[::-1], vol.dtype.name, compression)
    st.save_block(name, vol, (0, 0, 0, 0, 0))
    return st


def _storage(layout):
    return "N5" if layout == "n5" else "ZARR"


def _read(root, layout, name):
    return (bn5.N5Store(root) if layout == "n5" else bz.ZarrStore(root)).read_volume(name)


def _chain(vol, steps):
    out = []
    for s in commands.parse_downsample_steps(steps):
        vol = fo.downsample2x(vol, s)
        out.append(vol)
    return out


def _files(root):
    """{relative path: bytes} of every file of a container."""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(dp, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


# ------------------------------------------------------------------------------------------ downsample
@pytest.mark.parametrize("dtype", ["uint8", "uint16", "float32"])
@pytest.mark.parametrize("layout", ["n5", "zarr3", "zarr5"])
def test_every_level_is_the_chained_2x_step(tmp_path, dtype, layout):
    # odd dims whose last storage blocks are one voxel thick in x and z, thinner than the step
    vol = _volume((49, 37, 21), dtype, seed=1)
    root = str(tmp_path / "c")
    _write_input(root, layout, vol, (8, 8, 4))
    ctx = FakeContext()
    assert commands.downsample(root, ctx, "s0", OUT, STEPS, storage=_storage(layout)) == OUT
    want = _chain(vol, STEPS)
    for name, w in zip(OUT, want):
        got = _read(root, layout, name)
        assert got.dtype == np.dtype(dtype) and got.shape == w.shape and np.array_equal(got, w), name
    assert [w.shape[::-1] for w in want] == [(24, 18, 21), (12, 9, 10), (12, 4, 5)]
    assert ctx.calls["downsample"] > 0


@pytest.mark.parametrize("layout", ["n5", "zarr5"])
def test_block_scale_does_not_change_the_datasets(tmp_path, layout):
    vol = _volume((75, 66, 26), "uint16", seed=2)
    files = []
    for scale in ((1, 1, 1), (3, 2, 1), (4, 4, 2)):
        root = str(tmp_path / ("c%d%d%d" % scale))
        _write_input(root, layout, vol, (8, 8, 4))
        commands.downsample(root, FakeContext(), "s0", OUT, STEPS, storage=_storage(layout), block_scale=scale)
        files.append(_files(root))
    assert files[0] == files[1] == files[2]


def test_resident_levels_are_derived_on_the_device(tmp_path, monkeypatch):
    """(4, 4, 2) on 8 x 8 x 4 blocks: the compute blocks of s1 cover whole storage blocks of s2 (step 2, 2, 2) but not
    of s3, so s2 comes from the resident s1 block and s3 from the stored s2; (3, 2, 1) re-reads every level."""
    reads = []
    orig = bn5.N5Store.read_region
    monkeypatch.setattr(bn5.N5Store, "read_region", lambda self, path, mn, sz: reads.append(path) or orig(self, path, mn, sz))
    read = {}
    for scale in ((3, 2, 1), (4, 4, 2)):
        root = str(tmp_path / ("c%d%d%d" % scale))
        _write_input(root, "n5", _volume((75, 66, 26), "uint16", seed=2), (8, 8, 4))
        reads.clear()
        commands.downsample(root, FakeContext(), "s0", OUT, STEPS, block_scale=scale)
        read[scale] = sorted(set(reads))
    assert read[(3, 2, 1)] == ["s0", "s1", "s2"] and read[(4, 4, 2)] == ["s0", "s2"]


@pytest.mark.parametrize("layout", ["n5", "zarr3"])
def test_metadata_is_copied_from_the_input(tmp_path, layout):
    vol = _volume((40, 30, 12), "float32", seed=3)
    root = str(tmp_path / "c")
    st = _write_input(root, layout, vol, (16, 8, 4), compression="gzip")
    commands.downsample(root, FakeContext(), "s0", ["s1", "s2"], [(2, 2, 1), (2, 1, 2)], storage=_storage(layout))
    if layout == "n5":
        a0 = st.dataset_attributes("s0")
        for name, dims in (("s1", [20, 15, 12]), ("s2", [10, 15, 6])):
            a = st.dataset_attributes(name)
            assert a == dict(dimensions=dims, blockSize=a0["blockSize"], dataType="float32", compression=a0["compression"])
        assert a0["compression"] == {"type": "gzip", "level": 1}
    else:
        m0 = st.array_meta("s0")
        for name, shape in (("s1", [12, 15, 20]), ("s2", [6, 15, 10])):
            assert st.array_meta(name) == dict(m0, shape=shape)


def test_dry_run_plans_and_writes_nothing(tmp_path):
    root = str(tmp_path / "c")
    _write_input(root, "n5", _volume((49, 37, 21), "uint8"), (8, 8, 4))
    before = _files(root)
    assert commands.downsample(root, FakeContext(), "s0", "s1; s2; s3", STEPS, dry_run=True) == [
        ("s1", (24, 18, 21)), ("s2", (12, 9, 10)), ("s3", (12, 4, 5))]
    assert _files(root) == before


@pytest.mark.parametrize("kw, exc, text", [
    (dict(downsampling="2,2,1; 3,3,1"), ValueError, "not 1 or 2"),
    (dict(downsampling="2,2,1"), ValueError, "as many"),
    (dict(downsampling="2,2,1; 2,2"), ValueError, "triples"),
    (dict(downsampling="2,2,2; 2,2,2"), ValueError, "empty axis"),               # z: 3 -> 1 -> 0
    (dict(datasets_out=["s1", "s0"]), ValueError, "different"),
    (dict(shard=(0, 2)), ValueError, "barrier"),
    (dict(storage="HDF5"), ValueError, "N5 or ZARR"),
])
def test_downsample_rejects(tmp_path, kw, exc, text):
    root = str(tmp_path / "c")
    _write_input(root, "n5", _volume((20, 16, 3), "uint16"), (8, 8, 4))
    args = dict(n5_path=root, ctx=FakeContext(), dataset_in="s0", datasets_out=["s1", "s2"], downsampling="2,2,1; 2,2,1")
    args.update(kw)
    before = _files(root)
    with pytest.raises(exc, match=text):
        commands.downsample(**args)
    assert _files(root) == before


def test_int16_and_five_d_zarr_with_two_channels_are_rejected(tmp_path):
    root = str(tmp_path / "n")
    st = bn5.N5Store(root, create=True)
    st.write_volume("s0", np.zeros((4, 8, 8), dtype=np.int16), (8, 8, 4))
    with pytest.raises(NotImplementedError, match="int16"):
        commands.downsample(root, FakeContext(), "s0", ["s1"], "2,2,1")
    root = str(tmp_path / "z")
    zs = bz.ZarrStore(root, create=True)
    zs.create_array("s0", [1, 2, 4, 8, 8], [1, 1, 4, 8, 8], "uint16", "zstd")
    with pytest.raises(ValueError, match="neither"):
        commands.downsample(root, FakeContext(), "s0", ["s1"], "2,2,1", storage="ZARR")
    assert not os.path.exists(os.path.join(root, "s1"))


@pytest.mark.parametrize("layout", ["n5", "zarr5"])
def test_all_zero_blocks_are_not_written(tmp_path, layout):
    vol = _volume((64, 32, 16), "uint16", seed=4)
    vol[:, :, :32] = 0                                         # x < 32 of s0 is x < 16 of s1, x < 8 of s2
    root = str(tmp_path / "c")
    _write_input(root, layout, vol, (8, 8, 4))
    commands.downsample(root, FakeContext(), "s0", ["s1", "s2"], "2,2,1; 2,2,2", storage=_storage(layout))
    for name, w, gx_zero in zip(["s1", "s2"], _chain(vol, "2,2,1; 2,2,2"), (2, 1)):
        dims = w.shape[::-1]
        grid = [-(-dims[d] // (8, 8, 4)[d]) for d in range(3)]
        for gz in range(grid[2]):
            for gy in range(grid[1]):
                for gx in range(grid[0]):
                    key = [str(gx), str(gy), str(gz)] if layout == "n5" else ["0", "0", str(gz), str(gy), str(gx)]
                    assert os.path.exists(os.path.join(root, name, *key)) == (gx >= gx_zero), (name, gx, gy, gz)
        assert np.array_equal(_read(root, layout, name), w)


@pytest.mark.parametrize("layout", ["n5", "zarr5"])
def test_nonrigid_fusion_output_layouts(tmp_path, layout):
    """The dataset nonrigid_fusion writes: 3-D N5 or (1, 1, z, y, x) Zarr, zstd, an `offset` attribute, and no block
    files where no view reaches."""
    dims, bs = (96, 70, 20), (32, 32, 16)
    vol = _volume(dims, "float32", seed=5)
    vol[:, 32:64, :] = 0                                       # an unreached slab
    root = str(tmp_path / "fused")
    if layout == "n5":
        st = bn5.N5Store(root, create=True)
        st.create_dataset("fused/s0", dims, bs, np.float32, "zstd")
    else:
        st = bz.ZarrStore(root, create=True)
        st.create_array("fused/s0", [1, 1] + list(dims[::-1]), [1, 1] + list(bs[::-1]), "float32", "zstd")
    st.set_attributes("fused/s0", {"offset": [-5, 3, 0]})
    sink = commands._Sink(st, layout != "n5", 0, 0)
    for off, size, gpos in commands.bf.grid_create(list(dims), [64, 64, 16], list(bs)):
        blk = vol[off[2]:off[2] + size[2], off[1]:off[1] + size[1], off[0]:off[0] + size[0]]
        for o, s, g in commands._storage_cells(((0, 0, 0), size, gpos), bs):
            if blk[o[2]:o[2] + s[2], o[1]:o[1] + s[1], o[0]:o[0] + s[0]].any():
                sink.save("fused/s0", np.ascontiguousarray(blk[o[2]:o[2] + s[2], o[1]:o[1] + s[1], o[0]:o[0] + s[0]]), g)
    out = commands.downsample(root, FakeContext(), "fused/s0", ["fused/s1", "fused/s2"], "2,2,1; 2,2,2",
                              storage=_storage(layout))
    assert out == ["fused/s1", "fused/s2"]
    for name, w in zip(out, _chain(vol, "2,2,1; 2,2,2")):
        assert np.array_equal(_read(root, layout, name), w)


def _shard_worker(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    for scale in ((1, 1, 1), (4, 4, 2)):
        commands.downsample(os.path.join(root, "c%d%d%d" % scale), FakeContext(), "s0", OUT, STEPS, block_scale=scale,
                            shard=(rank, world), barrier=dist.barrier)
    dist.barrier()
    if rank == 0:
        q.put("done")
    dist.barrier()
    dist.destroy_process_group()


def test_world2_shard_writes_the_same_bytes(tmp_path):
    import torch.multiprocessing as mp
    vol = _volume((75, 66, 26), "uint16", seed=6)
    vol[:10] = 0
    one, two = tmp_path / "one", tmp_path / "two"
    for d in (one, two):
        for scale in ((1, 1, 1), (4, 4, 2)):
            _write_input(str(d / ("c%d%d%d" % scale)), "n5", vol, (8, 8, 4))
    for scale in ((1, 1, 1), (4, 4, 2)):
        commands.downsample(str(one / ("c%d%d%d" % scale)), FakeContext(), "s0", OUT, STEPS, block_scale=scale)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, str(two), q)) for r in range(2)]
    for p in procs:
        p.start()
    assert q.get(timeout=300) == "done"
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    a, b = _files(str(one)), _files(str(two))
    assert a == b and len(a) > 100


# ------------------------------------------------------------------------------------------ clear-interestpoints
def _ip_scene(root):
    """Two views of beads with correspondences from match_interestpoints, plus a second label `nuclei` on view 0
    only, all listed in the XML."""
    xml, truth = planted_scene(root, tile=(120, 100, 40))
    commands.match_interestpoints(xml, MatchFakeContext(), ["beads"], **RUN)
    st = bn5.N5Store(os.path.join(str(root), "interestpoints.n5"))
    g = "tpId_0_viewSetupId_0/nuclei/interestpoints"
    st.write_list(g + "/id", np.arange(5, dtype=np.uint64).reshape(-1, 1), 300000, "zstd")
    st.write_list(g + "/loc", np.arange(15, dtype=np.float64).reshape(-1, 3), 300000, "zstd")
    data = spimdata.SpimData2.load(xml)
    data.set_interest_points("beads", "DOG", {v: f"tpId_{v[0]}_viewSetupId_{v[1]}/beads" for v in truth})
    data.set_interest_points("nuclei", "DOG", {(0, 0): "tpId_0_viewSetupId_0/nuclei"})
    data.save(xml, backup=False)
    return xml, sorted(truth)


def _points(root, view, label):
    st = bn5.N5Store(os.path.join(str(root), "interestpoints.n5"))
    return st.read_list(f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}/interestpoints/loc")


def test_clear_interestpoints_dry_run_counts_and_keeps_everything(tmp_path):
    xml, views = _ip_scene(tmp_path)
    rows = read_rows(tmp_path, views)
    before = _files(str(tmp_path))
    rep = commands.clear_interestpoints(xml, dry_run=True)
    assert rep == {views[0]: {"beads": (len(_points(tmp_path, views[0], "beads")), len(rows[views[0]])), "nuclei": (5, 0)},
                   views[1]: {"beads": (len(_points(tmp_path, views[1], "beads")), len(rows[views[1]]))}}
    assert min(len(r) for r in rows.values()) > 20
    assert _files(str(tmp_path)) == before
    assert commands.clear_interestpoints(xml, correspondences_only=True, dry_run=True) == rep
    assert _files(str(tmp_path)) == before


def test_clear_correspondences_only(tmp_path):
    xml, views = _ip_scene(tmp_path)
    pts = {(v, lab): _points(tmp_path, v, lab) for v in views for lab in ("beads",)}
    xml_bytes = open(xml, "rb").read()
    rep = commands.clear_interestpoints(xml, correspondences_only=True)
    assert rep[views[0]]["beads"][1] > 0
    assert open(xml, "rb").read() == xml_bytes
    st = bn5.N5Store(os.path.join(str(tmp_path), "interestpoints.n5"))
    for (v, lab), p in pts.items():
        assert np.array_equal(_points(tmp_path, v, lab), p)
    for v, lab in [(views[0], "beads"), (views[1], "beads"), (views[0], "nuclei")]:
        g = f"tpId_{v[0]}_viewSetupId_{v[1]}/{lab}"
        assert st.read_correspondences(g) == []
        assert st.get_attributes(g + "/correspondences")["idMap"] == {}
        assert st.get_attributes(g + "/correspondences/data")["dimensions"] == [0]
    assert commands.clear_interestpoints(xml, dry_run=True) == {
        views[0]: {"beads": (len(pts[(views[0], "beads")]), 0), "nuclei": (5, 0)},
        views[1]: {"beads": (len(pts[(views[1], "beads")]), 0)}}


def test_clear_everything(tmp_path):
    xml, views = _ip_scene(tmp_path)
    commands.clear_interestpoints(xml)
    assert not os.path.exists(tmp_path / "interestpoints.n5")
    root = ET.parse(xml).getroot()
    assert len(root.find("ViewInterestPoints")) == 0 and not list(root.iter("ViewInterestPointsFile"))
    assert list(ET.parse(xml + "~1").getroot().iter("ViewInterestPointsFile"))
    assert spimdata.SpimData2.load(xml).interest_points() == {}
    assert commands.clear_interestpoints(xml) == {}


def test_matching_after_clearing_equals_matching_a_fresh_scene(tmp_path):
    fresh, used = tmp_path / "fresh", tmp_path / "used"
    for d in (fresh, used):
        d.mkdir()
    xml_f, _ = planted_scene(fresh, tile=(120, 100, 40))
    commands.match_interestpoints(xml_f, MatchFakeContext(), ["beads"], **RUN)
    xml_u, views = _ip_scene(used)
    st = bn5.N5Store(os.path.join(str(used), "interestpoints.n5"))
    # stored rows a new match would not produce: without clearing they would stay
    st.write_correspondences("tpId_0_viewSetupId_0/beads", [(0, (0, 1), "beads", 1), (2, (0, 1), "beads", 3)])
    commands.clear_interestpoints(xml_u, correspondences_only=True)
    commands.match_interestpoints(xml_u, MatchFakeContext(), ["beads"], **RUN)
    want = read_rows(fresh, views)
    assert read_rows(used, views) == want and all(len(r) > 20 for r in want.values())


# ------------------------------------------------------------------------------------------ clear-registrations
def _affine(k):
    m = np.zeros((3, 4))
    m[:, :3] = np.eye(3) * (1.0 + 0.5 * k)
    m[:, 3] = (k, -2.0 * k, 0.25 * k)
    return m


def _reg_scene(tmp_path):
    """Views (0, s), s = 0..3, with s + 1 transforms named `v{s}t{k}`, k = 0 first in the list."""
    tiles = [dict(setup=s, size_xyz=(10, 10, 10), translation_xyz=(0, 0, 0)) for s in range(4)]
    xml = str(tmp_path / "dataset.xml")
    spimdata.write_dataset_xml(xml, "dataset.n5", tiles)
    tree = ET.parse(xml)
    regs = {}
    for vr in tree.getroot().iter("ViewRegistration"):
        s = int(vr.get("setup"))
        for vt in vr.findall("ViewTransform"):
            vr.remove(vt)
        regs[(0, s)] = []
        for k in range(s + 1):
            vt = ET.SubElement(vr, "ViewTransform", type="affine")
            ET.SubElement(vt, "Name").text = f"v{s}t{k}"
            ET.SubElement(vt, "affine").text = " ".join(repr(float(v)) for v in _affine(10 * s + k).ravel())
            regs[(0, s)].append((f"v{s}t{k}", _affine(10 * s + k)))
    tree.write(xml, encoding="UTF-8", xml_declaration=True)
    return xml, regs


def _same(a, b):
    return [n for n, _ in a] == [n for n, _ in b] and all(np.array_equal(x, y) for (_, x), (_, y) in zip(a, b))


@pytest.mark.parametrize("kw, cut", [(dict(remove=2), lambda n: min(2, n)), (dict(keep=2), lambda n: max(n - 2, 0)),
                                     (dict(remove=0), lambda n: 0), (dict(keep=0), lambda n: n),
                                     (dict(remove=9), lambda n: n)])
def test_keep_and_remove(tmp_path, kw, cut):
    xml, regs = _reg_scene(tmp_path)
    removed = commands.clear_registrations(xml, **kw)
    after = spimdata.SpimData2.load(xml).registrations
    for v, lst in regs.items():
        assert _same(removed[v], lst[:cut(len(lst))]) and _same(after[v], lst[cut(len(lst)):]), v


def test_only_the_selected_views_change(tmp_path):
    xml, regs = _reg_scene(tmp_path)
    removed = commands.clear_registrations(xml, remove=1, view_selection=dict(vi=["0,2", "0,3"]))
    assert sorted(removed) == [(0, 2), (0, 3)]
    after = spimdata.SpimData2.load(xml).registrations
    for v, lst in regs.items():
        assert _same(after[v], lst[1:] if v[1] >= 2 else lst), v


@pytest.mark.parametrize("kw", [dict(), dict(keep=1, remove=1), dict(keep=-1), dict(remove=-1)])
def test_clear_registrations_rejects(tmp_path, kw):
    xml, _ = _reg_scene(tmp_path)
    before = open(xml, "rb").read()
    with pytest.raises(ValueError, match="--keep OR --remove"):
        commands.clear_registrations(xml, **kw)
    assert open(xml, "rb").read() == before


def test_clear_registrations_dry_run_leaves_the_file(tmp_path):
    xml, regs = _reg_scene(tmp_path)
    before = open(xml, "rb").read()
    removed = commands.clear_registrations(xml, keep=1, dry_run=True)
    assert open(xml, "rb").read() == before and not os.path.exists(xml + "~1")
    for v, lst in regs.items():
        assert _same(removed[v], lst[:len(lst) - 1])


# ------------------------------------------------------------------------------------------ transform-points
def _tp_scene(tmp_path):
    """View (0, 0): affine A (rotation about z, then x + 1, z - 2) o translation (10, -4, 3) o calibration diag(1, 1, 2);
    view (0, 1): the identity."""
    tiles = [dict(setup=s, size_xyz=(10, 10, 10), translation_xyz=(0, 0, 0)) for s in range(2)]
    xml = str(tmp_path / "dataset.xml")
    spimdata.write_dataset_xml(xml, "dataset.n5", tiles)
    tree = ET.parse(xml)
    for vr in tree.getroot().iter("ViewRegistration"):
        for vt in vr.findall("ViewTransform"):
            vr.remove(vt)
        lst = [("affine", [0, -1, 0, 1, 1, 0, 0, 0, 0, 0, 1, -2]), ("translation", [1, 0, 0, 10, 0, 1, 0, -4, 0, 0, 1, 3]),
               ("calibration", [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 2, 0])] if vr.get("setup") == "0" else \
            [("calibration", [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])]
        for name, m in lst:
            vt = ET.SubElement(vr, "ViewTransform", type="affine")
            ET.SubElement(vt, "Name").text = name
            ET.SubElement(vt, "affine").text = " ".join(repr(float(v)) for v in m)
    tree.write(xml, encoding="UTF-8", xml_declaration=True)
    return xml


def test_hand_computed_composition(tmp_path, capsys):
    xml = _tp_scene(tmp_path)
    # (1, 2, 3) -> calibration (1, 2, 6) -> translation (11, -2, 9) -> affine (-(-2) + 1, 11, 9 - 2)
    w = commands.transform_points(xml, (0, 0), points=["1,2,3", (0.5, 0, -1)])
    assert np.array_equal(w, [[3.0, 11.0, 7.0], [5.0, 10.5, -1.0]])
    assert capsys.readouterr().out == "3.0,11.0,7.0\n5.0,10.5,-1.0\n"


def test_csv_lines_that_do_not_match_are_ignored(tmp_path, capsys):
    xml = _tp_scene(tmp_path)
    csv = tmp_path / "in.csv"
    csv.write_text("x,y,z\n1,2,3\n\n   \n1e-5,0,0\n  4.5 , -1 , 0 \n0.00001,250,-7,\nNaN,1,1\n12,3,4,99\n")
    out = tmp_path / "out.csv"
    w = commands.transform_points(xml, "0,1", points=["0,0,1e7"], csv_in=str(csv), csv_out=str(out))
    assert np.array_equal(w, [[1, 2, 3], [4.5, -1, 0], [1e-5, 250, -7], [12, 3, 4], [0, 0, 1e7]])
    assert out.read_text() == "1.0,2.0,3.0\n4.5,-1.0,0.0\n1.0E-5,250.0,-7.0\n12.0,3.0,4.0\n0.0,0.0,1.0E7\n"
    assert capsys.readouterr().out == ""


def test_java_number_format():
    assert [commands.java_double(v) for v in (1.0, 1e-5, -0.0, 0.0, 1234567.5, 1e7, -0.001, 0.00099)] == [
        "1.0", "1.0E-5", "-0.0", "0.0", "1234567.5", "1.0E7", "-0.001", "9.9E-4"]


def test_transform_points_rejects(tmp_path):
    xml = _tp_scene(tmp_path)
    csv = tmp_path / "in.csv"
    csv.write_text("x,y,z\n1e-5,1,1\n")
    with pytest.raises(ValueError, match="No points"):
        commands.transform_points(xml, (0, 0), csv_in=str(csv))
    with pytest.raises(ValueError, match="x,y,z"):
        commands.transform_points(xml, (0, 0), points=["1,2"])
    with pytest.raises(ValueError, match="not in"):
        commands.transform_points(xml, (0, 7), points=["1,2,3"])
