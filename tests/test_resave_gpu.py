"""resave on the device: the containers it writes equal, chunk for decoded chunk, those of the oracle-backed context at
every level (with the pyramid resident, mixed, and built from the stored levels), and the chain resave -> stitching /
detect / match / affine-fusion / non-rigid fusion giving identical outputs on the N5 and the OME-ZARR copy of one
dataset."""
import os

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata
from bsgpu import zarr as bz
from bsgpu import zstd as bzstd
from tests import synth
from tests.fake_ctx import FakeContext
from tests.test_resave_cpu import half_pixel_chain

pytestmark = pytest.mark.gpu


def _dataset(tmp_path, sizes=((200, 180, 70), (190, 170, 66))):
    G = synth.field((72, 190, 400), seed=5, sigma=1.2)
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles, vols = [], {}
    for s, size in enumerate(sizes):
        vols[s] = synth.tile_from(G, (1, 2, 160 * s + 3), size[::-1], 40 + s, noise=5.0)
        bn5.write_bdv_setup(store, s, 0, vols[s], (64, 64, 32), compression="zstd")
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(160 * s, 0, 0)))
    return spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles), vols


def _decoded_files(root):
    """{relative path: bytes} of every file under a container, chunk payloads decompressed."""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(dp, f)
            b = open(p, "rb").read()
            if not f.startswith(".") and f != "attributes.json":
                if b[:4] == bzstd.MAGIC.to_bytes(4, "little"):
                    b = bzstd.decompress(b)
                elif b[4 + 12:4 + 16] == bzstd.MAGIC.to_bytes(4, "little"):     # N5: 16-byte header, then zstd
                    b = b[:16] + bzstd.decompress(b[16:])
            out[os.path.relpath(p, root)] = b
    return out


STEPS = [(1, 1, 1), (2, 2, 1), (4, 4, 2)]


@pytest.mark.parametrize("n5", [False, True])
@pytest.mark.parametrize("block_scale", [(4, 4, 2), (2, 2, 2), (1, 1, 1)])   # resident / mixed / from the stored levels
def test_device_resave_equals_fake_context(ctx, tmp_path, n5, block_scale):
    xml, vols = _dataset(tmp_path)
    out = {}
    for name, c in (("gpu", ctx), ("fake", FakeContext())):
        os.makedirs(tmp_path / name)
        commands.resave(xml, c, xml_out=str(tmp_path / name / "dataset.xml"), n5=n5, block_size=(64, 64, 16),
                        block_scale=block_scale, downsampling=STEPS)
        out[name] = _decoded_files(str(tmp_path / name / ("dataset.n5" if n5 else "dataset.ome.zarr")))
    assert sorted(out["gpu"]) == sorted(out["fake"]) and len(out["gpu"]) > 20
    for k in out["gpu"]:
        assert out["gpu"][k] == out["fake"][k], k
    x = str(tmp_path / "gpu" / "dataset.xml")
    from bsgpu import viewsource
    src = viewsource.open_views(spimdata.SpimData2.load(x))
    for s, vol in vols.items():
        for lvl, w in enumerate(half_pixel_chain(vol, STEPS)):
            assert np.array_equal(src.read_volume((0, s), lvl), w)


def test_chain_on_n5_and_zarr_copies(ctx, tmp_path):
    from tests.test_interestpoints_gpu import _beads
    rng = np.random.default_rng(9)
    world = np.stack([rng.uniform(6, 186, 90), rng.uniform(6, 90, 90), rng.uniform(3, 21, 90)], 1)
    tiles = []
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    for s, t in enumerate((0.0, 64.0)):
        local = world - (t, 0, 0)
        inside = local[(local[:, 0] > 3) & (local[:, 0] < 125)]
        vol = _beads((24, 96, 128), [tuple(p) for p in inside], 1 + s, sigma_xy=1.6, sigma_z=1.6)
        bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 16))
        tiles.append(dict(setup=s, size_xyz=(128, 96, 24), tile=s, translation_xyz=(t + (1.5 if s else 0.0), 0, 0)))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    kw = dict(block_size=(32, 32, 8), block_scale=(2, 2, 3), downsampling="1,1,1; 2,2,1; 4,4,2")
    got = {}
    for name, n5 in (("n", True), ("z", False)):
        os.makedirs(tmp_path / name)
        x = str(tmp_path / name / "dataset.xml")
        commands.resave(xml, ctx, xml_out=x, n5=n5, **kw)
        raw = commands.stitching(x, ctx, downsampling=(2, 2, 1))
        det = commands.detect_interestpoints(x, ctx, "beads", sigma=1.6, threshold=0.01, min_intensity=0.0,
                                             max_intensity=1000.0, downsample_xy=2, block_size=(64, 64, 24))
        det1 = commands.detect_interestpoints(x, ctx, "beads1", sigma=1.6, threshold=0.01, min_intensity=0.0,
                                              max_intensity=1000.0, downsample_xy=1, block_size=(64, 64, 24))
        res = commands.match_interestpoints(x, ctx, ["beads1"], "PRECISE_TRANSLATION", ransac_min_num_inliers=8,
                                            transformation_model="TRANSLATION", regularization_model="NONE")
        fused = str(tmp_path / name / "fused.zarr")
        commands.create_fusion_container(x, fused, block_size=(64, 32, 16), dtype="uint16", min_intensity=0.0,
                                         max_intensity=1000.0, downsamplings=[(2, 2, 1)])
        commands.affine_fusion(fused, ctx, "AVG_BLEND")
        nr = str(tmp_path / name / "nonrigid.n5")
        written = commands.nonrigid_fusion(x, ctx, nr, "fused/s0", ["beads1"], block_size=(64, 64, 24))
        fz = bz.ZarrStore(fused)
        got[name] = dict(
            stitching=[(r.pair, np.asarray(r.transform).tolist(), r.r) for r in raw if r is not None],
            detect={k: v[0].tolist() for k, v in det.items()}, detect1={k: v[0].tolist() for k, v in det1.items()},
            match={k: np.asarray(v).tolist() for k, v in res.items()},
            fused=[fz.read_volume("0"), fz.read_volume("1")], written=written,
            nonrigid=bn5.N5Store(nr).read_volume("fused/s0"))
    n, z = got["n"], got["z"]
    for k in ("stitching", "detect", "detect1", "match", "written"):
        assert n[k] == z[k], k
    assert len(n["stitching"]) == 1 and len(n["detect"]) == 2 and sum(len(v) for v in n["match"].values()) >= 8
    assert all(np.array_equal(a, b) for a, b in zip(n["fused"], z["fused"])) and n["fused"][0].max() > 0
    assert np.array_equal(n["nonrigid"], z["nonrigid"]) and n["nonrigid"].max() > 0
