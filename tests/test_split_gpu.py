"""split-images feeding the device paths: affine-fusion of the split project equals the unsplit fusion bit for bit (and
the oracle-backed context's files), DoG detection on the sub-views finds the unsplit points away from the cut faces,
resave copies every sub-view's window, and the solver keeps the pieces of one view together through the fake points."""
import os

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata, viewsource
from oracle import dog_oracle
from tests.fake_ctx import FakeContext
from tests.test_interestpoints_gpu import _beads
from tests.test_split_cpu import STEPS, make_dataset

pytestmark = pytest.mark.gpu


def _fused_files(root):
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(dp, f)
            if f not in ("attributes.json", ".zattrs"):
                out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def _fuse(xml, path, c, fusion_type):
    commands.create_fusion_container(xml, path, block_size=(64, 32, 8), dtype="uint16", min_intensity=0.0,
                                     max_intensity=65535.0, downsamplings=[(2, 2, 1)])
    commands.affine_fusion(path, c, fusion_type)
    return _fused_files(path)


@pytest.mark.parametrize("n5", [True, False])
@pytest.mark.parametrize("fusion_type", ["MAX_INTENSITY", "LOWEST_VIEWID_WINS"])
def test_fusion_of_split_equals_unsplit(ctx, tmp_path, n5, fusion_type):
    xml, _ = make_dataset(str(tmp_path), sizes=((150, 90, 20), (141, 85, 18)), shift=100, n5=n5)
    split = str(tmp_path / "split.xml")
    commands.split_images(xml, "48,32,16", "16,8,4", xml_out=split)
    ext = "n5" if n5 else "zarr"
    whole = _fuse(xml, str(tmp_path / f"whole.{ext}"), ctx, fusion_type)
    dev = _fuse(split, str(tmp_path / f"split.{ext}"), ctx, fusion_type)
    fake = _fuse(split, str(tmp_path / f"fake.{ext}"), FakeContext(), fusion_type)
    assert sorted(whole) == sorted(dev) == sorted(fake) and len(whole) > 10
    for k in whole:
        assert dev[k] == whole[k], k
        assert dev[k] == fake[k], k


def _bead_dataset(root):
    rng = np.random.default_rng(4)
    world = np.stack([rng.uniform(4, 236, 160), rng.uniform(4, 92, 160), rng.uniform(3, 29, 160)], 1)
    os.makedirs(root)
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles = []
    for s, t in enumerate((0, 112)):
        local = world - (t, 0, 0)
        vol = _beads((32, 96, 128), [tuple(p) for p in local], 1 + s, sigma_xy=1.6, sigma_z=1.6)
        bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 16))
        tiles.append(dict(setup=s, size_xyz=(128, 96, 32), tile=s, translation_xyz=(t, 0, 0)))
    xml = spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)
    out = os.path.join(root, "p", "dataset.xml")
    os.makedirs(os.path.dirname(out))
    commands.resave(xml, FakeContext(), xml_out=out, n5=True, block_size=(32, 32, 16), block_scale=(1, 1, 1),
                    downsampling=STEPS)
    return out


@pytest.mark.parametrize("dsxy", [1, 2])
def test_detection_on_split_matches_unsplit(ctx, tmp_path, dsxy):
    xml = _bead_dataset(str(tmp_path / "d"))
    split = str(tmp_path / "d" / "p" / "split.xml")
    res = commands.split_images(xml, "64,48,32", "24,16,0", xml_out=split)
    kw = dict(sigma=1.6, threshold=0.01, min_intensity=0.0, max_intensity=1000.0, downsample_xy=dsxy,
              block_size=(48, 48, 16), dry_run=True)
    whole = commands.detect_interestpoints(xml, ctx, "beads", **kw)
    parts = commands.detect_interestpoints(split, ctx, "beads", **kw)
    d0, d1 = spimdata.SpimData2.load(xml), spimdata.SpimData2.load(split)
    sb = dog_oracle.compute_sigmas(1.6)[1]
    margin = (len(dog_oracle.gauss_kernel(sb)) // 2 + 2) * dsxy

    def world(data, v, loc):
        M = data.model(*v)
        return loc @ M[:, :3].T + M[:, 3]

    def interior(p, mn, mx, dims):
        return all((mn[d] == 0 or p[d] - mn[d] > margin) and (mx[d] == dims[d] - 1 or mx[d] - p[d] > margin)
                   for d in range(3))

    checked = found = 0
    for nid, (old, mn, mx) in res["views"].items():
        dims = d0.setups[old].size
        wp = world(d0, (0, old), whole[(0, old)][0])
        sp = world(d1, (0, nid), parts[(0, nid)][0])
        keep = [k for k, p in enumerate(parts[(0, nid)][0]) if interior(p + mn, mn, mx, dims)]
        for k in keep:
            assert np.min(np.max(np.abs(wp - sp[k]), axis=1)) <= 1e-9
            checked += 1
        for k, q in enumerate(whole[(0, old)][0]):
            if interior(q, mn, mx, dims) and np.all(q >= mn) and np.all(q <= mx):
                assert len(sp) and np.min(np.max(np.abs(sp - wp[k]), axis=1)) <= 1e-9
                found += 1
    assert checked > 50 and found > 50


def test_resave_of_split_copies_windows(ctx, tmp_path):
    xml, _ = make_dataset(str(tmp_path), sizes=((150, 90, 20), (141, 85, 18)), shift=100)
    split = str(tmp_path / "split.xml")
    res = commands.split_images(xml, "48,32,16", "16,8,4", xml_out=split)
    out = str(tmp_path / "r" / "dataset.xml")
    os.makedirs(os.path.dirname(out))
    commands.resave(split, ctx, xml_out=out, n5=True, block_size=(32, 32, 8), downsampling=STEPS)
    parent = viewsource.open_views(spimdata.SpimData2.load(xml))
    copy = viewsource.open_views(spimdata.SpimData2.load(out))
    assert isinstance(copy, viewsource.N5Views)
    for nid, (old, mn, mx) in res["views"].items():
        pv = parent.read_volume((0, old), 0)
        assert np.array_equal(copy.read_volume((0, nid), 0), pv[mn[2]:mx[2] + 1, mn[1]:mx[1] + 1, mn[0]:mx[0] + 1])


def test_fake_points_keep_pieces_together(ctx, tmp_path):
    xml, _ = make_dataset(str(tmp_path), sizes=((150, 90, 20), (141, 85, 18)), shift=100, pyramid=False)
    split = str(tmp_path / "split.xml")
    err = 0.5
    res = commands.split_images(xml, "64,48,20", "24,16,4", xml_out=split, fake_interest_points=True, fip_error=err,
                                fip_exclusion_radius=4.0)
    assert sum(res["fake_points"].values()) > 100
    out = commands.solver(split, ctx, "IP", labels=["splitPoints"], transformation_model="TRANSLATION",
                          regularization_model="NONE")
    models = out["models"]
    for a, (oa, _, _) in res["views"].items():
        for b, (ob, _, _) in res["views"].items():
            if oa == ob and a < b:
                d = np.asarray(models[(0, a)])[:, 3] - np.asarray(models[(0, b)])[:, 3]
                assert np.all(np.abs(d) <= 2 * err), (a, b, d)
