"""TIFF datasets (`spimreconstruction.filemap2`) on the device: the same seeded bead views as a `bdv.n5` dataset and as
Deflate + Predictor 2 TIFF files give identical resave levels, stitching results, interest points, affine-fusion
blocks (the windowed z-slab path, with windows that cover part of each view) and non-rigid fusion blocks.  Only the
byte source differs, so every output is bit for bit the same."""
import os

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata
from bsgpu import zarr as bz
from tests.tiff_files import twin_datasets

pytestmark = pytest.mark.gpu


def _files(root):
    return {os.path.relpath(os.path.join(dp, f), root): open(os.path.join(dp, f), "rb").read()
            for dp, _, fs in os.walk(root) for f in fs}


def _twins(tmp_path):
    from tests.test_interestpoints_gpu import _beads
    rng = np.random.default_rng(11)
    world = np.stack([rng.uniform(6, 186, 120), rng.uniform(6, 90, 120), rng.uniform(3, 37, 120)], 1)
    vols, trans = {}, {}
    for s, t in enumerate((0.0, 64.0)):
        local = world - (t, 0, 0)
        inside = local[(local[:, 0] > 3) & (local[:, 0] < 125)]
        vols[s] = _beads((40, 96, 128), [tuple(p) for p in inside], 1 + s, sigma_xy=1.6, sigma_z=1.6)
        trans[s] = (t + (1.5 if s else 0.0), 0.0, 0.0)
    assert all(v.dtype == np.uint16 for v in vols.values())          # the windowed fusion path takes uint16
    return twin_datasets(str(tmp_path), vols, trans, compression=8, predictor=2, rows_per_strip=16)


def test_tiff_dataset_equals_n5_twin_on_the_device(ctx, tmp_path):
    xn, xt = _twins(tmp_path)
    got = {}
    for name, x in (("n", xn), ("t", xt)):
        d = os.path.dirname(x)
        out = dict(resave={})
        for n5 in (True, False):
            os.makedirs(os.path.join(d, f"r{int(n5)}"))
            commands.resave(x, ctx, xml_out=os.path.join(d, f"r{int(n5)}", "dataset.xml"), n5=n5,
                            block_size=(32, 32, 8), block_scale=(2, 2, 3), downsampling="1,1,1; 2,2,1; 4,4,2")
            out["resave"][n5] = _files(os.path.join(d, f"r{int(n5)}", "dataset.n5" if n5 else "dataset.ome.zarr"))
        raw = commands.stitching(x, ctx, downsampling=(1, 1, 1))
        out["stitching"] = [(r.pair, np.asarray(r.transform).tolist(), r.r) for r in raw if r is not None]
        out["stitching_xml"] = [(r["pair"], r["shift"].tolist(), r["r"], r["bbox"])
                                for r in spimdata.SpimData2.load(x).stitching_results()]
        det = commands.detect_interestpoints(x, ctx, "beads", sigma=1.6, threshold=0.01, min_intensity=0.0,
                                             max_intensity=1000.0, downsample_xy=1, block_size=(64, 64, 24))
        out["detect"] = {k: v[0].tolist() for k, v in det.items()}
        res = commands.match_interestpoints(x, ctx, ["beads"], "PRECISE_TRANSLATION", ransac_min_num_inliers=8,
                                            transformation_model="TRANSLATION", regularization_model="NONE")
        out["match"] = {k: np.asarray(v).tolist() for k, v in res.items()}
        fused = os.path.join(d, "fused.zarr")
        # 8-plane z-slabs over 40-plane views: every slab stages a partial source window
        commands.create_fusion_container(x, fused, block_size=(64, 32, 8), dtype="uint16", min_intensity=0.0,
                                         max_intensity=1000.0, downsamplings=[(2, 2, 1)])
        commands.affine_fusion(fused, ctx, "AVG_BLEND", block_scale=(2, 2, 1))
        fz = bz.ZarrStore(fused)
        out["fused"] = [fz.read_volume("0"), fz.read_volume("1")]
        nr = os.path.join(d, "nonrigid.n5")
        out["written"] = commands.nonrigid_fusion(x, ctx, nr, "fused/s0", ["beads"], block_size=(64, 64, 24))
        out["nonrigid"] = bn5.N5Store(nr).read_volume("fused/s0")
        got[name] = out
    n, t = got["n"], got["t"]
    for n5 in (True, False):
        assert len(n["resave"][n5]) > 10 and t["resave"][n5] == n["resave"][n5], n5
    for k in ("stitching", "stitching_xml", "detect", "match", "written"):
        assert n[k] == t[k], k
    assert len(n["stitching"]) == 1 and len(n["stitching_xml"]) >= 1
    assert len(n["detect"]) == 2 and all(len(v) > 20 for v in n["detect"].values())
    assert sum(len(v) for v in n["match"].values()) >= 8
    assert all(np.array_equal(a, b) for a, b in zip(n["fused"], t["fused"])) and n["fused"][0].max() > 0
    assert np.array_equal(n["nonrigid"], t["nonrigid"]) and n["nonrigid"].max() > 0
