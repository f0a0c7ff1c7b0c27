"""split-images on the CPU: the interval plan (hand-computed cases and an invariant sweep), the project it writes (setups,
tiles, illuminations, registrations, missing views, the split loader and its paths, backups, dry runs), the sub-view
reads of N5 and OME-ZARR pyramids, split of a split, the interest points carried over, the fake points, and
split -> affine-fusion against the unsplit fusion through the oracle-backed context."""
import os

import numpy as np
import pytest

from bsgpu import commands, n5 as bn5, spimdata, split as bsplit, viewsource
from tests import synth
from tests.fake_ctx import FakeContext

STEPS = [(1, 1, 1), (2, 2, 1)]


def make_dataset(root, sizes=((71, 45, 12), (66, 41, 10)), shift=50, n5=True, pyramid=True, seed=3):
    """Two uint16 tiles at integer translations (shift, 0, 0) apart, re-saved with a (1,1,1), (2,2,1) pyramid into
    `root/p/dataset.xml` (N5 or OME-ZARR) when ``pyramid``.  Returns (xml path, {setup: level-0 volume})."""
    os.makedirs(root, exist_ok=True)
    G = synth.field((max(s[2] for s in sizes) + 2, max(s[1] for s in sizes) + 3,
                     shift * (len(sizes) - 1) + max(s[0] for s in sizes) + 3), seed=seed, sigma=1.0)
    store = bn5.N5Store(os.path.join(root, "dataset.n5"), create=True)
    tiles, vols = [], {}
    for s, size in enumerate(sizes):
        vols[s] = synth.tile_from(G, (1, 2, shift * s + 2), size[::-1], 20 + s, noise=5.0)
        bn5.write_bdv_setup(store, s, 0, vols[s], (16, 16, 8))
        tiles.append(dict(setup=s, size_xyz=size, tile=s, translation_xyz=(shift * s, 0, 0)))
    xml = spimdata.write_dataset_xml(os.path.join(root, "dataset.xml"), "dataset.n5", tiles)
    if not pyramid:
        return xml, vols
    out = os.path.join(root, "p", "dataset.xml")
    os.makedirs(os.path.dirname(out))
    commands.resave(xml, FakeContext(), xml_out=out, n5=n5, block_size=(16, 16, 8), block_scale=(1, 1, 1),
                    downsampling=STEPS)
    return out, vols


# ------------------------------------------------------------------------------------------------ planning
@pytest.mark.parametrize("L, s, o, m, opt, want", [
    (30, 40, 10, 1, True, [(0, 29)]),
    (100, 40, 10, 1, False, [(0, 39), (30, 69), (60, 99)]),
    (100, 40, 10, 1, True, [(0, 39), (30, 69), (60, 99)]),
    (110, 40, 10, 1, False, [(0, 39), (30, 69), (60, 99), (90, 109)]),
    (110, 40, 10, 1, True, [(0, 34), (25, 59), (50, 84), (75, 109)]),
    (70, 48, 16, 4, False, [(0, 47), (32, 69)]),
    (70, 48, 16, 4, True, [(0, 43), (28, 69)]),
    (41, 40, 0, 1, False, [(0, 39), (40, 40)]),
])
def test_intervals_hand_computed(L, s, o, m, opt, want):
    assert bsplit.intervals(L, s, o, m, opt) == want


def test_interval_invariants_sweep():
    rng = np.random.default_rng(0)
    for _ in range(3000):
        m = int(rng.choice([1, 2, 4, 8]))
        s = m * int(rng.integers(1, 20))
        o = m * int(rng.integers(0, s // m))
        L = int(rng.integers(1, 12 * s))
        a = bsplit.intervals(L, s, o, m, False)
        b = bsplit.intervals(L, s, o, m, True)
        assert len(a) == len(b)                                  # optimisation keeps the count
        for iv in (a, b):
            assert iv[0][0] == 0 and iv[-1][1] == L - 1
            for k, (lo, hi) in enumerate(iv):
                assert lo % m == 0 and lo <= hi and hi - lo + 1 <= s and hi < L
                if k:
                    assert lo > iv[k - 1][0] and iv[k - 1][1] - lo + 1 >= o and lo <= iv[k - 1][1] + 1


def test_overlap_errors(tmp_path):
    with pytest.raises(ValueError, match="smaller than the image size"):
        bsplit.intervals(100, 32, 32, 1)
    assert bsplit.intervals(30, 32, 32, 1) == [(0, 29)]           # an axis that is not split takes any overlap <= size
    xml, _ = make_dataset(str(tmp_path), pyramid=False)
    with pytest.raises(ValueError, match="cannot be bigger"):
        commands.split_images(xml, "32,32,8", "33,8,8")
    with pytest.raises(ValueError, match="smaller than the image size"):
        commands.split_images(xml, (32, 32, 8), (32, 8, 8))
    with pytest.raises(NotImplementedError):
        commands.split_images(xml, (32, 32, 8), (8, 8, 8), display_result=True)


def test_step_rounds_size_and_overlap(tmp_path):
    xml, _ = make_dataset(str(tmp_path))
    res = commands.split_images(xml, "31,17,5", "3,3,1", dry_run=True)
    assert res["step"] == (2, 2, 1) and res["size"] == (32, 18, 5) and res["overlap"] == (4, 4, 1)
    for old, mn, mx in res["views"].values():
        assert mn[0] % 2 == 0 and mn[1] % 2 == 0


# ------------------------------------------------------------------------------------------------ the project
def _tile_attributes(xml):
    d = spimdata.SpimData2.load(xml)
    d.set_attribute_entries("tile", {0: dict(name="left", location=np.array([0.0, 0.0, 0.0])),
                                     1: dict(name="right", location=np.array([50.0, 0.0, 0.0]))})
    d.set_missing_views({(0, 1)})
    d.set_bounding_box("roi", (1, 2, 3), (40, 30, 9))
    d.set_stitching_results([dict(pair=((0, 0), (0, 1)), shift=np.eye(3, 4), r=0.9, hash=1.0, bbox_min=[0, 0, 0],
                                  bbox_max=[1, 1, 1])])
    d.save(xml, backup=False)


def test_project_round_trip(tmp_path):
    xml, _ = make_dataset(str(tmp_path), pyramid=False)
    _tile_attributes(xml)
    old = spimdata.SpimData2.load(xml)
    out = str(tmp_path / "other" / "split.xml")
    res = commands.split_images(xml, "32,32,8", "8,8,4", xml_out=out, assign_illuminations=True)
    new = spimdata.SpimData2.load(out)
    # 71 x 45 x 12 -> 3 x 2 x 2 boxes, 66 x 41 x 10 -> 3 x 2 x 2: ids 0..11 of setup 0, then 12..23 of setup 1
    assert sorted(new.setups) == list(range(24)) and res["views"][0][0] == 0 and res["views"][12][0] == 1
    spread = 12
    for nid, (o, mn, mx) in res["views"].items():
        vs = new.setups[nid]
        assert vs.size == tuple(int(mx[d] - mn[d] + 1) for d in range(3))
        k = nid - 12 * o
        assert vs.attributes["tile"] == o * spread + k and vs.attributes["illumination"] == o
        assert vs.attributes["channel"] == 0 and vs.attributes["angle"] == 0
        if (0, o) not in old.missing_views():
            assert new.registrations[(0, nid)][-1][0] == "Image Splitting"
            T = np.hstack([np.eye(3), np.asarray(mn, dtype=np.float64)[:, None]])
            assert np.allclose(new.model(0, nid), old.model(0, o) @ np.vstack([T, [0, 0, 0, 1]]), atol=0)
    assert new.missing_views() == {(0, n) for n in range(12, 24)}
    tiles = new.attribute_entries("tile")
    assert sorted(tiles) == sorted(o * spread + (n - 12 * o) for n, (o, _, _) in res["views"].items())
    mn13 = np.asarray(res["views"][13][1], dtype=np.float64)
    assert tiles[13]["name"] == "13" and np.array_equal(tiles[13]["location"], np.array([50.0, 0, 0]) + mn13)
    assert {i: e["name"] for i, e in new.attribute_entries("illumination").items()} == {0: "left", 1: "right"}
    assert "roi" in new.bounding_boxes() and new.stitching_results() == []
    # the loader: the input's bdv.n5 element, re-based from the other directory, and one definition per new setup
    il = new.root.find("SequenceDescription/ImageLoader")
    assert il.get("format") == "split.viewerimgloader" and il.find("ImageLoader").get("format") == "bdv.n5"
    assert il.find("ImageLoader/n5").text == os.path.join("..", "dataset.n5")
    assert new.image_loader(nested=True) == ("bdv.n5", str(tmp_path / "dataset.n5"))
    assert {k: (o, tuple(a), tuple(b)) for k, (o, a, b) in new.split_setups().items()} == res["views"]
    d = il.find("SetupIds").findall("SetupIdDefinition")[1]
    assert [c.tag for c in d] == ["NewId", "OldId", "min", "max"]
    # two illuminations cannot take the tile ids
    d2 = spimdata.SpimData2.load(xml)
    for vs in d2.root.find("SequenceDescription/ViewSetups").findall("ViewSetup"):
        vs.find("attributes/illumination").text = vs.findtext("id")
    d2.save(xml, backup=False)
    with pytest.raises(ValueError, match="more than one illumination"):
        commands.split_images(xml, "32,32,8", "8,8,4", xml_out=out, assign_illuminations=True)


def test_backup_and_dry_run(tmp_path):
    xml, _ = make_dataset(str(tmp_path), pyramid=False)
    before = open(xml, "rb").read()
    files = sorted(os.listdir(tmp_path))
    res = commands.split_images(xml, "32,32,8", "8,8,4", dry_run=True)
    assert len(res["views"]) == 24 and open(xml, "rb").read() == before and sorted(os.listdir(tmp_path)) == files
    commands.split_images(xml, "32,32,8", "8,8,4")
    assert open(xml + "~1", "rb").read() == before
    assert len(spimdata.SpimData2.load(xml).setups) == 24


# ------------------------------------------------------------------------------------------------ reads
@pytest.mark.parametrize("n5", [True, False])
def test_sub_view_reads_every_level(tmp_path, n5):
    xml, _ = make_dataset(str(tmp_path), n5=n5)
    parent_src = viewsource.open_views(spimdata.SpimData2.load(xml))
    out = str(tmp_path / "split.xml")
    res = commands.split_images(xml, "32,16,8", "8,4,2", xml_out=out)
    src = viewsource.open_views(spimdata.SpimData2.load(out))
    assert isinstance(src, viewsource.SplitViews) and src.inner.format == ("bdv.n5" if n5 else "bdv.multimg.zarr")
    clipped = 0
    for nid, (old, mn, mx) in res["views"].items():
        assert src.mipmap_info((0, nid))[0] == parent_src.mipmap_info((0, old))[0] == STEPS
        for lvl, f in enumerate(STEPS):
            pv = parent_src.read_volume((0, old), lvl)
            lo = [mn[d] // f[d] for d in range(3)]
            hi = [min(mx[d] // f[d], pv.shape[2 - d] - 1) for d in range(3)]
            clipped += any(mx[d] // f[d] > pv.shape[2 - d] - 1 for d in range(3))
            want = pv[lo[2]:hi[2] + 1, lo[1]:hi[1] + 1, lo[0]:hi[0] + 1]
            got = src.read_volume((0, nid), lvl)
            assert np.array_equal(got, want) and src.level_dims((0, nid), lvl) == want.shape[::-1]
            # a region reaching outside the sub-view reads zeros there, not the parent's neighbouring voxels
            reg = src.read_region((0, nid), lvl, (-3, 2, 0), (want.shape[2] + 6, 3, 2))
            exp = np.zeros_like(reg)
            part = want[0:2, 2:5, :]
            exp[:part.shape[0], :part.shape[1], 3:3 + want.shape[2]] = part
            assert np.array_equal(reg, exp)
    assert clipped > 0                         # an odd parent edge is clipped at level 1


def test_split_of_split_flattens(tmp_path):
    xml, _ = make_dataset(str(tmp_path))
    parent_src = viewsource.open_views(spimdata.SpimData2.load(xml))
    a, b = str(tmp_path / "a.xml"), str(tmp_path / "sub" / "b.xml")
    ra = commands.split_images(xml, "40,32,8", "8,8,2", xml_out=a)
    rb = commands.split_images(a, "20,16,8", "4,4,2", xml_out=b)
    db = spimdata.SpimData2.load(b)
    il = db.root.find("SequenceDescription/ImageLoader")
    assert il.find("ImageLoader").get("format") == "bdv.n5" and il.find("ImageLoader/ImageLoader") is None
    defs = db.split_setups()
    src = viewsource.open_views(db)
    for nid, (mid, mn, mx) in rb["views"].items():
        orig, amn, _ = ra["views"][mid]
        o, cmn, cmx = defs[nid]
        assert o == orig and np.array_equal(cmn, np.add(amn, mn)) and np.array_equal(cmx, np.add(amn, mx))
        once = viewsource.SplitViews(parent_src, {nid: (orig, cmn, cmx)})
        for lvl in range(2):
            assert np.array_equal(src.read_volume((0, nid), lvl), once.read_volume((0, nid), lvl))
        # the composed registration equals the original's with the composed offset
        T = np.vstack([np.hstack([np.eye(3), cmn.astype(np.float64)[:, None]]), [0, 0, 0, 1]])
        assert np.allclose(db.model(0, nid), spimdata.SpimData2.load(xml).model(0, orig) @ T, atol=0)


# ------------------------------------------------------------------------------------------------ interest points
def _with_points(xml, seed=1, n=60):
    d = spimdata.SpimData2.load(xml)
    base = os.path.dirname(os.path.abspath(xml))
    st = bn5.N5Store(os.path.join(base, "interestpoints.n5"), create=True)
    rng = np.random.default_rng(seed)
    pts = {}
    for s, vs in d.setups.items():
        for label in ("beads", "nuclei"):
            loc = rng.uniform(0, 1, (n, 3)) * (np.asarray(vs.size) - 1)
            loc[0] = [32.0, 0.0, 4.0]                              # on a box face: kept by both closed boxes
            ids = rng.permutation(1000)[:n]
            g = f"tpId_0_viewSetupId_{s}/{label}"
            commands._write_view_points(st, g, ids, loc, rng.uniform(0, 9, n).astype(np.float32) if label == "beads" else None)
            st.write_correspondences(g, [(int(ids[0]), (0, 1 - s), label, 7)])
            pts[(s, label)] = (ids, loc)
    for label in ("beads", "nuclei"):
        d.set_interest_points(label, f"DOG {label}", {(0, s): f"tpId_0_viewSetupId_{s}/{label}" for s in d.setups})
    d.save(xml, backup=False)
    return pts


def test_interest_points_carried_over(tmp_path):
    xml, _ = make_dataset(str(tmp_path), pyramid=False)
    pts = _with_points(xml)
    res = commands.split_images(xml, "32,32,8", "8,8,4")          # in place: new ids reuse old ones
    new = spimdata.SpimData2.load(xml)
    st = bn5.N5Store(str(tmp_path / "interestpoints.n5"))
    ips = new.interest_points()
    on_face = 0
    for nid, (old, mn, mx) in res["views"].items():
        assert sorted(ips[(0, nid)]) == ["beads", "nuclei"] and ips[(0, nid)]["beads"]["params"] == "DOG beads"
        for label in ("beads", "nuclei"):
            ids, loc = pts[(old, label)]
            inside = np.all((loc >= mn) & (loc <= mx), axis=1)
            got_ids, got_loc, inten = commands._read_view_points(st, ips[(0, nid)][label]["path"])
            assert np.array_equal(got_ids, ids[inside]) and np.array_equal(got_loc, loc[inside] - mn)
            assert (inten is not None) == (label == "beads")
            assert st.read_correspondences(ips[(0, nid)][label]["path"]) == []
            on_face += bool(inside[0])
    assert on_face >= 4                                             # the face point is in more than one sub-view


# ------------------------------------------------------------------------------------------------ fake points
FIP = dict(fake_interest_points=True, fip_density=2000.0, fip_min_num_points=5, fip_max_num_points=40, fip_error=0.5,
           fip_exclusion_radius=3.0)


def _fip_files(root):
    out = {}
    for dp, _, fs in os.walk(os.path.join(root, "interestpoints.n5")):
        for f in fs:
            out[os.path.relpath(os.path.join(dp, f), root)] = open(os.path.join(dp, f), "rb").read()
    return out


def test_fake_points(tmp_path):
    xml, _ = make_dataset(str(tmp_path), pyramid=False)
    pts = _with_points(xml, n=30)
    out = str(tmp_path / "a" / "split.xml")
    res = commands.split_images(xml, "32,32,8", "8,8,4", xml_out=out, **FIP)
    new = spimdata.SpimData2.load(out)
    st = bn5.N5Store(str(tmp_path / "a" / "interestpoints.n5"))
    ips = new.interest_points()
    assert all("splitPoints" in ips[(0, nid)] for nid in res["views"])
    fake = {nid: commands._read_view_points(st, ips[(0, nid)]["splitPoints"]["path"]) for nid in res["views"]}
    r = FIP["fip_exclusion_radius"]
    for nid, (old, mn, mx) in res["views"].items():
        ids, loc, _ = fake[nid]
        assert np.array_equal(ids, np.arange(len(loc)))
        par = loc + mn
        existing = np.concatenate([pts[(old, lab)][1] for lab in ("beads", "nuclei")])
        assert np.min(np.linalg.norm(par[:, None] - existing[None], axis=2)) >= r
        dd = np.linalg.norm(par[:, None] - par[None], axis=2) + np.eye(len(par)) * 1e9
        assert len(par) < 2 or dd.min() >= r
    # counts follow density / min / max, unless the 100 n draws ran out
    for (tp, a, b), cnt in res["fake_points"].items():
        (oa, mna, mxa), (ob, mnb, mxb) = res["views"][a], res["views"][b]
        assert oa == ob and a < b
        vox = np.prod(np.minimum(mxa, mxb) - np.maximum(mna, mnb) + 1)
        want = min(40, max(5, int(np.ceil(2000.0 * vox / 1e6))))
        assert cnt <= want
    assert sum(res["fake_points"].values()) > 0.8 * sum(
        min(40, max(5, int(np.ceil(2000.0 * np.prod(np.minimum(res["views"][a][2], res["views"][b][2]) -
                                                       np.maximum(res["views"][a][1], res["views"][b][1]) + 1) / 1e6))))
        for (_, a, b) in res["fake_points"])
    # correspondences: symmetric, and the copies agree to fip_error
    n_corr = 0
    for nid, (old, mn, mx) in res["views"].items():
        g = ips[(0, nid)]["splitPoints"]["path"]
        for pid, pv, pl, qid in st.read_correspondences(g):
            assert pl == "splitPoints" and pv[0] == 0
            back = st.read_correspondences(ips[pv]["splitPoints"]["path"])
            assert (qid, (0, nid), "splitPoints", pid) in back
            omn = np.asarray(res["views"][pv[1]][1])
            assert np.all(np.abs(fake[pv[1]][1][qid] + omn - fake[nid][1][pid] - mn) <= FIP["fip_error"] + 1e-12)
            n_corr += 1
    assert n_corr == 2 * sum(res["fake_points"].values())
    # deterministic: a second run writes identical files
    out2 = str(tmp_path / "b" / "split.xml")
    commands.split_images(xml, "32,32,8", "8,8,4", xml_out=out2, **FIP)
    assert _fip_files(str(tmp_path / "a")) == _fip_files(str(tmp_path / "b"))
    # an existing label clashes
    with pytest.raises(ValueError, match="already exists"):
        commands.split_images(xml, "32,32,8", "8,8,4", xml_out=out2, **dict(FIP, fip_label="beads"))


def test_fake_point_counts_min_max():
    boxes = [(np.array([0, 0, 0]), np.array([39, 39, 9])), (np.array([30, 0, 0]), np.array([69, 39, 9]))]
    vox = 10 * 40 * 10
    for dens, lo, hi in ((1.0, 7, 50), (1e6, 3, 9), (2e4, 3, 500)):
        fakes, pairs = bsplit.fake_points(0, 0, boxes, np.zeros((0, 3)), dens, lo, hi, 0.5, 0.5)
        assert len(pairs[(0, 1)]) == min(hi, max(lo, int(np.ceil(dens * vox / 1e6))))
    # a radius that leaves no room: the pair stops after 100 n draws with fewer points
    fakes, pairs = bsplit.fake_points(0, 0, boxes, np.zeros((0, 3)), 1.0, 50, 50, 0.5, 100.0)
    assert len(pairs[(0, 1)]) == 1


# ------------------------------------------------------------------------------------------------ chain
@pytest.mark.parametrize("fusion_type", ["MAX_INTENSITY", "LOWEST_VIEWID_WINS"])
def test_split_then_fusion_equals_unsplit(tmp_path, fusion_type):
    xml, _ = make_dataset(str(tmp_path))
    split = str(tmp_path / "split.xml")
    commands.split_images(xml, "32,16,8", "8,4,2", xml_out=split)
    fused = {}
    for name, x in (("whole", xml), ("split", split)):
        path = str(tmp_path / f"{name}.n5")
        commands.create_fusion_container(x, path, block_size=(32, 16, 8), dtype="uint16", min_intensity=0.0,
                                         max_intensity=65535.0, downsamplings=[(2, 2, 1)])
        commands.affine_fusion(path, FakeContext(), fusion_type, block_scale=(1, 1, 1))
        st = bn5.N5Store(path)
        fused[name] = [st.read_volume("ch0tp0/s0"), st.read_volume("ch0tp0/s1")]
    assert fused["whole"][0].max() > 0
    for a, b in zip(fused["whole"], fused["split"]):
        assert np.array_equal(a, b)
