"""match-interestpoints without a GPU: the oracle's known answers (PARITY_GAPS M4-M8), the host logic (tasks, the M3
filter, correspondences written and read back) and the command end to end through an oracle-backed context."""
import os
import socket
import xml.etree.ElementTree as ET

import numpy as np
import pytest
from scipy.spatial import cKDTree

from bsgpu import commands, matching as bm, n5 as bn5, spimdata
from oracle import match_oracle as mo
from tests.fake_ctx import FakeContext


class MatchFakeContext(FakeContext):
    """FakeContext whose descriptor methods call oracle/match_oracle.py."""

    def __init__(self):
        super().__init__()
        self.sets = {}

    def descriptors_build(self, xyz, num_neighbors=3, redundancy=1):
        if num_neighbors < 3 or redundancy < 0 or num_neighbors + redundancy > 6:
            raise ValueError("bad (num_neighbors, redundancy)")
        h = self.next
        self.next += 1
        self.sets[h] = (np.asarray(xyz, dtype=np.float64).reshape(-1, 3), num_neighbors, redundancy)
        return h

    def descriptors_neighbors(self, h):
        xyz, n, r = self.sets[h]
        return mo.knn(xyz, n + r)

    def descriptors_match(self, ha, hb, search_radius=None):
        (xa, n, r), (xb, n2, r2) = self.sets[ha], self.sets[hb]
        assert (n, r) == (n2, r2)
        return mo.match(xa, xb, n, r, search_radius)

    def descriptors_free(self, h):
        del self.sets[h]


# ------------------------------------------------------------------------------------------ planted scenes
def rot_z(deg, centre):
    th = np.deg2rad(deg)
    R = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
    c = np.asarray(centre, dtype=np.float64)
    return np.hstack([R, (c - R @ c)[:, None]])


def compose(A, B):
    """A after B, 3 x 4 each."""
    return np.hstack([A[:, :3] @ B[:, :3], (A[:, :3] @ B[:, 3] + A[:, 3])[:, None]])


SPURIOUS_CLEARANCE = 8.0


def planted_scene(root, grid=(2, 1), tile=(200, 160, 60), overlap=0.3, spacing=14.0, keep=0.6, jitter=0.3, spurious=0.1,
                  off_px=3.0, rot_deg=1.0, seed=3, label="beads"):
    """Tiles of one bead cloud (lattice sites every ``spacing`` px, each kept with probability ``keep`` and moved by up to
    spacing / 4 per axis): true transforms are the nominal grid translations; the XML registrations are those
    composed with a few px of offset and rot_deg about z; every view stores the beads inside it (+ jitter) and
    spurious * n extra random points.  Returns (xml, truth): truth[view] maps point id -> bead index (-1 spurious)."""
    rng = np.random.default_rng(seed)
    step = [int(round(tile[d] * (1 - overlap))) for d in range(2)]
    extent = np.array([step[0] * (grid[0] - 1) + tile[0], step[1] * (grid[1] - 1) + tile[1], tile[2]], dtype=np.float64)
    # beads: a random subset of a jittered lattice, so that two beads are never within RANSAC's max_error of each other
    axes = [np.arange(spacing / 2, extent[d] - spacing / 2, spacing) for d in range(3)]
    sites = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    sites = sites[rng.random(len(sites)) < keep]
    beads = sites + rng.uniform(-spacing / 4, spacing / 4, sites.shape)
    tiles, truth, points = [], {}, {}
    setup = 0
    for gy in range(grid[1]):
        for gx in range(grid[0]):
            t = np.array([gx * step[0], gy * step[1], 0.0])
            loc = beads - t
            inside = np.nonzero(np.all((loc >= 0) & (loc <= np.array(tile) - 1), axis=1))[0]
            pts = loc[inside] + rng.normal(0.0, jitter, (len(inside), 3))
            ns = int(round(spurious * len(inside)))
            # spurious points keep clear of every bead, so no model can take one for a bead within max_error
            tree, extra = cKDTree(loc[inside]), np.zeros((0, 3))
            while len(extra) < ns:
                c = rng.uniform(0, 1, (2 * ns, 3)) * (np.array(tile) - 1)
                extra = np.vstack([extra, c[tree.query(c)[0] > SPURIOUS_CLEARANCE]])[:ns]
            pts = np.vstack([pts, extra])
            bead_of = np.concatenate([inside, -np.ones(ns, dtype=np.int64)])
            order = rng.permutation(len(pts))
            points[(0, setup)] = pts[order]
            truth[(0, setup)] = bead_of[order]
            reg = compose(rot_z(rot_deg * (1 if setup % 2 else -1), t + np.array(tile) / 2),
                          np.hstack([np.eye(3), (t + rng.uniform(-off_px, off_px, 3))[:, None]]))
            tiles.append(dict(setup=setup, size_xyz=tile, tile=setup, translation_xyz=(0, 0, 0), reg=reg))
            setup += 1
    xml = os.path.join(str(root), "dataset.xml")
    spimdata.write_dataset_xml(xml, "dataset.n5", tiles)
    tree = ET.parse(xml)
    for vr in tree.getroot().iter("ViewRegistration"):
        reg = tiles[int(vr.get("setup"))]["reg"]
        vr.find("ViewTransform").find("affine").text = " ".join(repr(float(v)) for v in reg.ravel())
    tree.write(xml, encoding="UTF-8", xml_declaration=True)
    store = bn5.N5Store(os.path.join(str(root), "interestpoints.n5"), create=True)
    for v, pts in points.items():
        write_points(store, v, label, pts)
    return xml, truth


def write_points(store, view, label, loc):
    group = f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}"
    loc = np.asarray(loc, dtype=np.float64).reshape(-1, 3)
    store.set_attributes(group + "/interestpoints", {"pointcloud": "1.0.0", "type": "list", "list version": "1.0.0"})
    store.write_list(group + "/interestpoints/id", np.arange(len(loc), dtype=np.uint64).reshape(-1, 1), 300000, "zstd")
    store.write_list(group + "/interestpoints/loc", loc, 300000, "zstd")


def read_rows(root, views, label="beads"):
    st = bn5.N5Store(os.path.join(str(root), "interestpoints.n5"))
    return {v: st.read_correspondences(f"tpId_{v[0]}_viewSetupId_{v[1]}/{label}") for v in views}


# ------------------------------------------------------------------------------------------ oracle known answers
def test_knn_tie_order_on_an_integer_lattice():
    g = np.stack(np.meshgrid(np.arange(4), np.arange(3), np.arange(2), indexing="ij"), -1).reshape(-1, 3).astype(float)
    idx, d2 = mo.knn(g, 6)
    fi, fd = mo.knn_full_sort(g, 6)
    assert np.array_equal(idx, fi) and np.array_equal(d2, fd)
    # point (0,0,0) = index 0: distance-1 neighbours (0,0,1)=1, (0,1,0)=2, (1,0,0)=6 in index order, then distance 2
    assert idx[0].tolist() == [1, 2, 6, 3, 7, 8] and d2[0].tolist() == [1, 1, 1, 2, 2, 2]
    dup = np.vstack([g[:5], g[:1]])                                   # distance-0 neighbours are legal
    assert mo.knn(dup, 3)[0][0].tolist() == [5, 1, 2]


def test_descriptor_distance_zero_for_a_translated_copy():
    rng = np.random.default_rng(1)
    a = rng.integers(0, 400, (40, 3)) / 8.0                            # dyadic: the translated copy is exact
    bb, best, second = mo.match(a, a + (7.25, -3.0, 11.5))
    assert np.array_equal(bb, np.arange(40)) and np.all(best == 0.0) and np.all(second > 0)


def test_hand_computed_distance_prefers_a_later_subset_pair():
    u = np.array([[1.0, 0, 0], [0, 2, 0], [0, 0, 3], [4, 4, 4]])
    v = np.array([[9.0, 9, 9], [1, 0, 0], [0, 2, 0], [0, 0, 3]])
    # s = (0, 1, 2) of u against t = (1, 2, 3) of v matches exactly; the first pair ((0,1,2), (0,1,2)) does not
    assert mo.descriptor_distance(u, v, 3) == 0.0
    first = mo.sq3(u[0] - v[0]) + mo.sq3(u[1] - v[1]) + mo.sq3(u[2] - v[2])
    assert first > 0 and mo.subsets(3, 4)[0] == (0, 1, 2) and mo.subsets(3, 4)[-1] == (1, 2, 3)


def test_ratio_test_at_the_boundary():
    kept = mo.ratio_test([0, 1, 2, -1, 4], [1.0, 1.0, 0.0, 0.0, 3.5e38], [3.0, 3.0000001, 0.0, 1.0, np.inf], 3.0)
    assert kept == [1]
    assert bm.ratio_test(np.array([0, 1, 2, -1, 4]), np.array([1.0, 1.0, 0.0, 0.0, 3.5e38]),
                         np.array([3.0, 3.0000001, 0.0, 1.0, np.inf]), 3.0).tolist() == kept


def _affine_truth():
    A = np.array([[1.02, 0.05, -0.01], [-0.03, 0.97, 0.02], [0.01, 0.04, 1.05]])
    return np.hstack([A, [[5.0], [-7.5], [2.25]]])


@pytest.mark.parametrize("kind", ["TRANSLATION", "RIGID", "AFFINE"])
def test_fits_exact_on_noiseless_points(kind):
    rng = np.random.default_rng(2)
    a = rng.uniform(-40, 40, (9, 3))
    M = {"TRANSLATION": np.hstack([np.eye(3), [[3.0], [-1.0], [0.5]]]), "RIGID": rot_z(17.0, (4, 5, 6)),
         "AFFINE": _affine_truth()}[kind]
    b = a @ M[:, :3].T + M[:, 3]
    assert np.abs(mo.fit(kind, a, b) - M).max() < 1e-12
    got, ok = bm.Model(kind, "NONE").fit(a[None], b[None])
    assert ok[0] and np.abs(got[0] - M).max() < 1e-12


def test_interpolated_model_is_the_blend():
    rng = np.random.default_rng(3)
    a = rng.uniform(-40, 40, (12, 3))
    b = a @ _affine_truth()[:, :3].T + _affine_truth()[:, 3] + rng.normal(0, 0.5, (12, 3))
    want = 0.9 * mo.fit("AFFINE", a, b) + 0.1 * mo.fit("RIGID", a, b)
    assert np.abs(mo.fit_model("AFFINE", "RIGID", 0.1, a, b) - want).max() < 1e-12
    got, ok = bm.Model("AFFINE", "RIGID", 0.1).fit(a[None], b[None])
    assert ok[0] and np.abs(got[0] - want).max() < 1e-10 and bm.Model().min_matches == 4


def _planted_candidates(seed=4, n=60, outliers=0.4):
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 200, (n, 3))
    b = a @ _affine_truth()[:, :3].T + _affine_truth()[:, 3] + rng.normal(0, 0.2, (n, 3))
    bad = rng.permutation(n)[:int(outliers * n)]
    b[bad] += rng.uniform(20, 60, (len(bad), 3)) * rng.choice([-1, 1], (len(bad), 3))
    return a, b, sorted(set(range(n)) - set(bad.tolist()))


def test_ransac_returns_the_planted_inliers_deterministically():
    a, b, good = _planted_candidates()
    inl, M = mo.ransac(a, b, iterations=300)
    assert inl == good and mo.ransac(a, b, iterations=300)[0] == inl
    got, gM = bm.ransac(a, b, bm.Model(), iterations=300)
    assert got.tolist() == good and np.abs(gM - M).max() < 1e-9
    # the chunk size does not change the sample stream
    assert bm.ransac(a, b, bm.Model(), iterations=300, chunk=7)[0].tolist() == good


def test_ransac_rejects_by_count_and_ratio():
    a, b, good = _planted_candidates()
    assert mo.ransac(a, b, iterations=200, min_num_inliers=len(good) + 1) == ([], None)
    assert bm.ransac(a, b, bm.Model(), iterations=200, min_num_inliers=len(good) + 1)[1] is None
    assert mo.ransac(a, b, iterations=200, min_inlier_ratio=0.7) == ([], None)
    assert bm.ransac(a, b, bm.Model(), iterations=200, min_inlier_ratio=0.7)[1] is None


# ------------------------------------------------------------------------------------------ host logic
def test_pairs_and_tasks():
    dims = {(0, s): (100, 100, 10) for s in range(3)}
    dims[(1, 0)] = (100, 100, 10)
    T = lambda x: np.hstack([np.eye(3), [[x], [0.0], [0.0]]])   # noqa: E731
    regs = {(0, 0): T(0), (0, 1): T(99), (0, 2): T(200), (1, 0): T(0)}
    assert commands.match_pairs(dims, regs, list(regs)) == [((0, 0), (0, 1))]          # closed boxes touch at x = 99
    assert commands.match_pairs(dims, regs, list(regs), "ALL_AGAINST_ALL") == [
        ((0, 0), (0, 1)), ((0, 0), (0, 2)), ((0, 1), (0, 2))]
    p = [((0, 0), (0, 1))]
    assert commands.match_tasks(p, ["a", "b"]) == [((0, 0), "a", (0, 1), "a"), ((0, 0), "b", (0, 1), "b")]
    assert commands.match_tasks(p, ["a", "b"], True) == [((0, 0), la, (0, 1), lb) for la in "ab" for lb in "ab"]


def test_overlap_filter_keeps_points_in_the_partner_box():
    reg = np.hstack([np.eye(3), [[10.0], [0.0], [0.0]]])
    w = np.array([[9.9, 5, 5], [10.0, 0, 0], [29.0, 19, 9], [29.01, 5, 5], [15, -0.1, 5]])
    assert commands.overlap_filter(w, (20, 20, 10), reg).tolist() == [False, True, True, False, False]


def test_correspondence_writer_round_trip_append_and_clear(tmp_path):
    store = bn5.N5Store(str(tmp_path / "interestpoints.n5"), create=True)
    rows = [(0, (0, 2), "nuclei", 4), (3, (0, 1), "beads", 7)]
    store.write_correspondences("tpId_0_viewSetupId_0/beads", rows)
    a = store.get_attributes("tpId_0_viewSetupId_0/beads/correspondences")
    assert a["idMap"] == {"0,1,beads": 0, "0,2,nuclei": 1}
    assert store.read_correspondences("tpId_0_viewSetupId_0/beads") == rows
    store.write_correspondences("tpId_0_viewSetupId_1/beads", [])
    assert store.dataset_attributes("tpId_0_viewSetupId_1/beads/correspondences/data")["dimensions"] == [0]
    for v in ((0, 0), (0, 1), (0, 2)):
        write_points(store, v, "beads", np.arange(30.0).reshape(10, 3) + 100 * v[1])
    ips = commands._MatchPoints(store, [(0, 0), (0, 1), (0, 2)], ["beads"], {v: np.hstack([np.eye(3), np.zeros((3, 1))])
                                                                           for v in ((0, 0), (0, 1), (0, 2))})
    task = ((0, 0), "beads", (0, 1), "beads")
    commands.write_match_correspondences(store, ips, [(0, 0), (0, 1), (0, 2)], ["beads"],
                                         {task: np.array([[3, 7], [1, 2]])})
    got = read_rows(tmp_path, [(0, 0), (0, 1), (0, 2)])
    # appended without the duplicate (3, (0,1), beads, 7), sorted by (id, partner tp, setup, label, id)
    assert got[(0, 0)] == [(0, (0, 2), "nuclei", 4), (1, (0, 1), "beads", 2), (3, (0, 1), "beads", 7)]
    assert got[(0, 1)] == [(2, (0, 0), "beads", 1), (7, (0, 0), "beads", 3)] and got[(0, 2)] == []
    ips = commands._MatchPoints(store, [(0, 0), (0, 1), (0, 2)], ["beads"], ips_regs := {
        v: np.hstack([np.eye(3), np.zeros((3, 1))]) for v in ((0, 0), (0, 1), (0, 2))})
    commands.write_match_correspondences(store, ips, [(0, 0), (0, 1), (0, 2)], ["beads"], {task: np.array([[5, 5]])},
                                         clear=True)
    got = read_rows(tmp_path, [(0, 0), (0, 1)])
    assert got[(0, 0)] == [(5, (0, 1), "beads", 5)] and got[(0, 1)] == [(5, (0, 0), "beads", 5)]
    # the non-rigid fusion reads the written rows: targets average the direct partners
    t, _ = commands._InterestPoints(store, [(0, 0), (0, 1)], ["beads"], ips_regs).targets((0, 0), [(0, 0), (0, 1)])
    assert np.allclose(t, [[(15.0 + 115.0) / 2, (16.0 + 116.0) / 2, (17.0 + 117.0) / 2]])


@pytest.mark.parametrize("kw, text", [
    (dict(method="FAST_ROTATION"), "FAST_ROTATION"), (dict(method="FAST_TRANSLATION"), "FAST_TRANSLATION"),
    (dict(method="ICP"), "ICP"), (dict(group_tiles=True), "--groupTiles"), (dict(group_illums=True), "--groupIllums"),
    (dict(group_channels=True), "--groupChannels"), (dict(split_timepoints=True), "--splitTimepoints"),
    (dict(registration_tp="TIMEPOINTS_ALL_TO_ALL"), "-rtp"), (dict(ransac_multi_consensus=True), "-rmc"),
])
def test_unbuilt_flags_raise(kw, text):
    args = dict(xml_path="missing.xml", ctx=None, labels=["beads"], method="PRECISE_TRANSLATION")
    args.update(kw)
    with pytest.raises(NotImplementedError, match=text):
        commands.match_interestpoints(**args)


# ------------------------------------------------------------------------------------------ command end to end
RUN = dict(method="PRECISE_TRANSLATION", interestpoints_for_reg="OVERLAPPING_ONLY", ransac_iterations=2000)


def check_scene(root, truth, results, min_recall=0.6):
    """Every written correspondence is a true pair, and at least min_recall of the true overlap pairs are found."""
    views = sorted(truth)
    rows = read_rows(root, views)
    for v in views:
        for pid, pv, _, qid in rows[v]:
            assert truth[v][pid] >= 0 and truth[v][pid] == truth[pv][qid], (v, pid, pv, qid)
    for (va, _, vb, _), pairs in results.items():
        common = set(truth[va][truth[va] >= 0].tolist()) & set(truth[vb][truth[vb] >= 0].tolist())
        if len(common) < 50:
            continue
        assert len(pairs) >= min_recall * len(common), (va, vb, len(pairs), len(common))
    return rows


def test_command_on_a_planted_scene(tmp_path):
    xml, truth = planted_scene(tmp_path)
    res = commands.match_interestpoints(xml, MatchFakeContext(), ["beads"], **RUN)
    assert list(res) == [((0, 0), "beads", (0, 1), "beads")]
    rows = check_scene(tmp_path, truth, res)
    assert len(rows[(0, 0)]) == len(res[((0, 0), "beads", (0, 1), "beads")]) > 50


def test_dry_run_writes_nothing(tmp_path):
    xml, _ = planted_scene(tmp_path, tile=(120, 100, 40))
    res = commands.match_interestpoints(xml, MatchFakeContext(), ["beads"], dry_run=True, **RUN)
    assert len(res) == 1
    assert not os.path.exists(tmp_path / "interestpoints.n5" / "tpId_0_viewSetupId_0" / "beads" / "correspondences")


def _shard_worker(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)

    def allgather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out
    commands.match_interestpoints(os.path.join(root, "dataset.xml"), MatchFakeContext(), ["beads"],
                                  shard=(rank, world), allgather=allgather, **RUN)
    dist.barrier()
    if rank == 0:
        q.put("done")
    dist.barrier()
    dist.destroy_process_group()


def test_world2_shard_writes_the_same_rows(tmp_path):
    import torch.multiprocessing as mp
    one, two = tmp_path / "one", tmp_path / "two"
    for d in (one, two):
        d.mkdir()
        planted_scene(d, grid=(3, 1), tile=(120, 100, 40))
    _, truth = planted_scene(tmp_path / "one", grid=(3, 1), tile=(120, 100, 40))
    commands.match_interestpoints(str(one / "dataset.xml"), MatchFakeContext(), ["beads"], **RUN)
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
    views = sorted(truth)
    assert read_rows(one, views) == read_rows(two, views) and sum(len(r) for r in read_rows(one, views).values()) > 0
