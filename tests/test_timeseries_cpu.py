"""Registration across timepoints without a GPU: the -rtp pair constellations of match-interestpoints, the automatic
fixed views of the solver, and both commands end to end on a planted time-lapse through oracle-backed contexts."""
import os
import socket
import xml.etree.ElementTree as ET

import numpy as np
import pytest
from scipy.spatial import cKDTree

from bsgpu import commands, n5 as bn5, solver as bsv, spimdata
from tests.test_match_cpu import SPURIOUS_CLEARANCE, MatchFakeContext, compose, read_rows, rot_z, write_points
from tests.test_solver_cpu import SolverFakeContext

RUN = dict(method="PRECISE_TRANSLATION", interestpoints_for_reg="OVERLAPPING_ONLY", ransac_iterations=2000)


# ------------------------------------------------------------------------------------------ planted time-lapse
def apply(M, x):
    return np.asarray(x, dtype=np.float64) @ M[:, :3].T + M[:, 3]


def timeseries_scene(root, timepoints=3, tile=(200, 160, 60), overlap=0.3, spacing=14.0, keep=0.6, jitter=0.3,
                     spurious=0.1, drift_px=3.0, rot_deg=0.8, seed=5, label="beads"):
    """One bead cloud seen by two tiles side by side in x at every timepoint.  At timepoint t the cloud is moved by a
    rigid drift D_t (up to ``drift_px`` per axis and ``rot_deg`` about z through the cloud's centre); the XML holds the
    same exact grid translations at every timepoint, so the drift is what registration across time has to find.  Beads
    are a kept subset of a jittered lattice (never within RANSAC's max_error of each other); every view stores the
    beads inside it (+ ``jitter``) and ``spurious`` * n extra points kept clear of every bead.
    Returns (xml, truth, drift): truth[view] maps point id -> bead index (-1 spurious), drift[t] is D_t (3 x 4), and
    drift["beads"] the undrifted bead positions."""
    rng = np.random.default_rng(seed)
    step = int(round(tile[0] * (1 - overlap)))
    extent = np.array([step + tile[0], tile[1], tile[2]], dtype=np.float64)
    axes = [np.arange(spacing / 2, extent[d] - spacing / 2, spacing) for d in range(3)]
    sites = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    sites = sites[rng.random(len(sites)) < keep]
    beads = sites + rng.uniform(-spacing / 4, spacing / 4, sites.shape)
    drift, truth = {"beads": beads}, {}
    store = bn5.N5Store(os.path.join(str(root), "interestpoints.n5"), create=True)
    for t in range(timepoints):
        shift = np.hstack([np.eye(3), rng.uniform(-drift_px, drift_px, (3, 1))])
        drift[t] = compose(shift, rot_z(rng.uniform(-rot_deg, rot_deg), extent / 2))
        moved = apply(drift[t], beads)
        for s in range(2):
            loc = moved - (s * step, 0.0, 0.0)
            inside = np.nonzero(np.all((loc >= 0) & (loc <= np.array(tile) - 1), axis=1))[0]
            pts = loc[inside] + rng.normal(0.0, jitter, (len(inside), 3))
            ns = int(round(spurious * len(inside)))
            tree, extra = cKDTree(loc[inside]), np.zeros((0, 3))
            while len(extra) < ns:
                c = rng.uniform(0, 1, (2 * ns, 3)) * (np.array(tile) - 1)
                extra = np.vstack([extra, c[tree.query(c)[0] > SPURIOUS_CLEARANCE]])[:ns]
            order = rng.permutation(len(inside) + ns)
            write_points(store, (t, s), label, np.vstack([pts, extra])[order])
            truth[(t, s)] = np.concatenate([inside, -np.ones(ns, dtype=np.int64)])[order]
    xml = os.path.join(str(root), "dataset.xml")
    spimdata.write_dataset_xml(xml, "dataset.n5", [dict(setup=s, size_xyz=tile, tile=s,
                                                        translation_xyz=(s * step, 0, 0)) for s in range(2)])
    repeat_timepoint(xml, timepoints)
    return xml, truth, drift


def repeat_timepoint(xml, timepoints):
    """Give the one-timepoint project ``xml`` timepoints 0 .. n-1, every one with timepoint 0's registrations."""
    tree = ET.parse(xml)
    vrs = tree.getroot().find("ViewRegistrations")
    first = list(vrs)
    for t in range(1, timepoints):
        for vr in first:
            copy = ET.fromstring(ET.tostring(vr))
            copy.set("timepoint", str(t))
            vrs.append(copy)
    tree.getroot().find("SequenceDescription").find("Timepoints").find("integerpattern").text = f"0-{timepoints - 1}"
    tree.write(xml, encoding="UTF-8", xml_declaration=True)


def check_rows(root, truth, results, min_recall=0.6):
    """Every written row, same-time or cross-time, links one planted bead; every task whose views share at least 50
    beads finds at least ``min_recall`` of them.  Returns the rows and the number of cross-time tasks checked."""
    views = sorted(truth)
    rows = read_rows(root, views)
    for v in views:
        for pid, pv, _, qid in rows[v]:
            assert truth[v][pid] >= 0 and truth[v][pid] == truth[pv][qid], (v, pid, pv, qid)
    cross = 0
    for (va, _, vb, _), pairs in results.items():
        common = set(truth[va][truth[va] >= 0].tolist()) & set(truth[vb][truth[vb] >= 0].tolist())
        if len(common) < 50:
            continue
        assert len(pairs) >= min_recall * len(common), (va, vb, len(pairs), len(common))
        cross += va[0] != vb[0]
    return rows, cross


# ------------------------------------------------------------------------------------------ pair constellations
V6 = [(t, s) for t in range(3) for s in range(2)]


def _hand_setup():
    """3 timepoints x 2 setups whose boxes all overlap (setup 1 sits 50 px right of setup 0)."""
    T = lambda x: np.hstack([np.eye(3), [[x], [0.0], [0.0]]])   # noqa: E731
    dims = {v: (100, 100, 10) for v in V6}
    regs = {v: T(50.0 * v[1]) for v in V6}
    return dims, regs


def P(a, b):
    return ((a // 10, a % 10), (b // 10, b % 10))


def test_pair_constellations_by_hand():
    dims, regs = _hand_setup()
    pairs = lambda *a, **k: commands.match_pairs(dims, regs, V6[::-1], *a, **k)   # noqa: E731
    individually = [P(0, 1), P(10, 11), P(20, 21)]
    assert pairs() == individually == commands.match_pairs(dims, regs, V6, "OVERLAPPING_ONLY")
    assert pairs("OVERLAPPING_ONLY", "timepoints_individually") == individually
    assert pairs(registration_tp="ALL_TO_ALL") == [
        P(0, 1), P(0, 10), P(0, 11), P(0, 20), P(0, 21),
        P(1, 10), P(1, 11), P(1, 20), P(1, 21),
        P(10, 11), P(10, 20), P(10, 21),
        P(11, 20), P(11, 21),
        P(20, 21)]
    assert pairs(registration_tp="ALL_TO_ALL_WITH_RANGE", range_tp=0) == individually
    assert pairs(registration_tp="All_To_All_With_Range", range_tp=1) == [
        P(0, 1), P(0, 10), P(0, 11),
        P(1, 10), P(1, 11),
        P(10, 11), P(10, 20), P(10, 21),
        P(11, 20), P(11, 21),
        P(20, 21)]
    assert pairs(registration_tp="ALL_TO_ALL_WITH_RANGE") == pairs(registration_tp="ALL_TO_ALL")   # default range 5
    assert pairs(registration_tp="TO_REFERENCE_TIMEPOINT", reference_tp=1) == [
        P(0, 10), P(0, 11),
        P(1, 10), P(1, 11),
        P(10, 11), P(10, 20), P(10, 21),
        P(11, 20), P(11, 21)]
    # the default reference is the timepoint of the first view
    assert pairs(registration_tp="TO_REFERENCE_TIMEPOINT") == [
        P(0, 1), P(0, 10), P(0, 11), P(0, 20), P(0, 21),
        P(1, 10), P(1, 11), P(1, 20), P(1, 21)]


def test_constellations_then_overlap_under_each_views_registration():
    dims, regs = _hand_setup()
    regs = {v: np.hstack([np.eye(3), [[200.0 * v[1]], [0.0], [0.0]]]) for v in V6}   # setups 0 and 1 apart
    regs[(2, 1)] = np.hstack([np.eye(3), [[60.0], [0.0], [0.0]]])                   # tp 2 setup 1 moved onto setup 0
    assert commands.match_pairs(dims, regs, V6) == [P(20, 21)]
    assert commands.match_pairs(dims, regs, V6, "OVERLAPPING_ONLY", "ALL_TO_ALL") == [
        P(0, 10), P(0, 20), P(0, 21), P(1, 11), P(10, 20), P(10, 21), P(20, 21)]
    assert commands.match_pairs(dims, regs, V6, "ALL_AGAINST_ALL", "ALL_TO_ALL_WITH_RANGE", range_tp=1) == [
        P(0, 1), P(0, 10), P(0, 11), P(1, 10), P(1, 11), P(10, 11), P(10, 20), P(10, 21), P(11, 20), P(11, 21),
        P(20, 21)]


def test_constellation_errors():
    dims, regs = _hand_setup()
    with pytest.raises(ValueError, match="Specified reference timepoint is not part of the ViewIds"):
        commands.match_pairs(dims, regs, V6, registration_tp="TO_REFERENCE_TIMEPOINT", reference_tp=3)
    with pytest.raises(ValueError, match="rangeTP"):
        commands.match_pairs(dims, regs, V6, registration_tp="ALL_TO_ALL_WITH_RANGE", range_tp=-1)
    with pytest.raises(NotImplementedError, match="-rtp"):
        commands.match_pairs(dims, regs, V6, registration_tp="REFERENCE")
    assert commands.reference_timepoint([(4, 1), (2, 3), (2, 0)]) == 2
    assert commands.reference_timepoint([(4, 1), (2, 3)], 4) == 4


@pytest.mark.parametrize("name", ["TIMEPOINTS_TO_REFERENCE", "ALL_TO_ALL_RANGE", "REFERENCE_TIMEPOINT"])
def test_unknown_names_raise_before_the_xml_is_read(name):
    with pytest.raises(NotImplementedError, match="-rtp"):
        commands.match_interestpoints("missing.xml", None, ["beads"], "PRECISE_TRANSLATION", registration_tp=name)
    with pytest.raises(NotImplementedError, match="-rtp"):
        commands.solver("missing.xml", None, "IP", labels=["beads"], registration_tp=name)


def test_command_argument_errors_and_the_default_reference(tmp_path):
    xml, truth, _ = timeseries_scene(tmp_path, tile=(120, 100, 40))
    ctx = MatchFakeContext()
    with pytest.raises(ValueError, match="Specified reference timepoint is not part of the ViewIds"):
        commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="TO_REFERENCE_TIMEPOINT", reference_tp=7,
                                      **RUN)
    with pytest.raises(ValueError, match="Specified reference timepoint is not part of the ViewIds"):
        commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="TO_REFERENCE_TIMEPOINT", reference_tp=0,
                                      view_selection=dict(timepoint_ids="1,2"), **RUN)
    with pytest.raises(ValueError, match="rangeTP"):
        commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="ALL_TO_ALL_WITH_RANGE", range_tp=-2, **RUN)
    with pytest.raises(ValueError, match="Specified reference timepoint is not part of the ViewIds"):
        commands.solver(xml, SolverFakeContext(), "IP", labels=["beads"], registration_tp="TO_REFERENCE_TIMEPOINT",
                        reference_tp=5)
    # with --timepointId 1,2 the default reference is timepoint 1: no pair of two views at timepoint 2
    res = commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="to_reference_timepoint", dry_run=True,
                                        view_selection=dict(timepoint_ids="1,2"), **RUN)
    assert [(a, b) for a, _, b, _ in res] == [P(10, 11), P(10, 20), P(10, 21), P(11, 20), P(11, 21)]


# ------------------------------------------------------------------------------------------ fixed views
def test_fixed_views_auto_per_mode():
    views = [(2, 0), (0, 5), (1, 3), (0, 2), (1, 1)]
    assert bsv.fixed_views_auto(views) == {(0, 2), (1, 1), (2, 0)}
    assert bsv.fixed_views_auto(views, "TIMEPOINTS_INDIVIDUALLY") == {(0, 2), (1, 1), (2, 0)}
    assert bsv.fixed_views_auto(views, "TO_REFERENCE_TIMEPOINT", 1) == {(1, 1)}
    assert bsv.fixed_views_auto(views, "to_reference_timepoint", 2) == {(2, 0)}
    assert bsv.fixed_views_auto(views, "TO_REFERENCE_TIMEPOINT", 4) == set()
    assert bsv.fixed_views_auto(views, "ALL_TO_ALL") == {(0, 2)}
    assert bsv.fixed_views_auto(views, "ALL_TO_ALL_WITH_RANGE") == {(0, 2)}


# ------------------------------------------------------------------------------------------ commands end to end
@pytest.mark.parametrize("rtp, ref, want", [
    ("ALL_TO_ALL", None, [P(a, b) for i, a in enumerate((0, 1, 10, 11, 20, 21)) for b in (0, 1, 10, 11, 20, 21)[i + 1:]]),
    ("TO_REFERENCE_TIMEPOINT", 1, [P(0, 10), P(0, 11), P(1, 10), P(1, 11), P(10, 11), P(10, 20), P(10, 21), P(11, 20),
                                   P(11, 21)]),
])
def test_command_across_timepoints(tmp_path, rtp, ref, want):
    xml, truth, _ = timeseries_scene(tmp_path)
    res = commands.match_interestpoints(xml, MatchFakeContext(), ["beads"], registration_tp=rtp, reference_tp=ref, **RUN)
    assert [(a, b) for a, _, b, _ in res] == want
    rows, cross = check_rows(tmp_path, truth, res)
    assert cross == sum(a[0] != b[0] for a, b in want)
    # cross-time rows are written on both sides and read back through the solver's and non-rigid fusion's reader
    assert any(pv[0] != 0 for _, pv, _, _ in rows[(0, 0)])
    regs = {v: spimdata.SpimData2.load(xml).model(*v) for v in truth}
    ips = commands._InterestPoints(bn5.N5Store(str(tmp_path / "interestpoints.n5")), sorted(truth), ["beads"], regs)
    for (va, _, vb, _), pairs in res.items():
        got = {(pid, qid) for pid, pv, _, qid in ips.corr[(va, "beads")] if pv == vb}
        assert got == {tuple(p) for p in pairs.tolist()}, (va, vb)


def test_dry_run_across_timepoints_writes_nothing(tmp_path):
    xml, _, _ = timeseries_scene(tmp_path, tile=(120, 100, 40))
    res = commands.match_interestpoints(xml, MatchFakeContext(), ["beads"], registration_tp="ALL_TO_ALL", dry_run=True,
                                        **RUN)
    assert len(res) == 15 and any(len(p) for (a, _, b, _), p in res.items() if a[0] != b[0])
    for t in range(3):
        assert not os.path.exists(tmp_path / "interestpoints.n5" / f"tpId_{t}_viewSetupId_0" / "beads" / "correspondences")


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
                                  registration_tp="ALL_TO_ALL", shard=(rank, world), allgather=allgather, **RUN)
    dist.barrier()
    if rank == 0:
        q.put("done")
    dist.barrier()
    dist.destroy_process_group()


def test_world2_shard_across_timepoints_writes_the_same_rows(tmp_path):
    import torch.multiprocessing as mp
    one, two = tmp_path / "one", tmp_path / "two"
    for d in (one, two):
        d.mkdir()
        _, truth, _ = timeseries_scene(d, tile=(120, 100, 40))
    commands.match_interestpoints(str(one / "dataset.xml"), MatchFakeContext(), ["beads"], registration_tp="ALL_TO_ALL",
                                  **RUN)
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
    rows = read_rows(one, views)
    assert rows == read_rows(two, views) and any(pv[0] != v[0] for v in views for _, pv, _, _ in rows[v])


def check_drift(models, drift, truth, reference_tp, tol=0.5):
    """The reference timepoint's views keep the identity; every other view's model maps the beads it sees (their drifted
    world positions) onto the reference timepoint's positions of the same beads within ``tol`` px."""
    want = apply(drift[reference_tp], drift["beads"])
    for v, M in models.items():
        if v[0] == reference_tp:
            assert np.allclose(M, np.eye(3, 4), atol=1e-9), v
            continue
        b = truth[v][truth[v] >= 0]
        err = np.linalg.norm(apply(M, apply(drift[v[0]], drift["beads"][b])) - want[b], axis=1)
        assert err.max() < tol, (v, err.max())


def match_and_solve(root, ctx, solver_ctx, tm="RIGID"):
    """TO_REFERENCE_TIMEPOINT matching with the reference in the middle, then the -s IP solve of every timepoint as
    one tile."""
    xml = os.path.join(str(root), "dataset.xml")
    commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="TO_REFERENCE_TIMEPOINT", reference_tp=1, **RUN)
    return commands.solver(xml, solver_ctx, "IP", labels=["beads"], transformation_model=tm, regularization_model="NONE",
                           max_plateau_width=20, split_timepoints=True, registration_tp="TO_REFERENCE_TIMEPOINT",
                           reference_tp=1)


def test_solver_corrects_the_drift_to_the_reference_timepoint(tmp_path):
    xml, truth, drift = timeseries_scene(tmp_path)
    res = match_and_solve(tmp_path, MatchFakeContext(), SolverFakeContext())
    assert set(res["models"]) == set(truth) and res["stats"]["unconnected_views"] == []
    for t in range(3):                                  # one tile per timepoint
        assert np.array_equal(res["models"][(t, 0)], res["models"][(t, 1)])
    check_drift(res["models"], drift, truth, 1)
    data = spimdata.SpimData2.load(xml)
    assert data.registrations[(0, 1)][0][0] == "RigidModel3D"
    assert np.allclose(data.model(0, 1), compose(res["models"][(0, 1)], np.hstack([np.eye(3), [[140.0], [0], [0]]])))
