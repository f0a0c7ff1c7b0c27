"""solver host logic without a GPU: weighted fits, match creation from stitching results and correspondences, grouping,
fixed views, colouring, the stopping rule, link removal, the XML write and the command end to end through an
oracle-backed context."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import solver_oracle as so
from tests.fake_ctx import FakeContext


class SolverFakeContext(FakeContext):
    """FakeContext whose relaxation is the float64 oracle."""

    def __init__(self):
        super().__init__()
        self.solves = 0

    def solve_tiles(self, *args, **kw):
        self.solves += 1
        return so.solve_tiles(*args, **kw)


def _rot(axis, ang):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _T(t):
    M = np.eye(3, 4)
    M[:, 3] = t
    return M


def _apply(M, x):
    return x @ M[:, :3].T + M[:, 3]


# ------------------------------------------------------------------------------------------ fits (closed forms)
def test_weighted_fits_known_answers():
    from bsgpu import matching as bm
    rng = np.random.default_rng(1)
    x = rng.uniform(-50, 50, (40, 3)) + 1e4
    w = rng.uniform(0.1, 2.0, 40)
    # translation: the weighted mean difference
    y = x + rng.normal(0, 1.0, x.shape) + (3.0, -2.0, 1.0)
    M, ok = bm._fit("TRANSLATION", x[None], y[None], w[None])
    assert ok[0] and np.allclose(M[0][:, 3], (w[:, None] * (y - x)).sum(0) / w.sum(), atol=1e-9)
    # rigid and affine recover planted models exactly
    R = np.eye(3, 4)
    R[:, :3] = _rot((1, 2, 3), 0.2)
    R[:, 3] = (5, -7, 11)
    A = R.copy()
    A[:, :3] = A[:, :3] @ np.diag([1.05, 0.97, 1.01]) + 0.01
    for kind, G in (("RIGID", R), ("AFFINE", A)):
        F, ok = bm._fit(kind, x[None], _apply(G, x)[None], w[None])
        assert ok[0] and np.allclose(F[0], G, atol=1e-8), kind
        Fo, oko = so.fit(kind, x, _apply(G, x), w)
        assert oko and np.allclose(Fo, G, atol=1e-8)
    # the weighted fits equal the per-match oracle on noisy data, interpolated too
    y = _apply(A, x) + rng.normal(0, 0.5, x.shape)
    for tm in ("TRANSLATION", "RIGID", "AFFINE"):
        for rm in ("NONE", "IDENTITY", "TRANSLATION", "RIGID", "AFFINE"):
            F, ok = bm.Model(tm, rm, 0.1).fit(x[None], y[None], w[None])
            Fo = so.fit_model(tm, rm, 0.1, x, y, w)
            assert ok[0] and Fo is not None and np.allclose(F[0], Fo, rtol=1e-9, atol=1e-7), (tm, rm)
    # weights 1 give the unweighted fit; weights=None is the unchanged path
    for kind in ("TRANSLATION", "RIGID", "AFFINE"):
        F1, _ = bm._fit(kind, x[None], y[None], np.ones((1, 40)))
        F0, _ = bm._fit(kind, x[None], y[None])
        assert np.allclose(F1, F0, atol=1e-8)
    # singular: collinear points for RIGID / AFFINE, zero weight for everything
    line = np.outer(np.arange(10.0), (1.0, 2.0, 3.0))
    for kind in ("RIGID", "AFFINE"):
        assert not bm._fit(kind, line[None], line[None] + 1, np.ones((1, 10)))[1][0]
        assert so.fit(kind, line, line + 1, np.ones(10))[1] is False
    assert not bm._fit("TRANSLATION", x[None], y[None], np.zeros((1, 40)))[1][0]


def _chain_problem(truth, n_corner=8, seed=0):
    """Tiles in a chain: matches between tile i and i + 1 at random points, exact under the planted models."""
    from bsgpu import solver as bsv
    rng = np.random.default_rng(seed)
    ta, tb, p, q, w = [], [], [], [], []
    for i in range(len(truth) - 1):
        c = rng.uniform(0, 100, (n_corner, 3)) + 100.0 * i
        # world truth point c; tile i sees it at truth_i^-1(c), tile i+1 at truth_{i+1}^-1(c)
        for t, lst in ((i, p), (i + 1, q)):
            Mi = np.linalg.inv(np.vstack([truth[t], [0, 0, 0, 1]]))[:3]
            lst.append(_apply(Mi, c))
        ta.append(np.full(n_corner, i))
        tb.append(np.full(n_corner, i + 1))
        w.append(np.full(n_corner, 1.0))
    return bsv.build_problem(len(truth), np.concatenate(ta), np.concatenate(tb), np.concatenate(p), np.concatenate(q),
                             np.concatenate(w))


@pytest.mark.parametrize("tm", ["TRANSLATION", "RIGID", "AFFINE"])
def test_two_and_three_tiles_recover_planted_models(tm):
    from bsgpu import matching as bm
    from bsgpu import solver as bsv
    for n in (2, 3):
        truth = [np.eye(3, 4)]
        for i in range(1, n):
            G = _T((3.0 * i, -2.0, 1.0 + i))
            if tm != "TRANSLATION":
                G[:, :3] = _rot((0, 0, 1), 0.05 * i)
            if tm == "AFFINE":
                G[:, :3] = G[:, :3] @ np.diag([1.02, 1.0, 0.99])
            truth.append(G)
        prob = _chain_problem(truth)
        prob.fixed = np.array([1] + [0] * (n - 1), np.int32)
        M, removed, st = bsv.solve(SolverFakeContext(), prob, bm.Model(tm, "NONE"), max_plateau_width=20)
        assert not removed and st["iterations"] >= 21
        for t in range(n):
            assert np.allclose(M[t], truth[t], atol=1e-6), (tm, n, t)


# ------------------------------------------------------------------------------------------ matches, grouping
def _xml(tmp_path, tiles):
    from bsgpu import spimdata
    return spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)


def _row_of_three(tmp_path, channels=1):
    tiles = []
    for t in range(3):
        for c in range(channels):
            tiles.append(dict(setup=t * channels + c, size_xyz=(100, 80, 60), tile=t, channel=c,
                              translation_xyz=(80.0 * t, 0, 0)))
    return _xml(tmp_path, tiles)


def _store_result(data, a, b, R, r, bmin, bmax):
    from bsgpu.spimdata import SpimData2
    ga, gb = data._as_group(a), data._as_group(b)
    h = SpimData2.transform_hash(data.registrations[ga[0]], data.registrations[gb[0]])
    data.set_stitching_results([dict(pair=(a, b), shift=R, r=r, hash=h, bbox_min=bmin, bbox_max=bmax)])


def test_stitching_matches_corners_weights_inverse_and_stale_hash(tmp_path):
    from bsgpu import solver as bsv
    from bsgpu.spimdata import SpimData2
    xml = _row_of_three(tmp_path)
    data = SpimData2.load(xml)
    R = _T((3.0, -2.0, 1.0))
    R[:, :3] = _rot((0, 0, 1), 0.01)
    _store_result(data, (0, 0), (0, 1), R, 0.9, (80, 0, 0), (99, 79, 59))
    _store_result(data, (0, 1), (0, 2), _T((1, 1, 0)), 0.7, (160, 0, 0), (179, 79, 59))
    data.save()
    data = SpimData2.load(xml)
    views = data.view_ids()
    tile_of = {v: i for i, v in enumerate(views)}
    ta, tb, p, q, w, stale = bsv.stitching_matches(data, tile_of, views)
    assert stale == 0 and len(ta) == 16 and ta[:8].tolist() == [0] * 8 and tb[:8].tolist() == [1] * 8
    corners = {(x, y, z) for x in (80, 99) for y in (0, 79) for z in (0, 59)}
    assert {tuple(c) for c in p[:8]} == corners
    assert np.allclose(_apply(R, q[:8]), p[:8]) and np.all(w[:8] == 0.9) and np.all(w[8:] == 0.7)
    # a changed registration of a first view makes its results stale
    data.registrations[(0, 1)][0] = ("moved", _T((81.0, 0, 0)))
    ta, tb, p, q, w, stale = bsv.stitching_matches(data, tile_of, views)
    assert stale == 2 and len(ta) == 0


def test_grouping_keys(tmp_path):
    from bsgpu import solver as bsv
    from bsgpu.spimdata import SpimData2
    data = SpimData2.load(_row_of_three(tmp_path, channels=2))
    views = data.view_ids()
    k = bsv.tile_keys(data, views)
    assert len(set(k.values())) == 6
    k = bsv.tile_keys(data, views, group_channels=True)
    assert len(set(k.values())) == 3 and k[(0, 0)] == k[(0, 1)] != k[(0, 2)]
    k = bsv.tile_keys(data, views, group_tiles=True)
    assert len(set(k.values())) == 2 and k[(0, 0)] == k[(0, 2)] == k[(0, 4)]
    k = bsv.tile_keys(data, views, split_timepoints=True)
    assert len(set(k.values())) == 1


def test_colouring_is_valid_and_greedy():
    from bsgpu import solver as bsv
    rng = np.random.default_rng(3)
    for n in (1, 2, 7, 40):
        links = np.array(sorted({tuple(sorted(rng.choice(n, 2, replace=False))) for _ in range(3 * n)} if n > 1 else []),
                         dtype=np.int64).reshape(-1, 2)
        col, off, order = bsv.colouring(n, links)
        assert all(col[a] != col[b] for a, b in links)
        assert sorted(order.tolist()) == list(range(n)) and off[0] == 0 and off[-1] == n
        for c in range(len(off) - 1):
            ts = order[off[c]:off[c + 1]]
            assert np.all(col[ts] == c) and np.all(np.diff(ts) > 0)
        for t in range(n):                        # greedy: every smaller colour is taken by a lower neighbour
            lower = {int(col[u]) for a, b in links for u in (a, b) if t in (a, b) and u != t and u < t}
            assert all(c in lower for c in range(col[t]))


def test_stopping_rule_on_a_synthetic_sequence():
    from bsgpu import solver as bsv
    width = 8
    E = [10.0 / (i + 1) for i in range(8)]
    assert all(bsv.proceed(E[:i + 1], 5.0, width) for i in range(8))   # never stops within the plateau width
    seq = E + [1.0] * 20
    stop = next(i + 1 for i in range(len(seq)) if not bsv.proceed(seq[:i + 1], 5.0, width))
    # E_i = 1 from i = 9; |E_i - E_{i-d}| / d must be <= 1e-4 for d = 8, 4, 2, 1: i - 8 >= 9
    assert stop == 17
    assert stop == next(i + 1 for i in range(len(seq)) if not so.proceed(seq[:i + 1], 5.0, width))
    assert bsv.proceed([7.0] * 30, 5.0, width)                          # above max_error: go on
    assert not bsv.proceed([7.0] * 30, float("inf"), width)
    slope = [1.0 + 2e-4 * i for i in range(30)]                           # slope 2e-4 per iteration: go on
    assert bsv.proceed(slope, 5.0, width) and not bsv.proceed([1.0 + 5e-5 * i for i in range(30)], 5.0, width)


def test_link_removal_rule():
    from bsgpu import solver as bsv
    # square 0-1-2-3-0 plus a pendant tile 4 on tile 0
    links = np.array([[0, 1], [0, 3], [0, 4], [1, 2], [2, 3]])
    prob = bsv.Problem(5, links, np.arange(6), np.zeros((5, 3)), np.zeros((5, 3)), np.ones(5))
    assert bsv.worst_link(prob, np.array([1.0, 2.0, 9.0, 3.0, 0.5])) == 3     # 0-4 would cut tile 4 off
    assert bsv.worst_link(prob, np.array([5.0, 5.0, 0.0, 1.0, 1.0])) == 0     # first of equal maxima
    chain = bsv.Problem(2, np.array([[0, 1]]), np.arange(2), np.zeros((1, 3)), np.zeros((1, 3)), np.ones(1))
    assert bsv.worst_link(chain, np.array([9.0])) is None
    assert bsv.not_converged(np.array([0.1, 0.1, 0.1, 3.0]), 3.5, 7.0)
    assert not bsv.not_converged(np.array([0.5, 0.6, 0.7]), 3.5, 7.0)
    assert bsv.not_converged(np.array([8.0, 8.0]), 3.5, 7.0)
    dropped = bsv.drop_link(prob, 1)
    assert dropped.links.tolist() == [[0, 1], [0, 4], [1, 2], [2, 3]] and dropped.match_offsets.tolist() == [0, 1, 2, 3, 4]


def test_label_weights_and_correspondence_matches(tmp_path):
    from bsgpu import commands, n5 as bn5, solver as bsv
    from bsgpu.spimdata import SpimData2
    from tests.test_match_cpu import write_points
    xml = _xml(tmp_path, [dict(setup=s, size_xyz=(100, 100, 50), translation_xyz=(60.0 * s, 0, 0)) for s in range(2)])
    store = bn5.N5Store(str(tmp_path / "interestpoints.n5"), create=True)
    rng = np.random.default_rng(4)
    loc0 = rng.uniform(60, 100, (12, 3)) * (1, 1, 0.5)
    loc1 = loc0 - (60.0 - 2.0, 0, 0)                       # view 1 sits 2 px further right than its registration says
    for lab, sl in (("beads", slice(0, 8)), ("nuclei", slice(8, 12))):
        write_points(store, (0, 0), lab, loc0[sl])
        write_points(store, (0, 1), lab, loc1[sl])
        n = sl.stop - sl.start
        rows0 = [(i, (0, 1), lab, i) for i in range(n)]
        rows1 = [(i, (0, 0), lab, i) for i in range(n)]
        store.write_correspondences(f"tpId_0_viewSetupId_0/{lab}", rows0)
        store.write_correspondences(f"tpId_0_viewSetupId_1/{lab}", rows1)
    data = SpimData2.load(xml)
    views = data.view_ids()
    regs = {v: data.model(*v) for v in views}
    ips = commands._InterestPoints(store, views, ["beads", "nuclei"], regs, tables=True)
    ta, tb, p, q, w = bsv.ip_matches(ips, {v: i for i, v in enumerate(views)}, views, ["beads", "nuclei"], [1.0, 0.25])
    assert len(ta) == 12 and sorted(w.tolist()) == [0.25] * 4 + [1.0] * 8        # once per pair, the label's weight
    assert np.allclose(q - p, (2.0, 0, 0))
    ta, *_ = bsv.ip_matches(ips, {v: i for i, v in enumerate(views)}, views, ["beads"], [1.0])
    assert len(ta) == 8

    ctx = SolverFakeContext()
    res = commands.solver(xml, ctx, "IP", labels=["beads", "nuclei"], label_weights=[1.0, 0.25],
                          transformation_model="TRANSLATION", regularization_model="NONE", max_plateau_width=10)
    assert np.allclose(res["models"][(0, 1)], _T((-2.0, 0, 0)), atol=1e-9)
    assert np.allclose(SpimData2.load(xml).model(0, 1), _T((58.0, 0, 0)), atol=1e-9)


# ------------------------------------------------------------------------------------------ the command
def _stitched_row(tmp_path, channels=1):
    from bsgpu.spimdata import SpimData2
    xml = _row_of_three(tmp_path, channels)
    data = SpimData2.load(xml)
    g = [tuple((0, t * channels + c) for c in range(channels)) for t in range(3)]
    a = [x if channels > 1 else x[0] for x in g]
    _store_result(data, a[0], a[1], _T((3.0, -2.0, 1.0)), 0.9, (80, 0, 0), (99, 79, 59))
    _store_result(data, a[1], a[2], _T((1.0, 1.0, 0.0)), 0.8, (160, 0, 0), (179, 79, 59))
    data.save(backup=False)
    return xml


def test_solver_stitching_end_to_end_writes_preconcatenated_registrations(tmp_path):
    from bsgpu import commands
    from bsgpu.spimdata import SpimData2
    xml = _stitched_row(tmp_path)
    before = open(xml).read()
    ctx = SolverFakeContext()
    kw = dict(transformation_model="TRANSLATION", regularization_model="NONE", max_plateau_width=10)
    res = commands.solver(xml, ctx, "STITCHING", dry_run=True, **kw)
    assert open(xml).read() == before and not os.path.exists(xml + "~1")        # dry run: file untouched
    want = {(0, 0): _T((0, 0, 0)), (0, 1): _T((3, -2, 1)), (0, 2): _T((4, -1, 1))}
    assert set(res["models"]) == set(want) and all(np.allclose(res["models"][v], want[v], atol=1e-9) for v in want)
    res = commands.solver(xml, ctx, "STITCHING", **kw)
    assert open(xml + "~1").read() == before
    data = SpimData2.load(xml)
    for v in want:
        name, M = data.registrations[v][0]
        assert name == "TranslationModel3D" and np.allclose(M, want[v], atol=1e-9)
        assert len(data.registrations[v]) == 3
        assert np.allclose(data.model(*v), want[v] + _T((80.0 * v[1], 0, 0)) - np.eye(3, 4), atol=1e-9)
    # the registrations changed, so every stored result is stale now: nothing is solved or written
    res2 = commands.solver(xml, ctx, "STITCHING", **kw)
    assert res2["models"] == {} and res2["stats"]["stale_results"] == 2
    assert len(SpimData2.load(xml).registrations[(0, 1)]) == 3


def test_solver_fixed_views_auto_explicit_disabled_and_grouping(tmp_path):
    from bsgpu import commands
    xml = _stitched_row(tmp_path, channels=2)
    kw = dict(transformation_model="TRANSLATION", regularization_model="NONE", max_plateau_width=10, dry_run=True)
    ctx = SolverFakeContext()
    res = commands.solver(xml, ctx, "STITCHING", **kw)          # channels grouped by default: 3 tiles, views share
    m = res["models"]
    assert len(m) == 6 and np.allclose(m[(0, 2)], m[(0, 3)]) and np.allclose(m[(0, 0)], np.eye(3, 4))
    assert np.allclose(m[(0, 2)], _T((3, -2, 1)), atol=1e-9)
    res = commands.solver(xml, ctx, "STITCHING", fixed_views=["0,4"], **kw)
    assert np.allclose(res["models"][(0, 5)], np.eye(3, 4)) and np.allclose(res["models"][(0, 0)], _T((-4, 1, -1)), atol=1e-9)
    res = commands.solver(xml, ctx, "STITCHING", disable_fixed_views=True, **kw)
    m = res["models"]
    assert np.allclose(m[(0, 2)][:, 3] - m[(0, 0)][:, 3], (3, -2, 1), atol=1e-6)
    # ungrouped channels: the views of channel 1 have no stored result and keep their registration
    res = commands.solver(xml, ctx, "STITCHING", group_channels=False, group_illums=False, **kw)
    assert len(res["models"]) == 3 and res["stats"]["unconnected_views"] == [(0, 1), (0, 3), (0, 5)]


def test_solver_iterative_removes_the_inconsistent_link(tmp_path):
    from bsgpu import commands, solver as bsv
    from bsgpu.spimdata import SpimData2
    tiles = [dict(setup=3 * j + i, size_xyz=(100, 100, 40), translation_xyz=(80.0 * i, 80.0 * j, 0)) for j in range(3)
             for i in range(3)]
    xml = _xml(tmp_path, tiles)
    data = SpimData2.load(xml)
    truth = {s: np.array([(s * 7) % 3 - 1.0, (s * 5) % 3 - 1.0, 0.5 * (s % 2)]) for s in range(9)}
    for j in range(3):
        for i in range(3):
            s = 3 * j + i
            for (u, ov_min, ov_max) in ((s + 1, (80.0 * (i + 1), 80.0 * j, 0), (80.0 * i + 99, 80.0 * j + 99, 39)) if i < 2 else (None,) * 3,
                                        (s + 3, (80.0 * i, 80.0 * (j + 1), 0), (80.0 * i + 99, 80.0 * j + 99, 39)) if j < 2 else (None,) * 3):
                if u is not None:
                    _store_result(data, (0, s), (0, u), _T(truth[u] - truth[s]), 0.9, ov_min, ov_max)
    _store_result(data, (0, 0), (0, 8), _T((60.0, -70.0, 30.0)), 0.95, (80, 80, 0), (99, 99, 39))   # bogus
    data.save(backup=False)
    kw = dict(transformation_model="TRANSLATION", regularization_model="NONE", max_plateau_width=20, dry_run=True)
    res = commands.solver(xml, SolverFakeContext(), "STITCHING", method="ONE_ROUND_ITERATIVE", **kw)
    assert res["removed"] == [([(0, 0)], [(0, 8)])]
    for s in range(9):
        assert np.allclose(res["models"][(0, s)][:, 3], truth[s] - truth[0], atol=1e-4), s
    res = commands.solver(xml, SolverFakeContext(), "STITCHING", **kw)
    assert res["removed"] == [] and not np.allclose(res["models"][(0, 8)][:, 3], truth[8] - truth[0], atol=0.25)
    assert bsv.model_name("AFFINE", "RIGID") == "InterpolatedAffineModel3D"


def test_unbuilt_flags_raise(tmp_path):
    from bsgpu import commands
    xml = _stitched_row(tmp_path)
    for kw in (dict(method="TWO_ROUND_SIMPLE"), dict(method="TWO_ROUND_ITERATIVE"),
               dict(registration_tp="TIMEPOINTS_TO_REFERENCE")):
        with pytest.raises(NotImplementedError):
            commands.solver(xml, SolverFakeContext(), "STITCHING", **kw)
    with pytest.raises(ValueError):
        commands.solver(xml, SolverFakeContext(), "IP")
    with pytest.raises(ValueError):
        commands.solver(xml, SolverFakeContext(), "IP", labels=["a", "b"], label_weights=[1.0])


def test_solve_struct_layout_matches_header(tmp_path):
    """sizeof / offsetof of bs_solve_params and bs_solve_stats from the real header == the ctypes mirrors."""
    import subprocess
    import bsgpu
    n = bsgpu.native
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "sz.c"
    src.write_text('''#include <stdio.h>
#include <stddef.h>
#include "bsgpu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(bs_solve_params), sizeof(bs_solve_stats),
         offsetof(bs_solve_params, lambda), offsetof(bs_solve_params, max_error), offsetof(bs_solve_params, max_plateau_width),
         offsetof(bs_solve_stats, skipped_fits), offsetof(bs_solve_stats, error), offsetof(bs_solve_stats, models_in_shared));
  return 0; }''')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(n.SolveParamsC), C.sizeof(n.SolveStatsC), n.SolveParamsC.lam.offset, n.SolveParamsC.max_error.offset,
            n.SolveParamsC.max_plateau_width.offset, n.SolveStatsC.skipped_fits.offset, n.SolveStatsC.error.offset,
            n.SolveStatsC.models_in_shared.offset]
    assert got == want
