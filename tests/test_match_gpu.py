"""match-interestpoints on the device: bs_descriptors_build neighbours and bs_descriptors_match results equal to
oracle/match_oracle.py (indices exactly, values within 1e-12 relative), argument errors, the command on a planted
scene against the oracle-backed context, and the chain detect -> match -> non-rigid fusion."""
import numpy as np
import pytest

import bsgpu
from oracle import match_oracle as mo

pytestmark = pytest.mark.gpu

LEGAL = [(n, r) for n in range(3, 7) for r in range(0, 4) if n + r <= 6]


def _cloud(n, seed, lattice=False):
    rng = np.random.default_rng(seed)
    if lattice:
        return rng.integers(0, 6, (n, 3)).astype(np.float64)      # many exact ties and duplicates
    return rng.uniform(0, 200, (n, 3))


def _rel_close(got, want):
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.all(np.abs(got[fin] - want[fin]) <= 1e-12 * np.maximum(np.abs(want[fin]), 1e-300))


@pytest.mark.parametrize("n_nb, red", LEGAL)
@pytest.mark.parametrize("size, lattice", [("k+1", False), (7, True), (1000, False), (1000, True)])
def test_knn_matches_oracle(ctx, n_nb, red, size, lattice):
    k = n_nb + red
    n = k + 1 if size == "k+1" else size
    xyz = _cloud(n, 10 + n + k, lattice)
    h = ctx.descriptors_build(xyz, n_nb, red)
    try:
        idx, d2 = ctx.descriptors_neighbors(h)
    finally:
        ctx.descriptors_free(h)
    wi, wd = mo.knn(xyz, k)
    assert np.array_equal(idx, wi)
    _rel_close(d2, wd)


def test_knn_30000(ctx):
    xyz = _cloud(30000, 5)
    h = ctx.descriptors_build(xyz, 3, 1)
    try:
        idx, d2 = ctx.descriptors_neighbors(h)
    finally:
        ctx.descriptors_free(h)
    wi, wd = mo.knn(xyz, 4, chunk=1024)
    assert np.array_equal(idx, wi)
    _rel_close(d2, wd)


def _match(ctx, a, b, n_nb=3, red=1, radius=None):
    ha = ctx.descriptors_build(a, n_nb, red)
    hb = ctx.descriptors_build(b, n_nb, red)
    try:
        return ctx.descriptors_match(ha, hb, radius)
    finally:
        ctx.descriptors_free(ha)
        ctx.descriptors_free(hb)


def _check_match(got, want):
    assert np.array_equal(got[0], want[0])
    _rel_close(got[1], want[1])
    _rel_close(got[2], want[2])


@pytest.mark.parametrize("na, nb", [(1000, 777), (129, 3001), (5, 6)])
@pytest.mark.parametrize("n_nb, red", [(3, 1), (3, 0), (4, 2), (6, 0)])
def test_match_matches_oracle(ctx, na, nb, n_nb, red):
    rng = np.random.default_rng(na + nb + n_nb)
    b = _cloud(nb, 20 + nb)
    a = np.vstack([b[:na // 2] + (3.5, -1.25, 2.0) + rng.normal(0, 0.2, (min(na // 2, nb), 3)),
                   _cloud(na - min(na // 2, nb), 30 + na)])
    _check_match(_match(ctx, a, b, n_nb, red), mo.match(a, b, n_nb, red))


def test_match_small_b_and_single_eligible_and_radius(ctx):
    a = _cloud(300, 1)
    got = _match(ctx, a, _cloud(4, 2))                                  # N_B <= k: no descriptors in B
    assert np.all(got[0] == -1) and np.all(np.isinf(got[1])) and np.all(np.isinf(got[2]))
    # lattice points with a radius that lands exactly on neighbours at distance 5 = |(3, 4, 0)|
    g = np.stack(np.meshgrid(np.arange(0, 40, 3.0), np.arange(0, 40, 4.0), np.arange(0, 12, 5.0), indexing="ij"), -1)
    g = g.reshape(-1, 3) + np.random.default_rng(3).integers(0, 2, (g.size // 3, 3))
    for r in (5.0, 0.0, 1e9):
        gb = g + np.array([3.0, 4.0, 0.0]) * (r == 5.0)
        _check_match(_match(ctx, g, gb, radius=r), mo.match(g, gb, search_radius=r))
    # a single eligible B point: second = inf
    b = np.vstack([_cloud(50, 4), [[1000.0, 1000.0, 1000.0]]])
    want = mo.match(b[-1:] + 0.0, b, search_radius=1.0)               # A has one point: no descriptors
    assert want[0][0] == -1
    a2 = np.vstack([b[:20], [[1000.0, 1000.0, 1000.0]]])
    got = _match(ctx, a2, b, radius=0.5)
    _check_match(got, mo.match(a2, b, search_radius=0.5))
    assert np.all(np.isinf(got[2][:20]))


def test_mismatched_parameters_raise_and_context_survives(ctx):
    a = _cloud(100, 7)
    ha = ctx.descriptors_build(a, 3, 1)
    hb = ctx.descriptors_build(a, 4, 1)
    try:
        with pytest.raises(bsgpu.BsError):
            ctx.descriptors_match(ha, hb)
        with pytest.raises(bsgpu.BsError):
            ctx.descriptors_build(a, 2, 1)
        with pytest.raises(bsgpu.BsError):
            ctx.descriptors_build(a, 4, 3)
        got = ctx.descriptors_match(ha, ha)
        assert np.array_equal(got[0], np.arange(100))
    finally:
        ctx.descriptors_free(ha)
        ctx.descriptors_free(hb)


# ------------------------------------------------------------------------------------------ the command
def test_command_on_a_planted_2x2_scene(ctx, tmp_path):
    from bsgpu import commands
    from tests.test_match_cpu import MatchFakeContext, RUN, check_scene, planted_scene, read_rows
    (tmp_path / "gpu").mkdir()
    (tmp_path / "fake").mkdir()
    kw = dict(grid=(2, 2), tile=(400, 400, 100), overlap=0.3, spacing=14.0, keep=0.5)
    xml, truth = planted_scene(tmp_path / "gpu", **kw)
    assert sum(len(t) for t in truth.values()) > 0
    res = commands.match_interestpoints(xml, ctx, ["beads"], **RUN)
    check_scene(tmp_path / "gpu", truth, res)
    fxml, _ = planted_scene(tmp_path / "fake", **kw)
    commands.match_interestpoints(fxml, MatchFakeContext(), ["beads"], **RUN)
    assert read_rows(tmp_path / "gpu", sorted(truth)) == read_rows(tmp_path / "fake", sorted(truth))


def test_chain_detect_match_nonrigid(ctx, tmp_path):
    from bsgpu import commands, n5 as bn5, spimdata
    from tests.test_interestpoints_gpu import _beads
    rng = np.random.default_rng(9)
    # one bead cloud in world, two tiles overlapping by 64 px in x
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
    commands.detect_interestpoints(xml, ctx, "beads", sigma=1.6, threshold=0.01, min_intensity=0.0, max_intensity=1000.0,
                                   downsample_xy=1, block_size=(64, 64, 24))
    res = commands.match_interestpoints(xml, ctx, ["beads"], "PRECISE_TRANSLATION", ransac_min_num_inliers=8,
                                        transformation_model="TRANSLATION", regularization_model="NONE")
    assert len(res) == 1 and all(len(p) >= 8 for p in res.values()), {k: len(v) for k, v in res.items()}
    written = commands.nonrigid_fusion(xml, ctx, str(tmp_path / "fused.n5"), "fused/s0", ["beads"],
                                       block_size=(64, 64, 24))
    assert len(written) > 0
