"""solver on the device: bs_solve_tiles against oracle/solver_oracle.py after 1, 2 and 50 iterations on chains, grids and
random graphs for every model x regularizer; convergence, the iteration count, bit-identical repeats and argument errors;
and the command chains stitching -> solver -> affine-fusion, ONE_ROUND_ITERATIVE link removal and detect -> match ->
solver."""
import zlib

import numpy as np
import pytest

import bsgpu
from oracle import solver_oracle as so
from tests import synth

pytestmark = pytest.mark.gpu

MODELS = [(tm, rm) for tm in ("TRANSLATION", "RIGID", "AFFINE") for rm in ("NONE", "IDENTITY", "TRANSLATION", "RIGID", "AFFINE")]


def _rot(axis, ang):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _graph(kind, rng):
    """(n_tiles, links, tile centres)."""
    if kind == "chain":
        n = 6
        pos = np.array([[100.0 * i, 0, 0] for i in range(n)])
        links = [(i, i + 1) for i in range(n - 1)]
    elif kind in ("grid2", "grid3"):
        dims = (4, 3, 1) if kind == "grid2" else (3, 3, 2)
        idx = {}
        for z in range(dims[2]):
            for y in range(dims[1]):
                for x in range(dims[0]):
                    idx[(x, y, z)] = len(idx)
        pos = np.array([[100.0 * x, 100.0 * y, 60.0 * z] for (x, y, z) in idx])
        links = [(idx[k], idx[(k[0] + dx, k[1] + dy, k[2] + dz)]) for k in idx for dx, dy, dz in ((1, 0, 0), (0, 1, 0), (0, 0, 1))
                 if (k[0] + dx, k[1] + dy, k[2] + dz) in idx]
    else:
        n = 12
        pos = rng.uniform(0, 300, (n, 3))
        links = sorted({tuple(sorted(rng.choice(n, 2, replace=False))) for _ in range(25)} | {(i, i + 1) for i in range(n - 1)})
    return len(pos), links, pos + 1e4


def _problem(kind, seed, noise=0.3, singular=False, truth_model="AFFINE"):
    """Matches of planted models (tile t sees world point c at truth_t^-1(c)) plus noise.  ``singular``: the last tile
    keeps one link, to the tile before it, whose noise-free matches lie on a line, so RIGID and AFFINE fits of that
    tile are singular."""
    from bsgpu import solver as bsv
    rng = np.random.default_rng(seed)
    n, links, pos = _graph(kind, rng)
    if singular:
        links = [l for l in links if n - 1 not in l] + [(n - 2, n - 1)]
    truth = []
    for t in range(n):
        G = np.eye(3, 4)
        if truth_model != "TRANSLATION":
            G[:, :3] = _rot(rng.normal(size=3), 0.02 * rng.normal())
        if truth_model == "AFFINE":
            G[:, :3] = G[:, :3] @ (np.eye(3) + 0.005 * rng.normal(size=(3, 3)))
        G[:, 3] = rng.normal(0, 3, 3) + pos[t] - G[:, :3] @ pos[t]
        truth.append(G)
    inv = [np.linalg.inv(np.vstack([G, [0, 0, 0, 1]]))[:3] for G in truth]
    ta, tb, p, q, w = [], [], [], [], []
    for a, b in links:
        m = int(rng.integers(6, 40))
        line = singular and b == n - 1
        c = (pos[a] + pos[b]) / 2 + (np.outer(np.linspace(-30, 30, m), (1.0, 0.3, 0.2)) if line else rng.uniform(-30, 30, (m, 3)))
        sd = 0.0 if line else noise
        ta.append(np.full(m, a))
        tb.append(np.full(m, b))
        p.append(c @ inv[a][:, :3].T + inv[a][:, 3] + rng.normal(0, sd, (m, 3)))
        q.append(c @ inv[b][:, :3].T + inv[b][:, 3] + rng.normal(0, sd, (m, 3)))
        w.append(rng.uniform(0.5, 1.5, m))
    return bsv.build_problem(n, *(np.concatenate(x) for x in (ta, tb, p, q, w))), truth


def _args(prob, fixed):
    from bsgpu import solver as bsv
    _, off, order = bsv.colouring(prob.n_tiles, prob.links)
    return (off, order, fixed, prob.links, prob.match_offsets, prob.p, prob.q, prob.w)


def _close(got, want, rtol=1e-9):
    scale = max(1.0, float(np.abs(want).max()))
    assert np.all(np.abs(got - want) <= rtol * scale), float(np.abs(got - want).max())


@pytest.mark.parametrize("kind", ["chain", "grid2", "grid3", "random"])
@pytest.mark.parametrize("tm, rm", MODELS)
def test_device_equals_oracle_after_k_iterations(ctx, kind, tm, rm):
    from bsgpu import matching as bm
    from bsgpu import solver as bsv
    singular = kind == "random" and tm != "TRANSLATION"
    prob, _ = _problem(kind, seed=zlib.crc32(f"{kind}{tm}{rm}".encode()) % 1000, singular=singular)
    for fixed_first in (True, False):
        fixed = np.zeros(prob.n_tiles, np.int32)
        fixed[0] = 1 if fixed_first else 0
        prob.fixed = fixed
        M0 = bsv.prealign(prob, bm.Model(tm, rm, 0.1))
        for k in (1, 2, 50):
            kw = dict(transformation=tm, regularization=rm, lam=0.1, max_error=5.0, max_iterations=k, max_plateau_width=1000)
            g = ctx.solve_tiles(*_args(prob, fixed), M0, **kw)
            o = so.solve_tiles(*_args(prob, fixed), M0, **kw)
            _close(g[0], o[0])
            assert g[1]["iterations"] == o[1]["iterations"] == k and g[1]["skipped_fits"] == o[1]["skipped_fits"]
            _close(g[2], o[2], 1e-8)
            _close(g[3], o[3], 1e-8)
            _close(g[4], o[4], 1e-8)
            if singular:
                assert g[1]["skipped_fits"] >= k


def test_convergence_recovers_planted_models_and_follows_the_oracle(ctx):
    from bsgpu import matching as bm
    from bsgpu import solver as bsv
    for tm in ("TRANSLATION", "RIGID", "AFFINE"):
        prob, truth = _problem("grid2", seed=5, noise=0.0, truth_model=tm)
        prob.fixed = np.zeros(prob.n_tiles, np.int32)
        prob.fixed[0] = 1
        M, _, st = bsv.solve(ctx, prob, bm.Model(tm, "NONE"), max_error=1e-9, max_iterations=20000, max_plateau_width=200)
        assert st["stopped"]
        # tile 0 is fixed, so tile t must become truth_0^-1 truth_t: compare where the matches are
        T0i = np.linalg.inv(np.vstack([truth[0], [0, 0, 0, 1]]))
        for t in range(prob.n_tiles):
            want = (T0i @ np.vstack([truth[t], [0, 0, 0, 1]]))[:3]
            x = np.concatenate([prob.p, prob.q])
            err = np.abs(x @ (M[t][:, :3] - want[:, :3]).T + (M[t][:, 3] - want[:, 3]))
            assert err.max() < 1e-6, (tm, t, err.max())
    # noisy: device and oracle converge to the same solution and stop within one iteration of each other
    prob, _ = _problem("grid3", seed=7, noise=0.5)
    prob.fixed = np.zeros(prob.n_tiles, np.int32)
    prob.fixed[0] = 1
    M0 = bsv.prealign(prob, bm.Model("AFFINE", "RIGID", 0.1))
    kw = dict(transformation="AFFINE", regularization="RIGID", lam=0.1, max_error=5.0, max_iterations=10000,
              max_plateau_width=200)
    g = ctx.solve_tiles(*_args(prob, prob.fixed), M0, **kw)
    o = so.solve_tiles(*_args(prob, prob.fixed), M0, **kw)
    assert abs(g[1]["iterations"] - o[1]["iterations"]) <= 1 and g[1]["stopped"] and o[1]["stopped"]
    x = np.concatenate([prob.p, prob.q])
    for t in range(prob.n_tiles):
        d = np.abs(x @ (g[0][t][:, :3] - o[0][t][:, :3]).T + (g[0][t][:, 3] - o[0][t][:, 3]))
        assert d.max() < 1e-2, (t, d.max())


def test_repeat_runs_are_bit_identical_and_errors_leave_the_context_usable(ctx):
    from bsgpu import matching as bm
    from bsgpu import solver as bsv
    prob, _ = _problem("grid3", seed=11, noise=0.4)
    fixed = np.zeros(prob.n_tiles, np.int32)
    fixed[0] = 1
    prob.fixed = fixed
    M0 = bsv.prealign(prob, bm.Model("AFFINE", "RIGID", 0.1))
    kw = dict(transformation="AFFINE", regularization="RIGID", lam=0.1, max_iterations=300, max_plateau_width=50)
    a = ctx.solve_tiles(*_args(prob, fixed), M0, **kw)
    b = ctx.solve_tiles(*_args(prob, fixed), M0, **kw)
    for x, y in zip((a[0], a[2], a[3], a[4]), (b[0], b[2], b[3], b[4])):
        assert np.array_equal(x, y)
    assert a[1] == b[1]
    off, order, _, links, mo, p, q, w = _args(prob, fixed)
    bad = [
        dict(colour_offsets=[0, prob.n_tiles], colour_tiles=np.arange(prob.n_tiles)),    # links inside one colour
        dict(links=np.where(links == 1, prob.n_tiles + 3, links)),                      # tile out of range
        dict(w=-w),
        dict(p=np.where(np.arange(len(p))[:, None] == 3, np.nan, p)),
        dict(transformation="IDENTITY"),
        dict(max_iterations=0),
        dict(lam=1.5),
    ]
    for change in bad:
        args = dict(colour_offsets=off, colour_tiles=order, fixed=fixed, links=links, match_offsets=mo, p=p, q=q, w=w,
                    models=M0, **kw)
        args.update(change)
        with pytest.raises(bsgpu.BsError) as e:
            ctx.solve_tiles(**args)
        assert e.value.code == -1
    c = ctx.solve_tiles(*_args(prob, fixed), M0, **kw)
    assert np.array_equal(c[0], a[0])


# ------------------------------------------------------------------------------------------ command chains
def _grid_dataset(tmp_path, n=96, ov=32, seed=21):
    """3 x 3 x 1 tiles of one field; tile s truly sits at its nominal position + err[s] (integer px), the XML has the
    nominal positions."""
    from bsgpu import n5 as bn5, spimdata
    step = n - ov
    G = synth.field((n + 16, 2 * step + n + 16, 2 * step + n + 16), seed=seed, sigma=1.0)
    rng = np.random.default_rng(seed)
    err = {s: (np.array([0, 0, 0]) if s == 0 else rng.integers(-3, 4, 3)) for s in range(9)}
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles, vols = [], {}
    for j in range(3):
        for i in range(3):
            s = 3 * j + i
            e = err[s]
            vol = synth.tile_from(G, (8 + e[2], 8 + step * j + e[1], 8 + step * i + e[0]), (n, n, n), 100 + s)
            vols[s] = vol
            bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 64))
            tiles.append(dict(setup=s, size_xyz=(n, n, n), tile=s, translation_xyz=(step * i, step * j, 0)))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    truth = {(0, s): synth.translation((step * (s % 3) + err[s][0], step * (s // 3) + err[s][1], err[s][2]))
             for s in range(9)}
    return xml, truth, vols


def test_chain_stitching_solver_fusion_and_iterative_link_removal(ctx, tmp_path):
    from bsgpu import commands, n5 as bn5
    from bsgpu.spimdata import SpimData2
    from oracle import fusion_oracle as fo
    xml, truth, vols = _grid_dataset(tmp_path)
    commands.stitching(xml, ctx, downsampling=(1, 1, 1))
    assert len(SpimData2.load(xml).stitching_results()) >= 12
    base = open(xml).read()

    # ONE_ROUND_ITERATIVE drops exactly one inserted bogus result; ONE_ROUND_SIMPLE cannot
    data = SpimData2.load(xml)
    h = SpimData2.transform_hash(data.registrations[(0, 0)], data.registrations[(0, 8)])
    data.set_stitching_results([dict(pair=((0, 0), (0, 8)), shift=synth.translation((150.0, -170.0, 90.0)), r=0.95, hash=h,
                                     bbox_min=(64, 64, 0), bbox_max=(95, 95, 95))])
    data.save(backup=False)
    kw = dict(transformation_model="TRANSLATION", regularization_model="NONE", dry_run=True)
    it = commands.solver(xml, ctx, "STITCHING", method="ONE_ROUND_ITERATIVE", **kw)
    assert it["removed"] == [([(0, 0)], [(0, 8)])]
    simple = commands.solver(xml, ctx, "STITCHING", **kw)
    for v, T in truth.items():
        M = it["models"][v] @ np.vstack([SpimData2.load(xml).model(*v), [0, 0, 0, 1]])
        assert np.abs(M - T).max() < 0.25, (v, M - T)
    assert max(np.abs(simple["models"][v] @ np.vstack([SpimData2.load(xml).model(*v), [0, 0, 0, 1]]) - truth[v]).max()
               for v in truth) > 0.25
    open(xml, "w").write(base)

    res = commands.solver(xml, ctx, "STITCHING", transformation_model="TRANSLATION", regularization_model="NONE")
    assert res["stats"]["stale_results"] == 0 and len(res["models"]) == 9
    data = SpimData2.load(xml)
    for v, T in truth.items():
        assert np.abs(data.model(*v) - T).max() < 0.25, (v, data.model(*v) - T)
    solved = open(xml).read()
    again = commands.solver(xml, ctx, "STITCHING", transformation_model="TRANSLATION", regularization_model="NONE")
    assert again["models"] == {} and again["stats"]["stale_results"] >= 12 and open(xml).read() == solved

    out = str(tmp_path / "fused.n5")
    commands.create_fusion_container(xml, out, block_size=(64, 64, 32))
    ds = commands.affine_fusion(out, ctx, "AVG_BLEND", block_scale=(2, 2, 1))
    st, meta = bn5.read_fusion_container(out)
    fused = st.read_volume(ds[0])
    lo = np.asarray(meta["bb_min"])
    views = []
    for s in range(9):
        M = SpimData2.load(xml).model(0, s)
        border, rng = fo.adjust_blending(M)
        views.append(fo.View(vols[s], M, border, rng))
    want = fo.fuse_block(views, lo, fused.shape[::-1], fo.AVG_BLEND)
    err = np.abs(fused - want) / np.maximum(np.abs(want), 1.0)
    assert (err > 1e-4).mean() < 1e-3
    tviews = [fo.View(vols[s], truth[(0, s)], *fo.adjust_blending(truth[(0, s)])) for s in range(9)]
    twant = fo.fuse_block(tviews, lo, fused.shape[::-1], fo.AVG_BLEND)
    inner = (slice(8, -8),) * 3
    assert np.corrcoef(fused[inner].ravel(), twant[inner].ravel())[0, 1] > 0.99


def test_chain_detect_match_solver_recovers_a_planted_rotation(ctx, tmp_path):
    from bsgpu import commands, n5 as bn5, spimdata
    from bsgpu.spimdata import SpimData2
    from tests.test_interestpoints_gpu import _beads
    from tests.test_match_cpu import compose, rot_z
    rng = np.random.default_rng(19)
    world = np.stack([rng.uniform(6, 250, 260), rng.uniform(6, 122, 260), rng.uniform(3, 29, 260)], 1)
    store = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    tiles, true = [], {}
    for s, t in enumerate((0.0, 96.0)):
        local = world - (t, 0, 0)
        inside = local[(local[:, 0] > 3) & (local[:, 0] < 157)]
        vol = _beads((32, 128, 160), [tuple(p) for p in inside], 1 + s, sigma_xy=1.6, sigma_z=1.6)
        bn5.write_bdv_setup(store, s, 0, vol, (64, 64, 32))
        tiles.append(dict(setup=s, size_xyz=(160, 128, 32), tile=s, translation_xyz=(t, 0, 0)))
        true[(0, s)] = synth.translation((t, 0, 0))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    data = SpimData2.load(xml)
    wrong = compose(rot_z(0.8, (96 + 80, 64, 16)), synth.translation((97.5, -1.0, 0.5)))
    data.registrations[(0, 1)] = [("Translation to Regular Grid", wrong)]
    for vr in data.root.iter("ViewRegistration"):
        if vr.get("setup") == "1":
            vr.find("ViewTransform").find("affine").text = " ".join(repr(float(v)) for v in wrong.ravel())
    data.save(backup=False)
    commands.detect_interestpoints(xml, ctx, "beads", sigma=1.6, threshold=0.01, min_intensity=0.0, max_intensity=1000.0,
                                   downsample_xy=1, block_size=(64, 64, 32))
    m = commands.match_interestpoints(xml, ctx, ["beads"], "PRECISE_TRANSLATION", ransac_min_num_inliers=8)
    assert all(len(p) >= 20 for p in m.values()), {k: len(v) for k, v in m.items()}
    res = commands.solver(xml, ctx, "IP", labels=["beads"], transformation_model="AFFINE", regularization_model="RIGID",
                          regularization_lambda=0.1)
    data = SpimData2.load(xml)
    corners = np.array([[x, y, z] for x in (0, 159) for y in (0, 127) for z in (0, 31)], dtype=np.float64)
    for v, T in true.items():
        M = data.model(*v)
        d = np.linalg.norm(corners @ (M[:, :3] - T[:, :3]).T + (M[:, 3] - T[:, 3]), axis=1)
        assert d.max() < 0.5, (v, d)
    assert res["stats"]["iterations"] > 200
