"""Intensity correction on the CPU: known answers of the oracle and the host logic, and match-intensities,
solve-intensities and affine-fusion --intensityN5Path end to end through an oracle-backed context."""
import numpy as np
import pytest

from bsgpu import commands, intensity as bint, n5 as bn5, spimdata
from oracle import intensity_oracle as io
from tests.intensity_scene import (DEFAULT_GRID, WIDE_SLOTS, IntensityFakeContext, apply_bound, apply_case,
                                   candidate_value_bound, integer_scene, later_round_bucket, overlap_disagreement,
                                   planted_dataset, shifted_grid_scene)


def test_cell_index_at_the_edges():
    d, n = 64.0, 4
    p = np.array([-0.0, 0.0, 15.999, 16.0, 47.99, 48.0, 63.0, 64.0, 70.0])
    assert io.cell_index(p, n, d).tolist() == [0, 0, 0, 1, 2, 3, 3, 3, 3]
    assert io.cell_index([-5.0], n, d).tolist() == [0]


def test_coefficient_field_is_the_cell_value_at_centres_and_clamps():
    n = (4, 2, 1)
    full = (64, 32, 8)
    ca = np.arange(8, dtype=np.float64).reshape(1, 2, 4) + 1.0
    cb = np.zeros_like(ca)
    vol = np.ones((8, 32, 64), np.float32)
    out = io.apply(vol, (0, 0, 0), np.eye(3, 4), full, ca, cb)
    # cell centres at (c + 0.5) d / n - 0.5: y 7.5 and 23.5 here, so y 0..7 and 24..31 take one row of cells
    for cy, y in ((0, 0), (0, 7), (1, 24), (1, 31)):
        assert out[0, y, 0] == ca[0, cy, 0]              # clamped below the first centre
        assert out[0, y, 63] == ca[0, cy, 3]             # clamped beyond the last centre
        assert ca[0, cy, 0] < out[0, y, 8] < ca[0, cy, 1]
    # exactly on a centre: full 32 in y with 2 cells -> centres 7.5 and 23.5; use n = 2 over 34 px (centres 8, 25)
    out2 = io.apply(np.ones((1, 1, 34), np.float32), (0, 0, 0), np.eye(3, 4), (34, 1, 1), np.array([[[2.0, 5.0]]]),
                    np.array([[[0.0, 0.0]]]))
    assert out2[0, 0, 8] == 2.0 and out2[0, 0, 25] == 5.0 and out2[0, 0, 0] == 2.0 and out2[0, 0, 33] == 5.0


def test_splitmix64_stream_against_hand_values():
    # splitmix64 reference values (Vigna): state 0 -> first output
    assert io.splitmix64(0) == 0xE220A8397B1DCDAF
    assert io.splitmix64(1) == 0x910A2DEC89025CC1
    i, j = io.draw(7, 0, 10)
    assert 0 <= i < 10 and 0 <= j < 10 and i != j
    for h in range(200):
        i, j = io.draw(3, h, 2)
        assert {i, j} == {0, 1}


def test_filter_and_acceptance_at_their_boundaries():
    x = np.arange(20, dtype=np.float64)
    y = 2 * x + 1
    inl = bint.filter_accept(x, y, 2.0, 1.0, 0.5, 3.0, 0.1, 20)
    assert inl is not None and inl.all()
    assert bint.filter_accept(x, y, 2.0, 1.0, 0.5, 3.0, 0.1, 21) is None          # min_num_inliers
    y2 = y.copy()
    y2[:10] += 100.0                                                               # half are outliers
    assert bint.filter_accept(x, y2, 2.0, 1.0, 0.5, 3.0, 0.5, 2) is not None       # exactly the ratio
    assert bint.filter_accept(x, y2, 2.0, 1.0, 0.5, 3.0, 0.51, 2) is None
    assert bint.filter_accept(np.ones(5), np.ones(5), 1.0, 0.0, 0.5, 3.0, 0.1, 2) is None   # singular fit
    assert bint.filter_accept(x[:1], y[:1], 2.0, 1.0, 0.5, 3.0, 0.1, 0) is None             # at least 2
    # the oracle agrees
    assert (io.filter_accept(x, y2, 2.0, 1.0, 0.5, 3.0, 0.5, 2) == bint.filter_accept(x, y2, 2.0, 1.0, 0.5, 3.0, 0.5, 2)).all()


def test_pair_rule_across_timepoints():
    b = {(0, 0): (np.zeros(3), np.full(3, 10.0)), (0, 1): (np.full(3, 10.0), np.full(3, 20.0)),
         (1, 0): (np.full(3, 5.0), np.full(3, 6.0)), (1, 1): (np.full(3, 30.0), np.full(3, 40.0))}
    views = sorted(b)
    assert bint.pairs(views, b) == [((0, 0), (0, 1)), ((0, 0), (1, 0))]
    lo, hi = bint.render_range(np.array([0.3, 1.0, -0.1]), np.array([4.9, 2.0, 0.1]), 0.5)
    assert lo.tolist() == [1, 1, 0] and hi.tolist() == [2, 1, 0]


@pytest.mark.parametrize("storage,path", [("N5", "c.n5"), ("ZARR", "c.zarr")])
def test_coefficient_round_trip(tmp_path, storage, path):
    p = str(tmp_path / path)
    assert bint.guess_storage(p) == storage
    rng = np.random.default_rng(1)
    co = {(0, 3): (rng.random((2, 3, 4)), rng.random((2, 3, 4))), (1, 5): (np.ones((2, 3, 4)), np.zeros((2, 3, 4)))}
    bint.write_coefficients(p, storage, "grp", "intensity", co)
    for v, (a, b) in co.items():
        ga, gb = bint.read_coefficients(p, storage, "grp", "intensity", v)
        assert np.array_equal(ga, a) and np.array_equal(gb, b)
    assert bint.read_coefficients(p, storage, "grp", "intensity", (2, 3)) is None
    assert bint.coefficient_dataset("", (4, 7), "intensity") == "setup7/timepoint4/intensity"


def test_histogram_and_hdf5_raise(tmp_path):
    xml, _ = planted_dataset(tmp_path, tile=(32, 32, 8), overlap=8)
    with pytest.raises(NotImplementedError):
        commands.match_intensities(xml, IntensityFakeContext(), str(tmp_path / "m.n5"), method="HISTOGRAM")
    with pytest.raises(NotImplementedError):
        bint.guess_storage(str(tmp_path / "c.h5"))
    with pytest.raises(NotImplementedError):
        commands.solve_intensities(xml, str(tmp_path / "c.hdf5"), str(tmp_path / "m.n5"))


def _run_chain(tmp_path, gains, n_cells=(4, 4, 2)):
    xml, raw = planted_dataset(tmp_path, gains=gains)
    ctx = IntensityFakeContext()
    m = str(tmp_path / "matches.n5")
    kw = dict(num_coefficients=n_cells, render_scale=0.5, min_num_candidates=200, num_iterations=150)
    got = commands.match_intensities(xml, ctx, m, **kw)
    co = commands.solve_intensities(xml, str(tmp_path / "coeff.n5"), m, num_coefficients=n_cells, max_iterations=300)
    return xml, raw, ctx, got, co


def test_planted_gain_is_recovered_end_to_end(tmp_path):
    xml, raw, ctx, got, co = _run_chain(tmp_path, gains=True)
    assert len(got) == 6 and sum(len(c) for c in got.values()) >= 8     # 4 edge + 2 diagonal pairs
    data = spimdata.SpimData2.load(xml)
    views = data.view_ids()
    regs = {v: data.model(*v) for v in views}
    dims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in views}
    store = bn5.N5Store(str(tmp_path / "dataset.n5"))
    stored = {v: store.read_volume(bn5.bdv_dataset(v[1], v[0], 0)).astype(np.float32) for v in views}
    corrected = {v: io.apply(stored[v], (0, 0, 0), np.eye(3, 4), dims[v], *co[v]) for v in views}
    prs = bint.pairs(views, {v: bint.view_bounds(dims[v], regs[v]) for v in views})
    before = overlap_disagreement(stored, regs, dims, prs)
    after = overlap_disagreement(corrected, regs, dims, prs)
    assert after <= 0.25 * before, (before, after)

    # affine-fusion with the coefficients: the fused overlap no longer jumps between tiles
    out = str(tmp_path / "fused.n5")
    commands.create_fusion_container(xml, out, block_size=(32, 32, 16))
    commands.affine_fusion(out, ctx, intensity_n5_path=str(tmp_path / "coeff.n5"))
    out0 = str(tmp_path / "plain.n5")
    commands.create_fusion_container(xml, out0, block_size=(32, 32, 16))
    commands.affine_fusion(out0, ctx)
    with pytest.raises(ValueError, match="setup"):
        commands.affine_fusion(out0, ctx, intensity_n5_path=str(tmp_path / "missing.n5"), intensity_n5_storage="N5")


def test_no_planted_gain_gives_identity_coefficients(tmp_path):
    _, _, _, got, co = _run_chain(tmp_path, gains=False)
    assert sum(len(c) for c in got.values()) > 0
    for a, b in co.values():
        assert np.abs(a - 1.0).max() < 1e-9 and np.abs(b).max() < 1e-9


def test_num_coefficients_mismatch_warns_and_uses_the_stored_size(tmp_path):
    xml, _ = planted_dataset(tmp_path, tile=(48, 48, 16), overlap=16)
    m = str(tmp_path / "matches.n5")
    commands.match_intensities(xml, IntensityFakeContext(), m, num_coefficients=(2, 2, 1), render_scale=0.5,
                               min_num_candidates=50, num_iterations=50)
    with pytest.warns(UserWarning, match="numCoefficients"):
        co = commands.solve_intensities(xml, str(tmp_path / "c.zarr"), m, num_coefficients=(8, 8, 8), max_iterations=20)
    assert all(a.shape == (1, 2, 2) for a, _ in co.values())


# ------------------------------------------------------------------------------------------------ float64 references
@pytest.mark.parametrize("scene", ["default_grid", "wide_slots", "integer_200", "integer_nan"])
def test_candidates_reference_agrees_with_the_oracle(scene):
    """On the exact-geometry scenes of the kernel tests the float64 reference keeps the same points under the same
    keys as the bit-level oracle, and its values are within 16 u max|corner| (PARITY_GAPS row 37)."""
    if scene.startswith("integer"):
        A, B, va, vb, rmin, rmax = integer_scene()
        th = (1.0, 200.0 if scene == "integer_200" else float("nan"))
    else:
        A, B, va, vb, rmin, rmax = shifted_grid_scene(**(DEFAULT_GRID if scene == "default_grid" else WIDE_SLOTS))
        th = (1.0, float("nan"))
    want = io.candidates(A, va, B, vb, 1.0, rmin, rmax, *th)
    keys, offs, cnts, vals, cmax = io.candidates_reference(A, va, B, vb, 1.0, rmin, rmax, *th, corners=True)
    for g, w in zip((keys, offs, cnts), want[:3]):
        assert np.array_equal(g, w)
    assert np.all(np.abs(want[3] - vals) <= candidate_value_bound(cmax))
    assert len(keys) >= 32 and len(vals) > 10000


def test_integer_scene_sits_on_every_boundary():
    """The integer scene reaches what its GPU test relies on: values exactly at min_threshold 1 and max_threshold
    200 among the kept points (so > instead of >= changes the output), and render points exactly on p = d - 1 and on
    cell borders p n / d in Z of both views."""
    A, B, va, vb, rmin, rmax = integer_scene()
    _, _, _, vals = io.candidates_reference(A, va, B, vb, 1.0, rmin, rmax, 1.0, 200.0)
    assert (vals == 1.0).any() and (vals == 200.0).any()
    strict = io.candidates_reference(A, va, B, vb, 1.0, rmin, rmax, np.nextafter(1.0, 2.0), np.nextafter(200.0, 0.0))
    assert len(strict[3]) < len(vals)
    g = np.stack(np.meshgrid(*[np.arange(rmin[k], rmax[k] + 1) for k in range(3)], indexing="ij")).reshape(3, -1)
    for v in (va, vb):
        m = np.asarray(v["world_to_px"]).reshape(3, 4)
        p = m[:, :3] @ g + m[:, 3:]
        d, n = np.asarray(v["full_dims"])[:, None], np.asarray(v["n_cells"])[:, None]
        assert (p == d - 1).any()
        border = (p * n % d == 0) & (p > 0)
        assert border.any(axis=1).all()


@pytest.mark.parametrize("x", [1, 257, 600])
@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_apply_reference_agrees_with_the_oracle(x, level, dtype):
    vol, wmin, mt, full, ca, cb = apply_case(x, level, dtype)
    want = io.apply(vol, wmin, mt, full, ca, cb)
    ref = io.apply_reference(vol, wmin, mt, full, ca, cb)
    assert np.all(np.abs(want - ref) <= apply_bound(vol, wmin, mt, full, ca, cb))


def test_apply_reference_is_the_cell_value_at_centres_and_clamps():
    # 2 cells over 34 px: centres at 8 and 25, constant beyond them; halfway between them the mean
    ca, cb = np.array([[[2.0, 5.0]]]), np.array([[[-1.0, 3.0]]])
    out = io.apply_reference(np.full((1, 1, 34), 2.0), (0, 0, 0), np.eye(3, 4), (34, 1, 1), ca, cb)[0, 0]
    assert out[0] == out[8] == 3.0 and out[25] == out[33] == 13.0
    assert np.isclose(out[16], 2 * (2 + 3 * 8 / 17) - 1 + 4 * 8 / 17, rtol=1e-15)
    # a 2x level: level voxel l sits at full-resolution q = 2 l + 0.5, so l = 4 is at fractional cell 9 * 2 / 34 - 0.5
    mt = np.array([[2, 0, 0, 0.5], [0, 1, 0, 0], [0, 0, 1, 0]], np.float64)
    u = 9 * 2 / 34 - 0.5
    got = io.apply_reference(np.ones((1, 1, 17)), (0, 0, 0), mt, (34, 1, 1), ca, cb)[0, 0, 4]
    assert np.isclose(got, (2 + 3 * u) + (-1 + 4 * u), rtol=1e-15)


def test_later_round_bucket_has_one_triple_found_first_at_h_1024():
    x, y = later_round_bucket()
    for iters, want in ((1024, 2), (1025, 3)):
        a, b, c = io.ransac_bucket(np.stack([x, y], 1), 0, iters, 1e-3)
        assert c == want
    assert (a, b) == (2.0, 3.0)
