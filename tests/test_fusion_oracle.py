"""Known-answer pins for oracle/fusion_oracle.py (analytic expectations, SURVEY.md section 7.2)."""
import math
import os

import numpy as np
import pytest

from oracle import fusion_oracle as fo
from tests import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fusion_golden.npz")


def _view(vol, M, **kw):
    border, rng = fo.adjust_blending(M)
    return fo.View(vol, M, border, rng, **kw)


def test_single_view_identity_returns_input():
    vol = synth.tile_from(synth.field((12, 14, 16), seed=1), (0, 0, 0), (12, 14, 16), 1)
    out = fo.fuse_block([_view(vol, synth.translation((0, 0, 0)))], (0, 0, 0), (16, 14, 12), fo.AVG)
    assert np.array_equal(out, vol.astype(np.float32))
    # AVG_BLEND: weight is exactly 0 on the faces (dist == 0), identical inside
    out = fo.fuse_block([_view(vol, synth.translation((0, 0, 0)))], (0, 0, 0), (16, 14, 12), fo.AVG_BLEND)
    assert np.allclose(out[1:-1, 1:-1, 1:-1], vol.astype(np.float32)[1:-1, 1:-1, 1:-1], rtol=3e-7, atol=0)
    assert not out[0].any() and not out[:, 0].any() and not out[:, :, -1].any()


def test_linear_ramp_is_reproduced_regardless_of_weights():
    """Two views of the same linear ramp with a non-integer relative translation: trilinear
    interpolation is exact on a ramp, so the fused overlap equals the ramp for any weights."""
    z, y, x = np.meshgrid(np.arange(30), np.arange(34), np.arange(60), indexing="ij")
    t2 = (20.25, 1.5, -0.75)

    def ramp(X, Y, Z):
        return (3.0 * X + 5.0 * Y + 7.0 * Z + 100.0).astype(np.float32)

    v1 = ramp(x, y, z)
    v2 = ramp(x + t2[0], y + t2[1], z + t2[2])
    views = [_view(v1, synth.translation((0, 0, 0))), _view(v2, synth.translation(t2))]
    bmin, bsz = (22, 4, 2), (30, 24, 20)
    for ft in (fo.AVG, fo.AVG_BLEND):
        out = fo.fuse_block(views, bmin, bsz, ft)
        Z, Y, X = np.meshgrid(np.arange(bsz[2]) + bmin[2], np.arange(bsz[1]) + bmin[1],
                              np.arange(bsz[0]) + bmin[0], indexing="ij")
        assert np.allclose(out, ramp(X, Y, Z), rtol=2e-6)


def test_blend_weight_formula_and_partition():
    src = np.zeros((1, 5, 3), np.float32)
    src[0, :, 0] = [0.0, 10.0, 20.0, 40.0, 99.0]
    src[0, :, 1] = 50.0
    src[0, :, 2] = 50.0
    w = fo.blend_weight(src, (100, 101, 101), (0, 0, 0), (40, 40, 40))[0]
    assert w[0] == 0.0 and w[4] == 0.0                      # on the faces
    assert w[3] == 1.0                                       # dist >= range
    assert abs(w[1] - (math.cos(0.75 * math.pi) + 1) / 2) < 1e-7
    assert abs(w[2] - 0.5) < 1e-7
    # normalised weights of two views sum to one wherever either is positive
    vol = np.full((8, 8, 40), 500, np.uint16)
    views = [_view(vol, synth.translation((0, 0, 0))), _view(vol, synth.translation((25, 0, 0)))]
    out = fo.fuse_block(views, (0, 0, 0), (65, 8, 8), fo.AVG_BLEND)
    inner = out[1:-1, 1:-1, 1:-1]
    assert np.allclose(inner[inner > 0], 500.0, rtol=1e-6)


def test_lut_cosine_close_to_analytic():
    src = np.zeros((1, 200, 3), np.float32)
    src[0, :, 0] = np.linspace(0.1, 39.9, 200)
    src[0, :, 1:] = 50
    a = fo.blend_weight(src, (100, 101, 101), (0, 0, 0), (40, 40, 40), 0)
    b = fo.blend_weight(src, (100, 101, 101), (0, 0, 0), (40, 40, 40), 30)
    assert np.abs(a - b).max() < 1.5e-3 and np.abs(a - b).max() > 1e-5


def test_winner_fusion_types():
    lo = np.full((6, 6, 20), 100, np.uint16)
    hi = np.full((6, 6, 20), 900, np.uint16)
    views = [_view(lo, synth.translation((0, 0, 0))), _view(hi, synth.translation((10, 0, 0)))]
    args = ((0, 1, 1), (30, 4, 4))
    assert fo.fuse_block(views, *args, fo.MAX_INTENSITY)[0, 0, 15] == 900
    assert fo.fuse_block(views, *args, fo.LOWEST_VIEWID_WINS)[0, 0, 15] == 100
    assert fo.fuse_block(views, *args, fo.HIGHEST_VIEWID_WINS)[0, 0, 15] == 900
    cl = fo.fuse_block(views, *args, fo.CLOSEST_PIXEL_WINS)
    assert cl[0, 0, 12] == 100 and cl[0, 0, 17] == 900     # nearer to the centre of its view wins
    assert fo.fuse_block(views, *args, fo.AVG)[0, 0, 15] == 500
    assert fo.fuse_block(views, *args, fo.AVG)[0, 0, 5] == 100


def test_converters_round_and_clamp():
    v = np.array([[[-5.0, 0.0, 0.49, 0.5, 254.5, 300.0]]], np.float32)
    assert list(fo.convert_output(v, "uint8", 0.0, 255.0).ravel()) == [0, 0, 0, 1, 255, 255]
    v = np.array([[[100.0, 150.0, 200.0]]], np.float32)
    assert list(fo.convert_output(v, "uint16", 100.0, 200.0).ravel()) == [0, 32768, 65535]


def test_block_seam_invariance_oracle():
    G = synth.field((24, 30, 80), seed=2)
    vols = [synth.tile_from(G, (0, 0, 0), (20, 26, 40), 3), synth.tile_from(G, (2, 1, 30), (20, 26, 40), 4)]
    views = [_view(vols[0], synth.translation((0.3, 0.1, -0.2))), _view(vols[1], synth.translation((30.2, 1.4, 2.1)))]
    whole = fo.fuse_block(views, (0, 0, 0), (64, 24, 16), fo.AVG_BLEND)
    left = fo.fuse_block(views, (0, 0, 0), (32, 24, 16), fo.AVG_BLEND)
    right = fo.fuse_block(views, (32, 0, 0), (32, 24, 16), fo.AVG_BLEND)
    assert np.array_equal(whole, np.concatenate([left, right], axis=2))


def test_adjust_blending_scales_with_anisotropy():
    M = np.diag([1.0, 1.0, 2.5]) @ synth.translation((1, 2, 3))
    border, rng = fo.adjust_blending(M)
    assert np.allclose(rng, [40, 40, 16]) and np.all(border == 0)


def test_invert_affine_roundtrip():
    M = (np.vstack([synth.rot_z(12.0, (5, 6, 7)), [0, 0, 0, 1]]) @ np.vstack([synth.translation((3, -4, 5)), [0, 0, 0, 1]]))[:3]
    I = np.vstack([fo.invert_affine(M), [0, 0, 0, 1]]) @ np.vstack([M, [0, 0, 0, 1]])
    assert np.allclose(I, np.eye(4), atol=1e-12)


def test_content_weights_of_constant_are_zero_and_positive_on_texture():
    c = fo.content_weights(np.full((12, 12, 12), 300, np.uint16), 1.0, 2.0)
    assert np.abs(c).max() < 1e-3
    vol = synth.tile_from(synth.field((16, 16, 16), seed=5), (0, 0, 0), (16, 16, 16), 5)
    assert fo.content_weights(vol, 1.0, 2.0).min() > 0


def test_golden_fusion_block():
    from tests.golden import make_golden
    want = np.load(GOLDEN)["avg_blend"]
    got = make_golden.fusion_case()
    assert np.array_equal(got, want)


def test_downsample_known_answers():
    v = np.arange(2 * 2 * 4, dtype=np.float32).reshape(2, 2, 4)
    assert np.array_equal(fo.downsample2x(v, (2, 1, 1)), [[[0.5, 2.5], [4.5, 6.5]], [[8.5, 10.5], [12.5, 14.5]]])
    assert fo.downsample2x(v, (2, 2, 2)).shape == (1, 1, 2) and fo.downsample2x(v, (2, 2, 2))[0, 0, 0] == 6.5
    u = np.array([[[1, 2, 3, 4, 9]]], dtype=np.uint16)
    assert list(fo.downsample2x(u, (2, 1, 1)).ravel()) == [2, 4]    # (1+2+1)>>1, (3+4+1)>>1, odd tail dropped


def test_c_restatement_matches_numpy_oracle():
    """oracle/c/fusion_oracle.c (the CPU-baseline arm) against the numpy oracle on a jittered 3-view scene."""
    from oracle import c_fusion
    G = synth.field((30, 44, 120), seed=4, sigma=1.5)
    views = []
    for i, t in enumerate([(0.3, 0.1, -0.2), (31.7, 1.4, 2.1), (64.2, -2.2, 0.6)]):
        vol = synth.tile_from(G, (2, 3, int(t[0]) + 4), (24, 36, 44), 20 + i, noise=5.0)
        M = synth.translation(t)
        border, rng = fo.adjust_blending(M)
        views.append(fo.View(vol, M, border, rng))
    for ft in (fo.AVG, fo.AVG_BLEND):
        want = fo.fuse_block(views, (-2, -1, -1), (112, 40, 28), ft)
        got = c_fusion.fuse_block(views, (-2, -1, -1), (112, 40, 28), ft)
        assert np.allclose(got, want, rtol=2e-6, atol=1e-4)
        assert np.array_equal(got == 0, want == 0)
    assert c_fusion.num_threads() >= 1


def test_mask_block_semantics():
    """--masks: closed interval [0 - off, dim - 1 + off] on every axis of any view; 255 / 65535 / 1.0."""
    M0 = synth.translation((2.0, 0.0, 0.0))
    M1 = synth.translation((30.5, 3.0, 1.0))
    geom = [(M0, (20, 10, 6)), (M1, (10, 10, 6))]
    m = fo.mask_block(geom, (0, 0, 0), (48, 16, 8), (0.0, 0.0, 0.0), "uint8")
    assert m.dtype == np.uint8 and set(np.unique(m)) == {0, 255}
    assert m[0, 0, 2] == 255 and m[0, 0, 1] == 0 and m[0, 0, 21] == 255 and m[0, 0, 22] == 0      # view 0: x in [2, 21]
    assert m[1, 3, 31] == 255 and m[1, 3, 30] == 0 and m[1, 3, 39] == 255 and m[1, 3, 40] == 0     # view 1: x in [30.5, 39.5]
    assert m[0, 3, 31] == 0 and m[7, 3, 31] == 0                                                   # z in [1, 6]
    g = fo.mask_block(geom, (0, 0, 0), (48, 16, 8), (1.0, 0.0, 0.5), "uint16")
    assert g.dtype == np.uint16 and g[0, 0, 1] == 65535 and g[0, 0, 0] == 0 and g[0, 0, 22] == 65535
    assert g[0, 3, 31] == 0 and g[1, 3, 30] == 65535                                               # z grows by 0.5 only
    f = fo.mask_block(geom, (0, 0, 0), (48, 16, 8), (0.0, 0.0, 0.0), "float32")
    assert f.dtype == np.float32 and np.array_equal(f > 0, m > 0) and f.max() == 1.0
    assert not fo.mask_block([], (0, 0, 0), (4, 4, 4)).any()


def test_content_weights_reference_agrees_with_the_float32_oracle():
    """The float64 content weights equal the float32 pipeline within the rounding of its stored intermediates, also on
    axes of length 1 (mirror-single of a single sample is that sample) and on float32 input with negative values."""
    rng = np.random.default_rng(0)
    u = 2.0 ** -24
    for shape in [(12, 14, 16), (1, 14, 16), (12, 1, 16), (12, 14, 1), (9, 7, 33)]:
        vol = (rng.normal(0, 50, shape) + 20).astype(np.float32)
        for s1, s2 in ((2.0, 4.0), (1.0, 2.0)):
            c, f, g1, d = fo.content_weights_reference(vol, s1, s2)
            assert np.array_equal(f, vol.astype(np.float64))
            bar = u * (c + fo._gauss3_f64(2 * np.abs(d) * (np.abs(f) + 2 * np.abs(g1)), fo.gauss_kernel(s2)))
            assert np.all(np.abs(fo.content_weights(vol, s1, s2) - c) <= 2 * bar), (shape, s1, s2)
    # a single sample along x: the blur along x is the identity
    line = rng.normal(0, 5, (6, 7, 1)).astype(np.float32)
    assert np.allclose(fo._gauss3_f64(line, fo.gauss_kernel(3.0)), fo._gauss3_f64(line[:, :, 0:1], fo.gauss_kernel(3.0)))
