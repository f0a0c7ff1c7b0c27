"""GPU: the forward x transforms of the 540-point plan (k_fft_x_r2c_col540, and the x role of the fused
k_fft_xy_col540) at crop widths that move the range of row positions they read without the blending table.

With the extension 10, positions 27..512 of a padded x line lie inside the crop for dx >= 503: there a line of y and
z weight 1 takes the samples straight from its row.  dx = 496 keeps every position on the table, dx = 504 leaves a
single crop sample past position 512, and dx = 520 has no zero tail; all pad to 540.  Pass 0 is held to the float64
reference of test_pcm_xpass_col540_gpu.py, and debug pass 5 (fused) to pass 0 followed by pass 1 bit for bit, also
with the hand-off window at 2 and 3 planes over many more planes than that, and with all-zero rows in the crops'
interior and in their y and z border lines.
"""
import numpy as np
import pytest

from oracle import pcm_passes as pp
from tests import synth
from tests.pcm_switches import set_switches

pytestmark = pytest.mark.gpu

BAR = 8.0
ULP32 = 2.0 ** -24
XY = "k_fft_xy_col540"


def _crops(dims, seed, blank=()):
    """Two seeded uint16 crops [z, y, x]; ``blank`` = (image, z, y) rows set to 0."""
    shape = dims[::-1]
    out = [np.clip(np.rint(synth.field(shape, seed=seed + i)), 0, 65535).astype(np.uint16) for i in range(2)]
    for im, z, y in blank:
        out[im][z, y, :] = 0
    return out


def _device(a):
    import torch
    t = torch.from_numpy(a.view(np.int16)).cuda()
    torch.cuda.synchronize()
    return t


def _same_bits(x, y):
    return x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))


def _check_pass0(got, a):
    err, live = pp.line_rel_l2(got, pp.pass0(a), 2)
    err32, _ = pp.line_rel_l2(pp.pass0_f32(a), pp.pass0(a), 2)
    assert err.max() <= BAR * max(err32[live].max(), ULP32), (err.max(), err32.max())
    assert np.all(np.moveaxis(got, 2, -1)[~live] == 0)


# rows of zeros: interior line (z 20, y 200), y border line (y 3), z border line (z 1), and one in both borders
BLANK = ((0, 20, 200), (1, 20, 201), (0, 5, 3), (1, 1, 300), (0, 0, 511), (1, 60, 0))


@pytest.mark.parametrize("dx", [496, 504, 520])
def test_x_pass_matches_reference(ctx, monkeypatch, dx):
    dims = (dx, 30, 7)
    a, b = _crops(dims, dx, blank=((0, 3, 5), (1, 0, 29), (0, 6, 12)))
    set_switches(monkeypatch, {"BS_FFT_X_COL540": 2})
    out_a, out_b, info = ctx.pcm_debug_pass(0, dims, _device(a), _device(b))
    assert info == "k_fft_x_r2c_col540", info
    _check_pass0(out_a, a)
    _check_pass0(out_b, b)


@pytest.mark.parametrize("dx,dz,env,blank", [
    (504, 61, {}, ()),
    (520, 61, {}, ()),
    (496, 9, {}, ()),
    (504, 61, {"BS_FFT_XY_WINDOW": 2}, ()),
    (520, 45, {"BS_FFT_XY_WINDOW": 3}, ()),
    (512, 61, {"BS_FFT_XY_WINDOW": 2, "BS_FFT_XY_KX": 100}, BLANK),
    (504, 61, {}, BLANK),
])
def test_fused_matches_two_passes(ctx, monkeypatch, dx, dz, env, blank):
    dims = (dx, 512, dz)
    a, b = _crops(dims, 7 * dx + dz, blank)
    ta, tb = _device(a), _device(b)
    set_switches(monkeypatch, env)
    fa, fb, info = ctx.pcm_debug_pass(5, dims, ta, tb)
    assert info == XY, info
    set_switches(monkeypatch, {"BS_FFT_XY_FUSE": 0})
    xa, xb, _ = ctx.pcm_debug_pass(0, dims, ta, tb)
    ya, yb, _ = ctx.pcm_debug_pass(1, dims, xa, xb)
    for got, ref in ((fa, ya), (fb, yb)):
        assert not np.isnan(got).any()
        assert _same_bits(got, ref), f"{np.count_nonzero(got != ref)} bins differ"
