"""GPU: the two-for-one x passes of the 540-point plan (k_fft_x_r2c_col540, k_fft_x_c2r_col540) against the float64
reference of each pass (oracle/pcm_passes.py), and the dispatch rule that chooses them.

BS_FFT_X_COL540=2 forces the Col540 x kernels wherever the geometry allows, so small volumes reach them; the bar is
the one of test_pcm_fft_passes_gpu.py: worst-line relative L2 within BAR x scipy float32's, bit-exact zeros on lines
whose reference is zero (device spectra poisoned with NaN beforehand), no NaN.
"""
import numpy as np
import pytest

from oracle import pcm_oracle as po
from oracle import pcm_passes as pp
from tests import synth

pytestmark = pytest.mark.gpu

ENV = ("BS_FFT_X_COL540", "BS_FFT_X_WARP", "BS_FFT_R2C_TMA", "BS_FFT_R2C_LINES_LOG2", "BS_FFT_XLINES_LOG2",
       "BS_FFT_STATIC")
BAR = 8.0
ULP32 = 2.0 ** -24
_DT = {"u16": (np.uint16, 0), "f32": (np.float32, 1), "u8": (np.uint8, 2)}
R2C, C2R = "k_fft_x_r2c_col540", "k_fft_x_c2r_col540"
FORCE = {"BS_FFT_X_COL540": 2}


def _set_env(monkeypatch, env):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def _crops(dims, dtype, seed):
    np_dt, _ = _DT[dtype]
    shape = dims[::-1]
    if np_dt == np.uint8:
        a, b = (synth.field(shape, seed=seed + i, mean=120.0, std=40.0) for i in range(2))
    else:
        a, b = (synth.field(shape, seed=seed + i) for i in range(2))
    if np_dt != np.float32:
        a, b = (np.clip(np.rint(v), 0, np.iinfo(np_dt).max).astype(np_dt) for v in (a, b))
    return a, b


def _device(arr, misalign):
    """A device copy of ``arr`` whose base address is ``misalign`` elements past a 256-byte aligned allocation."""
    import torch
    flat = arr.ravel()
    view = flat.view(np.int16) if flat.dtype == np.uint16 else flat
    t = torch.zeros(flat.size + 16, dtype=torch.from_numpy(view[:1].copy()).dtype, device="cuda")
    t[misalign:misalign + flat.size] = torch.from_numpy(view.copy()).cuda()
    torch.cuda.synchronize()
    return t, t.data_ptr() + misalign * flat.itemsize


def _check_linear(got, ref, f32, axis, what):
    err, live = pp.line_rel_l2(got, ref, axis)
    err32, _ = pp.line_rel_l2(f32, ref, axis)
    bar = BAR * max(err32[live].max(), ULP32)
    worst = np.unravel_index(np.argmax(err), err.shape)
    assert err.max() <= bar, f"{what}: worst line {worst} rel L2 {err.max():.3g}, scipy float32 {err32.max():.3g}"
    dead = np.moveaxis(got, axis, -1)[~live]
    assert np.all(dead == 0), f"{what}: {int(np.sum(np.any(dead != 0, axis=-1)))} zero-reference lines are not 0"


def _pass0(ctx, dims, dtype="u16", misalign=0, seed=None, blank=None):
    """Run pass 0 on two seeded crops; ``blank`` = (image, z, y) rows of one crop set to 0.  Returns (a, b, A, B, info)."""
    a, b = _crops(dims, dtype, sum(dims) if seed is None else seed)
    for im, z, y in blank or ():
        (a, b)[im][z, y, :] = 0
    (ta, pa), (tb, pb) = _device(a, misalign), _device(b, misalign)
    out_a, out_b, info = ctx.pcm_debug_pass(0, dims, pa, pb, dtype=_DT[dtype][1])
    del ta, tb
    return a, b, out_a, out_b, info


def _spectrum(dims, seed):
    """Random pass-4 input, [Pz, Py, M+1]: about 10 % of the x lines all zero, bins 0 and M real (a C2R input)."""
    P = po.padded_dims(dims, (10, 10, 10))
    M = P[0] // 2
    rng = np.random.default_rng(seed)
    s = (rng.standard_normal((P[2], P[1], M + 1)) + 1j * rng.standard_normal((P[2], P[1], M + 1))).astype(np.complex64)
    s[rng.random((P[2], P[1])) < 0.1] = 0
    s[..., 0] = s[..., 0].real
    s[..., M] = s[..., M].real
    return s, P


# (512, 100, 60): Py x Pz = 120 x 80 -> 600 r2c / 300 c2r tiles (several per SM, not a multiple of the SM count),
#   and Py = 120 is not a multiple of 16, so tiles straddle z-planes
# (520, 13, 7): dy, dz below the extension (mirrored borders), Ey = 39 < Py = 40 and Ez = 21 < Pz = 24: zero lines
#   inside tiles and whole zero planes
# (520, 25, 5): Py x Pz = 45 x 15 = 675 lines, odd: the last c2r tile ends on half a pair
GEOMS = ((512, 100, 60), (520, 13, 7), (520, 25, 5))


@pytest.mark.parametrize("dims", GEOMS)
def test_r2c_col540(ctx, monkeypatch, dims):
    _set_env(monkeypatch, FORCE)
    a, b, out_a, out_b, info = _pass0(ctx, dims)
    assert info == R2C, info
    assert np.isfinite(out_a).all() and np.isfinite(out_b).all()
    _check_linear(out_a, pp.pass0(a), pp.pass0_f32(a), 2, info + " (A)")
    _check_linear(out_b, pp.pass0(b), pp.pass0_f32(b), 2, info + " (B)")


def test_r2c_col540_blank_rows_stay_zero(ctx, monkeypatch):
    """A row that is zero in one crop only: its spectrum is exactly 0, not the partner row's rounding noise."""
    _set_env(monkeypatch, FORCE)
    dims = (520, 13, 7)
    a, b, out_a, out_b, info = _pass0(ctx, dims, blank=((0, 3, 5), (1, 4, 9), (0, 0, 0)))
    assert info == R2C, info
    _check_linear(out_a, pp.pass0(a), pp.pass0_f32(a), 2, info + " (A)")
    _check_linear(out_b, pp.pass0(b), pp.pass0_f32(b), 2, info + " (B)")


@pytest.mark.parametrize("dims", GEOMS)
def test_c2r_col540(ctx, monkeypatch, dims):
    _set_env(monkeypatch, FORCE)
    s, P = _spectrum(dims, sum(dims) + 4)
    out, _, info = ctx.pcm_debug_pass(4, dims, s)
    assert info == C2R, info
    assert np.isfinite(out).all()
    _check_linear(out, pp.pass4(s, P[0]), pp.pass4_f32(s, P[0]), 2, info)


@pytest.mark.parametrize("dims,dtype,misalign,kernel", [
    ((520, 6, 3), "u16", 1, "k_fft_x_r2c_w<FftW270S>"),
    ((512, 6, 3), "u8", 0, "k_fft_x_r2c_w<FftW270S> tma"),
    ((520, 6, 3), "f32", 0, "k_fft_x_r2c_w<FftW270S> tma"),
    ((519, 6, 3), "u16", 0, "k_fft_x_r2c_w<FftW270S>"),   # rows of 1038 bytes
], ids=["misaligned", "u8", "f32", "odd-row"])
def test_r2c_falls_back(ctx, monkeypatch, dims, dtype, misalign, kernel):
    """Crops the staged-row kernel does not take keep today's kernel even when the Col540 kernels are forced."""
    _set_env(monkeypatch, FORCE)
    a, b, out_a, out_b, info = _pass0(ctx, dims, dtype, misalign)
    assert info == kernel, info
    _check_linear(out_a, pp.pass0(a), pp.pass0_f32(a), 2, info + " (A)")


def test_default_rule_by_tile_count(ctx, monkeypatch):
    """Default switch: fewer tiles than SMs keep the warp kernels, enough tiles take the Col540 kernels; 0 never."""
    small, large = (520, 6, 3), (512, 100, 60)
    warp_r2c = "k_fft_x_r2c_w<FftW270S> tma"
    for env, dims, r2c, c2r in (({}, small, warp_r2c, "k_fft_x_c2r_w<FftW270>"),
                                ({}, large, R2C, C2R),
                                ({"BS_FFT_X_COL540": 0}, large, warp_r2c, "k_fft_x_c2r_w<FftW270>")):
        _set_env(monkeypatch, env)
        assert _pass0(ctx, dims)[4] == r2c, (env, dims)
        s, _ = _spectrum(dims, 1)
        assert ctx.pcm_debug_pass(4, dims, s)[2] == c2r, (env, dims)


def test_col540_runs_are_bit_identical(ctx, monkeypatch):
    _set_env(monkeypatch, FORCE)
    dims = (512, 100, 60)
    first = _pass0(ctx, dims, seed=3)
    again = _pass0(ctx, dims, seed=3)
    assert first[4] == again[4] == R2C
    assert np.array_equal(first[2], again[2]) and np.array_equal(first[3], again[3])
    s, _ = _spectrum(dims, 3)
    o1, _, i1 = ctx.pcm_debug_pass(4, dims, s)
    o2, _, i2 = ctx.pcm_debug_pass(4, dims, s)
    assert i1 == i2 == C2R and np.array_equal(o1, o2)


@pytest.mark.parametrize("env", [{}, FORCE], ids=["default", "forced"])
def test_pipeline_pair_on_col540(ctx, monkeypatch, env):
    """A whole pair at a geometry where the default switch picks both Col540 kernels, against the oracle."""
    _set_env(monkeypatch, env)
    shape = (60, 60, 504)   # (z, y, x): padded 80 x 80 x 540, rows of 1008 bytes
    a, b = synth.shifted_pair(shape, (6, -4, 3), seed=91, margin=16)
    dims = shape[::-1]
    assert _pass0(ctx, dims)[4] == R2C
    assert ctx.pcm_debug_pass(4, dims, _spectrum(dims, 2)[0])[2] == C2R
    o = po.pcm_shift(a, b)
    g = ctx.pcm_pair(a, b)
    assert g.pad == o.pad and g.pad[0] == 540
    assert g.found and o.found
    assert g.shift_int == o.shift_int and g.peak_index == o.peak_index
    assert g.n_overlap_px == o.n_overlap_px and abs(g.r - o.r) < 1e-9
    assert np.allclose(g.shift_sub, o.shift_sub, atol=1e-3), (g.shift_sub, o.shift_sub)
