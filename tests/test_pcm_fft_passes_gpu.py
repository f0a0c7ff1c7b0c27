"""GPU: every FFT pass of the PCM pipeline, and every kernel instantiation its dispatcher can choose, against the
float64 reference of that pass (oracle/pcm_passes.py).

bs_pcm_debug_pass runs one pass with exactly the launch bs_pcm_* uses and reports the instantiation it chose; each
case below sets the BS_FFT_* switches, asserts that instantiation, and compares the output line by line:

  * linear passes (0, 1, 3, 4) and ordinary cross-power lines: the worst line's relative L2 error against float64 must
    be within BAR times the worst-line error of scipy's single-precision FFT on the same input;
  * cross-power lines built around the 1e-5 threshold, and all-zero / 1e-30 lines: the exact outcome (unit or 0);
  * lines whose reference is identically zero: bit-exact 0, with the device spectra poisoned with NaN beforehand;
  * no NaN anywhere.
"""
import re

import numpy as np
import pytest

from oracle import pcm_oracle as po
from oracle import pcm_passes as pp
from tests import synth
from tests.pcm_switches import set_switches

pytestmark = pytest.mark.gpu

#: allowed worst-line error, in multiples of scipy's single-precision worst-line error (floored at one float32 ulp,
#: so that a length scipy happens to transform exactly does not make the bar 0)
BAR = 8.0
ULP32 = 2.0 ** -24
RADICES = {16, 15, 12, 10, 9, 8, 6, 5, 4, 3, 2}
#: generic (runtime-planned) kernel families whose plans must, together, use every radix of the planner
FAMILIES = {
    "warp-x": ("k_fft_x_r2c_w<FftWGeneric>", "k_fft_x_c2r_w<FftWGeneric>"),
    "cta-x": ("k_fft_x_r2c", "k_fft_x_r2c_tma", "k_fft_x_c2r"),
    "strided-pipe": ("k_fft_strided_pipe",),
    "strided": ("k_fft_strided",),
}
#: k_fft_strided only runs y lengths whose pipelined tiles do not fit shared memory (1161..1709 and 2236..3228 with
#: the default tiles, 594..880 with 16-column tiles, 4151..5811); no 5-smooth length there has a radix-8 plan
UNREACHABLE = {"strided": {8}}
_DT = {"u16": (np.uint16, 0), "f32": (np.float32, 1), "u8": (np.uint8, 2)}


def crop_for(P, even=False):
    """Largest crop size whose padded size (extension 10) is P."""
    for d in range(P, 0, -1):
        if po.good_fft_size(po.extended_size(d, 10), even) == P:
            return d
    raise ValueError(P)


def case(pass_no, dims, kernel, dtype="u16", env=None, misalign=0, tag=""):
    env = env or {}
    name = f"p{pass_no}-{kernel}-{dtype}-{'x'.join(map(str, dims))}" + "".join(f"-{k[7:]}{v}" for k, v in env.items())
    return pytest.param(pass_no, tuple(dims), kernel, dtype, env, misalign, id=name + tag)


# M (= Px / 2) or padded y lengths whose plans together use every radix: 180 15x12, 40 10x4, 96 16x6, 27 9x3,
# 120 15x8, 80 5x16, 32 16x2
GEN = (180, 40, 96, 27, 120, 80, 32)
STATIC0 = {"BS_FFT_STATIC": 0}
CTA = {"BS_FFT_X_WARP": 0}
CTA_NOTMA = {"BS_FFT_X_WARP": 0, "BS_FFT_R2C_TMA": 0}
# edge geometries: (10, 13, 4): M = 15 (pitch tail 0), Ey = 33 < Py = 36, dz < extension; (12, 1, 13): M = 16 (pitch
# tail 15), dy = 1, Ez < Pz; (1, 4, 1): every axis below the extension, d = 1
EDGES = ((10, 13, 4), (12, 1, 13), (1, 4, 1))

CASES = [
    # ---- pass 0: x r2c
    case(0, (520, 6, 3), "k_fft_x_r2c_w<FftW270S> tma"),
    case(0, (519, 6, 3), "k_fft_x_r2c_w<FftW270S>"),
    case(0, (520, 6, 3), "k_fft_x_r2c_w<FftW270S>", misalign=1, tag="-misaligned"),
    case(0, (520, 6, 3), "k_fft_x_r2c_w<FftW270S> tma", dtype="f32"),
    case(0, (512, 6, 3), "k_fft_x_r2c_w<FftW270S> tma", dtype="u8"),
    case(0, (520, 6, 3), "k_fft_x_r2c_w<FftW270S>", dtype="u8"),
    case(0, (520, 6, 3), "k_fft_x_r2c_w<FftWGeneric> tma", env=STATIC0),
    *[case(0, (crop_for(2 * m, True), 5, 2), "k_fft_x_r2c_w<FftWGeneric>") for m in GEN],
    case(0, (crop_for(2 * 180, True), 5, 2), "k_fft_x_r2c", env=CTA, misalign=1, tag="-misaligned"),
    *[case(0, (crop_for(2 * m, True), 5, 2), "k_fft_x_r2c", env=CTA_NOTMA) for m in GEN],
    case(0, (340, 5, 2), "k_fft_x_r2c_tma", dtype="f32", env=CTA),
    case(0, (784, 7, 2), "k_fft_x_r2c_tma"),                 # M = 405 > 319: CTA kernels by default
    case(0, (790, 7, 2), "k_fft_x_r2c"),                     # ... without TMA (row of 1580 B)
    case(0, (790, 7, 2), "k_fft_x_r2c", dtype="f32"),
    case(0, (4000, 3, 1), "k_fft_x_r2c"),                    # M = 2025: 4 lines per CTA
    case(0, (4000, 3, 1), "k_fft_x_r2c_tma", dtype="u8"),    # ... and its staged rows still fit
    *[case(0, d, "k_fft_x_r2c_w<FftWGeneric>") for d in EDGES],
    *[case(0, d, "k_fft_x_r2c", env=CTA_NOTMA) for d in EDGES],
    # ---- pass 1: y forward of both spectra
    case(1, (12, 520, 3), "k_fft_col540"),
    case(1, (520, 520, 2), "k_fft_col540"),
    case(1, (12, 520, 3), "k_fft_strided_pipe", env=STATIC0),
    *[case(1, (10, crop_for(p), 2), "k_fft_strided_pipe") for p in GEN],
    # k_fft_strided: Py = 1200 (15x5x16), 1458 (9x9x9x2), 1620 (15x9x12), 1440 (15x16x6), 2400 (15x16x10, 4-column
    # tiles); with 16-column tiles Py = 600 (15x10x4) and 675 (15x15x3)
    case(1, (12, 1180, 1), "k_fft_strided"),
    *[case(1, (10, crop_for(p), 1), "k_fft_strided") for p in (1458, 1620, 1440, 2400)],
    *[case(1, (10, crop_for(p), 1), "k_fft_strided", env={"BS_FFT_YTILE_LOG2": 4}) for p in (600, 675)],
    *[case(1, d, "k_fft_strided_pipe") for d in EDGES],
    # ---- pass 2: z cross-power
    case(2, (12, 6, 520), "k_fft_xpower_col540"),
    case(2, (10, 13, 520), "k_fft_xpower_col540"),
    case(2, (12, 6, 520), "k_fft_xpower_pipe", env=STATIC0),
    case(2, (12, 5, 44), "k_fft_xpower_pipe"),
    case(2, (12, 5, 25), "k_fft_xpower_pipe", env={"BS_FFT_ZTILE_LOG2": 2}),
    *[case(2, d, "k_fft_xpower_pipe") for d in EDGES],
    # ---- pass 3: y forward of the product
    case(3, (12, 520, 3), "k_fft_col540"),
    case(3, (12, 520, 3), "k_fft_strided_pipe", env=STATIC0),
    case(3, (10, 25, 3), "k_fft_strided_pipe"),
    case(3, (12, 1180, 1), "k_fft_strided"),
    case(3, (10, crop_for(600), 1), "k_fft_strided", env={"BS_FFT_YTILE_LOG2": 4}),
    *[case(3, d, "k_fft_strided_pipe") for d in EDGES],
    # ---- pass 4: x c2r
    case(4, (520, 6, 3), "k_fft_x_c2r_w<FftW270>"),
    case(4, (520, 6, 3), "k_fft_x_c2r_w<FftWGeneric>", env=STATIC0),
    *[case(4, (crop_for(2 * m, True), 5, 2), "k_fft_x_c2r_w<FftWGeneric>") for m in GEN],
    *[case(4, (crop_for(2 * m, True), 5, 2), "k_fft_x_c2r", env=CTA) for m in GEN],
    case(4, (790, 7, 2), "k_fft_x_c2r"),
    case(4, (4000, 3, 1), "k_fft_x_c2r"),
    *[case(4, d, "k_fft_x_c2r_w<FftWGeneric>") for d in EDGES],
    *[case(4, d, "k_fft_x_c2r", env=CTA) for d in EDGES],
]


def _kernel(info):
    """The info string without the plan radices."""
    return re.sub(r" \d+(x\d+)*$", "", info)


def _radices(info):
    m = re.search(r" (\d+(?:x\d+)*)$", info)
    return {int(r) for r in m.group(1).split("x")} if m else set()


def _geometry(dims):
    P = po.padded_dims(dims, (10, 10, 10))
    return P, P[0] // 2


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


def _random_spectrum(rng, shape, zero_lines_axis):
    """Random complex64 spectrum; about 10 % of the lines along ``zero_lines_axis`` are all zero."""
    s = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)
    lines = np.moveaxis(s, zero_lines_axis, -1)
    lines[rng.random(lines.shape[:-1]) < 0.1] = 0
    return s


# z lines of the cross-power pass, by kind (A and B are built in float64 from their z spectra)
ORDINARY, A_ABOVE, A_BELOW, B_ABOVE, B_BELOW, BOTH_ZERO, A_TINY, A_HUGE, B_HUGE, A_AT = range(10)
UNIT = (A_ABOVE, B_ABOVE, A_AT)
ZERO = (A_BELOW, B_BELOW, BOTH_ZERO, A_TINY)
MEASURED = (ORDINARY, A_HUGE, B_HUGE)


def _z_lines(P, M, seed):
    """Inputs of pass 2 whose z transforms have known bins: ordinary lines (every bin within one decade of a line
    scale between 1e-2 and 1e4), single-bin lines with |bin| = 1e-5 (1 +- 1e-3) against an ordinary single bin,
    all-zero lines, lines with every bin near 1e-30 or 1e20, and lines whose bin 0 is exactly the float32 threshold
    (a delta at z = 0 of value 1e-5f: its transform is exact at bin 0, and |c| == threshold keeps the bin)."""
    rng = np.random.default_rng(seed)
    Pz, n = P[2], P[1] * (M + 1)
    kind = rng.permutation(np.arange(n) % 10)
    FA = np.zeros((Pz, n), np.complex128)
    FB = np.zeros((Pz, n), np.complex128)

    def ordinary(scale):
        return scale * 10 ** rng.uniform(-0.5, 0.5, Pz) * np.exp(2j * np.pi * rng.random(Pz))

    def single(mag):
        v = np.zeros(Pz, np.complex128)
        v[k0] = mag * np.exp(2j * np.pi * rng.random())
        return v

    for j in range(n):
        k0 = int(rng.integers(Pz))
        kj = kind[j]
        if kj == ORDINARY:
            FA[:, j], FB[:, j] = ordinary(10 ** rng.uniform(-1.5, 3.5)), ordinary(10 ** rng.uniform(-1.5, 3.5))
        elif kj in (A_ABOVE, A_BELOW):
            FA[:, j] = single(1e-5 * (1 + 1e-3 if kj == A_ABOVE else 1 - 1e-3))
            FB[:, j] = single(rng.uniform(1, 10))
        elif kj in (B_ABOVE, B_BELOW):
            FA[:, j] = single(rng.uniform(1, 10))
            FB[:, j] = single(1e-5 * (1 + 1e-3 if kj == B_ABOVE else 1 - 1e-3))
        elif kj == A_TINY:
            FA[:, j], FB[:, j] = ordinary(1e-30), ordinary(1.0)
        elif kj == A_HUGE:
            FA[:, j], FB[:, j] = ordinary(1e20), ordinary(1.0)
        elif kj == B_HUGE:
            FA[:, j], FB[:, j] = ordinary(1.0), ordinary(1e20)
        elif kj == A_AT:
            k0 = 0
            FB[:, j] = single(rng.uniform(1, 2))
    shape = (Pz, P[1], M + 1)
    a = np.fft.ifft(FA, axis=0)
    a[0, kind == A_AT] = np.float32(po.NORMALIZATION_THRESHOLD)
    a = a.astype(np.complex64).reshape(shape)
    b = np.fft.ifft(FB, axis=0).astype(np.complex64).reshape(shape)
    return a, b, kind.reshape(P[1], M + 1)


def _check_linear(got, ref, f32, axis, what):
    """Worst-line relative L2 within BAR x scipy's; lines with an all-zero reference exactly 0."""
    err, live = pp.line_rel_l2(got, ref, axis)
    err32, _ = pp.line_rel_l2(f32, ref, axis)
    bar = BAR * max(err32[live].max(), ULP32)
    worst = np.unravel_index(np.argmax(err), err.shape)
    assert err.max() <= bar, f"{what}: worst line {worst} rel L2 {err.max():.3g}, scipy float32 {err32.max():.3g}"
    dead = np.moveaxis(got, axis, -1)[~live]
    assert np.all(dead == 0), f"{what}: {int(np.sum(np.any(dead != 0, axis=-1)))} zero-padding lines are not 0"


@pytest.mark.parametrize("pass_no,dims,kernel,dtype,env,misalign", CASES)
def test_fft_pass(ctx, monkeypatch, pass_no, dims, kernel, dtype, env, misalign):
    set_switches(monkeypatch, env)
    P, M = _geometry(dims)
    seed = sum(dims) * 7 + pass_no
    rng = np.random.default_rng(seed)
    if pass_no == 0:
        a, b = _crops(dims, dtype, seed)
        (ta, pa), (tb, pb) = _device(a, misalign), _device(b, misalign)
        out_a, out_b, info = ctx.pcm_debug_pass(0, dims, pa, pb, dtype=_DT[dtype][1])
        del ta, tb
    elif pass_no == 1:
        a, b = (_random_spectrum(rng, (P[2], P[1], M + 1), 1) for _ in range(2))
        out_a, out_b, info = ctx.pcm_debug_pass(1, dims, a, b)
    elif pass_no == 2:
        a, b, kind = _z_lines(P, M, seed)
        out_a, out_b, info = ctx.pcm_debug_pass(2, dims, a, b)
    elif pass_no == 3:
        a = _random_spectrum(rng, (P[2], P[1], M + 1), 1)
        out_a, out_b, info = ctx.pcm_debug_pass(3, dims, a)
    else:
        a = _random_spectrum(rng, (P[2], P[1], M + 1), 2)
        a[..., 0] = a[..., 0].real            # a C2R input: bins 0 and M of each line are real
        a[..., M] = a[..., M].real
        out_a, out_b, info = ctx.pcm_debug_pass(4, dims, a)
    assert _kernel(info) == kernel, info
    assert np.isfinite(out_a).all() and (out_b is None or np.isfinite(out_b).all()), info

    if pass_no == 0:
        _check_linear(out_a, pp.pass0(a), pp.pass0_f32(a), 2, info + " (A)")
        _check_linear(out_b, pp.pass0(b), pp.pass0_f32(b), 2, info + " (B)")
    elif pass_no == 1:
        _check_linear(out_a, pp.pass1(a), pp.pass1_f32(a), 1, info + " (A)")
        _check_linear(out_b, pp.pass1(b), pp.pass1_f32(b), 1, info + " (B)")
    elif pass_no == 3:
        _check_linear(out_a, pp.pass3(a), pp.pass3_f32(a), 1, info)
    elif pass_no == 4:
        _check_linear(out_a, pp.pass4(a, P[0]), pp.pass4_f32(a, P[0]), 2, info)
    else:
        ref, f32 = pp.pass2(a, b), pp.pass2_f32(a, b)
        err, _ = pp.line_rel_l2(out_a, ref, 0)
        err32, _ = pp.line_rel_l2(f32, ref, 0)
        meas = np.isin(kind, MEASURED)
        bar = BAR * max(err32[meas].max(), ULP32)
        for k in MEASURED:
            sel = kind == k
            if sel.any():
                assert err[sel].max() <= bar, f"{info}: kind {k} worst rel L2 {err[sel].max():.3g}, bar {bar:.3g}"
        for k in UNIT:
            sel = kind == k
            if sel.any():
                assert np.abs(np.abs(out_a[:, sel]) - 1).max() < 1e-4, f"{info}: kind {k} is not unit"
                assert err[sel].max() < 1e-4, f"{info}: kind {k} worst rel L2 {err[sel].max():.3g}"
        assert np.all(out_a[:, np.isin(kind, ZERO)] == 0), info


def test_generic_plans_cover_every_radix(ctx, monkeypatch):
    """For each runtime-planned kernel family, the plans the cases above run use every radix of the planner."""
    seen = {f: set() for f in FAMILIES}
    for p in CASES:
        pass_no, dims, kernel, dtype, env, misalign = p.values
        fam = [f for f, ks in FAMILIES.items() if kernel in ks]
        if not fam:
            continue
        set_switches(monkeypatch, env)
        P, M = _geometry(dims)
        if pass_no == 0:
            a, b = _crops(dims, dtype, 1)
            (ta, pa), (tb, pb) = _device(a, misalign), _device(b, misalign)
            info = ctx.pcm_debug_pass(0, dims, pa, pb, dtype=_DT[dtype][1])[2]
            del ta, tb
        else:
            z = np.zeros((P[2], P[1], M + 1), np.complex64)
            info = ctx.pcm_debug_pass(pass_no, dims, z, z)[2]
        assert _kernel(info) == kernel, info
        seen[fam[0]] |= _radices(info)
    for f, r in seen.items():
        assert r == RADICES - UNREACHABLE.get(f, set()), (f, sorted(RADICES - r))


def test_debug_pass_rejects_bad_arguments(ctx):
    import bsgpu
    z = np.zeros((3, 12, 17), np.complex64)
    with pytest.raises(bsgpu.BsError):
        ctx.pcm_debug_pass(5, (12, 4, 1), z, z)
    with pytest.raises(ValueError):
        ctx.pcm_debug_pass(1, (12, 4, 1), z[:, :5], z)
