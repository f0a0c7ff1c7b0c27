"""GPU parity tests, hot path 1: libbsgpu (through the C ABI) against oracle/pcm_oracle.py.

Bars (BASELINE.json north_star): integer peak / shift bit-identical; sub-pixel within 1e-3 px;
Pearson r (exact integer sums on the device) within 1e-9.  PCM volumes: relative L2 error against the float64
PCM (oracle/pcm_passes.py) within PCM_BAR times the float32 oracle's own error on the same pair.
"""
import numpy as np
import pytest

from oracle import pcm_oracle as po
from oracle import pcm_passes as pp
from tests import synth

pytestmark = pytest.mark.gpu

#: allowed relative L2 error of the device PCM, in multiples of the float32 oracle's error (about 1e-5 or less)
PCM_BAR = 4.0


def _check_pcm_volume(pg, a, b):
    """Device PCM against the float64 PCM: relative L2 within PCM_BAR x the float32 oracle's, same argmax."""
    ref = pp.pcm(a, b)
    pc = po.calculate_pcm(a, b, workers=-1)
    assert pg.shape == pc.shape == ref.shape
    e32, eg = pp.rel_l2(pc, ref), pp.rel_l2(pg, ref)
    assert eg <= PCM_BAR * e32, (eg, e32)
    assert np.unravel_index(np.argmax(pg), pg.shape) == np.unravel_index(np.argmax(ref), ref.shape)


def _check(ctx, a, b, **kw):
    import bsgpu  # noqa: F401
    ext = kw.get("extension", (10, 10, 10))
    o = po.pcm_shift(a, b, peaks_to_check=kw.get("peaks", 5), do_subpixel=kw.get("subpixel", True),
                     min_overlap_frac=kw.get("min_overlap", 0.25), extension=ext)
    p = ctx.pcm_params(kw.get("peaks", 5), kw.get("subpixel", True), kw.get("min_overlap", 0.25), ext)
    g = ctx.pcm_pair(a, b, p)
    assert g.pad == o.pad
    assert g.found == o.found
    if o.found:
        assert g.shift_int == o.shift_int, (g, o.shift_int, o.candidates[:6])
        assert g.peak_index == o.peak_index
        assert g.n_overlap_px == o.n_overlap_px
        assert abs(g.r - o.r) < 1e-9
        assert np.allclose(g.shift_sub, o.shift_sub, atol=1e-3), (g.shift_sub, o.shift_sub)
    return g, o


def test_pcm_volume_matches_oracle(ctx):
    a, b = synth.shifted_pair((40, 48, 56), (3, -2, 1), seed=1)
    _check_pcm_volume(ctx.pcm_debug_pcm(a, b), a, b)


@pytest.mark.parametrize("shape,shift,seed", [
    ((64, 64, 64), (3, -2, 1), 1),
    ((64, 64, 64), (0, 0, 0), 2),
    ((48, 80, 96), (-7, 5, 11), 3),
    ((96, 64, 50), (12, -9, 4), 4),
    ((33, 45, 71), (-5, 6, -3), 5),     # odd sizes -> radix 3/5 paths, ragged line groups
    ((128, 128, 128), (20, -20, 3), 6),
])
def test_planted_integer_shift(ctx, shape, shift, seed):
    a, b = synth.shifted_pair(shape, shift, seed=seed)
    g, o = _check(ctx, a, b)
    assert g.found and g.shift_int == shift  # known answer, not just oracle agreement


def test_identical_images(ctx):
    a, _ = synth.shifted_pair((64, 64, 64), (0, 0, 0), seed=7)
    g, o = _check(ctx, a, a.copy())
    assert g.shift_int == (0, 0, 0) and abs(g.r - 1.0) < 1e-12


def test_float32_input(ctx):
    a, b = synth.shifted_pair((48, 48, 48), (4, 3, -2), seed=8, dtype=np.float32)
    g, o = _check(ctx, a, b)
    assert g.shift_int == (4, 3, -2)


def test_no_subpixel_and_peak_count(ctx):
    a, b = synth.shifted_pair((64, 64, 64), (2, 2, 2), seed=9)
    g, o = _check(ctx, a, b, subpixel=False, peaks=1)
    assert g.shift_sub == tuple(float(v) for v in g.shift_int)
    _check(ctx, a, b, peaks=12)


def test_constant_image_returns_r0(ctx):
    a = np.full((32, 32, 32), 1000, dtype=np.uint16)
    g, o = _check(ctx, a, a.copy())
    if g.found:
        assert g.r == 0.0


def test_min_overlap_rejects_everything(ctx):
    a, b = synth.shifted_pair((32, 32, 32), (1, 1, 1), seed=10)
    g, o = _check(ctx, a, b, min_overlap=2.0)   # nothing can overlap by 200 %
    assert not g.found


def test_thin_volume_2d_like(ctx):
    # singleton z: extension min(10, 1) = 1 -> padded size 3
    a, b = synth.shifted_pair((1, 96, 96), (5, -4, 0), seed=11)
    g, o = _check(ctx, a, b)
    assert g.shift_int == (5, -4, 0)


def test_batch_host_pipeline_equals_single(ctx):
    pairs = [synth.shifted_pair((48, 56, 64), s, seed=20 + i) for i, s in enumerate([(1, 2, 3), (-4, 0, 2), (6, -6, 1)])]
    single = [ctx.pcm_pair(a, b) for a, b in pairs]
    batch = ctx.pcm_batch([p[0] for p in pairs], [p[1] for p in pairs])
    for s, b in zip(single, batch):
        assert s == b


def test_device_resident_input(ctx):
    import torch
    a, b = synth.shifted_pair((64, 64, 64), (3, 1, -2), seed=30)
    ta = torch.from_numpy(a.view(np.int16)).cuda()
    tb = torch.from_numpy(b.view(np.int16)).cuda()
    torch.cuda.synchronize()
    g = ctx.pcm_pair(ta, tb)
    h = ctx.pcm_pair(a, b)
    assert g == h and g.shift_int == (3, 1, -2)


def test_bad_arguments(ctx):
    import bsgpu
    a = np.zeros((8, 8, 8), np.uint16)
    with pytest.raises(bsgpu.BsError):
        ctx.pcm_pair(a, a, ctx.pcm_params(peaks_to_check=0))
    with pytest.raises(bsgpu.BsError):
        ctx.pcm_pair(a, a, ctx.pcm_params(peaks_to_check=1000))


#: shapes and planted shifts of the mixed-size batches: the dims change from one pair to the next
MIXED_SPECS = [((40, 48, 56), (2, -1, 3)), ((64, 64, 64), (-3, 4, 1)), ((33, 45, 71), (1, 1, -2)), ((40, 48, 56), (0, 5, -4))]


def _mixed_pairs():
    return [synth.shifted_pair(sh, s, seed=60 + i) for i, (sh, s) in enumerate(MIXED_SPECS)]


def test_mixed_size_batch_regrows_workspace(ctx):
    """Pairs of different sizes in one call: workspace, twiddle tables and profiles are rebuilt per size."""
    pairs = _mixed_pairs()
    batch = ctx.pcm_batch([p[0] for p in pairs], [p[1] for p in pairs])
    for (sh, s), r, (a, b) in zip(MIXED_SPECS, batch, pairs):
        o = po.pcm_shift(a, b)
        assert r.found and r.shift_int == o.shift_int == s and r.pad == o.pad
        assert np.allclose(r.shift_sub, o.shift_sub, atol=1e-3) and abs(r.r - o.r) < 1e-9


def test_mixed_size_batch_device_inputs(ctx):
    """The same mixed sizes as device-resident crops: each result equals the pair run alone."""
    import torch
    pairs = _mixed_pairs()
    dev = [[torch.from_numpy(x.view(np.int16)).cuda() for x in p] for p in pairs]
    torch.cuda.synchronize()
    assert ctx.pcm_batch([d[0] for d in dev], [d[1] for d in dev]) == [ctx.pcm_pair(a, b) for a, b in pairs]


def test_mixed_size_volumes_batch(ctx):
    """pcm_volumes_batch over resident volumes whose overlap dims change twice (A B A); pair B's first crop is cut
    from a larger volume on the device.  Each result equals the pair run alone."""
    pairs = _mixed_pairs()
    pairs = [pairs[0], pairs[1], pairs[3]]
    a1, b1 = pairs[1]
    big = np.zeros((a1.shape[0] + 3, a1.shape[1] + 5, a1.shape[2] + 7), a1.dtype)
    big[1:1 + a1.shape[0], 2:2 + a1.shape[1], 3:3 + a1.shape[2]] = a1
    vols = [pairs[0], (big, b1), pairs[2]]
    mins = [((0, 0, 0), (0, 0, 0)), ((3, 2, 1), (0, 0, 0)), ((0, 0, 0), (0, 0, 0))]
    handles = [(ctx.volume_upload(v1), ctx.volume_upload(v2)) for v1, v2 in vols]
    jobs = [(h1, h2, m1, m2, a.shape[::-1]) for (h1, h2), (m1, m2), (a, _) in zip(handles, mins, pairs)]
    try:
        got = ctx.pcm_volumes_batch(jobs)
    finally:
        for h in handles:
            ctx.volume_free(h[0])
            ctx.volume_free(h[1])
    assert got == [ctx.pcm_pair(a, b) for a, b in pairs]


def _pcm_via(ctx, entry, a, b, params=None, dtype=None):
    """Phase correlation of one host pair through one entry point (debug_pcm: the PCM volume); `dtype`, when given,
    is the code handed to the library as is."""
    if entry == "host":
        return ctx.pcm_batch([a], [b], params, dtype=dtype)[0]
    if entry == "device":
        import torch
        ta, tb = (torch.from_numpy(x.view(np.int16)).cuda() for x in (a, b))
        torch.cuda.synchronize()
        return ctx.pcm_batch([ta], [tb], params, dtype=dtype)[0]
    if entry == "volumes":
        h1, h2 = ctx.volume_upload(a), ctx.volume_upload(b)
        try:
            return ctx.pcm_volumes_batch([(h1, h2, (0, 0, 0), (0, 0, 0), a.shape[::-1])], params)[0]
        finally:
            ctx.volume_free(h1)
            ctx.volume_free(h2)
    return ctx.pcm_debug_pcm(a, b)


@pytest.mark.parametrize("entry", ["host", "device", "volumes", "debug_pcm"])
def test_bad_parameters_rejected_on_every_entry_point(ctx, entry):
    """interpolate_xcorr, peaks_to_check outside [1, 32] and an unknown dtype code (where the caller passes one) are
    refused by every PCM entry point, and the context then still returns the right result for a valid pair."""
    import ctypes as C
    import bsgpu
    a, b = synth.shifted_pair((24, 32, 40), (2, -3, 1), seed=110)
    want = _pcm_via(ctx, entry, a, b)
    bad = []   # (message, call)
    if entry == "debug_pcm":   # takes only the extension of the parameters; the wrapper derives the dtype from a
        _check_pcm_volume(want, a, b)
        out, pad = np.empty_like(want), (C.c_int * 3)()
        dims, ext = (C.c_longlong * 3)(*a.shape[::-1]), (C.c_int * 3)(10, 10, 10)
        bad.append(("dtype", lambda: ctx._check(ctx.lib.bs_pcm_debug_pcm(ctx.h, a.ctypes.data, b.ctypes.data, dims, 99,
                                                                          ext, out.ctypes.data, pad))))
    else:
        assert want.found and want.shift_int == (2, -3, 1)
        for field, value in (("interpolate_xcorr", 1), ("peaks_to_check", 0), ("peaks_to_check", 33)):
            p = ctx.pcm_params()
            setattr(p, field, value)
            bad.append((field, lambda p=p: _pcm_via(ctx, entry, a, b, params=p)))
    if entry in ("host", "device"):
        bad.append(("dtype", lambda: _pcm_via(ctx, entry, a, b, dtype=99)))
    for msg, call in bad:
        with pytest.raises(bsgpu.BsError, match=msg):
            call()
        got = _pcm_via(ctx, entry, a, b)
        assert np.array_equal(got, want) if entry == "debug_pcm" else got == want


def test_large_single_axis_generic_path(ctx):
    """A long, thin crop (x pad 810 = 2*3^4*5, M = 405 > 319): CTA-level x kernels + generic plans."""
    a, b = synth.shifted_pair((12, 20, 780), (9, -2, 1), seed=70, margin=12)
    g, o = _check(ctx, a, b)           # GPU == oracle (bit-identical shift, 1e-3 sub-pixel)
    assert g.shift_int[:2] == (9, -2)  # 12 z-slices carry too little signal to pin the z component


def test_long_aligned_rows_cta_tma_path(ctx):
    """x pad 810 (M = 405 > 319) with 16-byte-multiple rows (784 * 2 B): the CTA-level TMA-staged
    r2c kernel with a runtime-planned FFT."""
    a, b = synth.shifted_pair((10, 24, 784), (-6, 3, 0), seed=71, margin=12)
    g, o = _check(ctx, a, b)
    assert g.pad[0] == 810 and g.shift_int[:2] == (-6, 3)


def test_oversized_dims_rejected_before_any_copy(ctx):
    """Maximum sizes: an axis beyond 16384 is refused up front (nothing is read from the host buffers)."""
    import bsgpu
    a = np.zeros((8, 8, 8), np.uint16)
    with pytest.raises(bsgpu.BsError) as e:
        ctx.pcm_pair(a, a, dims_xyz=(20000, 8, 8))
    assert "out of range" in str(e.value)
    assert ctx.pcm_batch([], []) == []          # empty batch is a no-op


# ---- the code paths bench.py runs: compile-time plans for padded length 540 (x: FftWStatic<270>, y/z:
# k_fft_col540 y pass and k_fft_xpower_col540 z cross-power pass on RegFft2<20, 27>).  The static plans are
# selected per axis, so three thin crops reach each of them cheaply; the full 512^3 pair is the bench unit.
@pytest.mark.parametrize("shape,shift", [
    ((24, 24, 500), (7, -3, 2)),     # x pads to 540  -> k_fft_x_r2c_w / k_fft_x_c2r_w <FftWStatic<270>>
    ((24, 500, 24), (-2, 9, 1)),     # y pads to 540  -> k_fft_col540
    ((500, 24, 24), (3, 2, -11)),    # z pads to 540  -> k_fft_xpower_col540 (cross-power)
    ((500, 500, 24), (1, -8, 6)),    # y and z static, x generic
])
def test_static_540_plans_thin_crops(ctx, shape, shift):
    a, b = synth.shifted_pair(shape, shift, seed=80 + shape[0] % 7, margin=16)
    g, o = _check(ctx, a, b)
    assert 540 in g.pad
    _check_pcm_volume(ctx.pcm_debug_pcm(a, b), a, b)


def test_static_540_thin_subpixel(ctx):
    a, b = synth.subpixel_pair((24, 500, 500), (4.3, -6.25, 1.4), seed=85, margin=16)
    g, o = _check(ctx, a, b)
    assert g.pad[0] == 540 and g.pad[1] == 540
    assert g.shift_int[:2] == (4, -6)
    assert abs(g.shift_sub[0] - 4.3) < 0.15 and abs(g.shift_sub[1] + 6.25) < 0.15   # known answer (fit bias)


def test_full_512_pair_subpixel_bench_unit(ctx):
    """One full BASELINE configs[1] unit: 512^3 uint16 pair with a planted SUB-PIXEL shift, all three axes
    on the static 540 plans -- every kernel bench.py times, against the oracle (sub 1e-3, r 1e-9, index
    bit-identical, PCM volume 2e-4)."""
    a, b = synth.subpixel_pair((512, 512, 512), (11.37, -4.62, 7.3), seed=90, margin=20)
    o = po.pcm_shift(a, b, workers=-1)
    g = ctx.pcm_pair(a, b)
    assert g.pad == o.pad == (540, 540, 540)
    assert g.found and o.found
    assert g.shift_int == o.shift_int and g.peak_index == o.peak_index
    assert g.n_overlap_px == o.n_overlap_px and abs(g.r - o.r) < 1e-9
    assert np.allclose(g.shift_sub, o.shift_sub, atol=1e-3), (g.shift_sub, o.shift_sub)
    assert np.allclose(g.shift_sub, (11.37, -4.62, 7.3), atol=0.2)
    # The float64 PCM of this size needs several GB of host memory, so the volume keeps the float32 oracle's
    # max-norm bar; the per-pass tests (test_pcm_fft_passes_gpu.py) cover the 540-point kernels in float64.
    pg = ctx.pcm_debug_pcm(a, b)
    pc = po.calculate_pcm(a, b, workers=-1)
    assert np.abs(pg - pc).max() < 2e-4 * np.abs(pc).max()


def _pinned(arr):
    import torch
    t = torch.from_numpy(arr.view(np.int16) if arr.dtype == np.uint16 else arr).pin_memory()
    return t, (t.numpy().view(np.uint16) if arr.dtype == np.uint16 else t.numpy())


def test_volumes_batch_crops_on_device(ctx):
    """Tiles are uploaded once (async, pinned) and every pair's overlap crop is cut on the device:
    bit-identical to running the host-cropped pair."""
    G = synth.field((96, 120, 200), seed=101, sigma=1.5)
    tA = synth.tile_from(G, (8, 10, 12), (64, 72, 96), 1)
    tB = synth.tile_from(G, (8 + 2, 10 - 3, 12 + 70), (64, 72, 96), 2)     # true offset of B in A's frame: (70, -3, 2)
    keep = [_pinned(tA), _pinned(tB)]
    hA, hB = ctx.volume_upload_async(keep[0][1]), ctx.volume_upload_async(keep[1][1])
    # nominal registration says B starts at x = 66: overlap = A[66:96] x B[0:30] (x), full y / z
    jobs = [(hA, hB, (66, 0, 0), (0, 0, 0), (30, 72, 64)),
            (hA, hA, (0, 0, 0), (0, 0, 0), (96, 72, 64)),          # whole volumes: no crop copy
            (hB, hA, (0, 0, 0), (66, 0, 0), (30, 72, 64))]
    got = ctx.pcm_volumes_batch(jobs)
    a, b = np.ascontiguousarray(tA[:, :, 66:96]), np.ascontiguousarray(tB[:, :, 0:30])
    assert got[0] == ctx.pcm_pair(a, b)
    o = po.pcm_shift(a, b)
    assert got[0].found and got[0].shift_int == o.shift_int and abs(got[0].r - o.r) < 1e-9
    assert got[0].shift_int == (4, -3, 2)       # planted: b[p] = a[p + (4, -3, 2)] (true x offset 70 vs nominal 66)
    assert got[1].shift_int == (0, 0, 0) and abs(got[1].r - 1.0) < 1e-12
    assert got[2] == ctx.pcm_pair(b, a)
    ctx.volume_free(hA)
    ctx.volume_free(hB)
    # recycled pool buffer: a second upload of the same size reuses the device allocation
    hC = ctx.volume_upload_async(keep[0][1])
    assert ctx.pcm_volumes_batch([(hC, hC, (0, 0, 0), (0, 0, 0), (96, 72, 64))])[0].shift_int == (0, 0, 0)
    ctx.volume_free(hC)
    import bsgpu
    with pytest.raises(bsgpu.BsError):
        ctx.pcm_volumes_batch([(12345, 12345, (0, 0, 0), (0, 0, 0), (8, 8, 8))])
