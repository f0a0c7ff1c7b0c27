"""The two separable-Gaussian stencil paths on the device against float64 references.

DoG detection (csrc/dog.cu): the DoG box the extremum stage reads (bs_dog_debug_dog), for every blur variant forced in
turn, against oracle/dog_oracle.dog_reference; the variants bit-identical to each other; detections independent of the
block grid; the extremum stage exact given the device's DoG; the threshold compares.
Content weights (csrc/content.cu): bs_content_weights against oracle/fusion_oracle.content_weights_reference up to the
shared-memory length limits, and a clean error one past them.

Each bar is a worst-case float32 rounding bound per voxel.  Each test also checks that a wrong reference (an outermost
tap dropped, a border fold off by one) breaks its bar by at least TEETH on its own inputs.
"""
import os
import re

import numpy as np
import pytest

from oracle import dog_oracle as do
from oracle import fusion_oracle as fo
from tests import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24          # float32 unit roundoff
TEETH = 50.0            # a wrong reference must miss the bar by this factor on at least one voxel

# ------------------------------------------------------------------------------------------ DoG
# One blur pass of radius r rounds r + 1 fmaf steps and one pair add per tap pair: at most (r + 2) u relative to
# G * |I'|, and the three passes add up to 3 (r + 2) u.  A - B and the 1 / (k - 1) scale round once each, so the DoG
# error is at most (3 rb + 8) u kinv (G_sa * |I'| + G_sb * |I'|), which is <= 2 (2 rb + 3) (...) for rb >= 2 (every
# sigma >= 0.6).  The reference uses the same float32 taps, I' and scale, so nothing else differs.
DOG_BAR_C = 2.0
DOG_SHAPE = (28, 36, 40)                  # [z, y, x]
SIGMAS = (0.6, 1.8, 2.0, 3.5, 3.6, 8.0, 17.0)
BLUR_GENERIC, BLUR_WIN6, BLUR_WIN12 = 1, 2, 3
BLUR_NAMES = {BLUR_GENERIC: "k_dog_blur", BLUR_WIN6: "k_dog_blur_x<6>", BLUR_WIN12: "k_dog_blur_x<12>"}


def _radii(sigma):
    sa, sb, kinv = do.compute_sigmas(sigma)
    return len(do.gauss_kernel(sa)) // 2, len(do.gauss_kernel(sb)) // 2, kinv


def _variants(rb):
    """The blurs that can run kernel radius rb."""
    return [BLUR_GENERIC] + ([BLUR_WIN6] if rb <= 6 else []) + ([BLUR_WIN12] if rb <= 12 else [])


def _production(rb):
    return BLUR_WIN6 if rb <= 6 else (BLUR_WIN12 if rb <= 12 else BLUR_GENERIC)


def _ratio(err, bar):
    """max err / bar over the voxels (inf where the bar is 0 and the error is not)."""
    if np.any((bar == 0) & (err > 0)):
        return np.inf
    pos = bar > 0
    return float((err[pos] / bar[pos]).max()) if pos.any() else 0.0


def _field(seed, noise, shape=DOG_SHAPE):
    return synth.tile_from(synth.field(shape, seed=seed, sigma=2.0), (0, 0, 0), shape, seed, noise=noise)


@pytest.fixture(scope="module")
def dog_sources():
    """name -> (image [z, y, x], min_intensity, max_intensity)."""
    field = _field(11, 20.0)
    f32 = ((field.astype(np.float32) - 1200.0) / 7.0).astype(np.float32)      # about -170 .. 180: I' < 0 and > 1
    imp = np.zeros(DOG_SHAPE, np.uint8)                                       # sparse impulses: G*|I'| is 0 or small
    imp[14, 18, 20] = imp[2, 33, 3] = 255                                     # away from and near the faces
    tiny = np.random.default_rng(3).integers(0, 4000, (2, 3, 5)).astype(np.uint16)   # smaller than any halo
    return {"u16": (field, 0.0, 3000.0), "f32": (f32, 10.0, 150.0), "u8": (imp, 0.0, 255.0), "tiny": (tiny, 0.0, 4000.0)}


def _dog_cases(halo):
    """(source, interval_min xyz, interval_size xyz)."""
    Z, Y, X = DOG_SHAPE
    cases = [
        ("u8", (0, 0, 0), (X, Y, Z)),                     # the whole volume: every face
        ("u16", (9, 8, 7), (17, 13, 11)),                 # interior
        ("f32", (0, 0, 0), (12, 10, 9)),                  # near faces
        ("u16", (X - 13, Y - 11, Z - 6), (13, 11, 6)),    # far faces
        ("u8", (X - 9, 0, Z - 8), (9, 12, 8)),            # far x, near y, far z
        ("f32", (5, 20, 3), (11, 1, 14)),                 # one voxel along y
        ("u16", (30, 2, Z - 1), (1, 9, 1)),               # one voxel along x and z, on the far z face
        ("tiny", (0, 0, 0), (5, 3, 2)),                   # the mirror folds over several periods
        ("tiny", (4, 1, 1), (1, 2, 1)),
    ]
    for m in (0, 1, 7):     # region x = size + 2 halo: = 0 (mod 8) needs no row padding, 1 and 7 do
        cases.append(("f32" if m else "u16", (3, 4, 5), ((m - 2 * halo) % 8 + 8, 6, 5)))
    return cases


@pytest.mark.parametrize("sigma", SIGMAS)
def test_dog_box_matches_float64_and_blur_variants_agree(ctx, dog_sources, sigma):
    ra, rb, kinv = _radii(sigma)
    variants = _variants(rb)
    handles = {k: ctx.volume_upload(v[0]) for k, v in dog_sources.items()}
    worst = {b: 0.0 for b in variants}
    teeth_tap = teeth_fold = 0.0
    try:
        for name, mn, sz in _dog_cases(max(ra, rb) + 1):
            img, lo, hi = dog_sources[name]
            ref, ga, gb = do.dog_reference(img, mn, sz, sigma, lo, hi)
            bar = DOG_BAR_C * U * kinv * (2 * rb + 3) * (ga + gb)
            boxes = {}
            for b in variants:
                got, info = ctx.dog_debug_dog(handles[name], mn, sz, sigma, lo, hi, blur=b)
                assert info == f"{BLUR_NAMES[b]} ra={ra} rb={rb}"
                r = _ratio(np.abs(got - ref), bar)
                assert r <= 1.0, (name, mn, sz, info, r)
                worst[b] = max(worst[b], r)
                boxes[b] = got
            # the production choice is one of them, and every variant that can run rb gives the same bits
            got, info = ctx.dog_debug_dog(handles[name], mn, sz, sigma, lo, hi)
            assert info.split(" ")[0] == BLUR_NAMES[_production(rb)]
            for b in variants:
                assert np.array_equal(boxes[b], got), (name, mn, sz, BLUR_NAMES[b], info)
            if name in ("u8", "tiny"):
                tap, _, _ = do.dog_reference(img, mn, sz, sigma, lo, hi, drop_outer_tap_axis=0)
                fold, _, _ = do.dog_reference(img, mn, sz, sigma, lo, hi, pad_mode="reflect")
                teeth_tap = max(teeth_tap, _ratio(np.abs(tap - ref), bar))
                teeth_fold = max(teeth_fold, _ratio(np.abs(fold - ref), bar))
    finally:
        for h in handles.values():
            ctx.volume_free(h)
    print(f"\nDoG sigma {sigma} ra={ra} rb={rb}: worst |err| / bar " +
          ", ".join(f"{BLUR_NAMES[b]} {worst[b]:.4f}" for b in variants) + f"; teeth tap {teeth_tap:.0f} fold {teeth_fold:.0f}")
    assert teeth_tap >= TEETH and teeth_fold >= TEETH


def test_forced_window_too_small_is_an_argument_error(ctx):
    import bsgpu
    h = ctx.volume_upload(_field(11, 20.0))
    try:
        for sigma, blur in ((2.0, BLUR_WIN6), (3.6, BLUR_WIN12), (1.8, 4)):
            with pytest.raises(bsgpu.BsError):
                ctx.dog_debug_dog(h, (0, 0, 0), (8, 8, 8), sigma, 0.0, 3000.0, blur=blur)
        box, info = ctx.dog_debug_dog(h, (0, 0, 0), (8, 8, 8), 1.8, 0.0, 3000.0, blur=BLUR_WIN6)
        assert info == "k_dog_blur_x<6> ra=5 rb=6" and box.shape == (10, 10, 10)
    finally:
        ctx.volume_free(h)


@pytest.mark.parametrize("sigma", [1.8, 3.5, 8.0])      # window R 6, window R 12, generic
def test_dog_block_grid_union_is_the_whole_interval(ctx, sigma):
    """Unequal 2 x 3 x 2 blocks of a 96 x 80 x 64 field detect exactly what the whole interval does: a halo one voxel
    short on any axis would change the DoG next to a block face."""
    vol = _field(21, 30.0, (64, 80, 96))
    h = ctx.volume_upload(vol)
    kw = dict(sigma=sigma, threshold=0.0, max_intensity=3000.0, find_max=True, find_min=True)
    try:
        whole = ctx.dog_detect(h, (0, 0, 0), (96, 80, 64), **kw)
        parts = []
        for x0, x1 in ((0, 41), (41, 96)):
            for y0, y1 in ((0, 23), (23, 50), (50, 80)):
                for z0, z1 in ((0, 37), (37, 64)):
                    parts += ctx.dog_detect(h, (x0, y0, z0), (x1 - x0, y1 - y0, z1 - z0), **kw)
    finally:
        ctx.volume_free(h)
    parts.sort(key=lambda p: (p[2][2], p[2][1], p[2][0]))
    assert len(whole) > 20
    assert parts == whole


@pytest.mark.parametrize("sigma", [1.8, 2.6])      # window R 6, window R 12
def test_extremum_stage_is_exact_on_the_device_dog(ctx, sigma):
    """Given the device's DoG box, oracle.extrema reproduces dog_detect exactly: same voxels and is_max, loc and value to
    1e-12 (both are double arithmetic on the same floats), for MAX / MIN / BOTH with and without localisation."""
    vol = _field(7, 60.0)
    h = ctx.volume_upload(vol)
    mn, sz = (2, 3, 1), (36, 31, 26)
    try:
        box, _ = ctx.dog_debug_dog(h, mn, sz, sigma, 0.0, 3000.0)
        thr = float(np.quantile(np.abs(box), 0.1))
        for fmax, fmin in ((True, False), (False, True), (True, True)):
            for loc in (True, False):
                kw = dict(threshold=thr, find_max=fmax, find_min=fmin, localization=loc)
                got = ctx.dog_detect(h, mn, sz, sigma=sigma, max_intensity=3000.0, **kw)
                want = do.extrema(box, mn, **kw)
                assert len(want) >= 3, kw
                assert [(g[2], g[3]) for g in got] == [(w[2], w[3]) for w in want], kw
                assert max(np.abs(np.subtract(g[0], w[0])).max() for g, w in zip(got, want)) <= 1e-12
                assert max(abs(g[1] - w[1]) for g, w in zip(got, want)) <= 1e-12
    finally:
        ctx.volume_free(h)


# ---- threshold semantics (PARITY_GAPS #26): kept at |value| >= threshold in double, candidates at
# |DoG| >= float32(threshold / 3) with localisation (float32(threshold) without)
_KW = dict(sigma=1.8, min_intensity=0.0, max_intensity=3000.0, find_max=True, find_min=True)


def test_detection_at_exactly_its_threshold_is_kept(ctx):
    vol = _field(5, 10.0)
    h = ctx.volume_upload(vol)
    full = ((0, 0, 0), DOG_SHAPE[::-1])
    try:
        pts = ctx.dog_detect(h, *full, threshold=0.001, **_KW)
        assert len(pts) >= 20
        rounds_up = 0
        for p in pts[:24]:
            t = abs(p[1])
            rounds_up += float(np.float32(t)) > t       # the values a float32 compare used to drop
            again = ctx.dog_detect(h, *full, threshold=t, **_KW)
            assert p in again, p
        assert rounds_up >= 3
    finally:
        ctx.volume_free(h)


def test_unlocalised_threshold_just_above_the_value_drops_it(ctx):
    vol = _field(5, 10.0)
    h = ctx.volume_upload(vol)
    full = ((0, 0, 0), DOG_SHAPE[::-1])
    try:
        pts = ctx.dog_detect(h, *full, threshold=0.001, localization=False, **_KW)
        assert len(pts) >= 10
        for p in pts[:10]:
            v = abs(p[1])
            above = float(np.nextafter(v, np.inf))
            assert float(np.float32(above)) == v
            assert p in ctx.dog_detect(h, *full, threshold=v, localization=False, **_KW)
            assert p[2] not in [q[2] for q in ctx.dog_detect(h, *full, threshold=above, localization=False, **_KW)]
    finally:
        ctx.volume_free(h)


def test_zero_threshold_on_a_constant_volume_returns_every_voxel(ctx):
    h = ctx.volume_upload(np.full((6, 7, 9), 700, np.uint16))
    mn, sz = (1, 2, 0), (7, 4, 5)
    every = sorted((x, y, z) for z in range(5) for y in range(2, 6) for x in range(1, 8))
    try:
        # a constant DoG ties with all its neighbours: every voxel is an extremum; max_points 5 < 140 takes the
        # buffer growth path
        got = ctx.dog_detect(h, mn, sz, threshold=0.0, max_points=5, **_KW)
        assert sorted(g[2] for g in got) == every
        # I' = 0: the DoG is exactly 0 and every voxel is a maximum at threshold 0
        got = ctx.dog_detect(h, mn, sz, sigma=3.6, threshold=0.0, min_intensity=700.0, max_intensity=3000.0, max_points=5)
        assert sorted(g[2] for g in got) == every and all(g[3] and g[1] == 0.0 for g in got)
    finally:
        ctx.volume_free(h)


def test_candidate_threshold_is_float32_of_threshold_over_3(ctx):
    """With localisation a voxel of DoG v is a candidate when |v| >= float32(threshold / 3).  For voxels whose
    localised value exceeds 3 |v|, threshold 3 |v| keeps them (a tie); 3 |v| (1 + 2^-30) keeps them too (the quotient
    rounds to |v| in float32); 3 nextafter_f32(|v|) drops them although their value passes the final test."""
    sigma = 0.8
    vol = _field(4, 60.0)
    h = ctx.volume_upload(vol)
    full = ((0, 0, 0), DOG_SHAPE[::-1])
    try:
        box, _ = ctx.dog_debug_dog(h, *full, sigma, 0.0, 3000.0)
        pts = do.extrema(box, full[0], threshold=0.0, find_max=True, find_min=True)
        val_of = {p[2]: abs(p[1]) for p in pts}
        picks = [p[2] for p in pts if 0 < 3 * abs(float(box[p[2][2] + 1, p[2][1] + 1, p[2][0] + 1])) * (1 + 1e-6) < abs(p[1])]
        assert len(picks) >= 1
        for (x, y, z) in picks[:4]:
            a = abs(float(box[z + 1, y + 1, x + 1]))
            t_tie, t_mid = 3.0 * a, 3.0 * a * (1 + 2.0 ** -30)
            t_hi = 3.0 * float(np.nextafter(np.float32(a), np.float32(np.inf)))
            assert t_mid / 3 > a and float(np.float32(t_mid / 3)) == a and t_hi <= val_of[(x, y, z)]
            for t, kept in ((t_tie, True), (t_mid, True), (t_hi, False)):
                got = ctx.dog_detect(h, (x, y, z), (1, 1, 1), sigma=sigma, threshold=t, max_intensity=3000.0,
                                     find_max=True, find_min=True)
                assert [g[2] for g in got] == ([(x, y, z)] if kept else []), (x, y, z, t, kept)
    finally:
        ctx.volume_free(h)


# ------------------------------------------------------------------------------------------ content weights
# The device accumulates every tap sum in double; only the float32 stores round.  c rounds in d = f - g, d * d and
# the three passes of G_s2 (at most 6 u c); G_s1 f rounds in its three passes, and a change e of it moves c by
# G_s2 * (2 |d| e).  With the stored intermediates bounded by |f| + 2 |G_s1 f|, 8 covers both terms.
CW_BAR_C = 8.0


def _ga_smem_max():
    src = open(os.path.join(ROOT, "bigstitcher-spark_b200", "csrc", "content.cu")).read()
    return int(re.search(r"#define GA_SMEM_MAX (\d+)", src).group(1))


def _content_limits(sigmas):
    """Largest x, and largest y / z, that bs_content_weights accepts: content.cu's shared-memory formulas (double tap
    table of 4 G + 8, G = (2 r + 7) / 4 sample groups; x pass one line of 4 ceil(x / 4) + 4 G + 4 floats, strided pass
    32 columns of 4 ceil(len / 4) + 4 G + 4 floats) against GA_SMEM_MAX, for both sigmas."""
    smem = _ga_smem_max()
    xs, ls = [], []
    for s in sigmas:
        r = len(fo.gauss_kernel(s)) // 2
        G = (2 * r + 1 + 6) // 4
        free = smem - (4 * G + 8) * 8
        xs.append(4 * ((free // 4 - 4 * G - 4) // 4))
        ls.append(4 * ((free // 128 - 4 * G - 4) // 4))
    return min(xs), min(ls)


def _x_lines(x, sigma):
    """Rows per CTA of k_gauss_x."""
    r = len(fo.gauss_kernel(sigma)) // 2
    G = (2 * r + 1 + 6) // 4
    return min(8, (_ga_smem_max() - (4 * G + 8) * 8) // ((4 * ((x + 3) // 4) + 4 * G + 4) * 4))


def _cw_source(kind, xyz, seed):
    rng = np.random.default_rng(seed)
    shape = tuple(xyz[::-1])
    if kind == "u16":
        return rng.integers(0, 4000, shape).astype(np.uint16)
    if kind == "u8":
        return rng.integers(0, 256, shape).astype(np.uint8)
    return (rng.normal(0.0, 50.0, shape) + 20.0).astype(np.float32)     # float32 with negative values


X_MAX, L_MAX = _content_limits((20.0, 40.0))
CW_CASES = {
    (2.0, 4.0): [("f32", (1, 40, 30)), ("u8", (37, 1, 25)), ("u16", (33, 29, 1)), ("f32", (95, 14, 9)), ("u16", (33, 20, 12))],
    (20.0, 40.0): [("f32", (33, 20, 12)), ("u8", (1, 40, 30)), ("u16", (95, 1, 9)), ("f32", (33, 29, 1)),
                   ("u16", (7300, 3, 2)), ("f32", (X_MAX, 2, 1)), ("u8", (33, L_MAX, 2)), ("u16", (40, 2, L_MAX))],
}


def test_content_limits_follow_from_the_shared_memory_formulas():
    assert (X_MAX, L_MAX) == (57360, 1552) and _x_lines(7300, 40.0) == 7 and _x_lines(X_MAX, 40.0) == 1


@pytest.mark.parametrize("sigmas", list(CW_CASES))
def test_content_weights_match_float64(ctx, sigmas):
    s1, s2 = sigmas
    worst = teeth = 0.0
    for i, (kind, xyz) in enumerate(CW_CASES[sigmas]):
        vol = _cw_source(kind, xyz, 100 + i)
        h = ctx.volume_upload(vol)
        c = ctx.content_weights(h, s1, s2)
        got = ctx.volume_download(c, xyz)
        ctx.volume_free(c)
        ctx.volume_free(h)
        ref, f, g1, d = fo.content_weights_reference(vol, s1, s2)
        bar = CW_BAR_C * U * (ref + fo._gauss3_f64(2 * np.abs(d) * (np.abs(f) + 2 * np.abs(g1)), fo.gauss_kernel(s2)))
        r = _ratio(np.abs(got - ref), bar)
        assert r <= 1.0, (kind, xyz, r)
        worst = max(worst, r)
        wrong, *_ = fo.content_weights_reference(vol, s1, s2, drop_outer_tap_axis=int(np.argmax(xyz)))
        teeth = max(teeth, _ratio(np.abs(wrong - ref), bar))
        print(f"\ncontent {s1}/{s2} {kind} {xyz} (x-pass lines {_x_lines(xyz[0], s2)}): |err| / bar {r:.4f}")
    print(f"content {s1}/{s2}: worst |err| / bar {worst:.4f}, teeth {teeth:.0f}")
    assert teeth >= TEETH


def test_content_weights_one_past_each_limit_is_a_clean_error(ctx):
    import bsgpu
    for xyz in ((X_MAX + 1, 1, 1), (2, L_MAX + 1, 1), (2, 1, L_MAX + 1)):
        h = ctx.volume_upload(np.ones(xyz[::-1], np.float32))
        try:
            with pytest.raises(bsgpu.BsError) as e:
                ctx.content_weights(h, 20.0, 40.0)
            assert "shared memory" in str(e.value)
        finally:
            ctx.volume_free(h)
    # the context still computes a correct volume afterwards
    vol = _cw_source("f32", (33, 20, 12), 7)
    h = ctx.volume_upload(vol)
    c = ctx.content_weights(h, 20.0, 40.0)
    got = ctx.volume_download(c, (33, 20, 12))
    ctx.volume_free(c)
    ctx.volume_free(h)
    ref, f, g1, d = fo.content_weights_reference(vol, 20.0, 40.0)
    bar = CW_BAR_C * U * (ref + fo._gauss3_f64(2 * np.abs(d) * (np.abs(f) + 2 * np.abs(g1)), fo.gauss_kernel(40.0)))
    assert _ratio(np.abs(got - ref), bar) <= 1.0
