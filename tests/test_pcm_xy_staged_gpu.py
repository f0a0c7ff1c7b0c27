"""GPU: the fused forward FFT kernel k_fft_xy_col540 at the benchmark's shape, whose y role stages its tiles by
tensor-map copies into a ring of three shared-memory buffers.

Debug pass 5 (passes 0 + 1 fused) must match pass 0 followed by pass 1 (BS_FFT_XY_FUSE=0) bit for bit on
512^3 uint16 crops (padded to 540^3).  At that shape every y CTA takes hundreds of tiles, many more than the three
buffers, so every buffer and both parities of its mbarrier turn over many times.  The hand-off window runs at its
minimum of 2 planes, at 3 and at the default; the role split at the default and 8 CTAs either side of it, so that
either role can be the one that waits; and one pair of crops has runs of all-zero z-planes.
"""
import numpy as np
import pytest

from tests.pcm_switches import set_switches

pytestmark = pytest.mark.gpu

XY = "k_fft_xy_col540"
DIMS = (512, 512, 512)
KX_132 = 82   # the default x-role CTAs of 132 SMs (xy_split in csrc/pcm.cu), scaled to the SM count the same way


def _crops(kind):
    rng = np.random.default_rng(7)
    shape = DIMS[::-1]
    a = rng.integers(0, 4096, size=shape, dtype=np.uint16)
    b = rng.integers(0, 4096, size=shape, dtype=np.uint16)
    if kind == "zero_planes":
        a[:24] = 0          # the first planes: the y role starts on planes the x role filled with zeros
        a[300:340] = 0
        b[200:260] = 0
        b[-5:] = 0
    return a, b


def _device(a):
    import torch
    t = torch.from_numpy(a.view(np.int16)).cuda()
    torch.cuda.synchronize()
    return t


def _default_kx():
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min(sm - 1, (KX_132 * sm + 66) // 132)), sm


@pytest.fixture(scope="module")
def pair(ctx):
    """pair(kind): device crops and the reference spectra of pass 0 then pass 1, kept for one kind at a time."""
    cache = {}

    def get(kind):
        if kind not in cache:
            cache.clear()
            ta, tb = (_device(x) for x in _crops(kind))
            with pytest.MonkeyPatch.context() as mp:
                set_switches(mp, {"BS_FFT_XY_FUSE": 0})
                xa, xb, _ = ctx.pcm_debug_pass(0, DIMS, ta, tb)
                ya, yb, _ = ctx.pcm_debug_pass(1, DIMS, xa, xb)
            cache[kind] = ta, tb, (ya, yb)
        return cache[kind]
    return get


@pytest.mark.parametrize("kind,setting", [("random", s) for s in ("default", "window2", "window3", "kx-8", "kx+8")] +
                         [("zero_planes", s) for s in ("default", "window2")])
def test_staged_y_role_matches_two_passes(ctx, monkeypatch, pair, kind, setting):
    ta, tb, ref = pair(kind)
    kx, sm = _default_kx()
    env = {"window2": {"BS_FFT_XY_WINDOW": 2}, "window3": {"BS_FFT_XY_WINDOW": 3},
           "kx-8": {"BS_FFT_XY_KX": kx - 8}, "kx+8": {"BS_FFT_XY_KX": kx + 8}}.get(setting, {})
    # y tiles: 540 planes x 2 spectra x 17 column tiles, over the y CTAs
    assert 540 * 34 // (sm - kx + 8) > 3
    set_switches(monkeypatch, env)
    fa, fb, info = ctx.pcm_debug_pass(5, DIMS, ta, tb)
    assert info == XY, info
    for got, want in zip((fa, fb), ref):
        assert got.shape == want.shape
        same = np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert same, f"{np.count_nonzero(got != want)} bins differ"
