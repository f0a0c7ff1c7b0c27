"""GPU: the z cross-power pass k_fft_xpower_col540 on geometries where each persistent CTA runs several tiles.

The kernel streams its tiles through three rotating shared-memory buffers, each with an mbarrier whose phase parity
flips every time the buffer is filled.  The small pass-2 cases of test_pcm_fft_passes_gpu.py have fewer tiles than the
device has SMs, so every CTA runs one tile and neither the rotation nor the second parity of any mbarrier is reached.
The geometries here are chosen from the device's SM count:

  * many: at least four tiles per SM (every CTA cycles A through both of its buffers at least twice, so every
    mbarrier completes phases of both parities), a tile count that is not a multiple of the SM count, and a last
    x-tile with 15 pitch-tail columns;
  * above: a few more tiles than SMs, so most CTAs exit after one tile while the others run a second;
  * below: fewer tiles than SMs.

Each case is checked against the float64 reference of the pass (oracle/pcm_passes.py) with the bars of
test_pcm_fft_passes_gpu.py, and run twice to require bit-identical output.
"""
import numpy as np
import pytest

from oracle import pcm_oracle as po
from oracle import pcm_passes as pp
from tests.pcm_switches import set_switches
from tests.test_pcm_fft_passes_gpu import BAR, MEASURED, ULP32, UNIT, ZERO, _z_lines

pytestmark = pytest.mark.gpu

DZ = 520    # pads to Pz = 540, the static z plan
DX = {1: 10, 2: 12}   # x-tiles per row -> crop x: 10 pads to Px = 30 (M + 1 = 16), 12 to Px = 32 (M + 1 = 17, tail 15)


def _n_tiles(dims):
    P = po.padded_dims(dims, (10, 10, 10))
    assert P[2] == 540
    pitch = (P[0] // 2 + 1 + 15) // 16 * 16
    return pitch // 16 * P[1]


def _dims(kind, sm):
    """Smallest (or for "below", largest) crop of the kind for a device with ``sm`` SMs."""
    if kind == "many":
        ok = lambda n: n >= 4 * sm and n % sm != 0
        tx, order = 2, range(1, 4096)
    elif kind == "above":
        ok = lambda n: sm < n < 2 * sm
        tx, order = 1, range(1, 4096)
    else:
        ok = lambda n: n < sm
        tx, order = 1, range(sm, 0, -1)
    for dy in order:
        dims = (DX[tx], dy, DZ)
        if ok(_n_tiles(dims)):
            return dims
    raise ValueError((kind, sm))


@pytest.mark.parametrize("kind", ["many", "above", "below"])
def test_zpass_rotating_buffers(ctx, monkeypatch, kind):
    import torch
    set_switches(monkeypatch)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    dims = _dims(kind, sm)
    n_tiles = _n_tiles(dims)
    P = po.padded_dims(dims, (10, 10, 10))
    M = P[0] // 2
    a, b, kind_of = _z_lines(P, M, seed=sum(dims))
    out, _, info = ctx.pcm_debug_pass(2, dims, a, b)
    what = f"{info} dims {dims}, {n_tiles} tiles on {sm} SMs"
    assert info == "k_fft_xpower_col540", what
    assert not np.isnan(out).any(), what

    ref, f32 = pp.pass2(a, b), pp.pass2_f32(a, b)
    err, _ = pp.line_rel_l2(out, ref, 0)
    err32, _ = pp.line_rel_l2(f32, ref, 0)
    bar = BAR * max(err32[np.isin(kind_of, MEASURED)].max(), ULP32)
    for k in MEASURED:
        sel = kind_of == k
        if sel.any():
            assert err[sel].max() <= bar, f"{what}: kind {k} worst rel L2 {err[sel].max():.3g}, bar {bar:.3g}"
    for k in UNIT:
        sel = kind_of == k
        if sel.any():
            assert np.abs(np.abs(out[:, sel]) - 1).max() < 1e-4, f"{what}: kind {k} is not unit"
            assert err[sel].max() < 1e-4, f"{what}: kind {k} worst rel L2 {err[sel].max():.3g}"
    assert np.all(out[:, np.isin(kind_of, ZERO)] == 0), what

    again, _, _ = ctx.pcm_debug_pass(2, dims, a, b)
    assert np.array_equal(out.view(np.uint64), again.view(np.uint64)), f"{what}: second run differs"
