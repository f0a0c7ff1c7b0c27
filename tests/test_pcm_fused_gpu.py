"""GPU: the fused forward FFT kernel of the 540-point plan against the passes it replaces.

k_fft_xy_col540 runs the x R2C pass and the forward y pass in one launch (debug pass 5).  Each transform keeps the
arithmetic of the standalone kernels, so the bar is bit identity with pass 0 followed by pass 1, run with
BS_FFT_XY_FUSE=0.  The crops are 512 x 512 in x and y (padded to 540) with a small z extent, so the fused kernel
applies at the default rule; the z extents cover fewer planes than the hand-off window, a partial last x tile
(540 Pz not a multiple of 16), and many more planes than the window, so that the x role waits for it; the window
is also forced down to its minimum of 2 planes.
"""
import dataclasses

import numpy as np
import pytest

from tests import synth

pytestmark = pytest.mark.gpu

ENV = ("BS_FFT_XY_FUSE", "BS_FFT_XY_KX", "BS_FFT_XY_WINDOW", "BS_FFT_X_COL540", "BS_FFT_STATIC")
XY = "k_fft_xy_col540"
# dz -> Pz with the extension 10: 3 -> 9 (odd, below the window), 4 -> 12, 61 -> 81 (odd, several windows deep)
DZ = [3, 4, 61]


def _set_env(monkeypatch, **env):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def _geometry(dims):
    from bsgpu.native import good_fft_size
    P = [good_fft_size(d + (2 * d if d < 10 else 20), i == 0) for i, d in enumerate(dims)]
    return P, P[0] // 2


def _device_crops(dims, seed):
    import torch
    shape = dims[::-1]
    out = []
    for i in range(2):
        a = np.clip(np.rint(synth.field(shape, seed=seed + i)), 0, 65535).astype(np.uint16)
        out.append(torch.from_numpy(a.view(np.int16)).cuda())
    torch.cuda.synchronize()
    return out


def _same_bits(x, y):
    return x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("dz,env", [(dz, {}) for dz in DZ] +
                         [(61, {"BS_FFT_XY_WINDOW": 2}), (61, {"BS_FFT_XY_KX": 100})])
def test_forward_matches_two_passes(ctx, monkeypatch, dz, env):
    dims = (512, 512, dz)
    ta, tb = _device_crops(dims, 11 * dz)
    _set_env(monkeypatch, **env)
    fa, fb, info = ctx.pcm_debug_pass(5, dims, ta, tb)
    assert info == XY, info
    _set_env(monkeypatch, BS_FFT_XY_FUSE=0)
    xa, xb, _ = ctx.pcm_debug_pass(0, dims, ta, tb)
    ya, yb, _ = ctx.pcm_debug_pass(1, dims, xa, xb)
    for got, ref in ((fa, ya), (fb, yb)):
        assert not np.isnan(got).any()
        assert _same_bits(got, ref), f"Pz {got.shape[0]}: {np.count_nonzero(got != ref)} bins differ"


def test_fused_pass_repeats_bit_identically(ctx, monkeypatch):
    dims = (512, 512, 61)
    ta, tb = _device_crops(dims, 3)
    _set_env(monkeypatch)
    first = ctx.pcm_debug_pass(5, dims, ta, tb)[:2]
    again = ctx.pcm_debug_pass(5, dims, ta, tb)[:2]
    for x, y in zip(first, again):
        assert _same_bits(x, y)


def test_dispatch_rule(ctx, monkeypatch):
    dims = (512, 512, 4)
    ta, tb = _device_crops(dims, 1)
    _set_env(monkeypatch)
    assert ctx.pcm_debug_pass(5, dims, ta, tb)[2] == XY
    # the switch keeps the five-pass chain
    _set_env(monkeypatch, BS_FFT_XY_FUSE=0)
    assert ctx.pcm_debug_pass(5, dims, ta, tb)[2] == "k_fft_x_r2c_col540 + k_fft_col540"
    # Py != 540: the y pass is not Col540's
    _set_env(monkeypatch)
    dims_y = (512, 480, 4)
    ua, ub = _device_crops(dims_y, 2)
    assert _geometry(dims_y)[0][1] != 540
    info = ctx.pcm_debug_pass(5, dims_y, ua, ub)[2]
    assert info.startswith("k_fft_x_r2c_col540 + ") and XY not in info, info
    # Pz = 3: 102 x tiles of 16 lines, fewer than the SMs
    dims_z = (512, 512, 1)
    va, vb = _device_crops(dims_z, 3)
    assert _geometry(dims_z)[0][2] == 3
    info = ctx.pcm_debug_pass(5, dims_z, va, vb)[2]
    assert XY not in info and "k_fft_x_r2c_col540" not in info and " + k_fft_col540" in info, info


def test_pair_results_identical(ctx, monkeypatch):
    from bsgpu import synthetic
    imgs1, imgs2, _ = synthetic.make_pcm_workload(1, n=512, device="cuda", seed=9, n_fields=1)
    p = ctx.pcm_params(peaks_to_check=5, do_subpixel=True, min_overlap_frac=0.25, extension=(10, 10, 10))
    res = {}
    for fuse in (0, 1):
        _set_env(monkeypatch, BS_FFT_XY_FUSE=fuse)
        res[fuse] = dataclasses.asdict(ctx.pcm_pair(imgs1[0], imgs2[0], p, dtype=None))
    assert res[1]["found"]
    assert res[0] == res[1]


def test_debug_pass_rejects_host_crops_and_unknown_passes(ctx):
    import bsgpu
    host = np.zeros((1, 4, 12), np.uint16)
    for pass_no in (0, 5):   # the x kernels read the crops directly: they must be device memory
        with pytest.raises(bsgpu.BsError, match="device crops"):
            ctx.pcm_debug_pass(pass_no, (12, 4, 1), host, host)
    z = np.zeros((3, 12, 17), np.complex64)
    with pytest.raises(bsgpu.BsError, match="not in"):
        ctx.pcm_debug_pass(6, (12, 4, 1), z, z)
