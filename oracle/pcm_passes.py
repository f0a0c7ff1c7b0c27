"""Float64 reference of each FFT pass of the device PCM pipeline (include/bsgpu.h, bs_pcm_debug_pass).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle/``.  Spectra are [Pz, Py, M+1] arrays (x fastest, M = Px / 2),
every transform is an unnormalised forward DFT along one axis, computed in complex128:

  pass 0  rfft along x of pcm_oracle.blend_extend_pad's float32 volume
  pass 1  fft along y (both spectra)
  pass 2  fft_z(conj(n(fft_z A)) * n(fft_z B)), n(c) = c / |c| or 0 when |c| < the normalisation threshold
  pass 3  fft along y
  pass 4  irfft(conj(H), Px) / (Py * Pz) along x

The conjugations make passes 3 and 4 inverse transforms, so ``pcm`` (the five composed) equals
pcm_oracle.calculate_pcm evaluated in float64.  The helpers at the end compute the per-line error measures the
GPU tests use.
"""
from __future__ import annotations

import numpy as np
import scipy.fft as sfft

from oracle import pcm_oracle as po

#: |c| threshold of the unit-magnitude normalisation, as the float32 value both the oracle and the device use
THRESHOLD = float(np.float32(po.NORMALIZATION_THRESHOLD))


def padded_volume(img: np.ndarray, extension=(po.DEFAULT_EXTENSION,) * 3) -> np.ndarray:
    """float32 [Pz, Py, Px] input of pass 0 (blended mirrored extension + zero pad)."""
    P = po.padded_dims(img.shape[::-1], extension)
    return po.blend_extend_pad(img, extension, P)


def normalize(c: np.ndarray) -> np.ndarray:
    mag = np.abs(c)
    out = np.zeros_like(c)
    np.divide(c, mag, out=out, where=mag >= THRESHOLD)
    return out


def pass0(img: np.ndarray, extension=(po.DEFAULT_EXTENSION,) * 3) -> np.ndarray:
    return np.fft.rfft(padded_volume(img, extension).astype(np.float64), axis=2)


def pass1(spec: np.ndarray) -> np.ndarray:
    return np.fft.fft(np.asarray(spec, np.complex128), axis=1)


def pass2(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    fa = normalize(np.fft.fft(np.asarray(a, np.complex128), axis=0))
    fb = normalize(np.fft.fft(np.asarray(b, np.complex128), axis=0))
    return np.fft.fft(np.conj(fa) * fb, axis=0)


def pass3(spec: np.ndarray) -> np.ndarray:
    return np.fft.fft(np.asarray(spec, np.complex128), axis=1)


def pass4(spec: np.ndarray, px: int) -> np.ndarray:
    h = np.asarray(spec, np.complex128)
    return np.fft.irfft(np.conj(h), n=px, axis=2) / (h.shape[0] * h.shape[1])


def pcm(img1: np.ndarray, img2: np.ndarray, extension=(po.DEFAULT_EXTENSION,) * 3) -> np.ndarray:
    """The five passes composed: float64 PCM [Pz, Py, Px]."""
    px = po.padded_dims(img1.shape[::-1], extension)[0]
    a = pass1(pass0(img1, extension))
    b = pass1(pass0(img2, extension))
    return pass4(pass3(pass2(a, b)), px)


# ---- what scipy's single-precision FFT makes of the same pass (the yardstick of the GPU bars)
def pass0_f32(img, extension=(po.DEFAULT_EXTENSION,) * 3):
    return sfft.rfft(padded_volume(img, extension), axis=2)


def pass1_f32(spec):
    return sfft.fft(np.asarray(spec, np.complex64), axis=1)


def pass2_f32(a, b):
    def n32(c):
        mag = np.abs(c)
        out = np.zeros_like(c)
        np.divide(c, mag, out=out, where=mag >= np.float32(po.NORMALIZATION_THRESHOLD))
        return out
    fa = n32(sfft.fft(np.asarray(a, np.complex64), axis=0))
    fb = n32(sfft.fft(np.asarray(b, np.complex64), axis=0))
    return sfft.fft(np.conj(fa) * fb, axis=0)


pass3_f32 = pass1_f32


def pass4_f32(spec, px):
    h = np.asarray(spec, np.complex64)
    return (sfft.irfft(np.conj(h), n=px, axis=2) / np.float32(h.shape[0] * h.shape[1])).astype(np.float32)


# ---- error measures
def line_rel_l2(got: np.ndarray, ref: np.ndarray, axis: int):
    """Per-line relative L2 error ||got - ref|| / ||ref|| along ``axis``, and the mask of lines whose reference is
    not identically zero (the error is only defined there)."""
    g = np.moveaxis(np.asarray(got), axis, -1).astype(np.complex128)
    r = np.moveaxis(np.asarray(ref), axis, -1).astype(np.complex128)
    num = np.sqrt(np.sum(np.abs(g - r) ** 2, axis=-1))
    den = np.sqrt(np.sum(np.abs(r) ** 2, axis=-1))
    live = den > 0
    err = np.zeros_like(den)
    err[live] = num[live] / den[live]
    return err, live


def rel_l2(got: np.ndarray, ref: np.ndarray) -> float:
    """Relative L2 error of a whole array."""
    g = np.asarray(got, np.float64)
    r = np.asarray(ref, np.float64)
    return float(np.linalg.norm((g - r).ravel()) / np.linalg.norm(r.ravel()))
