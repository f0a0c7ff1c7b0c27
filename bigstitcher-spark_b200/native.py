"""ctypes binding of libbsgpu.so (the C ABI declared in include/bsgpu.h).

This is the reference-side binding a maintainer would write in JNI (INTEGRATION.md shows the
Java stub); in this image there is no JVM, so the host side above the C ABI is Python.
There is NO CPU fallback: if the shared library is missing or no H100 is visible the calls
raise ``BsError`` -- they never route through oracle/.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbsgpu.so")

DTYPE_U16, DTYPE_F32, DTYPE_U8 = 0, 1, 2
_NP2BS = {np.dtype(np.uint16): DTYPE_U16, np.dtype(np.float32): DTYPE_F32, np.dtype(np.uint8): DTYPE_U8}
_BS2NP = {v: k for k, v in _NP2BS.items()}

(FUSE_AVG, FUSE_AVG_BLEND, FUSE_AVG_CONTENT, FUSE_AVG_BLEND_CONTENT, FUSE_MAX_INTENSITY,
 FUSE_LOWEST_VIEWID_WINS, FUSE_HIGHEST_VIEWID_WINS, FUSE_CLOSEST_PIXEL_WINS) = range(8)
FUSION_TYPES = {
    "AVG": FUSE_AVG, "AVG_BLEND": FUSE_AVG_BLEND, "AVG_CONTENT": FUSE_AVG_CONTENT,
    "AVG_BLEND_CONTENT": FUSE_AVG_BLEND_CONTENT, "MAX_INTENSITY": FUSE_MAX_INTENSITY,
    "LOWEST_VIEWID_WINS": FUSE_LOWEST_VIEWID_WINS, "HIGHEST_VIEWID_WINS": FUSE_HIGHEST_VIEWID_WINS,
    "CLOSEST_PIXEL_WINS": FUSE_CLOSEST_PIXEL_WINS,
}


class BsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libbsgpu error {code}: {msg}")
        self.code = code


class PcmParams(C.Structure):
    _fields_ = [("peaks_to_check", C.c_int), ("do_subpixel", C.c_int), ("interpolate_xcorr", C.c_int),
                ("min_overlap_frac", C.c_double), ("extension", C.c_int * 3)]


class PcmResultC(C.Structure):
    _fields_ = [("found", C.c_int), ("shift_int", C.c_longlong * 3), ("shift_sub", C.c_double * 3),
                ("r", C.c_double), ("n_overlap_px", C.c_longlong), ("peak_index", C.c_longlong * 3),
                ("pcm_value", C.c_double), ("pad", C.c_int * 3), ("n_candidates", C.c_int),
                ("pearson_px", C.c_longlong)]


class ViewC(C.Structure):
    _fields_ = [("src_to_world", C.c_double * 12), ("vol_handle", C.c_ulonglong),
                ("content_handle", C.c_ulonglong), ("blend_border", C.c_float * 3),
                ("blend_range", C.c_float * 3), ("full_dims", C.c_longlong * 3), ("window_min", C.c_longlong * 3)]


class NonrigidViewC(C.Structure):
    _fields_ = [("view", ViewC), ("n_points", C.c_int), ("pad", C.c_int),
                ("target_world_xyz", C.POINTER(C.c_double)), ("local_xyz", C.POINTER(C.c_double))]


class DogParamsC(C.Structure):
    _fields_ = [("sigma", C.c_double), ("threshold", C.c_double), ("min_intensity", C.c_double),
                ("max_intensity", C.c_double), ("find_max", C.c_int), ("find_min", C.c_int),
                ("localization", C.c_int), ("pad", C.c_int)]


class DogPointC(C.Structure):
    _fields_ = [("loc", C.c_double * 3), ("value", C.c_double), ("voxel", C.c_longlong * 3), ("is_max", C.c_int),
                ("pad", C.c_int)]


class SolveParamsC(C.Structure):
    _fields_ = [("transformation", C.c_int), ("regularization", C.c_int), ("lam", C.c_double), ("max_error", C.c_double),
                ("max_iterations", C.c_int), ("max_plateau_width", C.c_int)]


class SolveStatsC(C.Structure):
    _fields_ = [("iterations", C.c_int), ("stopped", C.c_int), ("skipped_fits", C.c_longlong), ("error", C.c_double),
                ("blocks", C.c_int), ("models_in_shared", C.c_int)]


#: model kinds of bs_solve_params (BS_MODEL_* in include/bsgpu.h)
SOLVE_MODELS = {"NONE": -1, "IDENTITY": 0, "TRANSLATION": 1, "RIGID": 2, "AFFINE": 3}


class IntensityViewC(C.Structure):
    _fields_ = [("vol_handle", C.c_ulonglong), ("world_to_px", C.c_double * 12), ("px_to_level", C.c_double * 12),
                ("full_dims", C.c_longlong * 3), ("n_cells", C.c_int * 3), ("pad", C.c_int)]


class IntensityParamsC(C.Structure):
    _fields_ = [("render_scale", C.c_double), ("min_threshold", C.c_double), ("max_threshold", C.c_double),
                ("render_min", C.c_longlong * 3), ("render_max", C.c_longlong * 3), ("chunk_points", C.c_longlong)]


class PcmJobC(C.Structure):
    _fields_ = [("vol1", C.c_ulonglong), ("vol2", C.c_ulonglong), ("min1", C.c_longlong * 3),
                ("min2", C.c_longlong * 3), ("dims", C.c_longlong * 3)]


def _out_dtype(params):
    """numpy dtype of a fused block: byte order follows params.out_big_endian (the bytes are what the device wrote)."""
    dt = np.dtype(_BS2NP[params.out_dtype])
    return dt.newbyteorder(">") if getattr(params, "out_big_endian", 0) and dt.itemsize > 1 else dt


class FuseParamsC(C.Structure):
    _fields_ = [("fusion_type", C.c_int), ("interpolation", C.c_int), ("out_dtype", C.c_int),
                ("blend_lut_n", C.c_int), ("min_intensity", C.c_double), ("max_intensity", C.c_double),
                ("out_big_endian", C.c_int), ("reserved", C.c_int)]


@dataclass
class PcmResult:
    found: bool
    shift_int: tuple
    shift_sub: tuple
    r: float
    n_overlap_px: int
    peak_index: tuple
    pcm_value: float
    pad: tuple
    n_candidates: int
    pearson_px: int = 0


_lib = None

#: every symbol include/bsgpu.h declares (checked by tests/test_abi.py against the header)
SYMBOLS = [
    "bs_version", "bs_init", "bs_destroy", "bs_last_error", "bs_synchronize", "bs_launch_count",
    "bs_profile_enable", "bs_profile_reset", "bs_profile_get", "bs_host_alloc", "bs_host_free",
    "bs_pcm_default_params", "bs_pcm_pair", "bs_pcm_batch", "bs_pcm_volumes_batch", "bs_good_fft_size", "bs_pcm_debug_pcm",
    "bs_pcm_debug_pearson", "bs_pcm_debug_pass",
    "bs_fuse_default_params", "bs_volume_upload", "bs_volume_upload_async", "bs_volume_wrap", "bs_volume_free",
    "bs_content_weights", "bs_volume_info", "bs_volume_download", "bs_volume_devptr", "bs_downsample", "bs_fuse_block", "bs_fuse_blocks",
    "bs_fuse_block_to_volume", "bs_fuse_accumulate", "bs_fuse_finish", "bs_mask_blocks", "bs_dog_default_params", "bs_dog_detect",
    "bs_dog_debug_dog", "bs_comm_unique_id", "bs_comm_init", "bs_comm_destroy", "bs_fuse_allreduce",
    "bs_downsample_float", "bs_median_divide", "bs_sample_nlinear", "bs_nonrigid_fuse_blocks", "bs_nonrigid_debug_grid",
    "bs_descriptors_build", "bs_descriptors_free", "bs_descriptors_neighbors", "bs_descriptors_match",
    "bs_solve_tiles",
    "bs_intensity_pair_candidates", "bs_intensity_candidates_get", "bs_intensity_candidates_free", "bs_intensity_ransac",
    "bs_intensity_apply", "bs_min_filter", "bs_volume_min_max", "bs_threshold_bbox", "bs_psf_accumulate",
]

#: fixed parameters of the reference's non-rigid fusion (J/SparkNonRigidFusion.java:373-383): control-point distance
NONRIGID_CP_DISTANCE = 10

#: largest num_neighbors + redundancy bs_descriptors_build accepts (BS_MATCH_MAX_NEIGHBORS in include/bsgpu.h)
MATCH_MAX_NEIGHBORS = 6

#: largest --medianFilter radius bs_median_divide accepts (BS_MEDIAN_MAX_RADIUS in include/bsgpu.h)
MEDIAN_MAX_RADIUS = 32


def load_library():
    """dlopen libbsgpu.so and declare prototypes.  Raises BsError if the extension was not
    built (run ``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BsError(-2, f"{LIB_PATH} is missing: build it with __graft_entry__.build(); "
                          "there is no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    vp, ip, ll, ull, dbl = C.c_void_p, C.c_int, C.c_longlong, C.c_ulonglong, C.c_double
    P = C.POINTER
    lib.bs_version.restype = ip
    lib.bs_init.argtypes = [P(vp), ip, vp]
    lib.bs_destroy.argtypes = [vp]
    lib.bs_destroy.restype = None
    lib.bs_last_error.argtypes = [vp]
    lib.bs_last_error.restype = C.c_char_p
    lib.bs_synchronize.argtypes = [vp]
    lib.bs_launch_count.argtypes = [vp]
    lib.bs_launch_count.restype = ll
    lib.bs_profile_enable.argtypes = [vp, ip]
    lib.bs_profile_reset.argtypes = [vp]
    lib.bs_profile_get.argtypes = [vp, C.c_char_p, P(dbl), P(ll)]
    lib.bs_host_alloc.argtypes = [vp, ull, P(vp)]
    lib.bs_host_free.argtypes = [vp, vp]
    lib.bs_pcm_default_params.argtypes = [P(PcmParams)]
    lib.bs_pcm_default_params.restype = None
    lib.bs_pcm_pair.argtypes = [vp, vp, vp, P(ll), ip, P(PcmParams), ip, P(PcmResultC)]
    lib.bs_pcm_batch.argtypes = [vp, ip, P(vp), P(vp), P(ll), ip, P(PcmParams), ip, P(PcmResultC)]
    lib.bs_good_fft_size.argtypes = [ip, ip]
    lib.bs_pcm_debug_pcm.argtypes = [vp, vp, vp, P(ll), ip, P(ip), vp, P(ip)]
    lib.bs_pcm_debug_pearson.argtypes = [vp, vp, vp, P(ll), ip, ip, P(ip), vp]
    lib.bs_pcm_debug_pass.argtypes = [vp, ip, P(ll), ip, P(ip), vp, vp, vp, vp, ip, P(ip), C.c_char_p]
    lib.bs_fuse_default_params.argtypes = [P(FuseParamsC)]
    lib.bs_fuse_default_params.restype = None
    lib.bs_volume_upload.argtypes = [vp, vp, P(ll), ip, P(ull)]
    lib.bs_volume_upload_async.argtypes = [vp, vp, P(ll), ip, P(ull)]
    lib.bs_pcm_volumes_batch.argtypes = [vp, ip, P(PcmJobC), P(PcmParams), P(PcmResultC)]
    lib.bs_volume_wrap.argtypes = [vp, vp, P(ll), ip, P(ull)]
    lib.bs_volume_free.argtypes = [vp, ull]
    lib.bs_content_weights.argtypes = [vp, ull, dbl, dbl, P(ull)]
    lib.bs_volume_info.argtypes = [vp, ull, P(ll), P(ip)]
    lib.bs_volume_download.argtypes = [vp, ull, vp, ull]
    lib.bs_volume_devptr.argtypes = [vp, ull, P(vp)]
    lib.bs_downsample.argtypes = [vp, ull, P(ip), P(ull)]
    lib.bs_fuse_block.argtypes = [vp, P(ViewC), ip, P(ll), P(ll), P(FuseParamsC), vp, ip]
    lib.bs_fuse_blocks.argtypes = [vp, P(ViewC), ip, ip, P(ll), P(ll), P(FuseParamsC), P(vp), ip]
    lib.bs_mask_blocks.argtypes = [vp, P(ViewC), ip, ip, P(ll), P(ll), P(C.c_double), ip, ip, P(vp), ip]
    lib.bs_fuse_block_to_volume.argtypes = [vp, P(ViewC), ip, P(ll), P(ll), P(FuseParamsC), P(ull)]
    lib.bs_fuse_accumulate.argtypes = [vp, P(ViewC), ip, P(ll), P(ll), P(FuseParamsC), vp, vp]
    lib.bs_fuse_finish.argtypes = [vp, vp, vp, ll, P(FuseParamsC), vp, ip]
    lib.bs_comm_unique_id.argtypes = [C.c_char_p]
    lib.bs_comm_init.argtypes = [vp, ip, ip, C.c_char_p]
    lib.bs_comm_destroy.argtypes = [vp]
    lib.bs_fuse_allreduce.argtypes = [vp, vp, vp, ll]
    lib.bs_dog_default_params.argtypes = [P(DogParamsC)]
    lib.bs_dog_default_params.restype = None
    lib.bs_dog_detect.argtypes = [vp, ull, P(ll), P(ll), P(DogParamsC), P(DogPointC), ip, P(ip)]
    lib.bs_dog_debug_dog.argtypes = [vp, ull, P(ll), P(ll), P(DogParamsC), ip, vp, C.c_char_p]
    lib.bs_downsample_float.argtypes = [vp, ull, P(ip), P(ull)]
    lib.bs_median_divide.argtypes = [vp, ull, ip, P(ull)]
    lib.bs_sample_nlinear.argtypes = [vp, ull, ip, P(dbl), vp]
    lib.bs_nonrigid_fuse_blocks.argtypes = [vp, P(NonrigidViewC), ip, ip, P(ll), P(ll), P(ll), P(FuseParamsC), P(vp), ip]
    lib.bs_nonrigid_debug_grid.argtypes = [vp, P(NonrigidViewC), P(ll), P(ll), P(ll), P(dbl), P(ll)]
    lib.bs_descriptors_build.argtypes = [vp, P(dbl), ip, ip, ip, P(ull)]
    lib.bs_descriptors_free.argtypes = [vp, ull]
    lib.bs_descriptors_neighbors.argtypes = [vp, ull, P(ip), P(dbl)]
    lib.bs_descriptors_match.argtypes = [vp, ull, ull, dbl, P(ip), P(dbl), P(dbl)]
    lib.bs_solve_tiles.argtypes = [vp, ip, ip, P(ip), P(ip), P(ip), ip, P(ip), P(ll), P(dbl), P(dbl), P(dbl),
                                   P(SolveParamsC), P(dbl), P(SolveStatsC), P(dbl), P(dbl), P(dbl)]
    lib.bs_intensity_pair_candidates.argtypes = [vp, P(IntensityViewC), P(IntensityViewC), P(IntensityParamsC), P(ull),
                                                 P(ll), P(ll)]
    lib.bs_intensity_candidates_get.argtypes = [vp, ull, P(ll), P(ll), P(ll), vp]
    lib.bs_intensity_candidates_free.argtypes = [vp, ull]
    lib.bs_intensity_ransac.argtypes = [vp, ull, ll, ip, dbl, P(dbl), P(dbl), P(ip)]
    lib.bs_intensity_apply.argtypes = [vp, ull, P(ll), P(ll), P(dbl), P(ip), P(dbl), P(dbl), P(ull)]
    lib.bs_min_filter.argtypes = [vp, ull, P(ip), P(ull)]
    lib.bs_volume_min_max.argtypes = [vp, ull, P(dbl)]
    lib.bs_threshold_bbox.argtypes = [vp, ull, dbl, P(ll), P(ll), P(ll)]
    lib.bs_psf_accumulate.argtypes = [vp, ull, P(ll), P(ll), P(dbl), ip, P(ip), P(dbl)]
    _lib = lib
    return lib


def good_fft_size(n: int, even: bool = False) -> int:
    return load_library().bs_good_fft_size(int(n), 1 if even else 0)


def _ptr_of(x):
    """(address, is_device, keepalive) for a numpy array / torch tensor / int device pointer."""
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise ValueError("array must be C-contiguous [z, y, x]")
        return x.ctypes.data, False, x
    if isinstance(x, int):
        return x, True, None
    if hasattr(x, "data_ptr"):  # torch tensor
        if not x.is_contiguous():
            raise ValueError("tensor must be contiguous")
        return x.data_ptr(), bool(x.is_cuda), x
    raise TypeError(f"unsupported buffer type {type(x)}")


def _bs_dtype(x, dtype=None):
    if dtype is not None:
        return dtype
    if isinstance(x, np.ndarray):
        return _NP2BS[x.dtype]
    import torch
    return {torch.uint16: DTYPE_U16, torch.int16: DTYPE_U16, torch.float32: DTYPE_F32,
            torch.uint8: DTYPE_U8}[x.dtype]


class Context:
    """One bs_ctx: bound to a device and a compute stream."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.bs_init(C.byref(h), int(device), C.c_void_p(stream) if stream else None)
        if rc != 0:
            raise BsError(rc, self.lib.bs_last_error(None).decode())
        self.h = h
        self.device = device
        self._desc_shape = {}      # descriptor handle -> (n, k)

    # -- plumbing
    def _check(self, rc):
        if rc != 0:
            raise BsError(rc, self.lib.bs_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.bs_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        self._check(self.lib.bs_synchronize(self.h))

    def launch_count(self) -> int:
        return int(self.lib.bs_launch_count(self.h))

    def profile_enable(self, on=True):
        self._check(self.lib.bs_profile_enable(self.h, 1 if on else 0))

    def profile_reset(self):
        self._check(self.lib.bs_profile_reset(self.h))

    def profile_get(self, tag: str):
        ms = C.c_double()
        n = C.c_longlong()
        self._check(self.lib.bs_profile_get(self.h, tag.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # -- hot path 1
    @staticmethod
    def pcm_params(peaks_to_check=5, do_subpixel=True, min_overlap_frac=0.25, extension=(10, 10, 10)):
        p = PcmParams()
        p.peaks_to_check = int(peaks_to_check)
        p.do_subpixel = 1 if do_subpixel else 0
        p.interpolate_xcorr = 0
        p.min_overlap_frac = float(min_overlap_frac)
        p.extension[:] = [int(e) for e in extension]
        return p

    @staticmethod
    def _result(r: PcmResultC) -> PcmResult:
        return PcmResult(bool(r.found), tuple(r.shift_int), tuple(r.shift_sub), r.r, r.n_overlap_px,
                         tuple(r.peak_index), r.pcm_value, tuple(r.pad), r.n_candidates, r.pearson_px)

    def pcm_pair(self, img1, img2, params: PcmParams | None = None, dims_xyz=None, dtype=None) -> PcmResult:
        """Phase correlation of one equal-size crop pair ([z,y,x] arrays, host or device)."""
        return self.pcm_batch([img1], [img2], params, [dims_xyz] if dims_xyz else None, dtype)[0]

    def pcm_batch(self, imgs1, imgs2, params: PcmParams | None = None, dims_xyz=None, dtype=None):
        n = len(imgs1)
        if len(imgs2) != n:
            raise ValueError("imgs1 / imgs2 length mismatch")
        params = params or self.pcm_params()
        a1 = (C.c_void_p * n)()
        a2 = (C.c_void_p * n)()
        dims = (C.c_longlong * (3 * n))()
        keep = []
        on_dev = None
        bs_dt = None
        for i in range(n):
            p1, d1, k1 = _ptr_of(imgs1[i])
            p2, d2, k2 = _ptr_of(imgs2[i])
            if d1 != d2 or (on_dev is not None and d1 != on_dev):
                raise ValueError("all images of a batch must live on the same side (host or device)")
            on_dev = d1
            keep += [k1, k2]
            a1[i], a2[i] = p1, p2
            if dims_xyz is not None:
                dx = dims_xyz[i]
            else:
                if tuple(imgs1[i].shape) != tuple(imgs2[i].shape):
                    raise ValueError("crops of a pair must have equal shape")
                dx = tuple(imgs1[i].shape)[::-1]
            dims[3 * i:3 * i + 3] = [int(v) for v in dx]
            dt = _bs_dtype(imgs1[i], dtype)
            if bs_dt is not None and dt != bs_dt:
                raise ValueError("mixed dtypes in one batch")
            bs_dt = dt
        out = (PcmResultC * n)()
        self._check(self.lib.bs_pcm_batch(self.h, n, a1, a2, dims, bs_dt or 0, C.byref(params),
                                          1 if on_dev else 0, out))
        return [self._result(out[i]) for i in range(n)]

    def pcm_volumes_batch(self, jobs, params: PcmParams | None = None):
        """jobs: iterable of (vol1, vol2, min1_xyz, min2_xyz, dims_xyz) on resident volumes; the overlap crops are
        cut on the device (a tile is uploaded once and reused by all its pairs)."""
        jobs = list(jobs)
        params = params or self.pcm_params()
        arr = (PcmJobC * max(1, len(jobs)))()
        for i, (v1, v2, m1, m2, d) in enumerate(jobs):
            arr[i].vol1, arr[i].vol2 = int(v1), int(v2)
            arr[i].min1[:] = [int(x) for x in m1]
            arr[i].min2[:] = [int(x) for x in m2]
            arr[i].dims[:] = [int(x) for x in d]
        out = (PcmResultC * max(1, len(jobs)))()
        self._check(self.lib.bs_pcm_volumes_batch(self.h, len(jobs), arr, C.byref(params), out))
        return [self._result(out[i]) for i in range(len(jobs))]

    def pcm_debug_pcm(self, img1: np.ndarray, img2: np.ndarray, extension=(10, 10, 10)) -> np.ndarray:
        dims = (C.c_longlong * 3)(*img1.shape[::-1])
        ext = (C.c_int * 3)(*extension)
        pad = (C.c_int * 3)()
        P = [good_fft_size(d + (2 * d if d < e else 2 * e), i == 0)
             for i, (d, e) in enumerate(zip(img1.shape[::-1], extension))]
        out = np.empty((P[2], P[1], P[0]), dtype=np.float32)
        self._check(self.lib.bs_pcm_debug_pcm(self.h, img1.ctypes.data, img2.ctypes.data, dims,
                                              _NP2BS[img1.dtype], ext, out.ctypes.data, pad))
        assert tuple(pad) == tuple(P)
        return out

    def pcm_debug_pass(self, pass_no: int, dims_xyz, in_a, in_b=None, dtype=None, extension=(10, 10, 10), poison=True):
        """Run one FFT pass of the PCM pipeline with the production launch (include/bsgpu.h bs_pcm_debug_pass states
        what each pass computes).  Passes 0 and 5 take two device crops ([z,y,x] CUDA tensors or int device pointers
        with ``dtype``); passes 1-4 take host complex64 spectra [Pz, Py, M+1].  Returns (out_a, out_b, info):
        complex64 spectra (out_b is None from pass 2 to 4), or for pass 4 the float32 PCM [Pz, Py, Px] as out_a."""
        dims = (C.c_longlong * 3)(*[int(v) for v in dims_xyz])
        ext = (C.c_int * 3)(*[int(e) for e in extension])
        P = [good_fft_size(d + (2 * d if d < e else 2 * e), i == 0) for i, (d, e) in enumerate(zip(dims_xyz, extension))]
        M = P[0] // 2
        spec_shape = (P[2], P[1], M + 1)
        keep = []
        if pass_no in (0, 5):
            # the library rejects crops that are not device memory or not of an image dtype
            (pa, _, ka), (pb, _, kb) = _ptr_of(in_a), _ptr_of(in_b)
            keep += [ka, kb]
            try:
                dt = _bs_dtype(in_a, dtype)
            except KeyError:
                dt = -1
        else:
            dt = DTYPE_F32
            ins = [in_a] + ([in_b] if pass_no <= 2 else [])
            for x in ins:
                x = np.ascontiguousarray(x, dtype=np.complex64)
                if x.shape != spec_shape:
                    raise ValueError(f"pass {pass_no} takes complex64 spectra of shape {spec_shape}, got {x.shape}")
                keep.append(x)
            pa = keep[0].ctypes.data
            pb = keep[1].ctypes.data if len(keep) > 1 else None
        out_a = np.empty((P[2], P[1], P[0]), np.float32) if pass_no == 4 else np.empty(spec_shape, np.complex64)
        out_b = np.empty(spec_shape, np.complex64) if pass_no in (0, 1, 5) else None
        pad = (C.c_int * 3)()
        info = C.create_string_buffer(128)
        self._check(self.lib.bs_pcm_debug_pass(self.h, int(pass_no), dims, dt, ext, pa, pb, out_a.ctypes.data,
                                               out_b.ctypes.data if out_b is not None else None, 1 if poison else 0,
                                               pad, info))
        assert tuple(pad) == tuple(P)
        return out_a, out_b, info.value.decode()

    def pcm_debug_pearson(self, img1, img2, boxes, dtype=None) -> np.ndarray:
        """Pearson sums of explicit candidate boxes on two equal-shape crops on the device ([z,y,x] CUDA tensors),
        computed by the production Pearson launch.  boxes: (n, 9) ints {o1 xyz, o2 xyz, sz xyz}.  Returns
        (n, 5) {sum a, sum b, sum a^2, sum b^2, sum ab}: uint64 for integer input, float64 for float32."""
        p1, d1, _ = _ptr_of(img1)
        p2, d2, _ = _ptr_of(img2)
        if not (d1 and d2):
            raise ValueError("pcm_debug_pearson takes device tensors")
        if tuple(img1.shape) != tuple(img2.shape):
            raise ValueError("crops of a pair must have equal shape")
        dims = (C.c_longlong * 3)(*[int(v) for v in tuple(img1.shape)[::-1]])
        bx = np.ascontiguousarray(np.asarray(boxes, dtype=np.int32).reshape(-1, 9))
        dt = _bs_dtype(img1, dtype)
        out = np.zeros((max(len(bx), 1), 5), dtype=np.float64 if dt == DTYPE_F32 else np.uint64)
        self._check(self.lib.bs_pcm_debug_pearson(self.h, p1, p2, dims, dt, len(bx),
                                                  bx.ctypes.data_as(C.POINTER(C.c_int)), out.ctypes.data))
        return out[:len(bx)]

    # -- hot path 2
    def volume_upload(self, vol: np.ndarray) -> int:
        dims = (C.c_longlong * 3)(*vol.shape[::-1])
        h = C.c_ulonglong()
        vol = np.ascontiguousarray(vol)
        self._check(self.lib.bs_volume_upload(self.h, vol.ctypes.data, dims, _NP2BS[vol.dtype], C.byref(h)))
        return h.value

    def volume_upload_async(self, vol) -> int:
        """Queue the H2D copy of a PINNED host array (numpy view of a pinned buffer / pinned torch tensor) on the
        copy stream; later calls using the handle wait for it on the device.  The array must stay alive."""
        p, on_dev, _ = _ptr_of(vol)
        if on_dev:
            raise ValueError("volume_upload_async needs a host buffer")
        dims = (C.c_longlong * 3)(*tuple(vol.shape)[::-1])
        h = C.c_ulonglong()
        self._check(self.lib.bs_volume_upload_async(self.h, p, dims, _bs_dtype(vol), C.byref(h)))
        return h.value

    def volume_wrap(self, dev_ptr, dims_xyz, dtype) -> int:
        p, is_dev, _ = _ptr_of(dev_ptr)
        dims = (C.c_longlong * 3)(*[int(v) for v in dims_xyz])
        h = C.c_ulonglong()
        self._check(self.lib.bs_volume_wrap(self.h, p, dims, dtype, C.byref(h)))
        return h.value

    def volume_empty(self, dims_xyz):
        """A new resident float32 volume of uninitialised device memory, allocated by torch on this context's device
        and wrapped (bs_volume_wrap).  Returns (handle, tensor [z, y, x]); the tensor owns the memory and must outlive
        the handle."""
        import torch
        t = torch.empty(tuple(int(v) for v in dims_xyz)[::-1], dtype=torch.float32, device=f"cuda:{self.device}")
        return self.volume_wrap(t, dims_xyz, DTYPE_F32), t

    def memory_free(self) -> int:
        """Free bytes on this context's device."""
        import torch
        return int(torch.cuda.mem_get_info(self.device)[0])

    def downsample(self, handle: int, factors_xyz) -> int:
        f = (C.c_int * 3)(*[int(v) for v in factors_xyz])
        h = C.c_ulonglong()
        self._check(self.lib.bs_downsample(self.h, handle, f, C.byref(h)))
        return h.value

    def volume_devptr(self, handle: int) -> int:
        p = C.c_void_p()
        self._check(self.lib.bs_volume_devptr(self.h, handle, C.byref(p)))
        return int(p.value)

    def volume_free(self, handle: int):
        self._check(self.lib.bs_volume_free(self.h, handle))

    def content_weights(self, handle: int, sigma1=20.0, sigma2=40.0) -> int:
        h = C.c_ulonglong()
        self._check(self.lib.bs_content_weights(self.h, handle, float(sigma1), float(sigma2), C.byref(h)))
        return h.value

    def volume_info(self, handle: int):
        """(dims_xyz, numpy dtype) of a resident volume."""
        dims = (C.c_longlong * 3)()
        dt = C.c_int()
        self._check(self.lib.bs_volume_info(self.h, handle, dims, C.byref(dt)))
        return tuple(int(v) for v in dims), _BS2NP[dt.value]

    def volume_download(self, handle: int, dims_xyz=None, dtype=None) -> np.ndarray:
        """Shape and dtype come from the handle; ``dims_xyz`` / ``dtype`` are only checked when given."""
        dims, dt = self.volume_info(handle)
        if dims_xyz is not None and tuple(int(v) for v in dims_xyz) != dims:
            raise ValueError(f"volume {handle} has dims {dims}, caller expected {tuple(dims_xyz)}")
        if dtype is not None and np.dtype(dtype) != dt:
            raise ValueError(f"volume {handle} has dtype {dt}, caller expected {np.dtype(dtype)}")
        out = np.empty(dims[::-1], dtype=dt)
        self._check(self.lib.bs_volume_download(self.h, handle, out.ctypes.data, out.nbytes))
        return out

    # -- next row: DoG interest points
    def dog_detect(self, handle: int, interval_min_xyz, interval_size_xyz, sigma=1.8, threshold=0.008, min_intensity=0.0,
                   max_intensity=65535.0, find_max=True, find_min=False, localization=True, max_points=1 << 16):
        """DoG detections of one block of a resident view: list of (loc_xyz, value, voxel_xyz, is_max) sorted by
        (z, y, x).  The buffer grows until every detection fits."""
        p = DogParamsC(float(sigma), float(threshold), float(min_intensity), float(max_intensity),
                       1 if find_max else 0, 1 if find_min else 0, 1 if localization else 0, 0)
        mn = (C.c_longlong * 3)(*[int(v) for v in interval_min_xyz])
        sz = (C.c_longlong * 3)(*[int(v) for v in interval_size_xyz])
        while True:
            buf = (DogPointC * max(1, max_points))()
            n = C.c_int()
            self._check(self.lib.bs_dog_detect(self.h, handle, mn, sz, C.byref(p), buf, max_points, C.byref(n)))
            if n.value <= max_points:
                break
            max_points = n.value
        return [(tuple(buf[i].loc), buf[i].value, tuple(buf[i].voxel), bool(buf[i].is_max)) for i in range(n.value)]

    def dog_debug_dog(self, handle: int, interval_min_xyz, interval_size_xyz, sigma=1.8, min_intensity=0.0,
                      max_intensity=65535.0, blur=0):
        """The DoG box dog_detect's extremum stage reads for this interval (include/bsgpu.h bs_dog_debug_dog): float32
        [sz + 2, sy + 2, sx + 2] over [min - 1, min + size + 1) per axis, and the blur instantiation launched.
        blur: 0 production choice, 1 generic, 2 window R 6, 3 window R 12."""
        p = DogParamsC(float(sigma), 0.0, float(min_intensity), float(max_intensity), 1, 0, 1, 0)
        mn = (C.c_longlong * 3)(*[int(v) for v in interval_min_xyz])
        sz = (C.c_longlong * 3)(*[int(v) for v in interval_size_xyz])
        out = np.empty([int(v) + 2 for v in interval_size_xyz][::-1], dtype=np.float32)
        info = C.create_string_buffer(128)
        self._check(self.lib.bs_dog_debug_dog(self.h, handle, mn, sz, C.byref(p), int(blur), out.ctypes.data, info))
        return out, info.value.decode()

    # -- detect-interestpoints helpers
    def downsample_float(self, handle: int, factors_xyz) -> int:
        """New float32 volume: the LazyDownsample2x chain (every x halving, then y, then z; 0.5f * (a + b), floor dims)
        of a resident volume; ``factors_xyz`` are powers of two <= 128 (all 1: a float copy)."""
        f = (C.c_int * 3)(*[int(v) for v in factors_xyz])
        h = C.c_ulonglong()
        self._check(self.lib.bs_downsample_float(self.h, handle, f, C.byref(h)))
        return h.value

    def median_divide(self, handle: int, radius: int) -> int:
        """New float32 volume: every z-slice divided by its circular (ImageJ RankFilters) median of ``radius``, 0 where
        the median is <= 0 (``--medianFilter``)."""
        h = C.c_ulonglong()
        self._check(self.lib.bs_median_divide(self.h, handle, int(radius), C.byref(h)))
        return h.value

    def sample_nlinear(self, handle: int, loc_xyz) -> np.ndarray:
        """float32 n-linear samples (border extension) of a resident volume at (n, 3) pixel coordinates {x, y, z}."""
        loc = np.ascontiguousarray(np.asarray(loc_xyz, dtype=np.float64).reshape(-1, 3))
        out = np.empty(len(loc), dtype=np.float32)
        self._check(self.lib.bs_sample_nlinear(self.h, handle, len(loc), loc.ctypes.data_as(C.POINTER(C.c_double)),
                                               out.ctypes.data))
        return out

    @staticmethod
    def fuse_params(fusion_type=FUSE_AVG_BLEND, interpolation=1, out_dtype=DTYPE_F32, blend_lut_n=0,
                    min_intensity=0.0, max_intensity=65535.0, out_big_endian=False):
        p = FuseParamsC()
        p.fusion_type = FUSION_TYPES[fusion_type] if isinstance(fusion_type, str) else int(fusion_type)
        p.interpolation = int(interpolation)
        p.out_dtype = int(out_dtype)
        p.blend_lut_n = int(blend_lut_n)
        p.min_intensity = float(min_intensity)
        p.max_intensity = float(max_intensity)
        p.out_big_endian = 1 if out_big_endian else 0
        return p

    @staticmethod
    def make_views(views):
        """views: iterable of dicts(src_to_world=12 doubles, vol_handle, content_handle=0,
        blend_border=(3,), blend_range=(3,))."""
        views = list(views)
        arr = (ViewC * max(1, len(views)))()
        for i, v in enumerate(views):
            arr[i].src_to_world[:] = [float(x) for x in np.asarray(v["src_to_world"]).ravel()]
            arr[i].vol_handle = int(v["vol_handle"])
            arr[i].content_handle = int(v.get("content_handle", 0))
            arr[i].blend_border[:] = [float(x) for x in v.get("blend_border", (0, 0, 0))]
            arr[i].blend_range[:] = [float(x) for x in v.get("blend_range", (40, 40, 40))]
            arr[i].full_dims[:] = [int(x) for x in v.get("full_dims", (0, 0, 0))]
            arr[i].window_min[:] = [int(x) for x in v.get("window_min", (0, 0, 0))]
        return arr, len(views)

    def fuse_block(self, views, block_min_xyz, block_size_xyz, params: FuseParamsC | None = None, out=None):
        """Fuse one block; returns a numpy array [z,y,x] (or fills ``out``: numpy array or
        device tensor / pointer)."""
        params = params or self.fuse_params()
        arr, n = views if isinstance(views, tuple) else self.make_views(views)
        bmin = (C.c_longlong * 3)(*[int(v) for v in block_min_xyz])
        bsz = (C.c_longlong * 3)(*[int(v) for v in block_size_xyz])
        if out is None:
            out = np.empty(tuple(int(v) for v in block_size_xyz)[::-1], dtype=_out_dtype(params))
        p, on_dev, _ = _ptr_of(out)
        self._check(self.lib.bs_fuse_block(self.h, arr, n, bmin, bsz, C.byref(params), p, 1 if on_dev else 0))
        return out

    def fuse_blocks(self, views, block_mins_xyz, block_sizes_xyz, params: FuseParamsC | None = None, outs=None):
        """Fuse a list of blocks in one call (one plan pass + one launch).  ``outs``: list of numpy arrays or
        device tensors / pointers (all on the same side); allocated as numpy arrays when None."""
        params = params or self.fuse_params()
        arr, n = views if isinstance(views, tuple) else self.make_views(views)
        nb = len(block_mins_xyz)
        bmin = (C.c_longlong * (3 * max(nb, 1)))()
        bsz = (C.c_longlong * (3 * max(nb, 1)))()
        for i in range(nb):
            bmin[3 * i:3 * i + 3] = [int(v) for v in block_mins_xyz[i]]
            bsz[3 * i:3 * i + 3] = [int(v) for v in block_sizes_xyz[i]]
        if outs is None:
            outs = [np.empty(tuple(int(v) for v in s)[::-1], dtype=_out_dtype(params)) for s in block_sizes_xyz]
        ptrs = (C.c_void_p * max(nb, 1))()
        on_dev = None
        keep = []
        for i, o in enumerate(outs):
            p, d, k = _ptr_of(o)
            if on_dev is not None and d != on_dev:
                raise ValueError("all outputs must live on the same side (host or device)")
            on_dev = d
            ptrs[i] = p
            keep.append(k)
        self._check(self.lib.bs_fuse_blocks(self.h, arr, n, nb, bmin, bsz, C.byref(params), ptrs, 1 if on_dev else 0))
        return outs

    def mask_blocks(self, views, block_mins_xyz, block_sizes_xyz, mask_offset=(0.0, 0.0, 0.0), out_dtype=DTYPE_U8,
                    out_big_endian=False):
        """`--masks` mode for a list of blocks: arrays [z,y,x] that are 255 / 65535 / 1.0 where any view covers the
        voxel (views need src_to_world and full_dims or a resident volume; no image data is read)."""
        arr, n = views if isinstance(views, tuple) else self.make_views(views)
        nb = len(block_mins_xyz)
        bmin = (C.c_longlong * (3 * max(nb, 1)))()
        bsz = (C.c_longlong * (3 * max(nb, 1)))()
        for i in range(nb):
            bmin[3 * i:3 * i + 3] = [int(v) for v in block_mins_xyz[i]]
            bsz[3 * i:3 * i + 3] = [int(v) for v in block_sizes_xyz[i]]
        dt = np.dtype(_BS2NP[out_dtype])
        if out_big_endian and dt.itemsize > 1:
            dt = dt.newbyteorder(">")
        outs = [np.empty(tuple(int(v) for v in s)[::-1], dtype=dt) for s in block_sizes_xyz]
        ptrs = (C.c_void_p * max(nb, 1))(*[o.ctypes.data for o in outs])
        off = (C.c_double * 3)(*[float(v) for v in mask_offset])
        self._check(self.lib.bs_mask_blocks(self.h, arr, n, nb, bmin, bsz, off, int(out_dtype), 1 if out_big_endian else 0, ptrs, 0))
        return outs

    def fuse_block_to_volume(self, views, block_min_xyz, block_size_xyz, params: FuseParamsC | None = None) -> int:
        """Fuse one block into a new resident volume; returns its handle."""
        params = params or self.fuse_params()
        arr, n = views if isinstance(views, tuple) else self.make_views(views)
        bmin = (C.c_longlong * 3)(*[int(v) for v in block_min_xyz])
        bsz = (C.c_longlong * 3)(*[int(v) for v in block_size_xyz])
        h = C.c_ulonglong()
        self._check(self.lib.bs_fuse_block_to_volume(self.h, arr, n, bmin, bsz, C.byref(params), C.byref(h)))
        return h.value

    def fuse_accumulate(self, views, block_min_xyz, block_size_xyz, params, sum_wi, sum_w):
        arr, n = views if isinstance(views, tuple) else self.make_views(views)
        bmin = (C.c_longlong * 3)(*[int(v) for v in block_min_xyz])
        bsz = (C.c_longlong * 3)(*[int(v) for v in block_size_xyz])
        p1, d1, _ = _ptr_of(sum_wi)
        p2, d2, _ = _ptr_of(sum_w)
        if not (d1 and d2):
            raise ValueError("accumulators must be device buffers")
        self._check(self.lib.bs_fuse_accumulate(self.h, arr, n, bmin, bsz, C.byref(params), p1, p2))

    # -- nonrigid-fusion
    @staticmethod
    def make_nonrigid_views(views):
        """views: iterable of make_views dicts plus target_world_xyz and local_xyz ((n, 3) float64 each).  Returns the
        ctypes array, its length and the point arrays that must stay alive for the call."""
        views = list(views)
        base, n = Context.make_views(views)
        arr = (NonrigidViewC * max(1, n))()
        keep = []
        for i, v in enumerate(views):
            t = np.ascontiguousarray(np.asarray(v.get("target_world_xyz", np.zeros((0, 3))), dtype=np.float64).reshape(-1, 3))
            l = np.ascontiguousarray(np.asarray(v.get("local_xyz", np.zeros((0, 3))), dtype=np.float64).reshape(-1, 3))
            if t.shape != l.shape:
                raise ValueError("target_world_xyz and local_xyz must have the same shape")
            keep += [t, l]
            arr[i].view = base[i]
            arr[i].n_points = len(t)
            arr[i].target_world_xyz = t.ctypes.data_as(C.POINTER(C.c_double))
            arr[i].local_xyz = l.ctypes.data_as(C.POINTER(C.c_double))
        return arr, n, keep

    def nonrigid_fuse_blocks(self, views, block_mins_xyz, block_sizes_xyz, params: FuseParamsC | None = None,
                             cp_distance=(NONRIGID_CP_DISTANCE,) * 3, outs=None):
        """Non-rigid AVG_BLEND fusion of a list of blocks (include/bsgpu.h bs_nonrigid_fuse_blocks).  ``views``: dicts
        as for make_nonrigid_views; ``outs``: numpy arrays or device tensors / pointers, allocated when None."""
        params = params or self.fuse_params()
        arr, n, keep = self.make_nonrigid_views(views)
        nb = len(block_mins_xyz)
        bmin = (C.c_longlong * (3 * max(nb, 1)))()
        bsz = (C.c_longlong * (3 * max(nb, 1)))()
        for i in range(nb):
            bmin[3 * i:3 * i + 3] = [int(v) for v in block_mins_xyz[i]]
            bsz[3 * i:3 * i + 3] = [int(v) for v in block_sizes_xyz[i]]
        if outs is None:
            outs = [np.empty(tuple(int(v) for v in s)[::-1], dtype=_out_dtype(params)) for s in block_sizes_xyz]
        ptrs = (C.c_void_p * max(nb, 1))()
        on_dev = None
        for i, o in enumerate(outs):
            p, d, k = _ptr_of(o)
            if on_dev is not None and d != on_dev:
                raise ValueError("all outputs must live on the same side (host or device)")
            on_dev = d
            ptrs[i] = p
            keep.append(k)
        cpd = (C.c_longlong * 3)(*[int(v) for v in cp_distance])
        self._check(self.lib.bs_nonrigid_fuse_blocks(self.h, arr, n, nb, bmin, bsz, cpd, C.byref(params), ptrs,
                                                     1 if on_dev else 0))
        return outs

    def nonrigid_debug_grid(self, view, block_min_xyz, block_size_xyz, cp_distance=(NONRIGID_CP_DISTANCE,) * 3):
        """The mapped source coordinate of every control point of one view for one block: float64
        [gz, gy, gx, 3] ({x, y, z} last); control point (i, j, k) sits at world block_min + ((i, j, k) - 1) * cpd."""
        arr, _, keep = self.make_nonrigid_views([view])
        bmin = (C.c_longlong * 3)(*[int(v) for v in block_min_xyz])
        bsz = (C.c_longlong * 3)(*[int(v) for v in block_size_xyz])
        cpd = (C.c_longlong * 3)(*[int(v) for v in cp_distance])
        gd = (C.c_longlong * 3)()
        self._check(self.lib.bs_nonrigid_debug_grid(self.h, arr, bmin, bsz, cpd, None, gd))
        out = np.empty((gd[2], gd[1], gd[0], 3), dtype=np.float64)
        self._check(self.lib.bs_nonrigid_debug_grid(self.h, arr, bmin, bsz, cpd, out.ctypes.data_as(C.POINTER(C.c_double)), gd))
        return out

    # -- match-interestpoints
    def descriptors_build(self, xyz, num_neighbors=3, redundancy=1) -> int:
        """Resident local descriptors of (n, 3) float64 world points: every point's num_neighbors + redundancy nearest
        other points in (squared distance, index) order, kept as relative vectors (include/bsgpu.h)."""
        p = np.ascontiguousarray(np.asarray(xyz, dtype=np.float64).reshape(-1, 3))
        h = C.c_ulonglong()
        self._check(self.lib.bs_descriptors_build(self.h, p.ctypes.data_as(C.POINTER(C.c_double)), len(p),
                                                  int(num_neighbors), int(redundancy), C.byref(h)))
        self._desc_shape[h.value] = (len(p), int(num_neighbors) + int(redundancy))
        return h.value

    def descriptors_neighbors(self, handle: int):
        """(idx int32 (n, k), d2 float64 (n, k)) of a descriptor set; -1 / inf everywhere when n <= k."""
        n, k = self._desc_shape[handle]
        idx = np.empty((n, k), dtype=np.int32)
        d2 = np.empty((n, k), dtype=np.float64)
        self._check(self.lib.bs_descriptors_neighbors(self.h, handle, idx.ctypes.data_as(C.POINTER(C.c_int)),
                                                      d2.ctypes.data_as(C.POINTER(C.c_double))))
        return idx, d2

    def descriptors_match(self, ha: int, hb: int, search_radius=None):
        """Exhaustive descriptor search A -> B: (best_b int32 (nA,), best float64, second float64); best_b = -1 where no
        point of B qualifies.  ``search_radius`` None: every point of B."""
        n = self._desc_shape[ha][0]
        best_b = np.empty(n, dtype=np.int32)
        best = np.empty(n, dtype=np.float64)
        second = np.empty(n, dtype=np.float64)
        r = -1.0 if search_radius is None else float(search_radius)
        self._check(self.lib.bs_descriptors_match(self.h, ha, hb, r, best_b.ctypes.data_as(C.POINTER(C.c_int)),
                                                  best.ctypes.data_as(C.POINTER(C.c_double)),
                                                  second.ctypes.data_as(C.POINTER(C.c_double))))
        return best_b, best, second

    def descriptors_free(self, handle: int):
        self._check(self.lib.bs_descriptors_free(self.h, handle))
        self._desc_shape.pop(handle, None)

    # -- solver
    def solve_tiles(self, colour_offsets, colour_tiles, fixed, links, match_offsets, p, q, w, models,
                    transformation="AFFINE", regularization="RIGID", lam=0.1, max_error=5.0, max_iterations=10000,
                    max_plateau_width=200):
        """The device relaxation of one solve (include/bsgpu.h bs_solve_tiles) from the starting ``models`` (T, 3, 4).
        Returns (models (T, 3, 4), stats dict, tile_error (T,), link_mean (L,), link_max (L,))."""
        def arr(x, dt, shape=(-1,)):
            return np.ascontiguousarray(np.asarray(x, dtype=dt).reshape(shape))
        co, ct, fx = arr(colour_offsets, np.int32), arr(colour_tiles, np.int32), arr(fixed, np.int32)
        lk, mo = arr(links, np.int32, (-1, 2)), arr(match_offsets, np.int64)
        pp, qq, ww = arr(p, np.float64, (-1, 3)), arr(q, np.float64, (-1, 3)), arr(w, np.float64)
        M = np.array(models, dtype=np.float64).reshape(-1, 3, 4).copy()
        T, L = len(M), len(lk)
        if len(co) < 1:
            raise ValueError("colour_offsets needs at least one entry")
        prm = SolveParamsC(SOLVE_MODELS[transformation.upper()], SOLVE_MODELS[regularization.upper()], float(lam),
                           float(max_error), int(max_iterations), int(max_plateau_width))
        st = SolveStatsC()
        te, lm, lx = np.zeros(T), np.zeros(max(L, 1)), np.zeros(max(L, 1))
        I, LL, D = C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_double)
        if L and len(mo) != L + 1:
            raise ValueError("match_offsets needs n_links + 1 entries")
        self._check(self.lib.bs_solve_tiles(self.h, T, len(co) - 1, co.ctypes.data_as(I), ct.ctypes.data_as(I),
                                            fx.ctypes.data_as(I), L, lk.ctypes.data_as(I), mo.ctypes.data_as(LL),
                                            pp.ctypes.data_as(D), qq.ctypes.data_as(D), ww.ctypes.data_as(D), C.byref(prm),
                                            M.ctypes.data_as(D), C.byref(st), te.ctypes.data_as(D), lm.ctypes.data_as(D),
                                            lx.ctypes.data_as(D)))
        stats = dict(iterations=st.iterations, error=st.error, skipped_fits=st.skipped_fits, stopped=bool(st.stopped),
                     blocks=st.blocks, models_in_shared=bool(st.models_in_shared))
        return M, stats, te, lm[:L], lx[:L]

    # -- intensity correction
    @staticmethod
    def _intensity_view(v):
        c = IntensityViewC()
        c.vol_handle = int(v["vol_handle"])
        c.world_to_px[:] = [float(x) for x in np.asarray(v["world_to_px"], dtype=np.float64).ravel()]
        c.px_to_level[:] = [float(x) for x in np.asarray(v["px_to_level"], dtype=np.float64).ravel()]
        c.full_dims[:] = [int(x) for x in v["full_dims"]]
        c.n_cells[:] = [int(x) for x in v["n_cells"]]
        return c

    def intensity_candidates(self, view_a, view_b, render_scale, render_min, render_max, min_threshold=1.0,
                             max_threshold=float("nan"), chunk_points=0):
        """Candidates of one view pair (include/bsgpu.h bs_intensity_pair_candidates), kept resident.  ``view_a`` /
        ``view_b``: dicts(vol_handle, world_to_px (3, 4), px_to_level (3, 4), full_dims, n_cells).  Returns
        (handle, keys int64, offsets int64, counts int64, values float32 (n, 2)); free the handle with
        intensity_candidates_free."""
        a, b = self._intensity_view(view_a), self._intensity_view(view_b)
        p = IntensityParamsC(float(render_scale), float(min_threshold), float(max_threshold),
                             (C.c_longlong * 3)(*[int(v) for v in render_min]),
                             (C.c_longlong * 3)(*[int(v) for v in render_max]), int(chunk_points))
        h, nb, nv = C.c_ulonglong(), C.c_longlong(), C.c_longlong()
        self._check(self.lib.bs_intensity_pair_candidates(self.h, C.byref(a), C.byref(b), C.byref(p), C.byref(h),
                                                          C.byref(nb), C.byref(nv)))
        keys, off, cnt = (np.empty(max(nb.value, 1), dtype=np.int64) for _ in range(3))
        vals = np.empty((max(nv.value, 1), 2), dtype=np.float32)
        LL = C.POINTER(C.c_longlong)
        self._check(self.lib.bs_intensity_candidates_get(self.h, h.value, keys.ctypes.data_as(LL), off.ctypes.data_as(LL),
                                                         cnt.ctypes.data_as(LL), vals.ctypes.data))
        return h.value, keys[:nb.value], off[:nb.value], cnt[:nb.value], vals[:nv.value]

    def intensity_candidates_free(self, handle: int):
        self._check(self.lib.bs_intensity_candidates_free(self.h, handle))

    def intensity_ransac(self, handle: int, n_buckets: int, min_num_candidates=1000, num_iterations=1000, max_epsilon=5.1):
        """Best RANSAC hypothesis per bucket of a resident candidate set: (a, b, count) arrays; count -1 for buckets
        below ``min_num_candidates``."""
        n = max(int(n_buckets), 1)
        a, b, cnt = np.empty(n), np.empty(n), np.empty(n, dtype=np.int32)
        D = C.POINTER(C.c_double)
        self._check(self.lib.bs_intensity_ransac(self.h, handle, int(min_num_candidates), int(num_iterations),
                                                 float(max_epsilon), a.ctypes.data_as(D), b.ctypes.data_as(D),
                                                 cnt.ctypes.data_as(C.POINTER(C.c_int))))
        return a[:n_buckets], b[:n_buckets], cnt[:n_buckets]

    def intensity_apply(self, handle: int, full_dims_xyz, level_to_full, coeff_a, coeff_b, window_min_xyz=(0, 0, 0)) -> int:
        """New float32 volume a(q) v + b(q) of a resident (window of a) level volume; ``coeff_a`` / ``coeff_b``:
        cell values [nz, ny, nx]."""
        ca = np.ascontiguousarray(coeff_a, dtype=np.float64)
        cb = np.ascontiguousarray(coeff_b, dtype=np.float64)
        if ca.ndim != 3 or ca.shape != cb.shape:
            raise ValueError("coefficients must be two [nz, ny, nx] arrays of one shape")
        fd = (C.c_longlong * 3)(*[int(v) for v in full_dims_xyz])
        wm = (C.c_longlong * 3)(*[int(v) for v in window_min_xyz])
        m = (C.c_double * 12)(*[float(x) for x in np.asarray(level_to_full, dtype=np.float64).ravel()])
        n = (C.c_int * 3)(*ca.shape[::-1])
        h = C.c_ulonglong()
        D = C.POINTER(C.c_double)
        self._check(self.lib.bs_intensity_apply(self.h, handle, fd, wm, m, n, ca.ctypes.data_as(D), cb.ctypes.data_as(D),
                                                C.byref(h)))
        return h.value

    # -- estimate-bounding-box
    def min_filter(self, handle: int, radius_xyz) -> int:
        """New float32 volume: the minimum over the box of ``radius_xyz`` around every voxel, clipped to the volume
        (NaN neighbours ignored) of a resident float32 volume."""
        r = (C.c_int * 3)(*[int(v) for v in radius_xyz])
        h = C.c_ulonglong()
        self._check(self.lib.bs_min_filter(self.h, handle, r, C.byref(h)))
        return h.value

    def volume_min_max(self, handle: int):
        """(min, max) of a resident float32 volume over its voxels that are not NaN; (nan, nan) when there are none."""
        out = (C.c_double * 2)()
        self._check(self.lib.bs_volume_min_max(self.h, handle, out))
        return out[0], out[1]

    def threshold_bbox(self, handle: int, t: float):
        """(min_xyz, max_xyz, count) of the voxels of a resident float32 volume that are > ``t`` (compared in double);
        (-1, -1, -1) twice and 0 when there are none."""
        mn, mx, n = (C.c_longlong * 3)(), (C.c_longlong * 3)(), C.c_longlong()
        self._check(self.lib.bs_threshold_bbox(self.h, handle, float(t), mn, mx, C.byref(n)))
        return tuple(mn), tuple(mx), n.value

    # -- extract-psfs
    def psf_accumulate(self, handle: int, window_min_xyz, full_dims_xyz, points_xyz, psf_size_xyz, sum=None):
        """Add, for every point in the order given, the n-linear samples (PARITY_GAPS #37, border extension of the
        full view of size ``full_dims_xyz``) of the PSF box of odd size ``psf_size_xyz`` around the point to ``sum``
        (float64 [sz, sy, sx], updated in place; zeros when None) and return it.  The resident volume is the window of
        the view's full-resolution level that starts at ``window_min_xyz``; points are full-resolution pixels."""
        s = [int(v) for v in psf_size_xyz]
        if sum is None:
            sum = np.zeros(s[::-1], dtype=np.float64)
        if sum.dtype != np.float64 or not sum.flags.c_contiguous or sum.size != int(np.prod(s)):
            raise ValueError(f"psf_accumulate: sum must be a C-contiguous float64 array of {s[::-1]}")
        pts = np.ascontiguousarray(np.asarray(points_xyz, dtype=np.float64).reshape(-1, 3))
        self._check(self.lib.bs_psf_accumulate(
            self.h, handle, (C.c_longlong * 3)(*[int(v) for v in window_min_xyz]),
            (C.c_longlong * 3)(*[int(v) for v in full_dims_xyz]), pts.ctypes.data_as(C.POINTER(C.c_double)), len(pts),
            (C.c_int * 3)(*s), sum.ctypes.data_as(C.POINTER(C.c_double))))
        return sum

    @staticmethod
    def comm_unique_id() -> bytes:
        """rank 0: a fresh 128-byte NCCL id to hand to every rank (any host channel)."""
        lib = load_library()
        buf = C.create_string_buffer(128)
        rc = lib.bs_comm_unique_id(buf)
        if rc != 0:
            raise BsError(rc, lib.bs_last_error(None).decode())
        return buf.raw

    def comm_init(self, n_ranks: int, rank: int, unique_id: bytes):
        self._check(self.lib.bs_comm_init(self.h, int(n_ranks), int(rank), unique_id))

    def comm_destroy(self):
        self._check(self.lib.bs_comm_destroy(self.h))

    def fuse_allreduce(self, sum_wi, sum_w, n_elems):
        """In-place SUM of both partial buffers over the ranks of bs_comm_init (NCCL, on this context's stream)."""
        p1, d1, _ = _ptr_of(sum_wi)
        p2, d2, _ = _ptr_of(sum_w)
        if not (d1 and d2):
            raise ValueError("accumulators must be device buffers")
        self._check(self.lib.bs_fuse_allreduce(self.h, p1, p2, int(n_elems)))

    def fuse_finish(self, sum_wi, sum_w, n_elems, params, out):
        p1, _, _ = _ptr_of(sum_wi)
        p2, _, _ = _ptr_of(sum_w)
        p, on_dev, _ = _ptr_of(out)
        self._check(self.lib.bs_fuse_finish(self.h, p1, p2, int(n_elems), C.byref(params), p, 1 if on_dev else 0))
        return out
