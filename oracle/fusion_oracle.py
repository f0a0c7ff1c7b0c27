"""CPU oracle for hot path 2: per-block affine resample-and-blend fusion.

TEST INFRASTRUCTURE ONLY (see oracle/pcm_oracle.py header): never imported by the product.

PARITY UNPINNED.  The arithmetic lives in net.preibisch:multiview-reconstruction:8.0.0
(process.fusion.blk.BlkAffineFusion, process.fusion.transformed.TransformVirtual,
process.fusion.FusionTools; pom.xml:106) on top of imglib2-algorithm 0.18.2
(algorithm.blocks.transform.Transform, blocks.convert.Convert; pom.xml:101); none of it is
under /root/reference and the reference's tests assert nothing (SURVEY.md 4, 8c).  This
restates SURVEY.md Appendix A.2 at the call-site contract of
src/main/java/net/preibisch/bigstitcher/spark/SparkAffineFusion.java:602-627
(initWithIntensityCoefficients(conv, imgLoader, viewIds, registrations, descriptions,
fusionType, NaN, null, 1 /*linear*/, coefficients=null, boundingBox, type, blockSize) then
BlockAlgoUtils.arrayImg(supplier, [blockMin, blockMax])).  Uncertain choices are named
constants and listed in PARITY_GAPS.md.

Arrays are [z, y, x]; triples in the public API are (x, y, z) like the reference's long[]s.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

# FusionType ordinals (mvrecon FusionGUI.FusionType; CLI help SparkAffineFusion.java:124)
AVG, AVG_BLEND, AVG_CONTENT, AVG_BLEND_CONTENT, MAX_INTENSITY, LOWEST_VIEWID_WINS, \
    HIGHEST_VIEWID_WINS, CLOSEST_PIXEL_WINS = range(8)

#: FusionTools.defaultBlendingRange / defaultBlendingBorder (A.2 step 3, "(?)")
DEFAULT_BLENDING_RANGE = 40.0
DEFAULT_BLENDING_BORDER = 0.0
#: content-based weights: c = G_s2 * (I - G_s1 * I)^2  (A.2 step 3, "(?)")
DEFAULT_CONTENT_SIGMA1 = 20.0
DEFAULT_CONTENT_SIGMA2 = 40.0
#: size of upstream's (recalled) cosine lookup table in the blk code path; 0 = analytic cosine
BLEND_LUT_N = 30


def invert_affine(m12):
    """Invert a row-packed 3x4 affine (double)."""
    M = np.asarray(m12, dtype=np.float64).reshape(3, 4)
    A = M[:, :3]
    t = M[:, 3]
    Ai = np.linalg.inv(A)
    out = np.empty((3, 4))
    out[:, :3] = Ai
    out[:, 3] = -Ai @ t
    return out


def axis_scales(m12):
    """TransformationTools.scaling: per source axis, length of the transformed unit step
    (column norms of the linear part)."""
    M = np.asarray(m12, dtype=np.float64).reshape(3, 4)
    return np.sqrt((M[:, :3] ** 2).sum(axis=0))


def adjust_blending(m12, blending=DEFAULT_BLENDING_RANGE, border=DEFAULT_BLENDING_BORDER):
    """FusionTools.adjustBlending: range/border (float[3]) divided by (float) axis scale."""
    s = axis_scales(m12).astype(np.float32)
    b = (np.full(3, blending, dtype=np.float32) / s).astype(np.float32)
    bo = (np.full(3, border, dtype=np.float32) / s).astype(np.float32)
    return bo, b


def _cos_lut(n):
    lut = np.empty(n + 2, dtype=np.float32)
    for i in range(n + 1):
        lut[i] = np.float32((math.cos((1.0 - i / n) * math.pi) + 1.0) / 2.0)
    lut[n + 1] = lut[n]
    return lut


def blend_weight(src, dims_xyz, border, blending, lut_n=0):
    """Cosine blending weight per view (BlendingRealRandomAccess.computeWeight semantics):
    per axis l = source coordinate (float32), dist = max(0, min(l - border, dim-1 - l -
    border)); dist == 0 -> weight 0; relDist = dist/blending; relDist < 1 -> multiply by
    (cos((1-relDist)*pi)+1)/2 (evaluated in double, product kept in float32).
    ``src``: float32 array [..., 3] (x, y, z).  ``lut_n`` > 0 evaluates the cosine through a
    linear-interpolated table with n segments instead."""
    w = np.ones(src.shape[:-1], dtype=np.float32)
    zero = np.zeros(src.shape[:-1], dtype=bool)
    lut = _cos_lut(lut_n) if lut_n > 0 else None
    for d in range(3):
        l = src[..., d]
        dist = np.maximum(np.float32(0), np.minimum(l - np.float32(border[d]),
                                                    np.float32(dims_xyz[d] - 1) - l - np.float32(border[d])))
        zero |= dist == 0
        rel = (dist / np.float32(blending[d])).astype(np.float32)
        inside = rel < 1
        if lut is None:
            f = (np.cos((1.0 - rel.astype(np.float64)) * math.pi) + 1.0) / 2.0
            wf = (w.astype(np.float64) * f).astype(np.float32)
        else:
            relc = np.where(inside, rel, np.float32(0))
            pos = (relc * np.float32(lut_n)).astype(np.float32)
            i = pos.astype(np.int32)
            s = pos - i.astype(np.float32)
            f = lut[i] * (np.float32(1.0) - s) + lut[i + 1] * s
            wf = (w * f).astype(np.float32)
        w = np.where(inside, wf, w)
    w[zero] = 0
    return w


def inside_mask(src, dims_xyz):
    """AVG mask: 1 inside the closed interval [0, dim-1] on every axis."""
    m = np.ones(src.shape[:-1], dtype=bool)
    for d in range(3):
        m &= (src[..., d] >= 0) & (src[..., d] <= np.float32(dims_xyz[d] - 1))
    return m


def trilinear(img, src):
    """n-linear interpolation (interpolation arg 1) of ``img`` [z,y,x] converted to float32
    at float32 positions ``src`` [...,3]; border (clamp) extension; x then y then z lerps as
    a + f*(b-a) in float32."""
    dz, dy, dx = img.shape
    sx, sy, sz = src[..., 0], src[..., 1], src[..., 2]
    fx0 = np.floor(sx)
    fy0 = np.floor(sy)
    fz0 = np.floor(sz)
    rx = (sx - fx0).astype(np.float32)
    ry = (sy - fy0).astype(np.float32)
    rz = (sz - fz0).astype(np.float32)
    x0 = fx0.astype(np.int64)
    y0 = fy0.astype(np.int64)
    z0 = fz0.astype(np.int64)

    def cl(v, n):
        return np.clip(v, 0, n - 1)

    x0c, x1c = cl(x0, dx), cl(x0 + 1, dx)
    y0c, y1c = cl(y0, dy), cl(y0 + 1, dy)
    z0c, z1c = cl(z0, dz), cl(z0 + 1, dz)

    def g(zz, yy, xx):
        return img[zz, yy, xx].astype(np.float32)

    def lerp(a, b, f):
        return (a + f * (b - a)).astype(np.float32)

    c00 = lerp(g(z0c, y0c, x0c), g(z0c, y0c, x1c), rx)
    c01 = lerp(g(z0c, y1c, x0c), g(z0c, y1c, x1c), rx)
    c10 = lerp(g(z1c, y0c, x0c), g(z1c, y0c, x1c), rx)
    c11 = lerp(g(z1c, y1c, x0c), g(z1c, y1c, x1c), rx)
    c0 = lerp(c00, c01, ry)
    c1 = lerp(c10, c11, ry)
    return lerp(c0, c1, rz)


def nearest(img, src):
    dz, dy, dx = img.shape
    xi = np.clip(np.floor(src[..., 0] + np.float32(0.5)).astype(np.int64), 0, dx - 1)
    yi = np.clip(np.floor(src[..., 1] + np.float32(0.5)).astype(np.int64), 0, dy - 1)
    zi = np.clip(np.floor(src[..., 2] + np.float32(0.5)).astype(np.int64), 0, dz - 1)
    return img[zi, yi, xi].astype(np.float32)


def gauss_kernel(sigma):
    """Truncated, normalised Gaussian (imglib2 Gauss3 half-kernel size max(2, int(3*sigma+0.5)+1))."""
    size = max(2, int(3 * sigma + 0.5) + 1)
    x = np.arange(-(size - 1), size, dtype=np.float64)
    k = np.exp(-0.5 * (x / sigma) ** 2)
    return (k / k.sum()).astype(np.float32)


def gauss3(vol, sigma):
    """Separable Gaussian, float32, mirror-single border (Views.extendMirrorSingle)."""
    from scipy.ndimage import correlate1d
    k = gauss_kernel(sigma)
    out = vol.astype(np.float32)
    for ax in (2, 1, 0):
        out = correlate1d(out, k, axis=ax, mode="mirror").astype(np.float32)
    return out


def content_weights(img, sigma1=DEFAULT_CONTENT_SIGMA1, sigma2=DEFAULT_CONTENT_SIGMA2):
    """Content-based weight volume c = G_s2 * (I - G_s1 * I)^2 on the source image."""
    f = img.astype(np.float32)
    d = (f - gauss3(f, sigma1)).astype(np.float32)
    return gauss3((d * d).astype(np.float32), sigma2)


def _mirror_single_index(i, n):
    """Views.extendMirrorSingle: ... c b | a b c ... (the border pixel is not repeated); a length-1 axis is constant."""
    if n == 1:
        return np.zeros_like(i)
    period = 2 * n - 2
    i = np.mod(i, period)
    return np.where(i < n, i, period - i)


def _gauss3_f64(vol, k, drop_outer_tap_axis=None):
    """Separable correlation with the taps ``k`` in float64, mirror-single border, x then y then z."""
    r = len(k) // 2
    out = np.asarray(vol, dtype=np.float64)
    for d in (0, 1, 2):             # x, y, z
        ax = 2 - d
        kk = np.array(k, dtype=np.float64)
        if d == drop_outer_tap_axis:
            kk[0] = kk[-1] = 0.0
        n = out.shape[ax]
        ext = np.take(out, _mirror_single_index(np.arange(-r, n + r), n), axis=ax)
        acc = np.zeros(out.shape)
        sl = [slice(None)] * 3
        for t, kt in enumerate(kk):
            sl[ax] = slice(t, t + n)
            acc += kt * ext[tuple(sl)]
        out = acc
    return out


def content_weights_reference(img, sigma1=DEFAULT_CONTENT_SIGMA1, sigma2=DEFAULT_CONTENT_SIGMA2, drop_outer_tap_axis=None):
    """Float64 reference of content_weights: the float32 taps of gauss_kernel, mirror-single borders, no intermediate
    rounding.  Returns (c, f, G_s1 f, d = f - G_s1 f), float64 [z, y, x]; f, G_s1 f and d set the error bar of a float32
    implementation.  ``drop_outer_tap_axis`` (0 = x, 1 = y, 2 = z) zeroes the outermost taps of both kernels on that axis:
    a wrong reference, used to show that a test's bar can tell it apart."""
    f = np.asarray(img, dtype=np.float32).astype(np.float64)
    g1 = _gauss3_f64(f, gauss_kernel(sigma1), drop_outer_tap_axis)
    d = f - g1
    return _gauss3_f64(d * d, gauss_kernel(sigma2), drop_outer_tap_axis), f, g1, d


@dataclass
class View:
    img: np.ndarray            # [z, y, x] uint16 or float32
    src_to_world: np.ndarray   # 12 doubles, row-packed 3x4 (registration * mipmap transform)
    blend_border: tuple = None  # float[3] in source px (after adjust_blending)
    blend_range: tuple = None
    content: np.ndarray = None  # optional float32 content-weight volume [z, y, x]


def source_coords(view: View, block_min_xyz, block_size_xyz):
    """Per output voxel, world -> source pixel coordinates in double, cast to float32.
    Output voxel (i,j,k) sits at world block_min + (i,j,k) (SparkAffineFusion.java:520-534)."""
    inv = invert_affine(view.src_to_world)
    bx, by, bz = block_size_xyz
    wx = np.arange(bx, dtype=np.float64) + block_min_xyz[0]
    wy = np.arange(by, dtype=np.float64) + block_min_xyz[1]
    wz = np.arange(bz, dtype=np.float64) + block_min_xyz[2]
    Z, Y, X = np.meshgrid(wz, wy, wx, indexing="ij")
    src = np.empty((bz, by, bx, 3), dtype=np.float32)
    for r in range(3):
        # same association as the device code: fma(m0, x, fma(m1, y, fma(m2, z, t)))
        src[..., r] = (inv[r, 0] * X + (inv[r, 1] * Y + (inv[r, 2] * Z + inv[r, 3]))).astype(np.float32)
    return src


def fuse_block(views, block_min_xyz, block_size_xyz, fusion_type=AVG_BLEND, interpolation=1,
               out_dtype="float32", min_intensity=0.0, max_intensity=65535.0, blend_lut_n=0):
    """Fuse one output block; returns [bz, by, bx] array of ``out_dtype``.

    Views must be given in ascending ViewId order (Collections.sort(sortedViewIds), which
    LOWEST/HIGHEST_VIEWID_WINS rely on).
    """
    bx, by, bz = block_size_xyz
    shape = (bz, by, bx)
    sum_i = np.zeros(shape, dtype=np.float32)
    sum_w = np.zeros(shape, dtype=np.float32)
    best = np.zeros(shape, dtype=np.float32)       # MAX / *_WINS result
    best_w = np.zeros(shape, dtype=np.float32)     # CLOSEST: best weight so far
    have = np.zeros(shape, dtype=bool)
    for v in views:
        dims_xyz = v.img.shape[::-1]
        src = source_coords(v, block_min_xyz, block_size_xyz)
        inside = inside_mask(src, dims_xyz)
        if not inside.any():
            continue
        val = trilinear(v.img, src) if interpolation == 1 else nearest(v.img, src)
        if fusion_type in (AVG_BLEND, AVG_BLEND_CONTENT, CLOSEST_PIXEL_WINS):
            border = v.blend_border if v.blend_border is not None else adjust_blending(v.src_to_world)[0]
            rng = v.blend_range if v.blend_range is not None else adjust_blending(v.src_to_world)[1]
            w = blend_weight(src, dims_xyz, border, rng, blend_lut_n)
        else:
            w = inside.astype(np.float32)
        w = np.where(inside, w, np.float32(0)).astype(np.float32)
        if fusion_type in (AVG_CONTENT, AVG_BLEND_CONTENT):
            if v.content is None:
                raise ValueError("content-based fusion needs View.content")
            cw = trilinear(v.content, src) if interpolation == 1 else nearest(v.content, src)
            w = (w * cw).astype(np.float32)
        if fusion_type in (AVG, AVG_BLEND, AVG_CONTENT, AVG_BLEND_CONTENT):
            sum_i = (sum_i + w * val).astype(np.float32)
            sum_w = (sum_w + w).astype(np.float32)
        elif fusion_type == MAX_INTENSITY:
            m = w > 0
            best = np.where(m & (~have | (val > best)), val, best)
            have |= m
        elif fusion_type == LOWEST_VIEWID_WINS:
            m = (w > 0) & ~have
            best = np.where(m, val, best)
            have |= m
        elif fusion_type == HIGHEST_VIEWID_WINS:
            m = w > 0
            best = np.where(m, val, best)
            have |= m
        elif fusion_type == CLOSEST_PIXEL_WINS:
            m = (w > 0) & (w > best_w)
            best = np.where(m, val, best)
            best_w = np.where(m, w, best_w)
            have |= m
        else:
            raise ValueError(fusion_type)
    if fusion_type in (AVG, AVG_BLEND, AVG_CONTENT, AVG_BLEND_CONTENT):
        out = np.zeros(shape, dtype=np.float32)
        np.divide(sum_i, sum_w, out=out, where=sum_w > 0)
    else:
        out = np.where(have, best, np.float32(0)).astype(np.float32)
    return convert_output(out, out_dtype, min_intensity, max_intensity)


def accumulate_block(views, block_min_xyz, block_size_xyz, fusion_type=AVG_BLEND, interpolation=1, blend_lut_n=0):
    """Partial sums [sum w*I, sum w] of a view subset (the view-sharded mode of SURVEY.md 8e);
    summing them over disjoint subsets and dividing equals fuse_block up to float re-association."""
    bx, by, bz = block_size_xyz
    sum_i = np.zeros((bz, by, bx), dtype=np.float32)
    sum_w = np.zeros((bz, by, bx), dtype=np.float32)
    for v in views:
        dims_xyz = v.img.shape[::-1]
        src = source_coords(v, block_min_xyz, block_size_xyz)
        inside = inside_mask(src, dims_xyz)
        if not inside.any():
            continue
        val = trilinear(v.img, src) if interpolation == 1 else nearest(v.img, src)
        if fusion_type in (AVG_BLEND, AVG_BLEND_CONTENT):
            w = blend_weight(src, dims_xyz, v.blend_border, v.blend_range, blend_lut_n)
        else:
            w = inside.astype(np.float32)
        w = np.where(inside, w, np.float32(0)).astype(np.float32)
        if fusion_type in (AVG_CONTENT, AVG_BLEND_CONTENT):
            w = (w * trilinear(v.content, src)).astype(np.float32)
        sum_i = (sum_i + w * val).astype(np.float32)
        sum_w = (sum_w + w).astype(np.float32)
    return sum_i, sum_w


def convert_output(out, out_dtype, min_intensity, max_intensity):
    """float32 stays; RealUnsignedByte/ShortConverter(min,max): round((v-min)/(max-min)*
    {255|65535}) clamped (SparkAffineFusion.java:493-517).  Rounding is Java Math.round-like
    floor(x + 0.5) on the double value."""
    if out_dtype in ("float32", np.float32):
        return out
    top = 255.0 if out_dtype in ("uint8", np.uint8) else 65535.0
    a = (out.astype(np.float64) - min_intensity) / (max_intensity - min_intensity) * top
    a = np.floor(a + 0.5)
    a = np.clip(a, 0, top)
    return a.astype(np.uint8 if top == 255.0 else np.uint16)


def downsample2x(vol, factors_xyz):
    """One pyramid step (N5ApiTools.writeDownsampledBlock / LazyHalfPixelDownsample2x restated; next
    row 8f-3): per axis with factor 2, out[i] = avg(in[2i], in[2i+1]), x then y then z; float32:
    0.5*(a+b); integer types: (a+b+1)>>1 per step (rounding rule recalled, PARITY_GAPS #23)."""
    out = vol
    for ax, f in zip((2, 1, 0), factors_xyz):
        if f == 1:
            continue
        n = out.shape[ax] // 2
        a = np.take(out, np.arange(0, 2 * n, 2), axis=ax)
        b = np.take(out, np.arange(1, 2 * n, 2), axis=ax)
        if out.dtype == np.float32:
            out = (np.float32(0.5) * (a + b)).astype(np.float32)
        else:
            out = ((a.astype(np.uint32) + b.astype(np.uint32) + 1) >> 1).astype(vol.dtype)
    return out


def mask_block(views_geom, block_min_xyz, block_size_xyz, mask_offset=(0.0, 0.0, 0.0), dtype="uint8"):
    """`--masks` mode (src/main/java/net/preibisch/bigstitcher/spark/fusion/GenerateComputeBlockMasks.java:119-176):
    a voxel is on when its back-projection l = M^-1 (world) satisfies min_d <= l_d <= max_d for EVERY axis of ANY view,
    min = 0 - offset, max = dim - 1 + offset (:127-128, :141-147); on = 255 / 65535 / 1.0f (:154-176).
    ``views_geom``: [(src_to_world 3x4, dims_xyz)]."""
    bx, by, bz = (int(v) for v in block_size_xyz)
    z, y, x = np.meshgrid(np.arange(bz, dtype=np.float64) + block_min_xyz[2], np.arange(by, dtype=np.float64) + block_min_xyz[1],
                          np.arange(bx, dtype=np.float64) + block_min_xyz[0], indexing="ij")
    on = np.zeros((bz, by, bx), dtype=bool)
    off = np.asarray(mask_offset, dtype=np.float64)
    for M, dims in views_geom:
        inv = np.linalg.inv(np.vstack([np.asarray(M, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]]))
        inside = np.ones_like(on)
        for d in range(3):
            l = inv[d, 0] * x + inv[d, 1] * y + inv[d, 2] * z + inv[d, 3]
            inside &= ~((l < 0.0 - off[d]) | (l > (dims[d] - 1) + off[d]))
        on |= inside
    top = {"uint8": 255, "uint16": 65535, "float32": 1.0}[dtype]
    return np.where(on, top, 0).astype(dtype)
