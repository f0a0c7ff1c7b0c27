// Pieces shared by the fusion translation units (fuse.cu: generic tile kernel; fuse_tma.cu: TMA-staged
// z-marching kernels; nonrigid.cu: moving-least-squares grids and non-rigid fusion).
#pragma once
#include <cmath>

#include "bs_internal.cuh"

#define FUSE_MAX_LUT 256

template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p, size_t i) {
    return (float)__ldg(p + i);
}

// n-linear (LINEAR) or nearest-neighbour sample of a dense x-fastest volume at (sx, sy, sz); the upper taps are
// clamped to the volume (border extension), the caller keeps the coordinate >= 0
template <typename T, bool LINEAR>
__device__ __forceinline__ float sample(const T* __restrict__ d, int dx, int dy, int dz, float sx, float sy,
                                        float sz) {
    if (LINEAR) {
        float fx = floorf(sx), fy = floorf(sy), fz = floorf(sz);
        float rx = sx - fx, ry = sy - fy, rz = sz - fz;
        int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
        int x1 = min(x0 + 1, dx - 1), y1 = min(y0 + 1, dy - 1), z1 = min(z0 + 1, dz - 1);
        size_t r00 = ((size_t)z0 * dy + y0) * dx, r01 = ((size_t)z0 * dy + y1) * dx;
        size_t r10 = ((size_t)z1 * dy + y0) * dx, r11 = ((size_t)z1 * dy + y1) * dx;
        float a000 = ld_as_float(d, r00 + x0), a001 = ld_as_float(d, r00 + x1);
        float a010 = ld_as_float(d, r01 + x0), a011 = ld_as_float(d, r01 + x1);
        float a100 = ld_as_float(d, r10 + x0), a101 = ld_as_float(d, r10 + x1);
        float a110 = ld_as_float(d, r11 + x0), a111 = ld_as_float(d, r11 + x1);
        float c00 = a000 + rx * (a001 - a000);
        float c01 = a010 + rx * (a011 - a010);
        float c10 = a100 + rx * (a101 - a100);
        float c11 = a110 + rx * (a111 - a110);
        float c0 = c00 + ry * (c01 - c00);
        float c1 = c10 + ry * (c11 - c10);
        return c0 + rz * (c1 - c0);
    } else {
        int xi = min(max((int)floorf(sx + 0.5f), 0), dx - 1);
        int yi = min(max((int)floorf(sy + 0.5f), 0), dy - 1);
        int zi = min(max((int)floorf(sz + 0.5f), 0), dz - 1);
        return ld_as_float(d, ((size_t)zi * dy + yi) * dx + xi);
    }
}

template <bool LINEAR>
__device__ __forceinline__ float sample_any(const void* d, int dtype, int dx, int dy, int dz, float sx,
                                            float sy, float sz) {
    if (dtype == BS_DTYPE_U16) return sample<unsigned short, LINEAR>((const unsigned short*)d, dx, dy, dz, sx, sy, sz);
    if (dtype == BS_DTYPE_F32) return sample<float, LINEAR>((const float*)d, dx, dy, dz, sx, sy, sz);
    return sample<unsigned char, LINEAR>((const unsigned char*)d, dx, dy, dz, sx, sy, sz);
}

// Output element encoding: the kernels' OUT template value = output dtype | OUT_BE.  Big-endian output
// (bs_fuse_params.out_big_endian) is a compile-time property of the instantiation, so the native-order kernels carry
// no byte-order code at all and the big-endian ones pay one PRMT per store.
#define OUT_BE 8
#define OUT_DT(OUT) ((OUT) & 7)
__device__ __forceinline__ unsigned int bswap32(unsigned int v) { return __byte_perm(v, 0u, 0x0123); }
__device__ __forceinline__ unsigned int bswap16x2(unsigned int v) { return __byte_perm(v, 0u, 0x2301); }

// one output voxel: float32 as it is, integer types through the converter (v - cmin) * cscale, rounded as
// floor(x + 0.5) and clamped to [0, ctop]
template <int OUT>
__device__ __forceinline__ void bs_store_converted(void* out, size_t o, float res, double cmin, double cscale, double ctop) {
    constexpr bool BE = (OUT & OUT_BE) != 0;
    if (OUT_DT(OUT) == BS_DTYPE_F32) {
        if (BE) __stcs((unsigned int*)out + o, bswap32(__float_as_uint(res)));
        else __stcs((float*)out + o, res);
    } else {
        double c = floor(((double)res - cmin) * cscale + 0.5);
        c = fmin(fmax(c, 0.0), ctop);
        if (OUT_DT(OUT) == BS_DTYPE_U16) ((unsigned short*)out)[o] = (unsigned short)(BE ? bswap16x2((unsigned int)c) : (unsigned int)c);
        else ((unsigned char*)out)[o] = (unsigned char)c;
    }
}

// cosine blending weight along one axis (l = absolute source coordinate); false when weight is 0
__device__ __forceinline__ bool blend_axis(float l, float dm1, float border, float inv_range, int lut_n,
                                           const float* s_lut, float& w) {
    const float dist = fmaxf(0.f, fminf(l - border, (dm1 - l) - border));
    if (dist == 0.f) return false;
    const float rel = dist * inv_range;
    if (rel < 1.f) {
        float f;
        if (lut_n > 0) {
            const float pos = rel * (float)lut_n;
            const int i = (int)pos;
            const float s = pos - (float)i;
            f = s_lut[i] * (1.0f - s) + s_lut[i + 1] * s;
        } else {
            // (cos((1 - rel) pi) + 1) / 2 == sin^2(pi rel / 2): no cancellation for tiny weights.
            // sin(pi y), y = rel / 2 in [0, 0.5): odd Taylor polynomial to y^11 (rel. error < 1e-7)
            const float yh = 0.5f * rel, y2 = yh * yh;
            float p = -0.0073704309f;              // -pi^11 / 11!
            p = fmaf(p, y2, 0.0821458866f);         //  pi^9 / 9!
            p = fmaf(p, y2, -0.5992645293f);        // -pi^7 / 7!
            p = fmaf(p, y2, 2.5501640399f);         //  pi^5 / 5!
            p = fmaf(p, y2, -5.1677127800f);        // -pi^3 / 3!
            p = fmaf(p, y2, 3.1415926536f);         //  pi
            const float sn = p * yh;
            f = sn * sn;
        }
        w *= f;
    }
    return true;
}


// Same weight as blend_axis, as a factor: 0 when the sample is outside [0, dim-1] or its weight is zero
// (dist == 0), 1 on the plateau.  use_blend == false gives the AVG mask (1 on the closed interval).
__device__ __forceinline__ float blend_factor(float l, float dm1, float border, float inv_range, bool use_blend) {
    if (!(l >= 0.f && l <= dm1)) return 0.f;
    if (!use_blend) return 1.f;
    float w = 1.f;
    if (!blend_axis(l, dm1, border, inv_range, 0, nullptr, w)) return 0.f;
    return w;
}

static inline bool bs_invert34(const double* m, double* inv) {
    const double a = m[0], b = m[1], c = m[2], d = m[4], e = m[5], f = m[6], g = m[8], h = m[9], i = m[10];
    const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
    if (det == 0.0 || !std::isfinite(det)) return false;
    const double id = 1.0 / det;
    double A[9] = {(e * i - f * h) * id, (c * h - b * i) * id, (b * f - c * e) * id,
                   (f * g - d * i) * id, (a * i - c * g) * id, (c * d - a * f) * id,
                   (d * h - e * g) * id, (b * g - a * h) * id, (a * e - b * d) * id};
    for (int r = 0; r < 3; ++r) {
        inv[4 * r + 0] = A[3 * r + 0];
        inv[4 * r + 1] = A[3 * r + 1];
        inv[4 * r + 2] = A[3 * r + 2];
        inv[4 * r + 3] = -(A[3 * r + 0] * m[3] + A[3 * r + 1] * m[7] + A[3 * r + 2] * m[11]);
    }
    return true;
}

