// Next row 8f-4: Difference-of-Gaussian interest-point detection on one block of a resident view
// (DoGImgLib2.computeDoG, call site J/SparkInterestPointDetection.java:530-547; the reference exposes -- and
// nulls -- a CUDA hook right there: dog.cuda = null, :490-493; block + 1 px halo logic :397-424).
//
//   I' = (I - minIntensity) / (maxIntensity - minIntensity)                       (float, mirror-double extension)
//   s1 = sigma, s2 = sigma * k, k = 2^(1/4) (4 steps per octave), image sigma 0.5:
//   sa = sqrt(s1^2 - 0.25), sb = sqrt(s2^2 - 0.25)            (DoGImgLib2.computeSigmas)
//   DoG = (G_sa * I' - G_sb * I') / (k - 1)                   (truncated normalised kernels, half size
//                                                              max(2, int(3 s + 0.5) + 1), Gauss3.halfkernelsizes)
//   candidates: 3x3x3 extrema of the block's voxels with |DoG| >= threshold / 3, quadratic localisation
//   (central-difference gradient / Hessian), kept when |interpolated value| >= threshold.
//
// One source read: k_dog_load cuts block + 1 px + kernel halo out of the resident volume (normalised float),
// the x / y passes blur with BOTH kernels at once, the z pass writes the DoG directly, k_dog_extrema compacts the
// detections with a global counter.  HBM-bound stencil work, no tensor cores.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "bs_internal.cuh"

namespace {

__device__ __forceinline__ int mirror_double(long long i, int n) {
    // Views.extendMirrorDouble: ... c b a | a b c ... (the border pixel is repeated)
    const long long period = 2LL * n;
    i %= period;
    if (i < 0) i += period;
    return (int)(i < n ? i : period - 1 - i);
}

struct LoadArgs {
    const void* src;
    int dtype;
    int vdims[3];
    long long rmin[3];      // region origin in image coordinates (may be negative)
    int rdims[3];
    float offset, scale;    // I' = (I - offset) * scale
    float* out;
};

// grid (ceil(rdims[0] / 256), rdims[1], rdims[2]): no per-voxel index division; the mirror folding only runs for
// voxels outside the image (the halo of border blocks)
__global__ void __launch_bounds__(256) k_dog_load(const __grid_constant__ LoadArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= a.rdims[0]) return;
    const int y = blockIdx.y, z = blockIdx.z;
    const long long gx = a.rmin[0] + x, gy = a.rmin[1] + y, gz = a.rmin[2] + z;
    const int sx = (gx >= 0 && gx < a.vdims[0]) ? (int)gx : mirror_double(gx, a.vdims[0]);
    const int sy = (gy >= 0 && gy < a.vdims[1]) ? (int)gy : mirror_double(gy, a.vdims[1]);
    const int sz = (gz >= 0 && gz < a.vdims[2]) ? (int)gz : mirror_double(gz, a.vdims[2]);
    const size_t si = ((size_t)sz * a.vdims[1] + sy) * a.vdims[0] + sx;
    float v;
    if (a.dtype == BS_DTYPE_U16) v = (float)__ldg((const unsigned short*)a.src + si);
    else if (a.dtype == BS_DTYPE_F32) v = __ldg((const float*)a.src + si);
    else v = (float)__ldg((const unsigned char*)a.src + si);
    a.out[((size_t)z * a.rdims[1] + y) * a.rdims[0] + x] = (v - a.offset) * a.scale;
}

#define DOG_MAXR 64
struct BlurArgs {
    const float* in_a;      // x pass: the loaded region; later passes: blur A so far
    const float* in_b;      // blur B so far (== in_a for the x pass)
    float* out_a;
    float* out_b;           // nullptr in the z pass: out_a receives (A - B) * scale
    int dims[3];
    int axis;
    int ra, rb;
    float scale;
    float ka[2 * DOG_MAXR + 1], kb[2 * DOG_MAXR + 1];
};

// one thread per voxel; taps outside the region are clamped (only voxels at least r away from the region's faces
// are used downstream: the region carries a halo of max(ra, rb) + 1)
__global__ void __launch_bounds__(256) k_dog_blur(const __grid_constant__ BlurArgs a) {
    const long long n = (long long)a.dims[0] * a.dims[1] * a.dims[2];
    const long long stride = a.axis == 0 ? 1 : (a.axis == 1 ? a.dims[0] : (long long)a.dims[0] * a.dims[1]);
    const int len = a.dims[a.axis];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % a.dims[0]);
        const long long r = i / a.dims[0];
        const int y = (int)(r % a.dims[1]), z = (int)(r / a.dims[1]);
        const int p = a.axis == 0 ? x : (a.axis == 1 ? y : z);
        const long long base = i - (long long)p * stride;
        // symmetric pairing, outermost taps first: (in[p - t] + in[p + t]) * k[t].  Across a mirrored image border
        // the two sides see the same pairs, so mirrored outputs are bit-identical and a border extremum ties with
        // its mirror image exactly (ties are kept) -- the symmetric-kernel evaluation of imglib2 / scipy.
        float sa = 0.f, sb = 0.f;
        for (int t = a.ra; t >= 1; --t) {
            const int q0 = max(p - t, 0), q1 = min(p + t, len - 1);
            sa = fmaf(a.ka[a.ra - t], __ldg(a.in_a + base + (long long)q0 * stride) + __ldg(a.in_a + base + (long long)q1 * stride), sa);
        }
        sa = fmaf(a.ka[a.ra], __ldg(a.in_a + i), sa);
        for (int t = a.rb; t >= 1; --t) {
            const int q0 = max(p - t, 0), q1 = min(p + t, len - 1);
            sb = fmaf(a.kb[a.rb - t], __ldg(a.in_b + base + (long long)q0 * stride) + __ldg(a.in_b + base + (long long)q1 * stride), sb);
        }
        sb = fmaf(a.kb[a.rb], __ldg(a.in_b + i), sb);
        if (a.out_b) { a.out_a[i] = sa; a.out_b[i] = sb; }
        else a.out_a[i] = (sa - sb) * a.scale;
    }
}

// ------------------------------------------------------------------------------------------ sliding-window blur
// The same sums as k_dog_blur (symmetric pairs, outermost tap first, so results are bit-identical), but every thread
// produces DOG_CH consecutive outputs along the blur axis from a register window of DOG_CH + 2 R inputs: ~2.5 loads
// per output instead of 2 (2 r + 1).  Half kernels are zero-padded to the compile-time radius R (a zero tap adds an
// exact +0).  x pass: the region's row pitch is a multiple of 4 floats, windows are fetched as aligned float4;
// y / z passes: lanes run along x (coalesced rows).
#define DOG_CH 8
#define DOG_WIN_MAXR 12
struct BlurWinArgs {
    const float* in_a;
    const float* in_b;
    float* out_a;
    float* out_b;
    int dims[3];            // dims[0] is the padded row pitch (multiple of 8)
    float scale;
    float ka[DOG_WIN_MAXR + 1], kb[DOG_WIN_MAXR + 1];   // ka[t]: coefficient at distance t, zero beyond the real radius
};

template <int R, int W>
__device__ __forceinline__ float dog_win_sum(const float (&w)[W], const float* __restrict__ k, int c) {
    float s = 0.f;
#pragma unroll
    for (int t = R; t >= 1; --t) s = fmaf(k[t], w[c - t] + w[c + t], s);
    return fmaf(k[0], w[c], s);
}

// x pass: in_a == in_b (the loaded region); one thread = 8 consecutive x of one row
template <int R>
__global__ void __launch_bounds__(256) k_dog_blur_x(const __grid_constant__ BlurWinArgs a) {
    constexpr int WL = (R + 3) & ~3;               // window reach rounded up to whole float4
    constexpr int W = DOG_CH + 2 * WL;
    const int pitch = a.dims[0], nch = pitch / DOG_CH;
    const long long items = (long long)nch * a.dims[1] * a.dims[2];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int cx = (int)(i % nch);
        const long long row = i / nch;
        const float* src = a.in_a + row * pitch;
        const int x0 = cx * DOG_CH;
        float w[W];
#pragma unroll
        for (int q = 0; q < W / 4; ++q) {
            const int xs = x0 - WL + 4 * q;
            if (xs >= 0 && xs + 3 < pitch) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src + xs));
                w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) w[4 * q + e] = __ldg(src + min(max(xs + e, 0), pitch - 1));
            }
        }
        float ra[DOG_CH], rb[DOG_CH];
#pragma unroll
        for (int o = 0; o < DOG_CH; ++o) {
            ra[o] = dog_win_sum<R, W>(w, a.ka, WL + o);
            rb[o] = dog_win_sum<R, W>(w, a.kb, WL + o);
        }
        float4* oa = reinterpret_cast<float4*>(a.out_a + row * pitch + x0);
        float4* ob = reinterpret_cast<float4*>(a.out_b + row * pitch + x0);
        oa[0] = make_float4(ra[0], ra[1], ra[2], ra[3]); oa[1] = make_float4(ra[4], ra[5], ra[6], ra[7]);
        ob[0] = make_float4(rb[0], rb[1], rb[2], rb[3]); ob[1] = make_float4(rb[4], rb[5], rb[6], rb[7]);
    }
}

// y (AXIS 1) and z (AXIS 2) passes; LAST writes the DoG (A - B) * scale
template <int R, int AXIS, bool LAST>
__global__ void __launch_bounds__(256) k_dog_blur_yz(const __grid_constant__ BlurWinArgs a) {
    constexpr int W = DOG_CH + 2 * R;
    const int pitch = a.dims[0], len = a.dims[AXIS];
    const int nch = (len + DOG_CH - 1) / DOG_CH;
    const int other = AXIS == 1 ? a.dims[2] : a.dims[1];
    const long long stride = AXIS == 1 ? pitch : (long long)pitch * a.dims[1];
    const long long ostride = AXIS == 1 ? (long long)pitch * a.dims[1] : pitch;   // stride of the remaining axis
    const long long items = (long long)pitch * nch * other;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % pitch);
        const long long r = i / pitch;
        const int c = (int)(r % nch), o2 = (int)(r / nch);
        const int p0 = c * DOG_CH;
        const long long base = (long long)o2 * ostride + x;
        float wa[W], wb[W];
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const long long q = base + (long long)min(max(p0 - R + j, 0), len - 1) * stride;
            wa[j] = __ldg(a.in_a + q);
            wb[j] = __ldg(a.in_b + q);
        }
#pragma unroll
        for (int o = 0; o < DOG_CH; ++o) {
            if (p0 + o >= len) break;
            const float sa = dog_win_sum<R, W>(wa, a.ka, R + o), sb = dog_win_sum<R, W>(wb, a.kb, R + o);
            const long long q = base + (long long)(p0 + o) * stride;
            if (LAST) a.out_a[q] = (sa - sb) * a.scale;
            else { a.out_a[q] = sa; a.out_b[q] = sb; }
        }
    }
}

template <int R>
void dog_blur_windowed(bs_ctx* ctx, BlurWinArgs b, float* r0, float* r1, float* r2, float* r3, int blocks) {
    // x: r0 -> (r1, r2); y: (r1, r2) -> (r3, r0); z: (r3, r0) -> r1 = DoG
    b.in_a = r0; b.in_b = r0; b.out_a = r1; b.out_b = r2;
    { bs_launch_scope sc(ctx, "dog_blur"); k_dog_blur_x<R><<<blocks, 256, 0, ctx->stream>>>(b); }
    b.in_a = r1; b.in_b = r2; b.out_a = r3; b.out_b = r0;
    { bs_launch_scope sc(ctx, "dog_blur"); k_dog_blur_yz<R, 1, false><<<blocks, 256, 0, ctx->stream>>>(b); }
    b.in_a = r3; b.in_b = r0; b.out_a = r1; b.out_b = nullptr;
    { bs_launch_scope sc(ctx, "dog_blur"); k_dog_blur_yz<R, 2, true><<<blocks, 256, 0, ctx->stream>>>(b); }
}

struct DogWs {
    void* buf[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t cap[4] = {0, 0, 0, 0};
    void* pts = nullptr;
    size_t pts_cap = 0;
    int* count = nullptr;
};

struct ExtremaArgs {
    const float* dog;       // region volume
    int rdims[3];
    int e0[3];              // first candidate voxel inside the region (halo + 1)
    int cdims[3];           // candidate box
    long long rmin[3];      // region origin in image coordinates
    float thr_initial;      // candidates: |DoG| >= (float)(threshold / 3), a float32 compare
    double thr_final;       // kept: |value| >= threshold, compared in double like the oracle (PARITY_GAPS #26)
    int find_max, find_min, localize;
    bs_dog_point* out;
    int max_points;
    int* counter;
};

__device__ __forceinline__ bool solve3f(const double H[3][3], const double g[3], double d[3]) {
    const double a = H[0][0], b = H[0][1], c = H[0][2], e = H[1][1], f = H[1][2], i = H[2][2];
    const double det = a * (e * i - f * f) - b * (b * i - f * c) + c * (b * f - e * c);
    if (fabs(det) < 1e-30 || !isfinite(det)) return false;
    const double inv[3][3] = {{(e * i - f * f) / det, (c * f - b * i) / det, (b * f - c * e) / det},
                              {(c * f - b * i) / det, (a * i - c * c) / det, (b * c - a * f) / det},
                              {(b * f - c * e) / det, (b * c - a * f) / det, (a * e - b * b) / det}};
    for (int r = 0; r < 3; ++r) d[r] = -(inv[r][0] * g[0] + inv[r][1] * g[1] + inv[r][2] * g[2]);
    return true;
}

// grid (ceil(cdims[0] / 256), cdims[1], cdims[2])
__global__ void __launch_bounds__(256) k_dog_extrema(const __grid_constant__ ExtremaArgs a) {
    const long long sy = a.rdims[0], sz = (long long)a.rdims[0] * a.rdims[1];
    const int cx = blockIdx.x * blockDim.x + threadIdx.x;
    if (cx < a.cdims[0]) {
        const int cy = blockIdx.y, cz = blockIdx.z;
        const int x = a.e0[0] + cx, y = a.e0[1] + cy, z = a.e0[2] + cz;
        const float* p = a.dog + (long long)z * sz + (long long)y * sy + x;
        const float v = p[0];
        const bool cand_max = a.find_max && v >= a.thr_initial;
        const bool cand_min = a.find_min && -v >= a.thr_initial;
        if (!cand_max && !cand_min) return;
        bool is_max = cand_max, is_min = cand_min;
        float nb[27];
#pragma unroll
        for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
                for (int dx = -1; dx <= 1; ++dx) {
                    const float w = p[dz * sz + dy * sy + dx];
                    nb[(dz + 1) * 9 + (dy + 1) * 3 + (dx + 1)] = w;
                    if (dx | dy | dz) {
                        if (w > v) is_max = false;      // LocalExtrema.MaximumCheck: no neighbour may be larger
                        if (w < v) is_min = false;
                    }
                }
        if (!is_max && !is_min) return;
        double d[3] = {0.0, 0.0, 0.0};
        double val = v;
        if (a.localize) {
#define NB(ix, iy, iz) (double)nb[((iz) + 1) * 9 + ((iy) + 1) * 3 + ((ix) + 1)]
            const double g[3] = {0.5 * (NB(1, 0, 0) - NB(-1, 0, 0)), 0.5 * (NB(0, 1, 0) - NB(0, -1, 0)), 0.5 * (NB(0, 0, 1) - NB(0, 0, -1))};
            double H[3][3];
            H[0][0] = NB(1, 0, 0) - 2.0 * v + NB(-1, 0, 0);
            H[1][1] = NB(0, 1, 0) - 2.0 * v + NB(0, -1, 0);
            H[2][2] = NB(0, 0, 1) - 2.0 * v + NB(0, 0, -1);
            H[0][1] = H[1][0] = 0.25 * (NB(1, 1, 0) - NB(-1, 1, 0) - NB(1, -1, 0) + NB(-1, -1, 0));
            H[0][2] = H[2][0] = 0.25 * (NB(1, 0, 1) - NB(-1, 0, 1) - NB(1, 0, -1) + NB(-1, 0, -1));
            H[1][2] = H[2][1] = 0.25 * (NB(0, 1, 1) - NB(0, -1, 1) - NB(0, 1, -1) + NB(0, -1, -1));
#undef NB
            if (solve3f(H, g, d)) {
                for (int q = 0; q < 3; ++q) d[q] = fmin(fmax(d[q], -0.5), 0.5);   // no re-centring moves (PARITY_GAPS)
                val = v + 0.5 * (g[0] * d[0] + g[1] * d[1] + g[2] * d[2]);
            } else {
                d[0] = d[1] = d[2] = 0.0;
            }
            if (fabs(val) < a.thr_final) return;
        } else if (fabs((double)v) < a.thr_final) {
            return;
        }
        const int slot = atomicAdd(a.counter, 1);
        if (slot >= a.max_points) return;
        bs_dog_point& o = a.out[slot];
        o.voxel[0] = a.rmin[0] + x; o.voxel[1] = a.rmin[1] + y; o.voxel[2] = a.rmin[2] + z;
        o.loc[0] = (double)o.voxel[0] + d[0]; o.loc[1] = (double)o.voxel[1] + d[1]; o.loc[2] = (double)o.voxel[2] + d[2];
        o.value = val;
        o.is_max = is_max ? 1 : 0;
        o.pad = 0;
    }
}

std::vector<float> dog_kernel(double sigma, int* r_out) {
    const int size = std::max(2, (int)(3.0 * sigma + 0.5) + 1);
    const int r = size - 1;
    std::vector<double> k(2 * r + 1);
    double sum = 0.0;
    for (int i = -r; i <= r; ++i) {
        k[i + r] = std::exp(-0.5 * ((double)i / sigma) * ((double)i / sigma));
        sum += k[i + r];
    }
    std::vector<float> out(2 * r + 1);
    for (size_t i = 0; i < k.size(); ++i) out[i] = (float)(k[i] / sum);
    *r_out = r;
    return out;
}

// blur variants (bs_dog_debug_dog's `blur` argument; 0 = the production choice from rb)
enum { DOG_BLUR_AUTO = 0, DOG_BLUR_GENERIC = 1, DOG_BLUR_WIN6 = 2, DOG_BLUR_WIN12 = 3 };

// the region one block is computed on: interval + halo per axis, rows padded to a multiple of 8 floats
struct DogRegion {
    long long rmin[3];      // origin in image coordinates (may be negative)
    int rdims[3];           // rdims[0] is the padded row pitch
    int halo;               // max(ra, rb) + 1: kernel reach + the 3x3x3 neighbourhood
    const float* dog;       // (G_sa * I' - G_sb * I') / (k - 1) over the region (context workspace)
};

// Checks the interval and the intensity / sigma parameters, then runs k_dog_load and the three blur passes of one
// block on the context's stream: the single copy of these launches, shared by bs_dog_detect and bs_dog_debug_dog.
// Called with ctx->mu held.  info (may be NULL): the blur instantiation launched and the radii.
int dog_load_blur(bs_ctx* ctx, const char* who, const bs_volume& v, const long long interval_min[3],
                  const long long interval_size[3], const bs_dog_params* p, int blur, DogRegion* reg, char* info) {
    if (!(p->sigma > 0.5) || !(p->max_intensity > p->min_intensity))
        return bs_set_error(ctx, BS_ERR_ARG, "%s: need sigma > 0.5 (image sigma), max_intensity > min_intensity", who);
    for (int d = 0; d < 3; ++d)
        if (interval_size[d] <= 0 || interval_min[d] < 0 || interval_min[d] + interval_size[d] > v.dims[d])
            return bs_set_error(ctx, BS_ERR_ARG, "%s: interval outside the volume (axis %d)", who, d);
    // DoGImgLib2.computeSigmas: 4 steps per octave, image sigma 0.5
    const double k = std::pow(2.0, 0.25), image_sigma = 0.5;
    const double s1 = p->sigma, s2 = p->sigma * k;
    const double sa = std::sqrt(s1 * s1 - image_sigma * image_sigma), sb = std::sqrt(s2 * s2 - image_sigma * image_sigma);
    int ra, rb;
    const std::vector<float> ka = dog_kernel(sa, &ra), kb = dog_kernel(sb, &rb);
    if (rb > DOG_MAXR) return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "%s: sigma too large (kernel radius %d > %d)", who, rb, DOG_MAXR);
    if (blur == DOG_BLUR_AUTO) blur = rb <= 6 ? DOG_BLUR_WIN6 : (rb <= DOG_WIN_MAXR ? DOG_BLUR_WIN12 : DOG_BLUR_GENERIC);
    if (blur < DOG_BLUR_GENERIC || blur > DOG_BLUR_WIN12 || (blur == DOG_BLUR_WIN6 && rb > 6) || (blur == DOG_BLUR_WIN12 && rb > 12))
        return bs_set_error(ctx, BS_ERR_ARG, "%s: blur variant %d cannot run kernel radius %d", who, blur, rb);
    const int halo = std::max(ra, rb) + 1;
    long long nreg = 1;
    for (int d = 0; d < 3; ++d) {
        reg->rmin[d] = interval_min[d] - halo;
        const long long rd = interval_size[d] + 2LL * halo;
        if (rd > 0x7fffffffLL) return bs_set_error(ctx, BS_ERR_ARG, "%s: interval too large", who);
        reg->rdims[d] = (int)rd;
        nreg *= rd;
    }
    int* rdims = reg->rdims;
    if (rdims[1] > 65535 || rdims[2] > 65535)
        return bs_set_error(ctx, BS_ERR_ARG, "%s: block too large in y / z (%d x %d incl. halo, limit 65535): detect block-wise", who, rdims[1], rdims[2]);
    // the region's rows are padded to a multiple of 8 floats (more halo on the right: the extra columns hold real
    // mirror-extended image data, so every used voxel is unchanged) -> aligned float4 windows in the x pass
    nreg = nreg / rdims[0];
    rdims[0] = (rdims[0] + 7) & ~7;
    nreg *= rdims[0];
    reg->halo = halo;
    if (!ctx->dog) ctx->dog = new DogWs();
    DogWs* W = (DogWs*)ctx->dog;
    for (int i = 0; i < 4; ++i) {
        const int rc = bs_ensure_dev(ctx, &W->buf[i], &W->cap[i], sizeof(float) * (size_t)nreg);
        if (rc) return rc;
    }
    float *r0 = (float*)W->buf[0], *r1 = (float*)W->buf[1], *r2 = (float*)W->buf[2], *r3 = (float*)W->buf[3];
    const int blocks = (int)std::min<long long>((nreg + 255) / 256, (long long)ctx->sm_count * 32);
    {
        LoadArgs a;
        a.src = v.dev; a.dtype = v.dtype;
        for (int d = 0; d < 3; ++d) { a.vdims[d] = (int)v.dims[d]; a.rmin[d] = reg->rmin[d]; a.rdims[d] = rdims[d]; }
        a.offset = (float)p->min_intensity;
        a.scale = (float)(1.0 / (p->max_intensity - p->min_intensity));
        a.out = r0;
        bs_launch_scope sc(ctx, "dog_load");
        k_dog_load<<<dim3((unsigned)((rdims[0] + 255) / 256), (unsigned)rdims[1], (unsigned)rdims[2]), 256, 0, ctx->stream>>>(a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    const float dog_scale = (float)(1.0 / (k - 1.0));           // K_MIN1_INV
    if (blur != DOG_BLUR_GENERIC) {
        BlurWinArgs b;
        memset(&b, 0, sizeof(b));
        for (int d = 0; d < 3; ++d) b.dims[d] = rdims[d];
        b.scale = dog_scale;
        for (int t = 0; t <= ra; ++t) b.ka[t] = ka[(size_t)(ra + t)];
        for (int t = 0; t <= rb; ++t) b.kb[t] = kb[(size_t)(rb + t)];
        const int wblocks = (int)std::min<long long>((nreg / DOG_CH + 255) / 256 + 1, (long long)ctx->sm_count * 32);
        if (blur == DOG_BLUR_WIN6) dog_blur_windowed<6>(ctx, b, r0, r1, r2, r3, wblocks);
        else dog_blur_windowed<12>(ctx, b, r0, r1, r2, r3, wblocks);
        BS_CUDA(ctx, cudaGetLastError());
    } else {
        BlurArgs b;
        memset(&b, 0, sizeof(b));
        for (int d = 0; d < 3; ++d) b.dims[d] = rdims[d];
        b.ra = ra; b.rb = rb;
        memcpy(b.ka, ka.data(), sizeof(float) * ka.size());
        memcpy(b.kb, kb.data(), sizeof(float) * kb.size());
        b.scale = dog_scale;
        // x: r0 -> (r1, r2); y: (r1, r2) -> (r3, r0); z: (r3, r0) -> r1 = DoG
        const float* ina[3] = {r0, r1, r3};
        const float* inb[3] = {r0, r2, r0};
        float* outa[3] = {r1, r3, r1};
        float* outb[3] = {r2, r0, nullptr};
        for (int axis = 0; axis < 3; ++axis) {
            b.in_a = ina[axis]; b.in_b = inb[axis]; b.out_a = outa[axis]; b.out_b = outb[axis]; b.axis = axis;
            bs_launch_scope sc(ctx, "dog_blur");
            k_dog_blur<<<blocks, 256, 0, ctx->stream>>>(b);
            BS_CUDA(ctx, cudaGetLastError());
        }
    }
    reg->dog = r1;
    if (info) {
        const char* name = blur == DOG_BLUR_GENERIC ? "k_dog_blur" : (blur == DOG_BLUR_WIN6 ? "k_dog_blur_x<6>" : "k_dog_blur_x<12>");
        snprintf(info, 128, "%s ra=%d rb=%d", name, ra, rb);
    }
    return BS_OK;
}

}  // namespace

extern "C" {

void bs_dog_default_params(bs_dog_params* p) {
    if (!p) return;
    p->sigma = 1.8;
    p->threshold = 0.008;
    p->min_intensity = 0.0;
    p->max_intensity = 65535.0;
    p->find_max = 1;
    p->find_min = 0;
    p->localization = 1;
    p->pad = 0;
}

int bs_dog_detect(bs_ctx* ctx, unsigned long long vol_handle, const long long interval_min[3], const long long interval_size[3],
                  const bs_dog_params* p, bs_dog_point* out, int max_points, int* n_found) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!interval_min || !interval_size || !p || !n_found || (max_points > 0 && !out) || max_points < 0)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_dog_detect: bad argument");
    *n_found = 0;
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_dog_detect: unknown handle %llu", vol_handle);
    if (!(p->threshold >= 0.0)) return bs_set_error(ctx, BS_ERR_ARG, "bs_dog_detect: need threshold >= 0");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = bs_volume_acquire(ctx, it->second);
    if (rc) return rc;
    const bs_volume v = it->second;
    DogRegion reg;
    rc = dog_load_blur(ctx, "bs_dog_detect", v, interval_min, interval_size, p, DOG_BLUR_AUTO, &reg, nullptr);
    if (rc) return rc;
    DogWs* W = (DogWs*)ctx->dog;
    rc = bs_ensure_dev(ctx, &W->pts, &W->pts_cap, sizeof(bs_dog_point) * (size_t)std::max(1, max_points));
    if (rc) return rc;
    if (!W->count) BS_CUDA(ctx, cudaMalloc(&W->count, sizeof(int)));
    bs_dog_point* dpts = (bs_dog_point*)W->pts;
    int* dcount = W->count;
#define DOG_CUDA(call) BS_CUDA(ctx, call)
    DOG_CUDA(cudaMemsetAsync(dcount, 0, sizeof(int), ctx->stream));
    {
        ExtremaArgs a;
        a.dog = reg.dog;
        for (int d = 0; d < 3; ++d) {
            a.rdims[d] = reg.rdims[d]; a.e0[d] = reg.halo; a.cdims[d] = (int)interval_size[d]; a.rmin[d] = reg.rmin[d];
        }
        a.thr_final = p->threshold;
        a.thr_initial = p->localization ? (float)(p->threshold / 3.0) : (float)p->threshold;
        a.find_max = p->find_max; a.find_min = p->find_min; a.localize = p->localization ? 1 : 0;
        a.out = dpts; a.max_points = max_points; a.counter = dcount;
        bs_launch_scope sc(ctx, "dog_extrema");
        k_dog_extrema<<<dim3((unsigned)((interval_size[0] + 255) / 256), (unsigned)interval_size[1], (unsigned)interval_size[2]), 256, 0,
                        ctx->stream>>>(a);
    }
    DOG_CUDA(cudaGetLastError());
    int n = 0;
    DOG_CUDA(cudaMemcpyAsync(&n, dcount, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    DOG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int ncopy = std::min(n, max_points);
    if (ncopy > 0) {
        DOG_CUDA(cudaMemcpyAsync(out, dpts, sizeof(bs_dog_point) * (size_t)ncopy, cudaMemcpyDeviceToHost, ctx->stream));
        DOG_CUDA(cudaStreamSynchronize(ctx->stream));
        // the compaction order is not deterministic: sort by voxel (z, y, x)
        std::sort(out, out + ncopy, [](const bs_dog_point& x, const bs_dog_point& y) {
            if (x.voxel[2] != y.voxel[2]) return x.voxel[2] < y.voxel[2];
            if (x.voxel[1] != y.voxel[1]) return x.voxel[1] < y.voxel[1];
            return x.voxel[0] < y.voxel[0];
        });
    }
#undef DOG_CUDA
    *n_found = n;      // > max_points: the caller's buffer was too small, the first max_points (unsorted subset) were kept
    return BS_OK;
}

int bs_dog_debug_dog(bs_ctx* ctx, unsigned long long vol_handle, const long long interval_min[3],
                     const long long interval_size[3], const bs_dog_params* p, int blur, float* out, char info[128]) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!interval_min || !interval_size || !p || !out)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_dog_debug_dog: bad argument");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_dog_debug_dog: unknown handle %llu", vol_handle);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = bs_volume_acquire(ctx, it->second);
    if (rc) return rc;
    const bs_volume v = it->second;
    DogRegion reg;
    char buf[128] = "";
    rc = dog_load_blur(ctx, "bs_dog_debug_dog", v, interval_min, interval_size, p, blur, &reg, buf);
    if (rc) return rc;
    // the box the extremum stage reads: region voxels [halo - 1, halo + size + 1) per axis
    const size_t bx = (size_t)interval_size[0] + 2, by = (size_t)interval_size[1] + 2, bz = (size_t)interval_size[2] + 2;
    const size_t pitch = (size_t)reg.rdims[0] * sizeof(float);
    for (size_t z = 0; z < bz; ++z) {
        const float* src = reg.dog + ((size_t)(reg.halo - 1 + z) * reg.rdims[1] + (size_t)(reg.halo - 1)) * reg.rdims[0] + (reg.halo - 1);
        BS_CUDA(ctx, cudaMemcpy2DAsync(out + z * bx * by, bx * sizeof(float), src, pitch, bx * sizeof(float), by,
                                       cudaMemcpyDeviceToHost, ctx->stream));
    }
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (info) memcpy(info, buf, sizeof(buf));
    return BS_OK;
}

}  // extern "C"

void bs_dog_free(bs_ctx* ctx) {
    DogWs* W = (DogWs*)ctx->dog;
    if (!W) return;
    for (int i = 0; i < 4; ++i)
        if (W->buf[i]) cudaFree(W->buf[i]);
    if (W->pts) cudaFree(W->pts);
    if (W->count) cudaFree(W->count);
    delete W;
    ctx->dog = nullptr;
}
