// Content-based fusion weights (Preibisch et al.): c = G_s2 * (I - G_s1 * I)^2 on the source
// volume, precomputed once per view and sampled by the fusion kernel (SURVEY.md A.2 step 3;
// FusionType AVG_CONTENT / AVG_BLEND_CONTENT, J/SparkAffineFusion.java:124).
//
// Separable truncated Gaussian (half size max(2, int(3*sigma+0.5)+1), normalised), single-mirror
// border.  Each pass stages whole lines in shared memory: x pass = LINES rows per CTA, y/z pass =
// a [len][32] column block (x-fastest, so global accesses stay coalesced).
#include <cmath>
#include <vector>

#include "bs_internal.cuh"

#define GA_THREADS 256
#define GA_SMEM_MAX 232448

extern __shared__ __align__(16) float ga_sm[];

__device__ __forceinline__ int mirror_single(int i, int n) {
    if (n == 1) return 0;
    const int period = 2 * n - 2;
    i %= period;
    if (i < 0) i += period;
    return i < n ? i : period - i;
}

struct GaussArgs {
    const float* in;
    float* out;
    int dims[3];
    int axis;
    const float* kern;  // 2*r+1 taps
    int r;
    int lines;          // x pass: rows per CTA
};

// Both passes register-tile GA_T = 4 consecutive outputs along the blur axis: every staged sample is converted to double
// ONCE and feeds four accumulators (tap index = sample index - output index, taps outside [0, 2r] are zero-padded in the
// table), so a tap costs one DFMA plus a quarter of a shared load and of an F2F -- the first version converted both
// operands for every tap and was bound by the conversion pipe (0.19 s per 576^3 view at sigma 20 / 40).  The sum of every
// output still runs over its taps in ascending order, so the values are bit-identical to the tap-by-tap loop.
#define GA_T 4
__device__ __forceinline__ int ga_groups(int r) { return (2 * r + 1 + (GA_T - 1) + 3) / 4; }   // sample groups of 4 per output tile
__device__ __forceinline__ int ga_ktab(int r) { return 4 * ga_groups(r) + 8; }                  // padded double taps

// kd[i + 3] = tap i (0 <= i <= 2r), zeros around it
__device__ __forceinline__ void ga_fill_taps(double* kd, const float* __restrict__ kern, int r) {
    const int n = ga_ktab(r);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int u = i - 3;
        kd[i] = (u >= 0 && u <= 2 * r) ? (double)kern[u] : 0.0;
    }
}

// x pass: ga_sm = double taps | lines * wpad samples (wpad: multiple of 4, zero tail), a thread = 4 consecutive x
__global__ void __launch_bounds__(GA_THREADS) k_gauss_x(const __grid_constant__ GaussArgs a) {
    const int len = a.dims[0], r = a.r, w = len + 2 * r;
    const int G = ga_groups(r);
    const int nq = (len + GA_T - 1) / GA_T;
    const int wpad = 4 * nq + 4 * G + 4;
    double* kd = reinterpret_cast<double*>(ga_sm);
    float* buf = ga_sm + 2 * ga_ktab(r);
    ga_fill_taps(kd, a.kern, r);
    const long long nrows = (long long)a.dims[1] * a.dims[2];
    const long long row0 = (long long)blockIdx.x * a.lines;
    const int nl = (int)min((long long)a.lines, nrows - row0);
    for (int i = threadIdx.x; i < nl * wpad; i += blockDim.x) {
        const int l = i / wpad, p = i - l * wpad;
        buf[i] = p < w ? a.in[(row0 + l) * len + mirror_single(p - r, len)] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nl * nq; i += blockDim.x) {
        const int l = i / nq, q = i - l * nq;
        const float4* b4 = reinterpret_cast<const float4*>(buf + l * wpad + GA_T * q);
        double acc[GA_T] = {0.0, 0.0, 0.0, 0.0};
        for (int g = 0; g < G; ++g) {
            const float4 s4 = b4[g];
            const double sd[4] = {(double)s4.x, (double)s4.y, (double)s4.z, (double)s4.w};
            double k[7];
#pragma unroll
            for (int e = 0; e < 7; ++e) k[e] = kd[4 * g + e];
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int j = 0; j < GA_T; ++j) acc[j] = fma(k[3 + c - j], sd[c], acc[j]);
        }
        float* o = a.out + (row0 + l) * len + GA_T * q;
#pragma unroll
        for (int j = 0; j < GA_T; ++j)
            if (GA_T * q + j < len) o[j] = (float)acc[j];
    }
}

// y / z pass: CTA owns a column block of 32 x-values for a fixed index of the third axis; a thread = 4 consecutive
// outputs along the axis for one x
__global__ void __launch_bounds__(GA_THREADS) k_gauss_strided(const __grid_constant__ GaussArgs a) {
    const int len = a.dims[a.axis], r = a.r;
    const int G = ga_groups(r);
    const int nq = (len + GA_T - 1) / GA_T;
    const int rows = 4 * nq + 4 * G + 4;            // staged samples per column (zero tail)
    double* kd = reinterpret_cast<double*>(ga_sm);
    float* buf = ga_sm + 2 * ga_ktab(r);            // [rows][32]
    ga_fill_taps(kd, a.kern, r);
    const int x0 = blockIdx.x * 32;
    const int lane = threadIdx.x & 31, wy = threadIdx.x >> 5, nwy = blockDim.x >> 5;
    const int x = x0 + lane;
    const long long sy = a.dims[0], sz = (long long)a.dims[0] * a.dims[1];
    const long long stride = a.axis == 1 ? sy : sz;
    const long long base = (a.axis == 1 ? (long long)blockIdx.y * sz : (long long)blockIdx.y * sy) + x;
    const bool ok = x < a.dims[0];
    for (int p = wy; p < rows; p += nwy)
        buf[p * 32 + lane] = (ok && p < len + 2 * r) ? a.in[base + (long long)mirror_single(p - r, len) * stride] : 0.f;
    __syncthreads();
    if (!ok) return;
    for (int q = wy; q < nq; q += nwy) {
        const float* b = buf + (GA_T * q) * 32 + lane;
        double acc[GA_T] = {0.0, 0.0, 0.0, 0.0};
        for (int g = 0; g < G; ++g) {
            double k[7];
#pragma unroll
            for (int e = 0; e < 7; ++e) k[e] = kd[4 * g + e];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const double sd = (double)b[(4 * g + c) * 32];
#pragma unroll
                for (int j = 0; j < GA_T; ++j) acc[j] = fma(k[3 + c - j], sd, acc[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < GA_T; ++j)
            if (GA_T * q + j < len) a.out[base + (long long)(GA_T * q + j) * stride] = (float)acc[j];
    }
}

__global__ void k_to_float(const void* in, int dtype, float* out, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long st = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += st) {
        float v;
        if (dtype == BS_DTYPE_U16) v = (float)((const unsigned short*)in)[i];
        else if (dtype == BS_DTYPE_F32) v = ((const float*)in)[i];
        else v = (float)((const unsigned char*)in)[i];
        out[i] = v;
    }
}

__global__ void k_sqdiff(const float* f, const float* g, float* out, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long st = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += st) {
        const float d = f[i] - g[i];
        out[i] = d * d;
    }
}

static std::vector<float> gauss_kernel(double sigma, int* r_out) {
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

// gaussian blur src -> dst using tmp (all float volumes of `dims`); order x, y, z
static int gauss3(bs_ctx* ctx, const float* src, float* dst, float* tmp, const long long dims[3], double sigma,
                  float* kern_dev) {
    int r;
    std::vector<float> k = gauss_kernel(sigma, &r);
    BS_CUDA(ctx, cudaMemcpyAsync(kern_dev, k.data(), sizeof(float) * k.size(), cudaMemcpyHostToDevice, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // k is a stack-lifetime staging buffer
    GaussArgs a;
    a.kern = kern_dev;
    a.r = r;
    for (int d = 0; d < 3; ++d) a.dims[d] = (int)dims[d];
    // x: src -> dst
    {
        const int G = (2 * r + 1 + 3 + 3) / 4;                       // ga_groups(r)
        const size_t fixed = (size_t)(4 * G + 8) * sizeof(double);     // ga_ktab(r) double taps
        const size_t per_line = (size_t)(4 * ((dims[0] + 3) / 4) + 4 * G + 4) * sizeof(float);
        int lines = (int)std::min<size_t>(8, (GA_SMEM_MAX - fixed) / per_line);
        if (lines < 1) return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "content: x size too large for shared memory");
        a.in = src; a.out = dst; a.axis = 0; a.lines = lines;
        const long long nrows = dims[1] * dims[2];
        bs_launch_scope sc(ctx, "content_gauss");
        k_gauss_x<<<(unsigned)((nrows + lines - 1) / lines), GA_THREADS, fixed + lines * per_line, ctx->stream>>>(a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    // y: dst -> tmp ; z: tmp -> dst
    for (int axis = 1; axis <= 2; ++axis) {
        const int G = (2 * r + 1 + 3 + 3) / 4;
        const size_t smem = (size_t)(4 * G + 8) * sizeof(double) + (size_t)(4 * ((dims[axis] + 3) / 4) + 4 * G + 4) * 32 * sizeof(float);
        if (smem > GA_SMEM_MAX) return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "content: axis %d too long for shared memory", axis);
        a.in = axis == 1 ? dst : tmp;
        a.out = axis == 1 ? tmp : dst;
        a.axis = axis;
        a.lines = 0;
        dim3 grid((unsigned)((dims[0] + 31) / 32), (unsigned)(axis == 1 ? dims[2] : dims[1]), 1);
        bs_launch_scope sc(ctx, "content_gauss");
        k_gauss_strided<<<grid, GA_THREADS, smem, ctx->stream>>>(a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

extern "C" int bs_content_weights(bs_ctx* ctx, unsigned long long vol_handle, double sigma1, double sigma2,
                                  unsigned long long* content_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!content_handle || !(sigma1 > 0.0) || !(sigma2 > 0.0))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_content_weights: bad argument");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_content_weights: unknown handle %llu", vol_handle);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    const bs_volume src = it->second;
    BS_CUDA(ctx, cudaFuncSetAttribute((const void*)k_gauss_x, cudaFuncAttributeMaxDynamicSharedMemorySize, GA_SMEM_MAX));
    BS_CUDA(ctx, cudaFuncSetAttribute((const void*)k_gauss_strided, cudaFuncAttributeMaxDynamicSharedMemorySize, GA_SMEM_MAX));
    const long long n = src.dims[0] * src.dims[1] * src.dims[2];
    float *f = nullptr, *g = nullptr, *t = nullptr, *kern = nullptr;
    auto cleanup = [&]() {
        if (f) cudaFree(f);
        if (g) cudaFree(g);
        if (t) cudaFree(t);
        if (kern) cudaFree(kern);
    };
    cudaError_t e;
    if ((e = cudaMalloc(&f, sizeof(float) * n)) != cudaSuccess || (e = cudaMalloc(&g, sizeof(float) * n)) != cudaSuccess ||
        (e = cudaMalloc(&t, sizeof(float) * n)) != cudaSuccess || (e = cudaMalloc(&kern, sizeof(float) * 65536)) != cudaSuccess) {
        cleanup();
        return bs_set_error(ctx, BS_ERR_NOMEM, "bs_content_weights: cudaMalloc: %s", cudaGetErrorString(e));
    }
    const int blocks = ctx->sm_count * 8;
    int rc = BS_OK;
    {
        bs_launch_scope sc(ctx, "content_misc");
        k_to_float<<<blocks, 256, 0, ctx->stream>>>(src.dev, src.dtype, f, n);
    }
    if (3.0 * std::max(sigma1, sigma2) + 2 > 30000) rc = bs_set_error(ctx, BS_ERR_ARG, "bs_content_weights: sigma too large");
    if (!rc) rc = gauss3(ctx, f, g, t, src.dims, sigma1, kern);
    if (!rc) {
        bs_launch_scope sc(ctx, "content_misc");
        k_sqdiff<<<blocks, 256, 0, ctx->stream>>>(f, g, f, n);
    }
    if (!rc) rc = gauss3(ctx, f, g, t, src.dims, sigma2, kern);
    if (!rc) {
        e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) rc = bs_set_error(ctx, BS_ERR_CUDA, "bs_content_weights: %s", cudaGetErrorString(e));
    }
    if (rc) {
        cudaStreamSynchronize(ctx->stream);
        cleanup();
        return rc;
    }
    cudaFree(f);
    cudaFree(t);
    cudaFree(kern);
    bs_volume v;
    v.dev = g;
    v.dims[0] = src.dims[0]; v.dims[1] = src.dims[1]; v.dims[2] = src.dims[2];
    v.dtype = BS_DTYPE_F32;
    v.owned = true;
    *content_handle = ctx->next_handle++;
    ctx->vols[*content_handle] = v;
    return BS_OK;
}

// ------------------------------------------------------------------------------------------
// Next row f-3 (SURVEY.md 8f): 2x half-pixel averaging pyramid level on the device, right after
// fusion while the block is still resident (replaces re-reading s(l-1) from the container,
// J/SparkAffineFusion.java:703-782; N5ApiTools.writeDownsampledBlock / LazyHalfPixelDownsample2x,
// J/SparkDownsample.java:159-176).  One dimension after the other like the lazy upstream ops:
// out[i] = avg(in[2i], in[2i+1]); float: 0.5f*(a+b); integer types: (a+b+1)>>1 per step.
template <typename T>
__device__ __forceinline__ T avg2(T a, T b);
template <> __device__ __forceinline__ float avg2<float>(float a, float b) { return 0.5f * (a + b); }
template <> __device__ __forceinline__ unsigned short avg2<unsigned short>(unsigned short a, unsigned short b) {
    return (unsigned short)(((unsigned)a + (unsigned)b + 1u) >> 1);
}
template <> __device__ __forceinline__ unsigned char avg2<unsigned char>(unsigned char a, unsigned char b) {
    return (unsigned char)(((unsigned)a + (unsigned)b + 1u) >> 1);
}

template <typename T, typename Tout = T>
__global__ void k_downsample(const T* __restrict__ in, Tout* __restrict__ out, int dx, int dy, int dz, int ox, int oy,
                             int oz, int fx, int fy, int fz) {
    const long long n = (long long)ox * oy * oz;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % ox);
        const long long r = i / ox;
        const int y = (int)(r % oy), z = (int)(r / oy);
        Tout vz[2];
#pragma unroll
        for (int kz = 0; kz < 2; ++kz) {
            if (kz >= fz) { vz[kz] = vz[0]; continue; }
            Tout vy[2];
#pragma unroll
            for (int ky = 0; ky < 2; ++ky) {
                if (ky >= fy) { vy[ky] = vy[0]; continue; }
                const T* p = in + ((size_t)(z * fz + kz) * dy + (y * fy + ky)) * dx + (size_t)x * fx;
                vy[ky] = fx == 2 ? avg2<Tout>((Tout)p[0], (Tout)p[1]) : (Tout)p[0];
            }
            vz[kz] = fy == 2 ? avg2<Tout>(vy[0], vy[1]) : vy[0];
        }
        out[i] = fz == 2 ? avg2<Tout>(vz[0], vz[1]) : vz[0];
    }
}

extern "C" int bs_downsample(bs_ctx* ctx, unsigned long long vol_handle, const int factors[3],
                             unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!factors || !out_handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample: NULL argument");
    for (int d = 0; d < 3; ++d)
        if (factors[d] != 1 && factors[d] != 2) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample: factors must be 1 or 2");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample: unknown handle %llu", vol_handle);
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    const bs_volume src = it->second;
    bs_volume v;
    for (int d = 0; d < 3; ++d) {
        v.dims[d] = src.dims[d] / factors[d];
        if (v.dims[d] < 1) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample: dimension %d too small", d);
    }
    v.dtype = src.dtype;
    v.owned = true;
    const size_t es = src.dtype == BS_DTYPE_U16 ? 2 : src.dtype == BS_DTYPE_F32 ? 4 : 1;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaMalloc(&v.dev, (size_t)v.dims[0] * v.dims[1] * v.dims[2] * es));
    const long long n = v.dims[0] * v.dims[1] * v.dims[2];
    const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)ctx->sm_count * 16);
    {
        bs_launch_scope sc(ctx, "downsample");
        if (src.dtype == BS_DTYPE_U16)
            k_downsample<unsigned short><<<blocks, 256, 0, ctx->stream>>>((const unsigned short*)src.dev, (unsigned short*)v.dev, (int)src.dims[0], (int)src.dims[1], (int)src.dims[2], (int)v.dims[0], (int)v.dims[1], (int)v.dims[2], factors[0], factors[1], factors[2]);
        else if (src.dtype == BS_DTYPE_F32)
            k_downsample<float><<<blocks, 256, 0, ctx->stream>>>((const float*)src.dev, (float*)v.dev, (int)src.dims[0], (int)src.dims[1], (int)src.dims[2], (int)v.dims[0], (int)v.dims[1], (int)v.dims[2], factors[0], factors[1], factors[2]);
        else
            k_downsample<unsigned char><<<blocks, 256, 0, ctx->stream>>>((const unsigned char*)src.dev, (unsigned char*)v.dev, (int)src.dims[0], (int)src.dims[1], (int)src.dims[2], (int)v.dims[0], (int)v.dims[1], (int)v.dims[2], factors[0], factors[1], factors[2]);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_downsample: %s", cudaGetErrorString(e));
    }
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}

// --------------------------------------------------------------------------------------------------------------------
// Interest-point detection input (J/SparkInterestPointDetection.java:1085-1095): the remaining downsampling after the
// mipmap level is a chain of LazyDownsample2x steps to FloatType -- every x halving, then every y, then every z -- each
// the float pair average 0.5f * (a + b) of k_downsample with floor(d / 2) output dims.  One axis per launch, because
// the order of the roundings is part of the result.
static int ds_float_step(bs_ctx* ctx, const void* in, int dtype, float* out, const long long di[3], const long long dout[3],
                         const int f[3]) {
    const long long n = dout[0] * dout[1] * dout[2];
    const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)ctx->sm_count * 16);
    const int a[9] = {(int)di[0], (int)di[1], (int)di[2], (int)dout[0], (int)dout[1], (int)dout[2], f[0], f[1], f[2]};
    bs_launch_scope sc(ctx, "downsample");
    if (dtype == BS_DTYPE_U16)
        k_downsample<unsigned short, float><<<blocks, 256, 0, ctx->stream>>>((const unsigned short*)in, out, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8]);
    else if (dtype == BS_DTYPE_F32)
        k_downsample<float, float><<<blocks, 256, 0, ctx->stream>>>((const float*)in, out, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8]);
    else
        k_downsample<unsigned char, float><<<blocks, 256, 0, ctx->stream>>>((const unsigned char*)in, out, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8]);
    return cudaGetLastError() == cudaSuccess ? BS_OK : BS_ERR_CUDA;
}

extern "C" int bs_downsample_float(bs_ctx* ctx, unsigned long long vol_handle, const int factors[3],
                                   unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!factors || !out_handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample_float: NULL argument");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample_float: unknown handle %llu", vol_handle);
    const bs_volume src = it->second;
    std::vector<int> axes;                       // one entry per 2x step, in the reference's order
    long long dims[3] = {src.dims[0], src.dims[1], src.dims[2]};
    for (int d = 0; d < 3; ++d) {
        const int f = factors[d];
        if (f < 1 || f > 128 || (f & (f - 1)))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample_float: factor %d of axis %d is not a power of two <= 128", f, d);
        for (int g = f; g > 1; g >>= 1) {
            axes.push_back(d);
            dims[d] /= 2;
        }
        if (dims[d] < 1) return bs_set_error(ctx, BS_ERR_ARG, "bs_downsample_float: dimension %d too small", d);
    }
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    if (axes.empty()) axes.push_back(-1);        // no halving: a plain conversion to float
    const void* cur = src.dev;
    int cur_dtype = src.dtype;
    long long cd[3] = {src.dims[0], src.dims[1], src.dims[2]};
    float* prev = nullptr;                       // intermediate owned here (freed once the next step has run)
    int rc = BS_OK;
    for (int ax : axes) {
        int f[3] = {1, 1, 1};
        long long nd[3] = {cd[0], cd[1], cd[2]};
        if (ax >= 0) {
            f[ax] = 2;
            nd[ax] /= 2;
        }
        float* next = nullptr;
        cudaError_t e = cudaMalloc(&next, sizeof(float) * (size_t)(nd[0] * nd[1] * nd[2]));
        if (e != cudaSuccess) {
            rc = bs_set_error(ctx, BS_ERR_NOMEM, "bs_downsample_float: cudaMalloc: %s", cudaGetErrorString(e));
            break;
        }
        if (ds_float_step(ctx, cur, cur_dtype, next, cd, nd, f) != BS_OK) {
            rc = bs_set_error(ctx, BS_ERR_CUDA, "bs_downsample_float: launch failed");
            cudaFree(next);
            break;
        }
        if (prev) {                              // the step just queued reads it
            cudaStreamSynchronize(ctx->stream);
            cudaFree(prev);
        }
        prev = next;
        cur = next;
        cur_dtype = BS_DTYPE_F32;
        for (int d = 0; d < 3; ++d) cd[d] = nd[d];
    }
    if (!rc) {
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) rc = bs_set_error(ctx, BS_ERR_CUDA, "bs_downsample_float: %s", cudaGetErrorString(e));
    }
    if (rc) {
        cudaStreamSynchronize(ctx->stream);
        if (prev) cudaFree(prev);
        return rc;
    }
    bs_volume v;
    v.dev = prev;
    for (int d = 0; d < 3; ++d) v.dims[d] = cd[d];
    v.dtype = BS_DTYPE_F32;
    v.owned = true;
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}
