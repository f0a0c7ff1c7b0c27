// Interest-point detection helpers around bs_dog_detect (J/SparkInterestPointDetection.java:532-604):
//   bs_median_divide  --medianFilter r: every z-slice divided by its own circular median (LazyBackgroundSubtract)
//   bs_sample_nlinear --storeIntensities / --maxSpots: n-linear intensities of the detections (border extension)
//
// Median: one thread per output voxel, the slice tile plus an r-voxel mirror-double halo staged in shared memory as
// order-preserving uint32 keys.  The exact median (rank (n-1)/2 of the n footprint keys, n odd) is found by bitwise
// bisection: the answer is the largest key t with #{keys < t} <= rank, built from the high bit down.  Bits shared by
// the footprint's minimum and maximum key are fixed by one min/max pass, so a footprint spanning a narrow value range
// needs fewer counting passes.  Only comparisons are involved, so the median is one of the input values bit for bit and
// the result is bit-identical to any exact selection followed by the same IEEE division.
#include <cmath>

#include "bs_internal.cuh"

#define MD_TX 32
#define MD_TY 8

namespace {

__device__ __forceinline__ int mirror_double(int i, int n) {
    // Views.extendMirrorDouble / np.pad(mode="symmetric"): ... c b a | a b c ... (also several periods out)
    const int period = 2 * n;
    i %= period;
    if (i < 0) i += period;
    return i < n ? i : period - 1 - i;
}

__device__ __forceinline__ unsigned fkey(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float fkey_inv(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <typename T>
__device__ __forceinline__ float to_f(const T* p, long long i) { return (float)p[i]; }

struct MedianArgs {
    const void* in;
    float* out;
    int dims[3];
    int r;                               // kRadius of the ImageJ kernel (== the integer radius)
    int rank;                            // (n - 1) / 2
    int hw[2 * BS_MEDIAN_MAX_RADIUS + 1]; // half width of row dy + r
};

template <typename T>
__global__ void __launch_bounds__(MD_TX * MD_TY) k_median_divide(const __grid_constant__ MedianArgs a) {
    extern __shared__ unsigned md_keys[];
    const int r = a.r, W = MD_TX + 2 * r, H = MD_TY + 2 * r;
    const int nx = a.dims[0], ny = a.dims[1];
    const int x0 = blockIdx.x * MD_TX, y0 = blockIdx.y * MD_TY, z = blockIdx.z;
    const T* src = static_cast<const T*>(a.in) + (long long)z * nx * ny;
    const int tid = threadIdx.y * MD_TX + threadIdx.x;
    for (int i = tid; i < W * H; i += MD_TX * MD_TY) {
        const int ty = i / W, tx = i - ty * W;
        const int gx = mirror_double(x0 - r + tx, nx), gy = mirror_double(y0 - r + ty, ny);
        md_keys[i] = fkey(to_f(src, (long long)gy * nx + gx));
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= nx || y >= ny) return;
    const unsigned* c = md_keys + (threadIdx.y + r) * W + threadIdx.x + r;
    unsigned lo = 0xffffffffu, hi = 0u;
    for (int dy = -r; dy <= r; ++dy) {
        const unsigned* row = c + dy * W;
        const int h = a.hw[dy + r];
        for (int dx = -h; dx <= h; ++dx) {
            const unsigned k = row[dx];
            lo = min(lo, k);
            hi = max(hi, k);
        }
    }
    unsigned ans = lo;
    if (lo != hi) {
        const int nb = 32 - __clz(lo ^ hi);                 // bits below the common prefix of lo and hi
        ans = nb == 32 ? 0u : (lo >> nb) << nb;
        for (int b = nb - 1; b >= 0; --b) {
            const unsigned cand = ans | (1u << b);
            int cnt = 0;
            for (int dy = -r; dy <= r; ++dy) {
                const unsigned* row = c + dy * W;
                const int h = a.hw[dy + r];
                for (int dx = -h; dx <= h; ++dx) cnt += row[dx] < cand;
            }
            if (cnt <= a.rank) ans = cand;
        }
    }
    const float m = fkey_inv(ans), v = fkey_inv(c[0]);
    a.out[((long long)z * ny + y) * nx + x] = m > 0.f ? v / m : 0.f;
}

template <typename T>
__global__ void k_sample_nlinear(const T* __restrict__ vol, int nx, int ny, int nz, const double* __restrict__ loc, int n,
                                 float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double px = loc[3 * i], py = loc[3 * i + 1], pz = loc[3 * i + 2];
    const double fx = floor(px), fy = floor(py), fz = floor(pz);
    const double t[3] = {px - fx, py - fy, pz - fz};
    const long long b[3] = {(long long)fx, (long long)fy, (long long)fz};
    const int dims[3] = {nx, ny, nz};
    float acc = 0.f;
#pragma unroll
    for (int code = 0; code < 8; ++code) {     // x toggles fastest
        double w = 1.0;
        int idx[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const int bit = (code >> d) & 1;
            w *= bit ? t[d] : 1.0 - t[d];
            const long long p = b[d] + bit;     // Views.extendBorder
            idx[d] = (int)(p < 0 ? 0 : p >= dims[d] ? dims[d] - 1 : p);
        }
        const float v = (float)vol[((long long)idx[2] * ny + idx[1]) * nx + idx[0]];
        acc += (float)((double)v * w);          // FloatType.mul(double) then add
    }
    out[i] = acc;
}

}  // namespace

extern "C" int bs_median_divide(bs_ctx* ctx, unsigned long long vol_handle, int radius, unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!out_handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_median_divide: NULL argument");
    if (radius < 1 || radius > BS_MEDIAN_MAX_RADIUS)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_median_divide: radius %d outside [1, %d]", radius, BS_MEDIAN_MAX_RADIUS);
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_median_divide: unknown handle %llu", vol_handle);
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    const bs_volume src = it->second;
    if (src.dims[0] > 1 << 30 || src.dims[1] > 1 << 30 || src.dims[2] > 65535)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_median_divide: volume too large");
    // RankFilters.makeLineRadii(radius) for an integer radius: r2 = r*r + 1, kRadius = floor(sqrt(r2)), row dy spans
    // |dx| <= floor(sqrt(r2 - dy^2 + 1e-10))
    MedianArgs a;
    const int r2 = radius * radius + 1;
    const int kr = (int)std::sqrt(r2 + 1e-10);
    int n = 0;
    for (int dy = -kr; dy <= kr; ++dy) {
        a.hw[dy + kr] = (int)std::sqrt(r2 - dy * dy + 1e-10);
        n += 2 * a.hw[dy + kr] + 1;
    }
    a.r = kr;
    a.rank = (n - 1) / 2;
    a.in = src.dev;
    for (int d = 0; d < 3; ++d) a.dims[d] = (int)src.dims[d];
    bs_volume v;
    for (int d = 0; d < 3; ++d) v.dims[d] = src.dims[d];
    v.dtype = BS_DTYPE_F32;
    v.owned = true;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaMalloc(&v.dev, sizeof(float) * (size_t)(v.dims[0] * v.dims[1] * v.dims[2])));
    a.out = static_cast<float*>(v.dev);
    const size_t smem = sizeof(unsigned) * (size_t)(MD_TX + 2 * kr) * (MD_TY + 2 * kr);
    const dim3 grid((unsigned)((src.dims[0] + MD_TX - 1) / MD_TX), (unsigned)((src.dims[1] + MD_TY - 1) / MD_TY),
                    (unsigned)src.dims[2]);
    const dim3 block(MD_TX, MD_TY);
    {
        bs_launch_scope sc(ctx, "median");
        if (src.dtype == BS_DTYPE_U16) k_median_divide<unsigned short><<<grid, block, smem, ctx->stream>>>(a);
        else if (src.dtype == BS_DTYPE_F32) k_median_divide<float><<<grid, block, smem, ctx->stream>>>(a);
        else k_median_divide<unsigned char><<<grid, block, smem, ctx->stream>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_median_divide: %s", cudaGetErrorString(e));
    }
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}

extern "C" int bs_sample_nlinear(bs_ctx* ctx, unsigned long long vol_handle, int n, const double* loc_xyz, float* out) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n < 0 || (n > 0 && (!loc_xyz || !out))) return bs_set_error(ctx, BS_ERR_ARG, "bs_sample_nlinear: bad argument");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_sample_nlinear: unknown handle %llu", vol_handle);
    if (n == 0) return BS_OK;
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    const bs_volume src = it->second;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    void* buf = nullptr;
    const size_t loc_bytes = sizeof(double) * 3 * (size_t)n;
    BS_CUDA(ctx, cudaMalloc(&buf, loc_bytes + sizeof(float) * (size_t)n));
    double* dloc = static_cast<double*>(buf);
    float* dout = reinterpret_cast<float*>(static_cast<char*>(buf) + loc_bytes);
    cudaError_t e = cudaMemcpyAsync(dloc, loc_xyz, loc_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        const int nx = (int)src.dims[0], ny = (int)src.dims[1], nz = (int)src.dims[2];
        const unsigned blocks = (unsigned)((n + 255) / 256);
        bs_launch_scope sc(ctx, "sample");
        if (src.dtype == BS_DTYPE_U16)
            k_sample_nlinear<unsigned short><<<blocks, 256, 0, ctx->stream>>>((const unsigned short*)src.dev, nx, ny, nz, dloc, n, dout);
        else if (src.dtype == BS_DTYPE_F32)
            k_sample_nlinear<float><<<blocks, 256, 0, ctx->stream>>>((const float*)src.dev, nx, ny, nz, dloc, n, dout);
        else
            k_sample_nlinear<unsigned char><<<blocks, 256, 0, ctx->stream>>>((const unsigned char*)src.dev, nx, ny, nz, dloc, n, dout);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, dout, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(buf);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_sample_nlinear: %s", cudaGetErrorString(e));
    }
    cudaFree(buf);
    return BS_OK;
}
