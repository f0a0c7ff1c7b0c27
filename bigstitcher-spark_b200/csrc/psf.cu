// extract-psfs (mvrecon PSFExtraction, recalled): the sum over bead positions of the n-linearly sampled box around each
// bead, on a resident window of a view's full-resolution level.
//
// One thread per PSF voxel (offset o in [-h, h], x fastest).  The points stream through shared memory in tiles of
// PSF_TILE, in the order given; every thread samples each point p at p + o with the arithmetic of bs_sample_nlinear
// (PARITY_GAPS #37: double weights, each corner term (float)(v w), the eight terms summed in float, x toggling fastest,
// on the border extension of the FULL view) and adds the sample to a double register.  The sum starts from the value
// passed in, so a host that hands the points over in several calls, in order, gets the same double operations in the
// same order as one call: the result does not depend on how the points are split.
#include <climits>

#include "bs_internal.cuh"

namespace {

constexpr int PSF_THREADS = 64;     // few voxels (9 025 for 19 x 19 x 25): small CTAs spread them over more SMs
constexpr int PSF_TILE = 256;       // points staged per tile (3 doubles each)

struct PsfArgs {
    const void* vol;
    int wdims[3];                   // window size
    long long wmin[3];              // window origin in the full view
    long long full[3];              // full view size (border extension)
    const double* pts;              // [n][3] {x, y, z}
    int n;
    int s[3];                       // PSF size (odd)
    double* sum;                    // [sz][sy][sx]
};

template <typename T>
__device__ __forceinline__ float psf_sample(const T* __restrict__ vol, const PsfArgs& a, double px, double py, double pz) {
    const double p[3] = {px, py, pz};
    double t[3];
    long long b[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double f = floor(p[d]);
        t[d] = p[d] - f;
        b[d] = (long long)f;
    }
    float acc = 0.f;
#pragma unroll
    for (int code = 0; code < 8; ++code) {     // x toggles fastest
        double w = 1.0;
        int idx[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const int bit = (code >> d) & 1;
            w *= bit ? t[d] : 1.0 - t[d];
            long long q = b[d] + bit;           // Views.extendBorder of the full view
            q = q < 0 ? 0 : q >= a.full[d] ? a.full[d] - 1 : q;
            q -= a.wmin[d];                     // the host's window covers every tap; stay inside it regardless
            idx[d] = (int)(q < 0 ? 0 : q >= a.wdims[d] ? a.wdims[d] - 1 : q);
        }
        const float v = (float)vol[((long long)idx[2] * a.wdims[1] + idx[1]) * a.wdims[0] + idx[0]];
        acc += (float)((double)v * w);          // FloatType.mul(double) then add
    }
    return acc;
}

template <typename T>
__global__ void __launch_bounds__(PSF_THREADS) k_psf_accumulate(const __grid_constant__ PsfArgs a) {
    __shared__ double tile[3 * PSF_TILE];
    const int nvox = a.s[0] * a.s[1] * a.s[2];
    const int i = blockIdx.x * PSF_THREADS + threadIdx.x;
    const bool live = i < nvox;
    const int x = live ? i % a.s[0] : 0, y = live ? (i / a.s[0]) % a.s[1] : 0, z = live ? i / (a.s[0] * a.s[1]) : 0;
    const double ox = (double)(x - (a.s[0] - 1) / 2), oy = (double)(y - (a.s[1] - 1) / 2),
                 oz = (double)(z - (a.s[2] - 1) / 2);
    const T* __restrict__ vol = static_cast<const T*>(a.vol);
    double acc = live ? a.sum[i] : 0.0;
    for (int base = 0; base < a.n; base += PSF_TILE) {
        const int m = min(PSF_TILE, a.n - base);
        __syncthreads();
        for (int j = threadIdx.x; j < 3 * m; j += PSF_THREADS) tile[j] = a.pts[3LL * base + j];
        __syncthreads();
        if (!live) continue;
#pragma unroll 2
        for (int k = 0; k < m; ++k)
            acc += (double)psf_sample(vol, a, tile[3 * k] + ox, tile[3 * k + 1] + oy, tile[3 * k + 2] + oz);
    }
    if (live) a.sum[i] = acc;
}

}  // namespace

extern "C" int bs_psf_accumulate(bs_ctx* ctx, unsigned long long vol_handle, const long long window_min[3],
                                 const long long full_dims[3], const double* points_xyz, int n, const int psf_size[3],
                                 double* sum) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!window_min || !full_dims || !psf_size || !sum || n < 0 || (n > 0 && !points_xyz))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_psf_accumulate: NULL argument or n < 0");
    long long nvox = 1;
    for (int d = 0; d < 3; ++d) {
        if (psf_size[d] < 1 || psf_size[d] % 2 == 0)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_psf_accumulate: psf_size %d %d %d must be odd and >= 1",
                                psf_size[0], psf_size[1], psf_size[2]);
        nvox *= psf_size[d];
    }
    if (nvox > (1LL << 30)) return bs_set_error(ctx, BS_ERR_ARG, "bs_psf_accumulate: PSF of %lld voxels", nvox);
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_psf_accumulate: unknown handle %llu", vol_handle);
    const bs_volume& src0 = it->second;
    for (int d = 0; d < 3; ++d)
        if (window_min[d] < 0 || src0.dims[d] < 1 || src0.dims[d] > INT_MAX || window_min[d] + src0.dims[d] > full_dims[d])
            return bs_set_error(ctx, BS_ERR_ARG, "bs_psf_accumulate: window [%lld, %lld) of axis %d outside the view of "
                                "size %lld", window_min[d], window_min[d] + src0.dims[d], d, full_dims[d]);
    if (n == 0) return BS_OK;
    { int rc0 = bs_volume_acquire(ctx, it->second); if (rc0) return rc0; }
    const bs_volume src = it->second;
    PsfArgs a;
    a.vol = src.dev;
    a.n = n;
    for (int d = 0; d < 3; ++d) {
        a.wdims[d] = (int)src.dims[d];
        a.wmin[d] = window_min[d];
        a.full[d] = full_dims[d];
        a.s[d] = psf_size[d];
    }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    void* buf = nullptr;
    const size_t sum_bytes = sizeof(double) * (size_t)nvox, pts_bytes = sizeof(double) * 3 * (size_t)n;
    BS_CUDA(ctx, cudaMalloc(&buf, sum_bytes + pts_bytes));
    a.sum = static_cast<double*>(buf);
    a.pts = reinterpret_cast<const double*>(static_cast<char*>(buf) + sum_bytes);
    cudaError_t e = cudaMemcpyAsync(a.sum, sum, sum_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(const_cast<double*>(a.pts), points_xyz, pts_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        const unsigned blocks = (unsigned)((nvox + PSF_THREADS - 1) / PSF_THREADS);
        bs_launch_scope sc(ctx, "psf");
        if (src.dtype == BS_DTYPE_U16) k_psf_accumulate<unsigned short><<<blocks, PSF_THREADS, 0, ctx->stream>>>(a);
        else if (src.dtype == BS_DTYPE_F32) k_psf_accumulate<float><<<blocks, PSF_THREADS, 0, ctx->stream>>>(a);
        else k_psf_accumulate<unsigned char><<<blocks, PSF_THREADS, 0, ctx->stream>>>(a);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(sum, a.sum, sum_bytes, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(buf);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_psf_accumulate: %s", cudaGetErrorString(e));
    }
    cudaFree(buf);
    return BS_OK;
}
