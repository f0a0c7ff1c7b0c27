// estimate-bounding-box (mvrecon BoundingBoxMinFilterThreshold) on a resident float32 volume:
//   bs_min_filter      box minimum of radius r per axis, as three separable 1-D passes (x, then y, then z)
//   bs_volume_min_max  min and max of the volume (NaN ignored)
//   bs_threshold_bbox  index bounding box and count of the voxels > t
//
// Min filter: a direct window in shared memory.  Each CTA stages its output run plus an r-voxel halo on both sides of
// the filtered axis; every thread takes the fminf of the 2r + 1 staged values of its output.  Voxels outside the
// volume are staged as NaN, which fminf ignores, so the window is clipped to the volume exactly (for a box, a mirror or
// border extension gives the same minimum).  A radius larger than MF_MAX_R is split into passes of at most MF_MAX_R:
// min is associative and the clipped windows compose (radius a then b equals radius a + b), so the result is the same
// minimum and bit-identical to any other evaluation order.  Radii are first clipped to n - 1.
//
// Reductions: per-thread partials, warp shuffles, then one integer atomic per CTA and value (float min / max through
// order-preserving uint32 keys), so the results do not depend on scheduling.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <utility>

#include "bs_internal.cuh"

namespace {

constexpr int MF_MAX_R = 64;     // largest radius of one pass
constexpr int MFX_TX = 128;      // x pass: outputs per CTA row
constexpr int MFX_ROWS = 2;      // x pass: rows per CTA
constexpr int MFA_TI = 32;       // y / z pass: lanes along x (the contiguous direction)
constexpr int MFA_TY = 8;        // y / z pass: thread rows along the filtered axis
constexpr int MFA_TA = 64;       // y / z pass: outputs per CTA along the filtered axis

__device__ __forceinline__ unsigned fkey(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

float fkey_inv_host(unsigned k) {
    const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float f;
    std::memcpy(&f, &u, sizeof f);
    return f;
}

// x pass: rows of nx voxels, row index = y + ny * z
__global__ void __launch_bounds__(MFX_TX * MFX_ROWS)
k_min_filter_x(const float* __restrict__ in, float* __restrict__ out, int nx, long long rows, int r) {
    __shared__ float s[MFX_ROWS][MFX_TX + 2 * MF_MAX_R];
    const long long row = (long long)blockIdx.x * MFX_ROWS + threadIdx.y;
    const int x0 = blockIdx.y * MFX_TX;
    const float nan = __uint_as_float(0x7fc00000u);
    if (row < rows) {
        const float* src = in + row * nx;
        for (int i = threadIdx.x; i < MFX_TX + 2 * r; i += MFX_TX) {
            const int x = x0 - r + i;
            s[threadIdx.y][i] = (x >= 0 && x < nx) ? src[x] : nan;
        }
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    if (row >= rows || x >= nx) return;
    const float* w = s[threadIdx.y] + threadIdx.x;
    float m = w[0];
    for (int k = 1; k <= 2 * r; ++k) m = fminf(m, w[k]);
    out[row * nx + x] = m;
}

// y or z pass: voxel (o, a, i) at o * n * stride + a * stride + i, a the filtered axis of length n, i < stride
__global__ void __launch_bounds__(MFA_TI * MFA_TY)
k_min_filter_axis(const float* __restrict__ in, float* __restrict__ out, long long stride, int n, int r) {
    __shared__ float s[MFA_TA + 2 * MF_MAX_R][MFA_TI];
    const long long i0 = (long long)blockIdx.x * MFA_TI;
    const int a0 = blockIdx.y * MFA_TA;
    const long long base = (long long)blockIdx.z * n * stride;
    const float nan = __uint_as_float(0x7fc00000u);
    const int tid = threadIdx.y * MFA_TI + threadIdx.x;
    for (int j = tid; j < (MFA_TA + 2 * r) * MFA_TI; j += MFA_TI * MFA_TY) {
        const int row = j / MFA_TI, col = j - row * MFA_TI;
        const int a = a0 - r + row;
        const long long i = i0 + col;
        s[row][col] = (a >= 0 && a < n && i < stride) ? in[base + (long long)a * stride + i] : nan;
    }
    __syncthreads();
    const long long i = i0 + threadIdx.x;
    if (i >= stride) return;
    for (int q = threadIdx.y; q < MFA_TA; q += MFA_TY) {
        const int a = a0 + q;
        if (a >= n) break;
        float m = s[q][threadIdx.x];
        for (int k = 1; k <= 2 * r; ++k) m = fminf(m, s[q + k][threadIdx.x]);
        out[base + (long long)a * stride + i] = m;
    }
}

__device__ __forceinline__ unsigned warp_min_u(unsigned v) {
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ unsigned warp_max_u(unsigned v) {
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_min_i(int v) {
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_max_i(int v) {
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// keys[0] = min key, keys[1] = max key over the non-NaN voxels (0xffffffff / 0 when there are none)
__global__ void __launch_bounds__(256) k_min_max(const float* __restrict__ v, long long n, unsigned* keys) {
    unsigned lo = 0xffffffffu, hi = 0u;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float f = v[i];
        if (f == f) {
            const unsigned k = fkey(f);
            lo = min(lo, k);
            hi = max(hi, k);
        }
    }
    lo = warp_min_u(lo);
    hi = warp_max_u(hi);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&keys[0], lo);
        atomicMax(&keys[1], hi);
    }
}

struct BboxAcc {
    int mn[3];
    int mx[3];
    unsigned long long count;
};

// rows (y, z) of nx voxels; a voxel is kept when (double)v > t
__global__ void __launch_bounds__(256) k_threshold_bbox(const float* __restrict__ v, int nx, int ny, long long rows,
                                                        double t, BboxAcc* acc) {
    int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {-1, -1, -1};
    unsigned long long cnt = 0;
    const int lanes = blockDim.x;
    for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
        const float* src = v + row * nx;
        int rmn = INT_MAX, rmx = -1;
        for (int x = threadIdx.x; x < nx; x += lanes) {
            if ((double)src[x] > t) {
                rmn = min(rmn, x);
                rmx = max(rmx, x);
                ++cnt;
            }
        }
        if (rmx >= 0) {
            const int y = (int)(row % ny), z = (int)(row / ny);
            mn[0] = min(mn[0], rmn); mx[0] = max(mx[0], rmx);
            mn[1] = min(mn[1], y);   mx[1] = max(mx[1], y);
            mn[2] = min(mn[2], z);   mx[2] = max(mx[2], z);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        mn[d] = warp_min_i(mn[d]);
        mx[d] = warp_max_i(mx[d]);
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            atomicMin(&acc->mn[d], mn[d]);
            atomicMax(&acc->mx[d], mx[d]);
        }
        atomicAdd(&acc->count, cnt);
    }
}

// the resident float32 volume behind a handle, or an error
int f32_volume(bs_ctx* ctx, unsigned long long handle, const char* fn, bs_volume** out) {
    auto it = ctx->vols.find(handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "%s: unknown handle %llu", fn, handle);
    if (it->second.dtype != BS_DTYPE_F32) return bs_set_error(ctx, BS_ERR_ARG, "%s: the volume is not float32", fn);
    const long long* d = it->second.dims;
    if (d[0] > INT_MAX || d[1] > INT_MAX || d[2] > 65535)
        return bs_set_error(ctx, BS_ERR_ARG, "%s: volume too large", fn);
    int rc = bs_volume_acquire(ctx, it->second);
    if (rc) return rc;
    *out = &it->second;
    return BS_OK;
}

int grid_for(bs_ctx* ctx, long long work) {
    const long long cap = (long long)ctx->sm_count * 8;
    return (int)(work < 1 ? 1 : work < cap ? work : cap);
}

}  // namespace

extern "C" int bs_min_filter(bs_ctx* ctx, unsigned long long vol_handle, const int radius[3],
                             unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!radius || !out_handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_min_filter: NULL argument");
    for (int d = 0; d < 3; ++d)
        if (radius[d] < 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_min_filter: radius[%d] = %d < 0", d, radius[d]);
    bs_volume* src = nullptr;
    { int rc = f32_volume(ctx, vol_handle, "bs_min_filter", &src); if (rc) return rc; }
    const long long nx = src->dims[0], ny = src->dims[1], nz = src->dims[2];
    const size_t bytes = sizeof(float) * (size_t)(nx * ny * nz);
    // the passes: (axis, radius <= MF_MAX_R), radii clipped to n - 1
    std::vector<std::pair<int, int>> passes;
    for (int d = 0; d < 3; ++d)
        for (long long left = std::min<long long>(radius[d], src->dims[d] - 1); left > 0; left -= MF_MAX_R)
            passes.push_back({d, (int)std::min<long long>(left, MF_MAX_R)});
    bs_volume v;
    for (int d = 0; d < 3; ++d) v.dims[d] = src->dims[d];
    v.dtype = BS_DTYPE_F32;
    v.owned = true;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    void* tmp = nullptr;
    BS_CUDA(ctx, cudaMalloc(&v.dev, bytes));
    cudaError_t e = cudaSuccess;
    if (passes.size() > 1) e = cudaMalloc(&tmp, bytes);
    const float* cur = static_cast<const float*>(src->dev);
    if (e == cudaSuccess && passes.empty())
        e = cudaMemcpyAsync(v.dev, cur, bytes, cudaMemcpyDeviceToDevice, ctx->stream);
    for (size_t p = 0; p < passes.size() && e == cudaSuccess; ++p) {
        // alternate between the two buffers so that the last pass writes the output volume
        float* dst = static_cast<float*>((passes.size() - 1 - p) % 2 == 0 ? v.dev : tmp);
        const int axis = passes[p].first, r = passes[p].second;
        bs_launch_scope sc(ctx, "min_filter");
        if (axis == 0) {
            const long long rows = ny * nz;
            const dim3 grid((unsigned)((rows + MFX_ROWS - 1) / MFX_ROWS), (unsigned)((nx + MFX_TX - 1) / MFX_TX));
            k_min_filter_x<<<grid, dim3(MFX_TX, MFX_ROWS), 0, ctx->stream>>>(cur, dst, (int)nx, rows, r);
        } else {
            const long long stride = axis == 1 ? nx : nx * ny;
            const int n = (int)src->dims[axis];
            const dim3 grid((unsigned)((stride + MFA_TI - 1) / MFA_TI), (unsigned)((n + MFA_TA - 1) / MFA_TA),
                            (unsigned)(axis == 1 ? nz : 1));
            k_min_filter_axis<<<grid, dim3(MFA_TI, MFA_TY), 0, ctx->stream>>>(cur, dst, stride, n, r);
        }
        e = cudaGetLastError();
        cur = dst;
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (tmp) cudaFree(tmp);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, e == cudaErrorMemoryAllocation ? BS_ERR_NOMEM : BS_ERR_CUDA, "bs_min_filter: %s",
                            cudaGetErrorString(e));
    }
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}

extern "C" int bs_volume_min_max(bs_ctx* ctx, unsigned long long vol_handle, double out[2]) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!out) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_min_max: NULL argument");
    bs_volume* src = nullptr;
    { int rc = f32_volume(ctx, vol_handle, "bs_volume_min_max", &src); if (rc) return rc; }
    const long long n = src->dims[0] * src->dims[1] * src->dims[2];
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    unsigned* keys = nullptr;
    BS_CUDA(ctx, cudaMalloc(&keys, 2 * sizeof(unsigned)));
    const unsigned init[2] = {0xffffffffu, 0u};
    unsigned host[2];
    cudaError_t e = cudaMemcpyAsync(keys, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        bs_launch_scope sc(ctx, "min_max");
        k_min_max<<<grid_for(ctx, (n + 255) / 256), 256, 0, ctx->stream>>>(static_cast<const float*>(src->dev), n, keys);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(host, keys, sizeof(host), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(keys);
    if (e != cudaSuccess) return bs_set_error(ctx, BS_ERR_CUDA, "bs_volume_min_max: %s", cudaGetErrorString(e));
    if (host[0] == 0xffffffffu && host[1] == 0u) {       // no voxel, or every voxel NaN
        out[0] = out[1] = NAN;
    } else {
        out[0] = (double)fkey_inv_host(host[0]);
        out[1] = (double)fkey_inv_host(host[1]);
    }
    return BS_OK;
}

extern "C" int bs_threshold_bbox(bs_ctx* ctx, unsigned long long vol_handle, double t, long long min[3], long long max[3],
                                 long long* count) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!min || !max || !count) return bs_set_error(ctx, BS_ERR_ARG, "bs_threshold_bbox: NULL argument");
    bs_volume* src = nullptr;
    { int rc = f32_volume(ctx, vol_handle, "bs_threshold_bbox", &src); if (rc) return rc; }
    const long long rows = src->dims[1] * src->dims[2];
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BboxAcc* acc = nullptr;
    BS_CUDA(ctx, cudaMalloc(&acc, sizeof(BboxAcc)));
    BboxAcc h = {{INT_MAX, INT_MAX, INT_MAX}, {-1, -1, -1}, 0ull};
    cudaError_t e = cudaMemcpyAsync(acc, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        bs_launch_scope sc(ctx, "threshold_bbox");
        k_threshold_bbox<<<grid_for(ctx, rows), 256, 0, ctx->stream>>>(static_cast<const float*>(src->dev),
                                                                       (int)src->dims[0], (int)src->dims[1], rows, t, acc);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h, acc, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(acc);
    if (e != cudaSuccess) return bs_set_error(ctx, BS_ERR_CUDA, "bs_threshold_bbox: %s", cudaGetErrorString(e));
    *count = (long long)h.count;
    for (int d = 0; d < 3; ++d) {
        min[d] = h.count ? h.mn[d] : -1;
        max[d] = h.count ? h.mx[d] : -1;
    }
    return BS_OK;
}
