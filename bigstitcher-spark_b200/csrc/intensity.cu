// Intensity correction (match-intensities / affine-fusion --intensityN5Path): pair candidates, RANSAC hypotheses and
// the coefficient application.  Only the CUDA runtime; no CUB / Thrust.
//
// Candidates of one view pair (bs_intensity_pair_candidates): every point r of the render grid (world r / s) is
// back-projected into both views in FP64, sampled n-linearly on each view's level volume and bucketed by
// (cell of A, cell of B).  The output order is fixed without atomics deciding any position:
//   pass A, per z-chunk: k_render counts the points of every key (atomic adds; only the totals are used);
//   k_compact (one CTA): the present keys become slots in ascending key order, with bucket offsets;
//   pass B, per z-chunk: k_render stores key + values per point, k_seg_count counts each slot per segment of
//   kSeg points (one warp walks a segment in render order), k_seg_scan turns the counts into per-(segment, slot)
//   cursors that continue from the previous chunk, and k_scatter writes every value at its cursor, again walking each
//   segment in render order (ranks among equal slots from __match_any_sync).
// A chunked run therefore writes exactly what an unchunked one does.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "bs_internal.cuh"

namespace {

constexpr int kSeg = 4096;                      // points per segment of pass B
constexpr long long kDefaultChunk = 1LL << 24;  // render points per z-chunk (12 B each in pass B)
constexpr long long kMaxKeys = 1LL << 26;       // cells(A) * cells(B)
constexpr unsigned long long kSeed = 0x2545F4914F6CDD1DULL;

struct IView {
    const void* data;
    int dtype;
    int ldims[3];        // level volume
    double w2p[12];      // world -> full-resolution pixel
    double p2l[12];      // full-resolution pixel -> level pixel
    double fdims[3];     // full-resolution dims
    int n[3];            // cells per axis
};

struct RenderArgs {
    IView A, B;
    double tmin, tmax;   // tmax NaN: no upper threshold
    const double* w[3];  // world coordinate r / s of every render grid index, per axis
    long long nx, ny;    // render grid x / y extents
    long long z0;        // first render plane of this chunk (relative to r0[2])
    long long npts;      // points in this chunk
    int nb_cells;        // cells of B
};

__device__ __forceinline__ double affine_row(const double* m, int r, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4 * r], x), __dmul_rn(m[4 * r + 1], y)), __dmul_rn(m[4 * r + 2], z)),
                     m[4 * r + 3]);
}

template <typename T>
__device__ __forceinline__ float ldf(const T* p, size_t i) { return (float)__ldg(p + i); }

// n-linear sample with border extension on both sides (the float32 arithmetic of sample() in fuse_common.cuh)
template <typename T>
__device__ __forceinline__ float sample_clamped(const T* __restrict__ d, int dx, int dy, int dz, float sx, float sy, float sz) {
    const float fx = floorf(sx), fy = floorf(sy), fz = floorf(sz);
    const float rx = sx - fx, ry = sy - fy, rz = sz - fz;
    const int ix = (int)fx, iy = (int)fy, iz = (int)fz;
    const int x0 = min(max(ix, 0), dx - 1), x1 = min(max(ix + 1, 0), dx - 1);
    const int y0 = min(max(iy, 0), dy - 1), y1 = min(max(iy + 1, 0), dy - 1);
    const int z0 = min(max(iz, 0), dz - 1), z1 = min(max(iz + 1, 0), dz - 1);
    const size_t r00 = ((size_t)z0 * dy + y0) * dx, r01 = ((size_t)z0 * dy + y1) * dx;
    const size_t r10 = ((size_t)z1 * dy + y0) * dx, r11 = ((size_t)z1 * dy + y1) * dx;
    const float a000 = ldf(d, r00 + x0), a001 = ldf(d, r00 + x1), a010 = ldf(d, r01 + x0), a011 = ldf(d, r01 + x1);
    const float a100 = ldf(d, r10 + x0), a101 = ldf(d, r10 + x1), a110 = ldf(d, r11 + x0), a111 = ldf(d, r11 + x1);
    const float c00 = __fadd_rn(a000, __fmul_rn(rx, __fsub_rn(a001, a000)));
    const float c01 = __fadd_rn(a010, __fmul_rn(rx, __fsub_rn(a011, a010)));
    const float c10 = __fadd_rn(a100, __fmul_rn(rx, __fsub_rn(a101, a100)));
    const float c11 = __fadd_rn(a110, __fmul_rn(rx, __fsub_rn(a111, a110)));
    const float c0 = __fadd_rn(c00, __fmul_rn(ry, __fsub_rn(c01, c00)));
    const float c1 = __fadd_rn(c10, __fmul_rn(ry, __fsub_rn(c11, c10)));
    return __fadd_rn(c0, __fmul_rn(rz, __fsub_rn(c1, c0)));
}

// value and cell of one view at world (wx, wy, wz); false when the point is outside [0, d-1] or thresholded away
__device__ __forceinline__ bool view_point(const IView& V, double wx, double wy, double wz, double tmin, double tmax, float& v, int& cell) {
    double p[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        p[r] = affine_row(V.w2p, r, wx, wy, wz);
        if (!(p[r] >= 0.0 && p[r] <= V.fdims[r] - 1.0)) return false;
    }
    float q[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) q[r] = (float)affine_row(V.p2l, r, p[0], p[1], p[2]);
    if (V.dtype == BS_DTYPE_U16)
        v = sample_clamped((const unsigned short*)V.data, V.ldims[0], V.ldims[1], V.ldims[2], q[0], q[1], q[2]);
    else if (V.dtype == BS_DTYPE_F32)
        v = sample_clamped((const float*)V.data, V.ldims[0], V.ldims[1], V.ldims[2], q[0], q[1], q[2]);
    else
        v = sample_clamped((const unsigned char*)V.data, V.ldims[0], V.ldims[1], V.ldims[2], q[0], q[1], q[2]);
    if (!((double)v >= tmin)) return false;
    if (!isnan(tmax) && !((double)v <= tmax)) return false;
    int c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double f = floor(__ddiv_rn(__dmul_rn(p[r], (double)V.n[r]), V.fdims[r]));
        c[r] = (int)fmin(fmax(f, 0.0), (double)(V.n[r] - 1));
    }
    cell = c[0] + V.n[0] * (c[1] + V.n[1] * c[2]);
    return true;
}

__device__ __forceinline__ int render_key(const RenderArgs& a, long long i, float& va, float& vb) {
    const long long plane = a.nx * a.ny;
    const long long lz = a.z0 + i / plane, rem = i % plane;
    const long long ly = rem / a.nx, lx = rem % a.nx;
    const double wx = __ldg(a.w[0] + lx), wy = __ldg(a.w[1] + ly), wz = __ldg(a.w[2] + lz);
    int ca, cb;
    if (!view_point(a.A, wx, wy, wz, a.tmin, a.tmax, va, ca)) return -1;
    if (!view_point(a.B, wx, wy, wz, a.tmin, a.tmax, vb, cb)) return -1;
    return ca * a.nb_cells + cb;
}

// COUNT: counts[key] += 1; else: key and values per point of the chunk
template <bool COUNT>
__global__ void __launch_bounds__(256) k_render(RenderArgs a, unsigned int* __restrict__ counts, int* __restrict__ keys,
                                                float2* __restrict__ vals) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.npts; i += (long long)gridDim.x * blockDim.x) {
        float va = 0.f, vb = 0.f;
        const int k = render_key(a, i, va, vb);
        if (COUNT) {
            if (k >= 0) atomicAdd(counts + k, 1u);
        } else {
            keys[i] = k;
            vals[i] = make_float2(va, vb);
        }
    }
}

struct CompactOut {
    long long n_slots;
    long long n_values;
};

// one CTA of 1024 threads: slot_of_key (-1 for absent keys), slot -> key / offset / count, totals
__global__ void __launch_bounds__(1024) k_compact(const unsigned int* __restrict__ counts, long long nkeys,
                                                  int* __restrict__ slot_of_key, long long* __restrict__ slot_key,
                                                  long long* __restrict__ slot_off, long long* __restrict__ slot_cnt,
                                                  CompactOut* out) {
    __shared__ long long s_n[1024], s_v[1024];
    const long long per = (nkeys + 1023) / 1024;
    const long long k0 = min(nkeys, per * threadIdx.x), k1 = min(nkeys, k0 + per);
    long long n = 0, v = 0;
    for (long long k = k0; k < k1; ++k)
        if (counts[k]) {
            ++n;
            v += counts[k];
        }
    s_n[threadIdx.x] = n;
    s_v[threadIdx.x] = v;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {   // inclusive Hillis-Steele scan
        long long an = 0, av = 0;
        if (threadIdx.x >= d) {
            an = s_n[threadIdx.x - d];
            av = s_v[threadIdx.x - d];
        }
        __syncthreads();
        s_n[threadIdx.x] += an;
        s_v[threadIdx.x] += av;
        __syncthreads();
    }
    long long slot = s_n[threadIdx.x] - n, off = s_v[threadIdx.x] - v;
    for (long long k = k0; k < k1; ++k) {
        const unsigned c = counts[k];
        if (c) {
            slot_of_key[k] = (int)slot;
            slot_key[slot] = k;
            slot_off[slot] = off;
            slot_cnt[slot] = c;
            ++slot;
            off += c;
        } else {
            slot_of_key[k] = -1;
        }
    }
    if (threadIdx.x == 1023) {
        out->n_slots = s_n[1023];
        out->n_values = s_v[1023];
    }
}

// one warp per segment: counts of every slot in the segment -> hist[seg][slot]
__global__ void __launch_bounds__(32) k_seg_count(const int* __restrict__ keys, long long npts, const int* __restrict__ slot_of_key,
                                                  int n_slots, unsigned int* __restrict__ hist) {
    extern __shared__ unsigned int s_cnt[];
    const long long seg = blockIdx.x;
    for (int s = threadIdx.x; s < n_slots; s += 32) s_cnt[s] = 0;
    __syncwarp();
    const long long b0 = seg * kSeg, b1 = min(npts, b0 + kSeg);
    for (long long base = b0; base < b1; base += 32) {
        const long long i = base + threadIdx.x;
        const int k = i < b1 ? keys[i] : -1;
        const int slot = k >= 0 ? slot_of_key[k] : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, slot);
        if (slot >= 0 && (int)threadIdx.x == __ffs(peers) - 1) s_cnt[slot] += __popc(peers);
        __syncwarp();
    }
    for (int s = threadIdx.x; s < n_slots; s += 32) hist[seg * n_slots + s] = s_cnt[s];
}

// per slot: segment counts -> cursors (exclusive), continuing from cursor[slot] (carried across chunks)
__global__ void k_seg_scan(unsigned int* __restrict__ hist, long long n_seg, int n_slots, long long* __restrict__ cursor,
                           long long* __restrict__ seg_base) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    long long run = cursor[s];
    for (long long g = 0; g < n_seg; ++g) {
        const unsigned c = hist[g * n_slots + s];
        seg_base[g * n_slots + s] = run;
        run += c;
    }
    cursor[s] = run;
}

__global__ void __launch_bounds__(32) k_scatter(const int* __restrict__ keys, const float2* __restrict__ vals, long long npts,
                                                const int* __restrict__ slot_of_key, int n_slots,
                                                const long long* __restrict__ seg_base, float2* __restrict__ out) {
    extern __shared__ long long s_cur[];
    const long long seg = blockIdx.x;
    for (int s = threadIdx.x; s < n_slots; s += 32) s_cur[s] = seg_base[seg * n_slots + s];
    __syncwarp();
    const long long b0 = seg * kSeg, b1 = min(npts, b0 + kSeg);
    const unsigned lt = (1u << threadIdx.x) - 1u;
    for (long long base = b0; base < b1; base += 32) {
        const long long i = base + threadIdx.x;
        const int k = i < b1 ? keys[i] : -1;
        const int slot = k >= 0 ? slot_of_key[k] : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, slot);
        long long pos = 0;
        if (slot >= 0) {
            pos = s_cur[slot] + __popc(peers & lt);
            out[pos] = vals[i];
        }
        __syncwarp();
        if (slot >= 0 && (int)threadIdx.x == __ffs(peers) - 1) s_cur[slot] += __popc(peers);
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------ RANSAC hypotheses
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// the two candidates of hypothesis h and its model; false when x_i == x_j (skipped)
__device__ __forceinline__ bool hypothesis(const float2* __restrict__ c, long long n, unsigned long long key, long long h,
                                           double& a, double& b) {
    const unsigned long long base = kSeed ^ (key << 32);
    const long long i = (long long)(splitmix64(base ^ (unsigned long long)(2 * h)) % (unsigned long long)n);
    long long j = (long long)(splitmix64(base ^ (unsigned long long)(2 * h + 1)) % (unsigned long long)(n - 1));
    j += (j >= i);
    const double xi = c[i].x, yi = c[i].y, xj = c[j].x, yj = c[j].y;
    if (xi == xj) return false;
    a = __ddiv_rn(__dsub_rn(yj, yi), __dsub_rn(xj, xi));
    b = __dsub_rn(yi, __dmul_rn(a, xi));
    return true;
}

constexpr int kRansacThreads = 256;
constexpr int kHypPerThread = 4;
constexpr int kTile = 2048;   // candidates per shared-memory tile (double2: 32 KB)

struct RansacBucket {
    long long off, n;
    unsigned long long key;
};

__global__ void __launch_bounds__(kRansacThreads) k_ransac(const float2* __restrict__ vals, const RansacBucket* __restrict__ buckets,
                                                           int iterations, double eps, double* __restrict__ out_a,
                                                           double* __restrict__ out_b, int* __restrict__ out_cnt) {
    __shared__ double2 s_c[kTile];
    __shared__ unsigned long long s_best[kRansacThreads / 32];
    const RansacBucket B = buckets[blockIdx.x];
    const float2* c = vals + B.off;
    unsigned long long best = 0;   // (count + 1) << 32 | ~h : most inliers, then the lower h
    for (long long h0 = 0; h0 < iterations; h0 += (long long)kRansacThreads * kHypPerThread) {
        double a[kHypPerThread] = {}, b[kHypPerThread] = {};
        int cnt[kHypPerThread];
        bool ok[kHypPerThread];
        for (int k = 0; k < kHypPerThread; ++k) {
            const long long h = h0 + (long long)k * kRansacThreads + threadIdx.x;
            ok[k] = h < iterations && hypothesis(c, B.n, B.key, h, a[k], b[k]);
            cnt[k] = 0;
        }
        for (long long t0 = 0; t0 < B.n; t0 += kTile) {
            const int m = (int)min((long long)kTile, B.n - t0);
            __syncthreads();
            for (int i = threadIdx.x; i < m; i += kRansacThreads) {
                const float2 v = c[t0 + i];
                s_c[i] = make_double2((double)v.x, (double)v.y);
            }
            __syncthreads();
#pragma unroll 4
            for (int i = 0; i < m; ++i) {
                const double2 v = s_c[i];
#pragma unroll
                for (int k = 0; k < kHypPerThread; ++k) {
                    const double r = __dsub_rn(__dadd_rn(__dmul_rn(a[k], v.x), b[k]), v.y);
                    cnt[k] += fabs(r) < eps;
                }
            }
        }
        for (int k = 0; k < kHypPerThread; ++k) {
            if (!ok[k]) continue;
            const long long h = h0 + (long long)k * kRansacThreads + threadIdx.x;
            const unsigned long long p = ((unsigned long long)(cnt[k] + 1) << 32) | (0xffffffffULL - (unsigned long long)h);
            if (p > best) best = p;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long q = __shfl_xor_sync(0xffffffffu, best, o);
        if (q > best) best = q;
    }
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kRansacThreads / 32; ++w)
            if (s_best[w] > best) best = s_best[w];
        s_best[0] = best;
        if (best == 0) {   // every hypothesis was skipped
            out_a[blockIdx.x] = nan("");
            out_b[blockIdx.x] = nan("");
            out_cnt[blockIdx.x] = 0;
        } else {
            const long long h = (long long)(0xffffffffULL - (best & 0xffffffffULL));
            double a, b;
            hypothesis(c, B.n, B.key, h, a, b);
            out_a[blockIdx.x] = a;
            out_b[blockIdx.x] = b;
            out_cnt[blockIdx.x] = (int)(best >> 32) - 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------ application
struct ApplyArgs {
    int wdims[3];         // resident (window) volume
    float woff[3];        // window_min (level pixels)
    float m[12];          // level pixel -> full-resolution pixel
    float sc[3];          // n / full_dims
    int n[3];
    const float* ca;      // cell values, x-fastest
    const float* cb;
    float* out;
};

__device__ __forceinline__ float lerp_rn(float a0, float a1, float t) { return __fadd_rn(a0, __fmul_rn(t, __fsub_rn(a1, a0))); }

// one thread per voxel: x from the thread index, y and z from the grid (no 64-bit division per voxel)
template <typename T>
__global__ void __launch_bounds__(256) k_apply(const T* __restrict__ src, ApplyArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, z = blockIdx.z;
    if (x >= a.wdims[0]) return;
    const size_t i = ((size_t)z * a.wdims[1] + y) * a.wdims[0] + x;
    {
        const float l[3] = {__fadd_rn(a.woff[0], (float)x), __fadd_rn(a.woff[1], (float)y), __fadd_rn(a.woff[2], (float)z)};
        int i0[3], i1[3];
        float t[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float q = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a.m[4 * r], l[0]), __fmul_rn(a.m[4 * r + 1], l[1])),
                                                __fmul_rn(a.m[4 * r + 2], l[2])), a.m[4 * r + 3]);
            float u = __fsub_rn(__fmul_rn(__fadd_rn(q, 0.5f), a.sc[r]), 0.5f);
            u = fminf(fmaxf(u, 0.f), (float)(a.n[r] - 1));
            const float f = floorf(u);
            i0[r] = (int)f;
            i1[r] = min(i0[r] + 1, a.n[r] - 1);
            t[r] = __fsub_rn(u, f);
        }
        const int r00 = (i0[2] * a.n[1] + i0[1]) * a.n[0], r01 = (i0[2] * a.n[1] + i1[1]) * a.n[0];
        const int r10 = (i1[2] * a.n[1] + i0[1]) * a.n[0], r11 = (i1[2] * a.n[1] + i1[1]) * a.n[0];
        float cf[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float* g = k ? a.cb : a.ca;
            const float c00 = lerp_rn(__ldg(g + r00 + i0[0]), __ldg(g + r00 + i1[0]), t[0]);
            const float c01 = lerp_rn(__ldg(g + r01 + i0[0]), __ldg(g + r01 + i1[0]), t[0]);
            const float c10 = lerp_rn(__ldg(g + r10 + i0[0]), __ldg(g + r10 + i1[0]), t[0]);
            const float c11 = lerp_rn(__ldg(g + r11 + i0[0]), __ldg(g + r11 + i1[0]), t[0]);
            cf[k] = lerp_rn(lerp_rn(c00, c01, t[1]), lerp_rn(c10, c11, t[1]), t[2]);
        }
        const float v = (float)__ldg(src + i);
        __stcs(a.out + i, __fadd_rn(__fmul_rn(cf[0], v), cf[1]));
    }
}

// ------------------------------------------------------------------------------------------------ resident candidates
struct Cands {
    float2* vals = nullptr;     // device, grouped by bucket
    long long n_values = 0;
    std::vector<long long> keys, off, cnt;   // per bucket, ascending key
};

struct IntensityWs {
    std::map<unsigned long long, Cands> cands;
    unsigned long long next = 1;
};

IntensityWs* ws_of(bs_ctx* ctx) {
    if (!ctx->intensity) ctx->intensity = new IntensityWs();
    return static_cast<IntensityWs*>(ctx->intensity);
}

int fill_view(bs_ctx* ctx, const bs_intensity_view* v, IView& d, const char* which) {
    auto it = ctx->vols.find(v->vol_handle);
    if (it == ctx->vols.end())
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_pair_candidates: view %s has unknown vol_handle %llu", which, v->vol_handle);
    { int rc = bs_volume_acquire(ctx, it->second); if (rc) return rc; }
    const bs_volume& vol = it->second;
    d.data = vol.dev;
    d.dtype = vol.dtype;
    for (int k = 0; k < 3; ++k) {
        d.ldims[k] = (int)vol.dims[k];
        d.fdims[k] = (double)v->full_dims[k];
        d.n[k] = v->n_cells[k];
        if (v->full_dims[k] < 1 || v->n_cells[k] < 1)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_pair_candidates: view %s needs full_dims and n_cells >= 1", which);
    }
    memcpy(d.w2p, v->world_to_px, sizeof(d.w2p));
    memcpy(d.p2l, v->px_to_level, sizeof(d.p2l));
    return BS_OK;
}

// device scratch of one candidates call, freed on every exit
struct Scratch {
    std::vector<void*> p;
    ~Scratch() {
        for (void* q : p) cudaFree(q);
    }
    template <typename T>
    cudaError_t alloc(T** out, size_t bytes) {
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, bytes ? bytes : 1);
        if (e == cudaSuccess) p.push_back(q);
        *out = static_cast<T*>(q);
        return e;
    }
};

int grid_for(bs_ctx* ctx, long long n, int threads) {
    return (int)std::max(1LL, std::min((n + threads - 1) / threads, (long long)ctx->sm_count * 16));
}

}  // namespace

void bs_intensity_free(bs_ctx* ctx) {
    if (!ctx->intensity) return;
    IntensityWs* W = static_cast<IntensityWs*>(ctx->intensity);
    for (auto& kv : W->cands) cudaFree(kv.second.vals);
    delete W;
    ctx->intensity = nullptr;
}

extern "C" int bs_intensity_pair_candidates(bs_ctx* ctx, const bs_intensity_view* view_a, const bs_intensity_view* view_b,
                                            const bs_intensity_params* params, unsigned long long* handle,
                                            long long* n_buckets, long long* n_values) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!view_a || !view_b || !params || !handle)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_pair_candidates: NULL argument");
    if (!(params->render_scale > 0.0) || params->chunk_points < 0)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_pair_candidates: render_scale must be > 0, chunk_points >= 0");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    RenderArgs a;
    memset(&a, 0, sizeof(a));
    { int rc = fill_view(ctx, view_a, a.A, "A"); if (rc) return rc; }
    { int rc = fill_view(ctx, view_b, a.B, "B"); if (rc) return rc; }
    const long long na = (long long)a.A.n[0] * a.A.n[1] * a.A.n[2], nb = (long long)a.B.n[0] * a.B.n[1] * a.B.n[2];
    if (na * nb > kMaxKeys)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_pair_candidates: %lld x %lld cell pairs exceed %lld", na, nb, kMaxKeys);
    a.nb_cells = (int)nb;
    a.tmin = params->min_threshold;
    a.tmax = params->max_threshold;
    long long ext[3];
    for (int k = 0; k < 3; ++k) ext[k] = params->render_max[k] - params->render_min[k] + 1;
    Cands C;
    IntensityWs* W = ws_of(ctx);
    if (ext[0] > 0 && ext[1] > 0 && ext[2] > 0) {
        Scratch S;
        // world coordinates r / s (IEEE division, as __ddiv_rn), one table per axis
        std::vector<double> hw((size_t)(ext[0] + ext[1] + ext[2]));
        for (int k = 0, o = 0; k < 3; o += (int)ext[k], ++k)
            for (long long r = 0; r < ext[k]; ++r) hw[o + r] = (double)(params->render_min[k] + r) / params->render_scale;
        double* dw;
        BS_CUDA(ctx, S.alloc(&dw, sizeof(double) * hw.size()));
        BS_CUDA(ctx, cudaMemcpyAsync(dw, hw.data(), sizeof(double) * hw.size(), cudaMemcpyHostToDevice, ctx->stream));
        a.w[0] = dw;
        a.w[1] = dw + ext[0];
        a.w[2] = dw + ext[0] + ext[1];
        a.nx = ext[0];
        a.ny = ext[1];
        const long long plane = ext[0] * ext[1];
        const long long chunk = params->chunk_points > 0 ? params->chunk_points : kDefaultChunk;
        const long long zc = std::max(1LL, chunk / plane);                 // planes per chunk
        const long long nkeys = na * nb;
        unsigned int* counts;
        int *slot_of_key, *keys;
        long long *skey, *soff, *scnt;
        float2* vals;
        CompactOut* co;
        BS_CUDA(ctx, S.alloc(&counts, sizeof(unsigned) * nkeys));
        BS_CUDA(ctx, S.alloc(&slot_of_key, sizeof(int) * nkeys));
        BS_CUDA(ctx, S.alloc(&co, sizeof(CompactOut)));
        BS_CUDA(ctx, cudaMemsetAsync(counts, 0, sizeof(unsigned) * nkeys, ctx->stream));
        // ---- pass A: counts per key
        for (long long z = 0; z < ext[2]; z += zc) {
            a.z0 = z;
            a.npts = std::min(zc, ext[2] - z) * plane;
            bs_launch_scope sc(ctx, "intensity_render");
            k_render<true><<<grid_for(ctx, a.npts, 256), 256, 0, ctx->stream>>>(a, counts, nullptr, nullptr);
        }
        BS_CUDA(ctx, cudaGetLastError());
        // slot arrays are sized by an upper bound first (the number of present keys is known after k_compact)
        const long long slot_cap = std::min(nkeys, ext[0] * ext[1] * ext[2]);
        BS_CUDA(ctx, S.alloc(&skey, sizeof(long long) * slot_cap));
        BS_CUDA(ctx, S.alloc(&soff, sizeof(long long) * slot_cap));
        BS_CUDA(ctx, S.alloc(&scnt, sizeof(long long) * slot_cap));
        {
            bs_launch_scope sc(ctx, "intensity_render");
            k_compact<<<1, 1024, 0, ctx->stream>>>(counts, nkeys, slot_of_key, skey, soff, scnt, co);
        }
        BS_CUDA(ctx, cudaGetLastError());
        CompactOut h;
        BS_CUDA(ctx, cudaMemcpyAsync(&h, co, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        const int ns = (int)h.n_slots;
        C.n_values = h.n_values;
        if (ns > 0) {
            C.keys.resize(ns);
            C.off.resize(ns);
            C.cnt.resize(ns);
            BS_CUDA(ctx, cudaMemcpy(C.keys.data(), skey, sizeof(long long) * ns, cudaMemcpyDeviceToHost));
            BS_CUDA(ctx, cudaMemcpy(C.off.data(), soff, sizeof(long long) * ns, cudaMemcpyDeviceToHost));
            BS_CUDA(ctx, cudaMemcpy(C.cnt.data(), scnt, sizeof(long long) * ns, cudaMemcpyDeviceToHost));
            const size_t smem_cur = sizeof(long long) * (size_t)ns;
            int max_smem = 0;
            BS_CUDA(ctx, cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
            if (smem_cur > (size_t)max_smem)
                return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "bs_intensity_pair_candidates: %d buckets exceed one CTA's shared memory", ns);
            BS_CUDA(ctx, cudaFuncSetAttribute(k_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cur));
            BS_CUDA(ctx, cudaFuncSetAttribute(k_seg_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned) * ns)));
            // pass B may chunk more finely than pass A (the output does not depend on the chunking): the per-(segment,
            // slot) cursors stay below 2^25 entries
            const long long zb = std::max(1LL, std::min(zc, ((1LL << 25) / ns) * kSeg / plane));
            const long long cpts = std::min(zb, ext[2]) * plane;
            const long long nseg_cap = (cpts + kSeg - 1) / kSeg;
            unsigned int* hist;
            long long *cursor, *seg_base;
            BS_CUDA(ctx, S.alloc(&keys, sizeof(int) * cpts));
            BS_CUDA(ctx, S.alloc(&vals, sizeof(float2) * cpts));
            BS_CUDA(ctx, S.alloc(&hist, sizeof(unsigned) * nseg_cap * ns));
            BS_CUDA(ctx, S.alloc(&seg_base, sizeof(long long) * nseg_cap * ns));
            BS_CUDA(ctx, S.alloc(&cursor, sizeof(long long) * ns));
            BS_CUDA(ctx, cudaMemcpyAsync(cursor, soff, sizeof(long long) * ns, cudaMemcpyDeviceToDevice, ctx->stream));
            BS_CUDA(ctx, cudaMalloc(&C.vals, sizeof(float2) * C.n_values));
            // ---- pass B: order-preserving scatter, chunk by chunk
            for (long long z = 0; z < ext[2]; z += zb) {
                a.z0 = z;
                a.npts = std::min(zb, ext[2] - z) * plane;
                const long long nseg = (a.npts + kSeg - 1) / kSeg;
                bs_launch_scope sc(ctx, "intensity_render");
                k_render<false><<<grid_for(ctx, a.npts, 256), 256, 0, ctx->stream>>>(a, nullptr, keys, vals);
                k_seg_count<<<(unsigned)nseg, 32, sizeof(unsigned) * ns, ctx->stream>>>(keys, a.npts, slot_of_key, ns, hist);
                k_seg_scan<<<(ns + 255) / 256, 256, 0, ctx->stream>>>(hist, nseg, ns, cursor, seg_base);
                k_scatter<<<(unsigned)nseg, 32, smem_cur, ctx->stream>>>(keys, vals, a.npts, slot_of_key, ns, seg_base, C.vals);
            }
            cudaError_t e = cudaGetLastError();
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            if (e != cudaSuccess) {
                cudaFree(C.vals);
                return bs_set_error(ctx, BS_ERR_CUDA, "bs_intensity_pair_candidates: %s", cudaGetErrorString(e));
            }
        }
    }
    *handle = W->next++;
    if (n_buckets) *n_buckets = (long long)C.keys.size();
    if (n_values) *n_values = C.n_values;
    W->cands[*handle] = std::move(C);
    return BS_OK;
}

extern "C" int bs_intensity_candidates_get(bs_ctx* ctx, unsigned long long handle, long long* keys, long long* offsets,
                                           long long* counts, float* values) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    IntensityWs* W = ws_of(ctx);
    auto it = W->cands.find(handle);
    if (it == W->cands.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_candidates_get: unknown handle %llu", handle);
    const Cands& C = it->second;
    const size_t nb = C.keys.size();
    if (keys && nb) memcpy(keys, C.keys.data(), sizeof(long long) * nb);
    if (offsets && nb) memcpy(offsets, C.off.data(), sizeof(long long) * nb);
    if (counts && nb) memcpy(counts, C.cnt.data(), sizeof(long long) * nb);
    if (values && C.n_values) {
        BS_CUDA(ctx, cudaSetDevice(ctx->device));
        BS_CUDA(ctx, cudaMemcpyAsync(values, C.vals, sizeof(float2) * C.n_values, cudaMemcpyDeviceToHost, ctx->stream));
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return BS_OK;
}

extern "C" int bs_intensity_candidates_free(bs_ctx* ctx, unsigned long long handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    IntensityWs* W = ws_of(ctx);
    auto it = W->cands.find(handle);
    if (it == W->cands.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_candidates_free: unknown handle %llu", handle);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(it->second.vals);
    W->cands.erase(it);
    return BS_OK;
}

extern "C" int bs_intensity_ransac(bs_ctx* ctx, unsigned long long handle, long long min_num_candidates, int num_iterations,
                                   double max_epsilon, double* a_out, double* b_out, int* count_out) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    IntensityWs* W = ws_of(ctx);
    auto it = W->cands.find(handle);
    if (it == W->cands.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_ransac: unknown handle %llu", handle);
    if (num_iterations < 1 || !(max_epsilon >= 0.0))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_ransac: num_iterations must be >= 1 and max_epsilon >= 0");
    const Cands& C = it->second;
    const int nb = (int)C.keys.size();
    if (nb && (!a_out || !b_out || !count_out)) return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_ransac: NULL output");
    std::vector<RansacBucket> hb;
    std::vector<int> idx;
    for (int i = 0; i < nb; ++i) {
        a_out[i] = b_out[i] = nan("");
        count_out[i] = -1;
        if (C.cnt[i] >= std::max(2LL, min_num_candidates)) {
            hb.push_back({C.off[i], C.cnt[i], (unsigned long long)C.keys[i]});
            idx.push_back(i);
        }
    }
    if (hb.empty()) return BS_OK;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t ne = hb.size();
    Scratch S;
    RansacBucket* db;
    double *da, *dbb;
    int* dc;
    BS_CUDA(ctx, S.alloc(&db, sizeof(RansacBucket) * ne));
    BS_CUDA(ctx, S.alloc(&da, sizeof(double) * ne));
    BS_CUDA(ctx, S.alloc(&dbb, sizeof(double) * ne));
    BS_CUDA(ctx, S.alloc(&dc, sizeof(int) * ne));
    BS_CUDA(ctx, cudaMemcpyAsync(db, hb.data(), sizeof(RansacBucket) * ne, cudaMemcpyHostToDevice, ctx->stream));
    {
        bs_launch_scope sc(ctx, "intensity_ransac");
        k_ransac<<<(unsigned)ne, kRansacThreads, 0, ctx->stream>>>(C.vals, db, num_iterations, max_epsilon, da, dbb, dc);
    }
    BS_CUDA(ctx, cudaGetLastError());
    std::vector<double> ha(ne), hbv(ne);
    std::vector<int> hc(ne);
    BS_CUDA(ctx, cudaMemcpyAsync(ha.data(), da, sizeof(double) * ne, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(hbv.data(), dbb, sizeof(double) * ne, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(hc.data(), dc, sizeof(int) * ne, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (size_t k = 0; k < ne; ++k) {
        a_out[idx[k]] = ha[k];
        b_out[idx[k]] = hbv[k];
        count_out[idx[k]] = hc[k];
    }
    return BS_OK;
}

extern "C" int bs_intensity_apply(bs_ctx* ctx, unsigned long long vol_handle, const long long full_dims[3],
                                  const long long window_min[3], const double level_to_full[12], const int n_cells[3],
                                  const double* coeff_a, const double* coeff_b, unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!full_dims || !level_to_full || !n_cells || !coeff_a || !coeff_b || !out_handle)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_apply: NULL argument");
    auto it = ctx->vols.find(vol_handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_apply: unknown handle %llu", vol_handle);
    { int rc = bs_volume_acquire(ctx, it->second); if (rc) return rc; }
    const bs_volume src = it->second;
    ApplyArgs a;
    long long ncell = 1;
    if (src.dims[1] > 65535 || src.dims[2] > 65535)
        return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "bs_intensity_apply: y and z sizes above 65535");
    for (int k = 0; k < 3; ++k) {
        if (n_cells[k] < 1 || full_dims[k] < 1)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_intensity_apply: n_cells and full_dims must be >= 1");
        a.wdims[k] = (int)src.dims[k];
        a.woff[k] = window_min ? (float)window_min[k] : 0.f;
        a.n[k] = n_cells[k];
        a.sc[k] = (float)((double)n_cells[k] / (double)full_dims[k]);
        ncell *= n_cells[k];
    }
    for (int k = 0; k < 12; ++k) a.m[k] = (float)level_to_full[k];
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<float> hc((size_t)(2 * ncell));
    for (long long i = 0; i < ncell; ++i) {
        hc[i] = (float)coeff_a[i];
        hc[ncell + i] = (float)coeff_b[i];
    }
    const long long nvox = src.dims[0] * src.dims[1] * src.dims[2];
    bs_volume v;
    for (int k = 0; k < 3; ++k) v.dims[k] = src.dims[k];
    v.dtype = BS_DTYPE_F32;
    v.owned = true;
    float* dcoef = nullptr;
    BS_CUDA(ctx, cudaMalloc(&v.dev, sizeof(float) * (size_t)nvox));
    cudaError_t e = cudaMalloc(&dcoef, sizeof(float) * hc.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(dcoef, hc.data(), sizeof(float) * hc.size(), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        a.ca = dcoef;
        a.cb = dcoef + ncell;
        a.out = static_cast<float*>(v.dev);
        const dim3 grid((unsigned)((src.dims[0] + 255) / 256), (unsigned)src.dims[1], (unsigned)src.dims[2]);
        bs_launch_scope sc(ctx, "intensity_apply");
        if (src.dtype == BS_DTYPE_U16) k_apply<unsigned short><<<grid, 256, 0, ctx->stream>>>((const unsigned short*)src.dev, a);
        else if (src.dtype == BS_DTYPE_F32) k_apply<float><<<grid, 256, 0, ctx->stream>>>((const float*)src.dev, a);
        else k_apply<unsigned char><<<grid, 256, 0, ctx->stream>>>((const unsigned char*)src.dev, a);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (dcoef) cudaFree(dcoef);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_intensity_apply: %s", cudaGetErrorString(e));
    }
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}
