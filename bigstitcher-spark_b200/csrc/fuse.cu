// Hot path 2: fused affine-warp + n-linear sample + blend/content weight + accumulate
// (+ dtype convert) for one output block.  Replaces BlkAffineFusion.init... +
// BlockAlgoUtils.arrayImg at J/SparkAffineFusion.java:602-627.
//
// Layout: every source volume is a dense x-fastest array resident in HBM (uint16 / float32 /
// uint8); the output block is dense x-fastest.  One CTA renders a 32 x 8 x FUSE_ZT tile: a
// warp spans 32 consecutive x so that, for the (typical) near-axis-aligned registrations,
// the 8 taps of a warp fall into a handful of 64-128 B source segments served by L1/L2.
// Views are culled per CTA (tile corners -> source AABB) so only overlapping views are
// evaluated; per view the thread keeps the inverse affine in registers and walks z.
#include <cmath>
#include <cstring>

#include "bs_internal.cuh"
#include "fuse_common.cuh"

#define FUSE_TX 32
#define FUSE_TY 8
#define FUSE_ZT 8
#define FUSE_CHUNK 32

struct FuseViewDev {
    double inv[12];        // world -> source pixel
    const void* data;
    const float* content;
    int dims[3];
    int dtype;
    float border[3];
    float range[3];
};

struct FuseArgs {
    long long bmin[3];
    int size[3];
    int fusion_type;
    int lut_n;
    const float* lut;      // device, lut_n + 2 entries
    double cmin, cscale;   // integer output conversion: (v - cmin) * cscale
    double ctop;
    void* out;
    float* acc_wi;         // accumulate mode
    float* acc_w;
    int no_stage;          // debug: force the global-gather path (env BS_FUSE_NO_STAGE)
    const struct TilePlan* plan;   // per-tile view lists from fuse_plan_kernel (or nullptr)
};

// ---- staged footprint: a fixed FS_X x FS_Y x FS_Z float box per (CTA tile, view) in shared memory
#define FS_X 40
#define FS_Y 12
#define FS_Z 12
#define FS_N (FS_X * FS_Y * FS_Z)   // 5760 floats = 22.5 KB
extern __shared__ float fuse_dyn_smem[];  // second stage buffer (content weights), sized at launch

// Per (CTA tile, active view) constants, computed once in double by one thread and kept in
// shared memory: everything the per-voxel loop needs is float and tile-relative.
struct ViewTile {
    float m[9];        // linear part of world->source
    float o[3];        // source coordinate of the tile origin, relative to the box origin b0
    int b0[3];         // box origin in source pixels (staged: clamped so the box stays inside the volume)
    int dims[3];
    float border[3];
    float inv_range[3];
    float range[3];
    const void* data;
    const float* content;
    int dtype;
    int staged;
    int interior;      // every upper tap of the tile exists (no clamping at the volume's far faces)
    int plateau;       // every voxel of the tile is >= blend range away from all faces: weight == 1
    int vec4;          // staged rows can be read as aligned 8-byte ushort4 vectors
};

template <typename T>
__device__ __forceinline__ void stage_fixed(float* __restrict__ st, const T* __restrict__ d, const ViewTile& t,
                                            int tid) {
    // FS_N elements, constant index math, every load independent of the others
    const int dx = t.dims[0], dy = t.dims[1], dz = t.dims[2];
#pragma unroll 6
    for (int i = tid; i < FS_N; i += FUSE_TX * FUSE_TY) {
        const int xx = i % FS_X, r = i / FS_X;
        const int yy = r % FS_Y, zz = r / FS_Y;
        const int gx = min(t.b0[0] + xx, dx - 1), gy = min(t.b0[1] + yy, dy - 1), gz = min(t.b0[2] + zz, dz - 1);
        st[i] = (float)__ldg(d + ((size_t)gz * dy + gy) * dx + gx);
    }
}

// uint16 fast path: box origin and row pitch are multiples of 4 voxels and the box lies inside the
// volume along x -> 10 aligned 8-byte loads per row, 1440 per box (5.6 per thread, all independent)
__device__ __forceinline__ void stage_fixed_u16x4(float* __restrict__ st, const unsigned short* __restrict__ d,
                                                  const ViewTile& t, int tid) {
    const int dx = t.dims[0], dy = t.dims[1], dz = t.dims[2];
    constexpr int VPR = FS_X / 4;
#pragma unroll 6
    for (int i = tid; i < FS_N / 4; i += FUSE_TX * FUSE_TY) {
        const int xv = i % VPR, r = i / VPR;
        const int yy = r % FS_Y, zz = r / FS_Y;
        const int gy = min(t.b0[1] + yy, dy - 1), gz = min(t.b0[2] + zz, dz - 1);
        const uint2 q = __ldg(reinterpret_cast<const uint2*>(d + ((size_t)gz * dy + gy) * dx + t.b0[0]) + xv);
        float4 f;
        f.x = (float)(q.x & 0xffffu); f.y = (float)(q.x >> 16);
        f.z = (float)(q.y & 0xffffu); f.w = (float)(q.y >> 16);
        reinterpret_cast<float4*>(st)[i] = f;
    }
}

__device__ __forceinline__ void stage_fixed_any(float* st, const void* d, int dtype, const ViewTile& t, int tid) {
    if (dtype == BS_DTYPE_U16) {
        if (t.vec4) stage_fixed_u16x4(st, (const unsigned short*)d, t, tid);
        else stage_fixed(st, (const unsigned short*)d, t, tid);
    } else if (dtype == BS_DTYPE_F32) stage_fixed(st, (const float*)d, t, tid);
    else stage_fixed(st, (const unsigned char*)d, t, tid);
}

// n-linear sample from the staged box at box-relative coordinates (rx, ry, rz)
template <bool INTERIOR>
__device__ __forceinline__ float sample_staged(const float* __restrict__ st, const ViewTile& t, float rx, float ry,
                                               float rz) {
    const float fx = floorf(rx), fy = floorf(ry), fz = floorf(rz);
    const float tx = rx - fx, ty = ry - fy, tz = rz - fz;
    const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
    const float* p = st + (z0 * FS_Y + y0) * FS_X + x0;
    float a000, a001, a010, a011, a100, a101, a110, a111;
    if (INTERIOR) {  // immediate offsets
        a000 = p[0]; a001 = p[1]; a010 = p[FS_X]; a011 = p[FS_X + 1];
        a100 = p[FS_X * FS_Y]; a101 = p[FS_X * FS_Y + 1]; a110 = p[FS_X * FS_Y + FS_X]; a111 = p[FS_X * FS_Y + FS_X + 1];
    } else {
        const int ox = (t.b0[0] + x0 + 1 < t.dims[0]) ? 1 : 0;
        const int oy = (t.b0[1] + y0 + 1 < t.dims[1]) ? FS_X : 0;
        const int oz = (t.b0[2] + z0 + 1 < t.dims[2]) ? FS_X * FS_Y : 0;
        a000 = p[0]; a001 = p[ox]; a010 = p[oy]; a011 = p[oy + ox];
        a100 = p[oz]; a101 = p[oz + ox]; a110 = p[oz + oy]; a111 = p[oz + oy + ox];
    }
    const float c00 = a000 + tx * (a001 - a000);
    const float c01 = a010 + tx * (a011 - a010);
    const float c10 = a100 + tx * (a101 - a100);
    const float c11 = a110 + tx * (a111 - a110);
    const float c0 = c00 + ty * (c01 - c00);
    const float c1 = c10 + ty * (c11 - c10);
    return c0 + tz * (c1 - c0);
}

// Cull one view against one output tile and derive its tile constants (double precision once per
// (tile, view); the per-voxel loop is float and tile-relative).  Returns false when the view's
// source AABB of the tile misses [0, dim-1] (+-1e-3).
__device__ __forceinline__ bool make_view_tile(const FuseViewDev& v, double cx0, double cy0, double cz0, double ex,
                                               double ey, double ez, bool allow_stage, ViewTile& t) {
    bool hit = true, fits = allow_stage, interior = true, plateau = true;
    const double c0[3] = {cx0, cy0, cz0};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double m0 = v.inv[4 * r], m1 = v.inv[4 * r + 1], m2 = v.inv[4 * r + 2];
        const double org = fma(m0, c0[0], fma(m1, c0[1], fma(m2, c0[2], v.inv[4 * r + 3])));
        const double lo = org + fmin(0.0, m0 * ex) + fmin(0.0, m1 * ey) + fmin(0.0, m2 * ez);
        const double hi = org + fmax(0.0, m0 * ex) + fmax(0.0, m1 * ey) + fmax(0.0, m2 * ez);
        const int dim = v.dims[r];
        if (hi < -1e-3 || lo > (double)(dim - 1) + 1e-3) hit = false;
        // taps floor(s) .. floor(s)+1 of every in-range s; eps covers float rounding of s
        const double eps = 2e-3 + 2e-7 * fmax(fabs(lo), fabs(hi));
        const int f0 = max((int)floor(fmax(lo - eps, 0.0)), 0);
        const int f1 = min((int)floor(fmin(hi + eps, (double)(dim - 1))) + 1, dim - 1);
        const int cap = r == 0 ? FS_X : (r == 1 ? FS_Y : FS_Z);
        int g0 = f0;
        if (r == 0) g0 &= ~3;                      // 4-voxel aligned box origin along x (vector staging)
        if (f1 - g0 + 1 > cap - 1) fits = false;   // one spare row/column: a tap at weight 0 may touch f1 + 1
        if (f1 + 1 > dim - 1) interior = false;
        if (!(lo - eps - (double)v.border[r] >= (double)v.range[r] &&
              (double)(dim - 1) - (hi + eps) - (double)v.border[r] >= (double)v.range[r])) plateau = false;
        t.b0[r] = g0;
        t.o[r] = (float)(org - (double)g0);
        t.m[3 * r] = (float)m0; t.m[3 * r + 1] = (float)m1; t.m[3 * r + 2] = (float)m2;
        t.dims[r] = dim;
        t.border[r] = v.border[r];
        t.range[r] = v.range[r];
        t.inv_range[r] = 1.0f / v.range[r];
    }
    t.data = v.data;
    t.content = v.content;
    t.dtype = v.dtype;
    t.staged = fits ? 1 : 0;
    t.interior = interior ? 1 : 0;
    t.plateau = plateau ? 1 : 0;
    t.vec4 = (v.dtype == BS_DTYPE_U16 && (v.dims[0] & 3) == 0 && ((size_t)v.data & 7) == 0 &&
              t.b0[0] + FS_X <= v.dims[0]) ? 1 : 0;
    return hit;
}

// Plan pre-pass: one thread per output tile walks the (ViewId-sorted) view list and writes the
// tile's active views with their constants.  It takes the culling / double-precision set-up out of
// the fusion kernel's critical path (there it was a serial prologue of five barriers per CTA).
#define FUSE_PLAN_MAXV 8
struct TilePlan {
    int count;
    int overflow;        // more than FUSE_PLAN_MAXV active views: the fusion kernel culls this tile itself
    ViewTile v[FUSE_PLAN_MAXV];
};

__global__ void fuse_plan_kernel(const FuseViewDev* __restrict__ views, int nviews, FuseArgs a, TilePlan* plan,
                                 int gx, int gy, int gz, int linear) {
    const int tile = blockIdx.x * blockDim.x + threadIdx.x;
    if (tile >= gx * gy * gz) return;
    const int bx = tile % gx, by = (tile / gx) % gy, bz = tile / (gx * gy);
    const int z0 = bz * FUSE_ZT;
    const double cx0 = (double)(a.bmin[0] + (long long)bx * FUSE_TX);
    const double cy0 = (double)(a.bmin[1] + (long long)by * FUSE_TY);
    const double cz0 = (double)(a.bmin[2] + z0);
    const double ex = (double)(min(FUSE_TX, a.size[0] - bx * FUSE_TX) - 1);
    const double ey = (double)(min(FUSE_TY, a.size[1] - by * FUSE_TY) - 1);
    const double ez = (double)(min(FUSE_ZT, a.size[2] - z0) - 1);
    TilePlan& p = plan[tile];
    int count = 0, overflow = 0;
    for (int vi = 0; vi < nviews; ++vi) {
        ViewTile t;
        if (!make_view_tile(views[vi], cx0, cy0, cz0, ex, ey, ez, linear && a.no_stage == 0, t)) continue;
        if (count < FUSE_PLAN_MAXV) p.v[count++] = t;
        else overflow = 1;
    }
    p.count = count;
    p.overflow = overflow;
}

template <int OUT>
__device__ __forceinline__ void store_voxel(const FuseArgs& a, size_t o, float res) {
    bs_store_converted<OUT>(a.out, o, res, a.cmin, a.cscale, a.ctop);
}

// KIND 0: weighted average family (AVG, AVG_BLEND, *_CONTENT); KIND 1: winner family.
// ACCUM: add partial sums into acc_wi/acc_w instead of producing the final voxel.
//
// Per CTA tile (32 x 8 x FUSE_ZT output voxels) and per overlapping view, one thread derives
// the tile-relative float transform in double; the source footprint of the tile (40 x 12 x 12
// box starting at the footprint's lower corner) is copied once into shared memory as float
// with independent, row-coalesced loads, and the 8 taps of every voxel then come from shared
// memory.  Footprints that do not fit the box (down-scaling, strong rotation) and nearest-
// neighbour sampling gather from global memory through L1/L2 instead.
template <int KIND, bool LINEAR, int OUT, bool ACCUM>
__global__ void __launch_bounds__(FUSE_TX* FUSE_TY, 4)
fuse_kernel(const FuseViewDev* __restrict__ views, int nviews, FuseArgs a) {
    __shared__ int s_active[FUSE_CHUNK];
    __shared__ ViewTile s_vt[FUSE_CHUNK];
    __shared__ int s_nactive;
    __shared__ float s_lut[FUSE_MAX_LUT + 2];
    __shared__ __align__(16) float s_stage[FS_N];
    float* s_stage_c = fuse_dyn_smem;

    const int tid = threadIdx.y * FUSE_TX + threadIdx.x;
    constexpr int NT = FUSE_TX * FUSE_TY;
    const int x = blockIdx.x * FUSE_TX + threadIdx.x;
    const int y = blockIdx.y * FUSE_TY + threadIdx.y;
    const int z0 = blockIdx.z * FUSE_ZT;
    const bool valid = x < a.size[0] && y < a.size[1];
    const int ft = a.fusion_type;
    const bool use_blend = ft == BS_FUSE_AVG_BLEND || ft == BS_FUSE_AVG_BLEND_CONTENT || ft == BS_FUSE_CLOSEST_PIXEL_WINS;
    const bool use_content = KIND == 0 && (ft == BS_FUSE_AVG_CONTENT || ft == BS_FUSE_AVG_BLEND_CONTENT);

    if (a.lut_n > 0)
        for (int i = tid; i < a.lut_n + 2; i += NT) s_lut[i] = a.lut[i];

    // accumulators live in shared memory ([k][thread], private to the owning thread) so that the z loop
    // can stay ROLLED: the fully unrolled version was 9.4k SASS instructions and stalled on
    // instruction fetch (ncu: no_instruction was the top stall reason)
    __shared__ float s_acc0[FUSE_ZT][FUSE_TX * FUSE_TY];  // KIND0: sum w*I ; KIND1: best value
    __shared__ float s_acc1[FUSE_ZT][FUSE_TX * FUSE_TY];  // KIND0: sum w   ; KIND1: best weight / have flag
#pragma unroll
    for (int k = 0; k < FUSE_ZT; ++k) { s_acc0[k][tid] = 0.f; s_acc1[k][tid] = 0.f; }

    const float tx = (float)threadIdx.x, ty = (float)threadIdx.y;
    const int nz = min(FUSE_ZT, a.size[2] - z0);

    const TilePlan* tp = a.plan ? a.plan + ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x : nullptr;
    const bool planned = tp != nullptr && tp->overflow == 0;   // CTA-uniform
    for (int chunk = 0; chunk < (planned ? 1 : nviews); chunk += FUSE_CHUNK) {
        int nact;
        if (planned) {
            // tile constants were prepared by fuse_plan_kernel: copy them to shared memory
            __syncthreads();
            nact = tp->count;
            const int nwords = nact * (int)(sizeof(ViewTile) / 4);
            const int* src = reinterpret_cast<const int*>(tp->v);
            int* dst = reinterpret_cast<int*>(s_vt);
            for (int i = tid; i < nwords; i += NT) dst[i] = __ldg(src + i);
            __syncthreads();
            if (KIND == 0 && !ACCUM && nact <= 1) {
                // ---- fast path (the majority of tiles): zero or one view.  The weighted average of a
                // single view is the sample itself wherever its weight is positive, so the voxels are
                // written straight from the tap loop -- no accumulators, no epilogue.
                const size_t plane = (size_t)a.size[1] * a.size[0];
                size_t o = ((size_t)z0 * a.size[1] + y) * a.size[0] + x;
                if (nact == 0) {
                    if (valid)
                        for (int k = 0; k < nz; ++k, o += plane) store_voxel<OUT>(a, o, 0.f);
                    return;
                }
                const ViewTile& t = s_vt[0];
                const bool staged = t.staged != 0;
                if (staged) {
                    stage_fixed_any(s_stage, t.data, t.dtype, t, tid);
                    if (use_content) stage_fixed(s_stage_c, t.content, t, tid);
                    __syncthreads();
                }
                if (!valid) return;
                float rx = fmaf(t.m[0], tx, fmaf(t.m[1], ty, t.o[0]));
                float ry = fmaf(t.m[3], tx, fmaf(t.m[4], ty, t.o[1]));
                float rz = fmaf(t.m[6], tx, fmaf(t.m[7], ty, t.o[2]));
                const float sxk = t.m[2], syk = t.m[5], szk = t.m[8];
                const float bx = (float)t.b0[0], by = (float)t.b0[1], bz = (float)t.b0[2];
                const float dm1x = (float)(t.dims[0] - 1), dm1y = (float)(t.dims[1] - 1), dm1z = (float)(t.dims[2] - 1);
                const bool do_blend = use_blend && !t.plateau;
                const int mode = staged ? (t.interior ? 0 : 1) : 2;
#pragma unroll 1
                for (int k = 0; k < nz; ++k, rx += sxk, ry += syk, rz += szk, o += plane) {
                    const float fx = rx + bx, fy = ry + by, fz = rz + bz;
                    float res = 0.f;
                    if (fx >= 0.f && fx <= dm1x && fy >= 0.f && fy <= dm1y && fz >= 0.f && fz <= dm1z) {
                        float w = 1.f;
                        bool ok = true;
                        if (do_blend)
                            ok = blend_axis(fx, dm1x, t.border[0], t.inv_range[0], a.lut_n, s_lut, w) &&
                                 blend_axis(fy, dm1y, t.border[1], t.inv_range[1], a.lut_n, s_lut, w) &&
                                 blend_axis(fz, dm1z, t.border[2], t.inv_range[2], a.lut_n, s_lut, w);
                        if (ok && use_content) {
                            if (staged) w *= sample_staged<false>(s_stage_c, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                            else w *= sample<float, LINEAR>(t.content, t.dims[0], t.dims[1], t.dims[2], fx, fy, fz);
                        }
                        if (ok && w > 0.f) {
                            if (mode == 0) res = sample_staged<true>(s_stage, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                            else if (mode == 1) res = sample_staged<false>(s_stage, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                            else res = sample_any<LINEAR>(t.data, t.dtype, t.dims[0], t.dims[1], t.dims[2], fx, fy, fz);
                        }
                    }
                    store_voxel<OUT>(a, o, res);
                }
                return;
            }
        } else {
            __syncthreads();
            if (tid == 0) s_nactive = 0;
            __syncthreads();
            const double cx0 = (double)(a.bmin[0] + (long long)blockIdx.x * FUSE_TX);
            const double cy0 = (double)(a.bmin[1] + (long long)blockIdx.y * FUSE_TY);
            const double cz0 = (double)(a.bmin[2] + z0);
            const double ex = (double)(min(FUSE_TX, a.size[0] - (int)blockIdx.x * FUSE_TX) - 1);
            const double ey = (double)(min(FUSE_TY, a.size[1] - (int)blockIdx.y * FUSE_TY) - 1);
            const double ez = (double)(nz - 1);
            // cull: threads over the views of this chunk
            for (int vi = chunk + tid; vi < min(nviews, chunk + FUSE_CHUNK); vi += NT) {
                ViewTile t;
                if (make_view_tile(views[vi], cx0, cy0, cz0, ex, ey, ez, LINEAR && a.no_stage == 0, t))
                    s_active[atomicAdd(&s_nactive, 1)] = vi;
            }
            __syncthreads();
            nact = s_nactive;
            // deterministic view order (ascending ViewId): sort the short active list
            if (tid == 0) {
                for (int i = 1; i < nact; ++i) {
                    int key = s_active[i], j = i - 1;
                    while (j >= 0 && s_active[j] > key) { s_active[j + 1] = s_active[j]; --j; }
                    s_active[j + 1] = key;
                }
            }
            __syncthreads();
            for (int ai = tid; ai < nact; ai += NT)
                make_view_tile(views[s_active[ai]], cx0, cy0, cz0, ex, ey, ez, LINEAR && a.no_stage == 0, s_vt[ai]);
            __syncthreads();
        }

        for (int ai = 0; ai < nact; ++ai) {
            const ViewTile& t = s_vt[ai];
            const bool staged = t.staged != 0;
            if (staged) {
                __syncthreads();  // previous view's taps are done with the stage buffers
                stage_fixed_any(s_stage, t.data, t.dtype, t, tid);
                if (use_content) stage_fixed(s_stage_c, t.content, t, tid);
                __syncthreads();
            }
            if (!valid) continue;
            // box-relative source coordinate of this thread's column at k = 0, and its z step
            float rx = fmaf(t.m[0], tx, fmaf(t.m[1], ty, t.o[0]));
            float ry = fmaf(t.m[3], tx, fmaf(t.m[4], ty, t.o[1]));
            float rz = fmaf(t.m[6], tx, fmaf(t.m[7], ty, t.o[2]));
            const float sxk = t.m[2], syk = t.m[5], szk = t.m[8];
            const float bx = (float)t.b0[0], by = (float)t.b0[1], bz = (float)t.b0[2];
            const float dm1x = (float)(t.dims[0] - 1), dm1y = (float)(t.dims[1] - 1), dm1z = (float)(t.dims[2] - 1);
            const bool do_blend = use_blend && !t.plateau;
            const int mode = staged ? (t.interior ? 0 : 1) : 2;
#pragma unroll 1
            for (int k = 0; k < nz; ++k, rx += sxk, ry += syk, rz += szk) {
                const float fx = rx + bx, fy = ry + by, fz = rz + bz;  // absolute source coordinate
                if (!(fx >= 0.f && fx <= dm1x && fy >= 0.f && fy <= dm1y && fz >= 0.f && fz <= dm1z)) continue;
                float w = 1.f;
                if (do_blend) {
                    if (!blend_axis(fx, dm1x, t.border[0], t.inv_range[0], a.lut_n, s_lut, w)) continue;
                    if (!blend_axis(fy, dm1y, t.border[1], t.inv_range[1], a.lut_n, s_lut, w)) continue;
                    if (!blend_axis(fz, dm1z, t.border[2], t.inv_range[2], a.lut_n, s_lut, w)) continue;
                }
                float val;
                if (mode == 0) val = sample_staged<true>(s_stage, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                else if (mode == 1) val = sample_staged<false>(s_stage, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                else val = sample_any<LINEAR>(t.data, t.dtype, t.dims[0], t.dims[1], t.dims[2], fx, fy, fz);
                if (KIND == 0) {
                    if (use_content) {
                        if (staged) w *= sample_staged<false>(s_stage_c, t, fmaxf(rx, 0.f), fmaxf(ry, 0.f), fmaxf(rz, 0.f));
                        else w *= sample<float, LINEAR>(t.content, t.dims[0], t.dims[1], t.dims[2], fx, fy, fz);
                    }
                    s_acc0[k][tid] += w * val;
                    s_acc1[k][tid] += w;
                } else {
                    if (!(w > 0.f)) continue;
                    const float c0 = s_acc0[k][tid], c1 = s_acc1[k][tid];
                    if (ft == BS_FUSE_MAX_INTENSITY) {
                        if (c1 == 0.f || val > c0) s_acc0[k][tid] = val;
                        s_acc1[k][tid] = 1.f;
                    } else if (ft == BS_FUSE_LOWEST_VIEWID_WINS) {
                        if (c1 == 0.f) { s_acc0[k][tid] = val; s_acc1[k][tid] = 1.f; }
                    } else if (ft == BS_FUSE_HIGHEST_VIEWID_WINS) {
                        s_acc0[k][tid] = val; s_acc1[k][tid] = 1.f;
                    } else {  // CLOSEST_PIXEL_WINS: largest blending weight wins
                        if (w > c1) { s_acc0[k][tid] = val; s_acc1[k][tid] = w; }
                    }
                }
            }
        }
    }
    if (!valid) return;
#pragma unroll 1
    for (int k = 0; k < nz; ++k) {
        const size_t o = ((size_t)(z0 + k) * a.size[1] + y) * a.size[0] + x;
        const float c0 = s_acc0[k][tid], c1 = s_acc1[k][tid];
        if (ACCUM) {
            a.acc_wi[o] += c0;
            a.acc_w[o] += c1;
            continue;
        }
        float res;
        if (KIND == 0) res = c1 > 0.f ? c0 / c1 : 0.f;
        else res = c1 > 0.f ? c0 : 0.f;
        if (OUT == BS_DTYPE_F32) {
            __stcs((float*)a.out + o, res);
        } else {
            double c = floor(((double)res - a.cmin) * a.cscale + 0.5);
            c = fmin(fmax(c, 0.0), a.ctop);
            if (OUT == BS_DTYPE_U16) ((unsigned short*)a.out)[o] = (unsigned short)c;
            else ((unsigned char*)a.out)[o] = (unsigned char)c;
        }
    }
}

template <int OUT>
__global__ void fuse_finish_kernel(const float* __restrict__ swi, const float* __restrict__ sw, long long n,
                                   FuseArgs a) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float w = sw[i];
        float res = w > 0.f ? swi[i] / w : 0.f;
        if (OUT == BS_DTYPE_F32) {
            ((float*)a.out)[i] = res;
        } else {
            double c = floor(((double)res - a.cmin) * a.cscale + 0.5);
            c = fmin(fmax(c, 0.0), a.ctop);
            if (OUT == BS_DTYPE_U16) ((unsigned short*)a.out)[i] = (unsigned short)c;
            else ((unsigned char*)a.out)[i] = (unsigned char)c;
        }
    }
}

// ------------------------------------------------------------------------------------------
int bs_fuse_validate(bs_ctx* ctx, const bs_view* views, int n_views, const bs_fuse_params* p) {
    if (!views && n_views > 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: views is NULL");
    if (!p) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: NULL argument");
    if (n_views < 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: n_views < 0");
    if (p->fusion_type < BS_FUSE_AVG || p->fusion_type > BS_FUSE_CLOSEST_PIXEL_WINS)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: unknown fusion_type %d", p->fusion_type);
    if (p->interpolation != 0 && p->interpolation != 1)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: interpolation must be 0 or 1");
    if (p->out_dtype != BS_DTYPE_F32 && p->out_dtype != BS_DTYPE_U16 && p->out_dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: bad out_dtype %d", p->out_dtype);
    if (p->blend_lut_n < 0 || p->blend_lut_n > FUSE_MAX_LUT)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: blend_lut_n out of range [0,%d]", FUSE_MAX_LUT);
    if (p->out_dtype != BS_DTYPE_F32 && !(p->max_intensity > p->min_intensity))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: max_intensity must exceed min_intensity");
    for (int i = 0; i < n_views; ++i)
        if (ctx->vols.find(views[i].vol_handle) == ctx->vols.end())
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d has unknown vol_handle %llu", i, views[i].vol_handle);
    return BS_OK;
}

struct FusePrepared {
    FuseArgs args;
    int nviews;
    int slot;
    const FuseViewDev* views_dev;
};

// validate + upload view descriptors (and the cosine table); fills args except out pointers
static int fuse_prepare(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                        const long long block_size[3], const bs_fuse_params* p, FusePrepared* prep) {
    if (!views && n_views > 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: views is NULL");
    if (!block_min || !block_size || !p) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: NULL argument");
    if (n_views < 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: n_views < 0");
    for (int d = 0; d < 3; ++d)
        if (block_size[d] <= 0 || block_size[d] > 0x7fffffffLL)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: bad block_size[%d]=%lld", d, block_size[d]);
    if (p->fusion_type < BS_FUSE_AVG || p->fusion_type > BS_FUSE_CLOSEST_PIXEL_WINS)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: unknown fusion_type %d", p->fusion_type);
    if (p->interpolation != 0 && p->interpolation != 1)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: interpolation must be 0 or 1");
    if (p->out_dtype != BS_DTYPE_F32 && p->out_dtype != BS_DTYPE_U16 && p->out_dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: bad out_dtype %d", p->out_dtype);
    if (p->blend_lut_n < 0 || p->blend_lut_n > FUSE_MAX_LUT)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: blend_lut_n out of range [0,%d]", FUSE_MAX_LUT);
    if (p->out_dtype != BS_DTYPE_F32 && !(p->max_intensity > p->min_intensity))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: max_intensity must exceed min_intensity");
    const bool need_content = p->fusion_type == BS_FUSE_AVG_CONTENT || p->fusion_type == BS_FUSE_AVG_BLEND_CONTENT;

    std::vector<FuseViewDev> hv((size_t)n_views);
    for (int i = 0; i < n_views; ++i) {
        auto it = ctx->vols.find(views[i].vol_handle);
        if (it == ctx->vols.end())
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d has unknown vol_handle %llu", i, views[i].vol_handle);
        bs_volume& vol = it->second;
        { int rc = bs_volume_acquire(ctx, vol); if (rc) return rc; }
        if (views[i].full_dims[0] > 0)
            return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "bs_fuse: windowed views need uint16 sources with x size a multiple of 8, "
                                                            "n-linear interpolation and AVG / AVG_BLEND fusion");
        FuseViewDev& d = hv[i];
        if (!bs_invert34(views[i].src_to_world, d.inv))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d has a singular transform", i);
        d.data = vol.dev;
        d.dims[0] = (int)vol.dims[0]; d.dims[1] = (int)vol.dims[1]; d.dims[2] = (int)vol.dims[2];
        d.dtype = vol.dtype;
        d.content = nullptr;
        if (need_content) {
            auto ic = ctx->vols.find(views[i].content_handle);
            if (ic == ctx->vols.end() || ic->second.dtype != BS_DTYPE_F32 || ic->second.dims[0] != vol.dims[0] ||
                ic->second.dims[1] != vol.dims[1] || ic->second.dims[2] != vol.dims[2])
                return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d needs a float32 content volume of equal dims", i);
            d.content = (const float*)ic->second.dev;
        }
        for (int k = 0; k < 3; ++k) {
            d.border[k] = views[i].blend_border[k];
            d.range[k] = views[i].blend_range[k];
        }
    }
    const size_t lut_bytes = (size_t)(FUSE_MAX_LUT + 2) * sizeof(float);
    const size_t need = lut_bytes + hv.size() * sizeof(FuseViewDev);
    if (need > ctx->fuse_slot_bytes) {
        size_t sb = 1 << 16;
        while (sb < need) sb <<= 1;
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ctx->fuse_ring_dev) cudaFree(ctx->fuse_ring_dev);
        if (ctx->fuse_ring_host) cudaFreeHost(ctx->fuse_ring_host);
        ctx->fuse_ring_dev = ctx->fuse_ring_host = nullptr;
        ctx->fuse_slot_bytes = 0;
        BS_CUDA(ctx, cudaMalloc(&ctx->fuse_ring_dev, sb * bs_ctx::kFuseSlots));
        BS_CUDA(ctx, cudaHostAlloc(&ctx->fuse_ring_host, sb * bs_ctx::kFuseSlots, cudaHostAllocDefault));
        for (int i = 0; i < bs_ctx::kFuseSlots; ++i) {
            ctx->fuse_slot_used[i] = false;
            if (!ctx->fuse_slot_ev[i])
                BS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->fuse_slot_ev[i], cudaEventDisableTiming));
        }
        ctx->fuse_slot_bytes = sb;
    }
    const int slot = ctx->fuse_next_slot;
    ctx->fuse_next_slot = (slot + 1) % bs_ctx::kFuseSlots;
    if (ctx->fuse_slot_used[slot]) BS_CUDA(ctx, cudaEventSynchronize(ctx->fuse_slot_ev[slot]));
    unsigned char* hslot = (unsigned char*)ctx->fuse_ring_host + (size_t)slot * ctx->fuse_slot_bytes;
    unsigned char* dslot = (unsigned char*)ctx->fuse_ring_dev + (size_t)slot * ctx->fuse_slot_bytes;
    float* lut = (float*)hslot;
    const int n = p->blend_lut_n;
    if (n > 0) {
        for (int i = 0; i <= n; ++i) lut[i] = (float)((std::cos((1.0 - (double)i / n) * M_PI) + 1.0) / 2.0);
        lut[n + 1] = lut[n];
    }
    if (!hv.empty()) memcpy(hslot + lut_bytes, hv.data(), hv.size() * sizeof(FuseViewDev));
    BS_CUDA(ctx, cudaMemcpyAsync(dslot, hslot, need, cudaMemcpyHostToDevice, ctx->stream));
    prep->slot = slot;
    prep->views_dev = (const FuseViewDev*)(dslot + lut_bytes);

    FuseArgs& a = prep->args;
    memset(&a, 0, sizeof(a));
    for (int d = 0; d < 3; ++d) { a.bmin[d] = block_min[d]; a.size[d] = (int)block_size[d]; }
    a.fusion_type = p->fusion_type;
    a.lut_n = n;
    a.lut = (const float*)dslot;
    a.ctop = p->out_dtype == BS_DTYPE_U8 ? 255.0 : 65535.0;
    a.cmin = p->min_intensity;
    a.cscale = p->out_dtype == BS_DTYPE_F32 ? 1.0 : a.ctop / (p->max_intensity - p->min_intensity);
    {
        const char* e = getenv("BS_FUSE_NO_STAGE");
        a.no_stage = (e && *e && *e != '0') ? 1 : 0;
    }
    prep->nviews = n_views;
    return BS_OK;
}

template <int KIND, bool LINEAR, bool ACCUM>
static void launch_out(int out_dtype, dim3 grid, dim3 block, cudaStream_t s, const FuseViewDev* v, int n,
                       const FuseArgs& a) {
    const bool content = a.fusion_type == BS_FUSE_AVG_CONTENT || a.fusion_type == BS_FUSE_AVG_BLEND_CONTENT;
    const size_t dyn = content ? sizeof(float) * FS_N : 0;
    auto go = [&](auto kern) {
        if (dyn) cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
        kern<<<grid, block, dyn, s>>>(v, n, a);
    };
    if (ACCUM || out_dtype == BS_DTYPE_F32) go(fuse_kernel<KIND, LINEAR, BS_DTYPE_F32, ACCUM>);
    else if (out_dtype == BS_DTYPE_U16) go(fuse_kernel<KIND, LINEAR, BS_DTYPE_U16, false>);
    else go(fuse_kernel<KIND, LINEAR, BS_DTYPE_U8, false>);
}

static int fuse_launch(bs_ctx* ctx, const FusePrepared& prep, const bs_fuse_params* p, bool accum) {
    const FuseArgs& a = prep.args;
    dim3 block(FUSE_TX, FUSE_TY, 1);
    dim3 grid((a.size[0] + FUSE_TX - 1) / FUSE_TX, (a.size[1] + FUSE_TY - 1) / FUSE_TY,
              (a.size[2] + FUSE_ZT - 1) / FUSE_ZT);
    if (grid.y > 65535 || grid.z > 65535)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: block too large for one launch (y/z tiles > 65535)");
    const FuseViewDev* v = prep.views_dev;
    const bool winner = p->fusion_type >= BS_FUSE_MAX_INTENSITY;
    const bool lin = p->interpolation == 1;
    FuseArgs a2 = a;
    {
        const char* e = getenv("BS_FUSE_NO_PLAN");
        const long long ntiles = (long long)grid.x * grid.y * grid.z;
        if (!(e && *e && *e != '0') && prep.nviews > 0 && ntiles * (long long)sizeof(TilePlan) <= (256LL << 20)) {
            int rc = bs_ensure_dev(ctx, &ctx->fuse_plan, &ctx->fuse_plan_cap, (size_t)ntiles * sizeof(TilePlan));
            if (rc) return rc;
            a2.plan = (const TilePlan*)ctx->fuse_plan;
            bs_launch_scope scope(ctx, "fuse_plan");
            fuse_plan_kernel<<<(unsigned)((ntiles + 127) / 128), 128, 0, ctx->stream>>>(
                v, prep.nviews, a, (TilePlan*)ctx->fuse_plan, (int)grid.x, (int)grid.y, (int)grid.z, lin ? 1 : 0);
        }
    }
    {
        bs_launch_scope scope(ctx, "fuse");
        if (accum) {
            if (lin) launch_out<0, true, true>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
            else launch_out<0, false, true>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
        } else if (!winner) {
            if (lin) launch_out<0, true, false>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
            else launch_out<0, false, false>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
        } else {
            if (lin) launch_out<1, true, false>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
            else launch_out<1, false, false>(p->out_dtype, grid, block, ctx->stream, v, prep.nviews, a2);
        }
    }
    BS_CUDA(ctx, cudaGetLastError());
    BS_CUDA(ctx, cudaEventRecord(ctx->fuse_slot_ev[prep.slot], ctx->stream));
    ctx->fuse_slot_used[prep.slot] = true;
    return BS_OK;
}

extern "C" {

void bs_fuse_default_params(bs_fuse_params* p) {
    if (!p) return;
    p->fusion_type = BS_FUSE_AVG_BLEND;
    p->interpolation = 1;
    p->out_dtype = BS_DTYPE_F32;
    p->blend_lut_n = 0;
    p->min_intensity = 0.0;
    p->max_intensity = 65535.0;
    p->out_big_endian = 0;
    p->reserved = 0;
}

}  // extern "C"

// generic tile kernel for one block into a device buffer; the caller holds ctx->mu
int bs_fuse_legacy_block(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                         const long long block_size[3], const bs_fuse_params* params, void* out_dev) {
    FusePrepared prep;
    int rc = fuse_prepare(ctx, views, n_views, block_min, block_size, params, &prep);
    if (rc) return rc;
    prep.args.out = out_dev;
    return fuse_launch(ctx, prep, params, false);
}

extern "C" {

int bs_fuse_accumulate(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                       const long long block_size[3], const bs_fuse_params* params, float* sum_wi_dev,
                       float* sum_w_dev) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!sum_wi_dev || !sum_w_dev) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_accumulate: NULL accumulator");
    if (params && params->fusion_type >= BS_FUSE_MAX_INTENSITY)
        return bs_set_error(ctx, BS_ERR_UNSUPPORTED,
                            "bs_fuse_accumulate: only the weighted-average fusion types reduce by sum");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    FusePrepared prep;
    int rc = fuse_prepare(ctx, views, n_views, block_min, block_size, params, &prep);
    if (rc) return rc;
    prep.args.acc_wi = sum_wi_dev;
    prep.args.acc_w = sum_w_dev;
    return fuse_launch(ctx, prep, params, true);
}

int bs_fuse_finish(bs_ctx* ctx, const float* sum_wi_dev, const float* sum_w_dev, long long n,
                   const bs_fuse_params* params, void* out, int out_on_device) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!sum_wi_dev || !sum_w_dev || !out || !params || n <= 0)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_finish: bad argument");
    if (params->out_big_endian)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_finish: out_big_endian is only supported by bs_fuse_block(s)");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    FuseArgs a;
    memset(&a, 0, sizeof(a));
    a.ctop = params->out_dtype == BS_DTYPE_U8 ? 255.0 : 65535.0;
    a.cmin = params->min_intensity;
    a.cscale = params->out_dtype == BS_DTYPE_F32 ? 1.0 : a.ctop / (params->max_intensity - params->min_intensity);
    const size_t bytes = (size_t)n * bs_out_elem_size(params->out_dtype);
    if (out_on_device) {
        a.out = out;
    } else {
        int rc = bs_ensure_dev(ctx, &ctx->fuse_out, &ctx->fuse_out_cap, bytes);
        if (rc) return rc;
        a.out = ctx->fuse_out;
    }
    int threads = 256;
    int blocks = (int)std::min<long long>((n + threads - 1) / threads, (long long)ctx->sm_count * 16);
    {
        bs_launch_scope scope(ctx, "fuse_finish");
        if (params->out_dtype == BS_DTYPE_F32) fuse_finish_kernel<BS_DTYPE_F32><<<blocks, threads, 0, ctx->stream>>>(sum_wi_dev, sum_w_dev, n, a);
        else if (params->out_dtype == BS_DTYPE_U16) fuse_finish_kernel<BS_DTYPE_U16><<<blocks, threads, 0, ctx->stream>>>(sum_wi_dev, sum_w_dev, n, a);
        else fuse_finish_kernel<BS_DTYPE_U8><<<blocks, threads, 0, ctx->stream>>>(sum_wi_dev, sum_w_dev, n, a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    if (!out_on_device) {
        BS_CUDA(ctx, cudaMemcpyAsync(out, ctx->fuse_out, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return BS_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------ --masks mode
namespace {
#define MASK_MAX_VIEWS 64
struct MaskArgs {
    double inv[MASK_MAX_VIEWS][12];    // world -> source pixel
    double lo[MASK_MAX_VIEWS][3], hi[MASK_MAX_VIEWS][3];
    int n_views;
    long long bmin[3];
    int bsize[3];
    int out_dtype, swap;
    void* out;
};

// one thread per voxel, x fastest; double arithmetic like the reference's AffineTransform3D.applyInverse.
// (HBM-bound on the output write; the view loop stops at the first hit.)
__global__ void __launch_bounds__(256) k_mask_block(const __grid_constant__ MaskArgs a, int first_pass) {
    const long long n = (long long)a.bsize[0] * a.bsize[1] * a.bsize[2];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % a.bsize[0]);
        const long long r = i / a.bsize[0];
        const int y = (int)(r % a.bsize[1]), z = (int)(r / a.bsize[1]);
        const double wx = (double)(a.bmin[0] + x), wy = (double)(a.bmin[1] + y), wz = (double)(a.bmin[2] + z);
        bool on = false;
        for (int v = 0; v < a.n_views && !on; ++v) {
            const double* m = a.inv[v];
            // separately rounded products and left-to-right sums (no fma contraction), as Java evaluates them
            const double lx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], wx), __dmul_rn(m[1], wy)), __dmul_rn(m[2], wz)), m[3]);
            const double ly = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4], wx), __dmul_rn(m[5], wy)), __dmul_rn(m[6], wz)), m[7]);
            const double lz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[8], wx), __dmul_rn(m[9], wy)), __dmul_rn(m[10], wz)), m[11]);
            on = !(lx < a.lo[v][0] || lx > a.hi[v][0] || ly < a.lo[v][1] || ly > a.hi[v][1] || lz < a.lo[v][2] || lz > a.hi[v][2]);
        }
        if (!on && !first_pass) continue;          // later view groups only ever switch voxels on
        if (a.out_dtype == BS_DTYPE_F32) {
            const unsigned int one = a.swap ? 0x0000803fu : 0x3f800000u;
            ((unsigned int*)a.out)[i] = on ? one : 0u;
        } else if (a.out_dtype == BS_DTYPE_U16) {
            ((unsigned short*)a.out)[i] = on ? (unsigned short)0xffffu : (unsigned short)0u;
        } else {
            ((unsigned char*)a.out)[i] = on ? (unsigned char)255 : (unsigned char)0;
        }
    }
}
}  // namespace

extern "C" int bs_mask_blocks(bs_ctx* ctx, const bs_view* views, int n_views, int n_blocks, const long long* block_min,
                              const long long* block_size, const double mask_offset[3], int out_dtype, int out_big_endian,
                              void* const* outs, int out_on_device) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n_views < 0 || (n_views > 0 && !views) || n_blocks < 0 || !mask_offset || (n_blocks > 0 && (!block_min || !block_size || !outs)))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: bad argument");
    if (out_dtype != BS_DTYPE_F32 && out_dtype != BS_DTYPE_U16 && out_dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: bad out_dtype %d", out_dtype);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    // per view: inverse registration and the grown pixel interval
    std::vector<double> inv((size_t)std::max(n_views, 1) * 12), lo((size_t)std::max(n_views, 1) * 3), hi((size_t)std::max(n_views, 1) * 3);
    for (int v = 0; v < n_views; ++v) {
        long long dims[3];
        if (views[v].full_dims[0] > 0) {
            for (int d = 0; d < 3; ++d) dims[d] = views[v].full_dims[d];
        } else {
            auto it = ctx->vols.find(views[v].vol_handle);
            if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: view %d has neither full_dims nor a volume", v);
            for (int d = 0; d < 3; ++d) dims[d] = it->second.dims[d];
        }
        if (!bs_invert34(views[v].src_to_world, &inv[(size_t)v * 12]))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: view %d has a singular transform", v);
        for (int d = 0; d < 3; ++d) {
            lo[(size_t)v * 3 + d] = 0.0 - mask_offset[d];
            hi[(size_t)v * 3 + d] = (double)(dims[d] - 1) + mask_offset[d];
        }
    }
    const size_t es = bs_out_elem_size(out_dtype);
    for (int b = 0; b < n_blocks; ++b) {
        if (!outs[b]) return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: outs[%d] is NULL", b);
        long long nvox = 1;
        for (int d = 0; d < 3; ++d) {
            if (block_size[3 * b + d] <= 0 || block_size[3 * b + d] > 0x7fffffffLL)
                return bs_set_error(ctx, BS_ERR_ARG, "bs_mask_blocks: bad block_size");
            nvox *= block_size[3 * b + d];
        }
        void* dev = outs[b];
        if (!out_on_device) {
            int rc = bs_ensure_dev(ctx, &ctx->fuse_out, &ctx->fuse_out_cap, (size_t)nvox * es);
            if (rc) return rc;
            dev = ctx->fuse_out;
        }
        MaskArgs a;
        for (int d = 0; d < 3; ++d) { a.bmin[d] = block_min[3 * b + d]; a.bsize[d] = (int)block_size[3 * b + d]; }
        a.out_dtype = out_dtype;
        a.swap = (out_big_endian && es > 1) ? 1 : 0;
        a.out = dev;
        const int grid = (int)std::min<long long>((nvox + 255) / 256, (long long)ctx->sm_count * 16);
        // views in groups of MASK_MAX_VIEWS (kernel-parameter space); the first group also writes the zeros
        int v0 = 0;
        do {
            a.n_views = std::min(n_views - v0, MASK_MAX_VIEWS);
            for (int v = 0; v < a.n_views; ++v) {
                memcpy(a.inv[v], &inv[(size_t)(v0 + v) * 12], sizeof(double) * 12);
                memcpy(a.lo[v], &lo[(size_t)(v0 + v) * 3], sizeof(double) * 3);
                memcpy(a.hi[v], &hi[(size_t)(v0 + v) * 3], sizeof(double) * 3);
            }
            bs_launch_scope scope(ctx, "mask");
            k_mask_block<<<grid, 256, 0, ctx->stream>>>(a, v0 == 0 ? 1 : 0);
            v0 += MASK_MAX_VIEWS;
        } while (v0 < n_views);
        BS_CUDA(ctx, cudaGetLastError());
        if (!out_on_device) {
            BS_CUDA(ctx, cudaMemcpyAsync(outs[b], dev, (size_t)nvox * es, cudaMemcpyDeviceToHost, ctx->stream));
            BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
    }
    return BS_OK;
}
