// Hot path 2, main kernels: TMA-staged, z-marching affine fusion of a LIST of output blocks in one launch.
// Replaces BlkAffineFusion.init... + BlockAlgoUtils.arrayImg (J/SparkAffineFusion.java:602-627) for the
// weighted-average fusion types with n-linear interpolation on uint16 sources (the reference's default
// configuration); every other combination is served by the generic tile kernel in fuse.cu.
//
// Work decomposition.  Output tile = 64 x 16 x 8 voxels.  A CTA owns a z-run of tiles of one (x, y) tile
// column of one block and marches it.  Warp specialisation: one PRODUCER warp walks the plan of the CTA's
// tiles and, for every (tile, view), acquires a shared-memory slot, copies the view's tile constants into it
// and issues ONE 3-D tensor-map TMA load (cp.async.bulk.tensor, out-of-bounds zero fill) of the uint16
// source box the tile's taps can touch; eight CONSUMER warps wait on the slots' mbarriers, sample from
// shared memory, blend, and store.  All views of a tile are resident at the same time, so the view loop is
// the INNER loop: no per-voxel accumulator arrays, a rolled z loop, and (translation kernel) a rolling
// register window over z -- every staged source voxel is converted once per thread and every x / y
// interpolation is shared between the two z neighbours that need it.
//
//   translation kernel (world->source linear part == identity, the stitching case): thread = 2 x 2 (x, y)
//     voxels, taps fetched as 32-bit words (two uint16), x-lerps shared between x neighbours, y-lerps between
//     y neighbours, z-lerp against the previous plane kept in registers; blending weights are separable
//     (wx * wy per thread, wz per plane from the plan).
//   general kernel (any affine): per-voxel 8-tap sampling from the staged box, tile-relative float
//     coordinates; footprints that do not fit the box, or tiles with more views than slots, gather from
//     global memory instead.
//
// Plan pre-pass (plan_kernel): one thread per tile culls the block's candidate views (double precision) and
// writes the tile's view items (box origin, tile-relative transform, plateau / inside flags, z weights).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstring>

#include "bs_internal.cuh"
#include "fuse_common.cuh"

namespace {

constexpr int TT_X = 64, TT_Y = 16, TT_Z = 8;
constexpr int NTEAM = 256;                 // consumer threads per team (8 warps render one tile)
constexpr int NTEAMS = 2;                  // two teams work on alternate tiles of the CTA's run
constexpr int NCONS = NTEAM * NTEAMS;
constexpr int NTHREADS = NCONS + 32;       // + 1 producer warp
// TMA (tiled, no swizzle): the box start along the innermost dimension must be 16-byte aligned, i.e. a multiple
// of 8 uint16 (an unaligned x coordinate raises "illegal instruction"); negative / out-of-range coordinates are
// fine and zero-filled.  Boxes therefore start at floor8(x0) and carry up to 7 extra columns.
constexpr int BXT = 72, BYT = 17, BZT = 9;     // translation box (uint16 elements; (7 +) 65 x 17 x 9 needed)
constexpr int BXG = 80, BYG = 20, BZG = 12;    // general box (x origin is rounded down to a multiple of 8)
constexpr int SLOT_T = ((BXT * BYT * BZT * 2 + 127) / 128) * 128;   // 22144 B
constexpr int SLOT_G = ((BXG * BYG * BZG * 2 + 127) / 128) * 128;   // 34560 B
constexpr int NST_T = 8, NST_G = 5;        // box slots per CTA (1 CTA per SM)
constexpr int NTR = 4;                     // tile-record ring

enum { VI_PLAT_X = 1, VI_PLAT_Y = 2, VI_PLAT_Z = 4, VI_INSIDE = 8, VI_FITS = 16 };

struct __align__(64) ViewDev {
    double inv[12];               // world -> source pixel
    double wlo[3], whi[3];        // world AABB of the view (expanded), second cull test
    const void* data;
    const float* content;         // content-weight volume (float32, same dims as the volume) or nullptr
    const CUtensorMap* tm_t;      // device copies of the tensor maps (translation box / general box)
    const CUtensorMap* tm_g;
    int dims[3];                  // size of the (full) view: inside test, blending
    int pad0;
    float border[3], range[3];
    int wdims[3];                 // resident window [woff, woff + wdims) of the view (== dims, 0 when not windowed)
    int woff[3];
};

struct __align__(16) ViewItem {   // per (tile, view); 112 B
    int view;
    int flags;
    int b0[3];                    // TMA box origin in source pixels (may be negative: zero fill)
    float o[3];                   // translation: fractional offsets; general: box-relative source coordinate of tile voxel (0,0,0)
    union {
        float wz[8];              // translation: z weight of output plane k (0 = excluded)
        float m[9];               // general: linear part of world -> source
    };
    float dm1[3], border[3], inv_range[3];
    int tma[3];                   // box origin in WINDOW coordinates, x a multiple of 8 (the TMA coordinates)
    int ox;                       // translation: column of the tile's first tap inside the box (0..7)
    int pad[1];
};
static_assert(sizeof(ViewItem) == 128, "ViewItem layout");
constexpr int VI_WORDS = sizeof(ViewItem) / 4;

struct TileHdr { int first, count, mode, pad; };   // mode 0: no view, 1: resident (TMA), 2: gather from global

struct BlockDev {
    long long bmin[3];
    int size[3];
    int tiles[3];
    int ntiles;
    int tile_base;
    int cand_off, cand_n;
    void* out;
};

struct WorkRec { int block, tx, ty, tz0, ntz, pad[3]; };

struct TileRec {
    unsigned long long out;       // address of the tile's first voxel
    long long pitch_z;            // elements
    int pitch_y;
    int nx, ny, nz;
    int count, mode, it0, last;
    const ViewItem* items;
};

struct FuseArgs2 {
    const ViewDev* views;
    const BlockDev* blocks;
    const WorkRec* work;
    const TileHdr* hdr;
    const ViewItem* pool;
    int* work_ctr;                // dynamic work distribution (zeroed per launch)
    int nwork;
    int use_blend;
    int xyaff;                    // general kernel: every view is an xy-affine + z-translation (fast z-marching tiles)
    double cmin, cscale, ctop;
};

// ------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_box(void* dst, const CUtensorMap* tm, int x, int y, int z, unsigned long long* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(dst)), "l"(tm), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tmap_acquire(const CUtensorMap* tm) {
    // the descriptor lives in global memory (written by a host copy): make it visible to the tensormap proxy
    asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(tm) : "memory");
}

// The per-call tables (views, blocks, candidates, work records) travel from a mapped pinned buffer to device memory
// by this kernel, NOT by cudaMemcpyAsync: a DMA copy would queue on the host->device copy engine behind every tile
// upload already in flight (bs_volume_upload_async), and the plan / fusion kernels of the first blocks would wait for
// ALL of the step's uploads.
__global__ void fuse_meta_copy_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src_mapped, int n16) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += gridDim.x * blockDim.x) dst[i] = src_mapped[i];
}

// ------------------------------------------------------------------------------------------ plan pre-pass
struct CullOut { bool hit, fits; };

// translation == true: inv linear part is the identity.  Fills `it` when non-null.
__device__ __forceinline__ CullOut cull_view(const ViewDev& v, int vi, const double w0[3], const double ext[3], bool general,
                                             bool use_blend, ViewItem* it) {
    CullOut r{true, true};
    int flags = VI_INSIDE | VI_PLAT_X | VI_PLAT_Y | VI_PLAT_Z;
    int b0[3], tma[3] = {0, 0, 0}, ox = 0;
    float o[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (w0[a] + ext[a] < v.wlo[a] || w0[a] > v.whi[a]) r.hit = false;
        const double m0 = v.inv[4 * a], m1 = v.inv[4 * a + 1], m2 = v.inv[4 * a + 2], t = v.inv[4 * a + 3];
        const int dim = v.dims[a];
        const double dm1 = (double)(dim - 1);
        double lo, hi;
        if (!general) {
            const double ft = floor(t);
            const double b = w0[a] + ft;           // exact integer
            b0[a] = (int)b;
            o[a] = (float)(t - ft);
            tma[a] = b0[a] - v.woff[a];
            if (a == 0) { ox = tma[0] & 7; tma[0] &= ~7; }   // 16-byte aligned TMA box origin
            lo = b + (t - ft);
            hi = lo + ext[a];
        } else {
            const double org = fma(m0, w0[0], fma(m1, w0[1], fma(m2, w0[2], t)));
            lo = org + fmin(0.0, m0 * ext[0]) + fmin(0.0, m1 * ext[1]) + fmin(0.0, m2 * ext[2]);
            hi = org + fmax(0.0, m0 * ext[0]) + fmax(0.0, m1 * ext[1]) + fmax(0.0, m2 * ext[2]);
            const double eps = 2e-3 + 2e-7 * fmax(fabs(lo), fabs(hi));
            int f0 = max((int)floor(fmax(lo - eps, 0.0)), 0);
            if (a == 0) f0 = v.woff[0] + ((f0 - v.woff[0]) & ~7);   // 16-byte aligned TMA box origin (window coordinates)
            tma[a] = f0 - v.woff[a];
            const int f1 = min((int)floor(fmin(hi + eps, dm1)), dim - 1) + 1;
            const int cap = a == 0 ? BXG : (a == 1 ? BYG : BZG);
            if (f1 - f0 + 1 > cap) r.fits = false;
            b0[a] = f0;
            o[a] = (float)(org - (double)f0);
        }
        if (hi < -1e-3 || lo > dm1 + 1e-3) r.hit = false;
        const double eps = 2e-3 + 2e-7 * fmax(fabs(lo), fabs(hi));
        if (!(lo - eps >= 0.0 && hi + eps <= dm1)) flags &= ~VI_INSIDE;
        bool plat;
        if (use_blend)
            plat = (lo - eps - (double)v.border[a] >= (double)v.range[a]) &&
                   (dm1 - (hi + eps) - (double)v.border[a] >= (double)v.range[a]);
        else
            plat = (lo - eps >= 0.0 && hi + eps <= dm1);
        if (!plat) flags &= ~(VI_PLAT_X << a);
    }
    if (!r.hit || !it) return r;
    if (r.fits) flags |= VI_FITS;
    it->view = vi;
    it->flags = flags;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        it->b0[a] = b0[a];
        it->tma[a] = tma[a];
        it->o[a] = o[a];
        it->dm1[a] = (float)(v.dims[a] - 1);
        it->border[a] = v.border[a];
        it->inv_range[a] = 1.0f / v.range[a];
    }
    if (!general) {
#pragma unroll
        for (int k = 0; k < TT_Z; ++k)
            it->wz[k] = (flags & VI_PLAT_Z) ? 1.f
                                            : blend_factor((float)(b0[2] + k) + o[2], it->dm1[2], it->border[2],
                                                           it->inv_range[2], use_blend);
    } else {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            it->m[3 * a] = (float)v.inv[4 * a];
            it->m[3 * a + 1] = (float)v.inv[4 * a + 1];
            it->m[3 * a + 2] = (float)v.inv[4 * a + 2];
        }
    }
    it->ox = ox;
    it->pad[0] = 0;
    return r;
}

__global__ void fuse_plan2_kernel(const ViewDev* __restrict__ views, const BlockDev* __restrict__ blocks,
                                  const int* __restrict__ cand, TileHdr* __restrict__ hdr, ViewItem* __restrict__ pool,
                                  int* __restrict__ ctr /* [0] pool counter, [1] overflow flag */, int pool_cap,
                                  int use_blend, int general, int nst) {
    const BlockDev& B = blocks[blockIdx.y];
    const int local = blockIdx.x * blockDim.x + threadIdx.x;
    if (local >= B.ntiles) return;
    const int tx = local % B.tiles[0], ty = (local / B.tiles[0]) % B.tiles[1], tz = local / (B.tiles[0] * B.tiles[1]);
    const double w0[3] = {(double)(B.bmin[0] + (long long)tx * TT_X), (double)(B.bmin[1] + (long long)ty * TT_Y),
                          (double)(B.bmin[2] + (long long)tz * TT_Z)};
    const double ext[3] = {(double)(min(TT_X, B.size[0] - tx * TT_X) - 1), (double)(min(TT_Y, B.size[1] - ty * TT_Y) - 1),
                           (double)(min(TT_Z, B.size[2] - tz * TT_Z) - 1)};
    int cnt = 0;
    bool allfit = true;
    for (int c = 0; c < B.cand_n; ++c) {
        const int vi = cand[B.cand_off + c];
        const CullOut r = cull_view(views[vi], vi, w0, ext, general != 0, use_blend != 0, nullptr);
        if (r.hit) { ++cnt; allfit = allfit && r.fits; }
    }
    int mode = cnt == 0 ? 0 : ((cnt <= nst && allfit) ? 1 : 2);
    int first = 0;
    if (cnt) {
        first = atomicAdd(&ctr[0], cnt);
        if (first + cnt > pool_cap) { atomicExch(&ctr[1], 1); cnt = 0; mode = 0; first = 0; }
    }
    TileHdr h; h.first = first; h.count = cnt; h.mode = mode; h.pad = 0;
    hdr[B.tile_base + local] = h;
    if (!cnt) return;
    int e = 0;
    for (int c = 0; c < B.cand_n && e < cnt; ++c) {
        const int vi = cand[B.cand_off + c];
        ViewItem it;
        const CullOut r = cull_view(views[vi], vi, w0, ext, general != 0, use_blend != 0, &it);
        if (r.hit) pool[first + e++] = it;
    }
}

// ------------------------------------------------------------------------------------------ output
// (OUT = output dtype | OUT_BE, see fuse_common.cuh)
template <int OUT>
__device__ __forceinline__ unsigned int conv_int(const FuseArgs2& a, float res) {
    double c = floor(((double)res - a.cmin) * a.cscale + 0.5);
    return (unsigned int)fmin(fmax(c, 0.0), a.ctop);
}
template <int OUT>
__device__ __forceinline__ void store1(const FuseArgs2& a, void* p, float res) {
    constexpr bool BE = (OUT & OUT_BE) != 0;
    if (OUT_DT(OUT) == BS_DTYPE_F32) {
        if (BE) __stcs((unsigned int*)p, bswap32(__float_as_uint(res)));
        else __stcs((float*)p, res);
    } else {
        const unsigned int c = conv_int<OUT>(a, res);
        if (OUT_DT(OUT) == BS_DTYPE_U16) *(unsigned short*)p = (unsigned short)(BE ? bswap16x2(c) : c);
        else *(unsigned char*)p = (unsigned char)c;
    }
}
template <int DT> struct OutT_ { using type = float; };
template <> struct OutT_<BS_DTYPE_U16> { using type = unsigned short; };
template <> struct OutT_<BS_DTYPE_U8> { using type = unsigned char; };
template <int OUT> struct OutT { using type = typename OutT_<OUT_DT(OUT)>::type; };

// store two x-adjacent voxels (x even within the tile); vec: the pair is 8-/4-/2-byte aligned and both exist
template <int OUT>
__device__ __forceinline__ void store_pair(const FuseArgs2& a, typename OutT<OUT>::type* p, float r0, float r1, bool has1,
                                           bool vec) {
    constexpr bool BE = (OUT & OUT_BE) != 0;
    if (OUT_DT(OUT) == BS_DTYPE_F32) {
        if (BE) {
            const unsigned int u0 = bswap32(__float_as_uint(r0)), u1 = bswap32(__float_as_uint(r1));
            if (vec && has1) __stcs((uint2*)p, make_uint2(u0, u1));
            else { __stcs((unsigned int*)p, u0); if (has1) __stcs((unsigned int*)p + 1, u1); }
        } else if (vec && has1) {
            __stcs((float2*)p, make_float2(r0, r1));
        } else {
            __stcs((float*)p, r0);
            if (has1) __stcs((float*)p + 1, r1);
        }
    } else if (OUT_DT(OUT) == BS_DTYPE_U16) {
        unsigned int c = conv_int<OUT>(a, r0) | (conv_int<OUT>(a, r1) << 16);
        if (BE) c = bswap16x2(c);
        if (vec && has1) *(unsigned int*)p = c;
        else { p[0] = (unsigned short)(c & 0xffffu); if (has1) p[1] = (unsigned short)(c >> 16); }
    } else {
        const unsigned int c0 = conv_int<OUT>(a, r0), c1 = conv_int<OUT>(a, r1);
        if (vec && has1) *(unsigned short*)p = (unsigned short)(c0 | (c1 << 8));
        else { p[0] = (unsigned char)c0; if (has1) p[1] = (unsigned char)c1; }
    }
}

// sum(w I) / sum(w): one MUFU.RCP + FMUL (2 ulp) for ordinary weights, IEEE division for denormal-range sums
__device__ __forceinline__ float wdiv(float swi, float sw) {
    if (sw > 1e-30f) {
        float r;
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(sw));
        return swi * r;
    }
    return sw > 0.f ? swi / sw : 0.f;
}

template <typename T>
__device__ __forceinline__ float gather8(const T* __restrict__ d, int dx, int dy, int dz, float sx, float sy, float sz) {
    const float fx = floorf(sx), fy = floorf(sy), fz = floorf(sz);
    const float rx = sx - fx, ry = sy - fy, rz = sz - fz;
    const int x0 = min(max((int)fx, 0), dx - 1), y0 = min(max((int)fy, 0), dy - 1), z0 = min(max((int)fz, 0), dz - 1);
    const int x1 = min(x0 + 1, dx - 1), y1 = min(y0 + 1, dy - 1), z1 = min(z0 + 1, dz - 1);
    const size_t r00 = ((size_t)z0 * dy + y0) * dx, r01 = ((size_t)z0 * dy + y1) * dx;
    const size_t r10 = ((size_t)z1 * dy + y0) * dx, r11 = ((size_t)z1 * dy + y1) * dx;
    const float a000 = (float)__ldg(d + r00 + x0), a001 = (float)__ldg(d + r00 + x1);
    const float a010 = (float)__ldg(d + r01 + x0), a011 = (float)__ldg(d + r01 + x1);
    const float a100 = (float)__ldg(d + r10 + x0), a101 = (float)__ldg(d + r10 + x1);
    const float a110 = (float)__ldg(d + r11 + x0), a111 = (float)__ldg(d + r11 + x1);
    const float c00 = a000 + rx * (a001 - a000), c01 = a010 + rx * (a011 - a010);
    const float c10 = a100 + rx * (a101 - a100), c11 = a110 + rx * (a111 - a110);
    const float c0 = c00 + ry * (c01 - c00), c1 = c10 + ry * (c11 - c10);
    return c0 + rz * (c1 - c0);
}

// ------------------------------------------------------------------------------------------ translation tile
// one z plane of the staged box -> the thread's 2 x 2 x/y-interpolated values (x then y, a + f (b - a)).
// uint16 -> float without the conversion pipe: PRMT builds 0x4B00hhll = 2^23 + v, differences of two such
// floats are exact, and v itself is one FADD away.  sel01 packs taps (x0, x0+1) out of the two words the row
// loads (x0 even: w0; x0 odd: w0.hi, w1.lo), sel2 picks tap x0+2 from w1.
__device__ __forceinline__ void tr_plane(const unsigned int* __restrict__ rowbase, unsigned int sel01, unsigned int sel2,
                                         float fx, float fy, float (&c)[4]) {
    constexpr unsigned int MAG = 0x4B000000u;
    float r[3][2];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const unsigned int w0 = rowbase[j * (BXT / 2)], w1 = rowbase[j * (BXT / 2) + 1];
        const unsigned int p = __byte_perm(w0, w1, sel01);
        const float f0 = __uint_as_float(__byte_perm(p, MAG, 0x7610));
        const float f1 = __uint_as_float(__byte_perm(p, MAG, 0x7632));
        const float f2 = __uint_as_float(__byte_perm(w1, MAG, sel2));
        r[j][0] = fmaf(fx, f1 - f0, f0 - 8388608.f);
        r[j][1] = fmaf(fx, f2 - f1, f1 - 8388608.f);
    }
    c[0] = r[0][0] + fy * (r[1][0] - r[0][0]);
    c[1] = r[0][1] + fy * (r[1][1] - r[0][1]);
    c[2] = r[1][0] + fy * (r[2][0] - r[1][0]);
    c[3] = r[1][1] + fy * (r[2][1] - r[1][1]);
}

// content-based weights: the same 2 x 2 interpolation of one z plane, taps straight from the float32 content volume in
// global memory (L1 / L2: lanes cover 65 consecutive floats per row); indices are clamped like the oracle's border
// extension.  xi: the three clamped x indices, yo: the three clamped row offsets (y * dx), plane: content + z * dy * dx.
__device__ __forceinline__ void tr_plane_c(const float* __restrict__ plane, const int (&xi)[3], const int (&yo)[3], float fx, float fy,
                                           float (&c)[4]) {
    float r[3][2];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float* row = plane + yo[j];
        const float t0 = __ldg(row + xi[0]), t1 = __ldg(row + xi[1]), t2 = __ldg(row + xi[2]);
        r[j][0] = t0 + fx * (t1 - t0);
        r[j][1] = t1 + fx * (t2 - t1);
    }
    c[0] = r[0][0] + fy * (r[1][0] - r[0][0]);
    c[1] = r[0][1] + fy * (r[1][1] - r[0][1]);
    c[2] = r[1][0] + fy * (r[2][0] - r[1][0]);
    c[3] = r[1][1] + fy * (r[2][1] - r[1][1]);
}

// x / y blending factors of a tile's views, computed once per tile by the team (80 values per view: 64 x
// columns + 16 y rows) into a double-buffered shared table; returns the table to read from
constexpr int WT_N = TT_X + TT_Y;
__device__ __forceinline__ const float* team_weights(const FuseArgs2& a, const ViewItem* descs, const TileRec& T, int nst,
                                                     float* wtab, int& uses, int team, int tid) {
    float* tab = wtab + (uses & 1) * (NST_T * WT_N);
    ++uses;
    const bool ub = a.use_blend != 0;
    for (int i = tid; i < T.count * WT_N; i += NTEAM) {
        const int v = i / WT_N, j = i - v * WT_N;
        const ViewItem& d = descs[(T.it0 + v) % nst];
        float f = 1.f;
        if (j < TT_X) {
            if (!(d.flags & VI_PLAT_X)) f = blend_factor((float)(d.b0[0] + j) + d.o[0], d.dm1[0], d.border[0], d.inv_range[0], ub);
        } else {
            if (!(d.flags & VI_PLAT_Y)) f = blend_factor((float)(d.b0[1] + (j - TT_X)) + d.o[1], d.dm1[1], d.border[1], d.inv_range[1], ub);
        }
        tab[i] = f;
    }
    asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "r"(NTEAM) : "memory");
    return tab;
}

// PLAT (C == 1 only): the single view's weight is 1 on the whole tile -> the voxel is the sample itself
template <int C, int OUT, bool PLAT = false, bool CONTENT = false>
__device__ __forceinline__ void tr_tile(const FuseArgs2& a, const unsigned char* slots, const ViewItem* descs,
                                        const TileRec& T, float* wtab, int& uses, int team, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    const unsigned int* base[C];
    const float* wz[C];
    unsigned int sel01[C], sel2[C];
    float fx[C], fy[C], fz[C], wxy[C][4], prev[C][4];
    // content path: per view the volume, its plane pitch, the clamped tap columns / row offsets, first z, previous plane
    const float* cvol[CONTENT ? C : 1];
    int cxi[CONTENT ? C : 1][3], cyo[CONTENT ? C : 1][3], cz0[CONTENT ? C : 1], cdz[CONTENT ? C : 1];
    long long cpl[CONTENT ? C : 1];
    float cprev[CONTENT ? C : 1][4];
    bool need = false;
#pragma unroll
    for (int v = 0; v < C; ++v) {
        const int fl = descs[(T.it0 + v) % NST_T].flags;
        need = need || (fl & (VI_PLAT_X | VI_PLAT_Y)) != (VI_PLAT_X | VI_PLAT_Y);
    }
    const float* tab = nullptr;
    if (need) tab = team_weights(a, descs, T, NST_T, wtab, uses, team, tid);   // team-uniform branch
#pragma unroll
    for (int v = 0; v < C; ++v) {
        const int s = (T.it0 + v) % NST_T;
        const ViewItem& d = descs[s];
        const int ox = d.ox;                   // column of the tile's first tap inside the 8-aligned box
        base[v] = reinterpret_cast<const unsigned int*>(slots + (size_t)s * SLOT_T) + (2 * ly) * (BXT / 2) + lx + (ox >> 1);
        sel01[v] = (ox & 1) ? 0x5432u : 0x3210u;
        sel2[v] = (ox & 1) ? 0x7632u : 0x7610u;
        wz[v] = d.wz;
        fx[v] = d.o[0]; fy[v] = d.o[1]; fz[v] = d.o[2];
        float wx0 = 1.f, wx1 = 1.f, wy0 = 1.f, wy1 = 1.f;
        if (need) {
            const float* tv = tab + v * WT_N;
            wx0 = tv[2 * lx]; wx1 = tv[2 * lx + 1];
            wy0 = tv[TT_X + 2 * ly]; wy1 = tv[TT_X + 2 * ly + 1];
        }
        wxy[v][0] = wx0 * wy0; wxy[v][1] = wx1 * wy0; wxy[v][2] = wx0 * wy1; wxy[v][3] = wx1 * wy1;
        tr_plane(base[v], sel01[v], sel2[v], fx[v], fy[v], prev[v]);
        if (CONTENT) {
            const ViewDev& V = a.views[d.view];
            cvol[v] = V.content;
            cpl[v] = (long long)V.dims[0] * V.dims[1];
            cz0[v] = d.b0[2];
            cdz[v] = V.dims[2];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                cxi[v][i] = min(max(d.b0[0] + 2 * lx + i, 0), V.dims[0] - 1);
                cyo[v][i] = min(max(d.b0[1] + 2 * ly + i, 0), V.dims[1] - 1) * V.dims[0];
            }
            tr_plane_c(cvol[v] + (long long)min(max(cz0[v], 0), cdz[v] - 1) * cpl[v], cxi[v], cyo[v], fx[v], fy[v], cprev[v]);
        }
    }
    const int x = 2 * lx, y = 2 * ly;
    const bool ok0 = y < T.ny && x < T.nx, ok1 = y + 1 < T.ny && x < T.nx;
    const bool has1 = x + 1 < T.nx;
    OT* o0 = reinterpret_cast<OT*>(T.out) + (size_t)y * T.pitch_y + x;
    const bool vec = ((T.out | ((unsigned long long)T.pitch_y * sizeof(OT)) | ((unsigned long long)T.pitch_z * sizeof(OT))) & (2 * sizeof(OT) - 1)) == 0;
#pragma unroll 1
    for (int k = 0; k < T.nz; ++k) {
        float swi[4] = {0.f, 0.f, 0.f, 0.f}, sw[4] = {0.f, 0.f, 0.f, 0.f}, res[4];
#pragma unroll
        for (int v = 0; v < C; ++v) {
            float cur[4], ccur[4];
            if (CONTENT)    // issued first: the global loads fly while the shared-memory plane is interpolated
                tr_plane_c(cvol[v] + (long long)min(max(cz0[v] + k + 1, 0), cdz[v] - 1) * cpl[v], cxi[v], cyo[v], fx[v], fy[v], ccur);
            tr_plane(base[v] + (k + 1) * (BYT * BXT / 2), sel01[v], sel2[v], fx[v], fy[v], cur);
            const float wk = wz[v][k];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float val = prev[v][q] + fz[v] * (cur[q] - prev[v][q]);
                prev[v][q] = cur[q];
                if (PLAT) { res[q] = val; continue; }
                float w = wxy[v][q] * wk;
                if (CONTENT) {
                    w *= cprev[v][q] + fz[v] * (ccur[q] - cprev[v][q]);
                    cprev[v][q] = ccur[q];
                }
                if (C == 1) {
                    res[q] = w > 0.f ? val : 0.f;
                } else {
                    swi[q] = swi[q] + w * val;
                    sw[q] = sw[q] + w;
                }
            }
        }
        if (C > 1) {
#pragma unroll
            for (int q = 0; q < 4; ++q) res[q] = wdiv(swi[q], sw[q]);
        }
        OT* p = o0 + (size_t)k * T.pitch_z;
        if (ok0) store_pair<OUT>(a, p, res[0], res[1], has1, vec);
        if (ok1) store_pair<OUT>(a, p + T.pitch_y, res[2], res[3], has1, vec);
    }
}

// ------------------------------------------------------------------------------------------ general tile
// > 4 resident views (the 2 x 2 x 2 corners of a tile grid): rolled view loop, both z planes of every
// output plane recomputed (no per-view register state)
template <int OUT, bool CONTENT = false>
__device__ __forceinline__ void tr_tile_many(const FuseArgs2& a, const unsigned char* slots, const ViewItem* descs,
                                             const TileRec& T, float* wtab, int& uses, int team, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    const int x = 2 * lx, y = 2 * ly;
    const bool ok0 = y < T.ny && x < T.nx, ok1 = y + 1 < T.ny && x < T.nx;
    const bool has1 = x + 1 < T.nx;
    OT* o0 = reinterpret_cast<OT*>(T.out) + (size_t)y * T.pitch_y + x;
    const bool vec = ((T.out | ((unsigned long long)T.pitch_y * sizeof(OT)) | ((unsigned long long)T.pitch_z * sizeof(OT))) & (2 * sizeof(OT) - 1)) == 0;
    const float* tab = team_weights(a, descs, T, NST_T, wtab, uses, team, tid);
#pragma unroll 1
    for (int k = 0; k < T.nz; ++k) {
        float swi[4] = {0.f, 0.f, 0.f, 0.f}, sw[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int v = 0; v < T.count; ++v) {
            const int s = (T.it0 + v) % NST_T;
            const ViewItem& d = descs[s];
            const float wk = d.wz[k];
            if (wk == 0.f) continue;   // team-uniform
            const int ox = d.ox;
            const unsigned int sel01 = (ox & 1) ? 0x5432u : 0x3210u, sel2 = (ox & 1) ? 0x7632u : 0x7610u;
            const unsigned int* base = reinterpret_cast<const unsigned int*>(slots + (size_t)s * SLOT_T) +
                                       (k * BYT + 2 * ly) * (BXT / 2) + lx + (ox >> 1);
            const float fx = d.o[0], fy = d.o[1], fz = d.o[2];
            const float* tv = tab + v * WT_N;
            const float wx0 = tv[x], wx1 = tv[x + 1], wy0 = tv[TT_X + y], wy1 = tv[TT_X + y + 1];
            const float wxy[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};
            float c0[4], c1[4], w0[4], w1[4];
            if (CONTENT) {
                const ViewDev& V = a.views[d.view];
                int xi[3], yo[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    xi[i] = min(max(d.b0[0] + x + i, 0), V.dims[0] - 1);
                    yo[i] = min(max(d.b0[1] + y + i, 0), V.dims[1] - 1) * V.dims[0];
                }
                const long long pl = (long long)V.dims[0] * V.dims[1];
                tr_plane_c(V.content + (long long)min(max(d.b0[2] + k, 0), V.dims[2] - 1) * pl, xi, yo, fx, fy, w0);
                tr_plane_c(V.content + (long long)min(max(d.b0[2] + k + 1, 0), V.dims[2] - 1) * pl, xi, yo, fx, fy, w1);
            }
            tr_plane(base, sel01, sel2, fx, fy, c0);
            tr_plane(base + BYT * BXT / 2, sel01, sel2, fx, fy, c1);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float val = c0[q] + fz * (c1[q] - c0[q]);
                float w = wxy[q] * wk;
                if (CONTENT) w *= w0[q] + fz * (w1[q] - w0[q]);
                swi[q] = swi[q] + w * val;
                sw[q] = sw[q] + w;
            }
        }
        float res[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) res[q] = wdiv(swi[q], sw[q]);
        OT* p = o0 + (size_t)k * T.pitch_z;
        if (ok0) store_pair<OUT>(a, p, res[0], res[1], has1, vec);
        if (ok1) store_pair<OUT>(a, p + T.pitch_y, res[2], res[3], has1, vec);
    }
}

// more views than slots: every tap gathered from global memory (L1/L2)
template <int OUT, bool CONTENT = false>
__device__ __forceinline__ void tr_slow_tile(const FuseArgs2& a, const TileRec& T, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    const bool ub = a.use_blend != 0;
    OT* obase = reinterpret_cast<OT*>(T.out);
#pragma unroll 1
    for (int k = 0; k < T.nz; ++k) {
#pragma unroll 1
        for (int q = 0; q < 4; ++q) {
            const int x = 2 * lx + (q & 1), y = 2 * ly + (q >> 1);
            if (x >= T.nx || y >= T.ny) continue;
            float swi = 0.f, sw = 0.f;
#pragma unroll 1
            for (int v = 0; v < T.count; ++v) {
                const ViewItem& d = T.items[v];
                const ViewDev& V = a.views[d.view];
                const float sx = (float)(d.b0[0] + x) + d.o[0], sy = (float)(d.b0[1] + y) + d.o[1];
                const float sz = (float)(d.b0[2] + k) + d.o[2];
                float w = (blend_factor(sx, d.dm1[0], d.border[0], d.inv_range[0], ub) *
                           blend_factor(sy, d.dm1[1], d.border[1], d.inv_range[1], ub)) * d.wz[k];
                if (CONTENT && w > 0.f) w *= gather8(V.content, V.dims[0], V.dims[1], V.dims[2], sx, sy, sz);
                if (!(w > 0.f)) continue;
                const float val = gather8((const unsigned short*)V.data, V.wdims[0], V.wdims[1], V.wdims[2],
                                          sx - (float)V.woff[0], sy - (float)V.woff[1], sz - (float)V.woff[2]);
                swi = swi + w * val;
                sw = sw + w;
            }
            store1<OUT>(a, obase + (size_t)k * T.pitch_z + (size_t)y * T.pitch_y + x, wdiv(swi, sw));
        }
    }
}

// xy-affine views (world->source has no z coupling: m2 = m5 = m6 = m7 = 0, m8 = 1 -- rotations about z, xy scale /
// shear, any translation): a voxel COLUMN keeps its tap address, x / y fractions and x / y weights for the whole z run,
// the z fraction is one constant per view, and the x/y-interpolated value of plane k + 1 is the lower plane of the next
// step -- 4 taps + 3 lerps per voxel instead of 8 + 7, no per-voxel floor or address arithmetic.  <= 2 views per tile.
template <int C, int OUT>
__device__ __forceinline__ void xy_tile(const FuseArgs2& a, const unsigned char* slots, const ViewItem* descs,
                                        const TileRec& T, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    const bool ub = a.use_blend != 0;
    constexpr int PS = BXG * BYG;
    const unsigned short* col[C][4];
    float fx[C][4], fy[C][4], wxy[C][4], prev[C][4], fz[C], oz[C];
    int zb[C];
    const ViewItem* dd[C];
#pragma unroll
    for (int v = 0; v < C; ++v) {
        const int s = (T.it0 + v) % NST_G;
        const ViewItem& d = descs[s];
        dd[v] = &d;
        const unsigned short* box = reinterpret_cast<const unsigned short*>(slots + (size_t)s * SLOT_G);
        oz[v] = d.o[2];
        const float zf = floorf(oz[v]);
        fz[v] = oz[v] - zf;
        zb[v] = (int)zf;
        const float b0x = (float)d.b0[0], b0y = (float)d.b0[1];
        const int p0 = min(max(zb[v], 0), BZG - 1) * PS;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float X = (float)(lx + 32 * (q & 1)), Y = (float)(ly + 8 * (q >> 1));
            float rx = fmaf(d.m[0], X, fmaf(d.m[1], Y, d.o[0]));
            float ry = fmaf(d.m[3], X, fmaf(d.m[4], Y, d.o[1]));
            const float wx = (d.flags & VI_PLAT_X) ? 1.f : blend_factor(rx + b0x, d.dm1[0], d.border[0], d.inv_range[0], ub);
            const float wy = (d.flags & VI_PLAT_Y) ? 1.f : blend_factor(ry + b0y, d.dm1[1], d.border[1], d.inv_range[1], ub);
            wxy[v][q] = wx * wy;
            rx = fminf(fmaxf(rx, 0.f), (float)(BXG - 2));     // masked columns (weight 0) stay inside the box
            ry = fminf(fmaxf(ry, 0.f), (float)(BYG - 2));
            const int x0 = (int)rx, y0 = (int)ry;
            fx[v][q] = rx - (float)x0;
            fy[v][q] = ry - (float)y0;
            col[v][q] = box + y0 * BXG + x0;
            const unsigned short* p = col[v][q] + p0;
            const float a00 = (float)p[0], a01 = (float)p[1], a10 = (float)p[BXG], a11 = (float)p[BXG + 1];
            const float c0 = a00 + fx[v][q] * (a01 - a00), c1 = a10 + fx[v][q] * (a11 - a10);
            prev[v][q] = c0 + fy[v][q] * (c1 - c0);
        }
    }
    OT* obase = reinterpret_cast<OT*>(T.out);
#pragma unroll 1
    for (int k = 0; k < T.nz; ++k) {
        float swi[4] = {0.f, 0.f, 0.f, 0.f}, sw[4] = {0.f, 0.f, 0.f, 0.f}, res[4];
#pragma unroll
        for (int v = 0; v < C; ++v) {
            const ViewItem& d = *dd[v];
            float wk = 1.f;
            if (!(d.flags & VI_PLAT_Z))
                wk = blend_factor((oz[v] + (float)k) + (float)d.b0[2], d.dm1[2], d.border[2], d.inv_range[2], ub);
            const int p1 = min(max(zb[v] + k + 1, 0), BZG - 1) * PS;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const unsigned short* p = col[v][q] + p1;
                const float a00 = (float)p[0], a01 = (float)p[1], a10 = (float)p[BXG], a11 = (float)p[BXG + 1];
                const float c0 = a00 + fx[v][q] * (a01 - a00), c1 = a10 + fx[v][q] * (a11 - a10);
                const float cur = c0 + fy[v][q] * (c1 - c0);
                const float val = prev[v][q] + fz[v] * (cur - prev[v][q]);
                prev[v][q] = cur;
                const float w = wxy[v][q] * wk;
                if (C == 1) {
                    res[q] = w > 0.f ? val : 0.f;
                } else {
                    swi[q] = swi[q] + w * val;
                    sw[q] = sw[q] + w;
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int x = lx + 32 * (q & 1), y = ly + 8 * (q >> 1);
            if (x < T.nx && y < T.ny)
                store1<OUT>(a, obase + (size_t)k * T.pitch_z + (size_t)y * T.pitch_y + x, C == 1 ? res[q] : wdiv(swi[q], sw[q]));
        }
    }
}

template <int OUT>
__device__ __forceinline__ void gen_tile(const FuseArgs2& a, const unsigned char* slots, const ViewItem* descs,
                                         const TileRec& T, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    const bool ub = a.use_blend != 0;
    const bool resident = T.mode == 1;
    const float xs[2] = {(float)lx, (float)(lx + 32)}, ys[2] = {(float)ly, (float)(ly + 8)};
    OT* obase = reinterpret_cast<OT*>(T.out);
#pragma unroll 1
    for (int k = 0; k < T.nz; ++k) {
        float swi[4] = {0.f, 0.f, 0.f, 0.f}, sw[4] = {0.f, 0.f, 0.f, 0.f};
        const float zk = (float)k;
#pragma unroll 1
        for (int v = 0; v < T.count; ++v) {
            const int s = (T.it0 + v) % NST_G;
            const ViewItem& d = resident ? descs[s] : T.items[v];
            const unsigned short* box = reinterpret_cast<const unsigned short*>(slots + (size_t)s * SLOT_G);
            const float m0 = d.m[0], m1 = d.m[1], m3 = d.m[3], m4 = d.m[4], m6 = d.m[6], m7 = d.m[7];
            const float bz0 = fmaf(d.m[2], zk, d.o[0]), bz1 = fmaf(d.m[5], zk, d.o[1]), bz2 = fmaf(d.m[8], zk, d.o[2]);
            const float b0x = (float)d.b0[0], b0y = (float)d.b0[1], b0z = (float)d.b0[2];
            const int flags = d.flags;
            const bool inside_all = (flags & VI_INSIDE) != 0;
            const bool plateau = (flags & (VI_PLAT_X | VI_PLAT_Y | VI_PLAT_Z)) == (VI_PLAT_X | VI_PLAT_Y | VI_PLAT_Z);
            const void* gdata = nullptr;
            int gdx = 0, gdy = 0, gdz = 0;
            float gox = 0.f, goy = 0.f, goz = 0.f;
            if (!resident) {
                const ViewDev& V = a.views[d.view];
                gdata = V.data; gdx = V.wdims[0]; gdy = V.wdims[1]; gdz = V.wdims[2];
                gox = (float)V.woff[0]; goy = (float)V.woff[1]; goz = (float)V.woff[2];
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float X = xs[q & 1], Y = ys[q >> 1];
                float rx = fmaf(m0, X, fmaf(m1, Y, bz0));
                float ry = fmaf(m3, X, fmaf(m4, Y, bz1));
                float rz = fmaf(m6, X, fmaf(m7, Y, bz2));
                float w = 1.f;
                bool ok = true;
                if (!inside_all || !plateau) {
                    const float ax = rx + b0x, ay = ry + b0y, az = rz + b0z;   // absolute source coordinate
                    if (!inside_all)
                        ok = ax >= 0.f && ax <= d.dm1[0] && ay >= 0.f && ay <= d.dm1[1] && az >= 0.f && az <= d.dm1[2];
                    if (ok && ub && !plateau) {
                        // per-axis plateau flags: a tile in a one-axis overlap zone evaluates one cosine, not three
                        if (!(flags & VI_PLAT_X)) ok = blend_axis(ax, d.dm1[0], d.border[0], d.inv_range[0], 0, nullptr, w);
                        if (ok && !(flags & VI_PLAT_Y)) ok = blend_axis(ay, d.dm1[1], d.border[1], d.inv_range[1], 0, nullptr, w);
                        if (ok && !(flags & VI_PLAT_Z)) ok = blend_axis(az, d.dm1[2], d.border[2], d.inv_range[2], 0, nullptr, w);
                    }
                    if (!inside_all) {   // keep the taps of masked voxels inside the staged box
                        rx = fminf(fmaxf(rx, 0.f), (float)(BXG - 2));
                        ry = fminf(fmaxf(ry, 0.f), (float)(BYG - 2));
                        rz = fminf(fmaxf(rz, 0.f), (float)(BZG - 2));
                    }
                }
                float val;
                if (resident) {
                    const int x0 = (int)rx, y0 = (int)ry, z0 = (int)rz;
                    const float tx = rx - (float)x0, ty = ry - (float)y0, tz = rz - (float)z0;
                    const unsigned short* p = box + (z0 * BYG + y0) * BXG + x0;
                    const float a000 = (float)p[0], a001 = (float)p[1], a010 = (float)p[BXG], a011 = (float)p[BXG + 1];
                    const float a100 = (float)p[BXG * BYG], a101 = (float)p[BXG * BYG + 1];
                    const float a110 = (float)p[BXG * BYG + BXG], a111 = (float)p[BXG * BYG + BXG + 1];
                    const float c00 = a000 + tx * (a001 - a000), c01 = a010 + tx * (a011 - a010);
                    const float c10 = a100 + tx * (a101 - a100), c11 = a110 + tx * (a111 - a110);
                    const float c0 = c00 + ty * (c01 - c00), c1 = c10 + ty * (c11 - c10);
                    val = c0 + tz * (c1 - c0);
                } else {
                    val = 0.f;
                    if (ok) val = gather8((const unsigned short*)gdata, gdx, gdy, gdz, rx + b0x - gox, ry + b0y - goy, rz + b0z - goz);
                }
                if (ok) {
                    swi[q] = swi[q] + w * val;
                    sw[q] = sw[q] + w;
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int x = lx + 32 * (q & 1), y = ly + 8 * (q >> 1);
            if (x < T.nx && y < T.ny) {
                const float res = wdiv(swi[q], sw[q]);
                store1<OUT>(a, obase + (size_t)k * T.pitch_z + (size_t)y * T.pitch_y + x, res);
            }
        }
    }
}

template <int OUT>
__device__ __forceinline__ void zero_tile(const FuseArgs2& a, const TileRec& T, int tid) {
    using OT = typename OutT<OUT>::type;
    const int lx = tid & 31, ly = tid >> 5;
    OT* obase = reinterpret_cast<OT*>(T.out);
    for (int k = 0; k < T.nz; ++k)
        for (int q = 0; q < 4; ++q) {
            const int x = lx + 32 * (q & 1), y = ly + 8 * (q >> 1);
            if (x < T.nx && y < T.ny) store1<OUT>(a, obase + (size_t)k * T.pitch_z + (size_t)y * T.pitch_y + x, 0.f);
        }
}

// ------------------------------------------------------------------------------------------ the kernel
extern __shared__ __align__(1024) unsigned char fuse2_smem[];

// Persistent: one CTA per SM; the producer warp draws work records (z-runs of one tile column) from a global
// counter and streams their tiles through the slot / tile-record rings without ever draining the pipeline;
// the two consumer teams take alternate tile records until each receives a terminator record.
template <bool GENERAL, int OUT, bool CONTENT = false>
__global__ void __launch_bounds__(NTHREADS, 1) fuse_tma_kernel(const __grid_constant__ FuseArgs2 a) {
    constexpr int NST = GENERAL ? NST_G : NST_T;
    constexpr int SLOT = GENERAL ? SLOT_G : SLOT_T;
    // NST boxes, 128-B aligned each (TMA destination)
    unsigned char* slots = fuse2_smem + ((128u - (smem_u32(fuse2_smem) & 127u)) & 127u);
    ViewItem* descs = reinterpret_cast<ViewItem*>(slots + (size_t)NST * SLOT);
    TileRec* recs = reinterpret_cast<TileRec*>(descs + NST);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(recs + NTR);
    unsigned long long* full = bars;                   // [NST]  producer -> consumers (TMA bytes + 1 arrive)
    unsigned long long* empty = bars + NST;            // [NST]  one team's 8 warps -> producer
    unsigned long long* tfull = bars + 2 * NST;        // [NTR]
    unsigned long long* tempty = bars + 2 * NST + NTR; // [NTR]
    float* wtab = reinterpret_cast<float*>(bars + 2 * NST + 2 * NTR);   // [NTEAMS][2][NST_T][WT_N]

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NTEAM / 32); }
        for (int i = 0; i < NTR; ++i) { mbar_init(&tfull[i], 1); mbar_init(&tempty[i], NTEAM / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wid == NCONS / 32) {
        // ---------------- producer warp: tile records + view items + TMA boxes, in ring order
        int it = 0, tseq = 0;
        unsigned long long fenced = 0ull;
        const size_t esz = OUT_DT(OUT) == BS_DTYPE_F32 ? 4 : (OUT_DT(OUT) == BS_DTYPE_U16 ? 2 : 1);
        for (;;) {
            int w = 0;
            if (lane == 0) w = atomicAdd(a.work_ctr, 1);
            w = __shfl_sync(0xffffffffu, w, 0);
            if (w >= a.nwork) break;
            const WorkRec W = a.work[w];
            const BlockDev& B = a.blocks[W.block];
            const int tile0 = B.tile_base + (W.tz0 * B.tiles[1] + W.ty) * B.tiles[0] + W.tx;
            const int tstride = B.tiles[0] * B.tiles[1];
            TileHdr myh = {0, 0, 0, 0};
            if (lane < W.ntz) myh = a.hdr[tile0 + lane * tstride];        // ntz <= 32 (host splits longer runs)
            for (int t = 0; t < W.ntz; ++t, ++tseq) {
                TileHdr h;
                h.first = __shfl_sync(0xffffffffu, myh.first, t);
                h.count = __shfl_sync(0xffffffffu, myh.count, t);
                h.mode = __shfl_sync(0xffffffffu, myh.mode, t);
                const int tz = W.tz0 + t;
                const int tr = tseq % NTR;
                mbar_wait(&tempty[tr], ((tseq / NTR) & 1) ^ 1);
                if (lane == 0) {
                    TileRec& R = recs[tr];
                    const size_t off = ((size_t)tz * TT_Z * B.size[1] + (size_t)W.ty * TT_Y) * B.size[0] + (size_t)W.tx * TT_X;
                    R.out = (unsigned long long)B.out + off * esz;
                    R.pitch_y = B.size[0];
                    R.pitch_z = (long long)B.size[0] * B.size[1];
                    R.nx = min(TT_X, B.size[0] - W.tx * TT_X);
                    R.ny = min(TT_Y, B.size[1] - W.ty * TT_Y);
                    R.nz = min(TT_Z, B.size[2] - tz * TT_Z);
                    R.count = h.count;
                    R.mode = h.mode;
                    R.it0 = it;
                    R.last = 0;
                    R.items = a.pool + h.first;
                }
                if (h.mode == 1) {
                    for (int e = 0; e < h.count; ++e, ++it) {
                        const int s = it % NST;
                        mbar_wait(&empty[s], ((it / NST) & 1) ^ 1);
                        const unsigned int* src = reinterpret_cast<const unsigned int*>(a.pool + h.first + e);
                        unsigned int* dst = reinterpret_cast<unsigned int*>(descs + s);
                        if (lane < VI_WORDS) dst[lane] = __ldg(src + lane);
                        __syncwarp();
                        if (lane == 0) {
                            const ViewItem& d = descs[s];
                            const ViewDev& V = a.views[d.view];
                            const CUtensorMap* tm = GENERAL ? V.tm_g : V.tm_t;
                            const bool known = d.view < 64 && ((fenced >> d.view) & 1ull);
                            if (!known) {
                                tmap_acquire(tm);
                                if (d.view < 64) fenced |= 1ull << d.view;
                            }
                            mbar_expect_tx(&full[s], (GENERAL ? BXG * BYG * BZG : BXT * BYT * BZT) * 2);
                            tma_load_box(slots + (size_t)s * SLOT, tm, d.tma[0], d.tma[1], d.tma[2], &full[s]);
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&tfull[tr]);
            }
        }
        // one terminator record per team (consecutive sequence numbers cover both parities)
        for (int g = 0; g < NTEAMS; ++g, ++tseq) {
            const int tr = tseq % NTR;
            mbar_wait(&tempty[tr], ((tseq / NTR) & 1) ^ 1);
            if (lane == 0) {
                recs[tr].mode = -1;
                recs[tr].count = 0;
                mbar_arrive(&tfull[tr]);
            }
            __syncwarp();
        }
        return;
    }

    // ---------------- consumer teams: team g renders tile records g, g + 2, ...
    const int team = tid / NTEAM, ttid = tid % NTEAM;
    float* wt = wtab + team * (2 * NST_T * WT_N);
    int uses = 0;
    for (int n = team;; n += NTEAMS) {
        const int tr = n % NTR;
        mbar_wait(&tfull[tr], (n / NTR) & 1);
        const TileRec T = recs[tr];
        if (T.mode < 0) break;
        if (T.mode == 1) {
            for (int v = 0; v < T.count; ++v) {
                const int it = T.it0 + v;
                mbar_wait(&full[it % NST], (it / NST) & 1);
            }
        }
        if (T.mode == 0) {
            zero_tile<OUT>(a, T, ttid);
        } else if (GENERAL) {
            if (a.xyaff && T.mode == 1 && T.count == 1) xy_tile<1, OUT>(a, slots, descs, T, ttid);
            else if (a.xyaff && T.mode == 1 && T.count == 2) xy_tile<2, OUT>(a, slots, descs, T, ttid);
            else gen_tile<OUT>(a, slots, descs, T, ttid);
        } else if (T.mode == 1) {
            if (CONTENT) {
                // content weights ride along from global memory; register state for <= 2 views, rolled beyond
                switch (T.count) {
                    case 1: tr_tile<1, OUT, false, true>(a, slots, descs, T, wt, uses, team, ttid); break;
                    case 2: tr_tile<2, OUT, false, true>(a, slots, descs, T, wt, uses, team, ttid); break;
                    default: tr_tile_many<OUT, true>(a, slots, descs, T, wt, uses, team, ttid); break;
                }
            } else {
                switch (T.count) {
                    case 1:
                        if ((descs[T.it0 % NST].flags & (VI_PLAT_X | VI_PLAT_Y | VI_PLAT_Z)) == (VI_PLAT_X | VI_PLAT_Y | VI_PLAT_Z))
                            tr_tile<1, OUT, true>(a, slots, descs, T, wt, uses, team, ttid);
                        else
                            tr_tile<1, OUT>(a, slots, descs, T, wt, uses, team, ttid);
                        break;
                    case 2: tr_tile<2, OUT>(a, slots, descs, T, wt, uses, team, ttid); break;
                    case 3: tr_tile<3, OUT>(a, slots, descs, T, wt, uses, team, ttid); break;
                    case 4: tr_tile<4, OUT>(a, slots, descs, T, wt, uses, team, ttid); break;
                    default: tr_tile_many<OUT>(a, slots, descs, T, wt, uses, team, ttid); break;
                }
            }
        } else {
            tr_slow_tile<OUT, CONTENT>(a, T, ttid);
        }
        __syncwarp();
        if (lane == 0) {
            if (T.mode == 1)
                for (int v = 0; v < T.count; ++v) mbar_arrive(&empty[(T.it0 + v) % NST]);
            mbar_arrive(&tempty[tr]);
        }
    }
}

}  // namespace

// ==========================================================================================
// host side
// ==========================================================================================
PFN_cuTensorMapEncodeTiled_v12000 bs_tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
    }
    return fn;
}

namespace {

// the two tensor maps of a uint16 volume (translation box, general box), copied once to device memory
bool ensure_tmaps(bs_ctx* ctx, bs_volume& vol) {
    if (vol.tma_state != 0) return vol.tma_state > 0;
    vol.tma_state = -1;
    if (vol.dtype != BS_DTYPE_U16 || (vol.dims[0] & 7) != 0 || ((size_t)vol.dev & 15) != 0) return false;
    auto enc = bs_tensor_map_encoder();
    if (!enc) return false;
    alignas(64) CUtensorMap tm[2];
    const cuuint64_t gdim[3] = {(cuuint64_t)vol.dims[0], (cuuint64_t)vol.dims[1], (cuuint64_t)vol.dims[2]};
    const cuuint64_t gstr[2] = {(cuuint64_t)vol.dims[0] * 2, (cuuint64_t)vol.dims[0] * vol.dims[1] * 2};
    const cuuint32_t estr[3] = {1, 1, 1};
    const cuuint32_t boxes[2][3] = {{BXT, BYT, BZT}, {BXG, BYG, BZG}};
    for (int i = 0; i < 2; ++i) {
        CUresult r = enc(&tm[i], CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, vol.dev, gdim, gstr, boxes[i], estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return false;
    }
    void* d = nullptr;
    if (cudaMalloc(&d, sizeof(tm)) != cudaSuccess) return false;
    if (cudaMemcpyAsync(d, tm, sizeof(tm), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) {   // tm is a stack object
        cudaFree(d);
        return false;
    }
    vol.tmaps_dev = d;
    vol.tma_state = 1;
    return true;
}

struct Fuse2Ws {
    static constexpr int kRing = 4;
    void* meta_host[kRing] = {};      // pinned staging of one call's tables
    size_t meta_host_cap[kRing] = {};
    cudaEvent_t meta_ev[kRing] = {};
    bool meta_used[kRing] = {};
    int next = 0;
    void* meta_dev = nullptr; size_t meta_dev_cap = 0;
    void* hdr = nullptr; size_t hdr_cap = 0;
    void* pool = nullptr; size_t pool_cap = 0;
    int* ctr = nullptr;
    void* stage[2] = {nullptr, nullptr};   // device staging of host outputs
    size_t stage_cap[2] = {0, 0};
    cudaEvent_t stage_done[2] = {};        // D2H of the staging buffer finished
    cudaEvent_t stage_ready[2] = {};       // kernel that filled it finished
    bool attr_done = false;
};

Fuse2Ws* ws_of(bs_ctx* ctx) {
    if (!ctx->fuse2) ctx->fuse2 = new Fuse2Ws();
    return (Fuse2Ws*)ctx->fuse2;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

template <bool GENERAL, bool CONTENT = false>
void launch_kernel(int out_dtype, bool big_endian, int grid, size_t smem, cudaStream_t s, const FuseArgs2& a) {
    if (out_dtype == BS_DTYPE_F32) {
        if (big_endian) fuse_tma_kernel<GENERAL, BS_DTYPE_F32 | OUT_BE, CONTENT><<<grid, NTHREADS, smem, s>>>(a);
        else fuse_tma_kernel<GENERAL, BS_DTYPE_F32, CONTENT><<<grid, NTHREADS, smem, s>>>(a);
    } else if (out_dtype == BS_DTYPE_U16) {
        if (big_endian) fuse_tma_kernel<GENERAL, BS_DTYPE_U16 | OUT_BE, CONTENT><<<grid, NTHREADS, smem, s>>>(a);
        else fuse_tma_kernel<GENERAL, BS_DTYPE_U16, CONTENT><<<grid, NTHREADS, smem, s>>>(a);
    } else {
        fuse_tma_kernel<GENERAL, BS_DTYPE_U8, CONTENT><<<grid, NTHREADS, smem, s>>>(a);
    }
}

constexpr size_t smem_bytes(bool general) {
    return (size_t)(general ? NST_G * SLOT_G : NST_T * SLOT_T) + (size_t)(general ? NST_G : NST_T) * sizeof(ViewItem) +
           NTR * sizeof(TileRec) + (2 * (general ? NST_G : NST_T) + 2 * NTR) * 8 +
           (size_t)NTEAMS * 2 * NST_T * WT_N * sizeof(float) + 1024;
}

bool eligible(bs_ctx* ctx, const bs_view* views, int n_views, const bs_fuse_params* p) {
    const char* e = getenv("BS_FUSE_LEGACY");
    if (e && *e && *e != '0') return false;
    const bool content = p->fusion_type == BS_FUSE_AVG_CONTENT || p->fusion_type == BS_FUSE_AVG_BLEND_CONTENT;
    if (!(p->fusion_type == BS_FUSE_AVG || p->fusion_type == BS_FUSE_AVG_BLEND || content)) return false;
    if (p->interpolation != 1 || p->blend_lut_n != 0) return false;
    for (int i = 0; i < n_views; ++i) {
        auto it = ctx->vols.find(views[i].vol_handle);
        if (it == ctx->vols.end()) return false;   // the legacy path reports the error
        if (!ensure_tmaps(ctx, it->second)) return false;
        if (content) {
            // content weights ride along in the translation kernel only: whole (non-windowed) views, identity linear part
            auto ic = ctx->vols.find(views[i].content_handle);
            if (ic == ctx->vols.end() || ic->second.dtype != BS_DTYPE_F32 || ic->second.dims[0] != it->second.dims[0] ||
                ic->second.dims[1] != it->second.dims[1] || ic->second.dims[2] != it->second.dims[2] || views[i].full_dims[0] > 0)
                return false;
            double inv[12];
            if (!bs_invert34(views[i].src_to_world, inv)) return false;
            if (!(inv[0] == 1.0 && inv[1] == 0.0 && inv[2] == 0.0 && inv[4] == 0.0 && inv[5] == 1.0 && inv[6] == 0.0 &&
                  inv[8] == 0.0 && inv[9] == 0.0 && inv[10] == 1.0))
                return false;
        }
        for (int k = 0; k < 3; ++k)
            if (!(views[i].blend_range[k] > 0.f) && p->fusion_type == BS_FUSE_AVG_BLEND) return false;
    }
    return true;
}

// Fuse blocks [b0, b1) into device buffers outs[b].  ctx->mu held.
int fuse2_launch(bs_ctx* ctx, const bs_view* views, int n_views, int nb, const long long* bmin, const long long* bsize,
                 const bs_fuse_params* p, void* const* outs_dev) {
    Fuse2Ws* W = ws_of(ctx);
    // ---- per-view tables
    std::vector<ViewDev> hv((size_t)n_views);
    bool general = false, xyaff = true;
    for (int i = 0; i < n_views; ++i) {
        bs_volume& vol = ctx->vols.find(views[i].vol_handle)->second;
        { int rc = bs_volume_acquire(ctx, vol); if (rc) return rc; }
        ViewDev& d = hv[i];
        memset(&d, 0, sizeof(d));
        if (!bs_invert34(views[i].src_to_world, d.inv))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d has a singular transform", i);
        double* m = d.inv;
        if (!(m[0] == 1.0 && m[1] == 0.0 && m[2] == 0.0 && m[4] == 0.0 && m[5] == 1.0 && m[6] == 0.0 && m[8] == 0.0 &&
              m[9] == 0.0 && m[10] == 1.0))
            general = true;
        // xy-affine + z translation (rotation about z, xy scale / shear): no z coupling, unit z step
        const double tiny = 1e-13 * (std::fabs(m[0]) + std::fabs(m[1]) + std::fabs(m[4]) + std::fabs(m[5]) + 1.0);
        if (std::fabs(m[2]) <= tiny && std::fabs(m[6]) <= tiny && std::fabs(m[8]) <= tiny && std::fabs(m[9]) <= tiny &&
            std::fabs(m[10] - 1.0) <= 1e-12) {
            m[2] = m[6] = m[8] = m[9] = 0.0;     // round-off of the inversion: snap to the exact structure
            m[10] = 1.0;
        } else {
            xyaff = false;
        }
        d.data = vol.dev;
        d.content = nullptr;
        if (p->fusion_type == BS_FUSE_AVG_CONTENT || p->fusion_type == BS_FUSE_AVG_BLEND_CONTENT) {
            bs_volume& cv = ctx->vols.find(views[i].content_handle)->second;
            { int rc = bs_volume_acquire(ctx, cv); if (rc) return rc; }
            d.content = (const float*)cv.dev;
        }
        d.tm_t = (const CUtensorMap*)vol.tmaps_dev;
        d.tm_g = (const CUtensorMap*)vol.tmaps_dev + 1;
        const bool windowed = views[i].full_dims[0] > 0;
        for (int k = 0; k < 3; ++k) {
            d.wdims[k] = (int)vol.dims[k];
            d.woff[k] = windowed ? (int)views[i].window_min[k] : 0;
            d.dims[k] = windowed ? (int)views[i].full_dims[k] : (int)vol.dims[k];
            if (windowed && (views[i].window_min[k] < 0 || views[i].window_min[k] + vol.dims[k] > views[i].full_dims[k] ||
                             views[i].full_dims[k] > 0x7fffffffLL))
                return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: view %d: window [%lld, +%lld) outside full_dims %lld", i,
                                    views[i].window_min[k], vol.dims[k], views[i].full_dims[k]);
            d.border[k] = views[i].blend_border[k];
            d.range[k] = views[i].blend_range[k];
        }
        // world AABB of the source box [-eps, dim-1+eps]^3, expanded
        const double* f = views[i].src_to_world;
        for (int r = 0; r < 3; ++r) {
            double lo = f[4 * r + 3], hi = f[4 * r + 3], mag = 0.0;
            for (int c = 0; c < 3; ++c) {
                const double e = f[4 * r + c] * (double)(d.dims[c] - 1);
                lo += std::min(0.0, e);
                hi += std::max(0.0, e);
                mag += std::fabs(f[4 * r + c]);
            }
            const double pad = 4e-3 * mag + 1e-6 * std::max(std::fabs(lo), std::fabs(hi)) + 1e-3;
            d.wlo[r] = lo - pad;
            d.whi[r] = hi + pad;
        }
    }
    {
        const char* e = getenv("BS_FUSE_GENERAL");
        if (e && *e && *e != '0') general = true;
    }
    // ---- blocks, candidates, work records, pool bound
    std::vector<BlockDev> hb((size_t)nb);
    std::vector<int> cand;
    long long ntiles_total = 0, pool_need = 0;
    for (int b = 0; b < nb; ++b) {
        BlockDev& B = hb[b];
        memset(&B, 0, sizeof(B));
        for (int k = 0; k < 3; ++k) {
            B.bmin[k] = bmin[3 * b + k];
            B.size[k] = (int)bsize[3 * b + k];
        }
        B.tiles[0] = (B.size[0] + TT_X - 1) / TT_X;
        B.tiles[1] = (B.size[1] + TT_Y - 1) / TT_Y;
        B.tiles[2] = (B.size[2] + TT_Z - 1) / TT_Z;
        const long long nt = (long long)B.tiles[0] * B.tiles[1] * B.tiles[2];
        if (ntiles_total + nt > 0x3fffffffLL)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: too many tiles in one call");
        B.ntiles = (int)nt;
        B.tile_base = (int)ntiles_total;
        ntiles_total += nt;
        B.out = outs_dev[b];
        B.cand_off = (int)cand.size();
        const int T3[3] = {TT_X, TT_Y, TT_Z};
        for (int i = 0; i < n_views; ++i) {
            long long cnt = 1;
            for (int k = 0; k < 3 && cnt; ++k) {
                const double lo = hv[i].wlo[k] - (double)B.bmin[k], hi = hv[i].whi[k] - (double)B.bmin[k];
                if (hi < 0.0 || lo > (double)(B.size[k] - 1)) { cnt = 0; break; }
                const long long t0 = std::max(0LL, (long long)std::floor(lo / T3[k]) - 0);
                const long long t1 = std::min((long long)B.tiles[k] - 1, (long long)std::floor(hi / T3[k]));
                cnt *= std::max(0LL, t1 - t0 + 1);
            }
            if (cnt) { cand.push_back(i); pool_need += cnt; }
        }
        B.cand_n = (int)cand.size() - B.cand_off;
    }
    if (nb > 65535) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: at most 65535 blocks per call");
    if (pool_need > 0x7fffffffLL / 2) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: plan too large, fuse fewer blocks per call");
    // z-run length: enough CTAs for every SM, at most 32 tiles per CTA
    int L = (int)std::min<long long>(32, std::max<long long>(2, ntiles_total / ((long long)ctx->sm_count * 8)));
    std::vector<WorkRec> work;
    {
        int max_runs = 0;
        for (int b = 0; b < nb; ++b) max_runs = std::max(max_runs, (hb[b].tiles[2] + L - 1) / L);
        for (int r = 0; r < max_runs; ++r)
            for (int b = 0; b < nb; ++b) {
                const BlockDev& B = hb[b];
                const int tz0 = r * L;
                if (tz0 >= B.tiles[2]) continue;
                for (int ty = 0; ty < B.tiles[1]; ++ty)
                    for (int tx = 0; tx < B.tiles[0]; ++tx) {
                        WorkRec w;
                        memset(&w, 0, sizeof(w));
                        w.block = b; w.tx = tx; w.ty = ty; w.tz0 = tz0; w.ntz = std::min(L, B.tiles[2] - tz0);
                        work.push_back(w);
                    }
            }
    }
    // ---- stage the tables
    const size_t off_views = 0;
    const size_t off_blocks = align_up(off_views + hv.size() * sizeof(ViewDev), 64);
    const size_t off_cand = align_up(off_blocks + hb.size() * sizeof(BlockDev), 64);
    const size_t off_work = align_up(off_cand + cand.size() * sizeof(int), 64);
    const size_t meta_bytes = align_up(off_work + work.size() * sizeof(WorkRec), 64) + 64;
    const int slot = W->next;
    W->next = (slot + 1) % Fuse2Ws::kRing;
    if (!W->meta_ev[slot]) BS_CUDA(ctx, cudaEventCreateWithFlags(&W->meta_ev[slot], cudaEventDisableTiming));
    if (W->meta_used[slot]) BS_CUDA(ctx, cudaEventSynchronize(W->meta_ev[slot]));
    if (W->meta_host_cap[slot] < meta_bytes) {
        if (W->meta_host[slot]) cudaFreeHost(W->meta_host[slot]);
        W->meta_host[slot] = nullptr;
        W->meta_host_cap[slot] = 0;
        const size_t cap = align_up(meta_bytes * 2, 1 << 16);
        BS_CUDA(ctx, cudaHostAlloc(&W->meta_host[slot], cap, cudaHostAllocMapped));
        W->meta_host_cap[slot] = cap;
    }
    int rc = bs_ensure_dev(ctx, &W->meta_dev, &W->meta_dev_cap, align_up(meta_bytes * 2, 1 << 16));
    if (rc) return rc;
    rc = bs_ensure_dev(ctx, &W->hdr, &W->hdr_cap, align_up((size_t)ntiles_total * sizeof(TileHdr) * 5 / 4, 1 << 16));
    if (rc) return rc;
    rc = bs_ensure_dev(ctx, &W->pool, &W->pool_cap, align_up((size_t)std::max<long long>(pool_need, 1) * sizeof(ViewItem) * 5 / 4, 1 << 16));
    if (rc) return rc;
    if (!W->ctr) BS_CUDA(ctx, cudaMalloc((void**)&W->ctr, 64));
    unsigned char* mh = (unsigned char*)W->meta_host[slot];
    if (!hv.empty()) memcpy(mh + off_views, hv.data(), hv.size() * sizeof(ViewDev));
    memcpy(mh + off_blocks, hb.data(), hb.size() * sizeof(BlockDev));
    if (!cand.empty()) memcpy(mh + off_cand, cand.data(), cand.size() * sizeof(int));
    memcpy(mh + off_work, work.data(), work.size() * sizeof(WorkRec));
    {
        void* mh_dev = nullptr;
        BS_CUDA(ctx, cudaHostGetDevicePointer(&mh_dev, mh, 0));
        const int n16 = (int)((meta_bytes + 15) / 16);
        bs_launch_scope scope(ctx, "fuse_meta");
        fuse_meta_copy_kernel<<<std::min(64, (n16 + 255) / 256), 256, 0, ctx->stream>>>((uint4*)W->meta_dev, (const uint4*)mh_dev, n16);
    }
    BS_CUDA(ctx, cudaGetLastError());
    BS_CUDA(ctx, cudaEventRecord(W->meta_ev[slot], ctx->stream));
    W->meta_used[slot] = true;
    BS_CUDA(ctx, cudaMemsetAsync(W->ctr, 0, 64, ctx->stream));

    const unsigned char* md = (const unsigned char*)W->meta_dev;
    const ViewDev* dviews = (const ViewDev*)(md + off_views);
    const BlockDev* dblocks = (const BlockDev*)(md + off_blocks);
    const int use_blend = (p->fusion_type == BS_FUSE_AVG_BLEND || p->fusion_type == BS_FUSE_AVG_BLEND_CONTENT) ? 1 : 0;
    const bool content = p->fusion_type == BS_FUSE_AVG_CONTENT || p->fusion_type == BS_FUSE_AVG_BLEND_CONTENT;
    int max_tiles = 0;
    for (int b = 0; b < nb; ++b) max_tiles = std::max(max_tiles, hb[b].ntiles);
    {
        bs_launch_scope scope(ctx, "fuse_plan");
        dim3 grid((max_tiles + 127) / 128, nb);
        fuse_plan2_kernel<<<grid, 128, 0, ctx->stream>>>(dviews, dblocks, (const int*)(md + off_cand), (TileHdr*)W->hdr,
                                                         (ViewItem*)W->pool, W->ctr, (int)pool_need, use_blend,
                                                         general ? 1 : 0, general ? NST_G : NST_T);
    }
    BS_CUDA(ctx, cudaGetLastError());
    if (!W->attr_done) {
        const int st = (int)smem_bytes(false), sg = (int)smem_bytes(true);
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U16>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U8>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_F32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<true, BS_DTYPE_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, sg));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<true, BS_DTYPE_U16>, cudaFuncAttributeMaxDynamicSharedMemorySize, sg));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<true, BS_DTYPE_U8>, cudaFuncAttributeMaxDynamicSharedMemorySize, sg));
        // big-endian instantiations (the same kernels with a byte swap in the store)
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_F32 | OUT_BE>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U16 | OUT_BE>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_F32 | OUT_BE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<false, BS_DTYPE_U16 | OUT_BE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, st));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<true, BS_DTYPE_F32 | OUT_BE>, cudaFuncAttributeMaxDynamicSharedMemorySize, sg));
        BS_CUDA(ctx, cudaFuncSetAttribute(fuse_tma_kernel<true, BS_DTYPE_U16 | OUT_BE>, cudaFuncAttributeMaxDynamicSharedMemorySize, sg));
        W->attr_done = true;
    }
    FuseArgs2 a;
    memset(&a, 0, sizeof(a));
    a.views = dviews;
    a.blocks = dblocks;
    a.work = (const WorkRec*)(md + off_work);
    a.hdr = (const TileHdr*)W->hdr;
    a.pool = (const ViewItem*)W->pool;
    a.use_blend = use_blend;
    {
        const char* e = getenv("BS_FUSE_NO_XYAFF");
        a.xyaff = (xyaff && !(e && *e && *e != '0')) ? 1 : 0;
    }
    a.work_ctr = W->ctr + 2;
    a.nwork = (int)work.size();
    a.ctop = p->out_dtype == BS_DTYPE_U8 ? 255.0 : 65535.0;
    a.cmin = p->min_intensity;
    a.cscale = p->out_dtype == BS_DTYPE_F32 ? 1.0 : a.ctop / (p->max_intensity - p->min_intensity);
    {
        bs_launch_scope scope(ctx, "fuse");
        const int grid = (int)std::min<size_t>(work.size(), (size_t)ctx->sm_count);
        const bool be = p->out_big_endian != 0;
        if (general) launch_kernel<true>(p->out_dtype, be, grid, smem_bytes(true), ctx->stream, a);
        else if (content) launch_kernel<false, true>(p->out_dtype, be, grid, smem_bytes(false), ctx->stream, a);
        else launch_kernel<false>(p->out_dtype, be, grid, smem_bytes(false), ctx->stream, a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    {
        const char* e = getenv("BS_FUSE_CHECK");
        if (e && *e && *e != '0') {
            int h[2] = {0, 0};
            BS_CUDA(ctx, cudaMemcpyAsync(h, W->ctr, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
            BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            if (h[1] || h[0] > pool_need)
                return bs_set_error(ctx, BS_ERR_CUDA, "bs_fuse: plan pool overflow (%d items, bound %lld)", h[0], pool_need);
        }
    }
    return BS_OK;
}

__global__ void fuse_bswap_kernel(void* data, size_t n, int es) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if (es == 4) ((unsigned int*)data)[i] = bswap32(((unsigned int*)data)[i]);
        else ((unsigned short*)data)[i] = (unsigned short)bswap16x2(((unsigned short*)data)[i]);
    }
}

int validate_blocks(bs_ctx* ctx, int nb, const long long* bmin, const long long* bsize, const bs_fuse_params* p) {
    if (!bmin || !bsize || !p) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: NULL argument");
    if (nb < 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: n_blocks < 0");
    for (int b = 0; b < nb; ++b)
        for (int d = 0; d < 3; ++d)
            if (bsize[3 * b + d] <= 0 || bsize[3 * b + d] > 0x7fffffffLL)
                return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse: bad block_size[%d]=%lld", d, bsize[3 * b + d]);
    return BS_OK;
}

// device outputs; chooses the TMA kernels or the generic tile kernel
int fuse_blocks_dev(bs_ctx* ctx, const bs_view* views, int n_views, int nb, const long long* bmin, const long long* bsize,
                    const bs_fuse_params* p, void* const* outs_dev) {
    int rc = bs_fuse_validate(ctx, views, n_views, p);
    if (rc) return rc;
    if (nb == 0) return BS_OK;
    if (eligible(ctx, views, n_views, p)) return fuse2_launch(ctx, views, n_views, nb, bmin, bsize, p, outs_dev);
    const size_t es = bs_out_elem_size(p->out_dtype);
    for (int b = 0; b < nb; ++b) {
        rc = bs_fuse_legacy_block(ctx, views, n_views, bmin + 3 * b, bsize + 3 * b, p, outs_dev[b]);
        if (rc) return rc;
        if (p->out_big_endian && es > 1) {   // the generic tile kernel stores native order: swap in place
            const size_t n = (size_t)bsize[3 * b] * bsize[3 * b + 1] * bsize[3 * b + 2];
            bs_launch_scope scope(ctx, "fuse_bswap");
            fuse_bswap_kernel<<<(unsigned int)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 16), 256, 0, ctx->stream>>>(outs_dev[b], n, (int)es);
            BS_CUDA(ctx, cudaGetLastError());
        }
    }
    return BS_OK;
}

}  // namespace

void bs_fuse2_free(bs_ctx* ctx) {
    Fuse2Ws* W = (Fuse2Ws*)ctx->fuse2;
    if (!W) return;
    for (int i = 0; i < Fuse2Ws::kRing; ++i) {
        if (W->meta_host[i]) cudaFreeHost(W->meta_host[i]);
        if (W->meta_ev[i]) cudaEventDestroy(W->meta_ev[i]);
    }
    if (W->meta_dev) cudaFree(W->meta_dev);
    if (W->hdr) cudaFree(W->hdr);
    if (W->pool) cudaFree(W->pool);
    if (W->ctr) cudaFree(W->ctr);
    for (int i = 0; i < 2; ++i) {
        if (W->stage[i]) cudaFree(W->stage[i]);
        if (W->stage_done[i]) cudaEventDestroy(W->stage_done[i]);
        if (W->stage_ready[i]) cudaEventDestroy(W->stage_ready[i]);
    }
    delete W;
    ctx->fuse2 = nullptr;
}

extern "C" {

int bs_fuse_blocks(bs_ctx* ctx, const bs_view* views, int n_views, int n_blocks, const long long* block_min,
                   const long long* block_size, const bs_fuse_params* params, void* const* outs, int out_on_device) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    int rc = validate_blocks(ctx, n_blocks, block_min, block_size, params);
    if (rc) return rc;
    if (n_blocks > 0 && !outs) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: outs is NULL");
    for (int b = 0; b < n_blocks; ++b)
        if (!outs[b]) return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_blocks: outs[%d] is NULL", b);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    if (out_on_device) return fuse_blocks_dev(ctx, views, n_views, n_blocks, block_min, block_size, params, outs);

    // host destinations: blocks are fused in groups into one of two device staging buffers; the D2H copies of
    // a group run on the D2H stream while the next group is being fused
    Fuse2Ws* W = ws_of(ctx);
    const size_t es = bs_out_elem_size(params->out_dtype);
    const size_t group_cap = (size_t)256 << 20;
    for (int i = 0; i < 2; ++i) {
        if (!W->stage_done[i]) BS_CUDA(ctx, cudaEventCreateWithFlags(&W->stage_done[i], cudaEventDisableTiming));
        if (!W->stage_ready[i]) BS_CUDA(ctx, cudaEventCreateWithFlags(&W->stage_ready[i], cudaEventDisableTiming));
    }
    int b0 = 0, g = 0;
    bool used[2] = {false, false};
    std::vector<void*> douts;
    while (b0 < n_blocks) {
        size_t bytes = 0;
        int b1 = b0;
        std::vector<size_t> offs;
        while (b1 < n_blocks) {
            const size_t nbytes = align_up((size_t)block_size[3 * b1] * block_size[3 * b1 + 1] * block_size[3 * b1 + 2] * es, 256);
            if (b1 > b0 && bytes + nbytes > group_cap) break;
            offs.push_back(bytes);
            bytes += nbytes;
            ++b1;
        }
        const int sb = g & 1;
        if (used[sb]) BS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, W->stage_done[sb], 0));
        if (W->stage_cap[sb] < bytes) {
            // growing a staging buffer: everything in flight on it must be finished
            BS_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
            rc = bs_ensure_dev(ctx, &W->stage[sb], &W->stage_cap[sb], bytes);
            if (rc) return rc;
        }
        douts.resize((size_t)(b1 - b0));
        for (int b = b0; b < b1; ++b) douts[(size_t)(b - b0)] = (unsigned char*)W->stage[sb] + offs[(size_t)(b - b0)];
        rc = fuse_blocks_dev(ctx, views, n_views, b1 - b0, block_min + 3 * b0, block_size + 3 * b0, params, douts.data());
        if (rc) return rc;
        BS_CUDA(ctx, cudaEventRecord(W->stage_ready[sb], ctx->stream));
        BS_CUDA(ctx, cudaStreamWaitEvent(ctx->d2h_stream, W->stage_ready[sb], 0));
        for (int b = b0; b < b1; ++b) {
            const size_t nbytes = (size_t)block_size[3 * b] * block_size[3 * b + 1] * block_size[3 * b + 2] * es;
            BS_CUDA(ctx, cudaMemcpyAsync(outs[b], douts[(size_t)(b - b0)], nbytes, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        }
        BS_CUDA(ctx, cudaEventRecord(W->stage_done[sb], ctx->d2h_stream));
        used[sb] = true;
        b0 = b1;
        ++g;
    }
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

int bs_fuse_block(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                  const long long block_size[3], const bs_fuse_params* params, void* out, int out_on_device) {
    if (!ctx) return BS_ERR_ARG;
    if (!out) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_block: out is NULL");
    }
    void* outs[1] = {out};
    return bs_fuse_blocks(ctx, views, n_views, 1, block_min, block_size, params, outs, out_on_device);
}

int bs_fuse_block_to_volume(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                            const long long block_size[3], const bs_fuse_params* params, unsigned long long* out_handle) {
    if (!ctx) return BS_ERR_ARG;
    if (!out_handle || !block_size || !params) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_block_to_volume: NULL argument");
    }
    void* dev = nullptr;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (int d = 0; d < 3; ++d)
            if (block_size[d] <= 0 || block_size[d] > 0x7fffffffLL)
                return bs_set_error(ctx, BS_ERR_ARG, "bs_fuse_block_to_volume: bad block_size");
        BS_CUDA(ctx, cudaSetDevice(ctx->device));
        BS_CUDA(ctx, cudaMalloc(&dev, (size_t)block_size[0] * block_size[1] * block_size[2] * bs_out_elem_size(params->out_dtype)));
    }
    int rc = bs_fuse_block(ctx, views, n_views, block_min, block_size, params, dev, 1);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (rc != BS_OK) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(dev);
        return rc;
    }
    bs_volume v;
    v.dev = dev;
    v.dims[0] = block_size[0]; v.dims[1] = block_size[1]; v.dims[2] = block_size[2];
    v.dtype = params->out_dtype;
    v.owned = true;
    *out_handle = ctx->next_handle++;
    ctx->vols[*out_handle] = v;
    return BS_OK;
}

}  // extern "C"
