// nonrigid-fusion: moving-least-squares (MLS) control-point grids and non-rigid AVG_BLEND fusion of a list of
// super-blocks.  Replaces NonRigidTools.fuseVirtualInterpolatedNonRigid (J/SparkNonRigidFusion.java:387-401).
//
// k_mls_grid: one thread per control point of one view.  The view's (target, local) pairs are staged through shared
//   memory in tiles (n-body pattern: every point is read from HBM once per CTA and broadcast to all its threads); each
//   thread accumulates the 22 weighted moments relative to its control point in double, then solves the 3x3 normal
//   equations of the weighted affine fit (or falls back to the view's inverse registration).
// k_nonrigid_fuse: one CTA per 32 x 8 x 4 output tile; per view the control points the tile needs are staged in shared
//   memory (float, relative to the box's first point), every voxel interpolates its source coordinate trilinearly,
//   samples the view n-linearly, weights it with the cosine blending and accumulates; then the converter and the store.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "bs_internal.cuh"
#include "fuse_common.cuh"

namespace {

struct NrView {
    double inv[12];        // world -> full-view pixel: the fallback of the MLS fit
    const double* pts;     // n x {tx, ty, tz, lx, ly, lz}
    int n;
    int dtype;
    const void* data;      // resident volume (window), nullptr for the grid-only diagnostic
    int dims[3];           // size of the full view: inside test, blending
    int wdims[3];          // resident window [woff, woff + wdims)
    int woff[3];
    float border[3], inv_range[3];
};

struct NrBlock {
    long long bmin[3];
    int size[3];
    int gdims[3];
    int cpd[3];
};

constexpr int MLS_THREADS = 128;
constexpr int MLS_TILE = 128;              // points per shared-memory tile (6 KB)
constexpr int NR_TX = 32, NR_TY = 8, NR_TZ = 4;
// control points one tile can touch: (tile extent - 1) / cpd + 2 per axis, largest at cpd = 1
constexpr int NR_BOX = (NR_TX + 1) * (NR_TY + 1) * (NR_TZ + 1);

__global__ void __launch_bounds__(MLS_THREADS) k_mls_grid(const NrView* __restrict__ views, const NrBlock B,
                                                          double* __restrict__ grid) {
    __shared__ double s_p[MLS_TILE * 6];
    const NrView& v = views[blockIdx.y];
    const int gd0 = B.gdims[0], gd1 = B.gdims[1];
    const int ncp = gd0 * gd1 * B.gdims[2];
    const int i = blockIdx.x * MLS_THREADS + threadIdx.x;
    const int gx = i % gd0, gy = (i / gd0) % gd1, gz = i / (gd0 * gd1);
    const double x[3] = {(double)(B.bmin[0] + (long long)(gx - 1) * B.cpd[0]),
                         (double)(B.bmin[1] + (long long)(gy - 1) * B.cpd[1]),
                         (double)(B.bmin[2] + (long long)(gz - 1) * B.cpd[2])};
    const int n = v.n;
    double S0 = 0.0, Su[3] = {0.0, 0.0, 0.0}, Sl[3] = {0.0, 0.0, 0.0};
    double Suu[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // xx xy xz yy yz zz
    double Sul[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int hit = -1;
    if (n >= 4) {                           // CTA-uniform: every thread of the CTA works on the same view
        for (int base = 0; base < n; base += MLS_TILE) {
            const int m = min(MLS_TILE, n - base);
            __syncthreads();
            for (int k = threadIdx.x; k < m * 6; k += MLS_THREADS) s_p[k] = __ldg(v.pts + (size_t)base * 6 + k);
            __syncthreads();
#pragma unroll 2
            for (int j = 0; j < m; ++j) {
                const double* p = s_p + 6 * j;
                const double u0 = p[0] - x[0], u1 = p[1] - x[1], u2 = p[2] - x[2];
                const double d2 = fma(u0, u0, fma(u1, u1, u2 * u2));
                if (d2 == 0.0) {
                    if (hit < 0) hit = base + j;
                    continue;
                }
                const double w = 1.0 / d2;
                const double l0 = p[3], l1 = p[4], l2 = p[5];
                const double wu0 = w * u0, wu1 = w * u1, wu2 = w * u2;
                S0 += w;
                Su[0] += wu0; Su[1] += wu1; Su[2] += wu2;
                Sl[0] = fma(w, l0, Sl[0]); Sl[1] = fma(w, l1, Sl[1]); Sl[2] = fma(w, l2, Sl[2]);
                Suu[0] = fma(wu0, u0, Suu[0]); Suu[1] = fma(wu0, u1, Suu[1]); Suu[2] = fma(wu0, u2, Suu[2]);
                Suu[3] = fma(wu1, u1, Suu[3]); Suu[4] = fma(wu1, u2, Suu[4]); Suu[5] = fma(wu2, u2, Suu[5]);
                Sul[0] = fma(wu0, l0, Sul[0]); Sul[1] = fma(wu0, l1, Sul[1]); Sul[2] = fma(wu0, l2, Sul[2]);
                Sul[3] = fma(wu1, l0, Sul[3]); Sul[4] = fma(wu1, l1, Sul[4]); Sul[5] = fma(wu1, l2, Sul[5]);
                Sul[6] = fma(wu2, l0, Sul[6]); Sul[7] = fma(wu2, l1, Sul[7]); Sul[8] = fma(wu2, l2, Sul[8]);
            }
        }
    }
    if (i >= ncp) return;
    double r[3];
    bool fallback = n < 4;
    if (!fallback && hit >= 0) {
        const double* l = v.pts + (size_t)hit * 6 + 3;
        r[0] = l[0]; r[1] = l[1]; r[2] = l[2];
    } else if (!fallback) {
        // centred moments: P = sum w (u - uc)(u - uc)^T, Q = sum w (u - uc)(l - lc)^T; the fit l = A (t - tc) + lc has
        // A = Q^T P^-1 and at the control point (u = 0) gives lc - Q^T P^-1 uc
        const double iS = 1.0 / S0;
        const double uc[3] = {Su[0] * iS, Su[1] * iS, Su[2] * iS};
        const double lc[3] = {Sl[0] * iS, Sl[1] * iS, Sl[2] * iS};
        const double a = Suu[0] - Su[0] * uc[0], b = Suu[1] - Su[0] * uc[1], c = Suu[2] - Su[0] * uc[2];
        const double d = Suu[3] - Su[1] * uc[1], e = Suu[4] - Su[1] * uc[2], f = Suu[5] - Su[2] * uc[2];
        // adjugate of the symmetric [[a b c] [b d e] [c e f]]
        const double A00 = d * f - e * e, A01 = c * e - b * f, A02 = b * e - c * d;
        const double A11 = a * f - c * c, A12 = b * c - a * e, A22 = a * d - b * b;
        const double det = a * A00 + b * A01 + c * A02;
        const double m = (a + d + f) * (1.0 / 3.0);
        if (!(det > 1e-10 * (m * m * m)) || !isfinite(det)) {
            fallback = true;
        } else {
            const double id = 1.0 / det;
            const double y0 = (A00 * uc[0] + A01 * uc[1] + A02 * uc[2]) * id;
            const double y1 = (A01 * uc[0] + A11 * uc[1] + A12 * uc[2]) * id;
            const double y2 = (A02 * uc[0] + A12 * uc[1] + A22 * uc[2]) * id;
            for (int k = 0; k < 3; ++k) {
                const double q0 = Sul[k] - Su[0] * lc[k], q1 = Sul[3 + k] - Su[1] * lc[k], q2 = Sul[6 + k] - Su[2] * lc[k];
                r[k] = lc[k] - (q0 * y0 + q1 * y1 + q2 * y2);
            }
        }
    }
    if (fallback)
        for (int k = 0; k < 3; ++k)
            r[k] = fma(v.inv[4 * k], x[0], fma(v.inv[4 * k + 1], x[1], fma(v.inv[4 * k + 2], x[2], v.inv[4 * k + 3])));
    double* o = grid + ((size_t)blockIdx.y * ncp + i) * 3;
    o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
}

template <int OUT>
__global__ void __launch_bounds__(NR_TX* NR_TY) k_nonrigid_fuse(const NrView* __restrict__ views, int nviews, const NrBlock B,
                                                              const double* __restrict__ grid, void* out, double cmin,
                                                              double cscale, double ctop) {
    __shared__ float s_g[NR_BOX * 3];
    constexpr int NT = NR_TX * NR_TY;
    const int tid = threadIdx.y * NR_TX + threadIdx.x;
    const int o0[3] = {(int)blockIdx.x * NR_TX, (int)blockIdx.y * NR_TY, (int)blockIdx.z * NR_TZ};
    const int ext[3] = {min(NR_TX, B.size[0] - o0[0]), min(NR_TY, B.size[1] - o0[1]), min(NR_TZ, B.size[2] - o0[2])};
    const int x = o0[0] + threadIdx.x, y = o0[1] + threadIdx.y;
    const bool valid = x < B.size[0] && y < B.size[1];
    // the tile's box of control points: grid indices c0 .. c0 + nb - 1 per axis (voxel o lies in cell o / cpd + 1)
    int c0[3], nb[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        c0[d] = o0[d] / B.cpd[d] + 1;
        nb[d] = (o0[d] + ext[d] - 1) / B.cpd[d] + 2 - c0[d] + 1;
    }
    const int sy = 3 * nb[0], sz = 3 * nb[0] * nb[1];
    const int cx = x / B.cpd[0] + 1 - c0[0], cy = y / B.cpd[1] + 1 - c0[1];
    const float fx = (float)(x % B.cpd[0]) / (float)B.cpd[0], fy = (float)(y % B.cpd[1]) / (float)B.cpd[1];
    const int nbox = nb[0] * nb[1] * nb[2];
    const size_t ncp = (size_t)B.gdims[0] * B.gdims[1] * B.gdims[2];
    float swi[NR_TZ], sw[NR_TZ];
#pragma unroll
    for (int k = 0; k < NR_TZ; ++k) { swi[k] = 0.f; sw[k] = 0.f; }

    for (int vi = 0; vi < nviews; ++vi) {
        const NrView& V = views[vi];
        const double* G = grid + (size_t)vi * ncp * 3;
        const double* g0 = G + (((size_t)c0[2] * B.gdims[1] + c0[1]) * B.gdims[0] + c0[0]) * 3;
        const double org0 = __ldg(g0), org1 = __ldg(g0 + 1), org2 = __ldg(g0 + 2);
        __syncthreads();   // the previous view's box is no longer read
        for (int k = tid; k < nbox; k += NT) {
            const int bx = k % nb[0], by = (k / nb[0]) % nb[1], bz = k / (nb[0] * nb[1]);
            const double* g = G + (((size_t)(c0[2] + bz) * B.gdims[1] + (c0[1] + by)) * B.gdims[0] + (c0[0] + bx)) * 3;
            s_g[3 * k] = (float)(__ldg(g) - org0);
            s_g[3 * k + 1] = (float)(__ldg(g + 1) - org1);
            s_g[3 * k + 2] = (float)(__ldg(g + 2) - org2);
        }
        __syncthreads();
        if (!valid) continue;
        const float of[3] = {(float)org0, (float)org1, (float)org2};
        const float dm1x = (float)(V.dims[0] - 1), dm1y = (float)(V.dims[1] - 1), dm1z = (float)(V.dims[2] - 1);
#pragma unroll
        for (int k = 0; k < NR_TZ; ++k) {
            if (k >= ext[2]) break;
            const int z = o0[2] + k;
            const int cz = z / B.cpd[2] + 1 - c0[2];
            const float fz = (float)(z % B.cpd[2]) / (float)B.cpd[2];
            const float* p = s_g + 3 * ((cz * nb[1] + cy) * nb[0] + cx);
            float s[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float c00 = p[c] + fx * (p[c + 3] - p[c]);
                const float c01 = p[c + sy] + fx * (p[c + sy + 3] - p[c + sy]);
                const float c10 = p[c + sz] + fx * (p[c + sz + 3] - p[c + sz]);
                const float c11 = p[c + sz + sy] + fx * (p[c + sz + sy + 3] - p[c + sz + sy]);
                const float e0 = c00 + fy * (c01 - c00), e1 = c10 + fy * (c11 - c10);
                s[c] = of[c] + (e0 + fz * (e1 - e0));
            }
            const float w = blend_factor(s[0], dm1x, V.border[0], V.inv_range[0], true) *
                            blend_factor(s[1], dm1y, V.border[1], V.inv_range[1], true) *
                            blend_factor(s[2], dm1z, V.border[2], V.inv_range[2], true);
            if (!(w > 0.f)) continue;
            // window-relative taps, clamped to the window (border extension; the caller's window covers every tap)
            const float wx = fminf(fmaxf(s[0] - (float)V.woff[0], 0.f), (float)(V.wdims[0] - 1));
            const float wy = fminf(fmaxf(s[1] - (float)V.woff[1], 0.f), (float)(V.wdims[1] - 1));
            const float wz = fminf(fmaxf(s[2] - (float)V.woff[2], 0.f), (float)(V.wdims[2] - 1));
            const float val = sample_any<true>(V.data, V.dtype, V.wdims[0], V.wdims[1], V.wdims[2], wx, wy, wz);
            swi[k] += w * val;
            sw[k] += w;
        }
    }
    if (!valid) return;
    const size_t plane = (size_t)B.size[1] * B.size[0];
    size_t o = ((size_t)o0[2] * B.size[1] + y) * B.size[0] + x;
#pragma unroll
    for (int k = 0; k < NR_TZ; ++k, o += plane) {
        if (k >= ext[2]) break;
        bs_store_converted<OUT>(out, o, sw[k] > 0.f ? swi[k] / sw[k] : 0.f, cmin, cscale, ctop);
    }
}

struct NrWs {
    void* views = nullptr;  size_t views_cap = 0;
    void* pts = nullptr;    size_t pts_cap = 0;
    void* grid = nullptr;   size_t grid_cap = 0;
    void* out = nullptr;    size_t out_cap = 0;
};

NrWs* ws_of(bs_ctx* ctx) {
    if (!ctx->nonrigid) ctx->nonrigid = new NrWs();
    return (NrWs*)ctx->nonrigid;
}

int check_block(bs_ctx* ctx, const long long bmin[3], const long long bsize[3], const long long cpd[3], NrBlock& B) {
    for (int d = 0; d < 3; ++d) {
        if (cpd[d] < 1 || cpd[d] > 0x3fffffffLL)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: cp_distance[%d] = %lld must be >= 1", d, cpd[d]);
        if (bsize[d] <= 0 || bsize[d] > 0x3fffffffLL)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: bad block_size[%d] = %lld", d, bsize[d]);
        B.bmin[d] = bmin[d];
        B.size[d] = (int)bsize[d];
        B.cpd[d] = (int)cpd[d];
        B.gdims[d] = (int)((bsize[d] - 1 + cpd[d] - 1) / cpd[d]) + 3;
    }
    if ((long long)B.gdims[0] * B.gdims[1] * B.gdims[2] > 0x7fffffffLL / 4)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: control-point grid too large");
    return BS_OK;
}

// validates the views and uploads their table and points; with_volumes: resolve and acquire the resident volumes
int upload_views(bs_ctx* ctx, const bs_nonrigid_view* views, int n_views, bool with_volumes, const NrView** dviews) {
    NrWs* W = ws_of(ctx);
    std::vector<NrView> hv((size_t)n_views);
    size_t total = 0;
    for (int i = 0; i < n_views; ++i) {
        if (views[i].n_points < 0 || (views[i].n_points > 0 && (!views[i].target_world_xyz || !views[i].local_xyz)))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: view %d has bad points", i);
        total += (size_t)views[i].n_points;
    }
    std::vector<double> hp(std::max<size_t>(total, 1) * 6);
    std::vector<size_t> first((size_t)n_views);
    size_t at = 0;
    for (int i = 0; i < n_views; ++i) {
        const bs_view& bv = views[i].view;
        NrView& d = hv[(size_t)i];
        memset(&d, 0, sizeof(d));
        if (!bs_invert34(bv.src_to_world, d.inv))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: view %d has a singular transform", i);
        d.n = views[i].n_points;
        first[(size_t)i] = at;
        for (int k = 0; k < d.n; ++k)
            for (int c = 0; c < 3; ++c) {
                hp[(at + k) * 6 + c] = views[i].target_world_xyz[3 * k + c];
                hp[(at + k) * 6 + 3 + c] = views[i].local_xyz[3 * k + c];
            }
        at += (size_t)d.n;
        if (!with_volumes) continue;
        auto it = ctx->vols.find(bv.vol_handle);
        if (it == ctx->vols.end())
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: view %d has unknown vol_handle %llu", i, bv.vol_handle);
        bs_volume& vol = it->second;
        { int rc = bs_volume_acquire(ctx, vol); if (rc) return rc; }
        const bool windowed = bv.full_dims[0] > 0;
        d.data = vol.dev;
        d.dtype = vol.dtype;
        for (int k = 0; k < 3; ++k) {
            d.wdims[k] = (int)vol.dims[k];
            d.woff[k] = windowed ? (int)bv.window_min[k] : 0;
            d.dims[k] = windowed ? (int)bv.full_dims[k] : (int)vol.dims[k];
            if (windowed && (bv.window_min[k] < 0 || bv.window_min[k] + vol.dims[k] > bv.full_dims[k] ||
                             bv.full_dims[k] > 0x7fffffffLL))
                return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: view %d: window [%lld, +%lld) outside full_dims %lld", i,
                                    bv.window_min[k], vol.dims[k], bv.full_dims[k]);
            d.border[k] = bv.blend_border[k];
            d.inv_range[k] = 1.0f / bv.blend_range[k];
        }
    }
    int rc = bs_ensure_dev(ctx, &W->pts, &W->pts_cap, hp.size() * sizeof(double));
    if (rc) return rc;
    rc = bs_ensure_dev(ctx, &W->views, &W->views_cap, std::max<size_t>(hv.size(), 1) * sizeof(NrView));
    if (rc) return rc;
    for (size_t i = 0; i < hv.size(); ++i) hv[i].pts = (const double*)W->pts + first[i] * 6;
    // pageable sources: both copies have consumed the host buffers when they return; stream order keeps the previous
    // call's kernels ahead of the overwrite
    BS_CUDA(ctx, cudaMemcpyAsync(W->pts, hp.data(), hp.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    if (!hv.empty())
        BS_CUDA(ctx, cudaMemcpyAsync(W->views, hv.data(), hv.size() * sizeof(NrView), cudaMemcpyHostToDevice, ctx->stream));
    *dviews = (const NrView*)W->views;
    return BS_OK;
}

int launch_grid(bs_ctx* ctx, const NrView* dviews, int n_views, const NrBlock& B, double** grid_out) {
    NrWs* W = ws_of(ctx);
    const size_t ncp = (size_t)B.gdims[0] * B.gdims[1] * B.gdims[2];
    int rc = bs_ensure_dev(ctx, &W->grid, &W->grid_cap, std::max<size_t>(ncp * n_views, 1) * 3 * sizeof(double));
    if (rc) return rc;
    *grid_out = (double*)W->grid;
    if (n_views == 0) return BS_OK;
    if (n_views > 65535) return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid: at most 65535 views per call");
    {
        bs_launch_scope scope(ctx, "mls_grid");
        k_mls_grid<<<dim3((unsigned)((ncp + MLS_THREADS - 1) / MLS_THREADS), (unsigned)n_views), MLS_THREADS, 0, ctx->stream>>>(
            dviews, B, (double*)W->grid);
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

template <int OUT>
void launch_fuse(dim3 g, cudaStream_t s, const NrView* v, int n, const NrBlock& B, const double* grid, void* out, double cmin,
                 double cscale, double ctop) {
    k_nonrigid_fuse<OUT><<<g, dim3(NR_TX, NR_TY), 0, s>>>(v, n, B, grid, out, cmin, cscale, ctop);
}

}  // namespace

void bs_nonrigid_free(bs_ctx* ctx) {
    NrWs* W = (NrWs*)ctx->nonrigid;
    if (!W) return;
    for (void* p : {W->views, W->pts, W->grid, W->out})
        if (p) cudaFree(p);
    delete W;
    ctx->nonrigid = nullptr;
}

extern "C" {

int bs_nonrigid_fuse_blocks(bs_ctx* ctx, const bs_nonrigid_view* views, int n_views, int n_blocks, const long long* block_min,
                            const long long* block_size, const long long cp_distance[3], const bs_fuse_params* p,
                            void* const* outs, int out_on_device) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!p || !cp_distance || n_views < 0 || n_blocks < 0 || (n_views > 0 && !views) ||
        (n_blocks > 0 && (!block_min || !block_size || !outs)))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: bad argument");
    if (p->fusion_type != BS_FUSE_AVG_BLEND)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: only AVG_BLEND fusion (got %d)", p->fusion_type);
    if (p->interpolation != 1)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: only n-linear interpolation (1)");
    if (p->out_dtype != BS_DTYPE_F32 && p->out_dtype != BS_DTYPE_U16 && p->out_dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: bad out_dtype %d", p->out_dtype);
    if (p->out_dtype != BS_DTYPE_F32 && !(p->max_intensity > p->min_intensity))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: max_intensity must exceed min_intensity");
    for (int d = 0; d < 3; ++d)
        if (cp_distance[d] < 1) return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: cp_distance must be >= 1");
    std::vector<NrBlock> blocks((size_t)n_blocks);
    for (int b = 0; b < n_blocks; ++b) {
        int rc = check_block(ctx, block_min + 3 * b, block_size + 3 * b, cp_distance, blocks[(size_t)b]);
        if (rc) return rc;
        if (!outs[b]) return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: outs[%d] is NULL", b);
        if ((blocks[(size_t)b].size[1] + NR_TY - 1) / NR_TY > 65535 || (blocks[(size_t)b].size[2] + NR_TZ - 1) / NR_TZ > 65535)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_fuse_blocks: block too large for one launch");
    }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    const NrView* dv = nullptr;
    int rc = upload_views(ctx, views, n_views, true, &dv);
    if (rc) return rc;
    NrWs* W = ws_of(ctx);
    const double ctop = p->out_dtype == BS_DTYPE_U8 ? 255.0 : 65535.0;
    const double cmin = p->min_intensity;
    const double cscale = p->out_dtype == BS_DTYPE_F32 ? 1.0 : ctop / (p->max_intensity - p->min_intensity);
    const size_t es = bs_out_elem_size(p->out_dtype);
    const bool be = p->out_big_endian != 0 && es > 1;
    for (int b = 0; b < n_blocks; ++b) {
        const NrBlock& B = blocks[(size_t)b];
        double* grid = nullptr;
        rc = launch_grid(ctx, dv, n_views, B, &grid);
        if (rc) return rc;
        const size_t bytes = (size_t)B.size[0] * B.size[1] * B.size[2] * es;
        void* dst = outs[b];
        if (!out_on_device) {
            rc = bs_ensure_dev(ctx, &W->out, &W->out_cap, bytes);
            if (rc) return rc;
            dst = W->out;
        }
        const dim3 g((B.size[0] + NR_TX - 1) / NR_TX, (B.size[1] + NR_TY - 1) / NR_TY, (B.size[2] + NR_TZ - 1) / NR_TZ);
        {
            bs_launch_scope scope(ctx, "nonrigid_fuse");
            if (p->out_dtype == BS_DTYPE_F32) {
                if (be) launch_fuse<BS_DTYPE_F32 | OUT_BE>(g, ctx->stream, dv, n_views, B, grid, dst, cmin, cscale, ctop);
                else launch_fuse<BS_DTYPE_F32>(g, ctx->stream, dv, n_views, B, grid, dst, cmin, cscale, ctop);
            } else if (p->out_dtype == BS_DTYPE_U16) {
                if (be) launch_fuse<BS_DTYPE_U16 | OUT_BE>(g, ctx->stream, dv, n_views, B, grid, dst, cmin, cscale, ctop);
                else launch_fuse<BS_DTYPE_U16>(g, ctx->stream, dv, n_views, B, grid, dst, cmin, cscale, ctop);
            } else {
                launch_fuse<BS_DTYPE_U8>(g, ctx->stream, dv, n_views, B, grid, dst, cmin, cscale, ctop);
            }
        }
        BS_CUDA(ctx, cudaGetLastError());
        if (!out_on_device) {
            BS_CUDA(ctx, cudaMemcpyAsync(outs[b], dst, bytes, cudaMemcpyDeviceToHost, ctx->stream));
            BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
    }
    return BS_OK;
}

int bs_nonrigid_debug_grid(bs_ctx* ctx, const bs_nonrigid_view* view, const long long block_min[3],
                           const long long block_size[3], const long long cp_distance[3], double* out, long long* grid_dims) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!view || !block_min || !block_size || !cp_distance || !grid_dims)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_nonrigid_debug_grid: NULL argument");
    NrBlock B;
    int rc = check_block(ctx, block_min, block_size, cp_distance, B);
    if (rc) return rc;
    for (int d = 0; d < 3; ++d) grid_dims[d] = B.gdims[d];
    if (!out) return BS_OK;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    const NrView* dv = nullptr;
    rc = upload_views(ctx, view, 1, false, &dv);
    if (rc) return rc;
    double* grid = nullptr;
    rc = launch_grid(ctx, dv, 1, B, &grid);
    if (rc) return rc;
    const size_t ncp = (size_t)B.gdims[0] * B.gdims[1] * B.gdims[2];
    BS_CUDA(ctx, cudaMemcpyAsync(out, grid, ncp * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

}  // extern "C"
