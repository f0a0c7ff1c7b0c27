// solver: the relaxation of TileConfiguration.optimize (J/Solver.java:352-395, mpicbg) over tiles joined by weighted
// point matches, in FP64 on the device.
//
// Every model here is linear, so a tile's fit needs only sums over its matches that factor into per-link moments and
// the partner's model: with p (own) and q (partner) shifted by the link's anchor o,
//   sum w p (M_u q)^T = Spq A_u^T + Sp (A_u o + t_u)^T,
// and W, Sp, Sq, Spp, Sqq, Spq are fixed for the whole solve.  k_link_moments takes them once (a segmented reduction over
// the matches, which arrive sorted by link); a fit then costs O(links of the tile), not O(matches).  The anchor keeps
// the second moments of world coordinates around 1e4 px from cancelling.
//
// k_solve is one persistent cooperative launch that runs every iteration without a host round trip:
//   1. per colour of the host's greedy colouring, one thread fits each tile of that colour (tiles of one colour share
//      no link, so this equals fitting them one after another), then a grid-wide sync;
//   2. one pass over every match, split into chunks of at most CHUNK matches of one link, one warp per chunk: the
//      distance |M_a p - M_b q| (models from shared memory when they fit), and per chunk sum w d and max d;
//   3. per tile, its links' chunk sums in a fixed order: tile error = sum w d / sum w;
//   4. every block takes E = mean tile error in the same fixed order, block 0 records it, and every block evaluates
//      the stopping rule on the same values, so all blocks leave the loop together.
// No floating-point atomics: two runs are bit-identical.  The only atomic counts skipped fits (integer).
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "bs_internal.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int SOLVE_THREADS = 256;
constexpr int MOM_THREADS = 128;
constexpr int CHUNK = 512;                       // matches per warp task of the distance pass
constexpr int MOM = 32;                          // doubles per link moment record
constexpr size_t SMEM_MODELS_MAX = 96 * 1024;    // models are staged in shared memory up to this size (1024 tiles)

// link moment record: W, n, o[3], Sp[3], Sq[3], Spp[6], Sqq[6], Spq[9] (row-major sum p_i q_j); symmetric 3 x 3 as
// xx, xy, xz, yy, yz, zz
enum { M_W = 0, M_N = 1, M_O = 2, M_SP = 5, M_SQ = 8, M_SPP = 11, M_SQQ = 17, M_SPQ = 23 };

__host__ __device__ constexpr int sym(int i, int j) {
    return i <= j ? (i == 0 ? j : (i == 1 ? 2 + j : 5)) : sym(j, i);
}

struct SolveArgs {
    int n_tiles, n_colours, n_links, n_chunks;
    const int* colour_offsets;
    const int* colour_tiles;
    const int* fixed;
    const int* links;             // 2 per link
    const int* tile_ptr;          // n_tiles + 1
    const int* tile_adj;          // link * 2 + side (side 0: the tile is the link's first tile)
    const int* chunk_link;
    const long long* chunk_begin;
    const long long* match_offsets;
    const int* link_chunk_ptr;    // n_links + 1
    const double* p;
    const double* q;
    const double* w;
    const double* mom;            // MOM per link
    double* models;               // 12 per tile
    double* chunk_swd;
    double* chunk_max;
    double* tile_err;
    double* hist;                 // E per iteration
    double* link_mean;
    double* link_max;
    unsigned long long* skipped;
    double* out_stats;            // iterations, stopped, E
    int tm, rm;
    double lam, max_error;
    int max_iterations, width, min_matches, models_in_smem;
};

__global__ void __launch_bounds__(MOM_THREADS) k_link_moments(const long long* __restrict__ off, const double* __restrict__ p,
                                                             const double* __restrict__ q, const double* __restrict__ w,
                                                             double* __restrict__ mom) {
    __shared__ double s_part[MOM_THREADS / 32][MOM - 3];
    const int l = blockIdx.x;
    const long long b = off[l], e = off[l + 1];
    double o[3] = {0.0, 0.0, 0.0};
    if (e > b) { o[0] = p[3 * b]; o[1] = p[3 * b + 1]; o[2] = p[3 * b + 2]; }
    double acc[MOM - 3];                           // W, n, Sp, Sq, Spp, Sqq, Spq (everything but the anchor)
#pragma unroll
    for (int k = 0; k < MOM - 3; ++k) acc[k] = 0.0;
    for (long long m = b + threadIdx.x; m < e; m += MOM_THREADS) {
        const double wm = w[m];
        double pp[3], qq[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) { pp[i] = p[3 * m + i] - o[i]; qq[i] = q[3 * m + i] - o[i]; }
        acc[0] += wm;
        acc[1] += 1.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            acc[2 + i] += wm * pp[i];
            acc[5 + i] += wm * qq[i];
#pragma unroll
            for (int j = i; j < 3; ++j) {
                acc[8 + sym(i, j)] += wm * pp[i] * pp[j];
                acc[14 + sym(i, j)] += wm * qq[i] * qq[j];
            }
#pragma unroll
            for (int j = 0; j < 3; ++j) acc[20 + 3 * i + j] += wm * pp[i] * qq[j];
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < MOM - 3; ++k) {
        double v = acc[k];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) s_part[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < MOM - 3) {
        double v = 0.0;
        for (int i = 0; i < MOM_THREADS / 32; ++i) v += s_part[i][threadIdx.x];
        const int k = threadIdx.x;
        mom[(size_t)l * MOM + (k < 2 ? k : k + 3)] = v;
    }
    if (threadIdx.x == 0) {
        mom[(size_t)l * MOM + M_O] = o[0];
        mom[(size_t)l * MOM + M_O + 1] = o[1];
        mom[(size_t)l * MOM + M_O + 2] = o[2];
    }
}

// ---------------------------------------------------------------------------------------------------- fits
struct TileSums {       // centred weighted moments of one tile in its own frame (origin o)
    double W, cx[3], cy[3], P[3][3], Q[3][3], o[3];
};

template <int P, int Q>
__device__ __forceinline__ void jacobi_rot(double a[4][4], double v[4][4]) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    const double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double x = a[k][P], y = a[k][Q];
        a[k][P] = c * x - s * y;
        a[k][Q] = s * x + c * y;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double x = a[P][k], y = a[Q][k];
        a[P][k] = c * x - s * y;
        a[Q][k] = s * x + c * y;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double x = v[k][P], y = v[k][Q];
        v[k][P] = c * x - s * y;
        v[k][Q] = s * x + c * y;
    }
}

// Horn: the rotation of the unit quaternion of N's largest eigenvalue (cyclic Jacobi on the 4 x 4 symmetric N)
__device__ __noinline__ void horn_rotation(const double S[3][3], double R[3][3]) {
    const double xx = S[0][0], xy = S[0][1], xz = S[0][2], yx = S[1][0], yy = S[1][1], yz = S[1][2], zx = S[2][0],
                 zy = S[2][1], zz = S[2][2];
    double a[4][4] = {{xx + yy + zz, yz - zy, zx - xz, xy - yx},
                      {yz - zy, xx - yy - zz, xy + yx, zx + xz},
                      {zx - xz, xy + yx, -xx + yy - zz, yz + zy},
                      {xy - yx, zx + xz, yz + zy, -xx - yy + zz}};
    double v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 32; ++sweep) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[0][3] * a[0][3] + a[1][2] * a[1][2] +
                           a[1][3] * a[1][3] + a[2][3] * a[2][3];
        const double dia = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2] + a[3][3] * a[3][3];
        if (off <= 1e-36 * dia || off == 0.0) break;
        jacobi_rot<0, 1>(a, v);
        jacobi_rot<0, 2>(a, v);
        jacobi_rot<0, 3>(a, v);
        jacobi_rot<1, 2>(a, v);
        jacobi_rot<1, 3>(a, v);
        jacobi_rot<2, 3>(a, v);
    }
    int k = 0;
#pragma unroll
    for (int i = 1; i < 4; ++i)
        if (a[i][i] > a[k][k]) k = i;
    double q0 = 0, q1 = 0, q2 = 0, q3 = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (i == k) { q0 = v[0][i]; q1 = v[1][i]; q2 = v[2][i]; q3 = v[3][i]; }
    R[0][0] = q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3; R[0][1] = 2 * (q1 * q2 - q0 * q3); R[0][2] = 2 * (q1 * q3 + q0 * q2);
    R[1][0] = 2 * (q2 * q1 + q0 * q3); R[1][1] = q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3; R[1][2] = 2 * (q2 * q3 - q0 * q1);
    R[2][0] = 2 * (q3 * q1 - q0 * q2); R[2][1] = 2 * (q3 * q2 + q0 * q1); R[2][2] = q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3;
}

// one model kind fitted to the sums; false = singular (the model keeps its value)
__device__ bool fit_kind(int kind, const TileSums& s, double M[12]) {
    double A[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    if (kind == BS_MODEL_IDENTITY) {
        for (int i = 0; i < 12; ++i) M[i] = (i % 5 == 0) ? 1.0 : 0.0;
        return true;
    }
    if (!(s.W > 0.0)) return false;
    bool ok = true;
    const double(&P)[3][3] = s.P;
    const double tr = P[0][0] + P[1][1] + P[2][2];
    if (kind == BS_MODEL_RIGID) {
        const double i2 = P[0][0] * P[1][1] - P[0][1] * P[0][1] + P[0][0] * P[2][2] - P[0][2] * P[0][2] +
                          P[1][1] * P[2][2] - P[1][2] * P[1][2];
        ok = i2 > 1e-12 * tr * tr;
        horn_rotation(s.Q, A);
    } else if (kind == BS_MODEL_AFFINE) {
        const double c00 = P[1][1] * P[2][2] - P[1][2] * P[2][1], c01 = P[1][2] * P[2][0] - P[1][0] * P[2][2],
                     c02 = P[1][0] * P[2][1] - P[1][1] * P[2][0];
        const double det = P[0][0] * c00 + P[0][1] * c01 + P[0][2] * c02;
        ok = isfinite(det) && det > 1e-12 * (tr / 3.0) * (tr / 3.0) * (tr / 3.0);
        if (!ok) return false;
        const double inv[3][3] = {{c00 / det, (P[0][2] * P[2][1] - P[0][1] * P[2][2]) / det, (P[0][1] * P[1][2] - P[0][2] * P[1][1]) / det},
                                  {c01 / det, (P[0][0] * P[2][2] - P[0][2] * P[2][0]) / det, (P[0][2] * P[1][0] - P[0][0] * P[1][2]) / det},
                                  {c02 / det, (P[0][1] * P[2][0] - P[0][0] * P[2][1]) / det, (P[0][0] * P[1][1] - P[0][1] * P[1][0]) / det}};
        // X = P^-1 Q (b_c = X^T a_c), A = X^T
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) A[j][i] = inv[i][0] * s.Q[0][j] + inv[i][1] * s.Q[1][j] + inv[i][2] * s.Q[2][j];
    }
    // y = A x + t in world coordinates: t = (cy + o) - A (cx + o)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        double ax = 0.0;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            M[4 * i + j] = A[i][j];
            ax += A[i][j] * (s.cx[j] + s.o[j]);
        }
        M[4 * i + 3] = (s.cy[i] + s.o[i]) - ax;
    }
    return ok;
}

__device__ __forceinline__ double ldm(const double* models, int t, int k, const double* s_models) {
    return s_models ? s_models[12 * t + k] : __ldcg(models + 12 * t + k);
}

// gather the tile's sums from its link moments and its partners' current models, fit, store (or count a skip)
__device__ __noinline__ void fit_tile(const SolveArgs& a, int t) {
    const int b0 = a.tile_ptr[t], b1 = a.tile_ptr[t + 1];
    TileSums s;
    double n = 0.0, sx[3] = {0, 0, 0}, sy[3] = {0, 0, 0}, sxx[3][3] = {}, sxy[3][3] = {};
    s.W = 0.0;
    const int l0 = a.tile_adj[b0] >> 1;
#pragma unroll
    for (int i = 0; i < 3; ++i) s.o[i] = __ldg(a.mom + (size_t)l0 * MOM + M_O + i);
    for (int e = b0; e < b1; ++e) {
        const int l = a.tile_adj[e] >> 1, side = a.tile_adj[e] & 1;
        const double* m = a.mom + (size_t)l * MOM;
        const int u = a.links[2 * l + (1 - side)];
        const double Wl = __ldg(m + M_W);
        n += __ldg(m + M_N);
        double Au[3][3], g[3], d[3], Sx[3], Sz[3], ASz[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double ol = __ldg(m + M_O + i);
            d[i] = ol - s.o[i];
            Sx[i] = __ldg(m + (side ? M_SQ : M_SP) + i);
            Sz[i] = __ldg(m + (side ? M_SP : M_SQ) + i);
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double go = 0.0;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                Au[i][j] = __ldcg(a.models + 12 * u + 4 * i + j);
                go += Au[i][j] * __ldg(m + M_O + j);
            }
            g[i] = go + __ldcg(a.models + 12 * u + 4 * i + 3) - s.o[i];
            ASz[i] = Au[i][0] * Sz[0] + Au[i][1] * Sz[1] + Au[i][2] * Sz[2];
        }
        s.W += Wl;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            sx[i] += Sx[i] + Wl * d[i];
            sy[i] += ASz[i] + Wl * g[i];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const double Sxx = __ldg(m + (side ? M_SQQ : M_SPP) + sym(i, j));
                sxx[i][j] += Sxx + Sx[i] * d[j] + d[i] * Sx[j] + Wl * d[i] * d[j];
                double sxz_au = 0.0;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    // sum x_i z_k: Spq[i][k] for side 0, Spq[k][i] for side 1
                    const double Sxz = __ldg(m + M_SPQ + (side ? 3 * k + i : 3 * i + k));
                    sxz_au += Sxz * Au[j][k];
                }
                sxy[i][j] += sxz_au + Sx[i] * g[j] + d[i] * ASz[j] + Wl * d[i] * g[j];
            }
        }
    }
    double R[12];
    bool ok = n >= (double)a.min_matches && s.W > 0.0;
    if (ok) {
#pragma unroll
        for (int i = 0; i < 3; ++i) { s.cx[i] = sx[i] / s.W; s.cy[i] = sy[i] / s.W; }
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                s.P[i][j] = sxx[i][j] - s.W * s.cx[i] * s.cx[j];
                s.Q[i][j] = sxy[i][j] - s.W * s.cx[i] * s.cy[j];
            }
        ok = fit_kind(a.tm, s, R);
        if (ok && a.rm >= 0) {
            double Rr[12];
            ok = fit_kind(a.rm, s, Rr);
#pragma unroll
            for (int k = 0; k < 12; ++k) R[k] = (1.0 - a.lam) * R[k] + a.lam * Rr[k];
        }
    }
    if (ok) {
#pragma unroll
        for (int k = 0; k < 12; ++k) a.models[12 * t + k] = R[k];
    } else {
        atomicAdd(a.skipped, 1ull);
    }
}

// ---------------------------------------------------------------------------------------------------- the solve
__global__ void __launch_bounds__(SOLVE_THREADS, 1) k_solve(SolveArgs a) {
    extern __shared__ double s_models[];
    __shared__ double s_red[SOLVE_THREADS / 32];
    cg::grid_group grid = cg::this_grid();
    const int gtid = blockIdx.x * SOLVE_THREADS + threadIdx.x, gthreads = gridDim.x * SOLVE_THREADS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gwarp = blockIdx.x * (SOLVE_THREADS / 32) + warp, gwarps = gridDim.x * (SOLVE_THREADS / 32);
    int it = 0, stopped = 0;
    double E = 0.0;
    while (it < a.max_iterations) {
        ++it;
        // 1. multicolour Gauss-Seidel sweep
        for (int c = 0; c < a.n_colours; ++c) {
            const int c0 = a.colour_offsets[c], c1 = a.colour_offsets[c + 1];
            for (int k = c0 + gtid; k < c1; k += gthreads) {
                const int t = a.colour_tiles[k];
                if (!a.fixed[t] && a.tile_ptr[t + 1] > a.tile_ptr[t]) fit_tile(a, t);
                else if (!a.fixed[t]) atomicAdd(a.skipped, 1ull);
            }
            grid.sync();
        }
        // 2. distances, per chunk sum w d and max d
        const double* sm = nullptr;
        if (a.models_in_smem) {
            for (int k = threadIdx.x; k < 12 * a.n_tiles; k += SOLVE_THREADS) s_models[k] = __ldcg(a.models + k);
            __syncthreads();
            sm = s_models;
        }
        for (int c = gwarp; c < a.n_chunks; c += gwarps) {
            const int l = a.chunk_link[c];
            const long long m0 = a.chunk_begin[c], m1 = min(m0 + CHUNK, a.match_offsets[l + 1]);
            const int ta = a.links[2 * l], tb = a.links[2 * l + 1];
            double Ma[12], Mb[12];
#pragma unroll
            for (int k = 0; k < 12; ++k) { Ma[k] = ldm(a.models, ta, k, sm); Mb[k] = ldm(a.models, tb, k, sm); }
            double swd = 0.0, mx = 0.0;
#pragma unroll 4
            for (long long m = m0 + lane; m < m1; m += 32) {
                const double px = __ldg(a.p + 3 * m), py = __ldg(a.p + 3 * m + 1), pz = __ldg(a.p + 3 * m + 2);
                const double qx = __ldg(a.q + 3 * m), qy = __ldg(a.q + 3 * m + 1), qz = __ldg(a.q + 3 * m + 2);
                const double wm = __ldg(a.w + m);
                const double dx = (Ma[0] * px + Ma[1] * py + Ma[2] * pz + Ma[3]) - (Mb[0] * qx + Mb[1] * qy + Mb[2] * qz + Mb[3]);
                const double dy = (Ma[4] * px + Ma[5] * py + Ma[6] * pz + Ma[7]) - (Mb[4] * qx + Mb[5] * qy + Mb[6] * qz + Mb[7]);
                const double dz = (Ma[8] * px + Ma[9] * py + Ma[10] * pz + Ma[11]) - (Mb[8] * qx + Mb[9] * qy + Mb[10] * qz + Mb[11]);
                const double d = sqrt(dx * dx + dy * dy + dz * dz);
                swd += wm * d;
                mx = fmax(mx, d);
            }
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) {
                swd += __shfl_xor_sync(0xffffffffu, swd, s);
                mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, s));
            }
            if (lane == 0) { a.chunk_swd[c] = swd; a.chunk_max[c] = mx; }
        }
        grid.sync();
        // 3. tile errors
        for (int t = gtid; t < a.n_tiles; t += gthreads) {
            double swd = 0.0, sw = 0.0;
            for (int e = a.tile_ptr[t]; e < a.tile_ptr[t + 1]; ++e) {
                const int l = a.tile_adj[e] >> 1;
                for (int c = a.link_chunk_ptr[l]; c < a.link_chunk_ptr[l + 1]; ++c) swd += __ldcg(a.chunk_swd + c);
                sw += __ldg(a.mom + (size_t)l * MOM + M_W);
            }
            a.tile_err[t] = sw > 0.0 ? swd / sw : 0.0;
        }
        grid.sync();
        // 4. E and the stopping rule, identically in every block
        double v = 0.0;
        for (int t = threadIdx.x; t < a.n_tiles; t += SOLVE_THREADS) v += __ldcg(a.tile_err + t);
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) s_red[warp] = v;
        __syncthreads();
        E = 0.0;
        for (int i = 0; i < SOLVE_THREADS / 32; ++i) E += s_red[i];
        E /= (double)a.n_tiles;
        __syncthreads();
        if (blockIdx.x == 0 && threadIdx.x == 0) a.hist[it - 1] = E;
        if (it > a.width) {
            bool go = E > a.max_error;
            for (int d = a.width; d >= 1; d >>= 1) go = go || fabs((E - __ldcg(a.hist + it - 1 - d)) / d) > 1e-4;
            if (!go) { stopped = 1; break; }
        }
    }
    // link statistics of the last iteration (ONE_ROUND_ITERATIVE's link removal reads them)
    for (int l = gtid; l < a.n_links; l += gthreads) {
        double swd = 0.0, mx = 0.0;
        for (int c = a.link_chunk_ptr[l]; c < a.link_chunk_ptr[l + 1]; ++c) {
            swd += __ldcg(a.chunk_swd + c);
            mx = fmax(mx, __ldcg(a.chunk_max + c));
        }
        const double W = __ldg(a.mom + (size_t)l * MOM + M_W);
        a.link_mean[l] = W > 0.0 ? swd / W : 0.0;
        a.link_max[l] = mx;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.out_stats[0] = (double)it;
        a.out_stats[1] = (double)stopped;
        a.out_stats[2] = E;
    }
}

struct DevBufs {
    std::vector<void*> ptrs;
    ~DevBufs() {
        for (void* p : ptrs) cudaFree(p);
    }
};

int min_matches_of(int kind) {
    return kind == BS_MODEL_AFFINE ? 4 : kind == BS_MODEL_RIGID ? 3 : kind == BS_MODEL_TRANSLATION ? 1 : 0;
}

}  // namespace

extern "C" {

int bs_solve_tiles(bs_ctx* ctx, int n_tiles, int n_colours, const int* colour_offsets, const int* colour_tiles,
                   const int* fixed, int n_links, const int* links, const long long* match_offsets, const double* p,
                   const double* q, const double* w, const bs_solve_params* params, double* models,
                   bs_solve_stats* stats, double* tile_error, double* link_mean, double* link_max) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
#define SOLVE_ARG(cond, ...) \
    if (!(cond)) return bs_set_error(ctx, BS_ERR_ARG, "bs_solve_tiles: " __VA_ARGS__)
    SOLVE_ARG(params && models && stats && tile_error, "NULL argument");
    SOLVE_ARG(n_tiles >= 1 && n_links >= 0 && n_colours >= 1 && n_colours <= n_tiles, "n_tiles %d, n_links %d, n_colours %d",
              n_tiles, n_links, n_colours);
    SOLVE_ARG(colour_offsets && colour_tiles && fixed && (n_links == 0 || (links && match_offsets && link_mean && link_max)),
              "NULL array");
    const bs_solve_params& P = *params;
    SOLVE_ARG(P.transformation >= BS_MODEL_TRANSLATION && P.transformation <= BS_MODEL_AFFINE, "transformation %d",
              P.transformation);
    SOLVE_ARG(P.regularization >= BS_MODEL_NONE && P.regularization <= BS_MODEL_AFFINE, "regularization %d", P.regularization);
    SOLVE_ARG(P.lambda >= 0.0 && P.lambda <= 1.0, "lambda %g outside [0, 1]", P.lambda);
    SOLVE_ARG(!std::isnan(P.max_error), "max_error is NaN");
    SOLVE_ARG(P.max_iterations >= 1 && P.max_plateau_width >= 0, "max_iterations %d, max_plateau_width %d",
              P.max_iterations, P.max_plateau_width);
    // colours: offsets ascending from 0 to n_tiles, tiles a permutation, no link inside one colour
    std::vector<int> colour((size_t)n_tiles, -1);
    SOLVE_ARG(colour_offsets[0] == 0 && colour_offsets[n_colours] == n_tiles, "colour offsets must run from 0 to n_tiles");
    for (int c = 0; c < n_colours; ++c) {
        SOLVE_ARG(colour_offsets[c + 1] >= colour_offsets[c], "colour offsets must ascend");
        for (int k = colour_offsets[c]; k < colour_offsets[c + 1]; ++k) {
            const int t = colour_tiles[k];
            SOLVE_ARG(t >= 0 && t < n_tiles && colour[t] < 0, "colour_tiles is not a permutation of the tiles");
            colour[t] = c;
        }
    }
    SOLVE_ARG(n_links == 0 || match_offsets[0] == 0, "match_offsets[0] must be 0");
    for (int l = 0; l < n_links; ++l) {
        const int ta = links[2 * l], tb = links[2 * l + 1];
        SOLVE_ARG(ta >= 0 && ta < n_tiles && tb >= 0 && tb < n_tiles && ta != tb, "link %d joins tiles %d and %d", l, ta, tb);
        SOLVE_ARG(colour[ta] != colour[tb], "link %d joins two tiles of colour %d", l, colour[ta]);
        SOLVE_ARG(match_offsets[l + 1] >= match_offsets[l], "match_offsets must ascend");
    }
    const long long n_matches = n_links ? match_offsets[n_links] : 0;
    SOLVE_ARG(n_matches == 0 || (p && q && w), "NULL match array");
    for (long long m = 0; m < n_matches; ++m) {
        SOLVE_ARG(std::isfinite(w[m]) && w[m] >= 0.0, "weight %lld is %g", m, w[m]);
        for (int i = 0; i < 3; ++i) SOLVE_ARG(std::isfinite(p[3 * m + i]) && std::isfinite(q[3 * m + i]), "match %lld is not finite", m);
    }
    for (long long k = 0; k < 12LL * n_tiles; ++k) SOLVE_ARG(std::isfinite(models[k]), "model %lld is not finite", k / 12);
#undef SOLVE_ARG

    // tile adjacency (ascending link per tile) and the chunks of the distance pass
    std::vector<int> tile_ptr((size_t)n_tiles + 1, 0), tile_adj((size_t)2 * n_links);
    for (int l = 0; l < n_links; ++l) { ++tile_ptr[links[2 * l] + 1]; ++tile_ptr[links[2 * l + 1] + 1]; }
    for (int t = 0; t < n_tiles; ++t) tile_ptr[t + 1] += tile_ptr[t];
    {
        std::vector<int> fill(tile_ptr.begin(), tile_ptr.end() - 1);
        for (int l = 0; l < n_links; ++l) {
            tile_adj[fill[links[2 * l]]++] = 2 * l;
            tile_adj[fill[links[2 * l + 1]]++] = 2 * l + 1;
        }
    }
    std::vector<int> chunk_link, link_chunk_ptr((size_t)n_links + 1, 0);
    std::vector<long long> chunk_begin;
    for (int l = 0; l < n_links; ++l) {
        for (long long m = match_offsets[l]; m < match_offsets[l + 1]; m += CHUNK) {
            chunk_link.push_back(l);
            chunk_begin.push_back(m);
        }
        link_chunk_ptr[l + 1] = (int)chunk_link.size();
    }
    const int n_chunks = (int)chunk_link.size();
    int max_colour = 0;
    for (int c = 0; c < n_colours; ++c) max_colour = std::max(max_colour, colour_offsets[c + 1] - colour_offsets[c]);

    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    DevBufs bufs;
    auto dalloc = [&](size_t bytes) -> void* {
        void* d = nullptr;
        if (cudaMalloc(&d, std::max<size_t>(bytes, 16)) != cudaSuccess) return nullptr;
        bufs.ptrs.push_back(d);
        return d;
    };
    auto up = [&](const void* h, size_t bytes) -> void* {
        void* d = dalloc(bytes);
        if (d && bytes && cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return nullptr;
        return d;
    };
    const int zero = 0;
    SolveArgs a{};
    a.n_tiles = n_tiles; a.n_colours = n_colours; a.n_links = n_links; a.n_chunks = n_chunks;
    a.colour_offsets = (const int*)up(colour_offsets, sizeof(int) * (n_colours + 1));
    a.colour_tiles = (const int*)up(colour_tiles, sizeof(int) * n_tiles);
    a.fixed = (const int*)up(fixed, sizeof(int) * n_tiles);
    a.links = (const int*)up(n_links ? links : &zero, sizeof(int) * 2 * n_links);
    a.tile_ptr = (const int*)up(tile_ptr.data(), sizeof(int) * tile_ptr.size());
    a.tile_adj = (const int*)up(tile_adj.data(), sizeof(int) * tile_adj.size());
    a.chunk_link = (const int*)up(chunk_link.data(), sizeof(int) * chunk_link.size());
    a.chunk_begin = (const long long*)up(chunk_begin.data(), sizeof(long long) * chunk_begin.size());
    a.match_offsets = (const long long*)up(n_links ? match_offsets : (const long long*)&zero, sizeof(long long) * (n_links ? n_links + 1 : 0));
    a.link_chunk_ptr = (const int*)up(link_chunk_ptr.data(), sizeof(int) * link_chunk_ptr.size());
    a.p = (const double*)up(p, sizeof(double) * 3 * n_matches);
    a.q = (const double*)up(q, sizeof(double) * 3 * n_matches);
    a.w = (const double*)up(w, sizeof(double) * n_matches);
    a.models = (double*)up(models, sizeof(double) * 12 * n_tiles);
    double* mom = (double*)dalloc(sizeof(double) * MOM * n_links);
    a.mom = mom;
    a.chunk_swd = (double*)dalloc(sizeof(double) * n_chunks);
    a.chunk_max = (double*)dalloc(sizeof(double) * n_chunks);
    a.tile_err = (double*)dalloc(sizeof(double) * n_tiles);
    a.hist = (double*)dalloc(sizeof(double) * P.max_iterations);
    a.link_mean = (double*)dalloc(sizeof(double) * n_links);
    a.link_max = (double*)dalloc(sizeof(double) * n_links);
    a.skipped = (unsigned long long*)dalloc(sizeof(unsigned long long));
    a.out_stats = (double*)dalloc(sizeof(double) * 3);
    for (const void* ptr : {(const void*)a.colour_offsets, (const void*)a.colour_tiles, (const void*)a.fixed, (const void*)a.links,
                            (const void*)a.tile_ptr, (const void*)a.tile_adj, (const void*)a.chunk_link, (const void*)a.chunk_begin,
                            (const void*)a.match_offsets, (const void*)a.link_chunk_ptr, (const void*)a.p, (const void*)a.q,
                            (const void*)a.w, (const void*)a.models, (const void*)mom, (const void*)a.chunk_swd,
                            (const void*)a.chunk_max, (const void*)a.tile_err, (const void*)a.hist, (const void*)a.link_mean,
                            (const void*)a.link_max, (const void*)a.skipped, (const void*)a.out_stats})
        if (!ptr) return bs_set_error(ctx, BS_ERR_NOMEM, "bs_solve_tiles: device allocation or copy failed");
    BS_CUDA(ctx, cudaMemsetAsync(a.chunk_swd, 0, sizeof(double) * std::max(n_chunks, 1), ctx->stream));
    BS_CUDA(ctx, cudaMemsetAsync(a.chunk_max, 0, sizeof(double) * std::max(n_chunks, 1), ctx->stream));
    BS_CUDA(ctx, cudaMemsetAsync(a.skipped, 0, sizeof(unsigned long long), ctx->stream));
    a.tm = P.transformation;
    a.rm = P.regularization;
    a.lam = P.lambda;
    a.max_error = P.max_error;
    a.max_iterations = P.max_iterations;
    a.width = P.max_plateau_width;
    a.min_matches = std::max(1, std::max(min_matches_of(P.transformation), P.regularization >= 0 ? min_matches_of(P.regularization) : 0));
    const size_t smem = sizeof(double) * 12 * (size_t)n_tiles;
    a.models_in_smem = smem <= SMEM_MODELS_MAX ? 1 : 0;
    const size_t dyn = a.models_in_smem ? smem : 0;

    if (n_links > 0) {
        bs_launch_scope scope(ctx, "solve_moments");
        k_link_moments<<<n_links, MOM_THREADS, 0, ctx->stream>>>(a.match_offsets, a.p, a.q, a.w, mom);
    }
    BS_CUDA(ctx, cudaGetLastError());
    // grid: as many co-resident blocks as the occupancy allows, but no more than the largest pass can use
    BS_CUDA(ctx, cudaFuncSetAttribute(k_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MODELS_MAX));
    int per_sm = 0;
    BS_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_solve, SOLVE_THREADS, dyn));
    if (per_sm < 1) return bs_set_error(ctx, BS_ERR_CUDA, "bs_solve_tiles: k_solve cannot be resident (%zu B shared)", dyn);
    const int need = std::max({(max_colour + SOLVE_THREADS - 1) / SOLVE_THREADS, (n_chunks + SOLVE_THREADS / 32 - 1) / (SOLVE_THREADS / 32),
                               (n_tiles + SOLVE_THREADS - 1) / SOLVE_THREADS, (n_links + SOLVE_THREADS - 1) / SOLVE_THREADS, 1});
    const int blocks = std::min(per_sm * ctx->sm_count, need);
    {
        bs_launch_scope scope(ctx, "solve");
        void* kargs[] = {&a};
        BS_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)k_solve, dim3(blocks), dim3(SOLVE_THREADS), kargs, dyn, ctx->stream));
    }
    double st[3];
    unsigned long long skipped = 0;
    BS_CUDA(ctx, cudaMemcpyAsync(models, a.models, sizeof(double) * 12 * n_tiles, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(tile_error, a.tile_err, sizeof(double) * n_tiles, cudaMemcpyDeviceToHost, ctx->stream));
    if (n_links) {
        BS_CUDA(ctx, cudaMemcpyAsync(link_mean, a.link_mean, sizeof(double) * n_links, cudaMemcpyDeviceToHost, ctx->stream));
        BS_CUDA(ctx, cudaMemcpyAsync(link_max, a.link_max, sizeof(double) * n_links, cudaMemcpyDeviceToHost, ctx->stream));
    }
    BS_CUDA(ctx, cudaMemcpyAsync(st, a.out_stats, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(&skipped, a.skipped, sizeof(skipped), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    stats->iterations = (int)st[0];
    stats->stopped = (int)st[1];
    stats->skipped_fits = (long long)skipped;
    stats->error = st[2];
    stats->blocks = blocks;
    stats->models_in_shared = a.models_in_smem;
    return BS_OK;
}

}  // extern "C"
