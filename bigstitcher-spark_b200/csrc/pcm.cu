// Hot path 1: phase correlation of one overlap-cropped tile pair, entirely on the device.
// Replaces TransformationTools.computeStitching's numeric core
// (PairwiseStitching.getShift -> PhaseCorrelation2.calculatePCM + getShift; call site
// J/SparkPairwiseStitching.java:247-255).  No cuFFT: the 3-D real FFT is five hand-written
// passes over an x-fastest half spectrum S[Pz][Py][pitch] (complex64, pitch = M+1 rounded up
// to 16 so every row is 128 B aligned):
//
//   k_fft_x_r2c      uint16/float crop -> blended mirrored extension + zero pad -> R2C along x
//   k_fft_col540     forward FFT along y, in place, both spectra in one launch
//   k_fft_xpower_col540  forward z FFT of A and B, unit-magnitude normalisation,
//                    conj(A)*B, forward z FFT of the product      [reads 2S, writes S]
//   k_fft_col540     forward y FFT of the product
//                    (other padded y / z sizes than 540: k_fft_strided_pipe / k_fft_xpower_pipe / k_fft_strided)
//   k_fft_x_c2r      conj + C2R along x, in place -> real PCM (row pitch 2*pitch floats)
//                    (Px = 540 with at least one tile per SM: k_fft_x_r2c_col540 / k_fft_x_c2r_col540, two lines per
//                    complex transform)
//   k_peaks          periodic 6-neighbour local maxima, per-CTA top-K
//   k_gather27       3x3x3 neighbourhoods of the K peaks (sub-pixel fit runs on the host)
//   k_pearson_u16    exact integer sums (uint64 atomics) for all surviving wrap candidates, slab-staged image 1
//                    (k_pearson: uint8 / float32 and unaligned uint16 crops)
//
// Inverse transforms are forward transforms of conjugated data (conj(F(conj X)) = N F^-1 X);
// the two conjugations between consecutive passes cancel, so only the product step and the
// C2R load conjugate.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "bs_internal.cuh"
#include "pcm_fft.cuh"

#define PCM_THREADS 256
#define PCM_KMAX 32
#define PCM_SMEM_MAX 232448  // 227 KB opt-in limit per CTA on sm_90

extern __shared__ __align__(128) float2 bs_sm[];   // 128: tensor-map copies into it need 128-byte aligned targets

// ------------------------------------------------------------------------------------------
// x pass, real -> complex
struct XR2CArgs {
    const void* img[2];
    float2* spec[2];
    int dtype;
    int dx, dy, dz;
    int Px, Py, Pz, M, pitch;
    int ex;        // offset of the crop inside the padded x axis (= min(extension, dx))
    int Ex, Ey, Ez;
    const int* idx_x; const float* w_x;
    const int* idx_y; const float* w_y;
    const int* idx_z; const float* w_z;
    const float2* tw;
    FftPlan plan;
    int lshift;
};

__device__ __forceinline__ float load_voxel(const void* p, int dtype, size_t i) {
    if (dtype == BS_DTYPE_U16) return (float)__ldg((const unsigned short*)p + i);
    if (dtype == BS_DTYPE_F32) return __ldg((const float*)p + i);
    return (float)__ldg((const unsigned char*)p + i);
}

// One warp owns a line at a time: the row's y/z profile is warp-uniform, interior samples are
// read as aligned ushort2 pairs, and each lane keeps XR_UNROLL independent loads in flight.
#define XR_UNROLL 5
template <class F>
__global__ void __launch_bounds__(PCM_THREADS) k_fft_x_r2c(const __grid_constant__ XR2CArgs a) {
    const int M = F::kStatic ? F::N : a.M;
    const int lshift = F::kStatic ? F::LSHIFT : a.lshift;
    const int LB = 1 << lshift, ls = LB + 1;
    const int Px = 2 * M;
    const int pitch = F::kStatic ? ((F::N + 1 + 15) / 16) * 16 : a.pitch;
    float2* tw = bs_sm;
    float2* b0 = bs_sm + Px;
    float2* b1 = b0 + M * ls;
    const int zp = blockIdx.y, y0 = blockIdx.x * LB, im = blockIdx.z;
    float2* __restrict__ spec = a.spec[im];
    const size_t rowbase = ((size_t)zp * a.Py + y0) * pitch;
    const int nlines = min(LB, a.Py - y0);
    if (zp >= a.Ez || y0 >= a.Ey) {  // every line of this CTA lies in the zero padding
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4* d4 = reinterpret_cast<float4*>(spec + rowbase);
        for (int i = threadIdx.x; i < nlines * (pitch >> 1); i += blockDim.x) d4[i] = z4;
        return;
    }
    for (int i = threadIdx.x; i < Px; i += blockDim.x) tw[i] = a.tw[i];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int NW = PCM_THREADS / 32;
    const float wz = a.w_z[zp];
    const int sz = a.idx_z[zp];
    const void* img = a.img[im];
    const int e0 = a.ex;
    const bool vec_ok = a.dtype == BS_DTYPE_U16 && !(e0 & 1) && !(a.dx & 1) && !((size_t)img & 3);
    // two lines per warp pass -> 2 * XR_UNROLL independent loads in flight per lane
    for (int lA = wid; lA < LB; lA += 2 * NW) {
        bool live[2];
        float gyz[2], wy[2];
        size_t rb[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int l = lA + h * NW, yp = y0 + l;
            live[h] = l < LB && l < nlines && yp < a.Ey;
            wy[h] = 0.f;
            rb[h] = 0;
            if (live[h]) {
                wy[h] = a.w_y[yp];
                rb[h] = ((size_t)sz * a.dy + a.idx_y[yp]) * a.dx;
            }
            gyz[h] = wy[h] * wz;  // == (1 * wy) * wz for interior samples
        }
        for (int n0 = 0; n0 < M; n0 += 32 * XR_UNROLL) {
            float2 v[2][XR_UNROLL];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int u = 0; u < XR_UNROLL; ++u) {
                    const int n = n0 + u * 32 + lane;
                    v[h][u] = make_float2(0.f, 0.f);
                    if (live[h] && n < M) {
                        const int xp = 2 * n;
                        if (xp >= e0 && xp + 1 < e0 + a.dx) {
                            if (vec_ok) {
                                const ushort2 t = __ldg(reinterpret_cast<const ushort2*>(
                                    (const unsigned short*)img + rb[h] + (xp - e0)));
                                v[h][u] = make_float2((float)t.x * gyz[h], (float)t.y * gyz[h]);
                            } else {
                                v[h][u] = make_float2(load_voxel(img, a.dtype, rb[h] + (xp - e0)) * gyz[h],
                                                      load_voxel(img, a.dtype, rb[h] + (xp - e0) + 1) * gyz[h]);
                            }
                        } else if (xp < a.Ex) {  // blended mirrored margin (a few samples per line)
                            const float g0 = (a.w_x[xp] * wy[h]) * wz, g1 = (a.w_x[xp + 1] * wy[h]) * wz;
                            if (g0 != 0.f) v[h][u].x = load_voxel(img, a.dtype, rb[h] + a.idx_x[xp]) * g0;
                            if (g1 != 0.f) v[h][u].y = load_voxel(img, a.dtype, rb[h] + a.idx_x[xp + 1]) * g1;
                        }
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int l = lA + h * NW;
                if (l < LB) {
#pragma unroll
                    for (int u = 0; u < XR_UNROLL; ++u) {
                        const int n = n0 + u * 32 + lane;
                        if (n < M) b0[n * ls + l] = v[h][u];
                    }
                }
            }
        }
    }
    __syncthreads();
    const float2* res = F::run(b0, b1, tw, a.plan, lshift, ls, 2);
    // untangle the packed half-length transform into the real-input spectrum X[0..M]
    for (int l = wid; l < nlines; l += NW) {
        float2* srow = spec + rowbase + (size_t)l * pitch;
        for (int k = lane; k < pitch; k += 32) {
            float2 X = make_float2(0.f, 0.f);
            if (k <= M) {
                const int k0 = (k == M) ? 0 : k;
                const int k1 = (k == 0 || k == M) ? 0 : M - k;
                const float2 Zk = res[k0 * ls + l];
                float2 Zm = res[k1 * ls + l];
                Zm.y = -Zm.y;
                const float2 E = make_float2(0.5f * (Zk.x + Zm.x), 0.5f * (Zk.y + Zm.y));
                const float2 D = make_float2(0.5f * (Zk.x - Zm.x), 0.5f * (Zk.y - Zm.y));
                const float2 wD = cmulf(tw[k], D);
                X = make_float2(E.x + wD.y, E.y - wD.x);  // E - i*w*D
            }
            __stcg(srow + k, X);
        }
    }
}

// ------------------------------------------------------------------------------------------
// x pass, real -> complex, persistent + TMA: each CTA loops over line groups; the raw uint16 /
// float rows of the NEXT group are pulled into shared memory by the TMA unit (1-D bulk copies
// completing on an mbarrier) while the current group is windowed, transformed and stored.
__device__ __forceinline__ unsigned int smem_u32(const void* p) {
    return (unsigned int)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
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
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, unsigned int bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct XR2CTmaArgs {
    XR2CArgs x;
    int n_groups;      // line groups per plane
    int n_items;       // 2 * Pz * n_groups
    int row_bytes;     // dx * element size (multiple of 16)
    int esize;
};

template <class F>
__global__ void __launch_bounds__(PCM_THREADS) k_fft_x_r2c_tma(const __grid_constant__ XR2CTmaArgs t) {
    const XR2CArgs& a = t.x;
    const int M = F::kStatic ? F::N : a.M;
    const int lshift = F::kStatic ? F::LSHIFT : a.lshift;
    const int LB = 1 << lshift, ls = LB + 1;
    const int Px = 2 * M;
    const int pitch = F::kStatic ? ((F::N + 1 + 15) / 16) * 16 : a.pitch;
    float2* tw = bs_sm;
    float2* b0 = bs_sm + Px;
    float2* b1 = b0 + M * ls;
    unsigned char* raw = reinterpret_cast<unsigned char*>(b1 + M * ls);     // 2 * LB * row_bytes, 16-B aligned
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(raw + 2 * (size_t)LB * t.row_bytes);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int NW = PCM_THREADS / 32;

    for (int i = threadIdx.x; i < Px; i += blockDim.x) tw[i] = a.tw[i];
    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // item -> (image, plane, line group); consecutive items share the plane
    auto decode = [&](int w, int& im, int& zp, int& y0) {
        const int g = w % t.n_groups;
        const int r = w / t.n_groups;
        zp = r % a.Pz;
        im = r / a.Pz;
        y0 = g * LB;
    };
    // producer: issue the bulk copies of item w into stage buffer `buf` (thread 0 only)
    auto prefetch = [&](int w, int buf) {
        int im, zp, y0;
        decode(w, im, zp, y0);
        if (zp >= a.Ez || y0 >= a.Ey) return;
        const int nl = min(min(LB, a.Py - y0), a.Ey - y0);
        mbar_expect_tx(&bars[buf], (unsigned int)(nl * t.row_bytes));
        const unsigned char* img = reinterpret_cast<const unsigned char*>(a.img[im]);
        const int sz = a.idx_z[zp];
        for (int l = 0; l < nl; ++l) {
            const size_t row = (size_t)sz * a.dy + a.idx_y[y0 + l];
            tma_bulk_g2s(raw + ((size_t)buf * LB + l) * t.row_bytes, img + row * t.row_bytes, (unsigned int)t.row_bytes,
                         &bars[buf]);
        }
    };

    unsigned int phase[2] = {0u, 0u};
    int it = 0;
    if (threadIdx.x == 0 && (int)blockIdx.x < t.n_items) prefetch(blockIdx.x, 0);
    for (int w = blockIdx.x; w < t.n_items; w += gridDim.x, ++it) {
        const int buf = it & 1;
        int im, zp, y0;
        decode(w, im, zp, y0);
        const int wn = w + gridDim.x;
        if (threadIdx.x == 0 && wn < t.n_items) prefetch(wn, buf ^ 1);
        float2* __restrict__ spec = a.spec[im];
        const size_t rowbase = ((size_t)zp * a.Py + y0) * pitch;
        const int nlines = min(LB, a.Py - y0);
        if (zp >= a.Ez || y0 >= a.Ey) {  // zero padding: no loads were issued for this item
            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            float4* d4 = reinterpret_cast<float4*>(spec + rowbase);
            for (int i = threadIdx.x; i < nlines * (pitch >> 1); i += blockDim.x) d4[i] = z4;
            continue;
        }
        mbar_wait(&bars[buf], phase[buf]);
        phase[buf] ^= 1u;
        const float wz = a.w_z[zp];
        const int e0 = a.ex;
        const unsigned char* rb = raw + (size_t)buf * LB * t.row_bytes;
        // window + pack from the staged rows
        for (int l = wid; l < LB; l += NW) {
            const int yp = y0 + l;
            const bool live = l < nlines && yp < a.Ey;
            const float wy = live ? a.w_y[yp] : 0.f;
            const float gyz = wy * wz;
            const unsigned char* row = rb + (size_t)l * t.row_bytes;
            for (int n = lane; n < M; n += 32) {
                float2 v = make_float2(0.f, 0.f);
                if (live) {
                    const int xp = 2 * n;
                    if (xp >= e0 && xp + 1 < e0 + a.dx) {
                        const int xs = xp - e0;
                        float p0, p1;
                        if (a.dtype == BS_DTYPE_U16) {
                            p0 = (float)reinterpret_cast<const unsigned short*>(row)[xs];
                            p1 = (float)reinterpret_cast<const unsigned short*>(row)[xs + 1];
                        } else if (a.dtype == BS_DTYPE_F32) {
                            p0 = reinterpret_cast<const float*>(row)[xs];
                            p1 = reinterpret_cast<const float*>(row)[xs + 1];
                        } else {
                            p0 = (float)row[xs];
                            p1 = (float)row[xs + 1];
                        }
                        v = make_float2(p0 * gyz, p1 * gyz);
                    } else if (xp < a.Ex) {
                        const float g0 = (a.w_x[xp] * wy) * wz, g1 = (a.w_x[xp + 1] * wy) * wz;
                        const int i0 = a.idx_x[xp], i1 = a.idx_x[xp + 1];
                        float p0, p1;
                        if (a.dtype == BS_DTYPE_U16) {
                            p0 = (float)reinterpret_cast<const unsigned short*>(row)[i0];
                            p1 = (float)reinterpret_cast<const unsigned short*>(row)[i1];
                        } else if (a.dtype == BS_DTYPE_F32) {
                            p0 = reinterpret_cast<const float*>(row)[i0];
                            p1 = reinterpret_cast<const float*>(row)[i1];
                        } else {
                            p0 = (float)row[i0];
                            p1 = (float)row[i1];
                        }
                        v = make_float2(g0 != 0.f ? p0 * g0 : 0.f, g1 != 0.f ? p1 * g1 : 0.f);
                    }
                }
                b0[n * ls + l] = v;
            }
        }
        __syncthreads();
        const float2* res = F::run(b0, b1, tw, a.plan, lshift, ls, 2);
        for (int l = wid; l < nlines; l += NW) {
            float2* srow = spec + rowbase + (size_t)l * pitch;
            for (int k = lane; k < pitch; k += 32) {
                float2 X = make_float2(0.f, 0.f);
                if (k <= M) {
                    const int k0 = (k == M) ? 0 : k;
                    const int k1 = (k == 0 || k == M) ? 0 : M - k;
                    const float2 Zk = res[k0 * ls + l];
                    float2 Zm = res[k1 * ls + l];
                    Zm.y = -Zm.y;
                    const float2 E = make_float2(0.5f * (Zk.x + Zm.x), 0.5f * (Zk.y + Zm.y));
                    const float2 D = make_float2(0.5f * (Zk.x - Zm.x), 0.5f * (Zk.y - Zm.y));
                    const float2 wD = cmulf(tw[k], D);
                    X = make_float2(E.x + wD.y, E.y - wD.x);
                }
                __stcg(srow + k, X);
            }
        }
        __syncthreads();  // b0/b1 and the consumed stage buffer may be overwritten from here on
    }
}

// ------------------------------------------------------------------------------------------
struct XC2RArgs {
    float2* spec;
    int Px, Py, Pz, M, pitch;
    const float2* tw;
    FftPlan plan;
    int lshift;
    float scale;
};

// Warp-private x passes: one warp owns one line at a time (window, FFT, untangle, store) with
// only __syncwarp() between steps; the raw row of the warp's NEXT line is fetched by a 1-D bulk
// TMA copy into the warp's own double buffer (own mbarrier), so there is no block-wide barrier
// in the steady state and the 8 warps of a CTA overlap each other's memory and math phases.
struct XWArgs {
    XR2CArgs x;
    int row_bytes;     // dx * element size; multiple of 16 when use_tma
    int use_tma;
    long long n_lines; // 2 * Pz * Py
};

__device__ __forceinline__ float raw_elem(const unsigned char* row, int dtype, int i) {
    if (dtype == BS_DTYPE_U16) return (float)reinterpret_cast<const unsigned short*>(row)[i];
    if (dtype == BS_DTYPE_F32) return reinterpret_cast<const float*>(row)[i];
    return (float)row[i];
}

template <class F>
__global__ void __launch_bounds__(PCM_THREADS, 4) k_fft_x_r2c_w(const __grid_constant__ XWArgs t) {
    const XR2CArgs& a = t.x;
    const int M = F::kStatic ? F::N : a.M;
    const int Px = 2 * M;
    const int pitch = F::kStatic ? ((F::N + 1 + 15) / 16) * 16 : a.pitch;
    constexpr int NW = PCM_THREADS / 32;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // smem: tw[Px] | per warp: A[M], B[M] | per warp raw[2][row_bytes] | per warp mbar[2]
    float2* tw = bs_sm;
    float2* A = bs_sm + Px + (size_t)wid * 2 * M;
    float2* B = A + M;
    unsigned char* raw = reinterpret_cast<unsigned char*>(bs_sm + Px + (size_t)NW * 2 * M) + (size_t)wid * 2 * t.row_bytes;
    unsigned long long* bars =
        reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(bs_sm + Px + (size_t)NW * 2 * M) +
                                              (size_t)NW * 2 * t.row_bytes) + 2 * wid;
    constexpr int UTW = F::N / 2 + 1;        // untangle twiddles tw[0 .. M/2]
    if constexpr (F::kSmemTw) {
        // the Px-entry table area holds: untangle twiddles | compact per-stage tables (conflict-free reads)
        static_assert(UTW + F::Tw::total <= 2 * F::N, "stage tables must fit the twiddle area");
        for (int i = threadIdx.x; i < UTW; i += blockDim.x) tw[i] = a.tw[i];
        F::Tw::build(tw + UTW, a.tw, threadIdx.x, blockDim.x);
    } else {
        for (int i = threadIdx.x; i < Px; i += blockDim.x) tw[i] = a.tw[i];
    }
    if (t.use_tma && lane == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // static plan: FFT twiddles and the untangle twiddles of this lane live in registers for the whole kernel
    typename F::Tw twr;
    twr.init(F::kSmemTw ? tw + UTW : tw, lane);
    constexpr bool kRegU = F::kStatic && !F::kSmemTw;
    constexpr int UIT = F::kStatic ? (F::N / 2 + 1 + 31) / 32 : 1;
    float2 utw[kRegU ? UIT : 1];
    if constexpr (kRegU) {
#pragma unroll
        for (int i = 0; i < UIT; ++i) utw[i] = tw[min(lane + 32 * i, M)];
    }

    const long long gw = (long long)blockIdx.x * NW + wid, gstride = (long long)gridDim.x * NW;
    const int e0 = a.ex;
    // line -> (image, plane, row); returns the source row index or -1 for an all-zero line
    auto src_row = [&](long long line, int& im, int& zp, int& yp) -> long long {
        yp = (int)(line % a.Py);
        const long long r = line / a.Py;
        zp = (int)(r % a.Pz);
        im = (int)(r / a.Pz);
        if (zp >= a.Ez || yp >= a.Ey) return -1;
        return (long long)a.idx_z[zp] * a.dy + a.idx_y[yp];
    };
    auto prefetch = [&](long long line, int buf) {  // lane 0 only
        int im, zp, yp;
        const long long row = src_row(line, im, zp, yp);
        if (row < 0) return;
        const unsigned char* img = reinterpret_cast<const unsigned char*>(a.img[im]);
        mbar_expect_tx(&bars[buf], (unsigned int)t.row_bytes);
        tma_bulk_g2s(raw + (size_t)buf * t.row_bytes, img + (size_t)row * t.row_bytes, (unsigned int)t.row_bytes, &bars[buf]);
    };

    unsigned int phase0 = 0u, phase1 = 0u;
    int it = 0;
    if (t.use_tma && lane == 0 && gw < t.n_lines) prefetch(gw, 0);
    for (long long line = gw; line < t.n_lines; line += gstride, ++it) {
        const int buf = it & 1;
        if (t.use_tma && lane == 0 && line + gstride < t.n_lines) prefetch(line + gstride, buf ^ 1);
        int im, zp, yp;
        const long long row = src_row(line, im, zp, yp);
        float2* srow = a.spec[im] + ((size_t)zp * a.Py + yp) * pitch;
        if (row < 0) {
            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int i = lane; i < (pitch >> 1); i += 32) reinterpret_cast<float4*>(srow)[i] = z4;
            continue;
        }
        const float wy = a.w_y[yp], wz = a.w_z[zp];
        const float gyz = wy * wz;
        const unsigned char* rrow;
        if (t.use_tma) {
            mbar_wait(&bars[buf], buf ? phase1 : phase0);
            if (buf) phase1 ^= 1u; else phase0 ^= 1u;
            rrow = raw + (size_t)buf * t.row_bytes;
        } else {
            rrow = reinterpret_cast<const unsigned char*>(a.img[im]) + (size_t)row * t.row_bytes;  // global
        }
        if (a.dtype == BS_DTYPE_U16 && !(e0 & 1) && !((size_t)rrow & 3)) {
            // interior pairs are aligned 32-bit words of the staged row
            const unsigned int* r32 = reinterpret_cast<const unsigned int*>(rrow);
            const int n_lo = e0 >> 1, n_hi = (e0 + a.dx) >> 1;   // pairs fully inside [e0, e0 + dx)
            for (int n = lane; n < M; n += 32) {
                float2 v = make_float2(0.f, 0.f);
                if (n >= n_lo && n < n_hi) {
                    const unsigned int w = r32[n - n_lo];
                    v = make_float2((float)(w & 0xffffu) * gyz, (float)(w >> 16) * gyz);
                } else if (2 * n < a.Ex) {
                    const int xp = 2 * n;
                    const float g0 = (a.w_x[xp] * wy) * wz, g1 = (a.w_x[xp + 1] * wy) * wz;
                    const float p0 = raw_elem(rrow, BS_DTYPE_U16, a.idx_x[xp]), p1 = raw_elem(rrow, BS_DTYPE_U16, a.idx_x[xp + 1]);
                    v = make_float2(g0 != 0.f ? p0 * g0 : 0.f, g1 != 0.f ? p1 * g1 : 0.f);
                }
                A[n] = v;
            }
        } else {
            for (int n = lane; n < M; n += 32) {
                float2 v = make_float2(0.f, 0.f);
                const int xp = 2 * n;
                if (xp >= e0 && xp + 1 < e0 + a.dx) {
                    v = make_float2(raw_elem(rrow, a.dtype, xp - e0) * gyz, raw_elem(rrow, a.dtype, xp - e0 + 1) * gyz);
                } else if (xp < a.Ex) {
                    const float g0 = (a.w_x[xp] * wy) * wz, g1 = (a.w_x[xp + 1] * wy) * wz;
                    const float p0 = raw_elem(rrow, a.dtype, a.idx_x[xp]), p1 = raw_elem(rrow, a.dtype, a.idx_x[xp + 1]);
                    v = make_float2(g0 != 0.f ? p0 * g0 : 0.f, g1 != 0.f ? p1 * g1 : 0.f);
                }
                A[n] = v;
            }
        }
        __syncwarp();
        const float2* res = F::run(A, B, tw, twr, a.plan, 2, lane);
        // untangle: X[k] and X[M-k] share E, D and the twiddle (w_{M-k} = -conj(w_k))
        auto untangle = [&](int k, float2 w) {
            const float2 Zk = res[k];
            const float2 Zm = p_mul(res[k == 0 ? 0 : M - k], make_float2(1.f, -1.f));   // conj
            const float2 S = caddf(Zk, Zm), Dd = csubf(Zk, Zm);        // 2E, 2D
            const float2 wD = cmulf(w, Dd);
            __stcg(srow + k, cscale(0.5f, cadd_mi(S, wD)));            // E - i w D
            if (2 * k != M) __stcg(srow + (M - k), p_mul(cadd_pi(S, wD), make_float2(0.5f, -0.5f)));   // conj(E + i w D)
        };
        if (F::kStatic) {
#pragma unroll
            for (int i = 0; i < UIT; ++i) {
                const int k = lane + 32 * i;
                if (2 * k <= M) untangle(k, kRegU ? utw[kRegU ? i : 0] : tw[k]);
            }
        } else {
            for (int k = lane; 2 * k <= M; k += 32) untangle(k, tw[k]);
        }
        for (int k = M + 1 + lane; k < pitch; k += 32) __stcg(srow + k, make_float2(0.f, 0.f));
        __syncwarp();  // A/B and the consumed raw buffer are free again
    }
}

#define XW_MAXV 10   // float2 per lane covering a row of up to 32 * XW_MAXV spectrum entries
template <class F>
__global__ void __launch_bounds__(PCM_THREADS, 3) k_fft_x_c2r_w(const __grid_constant__ XC2RArgs a) {
    const int M = F::kStatic ? F::N : a.M;
    const int Px = 2 * M;
    const int pitch = F::kStatic ? ((F::N + 1 + 15) / 16) * 16 : a.pitch;
    constexpr int NW = PCM_THREADS / 32;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float2* tw = bs_sm;
    float2* A = bs_sm + Px + (size_t)wid * 2 * (M + 1);   // M + 1 entries each
    float2* B = A + (M + 1);
    for (int i = threadIdx.x; i < Px; i += blockDim.x) tw[i] = a.tw[i];
    __syncthreads();
    typename F::Tw twr;
    twr.init(tw, lane);
    constexpr int UIT = F::kStatic ? (F::N / 2 + 1 + 31) / 32 : 1;
    const long long n_lines = (long long)a.Py * a.Pz;
    const long long gw = (long long)blockIdx.x * NW + wid, gstride = (long long)gridDim.x * NW;
    float2 nxt[XW_MAXV];
    auto load_row = [&](long long line) {
        const float2* srow = a.spec + (size_t)line * pitch;
#pragma unroll
        for (int u = 0; u < XW_MAXV; ++u) {
            const int k = lane + 32 * u;
            nxt[u] = (k <= M) ? __ldcg(srow + k) : make_float2(0.f, 0.f);
        }
    };
    if (gw < n_lines) load_row(gw);
    for (long long line = gw; line < n_lines; line += gstride) {
        // spectrum row -> B (conjugated: partial inverse along y,z = conj of forward transforms of conj data)
#pragma unroll
        for (int u = 0; u < XW_MAXV; ++u) {
            const int k = lane + 32 * u;
            if (k <= M) B[k] = make_float2(nxt[u].x, -nxt[u].y);
        }
        __syncwarp();
        if (line + gstride < n_lines) load_row(line + gstride);   // prefetch into registers
        // tangle: A[k] and A[M-k] share E, D and the twiddle (E' = conj E, D' = -conj D, conj w' = -w):
        //   A[k] = conj(E + i O), A[M-k] = (E.x + O.y, E.y - O.x) with O = D conj(w_k)
        auto tangle = [&](int k, float2 wc) {
            const float2 Xk = B[k];
            const float2 Xm = p_mul(B[M - k], make_float2(1.f, -1.f));
            const float2 S = caddf(Xk, Xm), Dd = csubf(Xk, Xm);       // 2E, 2D
            const float2 O = cmulf(Dd, wc);                            // 2 O
            A[k] = p_mul(cadd_pi(S, O), make_float2(0.5f, -0.5f));     // conj(E + i O)
            if (k != 0 && 2 * k != M) A[M - k] = cscale(0.5f, cadd_mi(S, O));   // E - i O = (E.x + O.y, E.y - O.x)
        };
        if (F::kStatic) {
#pragma unroll
            for (int i = 0; i < UIT; ++i) {
                const int k = lane + 32 * i;
                if (2 * k <= M) tangle(k, p_mul(tw[k], make_float2(1.f, -1.f)));   // contiguous table read, conflict-free
            }
        } else {
            for (int k = lane; 2 * k <= M; k += 32) tangle(k, p_mul(tw[k], make_float2(1.f, -1.f)));
        }
        __syncwarp();
        const float2* res = F::run(A, B, tw, twr, a.plan, 2, lane);
        float2* row = a.spec + (size_t)line * pitch;
        for (int n = lane; n < M; n += 32) {
            const float2 r = res[n];
            __stcg(row + n, make_float2(r.x * a.scale, -r.y * a.scale));
        }
        __syncwarp();
    }
}

typedef FftWStatic<270, 2, 9, 6, 5> FftW270;     // register twiddles (c2r: 3 CTAs / SM)
typedef FftWStaticS<270, 2, 9, 6, 5> FftW270S;   // shared-memory stage tables (r2c: 4 CTAs / SM)

// ------------------------------------------------------------------------------------------
// strided passes (y and z)
struct StridedArgs {
    float2* a;
    float2* b;
    long long estride;   // float2 units between consecutive elements along the FFT axis
    long long ostride;   // float2 units between consecutive blockIdx.y
    const float2* tw;
    FftPlan plan;
    int tshift;          // log2(tile width in float2)
    float thresh;        // normalisation threshold (cross-power passes)
};

template <int UNR>
__device__ __forceinline__ void tile_load(float2* dst, const float2* g, long long estride, int N, int tshift) {
    const int vshift = tshift - 1;           // float4 vectors per row = TW/2
    const int vmask = (1 << vshift) - 1;
    const int nvec = N << vshift;
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int i0 = threadIdx.x; i0 < nvec; i0 += blockDim.x * UNR) {
        float4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int i = i0 + u * blockDim.x;
            if (i < nvec) v[u] = __ldcg(reinterpret_cast<const float4*>(g + (long long)(i >> vshift) * estride) + (i & vmask));
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int i = i0 + u * blockDim.x;
            if (i < nvec) d4[i] = v[u];
        }
    }
}

__device__ __forceinline__ void tile_store(float2* g, const float2* src, long long estride, int N, int tshift) {
    const int vshift = tshift - 1;
    const int vmask = (1 << vshift) - 1;
    const int nvec = N << vshift;
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll 4
    for (int i = threadIdx.x; i < nvec; i += blockDim.x)
        __stcg(reinterpret_cast<float4*>(g + (long long)(i >> vshift) * estride) + (i & vmask), s4[i]);
}

// x / |x|, or 0 when |x| < thresh: the one unit-magnitude normalisation of the cross-power passes.  |x|^2 is formed
// from h = x * 2^-46 (exact), so it does not overflow for |x| up to ~1.3e33 (x * x would past ~1.8e19), and above the
// threshold it stays a normal number (thresh^2 * 2^-92 ~ 2e-38 > FLT_MIN): the reciprocal square root needs no
// denormal fix-up, and h / |h| equals x / |x| bit for bit.
__device__ __forceinline__ float rsqrt_ftz(float v) {
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ float2 unit_or_zero(float2 x, float thresh) {
    const float2 h = make_float2(x.x * 0x1p-46f, x.y * 0x1p-46f);
    const float m2 = h.x * h.x + h.y * h.y;
    if (m2 < (thresh * thresh) * 0x1p-92f) return make_float2(0.f, 0.f);   // |x| < threshold
    const float inv = rsqrt_ftz(m2);
    return make_float2(h.x * inv, h.y * inv);
}

// forward FFT in place on (blockIdx.z ? b : a), one tile per CTA (y lengths whose pipelined tiles do not fit)
template <class F>
__global__ void __launch_bounds__(PCM_THREADS, 3) k_fft_strided(const __grid_constant__ StridedArgs a) {
    const int tshift = F::kStatic ? F::LSHIFT : a.tshift;
    const int TW = 1 << tshift, N = F::kStatic ? F::N : a.plan.n;
    const int twpad = (N + 1) & ~1;
    float2* tw = bs_sm;
    float2* B0 = bs_sm + twpad;
    float2* B1 = B0 + (size_t)N * TW;
    const size_t base = (size_t)blockIdx.y * a.ostride + (size_t)blockIdx.x * TW;
    for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = a.tw[i];
    float2* g = (blockIdx.z ? a.b : a.a) + base;
    tile_load<9>(B0, g, a.estride, N, tshift);
    __syncthreads();
    const float2* res = F::run(B0, B1, tw, a.plan, tshift, TW, 1);
    tile_store(g, res, a.estride, N, tshift);
}

// Persistent, software-pipelined variant of k_fft_strided: each CTA walks its tiles with three rotating
// shared-memory buffers; the NEXT tile is pulled in with cp.async (LDGSTS, 16 B per thread and
// request, no register staging) while the current one is transformed and stored.
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct StridedPipeArgs {
    StridedArgs s;
    int tiles_x;     // pitch / TW
    int n_other;     // blockIdx.y extent of the non-persistent kernel
    int n_tiles;     // tiles_x * n_other * n_img
};

template <class F>
__global__ void __launch_bounds__(PCM_THREADS, 2) k_fft_strided_pipe(const __grid_constant__ StridedPipeArgs p) {
    const StridedArgs& a = p.s;
    const int tshift = F::kStatic ? F::LSHIFT : a.tshift;
    const int TW = 1 << tshift, N = F::kStatic ? F::N : a.plan.n;
    const int twpad = (N + 1) & ~1;
    float2* tw = bs_sm;
    float2* B[3];
    B[0] = bs_sm + twpad;
    B[1] = B[0] + (size_t)N * TW;
    B[2] = B[1] + (size_t)N * TW;
    for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = a.tw[i];
    const int vshift = tshift - 1, vmask = (1 << vshift) - 1, nvec = N << vshift;

    auto tile_ptr = [&](int t) -> float2* {
        const int tx = t % p.tiles_x;
        const int r = t / p.tiles_x;
        const int o = r % p.n_other, im = r / p.n_other;
        return (im ? a.b : a.a) + (size_t)o * a.ostride + (size_t)tx * TW;
    };
    auto prefetch = [&](int t, float2* dst) {
        const float2* g = tile_ptr(t);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
            cp_async16(d4 + i, reinterpret_cast<const float4*>(g + (long long)(i >> vshift) * a.estride) + (i & vmask));
        cp_async_commit();
    };

    int t = blockIdx.x;
    if (t < p.n_tiles) prefetch(t, B[0]);
    for (int it = 0; t < p.n_tiles; t += gridDim.x, ++it) {
        float2* cur = B[(2 * it) % 3];
        float2* pong = B[(2 * it + 1) % 3];
        float2* nxt = B[(2 * it + 2) % 3];
        const int tn = t + gridDim.x;
        if (tn < p.n_tiles) {
            prefetch(tn, nxt);
            cp_async_wait<1>();   // everything but the newest group (the next tile) has landed
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float2* res = F::run(cur, pong, tw, a.plan, tshift, TW, 1);
        tile_store(tile_ptr(t), res, a.estride, N, tshift);
        __syncthreads();   // res / cur may be overwritten by the next iteration's prefetch and FFT
    }
}

// Persistent, software-pipelined cross-power pass (z): three tile buffers (so two CTAs still fit an SM), the loads
// are cp.async groups that overlap the transforms:
//   A(t) lands -> FFT A   | B(t) still in flight
//   B(t) lands -> FFT B -> normalise, conj(A) * B
//   B's buffer is free    -> prefetch A(t+1) under the transform of the product
//   the transform's scratch buffer is free -> prefetch B(t+1) under the store and FFT A(t+1)
template <class F>
__global__ void __launch_bounds__(PCM_THREADS, 2) k_fft_xpower_pipe(const __grid_constant__ StridedPipeArgs p) {
    const StridedArgs& a = p.s;
    const int tshift = F::kStatic ? F::LSHIFT : a.tshift;
    const int TW = 1 << tshift, N = F::kStatic ? F::N : a.plan.n;
    const int twpad = (N + 1) & ~1;
    float2* tw = bs_sm;
    float2* bufA = bs_sm + twpad;
    float2* bufB = bufA + (size_t)N * TW;
    float2* pong = bufB + (size_t)N * TW;
    for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = a.tw[i];
    const int vshift = tshift - 1, vmask = (1 << vshift) - 1, nvec = N << vshift;
    auto tile_off = [&](int t) -> size_t {
        const int tx = t % p.tiles_x, o = t / p.tiles_x;
        return (size_t)o * a.ostride + (size_t)tx * TW;
    };
    auto prefetch = [&](const float2* g, float2* dst) {
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
            cp_async16(d4 + i, reinterpret_cast<const float4*>(g + (long long)(i >> vshift) * a.estride) + (i & vmask));
        cp_async_commit();
    };
    int t = blockIdx.x;
    if (t < p.n_tiles) {
        prefetch(a.a + tile_off(t), bufA);
        prefetch(a.b + tile_off(t), bufB);
    }
    for (; t < p.n_tiles; t += gridDim.x) {
        const int tn = t + gridDim.x;
        const bool has_next = tn < p.n_tiles;
        cp_async_wait<1>();            // A(t) landed (B(t) is the newest group)
        __syncthreads();
        float2* rA = F::run(bufA, pong, tw, a.plan, tshift, TW, 1);
        float2* freeA = (rA == bufA) ? pong : bufA;
        cp_async_wait<0>();            // B(t) landed
        __syncthreads();
        float2* rB = F::run(bufB, freeA, tw, a.plan, tshift, TW, 1);
        float2* free2 = (rB == bufB) ? freeA : bufB;
        const int tot = N * TW;
        for (int i = threadIdx.x; i < tot; i += blockDim.x) {
            const float2 x = unit_or_zero(rA[i], a.thresh);
            const float2 y = unit_or_zero(rB[i], a.thresh);
            rA[i] = make_float2(x.x * y.x + x.y * y.y, x.x * y.y - x.y * y.x);  // conj(x) * y
        }
        __syncthreads();
        if (has_next) prefetch(a.a + tile_off(tn), rB);          // rB's buffer is free from here on
        float2* rQ = F::run(rA, free2, tw, a.plan, tshift, TW, 1);
        float2* otherQ = (rQ == rA) ? free2 : rA;
        if (has_next) prefetch(a.b + tile_off(tn), otherQ);      // scratch of the last transform is free
        tile_store(a.a + tile_off(t), rQ, a.estride, N, tshift);
        __syncthreads();               // rQ is read out: it becomes the next iteration's scratch
        bufA = rB; bufB = otherQ; pong = rQ;
    }
}

// ------------------------------------------------------------------------------------------
// Strided passes of the static 540-point plan (540 = 20 x 27, RegFft2): tiles of 540 rows x TC columns, one
// shared-memory exchange and one block barrier per transform.  Persistent CTAs.  The y pass keeps the data in
// registers from the global load to the global store; the next tile's loads go out into the stage-1 registers as
// soon as the current tile's stage 1 has written them to the exchange buffer, so they are in flight under stage 2
// and the stores (a
// register double buffer would need twice the stage-1 registers; a cp.async staging tile would add two
// shared-memory passes per element and cost the occupancy a second 69 KB buffer allows).
//
// TC = 16 (128 B row segments), NT = 320: stage 1 has 27 x 16 = 432 items of 20 points (threads 0..111 take two),
// stage 2 has 20 x 16 = 320 items of 27 points (one per thread).  One CTA per SM (three 69 KB tile buffers in the z
// pass).
#define COL540_TC 16
#define COL540_NT 320
typedef RegFft2<20, 27, COL540_TC, COL540_NT> Col540;      // forward: 20 first, then 27
typedef RegFft2<27, 20, COL540_TC, COL540_NT> Col540Q;     // cross-power product: starts on Col540's output
static_assert(Col540Q::IT1 == Col540::IT2 && Col540Q::I1 == Col540::I2, "product transform must start in registers");

__device__ __forceinline__ void col540_tw(float2* tw, const float2* __restrict__ g) {
    for (int i = threadIdx.x; i < Col540::N; i += blockDim.x) tw[i] = g[i];
}

// ------------------------------------------------------------------------------------------
// Plane hand-off between the two roles of the fused kernel k_fft_xy_col540.  One role (the producer) stores z-planes
// of the spectra, the other (the consumer) transforms them along y as soon as each plane is complete, while the plane
// is still in L2.  Two counters per plane, zeroed before the launch: ready[z] counts the units the producer has stored
// into plane z, done[z] the units the consumer has taken out of it.  The producer stores into plane z only once plane
// z - window is taken, which bounds the data waiting in L2 to about `window` planes whatever the split of the CTAs
// between the roles.  done[] only bounds that residency: the producer never stores into a plane again once it is
// complete, so the consumer may count a unit as soon as it has loaded it.
// Every wait is bounded: when a wait expires, its thread records the kernel's code in *err and the CTA stops
// without writing; the other CTAs see *err and stop as well, and the host turns the code into an error.
#define PCM_HANDOFF_POLLS (1u << 24)
struct Handoff {
    int* ready = nullptr;   // [Pz]; nullptr in the standalone kernels, where every hook below is a no-op
    int* done = nullptr;    // [Pz]
    int* err = nullptr;
    int code = 0;
    int ready_full = 0, done_full = 0;   // units of a whole plane on each counter
    int window = 0;                      // >= 2: a tile's stores may reach into the plane after the one it waits for
};

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// one thread: poll *c until it reaches `full`; false when the poll budget is spent or another wait has expired
__device__ __forceinline__ bool handoff_wait(const int* c, int full, const Handoff& h) {
    unsigned int ns = 32;
    for (unsigned int i = 0; i < PCM_HANDOFF_POLLS; ++i) {
        if (ld_acquire_gpu(c) >= full) {
            __threadfence();   // the whole CTA reads the plane after the barrier that follows
            return true;
        }
        if (*(volatile int*)h.err) return false;
        __nanosleep(ns);
        ns = min(2 * ns, 256u);
    }
    atomicCAS(h.err, 0, h.code);
    return false;
}
// consumer: plane z is complete
__device__ __forceinline__ bool handoff_ready(const Handoff& h, int z) {
    return !h.ready || handoff_wait(h.ready + z, h.ready_full, h);
}
// producer: plane z may be stored into (plane z - window has been read out)
__device__ __forceinline__ bool handoff_window(const Handoff& h, int z) {
    return !h.ready || z < h.window || handoff_wait(h.done + z - h.window, h.done_full, h);
}
// one thread, after a barrier that follows the CTA's stores into plane z: n more units of it are complete
__device__ __forceinline__ void handoff_publish(const Handoff& h, int z, int n) {
    if (!h.ready) return;
    __threadfence();
    atomicAdd(h.ready + z, n);
}
// one thread, once the CTA has loaded n units of plane z
__device__ __forceinline__ void handoff_consume(const Handoff& h, int z, int n) {
    if (h.ready) atomicAdd(h.done + z, n);
}
// f(z, n) for each plane z of Py lines that lines [l0, l1) touch, with the n lines that fall into it
template <class Fn>
__device__ __forceinline__ void for_planes(int l0, int l1, int Py, Fn&& f) {
    for (int z = l0 / Py; z * Py < l1; ++z) f(z, min(l1, (z + 1) * Py) - max(l0, z * Py));
}

// Forward y FFT, in place, of tiles t, t + stride, ... < n_tiles on F (RegFft2<20, 27>), ptr(t) the tile's first
// element.  X0 holds two exchange buffers (one barrier per tile); the next tile's loads go out into the stage-1
// registers once stage 1 has written them out (in the fused roles after the barrier, which carries the hand-off
// wait), and are in flight under stage 2 and the stores.
//   Y_ALONE     k_fft_col540
//   Y_CONSUMER  y role of k_fft_xy_col540: a tile's loads wait for its plane; thread 0 counts a tile as taken
//               after its own stage 1, before it waits for the next tile's plane, so a tile's count never waits on
//               a later plane; the spectra go to DRAM as streaming (evict-first) stores so as not to push the x
//               output that is still waiting out of L2
enum { Y_ALONE, Y_CONSUMER };
template <class F, int MODE, class Ptr>
__device__ __forceinline__ void col540_y_tiles(float2* X0, float2* tw, const float2* __restrict__ tw_g, int t, int stride,
                                               int n_tiles, long long estride, int tiles_per_plane, Ptr ptr,
                                               const Handoff& h) {
    static_assert(F::N == 540, "RegFft2<20, 27>");
    bool ok = true;
    if (MODE == Y_CONSUMER && threadIdx.x == 0 && t < n_tiles) ok = handoff_ready(h, t / tiles_per_plane);
    if (MODE == Y_CONSUMER && __syncthreads_or(!ok)) return;
    typename F::In v;
    if (t < n_tiles) F::load(v, ptr(t), estride);
    col540_tw(tw, tw_g);
    __syncthreads();
    for (int it = 0; t < n_tiles; t += stride, ++it) {
        float2* x = X0 + (it & 1) * F::XSIZE;
        F::stage1(v, x, tw);
        const int tn = t + stride;
        if (MODE == Y_ALONE) {
            if (tn < n_tiles) F::load(v, ptr(tn), estride);
            __syncthreads();
        } else {
            if (threadIdx.x == 0) {
                handoff_consume(h, t / tiles_per_plane, 1);
                if (tn < n_tiles) ok = handoff_ready(h, tn / tiles_per_plane);
            }
            if (__syncthreads_or(!ok)) return;
            if (tn < n_tiles) F::load(v, ptr(tn), estride);   // the next tile's plane is complete from here on
        }
        F::stage2(x, [&](const float2 (&w)[27], int, int k1, int c) {
            float2* g = ptr(t);
            if (MODE == Y_CONSUMER) {
                float2* p = g + (long long)k1 * estride + c;
#pragma unroll
                for (int k2 = 0; k2 < 27; ++k2) __stcs(p + (long long)(20 * k2) * estride, w[k2]);
            } else {
                F::store(w, g, estride, k1, c);
            }
        });
    }
}

// forward y FFT in place, tiles of both spectra (p.n_tiles = tiles_x * n_other * n_img)
__global__ void __launch_bounds__(COL540_NT, 1) k_fft_col540(const __grid_constant__ StridedPipeArgs p) {
    const StridedArgs& a = p.s;
    float2* tw = bs_sm;
    auto tile_ptr = [&](int t) -> float2* {
        const int tx = t % p.tiles_x, r = t / p.tiles_x;
        const int o = r % p.n_other, im = r / p.n_other;
        return (im ? a.b : a.a) + (size_t)o * a.ostride + (size_t)tx * COL540_TC;
    };
    col540_y_tiles<Col540, Y_ALONE>(bs_sm + Col540::N, tw, a.tw, blockIdx.x, gridDim.x, p.n_tiles, a.estride, 1, tile_ptr,
                                    Handoff());
}

// z cross-power: forward z FFT of A and B, unit-magnitude normalisation and conj(A) * B, then the forward FFT of
// the product as RegFft2<27, 20>, which starts on the registers holding the product.
//
// The tiles reach shared memory by tensor-map TMA copies issued by one thread and completing on the buffer's
// mbarrier, so a load is in flight from the moment its buffer is released until the tile needs it, with no registers
// held for it.  Three 69 KB buffers: B always lands in buffer 1, A alternates between buffers 0 and 2.  Per tile t,
// with A(t) in XA, B(t) landing in XB and XZ free:
//   A: stage 1 in place in XA | barrier | copy A(t+1) into XZ, stage 2 in place (the spectrum stays in XA)
//   B: stage 1 in place in XB | barrier | stage 2 with the normalisation and conj(A) * B into registers
//   barrier (XA, XB read out) | copy B(t+1) into XB, product stage 1 into XA | barrier | product stage 2 + stores
// so A(t+1) has five phases to land and B(t+1) four.  XA becomes the next tile's free buffer.
//
// A tile is 540 rows of 128 B, one z-stride apart.  As 1-D bulk copies that is 1080 copies per tile pair, and the
// copy engine's per-copy cost made the pass 2.8x slower than register loads (H100 80GB HBM3, 700 W).  A 3-D tensor map
// of each spectrum ([Pz][Py][2 pitch] floats, encoded per launch) moves the tile in COL540_ZBOXES boxes of
// 32 floats x 1 x 180 rows.
#define COL540_ZBOXES 3
static_assert(Col540::N % COL540_ZBOXES == 0 && Col540::N / COL540_ZBOXES <= 256, "a TMA box has at most 256 rows");
struct XpowerCol540Args {
    CUtensorMap tm[2];   // spectra A and B
    StridedPipeArgs p;
};

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int x, int y, int z, unsigned long long* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(dst)), "l"(tm), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
        : "memory");
}

__global__ void __launch_bounds__(COL540_NT, 1) k_fft_xpower_col540(const __grid_constant__ XpowerCol540Args P) {
    const StridedPipeArgs& p = P.p;
    const StridedArgs& a = p.s;
    float2* X0 = bs_sm;   // the copies need 128-byte aligned targets: buffers first
    float2* tw = X0 + 3 * Col540::XSIZE;
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(tw + Col540::N);
    auto tile_off = [&](int t) -> size_t {
        return (size_t)(t / p.tiles_x) * a.ostride + (size_t)(t % p.tiles_x) * COL540_TC;
    };
    // thread 0: copy tile t of spectrum im into buffer b.  The fence orders the generic-proxy accesses to b before
    // the barrier that released it ahead of the async-proxy writes of the copy.
    auto fetch = [&](int im, int t, int b) {
        constexpr int rows = Col540::N / COL540_ZBOXES;
        fence_proxy_async_smem();
        mbar_expect_tx(&bars[b], Col540::XSIZE * sizeof(float2));
        float2* dst = X0 + b * Col540::XSIZE;
        const int x = (t % p.tiles_x) * 2 * COL540_TC, y = t / p.tiles_x;
#pragma unroll
        for (int k = 0; k < COL540_ZBOXES; ++k) tma_load_3d(dst + k * rows * COL540_TC, &P.tm[im], x, y, k * rows, &bars[b]);
    };
    if (threadIdx.x == 0) {
        for (int b = 0; b < 3; ++b) mbar_init(&bars[b], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    col540_tw(tw, a.tw);
    __syncthreads();
    int t = blockIdx.x;
    if (threadIdx.x == 0 && t < p.n_tiles) {
        fetch(0, t, 0);
        fetch(1, t, 1);
    }
    int ia = 0;                // A's buffer; the free one is 2 - ia
    unsigned int phase = 0u;   // bit b: parity of bars[b]'s next phase (the roles rotate, so it is kept per buffer)
    Col540::In v;
    Col540Q::In q;   // q[u] = product column of Col540's stage-2 item u
    for (; t < p.n_tiles; t += gridDim.x, ia = 2 - ia) {
        const int tn = t + gridDim.x;
        float2* XA = X0 + ia * Col540::XSIZE;
        float2* XB = X0 + Col540::XSIZE;
        mbar_wait(&bars[ia], (phase >> ia) & 1u);
        phase ^= 1u << ia;
        Col540::load_shared(v, XA);
        Col540::stage1(v, XA, tw);
        __syncthreads();   // also: the previous tile's product stage 2 has read XZ out
        if (threadIdx.x == 0 && tn < p.n_tiles) fetch(0, tn, 2 - ia);
        Col540::stage2(XA, [&](const float2 (&w)[27], int, int k1, int c) {
            float2* s = Col540::slot(XA, k1, c);
#pragma unroll
            for (int k2 = 0; k2 < 27; ++k2) s[k2 * COL540_TC] = w[k2];
        });
        mbar_wait(&bars[1], (phase >> 1) & 1u);
        phase ^= 2u;
        Col540::load_shared(v, XB);
        Col540::stage1(v, XB, tw);
        __syncthreads();
        Col540::stage2(XB, [&](const float2 (&w)[27], int u, int k1, int c) {
            const float2* s = Col540::slot(XA, k1, c);
#pragma unroll
            for (int k2 = 0; k2 < 27; ++k2) {
                const float2 x = unit_or_zero(s[k2 * COL540_TC], a.thresh);
                const float2 y = unit_or_zero(w[k2], a.thresh);
                q[u][k2] = make_float2(x.x * y.x + x.y * y.y, x.x * y.y - x.y * y.x);  // conj(x) * y
            }
        });
        __syncthreads();
        if (threadIdx.x == 0 && tn < p.n_tiles) fetch(1, tn, 1);
        Col540Q::stage1(q, XA, tw);
        __syncthreads();
        float2* g = a.a + tile_off(t);
        Col540Q::stage2(XA, [&](const float2 (&w)[20], int, int k1, int c) { Col540Q::store(w, g, a.estride, k1, c); });
    }
}

// ------------------------------------------------------------------------------------------
// x passes of the 540-point plan on Col540, two real lines per complex transform.  A tile's 16 columns are 16
// line pairs, so one RegFft2<20, 27> tile transform does the work of 32 real 540-point lines.  Stage 2 writes the
// transform in natural order into Y[c * COL540_XLP + k]; COL540_XLP is odd, so the 16 columns a half-warp writes
// fall on distinct banks, and the rows read back out of Y are contiguous.
//
// 448 threads (14 warps), not the 320 of the y / z passes: each thread holds one of the 432 stage-1 items instead of
// 112 threads holding two while the other 208 wait at the barrier, and the extra warps hide the shared-memory
// latency of building the points.  113-116 registers, no spills (the 146-register cap of 448 threads).  At 320 threads
// the r2c pass took 1.06 ms per bench pair, at 448 0.81 (H100 80GB HBM3, 700 W).
#define COL540_XLP 541
#define COL540_SP 546   // c2r: float2 between staged row pairs (2 x 272 + 2: pair c starts 2c banks further on)
#define COL540X_NT 448
typedef RegFft2<20, 27, COL540_TC, COL540X_NT> Col540X;
static_assert(Col540X::IT1 == 1 && Col540X::IT2 == 1, "one item per thread in each stage");

// Forward x pass of uint16 crops.  Column c of tile t is the line position L = 16 t + c (L = zp Py + yp) of both
// images: z[n] = a[n] + i b[n], with a, b the blended mirrored extension of the two crops' row (the same idx / w rule
// as k_fft_x_r2c_w).  With Z = FFT540(z) the two half spectra are
//   A[k] = (Z[k] + conj Z[540 - k]) / 2,   B[k] = (Z[k] - conj Z[540 - k]) / 2i,   k = 0..270.
// A line whose windowed samples are all zero gets an exactly zero spectrum, as it does from a one-line transform,
// rather than the partner's rounding noise.  The raw rows of tile t+1 are staged by 16-byte cp.async copies (rows
// 16-byte aligned) while tile t is transformed.
// Per tile: stage-1 load from the staged rows, stage 1 into X | barrier | stage 2 into Y | barrier (Y complete, the
// next tile's rows landed) | separation and whole-row stores from Y.
struct XR2CCol540Args {
    XR2CArgs x;
    int row_bytes;    // dx * 2, a multiple of 16
    int raw_stride;   // bytes between staged rows: row_bytes padded so that 16 rows fall on 8 different banks
    int n_tiles;      // ceil(Py * Pz / 16)
};

// Tiles t, t + stride, ... of the pass.  As the producer of k_fft_xy_col540, a tile's stores wait for the window of
// the last plane they reach, and the tile's lines are published per plane at the next tile's B1 (the last tile's
// after a barrier of its own).
__device__ __forceinline__ void x_r2c_col540_tiles(const XR2CCol540Args& P, int t, int stride, const Handoff& h) {
    const XR2CArgs& a = P.x;
    constexpr int TC = COL540_TC, N = Col540X::N, pitch = 272;
    float2* X = bs_sm;
    float2* Y = X + Col540X::XSIZE;
    float2* tw = Y + TC * COL540_XLP;
    int2* xw = reinterpret_cast<int2*>(tw + N);   // (idx_x, w_x bits) per padded x position
    int* nz = reinterpret_cast<int*>(xw + N);     // [buffer][image][16 lines]: the windowed line has a nonzero sample
    unsigned char* raw = reinterpret_cast<unsigned char*>(nz + 4 * TC);   // [buffer][image][16 lines][raw_stride]
    const int n_lines = a.Py * a.Pz;
    const int chunks = P.row_bytes >> 4;
    // all threads: stage the rows of tile t into raw buffer b.  TPR threads per (image, line) row, so each thread
    // looks up one source row per tile (the memory clobber of each copy would serialise per-chunk lookups); all-zero
    // lines are not read, so not copied.
    constexpr int TPR = COL540X_NT / (2 * TC);
    static_assert(COL540X_NT % (2 * TC) == 0, "whole rows per thread group");
    auto stage = [&](int t, int b) {
        const int im = threadIdx.x / (TPR * TC), l = (threadIdx.x / TPR) % TC;
        const int L = t * TC + l;
        const int zp = L / a.Py, yp = L - zp * a.Py;
        if (L < n_lines && zp < a.Ez && yp < a.Ey) {
            const size_t row = (size_t)__ldg(a.idx_z + zp) * a.dy + __ldg(a.idx_y + yp);
            const unsigned char* src = reinterpret_cast<const unsigned char*>(a.img[im]) + row * P.row_bytes;
            unsigned char* dst = raw + ((size_t)(b * 2 + im) * TC + l) * P.raw_stride;
            for (int ch = threadIdx.x % TPR; ch < chunks; ch += TPR) cp_async16(dst + ch * 16, src + ch * 16);
        }
        cp_async_commit();
    };
    for (int i = threadIdx.x; i < N; i += COL540X_NT) {
        tw[i] = a.tw[i];
        xw[i] = make_int2(a.idx_x[i], __float_as_int(a.w_x[i]));
    }
    if (threadIdx.x < 4 * TC) nz[threadIdx.x] = 0;
    if (t < P.n_tiles) stage(t, 0);
    cp_async_wait<0>();
    __syncthreads();
    const int c = threadIdx.x % TC;   // this thread's column in both of its stage-1 items and its stage-2 item
    auto publish = [&](int tp) {      // thread 0, after a barrier that follows tile tp's stores
        for_planes(tp * TC, min(tp * TC + TC, n_lines), a.Py, [&](int z, int n) { handoff_publish(h, z, n); });
    };
    int it = 0;
    for (; t < P.n_tiles; t += stride, ++it) {
        const int b = it & 1;
        const int L = t * TC + c;
        const int zp = L / a.Py, yp = L - zp * a.Py;
        const bool live = L < n_lines && zp < a.Ez && yp < a.Ey;
        const float wy = live ? __ldg(a.w_y + yp) : 0.f, wz = live ? __ldg(a.w_z + zp) : 0.f;
        if (t + stride < P.n_tiles) stage(t + stride, b ^ 1);   // buffer b^1 was read before the last B1
        const unsigned short* ra = reinterpret_cast<const unsigned short*>(raw + ((size_t)b * 2 * TC + c) * P.raw_stride);
        const unsigned short* rb = reinterpret_cast<const unsigned short*>(raw + ((size_t)(b * 2 + 1) * TC + c) * P.raw_stride);
        Col540X::In v;
        bool nza = false, nzb = false;
#pragma unroll
        for (int u = 0; u < Col540X::IT1; ++u) {
            if (!Col540X::live1(u)) continue;
            const int n2 = (threadIdx.x + u * COL540X_NT) / TC;
#pragma unroll
            for (int n1 = 0; n1 < 20; ++n1) {
                float2 z = make_float2(0.f, 0.f);
                if (live) {
                    const int2 e = xw[27 * n1 + n2];
                    const float g = (__int_as_float(e.y) * wy) * wz;
                    if (g != 0.f) z = make_float2((float)ra[e.x] * g, (float)rb[e.x] * g);
                }
                nza |= z.x != 0.f;
                nzb |= z.y != 0.f;
                v[u][n1] = z;
            }
        }
        if (nza) nz[(b * 2) * TC + c] = 1;
        if (nzb) nz[(b * 2 + 1) * TC + c] = 1;
        Col540X::stage1(v, X, tw);
        __syncthreads();   // B1: X complete; the previous tile's separation has read Y and nz[b ^ 1] out
        if (threadIdx.x == 0 && it) publish(t - stride);
        if (threadIdx.x < 2 * TC) nz[(b ^ 1) * 2 * TC + threadIdx.x] = 0;
        Col540X::stage2(X, [&](const float2 (&w)[27], int, int k1, int cc) {
            float2* y = Y + cc * COL540_XLP + k1;
#pragma unroll
            for (int k2 = 0; k2 < 27; ++k2) y[20 * k2] = w[k2];
        });
        cp_async_wait<0>();
        bool ok = true;
        if (threadIdx.x == 0) ok = handoff_window(h, (min(t * TC + TC, n_lines) - 1) / a.Py);
        // B2: Y complete (X free again), this thread's and every other thread's next rows landed
        if (__syncthreads_or(!ok)) return;
        for (int j = threadIdx.x; j < TC * pitch; j += COL540X_NT) {
            const int l = j / pitch, k = j - l * pitch;
            const int Lj = t * TC + l;
            if (Lj >= n_lines) break;   // j only grows
            float2 A = make_float2(0.f, 0.f), B = A;
            if (k <= N / 2) {
                const float2 Zk = Y[l * COL540_XLP + k], Zm = Y[l * COL540_XLP + (k ? N - k : 0)];
                if (nz[(b * 2) * TC + l]) A = make_float2(0.5f * (Zk.x + Zm.x), 0.5f * (Zk.y - Zm.y));
                if (nz[(b * 2 + 1) * TC + l]) B = make_float2(0.5f * (Zk.y + Zm.y), -0.5f * (Zk.x - Zm.x));
            }
            __stcg(a.spec[0] + (size_t)Lj * pitch + k, A);
            __stcg(a.spec[1] + (size_t)Lj * pitch + k, B);
        }
    }
    if (h.ready && it) {
        __syncthreads();
        if (threadIdx.x == 0) publish(t - stride);
    }
}

__global__ void __launch_bounds__(COL540X_NT, 1) k_fft_x_r2c_col540(const __grid_constant__ XR2CCol540Args P) {
    x_r2c_col540_tiles(P, blockIdx.x, gridDim.x, Handoff());
}

// Inverse x pass, in place: a tile is 32 consecutive spectrum rows (16 pairs of lines), staged by one 1-D bulk copy
// per pair into rows of COL540_SP float2.  Column c transforms
//   W[n] = S_2c[n] - i S_2c+1[n],   S[n] = s[n] (n <= 270), conj s[540 - n] (n > 270)
// for the two stored half spectra s, i.e. conj of Z = X_2c + i X_2c+1 with X = conj s the spectra the pass inverts.
// FFT(W) = conj(540 ifft(Z)), so with R = FFT(W) the real lines are x_2c = R.x / (Px Py Pz) and
// x_2c+1 = -R.y / (Px Py Pz).  The imaginary parts of bins 0 and 270 are dropped, as a C2R transform does: they
// would otherwise leak into the partner line.  A line whose (kept) spectrum is all zero is stored as exact zeros.
// After stage 1 the staged pair rows are free and stage 2 writes R there
// in natural order, from which whole output rows are stored.
struct XC2RCol540Args {
    XC2RArgs x;
    int n_tiles;   // ceil(Py * Pz / 32)
};

__global__ void __launch_bounds__(COL540X_NT, 1) k_fft_x_c2r_col540(const __grid_constant__ XC2RCol540Args P) {
    const XC2RArgs& a = P.x;
    constexpr int TC = COL540_TC, N = Col540X::N, M = N / 2, pitch = 272;
    static_assert(TC * COL540_XLP <= TC * COL540_SP && COL540_SP >= 2 * pitch && COL540_SP % 2 == 0, "pair rows");
    float2* S0 = bs_sm;   // two staging buffers of TC * COL540_SP (bulk-copy targets: first)
    float2* X = S0 + 2 * TC * COL540_SP;
    float2* tw = X + Col540X::XSIZE;
    int* nz = reinterpret_cast<int*>(tw + N);   // [buffer][32 rows]: the row has a nonzero input
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(nz + 4 * TC);
    const int n_lines = a.Py * a.Pz;
    // warp 0: copy the row pairs of tile t into buffer b, one bulk copy per pair (lane c)
    auto fetch = [&](int t, int b) {
        const int rows = min(2 * TC, n_lines - t * 2 * TC);
        const int lane = threadIdx.x;
        if (lane == 0) mbar_expect_tx(&bars[b], (unsigned int)(rows * pitch * sizeof(float2)));
        __syncwarp();
        const int r0 = 2 * lane;
        if (lane < TC && r0 < rows) {
            fence_proxy_async_smem();
            tma_bulk_g2s(S0 + (size_t)(b * TC + lane) * COL540_SP, a.spec + ((size_t)t * 2 * TC + r0) * pitch,
                         (unsigned int)(min(2, rows - r0) * pitch * sizeof(float2)), &bars[b]);
        }
    };
    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    col540_tw(tw, a.tw);
    if (threadIdx.x < 4 * TC) nz[threadIdx.x] = 0;
    __syncthreads();
    int t = blockIdx.x;
    if (threadIdx.x < 32 && t < P.n_tiles) fetch(t, 0);
    const int c = threadIdx.x % TC;
    const float s = 0.5f * a.scale;   // a.scale = 1 / (M Py Pz)
    unsigned int phase = 0u;
    for (int it = 0; t < P.n_tiles; t += gridDim.x, ++it) {
        const int b = it & 1;
        float2* Sb = S0 + (size_t)b * TC * COL540_SP;
        mbar_wait(&bars[b], (phase >> b) & 1u);
        phase ^= 1u << b;
        const int r = t * 2 * TC + 2 * c;   // this column's first row
        const bool la = r < n_lines, lb = r + 1 < n_lines;
        const float2* sa = Sb + c * COL540_SP;
        const float2* sb = sa + pitch;
        Col540X::In v;
        bool nzp = false, nzq = false;
#pragma unroll
        for (int u = 0; u < Col540X::IT1; ++u) {
            if (!Col540X::live1(u)) continue;
            const int n2 = (threadIdx.x + u * COL540X_NT) / TC;
#pragma unroll
            for (int n1 = 0; n1 < 20; ++n1) {
                // n = 27 n1 + n2 <= 270 exactly for n1 < 10 and for (n1, n2) = (10, 0)
                float2 p, q;
                if (n1 < 10) {
                    p = sa[27 * n1 + n2];
                    q = sb[27 * n1 + n2];
                    if (n1 == 0 && n2 == 0) p.y = q.y = 0.f;
                } else if (n1 == 10) {
                    const int m = n2 ? M - n2 : M;
                    p = sa[m];
                    q = sb[m];
                    p.y = n2 ? -p.y : 0.f;
                    q.y = n2 ? -q.y : 0.f;
                } else {
                    p = sa[N - 27 * n1 - n2];
                    q = sb[N - 27 * n1 - n2];
                    p.y = -p.y;
                    q.y = -q.y;
                }
                if (!la) p = make_float2(0.f, 0.f);
                if (!lb) q = make_float2(0.f, 0.f);
                nzp |= p.x != 0.f || p.y != 0.f;
                nzq |= q.x != 0.f || q.y != 0.f;
                v[u][n1] = make_float2(p.x + q.y, p.y - q.x);   // p - i q
            }
        }
        if (nzp) nz[b * 2 * TC + 2 * c] = 1;
        if (nzq) nz[b * 2 * TC + 2 * c + 1] = 1;
        Col540X::stage1(v, X, tw);
        __syncthreads();   // B1: X complete, Sb read out; the previous tile's stores have read S[b^1], nz[b^1] out
        if (threadIdx.x < 32 && t + (int)gridDim.x < P.n_tiles) fetch(t + gridDim.x, b ^ 1);
        if (threadIdx.x >= 32 && threadIdx.x < 64) nz[(b ^ 1) * 2 * TC + threadIdx.x - 32] = 0;
        Col540X::stage2(X, [&](const float2 (&w)[27], int, int k1, int cc) {
            float2* y = Sb + cc * COL540_XLP + k1;
#pragma unroll
            for (int k2 = 0; k2 < 27; ++k2) y[20 * k2] = w[k2];
        });
        __syncthreads();   // B2: R complete in Sb (X free again)
        for (int j = threadIdx.x; j < 2 * TC * M; j += COL540X_NT) {
            const int rr = j / M, q = j - rr * M;   // output row t * 32 + rr, floats 2q, 2q + 1
            if (t * 2 * TC + rr >= n_lines) break;
            const float2* y = Sb + (rr >> 1) * COL540_XLP + 2 * q;
            const float2 r0 = y[0], r1 = y[1];
            float2 o = (rr & 1) ? make_float2(-r0.y * s, -r1.y * s) : make_float2(r0.x * s, r1.x * s);
            if (!nz[b * 2 * TC + rr]) o = make_float2(0.f, 0.f);
            __stcg(a.spec + ((size_t)t * 2 * TC + rr) * pitch + q, o);
        }
    }
}

// ------------------------------------------------------------------------------------------
// The forward x and y passes in one persistent kernel, for Px = Py = 540.  The y transform of a z-plane needs only
// that plane's x output, so instead of one kernel per axis, with a round trip of both spectra through DRAM in
// between, the CTAs split into two roles that run concurrently and hand each plane over through L2 (Handoff above):
// CTAs [0, kx) run k_fft_x_r2c_col540's tiles (16 lines each, ascending line order, which is plane order) and publish
// the lines each tile stores per plane; the others run y tiles (540 rows x 16 columns) plane-major: the 17 column
// tiles of A and of B of plane z, then plane z + 1.  A y tile waits until its plane has all Py lines.
// The y role runs Col540X (RegFft2<20, 27> on 448 threads, one stage-1 item per thread): each item computes what
// k_fft_col540's does, so the spectra are bit-identical to the five-pass chain's.  It uses the x role's largest
// shared-memory regions as its two exchange buffers.
// Forward progress: all CTAs are co-resident (cooperative launch, one CTA per SM).  Each role takes its tiles in
// ascending plane order.  A y tile waits only on x tiles of its own plane (its count in done[] waits on nothing), and
// an x tile waits only on y tiles `window` >= 2 planes behind the last plane it stores into.  So the lowest plane p
// that is not yet taken can always proceed: the x tiles that reach into p (at most into p + 1) wait on planes below p,
// and every earlier tile of each CTA is in a plane no higher.
// The inverse pair (y, then x C2R) fused the same way measured slower than the two kernels (DESIGN.md), so it
// stays two launches.
struct XYCol540Args {
    XR2CCol540Args x;
    const float2* tw_y;
    int kx;   // CTAs of the x role
    Handoff h;
};

__global__ void __launch_bounds__(COL540X_NT, 1) k_fft_xy_col540(const __grid_constant__ XYCol540Args P) {
    if ((int)blockIdx.x < P.kx) {
        x_r2c_col540_tiles(P.x, blockIdx.x, P.kx, P.h);
        return;
    }
    const XR2CArgs& a = P.x.x;
    float2* X0 = bs_sm;                                           // r2c's X and Y regions
    float2* tw = X0 + Col540X::XSIZE + COL540_TC * COL540_XLP;   // r2c's twiddle region
    static_assert(COL540_TC * COL540_XLP >= Col540X::XSIZE, "exchange buffers");
    const int tiles_x = a.pitch / COL540_TC, per_plane = 2 * tiles_x;
    const long long ostride = (long long)a.Py * a.pitch;
    auto ptr = [&](int u) -> float2* {
        const int z = u / per_plane, j = u - z * per_plane, im = j / tiles_x;
        return a.spec[im] + z * ostride + (j - im * tiles_x) * COL540_TC;
    };
    col540_y_tiles<Col540X, Y_CONSUMER>(X0, tw, P.tw_y, blockIdx.x - P.kx, gridDim.x - P.kx, a.Pz * per_plane, a.pitch,
                                        per_plane, ptr, P.h);
}


// ------------------------------------------------------------------------------------------
// x pass, complex -> real, in place

template <class F>
__global__ void __launch_bounds__(PCM_THREADS) k_fft_x_c2r(const __grid_constant__ XC2RArgs a) {
    const int M = F::kStatic ? F::N : a.M;
    const int lshift = F::kStatic ? F::LSHIFT : a.lshift;
    const int LB = 1 << lshift, ls = LB + 1;
    const int Px = 2 * M;
    const int pitch = F::kStatic ? ((F::N + 1 + 15) / 16) * 16 : a.pitch;
    float2* tw = bs_sm;
    float2* T0 = bs_sm + Px;                 // (M+1) * ls
    float2* T1 = T0 + (size_t)(M + 1) * ls;  // M * ls
    const int zp = blockIdx.y, y0 = blockIdx.x * LB;
    const size_t rowbase = ((size_t)zp * a.Py + y0) * pitch;
    const int nlines = min(LB, a.Py - y0);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int NW = PCM_THREADS / 32;
    for (int i = threadIdx.x; i < Px; i += blockDim.x) tw[i] = a.tw[i];
    for (int l = wid; l < LB; l += NW) {
        const float2* srow = a.spec + rowbase + (size_t)l * pitch;
        for (int k0 = 0; k0 <= M; k0 += 32 * XR_UNROLL) {
            float2 v[XR_UNROLL];
#pragma unroll
            for (int u = 0; u < XR_UNROLL; ++u) {
                const int k = k0 + u * 32 + lane;
                v[u] = make_float2(0.f, 0.f);
                if (l < nlines && k <= M) v[u] = __ldcg(srow + k);
            }
#pragma unroll
            for (int u = 0; u < XR_UNROLL; ++u) {
                const int k = k0 + u * 32 + lane;
                // partial inverse along y,z = conj of the forward transforms of conj data
                if (k <= M) T0[k * ls + l] = make_float2(v[u].x, -v[u].y);
            }
        }
    }
    __syncthreads();
    for (int item = threadIdx.x; item < M * LB; item += blockDim.x) {
        const int k = item >> lshift, l = item & (LB - 1);
        const float2 Xk = T0[k * ls + l];
        float2 Xm = T0[(M - k) * ls + l];
        Xm.y = -Xm.y;
        const float2 E = make_float2(0.5f * (Xk.x + Xm.x), 0.5f * (Xk.y + Xm.y));
        const float2 D = make_float2(0.5f * (Xk.x - Xm.x), 0.5f * (Xk.y - Xm.y));
        float2 w = tw[k];
        w.y = -w.y;  // e^{+2 pi i k / P}
        const float2 O = cmulf(D, w);
        // Z = E + i*O ; store conj(Z) (inverse via forward transform of the conjugate)
        T1[k * ls + l] = make_float2(E.x - O.y, -(E.y + O.x));
    }
    __syncthreads();
    const float2* res = F::run(T1, T0, tw, a.plan, lshift, ls, 2);
    for (int l = wid; l < nlines; l += NW) {
        float2* row = a.spec + rowbase + (size_t)l * pitch;
        for (int n = lane; n < M; n += 32) {
            const float2 r = res[n * ls + l];
            __stcg(row + n, make_float2(r.x * a.scale, -r.y * a.scale));
        }
    }
}

// ------------------------------------------------------------------------------------------
// peak search: periodic axis-neighbour local maxima, top-K per CTA
struct PeakEntry {
    float val;
    int pad;
    long long idx;
};

struct PeakArgs {
    const float* pcm;
    int Px, Py, Pz;
    long long rowpitch;  // floats (multiple of 4, >= Px rounded up to 4)
    int K;
    PeakEntry* out;      // gridDim.x * K
};

__device__ __forceinline__ bool peak_better(float v, long long i, float v2, long long i2) {
    return v > v2 || (v == v2 && i < i2);
}

// A warp streams one row at a time with PK_UNROLL float4 loads in flight per lane.  The warp
// keeps ONE sorted top-K list in registers (lane i holds the i-th best; K <= 32) and its K-th
// value as a warp-uniform threshold, so after a few rows almost every voxel is rejected by a
// single compare; only survivors fetch their six periodic neighbours and are inserted with a
// ballot + shuffle shift.  Per-CTA merge of the 8 warp lists, then K entries per CTA go out.
#define PK_UNROLL 5

struct WarpTopK {
    float v;        // lane i: value of the i-th best (or -inf)
    long long i;    // its linear index (or LLONG_MAX)
    float thr;      // warp-uniform: value of the K-th best (-inf until the list is full)
};

__device__ __forceinline__ void warp_topk_insert(WarpTopK& t, int K, float nv, long long ni, int lane) {
    // rank of the new entry = number of current entries that are better
    const bool mine_better = peak_better(t.v, t.i, nv, ni);
    const unsigned better = __ballot_sync(0xffffffffu, mine_better && lane < K);
    const int pos = __popc(better);
    if (pos >= K) return;  // warp-uniform
    const float upv = __shfl_up_sync(0xffffffffu, t.v, 1);
    const long long upi = __shfl_up_sync(0xffffffffu, t.i, 1);
    if (lane == pos) { t.v = nv; t.i = ni; }
    else if (lane > pos && lane < K) { t.v = upv; t.i = upi; }
    t.thr = __shfl_sync(0xffffffffu, t.v, K - 1);
}

__global__ void __launch_bounds__(PCM_THREADS) k_peaks(const __grid_constant__ PeakArgs a) {
    const int K = a.K;
    const long long nrows = (long long)a.Py * a.Pz;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int NW = PCM_THREADS / 32;
    const int nvec = (a.Px + 3) >> 2;
    WarpTopK top;
    top.v = -INFINITY;
    top.i = 0x7fffffffffffffffLL;
    top.thr = -INFINITY;
    for (long long row = (long long)blockIdx.x * NW + wid; row < nrows; row += (long long)gridDim.x * NW) {
        const float* rp = a.pcm + row * a.rowpitch;
        const float4* rp4 = reinterpret_cast<const float4*>(rp);
        const int z = (int)(row / a.Py), y = (int)(row - (long long)z * a.Py);
        for (int v0 = 0; v0 < nvec; v0 += 32 * PK_UNROLL) {
            float4 q[PK_UNROLL];
#pragma unroll
            for (int u = 0; u < PK_UNROLL; ++u) {
                const int vi = v0 + u * 32 + lane;
                q[u] = vi < nvec ? __ldcs(rp4 + vi) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            }
            // phase 1 (unrolled, tiny): which of my 4 * PK_UNROLL values reach the warp threshold?
            unsigned int mask = 0u;
#pragma unroll
            for (int u = 0; u < PK_UNROLL; ++u) {
                const int vi = v0 + u * 32 + lane;
                const float c4[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c4[c] >= top.thr && c4[c] > -INFINITY && 4 * vi + c < a.Px) mask |= 1u << (4 * u + c);
            }
            // phase 2 (rolled, rare): neighbour test + insertion, one candidate per lane per round
            while (__any_sync(0xffffffffu, mask != 0u)) {
                bool cand = mask != 0u;
                int x = 0;
                float v = -INFINITY;
                if (cand) {
                    const int b = __ffs(mask) - 1;
                    mask &= mask - 1u;
                    x = 4 * (v0 + (b >> 2) * 32 + lane) + (b & 3);
                    v = rp[x];
                    cand = v >= top.thr;   // the threshold may have risen since phase 1
                    if (cand) cand = !(v < rp[x == 0 ? a.Px - 1 : x - 1] || v < rp[x == a.Px - 1 ? 0 : x + 1]);
                    if (cand) {
                        const float* rym = a.pcm + ((long long)z * a.Py + (y == 0 ? a.Py - 1 : y - 1)) * a.rowpitch;
                        const float* ryp = a.pcm + ((long long)z * a.Py + (y == a.Py - 1 ? 0 : y + 1)) * a.rowpitch;
                        const float* rzm = a.pcm + ((long long)(z == 0 ? a.Pz - 1 : z - 1) * a.Py + y) * a.rowpitch;
                        const float* rzp = a.pcm + ((long long)(z == a.Pz - 1 ? 0 : z + 1) * a.Py + y) * a.rowpitch;
                        cand = !(v < rym[x] || v < ryp[x] || v < rzm[x] || v < rzp[x]);
                    }
                }
                unsigned m = __ballot_sync(0xffffffffu, cand);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const float nv = __shfl_sync(0xffffffffu, v, src);
                    const int nx = __shfl_sync(0xffffffffu, x, src);
                    warp_topk_insert(top, K, nv, row * a.Px + nx, lane);
                }
            }
        }
    }
    // merge the warp lists of this CTA into warp 0's list, then write K entries
    __shared__ float s_v[NW * PCM_KMAX];
    __shared__ long long s_i[NW * PCM_KMAX];
    if (lane < K) { s_v[wid * PCM_KMAX + lane] = top.v; s_i[wid * PCM_KMAX + lane] = top.i; }
    __syncthreads();
    if (wid == 0) {
        for (int w = 1; w < NW; ++w)
            for (int e = 0; e < K; ++e) {
                const float nv = s_v[w * PCM_KMAX + e];
                if (nv == -INFINITY) break;  // lists are sorted; uniform across the warp
                warp_topk_insert(top, K, nv, s_i[w * PCM_KMAX + e], lane);
            }
        if (lane < K) {
            PeakEntry e;
            e.val = top.v;
            e.pad = 0;
            e.idx = (top.v == -INFINITY) ? -1 : top.i;
            a.out[(size_t)blockIdx.x * K + lane] = e;
        }
    }
}

// compile-time specialisations: padded 512^3 overlaps -> 540^3 (x half-length 270)
typedef FftStatic<270, 4, 17, 2, PCM_THREADS, 9, 6, 5> FftX270;
typedef FftStatic<270, 3, 9, 2, PCM_THREADS, 9, 6, 5> FftX270L8;

// ------------------------------------------------------------------------------------------
// Pearson sums for all candidate shifts in one launch
struct PearsonCand {
    int o1[3], o2[3], sz[3];
    int pad;
};

struct PearsonArgs {
    const void* img1;
    const void* img2;
    int dtype;
    int dx, dy, dz;
    const PearsonCand* cands;
    unsigned long long* sums_u;  // 5 per candidate: sa, sb, saa, sbb, sab
    double* sums_d;              // same for float input
};

// Generic path (uint8, float32, uint16 without 16-byte aligned bases): a warp owns PR_ROWS consecutive image-1 rows
// and evaluates every candidate on them, re-reading both images' rows from global memory per candidate.
#define PR_ROWS 16

// ------------------------------------------------------------------------------------------
// uint16 Pearson sums.  Work unit: a slab of up to PRS_ROWS consecutive image-1 rows, staged once into shared memory
// by a 1-D bulk copy (evict-first in L2) while the previous slab is consumed.  Persistent CTAs take slabs from a
// global counter in row (z-major) order, so all CTAs work inside a narrow z band and candidates with nearby (y, z)
// shifts share image-2 lines in L2.  For every candidate whose box meets the slab, a warp streams the matching
// image-2 row segments in 16-byte chunks aligned on the flat element index (so any row pitch works) and pairs them
// with the image-1 elements realigned from two 16-byte shared-memory reads.  Image 1 crosses DRAM once per pair,
// image 2 about once per candidate box.
#define PRS_ROWS 32
#define PRS_STAGE_ELEMS 16384     // bound on the staged rows per slab: 32 KB of uint16
#define PRS_PAD 8                 // elements in front of a staged slab (a chunk's realignment may start before it)

struct PearsonU16Args {
    const unsigned short* img1;   // both 16-byte aligned
    const unsigned short* img2;
    int dx, dy, dz;
    int slab_rows;                // image-1 rows per slab (<= PRS_ROWS, slab_rows * dx <= PRS_STAGE_ELEMS unless dx is larger)
    int stage_elems;              // uint16 elements per stage buffer, multiple of 8
    int nslabs;
    const PearsonCand* cands;
    unsigned long long* sums;     // 5 per candidate: sa, sb, saa, sbb, sab
    const int* ncand;
    int* counter;                 // slab counter, zero at launch
};

__device__ __forceinline__ unsigned long long l2_evict_first_policy() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void* dst, const void* src, unsigned int bytes, unsigned long long* bar,
                                                  unsigned long long policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}

// warp 0: stage slab s (flat image-1 elements [e0, e1)) into buf, where buf[PRS_PAD + e - (e0 & ~7)] = img1[e].
// Lane 0 issues the bulk copy of the 16-byte aligned middle; lanes 0-7 / 8-15 load the unaligned head / tail
// (< 8 elements each).
__device__ __forceinline__ void prs_stage(const PearsonU16Args& a, int s, long long nrows, unsigned short* buf,
                                          unsigned long long* bar, unsigned long long policy, int lane) {
    const long long r0 = (long long)s * a.slab_rows, r1 = min(r0 + a.slab_rows, nrows);
    const long long e0 = r0 * a.dx, e1 = r1 * a.dx, a0 = e0 & ~7LL;
    const long long b0 = (e0 + 7) & ~7LL, b1 = e1 & ~7LL;
    if (lane == 0) {
        const unsigned int bytes = b1 > b0 ? (unsigned int)((b1 - b0) * 2) : 0u;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the generic reads of the previous use came first
        mbar_expect_tx(bar, bytes);
        if (bytes) tma_bulk_g2s_hint(buf + PRS_PAD + (b0 - a0), a.img1 + b0, bytes, bar, policy);
    }
    const long long e = lane < 8 ? e0 + lane : max(b0, b1) + (lane - 8);
    if (lane < 16 && e < (lane < 8 ? min(b0, e1) : e1)) buf[PRS_PAD + (e - a0)] = a.img1[e];
}

// One lane's exact sums of one candidate.  The products go through the 2-way dot product IDP.2A (16-bit x 8-bit
// pairs into 32 bits): with b = b_lo + 256 b_hi, a * b = a * b_lo + 256 a * b_hi, so each product sum is kept as two
// uint32 partials p_lo + 256 p_hi.  One IDP adds at most 2 * 65535 * 255 = 33,422,850, so a partial holds 128 of
// them (4,278,124,800 < 2^32): 32 chunks of 8 elements (4 IDPs per partial each) between folds into uint64.
// sa / sb take one IDP against 0x0101 per word (bounded in prs_flush).
struct PrsAcc {
    unsigned int sa, sb;
    unsigned int aal, aah, bbl, bbh, abl, abh;
};
#define PRS_FOLD_CHUNKS 32        // chunks per lane between folds of the uint32 partials

__device__ __forceinline__ void prs_acc(const unsigned int A[4], const unsigned int B[4], PrsAcc& s) {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        // [x0 | x1] (two uint16) -> bytes [x0 lo, x1 lo, x0 hi, x1 hi]: _lo pairs with the low bytes, _hi the high
        const unsigned int Ap = __byte_perm(A[m], 0u, 0x3120), Bp = __byte_perm(B[m], 0u, 0x3120);
        s.sa = __dp2a_lo(A[m], 0x0101u, s.sa);
        s.sb = __dp2a_lo(B[m], 0x0101u, s.sb);
        s.aal = __dp2a_lo(A[m], Ap, s.aal);
        s.aah = __dp2a_hi(A[m], Ap, s.aah);
        s.bbl = __dp2a_lo(B[m], Bp, s.bbl);
        s.bbh = __dp2a_hi(B[m], Bp, s.bbh);
        s.abl = __dp2a_lo(A[m], Bp, s.abl);
        s.abh = __dp2a_hi(A[m], Bp, s.abh);
    }
}

// Fold the lanes' partials into uint64, add the warp's total to the candidate's shared-memory sums and restart the
// partials (warp-uniform).  Between flushes the warp covers at most 32 * PRS_FOLD_CHUNKS chunks (see prs_row), so its
// sa / sb stay below 8192 elements * 65535 < 2^32.
__device__ __forceinline__ void prs_flush(PrsAcc& s, unsigned long long* acc, int lane) {
    unsigned int sa = s.sa, sb = s.sb;
    unsigned long long saa = s.aal + ((unsigned long long)s.aah << 8), sbb = s.bbl + ((unsigned long long)s.bbh << 8),
                       sab = s.abl + ((unsigned long long)s.abh << 8);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        sa += __shfl_xor_sync(0xffffffffu, sa, off);
        sb += __shfl_xor_sync(0xffffffffu, sb, off);
        saa += __shfl_xor_sync(0xffffffffu, saa, off);
        sbb += __shfl_xor_sync(0xffffffffu, sbb, off);
        sab += __shfl_xor_sync(0xffffffffu, sab, off);
    }
    if (lane == 0) {
        if (sa) atomicAdd(acc + 0, (unsigned long long)sa);
        if (sb) atomicAdd(acc + 1, (unsigned long long)sb);
        if (saa) atomicAdd(acc + 2, saa);
        if (sbb) atomicAdd(acc + 3, sbb);
        if (sab) atomicAdd(acc + 4, sab);
    }
    s = PrsAcc{0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
}

// One image-2 row segment of one candidate, owned by a warp.  Chunk k covers image-2 elements g + 8k .. g + 8k + 7
// (g 16-byte aligned); elements lo .. hi - 1 of the chunk sequence belong to the segment.  s1 points at the staged
// image-1 element paired with chunk 0's first element, rounded down to 16 bytes; SH is the rounding (0..7).
// Chunks k >= kvec reach past the end of image 2 and are loaded element by element.
// A round takes one chunk per lane, and the row's last round up to two (its loads in flight before the arithmetic),
// so a segment of up to 64 chunks costs one round trip to image 2.  A lane takes ceil(nch / 32) chunks of the row.
// Segments of more than 32 * PRS_FOLD_CHUNKS = 1024 chunks (hi > 8192) fold every PRS_FOLD_CHUNKS - 1 rounds, which
// with a last round of two leaves at most PRS_FOLD_CHUNKS chunks per lane between folds.  Their rows are over 8185
// elements wide, so a slab holds at most 2 rows (slab_rows = PRS_STAGE_ELEMS / dx) and the warp owns only this one:
// the partials enter it at zero and leave it with at most PRS_FOLD_CHUNKS chunks per lane.  Everything else folds once per candidate in the caller:
// with slab_rows <= 8 a warp owns one row of <= 1024 chunks, with 9-16 two rows of <= 1820 elements and with 17-32
// four rows of <= 963 elements, <= 32 chunks per lane in every case.
template <int SH>
__device__ __forceinline__ void prs_row(const unsigned short* __restrict__ g, const unsigned short* s1, int lo, int hi,
                                        int nch, int kvec, int lane, PrsAcc& s, unsigned long long* acc) {
    for (int kb = 0, r = 1; kb < nch; kb += 32, ++r) {   // warp-uniform rounds
        const bool last = nch - kb <= 64;
        uint4 v[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = (u == 0 || last) ? kb + lane + 32 * u : nch;
            v[u] = make_uint4(0u, 0u, 0u, 0u);
            if (k < kvec) {
                v[u] = ldg_stream16(g + 8 * k);
            } else if (k < nch) {
                unsigned long long w0 = 0ull, w1 = 0ull;
                for (int j = max(lo - 8 * k, 0); j < min(hi - 8 * k, 8); ++j) {
                    const unsigned long long e = g[8 * k + j];
                    if (j < 4) w0 |= e << (16 * j);
                    else w1 |= e << (16 * (j - 4));
                }
                v[u] = make_uint4((unsigned int)w0, (unsigned int)(w0 >> 32), (unsigned int)w1, (unsigned int)(w1 >> 32));
            }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = (u == 0 || last) ? kb + lane + 32 * u : nch;
            if (k >= nch) break;
            const uint4 p = *reinterpret_cast<const uint4*>(s1 + 8 * k);
            const uint4 q = *reinterpret_cast<const uint4*>(s1 + 8 * k + 8);
            const unsigned int w[8] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w};
            unsigned int A[4], B[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
            for (int m = 0; m < 4; ++m)
                A[m] = (SH & 1) ? __funnelshift_r(w[SH / 2 + m], w[SH / 2 + m + 1], 16) : w[SH / 2 + m];
            const int l = lo - 8 * k, h = hi - 8 * k;
            if (l > 0 || h < 8) {            // first / last chunk of the segment: zero both sides outside it
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const unsigned int mk = ((2 * m >= l && 2 * m < h) ? 0x0000ffffu : 0u) |
                                            ((2 * m + 1 >= l && 2 * m + 1 < h) ? 0xffff0000u : 0u);
                    A[m] &= mk;
                    B[m] &= mk;
                }
            }
            prs_acc(A, B, s);
        }
        if (last) break;
        if (r % (PRS_FOLD_CHUNKS - 1) == 0) prs_flush(s, acc, lane);
    }
}

// dynamic smem: 2 stage buffers, the candidate list, 5 accumulators per candidate
__global__ void __launch_bounds__(PCM_THREADS, 3) k_pearson_u16(const __grid_constant__ PearsonU16Args a) {
    const int ncand = *a.ncand;   // written by k_pcm_select (no host round trip between peaks and Pearson)
    if (ncand <= 0) return;
    constexpr int NW = PCM_THREADS / 32, RPW = PRS_ROWS / NW;
    unsigned short* stage = reinterpret_cast<unsigned short*>(bs_sm);
    PearsonCand* s_cand = reinterpret_cast<PearsonCand*>(stage + 2 * (size_t)a.stage_elems);
    unsigned long long* s_acc = reinterpret_cast<unsigned long long*>(s_cand + ncand);
    __shared__ unsigned long long bars[2];
    __shared__ int s_slab[2];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long nrows = (long long)a.dy * a.dz, nel = nrows * a.dx;
    const unsigned long long policy = l2_evict_first_policy();
    for (int i = tid; i < 10 * ncand; i += blockDim.x) reinterpret_cast<int*>(s_cand)[i] = reinterpret_cast<const int*>(a.cands)[i];
    for (int i = tid; i < 5 * ncand; i += blockDim.x) s_acc[i] = 0ull;
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (wid == 0) {
        const int s = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(a.counter, 1) : 0, 0);
        if (lane == 0) s_slab[0] = s;
        if (s < a.nslabs) prs_stage(a, s, nrows, stage, &bars[0], policy, lane);
    }
    __syncthreads();
    for (int it = 0;; ++it) {
        const int buf = it & 1;
        const int s = s_slab[buf];
        if (s >= a.nslabs) break;
        if (wid == 0) {   // next slab's copy is in flight while this one is consumed
            const int sn = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(a.counter, 1) : 0, 0);
            if (lane == 0) s_slab[buf ^ 1] = sn;
            if (sn < a.nslabs) prs_stage(a, sn, nrows, stage + (size_t)(buf ^ 1) * a.stage_elems, &bars[buf ^ 1], policy, lane);
        }
        const long long r0 = (long long)s * a.slab_rows;
        const int nr = (int)min((long long)a.slab_rows, nrows - r0);
        const int z0 = (int)(r0 / a.dy), y0 = (int)(r0 - (long long)z0 * a.dy);
        const int zl = (int)((r0 + nr - 1) / a.dy);
        // staged image-1 element e0 + i (e0 = r0 * dx, the slab's first) sits at sbuf[soff + i]
        const unsigned short* sbuf = stage + (size_t)buf * a.stage_elems;
        const int soff = PRS_PAD + (int)((r0 * a.dx) & 7);
        mbar_wait(&bars[buf], (it >> 1) & 1);
        for (int c = 0; c < ncand; ++c) {
            const PearsonCand cd = s_cand[c];
            if (zl < cd.o1[2] || z0 >= cd.o1[2] + cd.sz[2]) continue;   // block-uniform
            PrsAcc acc = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
            bool any = false;
            // not unrolled: the 8 alignment cases of prs_row are inlined once each, not once per row (instruction
            // cache)
#pragma unroll 1
            for (int j = 0; j < RPW; ++j) {
                const int rr = wid + j * NW;
                int y = y0 + rr, z = z0;   // (y, z) of slab row rr
                while (y >= a.dy) { y -= a.dy; ++z; }
                const int yy = y - cd.o1[1], zz = z - cd.o1[2];
                if (rr >= nr || yy < 0 || yy >= cd.sz[1] || zz < 0 || zz >= cd.sz[2]) continue;
                any = true;
                const long long g2 = ((long long)(zz + cd.o2[2]) * a.dy + (yy + cd.o2[1])) * a.dx + cd.o2[0];
                const long long c2 = g2 & ~7LL;
                const int lo = (int)(g2 - c2), hi = lo + cd.sz[0];
                const int nch = (hi + 7) >> 3;
                const int kvec = (int)min((long long)nch, (nel - c2) >> 3);
                // staged index of the image-1 element paired with image-2 element c2 (>= soff - 7 >= 1)
                const int t = soff + rr * a.dx + cd.o1[0] - lo;
                const unsigned short* s1 = sbuf + (t & ~7);
                const unsigned short* g = a.img2 + c2;
                switch (t & 7) {
                    case 0: prs_row<0>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 1: prs_row<1>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 2: prs_row<2>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 3: prs_row<3>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 4: prs_row<4>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 5: prs_row<5>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 6: prs_row<6>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    default: prs_row<7>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                }
            }
            if (any) prs_flush(acc, s_acc + 5 * c, lane);   // warp-uniform
        }
        __syncthreads();   // every warp is done with this buffer before it is refilled
    }
    __syncthreads();
    for (int i = tid; i < 5 * ncand; i += blockDim.x)
        if (s_acc[i]) atomicAdd(a.sums + i, s_acc[i]);
}

template <typename T, typename ACC>
__device__ __forceinline__ void pearson_generic(const PearsonArgs& a, int ncand, ACC* s_acc) {
    const T* __restrict__ i1 = (const T*)a.img1;
    const T* __restrict__ i2 = (const T*)a.img2;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const long long nrows = (long long)a.dy * a.dz;
    const long long nchunks = (nrows + PR_ROWS - 1) / PR_ROWS;
    for (long long ch = (long long)blockIdx.x * nw + wid; ch < nchunks; ch += (long long)gridDim.x * nw) {
        const long long r0 = ch * PR_ROWS;
        for (int c = 0; c < ncand; ++c) {
            const PearsonCand cd = a.cands[c];
            ACC v[5] = {0, 0, 0, 0, 0};
            bool any = false;
            for (int rr = 0; rr < PR_ROWS; ++rr) {
                const long long r = r0 + rr;
                if (r >= nrows) break;
                const int z = (int)(r / a.dy), y = (int)(r - (long long)z * a.dy);
                const int yy = y - cd.o1[1], zz = z - cd.o1[2];
                if (yy < 0 || yy >= cd.sz[1] || zz < 0 || zz >= cd.sz[2]) continue;
                any = true;
                const T* p1 = i1 + (size_t)r * a.dx + cd.o1[0];
                const T* p2 = i2 + ((size_t)(zz + cd.o2[2]) * a.dy + (yy + cd.o2[1])) * a.dx + cd.o2[0];
                for (int x = lane; x < cd.sz[0]; x += 32) {
                    const ACC va = (ACC)__ldg(p1 + x), vb = (ACC)__ldg(p2 + x);
                    v[0] += va; v[1] += vb; v[2] += va * va; v[3] += vb * vb; v[4] += va * vb;
                }
            }
            if (!any) continue;
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                ACC t = v[k];
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) t += __shfl_down_sync(0xffffffffu, t, off);
                if (lane == 0) atomicAdd(&s_acc[5 * c + k], t);
            }
        }
    }
}

// dynamic smem: 5 accumulators per candidate (8 bytes each)
__global__ void __launch_bounds__(PCM_THREADS) k_pearson(const __grid_constant__ PearsonArgs a, const int* __restrict__ ncand_ptr) {
    const int ncand = *ncand_ptr;     // written by k_pcm_select (no host round trip between peaks and Pearson)
    if (ncand <= 0) return;
    unsigned long long* s_u = reinterpret_cast<unsigned long long*>(bs_sm);
    double* s_d = reinterpret_cast<double*>(bs_sm);
    for (int i = threadIdx.x; i < 5 * ncand; i += blockDim.x) s_u[i] = 0ull;  // 0.0 has the same bit pattern
    __syncthreads();
    if (a.dtype == BS_DTYPE_U16) pearson_generic<unsigned short, unsigned long long>(a, ncand, s_u);
    else if (a.dtype == BS_DTYPE_U8) pearson_generic<unsigned char, unsigned long long>(a, ncand, s_u);
    else pearson_generic<float, double>(a, ncand, s_d);
    __syncthreads();
    for (int i = threadIdx.x; i < 5 * ncand; i += blockDim.x) {
        if (a.dtype == BS_DTYPE_F32) { if (s_d[i] != 0.0) atomicAdd(a.sums_d + i, s_d[i]); }
        else if (s_u[i]) atomicAdd(a.sums_u + i, s_u[i]);
    }
}

// ------------------------------------------------------------------------------------------
// Device-side glue between peak search and Pearson verification: merge the per-CTA top-K lists, expand every
// peak into its 2^3 wrap candidates (PhaseCorrelation2Util.expandPeakToPossibleShifts for equal-size crops),
// keep those with enough overlap, gather the 3x3x3 neighbourhoods for the sub-pixel fit.  One small CTA; the
// host reads ONE result block per pair, after the Pearson kernel, and can do so a pair late.
struct PcmSelect {
    int np;                       // peaks kept (<= K)
    int nslots;                   // Pearson-verified candidates
    long long idx[PCM_KMAX];      // linear PCM index of peak i
    float val[PCM_KMAX];
    float nb[27 * PCM_KMAX];      // periodic 3x3x3 neighbourhoods
};

// candidate i (0..7) of a peak at PCM location loc: shift per axis is loc or loc - P; returns true when the
// candidate overlaps by at least min_px voxels (then pc / npx describe the overlap boxes)
__host__ __device__ inline bool pcm_expand_candidate(const long long loc[3], const int P[3], const int d[3], int i,
                                                     long long min_px, long long shift[3], PearsonCand* pc, long long* npx_out) {
    bool overlap = true;
    long long npx = 1;
    for (int a = 0; a < 3; ++a) {
        long long s = loc[a];
        if (((i >> a) & 1) == 0) s = s < 0 ? s + P[a] : s - P[a];
        shift[a] = s;
        const long long n = d[a];
        if (s >= 0) {
            if (s >= n) { overlap = false; continue; }
            pc->o1[a] = (int)s; pc->o2[a] = 0; pc->sz[a] = (int)(n - s < n ? n - s : n);
        } else {
            if (s <= -n) { overlap = false; continue; }
            pc->o1[a] = 0; pc->o2[a] = (int)-s; pc->sz[a] = (int)(n + s < n ? n + s : n);
        }
        npx *= pc->sz[a];
    }
    pc->pad = 0;
    *npx_out = npx;
    return overlap && npx >= min_px;
}

struct SelectArgs {
    const PeakEntry* peaks;       // n_entries per-CTA candidates (idx < 0: empty)
    int n_entries;
    int K;
    int P[3], d[3];
    long long rowpitch;
    const float* pcm;
    long long min_px;
    int do_subpixel;
    PcmSelect* sel;
    PearsonCand* cands;           // 8 * K
    unsigned long long* sums;     // 5 * 8 * K, zeroed here
    int* ncand;                   // [0]: candidate count, [1]: Pearson slab counter (zeroed here)
};

__global__ void __launch_bounds__(256) k_pcm_select(const __grid_constant__ SelectArgs a) {
    __shared__ float s_v[8];
    __shared__ long long s_i[8];
    __shared__ float s_pv[PCM_KMAX];
    __shared__ long long s_pi[PCM_KMAX];
    __shared__ int s_np, s_nslots;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    float lastv = INFINITY;
    long long lasti = -1;
    int np = 0;
    for (int j = 0; j < a.K; ++j) {
        // best entry that comes strictly after the previous pick in (value desc, index asc) order
        float bv = -INFINITY;
        long long bi = LLONG_MAX;
        for (int e = tid; e < a.n_entries; e += blockDim.x) {
            const PeakEntry pe = a.peaks[e];
            if (pe.idx < 0) continue;
            if (!peak_better(lastv, lasti, pe.val, pe.idx)) continue;
            if (bi == LLONG_MAX || peak_better(pe.val, pe.idx, bv, bi)) { bv = pe.val; bi = pe.idx; }
        }
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_down_sync(0xffffffffu, bv, o);
            const long long oi = __shfl_down_sync(0xffffffffu, bi, o);
            if (oi != LLONG_MAX && (bi == LLONG_MAX || peak_better(ov, oi, bv, bi))) { bv = ov; bi = oi; }
        }
        if (lane == 0) { s_v[wid] = bv; s_i[wid] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
                if (s_i[w] != LLONG_MAX && (bi == LLONG_MAX || peak_better(s_v[w], s_i[w], bv, bi))) { bv = s_v[w]; bi = s_i[w]; }
            s_v[0] = bv; s_i[0] = bi;
        }
        __syncthreads();
        bv = s_v[0]; bi = s_i[0];
        __syncthreads();
        if (bi == LLONG_MAX) break;
        if (tid == 0) { s_pv[np] = bv; s_pi[np] = bi; }
        lastv = bv; lasti = bi;
        ++np;
    }
    __syncthreads();
    if (tid == 0) {
        int nslots = 0;
        for (int pi = 0; pi < np; ++pi) {
            const long long li = s_pi[pi];
            const long long loc[3] = {li % a.P[0], (li / a.P[0]) % a.P[1], li / ((long long)a.P[0] * a.P[1])};
            for (int i = 0; i < 8; ++i) {
                long long shift[3], npx;
                PearsonCand pc;
                pc.o1[0] = pc.o1[1] = pc.o1[2] = pc.o2[0] = pc.o2[1] = pc.o2[2] = pc.sz[0] = pc.sz[1] = pc.sz[2] = 0;
                if (pcm_expand_candidate(loc, a.P, a.d, i, a.min_px, shift, &pc, &npx)) a.cands[nslots++] = pc;
            }
        }
        a.sel->np = np;
        a.sel->nslots = nslots;
        a.ncand[0] = nslots;
        a.ncand[1] = 0;   // k_pearson_u16's slab counter
        s_np = np; s_nslots = nslots;
    }
    __syncthreads();
    np = s_np;
    for (int i = tid; i < PCM_KMAX; i += blockDim.x) {
        a.sel->idx[i] = i < np ? s_pi[i] : -1;
        a.sel->val[i] = i < np ? s_pv[i] : 0.f;
    }
    for (int i = tid; i < 5 * s_nslots; i += blockDim.x) a.sums[i] = 0ull;
    if (a.do_subpixel)
        for (int t = tid; t < 27 * np; t += blockDim.x) {
            const int p = t / 27, o = t - p * 27;
            const long long li = s_pi[p];
            const int x = (int)(li % a.P[0]);
            const long long r = li / a.P[0];
            const int y = (int)(r % a.P[1]), z = (int)(r / a.P[1]);
            const int dz = o / 9 - 1, dy = (o / 3) % 3 - 1, dx = o % 3 - 1;
            const int xx = (x + dx + a.P[0]) % a.P[0], yy = (y + dy + a.P[1]) % a.P[1], zz = (z + dz + a.P[2]) % a.P[2];
            a.sel->nb[t] = a.pcm[((long long)zz * a.P[1] + yy) * a.rowpitch + xx];
        }
}

// ==========================================================================================
// host side
// ==========================================================================================
static const int kRadices[] = {16, 15, 12, 10, 9, 8, 6, 5, 4, 3, 2};

static void plan_search(int n, int depth, int* cur, int* best, int* best_len) {
    if (n == 1) {
        if (depth < *best_len) {
            *best_len = depth;
            memcpy(best, cur, sizeof(int) * depth);
        }
        return;
    }
    if (depth + 1 >= *best_len || depth >= BS_FFT_MAX_STAGES) return;
    for (int r : kRadices) {
        if (n % r) continue;
        if (depth > 0 && r > cur[depth - 1]) continue;  // non-increasing: canonical order
        cur[depth] = r;
        plan_search(n / r, depth + 1, cur, best, best_len);
    }
}

static bool make_plan(int n, FftPlan* p) {
    memset(p, 0, sizeof(*p));
    p->n = n;
    if (n == 1) { p->nst = 0; return true; }
    int cur[BS_FFT_MAX_STAGES], best[BS_FFT_MAX_STAGES], best_len = BS_FFT_MAX_STAGES + 1;
    plan_search(n, 0, cur, best, &best_len);
    if (best_len > BS_FFT_MAX_STAGES) return false;
    // odd radices first (conflict-free first-stage scatter), then descending
    std::stable_sort(best, best + best_len, [](int x, int y) { return (x & 1) > (y & 1); });
    p->nst = best_len;
    for (int i = 0; i < best_len; ++i) p->radix[i] = best[i];
    return true;
}

extern "C" int bs_good_fft_size(int n, int even) {
    int m = n < 2 ? 2 : n;
    for (;; ++m) {
        int k = m;
        for (int p : {2, 3, 5})
            while (k % p == 0) k /= p;
        if (k == 1 && (!even || m % 2 == 0)) return m;
    }
}

static int ext_size(int d, int ext) { return d + (d < ext ? 2 * d : 2 * ext); }

// per-axis source index + blending weight for every padded position (mirrors
// oracle/pcm_oracle.py:_axis_profile; BlendedExtendedMirroredRandomAccesible2 semantics)
static void axis_profile(int d, int ext, int P, std::vector<int>& idx, std::vector<float>& w) {
    const int e = std::min(ext, d);
    idx.assign(P, 0);
    w.assign(P, 0.f);
    const int period = std::max(2 * d - 2, 1);
    for (int p = 0; p < P; ++p) {
        const int s = p - e;
        if (s < -e || s > d - 1 + e) continue;
        const int dist = s < 0 ? -s : (s > d - 1 ? s - (d - 1) : 0);
        int m = 0;
        if (d > 1) {
            m = s % period;
            if (m < 0) m += period;
            if (m >= d) m = period - m;
        }
        idx[p] = m;
        w[p] = dist > 0 ? (float)(0.5 * (std::cos(M_PI * (double)dist / (double)e) + 1.0)) : 1.0f;
    }
}

struct PcmGeometry {
    int d[3], ext[3], P[3], E[3];
    int M, pitch;
    FftPlan plan_x, plan_y, plan_z;
    int lshift_x;   // log2 lines per CTA in the c2r kernel
    int lshift_r2c; // log2 lines per CTA in the r2c kernel (fewer lines -> more CTAs/SM to hide load latency)
    int tshift_y, tshift_z;
    size_t smem_x_r2c, smem_x_c2r, smem_y, smem_z;
    bool static_x, static_y, static_z;  // compile-time specialised kernels apply
};

struct PcmDeviceTables {
    int key[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // d[3], ext[3], P[3]
    int* idx[3] = {nullptr, nullptr, nullptr};
    float* w[3] = {nullptr, nullptr, nullptr};
    float2* tw[3] = {nullptr, nullptr, nullptr};
    int cap[3] = {0, 0, 0};
};

// one table set per context
static PcmDeviceTables* tables_of(bs_ctx* ctx) {
    if (!ctx->ws.tables) ctx->ws.tables = new PcmDeviceTables();
    return (PcmDeviceTables*)ctx->ws.tables;
}

void bs_pcm_slots_free(bs_ctx* ctx);
void bs_pcm_workspace_free(bs_ctx* ctx) {
    bs_pcm_slots_free(ctx);
    bs_pcm_workspace& ws = ctx->ws;
    if (ws.spec_a) cudaFree(ws.spec_a);
    if (ws.spec_b) cudaFree(ws.spec_b);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j)
            if (ws.crop[i][j]) cudaFree(ws.crop[i][j]);
    if (ws.small) cudaFree(ws.small);
    if (ws.small_host) cudaFreeHost(ws.small_host);
    if (ws.sync) cudaFree(ws.sync);
    for (int i = 0; i < 2; ++i) {
        if (ws.crop_ready[i]) cudaEventDestroy(ws.crop_ready[i]);
        if (ws.crop_free[i]) cudaEventDestroy(ws.crop_free[i]);
    }
    if (ws.tables) {
        PcmDeviceTables* t = (PcmDeviceTables*)ws.tables;
        for (int d = 0; d < 3; ++d) {
            if (t->idx[d]) cudaFree(t->idx[d]);
            if (t->w[d]) cudaFree(t->w[d]);
            if (t->tw[d]) cudaFree(t->tw[d]);
        }
        delete t;
    }
    ws = bs_pcm_workspace();
}

static int env_int(const char* name, int dflt) {
    const char* s = getenv(name);
    return s && *s ? atoi(s) : dflt;
}

static int pcm_geometry(bs_ctx* ctx, const long long dims[3], const int ext[3], PcmGeometry* g) {
    for (int d = 0; d < 3; ++d) {
        if (dims[d] <= 0 || dims[d] > 16384) return bs_set_error(ctx, BS_ERR_ARG, "pcm: dims[%d]=%lld out of range", d, dims[d]);
        if (ext[d] < 1 || ext[d] > 4096) return bs_set_error(ctx, BS_ERR_ARG, "pcm: extension[%d]=%d out of range", d, ext[d]);
        g->d[d] = (int)dims[d];
        g->ext[d] = ext[d];
        g->E[d] = ext_size(g->d[d], ext[d]);
        g->P[d] = bs_good_fft_size(g->E[d], d == 0);
    }
    g->M = g->P[0] / 2;
    g->pitch = ((g->M + 1 + 15) / 16) * 16;
    if (!make_plan(g->M, &g->plan_x) || !make_plan(g->P[1], &g->plan_y) || !make_plan(g->P[2], &g->plan_z))
        return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "pcm: cannot plan FFT for padded size %dx%dx%d", g->P[0], g->P[1], g->P[2]);
    // lines per CTA for the x kernels: largest power of two <= 16 that fits shared memory
    int ls = env_int("BS_FFT_XLINES_LOG2", 4);
    for (;; --ls) {
        const int LB = 1 << ls;
        g->smem_x_r2c = ((size_t)g->P[0] + 2 * (size_t)g->M * (LB + 1)) * sizeof(float2);
        g->smem_x_c2r = ((size_t)g->P[0] + (size_t)(2 * g->M + 1) * (LB + 1)) * sizeof(float2);
        if (g->smem_x_c2r <= PCM_SMEM_MAX && g->smem_x_r2c <= PCM_SMEM_MAX) break;
        if (ls == 0) return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "pcm: x size %d too large for shared memory", g->P[0]);
    }
    g->lshift_x = ls;
    g->lshift_r2c = std::min(ls, env_int("BS_FFT_R2C_LINES_LOG2", 3));
    g->smem_x_r2c = ((size_t)g->P[0] + 2 * (size_t)g->M * ((1 << g->lshift_r2c) + 1)) * sizeof(float2);
    auto strided = [&](int N, int nbuf, int pref, int* tshift, size_t* smem) -> bool {
        for (int ts = pref; ts >= 1; --ts) {
            const size_t b = ((size_t)((N + 1) & ~1) + (size_t)nbuf * N * (1 << ts)) * sizeof(float2);
            if (b <= PCM_SMEM_MAX) { *tshift = ts; *smem = b; return true; }
        }
        return false;
    };
    if (!strided(g->P[1], 2, env_int("BS_FFT_YTILE_LOG2", 3), &g->tshift_y, &g->smem_y) ||
        !strided(g->P[2], 3, env_int("BS_FFT_ZTILE_LOG2", 3), &g->tshift_z, &g->smem_z))
        return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "pcm: y/z size %dx%d too large for shared memory", g->P[1], g->P[2]);
    const bool allow_static = env_int("BS_FFT_STATIC", 1) != 0;
    g->static_x = allow_static && g->M == FftX270::N && (g->lshift_x == FftX270::LSHIFT || g->lshift_x == FftX270L8::LSHIFT) &&
                  (g->lshift_r2c == 3 || g->lshift_r2c == 4);
    // k_fft_col540 / k_fft_xpower_col540: the pitch (a multiple of 16) always divides into 16-column tiles
    g->static_y = allow_static && g->P[1] == Col540::N;
    g->static_z = allow_static && g->P[2] == Col540::N;
    return BS_OK;
}

static int pcm_tables(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables** out) {
    PcmDeviceTables* t = tables_of(ctx);
    *out = t;
    int key[9] = {g.d[0], g.d[1], g.d[2], g.ext[0], g.ext[1], g.ext[2], g.P[0], g.P[1], g.P[2]};
    if (!memcmp(key, t->key, sizeof(key))) return BS_OK;
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int d = 0; d < 3; ++d) {
        const int P = g.P[d];
        if (t->cap[d] < P) {
            if (t->idx[d]) { cudaFree(t->idx[d]); cudaFree(t->w[d]); cudaFree(t->tw[d]); }
            BS_CUDA(ctx, cudaMalloc(&t->idx[d], sizeof(int) * P));
            BS_CUDA(ctx, cudaMalloc(&t->w[d], sizeof(float) * P));
            BS_CUDA(ctx, cudaMalloc(&t->tw[d], sizeof(float2) * P));
            t->cap[d] = P;
        }
        std::vector<int> idx;
        std::vector<float> w;
        axis_profile(g.d[d], g.ext[d], P, idx, w);
        std::vector<float2> tw(P);
        for (int k = 0; k < P; ++k) {
            const double ang = -2.0 * M_PI * (double)k / (double)P;
            tw[k] = make_float2((float)std::cos(ang), (float)std::sin(ang));
        }
        BS_CUDA(ctx, cudaMemcpy(t->idx[d], idx.data(), sizeof(int) * P, cudaMemcpyHostToDevice));
        BS_CUDA(ctx, cudaMemcpy(t->w[d], w.data(), sizeof(float) * P, cudaMemcpyHostToDevice));
        BS_CUDA(ctx, cudaMemcpy(t->tw[d], tw.data(), sizeof(float2) * P, cudaMemcpyHostToDevice));
    }
    memcpy(t->key, key, sizeof(key));
    return BS_OK;
}

// ws.sync: the error word of k_fft_xy_col540's hand-off waits (PCM_HANDOFF_XY once one expired, else 0), reset once
// per pair, then [ready Pz][done Pz] counters, zeroed before each launch
#define PCM_SYNC_COUNTERS 32   // ints ahead of the counters (the error word on a line of its own)
enum { PCM_HANDOFF_OK = 0, PCM_HANDOFF_XY = 1 };

static int pcm_workspace(bs_ctx* ctx, const PcmGeometry& g) {
    bs_pcm_workspace& ws = ctx->ws;
    const size_t need = (size_t)g.P[2] * g.P[1] * g.pitch * sizeof(float2);
    if (ws.spec_bytes < need) {
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ws.spec_a) cudaFree(ws.spec_a);
        if (ws.spec_b) cudaFree(ws.spec_b);
        ws.spec_a = ws.spec_b = nullptr;
        ws.spec_bytes = 0;
        BS_CUDA(ctx, cudaMalloc(&ws.spec_a, need));
        BS_CUDA(ctx, cudaMalloc(&ws.spec_b, need));
        ws.spec_bytes = need;
    }
    const size_t small_need = 4 << 20;   // PCM_SLOTS result slots (per-CTA peak lists, select block, candidates, sums)
    if (!ws.small) {
        BS_CUDA(ctx, cudaMalloc(&ws.small, small_need));
        BS_CUDA(ctx, cudaHostAlloc(&ws.small_host, small_need, cudaHostAllocDefault));
        ws.small_bytes = small_need;
    }
    const size_t sync_need = sizeof(int) * (PCM_SYNC_COUNTERS + 2 * (size_t)g.P[2]);
    if (ws.sync_bytes < sync_need) {
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ws.sync) cudaFree(ws.sync);
        ws.sync = nullptr;
        ws.sync_bytes = 0;
        BS_CUDA(ctx, cudaMalloc(&ws.sync, sync_need));
        BS_CUDA(ctx, cudaMemset(ws.sync, 0, sync_need));
        ws.sync_bytes = sync_need;
    }
    return BS_OK;
}

static int pcm_reset_handoff(bs_ctx* ctx) {
    BS_CUDA(ctx, cudaMemsetAsync(ctx->ws.sync, 0, sizeof(int), ctx->stream));
    return BS_OK;
}
static int pcm_handoff_error(bs_ctx* ctx, int code) {
    if (code == PCM_HANDOFF_OK) return BS_OK;
    return bs_set_error(ctx, BS_ERR_CUDA, "pcm: k_fft_xy_col540: a plane hand-off wait expired (code %d)", code);
}
// wait for the stream, then check the error word
static int pcm_sync_handoff(bs_ctx* ctx) {
    int code = 0;
    BS_CUDA(ctx, cudaMemcpyAsync(&code, ctx->ws.sync, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return pcm_handoff_error(ctx, code);
}

static int set_smem(bs_ctx* ctx, const void* fn, size_t bytes) {
    BS_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PCM_SMEM_MAX));
    (void)bytes;
    return BS_OK;
}

// n_img: 1 or 2 spectra through k_fft_col540 (y), 0 for the cross-power k_fft_xpower_col540 (z)
static int launch_col540(bs_ctx* ctx, const StridedArgs& a, int tiles_x, int n_other, int n_img) {
    StridedPipeArgs pp;
    pp.s = a;
    pp.tiles_x = tiles_x;
    pp.n_other = n_other;
    pp.n_tiles = tiles_x * n_other * (n_img ? n_img : 1);
    const int nctas = std::min(pp.n_tiles, ctx->sm_count);   // one CTA per SM (shared memory, registers)
    if (n_img) {
        const size_t smem = (Col540::N + 2 * (size_t)Col540::XSIZE) * sizeof(float2);
        k_fft_col540<<<nctas, COL540_NT, smem, ctx->stream>>>(pp);
        return BS_OK;
    }
    // z pass: spectra [Pz = 540][Py = n_other][pitch] as floats, one 128 B x 1 x 180-row box per copy
    XpowerCol540Args xa;
    xa.p = pp;
    auto enc = bs_tensor_map_encoder();
    if (!enc) return bs_set_error(ctx, BS_ERR_CUDA, "pcm: cuTensorMapEncodeTiled is not available");
    const cuuint64_t gdim[3] = {(cuuint64_t)tiles_x * 2 * COL540_TC, (cuuint64_t)n_other, (cuuint64_t)Col540::N};
    const cuuint64_t gstr[2] = {(cuuint64_t)a.ostride * sizeof(float2), (cuuint64_t)a.estride * sizeof(float2)};
    const cuuint32_t box[3] = {2 * COL540_TC, 1, Col540::N / COL540_ZBOXES};
    const cuuint32_t estr[3] = {1, 1, 1};
    for (int i = 0; i < 2; ++i) {
        const CUresult r = enc(&xa.tm[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, i ? (void*)a.b : (void*)a.a, gdim, gstr, box,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return bs_set_error(ctx, BS_ERR_CUDA, "pcm: cuTensorMapEncodeTiled failed (%d)", (int)r);
    }
    // buffers, twiddles, one mbarrier per buffer
    const size_t smem = (3 * (size_t)Col540::XSIZE + Col540::N) * sizeof(float2) + 3 * sizeof(unsigned long long);
    k_fft_xpower_col540<<<nctas, COL540_NT, smem, ctx->stream>>>(xa);
    return BS_OK;
}

static int pcm_kernel_attrs(bs_ctx* ctx) {
    if (ctx->pcm_attr_done) return BS_OK;
    int rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_strided<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c<FftX270>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c<FftX270L8>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_tma<FftX270L8>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_w<FftW270S>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_w<FftWGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r_w<FftW270>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r_w<FftWGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_tma<FftX270>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_tma<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r<FftX270L8>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_strided_pipe<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_xpower_pipe<FftGeneric>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_col540, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_xpower_col540, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r<FftX270>, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_r2c_col540, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_x_c2r_col540, 0))) return rc;
    if ((rc = set_smem(ctx, (const void*)k_fft_xy_col540, 0))) return rc;
    ctx->pcm_attr_done = true;
    return BS_OK;
}

// The five FFT passes.  Each launches one kernel on ctx->stream and, when `info` is not NULL, writes the
// instantiation it chose (plus the plan's radices for runtime-planned kernels), e.g.
// "k_fft_strided_pipe<FftGeneric> 15x12x3", into info[PCM_INFO_LEN].  bs_pcm_debug_pass runs them one at a time.
#define PCM_INFO_LEN 128
static void pass_info(char* info, const char* kernel, const FftPlan* plan) {
    if (!info) return;
    int n = snprintf(info, PCM_INFO_LEN, "%s", kernel);
    for (int i = 0; plan && i < plan->nst && n < PCM_INFO_LEN; ++i)
        n += snprintf(info + n, PCM_INFO_LEN - n, "%s%d", i ? "x" : " ", plan->radix[i]);
}

// The two-for-one Col540 x kernels (k_fft_x_r2c_col540 / k_fft_x_c2r_col540) run one persistent CTA per SM, so they
// take over from the warp-private kernels only when a pass has at least one tile per SM; below that the warp kernels
// spread the lines better.  BS_FFT_X_COL540: 1 (default) applies that rule, 0 never uses them, 2 uses them wherever
// the geometry allows.
static bool x_col540(bs_ctx* ctx, const PcmGeometry& g, int tiles) {
    const int mode = env_int("BS_FFT_X_COL540", 1);
    return mode && g.P[0] == Col540X::N && env_int("BS_FFT_STATIC", 1) && (mode == 2 || tiles >= ctx->sm_count);
}

static XR2CArgs r2c_args(bs_ctx* ctx, const void* d1, const void* d2, int dtype, const PcmGeometry& g,
                         PcmDeviceTables* t) {
    bs_pcm_workspace& ws = ctx->ws;
    XR2CArgs a;
    a.img[0] = d1; a.img[1] = d2;
    a.spec[0] = (float2*)ws.spec_a; a.spec[1] = (float2*)ws.spec_b;
    a.dtype = dtype;
    a.dx = g.d[0]; a.dy = g.d[1]; a.dz = g.d[2];
    a.Px = g.P[0]; a.Py = g.P[1]; a.Pz = g.P[2]; a.M = g.M; a.pitch = g.pitch;
    a.ex = std::min(g.ext[0], g.d[0]);
    a.Ex = g.E[0]; a.Ey = g.E[1]; a.Ez = g.E[2];
    a.idx_x = t->idx[0]; a.w_x = t->w[0];
    a.idx_y = t->idx[1]; a.w_y = t->w[1];
    a.idx_z = t->idx[2]; a.w_z = t->w[2];
    a.tw = t->tw[0];
    a.plan = g.plan_x;
    a.lshift = g.lshift_r2c;
    return a;
}

// k_fft_x_r2c_col540's arguments and dynamic shared memory; false when pass 0 does not take that kernel
static bool r2c_col540(bs_ctx* ctx, const XR2CArgs& a, int dtype, const PcmGeometry& g, XR2CCol540Args* c,
                       size_t* smem) {
    const int row_bytes = g.d[0] * (dtype == BS_DTYPE_U16 ? 2 : dtype == BS_DTYPE_F32 ? 4 : 1);
    const int col_tiles = (g.P[1] * g.P[2] + COL540_TC - 1) / COL540_TC;
    int raw_stride = (row_bytes + 15) & ~15;   // 16 staged rows on 8 different banks: 4 words times an odd number
    while ((raw_stride / 4) % 8 != 4) raw_stride += 16;
    *smem = (Col540X::XSIZE + (size_t)COL540_TC * COL540_XLP + 2 * (size_t)Col540X::N) * sizeof(float2) +
            4 * COL540_TC * (sizeof(int) + (size_t)raw_stride);
    c->x = a;
    c->row_bytes = row_bytes;
    c->raw_stride = raw_stride;
    c->n_tiles = col_tiles;
    return x_col540(ctx, g, col_tiles) && dtype == BS_DTYPE_U16 && (row_bytes % 16) == 0 && ((size_t)a.img[0] % 16) == 0 &&
           ((size_t)a.img[1] % 16) == 0 && *smem <= PCM_SMEM_MAX;
}

// pass 0: both crops -> blended mirrored extension + zero pad -> R2C along x into ws.spec_a / ws.spec_b
static int pcm_pass_x_r2c(bs_ctx* ctx, const void* d1, const void* d2, int dtype, const PcmGeometry& g,
                          PcmDeviceTables* t, char* info) {
    const XR2CArgs a = r2c_args(ctx, d1, d2, dtype, g, t);
    const int LB = 1 << g.lshift_r2c;
    dim3 grid((g.P[1] + LB - 1) / LB, g.P[2], 2);
    {
        bs_launch_scope sc(ctx, "fft_x_r2c");
        const int esize = dtype == BS_DTYPE_U16 ? 2 : dtype == BS_DTYPE_F32 ? 4 : 1;
        const int row_bytes = g.d[0] * esize;
        const size_t smem_tma = g.smem_x_r2c + 2 * (size_t)LB * row_bytes + 16;
        const bool tma_ok = env_int("BS_FFT_R2C_TMA", 1) != 0 && (row_bytes % 16) == 0 && ((size_t)d1 % 16) == 0 &&
                            ((size_t)d2 % 16) == 0 && smem_tma <= PCM_SMEM_MAX && (g.smem_x_r2c % 16) == 0;
        const int xmode = env_int("BS_FFT_X_WARP", 1);
        const size_t smem_w = ((size_t)g.P[0] + (size_t)(PCM_THREADS / 32) * 2 * g.M) * sizeof(float2) +
                              (tma_ok ? (size_t)(PCM_THREADS / 32) * (2 * (size_t)row_bytes + 16) : 0);
        XR2CCol540Args c;
        size_t smem_col;
        if (r2c_col540(ctx, a, dtype, g, &c, &smem_col)) {
            k_fft_x_r2c_col540<<<std::min(c.n_tiles, ctx->sm_count), COL540X_NT, smem_col, ctx->stream>>>(c);
            pass_info(info, "k_fft_x_r2c_col540", nullptr);
        } else if (xmode && g.M <= 32 * XW_MAXV - 1 && smem_w <= PCM_SMEM_MAX && (((size_t)g.P[0] + 16 * (size_t)g.M) * 8) % 16 == 0) {
            XWArgs w;
            w.x = a;
            w.row_bytes = row_bytes;
            w.use_tma = tma_ok ? 1 : 0;
            w.n_lines = 2LL * g.P[2] * g.P[1];
            const int per_sm = std::max(1, std::min(6, (int)(PCM_SMEM_MAX / (smem_w + 1024))));
            const int nctas = (int)std::min<long long>((w.n_lines + 7) / 8, (long long)ctx->sm_count * per_sm);
            if (g.M == FftW270S::N && env_int("BS_FFT_STATIC", 1)) {
                k_fft_x_r2c_w<FftW270S><<<nctas, PCM_THREADS, smem_w, ctx->stream>>>(w);
                pass_info(info, tma_ok ? "k_fft_x_r2c_w<FftW270S> tma" : "k_fft_x_r2c_w<FftW270S>", nullptr);
            } else {
                k_fft_x_r2c_w<FftWGeneric><<<nctas, PCM_THREADS, smem_w, ctx->stream>>>(w);
                pass_info(info, tma_ok ? "k_fft_x_r2c_w<FftWGeneric> tma" : "k_fft_x_r2c_w<FftWGeneric>", &g.plan_x);
            }
        } else if (tma_ok) {
            XR2CTmaArgs m;
            m.x = a;
            m.n_groups = (g.P[1] + LB - 1) / LB;
            m.n_items = 2 * g.P[2] * m.n_groups;
            m.row_bytes = row_bytes;
            m.esize = esize;
            const int per_sm = std::max(1, (int)(PCM_SMEM_MAX / (smem_tma + 1024)));
            const int nctas = std::min(m.n_items, ctx->sm_count * std::min(per_sm, 4));
            if (g.static_x && g.lshift_r2c == 3) {
                k_fft_x_r2c_tma<FftX270L8><<<nctas, PCM_THREADS, smem_tma, ctx->stream>>>(m);
                pass_info(info, "k_fft_x_r2c_tma<FftX270L8>", nullptr);
            } else if (g.static_x && g.lshift_r2c == 4) {
                k_fft_x_r2c_tma<FftX270><<<nctas, PCM_THREADS, smem_tma, ctx->stream>>>(m);
                pass_info(info, "k_fft_x_r2c_tma<FftX270>", nullptr);
            } else {
                k_fft_x_r2c_tma<FftGeneric><<<nctas, PCM_THREADS, smem_tma, ctx->stream>>>(m);
                pass_info(info, "k_fft_x_r2c_tma<FftGeneric>", &g.plan_x);
            }
        } else if (g.static_x && g.lshift_r2c == 3) {
            k_fft_x_r2c<FftX270L8><<<grid, PCM_THREADS, g.smem_x_r2c, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_r2c<FftX270L8>", nullptr);
        } else if (g.static_x && g.lshift_r2c == 4) {
            k_fft_x_r2c<FftX270><<<grid, PCM_THREADS, g.smem_x_r2c, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_r2c<FftX270>", nullptr);
        } else {
            k_fft_x_r2c<FftGeneric><<<grid, PCM_THREADS, g.smem_x_r2c, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_r2c<FftGeneric>", &g.plan_x);
        }
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

// passes 1 and 3: forward FFT along y, in place, on both spectra (n_img = 2) or on the product in ws.spec_a (1)
static int pcm_launch_y(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables* t, int n_img, const char* tag, char* info) {
    StridedArgs a;
    a.a = (float2*)ctx->ws.spec_a; a.b = (float2*)ctx->ws.spec_b;
    a.estride = g.pitch;
    a.ostride = (long long)g.P[1] * g.pitch;
    a.tw = t->tw[1];
    a.plan = g.plan_y;
    a.tshift = g.tshift_y;
    a.thresh = 0.f;
    dim3 grid(g.pitch >> g.tshift_y, g.P[2], n_img);
    {
        bs_launch_scope sc(ctx, tag);
        const size_t smem_pipe = ((size_t)((g.P[1] + 1) & ~1) + 3 * (size_t)g.P[1] * (1 << g.tshift_y)) * sizeof(float2);
        if (g.static_y) {
            int rc;
            if ((rc = launch_col540(ctx, a, g.pitch / COL540_TC, g.P[2], n_img))) return rc;
            pass_info(info, "k_fft_col540", nullptr);
        } else if (smem_pipe <= PCM_SMEM_MAX) {
            StridedPipeArgs pp;
            pp.s = a;
            pp.tiles_x = g.pitch >> g.tshift_y;
            pp.n_other = g.P[2];
            pp.n_tiles = pp.tiles_x * pp.n_other * n_img;
            const int per_sm = std::max(1, std::min(2, (int)(PCM_SMEM_MAX / (smem_pipe + 1024))));
            const int nctas = std::min(pp.n_tiles, ctx->sm_count * per_sm);
            k_fft_strided_pipe<FftGeneric><<<nctas, PCM_THREADS, smem_pipe, ctx->stream>>>(pp);
            pass_info(info, "k_fft_strided_pipe<FftGeneric>", &g.plan_y);
        } else {
            k_fft_strided<FftGeneric><<<grid, PCM_THREADS, g.smem_y, ctx->stream>>>(a);
            pass_info(info, "k_fft_strided<FftGeneric>", &g.plan_y);
        }
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

// pass 1: forward y FFT of both spectra
static int pcm_pass_y_fwd(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables* t, char* info) {
    return pcm_launch_y(ctx, g, t, 2, "fft_y", info);
}

// pass 2: forward z FFT of both spectra, unit-magnitude normalisation, conj(A) * B, forward z FFT of the product
// into ws.spec_a
static int pcm_pass_z_xpower(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables* t, char* info) {
    StridedArgs a;
    a.a = (float2*)ctx->ws.spec_a; a.b = (float2*)ctx->ws.spec_b;
    a.estride = (long long)g.P[1] * g.pitch;
    a.ostride = g.pitch;
    a.tw = t->tw[2];
    a.plan = g.plan_z;
    a.tshift = g.tshift_z;
    a.thresh = 1e-5f;  // PhaseCorrelation2Util.normalizeInterval threshold
    {
        bs_launch_scope sc(ctx, "fft_z_xpower");
        if (g.static_z) {
            int rc;
            if ((rc = launch_col540(ctx, a, g.pitch / COL540_TC, g.P[1], 0))) return rc;
            pass_info(info, "k_fft_xpower_col540", nullptr);
        } else {
            StridedPipeArgs pp;
            pp.s = a;
            pp.tiles_x = g.pitch >> g.tshift_z;
            pp.n_other = g.P[1];
            pp.n_tiles = pp.tiles_x * pp.n_other;
            const int per_sm = std::max(1, std::min(2, (int)(PCM_SMEM_MAX / (g.smem_z + 1024))));
            const int nctas = std::min(pp.n_tiles, ctx->sm_count * per_sm);
            k_fft_xpower_pipe<FftGeneric><<<nctas, PCM_THREADS, g.smem_z, ctx->stream>>>(pp);
            pass_info(info, "k_fft_xpower_pipe<FftGeneric>", &g.plan_z);
        }
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

// pass 3: forward y FFT of the product
static int pcm_pass_y_inv(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables* t, char* info) {
    return pcm_launch_y(ctx, g, t, 1, "fft_y_inv", info);
}

// pass 4: conj + C2R along x with scale 1 / (M * Py * Pz), in place -> real PCM in ws.spec_a (row pitch 2*pitch floats)
static int pcm_pass_x_c2r(bs_ctx* ctx, const PcmGeometry& g, PcmDeviceTables* t, char* info) {
    XC2RArgs a;
    a.spec = (float2*)ctx->ws.spec_a;
    a.Px = g.P[0]; a.Py = g.P[1]; a.Pz = g.P[2]; a.M = g.M; a.pitch = g.pitch;
    a.tw = t->tw[0];
    a.plan = g.plan_x;
    a.lshift = g.lshift_x;
    a.scale = (float)(1.0 / ((double)g.M * (double)g.P[1] * (double)g.P[2]));
    const int LB = 1 << g.lshift_x;
    dim3 grid((g.P[1] + LB - 1) / LB, g.P[2], 1);
    {
        bs_launch_scope sc(ctx, "fft_x_c2r");
        const size_t smem_w = ((size_t)g.P[0] + (size_t)(PCM_THREADS / 32) * 2 * (g.M + 1)) * sizeof(float2);
        const int col_tiles = (g.P[1] * g.P[2] + 2 * COL540_TC - 1) / (2 * COL540_TC);
        if (x_col540(ctx, g, col_tiles)) {
            XC2RCol540Args c;
            c.x = a;
            c.n_tiles = col_tiles;
            const size_t smem = (2 * (size_t)COL540_TC * COL540_SP + Col540X::XSIZE + Col540X::N) * sizeof(float2) +
                                4 * COL540_TC * sizeof(int) + 2 * sizeof(unsigned long long);
            k_fft_x_c2r_col540<<<std::min(col_tiles, ctx->sm_count), COL540X_NT, smem, ctx->stream>>>(c);
            pass_info(info, "k_fft_x_c2r_col540", nullptr);
        } else if (env_int("BS_FFT_X_WARP", 1) && g.M <= 32 * XW_MAXV - 1 && smem_w <= PCM_SMEM_MAX) {
            const long long n_lines = (long long)g.P[1] * g.P[2];
            const int per_sm = std::max(1, std::min(6, (int)(PCM_SMEM_MAX / (smem_w + 1024))));
            const int nctas = (int)std::min<long long>((n_lines + 7) / 8, (long long)ctx->sm_count * per_sm);
            if (g.M == FftW270::N && env_int("BS_FFT_STATIC", 1)) {
                k_fft_x_c2r_w<FftW270><<<nctas, PCM_THREADS, smem_w, ctx->stream>>>(a);
                pass_info(info, "k_fft_x_c2r_w<FftW270>", nullptr);
            } else {
                k_fft_x_c2r_w<FftWGeneric><<<nctas, PCM_THREADS, smem_w, ctx->stream>>>(a);
                pass_info(info, "k_fft_x_c2r_w<FftWGeneric>", &g.plan_x);
            }
        } else if (g.static_x && g.lshift_x == 3) {
            k_fft_x_c2r<FftX270L8><<<grid, PCM_THREADS, g.smem_x_c2r, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_c2r<FftX270L8>", nullptr);
        } else if (g.static_x) {
            k_fft_x_c2r<FftX270><<<grid, PCM_THREADS, g.smem_x_c2r, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_c2r<FftX270>", nullptr);
        } else {
            k_fft_x_c2r<FftGeneric><<<grid, PCM_THREADS, g.smem_x_c2r, ctx->stream>>>(a);
            pass_info(info, "k_fft_x_c2r<FftGeneric>", &g.plan_x);
        }
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

// k_fft_xy_col540 takes over from passes 0 + 1 when k_fft_x_r2c_col540 would run, Py = 540 (static_y) and one CTA
// of the fused kernel fits on every SM.  BS_FFT_XY_FUSE: 1 (default) applies that rule, 0 keeps the five-pass chain.
static int xy_fuse(bs_ctx* ctx, const PcmGeometry& g, const void* fn, size_t smem, bool* fuse) {
    *fuse = false;
    if (!env_int("BS_FFT_XY_FUSE", 1) || !g.static_y) return BS_OK;
    int occ = 0;
    BS_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, COL540X_NT, smem));
    *fuse = occ >= 1;
    return BS_OK;
}

// CTAs of k_fft_xy_col540's x role: 80 of 132 measured best (DESIGN.md), scaled to the SM count;
// BS_FFT_XY_KX overrides it
static int xy_split(bs_ctx* ctx) {
    return std::max(1, std::min(ctx->sm_count - 1, env_int("BS_FFT_XY_KX", (80 * ctx->sm_count + 66) / 132)));
}

// counters in ws.sync; window: as many planes of plane_bytes as fill half of L2 (BS_FFT_XY_WINDOW overrides)
static int make_handoff(bs_ctx* ctx, const PcmGeometry& g, int code, int ready_full, int done_full, size_t plane_bytes,
                        Handoff* h) {
    int l2 = 0;
    BS_CUDA(ctx, cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, ctx->device));
    h->err = (int*)ctx->ws.sync;
    h->ready = h->err + PCM_SYNC_COUNTERS;
    h->done = h->ready + g.P[2];
    h->code = code;
    h->ready_full = ready_full;
    h->done_full = done_full;
    h->window = std::max(2, env_int("BS_FFT_XY_WINDOW", (int)((size_t)l2 / 2 / plane_bytes)));
    BS_CUDA(ctx, cudaMemsetAsync(h->ready, 0, 2 * sizeof(int) * g.P[2], ctx->stream));
    return BS_OK;
}

// one CTA per SM, launched cooperatively: a grid that cannot be co-resident fails to launch instead of waiting on
// CTAs that never start
template <class Args>
static int launch_fused(bs_ctx* ctx, void (*fn)(Args), const Args& args, size_t smem) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctx->sm_count);
    cfg.blockDim = dim3(COL540X_NT);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    BS_CUDA(ctx, cudaLaunchKernelEx(&cfg, fn, args));
    return BS_OK;
}

static void join_info(char* info, const char* a, const char* b) {
    if (info) snprintf(info, PCM_INFO_LEN, "%s + %s", a, b);
}

// passes 0 + 1: k_fft_xy_col540 when the rule above takes them, else the two passes
static int pcm_pass_xy(bs_ctx* ctx, const void* d1, const void* d2, int dtype, const PcmGeometry& g, PcmDeviceTables* t,
                       char* info) {
    XYCol540Args f;
    size_t smem;
    bool fuse = false;
    int rc;
    if (r2c_col540(ctx, r2c_args(ctx, d1, d2, dtype, g, t), dtype, g, &f.x, &smem) &&
        (rc = xy_fuse(ctx, g, (const void*)k_fft_xy_col540, smem, &fuse)))
        return rc;
    if (!fuse) {
        char i0[PCM_INFO_LEN] = "", i1[PCM_INFO_LEN] = "";
        if ((rc = pcm_pass_x_r2c(ctx, d1, d2, dtype, g, t, i0))) return rc;
        if ((rc = pcm_pass_y_fwd(ctx, g, t, i1))) return rc;
        join_info(info, i0, i1);
        return BS_OK;
    }
    f.tw_y = t->tw[1];
    f.kx = xy_split(ctx);
    bs_launch_scope sc(ctx, "fft_xy");
    if ((rc = make_handoff(ctx, g, PCM_HANDOFF_XY, g.P[1], 2 * (g.pitch / COL540_TC),
                           2 * (size_t)g.P[1] * g.pitch * sizeof(float2), &f.h)) ||
        (rc = launch_fused(ctx, k_fft_xy_col540, f, smem)))
        return rc;
    pass_info(info, "k_fft_xy_col540", nullptr);
    return BS_OK;
}


// forward pipeline up to the real PCM in ws.spec_a (row pitch 2*pitch floats).  The caller resets the hand-off
// error word (pcm_reset_handoff) before and checks it once the stream has passed the pair.
static int pcm_compute_pcm(bs_ctx* ctx, const void* d1, const void* d2, int dtype, const PcmGeometry& g,
                           PcmDeviceTables* t) {
    int rc;
    if ((rc = pcm_kernel_attrs(ctx))) return rc;
    if ((rc = pcm_pass_xy(ctx, d1, d2, dtype, g, t, nullptr))) return rc;
    if ((rc = pcm_pass_z_xpower(ctx, g, t, nullptr))) return rc;
    if ((rc = pcm_pass_y_inv(ctx, g, t, nullptr))) return rc;
    return pcm_pass_x_c2r(ctx, g, t, nullptr);
}

static void solve3(const double H[3][3], const double rhs[3], double out[3]) {
    const double a = H[0][0], b = H[0][1], c = H[0][2], d = H[1][0], e = H[1][1], f = H[1][2], g = H[2][0],
                 h = H[2][1], i = H[2][2];
    const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
    out[0] = out[1] = out[2] = 0.0;
    if (det == 0.0 || !std::isfinite(det)) return;
    const double r0 = rhs[0], r1 = rhs[1], r2 = rhs[2];
    const double x = (r0 * (e * i - f * h) - b * (r1 * i - f * r2) + c * (r1 * h - e * r2)) / det;
    const double y = (a * (r1 * i - f * r2) - r0 * (d * i - f * g) + c * (d * r2 - r1 * g)) / det;
    const double z = (a * (e * r2 - r1 * h) - b * (d * r2 - r1 * g) + r0 * (d * h - e * g)) / det;
    if (std::isfinite(x) && std::isfinite(y) && std::isfinite(z)) { out[0] = x; out[1] = y; out[2] = z; }
}

// quadratic sub-pixel fit on a 3x3x3 neighbourhood nb[dz+1][dy+1][dx+1]
// (imglib2 SubpixelLocalization as used by PhaseCorrelationPeak2.calculateSubpixelLocalization)
static void subpixel_offset(const float* nb, double out[3]) {
    auto f = [&](int z, int y, int x) { return (double)nb[(z * 3 + y) * 3 + x]; };
    const double c = f(1, 1, 1);
    const double g[3] = {(f(1, 1, 2) - f(1, 1, 0)) / 2.0, (f(1, 2, 1) - f(1, 0, 1)) / 2.0, (f(2, 1, 1) - f(0, 1, 1)) / 2.0};
    double H[3][3];
    H[0][0] = f(1, 1, 2) - 2 * c + f(1, 1, 0);
    H[1][1] = f(1, 2, 1) - 2 * c + f(1, 0, 1);
    H[2][2] = f(2, 1, 1) - 2 * c + f(0, 1, 1);
    H[0][1] = H[1][0] = (f(1, 2, 2) - f(1, 2, 0) - f(1, 0, 2) + f(1, 0, 0)) / 4.0;
    H[0][2] = H[2][0] = (f(2, 1, 2) - f(2, 1, 0) - f(0, 1, 2) + f(0, 1, 0)) / 4.0;
    H[1][2] = H[2][1] = (f(2, 2, 1) - f(2, 0, 1) - f(0, 2, 1) + f(0, 0, 1)) / 4.0;
    const double rhs[3] = {-g[0], -g[1], -g[2]};
    solve3(H, rhs, out);
}

struct HostCand {
    long long shift[3];
    int peak;      // index into the peak list
    int order;     // upstream enumeration order
    long long npx;
    double r;
    int slot;      // slot in the device candidate list, -1 when below min overlap
};

static double pearson_from_int_sums(const unsigned long long s[5], long long n) {
    // n*Sxy - Sx*Sy etc. in exact 128-bit integer arithmetic, final ratio in double
    const __int128 N = n;
    const __int128 sa = s[0], sb = s[1], saa = s[2], sbb = s[3], sab = s[4];
    const __int128 cov = N * sab - sa * sb;
    const __int128 va = N * saa - sa * sa;
    const __int128 vb = N * sbb - sb * sb;
    if (va == 0 || vb == 0) return 0.0;  // getCorrelation: constant overlap -> 0
    return (double)cov / (std::sqrt((double)va) * std::sqrt((double)vb));
}

static double pearson_from_dbl_sums(const double s[5], long long n) {
    const double N = (double)n;
    const double cov = s[4] - s[0] * s[1] / N;
    const double va = s[2] - s[0] * s[0] / N;
    const double vb = s[3] - s[1] * s[1] / N;
    if (!(va > 0.0) || !(vb > 0.0)) return 0.0;
    return cov / std::sqrt(va * vb);
}

// full pipeline on device-resident crops
// Result slots: a pair's device-side result block (peaks, neighbourhoods, candidates, Pearson sums) is read
// back by ONE async copy; the host math of pair i (r from integer sums, candidate sort, sub-pixel solve) runs
// after pair i+1 has been enqueued, so the stream never drains between pairs.
#define PCM_SLOTS 2
struct PcmPending {
    bool active = false;
    PcmGeometry g;
    bs_pcm_params p;
    int dtype = 0;
    long long min_px = 0;
    size_t off_sel = 0, off_cands = 0, off_sums = 0, off_err = 0, slot_base = 0;
};

struct PcmSlotState {
    PcmPending pend[PCM_SLOTS];
    cudaEvent_t done[PCM_SLOTS] = {};
};
static std::mutex g_slot_mu;
static std::unordered_map<bs_ctx*, PcmSlotState*> g_slot_states;
static PcmSlotState* slots_of(bs_ctx* ctx) {
    std::lock_guard<std::mutex> lk(g_slot_mu);
    auto it = g_slot_states.find(ctx);
    if (it != g_slot_states.end()) return it->second;
    PcmSlotState* s = new PcmSlotState();
    g_slot_states[ctx] = s;
    return s;
}
void bs_pcm_slots_free(bs_ctx* ctx) {
    std::lock_guard<std::mutex> lk(g_slot_mu);
    auto it = g_slot_states.find(ctx);
    if (it == g_slot_states.end()) return;
    for (int i = 0; i < PCM_SLOTS; ++i)
        if (it->second->done[i]) cudaEventDestroy(it->second->done[i]);
    delete it->second;
    g_slot_states.erase(it);
}

static int pcm_check_params(bs_ctx* ctx, const bs_pcm_params* p, int dtype) {
    if (p->peaks_to_check < 1 || p->peaks_to_check > PCM_KMAX)
        return bs_set_error(ctx, BS_ERR_ARG, "pcm: peaks_to_check must be in [1,%d]", PCM_KMAX);
    if (p->interpolate_xcorr)
        return bs_set_error(ctx, BS_ERR_UNSUPPORTED, "pcm: interpolate_xcorr is not supported (reference default false)");
    if (dtype != BS_DTYPE_U16 && dtype != BS_DTYPE_F32 && dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "pcm: bad dtype %d", dtype);
    return BS_OK;
}

// Pearson sums of up to max_cands candidates (count in ncand[0]; ncand[1] zero) on the context's stream.
// uint16 crops with 16-byte aligned bases take the slab-staged kernel; everything else the generic one.
static int pearson_launch(bs_ctx* ctx, const void* d1, const void* d2, int dtype, const int d[3], const PearsonCand* cands,
                          int max_cands, void* sums, int* ncand) {
    const long long rows = (long long)d[1] * d[2];
    if (dtype == BS_DTYPE_U16 && !((size_t)d1 & 15) && !((size_t)d2 & 15)) {
        PearsonU16Args a;
        a.img1 = (const unsigned short*)d1;
        a.img2 = (const unsigned short*)d2;
        a.dx = d[0]; a.dy = d[1]; a.dz = d[2];
        a.slab_rows = std::max(1, std::min(PRS_ROWS, PRS_STAGE_ELEMS / d[0]));
        a.stage_elems = ((a.slab_rows * d[0] + 32) + 7) & ~7;
        a.nslabs = (int)((rows + a.slab_rows - 1) / a.slab_rows);
        a.cands = cands;
        a.sums = (unsigned long long*)sums;
        a.ncand = ncand;
        a.counter = ncand + 1;
        const size_t smem = sizeof(unsigned short) * 2 * (size_t)a.stage_elems + (sizeof(PearsonCand) + 40) * max_cands;
        if (!ctx->pearson_attr_done) {   // per device: the opt-in leaves room for the kernel's static shared memory
            cudaFuncAttributes fa;
            BS_CUDA(ctx, cudaFuncGetAttributes(&fa, k_pearson_u16));
            BS_CUDA(ctx, cudaFuncSetAttribute(k_pearson_u16, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)(PCM_SMEM_MAX - fa.sharedSizeBytes)));
            ctx->pearson_attr_done = true;
        }
        if (ctx->pearson_smem != smem) {
            int occ = 0;
            BS_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_pearson_u16, PCM_THREADS, smem));
            if (occ < 1) return bs_set_error(ctx, BS_ERR_ARG, "pcm: %d Pearson candidates do not fit in shared memory", max_cands);
            ctx->pearson_occ = occ;
            ctx->pearson_smem = smem;
        }
        const int ctas = (int)std::min<long long>(a.nslabs, (long long)ctx->sm_count * ctx->pearson_occ);
        bs_launch_scope sc(ctx, "pearson");
        k_pearson_u16<<<ctas, PCM_THREADS, smem, ctx->stream>>>(a);
    } else {
        PearsonArgs a;
        a.img1 = d1; a.img2 = d2;
        a.dtype = dtype;
        a.dx = d[0]; a.dy = d[1]; a.dz = d[2];
        a.cands = cands;
        a.sums_u = (unsigned long long*)sums;
        a.sums_d = (double*)sums;
        const long long chunks = (rows + PR_ROWS - 1) / PR_ROWS;
        const int ctas = (int)std::max<long long>(1, std::min<long long>((chunks + 7) / 8, (long long)ctx->sm_count * 8));
        bs_launch_scope sc(ctx, "pearson");
        k_pearson<<<ctas, PCM_THREADS, sizeof(unsigned long long) * 5 * max_cands, ctx->stream>>>(a, ncand);
    }
    BS_CUDA(ctx, cudaGetLastError());
    return BS_OK;
}

// everything of one pair that runs on the device, asynchronously, into result slot `slot`
static int pcm_enqueue(bs_ctx* ctx, const void* d1, const void* d2, const long long dims[3], int dtype,
                       const bs_pcm_params* p, int slot) {
    int rc = pcm_check_params(ctx, p, dtype);
    if (rc) return rc;
    PcmSlotState* S = slots_of(ctx);
    PcmPending& pd = S->pend[slot];
    if ((rc = pcm_geometry(ctx, dims, p->extension, &pd.g))) return rc;
    const PcmGeometry& g = pd.g;
    PcmDeviceTables* t;
    if ((rc = pcm_tables(ctx, g, &t))) return rc;
    if ((rc = pcm_workspace(ctx, g))) return rc;
    if ((rc = pcm_reset_handoff(ctx))) return rc;
    if ((rc = pcm_compute_pcm(ctx, d1, d2, dtype, g, t))) return rc;

    bs_pcm_workspace& ws = ctx->ws;
    const int K = p->peaks_to_check;
    // one resident wave of persistent CTAs (the kernel is latency bound: a second, partial wave halves the bytes in flight
    // for the tail of the launch)
    static int peak_occ = 0;
    if (!peak_occ) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&peak_occ, k_peaks, PCM_THREADS, 0) != cudaSuccess || peak_occ < 1) peak_occ = 4;
        peak_occ = std::min(peak_occ, env_int("BS_PEAKS_CTAS_PER_SM", 8));
    }
    const int peak_ctas = std::max(1, std::min(ctx->sm_count * peak_occ, (g.P[1] * g.P[2] + 7) / 8));
    // small-buffer layout of one slot (device and pinned mirror share offsets)
    const size_t slot_bytes = ws.small_bytes / PCM_SLOTS;
    pd.slot_base = (size_t)slot * slot_bytes;
    size_t off = 0;
    pd.off_sel = off;   off += (sizeof(PcmSelect) + 15) & ~(size_t)15;
    pd.off_cands = off; off += sizeof(PearsonCand) * 8 * PCM_KMAX;
    pd.off_sums = off;  off += sizeof(unsigned long long) * 5 * 8 * PCM_KMAX;
    const size_t readback = off;
    const size_t off_ncand = off; off += 16;
    pd.off_err = off;   off += 16;
    const size_t off_peaks = off; off += sizeof(PeakEntry) * (size_t)peak_ctas * K;
    if (off > slot_bytes) return bs_set_error(ctx, BS_ERR_NOMEM, "pcm: scratch too small");
    unsigned char* dsmall = (unsigned char*)ws.small + pd.slot_base;
    unsigned char* hsmall = (unsigned char*)ws.small_host + pd.slot_base;
    {
        PeakArgs a;
        a.pcm = (const float*)ws.spec_a;
        a.Px = g.P[0]; a.Py = g.P[1]; a.Pz = g.P[2];
        a.rowpitch = 2LL * g.pitch;
        a.K = K;
        a.out = (PeakEntry*)(dsmall + off_peaks);
        bs_launch_scope sc(ctx, "peaks");
        k_peaks<<<peak_ctas, PCM_THREADS, 0, ctx->stream>>>(a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    const long long n_px = (long long)g.d[0] * g.d[1] * g.d[2];
    pd.min_px = (long long)((double)n_px * p->min_overlap_frac);
    pd.p = *p;
    pd.dtype = dtype;
    {
        SelectArgs a;
        a.peaks = (const PeakEntry*)(dsmall + off_peaks);
        a.n_entries = peak_ctas * K;
        a.K = K;
        for (int d = 0; d < 3; ++d) { a.P[d] = g.P[d]; a.d[d] = g.d[d]; }
        a.rowpitch = 2LL * g.pitch;
        a.pcm = (const float*)ws.spec_a;
        a.min_px = pd.min_px;
        a.do_subpixel = p->do_subpixel ? 1 : 0;
        a.sel = (PcmSelect*)(dsmall + pd.off_sel);
        a.cands = (PearsonCand*)(dsmall + pd.off_cands);
        a.sums = (unsigned long long*)(dsmall + pd.off_sums);
        a.ncand = (int*)(dsmall + off_ncand);
        bs_launch_scope sc(ctx, "select");
        k_pcm_select<<<1, 256, 0, ctx->stream>>>(a);
    }
    BS_CUDA(ctx, cudaGetLastError());
    if ((rc = pearson_launch(ctx, d1, d2, dtype, g.d, (const PearsonCand*)(dsmall + pd.off_cands), 8 * K,
                             dsmall + pd.off_sums, (int*)(dsmall + off_ncand))))
        return rc;
    BS_CUDA(ctx, cudaMemcpyAsync(hsmall, dsmall, readback, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(hsmall + pd.off_err, ws.sync, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (!S->done[slot]) BS_CUDA(ctx, cudaEventCreateWithFlags(&S->done[slot], cudaEventDisableTiming));
    BS_CUDA(ctx, cudaEventRecord(S->done[slot], ctx->stream));
    pd.active = true;
    return BS_OK;
}

// host half of a pair: wait for its result block, derive r, sort the candidates, solve the sub-pixel fit
static int pcm_finish(bs_ctx* ctx, int slot, bs_pcm_result* out) {
    PcmSlotState* S = slots_of(ctx);
    PcmPending& pd = S->pend[slot];
    memset(out, 0, sizeof(*out));
    out->r = -INFINITY;
    if (!pd.active) return bs_set_error(ctx, BS_ERR_ARG, "pcm: no pending pair in slot %d", slot);
    pd.active = false;
    BS_CUDA(ctx, cudaEventSynchronize(S->done[slot]));
    const PcmGeometry& g = pd.g;
    for (int d = 0; d < 3; ++d) out->pad[d] = g.P[d];
    const unsigned char* hsmall = (const unsigned char*)ctx->ws.small_host + pd.slot_base;
    int rc = pcm_handoff_error(ctx, *(const int*)(hsmall + pd.off_err));
    if (rc) return rc;
    const PcmSelect* sel = (const PcmSelect*)(hsmall + pd.off_sel);
    const unsigned long long* hsums = (const unsigned long long*)(hsmall + pd.off_sums);
    const int np = sel->np;
    if (np == 0) return BS_OK;  // found = 0
    // same enumeration as k_pcm_select: slots are numbered in (peak, candidate) order
    std::vector<HostCand> cands;
    int nslots = 0;
    for (int pi = 0; pi < np; ++pi) {
        const long long li = sel->idx[pi];
        const long long loc[3] = {li % g.P[0], (li / g.P[0]) % g.P[1], li / ((long long)g.P[0] * g.P[1])};
        for (int i = 0; i < 8; ++i) {
            HostCand c;
            c.peak = pi;
            c.order = pi * 8 + i;
            c.r = -INFINITY;
            c.npx = 0;
            c.slot = -1;
            PearsonCand pc;
            memset(&pc, 0, sizeof(pc));
            long long npx = 0;
            if (pcm_expand_candidate(loc, g.P, g.d, i, pd.min_px, c.shift, &pc, &npx)) {
                out->pearson_px += npx;
                c.npx = npx;
                c.slot = nslots++;
            }
            cands.push_back(c);
        }
    }
    if (nslots != sel->nslots)
        return bs_set_error(ctx, BS_ERR_CUDA, "pcm: candidate enumeration mismatch (host %d, device %d)", nslots, sel->nslots);
    out->n_candidates = nslots;
    for (auto& c : cands) {
        if (c.slot < 0) continue;
        if (pd.dtype == BS_DTYPE_F32) c.r = pearson_from_dbl_sums((const double*)hsums + 5 * c.slot, c.npx);
        else c.r = pearson_from_int_sums(hsums + 5 * c.slot, c.npx);
    }
    // Collections.sort(peaks, reverseOrder(by crossCorr, then nPixel)) -- stable
    std::stable_sort(cands.begin(), cands.end(), [](const HostCand& x, const HostCand& y) {
        if (x.r != y.r) return x.r > y.r;
        return x.npx > y.npx;
    });
    const HostCand& best = cands[0];
    if (std::isinf(best.r)) return BS_OK;  // found = 0
    out->found = 1;
    out->r = best.r;
    out->n_overlap_px = best.npx;
    const long long li = sel->idx[best.peak];
    out->peak_index[0] = li % g.P[0];
    out->peak_index[1] = (li / g.P[0]) % g.P[1];
    out->peak_index[2] = li / ((long long)g.P[0] * g.P[1]);
    out->pcm_value = sel->val[best.peak];
    double sub[3] = {0, 0, 0};
    if (pd.p.do_subpixel) subpixel_offset(sel->nb + 27 * best.peak, sub);
    for (int d = 0; d < 3; ++d) {
        out->shift_int[d] = best.shift[d];
        out->shift_sub[d] = (double)best.shift[d] + sub[d];
    }
    return BS_OK;
}

static size_t crop_bytes_of(const long long dims[3], int dtype) {
    const size_t es = dtype == BS_DTYPE_U16 ? 2 : dtype == BS_DTYPE_F32 ? 4 : 1;
    return (size_t)dims[0] * dims[1] * dims[2] * es;
}

static int ensure_crop_buffers(bs_ctx* ctx, size_t bytes, int nbuf) {
    bs_pcm_workspace& ws = ctx->ws;
    if (ws.crop_bytes >= bytes && ws.crop[0][0] && (nbuf < 2 || ws.crop[1][0])) return BS_OK;
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    const size_t nb = std::max(bytes, ws.crop_bytes);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) {
            if (ws.crop[i][j]) cudaFree(ws.crop[i][j]);
            ws.crop[i][j] = nullptr;
        }
    ws.crop_bytes = 0;
    for (int i = 0; i < nbuf; ++i)
        for (int j = 0; j < 2; ++j) BS_CUDA(ctx, cudaMalloc(&ws.crop[i][j], nb));
    for (int i = 0; i < 2; ++i) {
        if (!ws.crop_ready[i]) BS_CUDA(ctx, cudaEventCreateWithFlags(&ws.crop_ready[i], cudaEventDisableTiming));
        if (!ws.crop_free[i]) BS_CUDA(ctx, cudaEventCreateWithFlags(&ws.crop_free[i], cudaEventDisableTiming));
    }
    ws.crop_bytes = nb;
    return BS_OK;
}

extern "C" {

void bs_pcm_default_params(bs_pcm_params* p) {
    if (!p) return;
    p->peaks_to_check = 5;
    p->do_subpixel = 1;
    p->interpolate_xcorr = 0;
    p->min_overlap_frac = 0.25;
    p->extension[0] = p->extension[1] = p->extension[2] = 10;
}

int bs_pcm_pair(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3], int dtype,
                const bs_pcm_params* params, int on_device, bs_pcm_result* out) {
    if (!ctx) return BS_ERR_ARG;
    const void* a1[1] = {img1};
    const void* a2[1] = {img2};
    return bs_pcm_batch(ctx, 1, a1, a2, dims, dtype, params, on_device, out);
}

int bs_pcm_batch(bs_ctx* ctx, int n, const void* const* img1, const void* const* img2, const long long* dims,
                 int dtype, const bs_pcm_params* params, int on_device, bs_pcm_result* out) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n < 0 || (n > 0 && (!img1 || !img2 || !dims || !params || !out)))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_batch: NULL argument");
    if (n == 0) return BS_OK;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n > 0 && (params->peaks_to_check < 1 || params->peaks_to_check > PCM_KMAX))
        return bs_set_error(ctx, BS_ERR_ARG, "pcm: peaks_to_check must be in [1,%d]", PCM_KMAX);
    for (int i = 0; i < n; ++i) {
        if (!img1[i] || !img2[i]) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_batch: pair %d has a NULL image", i);
        for (int d = 0; d < 3; ++d)
            if (dims[3 * i + d] <= 0) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_batch: pair %d has dims[%d] <= 0", i, d);
        // validate every pair's geometry BEFORE any byte is copied or any kernel is launched
        PcmGeometry g;
        const int rc = pcm_geometry(ctx, dims + 3 * i, params->extension, &g);
        if (rc) return rc;
    }
    // pair i's host half (result read-back, candidate sort, sub-pixel solve) runs after pair i+1 was enqueued.
    // A change of geometry rebuilds tables / workspace, so the previous pair is finished first.
    auto same_dims = [&](int i, int j) {
        return dims[3 * i] == dims[3 * j] && dims[3 * i + 1] == dims[3 * j + 1] && dims[3 * i + 2] == dims[3 * j + 2];
    };
    if (on_device) {
        int pending = -1;
        for (int i = 0; i < n; ++i) {
            if (pending >= 0 && !same_dims(i, pending)) {
                int rc = pcm_finish(ctx, pending & 1, out + pending);
                if (rc) return rc;
                pending = -1;
            }
            int rc = pcm_enqueue(ctx, img1[i], img2[i], dims + 3 * i, dtype, params, i & 1);
            if (rc) return rc;
            if (pending >= 0 && (rc = pcm_finish(ctx, pending & 1, out + pending))) return rc;
            pending = i;
        }
        if (pending >= 0) return pcm_finish(ctx, pending & 1, out + pending);
        return BS_OK;
    }
    // host inputs: double-buffered H2D on the copy stream, overlapped with the previous pair
    size_t maxb = 0;
    for (int i = 0; i < n; ++i) maxb = std::max(maxb, crop_bytes_of(dims + 3 * i, dtype));
    int rc = ensure_crop_buffers(ctx, maxb, n > 1 ? 2 : 1);
    if (rc) return rc;
    bs_pcm_workspace& ws = ctx->ws;
    auto enqueue_copy = [&](int i) -> int {
        const int b = i & 1;
        const size_t bytes = crop_bytes_of(dims + 3 * i, dtype);
        if (i >= 2) BS_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ws.crop_free[b], 0));
        BS_CUDA(ctx, cudaMemcpyAsync(ws.crop[b][0], img1[i], bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        BS_CUDA(ctx, cudaMemcpyAsync(ws.crop[b][1], img2[i], bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        BS_CUDA(ctx, cudaEventRecord(ws.crop_ready[b], ctx->copy_stream));
        return BS_OK;
    };
    if (n > 0 && (rc = enqueue_copy(0))) return rc;
    int pending = -1;
    for (int i = 0; i < n; ++i) {
        const int b = i & 1;
        if (i + 1 < n && (rc = enqueue_copy(i + 1))) return rc;
        if (pending >= 0 && !same_dims(i, pending)) {
            if ((rc = pcm_finish(ctx, pending & 1, out + pending))) return rc;
            pending = -1;
        }
        BS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ws.crop_ready[b], 0));
        rc = pcm_enqueue(ctx, ws.crop[b][0], ws.crop[b][1], dims + 3 * i, dtype, params, b);
        if (rc) return rc;
        BS_CUDA(ctx, cudaEventRecord(ws.crop_free[b], ctx->stream));
        if (pending >= 0 && (rc = pcm_finish(ctx, pending & 1, out + pending))) return rc;
        pending = i;
    }
    if (pending >= 0) return pcm_finish(ctx, pending & 1, out + pending);
    return BS_OK;
}

int bs_pcm_volumes_batch(bs_ctx* ctx, int n, const bs_pcm_job* jobs, const bs_pcm_params* params, bs_pcm_result* out) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n < 0 || (n > 0 && (!jobs || !params || !out))) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_volumes_batch: NULL argument");
    if (n == 0) return BS_OK;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    // validate everything before any launch
    size_t maxb = 0;
    bool need_crop = false;
    int dtype = -1;
    for (int i = 0; i < n; ++i) {
        const bs_pcm_job& j = jobs[i];
        auto i1 = ctx->vols.find(j.vol1), i2 = ctx->vols.find(j.vol2);
        if (i1 == ctx->vols.end() || i2 == ctx->vols.end())
            return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_volumes_batch: job %d has an unknown volume handle", i);
        if (i1->second.dtype != i2->second.dtype) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_volumes_batch: job %d mixes dtypes", i);
        if (dtype >= 0 && i1->second.dtype != dtype) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_volumes_batch: mixed dtypes in one batch");
        dtype = i1->second.dtype;
        for (int d = 0; d < 3; ++d) {
            if (j.dims[d] <= 0 || j.min1[d] < 0 || j.min2[d] < 0 || j.min1[d] + j.dims[d] > i1->second.dims[d] ||
                j.min2[d] + j.dims[d] > i2->second.dims[d])
                return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_volumes_batch: job %d: overlap interval outside the volume (axis %d)", i, d);
        }
        PcmGeometry g;
        int rc = pcm_geometry(ctx, j.dims, params->extension, &g);
        if (rc) return rc;
        const bool whole1 = j.dims[0] == i1->second.dims[0] && j.dims[1] == i1->second.dims[1] && j.dims[2] == i1->second.dims[2];
        const bool whole2 = j.dims[0] == i2->second.dims[0] && j.dims[1] == i2->second.dims[1] && j.dims[2] == i2->second.dims[2];
        if (!whole1 || !whole2) {
            need_crop = true;
            maxb = std::max(maxb, crop_bytes_of(j.dims, dtype));
        }
    }
    int rc = pcm_check_params(ctx, params, dtype);
    if (rc) return rc;
    if (need_crop && (rc = ensure_crop_buffers(ctx, maxb, 2))) return rc;
    bs_pcm_workspace& ws = ctx->ws;
    const size_t es = dtype == BS_DTYPE_U16 ? 2 : dtype == BS_DTYPE_F32 ? 4 : 1;
    // the overlap crop of a volume: the volume itself when the interval covers it, else a strided device copy
    auto crop = [&](bs_volume& v, const long long mn[3], const long long dims[3], void* dst, const void** out_ptr) -> int {
        if (dims[0] == v.dims[0] && dims[1] == v.dims[1] && dims[2] == v.dims[2]) { *out_ptr = v.dev; return BS_OK; }
        cudaMemcpy3DParms p;
        memset(&p, 0, sizeof(p));
        p.srcPtr = make_cudaPitchedPtr(v.dev, (size_t)v.dims[0] * es, (size_t)v.dims[0], (size_t)v.dims[1]);
        p.srcPos = make_cudaPos((size_t)mn[0] * es, (size_t)mn[1], (size_t)mn[2]);
        p.dstPtr = make_cudaPitchedPtr(dst, (size_t)dims[0] * es, (size_t)dims[0], (size_t)dims[1]);
        p.extent = make_cudaExtent((size_t)dims[0] * es, (size_t)dims[1], (size_t)dims[2]);
        p.kind = cudaMemcpyDeviceToDevice;
        BS_CUDA(ctx, cudaMemcpy3DAsync(&p, ctx->stream));
        ctx->launches++;
        *out_ptr = dst;
        return BS_OK;
    };
    auto same_dims = [&](int i, int j) {
        return jobs[i].dims[0] == jobs[j].dims[0] && jobs[i].dims[1] == jobs[j].dims[1] && jobs[i].dims[2] == jobs[j].dims[2];
    };
    int pending = -1;
    for (int i = 0; i < n; ++i) {
        const bs_pcm_job& j = jobs[i];
        bs_volume& v1 = ctx->vols.find(j.vol1)->second;
        bs_volume& v2 = ctx->vols.find(j.vol2)->second;
        if ((rc = bs_volume_acquire(ctx, v1)) || (rc = bs_volume_acquire(ctx, v2))) return rc;
        if (pending >= 0 && !same_dims(i, pending)) {
            if ((rc = pcm_finish(ctx, pending & 1, out + pending))) return rc;
            pending = -1;
        }
        const int b = i & 1;
        const void *p1 = nullptr, *p2 = nullptr;
        // crop buffers of slot b were last read by pair i-2's Pearson kernel: same stream, already ordered
        if ((rc = crop(v1, j.min1, j.dims, need_crop ? ws.crop[b][0] : nullptr, &p1))) return rc;
        if ((rc = crop(v2, j.min2, j.dims, need_crop ? ws.crop[b][1] : nullptr, &p2))) return rc;
        if ((rc = pcm_enqueue(ctx, p1, p2, j.dims, dtype, params, b))) return rc;
        if (pending >= 0 && (rc = pcm_finish(ctx, pending & 1, out + pending))) return rc;
        pending = i;
    }
    if (pending >= 0) return pcm_finish(ctx, pending & 1, out + pending);
    return BS_OK;
}

int bs_pcm_debug_pcm(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3], int dtype,
                     const int extension[3], float* out_pcm, int pad_out[3]) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!img1 || !img2 || !dims || !extension || !out_pcm)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pcm: NULL argument");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    PcmGeometry g;
    int rc = pcm_geometry(ctx, dims, extension, &g);
    if (rc) return rc;
    PcmDeviceTables* t;
    if ((rc = pcm_tables(ctx, g, &t))) return rc;
    if ((rc = pcm_workspace(ctx, g))) return rc;
    const size_t bytes = crop_bytes_of(dims, dtype);
    if ((rc = ensure_crop_buffers(ctx, bytes, 1))) return rc;
    bs_pcm_workspace& ws = ctx->ws;
    BS_CUDA(ctx, cudaMemcpyAsync(ws.crop[0][0], img1, bytes, cudaMemcpyHostToDevice, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(ws.crop[0][1], img2, bytes, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = pcm_reset_handoff(ctx))) return rc;
    if ((rc = pcm_compute_pcm(ctx, ws.crop[0][0], ws.crop[0][1], dtype, g, t))) return rc;
    BS_CUDA(ctx, cudaMemcpy2DAsync(out_pcm, sizeof(float) * g.P[0], ws.spec_a, sizeof(float2) * g.pitch,
                                   sizeof(float) * g.P[0], (size_t)g.P[1] * g.P[2], cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = pcm_sync_handoff(ctx))) return rc;
    if (pad_out) for (int d = 0; d < 3; ++d) pad_out[d] = g.P[d];
    return BS_OK;
}

int bs_pcm_debug_pass(bs_ctx* ctx, int pass, const long long dims[3], int dtype, const int extension[3], const void* in_a,
                      const void* in_b, void* out_a, void* out_b, int poison, int pad_out[3], char info[128]) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (pass < 0 || pass > 5) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pass: pass %d not in [0,5]", pass);
    const bool crops = pass == 0 || pass == 5;
    const bool two = pass <= 2 || pass == 5;    // read both spectra / crops
    const bool two_out = pass <= 1 || pass == 5;
    const bool real_out = pass == 4;
    if (!dims || !extension || !in_a || (two && !in_b) || !out_a || (two_out && !out_b))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pass: NULL argument");
    if (crops && dtype != BS_DTYPE_U16 && dtype != BS_DTYPE_F32 && dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pass: bad dtype %d", dtype);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int i = 0; crops && i < 2; ++i) {   // the x kernels read the crops directly
        cudaPointerAttributes pa;
        BS_CUDA(ctx, cudaPointerGetAttributes(&pa, i ? in_b : in_a));
        if (pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged)
            return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pass: pass %d takes device crops (in_%c)", pass,
                                i ? 'b' : 'a');
    }
    PcmGeometry g;
    int rc = pcm_geometry(ctx, dims, extension, &g);
    if (rc) return rc;
    PcmDeviceTables* t;
    if ((rc = pcm_tables(ctx, g, &t))) return rc;
    if ((rc = pcm_workspace(ctx, g))) return rc;
    if ((rc = pcm_kernel_attrs(ctx))) return rc;
    bs_pcm_workspace& ws = ctx->ws;
    const size_t spec_bytes = (size_t)g.P[2] * g.P[1] * g.pitch * sizeof(float2);
    const size_t row = (size_t)(g.M + 1) * sizeof(float2), rows = (size_t)g.P[1] * g.P[2];
    void* spec[2] = {ws.spec_a, ws.spec_b};
    const void* in[2] = {in_a, in_b};
    void* out[2] = {out_a, out_b};
    for (int i = 0; i < 2; ++i) BS_CUDA(ctx, cudaMemsetAsync(spec[i], poison ? 0xff : 0, spec_bytes, ctx->stream));
    if ((rc = pcm_reset_handoff(ctx))) return rc;
    if (!crops)
        for (int i = 0; i < (two ? 2 : 1); ++i)
            BS_CUDA(ctx, cudaMemcpy2DAsync(spec[i], sizeof(float2) * g.pitch, in[i], row, row, rows, cudaMemcpyHostToDevice,
                                           ctx->stream));
    char buf[PCM_INFO_LEN] = "";
    switch (pass) {
        case 0: rc = pcm_pass_x_r2c(ctx, in_a, in_b, dtype, g, t, buf); break;
        case 1: rc = pcm_pass_y_fwd(ctx, g, t, buf); break;
        case 2: rc = pcm_pass_z_xpower(ctx, g, t, buf); break;
        case 3: rc = pcm_pass_y_inv(ctx, g, t, buf); break;
        case 4: rc = pcm_pass_x_c2r(ctx, g, t, buf); break;
        default: rc = pcm_pass_xy(ctx, in_a, in_b, dtype, g, t, buf); break;
    }
    if (rc) return rc;
    if (real_out) {
        BS_CUDA(ctx, cudaMemcpy2DAsync(out_a, sizeof(float) * g.P[0], ws.spec_a, sizeof(float2) * g.pitch,
                                       sizeof(float) * g.P[0], rows, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        for (int i = 0; i < (two_out ? 2 : 1); ++i)
            BS_CUDA(ctx, cudaMemcpy2DAsync(out[i], row, spec[i], sizeof(float2) * g.pitch, row, rows,
                                           cudaMemcpyDeviceToHost, ctx->stream));
    }
    if ((rc = pcm_sync_handoff(ctx))) return rc;
    if (pad_out) for (int d = 0; d < 3; ++d) pad_out[d] = g.P[d];
    if (info) memcpy(info, buf, PCM_INFO_LEN);
    return BS_OK;
}

int bs_pcm_debug_pearson(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3], int dtype, int n,
                         const int* boxes, void* sums_out) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!img1 || !img2 || !dims || (n > 0 && (!boxes || !sums_out)))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pearson: NULL argument");
    if (n < 0 || n > 8 * PCM_KMAX)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pearson: n must be in [0,%d]", 8 * PCM_KMAX);
    if (dtype != BS_DTYPE_U16 && dtype != BS_DTYPE_F32 && dtype != BS_DTYPE_U8)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pearson: bad dtype %d", dtype);
    int d[3];
    for (int a = 0; a < 3; ++a) {
        if (dims[a] <= 0 || dims[a] > 16384) return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pearson: dims out of range");
        d[a] = (int)dims[a];
    }
    std::vector<PearsonCand> hc(std::max(n, 1));
    for (int i = 0; i < n; ++i) {
        const int* b = boxes + 9 * i;
        PearsonCand& c = hc[i];
        for (int a = 0; a < 3; ++a) {
            c.o1[a] = b[a]; c.o2[a] = b[3 + a]; c.sz[a] = b[6 + a];
            if (c.o1[a] < 0 || c.o2[a] < 0 || c.sz[a] < 0 || c.o1[a] + c.sz[a] > d[a] || c.o2[a] + c.sz[a] > d[a])
                return bs_set_error(ctx, BS_ERR_ARG, "bs_pcm_debug_pearson: box %d leaves the volume (axis %d)", i, a);
        }
        c.pad = 0;
    }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    // device block: candidates, sums, {count, slab counter}
    const size_t cb = sizeof(PearsonCand) * hc.size(), sb = sizeof(unsigned long long) * 5 * hc.size();
    unsigned char* dev = nullptr;
    BS_CUDA(ctx, cudaMalloc(&dev, cb + sb + 16));
    const int cnt[2] = {n, 0};
    int rc = BS_OK;
    cudaError_t e = cudaMemcpyAsync(dev, hc.data(), cb, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(dev + cb, 0, sb, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dev + cb + sb, cnt, sizeof(cnt), cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) rc = bs_set_error(ctx, BS_ERR_CUDA, "bs_pcm_debug_pearson: %s", cudaGetErrorString(e));
    if (!rc) rc = pearson_launch(ctx, img1, img2, dtype, d, (const PearsonCand*)dev, (int)hc.size(), dev + cb, (int*)(dev + cb + sb));
    if (!rc && n > 0) {
        e = cudaMemcpyAsync(sums_out, dev + cb, sizeof(unsigned long long) * 5 * n, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) rc = bs_set_error(ctx, BS_ERR_CUDA, "bs_pcm_debug_pearson: %s", cudaGetErrorString(e));
    }
    cudaStreamSynchronize(ctx->stream);
    cudaFree(dev);
    return rc;
}

}  // extern "C"
