// probe: where the time of the uint16 Pearson verification goes.  Two seeded 512^3 uint16 volumes and two candidate
// lists of the bench's size: (1) the wrap candidates (pcm_expand_candidate, min overlap 0.25) of one true peak near
// shift 0 and 4 noise peaks at seeded random locations of the 540^3 PCM; (2) as many candidates, all with shifts
// within +-4 voxels.  Timed per list (CUDA events, 20 launches after 3 warm-ups):
//   (r) a plain 16-byte read of both volumes (the card's streaming-read bandwidth);
//   (a) the previous traversal (k_pearson's old uint16 path);
//   (b) the slab-staged traversal of k_pearson_u16 with the arithmetic replaced by one XOR per word;
//   (c) (b) plus the exact sums taken the previous way (three 64-bit multiply-accumulates per element);
//   (d) (b) plus the exact sums from packed 16 x 8-bit dot products (IDP.2A) into 32-bit partials;
//   (e) (d) with the loop over a warp's rows not unrolled, and optionally one more chunk per lane in a row's last
//       round; "as built" is k_pearson_u16 itself.
// (c) and (d) at several slab heights and chunks per lane per round (U).
// "DRAM" bytes are the slab design's traffic: image 1 once plus image 2 once per candidate box (2 n + 2 sum npx).
// (c) - (e)'s sums are checked against (a)'s.  (b) - (e) are a copy of k_pearson_u16 from csrc/pcm.cu with the
// arithmetic, the chunks per lane and the row loop's unrolling as template parameters; keep them in step when the
// kernel changes.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a pearson_probe.cu -o pearson_probe && ./pearson_probe
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <type_traits>
#include <vector>

#define NT 256
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

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
};

// (a) the previous uint16 traversal: a warp owns PR_ROWS image-1 rows and re-reads them, and the shifted image-2
// rows, from global memory for every candidate
#define PR_ROWS 16
#define PR_MLP 8

__device__ __forceinline__ void pr_acc(unsigned int va, unsigned int vb, unsigned int& ra, unsigned int& rb,
                                       unsigned long long& saa, unsigned long long& sbb, unsigned long long& sab) {
    ra += va;
    rb += vb;
    saa += (unsigned long long)va * va;   // one IMAD.WIDE.U32 with 64-bit accumulate each
    sbb += (unsigned long long)vb * vb;
    sab += (unsigned long long)va * vb;
}

__device__ __forceinline__ void pearson_u16(const PearsonArgs& a, int ncand, unsigned long long* s_acc) {
    const unsigned short* __restrict__ i1 = (const unsigned short*)a.img1;
    const unsigned short* __restrict__ i2 = (const unsigned short*)a.img2;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const long long nrows = (long long)a.dy * a.dz;
    const long long nchunks = (nrows + PR_ROWS - 1) / PR_ROWS;
    const bool even_rows = !(a.dx & 1) && !((size_t)i1 & 3) && !((size_t)i2 & 3);
    for (long long ch = (long long)blockIdx.x * nw + wid; ch < nchunks; ch += (long long)gridDim.x * nw) {
        const long long r0 = ch * PR_ROWS;
        const int z0 = (int)(r0 / a.dy), y0 = (int)(r0 - (long long)z0 * a.dy);
        for (int c = 0; c < ncand; ++c) {
            const PearsonCand cd = a.cands[c];
            unsigned long long sa = 0, sb = 0, saa = 0, sbb = 0, sab = 0;
            bool any = false;
            // both x offsets even -> aligned ushort2 loads on both images
            const bool vec = even_rows && !((cd.o1[0] | cd.o2[0]) & 1);
            for (int rr = 0; rr < PR_ROWS; ++rr) {
                const long long r = r0 + rr;
                if (r >= nrows) break;
                int z = z0, y = y0 + rr;          // (z, y) of row r0 + rr without a 64-bit division per row
                while (y >= a.dy) { y -= a.dy; ++z; }
                const int yy = y - cd.o1[1], zz = z - cd.o1[2];
                if (yy < 0 || yy >= cd.sz[1] || zz < 0 || zz >= cd.sz[2]) continue;
                any = true;
                const unsigned short* p1 = i1 + (size_t)r * a.dx + cd.o1[0];
                const unsigned short* p2 = i2 + ((size_t)(zz + cd.o2[2]) * a.dy + (yy + cd.o2[1])) * a.dx + cd.o2[0];
                unsigned int ra = 0, rb = 0;
                const int n = cd.sz[0];
                if (vec) {
                    const unsigned int* q1 = reinterpret_cast<const unsigned int*>(p1);
                    const unsigned int* q2 = reinterpret_cast<const unsigned int*>(p2);
                    const int nv = n >> 1;
                    for (int x0 = lane; x0 < nv; x0 += 32 * PR_MLP) {   // PR_MLP words per image in flight per lane
                        unsigned int w1[PR_MLP], w2[PR_MLP];
#pragma unroll
                        for (int u = 0; u < PR_MLP; ++u) {
                            const int x = x0 + 32 * u;
                            w1[u] = x < nv ? __ldg(q1 + x) : 0u;
                            w2[u] = x < nv ? __ldg(q2 + x) : 0u;
                        }
#pragma unroll
                        for (int u = 0; u < PR_MLP; ++u) {
                            pr_acc(w1[u] & 0xffffu, w2[u] & 0xffffu, ra, rb, saa, sbb, sab);
                            pr_acc(w1[u] >> 16, w2[u] >> 16, ra, rb, saa, sbb, sab);
                        }
                    }
                    if ((n & 1) && lane == 0) pr_acc(__ldg(p1 + n - 1), __ldg(p2 + n - 1), ra, rb, saa, sbb, sab);
                } else if (even_rows && n >= 4) {
                    // exactly one x offset is odd: aligned words on one side, funnel-shifted pairs of
                    // aligned words on the other (element -1 and the following words stay inside the row)
                    // the aligned side is accumulated as "a", the funnel-shifted side as "b"; the
                    // a/b statistics are swapped once per row when image 1 is the shifted side
                    const bool odd1 = cd.o1[0] & 1;
                    const unsigned int* qa = reinterpret_cast<const unsigned int*>(odd1 ? p2 : p1);
                    const unsigned int* qm = reinterpret_cast<const unsigned int*>((odd1 ? p1 : p2) - 1);
                    const int nv = (n >> 1) - 1;  // last pair(s) handled below: qm[x + 1] must not leave the row
                    unsigned int ta = 0, tb = 0;
                    unsigned long long taa = 0, tbb = 0;
                    for (int x0 = lane; x0 < nv; x0 += 32 * PR_MLP) {
                        unsigned int wa[PR_MLP], m0[PR_MLP], m1[PR_MLP];
#pragma unroll
                        for (int u = 0; u < PR_MLP; ++u) {
                            const int x = x0 + 32 * u;
                            wa[u] = x < nv ? __ldg(qa + x) : 0u;
                            m0[u] = x < nv ? __ldg(qm + x) : 0u;
                            m1[u] = x < nv ? __ldg(qm + x + 1) : 0u;
                        }
#pragma unroll
                        for (int u = 0; u < PR_MLP; ++u) {
                            const unsigned int wm = __funnelshift_r(m0[u], m1[u], 16);
                            pr_acc(wa[u] & 0xffffu, wm & 0xffffu, ta, tb, taa, tbb, sab);
                            pr_acc(wa[u] >> 16, wm >> 16, ta, tb, taa, tbb, sab);
                        }
                    }
                    if (odd1) { ra += tb; rb += ta; saa += tbb; sbb += taa; }
                    else { ra += ta; rb += tb; saa += taa; sbb += tbb; }
                    for (int x = 2 * nv + lane; x < n; x += 32) pr_acc(__ldg(p1 + x), __ldg(p2 + x), ra, rb, saa, sbb, sab);
                } else {
#pragma unroll 4
                    for (int x = lane; x < n; x += 32) pr_acc(__ldg(p1 + x), __ldg(p2 + x), ra, rb, saa, sbb, sab);
                }
                sa += ra;
                sb += rb;
            }
            if (!any) continue;  // warp-uniform
            unsigned long long v[5] = {sa, sb, saa, sbb, sab};
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                unsigned long long t = v[k];
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) t += __shfl_down_sync(0xffffffffu, t, off);
                if (lane == 0 && t) atomicAdd(&s_acc[5 * c + k], t);
            }
        }
    }
}


__global__ void __launch_bounds__(NT) k_old(const __grid_constant__ PearsonArgs a, const int* ncand_ptr, unsigned long long* sums) {
    extern __shared__ unsigned long long s_u[];
    const int ncand = *ncand_ptr;
    for (int i = threadIdx.x; i < 5 * ncand; i += blockDim.x) s_u[i] = 0ull;
    __syncthreads();
    pearson_u16(a, ncand, s_u);
    __syncthreads();
    for (int i = threadIdx.x; i < 5 * ncand; i += blockDim.x)
        if (s_u[i]) atomicAdd(sums + i, s_u[i]);
}

// (b) - (d): the slab-staged traversal of k_pearson_u16 (csrc/pcm.cu), with the arithmetic switchable (MODE 0 / 1 / 2
// for (b) / (c) / (d)) and U chunks per lane per round
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity) {
    asm volatile("{\n.reg .pred p;\nWAIT_LOOP:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE;\nbra WAIT_LOOP;\nDONE:\n}\n"
                 ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
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

// (c): 64-bit multiply-accumulates
struct Acc64 {
    unsigned int sa, sb;
    unsigned long long saa, sbb, sab;
};
__device__ __forceinline__ void prs_acc(const unsigned int A[4], const unsigned int B[4], Acc64& s) {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const unsigned int a0 = A[m] & 0xffffu, a1 = A[m] >> 16, b0 = B[m] & 0xffffu, b1 = B[m] >> 16;
        s.sa += a0 + a1;
        s.sb += b0 + b1;
        s.saa += (unsigned long long)a0 * a0;   // IMAD.WIDE.U32 with 64-bit accumulate each
        s.saa += (unsigned long long)a1 * a1;
        s.sbb += (unsigned long long)b0 * b0;
        s.sbb += (unsigned long long)b1 * b1;
        s.sab += (unsigned long long)a0 * b0;
        s.sab += (unsigned long long)a1 * b1;
    }
}

// (d): IDP.2A into uint32 partials p_lo + 256 p_hi, 128 IDPs (32 chunks) per partial between folds
struct PrsAcc {
    unsigned int sa, sb;
    unsigned int aal, aah, bbl, bbh, abl, abh;
};
#define PRS_FOLD_CHUNKS 32
__device__ __forceinline__ void prs_acc(const unsigned int A[4], const unsigned int B[4], PrsAcc& s) {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
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

__device__ __forceinline__ void prs_add(unsigned int sa, unsigned int sb, unsigned long long saa, unsigned long long sbb,
                                        unsigned long long sab, unsigned long long* acc, int lane) {
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
}
__device__ __forceinline__ void prs_flush(Acc64& s, unsigned long long* acc, int lane) {
    prs_add(s.sa, s.sb, s.saa, s.sbb, s.sab, acc, lane);
    s = Acc64{0u, 0u, 0ull, 0ull, 0ull};
}
__device__ __forceinline__ void prs_flush(PrsAcc& s, unsigned long long* acc, int lane) {
    prs_add(s.sa, s.sb, s.aal + ((unsigned long long)s.aah << 8), s.bbl + ((unsigned long long)s.bbh << 8),
            s.abl + ((unsigned long long)s.abh << 8), acc, lane);
    s = PrsAcc{0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
}

// One image-2 row segment of one candidate, owned by a warp.  Chunk k covers image-2 elements g + 8k .. g + 8k + 7
// (g 16-byte aligned); elements lo .. hi - 1 of the chunk sequence belong to the segment.  s1 points at the staged
// image-1 element paired with chunk 0's first element, rounded down to 16 bytes; SH is the rounding (0..7).
// Chunks k >= kvec reach past the end of image 2 and are loaded element by element.  (d) folds every
// PRS_FOLD_CHUNKS / U rounds of segments longer than 32 * PRS_FOLD_CHUNKS chunks (never at the probe's dx = 512).
// TAIL: the row's last round takes up to U + 1 chunks per lane (k_pearson_u16: U = 1, TAIL).
template <int MODE, int U, bool TAIL, int SH, typename ACC>
__device__ __forceinline__ void prs_row(const unsigned short* __restrict__ g, const unsigned short* s1, int lo, int hi,
                                        int nch, int kvec, int lane, ACC& s, unsigned long long* acc) {
    constexpr int UM = U + (TAIL ? 1 : 0);
    constexpr int FOLD_ROUNDS = (PRS_FOLD_CHUNKS - (TAIL ? 1 : 0)) / U;
    for (int kb = 0, r = 1; kb < nch; kb += 32 * U, ++r) {   // warp-uniform rounds
        const bool last = TAIL && nch - kb <= 32 * UM;
        uint4 v[UM];
#pragma unroll
        for (int u = 0; u < UM; ++u) {        // all chunks' loads in flight before any arithmetic
            const int k = (u < U || last) ? kb + lane + 32 * u : nch;
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
        for (int u = 0; u < UM; ++u) {
            const int k = (u < U || last) ? kb + lane + 32 * u : nch;
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
            if (MODE) prs_acc(A, B, s);
            else s.sa ^= A[0] ^ A[1] ^ A[2] ^ A[3] ^ B[0] ^ B[1] ^ B[2] ^ B[3];
        }
        if (last) break;
        if (MODE == 2 && r % FOLD_ROUNDS == 0 && kb + 32 * U < nch) prs_flush(s, acc, lane);
    }
}

// dynamic smem: 2 stage buffers, the candidate list, 5 accumulators per candidate.  UNR: unrolling of the loop over a
// warp's rows (k_pearson_u16: 1, so that the 8 alignment cases of prs_row are inlined once each).
template <int MODE, int U, bool TAIL = false, int UNR = PRS_ROWS / (NT / 32)>
__global__ void __launch_bounds__(NT, 3) k_new(const __grid_constant__ PearsonU16Args a) {
    extern __shared__ __align__(16) unsigned char dyn_sm[];
    const int ncand = *a.ncand;   // written by k_pcm_select (no host round trip between peaks and Pearson)
    if (ncand <= 0) return;
    constexpr int NW = NT / 32, RPW = PRS_ROWS / NW;
    unsigned short* stage = reinterpret_cast<unsigned short*>(dyn_sm);
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
            typename std::conditional<MODE == 1, Acc64, PrsAcc>::type acc = {};
            bool any = false;
#pragma unroll UNR
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
                    case 0: prs_row<MODE, U, TAIL, 0>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 1: prs_row<MODE, U, TAIL, 1>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 2: prs_row<MODE, U, TAIL, 2>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 3: prs_row<MODE, U, TAIL, 3>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 4: prs_row<MODE, U, TAIL, 4>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 5: prs_row<MODE, U, TAIL, 5>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    case 6: prs_row<MODE, U, TAIL, 6>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
                    default: prs_row<MODE, U, TAIL, 7>(g, s1, lo, hi, nch, kvec, lane, acc, s_acc + 5 * c); break;
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

__global__ void k_fill(unsigned short* p, long long n, unsigned int seed) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        unsigned int h = (unsigned int)i * 2654435761u ^ seed;
        h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
        p[i] = (unsigned short)h;
    }
}

__global__ void __launch_bounds__(NT) k_read(const uint4* p, long long n16, unsigned int* out) {
    unsigned int x = 0;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n16; i += (long long)gridDim.x * NT) {
        const uint4 v = ldg_stream16(p + i);
        x ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (x == 0x9e3779b9u) *out = x;
}

// pcm_expand_candidate (csrc/pcm.cu) for equal-size crops
static bool expand(const long long loc[3], const int P[3], const int d[3], int i, long long min_px, PearsonCand* pc, long long* npx_out) {
    bool overlap = true;
    long long npx = 1;
    for (int a = 0; a < 3; ++a) {
        long long s = loc[a];
        if (((i >> a) & 1) == 0) s = s < 0 ? s + P[a] : s - P[a];
        const long long n = d[a];
        if (s >= 0) {
            if (s >= n) { overlap = false; continue; }
            pc->o1[a] = (int)s; pc->o2[a] = 0; pc->sz[a] = (int)(n - s);
        } else {
            if (s <= -n) { overlap = false; continue; }
            pc->o1[a] = 0; pc->o2[a] = (int)-s; pc->sz[a] = (int)(n + s);
        }
        npx *= pc->sz[a];
    }
    pc->pad = 0;
    *npx_out = npx;
    return overlap && npx >= min_px;
}

int main() {
    setvbuf(stdout, nullptr, _IONBF, 0);
    const int D = 512, P = 540;
    const int d[3] = {D, D, D}, Pd[3] = {P, P, P};
    const long long n = (long long)D * D * D;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    unsigned short *i1, *i2;
    CK(cudaMalloc(&i1, n * 2));
    CK(cudaMalloc(&i2, n * 2));
    k_fill<<<1024, 256>>>(i1, n, 0x1234u);
    k_fill<<<1024, 256>>>(i2, n, 0xabcdu);
    CK(cudaDeviceSynchronize());
    // candidate lists
    std::mt19937 rng(7);
    std::vector<PearsonCand> lists[2];
    const long long min_px = (long long)(0.25 * n);
    {
        long long peaks[5][3] = {{3, 537, 2}};
        for (int p = 1; p < 5; ++p) for (int a = 0; a < 3; ++a) peaks[p][a] = rng() % P;
        for (int p = 0; p < 5; ++p)
            for (int i = 0; i < 8; ++i) {
                PearsonCand c; long long npx;
                memset(&c, 0, sizeof(c));
                if (expand(peaks[p], Pd, d, i, min_px, &c, &npx)) lists[0].push_back(c);
            }
        for (size_t k = 0; k < lists[0].size(); ++k) {
            long long loc[3];
            for (int a = 0; a < 3; ++a) { const int s = (int)(rng() % 9) - 4; loc[a] = s < 0 ? s + P : s; }
            PearsonCand c; long long npx;
            memset(&c, 0, sizeof(c));
            for (int i = 0; i < 8; ++i) if (expand(loc, Pd, d, i, min_px, &c, &npx)) break;
            lists[1].push_back(c);
        }
    }
    PearsonCand* dc;
    unsigned long long* dsum;
    int* dcnt;
    unsigned int* dsink;
    CK(cudaMalloc(&dc, sizeof(PearsonCand) * 64));
    CK(cudaMalloc(&dsum, 8 * 5 * 64));
    CK(cudaMalloc(&dcnt, 16));
    CK(cudaMalloc(&dsink, 16));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const int iters = 20;
    printf("device %s, %d SMs, SM clock max %d MHz\n", prop.name, prop.multiProcessorCount, prop.clockRate / 1000);
    {   // (r)
        for (int w = 0; w < 3; ++w) { k_read<<<prop.multiProcessorCount * 8, NT>>>((const uint4*)i1, n / 8, dsink); k_read<<<prop.multiProcessorCount * 8, NT>>>((const uint4*)i2, n / 8, dsink); }
        CK(cudaEventRecord(e0));
        for (int i = 0; i < iters; ++i) { k_read<<<prop.multiProcessorCount * 8, NT>>>((const uint4*)i1, n / 8, dsink); k_read<<<prop.multiProcessorCount * 8, NT>>>((const uint4*)i2, n / 8, dsink); }
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        const double gbs = 4.0 * n * iters / (ms * 1e-3) / 1e9;
        printf("(r) read both volumes, 16 B loads     %7.3f ms  %7.1f GB/s  %.2f of 3.35 TB/s\n", ms / iters, gbs, gbs / 3350.0);
    }
    for (int L = 0; L < 2; ++L) {
        const std::vector<PearsonCand>& cl = lists[L];
        const int nc = (int)cl.size();
        long long px = 0;
        for (auto& c : cl) px += (long long)c.sz[0] * c.sz[1] * c.sz[2];
        const double dram = 2.0 * n + 2.0 * px, alg = 4.0 * px;
        printf("list %d (%s): %d candidates, %.0f M candidate voxels; DRAM model %.2f GB, 4 B/voxel %.2f GB\n", L + 1,
               L ? "all shifts within +-4" : "true peak + 4 seeded noise peaks, wrap candidates", nc, px / 1e6, dram / 1e9, alg / 1e9);
        CK(cudaMemcpy(dc, cl.data(), sizeof(PearsonCand) * nc, cudaMemcpyHostToDevice));
        std::vector<unsigned long long> ref(5 * nc), got(5 * nc);
        typedef void (*KNew)(PearsonU16Args);   // nullptr: (a)
        auto run = [&](const char* name, KNew kn, bool check, int slab_rows) -> int {
            PearsonArgs oa;
            oa.img1 = i1; oa.img2 = i2; oa.dtype = 0; oa.dx = D; oa.dy = D; oa.dz = D; oa.cands = dc;
            PearsonU16Args a;
            a.img1 = i1; a.img2 = i2; a.dx = D; a.dy = D; a.dz = D;
            a.slab_rows = slab_rows;
            a.stage_elems = ((slab_rows * D + 32) + 7) & ~7;
            a.nslabs = (int)(((long long)D * D + slab_rows - 1) / slab_rows);
            a.cands = dc; a.sums = dsum; a.ncand = dcnt; a.counter = dcnt + 1;
            const size_t smem = 2 * 2 * (size_t)a.stage_elems + 80 * nc;
            int ctas = prop.multiProcessorCount * 8;
            if (kn) {
                CK(cudaFuncSetAttribute((const void*)kn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                int occ = 0;
                CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)kn, NT, smem));
                ctas = std::min(a.nslabs, prop.multiProcessorCount * std::max(occ, 1));
            }
            const int cnt[2] = {nc, 0};
            auto launch = [&]() {
                cudaMemsetAsync(dsum, 0, 8 * 5 * nc);
                cudaMemcpyAsync(dcnt, cnt, 8, cudaMemcpyHostToDevice);
                if (!kn) k_old<<<ctas, NT, 8 * 5 * nc>>>(oa, dcnt, dsum);
                else kn<<<ctas, NT, smem>>>(a);
            };
            for (int w = 0; w < 3; ++w) launch();
            CK(cudaEventRecord(e0));
            for (int i = 0; i < iters; ++i) launch();
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaGetLastError());
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            ms /= iters;
            CK(cudaMemcpy(got.data(), dsum, 8 * 5 * nc, cudaMemcpyDeviceToHost));
            const char* chk = "";
            if (!kn) ref = got;
            else if (check) chk = got == ref ? "  sums == (a)" : "  SUMS DIFFER from (a)";
            printf("  %-44s %7.3f ms  DRAM model %7.1f GB/s (%.2f of 3.35 TB/s)  4 B/voxel frac %.2f  CTAs %d%s\n", name, ms,
                   dram / (ms * 1e-3) / 1e9, dram / (ms * 1e-3) / 3.35e12, alg / (ms * 1e-3) / 3.35e12, ctas, chk);
            return 0;
        };
        if (run("(a) previous traversal", nullptr, true, 32)) return 1;
        if (run("(b) slabs of 32 rows, no arithmetic, U=2", k_new<0, 2>, false, 32)) return 1;
        if (run("(c) slabs of 32 rows, 64-bit sums, U=2", k_new<1, 2>, true, 32)) return 1;
        if (run("(c) slabs of 16 rows, 64-bit sums, U=2", k_new<1, 2>, true, 16)) return 1;
        if (run("(c) slabs of 32 rows, 64-bit sums, U=3", k_new<1, 3>, true, 32)) return 1;
        if (run("(c) slabs of 16 rows, 64-bit sums, U=3", k_new<1, 3>, true, 16)) return 1;
        if (run("(d) slabs of 32 rows, IDP sums, U=1", k_new<2, 1>, true, 32)) return 1;
        if (run("(d) slabs of 16 rows, IDP sums, U=1", k_new<2, 1>, true, 16)) return 1;
        if (run("(d) slabs of 32 rows, IDP sums, U=2", k_new<2, 2>, true, 32)) return 1;
        if (run("(d) slabs of 16 rows, IDP sums, U=2", k_new<2, 2>, true, 16)) return 1;
        if (run("(d) slabs of 32 rows, IDP sums, U=3", k_new<2, 3>, true, 32)) return 1;
        if (run("(d) slabs of 16 rows, IDP sums, U=3", k_new<2, 3>, true, 16)) return 1;
        if (run("(e) (d) rows not unrolled, U=2", k_new<2, 2, false, 1>, true, 32)) return 1;
        if (run("(e) (d) rows not unrolled, U=1", k_new<2, 1, false, 1>, true, 32)) return 1;
        if (run("(e) U=1, last round of 2 (as built)", k_new<2, 1, true, 1>, true, 32)) return 1;
        if (run("(e) U=2, last round of 3", k_new<2, 2, true, 1>, true, 32)) return 1;
    }
    return 0;
}
