// Shared-memory mixed-radix Stockham FFT building blocks (sm_90a, no cuFFT).
//
// A "tile" is N complex elements x L lines held in shared memory with the LINE index
// innermost: element e of line l lives at buf[e * lstride + l].  Every butterfly therefore
// touches, for a half-warp, 16 consecutive float2 (128 B) -> bank-conflict free for any
// radix/stride, and for the strided (y / z) passes the tile is a verbatim copy of the global
// layout (x-fastest spectrum rows), so loads/stores are straight 16 B-vector copies.
//
// Radix-R butterflies (R in {2,3,4,5,6,8,9,10,12,15,16}) are fully unrolled in registers;
// composite radices are built at compile time by a Cooley-Tukey split with constexpr
// twiddles, so a 540-point transform needs only 3 shared-memory round trips (9 x 10 x 6).
#pragma once
#include <cuda_runtime.h>
#include <utility>

#define BS_FFT_MAX_STAGES 12

struct FftPlan {
    int n;
    int nst;
    int radix[BS_FFT_MAX_STAGES];
};

// ------------------------------------------------------------------ compile-time trigonometry
namespace cx {
constexpr double pi = 3.141592653589793238462643383279502884;
constexpr double sin_series(double x) {  // |x| <= pi/2
    double x2 = x * x, term = x, sum = x;
    for (int i = 1; i < 16; ++i) {
        term *= -x2 / ((2.0 * i) * (2.0 * i + 1.0));
        sum += term;
    }
    return sum;
}
constexpr double cos_series(double x) {
    double x2 = x * x, term = 1.0, sum = 1.0;
    for (int i = 1; i < 16; ++i) {
        term *= -x2 / ((2.0 * i - 1.0) * (2.0 * i));
        sum += term;
    }
    return sum;
}
// cos / sin of 2*pi*t/r, exact at multiples of a quarter turn
constexpr double cos2pi(int t, int r) {
    t %= r;
    if (t < 0) t += r;
    if ((4 * t) % r == 0) {
        int q = (4 * t) / r;
        return q == 0 ? 1.0 : q == 2 ? -1.0 : 0.0;
    }
    double a = 2.0 * pi * t / r;      // (0, 2pi)
    if (a > pi) a = 2.0 * pi - a;     // cos even around pi
    if (a > pi / 2) return -cos_series(pi - a);
    return cos_series(a);
}
constexpr double sin2pi(int t, int r) {
    t %= r;
    if (t < 0) t += r;
    if ((4 * t) % r == 0) {
        int q = (4 * t) / r;
        return q == 1 ? 1.0 : q == 3 ? -1.0 : 0.0;
    }
    double a = 2.0 * pi * t / r;
    double sgn = 1.0;
    if (a > pi) { a = 2.0 * pi - a; sgn = -1.0; }
    if (a > pi / 2) a = pi - a;
    return sgn * sin_series(a);
}
constexpr int pick_factor(int r) {
    // split composite radices into (A, r/A): prefer 4 for 8/12/16, else smallest prime
    if (r % 4 == 0 && r > 4) return 4;
    if (r % 2 == 0) return 2;
    if (r % 3 == 0) return 3;
    if (r % 5 == 0) return 5;
    return r;
}
}  // namespace cx

// ---------------------------------------------------------------------------- complex arithmetic
// Element-wise float2 primitives.  sm_90 has no packed FP32 pair instructions, so each half is one scalar
// FADD / FMUL / FFMA; the multiplications by +-1 in the helpers below fold into operand negations.
__device__ __forceinline__ float2 p_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 p_sub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 p_mul(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 p_fma(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 p_swap(float2 a) { return make_float2(a.y, a.x); }
__device__ __forceinline__ float2 p_bc(float s) { return make_float2(s, s); }

// a * b = a.x * b + a.y * (i b)
__device__ __forceinline__ float2 cmulf(float2 a, float2 b) {
    return p_fma(p_bc(a.y), p_mul(p_swap(b), make_float2(-1.f, 1.f)), p_mul(p_bc(a.x), b));
}
__device__ __forceinline__ float2 caddf(float2 a, float2 b) { return p_add(a, b); }
__device__ __forceinline__ float2 csubf(float2 a, float2 b) { return p_sub(a, b); }
// a + s * (-i b)  and  a + s * (i b)   (s real)
__device__ __forceinline__ float2 cadd_mi(float2 a, float2 b, float s = 1.f) { return p_fma(p_swap(b), make_float2(s, -s), a); }
__device__ __forceinline__ float2 cadd_pi(float2 a, float2 b, float s = 1.f) { return p_fma(p_swap(b), make_float2(-s, s), a); }
// a + s * b, s * a   (s real)
__device__ __forceinline__ float2 caxpy(float s, float2 b, float2 a) { return p_fma(p_bc(s), b, a); }
__device__ __forceinline__ float2 cscale(float s, float2 a) { return p_mul(p_bc(s), a); }
// multiply by -i / +i
__device__ __forceinline__ float2 mul_mi(float2 a) { return p_mul(p_swap(a), make_float2(1.f, -1.f)); }
__device__ __forceinline__ float2 mul_pi(float2 a) { return p_mul(p_swap(a), make_float2(-1.f, 1.f)); }

// v * W_R^T (forward twiddle e^{-2 pi i T / R}) with T, R compile-time
template <int T, int R>
__device__ __forceinline__ float2 mul_w(float2 v) {
    constexpr int t = ((T % R) + R) % R;
    if constexpr (t == 0) {
        return v;
    } else if constexpr ((4 * t) % R == 0) {
        constexpr int q = (4 * t) / R;
        if constexpr (q == 1) return mul_mi(v);
        else if constexpr (q == 2) return p_mul(v, make_float2(-1.f, -1.f));
        else return mul_pi(v);
    } else {
        constexpr float c = (float)cx::cos2pi(t, R);
        constexpr float s = (float)(-cx::sin2pi(t, R));
        return p_fma(p_swap(v), make_float2(-s, s), cscale(c, v));   // (v.x c - v.y s, v.y c + v.x s)
    }
}

template <int R>
__device__ __forceinline__ void dft(float2 (&x)[R]);

template <int R, int A, int... I>
__device__ __forceinline__ void apply_inner_twiddles(float2 (&t)[R], std::integer_sequence<int, I...>) {
    // t index I = n2 * A + k1  ->  multiply by W_R^(n2 * k1)
    ((t[I] = mul_w<(I / A) * (I % A), R>(t[I])), ...);
}

template <int R>
__device__ __forceinline__ void dft(float2 (&x)[R]) {
    if constexpr (R == 1) {
    } else if constexpr (R == 2) {
        float2 a = x[0], b = x[1];
        x[0] = caddf(a, b);
        x[1] = csubf(a, b);
    } else if constexpr (R == 3) {
        constexpr float s = (float)cx::sin2pi(1, 3);
        const float2 t1 = caddf(x[1], x[2]);
        const float2 t2 = caxpy(-0.5f, t1, x[0]);
        const float2 d = csubf(x[1], x[2]);
        x[0] = caddf(x[0], t1);
        x[1] = cadd_mi(t2, d, s);
        x[2] = cadd_pi(t2, d, s);
    } else if constexpr (R == 4) {
        const float2 a = caddf(x[0], x[2]), b = csubf(x[0], x[2]);
        const float2 c = caddf(x[1], x[3]), d = csubf(x[1], x[3]);
        x[0] = caddf(a, c);
        x[2] = csubf(a, c);
        x[1] = cadd_mi(b, d);
        x[3] = cadd_pi(b, d);
    } else if constexpr (R == 5) {
        constexpr float c1 = (float)cx::cos2pi(1, 5), c2 = (float)cx::cos2pi(2, 5);
        constexpr float s1 = (float)cx::sin2pi(1, 5), s2 = (float)cx::sin2pi(2, 5);
        const float2 t1 = caddf(x[1], x[4]), t2 = caddf(x[2], x[3]);
        const float2 t3 = csubf(x[1], x[4]), t4 = csubf(x[2], x[3]);
        const float2 a1 = caxpy(c2, t2, caxpy(c1, t1, x[0]));
        const float2 a2 = caxpy(c1, t2, caxpy(c2, t1, x[0]));
        const float2 b1 = caxpy(s2, t4, cscale(s1, t3));
        const float2 b2 = caxpy(-s1, t4, cscale(s2, t3));
        x[0] = caddf(x[0], caddf(t1, t2));
        x[1] = cadd_mi(a1, b1);
        x[4] = cadd_pi(a1, b1);
        x[2] = cadd_mi(a2, b2);
        x[3] = cadd_pi(a2, b2);
    } else {
        // Cooley-Tukey in registers: n = B*n1 + n2, k = k1 + A*k2
        constexpr int A = cx::pick_factor(R);
        constexpr int B = R / A;
        static_assert(A > 1 && A < R, "unsupported radix");
        float2 t[R];
#pragma unroll
        for (int n2 = 0; n2 < B; ++n2) {
            float2 s[A];
#pragma unroll
            for (int n1 = 0; n1 < A; ++n1) s[n1] = x[B * n1 + n2];
            dft<A>(s);
#pragma unroll
            for (int k1 = 0; k1 < A; ++k1) t[n2 * A + k1] = s[k1];
        }
        apply_inner_twiddles<R, A>(t, std::make_integer_sequence<int, R>{});
#pragma unroll
        for (int k1 = 0; k1 < A; ++k1) {
            float2 s[B];
#pragma unroll
            for (int n2 = 0; n2 < B; ++n2) s[n2] = t[n2 * A + k1];
            dft<B>(s);
#pragma unroll
            for (int k2 = 0; k2 < B; ++k2) x[k1 + A * k2] = s[k2];
        }
    }
}

// One Stockham stage of radix R over a tile: in -> out (both shared memory, element offsets
// relative to `sm`).  tw[k * twmul] = e^{-2 pi i k / N}.  lshift = log2(lines).
template <int R>
__device__ __forceinline__ void fft_stage(const float2* __restrict__ in, float2* __restrict__ out,
                                          const float2* __restrict__ tw, int N, int Ls, int lshift,
                                          int lstride, int twmul) {
    const int m = N / R;
    const int nitems = m << lshift;
    const int lmask = (1 << lshift) - 1;
    const int twstep = (N / (Ls * R)) * twmul;
    for (int item = threadIdx.x; item < nitems; item += blockDim.x) {
        const int j = item >> lshift;
        const int l = item & lmask;
        const int k = (Ls == 1) ? 0 : (j % Ls);
        float2 x[R];
        const float2* p = in + j * lstride + l;
#pragma unroll
        for (int q = 0; q < R; ++q) x[q] = p[q * m * lstride];
        if (Ls > 1) {
            const int ts = k * twstep;
#pragma unroll
            for (int q = 1; q < R; ++q) x[q] = cmulf(x[q], tw[q * ts]);
        }
        dft<R>(x);
        float2* o = out + ((j - k) * R + k) * lstride + l;
#pragma unroll
        for (int q = 0; q < R; ++q) o[q * Ls * lstride] = x[q];
    }
}

// Forward FFT of all lines of a tile.  Ping-pongs between `a` and `b`; returns the buffer
// holding the result (a when the stage count is even).  Ends with __syncthreads().
__device__ __forceinline__ float2* fft_tile(float2* a, float2* b, const float2* tw, const FftPlan& plan,
                                         int lshift, int lstride, int twmul) {
    int Ls = 1;
    const int N = plan.n;
    for (int s = 0; s < plan.nst; ++s) {
        const int r = plan.radix[s];
        switch (r) {
            case 2: fft_stage<2>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 3: fft_stage<3>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 4: fft_stage<4>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 5: fft_stage<5>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 6: fft_stage<6>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 8: fft_stage<8>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 9: fft_stage<9>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 10: fft_stage<10>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 12: fft_stage<12>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 15: fft_stage<15>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            case 16: fft_stage<16>(a, b, tw, N, Ls, lshift, lstride, twmul); break;
            default: break;
        }
        __syncthreads();
        Ls *= r;
        float2* t = a; a = b; b = t;
    }
    return a;
}


// ------------------------------------------------------------------------------------------
// Compile-time plans.  For the transform lengths that dominate real workloads (the padded
// sizes of 512^3 / 256^3 overlaps) every stride, trip count and twiddle step is a constant:
// shared-memory accesses use immediate offsets, `j % Ls` becomes a multiply-shift and the
// item loops are fully unrolled.  Other lengths run the generic runtime-planned path above.
template <int N, int R, int LS, int LSHIFT, int LSTRIDE, int TWMUL, int NT>
__device__ __forceinline__ void fft_stage_s(const float2* __restrict__ in, float2* __restrict__ out,
                                            const float2* __restrict__ tw) {
    constexpr int m = N / R;
    constexpr int nitems = m << LSHIFT;
    constexpr int lmask = (1 << LSHIFT) - 1;
    constexpr int twstep = (N / (LS * R)) * TWMUL;
    constexpr int iters = (nitems + NT - 1) / NT;
#pragma unroll
    for (int it = 0; it < iters; ++it) {
        const int item = threadIdx.x + it * NT;
        if ((nitems % NT) != 0 && it == iters - 1 && item >= nitems) break;
        const int j = item >> LSHIFT;
        const int l = item & lmask;
        const int k = (LS == 1) ? 0 : (j % LS);
        float2 x[R];
        const float2* p = in + j * LSTRIDE + l;
#pragma unroll
        for (int q = 0; q < R; ++q) x[q] = p[q * m * LSTRIDE];
        if (LS > 1) {
            const float2* t = tw + k * twstep;
#pragma unroll
            for (int q = 1; q < R; ++q) x[q] = cmulf(x[q], t[(q - 1) * k * twstep]);
        }
        dft<R>(x);
        float2* o = out + ((j - k) * R + k) * LSTRIDE + l;
#pragma unroll
        for (int q = 0; q < R; ++q) o[q * LS * LSTRIDE] = x[q];
    }
}

template <int N, int LS, int LSHIFT, int LSTRIDE, int TWMUL, int NT, int R, int... Rest>
__device__ __forceinline__ float2* fft_tile_s(float2* a, float2* b, const float2* tw) {
    fft_stage_s<N, R, LS, LSHIFT, LSTRIDE, TWMUL, NT>(a, b, tw);
    __syncthreads();
    if constexpr (sizeof...(Rest) == 0) return b;
    else return fft_tile_s<N, LS * R, LSHIFT, LSTRIDE, TWMUL, NT, Rest...>(b, a, tw);
}

// Policy types the kernels are templated on.
struct FftGeneric {
    static constexpr bool kStatic = false;
    static constexpr int N = 0, LSHIFT = 0;
    static __device__ __forceinline__ float2* run(float2* a, float2* b, const float2* tw, const FftPlan& plan,
                                                  int lshift, int lstride, int twmul) {
        return fft_tile(a, b, tw, plan, lshift, lstride, twmul);
    }
};

template <int N_, int LSHIFT_, int LSTRIDE_, int TWMUL_, int NT_, int... Rs>
struct FftStatic {
    static constexpr bool kStatic = true;
    static constexpr int N = N_, LSHIFT = LSHIFT_;
    static __device__ __forceinline__ float2* run(float2* a, float2* b, const float2* tw, const FftPlan&, int, int,
                                                  int) {
        return fft_tile_s<N_, 1, LSHIFT_, LSTRIDE_, TWMUL_, NT_, Rs...>(a, b, tw);
    }
};


// ------------------------------------------------------------------------------------------
// Register-resident two-stage transform of a column tile: TC columns of N = RA * RB points, element n of column
// c at g[n * estride + c].  Cooley-Tukey with n = RB n1 + n2 and k = k1 + RA k2:
//   stage 1  item (n2, c) holds x[RB n1 + n2], n1 < RA, in registers: dft<RA>, times W_N^(n2 k1), and ONE write
//            per element to the exchange buffer X[(k1 RB + n2) TC + c]
//   (one __syncthreads)
//   stage 2  item (k1, c) reads X[(k1 RB + n2) TC + c], n2 < RB, once: dft<RB> leaves X[k1 + RA k2] in register k2
// Items of a stage are i = threadIdx.x + u NT, with (n2 | k1) = i / TC and c = i % TC, so a warp touches 32 / TC
// consecutive row segments of TC columns: the global accesses are whole segments, the exchange writes are
// contiguous, and the exchange reads of one n2 are 32 / TC segments of TC float2 (the 2-wavefront minimum).
// Two-element twiddles n2 k1 < N index the table tw[e] = e^{-2 pi i e / N} (shared memory) directly.
//
// Stage 2 of RegFft2<RA, RB> leaves item (k1, c) holding x[k1 + RA k2] for k2 < RB, which is exactly the stage-1
// item (n2' = k1, c) of RegFft2<RB, RA> (input n = RA n1' + n2', n1' = k2): a second transform of the result
// starts on the registers the threads already hold, with no exchange in between.
template <int RA, int RB, int TC, int NT>
struct RegFft2 {
    static constexpr int N = RA * RB;
    static constexpr int I1 = RB * TC, IT1 = (I1 + NT - 1) / NT;   // stage-1 items, per thread
    static constexpr int I2 = RA * TC, IT2 = (I2 + NT - 1) / NT;   // stage-2 items, per thread
    static constexpr int XSIZE = N * TC;                           // exchange buffer, float2
    typedef float2 In[IT1][RA];

    static __device__ __forceinline__ bool live1(int u) { return I1 % NT == 0 || (int)threadIdx.x + u * NT < I1; }
    static __device__ __forceinline__ bool live2(int u) { return I2 % NT == 0 || (int)threadIdx.x + u * NT < I2; }

    static __device__ __forceinline__ void load(In& v, const float2* __restrict__ g, long long estride) {
#pragma unroll
        for (int u = 0; u < IT1; ++u) {
            if (!live1(u)) continue;
            const int i = threadIdx.x + u * NT;
            const float2* p = g + (long long)(i / TC) * estride + (i % TC);
#pragma unroll
            for (int n1 = 0; n1 < RA; ++n1) v[u][n1] = __ldcg(p + (long long)(RB * n1) * estride);
        }
    }
    // the same items from a tile staged in shared memory as X[n TC + c].  Item (n2, c) reads the RA slots that its
    // stage 1 writes (n = RB n1 + n2 and k1 RB + n2), so stage1(v, X, tw) may follow without a barrier.
    static __device__ __forceinline__ void load_shared(In& v, const float2* __restrict__ X) {
#pragma unroll
        for (int u = 0; u < IT1; ++u) {
            if (!live1(u)) continue;
            const float2* p = X + threadIdx.x + u * NT;
#pragma unroll
            for (int n1 = 0; n1 < RA; ++n1) v[u][n1] = p[RB * n1 * TC];
        }
    }
    static __device__ __forceinline__ void stage1(In& v, float2* __restrict__ X, const float2* __restrict__ tw) {
#pragma unroll
        for (int u = 0; u < IT1; ++u) {
            if (!live1(u)) continue;
            const int i = threadIdx.x + u * NT;
            const int n2 = i / TC, c = i % TC;
            dft<RA>(v[u]);
            X[n2 * TC + c] = v[u][0];
#pragma unroll
            for (int k1 = 1; k1 < RA; ++k1) X[(k1 * RB + n2) * TC + c] = cmulf(v[u][k1], tw[n2 * k1]);
        }
    }
    // stage 2, one item at a time (its RB outputs are live only until emit returns):
    // emit(w, u, k1, c) receives w[k2] = X[k1 + RA k2] of column c
    template <class Emit>
    static __device__ __forceinline__ void stage2(const float2* __restrict__ X, Emit&& emit) {
#pragma unroll
        for (int u = 0; u < IT2; ++u) {
            if (!live2(u)) continue;
            const int i = threadIdx.x + u * NT;
            const int k1 = i / TC, c = i % TC;
            const float2* p = X + k1 * RB * TC + c;
            float2 w[RB];
#pragma unroll
            for (int n2 = 0; n2 < RB; ++n2) w[n2] = p[n2 * TC];
            dft<RB>(w);
            emit(w, u, k1, c);
        }
    }
    static __device__ __forceinline__ void store(const float2 (&w)[RB], float2* __restrict__ g, long long estride, int k1,
                                                 int c) {
        float2* p = g + (long long)k1 * estride + c;
#pragma unroll
        for (int k2 = 0; k2 < RB; ++k2) __stcg(p + (long long)(RA * k2) * estride, w[k2]);
    }
    // the item's own exchange slots: X[(k1 RB + k2) TC + c] (write-back of a stage-2 result for the same thread)
    static __device__ __forceinline__ float2* slot(float2* X, int k1, int c) { return X + k1 * RB * TC + c; }
};


// ------------------------------------------------------------------------------------------
// Warp-private line FFT:ONE warp transforms ONE contiguous line (buf[e]) with only
// __syncwarp() between stages, so the x passes need no block-wide barriers at all and the 8
// warps of a CTA drift freely (one warp's loads overlap another's butterflies).
template <int R>
__device__ __forceinline__ void fft_stage_wg(const float2* __restrict__ in, float2* __restrict__ out,
                                             const float2* __restrict__ tw, int N, int Ls, int twmul, int lane) {
    const int m = N / R;
    const int twstep = (N / (Ls * R)) * twmul;
    for (int j = lane; j < m; j += 32) {
        const int k = (Ls == 1) ? 0 : (j % Ls);
        float2 x[R];
#pragma unroll
        for (int q = 0; q < R; ++q) x[q] = in[j + q * m];
        if (Ls > 1) {
            const int ts = k * twstep;
#pragma unroll
            for (int q = 1; q < R; ++q) x[q] = cmulf(x[q], tw[q * ts]);
        }
        dft<R>(x);
        float2* o = out + (j - k) * R + k;
#pragma unroll
        for (int q = 0; q < R; ++q) o[q * Ls] = x[q];
    }
    __syncwarp();
}

__device__ __forceinline__ float2* fft_line_wg(float2* a, float2* b, const float2* tw, const FftPlan& plan, int twmul,
                                               int lane) {
    int Ls = 1;
    const int N = plan.n;
    for (int s = 0; s < plan.nst; ++s) {
        const int r = plan.radix[s];
        switch (r) {
            case 2: fft_stage_wg<2>(a, b, tw, N, Ls, twmul, lane); break;
            case 3: fft_stage_wg<3>(a, b, tw, N, Ls, twmul, lane); break;
            case 4: fft_stage_wg<4>(a, b, tw, N, Ls, twmul, lane); break;
            case 5: fft_stage_wg<5>(a, b, tw, N, Ls, twmul, lane); break;
            case 6: fft_stage_wg<6>(a, b, tw, N, Ls, twmul, lane); break;
            case 8: fft_stage_wg<8>(a, b, tw, N, Ls, twmul, lane); break;
            case 9: fft_stage_wg<9>(a, b, tw, N, Ls, twmul, lane); break;
            case 10: fft_stage_wg<10>(a, b, tw, N, Ls, twmul, lane); break;
            case 12: fft_stage_wg<12>(a, b, tw, N, Ls, twmul, lane); break;
            case 15: fft_stage_wg<15>(a, b, tw, N, Ls, twmul, lane); break;
            case 16: fft_stage_wg<16>(a, b, tw, N, Ls, twmul, lane); break;
            default: break;
        }
        Ls *= r;
        float2* t = a; a = b; b = t;
    }
    return a;
}

// Per-lane twiddles of the static warp-private plan, kept in REGISTERS for the whole kernel: a lane's items of a
// stage are j = lane + 32 it, so its twiddles W^(q (j % LS) step) never change from line to line.  The x passes are
// shared-memory-bandwidth bound, and the stride-(q k step) table reads are bank conflicts; this removes every
// twiddle LDS from the steady state.
template <int N, int R, int LS>
struct WStageTw {
    static constexpr int m = N / R;
    static constexpr int iters = (m + 31) / 32;
    float2 w[LS > 1 ? iters : 1][LS > 1 ? R - 1 : 1];
    __device__ __forceinline__ float2 get(int it, int q, int) const { return w[it][q - 1]; }
    template <int TWMUL>
    __device__ __forceinline__ void init(const float2* __restrict__ tw, int lane) {
        if constexpr (LS > 1) {
            constexpr int twstep = (N / (LS * R)) * TWMUL;
#pragma unroll
            for (int it = 0; it < iters; ++it) {
                const int j = min(lane + 32 * it, m - 1);
                const int ts = (j % LS) * twstep;
#pragma unroll
                for (int q = 1; q < R; ++q) w[it][q - 1] = tw[q * ts];
            }
        }
    }
};

template <int N, int LS, int TWMUL, int R, int... Rest>
struct WLineTw {
    WStageTw<N, R, LS> head;
    WLineTw<N, LS * R, TWMUL, Rest...> tail;
    __device__ __forceinline__ void init(const float2* __restrict__ tw, int lane) {
        head.template init<TWMUL>(tw, lane);
        tail.init(tw, lane);
    }
};
template <int N, int LS, int TWMUL, int R>
struct WLineTw<N, LS, TWMUL, R> {
    WStageTw<N, R, LS> head;
    __device__ __forceinline__ void init(const float2* __restrict__ tw, int lane) { head.template init<TWMUL>(tw, lane); }
};

// The alternative for kernels that cannot spare the registers (the r2c pass needs 4 CTAs per SM to hide its row
// loads): compact per-stage tables in shared memory, tab[(q - 1) * LS + k] -- consecutive lanes (consecutive k)
// read consecutive entries, so the reads are conflict-free (the stride-(q k step) reads of the full table were not).
template <int N, int R, int LS, int OFF>
struct WStageTwS {
    const float2* tab;
    __device__ __forceinline__ float2 get(int, int q, int k) const { return tab[OFF + (q - 1) * LS + k]; }
};
template <int N, int LS, int TWMUL, int OFF, int R, int... Rest>
struct WLineTwS {
    static constexpr int cnt = LS > 1 ? (R - 1) * LS : 0;
    WStageTwS<N, R, LS, OFF> head;
    WLineTwS<N, LS * R, TWMUL, OFF + cnt, Rest...> tail;
    static constexpr int total = cnt + WLineTwS<N, LS * R, TWMUL, OFF + cnt, Rest...>::total;
    __device__ __forceinline__ void init(const float2* tab, int) { head.tab = tab; tail.init(tab, 0); }
    // block-cooperative: fill dst[OFF ...] from the full table twg[i] = e^{-2 pi i i / (N TWMUL)}
    static __device__ __forceinline__ void build(float2* dst, const float2* __restrict__ twg, int tid, int nt) {
        if constexpr (LS > 1) {
            constexpr int twstep = (N / (LS * R)) * TWMUL;
            for (int i = tid; i < cnt; i += nt) dst[OFF + i] = twg[(i / LS + 1) * (i % LS) * twstep];
        }
        WLineTwS<N, LS * R, TWMUL, OFF + cnt, Rest...>::build(dst, twg, tid, nt);
    }
};
template <int N, int LS, int TWMUL, int OFF, int R>
struct WLineTwS<N, LS, TWMUL, OFF, R> {
    static constexpr int cnt = LS > 1 ? (R - 1) * LS : 0;
    static constexpr int total = cnt;
    WStageTwS<N, R, LS, OFF> head;
    __device__ __forceinline__ void init(const float2* tab, int) { head.tab = tab; }
    static __device__ __forceinline__ void build(float2* dst, const float2* __restrict__ twg, int tid, int nt) {
        if constexpr (LS > 1) {
            constexpr int twstep = (N / (LS * R)) * TWMUL;
            for (int i = tid; i < cnt; i += nt) dst[OFF + i] = twg[(i / LS + 1) * (i % LS) * twstep];
        }
    }
};

template <int N, int R, int LS, class ST>
__device__ __forceinline__ void fft_stage_ws(const float2* __restrict__ in, float2* __restrict__ out, const ST& st, int lane) {
    constexpr int m = N / R;
    constexpr int iters = (m + 31) / 32;
#pragma unroll
    for (int it = 0; it < iters; ++it) {
        const int j = lane + 32 * it;
        if ((m % 32) != 0 && it == iters - 1 && j >= m) break;
        const int k = (LS == 1) ? 0 : (j % LS);
        float2 x[R];
#pragma unroll
        for (int q = 0; q < R; ++q) x[q] = in[j + q * m];
        if (LS > 1) {
#pragma unroll
            for (int q = 1; q < R; ++q) x[q] = cmulf(x[q], st.get(it, q, k));
        }
        dft<R>(x);
        float2* o = out + (j - k) * R + k;
#pragma unroll
        for (int q = 0; q < R; ++q) o[q * LS] = x[q];
    }
    __syncwarp();
}

template <int N, int LS, int TWMUL, int R, int... Rest, class LT>
__device__ __forceinline__ float2* fft_line_ws(float2* a, float2* b, const LT& tw, int lane) {
    fft_stage_ws<N, R, LS>(a, b, tw.head, lane);
    if constexpr (sizeof...(Rest) == 0) return b;
    else return fft_line_ws<N, LS * R, TWMUL, Rest...>(b, a, tw.tail, lane);
}

struct WNoTw {
    static constexpr int total = 0;
    __device__ __forceinline__ void init(const float2*, int) {}
};

struct FftWGeneric {
    static constexpr bool kStatic = false;
    static constexpr bool kSmemTw = false;
    static constexpr int N = 0;
    typedef WNoTw Tw;            // twiddles stay in the shared table
    static __device__ __forceinline__ float2* run(float2* a, float2* b, const float2* tw, const Tw&, const FftPlan& plan,
                                                  int twmul, int lane) {
        return fft_line_wg(a, b, tw, plan, twmul, lane);
    }
};

template <int N_, int TWMUL_, int... Rs>
struct FftWStatic {
    static constexpr bool kStatic = true;
    static constexpr bool kSmemTw = false;
    static constexpr int N = N_;
    typedef WLineTw<N_, 1, TWMUL_, Rs...> Tw;   // per-lane register twiddles, Tw::init once per kernel
    static __device__ __forceinline__ float2* run(float2* a, float2* b, const float2*, const Tw& twr, const FftPlan&, int,
                                                  int lane) {
        return fft_line_ws<N_, 1, TWMUL_, Rs...>(a, b, twr, lane);
    }
};

// same plan, twiddles in compact conflict-free shared-memory tables (Tw::build once per CTA, Tw::total entries)
template <int N_, int TWMUL_, int... Rs>
struct FftWStaticS {
    static constexpr bool kStatic = true;
    static constexpr bool kSmemTw = true;
    static constexpr int N = N_;
    typedef WLineTwS<N_, 1, TWMUL_, 0, Rs...> Tw;
    static __device__ __forceinline__ float2* run(float2* a, float2* b, const float2*, const Tw& twr, const FftPlan&, int,
                                                  int lane) {
        return fft_line_ws<N_, 1, TWMUL_, Rs...>(a, b, twr, lane);
    }
};
