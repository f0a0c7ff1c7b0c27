// match-interestpoints: the two quadratic steps of PRECISE_TRANSLATION (RGLDM) descriptor matching
// (J/SparkGeometricDescriptorMatching.java:594-605), both in FP64 so that neighbour and match indices are exact.
//
// k_knn: brute-force k nearest OTHER points of one set.  One thread per point; the set streams through shared memory
//   in tiles and every thread keeps its top-k (squared distance, index) sorted by insertion in registers.  It then
//   writes the point's descriptor record {p, q_1 - p, ..., q_k - p} (k ascending by (distance, index)).
// k_desc_match: one thread per A descriptor (held in registers); the B records stream through shared memory in
//   double-buffered tiles pulled in by 1-D bulk async copies (TMA) completing on an mbarrier, as the z cross-power
//   pass of the phase correlation does.  Per (a, b) the k^2 squared distances |u_i - v_j|^2 are computed once and the
//   C(k,n)^2 subset sums are taken from them.  Blocks split B when N_A alone cannot fill the GPU; k_desc_merge folds the
//   per-split (best, second, index) triples in split (= ascending b) order.
//
// Every distance is ((dx*dx + dy*dy) + dz*dz) and every subset sum is accumulated left to right, without FMA
// contraction, so the results are bitwise those of the float64 oracle that spells the same operations.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "bs_internal.cuh"

namespace {

constexpr int KNN_THREADS = 128;
constexpr int KNN_TILE = 256;            // points per shared-memory tile (6 KB)
constexpr int DM_THREADS = 128;
constexpr int DM_TILE = 64;              // B records per bulk copy

// descriptor record: position (3) + k relative vectors (3k), padded to an even count of doubles (16-byte multiple)
__host__ __device__ constexpr int rec_len(int k) { return ((3 + 3 * k) + 1) & ~1; }

__device__ __forceinline__ double sq3(double dx, double dy, double dz) {
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
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
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned int bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// the C(K, N) neighbour subsets in lexicographic order of rank, each ascending
template <int N, int K>
struct Combos {
    static constexpr int count() {
        int c = 1;
        for (int i = 0; i < N; ++i) c = c * (K - i) / (i + 1);
        return c;
    }
    static constexpr int NC = count();
    int c[NC][N];
    constexpr Combos() : c() {
        int cur[N] = {};
        for (int i = 0; i < N; ++i) cur[i] = i;
        for (int s = 0; s < NC; ++s) {
            for (int i = 0; i < N; ++i) c[s][i] = cur[i];
            int i = N - 1;
            while (i >= 0 && cur[i] == K - N + i) --i;
            if (i < 0) break;
            ++cur[i];
            for (int j = i + 1; j < N; ++j) cur[j] = cur[j - 1] + 1;
        }
    }
};

template <int K>
__global__ void __launch_bounds__(KNN_THREADS) k_knn(const double* __restrict__ xyz, int n, double* __restrict__ rec,
                                                    int* __restrict__ nidx, double* __restrict__ nd2) {
    __shared__ double s_p[KNN_TILE * 3];
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    const bool valid = i < n;
    double px = 0.0, py = 0.0, pz = 0.0;
    if (valid) { px = xyz[3 * i]; py = xyz[3 * i + 1]; pz = xyz[3 * i + 2]; }
    double bd[K];
    int bi[K];
#pragma unroll
    for (int q = 0; q < K; ++q) { bd[q] = INFINITY; bi[q] = -1; }
    for (int base = 0; base < n; base += KNN_TILE) {
        const int m = min(KNN_TILE, n - base);
        __syncthreads();
        for (int t = threadIdx.x; t < m * 3; t += KNN_THREADS) s_p[t] = xyz[(size_t)base * 3 + t];
        __syncthreads();
        if (!valid) continue;
        for (int j = 0; j < m; ++j) {
            const double d = sq3(s_p[3 * j] - px, s_p[3 * j + 1] - py, s_p[3 * j + 2] - pz);
            // j ascends, so a candidate equal to the current k-th has the larger index and stays out
            if (d < bd[K - 1] && base + j != i) {
                bd[K - 1] = d;
                bi[K - 1] = base + j;
#pragma unroll
                for (int q = K - 1; q > 0; --q)
                    if (bd[q] < bd[q - 1]) {
                        const double td = bd[q]; bd[q] = bd[q - 1]; bd[q - 1] = td;
                        const int ti = bi[q]; bi[q] = bi[q - 1]; bi[q - 1] = ti;
                    }
            }
        }
    }
    if (!valid) return;
    constexpr int R = rec_len(K);
    double* r = rec + (size_t)i * R;
    r[0] = px; r[1] = py; r[2] = pz;
#pragma unroll
    for (int q = 0; q < K; ++q) {
        const int j = bi[q];
        r[3 + 3 * q] = xyz[3 * j] - px;
        r[4 + 3 * q] = xyz[3 * j + 1] - py;
        r[5 + 3 * q] = xyz[3 * j + 2] - pz;
        nidx[(size_t)i * K + q] = j;
        nd2[(size_t)i * K + q] = bd[q];
    }
    if (R > 3 + 3 * K) r[R - 1] = 0.0;
}

struct MatchArgs {
    const double* a_rec;
    const double* b_rec;      // padded to a whole number of DM_TILE records
    int na, nb;
    int tiles_per_split;      // B tiles each blockIdx.y scans
    int use_radius;
    double r2;
    double* p_best;           // [split][na]
    double* p_second;
    int* p_idx;
};

template <int N, int K>
__global__ void __launch_bounds__(DM_THREADS) k_desc_match(const __grid_constant__ MatchArgs g) {
    constexpr int R = rec_len(K);
    constexpr Combos<N, K> CB{};
    constexpr int NC = Combos<N, K>::NC;
    __shared__ __align__(128) double s_b[2][DM_TILE * R];
    __shared__ __align__(8) unsigned long long bars[2];
    const int a = blockIdx.x * DM_THREADS + threadIdx.x;
    const bool valid = a < g.na;
    double pa[3], u[K][3];
    {
        const double* r = g.a_rec + (size_t)(valid ? a : 0) * R;
#pragma unroll
        for (int c = 0; c < 3; ++c) pa[c] = r[c];
#pragma unroll
        for (int q = 0; q < K; ++q)
#pragma unroll
            for (int c = 0; c < 3; ++c) u[q][c] = r[3 + 3 * q + c];
    }
    const int ntiles_b = (g.nb + DM_TILE - 1) / DM_TILE;
    const int t0 = blockIdx.y * g.tiles_per_split;
    const int t1 = min(ntiles_b, t0 + g.tiles_per_split);
    const int nt = max(0, t1 - t0);
    constexpr unsigned int TILE_BYTES = DM_TILE * R * sizeof(double);
    if (threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0 && nt > 0) {
        mbar_expect_tx(&bars[0], TILE_BYTES);
        bulk_g2s(s_b[0], g.b_rec + (size_t)t0 * DM_TILE * R, TILE_BYTES, &bars[0]);
    }
    double best = INFINITY, second = INFINITY;
    int bidx = -1;
    for (int it = 0; it < nt; ++it) {
        const int buf = it & 1;
        if (threadIdx.x == 0 && it + 1 < nt) {
            // the other buffer was last read in iteration it - 1, which ended with a block barrier
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&bars[buf ^ 1], TILE_BYTES);
            bulk_g2s(s_b[buf ^ 1], g.b_rec + (size_t)(t0 + it + 1) * DM_TILE * R, TILE_BYTES, &bars[buf ^ 1]);
        }
        mbar_wait(&bars[buf], (unsigned)(it >> 1) & 1u);
        const int b0 = (t0 + it) * DM_TILE;
        const int m = min(DM_TILE, g.nb - b0);
        if (valid) {
            for (int j = 0; j < m; ++j) {
                const double* r = s_b[buf] + j * R;
                if (g.use_radius && !(sq3(r[0] - pa[0], r[1] - pa[1], r[2] - pa[2]) <= g.r2)) continue;
                double d[K][K];
#pragma unroll
                for (int q = 0; q < K; ++q)
#pragma unroll
                    for (int p = 0; p < K; ++p)
                        d[q][p] = sq3(u[q][0] - r[3 + 3 * p], u[q][1] - r[4 + 3 * p], u[q][2] - r[5 + 3 * p]);
                double D = INFINITY;
#pragma unroll
                for (int s = 0; s < NC; ++s)
#pragma unroll
                    for (int t = 0; t < NC; ++t) {
                        double sum = d[CB.c[s][0]][CB.c[t][0]];
#pragma unroll
                        for (int e = 1; e < N; ++e) sum = __dadd_rn(sum, d[CB.c[s][e]][CB.c[t][e]]);
                        D = sum < D ? sum : D;
                    }
                if (D < best) {
                    second = best;
                    best = D;
                    bidx = b0 + j;
                } else if (D < second) {
                    second = D;
                }
            }
        }
        __syncthreads();
    }
    if (!valid) return;
    const size_t o = (size_t)blockIdx.y * g.na + a;
    g.p_best[o] = best;
    g.p_second[o] = second;
    g.p_idx[o] = bidx;
}

__global__ void k_desc_merge(const double* __restrict__ pb, const double* __restrict__ ps, const int* __restrict__ pi,
                             int na, int splits, double* __restrict__ best_out, double* __restrict__ second_out,
                             int* __restrict__ idx_out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= na) return;
    double best = INFINITY, second = INFINITY;
    int bidx = -1;
    for (int s = 0; s < splits; ++s) {   // split s covers lower b than split s + 1: ties keep the earlier index
        const size_t o = (size_t)s * na + a;
        const int i = pi[o];
        if (i < 0) continue;
        const double b = pb[o];
        second = fmin(second, ps[o]);
        if (b < best) {
            second = fmin(second, best);
            best = b;
            bidx = i;
        } else {
            second = fmin(second, b);
        }
    }
    best_out[a] = best;
    second_out[a] = second;
    idx_out[a] = bidx;
}

struct DescSet {
    int n = 0, nn = 0, red = 0, k = 0;
    double* xyz = nullptr;   // n x 3
    double* rec = nullptr;   // ceil(n / DM_TILE) * DM_TILE records of rec_len(k) doubles (zero padded)
    int* idx = nullptr;      // n x k
    double* d2 = nullptr;    // n x k
    bool has_desc() const { return n > k; }
};

struct MatchWs {
    std::unordered_map<unsigned long long, DescSet> sets;
    void* part = nullptr; size_t part_cap = 0;   // per-split best / second / index
    void* out = nullptr;  size_t out_cap = 0;    // merged best / second / index
};

MatchWs* ws_of(bs_ctx* ctx) {
    if (!ctx->match) ctx->match = new MatchWs();
    return (MatchWs*)ctx->match;
}

void free_set(DescSet& s) {
    for (void* p : {(void*)s.xyz, (void*)s.rec, (void*)s.idx, (void*)s.d2})
        if (p) cudaFree(p);
    s = DescSet();
}

template <int K>
void launch_knn(bs_ctx* ctx, const DescSet& s) {
    k_knn<K><<<(s.n + KNN_THREADS - 1) / KNN_THREADS, KNN_THREADS, 0, ctx->stream>>>(s.xyz, s.n, s.rec, s.idx, s.d2);
}

template <int N, int K>
void launch_match(bs_ctx* ctx, dim3 grid, const MatchArgs& a) {
    k_desc_match<N, K><<<grid, DM_THREADS, 0, ctx->stream>>>(a);
}

// (num_neighbors, k) -> the instantiation; false for an illegal pair
bool dispatch_match(bs_ctx* ctx, int n, int k, dim3 grid, const MatchArgs& a) {
#define BS_MATCH_CASE(N_, K_) \
    if (n == N_ && k == K_) { launch_match<N_, K_>(ctx, grid, a); return true; }
    BS_MATCH_CASE(3, 3) BS_MATCH_CASE(3, 4) BS_MATCH_CASE(3, 5) BS_MATCH_CASE(3, 6)
    BS_MATCH_CASE(4, 4) BS_MATCH_CASE(4, 5) BS_MATCH_CASE(4, 6)
    BS_MATCH_CASE(5, 5) BS_MATCH_CASE(5, 6)
    BS_MATCH_CASE(6, 6)
#undef BS_MATCH_CASE
    return false;
}

}  // namespace

void bs_match_free(bs_ctx* ctx) {
    MatchWs* W = (MatchWs*)ctx->match;
    if (!W) return;
    for (auto& kv : W->sets) free_set(kv.second);
    for (void* p : {W->part, W->out})
        if (p) cudaFree(p);
    delete W;
    ctx->match = nullptr;
}

extern "C" {

int bs_descriptors_build(bs_ctx* ctx, const double* xyz, int n, int num_neighbors, int redundancy,
                         unsigned long long* handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!handle || n < 0 || (n > 0 && !xyz))
        return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_build: bad argument");
    const int k = num_neighbors + redundancy;
    if (num_neighbors < 3 || redundancy < 0 || k > BS_MATCH_MAX_NEIGHBORS)
        return bs_set_error(ctx, BS_ERR_ARG,
                            "bs_descriptors_build: need 3 <= num_neighbors, 0 <= redundancy, num_neighbors + redundancy "
                            "<= %d (got %d, %d)", BS_MATCH_MAX_NEIGHBORS, num_neighbors, redundancy);
    for (long long i = 0; i < 3LL * n; ++i)
        if (!std::isfinite(xyz[i])) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_build: non-finite coordinate");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    DescSet s;
    s.n = n; s.nn = num_neighbors; s.red = redundancy; s.k = k;
    if (s.has_desc()) {
        const size_t nrec = (size_t)(n + DM_TILE - 1) / DM_TILE * DM_TILE;
        cudaError_t e = cudaMalloc(&s.xyz, (size_t)n * 3 * sizeof(double));
        if (e == cudaSuccess) e = cudaMalloc(&s.rec, nrec * rec_len(k) * sizeof(double));
        if (e == cudaSuccess) e = cudaMalloc(&s.idx, (size_t)n * k * sizeof(int));
        if (e == cudaSuccess) e = cudaMalloc(&s.d2, (size_t)n * k * sizeof(double));
        if (e == cudaSuccess) e = cudaMemsetAsync(s.rec, 0, nrec * rec_len(k) * sizeof(double), ctx->stream);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(s.xyz, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) {
            bs_launch_scope scope(ctx, "knn");
            switch (k) {
                case 3: launch_knn<3>(ctx, s); break;
                case 4: launch_knn<4>(ctx, s); break;
                case 5: launch_knn<5>(ctx, s); break;
                default: launch_knn<6>(ctx, s); break;
            }
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        // the pageable copy has consumed xyz when it returns; keep the set only once its kernel ran cleanly
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            free_set(s);
            return bs_set_error(ctx, e == cudaErrorMemoryAllocation ? BS_ERR_NOMEM : BS_ERR_CUDA,
                                "bs_descriptors_build: %s", cudaGetErrorString(e));
        }
    }
    *handle = ctx->next_handle++;
    ws_of(ctx)->sets[*handle] = s;
    return BS_OK;
}

int bs_descriptors_free(bs_ctx* ctx, unsigned long long handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    MatchWs* W = ws_of(ctx);
    auto it = W->sets.find(handle);
    if (it == W->sets.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_free: unknown handle %llu", handle);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    free_set(it->second);
    W->sets.erase(it);
    return BS_OK;
}

int bs_descriptors_neighbors(bs_ctx* ctx, unsigned long long handle, int* idx, double* d2) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    MatchWs* W = ws_of(ctx);
    auto it = W->sets.find(handle);
    if (it == W->sets.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_neighbors: unknown handle %llu", handle);
    const DescSet& s = it->second;
    const size_t cnt = (size_t)s.n * s.k;
    if (cnt > 0 && (!idx || !d2)) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_neighbors: NULL output");
    if (!s.has_desc()) {   // too few points: nobody has k other points
        for (size_t i = 0; i < cnt; ++i) { idx[i] = -1; d2[i] = INFINITY; }
        return BS_OK;
    }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaMemcpyAsync(idx, s.idx, cnt * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(d2, s.d2, cnt * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

int bs_descriptors_match(bs_ctx* ctx, unsigned long long ha, unsigned long long hb, double search_radius, int* best_b,
                         double* best, double* second) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    MatchWs* W = ws_of(ctx);
    auto ia = W->sets.find(ha), ib = W->sets.find(hb);
    if (ia == W->sets.end() || ib == W->sets.end())
        return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_match: unknown handle");
    const DescSet& A = ia->second;
    const DescSet& B = ib->second;
    if (A.nn != B.nn || A.red != B.red)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_match: A has (num_neighbors, redundancy) = (%d, %d), B (%d, %d)",
                            A.nn, A.red, B.nn, B.red);
    if (A.n > 0 && (!best_b || !best || !second)) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_match: NULL output");
    if (std::isnan(search_radius)) return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_match: search_radius is NaN");
    if (!A.has_desc() || !B.has_desc()) {
        for (int i = 0; i < A.n; ++i) { best_b[i] = -1; best[i] = INFINITY; second[i] = INFINITY; }
        return BS_OK;
    }
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    const int blocks_a = (A.n + DM_THREADS - 1) / DM_THREADS;
    const int tiles_b = (B.n + DM_TILE - 1) / DM_TILE;
    // split B when the A blocks alone cover less than two waves' worth of SMs
    int splits = std::min(tiles_b, std::max(1, (2 * ctx->sm_count + blocks_a - 1) / blocks_a));
    splits = std::min(splits, 65535);
    const int per = (tiles_b + splits - 1) / splits;
    splits = (tiles_b + per - 1) / per;
    const size_t np = (size_t)splits * A.n;
    int rc = bs_ensure_dev(ctx, &W->part, &W->part_cap, np * (2 * sizeof(double) + sizeof(int)));
    if (rc) return rc;
    rc = bs_ensure_dev(ctx, &W->out, &W->out_cap, (size_t)A.n * (2 * sizeof(double) + sizeof(int)));
    if (rc) return rc;
    MatchArgs a;
    a.a_rec = A.rec;
    a.b_rec = B.rec;
    a.na = A.n;
    a.nb = B.n;
    a.tiles_per_split = per;
    a.use_radius = search_radius >= 0.0 ? 1 : 0;
    a.r2 = search_radius >= 0.0 ? search_radius * search_radius : 0.0;
    a.p_best = (double*)W->part;
    a.p_second = a.p_best + np;
    a.p_idx = (int*)(a.p_second + np);
    double* o_best = (double*)W->out;
    double* o_second = o_best + A.n;
    int* o_idx = (int*)(o_second + A.n);
    {
        bs_launch_scope scope(ctx, "desc_match");
        if (!dispatch_match(ctx, A.nn, A.k, dim3((unsigned)blocks_a, (unsigned)splits), a))
            return bs_set_error(ctx, BS_ERR_ARG, "bs_descriptors_match: no instantiation for (%d, %d)", A.nn, A.k);
        k_desc_merge<<<(A.n + 255) / 256, 256, 0, ctx->stream>>>(a.p_best, a.p_second, a.p_idx, A.n, splits, o_best,
                                                                 o_second, o_idx);
    }
    BS_CUDA(ctx, cudaGetLastError());
    BS_CUDA(ctx, cudaMemcpyAsync(best, o_best, (size_t)A.n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(second, o_second, (size_t)A.n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaMemcpyAsync(best_b, o_idx, (size_t)A.n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

}  // extern "C"
