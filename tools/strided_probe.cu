// probe: the HBM bandwidth the strided FFT passes' access pattern allows, with no arithmetic.  An in-place
// read-modify-write of a 540 x 540 x 272 complex64 spectrum (z, y, x-fastest rows of pitch 272) in tiles of
// 540 rows x TC columns (TC = 8 -> 64 B row segments, TC = 16 -> 128 B), element stride `pitch` (the y pass) or
// `Py * pitch` (the z pass), loaded either directly into registers or with cp.async into shared memory.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a strided_probe.cu -o strided_probe && ./strided_probe
#include <cuda_runtime.h>
#include <cstdio>

#define N 540
#define PITCH 272
#define NT 256
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ float2* tile_base(float2* s, long long estride, long long ostride, int tc) {
    const int tiles_x = PITCH / tc;
    return s + (long long)(blockIdx.x / tiles_x) * ostride + (long long)(blockIdx.x % tiles_x) * tc;
}

// registers: 8-byte loads, a half-warp covers one row segment of 16 columns (two of 8)
template <int TC>
__global__ void __launch_bounds__(NT) k_reg(float2* s, long long estride, long long ostride) {
    constexpr int TOT = N * TC, IT = (TOT + NT - 1) / NT;
    float2* g = tile_base(s, estride, ostride, TC);
    float2 v[IT];
#pragma unroll
    for (int u = 0; u < IT; ++u) {
        const int i = threadIdx.x + u * NT;
        if (i < TOT) v[u] = __ldcg(g + (long long)(i / TC) * estride + (i % TC));
    }
#pragma unroll
    for (int u = 0; u < IT; ++u) {
        const int i = threadIdx.x + u * NT;
        if (i < TOT) __stcg(g + (long long)(i / TC) * estride + (i % TC), make_float2(v[u].x + 1.f, v[u].y));
    }
}

// cp.async: 16-byte requests into shared memory, then 16-byte stores from shared memory
template <int TC>
__global__ void __launch_bounds__(NT) k_cpasync(float2* s, long long estride, long long ostride) {
    extern __shared__ __align__(16) float4 sm4[];
    constexpr int VR = TC / 2, NV = N * VR;
    float2* g = tile_base(s, estride, ostride, TC);
    for (int i = threadIdx.x; i < NV; i += NT) {
        const float4* src = reinterpret_cast<const float4*>(g + (long long)(i / VR) * estride) + (i % VR);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(sm4 + i)), "l"(src) : "memory");
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    for (int i = threadIdx.x; i < NV; i += NT) {
        float4 v = sm4[i];
        v.x += 1.f;
        __stcg(reinterpret_cast<float4*>(g + (long long)(i / VR) * estride) + (i % VR), v);
    }
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const long long elems = (long long)N * N * PITCH;
    const double bytes = 2.0 * elems * sizeof(float2);   // every element read once and written once
    float2* s;
    CK(cudaMalloc(&s, elems * sizeof(float2)));
    CK(cudaMemset(s, 0, elems * sizeof(float2)));
    CK(cudaFuncSetAttribute(k_cpasync<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, N * 16 * 8));
    CK(cudaFuncSetAttribute(k_cpasync<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, N * 8 * 8));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    printf("device %s, %d SMs; array %d x %d x %d complex64 (%.0f MB), %.0f MB moved per sweep\n", prop.name,
           prop.multiProcessorCount, N, N, PITCH, elems * 8.0 / 1e6, bytes / 1e6);
    const int iters = 20;
    for (int axis = 0; axis < 2; ++axis) {          // 0: y (estride pitch), 1: z (estride Py * pitch)
        const long long estride = axis ? (long long)N * PITCH : PITCH;
        const long long ostride = axis ? PITCH : (long long)N * PITCH;
        for (int tc = 8; tc <= 16; tc *= 2)
            for (int style = 0; style < 2; ++style) {
                const int grid = (PITCH / tc) * N;
                auto launch = [&]() {
                    if (style == 0 && tc == 8) k_reg<8><<<grid, NT>>>(s, estride, ostride);
                    else if (style == 0) k_reg<16><<<grid, NT>>>(s, estride, ostride);
                    else if (tc == 8) k_cpasync<8><<<grid, NT, N * 8 * 8>>>(s, estride, ostride);
                    else k_cpasync<16><<<grid, NT, N * 16 * 8>>>(s, estride, ostride);
                };
                for (int w = 0; w < 3; ++w) launch();
                CK(cudaEventRecord(e0));
                for (int i = 0; i < iters; ++i) launch();
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                CK(cudaGetLastError());
                float ms = 0.f;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                const double gbs = bytes * iters / (ms * 1e-3) / 1e9;
                printf("axis %c  segment %3d B  %-8s  %7.3f ms/sweep  %7.1f GB/s  %.2f of 3.35 TB/s\n", axis ? 'z' : 'y',
                       tc * 8, style ? "cp.async" : "regs", ms / iters, gbs, gbs / 3350.0);
            }
    }
    CK(cudaFree(s));
    return 0;
}
