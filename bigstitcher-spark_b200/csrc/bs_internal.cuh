// Internal declarations shared by the translation units of libbsgpu.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "bsgpu.h"

struct bs_volume {
    void* dev = nullptr;
    long long dims[3] = {0, 0, 0};
    int dtype = 0;
    bool owned = false;
    cudaEvent_t ready = nullptr;  // async upload: H2D copy finished (waited for on the compute stream at first use)
    bool ready_waited = true;
    bool pooled = false;          // device buffer comes from / returns to the context's pool
    size_t pool_bytes = 0;
    void* tmaps_dev = nullptr;   // device copies of the volume's TMA tensor maps (fuse_tma.cu), lazily built
    int tma_state = 0;           // 0 not tried, 1 available, -1 not eligible (dtype / alignment / pitch)
};

struct bs_pool_entry {
    void* dev = nullptr;
    cudaEvent_t last_use = nullptr;   // end of everything that was queued on the buffer in its previous life
    void* tmaps_dev = nullptr;        // tensor maps stay valid while address, dims and dtype are unchanged
    long long dims[3] = {0, 0, 0};
    int dtype = 0;
};

struct bs_prof_entry {
    double ms = 0.0;
    long long launches = 0;
};

struct bs_pending_event {
    cudaEvent_t a, b;
    std::string tag;
};

struct PcmPending;   // pcm.cu: one result slot of the pair pipeline

// Workspace of the phase-correlation pipeline (grown on demand, reused between pairs).
struct bs_pcm_workspace {
    void* spec_a = nullptr;      // complex64 [Pz][Py][pitch]; also the real PCM (in place)
    void* spec_b = nullptr;
    size_t spec_bytes = 0;
    void* crop[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // double-buffered device crops (host input)
    size_t crop_bytes = 0;
    void* tables = nullptr;      // PcmDeviceTables*: twiddles + blend-extension profiles per axis
    void* small = nullptr;       // device scratch for peaks / pearson sums
    size_t small_bytes = 0;
    void* small_host = nullptr;  // pinned mirror
    PcmPending* slots = nullptr; // the result slots in small / small_host, each with its completion event
    void* sync = nullptr;        // int: hand-off error word, then the per-plane counters of the fused FFT kernels
    size_t sync_bytes = 0;
    cudaEvent_t crop_ready[2] = {nullptr, nullptr};
    cudaEvent_t crop_free[2] = {nullptr, nullptr};
};

struct bs_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t copy_stream = nullptr;   // host -> device copies
    cudaStream_t d2h_stream = nullptr;    // device -> host copies (PCIe is full duplex: never share the H2D stream)
    std::mutex mu;
    std::string err;
    std::unordered_map<unsigned long long, bs_volume> vols;
    unsigned long long next_handle = 1;
    long long launches = 0;
    bool prof = false;
    std::map<std::string, bs_prof_entry> prof_entries;
    std::vector<bs_pending_event> prof_pending;
    bs_pcm_workspace ws;
    void* fuse_plan = nullptr;        // per-tile view lists of the current fusion call
    size_t fuse_plan_cap = 0;
    void* fuse_out = nullptr;         // device staging for host outputs
    size_t fuse_out_cap = 0;
    void* fuse2 = nullptr;            // fuse_tma.cu workspace (Fuse2Ws)
    void* dog = nullptr;              // dog.cu workspace (region buffers, detection list)
    void* nonrigid = nullptr;         // nonrigid.cu workspace (view table, points, control-point grids)
    void* match = nullptr;            // match.cu workspace (resident descriptor sets, per-split match results)
    void* intensity = nullptr;        // intensity.cu workspace (resident pair candidates)
    void* nccl_comm = nullptr;        // comm.cu: ncclComm_t of the view-sharded exchange (bs_comm_init)
    int nccl_ranks = 0;
    // recycled device buffers of async-uploaded volumes, keyed by byte size
    std::multimap<size_t, bs_pool_entry> vol_pool;
    int sm_count = 132;
    bool pcm_attr_done = false;       // cudaFuncSetAttribute(max dynamic smem) done on this device
    bool pearson_attr_done = false;   // the same for k_pearson_u16 (set from its first launch)
    size_t pearson_smem = 0;          // dynamic smem of k_pearson_u16's last launch on this context ...
    int pearson_occ = 0;              // ... and its resident CTAs per SM
    int peak_occ = 0;                 // k_peaks' resident CTAs per SM, at most 8 (set from its first launch)
};

// bytes per voxel of a BS_DTYPE_*
static inline size_t bs_out_elem_size(int dt) { return dt == BS_DTYPE_F32 ? 4 : dt == BS_DTYPE_U16 ? 2 : 1; }

int bs_set_error(bs_ctx* ctx, int code, const char* fmt, ...);

#define BS_CUDA(ctx, call)                                                                   \
    do {                                                                                     \
        cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return bs_set_error((ctx), e__ == cudaErrorMemoryAllocation ? BS_ERR_NOMEM       \
                                                                        : BS_ERR_CUDA,       \
                                "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),     \
                                __FILE__, __LINE__);                                         \
    } while (0)

// RAII-less profiling bracket around one kernel launch.
struct bs_launch_scope {
    bs_ctx* ctx;
    cudaEvent_t a = nullptr, b = nullptr;
    const char* tag;
    bs_launch_scope(bs_ctx* c, const char* t) : ctx(c), tag(t) {
        ctx->launches++;
        if (ctx->prof) {
            cudaEventCreate(&a);
            cudaEventCreate(&b);
            cudaEventRecord(a, ctx->stream);
        }
    }
    ~bs_launch_scope() {
        if (a) {
            cudaEventRecord(b, ctx->stream);
            ctx->prof_pending.push_back({a, b, tag});
        }
    }
};

void bs_profile_drain(bs_ctx* ctx);

// device-buffer helper: (re)allocate when too small
int bs_ensure_dev(bs_ctx* ctx, void** p, size_t* cap, size_t need);

// make the compute stream wait for a volume's pending async upload (no-op afterwards)
int bs_volume_acquire(bs_ctx* ctx, bs_volume& v);
// pcm.cu
void bs_pcm_workspace_free(bs_ctx* ctx);
// fuse_tma.cu
void bs_fuse2_free(bs_ctx* ctx);
// Staging of one fusion call's tables (views, blocks, LUT, ...) into device memory on ctx->stream.
// bs_fuse_tables_reserve waits until the next pinned host slot is no longer read by an earlier copy and
// returns it (*host, `bytes` long, 16-byte aligned) with the device address the tables will have (*dev);
// bs_fuse_tables_commit queues the copy.  The device buffer is shared by all calls, so the kernels that read
// the tables must be queued on ctx->stream before the next call's commit.
int bs_fuse_tables_reserve(bs_ctx* ctx, size_t bytes, void** host, const void** dev);
int bs_fuse_tables_commit(bs_ctx* ctx);
// the driver's cuTensorMapEncodeTiled, or NULL when the driver does not provide it
PFN_cuTensorMapEncodeTiled_v12000 bs_tensor_map_encoder();
void bs_dog_free(bs_ctx* ctx);
// nonrigid.cu
void bs_nonrigid_free(bs_ctx* ctx);
// match.cu
void bs_match_free(bs_ctx* ctx);
// intensity.cu
void bs_intensity_free(bs_ctx* ctx);
// comm.cu
void bs_comm_free(bs_ctx* ctx);
// fuse.cu: generic tile kernel for one block into a device buffer (ctx->mu held by the caller; arguments
// validated by bs_fuse_validate and bs_fuse_validate_blocks)
int bs_fuse_legacy_block(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                         const long long block_size[3], const bs_fuse_params* params, void* out_dev);
// the argument checks shared by every fusion entry point
int bs_fuse_validate(bs_ctx* ctx, const bs_view* views, int n_views, const bs_fuse_params* p);
int bs_fuse_validate_blocks(bs_ctx* ctx, int nb, const long long* bmin, const long long* bsize, const bs_fuse_params* p);
// a block extent the fusion kernels' int sizes can hold
static inline bool bs_fuse_block_dim_ok(long long n) { return n > 0 && n <= 0x7fffffffLL; }
