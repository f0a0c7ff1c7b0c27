// libbsgpu.so: context lifecycle, error reporting, profiling, resident volumes.
#include <cstdarg>
#include <cstring>

#include "bs_internal.cuh"

static thread_local std::string g_init_error;

int bs_set_error(bs_ctx* ctx, int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx)
        ctx->err = buf;
    else
        g_init_error = buf;
    return code;
}

int bs_ensure_dev(bs_ctx* ctx, void** p, size_t* cap, size_t need) {
    if (*cap >= need && *p) return BS_OK;
    if (*p) {
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        BS_CUDA(ctx, cudaFree(*p));
        *p = nullptr;
        *cap = 0;
    }
    BS_CUDA(ctx, cudaMalloc(p, need));
    *cap = need;
    return BS_OK;
}

void bs_profile_drain(bs_ctx* ctx) {
    for (auto& pe : ctx->prof_pending) {
        cudaEventSynchronize(pe.b);
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, pe.a, pe.b) == cudaSuccess) {
            auto& e = ctx->prof_entries[pe.tag];
            e.ms += ms;
            e.launches += 1;
        }
        cudaEventDestroy(pe.a);
        cudaEventDestroy(pe.b);
    }
    ctx->prof_pending.clear();
}

int bs_volume_acquire(bs_ctx* ctx, bs_volume& v) {
    if (v.ready_waited) return BS_OK;
    BS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, v.ready, 0));
    v.ready_waited = true;
    return BS_OK;
}

extern "C" {

int bs_version(void) { return 107; }

int bs_init(bs_ctx** out, int device, void* stream) {
    if (!out) return bs_set_error(nullptr, BS_ERR_ARG, "bs_init: out is NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return bs_set_error(nullptr, BS_ERR_CUDA,
                            "bs_init: no CUDA device available (%s); libbsgpu has no CPU fallback",
                            e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    if (device < 0 || device >= n)
        return bs_set_error(nullptr, BS_ERR_ARG, "bs_init: device %d out of range [0,%d)", device, n);
    e = cudaSetDevice(device);
    if (e != cudaSuccess)
        return bs_set_error(nullptr, BS_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess)
        return bs_set_error(nullptr, BS_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return bs_set_error(nullptr, BS_ERR_UNSUPPORTED,
                            "bs_init: device %d is sm_%d%d; libbsgpu is built for sm_90a only", device,
                            prop.major, prop.minor);
    bs_ctx* ctx = new bs_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (stream) {
        ctx->stream = (cudaStream_t)stream;
        ctx->own_stream = false;
    } else {
        e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) {
            delete ctx;
            return bs_set_error(nullptr, BS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
        }
        ctx->own_stream = true;
    }
    e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
        delete ctx;
        return bs_set_error(nullptr, BS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    }
    e = cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        cudaStreamDestroy(ctx->copy_stream);
        if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
        delete ctx;
        return bs_set_error(nullptr, BS_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    }
    *out = ctx;
    return BS_OK;
}

void bs_destroy(bs_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamSynchronize(ctx->d2h_stream);
    bs_profile_drain(ctx);
    for (auto& kv : ctx->vols) {
        if (kv.second.owned && kv.second.dev) cudaFree(kv.second.dev);
        if (kv.second.tmaps_dev) cudaFree(kv.second.tmaps_dev);
        if (kv.second.ready) cudaEventDestroy(kv.second.ready);
    }
    for (auto& kv : ctx->vol_pool) {
        cudaFree(kv.second.dev);
        if (kv.second.tmaps_dev) cudaFree(kv.second.tmaps_dev);
        if (kv.second.last_use) cudaEventDestroy(kv.second.last_use);
    }
    bs_pcm_workspace_free(ctx);
    bs_fuse2_free(ctx);
    bs_dog_free(ctx);
    bs_nonrigid_free(ctx);
    bs_match_free(ctx);
    bs_intensity_free(ctx);
    bs_comm_free(ctx);
    if (ctx->fuse_out) cudaFree(ctx->fuse_out);
    if (ctx->fuse_plan) cudaFree(ctx->fuse_plan);
    cudaStreamDestroy(ctx->copy_stream);
    cudaStreamDestroy(ctx->d2h_stream);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* bs_last_error(bs_ctx* ctx) { return ctx ? ctx->err.c_str() : g_init_error.c_str(); }

int bs_synchronize(bs_ctx* ctx) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

long long bs_launch_count(bs_ctx* ctx) { return ctx ? ctx->launches : -1; }

int bs_profile_enable(bs_ctx* ctx, int on) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->prof = on != 0;
    return BS_OK;
}

int bs_profile_reset(bs_ctx* ctx) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    bs_profile_drain(ctx);
    ctx->prof_entries.clear();
    return BS_OK;
}

int bs_profile_get(bs_ctx* ctx, const char* tag, double* ms_total, long long* launches) {
    if (!ctx || !tag) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    bs_profile_drain(ctx);
    auto it = ctx->prof_entries.find(tag);
    if (ms_total) *ms_total = it == ctx->prof_entries.end() ? 0.0 : it->second.ms;
    if (launches) *launches = it == ctx->prof_entries.end() ? 0 : it->second.launches;
    return BS_OK;
}

int bs_host_alloc(bs_ctx* ctx, unsigned long long bytes, void** out) {
    if (!ctx || !out) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    BS_CUDA(ctx, cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    return BS_OK;
}

int bs_host_free(bs_ctx* ctx, void* p) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    BS_CUDA(ctx, cudaFreeHost(p));
    return BS_OK;
}

static size_t dtype_size(int dtype) {
    switch (dtype) {
        case BS_DTYPE_U16: return 2;
        case BS_DTYPE_F32: return 4;
        case BS_DTYPE_U8: return 1;
        default: return 0;
    }
}

int bs_volume_upload(bs_ctx* ctx, const void* host, const long long dims[3], int dtype,
                     unsigned long long* handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!host || !dims || !handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_upload: NULL argument");
    size_t es = dtype_size(dtype);
    if (!es || dims[0] <= 0 || dims[1] <= 0 || dims[2] <= 0)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_upload: bad dtype/dims");
    if (dims[0] > 0x7fffffffLL || dims[1] > 0x7fffffffLL || dims[2] > 0x7fffffffLL)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_upload: dims exceed int32");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t bytes = (size_t)dims[0] * dims[1] * dims[2] * es;
    bs_volume v;
    BS_CUDA(ctx, cudaMalloc(&v.dev, bytes));
    cudaError_t e = cudaMemcpyAsync(v.dev, host, bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_volume_upload: copy failed: %s", cudaGetErrorString(e));
    }
    v.dims[0] = dims[0]; v.dims[1] = dims[1]; v.dims[2] = dims[2];
    v.dtype = dtype;
    v.owned = true;
    *handle = ctx->next_handle++;
    ctx->vols[*handle] = v;
    return BS_OK;
}

int bs_volume_upload_async(bs_ctx* ctx, const void* host, const long long dims[3], int dtype,
                           unsigned long long* handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!host || !dims || !handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_upload_async: NULL argument");
    size_t es = dtype_size(dtype);
    if (!es || dims[0] <= 0 || dims[1] <= 0 || dims[2] <= 0 || dims[0] > 0x7fffffffLL || dims[1] > 0x7fffffffLL ||
        dims[2] > 0x7fffffffLL)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_upload_async: bad dtype/dims");
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)dims[0] * dims[1] * dims[2] * es;
    bs_volume v;
    auto it = ctx->vol_pool.find(bytes);
    if (it != ctx->vol_pool.end()) {
        bs_pool_entry pe = it->second;
        ctx->vol_pool.erase(it);
        v.dev = pe.dev;
        if (pe.last_use) {
            // kernels of the buffer's previous life must be done before the copy overwrites it
            BS_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, pe.last_use, 0));
            cudaEventDestroy(pe.last_use);
        }
        if (pe.tmaps_dev) {
            if (pe.dims[0] == dims[0] && pe.dims[1] == dims[1] && pe.dims[2] == dims[2] && pe.dtype == dtype) {
                v.tmaps_dev = pe.tmaps_dev;
                v.tma_state = 1;
            } else {
                BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                cudaFree(pe.tmaps_dev);
            }
        }
    } else {
        BS_CUDA(ctx, cudaMalloc(&v.dev, bytes));
    }
    cudaError_t e = cudaMemcpyAsync(v.dev, host, bytes, cudaMemcpyHostToDevice, ctx->copy_stream);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&v.ready, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(v.ready, ctx->copy_stream);
    if (e != cudaSuccess) {
        cudaFree(v.dev);
        return bs_set_error(ctx, BS_ERR_CUDA, "bs_volume_upload_async: %s", cudaGetErrorString(e));
    }
    v.ready_waited = false;
    v.dims[0] = dims[0]; v.dims[1] = dims[1]; v.dims[2] = dims[2];
    v.dtype = dtype;
    v.owned = true;
    v.pooled = true;
    v.pool_bytes = bytes;
    *handle = ctx->next_handle++;
    ctx->vols[*handle] = v;
    return BS_OK;
}

int bs_volume_wrap(bs_ctx* ctx, const void* dev, const long long dims[3], int dtype,
                   unsigned long long* handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!dev || !dims || !handle) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_wrap: NULL argument");
    if (!dtype_size(dtype) || dims[0] <= 0 || dims[1] <= 0 || dims[2] <= 0 ||
        dims[0] > 0x7fffffffLL || dims[1] > 0x7fffffffLL || dims[2] > 0x7fffffffLL)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_wrap: bad dtype/dims");
    bs_volume v;
    v.dev = const_cast<void*>(dev);
    v.dims[0] = dims[0]; v.dims[1] = dims[1]; v.dims[2] = dims[2];
    v.dtype = dtype;
    v.owned = false;
    *handle = ctx->next_handle++;
    ctx->vols[*handle] = v;
    return BS_OK;
}

int bs_volume_free(bs_ctx* ctx, unsigned long long handle) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->vols.find(handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_free: unknown handle %llu", handle);
    bs_volume& v = it->second;
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    if (v.pooled) {
        // no host synchronisation: the buffer (and its tensor maps, which stay valid for it) goes back to the
        // pool together with an event that marks the end of everything queued on it so far
        cudaEvent_t last = nullptr;
        BS_CUDA(ctx, cudaEventCreateWithFlags(&last, cudaEventDisableTiming));
        if (!v.ready_waited) BS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, v.ready, 0));
        BS_CUDA(ctx, cudaEventRecord(last, ctx->stream));
        bs_pool_entry pe;
        pe.dev = v.dev;
        pe.last_use = last;
        pe.tmaps_dev = v.tmaps_dev;
        pe.dims[0] = v.dims[0]; pe.dims[1] = v.dims[1]; pe.dims[2] = v.dims[2];
        pe.dtype = v.dtype;
        ctx->vol_pool.insert({v.pool_bytes, pe});
    } else if (v.owned || v.tmaps_dev) {
        BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (v.owned) BS_CUDA(ctx, cudaFree(v.dev));
        if (v.tmaps_dev) BS_CUDA(ctx, cudaFree(v.tmaps_dev));
    }
    if (v.ready) cudaEventDestroy(v.ready);
    ctx->vols.erase(it);
    return BS_OK;
}

int bs_volume_devptr(bs_ctx* ctx, unsigned long long handle, void** dev) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->vols.find(handle);
    if (it == ctx->vols.end() || !dev) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_devptr: unknown handle or NULL out");
    *dev = it->second.dev;
    return BS_OK;
}

int bs_volume_info(bs_ctx* ctx, unsigned long long handle, long long dims[3], int* dtype) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->vols.find(handle);
    if (it == ctx->vols.end()) return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_info: unknown handle %llu", handle);
    if (dims) for (int d = 0; d < 3; ++d) dims[d] = it->second.dims[d];
    if (dtype) *dtype = it->second.dtype;
    return BS_OK;
}

int bs_volume_download(bs_ctx* ctx, unsigned long long handle, void* host, unsigned long long capacity_bytes) {
    if (!ctx) return BS_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->vols.find(handle);
    if (it == ctx->vols.end() || !host)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_download: unknown handle or NULL host");
    bs_volume& v = it->second;
    size_t bytes = (size_t)v.dims[0] * v.dims[1] * v.dims[2] * dtype_size(v.dtype);
    if (capacity_bytes < bytes)
        return bs_set_error(ctx, BS_ERR_ARG, "bs_volume_download: buffer of %llu bytes, volume needs %zu", capacity_bytes, bytes);
    BS_CUDA(ctx, cudaSetDevice(ctx->device));
    { int rc = bs_volume_acquire(ctx, v); if (rc) return rc; }
    BS_CUDA(ctx, cudaMemcpyAsync(host, v.dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    BS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BS_OK;
}

}  // extern "C"
