// JNI shim of libbsgpu.so: marshalling only, one native method per bs_* entry point of include/bsgpu.h.
// Java side: jni/java/net/preibisch/bigstitcher/spark/gpu/BsNative.java (+ GpuStitching / GpuBlockSupplier glue that
// plugs into J/SparkPairwiseStitching.java:247-255 and J/SparkAffineFusion.java:602-627).
//
// This image has no JDK (no jni.h, no javac), so the shim cannot be compiled into a loadable library here; it is
// CMake-gated on find_package(JNI) (jni/CMakeLists.txt) and syntax-checked against tests/stub_jni/jni.h by
// tests/test_jni_shim.py.  Conventions:
//   * a bs_ctx* travels as a jlong; every failing bs_* call throws java.lang.RuntimeException(bs_last_error)
//     -- in hot path 2 that exception is what RetryTrackerSpark turns into a retry (J/util/RetryTrackerSpark.java:41-61);
//     hot path 1 reports "no shift" as found == 0 (the Java glue returns null, :274-279).
//   * voxel buffers are either primitive arrays (pinned for the duration of the call with
//     GetPrimitiveArrayCritical -- no copy) or direct ByteBuffers (bs_host_alloc'ed pinned memory for the async paths).
#include <jni.h>

#include <cstring>
#include <vector>

#include "bsgpu.h"

namespace {

inline bs_ctx* C(jlong h) { return reinterpret_cast<bs_ctx*>(h); }

// throws and returns true when rc signals an error
bool failed(JNIEnv* env, jlong ctx, int rc) {
    if (rc == BS_OK) return false;
    jclass ex = env->FindClass("java/lang/RuntimeException");
    if (ex) env->ThrowNew(ex, bs_last_error(C(ctx)));
    return true;
}

// a voxel buffer argument: primitive array (critical section) or direct ByteBuffer
struct Pinned {
    JNIEnv* env;
    jobject obj;
    void* p = nullptr;
    bool critical = false;
    Pinned(JNIEnv* e, jobject o) : env(e), obj(o) {
        if (!o) return;
        p = env->GetDirectBufferAddress(o);
        if (!p) {
            p = env->GetPrimitiveArrayCritical(static_cast<jarray>(o), nullptr);
            critical = p != nullptr;
        }
    }
    ~Pinned() { if (critical) env->ReleasePrimitiveArrayCritical(static_cast<jarray>(obj), p, 0); }
    Pinned(const Pinned&) = delete;
    Pinned& operator=(const Pinned&) = delete;
};

void get3(JNIEnv* env, jlongArray a, long long out[3]) {
    jlong t[3];
    env->GetLongArrayRegion(a, 0, 3, t);
    for (int i = 0; i < 3; ++i) out[i] = t[i];
}

// iparams = {peaksToCheck, doSubpixel, extX, extY, extZ}
bs_pcm_params pcm_params(JNIEnv* env, jintArray iparams, jdouble minOverlap) {
    jint ip[5];
    env->GetIntArrayRegion(iparams, 0, 5, ip);
    bs_pcm_params p;
    bs_pcm_default_params(&p);
    p.peaks_to_check = ip[0];
    p.do_subpixel = ip[1];
    p.extension[0] = ip[2]; p.extension[1] = ip[3]; p.extension[2] = ip[4];
    p.min_overlap_frac = minOverlap;
    return p;
}

constexpr int PCM_RESULT_DOUBLES = 20;
void pack_result(const bs_pcm_result& r, jdouble* d) {
    d[0] = r.found;
    for (int i = 0; i < 3; ++i) { d[1 + i] = (double)r.shift_int[i]; d[4 + i] = r.shift_sub[i]; d[9 + i] = (double)r.peak_index[i]; d[13 + i] = r.pad[i]; }
    d[7] = r.r; d[8] = (double)r.n_overlap_px; d[12] = r.pcm_value; d[16] = r.n_candidates; d[17] = (double)r.pearson_px;
    d[18] = d[19] = 0.0;
}

// views: models n*12 doubles, handles n*2 longs {volume, content}, blend n*6 floats {border, range}, windows n*6 longs
// {full_dims, window_min} (may be null)
std::vector<bs_view> unpack_views(JNIEnv* env, jint n, jdoubleArray models, jlongArray handles, jfloatArray blend, jlongArray windows) {
    std::vector<bs_view> v((size_t)n);
    if (n == 0) return v;
    std::vector<jdouble> m((size_t)n * 12);
    std::vector<jlong> h((size_t)n * 2, 0), w((size_t)n * 6, 0);
    std::vector<jfloat> b((size_t)n * 6, 0.f);
    env->GetDoubleArrayRegion(models, 0, n * 12, m.data());
    if (handles) env->GetLongArrayRegion(handles, 0, n * 2, h.data());
    if (blend) env->GetFloatArrayRegion(blend, 0, n * 6, b.data());
    if (windows) env->GetLongArrayRegion(windows, 0, n * 6, w.data());
    for (jint i = 0; i < n; ++i) {
        memset(&v[i], 0, sizeof(bs_view));
        for (int k = 0; k < 12; ++k) v[i].src_to_world[k] = m[(size_t)i * 12 + k];
        v[i].vol_handle = (unsigned long long)h[(size_t)i * 2];
        v[i].content_handle = (unsigned long long)h[(size_t)i * 2 + 1];
        for (int k = 0; k < 3; ++k) {
            v[i].blend_border[k] = b[(size_t)i * 6 + k];
            v[i].blend_range[k] = b[(size_t)i * 6 + 3 + k];
            v[i].full_dims[k] = w[(size_t)i * 6 + k];
            v[i].window_min[k] = w[(size_t)i * 6 + 3 + k];
        }
    }
    return v;
}

// iparams = {fusionType, interpolation, outDtype, blendLutN, outBigEndian}; dparams = {minIntensity, maxIntensity}
bs_fuse_params fuse_params(JNIEnv* env, jintArray iparams, jdoubleArray dparams) {
    jint ip[5];
    jdouble dp[2];
    env->GetIntArrayRegion(iparams, 0, 5, ip);
    env->GetDoubleArrayRegion(dparams, 0, 2, dp);
    bs_fuse_params p;
    bs_fuse_default_params(&p);
    p.fusion_type = ip[0]; p.interpolation = ip[1]; p.out_dtype = ip[2]; p.blend_lut_n = ip[3];
    p.min_intensity = dp[0]; p.max_intensity = dp[1];
    p.out_big_endian = ip[4];
    return p;
}

}  // namespace

#define JF(ret, name) extern "C" JNIEXPORT ret JNICALL Java_net_preibisch_bigstitcher_spark_gpu_BsNative_##name

// ---------------------------------------------------------------------------------------- lifecycle
JF(jint, version)(JNIEnv*, jclass) { return bs_version(); }

JF(jlong, init)(JNIEnv* env, jclass, jint device) {
    bs_ctx* ctx = nullptr;
    if (bs_init(&ctx, device, nullptr) != BS_OK) {
        jclass ex = env->FindClass("java/lang/RuntimeException");
        if (ex) env->ThrowNew(ex, bs_last_error(nullptr));
        return 0;
    }
    return reinterpret_cast<jlong>(ctx);
}

JF(void, destroy)(JNIEnv*, jclass, jlong ctx) { bs_destroy(C(ctx)); }
JF(jstring, lastError)(JNIEnv* env, jclass, jlong ctx) { return env->NewStringUTF(bs_last_error(C(ctx))); }
JF(void, synchronize)(JNIEnv* env, jclass, jlong ctx) { failed(env, ctx, bs_synchronize(C(ctx))); }
JF(jlong, launchCount)(JNIEnv*, jclass, jlong ctx) { return bs_launch_count(C(ctx)); }
JF(void, profileEnable)(JNIEnv* env, jclass, jlong ctx, jboolean on) { failed(env, ctx, bs_profile_enable(C(ctx), on ? 1 : 0)); }
JF(void, profileReset)(JNIEnv* env, jclass, jlong ctx) { failed(env, ctx, bs_profile_reset(C(ctx))); }

JF(jdoubleArray, profileGet)(JNIEnv* env, jclass, jlong ctx, jstring tag) {
    const char* t = env->GetStringUTFChars(tag, nullptr);
    double ms = 0.0;
    long long n = 0;
    const int rc = bs_profile_get(C(ctx), t, &ms, &n);
    env->ReleaseStringUTFChars(tag, t);
    if (failed(env, ctx, rc)) return nullptr;
    const jdouble out[2] = {ms, (double)n};
    jdoubleArray a = env->NewDoubleArray(2);
    env->SetDoubleArrayRegion(a, 0, 2, out);
    return a;
}

// pinned host memory as a direct ByteBuffer (for the async upload / streaming output paths)
JF(jobject, hostAlloc)(JNIEnv* env, jclass, jlong ctx, jlong bytes) {
    void* p = nullptr;
    if (failed(env, ctx, bs_host_alloc(C(ctx), (unsigned long long)bytes, &p))) return nullptr;
    return env->NewDirectByteBuffer(p, bytes);
}
JF(void, hostFree)(JNIEnv* env, jclass, jlong ctx, jobject buf) { failed(env, ctx, bs_host_free(C(ctx), env->GetDirectBufferAddress(buf))); }

// ---------------------------------------------------------------------------------------- resident volumes
JF(jlong, volumeUpload)(JNIEnv* env, jclass, jlong ctx, jobject data, jlongArray dims, jint dtype) {
    long long d[3];
    get3(env, dims, d);
    unsigned long long h = 0;
    int rc;
    {
        Pinned p(env, data);
        rc = bs_volume_upload(C(ctx), p.p, d, dtype, &h);   // synchronous: the critical section ends after the copy
    }
    return failed(env, ctx, rc) ? 0 : (jlong)h;
}

JF(jlong, volumeUploadAsync)(JNIEnv* env, jclass, jlong ctx, jobject pinnedBuffer, jlongArray dims, jint dtype) {
    long long d[3];
    get3(env, dims, d);
    unsigned long long h = 0;
    // only direct (bs_host_alloc'ed) buffers: the copy runs after this call returns
    void* p = env->GetDirectBufferAddress(pinnedBuffer);
    return failed(env, ctx, bs_volume_upload_async(C(ctx), p, d, dtype, &h)) ? 0 : (jlong)h;
}

JF(jlong, volumeWrap)(JNIEnv* env, jclass, jlong ctx, jlong devPtr, jlongArray dims, jint dtype) {
    long long d[3];
    get3(env, dims, d);
    unsigned long long h = 0;
    return failed(env, ctx, bs_volume_wrap(C(ctx), reinterpret_cast<const void*>(devPtr), d, dtype, &h)) ? 0 : (jlong)h;
}

JF(void, volumeFree)(JNIEnv* env, jclass, jlong ctx, jlong handle) { failed(env, ctx, bs_volume_free(C(ctx), (unsigned long long)handle)); }

JF(jlongArray, volumeInfo)(JNIEnv* env, jclass, jlong ctx, jlong handle) {
    long long d[3];
    int dt = 0;
    if (failed(env, ctx, bs_volume_info(C(ctx), (unsigned long long)handle, d, &dt))) return nullptr;
    const jlong out[4] = {d[0], d[1], d[2], dt};
    jlongArray a = env->NewLongArray(4);
    env->SetLongArrayRegion(a, 0, 4, out);
    return a;
}

JF(jlong, volumeDevptr)(JNIEnv* env, jclass, jlong ctx, jlong handle) {
    void* p = nullptr;
    return failed(env, ctx, bs_volume_devptr(C(ctx), (unsigned long long)handle, &p)) ? 0 : reinterpret_cast<jlong>(p);
}

JF(void, volumeDownload)(JNIEnv* env, jclass, jlong ctx, jlong handle, jobject dst, jlong capacityBytes) {
    int rc;
    {
        Pinned p(env, dst);
        rc = bs_volume_download(C(ctx), (unsigned long long)handle, p.p, (unsigned long long)capacityBytes);
    }
    failed(env, ctx, rc);
}

JF(jlong, contentWeights)(JNIEnv* env, jclass, jlong ctx, jlong handle, jdouble sigma1, jdouble sigma2) {
    unsigned long long h = 0;
    return failed(env, ctx, bs_content_weights(C(ctx), (unsigned long long)handle, sigma1, sigma2, &h)) ? 0 : (jlong)h;
}

JF(jlong, downsample)(JNIEnv* env, jclass, jlong ctx, jlong handle, jintArray factors) {
    jint f[3];
    env->GetIntArrayRegion(factors, 0, 3, f);
    const int ff[3] = {f[0], f[1], f[2]};
    unsigned long long h = 0;
    return failed(env, ctx, bs_downsample(C(ctx), (unsigned long long)handle, ff, &h)) ? 0 : (jlong)h;
}

// ---------------------------------------------------------------------------------------- hot path 1
JF(jint, goodFftSize)(JNIEnv*, jclass, jint n, jboolean even) { return bs_good_fft_size(n, even ? 1 : 0); }

// one overlap-cropped pair from Java arrays (short[] / float[] / byte[]): returns PCM_RESULT_DOUBLES doubles
JF(jdoubleArray, pcmPair)(JNIEnv* env, jclass, jlong ctx, jobject img1, jobject img2, jlongArray dims, jint dtype,
                          jintArray iparams, jdouble minOverlap) {
    long long d[3];
    get3(env, dims, d);
    const bs_pcm_params p = pcm_params(env, iparams, minOverlap);
    bs_pcm_result r;
    int rc;
    {
        Pinned a(env, img1), b(env, img2);
        rc = bs_pcm_pair(C(ctx), a.p, b.p, d, dtype, &p, 0, &r);
    }
    if (failed(env, ctx, rc)) return nullptr;
    jdouble out[PCM_RESULT_DOUBLES];
    pack_result(r, out);
    jdoubleArray arr = env->NewDoubleArray(PCM_RESULT_DOUBLES);
    env->SetDoubleArrayRegion(arr, 0, PCM_RESULT_DOUBLES, out);
    return arr;
}

// n pairs; imgs1 / imgs2: Object[] of direct ByteBuffers (pinned) -- primitive arrays cannot all be held critical
// at once; dims: n*3 longs.  Returns n * PCM_RESULT_DOUBLES doubles.
JF(jdoubleArray, pcmBatch)(JNIEnv* env, jclass, jlong ctx, jobjectArray imgs1, jobjectArray imgs2, jlongArray dims, jint dtype,
                           jintArray iparams, jdouble minOverlap) {
    const jsize n = env->GetArrayLength(imgs1);
    std::vector<const void*> a((size_t)n), b((size_t)n);
    std::vector<jlong> dj((size_t)n * 3);
    std::vector<long long> d((size_t)n * 3);
    env->GetLongArrayRegion(dims, 0, n * 3, dj.data());
    for (jsize i = 0; i < n; ++i) {
        a[(size_t)i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(imgs1, i));
        b[(size_t)i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(imgs2, i));
        for (int k = 0; k < 3; ++k) d[(size_t)i * 3 + k] = dj[(size_t)i * 3 + k];
    }
    const bs_pcm_params p = pcm_params(env, iparams, minOverlap);
    std::vector<bs_pcm_result> r((size_t)n);
    if (failed(env, ctx, bs_pcm_batch(C(ctx), n, a.data(), b.data(), d.data(), dtype, &p, 0, r.data()))) return nullptr;
    std::vector<jdouble> out((size_t)n * PCM_RESULT_DOUBLES);
    for (jsize i = 0; i < n; ++i) pack_result(r[(size_t)i], out.data() + (size_t)i * PCM_RESULT_DOUBLES);
    jdoubleArray arr = env->NewDoubleArray(n * PCM_RESULT_DOUBLES);
    env->SetDoubleArrayRegion(arr, 0, n * PCM_RESULT_DOUBLES, out.data());
    return arr;
}

// jobs: n * 11 longs {vol1, vol2, min1[3], min2[3], dims[3]} on resident volumes (tiles uploaded once)
JF(jdoubleArray, pcmVolumesBatch)(JNIEnv* env, jclass, jlong ctx, jlongArray jobs, jintArray iparams, jdouble minOverlap) {
    const jsize n = env->GetArrayLength(jobs) / 11;
    std::vector<jlong> j((size_t)n * 11);
    env->GetLongArrayRegion(jobs, 0, n * 11, j.data());
    std::vector<bs_pcm_job> jb((size_t)n);
    for (jsize i = 0; i < n; ++i) {
        const jlong* s = j.data() + (size_t)i * 11;
        jb[(size_t)i].vol1 = (unsigned long long)s[0];
        jb[(size_t)i].vol2 = (unsigned long long)s[1];
        for (int k = 0; k < 3; ++k) { jb[(size_t)i].min1[k] = s[2 + k]; jb[(size_t)i].min2[k] = s[5 + k]; jb[(size_t)i].dims[k] = s[8 + k]; }
    }
    const bs_pcm_params p = pcm_params(env, iparams, minOverlap);
    std::vector<bs_pcm_result> r((size_t)n);
    if (failed(env, ctx, bs_pcm_volumes_batch(C(ctx), n, jb.data(), &p, r.data()))) return nullptr;
    std::vector<jdouble> out((size_t)n * PCM_RESULT_DOUBLES);
    for (jsize i = 0; i < n; ++i) pack_result(r[(size_t)i], out.data() + (size_t)i * PCM_RESULT_DOUBLES);
    jdoubleArray arr = env->NewDoubleArray(n * PCM_RESULT_DOUBLES);
    env->SetDoubleArrayRegion(arr, 0, n * PCM_RESULT_DOUBLES, out.data());
    return arr;
}

// diagnostic: padded PCM volume into a float[] (pad[0]*pad[1]*pad[2]); returns the padded dims
JF(jlongArray, pcmDebugPcm)(JNIEnv* env, jclass, jlong ctx, jobject img1, jobject img2, jlongArray dims, jint dtype, jintArray extension,
                            jobject outPcm) {
    long long d[3];
    get3(env, dims, d);
    jint e[3];
    env->GetIntArrayRegion(extension, 0, 3, e);
    const int ext[3] = {e[0], e[1], e[2]};
    int pad[3] = {0, 0, 0};
    int rc;
    {
        Pinned a(env, img1), b(env, img2), o(env, outPcm);
        rc = bs_pcm_debug_pcm(C(ctx), a.p, b.p, d, dtype, ext, static_cast<float*>(o.p), pad);
    }
    if (failed(env, ctx, rc)) return nullptr;
    const jlong out[3] = {pad[0], pad[1], pad[2]};
    jlongArray arr = env->NewLongArray(3);
    env->SetLongArrayRegion(arr, 0, 3, out);
    return arr;
}

// diagnostic: one FFT pass of the PCM pipeline (include/bsgpu.h bs_pcm_debug_pass).  Pass 0: devA / devB are device
// crops (volumeDevptr) and inA / inB are ignored; passes 1-4: inA / inB are complex64 spectra (float[2 * Pz*Py*(M+1)],
// interleaved).  outA / outB: float[] spectra, or float[Pz*Py*Px] for pass 4.  padOut (may be null) receives {Px, Py, Pz};
// returns the kernel info string.
JF(jstring, pcmDebugPass)(JNIEnv* env, jclass, jlong ctx, jint pass, jlongArray dims, jint dtype, jintArray extension, jlong devA,
                          jlong devB, jobject inA, jobject inB, jobject outA, jobject outB, jint poison, jlongArray padOut) {
    long long d[3];
    get3(env, dims, d);
    jint e[3];
    env->GetIntArrayRegion(extension, 0, 3, e);
    const int ext[3] = {e[0], e[1], e[2]};
    int pad[3] = {0, 0, 0};
    char info[128] = "";
    int rc;
    {
        Pinned ia(env, inA), ib(env, inB), oa(env, outA), ob(env, outB);
        const void* a = pass == 0 ? reinterpret_cast<const void*>(devA) : ia.p;
        const void* b = pass == 0 ? reinterpret_cast<const void*>(devB) : ib.p;
        rc = bs_pcm_debug_pass(C(ctx), pass, d, dtype, ext, a, b, oa.p, ob.p, poison, pad, info);
    }
    if (failed(env, ctx, rc)) return nullptr;
    const jlong p[3] = {pad[0], pad[1], pad[2]};
    if (padOut) env->SetLongArrayRegion(padOut, 0, 3, p);
    return env->NewStringUTF(info);
}

// diagnostic: Pearson sums of n explicit boxes (n x {o1[3], o2[3], sz[3]}) on two device crops (volumeDevptr);
// sumsOut: long[5 n] (uint16 / uint8) or double[5 n] (float32)
JF(void, pcmDebugPearson)(JNIEnv* env, jclass, jlong ctx, jlong dev1, jlong dev2, jlongArray dims, jint dtype, jintArray boxes,
                          jobject sumsOut) {
    long long d[3];
    get3(env, dims, d);
    const int n = boxes ? env->GetArrayLength(boxes) / 9 : 0;
    int rc;
    {
        Pinned b(env, boxes), o(env, sumsOut);
        rc = bs_pcm_debug_pearson(C(ctx), reinterpret_cast<const void*>(dev1), reinterpret_cast<const void*>(dev2), d, dtype, n,
                                  static_cast<const int*>(b.p), o.p);
    }
    failed(env, ctx, rc);
}

// ---------------------------------------------------------------------------------------- hot path 2
// BlockSupplier<T>.copy(interval, dest): dest is the primitive array BlockAlgoUtils.arrayImg allocated
JF(void, fuseBlock)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles, jfloatArray blend,
                    jlongArray windows, jlongArray blockMin, jlongArray blockSize, jintArray iparams, jdoubleArray dparams, jobject dest) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, blend, windows);
    long long mn[3], sz[3];
    get3(env, blockMin, mn);
    get3(env, blockSize, sz);
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    int rc;
    {
        Pinned o(env, dest);
        rc = bs_fuse_block(C(ctx), v.data(), nViews, mn, sz, &p, o.p, 0);
    }
    failed(env, ctx, rc);
}

// a list of blocks in one launch; dests: Object[] of direct ByteBuffers (pinned), blockMins / blockSizes: n*3 longs
JF(void, fuseBlocks)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles, jfloatArray blend,
                     jlongArray windows, jlongArray blockMins, jlongArray blockSizes, jintArray iparams, jdoubleArray dparams,
                     jobjectArray dests) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, blend, windows);
    const jsize n = env->GetArrayLength(dests);
    std::vector<jlong> mnj((size_t)n * 3), szj((size_t)n * 3);
    env->GetLongArrayRegion(blockMins, 0, n * 3, mnj.data());
    env->GetLongArrayRegion(blockSizes, 0, n * 3, szj.data());
    std::vector<long long> mn(mnj.begin(), mnj.end()), sz(szj.begin(), szj.end());
    std::vector<void*> outs((size_t)n);
    for (jsize i = 0; i < n; ++i) outs[(size_t)i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(dests, i));
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    failed(env, ctx, bs_fuse_blocks(C(ctx), v.data(), nViews, n, mn.data(), sz.data(), &p, outs.data(), 0));
}

// --masks mode: views carry geometry only (models + windows{fullDims, 0}); maskOffset {x, y, z} in source pixels
JF(void, maskBlocks)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles, jlongArray windows,
                     jlongArray blockMins, jlongArray blockSizes, jdoubleArray maskOffset, jint outDtype, jint outBigEndian,
                     jobjectArray dests) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, nullptr, windows);
    const jsize n = env->GetArrayLength(dests);
    std::vector<jlong> mnj((size_t)n * 3), szj((size_t)n * 3);
    env->GetLongArrayRegion(blockMins, 0, n * 3, mnj.data());
    env->GetLongArrayRegion(blockSizes, 0, n * 3, szj.data());
    std::vector<long long> mn(mnj.begin(), mnj.end()), sz(szj.begin(), szj.end());
    std::vector<void*> outs((size_t)n);
    for (jsize i = 0; i < n; ++i) outs[(size_t)i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(dests, i));
    jdouble off[3];
    env->GetDoubleArrayRegion(maskOffset, 0, 3, off);
    failed(env, ctx, bs_mask_blocks(C(ctx), v.data(), nViews, n, mn.data(), sz.data(), off, outDtype, outBigEndian, outs.data(), 0));
}

JF(jlong, fuseBlockToVolume)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles, jfloatArray blend,
                             jlongArray windows, jlongArray blockMin, jlongArray blockSize, jintArray iparams, jdoubleArray dparams) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, blend, windows);
    long long mn[3], sz[3];
    get3(env, blockMin, mn);
    get3(env, blockSize, sz);
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    unsigned long long h = 0;
    return failed(env, ctx, bs_fuse_block_to_volume(C(ctx), v.data(), nViews, mn, sz, &p, &h)) ? 0 : (jlong)h;
}

// view-sharded mode: partial sums into device buffers the caller all-reduces (NCCL) and finishes
JF(void, fuseAccumulate)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles, jfloatArray blend,
                         jlongArray blockMin, jlongArray blockSize, jintArray iparams, jdoubleArray dparams, jlong sumWiDev, jlong sumWDev) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, blend, nullptr);
    long long mn[3], sz[3];
    get3(env, blockMin, mn);
    get3(env, blockSize, sz);
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    failed(env, ctx, bs_fuse_accumulate(C(ctx), v.data(), nViews, mn, sz, &p, reinterpret_cast<float*>(sumWiDev),
                                        reinterpret_cast<float*>(sumWDev)));
}

JF(void, fuseFinish)(JNIEnv* env, jclass, jlong ctx, jlong sumWiDev, jlong sumWDev, jlong n, jintArray iparams, jdoubleArray dparams,
                     jobject dest) {
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    int rc;
    {
        Pinned o(env, dest);
        rc = bs_fuse_finish(C(ctx), reinterpret_cast<const float*>(sumWiDev), reinterpret_cast<const float*>(sumWDev), n, &p, o.p, 0);
    }
    failed(env, ctx, rc);
}

// the exchange behind the C ABI: rank 0 draws the id, the Java driver ships the 128 bytes, every worker joins
JF(jbyteArray, commUniqueId)(JNIEnv* env, jclass) {
    unsigned char id[128];
    if (bs_comm_unique_id(id) != BS_OK) {
        jclass ex = env->FindClass("java/lang/RuntimeException");
        if (ex) env->ThrowNew(ex, bs_last_error(nullptr));
        return nullptr;
    }
    jbyteArray a = env->NewByteArray(128);
    env->SetByteArrayRegion(a, 0, 128, reinterpret_cast<const jbyte*>(id));
    return a;
}

JF(void, commInit)(JNIEnv* env, jclass, jlong ctx, jint nRanks, jint rank, jbyteArray id) {
    jbyte b[128];
    env->GetByteArrayRegion(id, 0, 128, b);
    failed(env, ctx, bs_comm_init(C(ctx), nRanks, rank, reinterpret_cast<const unsigned char*>(b)));
}

JF(void, commDestroy)(JNIEnv* env, jclass, jlong ctx) { failed(env, ctx, bs_comm_destroy(C(ctx))); }

JF(void, fuseAllreduce)(JNIEnv* env, jclass, jlong ctx, jlong sumWiDev, jlong sumWDev, jlong n) {
    failed(env, ctx, bs_fuse_allreduce(C(ctx), reinterpret_cast<float*>(sumWiDev), reinterpret_cast<float*>(sumWDev), n));
}

// ---------------------------------------------------------------------------------------- next row: DoG
// returns n * 8 doubles {locX, locY, locZ, value, voxelX, voxelY, voxelZ, isMax}
JF(jdoubleArray, dogDetect)(JNIEnv* env, jclass, jlong ctx, jlong handle, jlongArray intervalMin, jlongArray intervalSize,
                            jdoubleArray dparams /* sigma, threshold, minI, maxI */, jintArray iparams /* findMax, findMin, localization */) {
    long long mn[3], sz[3];
    get3(env, intervalMin, mn);
    get3(env, intervalSize, sz);
    jdouble dp[4];
    jint ip[3];
    env->GetDoubleArrayRegion(dparams, 0, 4, dp);
    env->GetIntArrayRegion(iparams, 0, 3, ip);
    bs_dog_params p;
    bs_dog_default_params(&p);
    p.sigma = dp[0]; p.threshold = dp[1]; p.min_intensity = dp[2]; p.max_intensity = dp[3];
    p.find_max = ip[0]; p.find_min = ip[1]; p.localization = ip[2];
    int cap = 1 << 16, n = 0;
    std::vector<bs_dog_point> pts;
    for (;;) {
        pts.resize((size_t)cap);
        if (failed(env, ctx, bs_dog_detect(C(ctx), (unsigned long long)handle, mn, sz, &p, pts.data(), cap, &n))) return nullptr;
        if (n <= cap) break;
        cap = n;
    }
    std::vector<jdouble> out((size_t)n * 8);
    for (int i = 0; i < n; ++i) {
        jdouble* o = out.data() + (size_t)i * 8;
        for (int k = 0; k < 3; ++k) { o[k] = pts[(size_t)i].loc[k]; o[4 + k] = (double)pts[(size_t)i].voxel[k]; }
        o[3] = pts[(size_t)i].value;
        o[7] = pts[(size_t)i].is_max;
    }
    jdoubleArray arr = env->NewDoubleArray(n * 8);
    env->SetDoubleArrayRegion(arr, 0, n * 8, out.data());
    return arr;
}

// diagnostic: the DoG box the extremum stage reads (include/bsgpu.h bs_dog_debug_dog); out: float[(sx + 2)(sy + 2)(sz + 2)],
// x fastest; blur 0 production, 1 generic, 2 window R 6, 3 window R 12; returns the blur instantiation launched
JF(jstring, dogDebugDog)(JNIEnv* env, jclass, jlong ctx, jlong handle, jlongArray intervalMin, jlongArray intervalSize,
                         jdoubleArray dparams /* sigma, minI, maxI */, jint blur, jobject out) {
    long long mn[3], sz[3];
    get3(env, intervalMin, mn);
    get3(env, intervalSize, sz);
    jdouble dp[3];
    env->GetDoubleArrayRegion(dparams, 0, 3, dp);
    bs_dog_params p;
    bs_dog_default_params(&p);
    p.sigma = dp[0]; p.min_intensity = dp[1]; p.max_intensity = dp[2];
    char info[128] = "";
    int rc;
    {
        Pinned o(env, out);
        rc = bs_dog_debug_dog(C(ctx), (unsigned long long)handle, mn, sz, &p, blur, static_cast<float*>(o.p), info);
    }
    if (failed(env, ctx, rc)) return nullptr;
    return env->NewStringUTF(info);
}

// ---------------------------------------------------------------------------------------- detect-interestpoints helpers
JF(jlong, downsampleFloat)(JNIEnv* env, jclass, jlong ctx, jlong handle, jintArray factors) {
    jint f[3];
    env->GetIntArrayRegion(factors, 0, 3, f);
    const int ff[3] = {f[0], f[1], f[2]};
    unsigned long long h = 0;
    return failed(env, ctx, bs_downsample_float(C(ctx), (unsigned long long)handle, ff, &h)) ? 0 : (jlong)h;
}

JF(jlong, medianDivide)(JNIEnv* env, jclass, jlong ctx, jlong handle, jint radius) {
    unsigned long long h = 0;
    return failed(env, ctx, bs_median_divide(C(ctx), (unsigned long long)handle, radius, &h)) ? 0 : (jlong)h;
}

// loc: double[3n] {x, y, z} per point; out: float[n] (or a direct ByteBuffer of n floats)
JF(void, sampleNlinear)(JNIEnv* env, jclass, jlong ctx, jlong handle, jdoubleArray loc, jobject out) {
    const jint n = env->GetArrayLength(loc) / 3;
    std::vector<jdouble> l((size_t)n * 3);
    env->GetDoubleArrayRegion(loc, 0, n * 3, l.data());
    int rc;
    {
        Pinned o(env, out);
        rc = bs_sample_nlinear(C(ctx), (unsigned long long)handle, n, l.data(), static_cast<float*>(o.p));
    }
    failed(env, ctx, rc);
}

// ---------------------------------------------------------------------------------------- nonrigid-fusion
// views as for fuseBlocks plus nPoints int[n], targets / locals double[3 * sum(nPoints)] (the views' points one after
// the other, {x, y, z} each); replaces NonRigidTools.fuseVirtualInterpolatedNonRigid (J/SparkNonRigidFusion.java:387-401)
namespace {
std::vector<bs_nonrigid_view> unpack_nonrigid(JNIEnv* env, jint n, const std::vector<bs_view>& v, const std::vector<jint>& np,
                                              jdoubleArray targets, jdoubleArray locals, std::vector<jdouble>& t,
                                              std::vector<jdouble>& l) {
    std::vector<bs_nonrigid_view> nv((size_t)n);
    size_t total = 0;
    for (jint i = 0; i < n; ++i) total += (size_t)np[(size_t)i];
    t.assign(total * 3, 0.0);
    l.assign(total * 3, 0.0);
    if (total) {
        env->GetDoubleArrayRegion(targets, 0, (jsize)(total * 3), t.data());
        env->GetDoubleArrayRegion(locals, 0, (jsize)(total * 3), l.data());
    }
    size_t at = 0;
    for (jint i = 0; i < n; ++i) {
        memset(&nv[(size_t)i], 0, sizeof(bs_nonrigid_view));
        nv[(size_t)i].view = v[(size_t)i];
        nv[(size_t)i].n_points = np[(size_t)i];
        nv[(size_t)i].target_world_xyz = t.data() + at * 3;
        nv[(size_t)i].local_xyz = l.data() + at * 3;
        at += (size_t)np[(size_t)i];
    }
    return nv;
}
}  // namespace

// cpDistance long[3] (the reference passes 10, 10, 10); dests: Object[] of direct ByteBuffers, one per block
JF(void, nonrigidFuseBlocks)(JNIEnv* env, jclass, jlong ctx, jint nViews, jdoubleArray models, jlongArray handles,
                             jfloatArray blend, jlongArray windows, jintArray nPoints, jdoubleArray targets, jdoubleArray locals,
                             jlongArray blockMins, jlongArray blockSizes, jlongArray cpDistance, jintArray iparams,
                             jdoubleArray dparams, jobjectArray dests) {
    std::vector<bs_view> v = unpack_views(env, nViews, models, handles, blend, windows);
    std::vector<jint> np((size_t)nViews, 0);
    if (nViews > 0) env->GetIntArrayRegion(nPoints, 0, nViews, np.data());
    std::vector<jdouble> t, l;
    std::vector<bs_nonrigid_view> nv = unpack_nonrigid(env, nViews, v, np, targets, locals, t, l);
    const jsize n = env->GetArrayLength(dests);
    std::vector<jlong> mnj((size_t)n * 3), szj((size_t)n * 3);
    env->GetLongArrayRegion(blockMins, 0, n * 3, mnj.data());
    env->GetLongArrayRegion(blockSizes, 0, n * 3, szj.data());
    std::vector<long long> mn(mnj.begin(), mnj.end()), sz(szj.begin(), szj.end());
    std::vector<void*> outs((size_t)n);
    for (jsize i = 0; i < n; ++i) outs[(size_t)i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(dests, i));
    long long cpd[3];
    get3(env, cpDistance, cpd);
    const bs_fuse_params p = fuse_params(env, iparams, dparams);
    failed(env, ctx, bs_nonrigid_fuse_blocks(C(ctx), nv.data(), nViews, n, mn.data(), sz.data(), cpd, &p, outs.data(), 0));
}

// one view: the mapped source coordinate of every control point, double[gz][gy][gx][3]; gridDims (long[3]) receives
// {gx, gy, gz}
JF(jdoubleArray, nonrigidDebugGrid)(JNIEnv* env, jclass, jlong ctx, jdoubleArray model, jint nPoints, jdoubleArray targets,
                                    jdoubleArray locals, jlongArray blockMin, jlongArray blockSize, jlongArray cpDistance,
                                    jlongArray gridDims) {
    std::vector<bs_view> v = unpack_views(env, 1, model, nullptr, nullptr, nullptr);
    std::vector<jdouble> t, l;
    std::vector<bs_nonrigid_view> nv = unpack_nonrigid(env, 1, v, std::vector<jint>(1, nPoints), targets, locals, t, l);
    long long mn[3], sz[3], cpd[3], gd[3];
    get3(env, blockMin, mn);
    get3(env, blockSize, sz);
    get3(env, cpDistance, cpd);
    if (failed(env, ctx, bs_nonrigid_debug_grid(C(ctx), nv.data(), mn, sz, cpd, nullptr, gd))) return nullptr;
    std::vector<jdouble> out((size_t)gd[0] * gd[1] * gd[2] * 3);
    if (failed(env, ctx, bs_nonrigid_debug_grid(C(ctx), nv.data(), mn, sz, cpd, out.data(), gd))) return nullptr;
    jlong g[3] = {gd[0], gd[1], gd[2]};
    env->SetLongArrayRegion(gridDims, 0, 3, g);
    jdoubleArray r = env->NewDoubleArray((jsize)out.size());
    env->SetDoubleArrayRegion(r, 0, (jsize)out.size(), out.data());
    return r;
}

// ---------------------------------------------------------------------------------------- match-interestpoints
// the two quadratic steps of RGLDMPairwise (J/SparkGeometricDescriptorMatching.java:594-605); xyz: double[3n] world
// coordinates {x, y, z} per point
JF(jlong, descriptorsBuild)(JNIEnv* env, jclass, jlong ctx, jdoubleArray xyz, jint numNeighbors, jint redundancy) {
    const jint n = env->GetArrayLength(xyz) / 3;
    std::vector<jdouble> p((size_t)n * 3);
    if (n > 0) env->GetDoubleArrayRegion(xyz, 0, n * 3, p.data());
    unsigned long long h = 0;
    return failed(env, ctx, bs_descriptors_build(C(ctx), p.data(), n, numNeighbors, redundancy, &h)) ? 0 : (jlong)h;
}

JF(void, descriptorsFree)(JNIEnv* env, jclass, jlong ctx, jlong handle) {
    failed(env, ctx, bs_descriptors_free(C(ctx), (unsigned long long)handle));
}

// idx: long[n * k], d2: double[n * k] (k = numNeighbors + redundancy of the set)
JF(void, descriptorsNeighbors)(JNIEnv* env, jclass, jlong ctx, jlong handle, jlongArray idx, jdoubleArray d2) {
    const jsize m = env->GetArrayLength(idx);
    std::vector<int> i((size_t)m);
    std::vector<jdouble> d((size_t)m);
    if (failed(env, ctx, bs_descriptors_neighbors(C(ctx), (unsigned long long)handle, i.data(), d.data()))) return;
    const std::vector<jlong> il(i.begin(), i.end());
    env->SetLongArrayRegion(idx, 0, m, il.data());
    env->SetDoubleArrayRegion(d2, 0, m, d.data());
}

// per point of A: bestB long[nA], best / second double[nA]; searchRadius < 0: unlimited
JF(void, descriptorsMatch)(JNIEnv* env, jclass, jlong ctx, jlong ha, jlong hb, jdouble searchRadius, jlongArray bestB,
                           jdoubleArray best, jdoubleArray second) {
    const jsize n = env->GetArrayLength(bestB);
    std::vector<int> bi((size_t)n);
    std::vector<jdouble> b((size_t)n), s((size_t)n);
    if (failed(env, ctx, bs_descriptors_match(C(ctx), (unsigned long long)ha, (unsigned long long)hb, searchRadius, bi.data(),
                                              b.data(), s.data())))
        return;
    const std::vector<jlong> bl(bi.begin(), bi.end());
    env->SetLongArrayRegion(bestB, 0, n, bl.data());
    env->SetDoubleArrayRegion(best, 0, n, b.data());
    env->SetDoubleArrayRegion(second, 0, n, s.data());
}

// ---------------------------------------------------------------------------------------------------------------- solver
// the relaxation of the global optimisation (J/Solver.java:352-395): iparams = {transformation, regularization,
// maxIterations, maxPlateauwidth} (BS_MODEL_*), dparams = {lambda, maxError}; links int[2 * nLinks], matchOffsets
// long[nLinks + 1], p / q double[3 * nMatches], w double[nMatches]; models double[12 * nTiles] in and out; returns
// {iterations, stopped, skippedFits, error}
JF(jdoubleArray, solveTiles)(JNIEnv* env, jclass, jlong ctx, jintArray colourOffsets, jintArray colourTiles, jintArray fixed,
                             jintArray links, jlongArray matchOffsets, jdoubleArray p, jdoubleArray q, jdoubleArray w,
                             jintArray iparams, jdoubleArray dparams, jdoubleArray models, jdoubleArray tileError,
                             jdoubleArray linkMean, jdoubleArray linkMax) {
    auto ints = [&](jintArray a) {
        std::vector<jint> v((size_t)env->GetArrayLength(a));
        if (!v.empty()) env->GetIntArrayRegion(a, 0, (jsize)v.size(), v.data());
        return std::vector<int>(v.begin(), v.end());
    };
    auto dbls = [&](jdoubleArray a) {
        std::vector<jdouble> v((size_t)env->GetArrayLength(a));
        if (!v.empty()) env->GetDoubleArrayRegion(a, 0, (jsize)v.size(), v.data());
        return v;
    };
    const std::vector<int> co = ints(colourOffsets), ct = ints(colourTiles), fx = ints(fixed), lk = ints(links), ip = ints(iparams);
    std::vector<jlong> mo((size_t)env->GetArrayLength(matchOffsets));
    if (!mo.empty()) env->GetLongArrayRegion(matchOffsets, 0, (jsize)mo.size(), mo.data());
    const std::vector<long long> moff(mo.begin(), mo.end());
    const std::vector<jdouble> pp = dbls(p), qq = dbls(q), ww = dbls(w), dp = dbls(dparams);
    std::vector<jdouble> m = dbls(models);
    const int n_tiles = (int)ct.size(), n_links = (int)lk.size() / 2;
    std::vector<jdouble> te((size_t)n_tiles), lm((size_t)n_links + 1), lx((size_t)n_links + 1);
    bs_solve_params prm;
    prm.transformation = ip[0]; prm.regularization = ip[1]; prm.max_iterations = ip[2]; prm.max_plateau_width = ip[3];
    prm.lambda = dp[0]; prm.max_error = dp[1];
    bs_solve_stats st;
    if (failed(env, ctx, bs_solve_tiles(C(ctx), n_tiles, (int)co.size() - 1, co.data(), ct.data(), fx.data(), n_links, lk.data(),
                                        moff.data(), pp.data(), qq.data(), ww.data(), &prm, m.data(), &st, te.data(), lm.data(),
                                        lx.data())))
        return nullptr;
    env->SetDoubleArrayRegion(models, 0, (jsize)m.size(), m.data());
    env->SetDoubleArrayRegion(tileError, 0, n_tiles, te.data());
    env->SetDoubleArrayRegion(linkMean, 0, n_links, lm.data());
    env->SetDoubleArrayRegion(linkMax, 0, n_links, lx.data());
    const jdouble out[4] = {(jdouble)st.iterations, (jdouble)st.stopped, (jdouble)st.skipped_fits, st.error};
    jdoubleArray r = env->NewDoubleArray(4);
    env->SetDoubleArrayRegion(r, 0, 4, out);
    return r;
}
