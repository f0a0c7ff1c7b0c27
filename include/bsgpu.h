/*
 * bsgpu.h -- flat C ABI of libbsgpu.so: H100 (sm_90a) implementation of the two hot
 * paths of JaneliaSciComp/BigStitcher-Spark.
 *
 * Reference call sites each entry point replaces (paths relative to the reference root,
 * J/ = src/main/java/net/preibisch/bigstitcher/spark/):
 *
 *   bs_pcm_*   <-  TransformationTools.computeStitching(...)  J/SparkPairwiseStitching.java:247-255
 *                  (inner numeric cut: PairwiseStitching.getShift -> PhaseCorrelation2.calculatePCM
 *                   + PhaseCorrelation2.getShift, BigStitcher 2.5.0, pom.xml:107);
 *                  parameters: PairwiseStitchingParameters J/SparkPairwiseStitching.java:200-202;
 *                  found == 0  <=>  Java `null` ("No shift found", :274-279).
 *   bs_fuse_*  <-  BlkAffineFusion.initWithIntensityCoefficients(...)  J/SparkAffineFusion.java:602-615
 *                  + BlockAlgoUtils.arrayImg(blockSupplier, interval)   J/SparkAffineFusion.java:620-627
 *                  (multiview-reconstruction 8.0.0 / imglib2-algorithm 0.18.2, pom.xml:101,106);
 *                  dtype converters J/SparkAffineFusion.java:493-517.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; bs_last_error(ctx) gives the text.
 *     No exception crosses the boundary.  There is NO CPU fallback: without a CUDA device
 *     bs_init fails with BS_ERR_CUDA.
 *   - volumes are dense, x-fastest (imglib2 flat order), zero-min; dims are {x, y, z}.
 *   - the caller owns every host buffer; the library owns device memory it allocates.
 *   - a bs_ctx is bound to one device and one compute stream; calls on the same ctx are
 *     serialised by an internal mutex, different ctxs are independent (one per Java worker
 *     thread or one per device; the Spark RDD collapses to a host work queue over ctxs).
 */
#ifndef BSGPU_H
#define BSGPU_H

#ifdef __cplusplus
extern "C" {
#endif

#define BS_OK            0
#define BS_ERR_ARG      -1   /* invalid argument */
#define BS_ERR_CUDA     -2   /* CUDA runtime error / no device */
#define BS_ERR_NOMEM    -3   /* device or host allocation failed */
#define BS_ERR_UNSUPPORTED -4

#define BS_DTYPE_U16 0
#define BS_DTYPE_F32 1
#define BS_DTYPE_U8  2

/* FusionType ordinals (mvrecon FusionGUI.FusionType; CLI help J/SparkAffineFusion.java:124-125) */
#define BS_FUSE_AVG                 0
#define BS_FUSE_AVG_BLEND           1   /* reference default */
#define BS_FUSE_AVG_CONTENT         2
#define BS_FUSE_AVG_BLEND_CONTENT   3
#define BS_FUSE_MAX_INTENSITY       4
#define BS_FUSE_LOWEST_VIEWID_WINS  5
#define BS_FUSE_HIGHEST_VIEWID_WINS 6
#define BS_FUSE_CLOSEST_PIXEL_WINS  7

typedef struct bs_ctx bs_ctx;

/* ---------------------------------------------------------------- lifecycle */
int bs_version(void);
/* device: CUDA ordinal.  stream: an existing cudaStream_t to launch on (e.g. the caller's
 * framework stream), or NULL to let the context create its own non-blocking stream. */
int bs_init(bs_ctx** out, int device, void* stream);
void bs_destroy(bs_ctx* ctx);
const char* bs_last_error(bs_ctx* ctx);   /* ctx may be NULL: last bs_init error of this thread */
int bs_synchronize(bs_ctx* ctx);
/* number of kernels this context has launched since creation (bench.py's gpu_launches) */
long long bs_launch_count(bs_ctx* ctx);

/* per-kernel device timing with CUDA events on the context's stream.  Enabling inserts an
 * event pair around every kernel launch; bs_profile_get returns the accumulated milliseconds
 * and launch count for a kernel tag ("fft_x_r2c", "fft_y", "fft_z_xpower", "fft_y_inv",
 * "fft_x_c2r", "peaks", "pearson", "fuse", "content_gauss", "downsample", "median", "sample", "mls_grid",
 * "nonrigid_fuse"). */
int bs_profile_enable(bs_ctx* ctx, int on);
int bs_profile_reset(bs_ctx* ctx);
int bs_profile_get(bs_ctx* ctx, const char* tag, double* ms_total, long long* launches);

/* pinned host memory helpers (the JNI side wraps them in direct ByteBuffers) */
int bs_host_alloc(bs_ctx* ctx, unsigned long long bytes, void** out);
int bs_host_free(bs_ctx* ctx, void* p);

/* ---------------------------------------------------------------- hot path 1: phase correlation */
typedef struct {
    int    peaks_to_check;      /* --peaksToCheck, default 5 (J/SparkPairwiseStitching.java:79-80) */
    int    do_subpixel;         /* !--disableSubpixelResolution (J/SparkPairwiseStitching.java:82-83) */
    int    interpolate_xcorr;   /* PairwiseStitchingParameters.interpolateCrossCorrelation; must be 0 */
    double min_overlap_frac;    /* PairwiseStitchingParameters.minOverlap, default 0.25 */
    int    extension[3];        /* blended-mirror extension in px, upstream fills 10 */
} bs_pcm_params;

typedef struct {
    int       found;            /* 0 <=> Java null */
    long long shift_int[3];     /* integer shift s: img1[p + s] <-> img2[p], {x,y,z} */
    double    shift_sub[3];     /* s + sub-pixel offset (== s when !do_subpixel) */
    double    r;                /* Pearson cross-correlation of the winning candidate */
    long long n_overlap_px;     /* its overlap voxel count */
    long long peak_index[3];    /* PCM index of the winning peak */
    double    pcm_value;        /* PCM value of that peak */
    int       pad[3];           /* padded FFT size used */
    int       n_candidates;     /* Pearson-verified candidates (>= min overlap) */
    long long pearson_px;       /* sum of their overlap voxel counts (byte accounting) */
} bs_pcm_result;

void bs_pcm_default_params(bs_pcm_params* p);

/* one overlap-cropped pair, equal dims (PairwiseStitching.getShift returns null otherwise).
 * on_device != 0: img1/img2 are device pointers on ctx's device (resident data);
 * on_device == 0: host pointers, copied H2D inside the call. */
int bs_pcm_pair(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3],
                int dtype, const bs_pcm_params* params, int on_device, bs_pcm_result* out);

/* n pairs (all with their own dims[n][3]); host inputs are staged through a double-buffered
 * H2D pipeline on a second stream so copies overlap the previous pair's kernels. */
int bs_pcm_batch(bs_ctx* ctx, int n, const void* const* img1, const void* const* img2,
                 const long long* dims /* n*3 */, int dtype, const bs_pcm_params* params,
                 int on_device, bs_pcm_result* out /* n */);

/* Pairs given as resident volumes plus the raster overlap intervals PairwiseStitching.getShift derives from the
 * two translations (BigStitcher 2.5.0; call site J/SparkPairwiseStitching.java:247-255): a tile is uploaded ONCE
 * (bs_volume_upload[_async]) and takes part in up to 26 pairs; the overlap crops are cut on the device. */
typedef struct {
    unsigned long long vol1, vol2;   /* resident volumes (same dtype) */
    long long min1[3], min2[3];      /* first voxel of the overlap in each volume's own pixel coordinates */
    long long dims[3];               /* overlap size (equal for both; getShift returns null otherwise) */
} bs_pcm_job;
int bs_pcm_volumes_batch(bs_ctx* ctx, int n, const bs_pcm_job* jobs, const bs_pcm_params* params, bs_pcm_result* out);

/* padded FFT length policy of this build (smallest 2^a3^b5^c >= n; even when even != 0) */
int bs_good_fft_size(int n, int even);

/* diagnostic: compute only the PCM of one pair into a host float buffer of pad[0]*pad[1]*pad[2]
 * elements (x-fastest); used by the parity tests to compare spectra-level results. */
int bs_pcm_debug_pcm(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3],
                     int dtype, const int extension[3], float* out_pcm, int pad_out[3]);

/* diagnostic: ONE pass of the PCM's FFT pipeline, with exactly the launch bs_pcm_* uses, on explicit inputs.
 * Geometry as in bs_pcm_debug_pcm: P = padded dims {x,y,z}, M = P[0] / 2.  A "spectrum" is a host complex64 array
 * [P[2]][P[1]][M+1] (x fastest; interleaved re, im float32).  All transforms are unnormalised forward DFTs
 * F(v)[k] = sum_n v[n] exp(-2 pi i k n / N) along one axis:
 *   pass 0  x R2C.   in_a / in_b: DEVICE pointers to the two crops (dims {x,y,z}, dtype); each is blended-mirror
 *                    extended and zero padded to P (oracle/pcm_oracle.py blend_extend_pad), then out = rfft along x.
 *                    out_a / out_b: the two spectra.
 *   pass 1  y.       in_a / in_b: two spectra; out = F_y(in) for each.
 *   pass 2  z cross-power.  in_a = A, in_b = B: out_a = F_z(conj(n(F_z A)) * n(F_z B)), n(c) = c / |c|, or 0 when
 *                    |c| < 1e-5.
 *   pass 3  y.       in_a: one spectrum; out_a = F_y(in_a).
 *   pass 4  x C2R.   in_a: one spectrum H; out_a: float32 [P[2]][P[1]][P[0]] with, per line,
 *                    out = irfft(conj(H), P[0]) / (P[1] P[2])   (numpy's irfft, 1 / P[0] normalised; the kernel
 *                    scales its half-length transform by 1 / (M P[1] P[2])).  As in any C2R the imaginary parts of
 *                    bins 0 and M are expected to be 0.
 *   pass 5  x R2C + y.   As pass 1 after pass 0, from the same inputs to the same outputs, as the pipeline runs the
 *                    two (one fused kernel, k_fft_xy_col540, where it applies; the two passes otherwise).
 * The conjugations make passes 3 and 4 the inverse transforms: pass4(pass3(pass2(pass1(pass0(a, b))))) is the PCM
 * irfftn(n(rfftn A) conj(n(rfftn B))) of bs_pcm_debug_pcm.
 * BS_ERR_ARG when the crops of passes 0 and 5 are not device memory.
 * in_b / out_b are ignored (may be NULL) for passes 3 and 4, out_b also for pass 2.  poison != 0 fills the device
 * spectra with NaN bytes first, so anything a pass fails to write shows up as NaN.  info (may be NULL) receives the
 * kernel instantiation launched, and for runtime-planned kernels the radices of the plan, e.g.
 * "k_fft_strided_pipe 15x12x3" (NUL-terminated, at most 128 bytes). */
int bs_pcm_debug_pass(bs_ctx* ctx, int pass, const long long dims[3], int dtype, const int extension[3],
                      const void* in_a, const void* in_b, void* out_a, void* out_b, int poison, int pad_out[3],
                      char info[128]);

/* diagnostic: the Pearson sums of an explicit candidate list, computed by the same launch bs_pcm_* uses.
 * img1/img2: DEVICE pointers to two crops of dims {x,y,z}.  boxes: n * 9 ints per candidate, {o1[3], o2[3], sz[3]}
 * ({x,y,z} each): voxel o1 + p of img1 pairs with o2 + p of img2 for 0 <= p < sz; n <= 256.  sums_out: n * 5 values
 * {sum a, sum b, sum a^2, sum b^2, sum ab}, uint64 for U16 / U8 and float64 for F32. */
int bs_pcm_debug_pearson(bs_ctx* ctx, const void* img1, const void* img2, const long long dims[3], int dtype, int n,
                         const int* boxes, void* sums_out);

/* ---------------------------------------------------------------- hot path 2: affine fusion */
typedef struct {
    double             src_to_world[12]; /* row-packed 3x4: source pixel -> world, i.e. the adjusted
                                            registration (TransformVirtual.adjustAllTransforms,
                                            J/SparkAffineFusion.java:486-491) times the mipmap transform
                                            (J/util/ViewUtil.java:232-234); inverted by the library */
    unsigned long long vol_handle;       /* resident source volume (bs_volume_upload/_wrap) */
    unsigned long long content_handle;   /* content-weight volume (bs_content_weights) or 0 */
    float              blend_border[3];  /* source px, after FusionTools.adjustBlending */
    float              blend_range[3];
    /* Windowed source (block-wise staging, J/fusion/OverlappingBlocks.java:133-161 / J/util/ViewUtil.java:210-371:
     * only the source cells a block touches are loaded): when full_dims[0] > 0 the resident volume holds the
     * sub-interval [window_min, window_min + volume dims) of a view whose real size is full_dims; src_to_world
     * still maps FULL-view pixel coordinates, the inside test and the blending weights use full_dims, taps are
     * fetched relative to window_min.  The caller guarantees the window covers every tap with non-zero weight
     * (taps outside read zero).  All zeros = the volume is the whole view. */
    long long          full_dims[3];
    long long          window_min[3];
} bs_view;

typedef struct {
    int    fusion_type;     /* BS_FUSE_* */
    int    interpolation;   /* 0 nearest neighbour, 1 n-linear (the reference passes 1) */
    int    out_dtype;       /* BS_DTYPE_F32 / U16 / U8 (J/SparkAffineFusion.java:493-517) */
    int    blend_lut_n;     /* 0: analytic cosine; n>0: n-segment linear-interpolated cosine table */
    double min_intensity;   /* converter range for integer outputs */
    double max_intensity;
    int    out_big_endian;  /* 1: 2- and 4-byte output elements leave the device byte-swapped, i.e. as the big-endian
                             * payload of an N5 block (DefaultBlockWriter), so the host writes the bytes as they come */
    int    reserved;
} bs_fuse_params;

void bs_fuse_default_params(bs_fuse_params* p);

int bs_volume_upload(bs_ctx* ctx, const void* host, const long long dims[3], int dtype,
                     unsigned long long* handle);
/* same, but asynchronous: `host` must be pinned (bs_host_alloc) and stay valid until the copy has run; the copy is
 * queued on the context's copy stream and every later call that uses the handle waits for it on the device, so
 * tile uploads overlap the kernels of earlier work (no host synchronisation).  Device buffers of volumes created
 * this way are recycled through a per-context pool by bs_volume_free. */
int bs_volume_upload_async(bs_ctx* ctx, const void* host, const long long dims[3], int dtype,
                           unsigned long long* handle);
/* register device memory owned by the caller (not freed by bs_volume_free) */
int bs_volume_wrap(bs_ctx* ctx, const void* dev, const long long dims[3], int dtype,
                   unsigned long long* handle);
int bs_volume_free(bs_ctx* ctx, unsigned long long handle);
/* c = G_sigma2 * (I - G_sigma1 * I)^2 on the source volume -> new float32 volume handle */
int bs_content_weights(bs_ctx* ctx, unsigned long long vol_handle, double sigma1, double sigma2,
                       unsigned long long* content_handle);
/* dims {x,y,z} and dtype of a resident volume (either may be NULL) */
int bs_volume_info(bs_ctx* ctx, unsigned long long handle, long long dims[3], int* dtype);
/* copies the whole volume to `host`; capacity_bytes is the size of the caller's buffer and must be at least the
 * volume's byte size (no silent overflow) */
int bs_volume_download(bs_ctx* ctx, unsigned long long handle, void* host, unsigned long long capacity_bytes);
/* next row 8f-3: one 2x half-pixel averaging pyramid step on a resident volume (factors 1 or 2 per
 * axis, output dims = floor(dims / factors), same dtype) -> new handle.  Replaces re-reading level
 * l-1 from the container for every pyramid level (J/SparkAffineFusion.java:703-782). */
int bs_downsample(bs_ctx* ctx, unsigned long long vol_handle, const int factors[3],
                  unsigned long long* out_handle);
/* device address of a resident volume, so that a second context on the same device (another worker
 * thread) can bs_volume_wrap it instead of uploading the tile twice */
int bs_volume_devptr(bs_ctx* ctx, unsigned long long handle, void** dev);

/* fuse one output block: voxel (i,j,k) is at world block_min + (i,j,k)
 * (block_min = gridBlock[0] + bbMin, J/SparkAffineFusion.java:520-534).  views must be in
 * ascending ViewId order.  out: block_size[0]*[1]*[2] elements of out_dtype, x-fastest;
 * out_on_device selects a device or host destination. */
int bs_fuse_block(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                  const long long block_size[3], const bs_fuse_params* params,
                  void* out, int out_on_device);

/* the same for a LIST of blocks in one call (one plan pass, one kernel launch for the whole list; host
 * destinations are staged through two device buffers so the D2H copies of one group of blocks overlap the
 * fusion of the next).  block_min / block_size: n_blocks x 3; outs: n_blocks destination pointers, each a
 * dense x-fastest block like bs_fuse_block's.  This is the work-queue form of the reference's
 * rdd.map(gridBlock -> fuse + save) (J/SparkAffineFusion.java:480-482, 602-670). */
int bs_fuse_blocks(bs_ctx* ctx, const bs_view* views, int n_views, int n_blocks, const long long* block_min,
                   const long long* block_size, const bs_fuse_params* params, void* const* outs, int out_on_device);

/* same, but the fused block stays on the device as a new resident volume (handle): the pyramid
 * levels are then derived with bs_downsample before anything is downloaded (next row 8f-3) */
int bs_fuse_block_to_volume(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                            const long long block_size[3], const bs_fuse_params* params,
                            unsigned long long* out_handle);

/* `affine-fusion --masks [--maskOffset x,y,z]` (J/fusion/GenerateComputeBlockMasks.java:84-176, called at
 * J/SparkAffineFusion.java:564-578): instead of fusing, every block voxel becomes "on" (255 / 65535 / 1.0f for
 * U8 / U16 / F32) when its back-projection into ANY view lies inside [0 - mask_offset, dim - 1 + mask_offset]
 * (source pixels, all three axes).  Only view geometry is used: src_to_world and full_dims (or, when full_dims is 0,
 * the dims of vol_handle).  Same block-list form and output conventions as bs_fuse_blocks. */
int bs_mask_blocks(bs_ctx* ctx, const bs_view* views, int n_views, int n_blocks, const long long* block_min,
                   const long long* block_size, const double mask_offset[3], int out_dtype, int out_big_endian,
                   void* const* outs, int out_on_device);

/* view-sharded mode (SURVEY 8e): accumulate this context's views into partial sums
 * sum_wi / sum_w (device float32, block_size elements each, NOT cleared), to be all-reduced
 * across devices by the caller (NCCL) and finished with bs_fuse_finish. */
int bs_fuse_accumulate(bs_ctx* ctx, const bs_view* views, int n_views, const long long block_min[3],
                       const long long block_size[3], const bs_fuse_params* params,
                       float* sum_wi_dev, float* sum_w_dev);
int bs_fuse_finish(bs_ctx* ctx, const float* sum_wi_dev, const float* sum_w_dev, long long n,
                   const bs_fuse_params* params, void* out, int out_on_device);
/* The exchange itself, inside the library: rank 0 draws a 128-byte NCCL id (bs_comm_unique_id) and hands it to the
 * other ranks by any host channel (the Spark driver / torch.distributed store); every rank joins with bs_comm_init;
 * bs_fuse_allreduce sums both partial buffers of the (overlap) region over all ranks in place -- one grouped NCCL
 * all-reduce over NVLink / NVSwitch, queued on the context's stream between bs_fuse_accumulate and bs_fuse_finish. */
int bs_comm_unique_id(unsigned char id[128]);
int bs_comm_init(bs_ctx* ctx, int n_ranks, int rank, const unsigned char id[128]);
int bs_comm_destroy(bs_ctx* ctx);
int bs_fuse_allreduce(bs_ctx* ctx, float* sum_wi_dev, float* sum_w_dev, long long n);

/* ---------------------------------------------------------------- next row: DoG interest points
 * DoGImgLib2.computeDoG on one block of a resident view (J/SparkInterestPointDetection.java:469-566; the reference
 * passes dog.cuda = null at :490-493 -- this is the device implementation behind that hook).  The caller walks the
 * reference's block grid and expands every block by one voxel inside the image (:397-424). */
typedef struct {
    double sigma;           /* -s, e.g. 1.8 */
    double threshold;       /* -t, e.g. 0.008 */
    double min_intensity;   /* -i0 */
    double max_intensity;   /* -i1 */
    int    find_max;        /* --type MAX / BOTH */
    int    find_min;        /* --type MIN / BOTH */
    int    localization;    /* 0 NONE, 1 QUADRATIC */
    int    pad;
} bs_dog_params;

typedef struct {
    double    loc[3];       /* sub-pixel location {x,y,z} in the view's pixel coordinates */
    double    value;        /* (interpolated) DoG value */
    long long voxel[3];     /* integer location of the extremum */
    int       is_max;
    int       pad;
} bs_dog_point;

void bs_dog_default_params(bs_dog_params* p);
/* detections of the block [interval_min, interval_min + interval_size) sorted by (z, y, x); *n_found may exceed
 * max_points (buffer too small: only max_points were written) */
int bs_dog_detect(bs_ctx* ctx, unsigned long long vol_handle, const long long interval_min[3], const long long interval_size[3],
                  const bs_dog_params* params, bs_dog_point* out, int max_points, int* n_found);

/* diagnostic: the DoG (G_sa * I' - G_sb * I') / (k - 1) that bs_dog_detect's extremum stage reads for this interval,
 * i.e. over [interval_min - 1, interval_min + interval_size + 1) per axis (mirror-double extension outside the image),
 * computed by the same load / blur launches.  out: host float32, (size + 2) per axis, x fastest.
 * blur: 0 = the production choice, 1 = generic k_dog_blur, 2 = window R 6, 3 = window R 12
 * (BS_ERR_ARG when the kernel radius does not fit the forced window).
 * info (may be NULL): the blur instantiation launched and the radii, e.g. "k_dog_blur_x<12> ra=6 rb=7". */
int bs_dog_debug_dog(bs_ctx* ctx, unsigned long long vol_handle, const long long interval_min[3],
                     const long long interval_size[3], const bs_dog_params* params, int blur, float* out, char info[128]);

/* ---------------------------------------------------------------- detect-interestpoints helpers (ABI 106)
 * The per-view steps SparkInterestPointDetection.call() runs around computeDoG (J/SparkInterestPointDetection.java:
 * 532-604, openAndDownsample :991-1111).  Each returns a NEW resident volume (free it with bs_volume_free) or host
 * values; the input volume is unchanged. */

/* the remaining downsampling after the mipmap level (J/SparkInterestPointDetection.java:1085-1095): LazyDownsample2x to
 * FloatType, first every x halving, then every y, then every z, each out[i] = 0.5f * (in[2i] + in[2i+1]) with
 * floor(d / 2) output dims.  vol: U16, U8 or F32; factors: powers of two <= 128 per axis (all 1: a float copy);
 * out: F32.  BS_ERR_ARG when an axis would shrink to 0. */
int bs_downsample_float(bs_ctx* ctx, unsigned long long vol_handle, const int factors[3], unsigned long long* out_handle);

/* --medianFilter r (LazyBackgroundSubtract, J/detection/LazyBackgroundSubtract.java:74-140, applied at
 * J/SparkInterestPointDetection.java:532-547): per z-slice, m = the exact median of the values under ImageJ's circular
 * RankFilters kernel of radius r (r2 = r*r + 1, row dy spans |dx| <= floor(sqrt(r2 - dy*dy + 1e-10)), an odd number of
 * points) over the slice's mirror-double extension; out = v / m when m > 0, else 0, in float32.  vol: U16, U8 or F32;
 * out: F32, same dims.  1 <= radius <= BS_MEDIAN_MAX_RADIUS, else BS_ERR_ARG.  Profile tag "median". */
#define BS_MEDIAN_MAX_RADIUS 32
int bs_median_divide(bs_ctx* ctx, unsigned long long vol_handle, int radius, unsigned long long* out_handle);

/* --storeIntensities / --maxSpots (J/SparkInterestPointDetection.java:577-604): n-linear interpolation of the resident
 * volume (converted to float) on its border extension at n host points loc_xyz[3n] (pixel coordinates {x,y,z}), like
 * imglib2's NLinearInterpolator on FloatType: double weights, each corner term rounded to float and summed in float.
 * out: n floats on the host.  Profile tag "sample". */
int bs_sample_nlinear(bs_ctx* ctx, unsigned long long vol_handle, int n, const double* loc_xyz, float* out);

/* ---------------------------------------------------------------- nonrigid-fusion (ABI 107)
 * NonRigidTools.fuseVirtualInterpolatedNonRigid on one super-block (J/SparkNonRigidFusion.java:387-401): per view a
 * moving-least-squares affine model from target WORLD to local PIXEL coordinates, weights w_i = 1 / |x - t_i|^2
 * (alpha = 1), evaluated in double at the control points block_min + (k - 1) * cp_distance, k = 0 .. grid_dims - 1,
 * grid_dims[d] = ceil((block_size[d] - 1) / cp_distance[d]) + 3 (the block plus one cell on every side).  A control
 * point on a target returns its local point; a view with fewer than 4 points, or a singular fit
 * (det P <= 1e-10 (trace P / 3)^3 for the weighted, centred second moments P of the targets), uses the inverse of
 * src_to_world.  Every output voxel trilinearly interpolates the mapped source coordinate of its 8 surrounding control
 * points, samples the view n-linearly (border extension), weights it with the cosine blending of the view's
 * blend_border / blend_range at that coordinate and is sum(w I) / sum(w) over the views (0 where sum(w) = 0): AVG_BLEND
 * with n-linear interpolation only.  Profile tags "mls_grid" and "nonrigid_fuse". */
typedef struct {
    bs_view view;                      /* src_to_world: the full-resolution registration; windows as in bs_fuse_blocks */
    int n_points;
    int pad;
    const double* target_world_xyz;    /* n_points x 3: corresponding-point targets, world coordinates */
    const double* local_xyz;           /* n_points x 3: the same points in the view's full-resolution pixels */
} bs_nonrigid_view;

/* same block-list form and output conventions as bs_fuse_blocks (out_big_endian included); views in ascending ViewId
 * order.  BS_ERR_ARG for a fusion_type other than AVG_BLEND, interpolation != 1 or a cp_distance < 1. */
int bs_nonrigid_fuse_blocks(bs_ctx* ctx, const bs_nonrigid_view* views, int n_views, int n_blocks,
                            const long long* block_min, const long long* block_size, const long long cp_distance[3],
                            const bs_fuse_params* params, void* const* outs, int out_on_device);

/* diagnostic: the mapped source coordinate of every control point of one view for one block, host float64
 * [grid_dims z][y][x][3] ({x, y, z} last), computed by the launch bs_nonrigid_fuse_blocks uses.  grid_dims receives
 * {gx, gy, gz}; out may be NULL to query the dims.  The view's vol_handle is not used. */
int bs_nonrigid_debug_grid(bs_ctx* ctx, const bs_nonrigid_view* view, const long long block_min[3],
                           const long long block_size[3], const long long cp_distance[3], double* out, long long* grid_dims);

/* ---------------------------------------------------------------- match-interestpoints
 * The two quadratic steps of PRECISE_TRANSLATION matching, RGLDMPairwise (J/SparkGeometricDescriptorMatching.java:594-605):
 * the local descriptors of each point set and the exhaustive descriptor search from A to B, both in FP64.  The ratio test,
 * RANSAC and the model fits stay on the host.  These entry points are additive: the ABI version stays 107. */
#define BS_MATCH_MAX_NEIGHBORS 6   /* num_neighbors + redundancy */

/* resident local descriptors of one point set (world coordinates, n x 3 doubles {x,y,z}): for every point p its
 * k = num_neighbors + redundancy nearest OTHER points, ordered by (squared distance, index), kept as the relative
 * vectors q_j - p in double.  3 <= num_neighbors, 0 <= redundancy, k <= BS_MATCH_MAX_NEIGHBORS, else BS_ERR_ARG.
 * n <= k is legal: the set has no descriptors.  Profile tag "knn". */
int bs_descriptors_build(bs_ctx* ctx, const double* xyz, int n, int num_neighbors, int redundancy, unsigned long long* handle);
int bs_descriptors_free(bs_ctx* ctx, unsigned long long handle);
/* diagnostic: neighbour indices [n][k] and squared distances [n][k] of bs_descriptors_build (-1 / +inf when n <= k) */
int bs_descriptors_neighbors(bs_ctx* ctx, unsigned long long handle, int* idx, double* d2);
/* for every point a of A: over the points b of B (only |p_b - p_a| <= search_radius when search_radius >= 0),
 * D(a, b) = min over the C(k,n)^2 pairs of neighbour subsets (s of a, t of b) of sum_j |u_{s_j} - v_{t_j}|^2;
 * best_b = argmin (ties -> lower b), best = D(a, best_b), second = min over b != best_b (+inf when none);
 * best_b = -1 when no b qualifies.  A and B must share (num_neighbors, redundancy).  Subsets are taken in lexicographic
 * order of neighbour rank, each in ascending-distance order.  Profile tag "desc_match". */
int bs_descriptors_match(bs_ctx* ctx, unsigned long long ha, unsigned long long hb, double search_radius,
                         int* best_b, double* best, double* second);

/* ---------------------------------------------------------------- solver
 * The relaxation of the global optimisation (TileConfiguration.optimize behind J/Solver.java:352-395) in FP64: tiles
 * joined by links, each link a list of weighted point matches p (its first tile) <-> q (its second tile), world
 * coordinates.  Each iteration fits every non-fixed tile, colour by colour, to M_t(own point) ~ M_u(partner point) with
 * its partners' current models (a multicolour Gauss-Seidel sweep: no link may join two tiles of one colour), then takes
 * every match's distance d = |M_a p - M_b q|, each tile's error sum w d / sum w over its links' matches and
 * E = the mean tile error.  After iteration i > max_plateau_width it stops unless E_i > max_error or
 * |E_i - E_{i-d}| / d > 1e-4 for some d = max_plateau_width, max_plateau_width / 2, ... >= 1.  The model is
 * transformation, or (1 - lambda) transformation + lambda regularization; fits are weighted.  A tile with fewer matches
 * than the model needs, zero total weight, or a singular fit (AFFINE: det P <= 1e-12 (trace P / 3)^3; RIGID: second
 * invariant of P <= 1e-12 trace(P)^2, P the tile's centred weighted second moments) keeps its model and is counted in
 * skipped_fits.  Bit-identical between runs.  Additive: the ABI version stays 107.  Profile tags "solve_moments",
 * "solve". */
#define BS_MODEL_NONE        -1   /* regularization only */
#define BS_MODEL_IDENTITY     0   /* regularization only */
#define BS_MODEL_TRANSLATION  1
#define BS_MODEL_RIGID        2
#define BS_MODEL_AFFINE       3

typedef struct {
    int    transformation;      /* BS_MODEL_TRANSLATION / RIGID / AFFINE (-tm) */
    int    regularization;      /* BS_MODEL_NONE / IDENTITY / TRANSLATION / RIGID / AFFINE (-rm) */
    double lambda;              /* --lambda, in [0, 1] */
    double max_error;           /* --maxError; +inf stops on the plateau alone */
    int    max_iterations;      /* --maxIterations, >= 1 */
    int    max_plateau_width;   /* --maxPlateauwidth, >= 0 */
} bs_solve_params;

typedef struct {
    int       iterations;       /* iterations run */
    int       stopped;          /* 1: the stopping rule ended the solve; 0: max_iterations did */
    long long skipped_fits;     /* fits that kept the tile's model, summed over iterations */
    double    error;            /* E of the last iteration */
    int       blocks;           /* CTAs of the persistent solve kernel */
    int       models_in_shared; /* 1: the distance pass read the models from shared memory */
} bs_solve_stats;

/* n_tiles >= 1 tiles in n_colours colours: colour c holds tiles colour_tiles[colour_offsets[c] .. colour_offsets[c + 1]).
 * fixed[n_tiles]: non-zero tiles keep their model.  links[2 * n_links]: the two tiles of each link; the matches of link l
 * are rows match_offsets[l] .. match_offsets[l + 1] of p, q (3 doubles {x, y, z} each) and w (weights >= 0).
 * models[12 * n_tiles]: row-packed 3 x 4 models, the starting values in and the solution out.  tile_error[n_tiles] and,
 * per link, link_mean (sum w d / sum w) and link_max (max d) receive the values of the last iteration.  BS_ERR_ARG for a
 * bad colouring, link, count, parameter or a non-finite input. */
int bs_solve_tiles(bs_ctx* ctx, int n_tiles, int n_colours, const int* colour_offsets, const int* colour_tiles,
                   const int* fixed, int n_links, const int* links, const long long* match_offsets, const double* p,
                   const double* q, const double* w, const bs_solve_params* params, double* models,
                   bs_solve_stats* stats, double* tile_error, double* link_mean, double* link_max);

/* ---------------------------------------------------------------- intensity correction
 * match-intensities (IntensityCorrection.matchRansac, J/SparkIntensityMatching.java:166-183) and the coefficient
 * application of affine-fusion --intensityN5Path (J/SparkAffineFusion.java:602-615).  Additive: the ABI version stays
 * 107 (the existing structs and functions are unchanged).  Profile tags "intensity_render", "intensity_ransac",
 * "intensity_apply". */
typedef struct {
    unsigned long long vol_handle;   /* resident WHOLE level volume of the view (U16 / F32 / U8) */
    double    world_to_px[12];       /* row-packed 3x4: world -> full-resolution pixel (inverse registration) */
    double    px_to_level[12];       /* full-resolution pixel -> pixel of the level volume (inverse mipmap transform) */
    long long full_dims[3];          /* full-resolution view size */
    int       n_cells[3];            /* --numCoefficients */
    int       pad;
} bs_intensity_view;

typedef struct {
    double    render_scale;          /* --renderScale s */
    double    min_threshold;         /* --minThreshold */
    double    max_threshold;         /* --maxThreshold, NaN: none */
    long long render_min[3];         /* render grid: integers r with render_min <= r <= render_max, world r / s */
    long long render_max[3];
    long long chunk_points;          /* render points per z-chunk, 0: the library default (the output does not depend on it) */
} bs_intensity_params;

/* Candidates of one view pair, kept resident under *handle (free with bs_intensity_candidates_free).  Per render point,
 * in FP64 with __dmul_rn / __dadd_rn / __ddiv_rn: w = r / s per axis; p = world_to_px . (w, 1) per row as
 * ((m0 wx + m1 wy) + m2 wz) + m3; the point is kept when every p_d of both views is in [0, full_dims_d - 1]; level
 * coordinates q = px_to_level . (p, 1) (same order), rounded to float32; value = n-linear float32 sample at q with
 * border extension on both sides (the arithmetic of sample() in csrc/fuse_common.cuh, taps clamped to the volume);
 * kept when both values are >= min_threshold and, unless NaN, <= max_threshold; cell_d = clamp(floor(p_d n_d /
 * full_dims_d), 0, n_d - 1), flattened x-fastest; key = cellA * cells(B) + cellB.  Buckets are in ascending key order,
 * values (v_A, v_B) float32 pairs grouped by bucket and in ascending render index (x-fastest) within one.  No order
 * depends on atomics; the output is the same for every chunk_points. */
int bs_intensity_pair_candidates(bs_ctx* ctx, const bs_intensity_view* view_a, const bs_intensity_view* view_b,
                                 const bs_intensity_params* params, unsigned long long* handle, long long* n_buckets,
                                 long long* n_values);
/* host copies: keys / offsets / counts [n_buckets] (offsets into values, in pairs), values [2 n_values]; any may be NULL */
int bs_intensity_candidates_get(bs_ctx* ctx, unsigned long long handle, long long* keys, long long* offsets,
                                long long* counts, float* values);
int bs_intensity_candidates_free(bs_ctx* ctx, unsigned long long handle);

/* RANSAC hypotheses (the sampling loop of mpicbg Model.ransac behind IntensityCorrection.matchRansac) of every bucket
 * with at least max(2, min_num_candidates) candidates: hypothesis h = 0 .. num_iterations - 1 draws candidates
 * i = splitmix64(SEED ^ (key << 32) ^ 2h) mod n, j = splitmix64(SEED ^ (key << 32) ^ (2h + 1)) mod (n - 1), j += (j >= i),
 * SEED = 0x2545F4914F6CDD1D, and is skipped when x_i == x_j; its model a = (y_j - y_i) / (x_j - x_i),
 * b = y_i - a x_i counts the inliers |(a x + b) - y| < max_epsilon (FP64, those operations in that order).  Per bucket:
 * the hypothesis with the most inliers, the lower h on a tie, as (a, b, count); count 0 and a = b = NaN when every
 * hypothesis was skipped; count -1 for buckets below the threshold.  Outputs have n_buckets entries. */
int bs_intensity_ransac(bs_ctx* ctx, unsigned long long handle, long long min_num_candidates, int num_iterations,
                        double max_epsilon, double* a, double* b, int* count);

/* v' = a(q) v + b(q) on a resident volume (U16 / F32 / U8) -> new F32 volume handle.  The volume is the window
 * [window_min, window_min + dims) (window_min NULL: zeros) of the level of a view of full-resolution size full_dims;
 * level_to_full is the mipmap transform.  In float32 (inputs rounded to float): l = window_min + voxel;
 * q_d = ((m0 l_x + m1 l_y) + m2 l_z) + m3; u_d = clamp((q_d + 0.5) (n_d / full_dims_d) - 0.5, 0, n_d - 1) (cell
 * centres at (c + 0.5) full_dims / n - 0.5); a and b are the n-linear interpolation of the cell values coeff_a /
 * coeff_b (x-fastest, n cells) at u, in the lerp order of sample(); v' = (a v) + b. */
int bs_intensity_apply(bs_ctx* ctx, unsigned long long vol_handle, const long long full_dims[3], const long long window_min[3],
                       const double level_to_full[12], const int n_cells[3], const double* coeff_a, const double* coeff_b,
                       unsigned long long* out_handle);

/* ---------------------------------------------------------------- estimate-bounding-box
 * The filter and reductions of mvrecon's BoundingBoxMinFilterThreshold on a resident FLOAT32 volume (the downsampled
 * fusion).  Additive: the ABI version stays 107.  BS_ERR_ARG for an unknown handle, a volume that is not F32 or larger
 * than 2^31 - 1 x 2^31 - 1 x 65535, a negative radius and NULL outputs. */

/* out = the minimum over the box |q - p|_inf <= radius (per axis {x, y, z}), clipped to the volume (a mirror or border
 * extension gives the same minimum); a NaN neighbour is ignored as by fminf (NaN only when the whole box is NaN).
 * Computed as 1-D passes along x, then y, then z; min is exact, so the result is bit-identical to any evaluation order.
 * A radius of 0 leaves that axis as it is.  New F32 volume handle; needs two volume-sized device buffers while it runs.
 * Profile tag "min_filter". */
int bs_min_filter(bs_ctx* ctx, unsigned long long vol_handle, const int radius[3], unsigned long long* out_handle);
/* out = {min, max} over the voxels that are not NaN; both NaN when there are none.  Profile tag "min_max". */
int bs_volume_min_max(bs_ctx* ctx, unsigned long long vol_handle, double out[2]);
/* the voxels with (double)v > t: their count and the smallest / largest index per axis {x, y, z} (-1 and a count of 0
 * when there are none).  Profile tag "threshold_bbox". */
int bs_threshold_bbox(bs_ctx* ctx, unsigned long long vol_handle, double t, long long min[3], long long max[3],
                      long long* count);

/* ---------------------------------------------------------------- extract-psfs
 * The bead average of mvrecon's PSFExtraction (recalled).  Additive: the ABI version stays 107.
 *
 * The resident volume (U8 / U16 / F32) is the window [window_min, window_min + dims) of a full-resolution view of size
 * full_dims.  For every PSF voxel o in [-h, h] (h = (psf_size - 1) / 2, x fastest) and every point p, in the order
 * given: sum[o] += (double) nlinear(p + o), where nlinear is bs_sample_nlinear's arithmetic (PARITY_GAPS #37: double
 * weights, each corner term (float)(v w), summed in float) on the border extension of the FULL view; the caller's
 * window must hold every tap that extension reaches.  sum: host [sz][sy][sx] doubles, read and written, so a caller
 * that passes the points in several calls, in order, gets exactly the one-call result.  n = 0 leaves sum as it is.
 * BS_ERR_ARG for an even or non-positive psf_size, n < 0, NULL pointers, an unknown handle, or a window outside
 * full_dims.  Profile tag "psf". */
int bs_psf_accumulate(bs_ctx* ctx, unsigned long long vol_handle, const long long window_min[3],
                      const long long full_dims[3], const double* points_xyz, int n, const int psf_size[3], double* sum);

#ifdef __cplusplus
}
#endif
#endif /* BSGPU_H */
