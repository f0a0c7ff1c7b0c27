package net.preibisch.bigstitcher.spark.gpu;

import java.nio.ByteBuffer;

/**
 * Native methods of libbsgpu_jni.so (jni/bs_jni.cpp), one per entry point of include/bsgpu.h.
 * A context ({@code long ctx}) is bound to one device and one stream; create one per worker thread
 * (the Spark RDD of pairs / blocks collapses to a plain work queue over contexts).
 * Every failing call throws RuntimeException(bs_last_error).
 */
public final class BsNative
{
	static { System.loadLibrary( "bsgpu_jni" ); }

	private BsNative() {}

	public static final int U16 = 0, F32 = 1, U8 = 2;
	/** FusionType ordinals (mvrecon FusionGUI.FusionType) */
	public static final int AVG = 0, AVG_BLEND = 1, AVG_CONTENT = 2, AVG_BLEND_CONTENT = 3, MAX_INTENSITY = 4,
			LOWEST_VIEWID_WINS = 5, HIGHEST_VIEWID_WINS = 6, CLOSEST_PIXEL_WINS = 7;
	/** layout of the double[] a pcm* call returns per pair */
	public static final int R_FOUND = 0, R_SHIFT_INT = 1, R_SHIFT_SUB = 4, R_R = 7, R_N_OVERLAP = 8, R_PEAK = 9,
			R_PCM_VALUE = 12, R_PAD = 13, R_N_CANDIDATES = 16, R_PEARSON_PX = 17, R_STRIDE = 20;

	public static native int version();
	public static native long init( int device );
	public static native void destroy( long ctx );
	public static native String lastError( long ctx );
	public static native void synchronize( long ctx );
	public static native long launchCount( long ctx );
	public static native void profileEnable( long ctx, boolean on );
	public static native void profileReset( long ctx );
	public static native double[] profileGet( long ctx, String tag );
	public static native ByteBuffer hostAlloc( long ctx, long bytes );
	public static native void hostFree( long ctx, ByteBuffer buffer );

	/** data: short[] / float[] / byte[] or a direct ByteBuffer; dims {x,y,z} */
	public static native long volumeUpload( long ctx, Object data, long[] dims, int dtype );
	public static native long volumeUploadAsync( long ctx, ByteBuffer pinned, long[] dims, int dtype );
	public static native long volumeWrap( long ctx, long devicePointer, long[] dims, int dtype );
	public static native void volumeFree( long ctx, long handle );
	/** {dimX, dimY, dimZ, dtype} */
	public static native long[] volumeInfo( long ctx, long handle );
	public static native long volumeDevptr( long ctx, long handle );
	public static native void volumeDownload( long ctx, long handle, Object dest, long capacityBytes );
	public static native long contentWeights( long ctx, long handle, double sigma1, double sigma2 );
	public static native long downsample( long ctx, long handle, int[] factors );

	public static native int goodFftSize( int n, boolean even );
	/** iparams {peaksToCheck, doSubpixel, extX, extY, extZ} */
	public static native double[] pcmPair( long ctx, Object img1, Object img2, long[] dims, int dtype, int[] iparams, double minOverlap );
	public static native double[] pcmBatch( long ctx, Object[] imgs1, Object[] imgs2, long[] dims, int dtype, int[] iparams, double minOverlap );
	/** jobs: n x {vol1, vol2, min1[3], min2[3], dims[3]} */
	public static native double[] pcmVolumesBatch( long ctx, long[] jobs, int[] iparams, double minOverlap );
	public static native long[] pcmDebugPcm( long ctx, Object img1, Object img2, long[] dims, int dtype, int[] extension, Object outPcm );
	/** device crops (volumeDevptr); boxes n x {o1[3], o2[3], sz[3]}; sumsOut long[5n] (integer input) or double[5n] (float32) */
	public static native void pcmDebugPearson( long ctx, long dev1, long dev2, long[] dims, int dtype, int[] boxes, Object sumsOut );
	/** one FFT pass (0..4) of the PCM pipeline: pass 0 reads the device crops devA / devB, passes 1..4 the interleaved
	 *  complex64 spectra inA / inB (float[2 * Pz*Py*(M+1)]); outA / outB float[] spectra (pass 4: float[Pz*Py*Px] PCM);
	 *  padOut (long[3], may be null) receives {Px, Py, Pz}; returns the kernel instantiation launched */
	public static native String pcmDebugPass( long ctx, int pass, long[] dims, int dtype, int[] extension, long devA, long devB,
			Object inA, Object inB, Object outA, Object outB, int poison, long[] padOut );

	/** models n*12, handles n*{volume, content}, blend n*{border[3], range[3]}, windows n*{fullDims[3], windowMin[3]} or null;
	 *  iparams {fusionType, interpolation, outDtype, blendLutN, outBigEndian (1: N5 block payload byte order)}; dparams {minIntensity, maxIntensity} */
	public static native void fuseBlock( long ctx, int nViews, double[] models, long[] handles, float[] blend, long[] windows,
			long[] blockMin, long[] blockSize, int[] iparams, double[] dparams, Object dest );
	public static native void fuseBlocks( long ctx, int nViews, double[] models, long[] handles, float[] blend, long[] windows,
			long[] blockMins, long[] blockSizes, int[] iparams, double[] dparams, Object[] dests );
	/** --masks: 255 / 65535 / 1.0f where any view's (grown) pixel grid covers the voxel (GenerateComputeBlockMasks) */
	public static native void maskBlocks( long ctx, int nViews, double[] models, long[] handles, long[] windows,
			long[] blockMins, long[] blockSizes, double[] maskOffset, int outDtype, int outBigEndian, Object[] dests );
	public static native long fuseBlockToVolume( long ctx, int nViews, double[] models, long[] handles, float[] blend, long[] windows,
			long[] blockMin, long[] blockSize, int[] iparams, double[] dparams );
	public static native void fuseAccumulate( long ctx, int nViews, double[] models, long[] handles, float[] blend,
			long[] blockMin, long[] blockSize, int[] iparams, double[] dparams, long sumWiDev, long sumWDev );
	/** view-sharded exchange: rank 0 draws the id, every rank joins, fuseAllreduce sums both partial buffers over NVLink */
	public static native byte[] commUniqueId();
	public static native void commInit( long ctx, int nRanks, int rank, byte[] id );
	public static native void commDestroy( long ctx );
	public static native void fuseAllreduce( long ctx, long sumWiDev, long sumWDev, long n );
	public static native void fuseFinish( long ctx, long sumWiDev, long sumWDev, long n, int[] iparams, double[] dparams, Object dest );

	/** n x {locX, locY, locZ, value, voxelX, voxelY, voxelZ, isMax}; dparams {sigma, threshold, minI, maxI}; iparams {findMax, findMin, localization} */
	public static native double[] dogDetect( long ctx, long handle, long[] intervalMin, long[] intervalSize, double[] dparams, int[] iparams );
	/** the DoG box the extremum stage reads, [min - 1, min + size + 1) per axis: out float[(sx+2)(sy+2)(sz+2)], x fastest;
	 *  dparams {sigma, minI, maxI}; blur 0 production, 1 generic, 2 window R 6, 3 window R 12; returns the blur launched */
	public static native String dogDebugDog( long ctx, long handle, long[] intervalMin, long[] intervalSize, double[] dparams, int blur, Object out );

	/** detect-interestpoints: LazyDownsample2x chain to float32 (x halvings, then y, then z); factors powers of two <= 128 */
	public static native long downsampleFloat( long ctx, long handle, int[] factors );
	/** --medianFilter: every z-slice divided by its ImageJ circular median of the radius (0 where the median is <= 0) */
	public static native long medianDivide( long ctx, long handle, int radius );
	/** n-linear intensities (border extension) at loc = n x {x, y, z} into out: float[n] or a direct ByteBuffer */
	public static native void sampleNlinear( long ctx, long handle, double[] loc, Object out );

	/** nonrigid-fusion (replaces NonRigidTools.fuseVirtualInterpolatedNonRigid): views as for fuseBlocks plus nPoints[n] and
	 *  targets / locals = 3 * sum(nPoints) doubles (world targets, full-resolution pixel locations); iparams / dparams as for
	 *  fuseBlock with fusionType AVG_BLEND and interpolation 1; cpDistance {10, 10, 10} in the reference */
	public static native void nonrigidFuseBlocks( long ctx, int nViews, double[] models, long[] handles, float[] blend, long[] windows,
			int[] nPoints, double[] targets, double[] locals, long[] blockMins, long[] blockSizes, long[] cpDistance,
			int[] iparams, double[] dparams, Object[] dests );
	/** the MLS-mapped source coordinate of every control point of one view for one block: double[gz][gy][gx][3]; gridDims receives {gx, gy, gz} */
	public static native double[] nonrigidDebugGrid( long ctx, double[] model, int nPoints, double[] targets, double[] locals,
			long[] blockMin, long[] blockSize, long[] cpDistance, long[] gridDims );

	/** match-interestpoints (replaces the descriptor steps of RGLDMPairwise): resident local descriptors of n world points
	 *  xyz = n x {x, y, z}; k = numNeighbors + redundancy <= 6 nearest other points per point */
	public static native long descriptorsBuild( long ctx, double[] xyz, int numNeighbors, int redundancy );
	public static native void descriptorsFree( long ctx, long handle );
	/** neighbour indices idx[n * k] and squared distances d2[n * k] of a descriptor set (-1 / +inf when n <= k) */
	public static native void descriptorsNeighbors( long ctx, long handle, long[] idx, double[] d2 );
	/** exhaustive search A -> B: per point of A the best B index (-1: none), its descriptor distance and the second best;
	 *  searchRadius < 0: unlimited */
	public static native void descriptorsMatch( long ctx, long ha, long hb, double searchRadius, long[] bestB, double[] best, double[] second );

	/** solver (replaces TileConfiguration.optimize behind Solver): tiles colourOffsets / colourTiles, fixed flags, links
	 *  int[2 * nLinks], matchOffsets long[nLinks + 1], p / q double[3 * nMatches], w double[nMatches]; iparams =
	 *  {transformation, regularization, maxIterations, maxPlateauwidth}, dparams = {lambda, maxError}; models double[12 * nTiles]
	 *  in and out; returns {iterations, stopped, skippedFits, error} */
	public static native double[] solveTiles( long ctx, int[] colourOffsets, int[] colourTiles, int[] fixed, int[] links,
			long[] matchOffsets, double[] p, double[] q, double[] w, int[] iparams, double[] dparams, double[] models,
			double[] tileError, double[] linkMean, double[] linkMax );
}
