"""The `call()` bodies of the reference's `stitching`, `create-fusion-container` and
`affine-fusion` commands with the Spark RDD collapsed to a plain host work queue over one
`native.Context` (BASELINE north_star), SpimData2 XML in, N5 / OME-Zarr blocks out.

  stitching               J/SparkPairwiseStitching.java:110-392
  create_fusion_container J/CreateFusionContainer.java:122-519   (N5 or OME-ZARR, named boxes, BDV projects, pyramid)
  affine_fusion           J/SparkAffineFusion.java:179-800       (s0 + multi-resolution pyramid)
  nonrigid_fusion         J/SparkNonRigidFusion.java:124-446     (MLS grids from interest-point correspondences)
  detect_interestpoints   J/SparkInterestPointDetection.java:173-964 (block-wise DoG, interestpoints.n5 + the XML)
  match_interestpoints    J/SparkGeometricDescriptorMatching.java:161-545 (PRECISE_TRANSLATION, correspondences)
  solver                  J/Solver.java:161-432                   (ONE_ROUND_SIMPLE / ONE_ROUND_ITERATIVE, registrations)
  resave                  J/SparkResaveN5.java:80-455             (OME-ZARR or BDV-N5 with the pyramid built on the device)
  match_intensities       J/SparkIntensityMatching.java:84-190    (pairwise intensity matches, RANSAC on the device)
  solve_intensities       J/IntensitySolver.java:50-123           (per-view intensity coefficients)
  downsample              J/SparkDownsample.java:60-190           (pyramid levels of an existing dataset, on the device)
  clear_interestpoints    J/ClearInterestPoints.java              (points + correspondences, or correspondences only)
  clear_registrations     J/ClearRegistrations.java               (drop the latest <ViewTransform>s)
  transform_points        J/TransformPoints.java                  (view pixel coordinates -> world, host only)
  split_images            J/SplitDatasets.java                    (overlapping sub-views, split loader, fake points)
  estimate_bounding_box   (no upstream command; BigStitcher's BoundingBoxMinFilterThreshold) (named box from the data)

Every command reads its images through viewsource.py, so `bdv.n5` and `bdv.multimg.zarr` datasets both work.

No argument parsing here (the picocli layer is out of scope); keyword names follow the CLI flags.
"""
from __future__ import annotations

import math
import os
import re
import shutil
from decimal import Decimal

import numpy as np

from . import fusion as bf
from . import n5 as bn5
from . import zarr as bzarr
from . import matching as bm
from . import intensity as bint
from . import native, solver as bsolver, split as bsplit, stitching as bst, viewsource as bvs
from .native import Context
from .spimdata import FILEMAP_LOADER, SpimData2, fusion_project


def stitching(xml_path, ctx: Context, downsampling=(2, 2, 1), peaks_to_check=5, disable_subpixel=False,
              min_r=0.3, max_r=1.0, max_shift_xyz=None, max_shift_total=None, dry_run=False,
              channel_combine="AVERAGE", illum_combine="PICK_BRIGHTEST", shard=(0, 1), allgather=None, view_selection=None):
    """`./stitching -x dataset.xml [-ds 2,2,1] [-p 5] [--channelCombine AVERAGE] [--illumCombine PICK_BRIGHTEST] ...`:
    phase-correlate every overlapping pair of tile GROUPS (a tile's channels / illuminations are combined,
    J/SparkPairwiseStitching.java:103-107,141-165,204-208) and store the filtered results in the XML's
    <StitchingResults>.  Returns all raw results.  ``view_selection``: keyword arguments of SpimData2.select_views
    (`--angleId`, `--tileId`, `--channelId`, `--illuminationId`, `--timepointId` or `-vi`, default all views).

    Multi-GPU (SURVEY 8e): pairs are independent, so rank r of w takes pairs[r::w] (``shard``) with no data-path
    collective; ``allgather(obj) -> [obj of every rank]`` (e.g. torch.distributed.all_gather_object) merges the
    20-doubles-per-pair results and rank 0 writes the XML."""
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    selected = data.select_views(**view_selection) if view_selection else None
    all_pairs = data.stitching_groups(selected)
    rank, world = shard
    pairs = all_pairs[rank::world]
    needed = sorted({v for p in pairs for g in p for v in g})
    tiles = {v: src.read_volume(v, 0) for v in needed}
    models = {v: data.model(*v) for v in needed}
    attributes = {v: data.setups[v[1]].attributes for v in needed}
    params = bst.PairwiseStitchingParameters(peaks_to_check=peaks_to_check, do_subpixel=not disable_subpixel)
    raw = bst.stitch_pairs(pairs, tiles, models, params, downsampling, ctx, attributes=attributes,
                           channel_combine=channel_combine, illum_combine=illum_combine)
    for (ga, gb), r in zip(pairs, raw):
        if r is not None:   # hash of the FIRST views' registrations (J/SparkPairwiseStitching.java:287-289)
            r.hash = SpimData2.transform_hash(data.registrations[ga[0]], data.registrations[gb[0]])
    if world > 1:
        parts = allgather(raw)
        merged = [None] * len(all_pairs)
        for r_, part in enumerate(parts):
            merged[r_::world] = part
        raw, pairs = merged, all_pairs
        if rank != 0:
            return raw
    # every compared pair loses its stored result (a->b and b->a), found or not (:323-325); then the new ones go in
    data.remove_stitching_results(pairs)
    kept = bst.filter_results(raw, min_r, max_r, max_shift_xyz, max_shift_total)
    data.set_stitching_results([dict(pair=r.pair, shift=r.transform, r=r.r, hash=r.hash, bbox_min=r.bbox_min,
                                     bbox_max=r.bbox_max) for r in kept])
    if not dry_run:
        data.save(xml_path)
    return raw


def estimate_multires_pyramid(dims_xyz, anisotropy_factor=float("nan"), min_size=64):
    """`--multiRes`: ExportN5Api.estimateMultiResPyramid (mvrecon; recalled, PARITY_GAPS): keep halving the axes
    whose accumulated voxel size is the smallest (so anisotropic z catches up) until no axis could be halved without
    dropping below ``min_size`` voxels.  Returns RELATIVE steps after s0."""
    cur = [int(v) for v in dims_xyz]
    voxel = [1.0, 1.0, 1.0 if math.isnan(anisotropy_factor) else float(anisotropy_factor)]
    steps = []
    while True:
        smallest = min(voxel)
        rel = [2 if (voxel[d] <= smallest * 1.5 and cur[d] // 2 >= min_size) else 1 for d in range(3)]
        if rel == [1, 1, 1]:
            break
        steps.append(tuple(rel))
        cur = [cur[d] // rel[d] for d in range(3)]
        voxel = [voxel[d] * rel[d] for d in range(3)]
    return steps


def views_bounding_box(data, view_ids, anisotropy_factor=float("nan")):
    """The box of all ``view_ids`` (Import.getBoundingBox without a name, J/util/Import.java:39-66): the union of the
    views' transformed bounding boxes (fusion.transformed_bounding_box) under their registrations, adjusted for
    ``anisotropy_factor``.  (lo, hi) float64 [3] of whole world coordinates, both inclusive."""
    lo = np.full(3, np.inf)
    hi = np.full(3, -np.inf)
    regs = bf.adjust_all_transforms({v: data.model(*v) for v in view_ids}, anisotropy_factor)
    for v, M in regs.items():
        bmin, bmax = bf.transformed_bounding_box(data.setups[v[1]].size, M)
        lo = np.minimum(lo, bmin)
        hi = np.maximum(hi, bmax)
    return lo, hi


def create_fusion_container(xml_path, out_path, block_size=(128, 128, 128), dtype="float32", min_intensity=None,
                            max_intensity=None, preserve_anisotropy=False, anisotropy_factor=float("nan"),
                            storage=None, downsamplings=(), multi_res=False, compression="zstd", bounding_box=None,
                            bdv=False, xml_out=None, num_channels=None, num_timepoints=None):
    """`./create-fusion-container -x dataset.xml -o fused.zarr [-s ZARR|N5] -d FLOAT32 --blockSize ... [--multiRes |
    -ds ...] [-c Zstandard] [-b name] [-ch n] [-tp n] [--bdv -xo fused.xml]`: the fusion target
    (Import.getBoundingBox, J/CreateFusionContainer.java:184-211, J/util/Import.java:39-66), datasets + metadata.
    Defaults follow the reference: OME-ZARR storage unless the path ends in .n5 (:67-69), Zstandard compression
    (:71-76).  ``downsamplings``: relative steps.

    ``bounding_box`` (`-b`): the named <BoundingBoxDefinition> of the XML instead of the box of all views; an unknown
    name raises ValueError.  With ``preserve_anisotropy`` its z range becomes floor(min_z / af) .. ceil(max_z / af)
    (:204-206), which needs ``anisotropy_factor``.

    ``num_channels`` / ``num_timepoints`` (`-ch` / `-tp`): the number of fused volumes per axis, default the XML's
    (:157-176).  affine_fusion then needs its ``channel`` and ``timepoint`` to fill them.

    ``bdv`` (`--bdv`, :391-487) also writes ``xml_out`` (`-xo`, required: ValueError without it), a BigStitcher
    project of the fused volumes (spimdata.fusion_project): one setup per channel, timepoints 0 .. n-1, read through a
    `bdv.n5` loader (N5: the volumes become `setup{c}/timepoint{t}/s{l}`) or a `bdv.multimg.zarr` loader whose
    `<zgroup>`s point at the container's root multiscale group with indices [c, t] (ZARR: the 5-D arrays are
    unchanged).  affine_fusion fills either layout.  Everything else, and the default containers, are unchanged."""
    if bdv and xml_out is None:
        raise ValueError("Please specify the output XML for the BDV dataset: -xo")
    data = SpimData2.load(xml_path)
    af = anisotropy_factor if preserve_anisotropy else float("nan")
    if bounding_box is None:
        lo, hi = views_bounding_box(data, data.view_ids(), af)
    else:
        boxes = data.bounding_boxes()
        if bounding_box not in boxes:
            raise ValueError(f"Bounding box '{bounding_box}' not present in XML.")
        lo, hi = (b.copy() for b in boxes[bounding_box])
        if preserve_anisotropy:
            if math.isnan(af):
                raise ValueError("a named bounding box with preserve_anisotropy needs anisotropy_factor")
            lo[2] = math.floor(lo[2] / af)
            hi[2] = math.ceil(hi[2] / af)
    if storage is None:   # guessed from the extension like the reference (J/SparkAffineFusion.java:206-225)
        storage = "N5" if out_path.rstrip("/").lower().endswith(".n5") else "ZARR"
    is_zarr = storage.upper() == "ZARR"
    dims = [int(hi[d] - lo[d] + 1) for d in range(3)]
    if multi_res and not downsamplings:
        downsamplings = estimate_multires_pyramid(dims, af)
    if dtype != "float32":   # J/CreateFusionContainer.java:226-242
        top = 255.0 if dtype == "uint8" else 65535.0
        min_intensity = 0.0 if min_intensity is None else min_intensity
        max_intensity = top if max_intensity is None else max_intensity
    nc = len(data.channels_ordered()) if num_channels is None else int(num_channels)
    nt = len(data.timepoints) if num_timepoints is None else int(num_timepoints)
    kw = dict(anisotropy_factor=af if preserve_anisotropy else None, num_channels=nc, num_timepoints=nt,
              compression=compression, downsamplings=downsamplings)
    if bdv:
        kw["output_xml"] = os.path.abspath(xml_out)
    create = bzarr.create_fusion_container_zarr if is_zarr else bn5.create_fusion_container
    store = create(out_path, os.path.abspath(xml_path), lo.astype(np.int64), hi.astype(np.int64), block_size, dtype,
                   min_intensity, max_intensity, **kw)
    if bdv:
        project = fusion_project(xml_out, dims, nc, nt, af if preserve_anisotropy else None)
        if is_zarr:
            # the level datasets are "0", "1", ... of the root group (J/CreateFusionContainer.java:443-449)
            project.set_image_loader("bdv.multimg.zarr", out_path, xml_out,
                                     {(t, c): ("", c, t) for c in range(nc) for t in range(nt)})
        else:
            project.set_image_loader("bdv.n5", out_path, xml_out)
        os.makedirs(os.path.dirname(os.path.abspath(xml_out)), exist_ok=True)
        project.save(xml_out)
    return store


# --------------------------------------------------------------------------------------------- affine-fusion
class _Sink:
    """N5Utils.saveBlock on the 3-D dataset (N5) or the 5-D view (OME-ZARR, J/SparkAffineFusion.java:630-670)."""

    def __init__(self, store, is_zarr, c, t):
        self.store, self.is_zarr, self.c, self.t = store, is_zarr, c, t

    def save(self, dataset, block, grid_pos):
        if self.is_zarr:
            self.store.save_block(dataset, block, tuple(grid_pos) + (self.c, self.t))
        else:
            self.store.save_block(dataset, block, grid_pos)

    def save_chunk(self, dataset, block, chunk_pos):
        """One storage block / chunk exactly as the device packed it (N5: already big-endian)."""
        if self.is_zarr:
            gx, gy, gz = chunk_pos
            self.store.write_chunk(dataset, (self.t, self.c, gz, gy, gx), block)
        else:
            self.store.write_block(dataset, chunk_pos, block)

    def read_region(self, dataset, mn, size):
        if self.is_zarr:
            return self.store.read_region(dataset, mn, size, self.c, self.t)
        return self.store.read_region(dataset, mn, size)

    def write_region(self, dataset, block, off_xyz, dims, bs):
        """[z,y,x] region at a block-aligned voxel offset (read-modify-write when it covers blocks only partly)."""
        z, y, x = block.shape
        for gz in range(off_xyz[2] // bs[2], -(-(off_xyz[2] + z) // bs[2])):
            for gy in range(off_xyz[1] // bs[1], -(-(off_xyz[1] + y) // bs[1])):
                for gx in range(off_xyz[0] // bs[0], -(-(off_xyz[0] + x) // bs[0])):
                    b0 = [gx * bs[0], gy * bs[1], gz * bs[2]]
                    ext = [min(bs[d], dims[d] - b0[d]) for d in range(3)]
                    if any(e <= 0 for e in ext):
                        continue
                    s0 = [max(off_xyz[d], b0[d]) for d in range(3)]
                    s1 = [min(off_xyz[0] + x, b0[0] + ext[0]), min(off_xyz[1] + y, b0[1] + ext[1]), min(off_xyz[2] + z, b0[2] + ext[2])]
                    part = block[s0[2] - off_xyz[2]:s1[2] - off_xyz[2], s0[1] - off_xyz[1]:s1[1] - off_xyz[1],
                                 s0[0] - off_xyz[0]:s1[0] - off_xyz[0]]
                    if list(part.shape[::-1]) == ext:
                        cur = part
                    else:
                        cur = self.read_region(dataset, b0, ext)
                        cur[s0[2] - b0[2]:s1[2] - b0[2], s0[1] - b0[1]:s1[1] - b0[1], s0[0] - b0[0]:s1[0] - b0[0]] = part
                    self.save(dataset, np.ascontiguousarray(cur), (gx, gy, gz))


def _compose(reg, mt):
    R = np.vstack([np.asarray(reg, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
    M = np.vstack([np.asarray(mt, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
    return (R @ M)[:3]


def _source_window(src_to_world, level_dims, wmin, wmax, margin=3):
    """Source-pixel interval of a level volume that the world box [wmin, wmax] can sample (n-linear taps + margin),
    clipped to the volume; x is widened to multiples of 8 voxels (16-byte TMA rows).  None when empty."""
    inv = np.linalg.inv(np.vstack([src_to_world, [0, 0, 0, 1]]))[:3]
    c = np.array([[x, y, z] for x in (wmin[0], wmax[0]) for y in (wmin[1], wmax[1]) for z in (wmin[2], wmax[2])], dtype=np.float64)
    s = c @ inv[:, :3].T + inv[:, 3]
    lo = np.floor(s.min(axis=0)).astype(np.int64) - margin
    hi = np.ceil(s.max(axis=0)).astype(np.int64) + margin
    dims = np.asarray(level_dims, dtype=np.int64)
    lo = np.maximum(lo, 0)
    hi = np.minimum(hi, dims - 1)
    if np.any(hi < lo):
        return None
    lo[0] = (lo[0] // 8) * 8
    hi[0] = min(dims[0] - 1, (hi[0] // 8) * 8 + 7)
    return lo, hi - lo + 1


def affine_fusion(out_path, ctx: Context, fusion_type="AVG_BLEND", block_scale=(2, 2, 1), channel=None, timepoint=None,
                  retries=5, blocks_per_call=16, interpolation=1, shard=(0, 1), barrier=None, masks=False,
                  mask_offset=(0.0, 0.0, 0.0), view_selection=None, intensity_n5_path=None, intensity_n5_storage=None,
                  intensity_n5_group="", intensity_n5_dataset="intensity"):
    """`./affine-fusion -o fused.zarr [-f AVG_BLEND] [--blockScale 2,2,1] [-c channelIndex] [-t timepointIndex]
    [--masks [--maskOffset x,y,z]]`:
    read the container metadata and, for every (channel, timepoint) volume (J/SparkAffineFusion.java:425-440), fuse
    its views super-block by super-block on the device, write the blocks with N5Utils.saveBlock semantics and build
    the multi-resolution pyramid (:703-782).  Returns the list of s0 datasets written.

    Every container create_fusion_container writes is filled: plain N5 / OME-ZARR and the BDV projects (FusionFormat
    "BDV/N5": volume (c, t) is MultiResolutionInfos[c + t * NumChannels], the BDV-N5 view (t, setup c); "BDV/OME-ZARR":
    the 5-D arrays at [t, c]).  The views come from InputXML.  When the container's NumChannels / NumTimepoints differ
    from the XML's (`-ch` / `-tp`), ``channel`` and ``timepoint`` are required and name the one container volume to
    fuse; every view of ``view_selection`` (default all) goes into it (J/SparkAffineFusion.java:255-264,327-340,439).

    Source staging is block-wise (OverlappingBlocks / ViewUtil.findOverlappingBlocks, J/fusion/OverlappingBlocks.java:
    133-161): the super-block grid is walked in z-slabs; for every slab only the source WINDOW of each overlapping
    view is read from its container -- at the mipmap level ViewUtil's best-resolution rule picks
    (J/util/ViewUtil.java:425-493) -- uploaded as a windowed view and freed after the slab.

    ``view_selection``: keyword arguments of SpimData2.select_views (the AbstractSelectableViews flags); every
    (channel, timepoint) volume fuses its views out of that selection (J/SparkAffineFusion.java:425-440).

    ``masks``: save only the coverage masks (J/SparkAffineFusion.java:564-578, GenerateComputeBlockMasks): no image
    data is read, a voxel is 255 / 65535 / 1.0 where any view's pixel grid (grown by ``mask_offset`` source pixels)
    covers it; the pyramid is then built from that s0 as usual.

    Multi-GPU (SURVEY 8e, "one N5 block-grid slab per device"): rank r of w (``shard``) fuses a contiguous run of
    z-slabs, no data-path collective; ``barrier()`` separates s0 from the pyramid levels that re-read it.

    ``intensity_n5_path`` (`--intensityN5Path`, with `--intensityN5Storage` / `--intensityN5Group` /
    `--intensityN5Dataset`, J/SparkAffineFusion.java:158-168, 542-559): the coefficients solve-intensities wrote.  Each
    view's level volume is then staged whole, corrected on the device to float32 (bs_intensity_apply, before the
    n-linear resampling) and fused from that; content weights come from the corrected volume.  ``masks`` ignores them.
    A selected view without a coefficient dataset raises ValueError.  None: nothing changes."""
    coeffs = None
    if intensity_n5_path is not None and not masks:
        coeffs = (intensity_n5_path, bint.guess_storage(intensity_n5_path, intensity_n5_storage), intensity_n5_group,
                  intensity_n5_dataset)
    is_zarr = os.path.exists(os.path.join(out_path, ".zgroup"))
    store, meta = (bzarr.read_fusion_container_zarr if is_zarr else bn5.read_fusion_container)(out_path)
    data = SpimData2.load(meta["input_xml"])
    src = bvs.open_views(data)
    nc, nt = int(meta["num_channels"]), int(meta["num_timepoints"])
    # a container sized by -ch / -tp: the caller names the volume and the views that go into it
    # (J/SparkAffineFusion.java:255-264,327-340,439)
    manual = nc != len(data.channels_ordered()) or nt != len(data.timepoints)
    if manual and (channel is None or timepoint is None):
        raise ValueError(f"container says {nc} channel(s) / {nt} timepoint(s), the XML has "
                         f"{len(data.channels_ordered())} / {len(data.timepoints)}: give channel and timepoint (the "
                         f"container volume to fuse) and, optionally, view_selection (the views fused into it)")
    if manual and not (0 <= int(channel) < nc and 0 <= int(timepoint) < nt):
        raise ValueError(f"channel {channel} / timepoint {timepoint} outside the container's {nc} x {nt} volumes")
    written = []
    done = set()
    selected = data.select_views(**view_selection) if view_selection else None
    for c in range(nc):
        for t in range(nt):
            ci = c if channel is None else int(channel)
            ti = t if timepoint is None else int(timepoint)
            if (ci, ti) in done:
                continue
            done.add((ci, ti))
            levels = meta["mr_infos"][0 if is_zarr else ci + ti * nc]
            vol_views = (selected or data.view_ids()) if manual else data.views_of(ci, ti, selected)
            if not vol_views:
                continue                                             # nothing selected for this volume
            _fuse_volume_blockwise(ctx, data, src, _Sink(store, is_zarr, ci, ti), meta, levels, vol_views,
                                   fusion_type, interpolation, block_scale, retries, blocks_per_call, shard, barrier,
                                   masks, mask_offset, coeffs)
            written.append(levels[0]["dataset"])
    return written


def _fuse_volume_blockwise(ctx, data, src, sink, meta, levels, view_ids, fusion_type, interpolation, block_scale,
                           retries, blocks_per_call, shard=(0, 1), barrier=None, masks=False, mask_offset=(0.0, 0.0, 0.0),
                           coeffs=None):
    af = meta["anisotropy_factor"] if meta["preserve_anisotropy"] else float("nan")
    regs = bf.adjust_all_transforms({v: data.model(*v) for v in view_ids}, af)
    bb_min = np.asarray(meta["bb_min"], dtype=np.int64)
    dims = [int(meta["bb_max"][d] - meta["bb_min"][d] + 1) for d in range(3)]
    bs = [int(v) for v in meta["block_size"]]
    compute = tuple(bs[d] * int(block_scale[d]) for d in range(3))
    ft = native.FUSION_TYPES[fusion_type] if isinstance(fusion_type, str) else int(fusion_type)
    od = {"float32": native.DTYPE_F32, "uint16": native.DTYPE_U16, "uint8": native.DTYPE_U8}[meta["dtype"]]
    params = ctx.fuse_params(ft, interpolation, od, 0, float(meta["min_intensity"] or 0.0), float(meta["max_intensity"] or 65535.0))
    np_dt = native._BS2NP[od]
    s0 = levels[0]["dataset"]
    # blocks that go straight to the container leave the device as STORAGE chunks in the container's byte order
    # (N5 payloads are big-endian): the host neither re-strides nor swaps them
    chunk_params = ctx.fuse_params(ft, interpolation, od, 0, float(meta["min_intensity"] or 0.0),
                                   float(meta["max_intensity"] or 65535.0), out_big_endian=not sink.is_zarr)
    # the fusion kernels work on 64 x 16 x 8 output tiles anchored at the block origin: storage blocks that are whole
    # tiles (the usual 128^3 / 64^3) are packed by the device, smaller ones would leave most of every tile empty
    pack_on_device = bs[0] % 64 == 0 and bs[1] % 16 == 0 and bs[2] % 8 == 0

    # ---- per view: mipmap level by the reference's rule, level volume size, source -> world of that level
    info = {}
    for v in view_ids:
        factors, mts = src.mipmap_info(v)
        lvl = bf.best_mipmap_level(regs[v], factors, mts)
        m = _compose(regs[v], mts[lvl])
        info[v] = dict(level=lvl, dims=src.level_dims(v, lvl), model=m, blending=bf.adjust_blending(m),
                       dtype=src.level_dtype(v, lvl))
    vdims = {v: info[v]["dims"] for v in view_ids}
    vregs = {v: info[v]["model"] for v in view_ids}
    windowed_ok = (ft in (native.FUSE_AVG, native.FUSE_AVG_BLEND) and interpolation == 1 and
                   all(info[v]["dtype"] == "uint16" and info[v]["dims"][0] % 8 == 0 for v in view_ids))
    correction = {}
    if coeffs is not None:
        # corrected sources are float32 whole-view volumes (the windowed fusion kernel reads uint16 windows only)
        windowed_ok = False
        for v, c in bint.view_coefficients(*coeffs, view_ids).items():
            factors, mts = src.mipmap_info(v)
            correction[v] = (c, mts[info[v]["level"]], tuple(int(d) for d in data.setups[v[1]].size))
    content = ft in (native.FUSE_AVG_CONTENT, native.FUSE_AVG_BLEND_CONTENT)

    # pyramid straight from the resident fused block when every super-block maps onto whole voxels of every level
    fast_pyramid = len(levels) > 1 and _maps_onto_level(compute, levels[-1]) and not masks

    grid = bf.grid_create(dims, compute, bs)
    slabs = {}
    for gb in grid:
        slabs.setdefault(gb[0][2], []).append(gb)
    rank, world = shard
    zs = sorted(slabs)
    per = -(-len(zs) // world)
    my_z = zs[rank * per:(rank + 1) * per]           # contiguous run of z-slabs per device
    whole = {}      # fallback residency (content weights, winner types, float sources ...): whole views, kept
    if masks:
        # geometry only: full-resolution registrations and view sizes (GenerateComputeBlockMasks.java:119-128)
        fdims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in view_ids}
        for z0 in my_z:
            todo, attempt = list(slabs[z0]), 0
            while todo:
                attempt += 1
                if attempt > retries:
                    raise RuntimeError(f"masks: {len(todo)} block(s) still failing after {retries} attempts")
                failed = []
                for gb in todo:
                    off, size, gpos = gb
                    mn = tuple(int(v) for v in bb_min + np.asarray(off, dtype=np.int64))
                    sz = tuple(int(v) for v in size)
                    # the views of THIS block (OverlappingViews on the block expanded by 2, like the fusing path): a
                    # mask offset never pulls in a view the block does not overlap
                    vids = bf.find_overlapping_views(fdims, regs, np.asarray(mn), np.asarray(mn) + np.asarray(sz) - 1, sorted(view_ids))
                    gviews = [dict(src_to_world=regs[v], vol_handle=0, full_dims=fdims[v]) for v in vids]
                    try:
                        blk = ctx.mask_blocks(gviews, [mn], [sz], mask_offset, od)[0]
                    except native.BsError:
                        failed.append(gb)
                        continue
                    sink.save(s0, blk, gpos)
                todo = failed
        my_z = []
    try:
        for z0 in my_z:
            blocks = slabs[z0]
            lo = bb_min + np.array([0, 0, z0])
            hi = bb_min + np.array([dims[0] - 1, dims[1] - 1, min(dims[2], z0 + compute[2]) - 1])
            vids = bf.find_overlapping_views(vdims, vregs, lo, hi, view_ids)
            staged, views = {}, {}
            try:
                for v in vids:
                    border, rng = info[v]["blending"]
                    if windowed_ok:
                        w = _source_window(info[v]["model"], info[v]["dims"], lo - bf.AFFINE_EXPANSION, hi + bf.AFFINE_EXPANSION)
                        if w is None:
                            continue
                        wmin, wsize = w
                        staged[v] = ctx.volume_upload(src.read_region(v, info[v]["level"], wmin, wsize))
                        views[v] = dict(src_to_world=info[v]["model"], vol_handle=staged[v], blend_border=border, blend_range=rng,
                                        full_dims=info[v]["dims"], window_min=tuple(int(x) for x in wmin))
                    else:
                        if v not in whole:
                            h = ctx.volume_upload(src.read_volume(v, info[v]["level"]))
                            if v in correction:
                                (ca, cb), mt, full = correction[v]
                                try:
                                    hc = ctx.intensity_apply(h, full, mt, ca, cb)
                                finally:
                                    ctx.volume_free(h)
                                h = hc
                            whole[v] = (h, ctx.content_weights(h) if content else 0)
                        views[v] = dict(src_to_world=info[v]["model"], vol_handle=whole[v][0], content_handle=whole[v][1],
                                        blend_border=border, blend_range=rng)
                # ---- the slab's super-blocks, `blocks_per_call` per launch, RetryTracker policy (<= 5 attempts)
                todo, attempt = list(blocks), 0
                while todo:
                    attempt += 1
                    if attempt > retries:
                        raise RuntimeError(f"fusion: {len(todo)} block(s) still failing after {retries} attempts")
                    failed = []
                    if fast_pyramid:
                        # every super-block is fused into a RESIDENT volume and its lower levels are derived on the
                        # device (bs_downsample) before anything is downloaded -- level l-1 is never re-read from
                        # the container (SURVEY 8f-3; the reference re-reads it, J/SparkAffineFusion.java:703-782)
                        for gb in todo:
                            try:
                                _fuse_block_with_pyramid(ctx, gb, bb_min, vdims, vregs, views, params, np_dt, sink, levels, bs)
                            except native.BsError:
                                failed.append(gb)
                    else:
                        for c0 in range(0, len(todo), blocks_per_call):
                            chunk = todo[c0:c0 + blocks_per_call]
                            if not pack_on_device:       # small storage blocks: fuse super-blocks, split on the host
                                try:
                                    outs = _fuse_chunk(ctx, chunk, bb_min, vdims, vregs, views, params, np_dt)
                                except native.BsError:
                                    failed.extend(chunk)
                                    continue
                                for (off, size, gpos), blk in zip(chunk, outs):
                                    sink.save(s0, blk, gpos)
                                continue
                            cells = [cell for gb in chunk for cell in _storage_cells(gb, bs)]
                            try:
                                outs = _fuse_chunk(ctx, cells, bb_min, vdims, vregs, views, chunk_params, np_dt)
                            except native.BsError:
                                failed.extend(chunk)
                                continue
                            for (off, size, gpos), blk in zip(cells, outs):
                                sink.save_chunk(s0, blk, gpos)
                    todo = failed
            finally:
                for h in staged.values():
                    ctx.volume_free(h)
    finally:
        for h, ch in whole.values():
            ctx.volume_free(h)
            if ch:
                ctx.volume_free(ch)

    # ---- pyramid s1 .. sN when super-blocks do not map onto whole voxels of every level
    _pyramid_from_stored(ctx, [(sink, levels, np_dt)], len(levels) if fast_pyramid else 1, compute, bs, shard, retries,
                         barrier)


def _fuse_block_with_pyramid(ctx, gb, bb_min, vdims, vregs, views, params, np_dt, sink, levels, bs):
    off, size, gpos = gb
    wmin = bb_min + np.asarray(off, dtype=np.int64)
    vids = bf.find_overlapping_views(vdims, vregs, wmin, wmin + np.asarray(size) - 1, sorted(views))
    cur_h = ctx.fuse_block_to_volume([views[v] for v in vids], tuple(int(v) for v in wmin), tuple(int(v) for v in size), params)
    _write_resident_levels(ctx, cur_h, gb, sink, levels, bs, np_dt)


# --------------------------------------------------------------------------------------------- pyramid (shared)
# The multi-resolution pyramid of a container volume, shared by affine-fusion and resave.  A level is the 2x half-pixel
# average of the level above (N5ApiTools.writeDownsampledBlock[5dOMEZARR], LazyHalfPixelDownsample2x), taken on the
# device by bs_downsample.  While a compute block is resident, every level it maps onto whole voxels of is derived from
# it before anything is downloaded; the other levels are built from the stored level l-1 once it is complete.
def _maps_onto_level(compute, level):
    """True when compute blocks (at multiples of ``compute``) cover whole voxels of ``level`` (so the chained
    downsampling of a block equals that of the volume)."""
    a = [int(v) for v in level["absoluteDownsampling"][:3]]
    return all(int(compute[d]) % a[d] == 0 for d in range(3))


def _write_resident_levels(ctx, cur_h, gb, sink, levels, bs, np_dt):
    """Write the resident compute block ``cur_h`` (grid block ``gb`` of level 0) to every level of ``levels``, deriving
    each from the previous one on the device; frees ``cur_h``.  Each level is downloaded and split into storage blocks
    on the host, read-modify-writing those it covers only partly."""
    off, size, gpos = gb
    try:
        cur_size, cur_off = [int(v) for v in size], [int(v) for v in off]
        for li, lv in enumerate(levels):
            if li > 0:
                rel = [int(v) for v in lv["relativeDownsampling"][:3]]
                nxt = [cur_size[d] // rel[d] for d in range(3)]
                if min(nxt) < 1:
                    break        # an edge block thinner than the step: no voxel of this (or any deeper) level
                nh = ctx.downsample(cur_h, rel)
                ctx.volume_free(cur_h)
                cur_h, cur_size, cur_off = nh, nxt, [cur_off[d] // rel[d] for d in range(3)]
            if li == 0:
                sink.save(lv["dataset"], ctx.volume_download(cur_h, cur_size, np_dt), gpos)
            else:
                sink.write_region(lv["dataset"], ctx.volume_download(cur_h, cur_size, np_dt), cur_off,
                                  [int(v) for v in lv["dimensions"][:3]], bs)
    finally:
        ctx.volume_free(cur_h)


def _pyramid_from_stored(ctx, volumes, first, compute, bs, shard=(0, 1), retries=5, barrier=None, resident=1):
    """Levels ``first`` .. N of every volume in ``volumes`` ([(sink, levels, numpy dtype)]): every compute block of level
    l is the 2x average of its region of level l-1, read back from the container and averaged on the device.  Rank r of
    w takes blocks [r::w] of each level; ``barrier()`` runs before each level so that level l-1 is complete on every
    rank.  Failed blocks are retried up to ``retries`` times (RetryTrackerSpark).

    ``resident`` > 1: levels first + 1 .. first + resident - 1 are derived from each compute block of level ``first``
    while it is on the device (_write_resident_levels); those compute blocks must cover whole storage blocks of them."""
    rank, world = shard
    li = first
    while li < max(len(lv) for _, lv, _ in volumes):
        n = resident if li == first else 1
        if barrier is not None:
            barrier()                                # level l-1 is complete on every rank
        work = []
        for sink, levels, np_dt in volumes:
            if li < len(levels):
                cdims = [int(v) for v in levels[li]["dimensions"][:3]]
                work += [(sink, levels, np_dt, gb) for gb in bf.grid_create(cdims, compute, bs)]
        todo, attempt = work[rank::world], 0
        while todo:
            attempt += 1
            if attempt > retries:
                raise RuntimeError(f"pyramid s{li}: {len(todo)} block(s) still failing after {retries} attempts")
            failed = []
            for item in todo:
                sink, levels, np_dt, (off, size, gpos) = item
                prev, cur = levels[li - 1], levels[li]
                rel = [int(v) for v in cur["relativeDownsampling"][:3]]
                h = None
                try:
                    srcblk = sink.read_region(prev["dataset"], [off[d] * rel[d] for d in range(3)], [size[d] * rel[d] for d in range(3)])
                    h = ctx.volume_upload(np.ascontiguousarray(srcblk))
                    # the downsampled block is freed by _write_resident_levels
                    _write_resident_levels(ctx, ctx.downsample(h, rel), (off, size, gpos), sink, levels[li:li + n], bs,
                                           np_dt)
                except native.BsError:
                    failed.append(item)
                finally:
                    if h is not None:
                        ctx.volume_free(h)
            todo = failed
        li += n


def _storage_cells(gb, bs):
    """The storage blocks of one super-block: [(offset, size, grid position)] in the container's block grid."""
    off, size, gpos = gb
    cells = []
    for kz in range(-(-size[2] // bs[2])):
        for ky in range(-(-size[1] // bs[1])):
            for kx in range(-(-size[0] // bs[0])):
                k = (kx, ky, kz)
                cells.append((tuple(int(off[d] + k[d] * bs[d]) for d in range(3)),
                              tuple(int(min(bs[d], size[d] - k[d] * bs[d])) for d in range(3)),
                              tuple(int(gpos[d] + k[d]) for d in range(3))))
    return cells


def _fuse_chunk(ctx, chunk, bb_min, vdims, vregs, views, params, np_dt):
    mins, sizes = [], []
    lo = np.array([np.inf] * 3)
    hi = np.array([-np.inf] * 3)
    for (off, size, _) in chunk:
        wmin = bb_min + np.asarray(off, dtype=np.int64)
        mins.append(tuple(int(v) for v in wmin))
        sizes.append(tuple(int(v) for v in size))
        lo = np.minimum(lo, wmin)
        hi = np.maximum(hi, wmin + np.asarray(size) - 1)
    vids = [v for v in bf.find_overlapping_views(vdims, vregs, lo.astype(np.int64), hi.astype(np.int64), sorted(views))]
    return ctx.fuse_blocks([views[v] for v in vids], mins, sizes, params)


# --------------------------------------------------------------------------------------------- detect-interestpoints
IP_POWERS = (1, 2, 4, 8, 16, 32, 64, 128)        # J/SparkInterestPointDetection.java:1005
IP_N5_BLOCK_LENGTH = 300000                      # InterestPointsN5.defaultBlockSize (recalled, PARITY_GAPS)
IP_N5_GROUP_ATTRIBUTES = {"pointcloud": "1.0.0", "type": "list", "list version": "1.0.0"}   # recalled, PARITY_GAPS


def java_double(v) -> str:
    """Double.toString: shortest round-trip digits, plain in [1e-3, 1e7), else computerized scientific ("1.0E-4")."""
    v = float(v)
    if math.isnan(v):
        return "NaN"
    if math.isinf(v):
        return "Infinity" if v > 0 else "-Infinity"
    if v == 0.0:
        return "-0.0" if math.copysign(1.0, v) < 0 else "0.0"
    if 1e-3 <= abs(v) < 1e7:
        return repr(v)
    sign, digits, exp = Decimal(repr(abs(v))).as_tuple()
    digits = list(digits)
    while len(digits) > 1 and digits[-1] == 0:
        digits.pop()
        exp += 1
    e = len(digits) - 1 + exp
    frac = "".join(str(d) for d in digits[1:]) or "0"
    return f"{'-' if v < 0 else ''}{digits[0]}.{frac}E{e}"


def _java(v) -> str:
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(v)
    return java_double(v)


def interestpoint_params(sigma, threshold, overlapping_only, find_min, find_max, downsample_xy, downsample_z,
                         min_intensity, max_intensity) -> str:
    """The params attribute of <ViewInterestPointsFile> (J/SparkInterestPointDetection.java:898-899)."""
    return (f"DOG (Spark) s={_java(float(sigma))} t={_java(float(threshold))} overlappingOnly={_java(bool(overlapping_only))} "
            f"min={_java(bool(find_min))} max={_java(bool(find_max))} downsampleXY={int(downsample_xy)} "
            f"downsampleZ={int(downsample_z)} minIntensity={_java(float(min_intensity))} "
            f"maxIntensity={_java(float(max_intensity))}")


def interestpoint_level(factors, downsample_xyz):
    """openAndDownsample's level choice (J/SparkInterestPointDetection.java:1026-1044): the LAST mipmap level whose
    rounded factors are all <= the requested ones and powers of two <= 128; returns (level, remaining factors) with
    remaining = requested / level factor per axis.  No requested downsampling reads level 0."""
    ds = [int(v) for v in downsample_xyz]
    if all(v == 1 for v in ds):
        return 0, (1, 1, 1)
    best = 0
    for lvl, f in enumerate(factors):
        r = [int(math.floor(float(v) + 0.5)) for v in f]       # Math.round
        if all(r[d] <= ds[d] and r[d] in IP_POWERS for d in range(3)):
            best = lvl
    r = [int(math.floor(float(v) + 0.5)) for v in factors[best]]
    return best, tuple(ds[d] // r[d] for d in range(3))


def interestpoint_transform(mipmap_transform, remaining_xyz):
    """Downsampled pixel -> full-resolution view pixel: mipmapTransform[level] o scale(remaining), no extra shift
    (J/SparkInterestPointDetection.java:1067-1081, applied by correctForDownsampling at :606-609)."""
    M = np.vstack([np.asarray(mipmap_transform, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
    S = np.diag([float(v) for v in remaining_xyz] + [1.0])
    return (M @ S)[:3]


def interestpoint_blocks(dims_xyz, block_size):
    """The DoG intervals of one view: the reference's Grid.create blocks in job order, each passed to bs_dog_detect
    as it is, but shrunk by one voxel on faces that lie on the view border.  The reference expands every block by one
    voxel inside the image and computeDoG tests only the interior of its interval (J/SparkInterestPointDetection.java:
    397-424, PARITY_GAPS), so every voxel but the view's outermost layer is tested exactly once."""
    out = []
    for off, size, _ in bf.grid_create([int(v) for v in dims_xyz], [int(v) for v in block_size]):
        lo = [max(off[d], 1) for d in range(3)]
        hi = [min(off[d] + size[d], int(dims_xyz[d]) - 1) for d in range(3)]
        if all(hi[d] > lo[d] for d in range(3)):
            out.append((tuple(lo), tuple(hi[d] - lo[d] for d in range(3))))
    return out


def _check_device_memory(ctx, nbytes, what, command="detect-interestpoints",
                         advice="use a larger --downsampleXY / --downsampleZ"):
    free = ctx.memory_free()
    if nbytes > free:
        raise MemoryError(f"{command}: {what} needs {nbytes / 2**30:.2f} GiB on device {ctx.device}, "
                          f"{free / 2**30:.2f} GiB are free; {advice}")


def _detect_view(ctx, src, view, level, remaining, mt, sigma, threshold, min_intensity, max_intensity, find_max,
                 find_min, localization, block_size, median_filter, need_intensities):
    ldims = list(src.level_dims(view, level))
    vox = int(np.prod(ldims))
    dvox = int(np.prod([max(ldims[d] // remaining[d], 0) for d in range(3)]))
    blk = int(np.prod([min(int(block_size[d]), ldims[d]) + 64 for d in range(3)]))
    _check_device_memory(ctx, vox * np.dtype(src.level_dtype(view, level)).itemsize + 4 * (2 * dvox + 4 * blk),
                         f"view {view} (level s{level}, {ldims[0]}x{ldims[1]}x{ldims[2]})")
    handles = []
    try:
        h = ctx.volume_upload(src.read_volume(view, level))
        handles.append(h)
        img = h
        if any(v > 1 for v in remaining):
            img = ctx.downsample_float(h, remaining)
            handles.append(img)
            ctx.volume_free(h)
            handles.remove(h)
        det = img
        if median_filter:
            det = ctx.median_divide(img, int(median_filter))
            handles.append(det)
        dims, _ = ctx.volume_info(det)
        locs = []
        for mn, sz in interestpoint_blocks(dims, block_size):
            pts = ctx.dog_detect(det, mn, sz, sigma=sigma, threshold=threshold, min_intensity=min_intensity,
                                 max_intensity=max_intensity, find_max=find_max, find_min=find_min,
                                 localization=localization)
            locs.extend(p[0] for p in pts)
        loc = np.array(locs, dtype=np.float64).reshape(-1, 3)
        inten = ctx.sample_nlinear(img, loc) if need_intensities else None
    finally:
        for hh in handles:
            ctx.volume_free(hh)
    T = interestpoint_transform(mt, remaining)
    return loc @ T[:, :3].T + T[:, 3], inten


def detect_interestpoints(xml_path, ctx: Context, label, sigma, threshold, min_intensity, max_intensity, type="MAX",
                          localization="QUADRATIC", downsample_xy=2, downsample_z=1, block_size=(512, 512, 128),
                          median_filter=None, store_intensities=False, max_spots=0, view_selection=None, dry_run=False,
                          shard=(0, 1), allgather=None, overlapping_only=False, only_compare_overlap_tiles=False,
                          max_spots_per_overlap=False, prefetch=False, keep_temporary_n5=False):
    """`./detect-interestpoints -x dataset.xml -l beads -s 1.8 -t 0.008 -i0 0 -i1 2048 [--type MAX|MIN|BOTH]
    [--localization NONE|QUADRATIC] [-dsxy 2] [-dsz 1] [--blockSize 512,512,128] [--medianFilter r]
    [--storeIntensities] [--maxSpots N]`: per selected view, read the mipmap level openAndDownsample picks, finish the
    downsampling on the device in float (bs_downsample_float), optionally divide every z-slice by its median
    (bs_median_divide), run bs_dog_detect over the reference's block grid, map the points to full-resolution pixels and
    write them to `interestpoints.n5` next to the XML plus a <ViewInterestPointsFile> per view (also views without
    points).  Returns {(tp, setup): (loc (n, 3) float64, intensities float32 (n,) or None)}.

    ``prefetch`` and ``keep_temporary_n5`` tune the reference's Spark execution and are accepted without effect.
    ``overlapping_only``, ``only_compare_overlap_tiles`` and ``max_spots_per_overlap`` are not implemented.

    Multi-GPU: rank r of w (``shard``) takes views[r::w]; ``allgather(obj) -> [obj of every rank]`` merges the results
    and rank 0 writes."""
    for flag, on in (("--overlappingOnly", overlapping_only), ("--onlyCompareOverlapTiles", only_compare_overlap_tiles),
                     ("--maxSpotsPerOverlap", max_spots_per_overlap)):
        if on:
            raise NotImplementedError(f"detect-interestpoints {flag} is not implemented")
    type = type.upper()
    if type not in ("MIN", "MAX", "BOTH") or localization.upper() not in ("NONE", "QUADRATIC"):
        raise ValueError(f"--type {type} / --localization {localization}")
    find_min, find_max = type in ("MIN", "BOTH"), type in ("MAX", "BOTH")
    for v in (downsample_xy, downsample_z):
        if int(v) not in IP_POWERS:
            raise ValueError(f"downsampling {v} is not a power of two <= 128")
    if median_filter is not None and not 0 < int(median_filter) <= native.MEDIAN_MAX_RADIUS:
        raise ValueError(f"--medianFilter {median_filter} outside [1, {native.MEDIAN_MAX_RADIUS}]")
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    views = data.select_views(**view_selection) if view_selection else data.view_ids()
    rank, world = shard
    results = {}
    for v in views[rank::world]:
        factors, mts = src.mipmap_info(v)
        level, remaining = interestpoint_level(factors, (downsample_xy, downsample_xy, downsample_z))
        loc, inten = _detect_view(ctx, src, v, level, remaining, mts[level], sigma, threshold, min_intensity, max_intensity,
                                  find_max, find_min, localization.upper() == "QUADRATIC", block_size, median_filter,
                                  store_intensities or max_spots > 0)
        if max_spots > 0 and len(loc) > max_spots:
            order = sorted(range(len(loc)), key=lambda i: -float(inten[i]))[:max_spots]   # stable, descending
            loc, inten = loc[order], inten[order]
        results[v] = (loc, inten if store_intensities else None)
    if world > 1:
        merged = {}
        for part in allgather(results):
            merged.update(part)
        results = {v: merged[v] for v in views if v in merged}
        if rank != 0:
            return results
    if dry_run:
        return results
    base = os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")
    store = bn5.N5Store(os.path.join(base, "interestpoints.n5"), create=True)
    paths = {}
    for (tp, setup), (loc, inten) in sorted(results.items()):
        group = f"tpId_{tp}_viewSetupId_{setup}/{label}"
        shutil.rmtree(os.path.join(store.root, group), ignore_errors=True)     # re-running a label replaces it
        store.set_attributes(group + "/interestpoints", IP_N5_GROUP_ATTRIBUTES)
        store.write_list(group + "/interestpoints/id", np.arange(len(loc), dtype=np.uint64).reshape(-1, 1),
                         IP_N5_BLOCK_LENGTH, "zstd")
        store.write_list(group + "/interestpoints/loc", loc.astype(np.float64), IP_N5_BLOCK_LENGTH, "zstd")
        if inten is not None:
            store.write_list(group + "/intensities", inten.astype(np.float32).reshape(-1, 1), IP_N5_BLOCK_LENGTH,
                             "zstd")
        paths[(tp, setup)] = group
    data.set_interest_points(label, interestpoint_params(sigma, threshold, overlapping_only, find_min, find_max,
                                                         downsample_xy, downsample_z, min_intensity, max_intensity),
                             paths)
    data.save(xml_path)
    return results


# --------------------------------------------------------------------------------------------- nonrigid-fusion
NONRIGID_FUSE_EXPAND = 50      # viewsToFuse: transformed bounding box expanded by 50 (J/SparkNonRigidFusion.java:333-340)
NONRIGID_USE_EXPAND = 25       # viewsToUse: both boxes expanded by 25 (J/SparkNonRigidFusion.java:349-371)


def nonrigid_views_for_block(view_dims, registrations, block_min, block_max, view_ids):
    """(viewsToFuse, viewsToUse) of one super-block (J/SparkNonRigidFusion.java:317-371): the views whose transformed
    bounding box, expanded by 50, overlaps the block; and every view whose box expanded by 25 overlaps the box of a
    fused view expanded by 25 (the fused views included)."""
    fuse = bf.find_overlapping_views(view_dims, registrations, block_min, block_max, view_ids, expand=NONRIGID_FUSE_EXPAND)
    boxes = {v: bf.transformed_bounding_box(view_dims[v], registrations[v]) for v in view_ids}
    e = NONRIGID_USE_EXPAND
    use = [v for v in view_ids
           if any(np.all(np.minimum(boxes[v][1] + e, boxes[f][1] + e) >= np.maximum(boxes[v][0] - e, boxes[f][0] - e))
                  for f in fuse)]
    return fuse, use


class _InterestPoints:
    """Every selected view's points and correspondences of the `-ip` labels, read once from interestpoints.n5, with
    their world positions (the view's registration applied to the full-resolution pixel location)."""

    def __init__(self, store: bn5.N5Store, view_ids, labels, registrations, tables=False):
        """``tables``: keep each view's correspondences as arrays (``table``, ``ids``) instead of the row list ``corr``."""
        self.labels = list(labels)
        self.loc, self.world, self.index, self.corr, self.table, self.ids = {}, {}, {}, {}, {}, {}
        for v in view_ids:
            for label in self.labels:
                group = f"tpId_{v[0]}_viewSetupId_{v[1]}/{label}"
                if "dimensions" not in store.get_attributes(group + "/interestpoints/loc"):
                    continue
                ids = store.read_list(group + "/interestpoints/id").reshape(-1).astype(np.int64)
                loc = store.read_list(group + "/interestpoints/loc").astype(np.float64).reshape(-1, 3)
                M = np.asarray(registrations[v], dtype=np.float64).reshape(3, 4)
                self.loc[(v, label)] = loc
                self.world[(v, label)] = loc @ M[:, :3].T + M[:, 3]
                self.ids[(v, label)] = ids
                if tables:
                    self.table[(v, label)] = store.read_correspondence_table(group)
                    continue
                self.index[(v, label)] = {int(i): k for k, i in enumerate(ids)}
                self.corr[(v, label)] = store.read_correspondences(group)

    def targets(self, view, views_to_use):
        """N2: (target world (n, 3), local pixel (n, 3)) of one view to fuse: every point with at least one
        correspondence whose partner is in ``views_to_use`` and has one of the labels; the target is the mean of the
        point's own world position and its direct partners' world positions."""
        use = set(views_to_use)
        ts, ls = [], []
        for label in self.labels:
            key = (view, label)
            if key not in self.loc:
                continue
            acc = np.zeros_like(self.world[key])
            cnt = np.zeros(len(acc), dtype=np.int64)
            for (pid, pv, pl, qid) in self.corr[key]:
                if pv in use and pl in self.labels and (pv, pl) in self.loc:
                    k = self.index[key][pid]
                    acc[k] += self.world[(pv, pl)][self.index[(pv, pl)][qid]]
                    cnt[k] += 1
            sel = cnt > 0
            ts.append((self.world[key][sel] + acc[sel]) / (cnt[sel] + 1)[:, None])
            ls.append(self.loc[key][sel])
        if not ts:
            return np.zeros((0, 3)), np.zeros((0, 3))
        return np.concatenate(ts), np.concatenate(ls)


def nonrigid_fusion(xml_path, ctx: Context, out_path, n5_dataset, interest_points, storage="N5",
                    block_size=(128, 128, 128), block_scale=(2, 2, 1), data_type="FLOAT32", min_intensity=None,
                    max_intensity=None, view_selection=None, bdv=None, xml_out=None, bounding_box=None, dry_run=False,
                    shard=(0, 1), retries=5, blocks_per_call=16, intensity_n5_path=None, intensity_n5_storage=None,
                    intensity_n5_group="", intensity_n5_dataset="intensity"):
    """`./nonrigid-fusion -x dataset.xml -o fused.n5 -d /ch0/s0 -ip beads [-ip nuclei] [-s N5|ZARR] [--blockSize ...]
    [--blockScale 2,2,1] [-p FLOAT32|UINT16|UINT8 --minIntensity --maxIntensity]` (J/SparkNonRigidFusion.java:124-446):
    the maximal bounding box of the selected views becomes dataset ``n5_dataset`` (Zstandard, attribute offset = bb.min);
    every super-block of Grid.create(dims, blockSize * blockScale, blockSize) that some view reaches is fused on the
    device with per-view moving-least-squares grids fitted to the corresponding interest points of the ``-ip`` labels
    (bs_nonrigid_fuse_blocks, AVG_BLEND, control points every 10 px) and saved; blocks no view reaches are not written.
    Returns the list of written grid positions.  ZARR output is the (t, c, z, y, x) array with singleton t and c.

    ``intensity_n5_path`` (`--intensityN5Path`, with `--intensityN5Storage` / `--intensityN5Group` /
    `--intensityN5Dataset`, as affine-fusion takes them; upstream nonrigid-fusion has no such option, PARITY_GAPS N6):
    the coefficients solve-intensities wrote.  Every staged s0 source window is corrected on the device to float32
    (bs_intensity_apply at the window's full-resolution position, before the n-linear resampling) and fused from that.
    The coefficients of every selected view are read before the output dataset is created, so a selected view without
    a coefficient dataset raises ValueError and leaves nothing behind.  None: nothing changes.

    ``--bdv`` / ``-xo``, named ``-b`` bounding boxes, multi-GPU sharding and ``--dryRun`` raise NotImplementedError."""
    for flag, on in (("--bdv", bdv is not None), ("-xo", xml_out is not None), ("-b", bounding_box is not None),
                     ("--dryRun", dry_run), ("multi-GPU sharding", shard[1] > 1)):
        if on:
            raise NotImplementedError(f"nonrigid-fusion {flag} is not implemented")
    dt = data_type.upper()
    if dt not in ("FLOAT32", "UINT16", "UINT8"):
        raise ValueError(f"-p {data_type}")
    if dt != "FLOAT32" and (min_intensity is None or max_intensity is None):
        raise ValueError("When selecting UINT8 or UINT16 you need to specify minIntensity and maxIntensity.")
    if not interest_points:
        raise ValueError("no interest points defined, exiting.")
    labels = list(interest_points)
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    views = sorted(data.select_views(**view_selection) if view_selection else data.view_ids())
    regs = {v: data.model(*v) for v in views}
    vdims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in views}
    coeffs = None
    if intensity_n5_path is not None:
        coeffs = bint.view_coefficients(intensity_n5_path, intensity_n5_storage, intensity_n5_group,
                                        intensity_n5_dataset, views)
    lo = np.full(3, np.iinfo(np.int64).max, dtype=np.int64)
    hi = np.full(3, np.iinfo(np.int64).min, dtype=np.int64)
    for v in views:
        bmin, bmax = bf.transformed_bounding_box(vdims[v], regs[v])
        lo, hi = np.minimum(lo, bmin), np.maximum(hi, bmax)
    dims = [int(hi[d] - lo[d] + 1) for d in range(3)]
    bs = [int(b) for b in block_size]
    np_dt = {"FLOAT32": np.float32, "UINT16": np.uint16, "UINT8": np.uint8}[dt]
    od = native._NP2BS[np.dtype(np_dt)]
    is_zarr = storage.upper() == "ZARR"
    if is_zarr:
        store = bzarr.ZarrStore(out_path, create=True)
        store.create_array(n5_dataset, [1, 1] + dims[::-1], [1, 1] + bs[::-1], np.dtype(np_dt).name, "zstd")
    else:
        store = bn5.N5Store(out_path, create=True)
        store.create_dataset(n5_dataset, dims, bs, np_dt, "zstd")
    store.set_attributes(n5_dataset, {"offset": [int(v) for v in lo]})
    sink = _Sink(store, is_zarr, 0, 0)
    params = ctx.fuse_params(native.FUSE_AVG_BLEND, 1, od, 0, float(min_intensity or 0.0),
                             float(max_intensity if max_intensity is not None else 65535.0))

    base = os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")
    ips = _InterestPoints(bn5.N5Store(os.path.join(base, "interestpoints.n5")), views, labels, regs)
    blending = {v: bf.adjust_blending(regs[v]) for v in views}

    # super-blocks grouped by (viewsToFuse, viewsToUse): one set of MLS point lists per group
    compute = [bs[d] * int(block_scale[d]) for d in range(3)]
    groups = {}
    for gb in bf.grid_create(dims, compute, bs):
        off, size, _ = gb
        mn = lo + np.asarray(off, dtype=np.int64)
        fuse, use = nonrigid_views_for_block(vdims, regs, mn, mn + np.asarray(size) - 1, views)
        if fuse:
            groups.setdefault((tuple(fuse), tuple(use)), []).append(gb)
    written = []
    cpd = (native.NONRIGID_CP_DISTANCE,) * 3
    for (fuse, use), gbs in groups.items():
        nviews = {}
        for v in fuse:
            t, l = ips.targets(v, use)
            border, rng = blending[v]
            nviews[v] = dict(src_to_world=regs[v], vol_handle=0, blend_border=border, blend_range=rng,
                             full_dims=vdims[v], target_world_xyz=t, local_xyz=l)
        todo, attempt = list(gbs), 0
        while todo:
            attempt += 1
            if attempt > retries:
                raise RuntimeError(f"nonrigid-fusion: {len(todo)} block(s) still failing after {retries} attempts")
            failed = []
            for c0 in range(0, len(todo), blocks_per_call):
                chunk = todo[c0:c0 + blocks_per_call]
                try:
                    outs = _nonrigid_chunk(ctx, src, chunk, lo, fuse, nviews, vdims, params, cpd, coeffs)
                except native.BsError:
                    failed.extend(chunk)
                    continue
                for (off, size, gpos), blk in zip(chunk, outs):
                    sink.save(n5_dataset, blk, gpos)
                    written.append(tuple(gpos))
            todo = failed
    return written


def _nonrigid_chunk(ctx, src, chunk, bb_min, fuse, nviews, vdims, params, cpd, coeffs=None):
    """Fuse a list of super-blocks that share their views.  Each view's source window is the range its control-point
    grids map to over the chunk (+2 px for the n-linear taps), read from level s0 and uploaded as a windowed view.
    ``coeffs`` ({view: (a, b)}): each window is replaced by its float32 correction (s0 is full resolution, so the
    window voxel l sits at q = window_min + l)."""
    mins = [tuple(int(v) for v in bb_min + np.asarray(off, dtype=np.int64)) for off, _, _ in chunk]
    sizes = [tuple(int(v) for v in size) for _, size, _ in chunk]
    staged, gviews = [], []
    try:
        for v in fuse:
            nv = nviews[v]
            glo = np.full(3, np.inf)
            ghi = np.full(3, -np.inf)
            for mn, sz in zip(mins, sizes):
                g = ctx.nonrigid_debug_grid(nv, mn, sz, cpd).reshape(-1, 3)
                glo, ghi = np.minimum(glo, g.min(axis=0)), np.maximum(ghi, g.max(axis=0))
            dims = np.asarray(vdims[v], dtype=np.int64)
            wlo = np.maximum(np.floor(glo).astype(np.int64) - 2, 0)
            whi = np.minimum(np.ceil(ghi).astype(np.int64) + 2, dims - 1)
            if np.any(whi < wlo):
                continue                                  # the view's grids never reach its pixels in this chunk
            h = ctx.volume_upload(src.read_region(v, 0, wlo, whi - wlo + 1))
            if coeffs is not None:
                try:
                    hc = ctx.intensity_apply(h, vdims[v], np.eye(3, 4), *coeffs[v], window_min_xyz=wlo)
                finally:
                    ctx.volume_free(h)
                h = hc
            staged.append(h)
            gviews.append(dict(nv, vol_handle=h, window_min=tuple(int(x) for x in wlo)))
        if not gviews:
            return [np.zeros(tuple(s)[::-1], dtype=native._out_dtype(params)) for s in sizes]
        return ctx.nonrigid_fuse_blocks(gviews, mins, sizes, params, cpd)
    finally:
        for h in staged:
            ctx.volume_free(h)


# --------------------------------------------------------------------------------------------- match-interestpoints
# -rtp / --registrationTP: which timepoints are registered against each other (J/abstractcmdline/AbstractRegistration.java)
REGISTRATION_TPS = ("TIMEPOINTS_INDIVIDUALLY", "TO_REFERENCE_TIMEPOINT", "ALL_TO_ALL", "ALL_TO_ALL_WITH_RANGE")


def reference_timepoint(view_ids, reference_tp=None):
    """--referenceTP (J/abstractcmdline/AbstractRegistration.java:95-104): the timepoint of the first view in (tp, setup)
    order by default; a given timepoint must be the timepoint of one of ``view_ids``."""
    views = sorted(view_ids)
    if reference_tp is None:
        return int(views[0][0])
    if int(reference_tp) not in {v[0] for v in views}:
        raise ValueError("Specified reference timepoint is not part of the ViewIds that are processed.")
    return int(reference_tp)


def match_pairs(view_dims, registrations, view_ids, view_reg="OVERLAPPING_ONLY", registration_tp="TIMEPOINTS_INDIVIDUALLY",
                reference_tp=None, range_tp=5):
    """M2, M10: the view pairs (A, B), A < B in (tp, setup) order, that the -rtp constellation forms:
    TIMEPOINTS_INDIVIDUALLY pairs views of one timepoint, ALL_TO_ALL every two views, ALL_TO_ALL_WITH_RANGE views whose
    timepoint ids are at most ``range_tp`` apart, TO_REFERENCE_TIMEPOINT the pairs with at least one view at
    ``reference_tp`` (default: the first view's timepoint).  Then OVERLAPPING_ONLY keeps the pairs whose closed
    transformed bounding boxes (each view under its own registration) intersect, ALL_AGAINST_ALL keeps every pair."""
    vr = view_reg.upper()
    if vr not in ("OVERLAPPING_ONLY", "ALL_AGAINST_ALL"):
        raise ValueError(f"-vr {view_reg}")
    rtp = registration_tp.upper()
    if rtp not in REGISTRATION_TPS:
        raise NotImplementedError(f"-rtp {registration_tp} is not implemented")
    if int(range_tp) < 0:
        raise ValueError(f"--rangeTP {range_tp}: the range must not be negative")
    views = sorted(view_ids)
    ref = reference_timepoint(views, reference_tp) if views else None
    formed = {"TIMEPOINTS_INDIVIDUALLY": lambda ta, tb: ta == tb,
              "ALL_TO_ALL": lambda ta, tb: True,
              "ALL_TO_ALL_WITH_RANGE": lambda ta, tb: abs(ta - tb) <= int(range_tp),
              "TO_REFERENCE_TIMEPOINT": lambda ta, tb: ref in (ta, tb)}[rtp]
    boxes = {v: bf.transformed_bounding_box(view_dims[v], registrations[v]) for v in views}
    pairs = []
    for i, a in enumerate(views):
        for b in views[i + 1:]:
            if not formed(a[0], b[0]):
                continue
            if vr == "ALL_AGAINST_ALL" or np.all(np.minimum(boxes[a][1], boxes[b][1]) >= np.maximum(boxes[a][0], boxes[b][0])):
                pairs.append((a, b))
    return pairs


def match_tasks(pairs, labels, match_across_labels=False):
    """MatcherPairwiseTools.getTasksList: per pair (A, B) the label tasks (l, l), or every (la, lb) with
    --matchAcrossLabels; tasks are (viewA, labelA, viewB, labelB)."""
    out = []
    for a, b in pairs:
        if match_across_labels:
            out += [(a, la, b, lb) for la in labels for lb in labels]
        else:
            out += [(a, la, b, la) for la in labels]
    return out


def overlap_filter(world, dims_other, reg_other):
    """M3 (-ipfr OVERLAPPING_ONLY): mask of the world points inside the other view's closed transformed bounding box."""
    lo, hi = bf.transformed_bounding_box(dims_other, reg_other)
    return np.all((world >= lo) & (world <= hi), axis=1)


def _match_task(ctx, ips, task, vdims, regs, overlapping_only, significance, search_radius, num_neighbors, redundancy,
                model, ransac_kw):
    """One task: descriptors of both point sets on the device, the exhaustive search, the ratio test and RANSAC.
    Returns the inliers as an int64 (K, 2) array of (id in A, id in B)."""
    va, la, vb, lb = task
    empty = np.zeros((0, 2), dtype=np.int64)
    if (va, la) not in ips.world or (vb, lb) not in ips.world:
        return empty
    wa, wb = ips.world[(va, la)], ips.world[(vb, lb)]
    ia, ib = ips.ids[(va, la)], ips.ids[(vb, lb)]
    if overlapping_only:
        ka, kb = overlap_filter(wa, vdims[vb], regs[vb]), overlap_filter(wb, vdims[va], regs[va])
        wa, ia, wb, ib = wa[ka], ia[ka], wb[kb], ib[kb]
    ha = ctx.descriptors_build(wa, num_neighbors, redundancy)
    try:
        hb = ctx.descriptors_build(wb, num_neighbors, redundancy)
        try:
            best_b, best, second = ctx.descriptors_match(ha, hb, search_radius)
        finally:
            ctx.descriptors_free(hb)
    finally:
        ctx.descriptors_free(ha)
    cand = bm.ratio_test(best_b, best, second, significance)
    if len(cand) == 0:
        return empty
    pb = np.asarray(best_b)[cand].astype(np.int64)
    inl, _ = bm.ransac(wa[cand], wb[pb], model, **ransac_kw)
    return np.stack([ia[cand[inl]], ib[pb[inl]]], axis=1).astype(np.int64) if len(inl) else empty


class _MatchPoints:
    """The points of every (view, label) a matching run needs: ids and world positions (M1, as _InterestPoints)."""

    def __init__(self, store: bn5.N5Store, view_ids, labels, registrations):
        base = _InterestPoints(store, view_ids, labels, registrations)
        self.world = base.world
        self.ids = {k: np.array(sorted(base.index[k], key=base.index[k].get), dtype=np.int64) for k in base.index}
        self.corr = base.corr


def match_interestpoints(xml_path, ctx: Context, labels, method, significance=3.0, search_radius=None, redundancy=1,
                         num_neighbors=3, clear_correspondences=False, match_across_labels=False,
                         interestpoints_for_reg="ALL", view_reg="OVERLAPPING_ONLY", transformation_model="AFFINE",
                         regularization_model="RIGID", regularization_lambda=0.1, ransac_iterations=None,
                         ransac_max_error=None, ransac_min_inlier_ratio=0.1, ransac_min_num_inliers=12,
                         ransac_multi_consensus=False, registration_tp="TIMEPOINTS_INDIVIDUALLY", group_tiles=False,
                         group_illums=False, group_channels=False, split_timepoints=False, view_selection=None,
                         dry_run=False, shard=(0, 1), allgather=None, reference_tp=None, range_tp=5):
    """`./match-interestpoints -x dataset.xml -l beads -m PRECISE_TRANSLATION [-s 3.0] [-r 1] [-n 3] [--searchRadius r]
    [--clearCorrespondences] [--matchAcrossLabels] [-ipfr ALL|OVERLAPPING_ONLY] [-vr OVERLAPPING_ONLY|ALL_AGAINST_ALL]
    [-tm AFFINE] [-rm RIGID] [--lambda 0.1] [-rit 10000] [-rme 5.0] [-rmir 0.1] [-rmni 12]
    [-rtp TIMEPOINTS_INDIVIDUALLY|TO_REFERENCE_TIMEPOINT|ALL_TO_ALL|ALL_TO_ALL_WITH_RANGE] [--referenceTP t]
    [--rangeTP 5]`, the non-grouped branch of J/SparkGeometricDescriptorMatching.java:161-342 and the save at :512-545:
    the view pairs are those of the -rtp constellation (``match_pairs``; across timepoints for every name but
    TIMEPOINTS_INDIVIDUALLY); for every task (view pair x label pair) the points are read from interestpoints.n5 and
    mapped to world (M1), optionally filtered to the partner's box (M3);
    descriptors and the exhaustive A -> B search run on the device (bs_descriptors_build / bs_descriptors_match), the
    ratio test (M6), RANSAC and its filter (M7, M8) on the host; the inliers become correspondences of both views (M9),
    written for every selected view x label unless ``dry_run``.  The XML is not touched.
    Returns {(viewA, labelA, viewB, labelB): int64 (K, 2) id pairs} for every task.

    Multi-GPU: rank r of w (``shard``) takes tasks[r::w]; ``allgather(obj) -> [obj of every rank]`` merges the results
    and rank 0 writes.  FAST_ROTATION, FAST_TRANSLATION, ICP, grouping, an -rtp name other than the four above and
    -rmc raise NotImplementedError."""
    m = method.upper()
    if m in ("FAST_ROTATION", "FAST_TRANSLATION", "ICP"):
        raise NotImplementedError(f"match-interestpoints -m {m} is not implemented")
    if m != "PRECISE_TRANSLATION":
        raise ValueError(f"-m {method}")
    for flag, on in (("--groupTiles", group_tiles), ("--groupIllums", group_illums), ("--groupChannels", group_channels),
                     ("--splitTimepoints", split_timepoints), ("-rmc", ransac_multi_consensus),
                     (f"-rtp {registration_tp}", registration_tp.upper() not in REGISTRATION_TPS)):
        if on:
            raise NotImplementedError(f"match-interestpoints {flag} is not implemented")
    ipfr = interestpoints_for_reg.upper()
    if ipfr not in ("ALL", "OVERLAPPING_ONLY"):
        raise ValueError(f"-ipfr {interestpoints_for_reg}")
    k = int(num_neighbors) + int(redundancy)
    if int(num_neighbors) < 3 or int(redundancy) < 0 or k > native.MATCH_MAX_NEIGHBORS:
        raise ValueError(f"-n {num_neighbors} -r {redundancy}: need n >= 3, r >= 0, n + r <= {native.MATCH_MAX_NEIGHBORS}")
    labels = list(labels)
    if not labels:
        raise ValueError("no interest point labels given")
    if ransac_iterations is None:                      # J/SparkGeometricDescriptorMatching.java:180-189
        ransac_iterations = 10000
    if ransac_max_error is None:
        ransac_max_error = 5.0
    model = bm.Model(transformation_model, regularization_model, regularization_lambda)
    ransac_kw = dict(iterations=int(ransac_iterations), max_error=float(ransac_max_error),
                     min_inlier_ratio=float(ransac_min_inlier_ratio), min_num_inliers=int(ransac_min_num_inliers))

    data = SpimData2.load(xml_path)
    views = sorted(data.select_views(**view_selection) if view_selection else data.view_ids())
    regs = {v: data.model(*v) for v in views}
    vdims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in views}
    tasks = match_tasks(match_pairs(vdims, regs, views, view_reg, registration_tp, reference_tp, range_tp), labels,
                        match_across_labels)
    base = os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")
    store = bn5.N5Store(os.path.join(base, "interestpoints.n5"))
    ips = _MatchPoints(store, views, labels, regs)

    rank, world = shard
    results = {}
    for task in tasks[rank::world]:
        results[task] = _match_task(ctx, ips, task, vdims, regs, ipfr == "OVERLAPPING_ONLY", float(significance),
                                    search_radius, int(num_neighbors), int(redundancy), model, ransac_kw)
    if world > 1:
        merged = {}
        for part in allgather(results):
            merged.update(part)
        results = {t: merged[t] for t in tasks if t in merged}
        if rank != 0:
            return results
    if dry_run:
        return results
    write_match_correspondences(store, ips, views, labels, results, clear_correspondences)
    return results


def write_match_correspondences(store, ips, views, labels, results, clear=False):
    """M9: each inlier (idA, idB) of task (A, la, B, lb) adds (idA, B, lb, idB) to (A, la) and (idB, A, la, idA) to
    (B, lb), appended to the stored rows (replacing them with ``clear``) without duplicates, sorted by (id, partner tp,
    partner setup, partner label, partner id); every selected view x label that has points is written."""
    rows = {}
    for v in views:
        for lab in labels:
            if (v, lab) in ips.world:
                rows[(v, lab)] = set() if clear else {(int(a), tuple(pv), pl, int(b)) for a, pv, pl, b in ips.corr[(v, lab)]}
    for (va, la, vb, lb), pairs in results.items():
        for ida, idb in np.asarray(pairs, dtype=np.int64).reshape(-1, 2):
            rows[(va, la)].add((int(ida), tuple(vb), lb, int(idb)))
            rows[(vb, lb)].add((int(idb), tuple(va), la, int(ida)))
    for (v, lab), rs in sorted(rows.items()):
        ordered = sorted(rs, key=lambda r: (r[0], r[1][0], r[1][1], r[2], r[3]))
        store.write_correspondences(f"tpId_{v[0]}_viewSetupId_{v[1]}/{lab}", ordered)


# --------------------------------------------------------------------------------------------- solver
def solver(xml_path, ctx: Context, source, labels=None, label_weights=None, method="ONE_ROUND_SIMPLE",
           transformation_model="AFFINE", regularization_model="RIGID", regularization_lambda=0.1, max_error=5.0,
           max_iterations=10000, max_plateau_width=200, relative_threshold=3.5, absolute_threshold=7.0, fixed_views=None,
           disable_fixed_views=False, group_tiles=None, group_illums=None, group_channels=None, split_timepoints=None,
           registration_tp="TIMEPOINTS_INDIVIDUALLY", view_selection=None, dry_run=False, reference_tp=None):
    """`./solver -x dataset.xml -s STITCHING|IP [-l beads [-lw 1.0]] [--method ONE_ROUND_SIMPLE|ONE_ROUND_ITERATIVE]
    [-tm AFFINE] [-rm RIGID] [--lambda 0.1] [--maxError 5.0] [--maxIterations 10000] [--maxPlateauwidth 200]
    [--relativeThreshold 3.5] [--absoluteThreshold 7.0] [-fv 'tp,setup' | --disableFixedViews] [--groupTiles]
    [--groupIllums] [--groupChannels] [--splitTimepoints]
    [-rtp TIMEPOINTS_INDIVIDUALLY|TO_REFERENCE_TIMEPOINT|ALL_TO_ALL|ALL_TO_ALL_WITH_RANGE] [--referenceTP t] [--dryRun]`
    (J/Solver.java:161-432): global optimisation of the stored stitching results or interest-point correspondences.
    The matches are built and the tiles pre-aligned on the host; the relaxation runs on the device (bs_solve_tiles).  Every view of a solved tile gets the tile's model as
    a new first <ViewTransform>; the XML is saved (with a ~1 backup) unless ``dry_run``.  Returns dict(models={view:
    3 x 4}, removed=[(views A, views B)] (ONE_ROUND_ITERATIVE), stats) -- stats holds iterations, the final error,
    skipped fits, stale stitching results and the views without links, which keep their registration.  -rtp only
    chooses the automatic fixed views (``solver.fixed_views_auto``); every stored link between selected views is used.

    TWO_ROUND_SIMPLE / TWO_ROUND_ITERATIVE and an -rtp name other than the four above raise NotImplementedError."""
    return bsolver.run(xml_path, ctx, source, labels, label_weights, method, transformation_model, regularization_model,
                       regularization_lambda, max_error, max_iterations, max_plateau_width, relative_threshold,
                       absolute_threshold, fixed_views, disable_fixed_views, group_tiles, group_illums, group_channels,
                       split_timepoints, registration_tp, view_selection, dry_run, reference_tp)


# --------------------------------------------------------------------------------------------- resave
RESAVE_COMPRESSION = {"zstd": "zstd", "zstandard": "zstd", "gzip": "gzip", "raw": "raw"}


# --------------------------------------------------------------------------------------------- intensity correction
def match_intensities(xml_path, ctx: Context, out_path, num_coefficients=(8, 8, 8), render_scale=0.25, min_threshold=1.0,
                      max_threshold=float("nan"), min_num_candidates=1000, method="RANSAC", num_iterations=1000,
                      max_epsilon=5.1, min_inlier_ratio=0.1, min_num_inliers=10, max_trust=3.0, view_selection=None,
                      dry_run=False, chunk_points=0):
    """`./match-intensities -x dataset.xml -o matches.n5 [--numCoefficients 8,8,8] [--renderScale 0.25] ...`
    (J/SparkIntensityMatching.java:84-190): for every selected pair i < j whose transformed bounds intersect (across
    timepoints), render the intersection at ``render_scale`` on the device, bucket the overlapping intensities by
    (cell of A, cell of B), run RANSAC on the device and the filter on the host, and write coefficientsSize plus the
    accepted inliers per (pair, cellA, cellB) under ``out_path`` (intensity.MatchesIO).  Returns
    {(viewA, viewB): [(cellA, cellB, inliers)]}.  ``dry_run`` computes the matches and writes nothing."""
    if str(method).upper() == "HISTOGRAM":
        raise NotImplementedError("match-intensities --method HISTOGRAM")
    if str(method).upper() != "RANSAC":
        raise ValueError(f"unknown method {method!r}")
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    views = data.select_views(**view_selection) if view_selection else data.view_ids()
    n_cells = tuple(int(v) for v in num_coefficients)
    regs = {v: data.model(*v) for v in views}
    dims = {v: tuple(int(d) for d in data.setups[v[1]].size) for v in views}
    bounds = {v: bint.view_bounds(dims[v], regs[v]) for v in views}
    todo = bint.pairs(views, bounds)
    io = None
    if not dry_run:
        io = bint.MatchesIO(out_path, create=True)
        io.write_coefficients_size(n_cells)
    levels = {}
    for v in views:
        factors, mts = src.mipmap_info(v)
        lvl = bint.render_level(regs[v], render_scale, factors, mts)
        levels[v] = (lvl, mts[lvl])
    resident = {}
    out = {}
    try:
        for a, b in todo:
            for v in (a, b):
                if v not in resident:
                    resident[v] = ctx.volume_upload(src.read_volume(v, levels[v][0]))
            lo = np.maximum(bounds[a][0], bounds[b][0])
            hi = np.minimum(bounds[a][1], bounds[b][1])
            rmin, rmax = bint.render_range(lo, hi, render_scale)
            va = bint.device_view(resident[a], regs[a], levels[a][1], dims[a], n_cells)
            vb = bint.device_view(resident[b], regs[b], levels[b][1], dims[b], n_cells)
            cells, _ = bint.match_pair(ctx, va, vb, render_scale, rmin, rmax, min_threshold, max_threshold,
                                       min_num_candidates, num_iterations, max_epsilon, min_inlier_ratio,
                                       min_num_inliers, max_trust, chunk_points)
            out[(a, b)] = cells
            if io is not None:
                io.write(a, b, cells)
            # a view's volume stays resident until its last pair
            for v in (a, b):
                if not any(v in p for p in todo[todo.index((a, b)) + 1:]):
                    ctx.volume_free(resident.pop(v))
    finally:
        for h in resident.values():
            ctx.volume_free(h)
    return out


def solve_intensities(xml_path, out_path, matches_path, num_coefficients=(8, 8, 8), max_iterations=1000, storage=None,
                      group="", dataset="intensity", view_selection=None):
    """`./solve-intensities -x dataset.xml --matchesPath matches.n5 -o coefficients.n5 [-s N5|ZARR]
    [--intensityN5Group ""] [--intensityN5Dataset intensity]` (J/IntensitySolver.java:50-123): read the pairwise
    matches of every selected pair, solve one 1-D model per (view, cell) on the host (intensity.solve) and write each
    view's coefficients to `{group}/setup{s}/timepoint{t}/{dataset}`.  A ``num_coefficients`` that differs from the one
    stored with the matches warns and the stored one is used.  Returns {view: (a, b)}."""
    storage = bint.guess_storage(out_path, storage)
    data = SpimData2.load(xml_path)
    views = data.select_views(**view_selection) if view_selection else data.view_ids()
    io = bint.MatchesIO(matches_path)
    stored = io.read_coefficients_size()
    bint.check_coefficients_size(stored, num_coefficients)
    matches = {}
    for i, a in enumerate(views):
        for b in views[i + 1:]:
            m = io.read(a, b)
            if m is not None:
                matches[(a, b)] = m
    coeffs = bint.solve(views, stored, matches, max_iterations)
    bint.write_coefficients(out_path, storage, group, dataset, coeffs)
    return coeffs


def propose_mipmaps(size_xyz, voxel_size_xyz=(1.0, 1.0, 1.0)):
    """Resave_HDF5.proposeMipmaps / bdv ProposeMipmaps restated (recalled, PARITY_GAPS R5): starting at (1, 1, 1), while
    the largest axis of the current level is over 256 pixels, double the factor of every axis whose voxel size is at
    most twice the smallest one (and that is still over 1 pixel), so anisotropic z catches up.  Absolute factors."""
    vs = [float(v) for v in voxel_size_xyz]
    vs = [v / min(vs) for v in vs]
    size = [int(v) for v in size_xyz]
    res, out = [1, 1, 1], []
    while True:
        out.append(tuple(res))
        if max(size) <= 256:
            return out
        grow = [d for d in range(3) if vs[d] <= 2.0 * min(vs) and size[d] > 1]
        for d in grow:
            res[d] *= 2
            vs[d] *= 2.0
            size[d] //= 2


def parse_downsampling(downsampling):
    """`-ds "1,1,1; 2,2,1; 4,4,1"` (or a list of triples): absolute factors per level.  The first must be 1,1,1
    (J/SparkResaveN5.java:211); each level must be 1x or 2x the previous one per axis, the steps bs_downsample takes
    (PARITY_GAPS R4).  Anything else raises ValueError."""
    if isinstance(downsampling, str):
        steps = [tuple(int(v) for v in s.split(",")) for s in downsampling.split(";") if s.strip()]
    else:
        steps = [tuple(int(v) for v in s) for s in downsampling]
    if not steps or any(len(s) != 3 for s in steps):
        raise ValueError(f"-ds {downsampling}: need x,y,z triples")
    if steps[0] != (1, 1, 1):
        raise ValueError("First downsampling step must be full resolution [1,1,...1], stopping.")
    for a, b in zip(steps, steps[1:]):
        if any(b[d] not in (a[d], 2 * a[d]) for d in range(3)):
            raise ValueError(f"-ds {downsampling}: step {b} after {a} is not 1x or 2x per axis")
    return steps


def _voxel_size(data, setup):
    for vs in data.root.find("SequenceDescription").find("ViewSetups").findall("ViewSetup"):
        if int(vs.findtext("id")) == int(setup):
            txt = vs.findtext("voxelSize/size")
            return tuple(float(v) for v in txt.split()) if txt else (1.0, 1.0, 1.0)
    return (1.0, 1.0, 1.0)


def resave(xml_path, ctx: Context, xml_out=None, n5=False, out_path=None, block_size=(128, 128, 64),
           block_scale=(16, 16, 1), downsampling=None, compression="zstd", compression_level=None, dry_run=False,
           shard=(0, 1), barrier=None, retries=5):
    """`./resave -x dataset.xml [-xo out.xml] [--N5] [-o dataset.ome.zarr] [--blockSize 128,128,64]
    [--blockScale 16,16,1] [-ds "1,1,1; 2,2,1; 4,4,1"] [-c Zstandard] [-cl 3] [--dryRun]` (J/SparkResaveN5.java:80-455):
    copy every view of the XML, through whichever loader it has, into a new OME-ZARR container (default
    `dataset.ome.zarr` next to ``xml_out``) or, with ``n5``, a BDV-N5 one (`dataset.n5`), with a multi-resolution
    pyramid, and point the XML's ImageLoader at it (``xml_out``, default the input XML, saved with a ~1 backup).

    Work is cut into compute blocks of ``block_size * block_scale`` on storage-block boundaries (Grid.create).  Each
    block's s0 is read once and uploaded; the leading pyramid levels it lies on whole storage blocks of (block_scale a
    multiple of the level's factors) are derived on the device (bs_downsample) while it is resident, so no rank ever
    writes part of a storage block.  The other levels are built from the stored level l-1 after ``barrier()``; with the
    default block_scale (16, 16, 1) that is every level of a pyramid that halves z.  ``downsampling``: absolute factors
    (parse_downsampling); default propose_mipmaps of the first view's setup.

    The output container must not be, contain or lie inside the input one (ValueError): re-saving a dataset next to its
    own XML in the format it already has would overwrite the data being read.

    Multi-GPU: rank 0 creates every dataset and writes all metadata, then ``barrier()`` (required when w > 1) lets the
    other ranks in; rank r of w takes compute blocks [r::w]; rank 0 writes the XML after a last ``barrier()``.
    ``dry_run`` stops after planning and writes nothing.  Returns dict(out_path, xml_out, downsamplings,
    compute_blocks)."""
    comp = RESAVE_COMPRESSION.get(str(compression).lower())
    if comp is None:
        raise NotImplementedError(f"compression {compression} (writable: Zstandard, Gzip, Raw)")
    rank, world = shard
    if world > 1 and barrier is None:
        raise ValueError("resave with more than one rank needs barrier(): rank 0 creates the datasets first")
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    views = data.view_ids()
    if not views:
        raise ValueError("No views to resave.")
    xml_out = xml_out or xml_path
    if out_path is None:
        out_path = os.path.join(os.path.dirname(os.path.abspath(xml_out)), "dataset.n5" if n5 else "dataset.ome.zarr")
    a = os.path.realpath(out_path)
    for root in src.roots:
        b = os.path.realpath(root)
        if a == b or a.startswith(b + os.sep) or b.startswith(a + os.sep):
            raise ValueError(f"resave output {out_path} overlaps the input container {root}; choose another -o / -xo")
    bs = [int(v) for v in block_size]
    compute = [bs[d] * int(block_scale[d]) for d in range(3)]
    if downsampling is None:     # N5ApiTools.mipMapInfoToDownsamplings(proposeMipmaps(...)): one pyramid for all views
        first = views[0]
        downsampling = propose_mipmaps(src.level_dims(first, 0), _voxel_size(data, first[1]))
    steps = parse_downsampling(downsampling)
    # every view is checked before anything is created
    meta = {}
    for v in views:
        dims0, dt = src.level_dims(v, 0), src.level_dtype(v, 0)
        if dt not in ("uint8", "uint16", "float32"):
            raise NotImplementedError(f"resave of {dt} view {v} (bs_downsample takes uint8, uint16, float32)")
        if any(int(dims0[d]) // steps[-1][d] < 1 for d in range(3)):
            raise ValueError(f"view {v} of {tuple(dims0)} voxels is too small for the downsampling {steps[-1]}")
        meta[v] = (dims0, dt)
    grid = [(v, gb) for v in views for gb in bf.grid_create(list(meta[v][0]), compute, bs)]
    plan = dict(out_path=out_path, xml_out=xml_out, downsamplings=steps, compute_blocks=len(grid))
    if dry_run:
        return plan

    # ---- datasets and metadata of every view, created once by rank 0 (setupBdvDatasetsN5 / setupBdvDatasetsOMEZARR,
    # on the driver before any worker runs, J/SparkResaveN5.java:222-262)
    if rank == 0:
        store = bn5.N5Store(out_path, create=True) if n5 else bzarr.ZarrStore(out_path, create=True)
        for v in views:
            dims0, dt = meta[v]
            if n5:
                bn5.set_bdv_attributes(store, v[1], v[0], steps, dt)
                for li, f in enumerate(steps):
                    store.create_dataset(bn5.bdv_dataset(v[1], v[0], li), [int(dims0[d]) // f[d] for d in range(3)], bs,
                                         np.dtype(dt), comp, compression_level)
            else:
                bzarr.create_multiscale_group(store, _resave_group(v), dims0, dt, bs, steps, comp, compression_level)
    if world > 1:
        barrier()                                    # the container exists on every rank
    store = bn5.N5Store(out_path) if n5 else bzarr.ZarrStore(out_path)
    vols = {}
    for v in views:
        dims0, dt = meta[v]
        levels = [dict(dataset=bn5.bdv_dataset(v[1], v[0], li) if n5 else f"{_resave_group(v)}/{li}",
                       dimensions=[int(dims0[d]) // f[d] for d in range(3)], absoluteDownsampling=list(f),
                       relativeDownsampling=[f[d] // (steps[li - 1][d] if li else 1) for d in range(3)])
                  for li, f in enumerate(steps)]
        vols[v] = (_Sink(store, not n5, 0, 0), levels, np.dtype(dt))

    # levels kept resident: the leading ones every compute block lies on whole storage blocks of
    n_res = 1
    while n_res < len(steps) and all(compute[d] % (steps[n_res][d] * bs[d]) == 0 for d in range(3)):
        n_res += 1

    # ---- s0 (+ resident levels), compute blocks [r::w], RetryTrackerSpark policy
    todo, attempt = grid[rank::world], 0
    while todo:
        attempt += 1
        if attempt > retries:
            raise RuntimeError(f"resave: {len(todo)} block(s) still failing after {retries} attempts")
        failed = []
        for v, gb in todo:
            sink, levels, dt = vols[v]
            off, size, _ = gb
            try:
                h = ctx.volume_upload(src.read_region(v, 0, off, size))
            except native.BsError:
                failed.append((v, gb))
                continue
            try:
                _write_resident_levels(ctx, h, gb, sink, levels[:n_res], bs, dt)
            except native.BsError:
                failed.append((v, gb))
        todo = failed
    _pyramid_from_stored(ctx, [vols[v] for v in views], n_res, compute, bs, shard, retries, barrier)

    if world > 1:
        barrier()                                    # every rank has written its blocks
    if rank == 0:
        data.set_image_loader("bdv.n5" if n5 else "bdv.multimg.zarr", out_path, xml_out,
                              {v: (_resave_group(v), 0, 0) for v in views} if not n5 else None)
        data.save(xml_out)
    return plan


def _resave_group(view):
    """The OME-ZARR group of a resaved view (PARITY_GAPS R3)."""
    return f"s{view[1]}-t{view[0]}.zarr"


# --------------------------------------------------------------------------------------------- downsample
DOWNSAMPLE_DTYPES = ("uint8", "uint16", "float32")          # what bs_downsample takes


def parse_downsample_steps(downsampling):
    """`-ds "2,2,1; 2,2,1; 2,2,2"` (or a list of triples): the consecutive steps of `downsample`, each RELATIVE to the
    level before.  A step must be 1 or 2 per axis (PARITY_GAPS U1); anything else raises ValueError."""
    if isinstance(downsampling, str):
        steps = [tuple(int(v) for v in s.split(",")) for s in downsampling.split(";") if s.strip()]
    else:
        steps = [tuple(int(v) for v in s) for s in downsampling]
    if not steps or any(len(s) != 3 for s in steps):
        raise ValueError(f"-ds {downsampling}: need x,y,z triples")
    for s in steps:
        if any(v not in (1, 2) for v in s):
            raise ValueError(f"-ds {downsampling}: step {s} is not 1 or 2 per axis")
    return steps


class _NonEmptySink(_Sink):
    """N5Utils.saveNonEmptyBlock (J/SparkDownsample.java:176): the storage blocks of a saved block whose voxels are all
    0 are not written, so they read back as 0 (PARITY_GAPS U2)."""

    def __init__(self, store, is_zarr, block_size):
        super().__init__(store, is_zarr, 0, 0)
        self.bs = [int(v) for v in block_size]

    def save(self, dataset, block, grid_pos):
        for off, size, gpos in _storage_cells(((0, 0, 0), block.shape[::-1], grid_pos), self.bs):
            part = block[off[2]:off[2] + size[2], off[1]:off[1] + size[1], off[0]:off[0] + size[0]]
            if part.any():
                super().save(dataset, np.ascontiguousarray(part), gpos)


def _downsample_input(n5_path, storage, dataset):
    """(store, is_zarr, dims xyz, block size xyz, dtype name, create(dataset, dims xyz)) of the input of `downsample`
    (PARITY_GAPS U3); ``create`` makes a dataset with the input's block size, data type and compression."""
    if storage.upper() == "ZARR":
        store = bzarr.ZarrStore(n5_path)
        m = store.array_meta(dataset)
        shape = [int(v) for v in m["shape"]]
        if not (len(shape) == 3 or (len(shape) == 5 and shape[:2] == [1, 1])):
            raise ValueError(f"{dataset}: Zarr shape {shape} is neither (z, y, x) nor (1, 1, z, y, x)")
        lead = shape[:-3]
        return (store, True, shape[-3:][::-1], [int(v) for v in m["chunks"][-3:][::-1]],
                np.dtype(m["dtype"]).newbyteorder("=").name,
                lambda ds, dims: store.create_array_like(ds, dataset, lead + list(dims)[::-1]))
    if storage.upper() != "N5":
        raise ValueError(f"-s {storage} (N5 or ZARR)")
    store = bn5.N5Store(n5_path)
    a = store.dataset_attributes(dataset)
    if len(a["dimensions"]) != 3:
        raise ValueError(f"{dataset}: {len(a['dimensions'])}-D N5 dataset, downsample takes 3-D ones")
    if a["compression"]["type"] not in ("raw", "gzip", "zstd"):
        raise NotImplementedError(f"{dataset}: N5 compression {a['compression']['type']} (writable: raw, gzip, zstd)")
    return (store, False, [int(v) for v in a["dimensions"]], [int(v) for v in a["blockSize"]], a["dataType"],
            lambda ds, dims: store.set_attributes(ds, {"dimensions": list(dims), "blockSize": a["blockSize"],
                                                       "dataType": a["dataType"], "compression": a["compression"]}))


def downsample(n5_path, ctx: Context, dataset_in, datasets_out, downsampling, storage="N5", block_scale=(1, 1, 1),
               dry_run=False, shard=(0, 1), barrier=None, retries=5):
    """`./downsample -i fused.n5 -di /ch0/s0 -do "/ch0/s1; /ch0/s2" -ds "2,2,1; 2,2,2" [-s N5|ZARR] [--blockScale 1,1,1]`
    (J/SparkDownsample.java:60-190): pyramid levels for an existing dataset, e.g. the single one nonrigid-fusion writes.
    Level l (``datasets_out[l-1]``) is ``downsampling[l-1]`` applied to level l-1 (``dataset_in`` for l = 1) by the
    device 2x step (bs_downsample, LazyHalfPixelDownsample2x per axis whose step is 2; parse_downsample_steps).  Each
    output gets the input's blockSize, dataType and compression and dims in_dims // step (:126-139); it is computed in
    blocks of Grid.create(out dims, blockSize * block_scale, blockSize) (:141-147) and storage blocks that come out all
    0 are not written (saveNonEmptyBlock, :176).  When those compute blocks also cover whole storage blocks of the next
    levels, the next levels are derived from each one while it is on the device instead of re-read from the container.

    N5 3-D datasets and Zarr arrays of shape (z, y, x) or (1, 1, z, y, x) -- the layout `nonrigid_fusion(...,
    storage="ZARR")` writes; any other shape raises ValueError.  uint8, uint16 and float32; other types raise
    NotImplementedError.  A step count that differs from the output count, or an output dim below 1, raises ValueError.

    Multi-GPU: rank 0 creates the datasets; rank r of w (``shard``) takes blocks [r::w] of each level and ``barrier()``
    (required when w > 1) runs before each level, so that the level it reads is complete.  ``dry_run`` returns the
    planned [(dataset, dims xyz)] and writes nothing.  Returns the list of datasets written."""
    if isinstance(datasets_out, str):
        datasets_out = [s.strip() for s in datasets_out.split(";") if s.strip()]
    datasets_out = list(datasets_out)
    steps = parse_downsample_steps(downsampling)
    if len(steps) != len(datasets_out):
        raise ValueError(f"{len(datasets_out)} output dataset(s) for {len(steps)} downsampling step(s): give as many "
                         f"-do as -ds")
    if len({dataset_in.strip("/")} | {d.strip("/") for d in datasets_out}) != len(datasets_out) + 1:
        raise ValueError(f"-di {dataset_in} / -do {datasets_out}: every dataset must be a different one")
    rank, world = shard
    if world > 1 and barrier is None:
        raise ValueError("downsample with more than one rank needs barrier(): rank 0 creates the datasets first")
    store, is_zarr, dims, bs, dt, create = _downsample_input(n5_path, storage, dataset_in)
    if dt not in DOWNSAMPLE_DTYPES:
        raise NotImplementedError(f"downsample of {dt} dataset {dataset_in} (bs_downsample takes uint8, uint16, float32)")
    levels = [dict(dataset=dataset_in, dimensions=dims, relativeDownsampling=[1, 1, 1])]
    for ds, step in zip(datasets_out, steps):
        cur = [levels[-1]["dimensions"][d] // step[d] for d in range(3)]
        if min(cur) < 1:
            raise ValueError(f"{ds}: {levels[-1]['dimensions']} // {list(step)} = {cur} has an empty axis")
        levels.append(dict(dataset=ds, dimensions=cur, relativeDownsampling=list(step)))
    plan = [(lv["dataset"], tuple(lv["dimensions"])) for lv in levels[1:]]
    if dry_run:
        return plan

    if rank == 0:
        for lv in levels[1:]:
            create(lv["dataset"], lv["dimensions"])
    compute = [bs[d] * int(block_scale[d]) for d in range(3)]
    # the levels after s1 whose storage blocks every compute block of s1 covers whole stay on the device
    resident, acc = 1, [1, 1, 1]
    while resident < len(steps):
        acc = [acc[d] * steps[resident][d] for d in range(3)]
        if any(compute[d] % (acc[d] * bs[d]) for d in range(3)):
            break
        resident += 1
    # the barrier before level 1 also lets every rank in once rank 0 has created the datasets
    _pyramid_from_stored(ctx, [(_NonEmptySink(store, is_zarr, bs), levels, np.dtype(dt))], 1, compute, bs, shard,
                         retries, barrier, resident)
    return datasets_out


# --------------------------------------------------------------------------------------------- clear-interestpoints
def clear_interestpoints(xml_path, correspondences_only=False, dry_run=False):
    """`./clear-interestpoints -x dataset.xml [--correspondencesOnly] [--dryRun]` (J/ClearInterestPoints.java): returns
    {view: {label: (interest points, correspondences)}} of every view with interest points in the XML, counted before
    anything is cleared.  Default: <ViewInterestPoints> is emptied, the XML saved (with a ~1 backup) and the whole
    `interestpoints.n5` next to it removed.  ``correspondences_only``: every view's and label's correspondences become
    the empty list (PARITY_GAPS N1: {0} data, empty idMap); the points and the XML stay.  ``dry_run``: counts only."""
    data = SpimData2.load(xml_path)
    base = os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")
    root = os.path.join(base, "interestpoints.n5")
    store = bn5.N5Store(root) if os.path.isdir(root) else None

    def count(path):
        dims = store.get_attributes(path).get("dimensions", [0]) if store is not None else [0]
        return int(dims[1]) if len(dims) == 2 else 0

    report = {}
    for v, labels in sorted(data.interest_points().items()):
        report[v] = {lab: (count(e["path"].rstrip("/") + "/interestpoints/loc"),
                          count(e["path"].rstrip("/") + "/correspondences/data"))
                     for lab, e in sorted(labels.items())}
    if dry_run:
        return report
    if correspondences_only:
        store = store or bn5.N5Store(root, create=True)
        for v, labels in sorted(data.interest_points().items()):
            for e in labels.values():
                store.write_correspondences(e["path"], [])
    else:
        data.clear_interest_points()
        data.save(xml_path)
        shutil.rmtree(root, ignore_errors=True)
    return report


# --------------------------------------------------------------------------------------------- clear-registrations
def clear_registrations(xml_path, keep=None, remove=None, view_selection=None, dry_run=False):
    """`./clear-registrations -x dataset.xml (--keep N | --remove N) [view selection] [--dryRun]`
    (J/ClearRegistrations.java): ``remove`` N drops the first N <ViewTransform>s of each selected view (the most
    recently applied, e.g. a solve), ``keep`` N drops from the front until N remain; a view with fewer is not an error.
    Exactly one of them, >= 0, or ValueError.  ``view_selection``: keyword arguments of SpimData2.select_views (default
    all views; PARITY_GAPS U5).  The XML is saved (with a ~1 backup) unless ``dry_run``.  Returns {view: [(name,
    3 x 4 affine)]} of the removed transforms, first removed first."""
    if (keep is None) == (remove is None) or (keep is not None and int(keep) < 0) or (remove is not None and int(remove) < 0):
        raise ValueError("Please specify --keep OR --remove as >=0.")
    data = SpimData2.load(xml_path)
    views = data.select_views(**view_selection) if view_selection else data.view_ids()
    removed = {}
    for v in views:
        n = len(data.registrations[v])
        drop = min(int(remove), n) if remove is not None else max(n - int(keep), 0)
        removed[v] = [data.remove_first_registration(v) for _ in range(drop)]
    if not dry_run:
        data.save(xml_path)
    return removed


# --------------------------------------------------------------------------------------------- transform-points
# TransformPoints keeps a CSV line when its trimmed text matches [\p{Space}*[-]*\d+\.?\d*\p{Space}*\,?]+ -- in Java
# one character class (the nested [-] is a union): whitespace, '*', '-', digits, '+', '.', '?' and ','
_CSV_POINT = re.compile(r"[ \t\n\x0b\f\r*\-0-9+.?,]+")
_JAVA_TRIM = "".join(chr(c) for c in range(33))                 # String.trim strips every char <= ' '


def _csv_doubles(text):
    """Import.csvStringToDoubleArray: split at ',' (trailing empty fields dropped, as String.split does), parse each."""
    parts = text.split(",")
    while parts and parts[-1] == "":
        parts.pop()
    return [float(p.strip(_JAVA_TRIM)) for p in parts]


def transform_points(xml_path, view, points=None, csv_in=None, csv_out=None):
    """`./transform-points -x dataset.xml -vi '0,5' [--csvIn in.csv] [-p x,y,z ...] [--csvOut out.csv]`
    (J/TransformPoints.java): map pixel coordinates of ``view`` ((tp, setup) or 'tp,setup') to world coordinates with
    its full registration model.  Points come from ``csv_in`` -- only lines whose trimmed text matches upstream's
    character-class pattern; others, such as `1e-5` or text, are ignored (PARITY_GAPS U6) -- and then from ``points``
    (`-p` strings 'x,y,z' or triples).  A point takes the first three values of its line.  No points raises ValueError.
    Writes `x,y,z` lines in Java's Double.toString format (java_double, PARITY_GAPS U7) to ``csv_out``, or to stdout.
    Returns the (n, 3) float64 world coordinates."""
    rows = []
    if csv_in is not None:
        with open(csv_in) as f:
            for line in f.read().splitlines():
                s = line.strip(_JAVA_TRIM)
                if s and _CSV_POINT.fullmatch(s):
                    rows.append(_csv_doubles(s))
    for p in points or ():
        if isinstance(p, str):
            if p.strip(_JAVA_TRIM):
                rows.append(_csv_doubles(p))
        else:
            rows.append([float(v) for v in p])
    if not rows:
        raise ValueError("No points defined (use either --csv and/or -p), stopping.")
    if any(len(r) < 3 for r in rows):
        raise ValueError(f"a point needs x,y,z: {next(r for r in rows if len(r) < 3)}")
    data = SpimData2.load(xml_path)
    v = tuple(int(t) for t in view.split(",")) if isinstance(view, str) else tuple(int(t) for t in view)
    if v not in data.registrations:
        raise ValueError(f"view {v} (timepoint, setup) is not in {xml_path}")
    M = data.model(*v)
    X = np.array([r[:3] for r in rows], dtype=np.float64)
    # AffineTransform3D.apply, term by term in its order
    W = np.stack([X[:, 0] * M[i, 0] + X[:, 1] * M[i, 1] + X[:, 2] * M[i, 2] + M[i, 3] for i in range(3)], axis=1)
    lines = [",".join(java_double(c) for c in w) for w in W]
    if csv_out is None:
        for line in lines:
            print(line)
    else:
        with open(csv_out, "w") as f:
            f.writelines(line + "\n" for line in lines)
    return W


# --------------------------------------------------------------------------------------------- split-images
def _ip_base(xml_path, data):
    return os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")


def _read_view_points(store, group):
    """(ids int64 (n,), loc float64 (n, 3), intensities float32 (n,) or None) of one label group of interestpoints.n5."""
    if store is None or "dimensions" not in store.get_attributes(group + "/interestpoints/loc"):
        return np.zeros(0, dtype=np.int64), np.zeros((0, 3)), None
    ids = store.read_list(group + "/interestpoints/id").reshape(-1).astype(np.int64)
    loc = store.read_list(group + "/interestpoints/loc").astype(np.float64).reshape(-1, 3)
    inten = None
    if "dimensions" in store.get_attributes(group + "/intensities"):
        inten = store.read_list(group + "/intensities").reshape(-1).astype(np.float32)
    return ids, loc, inten


def _write_view_points(store, group, ids, loc, inten=None):
    shutil.rmtree(os.path.join(store.root, group), ignore_errors=True)     # no stale correspondences under it
    store.set_attributes(group + "/interestpoints", IP_N5_GROUP_ATTRIBUTES)
    store.write_list(group + "/interestpoints/id", np.asarray(ids, dtype=np.uint64).reshape(-1, 1), IP_N5_BLOCK_LENGTH, "zstd")
    store.write_list(group + "/interestpoints/loc", np.asarray(loc, dtype=np.float64).reshape(-1, 3), IP_N5_BLOCK_LENGTH,
                     "zstd")
    if inten is not None:
        store.write_list(group + "/intensities", np.asarray(inten, dtype=np.float32).reshape(-1, 1), IP_N5_BLOCK_LENGTH,
                         "zstd")


def split_images(xml_path, target_image_size, target_overlap, xml_out=None, disable_optimization=False,
                 fake_interest_points=False, fip_density=100.0, fip_min_num_points=20, fip_max_num_points=500,
                 fip_error=0.5, fip_exclusion_radius=20.0, fip_label="splitPoints", assign_illuminations=False,
                 display_result=False, dry_run=False):
    """`./split-images -x dataset.xml -tis 512,512,256 -to 32,32,32 [-xo out.xml] [--disableOptimization] [-fip
    [--fipDensity 100] [--fipMinNumPoints 20] [--fipMaxNumPoints 500] [--fipError 0.5] [--fipExclusionRadius 20]]
    [--assignIlluminations] [--dryRun]` (J/SplitDatasets.java:74-168): cut every view into overlapping sub-views so
    that match-interestpoints + solver can give each piece its own model, and write the project of the pieces to
    ``xml_out`` (default: the input, with a ~1 backup).  Sizes are "x,y,z" strings or triples.

    The target size and overlap are rounded up to multiples of the step m, per axis the lcm of every view's mipmap
    factors; an overlap larger than the size, or equal to it on an axis that has to be split, raises ValueError.  The
    boxes and the new project follow split.intervals / split.split_project.  The new views are read through a
    `split.viewerimgloader` wrapping the input's loader (viewsource.SplitViews), so every command reads them.

    Interest points carry over: each sub-view gets, per label of its parent, the points inside its closed box shifted
    by -min, ids and intensities kept, written to interestpoints.n5 next to ``xml_out``; correspondences are dropped
    (re-run matching).  ``fake_interest_points`` (`-fip`) adds split.fake_points between overlapping sub-views of one
    view, with their correspondences, as label ``fip_label``, which must not exist yet (ValueError).

    A TIFF dataset (`spimreconstruction.filemap2`) raises NotImplementedError before anything is written: resave it
    first.  ``display_result`` (a GUI) raises NotImplementedError; ``dry_run`` returns the plan and writes nothing.  Returns
    dict(step=m, size=s, overlap=o, views={new setup: (old setup, min xyz, max xyz)}, fake_points={(tp, new a, new b):
    count})."""
    if display_result:
        raise NotImplementedError("split-images --displayResult (the BigStitcher GUI) is not available")
    size = bsplit.parse_size(target_image_size, "targetImageSize")
    overlap = bsplit.parse_size(target_overlap, "targetOverlap")
    data = SpimData2.load(xml_path)
    src = bvs.open_views(data)
    if src.format == FILEMAP_LOADER:
        raise NotImplementedError("split-images of a TIFF dataset (spimreconstruction.filemap2): resave it to N5 or "
                                  "OME-ZARR first")
    missing = data.missing_views()
    present = [v for v in data.view_ids() if v not in missing]
    m = bsplit.min_step(src, present)
    s = tuple(bsplit.closest_larger_divisible(size[d], m[d]) for d in range(3))
    o = tuple(bsplit.closest_larger_divisible(overlap[d], m[d]) for d in range(3))
    if any(o[d] > s[d] for d in range(3)):
        raise ValueError(f"overlap {o} cannot be bigger than size {s}.")
    plan, boxes_of = {}, {}
    for old in sorted(data.setups):
        boxes_of[old] = bsplit.boxes(data.setups[old].size, s, o, m, not disable_optimization)
        for k, (mn, mx) in enumerate(boxes_of[old]):
            plan[len(plan)] = (old, mn, mx, k)
    new_of = {(p[0], p[3]): nid for nid, p in plan.items()}
    xml_out = xml_out or xml_path
    new = bsplit.split_project(data, plan, assign_illuminations, xml_out)

    # ---- every parent's points are read before anything is written: new setup ids reuse old ones
    ips = data.interest_points()
    if fake_interest_points and any(fip_label in labels for labels in ips.values()):
        raise ValueError(f"interest point label '{fip_label}' already exists; choose another --fipLabel")
    root_in = os.path.join(_ip_base(xml_path, data), "interestpoints.n5")
    store_in = bn5.N5Store(root_in) if os.path.isdir(root_in) else None
    parent_points = {}                        # (tp, old) -> {label: (ids, loc, intensities, params)}
    for v, labels in sorted(ips.items()):
        if v in missing:
            continue
        parent_points[v] = {lab: _read_view_points(store_in, e["path"].rstrip("/")) + (e["params"],)
                            for lab, e in sorted(labels.items())}

    carried = {}                              # (label, params) -> {new view: (group, ids, loc, intensities)}
    for (tp, old), labels in parent_points.items():
        for k, (mn, mx) in enumerate(boxes_of[old]):
            nv = (tp, new_of[(old, k)])
            for lab, (ids, loc, inten, params) in labels.items():
                inside = np.all((loc >= mn) & (loc <= mx), axis=1)
                carried.setdefault((lab, params), {})[nv] = (
                    f"tpId_{tp}_viewSetupId_{nv[1]}/{lab}", ids[inside], loc[inside] - mn,
                    None if inten is None else inten[inside])

    fakes_out, fake_counts, fake_results = {}, {}, {}
    if fake_interest_points:
        for (tp, old) in present:
            labels = parent_points.get((tp, old), {})
            existing = np.concatenate([p[1] for p in labels.values()]) if labels else np.zeros((0, 3))
            fakes, pairs = bsplit.fake_points(tp, old, boxes_of[old], existing, fip_density, fip_min_num_points,
                                              fip_max_num_points, fip_error, fip_exclusion_radius)
            for i, pts in fakes.items():
                fakes_out[(tp, new_of[(old, i)])] = pts - boxes_of[old][i][0]
            for (i, j), got in pairs.items():
                va, vb = (tp, new_of[(old, i)]), (tp, new_of[(old, j)])
                fake_counts[(tp, va[1], vb[1])] = len(got)
                fake_results[(va, fip_label, vb, fip_label)] = np.asarray(got, dtype=np.int64).reshape(-1, 2)

    result = dict(step=m, size=s, overlap=o, views={nid: (p[0], tuple(int(v) for v in p[1]), tuple(int(v) for v in p[2]))
                                                    for nid, p in plan.items()}, fake_points=fake_counts)
    if dry_run:
        return result

    if carried or fakes_out:
        store = bn5.N5Store(os.path.join(_ip_base(xml_out, new), "interestpoints.n5"), create=True)
        for (lab, params), views in sorted(carried.items()):
            for group, ids, loc, inten in views.values():
                _write_view_points(store, group, ids, loc, inten)
            new.set_interest_points(lab, params, {v: g[0] for v, g in views.items()})
        if fakes_out:
            groups = {}
            for v, pts in sorted(fakes_out.items()):
                groups[v] = f"tpId_{v[0]}_viewSetupId_{v[1]}/{fip_label}"
                _write_view_points(store, groups[v], np.arange(len(pts)), pts)
            holder = type("FakePoints", (), dict(world={(v, fip_label): None for v in groups}, corr={}))
            write_match_correspondences(store, holder, sorted(groups), [fip_label], fake_results, clear=True)
            new.set_interest_points(fip_label, (
                f"Fake points for image splitting: density={_java(float(fip_density))}, "
                f"minPoints={int(fip_min_num_points)}, maxPoints={int(fip_max_num_points)}, error={_java(float(fip_error))}, "
                f"excludeRadius={_java(float(fip_exclusion_radius))}"), groups)
    os.makedirs(os.path.dirname(os.path.abspath(xml_out)), exist_ok=True)
    new.save(xml_out)
    return result


# --------------------------------------------------------------------------------------------- estimate-bounding-box
BBOX_SLAB = 32                 # downsampled z-planes fused per call
BBOX_BYTES_PER_VOXEL = 12      # fused volume, filter output and the filter's ping-pong buffer, float32 each


def bounding_box_grid(lo, hi, ds):
    """The downsampled grid over the world box [lo, hi] (PARITY_GAPS B2): (g_min, dims), int64 [3] each, with
    g_min = floor(lo / ds), g_max = ceil(hi / ds) and dims = g_max - g_min + 1; voxel i is world point ds (g_min + i)."""
    lo = np.asarray(lo, dtype=np.int64)
    hi = np.asarray(hi, dtype=np.int64)
    g_min = np.floor_divide(lo, ds)
    return g_min, -np.floor_divide(-hi, ds) - g_min + 1


def fuse_downsampled(ctx, data, src, view_ids, ds, g_min, dims, out):
    """AVG_BLEND fusion of ``view_ids`` with n-linear interpolation, in float32, on the grid of bounding_box_grid
    (PARITY_GAPS B2), written into ``out`` ([z, y, x] float32 of ``dims``: a device tensor, e.g. from
    Context.volume_empty).  Each view's model is its registration scaled by 1 / ds (fusion.adjust_all_transforms) composed
    with the mipmap level ViewUtil's best-resolution rule picks for it, blending from adjust_blending of that model.  The
    grid is fused in slabs of BBOX_SLAB z-planes.  Each view's level volume is staged whole, once, as float32: that runs
    the generic fusion kernel, because the uint16 TMA kernels sample models that magnify the source (ds > 1) at the
    wrong voxels (DESIGN.md, estimate-bounding-box)."""
    view_ids = sorted(view_ids)
    regs = bf.adjust_all_transforms({v: data.model(*v) for v in view_ids}, downsampling=float(ds))
    info = {}
    for v in view_ids:
        factors, mts = src.mipmap_info(v)
        lvl = bf.best_mipmap_level(regs[v], factors, mts)
        m = _compose(regs[v], mts[lvl])
        info[v] = dict(level=lvl, dims=src.level_dims(v, lvl), model=m, blending=bf.adjust_blending(m))
    vdims = {v: info[v]["dims"] for v in view_ids}
    vregs = {v: info[v]["model"] for v in view_ids}
    params = ctx.fuse_params("AVG_BLEND", 1, native.DTYPE_F32)
    g_min = np.asarray(g_min, dtype=np.int64)
    nx, ny, nz = (int(d) for d in dims)
    staged = {}
    try:
        for z0 in range(0, nz, BBOX_SLAB):
            sz = min(BBOX_SLAB, nz - z0)
            lo = g_min + np.array([0, 0, z0])
            hi = g_min + np.array([nx - 1, ny - 1, z0 + sz - 1])
            views = []
            for v in bf.find_overlapping_views(vdims, vregs, lo, hi, view_ids):
                if v not in staged:
                    staged[v] = ctx.volume_upload(src.read_volume(v, info[v]["level"]).astype(np.float32))
                border, rng = info[v]["blending"]
                views.append(dict(src_to_world=info[v]["model"], vol_handle=staged[v], blend_border=border,
                                  blend_range=rng))
            ctx.fuse_blocks(views, [tuple(int(x) for x in lo)], [(nx, ny, sz)], params, outs=[out[z0:z0 + sz]])
    finally:
        for h in staged.values():
            ctx.volume_free(h)


def estimate_bounding_box(xml_path, ctx: Context, name, background_intensity=5.0, discarded_object_size=25,
                          downsampling=4, view_selection=None, dry_run=False):
    """`./estimate-bounding-box -x dataset.xml -b name [--background 5] [--minObjectSize 25] [--downsampling 4]
    [view selection] [--dryRun]`: the "automatic bounding box through image filtering" of BigStitcher's GUI (mvrecon
    BoundingBoxMinFilterThreshold, recalled; PARITY_GAPS B1-B6), stored as the XML's <BoundingBoxDefinition> ``name``
    for `create-fusion-container -b name`.  BigStitcher-Spark has no such command.  The defaults are the GUI's, recalled.

    1. The selected views (``view_selection``: keyword arguments of SpimData2.select_views, default all) are fused at
       1 / ``downsampling`` on the device (fuse_downsampled) over the box of those views (views_bounding_box).
    2. t = mn + (mx - mn) ``background_intensity`` / 100 from the fused volume's min mn and max mx.
    3. A box minimum filter of radius r = max(1, floor(``discarded_object_size`` / downsampling + 0.5)) on every axis
       (bs_min_filter) removes objects narrower than about the size (beads); the box is clipped to the volume.
    4. The voxels of the filtered volume above t (strictly) give an index box; one downsampled voxel is added on every
       side, it is mapped back to world coordinates and intersected with the views' box.

    The definition replaces any earlier one of that name; the XML is saved with a `~1` backup unless ``dry_run``.
    Returns dict(min, max (world, inclusive), threshold, min_max (mn, mx), radius, dims (of the downsampled grid),
    count (voxels above t)).  ValueError, with the XML untouched, for an empty name, a downsampling that is not an
    integer >= 1, a background outside [0, 100], a negative object size, no selected views, and when no voxel is above
    the threshold.  MemoryError, before anything is fused, when the device cannot hold 12 bytes per grid voxel plus the
    float32 source levels."""
    if not name:
        raise ValueError("estimate-bounding-box: the bounding box needs a name (-b)")
    if isinstance(downsampling, bool) or int(downsampling) != downsampling or downsampling < 1:
        raise ValueError(f"estimate-bounding-box: --downsampling {downsampling} is not an integer >= 1")
    if not 0.0 <= float(background_intensity) <= 100.0:
        raise ValueError(f"estimate-bounding-box: --background {background_intensity} outside [0, 100]")
    if not float(discarded_object_size) >= 0.0:
        raise ValueError(f"estimate-bounding-box: --minObjectSize {discarded_object_size} is negative")
    ds = int(downsampling)
    data = SpimData2.load(xml_path)
    views = data.select_views(**view_selection) if view_selection else data.view_ids()
    if not views:
        raise ValueError("estimate-bounding-box: no views selected")
    lo, hi = (b.astype(np.int64) for b in views_bounding_box(data, views))
    g_min, dims = bounding_box_grid(lo, hi, ds)
    src = bvs.open_views(data)
    source_bytes = 0
    for v in views:
        factors, mts = src.mipmap_info(v)
        reg = bf.adjust_all_transforms({v: data.model(*v)}, downsampling=float(ds))[v]
        source_bytes += 4 * int(np.prod(src.level_dims(v, bf.best_mipmap_level(reg, factors, mts))))
    _check_device_memory(ctx, BBOX_BYTES_PER_VOXEL * int(np.prod(dims)) + source_bytes,
                         f"the {dims[0]}x{dims[1]}x{dims[2]} grid at downsampling {ds}", "estimate-bounding-box",
                         "use a larger --downsampling")
    radius = max(1, int(math.floor(float(discarded_object_size) / ds + 0.5)))
    fused, buf = ctx.volume_empty(dims)
    handles = [fused]
    try:
        fuse_downsampled(ctx, data, src, views, ds, g_min, dims, buf)
        mn, mx = ctx.volume_min_max(fused)
        t = mn + (mx - mn) * float(background_intensity) / 100.0
        handles.append(ctx.min_filter(fused, (radius, radius, radius)))
        i_min, i_max, count = ctx.threshold_bbox(handles[-1], t)
    finally:
        for h in handles:
            ctx.volume_free(h)
        del buf
    if count == 0:
        raise ValueError(f"estimate-bounding-box: no voxel of the filtered fusion is above the threshold {t!r} "
                         f"(min {mn!r}, max {mx!r}, --background {background_intensity}); the XML is unchanged")
    bb_min = np.maximum(ds * (g_min + np.asarray(i_min, dtype=np.int64) - 1), lo)
    bb_max = np.minimum(ds * (g_min + np.asarray(i_max, dtype=np.int64) + 1), hi)
    data.set_bounding_box(name, bb_min, bb_max, replace=True)
    if not dry_run:
        data.save(xml_path)
    return dict(min=[int(v) for v in bb_min], max=[int(v) for v in bb_max], threshold=t, min_max=(mn, mx),
                radius=radius, dims=[int(v) for v in dims], count=int(count))
