"""The `call()` bodies of the reference's `stitching`, `create-fusion-container` and
`affine-fusion` commands with the Spark RDD collapsed to a plain host work queue over one
`native.Context` (BASELINE north_star), SpimData2 XML in, N5 / OME-Zarr blocks out.

  stitching               J/SparkPairwiseStitching.java:110-392
  create_fusion_container J/CreateFusionContainer.java:122-519   (N5 or OME-ZARR, all channels / timepoints, pyramid)
  affine_fusion           J/SparkAffineFusion.java:179-800       (s0 + multi-resolution pyramid)
  nonrigid_fusion         J/SparkNonRigidFusion.java:124-446     (MLS grids from interest-point correspondences)
  detect_interestpoints   J/SparkInterestPointDetection.java:173-964 (block-wise DoG, interestpoints.n5 + the XML)
  match_interestpoints    J/SparkGeometricDescriptorMatching.java:161-545 (PRECISE_TRANSLATION, correspondences)
  solver                  J/Solver.java:161-432                   (ONE_ROUND_SIMPLE / ONE_ROUND_ITERATIVE, registrations)
  resave                  J/SparkResaveN5.java:80-455             (OME-ZARR or BDV-N5 with the pyramid built on the device)

Every command reads its images through viewsource.py, so `bdv.n5` and `bdv.multimg.zarr` datasets both work.

No argument parsing here (the picocli layer is out of scope); keyword names follow the CLI flags.
"""
from __future__ import annotations

import math
import os
import shutil
from decimal import Decimal

import numpy as np

from . import fusion as bf
from . import n5 as bn5
from . import zarr as bzarr
from . import matching as bm
from . import native, solver as bsolver, stitching as bst, viewsource as bvs
from .native import Context
from .spimdata import SpimData2


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


def create_fusion_container(xml_path, out_path, block_size=(128, 128, 128), dtype="float32", min_intensity=None,
                            max_intensity=None, preserve_anisotropy=False, anisotropy_factor=float("nan"),
                            storage=None, downsamplings=(), multi_res=False, compression="zstd"):
    """`./create-fusion-container -x dataset.xml -o fused.zarr [-s ZARR|N5] -d FLOAT32 --blockSize ... [--multiRes |
    -ds ...] [-c Zstandard]`: bounding box of all views (Import.getBoundingBox, J/CreateFusionContainer.java:184-211),
    NumChannels / NumTimepoints from the XML (:213-216), datasets + metadata.  Defaults follow the reference: OME-ZARR
    storage unless the path ends in .n5 (:67-69), Zstandard compression (:71-76).  ``downsamplings``: relative steps."""
    data = SpimData2.load(xml_path)
    lo = np.full(3, np.inf)
    hi = np.full(3, -np.inf)
    af = anisotropy_factor if preserve_anisotropy else float("nan")
    regs = bf.adjust_all_transforms({v: data.model(*v) for v in data.view_ids()}, af)
    for v, M in regs.items():
        bmin, bmax = bf.transformed_bounding_box(data.setups[v[1]].size, M)
        lo = np.minimum(lo, bmin)
        hi = np.maximum(hi, bmax)
    if storage is None:   # guessed from the extension like the reference (J/SparkAffineFusion.java:206-225)
        storage = "N5" if out_path.rstrip("/").lower().endswith(".n5") else "ZARR"
    dims = [int(hi[d] - lo[d] + 1) for d in range(3)]
    if multi_res and not downsamplings:
        downsamplings = estimate_multires_pyramid(dims, af)
    if dtype != "float32":   # J/CreateFusionContainer.java:226-242
        top = 255.0 if dtype == "uint8" else 65535.0
        min_intensity = 0.0 if min_intensity is None else min_intensity
        max_intensity = top if max_intensity is None else max_intensity
    kw = dict(anisotropy_factor=af if preserve_anisotropy else None, num_channels=len(data.channels_ordered()),
              num_timepoints=len(data.timepoints), compression=compression, downsamplings=downsamplings)
    if storage.upper() == "ZARR":
        return bzarr.create_fusion_container_zarr(out_path, os.path.abspath(xml_path), lo.astype(np.int64),
                                                  hi.astype(np.int64), block_size, dtype, min_intensity, max_intensity, **kw)
    return bn5.create_fusion_container(out_path, os.path.abspath(xml_path), lo.astype(np.int64), hi.astype(np.int64),
                                       block_size, dtype, min_intensity, max_intensity, **kw)


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
                  mask_offset=(0.0, 0.0, 0.0), view_selection=None):
    """`./affine-fusion -o fused.zarr [-f AVG_BLEND] [--blockScale 2,2,1] [-c channelIndex] [-t timepointIndex]
    [--masks [--maskOffset x,y,z]]`:
    read the container metadata and, for every (channel, timepoint) volume (J/SparkAffineFusion.java:425-440), fuse
    its views super-block by super-block on the device, write the blocks with N5Utils.saveBlock semantics and build
    the multi-resolution pyramid (:703-782).  Returns the list of s0 datasets written.

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
    z-slabs, no data-path collective; ``barrier()`` separates s0 from the pyramid levels that re-read it."""
    is_zarr = os.path.exists(os.path.join(out_path, ".zgroup"))
    store, meta = (bzarr.read_fusion_container_zarr if is_zarr else bn5.read_fusion_container)(out_path)
    data = SpimData2.load(meta["input_xml"])
    src = bvs.open_views(data)
    nc, nt = int(meta["num_channels"]), int(meta["num_timepoints"])
    if nc != len(data.channels_ordered()) or nt != len(data.timepoints):
        raise ValueError(f"container says {nc} channel(s) / {nt} timepoint(s), the XML has "
                         f"{len(data.channels_ordered())} / {len(data.timepoints)}")
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
            vol_views = data.views_of(ci, ti, selected)
            if not vol_views:
                continue                                             # nothing selected for this volume
            _fuse_volume_blockwise(ctx, data, src, _Sink(store, is_zarr, ci, ti), meta, levels, vol_views,
                                   fusion_type, interpolation, block_scale, retries, blocks_per_call, shard, barrier,
                                   masks, mask_offset)
            written.append(levels[0]["dataset"])
    return written


def _fuse_volume_blockwise(ctx, data, src, sink, meta, levels, view_ids, fusion_type, interpolation, block_scale,
                           retries, blocks_per_call, shard=(0, 1), barrier=None, masks=False, mask_offset=(0.0, 0.0, 0.0)):
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


def _pyramid_from_stored(ctx, volumes, first, compute, bs, shard=(0, 1), retries=5, barrier=None):
    """Levels ``first`` .. N of every volume in ``volumes`` ([(sink, levels, numpy dtype)]): every compute block of level
    l is the 2x average of its region of level l-1, read back from the container and averaged on the device.  Rank r of
    w takes blocks [r::w] of each level; ``barrier()`` runs before each level so that level l-1 is complete on every
    rank.  Failed blocks are retried up to ``retries`` times (RetryTrackerSpark)."""
    rank, world = shard
    for li in range(first, max(len(lv) for _, lv, _ in volumes)):
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
                h = h2 = None
                try:
                    srcblk = sink.read_region(prev["dataset"], [off[d] * rel[d] for d in range(3)], [size[d] * rel[d] for d in range(3)])
                    h = ctx.volume_upload(np.ascontiguousarray(srcblk))
                    h2 = ctx.downsample(h, rel)
                    sink.save(cur["dataset"], ctx.volume_download(h2, size, np_dt), gpos)
                except native.BsError:
                    failed.append(item)
                finally:
                    for hh in (h, h2):
                        if hh is not None:
                            ctx.volume_free(hh)
            todo = failed


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


def _check_device_memory(ctx, nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info(ctx.device)
    if nbytes > free:
        raise MemoryError(f"detect-interestpoints: {what} needs {nbytes / 2**30:.2f} GiB on device {ctx.device}, "
                          f"{free / 2**30:.2f} GiB are free; use a larger --downsampleXY / --downsampleZ")


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
                    shard=(0, 1), retries=5, blocks_per_call=16):
    """`./nonrigid-fusion -x dataset.xml -o fused.n5 -d /ch0/s0 -ip beads [-ip nuclei] [-s N5|ZARR] [--blockSize ...]
    [--blockScale 2,2,1] [-p FLOAT32|UINT16|UINT8 --minIntensity --maxIntensity]` (J/SparkNonRigidFusion.java:124-446):
    the maximal bounding box of the selected views becomes dataset ``n5_dataset`` (Zstandard, attribute offset = bb.min);
    every super-block of Grid.create(dims, blockSize * blockScale, blockSize) that some view reaches is fused on the
    device with per-view moving-least-squares grids fitted to the corresponding interest points of the ``-ip`` labels
    (bs_nonrigid_fuse_blocks, AVG_BLEND, control points every 10 px) and saved; blocks no view reaches are not written.
    Returns the list of written grid positions.  ZARR output is the (t, c, z, y, x) array with singleton t and c.

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
                    outs = _nonrigid_chunk(ctx, src, chunk, lo, fuse, nviews, vdims, params, cpd)
                except native.BsError:
                    failed.extend(chunk)
                    continue
                for (off, size, gpos), blk in zip(chunk, outs):
                    sink.save(n5_dataset, blk, gpos)
                    written.append(tuple(gpos))
            todo = failed
    return written


def _nonrigid_chunk(ctx, src, chunk, bb_min, fuse, nviews, vdims, params, cpd):
    """Fuse a list of super-blocks that share their views.  Each view's source window is the range its control-point
    grids map to over the chunk (+2 px for the n-linear taps), read from level s0 and uploaded as a windowed view."""
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
            staged.append(h)
            gviews.append(dict(nv, vol_handle=h, window_min=tuple(int(x) for x in wlo)))
        if not gviews:
            return [np.zeros(tuple(s)[::-1], dtype=native._out_dtype(params)) for s in sizes]
        return ctx.nonrigid_fuse_blocks(gviews, mins, sizes, params, cpd)
    finally:
        for h in staged:
            ctx.volume_free(h)


# --------------------------------------------------------------------------------------------- match-interestpoints
def match_pairs(view_dims, registrations, view_ids, view_reg="OVERLAPPING_ONLY"):
    """M2: the view pairs (A, B) of one timepoint, A < B in (tp, setup) order; OVERLAPPING_ONLY keeps the pairs whose
    closed transformed bounding boxes intersect, ALL_AGAINST_ALL keeps every pair."""
    vr = view_reg.upper()
    if vr not in ("OVERLAPPING_ONLY", "ALL_AGAINST_ALL"):
        raise ValueError(f"-vr {view_reg}")
    views = sorted(view_ids)
    boxes = {v: bf.transformed_bounding_box(view_dims[v], registrations[v]) for v in views}
    pairs = []
    for i, a in enumerate(views):
        for b in views[i + 1:]:
            if a[0] != b[0]:
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
                         dry_run=False, shard=(0, 1), allgather=None):
    """`./match-interestpoints -x dataset.xml -l beads -m PRECISE_TRANSLATION [-s 3.0] [-r 1] [-n 3] [--searchRadius r]
    [--clearCorrespondences] [--matchAcrossLabels] [-ipfr ALL|OVERLAPPING_ONLY] [-vr OVERLAPPING_ONLY|ALL_AGAINST_ALL]
    [-tm AFFINE] [-rm RIGID] [--lambda 0.1] [-rit 10000] [-rme 5.0] [-rmir 0.1] [-rmni 12]`, the non-grouped branch of
    J/SparkGeometricDescriptorMatching.java:161-342 and the save at :512-545: for every task (view pair x label pair)
    the points are read from interestpoints.n5 and mapped to world (M1), optionally filtered to the partner's box (M3);
    descriptors and the exhaustive A -> B search run on the device (bs_descriptors_build / bs_descriptors_match), the
    ratio test (M6), RANSAC and its filter (M7, M8) on the host; the inliers become correspondences of both views (M9),
    written for every selected view x label unless ``dry_run``.  The XML is not touched.
    Returns {(viewA, labelA, viewB, labelB): int64 (K, 2) id pairs} for every task.

    Multi-GPU: rank r of w (``shard``) takes tasks[r::w]; ``allgather(obj) -> [obj of every rank]`` merges the results
    and rank 0 writes.  FAST_ROTATION, FAST_TRANSLATION, ICP, grouping, -rtp other than TIMEPOINTS_INDIVIDUALLY and
    -rmc raise NotImplementedError."""
    m = method.upper()
    if m in ("FAST_ROTATION", "FAST_TRANSLATION", "ICP"):
        raise NotImplementedError(f"match-interestpoints -m {m} is not implemented")
    if m != "PRECISE_TRANSLATION":
        raise ValueError(f"-m {method}")
    for flag, on in (("--groupTiles", group_tiles), ("--groupIllums", group_illums), ("--groupChannels", group_channels),
                     ("--splitTimepoints", split_timepoints), ("-rmc", ransac_multi_consensus),
                     (f"-rtp {registration_tp}", registration_tp.upper() != "TIMEPOINTS_INDIVIDUALLY")):
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
    tasks = match_tasks(match_pairs(vdims, regs, views, view_reg), labels, match_across_labels)
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
           registration_tp="TIMEPOINTS_INDIVIDUALLY", view_selection=None, dry_run=False):
    """`./solver -x dataset.xml -s STITCHING|IP [-l beads [-lw 1.0]] [--method ONE_ROUND_SIMPLE|ONE_ROUND_ITERATIVE]
    [-tm AFFINE] [-rm RIGID] [--lambda 0.1] [--maxError 5.0] [--maxIterations 10000] [--maxPlateauwidth 200]
    [--relativeThreshold 3.5] [--absoluteThreshold 7.0] [-fv 'tp,setup' | --disableFixedViews] [--groupTiles]
    [--groupIllums] [--groupChannels] [--splitTimepoints] [--dryRun]` (J/Solver.java:161-432): global optimisation of
    the stored stitching results or interest-point correspondences.  The matches are built and the tiles pre-aligned on
    the host; the relaxation runs on the device (bs_solve_tiles).  Every view of a solved tile gets the tile's model as
    a new first <ViewTransform>; the XML is saved (with a ~1 backup) unless ``dry_run``.  Returns dict(models={view:
    3 x 4}, removed=[(views A, views B)] (ONE_ROUND_ITERATIVE), stats) -- stats holds iterations, the final error,
    skipped fits, stale stitching results and the views without links, which keep their registration.

    TWO_ROUND_SIMPLE / TWO_ROUND_ITERATIVE and -rtp other than TIMEPOINTS_INDIVIDUALLY raise NotImplementedError."""
    return bsolver.run(xml_path, ctx, source, labels, label_weights, method, transformation_model, regularization_model,
                       regularization_lambda, max_error, max_iterations, max_plateau_width, relative_threshold,
                       absolute_threshold, fixed_views, disable_fixed_views, group_tiles, group_illums, group_channels,
                       split_timepoints, registration_tp, view_selection, dry_run)


# --------------------------------------------------------------------------------------------- resave
RESAVE_COMPRESSION = {"zstd": "zstd", "zstandard": "zstd", "gzip": "gzip", "raw": "raw"}


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
    a, b = os.path.realpath(out_path), os.path.realpath(src.store.root)
    if a == b or a.startswith(b + os.sep) or b.startswith(a + os.sep):
        raise ValueError(f"resave output {out_path} overlaps the input container {src.store.root}; choose another -o / -xo")
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
                store.set_attributes(f"setup{v[1]}", {"downsamplingFactors": [list(s) for s in steps], "dataType": dt})
                store.set_attributes(f"setup{v[1]}/timepoint{v[0]}", {"resolution": [1.0, 1.0, 1.0], "multiScale": True})
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
