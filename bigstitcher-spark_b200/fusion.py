"""Host-side mirror of the reference's affine-fusion operator interface.

Mirrors what ``SparkAffineFusion``'s per-block task calls
(src/main/java/net/preibisch/bigstitcher/spark/SparkAffineFusion.java:480-676):

    Grid.create(dimensions, computeBlockSize, blockSize)          (:457-461)  -> grid_create
    TransformVirtual.adjustAllTransforms(...)                     (:486-491)  -> adjust_all_transforms
    OverlappingViews.findOverlappingViews(...)  (J/fusion/OverlappingViews.java:28-47) -> find_overlapping_views
    BlkAffineFusion.initWithIntensityCoefficients(...)            (:602-615)  -> BlkAffineFusion.init
    BlockAlgoUtils.arrayImg(blockSupplier, interval)              (:620-627)  -> BlockSupplier.copy
    RetryTrackerSpark (5 attempts)   (J/util/RetryTrackerSpark.java:28-31)    -> fuse_volume(retries=5)

Voxel arithmetic runs in libbsgpu.so (``native.Context.fuse_block``); this module only does
geometry, bookkeeping and residency management of source volumes on the device.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from . import native
from .native import Context

DEFAULT_BLENDING_RANGE = 40.0   # FusionTools.defaultBlendingRange
DEFAULT_BLENDING_BORDER = 0.0   # FusionTools.defaultBlendingBorder
AFFINE_EXPANSION = 2            # Intervals.expand(interval, 2), J/fusion/OverlappingViews.java:36-37


def grid_create(dimensions, grid_block_size, out_block_size=None):
    """mvrecon util.Grid.create: x-fastest enumeration of blocks of ``grid_block_size``;
    each entry = (offset px, size px clipped to dimensions, offset / out_block_size)
    (usage J/SparkAffineFusion.java:520-525,620-624,635,648)."""
    out_block_size = out_block_size or grid_block_size
    n = len(dimensions)
    counts = [int(math.ceil(dimensions[d] / grid_block_size[d])) for d in range(n)]
    blocks = []
    idx = [0] * n
    total = int(np.prod(counts))
    for _ in range(total):
        off = [idx[d] * grid_block_size[d] for d in range(n)]
        size = [min(grid_block_size[d], dimensions[d] - off[d]) for d in range(n)]
        gpos = [off[d] // out_block_size[d] for d in range(n)]
        blocks.append((tuple(off), tuple(size), tuple(gpos)))
        for d in range(n):
            idx[d] += 1
            if idx[d] < counts[d]:
                break
            idx[d] = 0
    return blocks


def adjust_all_transforms(registrations: dict, anisotropy_factor=float("nan"), downsampling=float("nan")):
    """TransformVirtual.adjustAllTransforms: copy each model; pre-concatenate scale(1,1,1/af)
    when anisotropy is preserved; downsampling is NaN on this path
    (J/SparkAffineFusion.java:486-491)."""
    out = {}
    for vid, m in registrations.items():
        M = np.asarray(m, dtype=np.float64).reshape(3, 4).copy()
        if not math.isnan(anisotropy_factor):
            S = np.diag([1.0, 1.0, 1.0 / anisotropy_factor])
            M = S @ M
        if not math.isnan(downsampling):
            M = np.diag([1.0 / downsampling] * 3) @ M
        out[vid] = M
    return out


def transformed_bounding_box(dims_xyz, m):
    """ViewUtil.getTransformedBoundingBox (J/util/ViewUtil.java:154-159):
    smallestContainingInterval(t.estimateBounds([0, dim-1]))."""
    M = np.asarray(m, dtype=np.float64).reshape(3, 4)
    c = np.array([[x, y, z] for x in (0, dims_xyz[0] - 1) for y in (0, dims_xyz[1] - 1)
                  for z in (0, dims_xyz[2] - 1)], dtype=np.float64)
    w = c @ M[:, :3].T + M[:, 3]
    return np.floor(w.min(axis=0)).astype(np.int64), np.ceil(w.max(axis=0)).astype(np.int64)


def find_overlapping_views(view_dims: dict, registrations: dict, block_min, block_max, view_ids=None,
                           expand=AFFINE_EXPANSION):
    """OverlappingViews.findOverlappingViews: transformed bbox intersects the block expanded by ``expand`` (2; the
    non-rigid fusion's viewsToFuse use 50, J/SparkNonRigidFusion.java:333-340)."""
    lo = np.asarray(block_min, dtype=np.int64) - int(expand)
    hi = np.asarray(block_max, dtype=np.int64) + int(expand)
    out = []
    for vid in (view_ids if view_ids is not None else sorted(registrations)):
        bmin, bmax = transformed_bounding_box(view_dims[vid], registrations[vid])
        if np.all(np.minimum(hi, bmax) >= np.maximum(lo, bmin)):
            out.append(vid)
    return out


def adjust_blending(m, blending=DEFAULT_BLENDING_RANGE, border=DEFAULT_BLENDING_BORDER):
    """FusionTools.adjustBlending: range / border divided by the (float) per-axis scale of the model."""
    M = np.asarray(m, dtype=np.float64).reshape(3, 4)
    s = np.sqrt((M[:, :3] ** 2).sum(axis=0)).astype(np.float32)
    return (np.full(3, border, np.float32) / s), (np.full(3, blending, np.float32) / s)


def best_mipmap_level(src_to_world, mipmap_resolutions, mipmap_transforms, accepted_error=np.float32(0.02)):
    """ViewUtil ... forBestResolution (J/util/ViewUtil.java:425-493): the largest total
    downsampling whose float32 step sizes stay < 1 + 0.02 or approximately equal the
    full-resolution step."""
    def step_size(model):
        return np.array([np.float32(np.linalg.norm(model[:3, d])) for d in range(3)], dtype=np.float32)
    M = np.vstack([np.asarray(src_to_world, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
    best_level, best_scaling, size_max = 0, 0.0, None
    for level, (factors, mt) in enumerate(zip(mipmap_resolutions, mipmap_transforms)):
        L = M @ np.vstack([np.asarray(mt, dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
        size = step_size(L)
        if level == 0:
            size_max = size
            best_scaling = float(np.prod(factors))
            continue
        valid = all((size[d] < np.float32(1.0) + accepted_error) or
                    (abs(float(size[d]) - float(size_max[d])) <= float(accepted_error)) for d in range(3))
        if valid and float(np.prod(factors)) > best_scaling:
            best_scaling = float(np.prod(factors))
            best_level = level
    return best_level


@dataclass
class BlockSupplier:
    """What BlkAffineFusion.init* returns: ``copy(interval)`` materialises one block
    (BlockAlgoUtils.arrayImg -> BlockSupplier.copy)."""
    ctx: Context
    view_ids: list
    view_dims: dict
    registrations: dict          # adjusted, source px -> world
    handles: dict                # vid -> device volume handle
    content_handles: dict
    bb_min: tuple
    fusion_type: int
    interpolation: int
    out_dtype: int
    min_intensity: float
    max_intensity: float
    blend_lut_n: int = 0
    blending: dict = field(default_factory=dict)

    def views_for(self, vids):
        vs = []
        for vid in vids:
            border, rng = self.blending[vid]
            vs.append(dict(src_to_world=self.registrations[vid], vol_handle=self.handles[vid],
                           content_handle=self.content_handles.get(vid, 0), blend_border=border, blend_range=rng))
        return vs

    def copy(self, interval_min, interval_max, out=None):
        """interval is zero-min inside the bounding box (blockMin/blockMax, J/SparkAffineFusion.java:620-624)."""
        imin = np.asarray(interval_min, dtype=np.int64)
        imax = np.asarray(interval_max, dtype=np.int64)
        size = imax - imin + 1
        wmin = imin + np.asarray(self.bb_min, dtype=np.int64)
        vids = find_overlapping_views(self.view_dims, self.registrations, wmin, wmin + size - 1, self.view_ids)
        params = self.ctx.fuse_params(self.fusion_type, self.interpolation, self.out_dtype, self.blend_lut_n,
                                      self.min_intensity, self.max_intensity)
        return self.ctx.fuse_block(self.views_for(vids), wmin, size, params, out=out)

    def copy_to_volume(self, interval_min, interval_max) -> int:
        """Like copy(), but the block stays on the device: returns a resident-volume handle."""
        imin = np.asarray(interval_min, dtype=np.int64)
        size = np.asarray(interval_max, dtype=np.int64) - imin + 1
        wmin = imin + np.asarray(self.bb_min, dtype=np.int64)
        vids = find_overlapping_views(self.view_dims, self.registrations, wmin, wmin + size - 1, self.view_ids)
        params = self.ctx.fuse_params(self.fusion_type, self.interpolation, self.out_dtype, self.blend_lut_n,
                                      self.min_intensity, self.max_intensity)
        return self.ctx.fuse_block_to_volume(self.views_for(vids), wmin, size, params)


class BlkAffineFusion:
    """net.preibisch.mvrecon.process.fusion.blk.BlkAffineFusion (call site
    J/SparkAffineFusion.java:602-615)."""

    @staticmethod
    def init(ctx: Context, images: dict, registrations: dict, fusion_type="AVG_BLEND", interpolation=1,
             bounding_box=None, out_dtype="float32", min_intensity=0.0, max_intensity=65535.0,
             blend_lut_n=0, content_sigmas=(20.0, 40.0), resident_handles: dict | None = None) -> BlockSupplier:
        """images: ViewId -> [z,y,x] numpy volume (uploaded once and kept resident) -- or pass
        ``resident_handles`` (ViewId -> (handle, dims_xyz)) for volumes already on the device.
        registrations: ViewId -> adjusted 3x4 model.  bounding_box = (min_xyz, max_xyz)."""
        ft = native.FUSION_TYPES[fusion_type] if isinstance(fusion_type, str) else int(fusion_type)
        od = {"float32": native.DTYPE_F32, "uint16": native.DTYPE_U16, "uint8": native.DTYPE_U8}[out_dtype] \
            if isinstance(out_dtype, str) else int(out_dtype)
        view_ids = sorted(registrations)  # Collections.sort(sortedViewIds)
        handles, dims, content = {}, {}, {}
        for vid in view_ids:
            if resident_handles and vid in resident_handles:
                handles[vid], dims[vid] = resident_handles[vid]
            else:
                vol = images[vid]
                handles[vid] = ctx.volume_upload(vol)
                dims[vid] = tuple(vol.shape)[::-1]
            if ft in (native.FUSE_AVG_CONTENT, native.FUSE_AVG_BLEND_CONTENT):
                content[vid] = ctx.content_weights(handles[vid], *content_sigmas)
        regs = {vid: np.asarray(registrations[vid], dtype=np.float64).reshape(3, 4) for vid in view_ids}
        blending = {vid: adjust_blending(regs[vid]) for vid in view_ids}
        bb_min = tuple(bounding_box[0]) if bounding_box is not None else (0, 0, 0)
        return BlockSupplier(ctx, view_ids, dims, regs, handles, content, bb_min, ft, interpolation, od,
                             min_intensity, max_intensity, blend_lut_n, blending)


def fuse_volume(supplier: BlockSupplier, dimensions, block_size=(128, 128, 128), block_scale=(2, 2, 1),
                retries=5, sink=None):
    """The collapsed RDD of J/SparkAffineFusion.java:480-696: a host work queue over the grid of
    super-blocks with the reference's retry policy; ``sink(grid_block, array)`` receives each
    fused super-block (N5Utils.saveBlock in the reference, :670)."""
    compute = tuple(block_size[d] * block_scale[d] for d in range(3))
    grid = grid_create(dimensions, compute, block_size)
    out = None if sink is not None else np.zeros(tuple(dimensions)[::-1], dtype=native._BS2NP[supplier.out_dtype])
    attempt = 0
    while grid:
        attempt += 1
        if attempt > retries:
            raise RuntimeError(f"fusion: {len(grid)} block(s) still failing after {retries} attempts")
        failed = []
        for gb in grid:
            off, size, _ = gb
            try:
                blk = supplier.copy(off, tuple(off[d] + size[d] - 1 for d in range(3)))
            except native.BsError:
                failed.append(gb)
                continue
            if sink is not None:
                sink(gb, blk)
            else:
                out[off[2]:off[2] + size[2], off[1]:off[1] + size[1], off[0]:off[0] + size[0]] = blk
        grid = failed
    return out
