"""CPU oracle of `nonrigid-fusion`: float64 numpy restatement of PARITY_GAPS N2-N5.

TEST INFRASTRUCTURE ONLY (see oracle/pcm_oracle.py header): never imported by the product.

The arithmetic lives in multiview-reconstruction (NonRigidTools.fuseVirtualInterpolatedNonRigid, the MLS models of
mpicbg), which is not in the reference tree; SparkNonRigidFusion.call() (J/SparkNonRigidFusion.java:124-446) fixes the
call site and its parameters.  The recalled choices are the named constants below and the rows N1-N5 of PARITY_GAPS.md.
The MLS fit is written from the weighted normal equations in absolute coordinates, independently of the device's
moments-about-the-control-point form.

Arrays are [z, y, x]; triples are (x, y, z).
"""
from __future__ import annotations

import numpy as np

from . import fusion_oracle as fo

#: J/SparkNonRigidFusion.java:373-383
CP_DISTANCE = 10
ALPHA = 1.0
#: viewsToFuse / viewsToUse expansions of the transformed bounding boxes (J/SparkNonRigidFusion.java:333-336, :357-363)
FUSE_EXPAND = 50
USE_EXPAND = 25
#: N3: fewer points than this -> the inverse of the view's affine registration
MIN_POINTS = 4
#: N3: the fit is singular when det(P) <= SINGULAR_RTOL * (trace(P) / 3)^3 (P: weighted centred second moments)
SINGULAR_RTOL = 1e-10


def _apply(m12, pts):
    M = np.asarray(m12, dtype=np.float64).reshape(3, 4)
    return np.asarray(pts, dtype=np.float64) @ M[:, :3].T + M[:, 3]


def _bbox(dims_xyz, m12):
    M = np.asarray(m12, dtype=np.float64).reshape(3, 4)
    c = np.array([[x, y, z] for x in (0, dims_xyz[0] - 1) for y in (0, dims_xyz[1] - 1) for z in (0, dims_xyz[2] - 1)],
                 dtype=np.float64) @ M[:, :3].T + M[:, 3]
    return np.floor(c.min(axis=0)), np.ceil(c.max(axis=0))


def views_for_block(view_dims, registrations, block_min, block_max, view_ids):
    """(viewsToFuse, viewsToUse) of a block [block_min, block_max] (J/SparkNonRigidFusion.java:317-371)."""
    box = {v: _bbox(view_dims[v], registrations[v]) for v in view_ids}

    def overlap(a_lo, a_hi, b_lo, b_hi):
        return all(a_lo[d] <= b_hi[d] and b_lo[d] <= a_hi[d] for d in range(3))

    fuse = [v for v in view_ids if overlap(box[v][0] - FUSE_EXPAND, box[v][1] + FUSE_EXPAND, block_min, block_max)]
    use = [v for v in view_ids if any(overlap(box[v][0] - USE_EXPAND, box[v][1] + USE_EXPAND,
                                              box[f][0] - USE_EXPAND, box[f][1] + USE_EXPAND) for f in fuse)]
    return fuse, use


def target_positions(view, labels, views_to_use, points, correspondences, registrations):
    """N2: the (targets, locals) of one view to fuse.  ``points[(view, label)] = (ids, loc (n, 3))`` in full-resolution
    pixels; ``correspondences[(view, label)] = [(id, partner_view, partner_label, partner_id), ...]``;
    ``registrations[view]`` = 3x4 pixel -> world.  A point qualifies when at least one correspondence has its partner in
    ``views_to_use`` with a label in ``labels``; its target is the mean of its own world position and those partners'."""
    targets, locals_ = [], []
    for label in labels:
        if (view, label) not in points:
            continue
        ids, loc = points[(view, label)]
        index = {int(i): k for k, i in enumerate(ids)}
        partners = {}
        for (pid, pv, pl, qid) in correspondences.get((view, label), []):
            if pv in views_to_use and pl in labels:
                qids, qloc = points[(pv, pl)]
                q = int(np.nonzero(np.asarray(qids) == qid)[0][0])
                partners.setdefault(int(pid), []).append(_apply(registrations[pv], qloc[q][None])[0])
        for pid in sorted(partners, key=lambda i: index[i]):
            own = loc[index[pid]]
            world = [_apply(registrations[view], own[None])[0]] + partners[pid]
            targets.append(np.mean(world, axis=0))
            locals_.append(np.asarray(own, dtype=np.float64))
    return np.asarray(targets, dtype=np.float64).reshape(-1, 3), np.asarray(locals_, dtype=np.float64).reshape(-1, 3)


def grid_dims(block_size_xyz, cpd=(CP_DISTANCE,) * 3):
    """N4: control points per axis: the block [0, size - 1] plus one cell on every side."""
    return tuple(int(-(-(int(s) - 1) // int(c))) + 3 for s, c in zip(block_size_xyz, cpd))


def control_points(block_min_xyz, block_size_xyz, cpd=(CP_DISTANCE,) * 3):
    """World positions [gz, gy, gx, 3] of the control points block_min + (k - 1) * cpd."""
    g = grid_dims(block_size_xyz, cpd)
    ax = [float(block_min_xyz[d]) + (np.arange(g[d], dtype=np.float64) - 1.0) * cpd[d] for d in range(3)]
    Z, Y, X = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return np.stack([X, Y, Z], axis=-1)


def mls(x, targets, locals_, src_to_world, alpha=ALPHA):
    """N3: the MLS affine map target world -> local pixel evaluated at the world points ``x`` (..., 3)."""
    x = np.asarray(x, dtype=np.float64)
    shape = x.shape
    x = x.reshape(-1, 3)
    inv = fo.invert_affine(src_to_world)
    out = x @ inv[:, :3].T + inv[:, 3]                    # the fallback
    t = np.asarray(targets, dtype=np.float64).reshape(-1, 3)
    l = np.asarray(locals_, dtype=np.float64).reshape(-1, 3)
    if len(t) < MIN_POINTS:
        return out.reshape(shape)
    for s in range(0, len(x), 256):
        xs = x[s:s + 256]
        d2 = ((xs[:, None, :] - t[None, :, :]) ** 2).sum(axis=-1)        # (m, n)
        for i in range(len(xs)):
            on = np.nonzero(d2[i] == 0.0)[0]
            if len(on):
                out[s + i] = l[on[0]]
                continue
            w = 1.0 / d2[i] ** alpha
            W = w.sum()
            tc = (w[:, None] * t).sum(axis=0) / W
            lc = (w[:, None] * l).sum(axis=0) / W
            dt, dl = t - tc, l - lc
            P = (w[:, None, None] * dt[:, :, None] * dt[:, None, :]).sum(axis=0)
            Q = (w[:, None, None] * dt[:, :, None] * dl[:, None, :]).sum(axis=0)
            det = np.linalg.det(P)
            if not (det > SINGULAR_RTOL * (np.trace(P) / 3.0) ** 3) or not np.isfinite(det):
                continue
            A = np.linalg.solve(P, Q).T                   # A P = Q^T
            out[s + i] = lc + A @ (xs[i] - tc)
    return out.reshape(shape)


def mls_grid(targets, locals_, src_to_world, block_min_xyz, block_size_xyz, cpd=(CP_DISTANCE,) * 3):
    """N4: the mapped source coordinate of every control point, float64 [gz, gy, gx, 3]."""
    return mls(control_points(block_min_xyz, block_size_xyz, cpd), targets, locals_, src_to_world)


def source_coords(grid, block_size_xyz, cpd=(CP_DISTANCE,) * 3):
    """N4: per output voxel the trilinear interpolation of its 8 surrounding control points (float64, then float32)."""
    idx, frac = [], []
    for d in range(3):
        o = np.arange(int(block_size_xyz[d]))
        idx.append(o // cpd[d] + 1)
        frac.append((o % cpd[d]) / float(cpd[d]))
    cz, cy, cx = np.meshgrid(idx[2], idx[1], idx[0], indexing="ij")
    fz, fy, fx = (f[..., None] for f in np.meshgrid(frac[2], frac[1], frac[0], indexing="ij"))
    g = lambda dz, dy, dx: grid[cz + dz, cy + dy, cx + dx]
    c00 = g(0, 0, 0) * (1 - fx) + g(0, 0, 1) * fx
    c01 = g(0, 1, 0) * (1 - fx) + g(0, 1, 1) * fx
    c10 = g(1, 0, 0) * (1 - fx) + g(1, 0, 1) * fx
    c11 = g(1, 1, 0) * (1 - fx) + g(1, 1, 1) * fx
    c0 = c00 * (1 - fy) + c01 * fy
    c1 = c10 * (1 - fy) + c11 * fy
    return (c0 * (1 - fz) + c1 * fz).astype(np.float32)


def fuse_block(views, block_min_xyz, block_size_xyz, cpd=(CP_DISTANCE,) * 3, out_dtype="float32", min_intensity=0.0,
               max_intensity=65535.0):
    """N5: non-rigid AVG_BLEND fusion of one block.  ``views``: ascending ViewId order of dicts(img [z,y,x] full
    resolution, src_to_world, targets, locals, blend_border, blend_range).  Returns [bz, by, bx] of ``out_dtype``."""
    bx, by, bz = (int(v) for v in block_size_xyz)
    sum_i = np.zeros((bz, by, bx), dtype=np.float32)
    sum_w = np.zeros((bz, by, bx), dtype=np.float32)
    for v in views:
        dims = v["img"].shape[::-1]
        grid = mls_grid(v["targets"], v["locals"], v["src_to_world"], block_min_xyz, block_size_xyz, cpd)
        src = source_coords(grid, block_size_xyz, cpd)
        inside = fo.inside_mask(src, dims)
        if not inside.any():
            continue
        border, rng = v.get("blend_border"), v.get("blend_range")
        if border is None:
            border, rng = fo.adjust_blending(v["src_to_world"])
        w = np.where(inside, fo.blend_weight(src, dims, border, rng), np.float32(0)).astype(np.float32)
        val = fo.trilinear(v["img"], src)
        sum_i = (sum_i + w * val).astype(np.float32)
        sum_w = (sum_w + w).astype(np.float32)
    out = np.zeros((bz, by, bx), dtype=np.float32)
    np.divide(sum_i, sum_w, out=out, where=sum_w > 0)
    return fo.convert_output(out, out_dtype, min_intensity, max_intensity)
