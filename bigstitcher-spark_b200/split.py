"""split-images (J/SplitDatasets.java:91-124; SplittingTools.splitImages and the Split_Views helpers it calls are
recalled, PARITY_GAPS P1-P8): the plan that cuts every view into overlapping boxes, the SpimData2 project of the boxes
read through a `split.viewerimgloader`, and the fake corresponding interest points that keep the pieces of one view
together.  Host bookkeeping only: the image data of the new views is read through viewsource.SplitViews by the existing
device paths.
"""
from __future__ import annotations

import copy
import math
import xml.etree.ElementTree as ET

import numpy as np

from .spimdata import SPLIT_LOADER, SpimData2, _fmt

SPLIT_TRANSFORM = "Image Splitting"


def parse_size(value, what):
    """"512,512,256" or a 3-tuple -> (x, y, z) ints."""
    parts = [p for p in value.split(",") if p.strip()] if isinstance(value, str) else list(value)
    if len(parts) != 3:
        raise ValueError(f"{what} needs three values x,y,z: {value!r}")
    out = tuple(int(p) for p in parts)
    if any(v < 0 for v in out):
        raise ValueError(f"{what} must not be negative: {value!r}")
    return out


def closest_larger_divisible(value, step):
    """Split_Views.closestLargerLongDivisableBy: the smallest multiple of ``step`` that is >= ``value``."""
    return -(-int(value) // int(step)) * int(step)


def min_step(src, views):
    """Split_Views.findMinStepSize: per axis the lcm of every view's mipmap factors, so a box starting at a multiple
    of it starts on a whole voxel of every level (PARITY_GAPS P2)."""
    m = [1, 1, 1]
    for v in views:
        for f in src.mipmap_info(v)[0]:
            m = [math.lcm(m[d], int(f[d])) for d in range(3)]
    return tuple(m)


def intervals(length, size, overlap, step, optimize=True):
    """The [start, end] (inclusive) intervals one axis of ``length`` voxels is cut into (PARITY_GAPS P1).  Without
    optimisation: starts 0, size - overlap, ... while start + size < length, then one last interval from the next start
    to the end.  With it: the same count n, every interval S long, S the smallest multiple of ``step`` with
    n (S - overlap) + overlap >= length, the last one clipped at the end.  ``size`` and ``overlap`` are multiples of
    ``step``, so every start is."""
    L, s, o, m = int(length), int(size), int(overlap), int(step)
    if L <= s:
        return [(0, L - 1)]
    if o >= s:
        raise ValueError(f"overlap {o} must be smaller than the image size {s} to split an axis of {L} voxels")
    starts, st = [], 0
    while st + s < L:
        starts.append(st)
        st += s - o
    if not optimize:
        return [(a, a + s - 1) for a in starts] + [(st, L - 1)]
    n = len(starts) + 1
    S = closest_larger_divisible(o + -(-(L - o) // n), m)
    return [(i * (S - o), min(i * (S - o) + S - 1, L - 1)) for i in range(n)]


def boxes(dims_xyz, size, overlap, step, optimize=True):
    """The boxes of one view: the product of the per-axis intervals, x fastest; [(min int64[3], max int64[3])]."""
    ax = [intervals(dims_xyz[d], size[d], overlap[d], step[d], optimize) for d in range(3)]
    return [(np.array([x[0], y[0], z[0]], dtype=np.int64), np.array([x[1], y[1], z[1]], dtype=np.int64))
            for z in ax[2] for y in ax[1] for x in ax[0]]


# --------------------------------------------------------------------------------------------- the new project
def split_project(data: SpimData2, plan, assign_illuminations, xml_out) -> SpimData2:
    """The SpimData2 of the sub-views.  ``plan``: {new setup: (old setup, min, max, local index)}, new ids in old-setup
    then box order.  Setups take the box size and the old setup's other fields; tile ids become old tile * spread +
    local index (spread = the most boxes of any old setup) and <Attributes name="tile"> is rebuilt with the box min added
    to each location (P3); ``assign_illuminations`` makes the old tile the illumination.  Each view's transform list
    gets a translation by the box min, applied first; missing views stay missing; the ImageLoader wraps the input's
    (flattened when it already is a split loader, P5).  Stitching results, intensity adjustments, PSFs and interest
    points are emptied, bounding boxes kept (P8).  Not saved."""
    tiles_old = data.attribute_entries("tile")
    if assign_illuminations and len({s.attributes.get("illumination", 0) for s in data.setups.values()}) > 1:
        raise ValueError("Cannot assign tiles as illuminations: the dataset has more than one illumination.")
    spread = max(p[3] for p in plan.values()) + 1
    new = SpimData2(ET.ElementTree(copy.deepcopy(data.root)), xml_out)
    root = new.root

    # ---- view setups
    vss = root.find("SequenceDescription").find("ViewSetups")
    old_el = {int(vs.findtext("id")): vs for vs in vss.findall("ViewSetup")}
    for vs in old_el.values():
        vss.remove(vs)
    tiles_new, illums = {}, {}
    for pos, (nid, (old, mn, mx, k)) in enumerate(sorted(plan.items())):
        vs = copy.deepcopy(old_el[old])
        vs.find("id").text = str(nid)
        if vs.find("name") is not None:
            vs.find("name").text = str(nid)
        vs.find("size").text = " ".join(str(int(mx[d] - mn[d] + 1)) for d in range(3))
        at = vs.find("attributes")
        if at is None:
            at = ET.SubElement(vs, "attributes")
        old_tile = data.setups[old].attributes.get("tile", old)
        tile = old_tile * spread + k
        _set_child(at, "tile", tile)
        if tiles_old is not None and tile not in tiles_new:
            e = tiles_old.get(old_tile, {})
            loc = e.get("location")
            tiles_new[tile] = dict(name=str(tile), location=None if loc is None else loc + mn)
        if assign_illuminations:
            _set_child(at, "illumination", old_tile)
            illums[old_tile] = dict(name=(tiles_old or {}).get(old_tile, {}).get("name") or str(old_tile))
        vss.insert(pos, vs)
    if tiles_old is not None:
        new.set_attribute_entries("tile", tiles_new)
    if assign_illuminations:
        new.set_attribute_entries("illumination", illums)

    # ---- registrations: the old list, then the box offset (the last entry is applied first)
    vrs = root.find("ViewRegistrations")
    old_vr = {(int(vr.get("timepoint")), int(vr.get("setup"))): vr for vr in vrs.findall("ViewRegistration")}
    for vr in old_vr.values():
        vrs.remove(vr)
    for (tp, old), vr in sorted(old_vr.items()):
        for nid, (o, mn, mx, k) in sorted(plan.items()):
            if o != old:
                continue
            e = copy.deepcopy(vr)
            e.set("setup", str(nid))
            vt = ET.SubElement(e, "ViewTransform", type="affine")
            ET.SubElement(vt, "Name").text = SPLIT_TRANSFORM
            ET.SubElement(vt, "affine").text = _fmt([1, 0, 0, mn[0], 0, 1, 0, mn[1], 0, 0, 1, mn[2]])
            vrs.append(e)

    new.set_missing_views({(tp, nid) for (tp, old) in data.missing_views()
                           for nid, p in plan.items() if p[0] == old})
    for tag in ("StitchingResults", "IntensityAdjustments", "PointSpreadFunctions", "ViewInterestPoints"):
        el = root.find(tag)
        for ch in (list(el) if el is not None else []):
            el.remove(ch)

    # ---- the split loader over the input's own loader: a split of a split composes onto the original views
    parent = data.split_setups()
    nested = data.root.find("SequenceDescription").find("ImageLoader")
    container = data.image_loader()[1]
    defs = {}
    for nid, (old, mn, mx, _) in plan.items():
        if parent:
            po, pmin, _ = parent[old]
            defs[nid] = (po, pmin + mn, pmin + mx)
        else:
            defs[nid] = (old, mn, mx)
    if nested.get("format") == SPLIT_LOADER:
        nested = nested.find("ImageLoader")
        container = data.image_loader(nested=True)[1]
    new.set_split_image_loader(nested, container, defs, xml_out)
    return SpimData2(new.tree, xml_out)


def _set_child(parent, tag, value):
    el = parent.find(tag)
    if el is None:
        el = ET.SubElement(parent, tag)
    el.text = str(int(value))


# --------------------------------------------------------------------------------------------- fake interest points
_M64 = (1 << 64) - 1


def splitmix64(z):
    """The splitmix64 finaliser of intensity.cu (PARITY I1), on Python ints."""
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def stream_key(*ids):
    k = 0
    for v in ids:
        k = splitmix64(k ^ (int(v) & _M64))
    return k


def draw(key, n, count):
    """Draw ``n`` of a counter-based stream: ``count`` uniforms in [0, 1) from counters n * count ...  (53-bit)."""
    return np.array([(splitmix64(key ^ (n * count + c)) >> 11) * (1.0 / (1 << 53)) for c in range(count)])


def _near(points, p, r2):
    return len(points) > 0 and float(np.min(np.sum((points - p) ** 2, axis=1))) < r2


def fake_points(tp, old, view_boxes, existing, density, min_points, max_points, error, radius):
    """The fake corresponding points of one view at one timepoint (PARITY_GAPS P7).  For every pair i < j of its boxes
    whose closed boxes intersect, n = min(max, max(min, ceil(density * V / 1e6))) points, V the intersection's voxel
    count: candidates p uniform in the intersection (parent pixels) with an error e uniform in [-error, error]^3, drawn
    from the stream keyed (tp, old, i, j); rejected when p or p + e lies closer than ``radius`` to an ``existing`` point
    of the parent, p to a fake point of box i or p + e to one of box j.  At most 100 n draws.  Returns ({box: (k, 3)
    parent-pixel positions, ids = row index}, {(i, j): [(id in i, id in j)]})."""
    existing = np.asarray(existing, dtype=np.float64).reshape(-1, 3)
    tree = None
    if len(existing):
        from scipy.spatial import cKDTree
        tree = cKDTree(existing)
    r2 = float(radius) ** 2
    fakes = {i: np.zeros((0, 3)) for i in range(len(view_boxes))}
    pairs = {}
    for i, (mni, mxi) in enumerate(view_boxes):
        for j in range(i + 1, len(view_boxes)):
            mnj, mxj = view_boxes[j]
            lo, hi = np.maximum(mni, mnj).astype(np.float64), np.minimum(mxi, mxj).astype(np.float64)
            if np.any(hi < lo):
                continue
            vox = float(np.prod(hi - lo + 1))
            n = min(int(max_points), max(int(min_points), math.ceil(float(density) * vox / 1e6)))
            key = stream_key(tp, old, i, j)
            got = []
            for k in range(100 * n):
                if len(got) >= n:
                    break
                u = draw(key, k, 6)
                p = lo + u[:3] * (hi - lo)
                q = p + (2.0 * u[3:] - 1.0) * float(error)
                if tree is not None and (tree.query(p)[0] < radius or tree.query(q)[0] < radius):
                    continue
                if _near(fakes[i], p, r2) or _near(fakes[j], q, r2):
                    continue
                fakes[i] = np.vstack([fakes[i], p])
                fakes[j] = np.vstack([fakes[j], q])
                got.append((len(fakes[i]) - 1, len(fakes[j]) - 1))
            pairs[(i, j)] = got
    return fakes, pairs
