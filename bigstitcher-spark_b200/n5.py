"""Minimal N5 reader / writer for the data formats either side of the hot path (SURVEY.md 8f-1,
Appendix B; n5 3.5.0, pom.xml:109-111).

Covers what `stitching` / `affine-fusion` touch: dataset `attributes.json`, block files
`<dataset>/<gx>/<gy>/<gz>` with the big-endian header (uint16 mode, uint16 ndim, ndim x uint32
block dims) followed by big-endian x-fastest elements, `raw`, `gzip` and `zstd` compression (zstd, the reference's default J/CreateFusionContainer.java:71-76,
through the in-repo codec zstd.py), the BDV-N5
input layout `setup{S}/timepoint{T}/s{L}` and the container root attributes `Bigstitcher-Spark/*`
(J/CreateFusionContainer.java:302-320,519; read back at J/SparkAffineFusion.java:241-307).
Host-side plumbing only -- no voxel arithmetic.
"""
from __future__ import annotations

import gzip
import json
import os
import shutil
import struct
import zlib

import numpy as np

from . import zstd as bzstd

BS_KEY = "Bigstitcher-Spark"


def bs_attrs(flat: dict) -> dict:
    """`setAttribute("/", "Bigstitcher-Spark/InputXML", v)` of N5 3.x treats '/' as a JSON path: the attributes
    are written as ONE nested object {"Bigstitcher-Spark": {"InputXML": v, ...}} (J/CreateFusionContainer.java:302-320)."""
    return {BS_KEY: dict(flat)}


def bs_attr_get(attrs: dict, key, default=None):
    """Read `Bigstitcher-Spark/<key>`: the nested form the reference writes, or the flat key with a literal slash
    that round-1 containers of this build used."""
    nested = attrs.get(BS_KEY)
    if isinstance(nested, dict) and key in nested:
        return nested[key]
    return attrs.get(BS_KEY + "/" + key, default)

_DTYPES = {"uint8": np.uint8, "uint16": np.uint16, "uint32": np.uint32, "uint64": np.uint64, "int16": np.int16,
           "float32": np.float32, "float64": np.float64}


def _dtype_name(dt):
    dt = np.dtype(dt)
    for k, v in _DTYPES.items():
        if np.dtype(v) == dt:
            return k
    raise ValueError(f"unsupported dtype {dt}")


class N5Store:
    """Filesystem N5 container."""

    def __init__(self, root: str, create: bool = False):
        self.root = root
        if create:
            os.makedirs(root, exist_ok=True)
            if not os.path.exists(os.path.join(root, "attributes.json")):
                self.set_attributes("", {"n5": "2.5.1"})
        elif not os.path.isdir(root):
            raise FileNotFoundError(root)

    # -- attributes
    def _attr_path(self, group):
        return os.path.join(self.root, group.strip("/"), "attributes.json")

    def get_attributes(self, group=""):
        p = self._attr_path(group)
        if not os.path.exists(p):
            return {}
        with open(p) as f:
            return json.load(f)

    def set_attributes(self, group, attrs: dict):
        p = self._attr_path(group)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        cur = self.get_attributes(group)
        for k, v in attrs.items():
            if k == BS_KEY and isinstance(v, dict) and isinstance(cur.get(k), dict):
                cur[k].update(v)
            else:
                cur[k] = v
        with open(p, "w") as f:
            json.dump(cur, f)

    # -- datasets
    def create_dataset(self, path, dimensions, block_size, dtype, compression="raw", level=None):
        comp = {"type": compression}
        if compression == "gzip":
            comp["level"] = 1  # reference default, J/util/N5Util.java:82-105
        elif compression == "zstd":
            comp["level"] = 3  # reference default (J/CreateFusionContainer.java:71-76, J/util/N5Util.java:91-92)
        if compression != "raw" and level is not None:
            comp["level"] = int(level)
        self.set_attributes(path, {"dimensions": [int(d) for d in dimensions],
                                   "blockSize": [int(b) for b in block_size],
                                   "dataType": _dtype_name(dtype), "compression": comp})

    def dataset_attributes(self, path):
        a = self.get_attributes(path)
        if "dimensions" not in a:
            raise KeyError(f"{path} is not an N5 dataset")
        return a

    def _block_path(self, path, grid_pos):
        return os.path.join(self.root, path.strip("/"), *[str(int(g)) for g in grid_pos])

    def write_block(self, path, grid_pos, block: np.ndarray):
        """block: [z, y, x] array (x fastest), at most blockSize in every dimension."""
        a = self.dataset_attributes(path)
        dt = np.dtype(_DTYPES[a["dataType"]])
        if block.dtype.newbyteorder("=") != dt:      # big-endian blocks (swapped on the device) pass through as they are
            raise ValueError(f"block dtype {block.dtype} != dataset dtype {dt}")
        dims_xyz = block.shape[::-1]
        header = struct.pack(">HH", 0, len(dims_xyz)) + b"".join(struct.pack(">I", int(d)) for d in dims_xyz)
        payload = np.ascontiguousarray(block).astype(dt.newbyteorder(">"), copy=False).tobytes()
        ctype = a["compression"]["type"]
        if ctype == "gzip":
            payload = gzip.compress(payload, compresslevel=a["compression"].get("level", 1))
        elif ctype == "zstd":
            payload = bzstd.compress(payload, a["compression"].get("level", bzstd.DEFAULT_LEVEL))
        elif ctype != "raw":
            raise NotImplementedError(f"compression {ctype} (not available in this image)")
        p = self._block_path(path, grid_pos)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(header + payload)

    def read_block(self, path, grid_pos):
        """Returns the [z, y, x] block or None when the block file does not exist."""
        a = self.dataset_attributes(path)
        p = self._block_path(path, grid_pos)
        if not os.path.exists(p):
            return None
        with open(p, "rb") as f:
            buf = f.read()
        mode, ndim = struct.unpack(">HH", buf[:4])
        if mode != 0:
            raise NotImplementedError("varlength / object N5 blocks")
        dims = struct.unpack(">" + "I" * ndim, buf[4:4 + 4 * ndim])
        payload = buf[4 + 4 * ndim:]
        ctype = a["compression"]["type"]
        if ctype == "gzip":
            payload = zlib.decompress(payload, 16 + zlib.MAX_WBITS)
        elif ctype == "zstd":
            payload = bzstd.decompress(payload)
        elif ctype != "raw":
            raise NotImplementedError(f"compression {ctype}")
        dt = np.dtype(_DTYPES[a["dataType"]])
        arr = np.frombuffer(payload, dtype=dt.newbyteorder(">"), count=int(np.prod(dims)))
        return arr.astype(dt).reshape(dims[::-1])

    def read_volume(self, path):
        """Whole dataset as a [z, y, x] array (missing blocks are zero)."""
        a = self.dataset_attributes(path)
        dims = a["dimensions"]
        bs = a["blockSize"]
        out = np.zeros(dims[::-1], dtype=_DTYPES[a["dataType"]])
        grid = [int(np.ceil(dims[d] / bs[d])) for d in range(3)]
        for gz in range(grid[2]):
            for gy in range(grid[1]):
                for gx in range(grid[0]):
                    b = self.read_block(path, (gx, gy, gz))
                    if b is None:
                        continue
                    z, y, x = b.shape
                    out[gz * bs[2]:gz * bs[2] + z, gy * bs[1]:gy * bs[1] + y, gx * bs[0]:gx * bs[0] + x] = b
        return out

    def read_region(self, path, min_xyz, size_xyz):
        """[z, y, x] array of the interval [min, min + size) -- only the storage blocks it touches are read
        (missing blocks / parts outside the dataset are zero)."""
        a = self.dataset_attributes(path)
        dims, bs = a["dimensions"], a["blockSize"]
        mn = [int(v) for v in min_xyz]
        sz = [int(v) for v in size_xyz]
        out = np.zeros(sz[::-1], dtype=_DTYPES[a["dataType"]])
        lo = [max(0, mn[d]) for d in range(3)]
        hi = [min(dims[d], mn[d] + sz[d]) for d in range(3)]     # exclusive
        if any(hi[d] <= lo[d] for d in range(3)):
            return out
        for gz in range(lo[2] // bs[2], -(-hi[2] // bs[2])):
            for gy in range(lo[1] // bs[1], -(-hi[1] // bs[1])):
                for gx in range(lo[0] // bs[0], -(-hi[0] // bs[0])):
                    b = self.read_block(path, (gx, gy, gz))
                    if b is None:
                        continue
                    b0 = (gx * bs[0], gy * bs[1], gz * bs[2])
                    bz, by, bx = b.shape
                    s0 = [max(lo[d], b0[d]) for d in range(3)]
                    s1 = [min(hi[0], b0[0] + bx), min(hi[1], b0[1] + by), min(hi[2], b0[2] + bz)]
                    if any(s1[d] <= s0[d] for d in range(3)):
                        continue
                    out[s0[2] - mn[2]:s1[2] - mn[2], s0[1] - mn[1]:s1[1] - mn[1], s0[0] - mn[0]:s1[0] - mn[0]] = \
                        b[s0[2] - b0[2]:s1[2] - b0[2], s0[1] - b0[1]:s1[1] - b0[1], s0[0] - b0[0]:s1[0] - b0[0]]
        return out

    def save_block(self, path, volume: np.ndarray, grid_offset):
        """N5Utils.saveBlock(img, writer, dataset, gridOffset) (J/SparkAffineFusion.java:670): split
        a super-block into storage blocks starting at grid position ``grid_offset`` and write them."""
        a = self.dataset_attributes(path)
        bs = a["blockSize"]
        dims = a["dimensions"]
        sz = volume.shape[::-1]
        n = [int(np.ceil(sz[d] / bs[d])) for d in range(3)]
        for kz in range(n[2]):
            for ky in range(n[1]):
                for kx in range(n[0]):
                    g = (grid_offset[0] + kx, grid_offset[1] + ky, grid_offset[2] + kz)
                    if any(g[d] * bs[d] >= dims[d] for d in range(3)):
                        continue
                    blk = volume[kz * bs[2]:(kz + 1) * bs[2], ky * bs[1]:(ky + 1) * bs[1], kx * bs[0]:(kx + 1) * bs[0]]
                    self.write_block(path, g, blk)

    def write_list(self, path, values: np.ndarray, block_length, compression="raw"):
        """A list of n k-vectors as the 2-D dataset {k, n} (k fastest) in blocks {k, block_length}, the layout of
        InterestPointsN5 and the --storeIntensities dataset; an empty list is the 1-D dataset {0}, block {1}, with
        no block files (J/SparkInterestPointDetection.java:917-925)."""
        values = np.asarray(values)
        if values.shape[0] == 0:
            self.create_dataset(path, [0], [1], values.dtype, compression)
            return
        k = values.shape[1]
        self.create_dataset(path, [k, values.shape[0]], [k, block_length], values.dtype, compression)
        for j, s0 in enumerate(range(0, values.shape[0], block_length)):
            self.write_block(path, (0, j), np.ascontiguousarray(values[s0:s0 + block_length]))

    def read_list(self, path) -> np.ndarray:
        """The (n, k) array of a dataset written by write_list ((0, 0) when empty)."""
        a = self.dataset_attributes(path)
        dims, bs = a["dimensions"], a["blockSize"]
        dt = _DTYPES[a["dataType"]]
        if len(dims) == 1:
            return np.zeros((0, 0), dtype=dt)
        out = np.zeros((dims[1], dims[0]), dtype=dt)
        for j in range(-(-dims[1] // bs[1])):
            b = self.read_block(path, (0, j))
            if b is not None:
                out[j * bs[1]:j * bs[1] + b.shape[0]] = b
        return out

    def read_correspondences(self, group):
        """Correspondences of one label of one view in interestpoints.n5 (``group`` = `tpId_{t}_viewSetupId_{s}/{label}`):
        the uint64 dataset `correspondences/data` {3, M} of (detectionId, correspondingDetectionId, idMap index) rows and
        the group attribute idMap {"tp,setup,label": index}.  Returns a list of (detection id, (tp, setup), label,
        corresponding detection id); [] when the view has no correspondences (dataset {0} or absent)."""
        rows, keys = self.read_correspondence_table(group)
        return [(int(a), keys[int(c)][0], keys[int(c)][1], int(b)) for a, b, c in rows]

    def read_correspondence_table(self, group):
        """The same correspondences as arrays: (uint64 (M, 3) rows of (detection id, corresponding detection id, idMap
        index), {idMap index: ((tp, setup), label)})."""
        path = group.rstrip("/") + "/correspondences"
        attrs = self.get_attributes(path)
        if "idMap" not in attrs or "dimensions" not in self.get_attributes(path + "/data"):
            return np.zeros((0, 3), dtype=np.uint64), {}
        keys = {}
        for k, idx in attrs["idMap"].items():
            tp, setup, label = k.split(",", 2)
            keys[int(idx)] = ((int(tp), int(setup)), label)
        return np.asarray(self.read_list(path + "/data"), dtype=np.uint64).reshape(-1, 3), keys

    def write_correspondences(self, group, rows):
        """The inverse of read_correspondences: ``rows`` [(detection id, (tp, setup), label, corresponding detection id)]
        become group attributes correspondences = "1.0.0" and idMap {"tp,setup,label": index} (numbered in sorted key
        order) and the zstd uint64 dataset `correspondences/data` {3, M} in the given row order; {0} when empty.  An
        earlier `correspondences` group is replaced."""
        path = group.rstrip("/") + "/correspondences"
        keys = sorted({(tuple(int(x) for x in pv), str(pl)) for _, pv, pl, _ in rows})
        idmap = {f"{pv[0]},{pv[1]},{pl}": i for i, (pv, pl) in enumerate(keys)}
        shutil.rmtree(os.path.join(self.root, path), ignore_errors=True)
        self.set_attributes(path, {"correspondences": "1.0.0", "idMap": idmap})
        data = np.array([(int(a), int(b), idmap[f"{int(pv[0])},{int(pv[1])},{pl}"]) for a, pv, pl, b in rows],
                        dtype=np.uint64).reshape(-1, 3)
        self.write_list(path + "/data", data, 300000, "zstd")

    def write_volume(self, path, volume: np.ndarray, block_size, compression="raw"):
        self.create_dataset(path, volume.shape[::-1], block_size, volume.dtype, compression)
        self.save_block(path, volume, (0, 0, 0))


# ---------------------------------------------------------------------------------------------
# BDV-N5 input layout and the fusion-container contract
def bdv_dataset(setup: int, timepoint: int, level: int = 0) -> str:
    """`setup{S}/timepoint{T}/s{L}` (J/util/Import.java:319-326)."""
    return f"setup{setup}/timepoint{timepoint}/s{level}"


def set_bdv_attributes(store: N5Store, setup: int, timepoint: int, factors, dtype):
    """The BDV-N5 metadata of one view (PARITY_GAPS R6): `setup{S}` gets the absolute `downsamplingFactors` of every
    level and `dataType`, `setup{S}/timepoint{T}` gets `resolution` [1, 1, 1] and `multiScale` true."""
    store.set_attributes(f"setup{setup}", {"downsamplingFactors": [list(f) for f in factors],
                                           "dataType": _dtype_name(dtype)})
    store.set_attributes(f"setup{setup}/timepoint{timepoint}", {"resolution": [1.0, 1.0, 1.0], "multiScale": True})


def write_bdv_setup(store: N5Store, setup: int, timepoint: int, volume: np.ndarray, block_size=(128, 128, 128),
                    downsampling_factors=((1, 1, 1),), compression="raw"):
    set_bdv_attributes(store, setup, timepoint, downsampling_factors, volume.dtype)
    store.write_volume(bdv_dataset(setup, timepoint, 0), volume, block_size, compression)


def create_fusion_container(root, input_xml, bb_min, bb_max, block_size=(128, 128, 128), dtype="float32",
                            min_intensity=None, max_intensity=None, num_timepoints=1, num_channels=1,
                            anisotropy_factor=None, compression="raw", downsamplings=(), output_xml=None):
    """`create-fusion-container -s N5` (J/CreateFusionContainer.java:302-320,490-519): per
    (channel, timepoint) dataset `ch{c}tp{t}/s0` plus the `Bigstitcher-Spark/*` root attributes
    that `affine-fusion` reads back (J/SparkAffineFusion.java:241-307).

    With ``output_xml`` (`--bdv -xo`, :391-487) the volumes are BDV-N5 views instead: view (t, setup c) at
    `setup{c}/timepoint{t}/s{l}` with the BDV-N5 attributes (set_bdv_attributes), FusionFormat "BDV/N5" and
    OutputXML = ``output_xml``.  Either way MultiResolutionInfos[c + t * num_channels] holds volume (c, t), the
    index affine-fusion reads (J/SparkAffineFusion.java:454)."""
    store = N5Store(root, create=True)
    dims = [int(bb_max[d] - bb_min[d] + 1) for d in range(3)]
    name = bdv_dataset if output_xml else (lambda c, t, lvl: f"ch{c}tp{t}/s{lvl}")
    mr = []
    for t in range(num_timepoints):
        for c in range(num_channels):
            ds = name(c, t, 0)
            store.create_dataset(ds, dims, block_size, _DTYPES[dtype], compression)
            levels = [{"dataset": ds, "dimensions": dims, "blockSize": list(block_size),
                       "relativeDownsampling": [1, 1, 1], "absoluteDownsampling": [1, 1, 1], "dataType": dtype}]
            # --multiRes: s1, s2, ... with relative 2x steps (N5ApiTools.setupMultiResolutionPyramid,
            # J/CreateFusionContainer.java:260-270)
            cur, absd = list(dims), [1, 1, 1]
            for lvl, rel in enumerate(downsamplings, start=1):
                cur = [cur[d] // int(rel[d]) for d in range(3)]
                absd = [absd[d] * int(rel[d]) for d in range(3)]
                dsl = name(c, t, lvl)
                store.create_dataset(dsl, cur, block_size, _DTYPES[dtype], compression)
                levels.append({"dataset": dsl, "dimensions": list(cur), "blockSize": list(block_size),
                               "relativeDownsampling": [int(v) for v in rel], "absoluteDownsampling": list(absd),
                               "dataType": dtype})
            if output_xml:
                set_bdv_attributes(store, c, t, [lv["absoluteDownsampling"] for lv in levels], _DTYPES[dtype])
            mr.append(levels)
    flat = {"FusionFormat": "BDV/N5" if output_xml else "N5", "InputXML": input_xml,
            "NumTimepoints": num_timepoints, "NumChannels": num_channels,
            "Boundingbox_min": [int(v) for v in bb_min], "Boundingbox_max": [int(v) for v in bb_max],
            "PreserveAnisotropy": anisotropy_factor is not None,
            "DataType": dtype.lower(),      # N5's DataType adapter (de)serialises lowercase names
            "BlockSize": list(block_size), "MultiResolutionInfos": mr}
    if anisotropy_factor is not None:
        flat["AnisotropyFactor"] = float(anisotropy_factor)
    if dtype != "float32":
        flat["MinIntensity"] = float(min_intensity)
        flat["MaxIntensity"] = float(max_intensity)
    if output_xml:
        flat["OutputXML"] = output_xml
    attrs = bs_attrs(flat)
    store.set_attributes("", attrs)
    return store


def parse_fusion_metadata(a: dict):
    """Bigstitcher-Spark/* -> the dict `affine-fusion` works with (J/SparkAffineFusion.java:241-307)."""
    g = lambda k, d=None: bs_attr_get(a, k, d)  # noqa: E731
    if g("FusionFormat") is None:
        raise KeyError("not a BigStitcher-Spark fusion container (no Bigstitcher-Spark/FusionFormat)")
    return {
        "format": g("FusionFormat"), "input_xml": g("InputXML"), "num_timepoints": g("NumTimepoints", 1),
        "num_channels": g("NumChannels", 1), "bb_min": g("Boundingbox_min"), "bb_max": g("Boundingbox_max"),
        "preserve_anisotropy": g("PreserveAnisotropy", False), "anisotropy_factor": g("AnisotropyFactor", float("nan")),
        "dtype": str(g("DataType", "float32")).lower(), "block_size": g("BlockSize"),
        "min_intensity": g("MinIntensity", 0.0), "max_intensity": g("MaxIntensity", 65535.0),
        "mr_infos": g("MultiResolutionInfos"),
    }


def read_fusion_container(root):
    """The metadata `affine-fusion` needs (J/SparkAffineFusion.java:241-307)."""
    store = N5Store(root)
    return store, parse_fusion_metadata(store.get_attributes(""))
