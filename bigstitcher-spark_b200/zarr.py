"""Minimal OME-Zarr (Zarr v2) writer / reader for the fusion output -- the reference's DEFAULT
container (J/CreateFusionContainer.java:67-69,331-389): one 5-D array per resolution level, N5-API
axis order x,y,z,c,t == Zarr array order t,c,z,y,x, chunks {1,1,bz,by,bx}, levels named "0","1",...
(:346), `multiscales` v0.4 metadata (:374-388), grid offsets {gx,gy,gz,c,t} at write time
(J/SparkAffineFusion.java:630-643).  Little-endian C-order chunks, always full chunk shape (edge
chunks padded with fill_value 0), dimension_separator "/"; compressor null (raw), gzip or zstd (the reference default,
through zstd.py).

The reader also takes 5-D arrays written by other tools (the `bdv.multimg.zarr` input of every command): dtypes in
any byte order ('<', '>', '|'), both dimension separators ('/' and '.', the Zarr v2 default), compressors null, zstd,
gzip and zlib, and a missing chunk reads as the array's fill_value.  Any other codec (blosc, ...) raises
NotImplementedError naming it.  3-D (z, y, x) arrays (what `downsample` reads and writes besides the 5-D ones) are
read and written by the same methods: their chunk index is the spatial part of (t, c, z, y, x).  ``read_multiscales``
turns an OME-NGFF 0.4 `multiscales` group into integer mipmap factors.  Host-side plumbing only.
"""
from __future__ import annotations

import gzip
import json
import os
import zlib

import numpy as np

from . import zstd as bzstd
from .n5 import bs_attrs, parse_fusion_metadata, BS_KEY

_ZDT = {"uint8": "|u1", "uint16": "<u2", "float32": "<f4"}


def _np_dtype(meta):
    """Native-order numpy dtype of an array's elements (the stored byte order is handled by the chunk codec)."""
    return np.dtype(meta["dtype"]).newbyteorder("=")


def _decode(meta, payload: bytes) -> bytes:
    comp = meta.get("compressor")
    if meta.get("filters"):
        raise NotImplementedError(f"Zarr filters {[f.get('id') for f in meta['filters']]}")
    if comp is None:
        return payload
    cid = comp.get("id")
    if cid == "zstd":
        return bzstd.decompress(payload)
    if cid == "gzip":
        return gzip.decompress(payload)
    if cid == "zlib":
        return zlib.decompress(payload)
    raise NotImplementedError(f"Zarr compressor {cid!r} (readable: null, zstd, gzip, zlib)")


class ZarrStore:
    def __init__(self, root: str, create: bool = False):
        self.root = root
        if create:
            os.makedirs(root, exist_ok=True)
            self._write_json("", ".zgroup", {"zarr_format": 2})
        elif not os.path.isdir(root):
            raise FileNotFoundError(root)

    def _write_json(self, group, name, obj):
        d = os.path.join(self.root, group.strip("/"))
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, name), "w") as f:
            json.dump(obj, f)

    def _read_json(self, group, name):
        p = os.path.join(self.root, group.strip("/"), name)
        if not os.path.exists(p):
            return {}
        with open(p) as f:
            return json.load(f)

    def get_attributes(self, group=""):
        return self._read_json(group, ".zattrs")

    def set_attributes(self, group, attrs: dict):
        cur = self.get_attributes(group)
        for k, v in attrs.items():
            if k == BS_KEY and isinstance(v, dict) and isinstance(cur.get(k), dict):
                cur[k].update(v)
            else:
                cur[k] = v
        self._write_json(group, ".zattrs", cur)

    def create_array(self, path, shape_tczyx, chunks_tczyx, dtype: str, compression="raw", level=None):
        if compression not in ("raw", "gzip", "zstd"):
            raise NotImplementedError(f"compression {compression} (not available in this image)")
        # numcodecs ids; zstd level 3 = the reference default (J/util/N5Util.java:91-92)
        comp = {"raw": None, "gzip": {"id": "gzip", "level": 1}, "zstd": {"id": "zstd", "level": 3}}[compression]
        if comp is not None and level is not None:
            comp["level"] = int(level)
        self._write_json(path, ".zarray", {"zarr_format": 2, "shape": [int(v) for v in shape_tczyx],
                                           "chunks": [int(v) for v in chunks_tczyx], "dtype": _ZDT[dtype],
                                           "compressor": comp, "fill_value": 0, "order": "C", "filters": None,
                                           "dimension_separator": "/"})

    def array_meta(self, path):
        m = self._read_json(path, ".zarray")
        if not m:
            raise KeyError(f"{path} is not a Zarr array")
        return m

    def create_array_like(self, path, like, shape):
        """An array of ``shape`` with the chunks, dtype, compressor, fill value, order, filters and dimension separator
        of the array ``like`` of this store.  Compressors other than null, zstd and gzip raise NotImplementedError."""
        m = dict(self.array_meta(like), shape=[int(v) for v in shape])
        cid = (m.get("compressor") or {}).get("id")
        if cid not in (None, "zstd", "gzip"):
            raise NotImplementedError(f"Zarr compressor {cid!r} (writable: null, zstd, gzip)")
        self._write_json(path, ".zarray", m)

    def _chunk_path(self, path, idx_tczyx, meta=None):
        m = meta or self.array_meta(path)
        sep = m.get("dimension_separator") or "."
        # a 3-D (z, y, x) array takes the spatial part of the (t, c, z, y, x) index
        key = sep.join(str(int(i)) for i in tuple(idx_tczyx)[-len(m["shape"]):])
        return os.path.join(self.root, path.strip("/"), *key.split("/"))

    def write_chunk(self, path, idx_tczyx, block_zyx: np.ndarray):
        """block_zyx: the valid [z,y,x] part of one chunk; padded to the full chunk shape.  A full chunk already in
        the array's byte order is written as it is."""
        m = self.array_meta(path)
        cz, cy, cx = m["chunks"][-3:]
        sdt = np.dtype(m["dtype"])
        if block_zyx.shape == (cz, cy, cx) and block_zyx.dtype == sdt and block_zyx.flags["C_CONTIGUOUS"]:
            payload = block_zyx.tobytes()
        else:
            full = np.zeros((cz, cy, cx), dtype=sdt)
            z, y, x = block_zyx.shape
            full[:z, :y, :x] = block_zyx
            payload = full.tobytes()
        if m["compressor"] is not None:
            if m["compressor"]["id"] == "zstd":
                payload = bzstd.compress(payload, m["compressor"].get("level", 3))
            else:
                payload = gzip.compress(payload, compresslevel=m["compressor"].get("level", 1))
        p = self._chunk_path(path, idx_tczyx, m)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(payload)

    def read_chunk(self, path, idx_tczyx):
        m = self.array_meta(path)
        if m.get("order", "C") != "C":
            raise NotImplementedError(f"Zarr order {m['order']!r} of {path}")
        p = self._chunk_path(path, idx_tczyx, m)
        cz, cy, cx = m["chunks"][-3:]
        dt = _np_dtype(m)
        if not os.path.exists(p):
            return np.full((cz, cy, cx), m.get("fill_value") or 0, dtype=dt)
        with open(p, "rb") as f:
            payload = _decode(m, f.read())
        return np.frombuffer(payload, dtype=np.dtype(m["dtype"]), count=cz * cy * cx).astype(dt).reshape(cz, cy, cx)

    def save_block(self, path, volume_zyx: np.ndarray, grid_offset_xyzct):
        """N5Utils.saveBlock on the 5-D view (J/SparkAffineFusion.java:630-643,670): split a
        [z,y,x] super-block into chunks starting at chunk index {gx,gy,gz} of channel c, timepoint t."""
        m = self.array_meta(path)
        gx, gy, gz, c, t = (int(v) for v in grid_offset_xyzct)
        sz, sy, sx = m["shape"][-3:]
        cz, cy, cx = m["chunks"][-3:]
        vz, vy, vx = volume_zyx.shape
        for kz in range(-(-vz // cz)):
            for ky in range(-(-vy // cy)):
                for kx in range(-(-vx // cx)):
                    iz, iy, ix = gz + kz, gy + ky, gx + kx
                    if iz * cz >= sz or iy * cy >= sy or ix * cx >= sx:
                        continue
                    blk = volume_zyx[kz * cz:(kz + 1) * cz, ky * cy:(ky + 1) * cy, kx * cx:(kx + 1) * cx]
                    blk = blk[:sz - iz * cz, :sy - iy * cy, :sx - ix * cx]
                    self.write_chunk(path, (t, c, iz, iy, ix), blk)

    def read_region(self, path, min_xyz, size_xyz, c=0, t=0):
        """[z, y, x] array of the interval [min, min + size) of channel c / timepoint t (zero outside the array)."""
        m = self.array_meta(path)
        sz, sy, sx = m["shape"][-3:]
        cz, cy, cx = m["chunks"][-3:]
        mn = [int(v) for v in min_xyz]
        n = [int(v) for v in size_xyz]
        out = np.zeros(n[::-1], dtype=_np_dtype(m))
        lo = [max(0, mn[d]) for d in range(3)]
        hi = [min((sx, sy, sz)[d], mn[d] + n[d]) for d in range(3)]
        if any(hi[d] <= lo[d] for d in range(3)):
            return out
        for iz in range(lo[2] // cz, -(-hi[2] // cz)):
            for iy in range(lo[1] // cy, -(-hi[1] // cy)):
                for ix in range(lo[0] // cx, -(-hi[0] // cx)):
                    ch = self.read_chunk(path, (t, c, iz, iy, ix))
                    b0 = (ix * cx, iy * cy, iz * cz)
                    s0 = [max(lo[d], b0[d]) for d in range(3)]
                    s1 = [min(hi[0], b0[0] + cx), min(hi[1], b0[1] + cy), min(hi[2], b0[2] + cz)]
                    out[s0[2] - mn[2]:s1[2] - mn[2], s0[1] - mn[1]:s1[1] - mn[1], s0[0] - mn[0]:s1[0] - mn[0]] = \
                        ch[s0[2] - b0[2]:s1[2] - b0[2], s0[1] - b0[1]:s1[1] - b0[1], s0[0] - b0[0]:s1[0] - b0[0]]
        return out

    def read_volume(self, path, c=0, t=0):
        m = self.array_meta(path)
        sz, sy, sx = m["shape"][-3:]
        cz, cy, cx = m["chunks"][-3:]
        out = np.zeros((sz, sy, sx), dtype=_np_dtype(m))
        for iz in range(-(-sz // cz)):
            for iy in range(-(-sy // cy)):
                for ix in range(-(-sx // cx)):
                    ch = self.read_chunk(path, (t, c, iz, iy, ix))
                    z0, y0, x0 = iz * cz, iy * cy, ix * cx
                    out[z0:z0 + cz, y0:y0 + cy, x0:x0 + cx] = ch[:sz - z0, :sy - y0, :sx - x0]
        return out


def mipmap_transform_default(abs_ds):
    """MipmapTransforms.getMipmapTransformDefault: scale f per axis and a half-pixel shift (f - 1) / 2
    (example at J/SparkInterestPointDetection.java:1073-1080)."""
    f = [float(v) for v in abs_ds]
    return [[f[0], 0, 0, (f[0] - 1) / 2], [0, f[1], 0, (f[1] - 1) / 2], [0, 0, f[2], (f[2] - 1) / 2]]


def read_multiscales(store: ZarrStore, group=""):
    """The levels of an OME-NGFF 0.4 multiscale group: [dict(path, factors (x, y, z) ints, dims (x, y, z))], level 0
    first.  A level's mipmap factors are its `scale` transformation divided by that of level 0, per spatial axis; they
    must be integers and the level's array must be floor or ceil of level 0's dims over them (ValueError otherwise)."""
    ms = store.get_attributes(group).get("multiscales")
    if not ms:
        raise KeyError(f"{os.path.join(store.root, group)} has no OME-NGFF multiscales attribute")
    ms = ms[0]
    names = [a["name"] if isinstance(a, dict) else str(a) for a in ms.get("axes", [])]
    ax = [names.index(n) for n in "xyz"] if all(n in names for n in "xyz") else [-1, -2, -3]
    levels = []
    for d in ms["datasets"]:
        scale = next((t["scale"] for t in d.get("coordinateTransformations", []) if t.get("type") == "scale"), None)
        path = (group.strip("/") + "/" + d["path"]).strip("/")
        shape = store.array_meta(path)["shape"]
        levels.append(dict(path=path, scale=[float(scale[a]) if scale else 1.0 for a in ax],
                           dims=tuple(int(shape[a]) for a in ax)))
    s0, d0 = levels[0]["scale"], levels[0]["dims"]
    for lv in levels:
        f = [lv["scale"][k] / s0[k] for k in range(3)]
        fi = [int(round(v)) for v in f]
        if any(abs(f[k] - fi[k]) > 1e-6 * max(1.0, f[k]) or fi[k] < 1 for k in range(3)):
            raise ValueError(f"{lv['path']}: mipmap factors {f} relative to level 0 are not integers")
        if any(lv["dims"][k] not in (d0[k] // fi[k], -(-d0[k] // fi[k])) for k in range(3)):
            raise ValueError(f"{lv['path']}: dims {lv['dims']} do not match level 0 dims {d0} over factors {fi}")
        lv["factors"] = tuple(fi)
        del lv["scale"]
    return levels


def create_multiscale_group(store: ZarrStore, group, dims_xyz, dtype, block_size, abs_factors, compression="zstd",
                            level=None):
    """One resaved view (J/SparkResaveN5.java:246-256, setupBdvDatasetsOMEZARR; layout recalled, PARITY_GAPS R3):
    the group holds one 5-D (1, 1, z, y, x) array per level, "0", "1", ..., chunks {1, 1, bz, by, bx}, dims
    floor(dims / factor), and `multiscales` v0.4 with scale = the absolute factors (pixel units) and the half-pixel
    translation (f - 1) / 2 of mipmap_transform_default."""
    datasets = []
    for lvl, f in enumerate(abs_factors):
        dims = [int(dims_xyz[d]) // int(f[d]) for d in range(3)]
        path = f"{group}/{lvl}"
        store.create_array(path, (1, 1, dims[2], dims[1], dims[0]), (1, 1, block_size[2], block_size[1], block_size[0]),
                           dtype, compression, level)
        mt = mipmap_transform_default(f)
        datasets.append({"path": str(lvl), "coordinateTransformations": [
            {"type": "scale", "scale": [1.0, 1.0, float(f[2]), float(f[1]), float(f[0])]},
            {"type": "translation", "translation": [0.0, 0.0, mt[2][3], mt[1][3], mt[0][3]]}]})
    store.set_attributes(group, {"multiscales": [{
        "version": "0.4", "name": group,
        "axes": [{"name": "t", "type": "time", "unit": "second"}, {"name": "c", "type": "channel"},
                 {"name": "z", "type": "space", "unit": "micrometer"}, {"name": "y", "type": "space", "unit": "micrometer"},
                 {"name": "x", "type": "space", "unit": "micrometer"}],
        "datasets": datasets}]})
    store._write_json(group, ".zgroup", {"zarr_format": 2})


def create_fusion_container_zarr(root, input_xml, bb_min, bb_max, block_size=(128, 128, 128), dtype="float32",
                                 min_intensity=None, max_intensity=None, num_timepoints=1, num_channels=1,
                                 anisotropy_factor=None, compression="raw", voxel_size=(1.0, 1.0, 1.0),
                                 downsamplings=(), output_xml=None):
    """`create-fusion-container -s ZARR` (J/CreateFusionContainer.java:331-389): one 5-D array per resolution level
    ("0", "1", ...: levelToName :346), the OME-NGFF v0.4 `multiscales` attribute with one scale + translation per
    level (:374-388) and the `Bigstitcher-Spark/*` root attributes.  ``downsamplings``: RELATIVE steps after s0
    (e.g. [(2,2,1), (2,2,2)]); the 5-D pyramid of N5ApiTools.setupMultiResolutionPyramid never downsamples c / t.
    With ``output_xml`` (`--bdv -xo`, :391-402) the arrays are the same; FusionFormat is "BDV/OME-ZARR" and
    OutputXML = ``output_xml``."""
    st = ZarrStore(root, create=True)
    dims = [int(bb_max[d] - bb_min[d] + 1) for d in range(3)]
    levels, datasets = [], []
    cur, absd = list(dims), [1, 1, 1]
    for lvl, rel in enumerate([(1, 1, 1)] + [tuple(int(v) for v in r) for r in downsamplings]):
        if lvl > 0:
            cur = [cur[d] // rel[d] for d in range(3)]
            absd = [absd[d] * rel[d] for d in range(3)]
        st.create_array(str(lvl), (num_timepoints, num_channels, cur[2], cur[1], cur[0]),
                        (1, 1, block_size[2], block_size[1], block_size[0]), dtype, compression)
        levels.append({"dataset": str(lvl), "dimensions": list(cur) + [num_channels, num_timepoints],
                       "blockSize": list(block_size) + [1, 1], "relativeDownsampling": list(rel) + [1, 1],
                       "absoluteDownsampling": list(absd) + [1, 1], "dataType": dtype})
        mt = mipmap_transform_default(absd)
        datasets.append({"path": str(lvl), "coordinateTransformations": [
            {"type": "scale", "scale": [1.0, 1.0, voxel_size[2] * absd[2], voxel_size[1] * absd[1], voxel_size[0] * absd[0]]},
            {"type": "translation", "translation": [0.0, 0.0, voxel_size[2] * mt[2][3], voxel_size[1] * mt[1][3],
                                                    voxel_size[0] * mt[0][3]]}]})
    multiscales = [{"version": "0.4", "name": "/",
                    "axes": [{"name": "t", "type": "time", "unit": "second"}, {"name": "c", "type": "channel"},
                             {"name": "z", "type": "space", "unit": "micrometer"},
                             {"name": "y", "type": "space", "unit": "micrometer"},
                             {"name": "x", "type": "space", "unit": "micrometer"}],
                    "datasets": datasets}]
    flat = {"FusionFormat": "BDV/OME-ZARR" if output_xml else "OME-ZARR", "InputXML": input_xml,
            "NumTimepoints": num_timepoints, "NumChannels": num_channels,
            "Boundingbox_min": [int(v) for v in bb_min], "Boundingbox_max": [int(v) for v in bb_max],
            "PreserveAnisotropy": anisotropy_factor is not None, "DataType": dtype.lower(),
            "BlockSize": list(block_size), "MultiResolutionInfos": [levels]}
    if anisotropy_factor is not None:
        flat["AnisotropyFactor"] = float(anisotropy_factor)
    if dtype != "float32":
        flat["MinIntensity"] = float(min_intensity)
        flat["MaxIntensity"] = float(max_intensity)
    if output_xml:
        flat["OutputXML"] = output_xml
    attrs = {"multiscales": multiscales}
    attrs.update(bs_attrs(flat))
    st.set_attributes("", attrs)
    return st


def read_fusion_container_zarr(root):
    st = ZarrStore(root)
    meta = parse_fusion_metadata(st.get_attributes(""))
    if meta["format"] not in ("OME-ZARR", "BDV/OME-ZARR"):
        raise KeyError("not a BigStitcher-Spark OME-ZARR fusion container")
    return st, meta
