"""TIFF stacks as the views of a `spimreconstruction.filemap2` dataset (the BigStitcher automatic loader's XML).
Host only: numpy and zlib.

Read: classic TIFF and BigTIFF in either byte order, strips or tiles, one sample per pixel, uint8 / uint16 / float32,
compression none (1), Deflate (8, 32946) and PackBits (32773), horizontal differencing (Predictor 2, wrapping in the
sample type) on the integer types.  Three layouts give the (c, z, t) planes of a file's series:

  * plain multi-page TIFF: one series, every page one z-plane, one channel, one frame;
  * ImageJ hyperstack (`ImageDescription` starting "ImageJ="): `images=`, `channels=`, `slices=`, `frames=`, pages
    in czt order, channel fastest; a single IFD with `images` > 1 is ImageJ's large-file form, every plane stored
    uncompressed right after the one before, from the first plane's strip offset;
  * single-file OME-TIFF (OME-XML in the first `ImageDescription`): series i is `<Image>` i, its planes placed by
    `<TiffData IFD= FirstZ= FirstC= FirstT= PlaneCount=>` in the `DimensionOrder` of its `<Pixels>`, or, without
    `<TiffData>`, the IFDs that follow the planes of the series before it.

Write: ``write_float32_stack``, an uncompressed float32 stack with an ImageJ description (the PSFs of extract-psfs).

Anything else raises NotImplementedError naming the file and what it has (PARITY_GAPS T4).  Regions read only the
pages, and the strips or tiles of those pages, that they touch; uncompressed rows are read straight into the output
buffer, one read per run of adjacent rows.
"""
from __future__ import annotations

import os
import re
import struct
import xml.etree.ElementTree as ET
import zlib

import numpy as np

# tags
_DESCRIPTION, _WIDTH, _LENGTH, _BITS, _COMPRESSION, _PHOTOMETRIC = 270, 256, 257, 258, 259, 262
_STRIP_OFFSETS, _SAMPLES, _ROWS_PER_STRIP, _STRIP_COUNTS, _PREDICTOR = 273, 277, 278, 279, 317
_TILE_WIDTH, _TILE_LENGTH, _TILE_OFFSETS, _TILE_COUNTS, _SAMPLE_FORMAT = 322, 323, 324, 325, 339

# field type -> (struct code, size); RATIONALs are kept as raw pairs
_TYPES = {1: ("B", 1), 2: ("s", 1), 3: ("H", 2), 4: ("I", 4), 5: ("I", 4), 6: ("b", 1), 7: ("B", 1), 8: ("h", 2),
          9: ("i", 4), 10: ("i", 4), 11: ("f", 4), 12: ("d", 8), 13: ("I", 4), 16: ("Q", 8), 17: ("q", 8), 18: ("Q", 8)}

_COMPRESSIONS = {1: "none", 8: "Deflate", 32946: "Deflate", 32773: "PackBits"}
_COMPRESSION_NAMES = {2: "CCITT RLE", 3: "CCITT G3", 4: "CCITT G4", 5: "LZW", 6: "old-style JPEG", 7: "JPEG",
                      34712: "JPEG 2000", 50000: "Zstandard", 34925: "LZMA"}
_DTYPES = {(1, 8): "uint8", (1, 16): "uint16", (3, 32): "float32"}
_SAMPLE_FORMAT_NAMES = {1: "uint", 2: "int", 3: "float"}


class Page:
    """One IFD: the plane's geometry, sample type and where its strips or tiles are."""

    def __init__(self, path, tags, order):
        self.path = path
        self.description = tags.get(_DESCRIPTION, b"")
        self.width, self.height = int(tags[_WIDTH][0]), int(tags[_LENGTH][0])
        spp = int(tags.get(_SAMPLES, (1,))[0])
        if spp != 1:
            photometric = int(tags.get(_PHOTOMETRIC, (1,))[0])
            raise NotImplementedError(f"{path}: {spp} samples per pixel" + (" (RGB)" if photometric == 2 else "") +
                                      "; only single-sample (grayscale) planes are read")
        fmt = int(tags.get(_SAMPLE_FORMAT, (1,))[0])
        bits = int(tags.get(_BITS, (1,))[0])
        name = _DTYPES.get((fmt, bits))
        if name is None:
            raise NotImplementedError(f"{path}: sample type {_SAMPLE_FORMAT_NAMES.get(fmt, fmt)}{bits} "
                                      "(readable: uint8, uint16, float32)")
        self.dtype = np.dtype(name).newbyteorder(order)
        self.compression = int(tags.get(_COMPRESSION, (1,))[0])
        if self.compression not in _COMPRESSIONS:
            raise NotImplementedError(f"{path}: compression {_COMPRESSION_NAMES.get(self.compression, self.compression)}"
                                      " (readable: none, Deflate, PackBits)")
        self.predictor = int(tags.get(_PREDICTOR, (1,))[0])
        if self.predictor == 2 and name == "float32":
            raise NotImplementedError(f"{path}: Predictor 2 (horizontal differencing) on float32 samples")
        if self.predictor not in (1, 2):
            raise NotImplementedError(f"{path}: Predictor {self.predictor}")
        if _TILE_OFFSETS in tags:
            self.tile = (int(tags[_TILE_WIDTH][0]), int(tags[_TILE_LENGTH][0]))          # (width, length)
            self.offsets, self.counts = tags[_TILE_OFFSETS], tags[_TILE_COUNTS]
        else:
            self.tile = None
            self.rows_per_strip = min(int(tags.get(_ROWS_PER_STRIP, (self.height,))[0]), self.height)
            self.offsets, self.counts = tags[_STRIP_OFFSETS], tags[_STRIP_COUNTS]
        self.offsets = np.asarray(self.offsets, dtype=np.int64)
        self.counts = np.asarray(self.counts, dtype=np.int64)

    def describe(self):
        return (self.width, self.height, self.dtype.name)


class TiffFile:
    """The IFD chain of one TIFF file.  ``fh``: an open binary file object to read through (default: the file)."""

    def __init__(self, path, fh=None):
        self.path = path
        if fh is None and not os.path.isfile(path):
            raise FileNotFoundError(f"TIFF file {path} not found")
        self.fh = fh if fh is not None else open(path, "rb")
        head = self._read(0, 16)
        if head[:2] not in (b"II", b"MM"):
            raise ValueError(f"{path} is not a TIFF file")
        self.order = "<" if head[:2] == b"II" else ">"
        magic = struct.unpack(self.order + "H", head[2:4])[0]
        if magic == 42:
            self.big, first = False, struct.unpack(self.order + "I", head[4:8])[0]
        elif magic == 43:
            self.big, first = True, struct.unpack(self.order + "Q", head[8:16])[0]
        else:
            raise ValueError(f"{path}: TIFF version {magic}")
        self.pages, seen = [], set()
        while first and first not in seen:
            seen.add(first)
            tags, first = self._ifd(first)
            self.pages.append(Page(path, tags, self.order))
        if not self.pages:
            raise ValueError(f"{path}: no image file directory")
        self._series = None

    def close(self):
        self.fh.close()

    def _read(self, offset, n):
        self.fh.seek(offset)
        return self.fh.read(n)

    def _ifd(self, offset):
        """({tag: values}, next IFD offset) of the IFD at ``offset``; ASCII values are bytes."""
        o = self.order
        cnt_fmt, ent, off_fmt = ("Q", 20, "Q") if self.big else ("H", 12, "I")
        csz = struct.calcsize(cnt_fmt)
        n = struct.unpack(o + cnt_fmt, self._read(offset, csz))[0]
        raw = self._read(offset + csz, n * ent + struct.calcsize(off_fmt))
        tags = {}
        inline = 8 if self.big else 4
        for i in range(n):
            e = raw[i * ent:(i + 1) * ent]
            tag, typ = struct.unpack(o + "HH", e[:4])
            count = struct.unpack(o + cnt_fmt.replace("H", "I"), e[4:4 + (8 if self.big else 4)])[0]
            if typ not in _TYPES:
                continue
            code, size = _TYPES[typ]
            nbytes = count * size * (2 if typ in (5, 10) else 1)
            val = e[-inline:]
            data = val[:nbytes] if nbytes <= inline else self._read(struct.unpack(o + off_fmt, val)[0], nbytes)
            if typ == 2:
                tags[tag] = data.split(b"\0", 1)[0]
            else:
                tags[tag] = np.frombuffer(data, dtype=np.dtype(o + code)).tolist() if count > 4 else \
                    struct.unpack(o + code * (count * (2 if typ in (5, 10) else 1)), data)
        nxt = struct.unpack(o + off_fmt, raw[n * ent:])[0]
        return tags, nxt

    # ------------------------------------------------------------------ layouts
    def series(self):
        """The series of the file, [Series], by its layout."""
        if self._series is None:
            desc = self.pages[0].description
            if desc.startswith(b"ImageJ="):
                self._series = [self._imagej(desc.decode("latin-1"))]
            elif b"<OME" in desc[:4096]:
                self._series = self._ome(desc.decode("utf-8"))
            else:
                self._series = [Series(self, {(0, z, 0): (z, 0) for z in range(len(self.pages))}, 1, len(self.pages), 1)]
        return self._series

    def _imagej(self, desc):
        kv = dict(m.groups() for m in re.finditer(r"^(\w+)=(.*)$", desc, re.M))
        c, z, t = (int(kv.get(k, 1)) for k in ("channels", "slices", "frames"))
        images = int(kv.get("images", c * z * t))
        if "slices" not in kv and c * t and images % (c * t) == 0:
            z = images // (c * t)
        if images != c * z * t:
            raise ValueError(f"{self.path}: ImageJ images={images} is not channels x slices x frames = {c * z * t}")
        if len(self.pages) == 1 and images > 1:
            p = self.pages[0]
            if p.compression != 1:
                raise NotImplementedError(f"{self.path}: ImageJ single-IFD planes with compression "
                                          f"{_COMPRESSIONS[p.compression]}")
            plane = p.width * p.height * p.dtype.itemsize
            planes = {(ci, zi, ti): (0, ((ti * z + zi) * c + ci) * plane)
                      for ti in range(t) for zi in range(z) for ci in range(c)}
        else:
            if len(self.pages) < images:
                raise ValueError(f"{self.path}: ImageJ images={images} but {len(self.pages)} pages")
            planes = {(ci, zi, ti): ((ti * z + zi) * c + ci, 0)
                      for ti in range(t) for zi in range(z) for ci in range(c)}
        return Series(self, planes, c, z, t)

    def _ome(self, desc):
        root = ET.fromstring(desc)
        out, next_ifd = [], 0
        name = os.path.basename(self.path)
        for image in root.findall("{*}Image"):
            px = image.find("{*}Pixels")
            order = px.get("DimensionOrder", "XYZCT")
            size = {k: int(px.get("Size" + k, 1)) for k in "ZCT"}
            axes = order[2:]                                       # fastest first, e.g. "CZT"
            if sorted(axes) != ["C", "T", "Z"]:
                raise ValueError(f"{self.path}: DimensionOrder {order}")

            def coords(k):                                         # plane index -> (c, z, t) in DimensionOrder
                v = {}
                for a in axes:
                    v[a] = k % size[a]
                    k //= size[a]
                return (v["C"], v["Z"], v["T"])

            def index(c, z, t):
                v, k, m = dict(C=c, Z=z, T=t), 0, 1
                for a in axes:
                    k += v[a] * m
                    m *= size[a]
                return k

            total = size["Z"] * size["C"] * size["T"]
            tds = px.findall("{*}TiffData")
            planes = {}
            if not tds:
                for k in range(total):
                    planes[coords(k)] = (next_ifd + k, 0)
                next_ifd += total
            for td in tds:
                uuid = td.find("{*}UUID")
                if uuid is not None and uuid.get("FileName") not in (None, name):
                    raise NotImplementedError(f"{self.path}: multi-file OME-TIFF (planes in {uuid.get('FileName')})")
                ifd = int(td.get("IFD", 0))
                count = int(td.get("PlaneCount", 1 if "IFD" in td.attrib else total))
                first = index(int(td.get("FirstC", 0)), int(td.get("FirstZ", 0)), int(td.get("FirstT", 0)))
                for j in range(count):
                    planes[coords(first + j)] = (ifd + j, 0)
            if len(planes) != total or max(p[0] for p in planes.values()) >= len(self.pages):
                raise ValueError(f"{self.path}: OME series {len(out)} places {len(planes)} of {total} planes "
                                 f"in {len(self.pages)} IFDs")
            next_ifd = max(p[0] for p in planes.values()) + 1
            out.append(Series(self, planes, size["C"], size["Z"], size["T"]))
        if not out:
            raise ValueError(f"{self.path}: OME-XML without <Image>")
        return out


class Series:
    """One series: planes {(c, z, t): (page index, byte shift of the page's strips)}, all of one geometry."""

    def __init__(self, tf, planes, channels, slices, frames):
        self.file, self.planes = tf, planes
        self.channels, self.slices, self.frames = channels, slices, frames
        pages = {tf.pages[i].describe() for i, _ in planes.values()}
        if len(pages) != 1:
            raise ValueError(f"{tf.path}: the planes of one series differ in size or type: {sorted(pages)}")
        self.width, self.height, dt = pages.pop()
        self.dtype = np.dtype(dt)
        self.dims = (self.width, self.height, self.slices)      # x, y, z

    def read_volume(self, c=0, t=0):
        return self.read_region((0, 0, 0), self.dims, c, t)

    def read_region(self, min_xyz, size_xyz, c=0, t=0):
        """[z, y, x] array of [min, min + size) of channel ``c``, frame ``t``; voxels outside the series are zero."""
        mn = [int(v) for v in min_xyz]
        sz = [int(v) for v in size_xyz]
        out = np.zeros(sz[::-1], dtype=self.dtype)
        lo = [max(0, mn[d]) for d in range(3)]
        hi = [min(self.dims[d], mn[d] + sz[d]) for d in range(3)]
        if any(hi[d] <= lo[d] for d in range(3)):
            return out
        for z in range(lo[2], hi[2]):
            page, shift = self.planes[(c, z, t)]
            dst = out[z - mn[2], lo[1] - mn[1]:hi[1] - mn[1], lo[0] - mn[0]:hi[0] - mn[0]]
            _read_plane(self.file, self.file.pages[page], shift, lo[1], hi[1], lo[0], hi[0], dst)
        return out


# ---------------------------------------------------------------------------------------------- decoding
def _packbits(data, n):
    out = bytearray()
    i, m = 0, len(data)
    while i < m and len(out) < n:
        h = data[i]
        if h < 128:
            out += data[i + 1:i + 2 + h]
            i += 2 + h
        elif h > 128:
            out += data[i + 1:i + 2] * (257 - h)
            i += 2
        else:
            i += 1
    return bytes(out)


def _decode(tf, page, offset, count, rows, width):
    """The (rows, width) native-order samples of one compressed strip or tile."""
    raw = tf._read(int(offset), int(count))
    n = rows * width * page.dtype.itemsize
    if page.compression == 32773:
        raw = _packbits(raw, n)
    elif page.compression != 1:
        raw = zlib.decompress(raw)
    if len(raw) < n:
        raise ValueError(f"{tf.path}: a strip or tile holds {len(raw)} bytes, {n} expected")
    a = np.frombuffer(raw, dtype=page.dtype, count=rows * width).reshape(rows, width).astype(page.dtype.newbyteorder("="))
    if page.predictor == 2:
        a = np.cumsum(a, axis=1, dtype=a.dtype)
    return a


def _read_plane(tf, page, shift, y0, y1, x0, x1, dst):
    """Rows [y0, y1) and columns [x0, x1) of a page into ``dst``, touching only the strips or tiles they lie in."""
    w, isz = page.width, page.dtype.itemsize
    if page.tile is not None:
        tw, tl = page.tile
        across = -(-w // tw)
        for ty in range(y0 // tl, -(-y1 // tl)):
            for tx in range(x0 // tw, -(-x1 // tw)):
                k = ty * across + tx
                t = _decode(tf, page, page.offsets[k] + shift, page.counts[k], tl, tw)
                a0, a1 = max(y0, ty * tl), min(y1, (ty + 1) * tl)
                b0, b1 = max(x0, tx * tw), min(x1, (tx + 1) * tw)
                dst[a0 - y0:a1 - y0, b0 - x0:b1 - x0] = t[a0 - ty * tl:a1 - ty * tl, b0 - tx * tw:b1 - tx * tw]
        return
    rps = page.rows_per_strip
    if page.compression == 1 and page.predictor == 1:
        # uncompressed: row r of strip k lies at offsets[k] + (r - k rps) w isz; each run of adjacent rows is one read
        # straight into the buffer
        row = w * isz
        r = np.arange(y0, y1)
        starts = page.offsets[r // rps] + shift + (r % rps) * row
        cuts = np.concatenate([[0], np.nonzero(np.diff(starts) != row)[0] + 1, [len(r)]])
        rows = np.empty((y1 - y0, w), dtype=page.dtype)
        buf = memoryview(rows.reshape(-1).view(np.uint8))
        for a, b in zip(cuts[:-1].tolist(), cuts[1:].tolist()):
            tf.fh.seek(int(starts[a]))
            if tf.fh.readinto(buf[a * row:b * row]) != (b - a) * row:
                raise ValueError(f"{tf.path}: truncated strip at byte {int(starts[a])}")
        dst[...] = rows[:, x0:x1]
        return
    for k in range(y0 // rps, -(-y1 // rps)):
        n = min(rps, page.height - k * rps)
        s = _decode(tf, page, page.offsets[k] + shift, page.counts[k], n, w)
        a0, a1 = max(y0, k * rps), min(y1, k * rps + n)
        dst[a0 - y0:a1 - y0] = s[a0 - k * rps:a1 - k * rps, x0:x1]


def write_float32_stack(path, vol):
    """Write ``vol`` [z, y, x] as an uncompressed little-endian float32 TIFF: one page per z-plane, one strip per page,
    and the ImageJ description `images=z slices=z` in the first page, so ImageJ / Fiji open it as a z-stack."""
    vol = np.ascontiguousarray(vol, dtype="<f4")
    if vol.ndim != 3 or 0 in vol.shape:
        raise ValueError(f"write_float32_stack: a non-empty [z, y, x] volume, not shape {vol.shape}")
    nz, h, w = vol.shape
    desc = f"ImageJ=1.11a\nimages={nz}\nslices={nz}\nloop=false\n".encode("ascii") + b"\0"
    plane = h * w * 4
    data_at = 8 + len(desc) + len(desc) % 2            # word-aligned pixel data, so every IFD is word-aligned too
    ifd_at = data_at + nz * plane
    out = bytearray(struct.pack("<2sHI", b"II", 42, ifd_at))
    out += desc + b"\0" * (len(desc) % 2)
    out += vol.tobytes()
    for z in range(nz):
        entries = [(_WIDTH, 4, 1, w), (_LENGTH, 4, 1, h), (_BITS, 3, 1, 32), (_COMPRESSION, 3, 1, 1),
                   (_PHOTOMETRIC, 3, 1, 1)]
        if z == 0:
            entries.append((_DESCRIPTION, 2, len(desc), 8))
        entries += [(_STRIP_OFFSETS, 4, 1, data_at + z * plane), (_SAMPLES, 3, 1, 1), (_ROWS_PER_STRIP, 4, 1, h),
                    (_STRIP_COUNTS, 4, 1, plane), (_SAMPLE_FORMAT, 3, 1, 3)]
        here = len(out)
        nxt = here + 2 + 12 * len(entries) + 4 if z + 1 < nz else 0
        out += struct.pack("<H", len(entries))
        for tag, typ, count, value in entries:
            inline = struct.pack("<HH", value, 0) if typ == 3 else struct.pack("<I", value)   # SHORTs left-justified
            out += struct.pack("<HHI", tag, typ, count) + inline
        out += struct.pack("<I", nxt)
    with open(path, "wb") as f:
        f.write(bytes(out))
