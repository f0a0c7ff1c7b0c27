"""TIFF files assembled byte by byte (TIFF 6.0, and BigTIFF: 8-byte offsets, 20-byte IFD entries), independently of
the reader under test, and twin datasets: the same seeded views as a `bdv.n5` dataset and as TIFF files behind a
`spimreconstruction.filemap2` XML."""
import os
import struct
import zlib

import numpy as np

from bsgpu import n5 as bn5, spimdata

_FORMAT = {"uint8": (1, 8), "uint16": (1, 16), "float32": (3, 32), "int16": (2, 16), "uint32": (1, 32)}


def _encode(a, order, compression, predictor, level):
    a = np.ascontiguousarray(a)
    if predictor == 2:
        d = a.copy()
        d[:, 1:] = a[:, 1:] - a[:, :-1]                      # wraps in the sample type
        a = d
    b = a.astype(a.dtype.newbyteorder(order)).tobytes()
    if compression in (8, 32946):
        b = zlib.compress(b, level)
    elif compression == 5:
        b = b"\x80\x00" + b                                  # not decodable as LZW; the reader must refuse it first
    return b


def tiff_bytes(planes, order="<", big=False, description=None, compression=1, predictor=1, rows_per_strip=None,
               tile=None, samples_per_pixel=1, contiguous=False, level=6):
    """The bytes of a TIFF holding ``planes`` (2-D arrays of one dtype), one IFD per plane, in strips of
    ``rows_per_strip`` rows (default: one strip) or ``tile`` = (width, length) tiles, the edge tiles padded with zeros.
    ``description`` goes to the first IFD.  ``contiguous``: ImageJ's large-file form, ONE IFD describing the first plane
    and every other plane stored raw right after it."""
    o = order
    out = bytearray(b"II" if o == "<" else b"MM")
    out += struct.pack(o + "HHHQ", 43, 8, 0, 0) if big else struct.pack(o + "HI", 42, 0)
    link = 8 if big else 4                                   # where the offset of the next IFD goes
    off_type = 16 if big else 4
    dt = np.dtype(planes[0].dtype)
    fmt, bits = _FORMAT[dt.name]
    for i, p in enumerate(planes[:1] if contiguous else planes):
        h, w = p.shape
        if tile is not None:
            tw, tl = tile
            chunks = []
            for y in range(0, h, tl):
                for x in range(0, w, tw):
                    t = np.zeros((tl, tw), dtype=dt)
                    part = p[y:y + tl, x:x + tw]
                    t[:part.shape[0], :part.shape[1]] = part
                    chunks.append(t)
        else:
            rps = rows_per_strip or h
            chunks = [p[y:y + rps] for y in range(0, h, rps)]
        offs, cnts = [], []
        for c in chunks:
            if samples_per_pixel > 1:
                c = np.repeat(c, samples_per_pixel, axis=1)
            b = _encode(c, o, compression, predictor, level)
            offs.append(len(out))
            cnts.append(len(b))
            out += b
        if contiguous:
            for q in planes[1:]:
                out += _encode(q, o, 1, 1, level)
        entries = [(256, 4, [w]), (257, 4, [h]), (258, 3, [bits] * samples_per_pixel), (259, 3, [compression]),
                   (262, 3, [2 if samples_per_pixel == 3 else 1]), (277, 3, [samples_per_pixel]),
                   (339, 3, [fmt] * samples_per_pixel)]
        if predictor != 1:
            entries.append((317, 3, [predictor]))
        if i == 0 and description is not None:
            entries.append((270, 2, description.encode() + b"\0"))
        if tile is not None:
            entries += [(322, 3, [tile[0]]), (323, 3, [tile[1]]), (324, off_type, offs), (325, off_type, cnts)]
        else:
            entries += [(273, off_type, offs), (278, 4, [rows_per_strip or h]), (279, off_type, cnts)]
        entries.sort()
        inline = 8 if big else 4
        packed = []
        for tag, typ, vals in entries:                       # out-of-line values go before the IFD
            data = vals if typ == 2 else struct.pack(o + {3: "H", 4: "I", 16: "Q"}[typ] * len(vals), *vals)
            count = len(vals)
            if len(data) > inline:
                if len(out) % 2:
                    out += b"\0"
                pos = len(out)
                out += data
                data = struct.pack(o + ("Q" if big else "I"), pos)
            packed.append(struct.pack(o + "HH", tag, typ) + struct.pack(o + ("Q" if big else "I"), count) +
                          data.ljust(inline, b"\0"))
        if len(out) % 2:
            out += b"\0"
        out[link:link + (8 if big else 4)] = struct.pack(o + ("Q" if big else "I"), len(out))
        out += struct.pack(o + ("Q" if big else "H"), len(packed)) + b"".join(packed)
        link = len(out)
        out += bytes(8 if big else 4)
    return bytes(out)


def write_tiff(path, planes, **kw):
    with open(path, "wb") as f:
        f.write(tiff_bytes(planes, **kw))
    return str(path)


def imagej_description(channels, slices, frames):
    return (f"ImageJ=1.54f\nimages={channels * slices * frames}\nchannels={channels}\nslices={slices}\n"
            f"frames={frames}\nhyperstack=true\nmode=grayscale\n")


def twin_datasets(root, vols, translations, block_size=(64, 64, 32), **tiff_kw):
    """``vols`` {setup: [z, y, x] array} as `root/n5/dataset.xml` (bdv.n5, raw blocks) and as `root/tif/dataset.xml`
    (one TIFF per view under root/tif/raw, written with ``tiff_kw``, filemap2 loader).  Returns (n5 xml, tiff xml)."""
    os.makedirs(os.path.join(root, "n5"))
    os.makedirs(os.path.join(root, "tif", "raw"))
    store = bn5.N5Store(os.path.join(root, "n5", "dataset.n5"), create=True)
    tiles, mappings = [], {}
    for s, vol in sorted(vols.items()):
        bn5.write_bdv_setup(store, s, 0, vol, block_size)
        tiles.append(dict(setup=s, size_xyz=vol.shape[::-1], tile=s, translation_xyz=translations[s]))
        mappings[(0, s)] = (write_tiff(os.path.join(root, "tif", "raw", f"tile{s}.tif"), list(vol), **tiff_kw), 0, 0)
    xn = spimdata.write_dataset_xml(os.path.join(root, "n5", "dataset.xml"), "dataset.n5", tiles)
    xt = spimdata.write_dataset_xml(os.path.join(root, "tif", "dataset.xml"), "unused", tiles)
    d = spimdata.SpimData2.load(xt)
    d.set_file_map_loader(mappings)
    d.save(xt, backup=False)
    return xn, xt
