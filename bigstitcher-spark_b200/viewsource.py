"""The image data of a SpimData2 dataset, whichever container holds it: volume and region reads and the mipmap
levels of every view.  Three loaders are read (Import / the BDV image loaders the reference opens through the XML):

  * `bdv.n5` -- BDV-N5: `setup{s}/timepoint{t}/s{l}` 3-D datasets, mipmap factors from the setup's
    `downsamplingFactors` attribute;
  * `bdv.multimg.zarr` -- AllenOMEZarrLoader (J/SparkResaveN5.java:434-445): one OME-NGFF multiscale group per view,
    levels "0", "1", ... of 5-D (t, c, z, y, x) arrays read at the view's (channel, timepoint) indices, mipmap factors
    from the levels' `scale` transformations (zarr.read_multiscales);
  * `spimreconstruction.filemap2` -- TIFF stacks as BigStitcher's automatic loader defines them: per view a file,
    a series and a channel (SpimData2.file_mappings), read by tiff.py, one level (TiffViews).

Mipmap transforms follow the half-pixel convention of MipmapTransforms.getMipmapTransformDefault for both
(zarr.mipmap_transform_default).  A `split.viewerimgloader` (split-images) wraps an N5 or OME-ZARR one: its views are
boxes of the wrapped views (SplitViews).  Any other loader raises NotImplementedError.  ``roots`` of every view source
lists the containers or files it reads.  Host-side plumbing only.
"""
from __future__ import annotations

import numpy as np

from . import n5 as bn5
from . import tiff as btiff
from . import zarr as bzarr
from .spimdata import FILEMAP_LOADER, SPLIT_LOADER


def open_views(data):
    """The view source of a loaded SpimData2."""
    fmt, path = data.image_loader()
    if fmt == "bdv.n5":
        return N5Views(path)
    if fmt == "bdv.multimg.zarr":
        return ZarrViews(path, data.zarr_groups())
    if fmt == FILEMAP_LOADER:
        return TiffViews(data.file_mappings())
    if fmt == SPLIT_LOADER:
        fmt, path = data.image_loader(nested=True)
        if fmt == "bdv.n5":
            return SplitViews(N5Views(path), data.split_setups())
        if fmt == "bdv.multimg.zarr":
            return SplitViews(ZarrViews(path, data.zarr_groups(nested=True)), data.split_setups())
    raise NotImplementedError(f"ImageLoader format {fmt}")


class N5Views:
    format = "bdv.n5"

    def __init__(self, root):
        self.store = bn5.N5Store(root)
        self.roots = [root]

    def mipmap_info(self, view):
        """(factors [(fx, fy, fz)] per level, mipmap transforms 3 x 4 per level) of a view."""
        a = self.store.get_attributes(f"setup{view[1]}")
        factors = [tuple(int(v) for v in f) for f in a.get("downsamplingFactors", [[1, 1, 1]])]
        return factors, [bzarr.mipmap_transform_default(f) for f in factors]

    def _attrs(self, view, level):
        return self.store.dataset_attributes(bn5.bdv_dataset(view[1], view[0], level))

    def level_dims(self, view, level):
        return tuple(int(d) for d in self._attrs(view, level)["dimensions"])

    def level_dtype(self, view, level) -> str:
        return self._attrs(view, level)["dataType"]

    def read_volume(self, view, level=0):
        return self.store.read_volume(bn5.bdv_dataset(view[1], view[0], level))

    def read_region(self, view, level, min_xyz, size_xyz):
        return self.store.read_region(bn5.bdv_dataset(view[1], view[0], level), min_xyz, size_xyz)


class ZarrViews:
    format = "bdv.multimg.zarr"

    def __init__(self, root, groups):
        self.store = bzarr.ZarrStore(root)
        self.roots = [root]
        self.groups = groups                     # {(tp, setup): (group path, channel index, timepoint index)}
        self._levels = {}

    def _view(self, view):
        key = (int(view[0]), int(view[1]))
        if key not in self.groups:
            raise KeyError(f"view {key} has no <zgroup> in the ImageLoader of {self.store.root}")
        if key not in self._levels:
            self._levels[key] = bzarr.read_multiscales(self.store, self.groups[key][0])
        return self.groups[key], self._levels[key]

    def mipmap_info(self, view):
        _, levels = self._view(view)
        factors = [lv["factors"] for lv in levels]
        return factors, [bzarr.mipmap_transform_default(f) for f in factors]

    def level_dims(self, view, level):
        return self._view(view)[1][level]["dims"]

    def level_dtype(self, view, level) -> str:
        _, levels = self._view(view)
        return bzarr._np_dtype(self.store.array_meta(levels[level]["path"])).name

    def read_volume(self, view, level=0):
        (_, c, t), levels = self._view(view)
        return self.store.read_volume(levels[level]["path"], c, t)

    def read_region(self, view, level, min_xyz, size_xyz):
        (_, c, t), levels = self._view(view)
        return self.store.read_region(levels[level]["path"], min_xyz, size_xyz, c, t)


class TiffViews:
    """TIFF stacks (`spimreconstruction.filemap2`): view (tp, setup) is channel ``channel`` of series ``series`` of its
    file, at frame tp when the series has more than one frame and at frame 0 for every timepoint when it has one
    (PARITY_GAPS T2).  One level, full resolution.  Files are opened on first use and kept open."""
    format = FILEMAP_LOADER

    def __init__(self, mappings):
        self.mappings = mappings                 # {(tp, setup): (file path, series, channel)}
        self.roots = sorted({m[0] for m in mappings.values()})
        self._files = {}

    def _view(self, view):
        """(Series, channel, frame) of a view."""
        key = (int(view[0]), int(view[1]))
        if key not in self.mappings:
            raise KeyError(f"view {key} has no <FileMapping> in the ImageLoader")
        path, series, channel = self.mappings[key]
        if path not in self._files:
            self._files[path] = btiff.TiffFile(path)
        all_series = self._files[path].series()
        if series >= len(all_series):
            raise ValueError(f"view {key}: {path} has {len(all_series)} series, not series {series}")
        s = all_series[series]
        frame = key[0] if s.frames > 1 else 0
        if channel >= s.channels or frame >= s.frames:
            raise ValueError(f"view {key}: series {series} of {path} has {s.channels} channels and {s.frames} frames; "
                             f"channel {channel}, frame {frame} asked")
        return s, channel, frame

    def mipmap_info(self, view):
        return [(1, 1, 1)], [bzarr.mipmap_transform_default((1, 1, 1))]

    def _level0(self, view, level):
        if int(level) != 0:
            raise ValueError(f"view {tuple(view)}: a TIFF view has only level 0, not level {level}")
        return self._view(view)

    def level_dims(self, view, level):
        return self._level0(view, level)[0].dims

    def level_dtype(self, view, level) -> str:
        return self._level0(view, level)[0].dtype.name

    def read_volume(self, view, level=0):
        s, c, t = self._level0(view, level)
        return s.read_volume(c, t)

    def read_region(self, view, level, min_xyz, size_xyz):
        s, c, t = self._level0(view, level)
        return s.read_region(min_xyz, size_xyz, c, t)


class SplitViews:
    """The sub-views split-images defines (`split.viewerimgloader`): view (tp, new setup) is the box [min, max] of view
    (tp, old setup) of the wrapped N5Views / ZarrViews.  Level l with factors f is the parent's level-l window from
    min / f to min(floor(max / f), parent dims - 1); min is a multiple of every factor, so the parent's half-pixel
    mipmap transforms stay exact.  Voxels outside the window read as zero, like those outside a dataset."""
    format = SPLIT_LOADER

    def __init__(self, inner, definitions):
        self.inner = inner
        self.store = inner.store
        self.roots = inner.roots
        self.definitions = definitions           # {new setup: (old setup, min xyz, max xyz)}

    def _parent(self, view):
        old, _, _ = self.definitions[int(view[1])]
        return (int(view[0]), old)

    def _window(self, view, level):
        """(parent view, window min, window size) of a level."""
        old, mn, mx = self.definitions[int(view[1])]
        parent = (int(view[0]), old)
        f = self.inner.mipmap_info(parent)[0][level]
        pdims = self.inner.level_dims(parent, level)
        lo = [int(mn[d]) // int(f[d]) for d in range(3)]
        hi = [min(int(mx[d]) // int(f[d]), int(pdims[d]) - 1) for d in range(3)]
        return parent, lo, [hi[d] - lo[d] + 1 for d in range(3)]

    def mipmap_info(self, view):
        return self.inner.mipmap_info(self._parent(view))

    def level_dims(self, view, level):
        return tuple(self._window(view, level)[2])

    def level_dtype(self, view, level) -> str:
        return self.inner.level_dtype(self._parent(view), level)

    def read_volume(self, view, level=0):
        parent, lo, size = self._window(view, level)
        return self.inner.read_region(parent, level, lo, size)

    def read_region(self, view, level, min_xyz, size_xyz):
        parent, lo, dims = self._window(view, level)
        mn = [int(v) for v in min_xyz]
        sz = [int(v) for v in size_xyz]
        a = [max(mn[d], 0) for d in range(3)]                       # the part inside the sub-view
        b = [min(mn[d] + sz[d], dims[d]) for d in range(3)]
        if any(b[d] <= a[d] for d in range(3)):
            return np.zeros(sz[::-1], dtype=self.level_dtype(view, level))
        part = self.inner.read_region(parent, level, [lo[d] + a[d] for d in range(3)], [b[d] - a[d] for d in range(3)])
        if a == mn and b == [mn[d] + sz[d] for d in range(3)]:
            return part
        out = np.zeros(sz[::-1], dtype=part.dtype)
        out[a[2] - mn[2]:b[2] - mn[2], a[1] - mn[1]:b[1] - mn[1], a[0] - mn[0]:b[0] - mn[0]] = part
        return out
