"""The image data of a SpimData2 dataset, whichever container holds it: volume and region reads and the mipmap
levels of every view.  Two loaders are read (Import / the BDV image loaders the reference opens through the XML):

  * `bdv.n5` -- BDV-N5: `setup{s}/timepoint{t}/s{l}` 3-D datasets, mipmap factors from the setup's
    `downsamplingFactors` attribute;
  * `bdv.multimg.zarr` -- AllenOMEZarrLoader (J/SparkResaveN5.java:434-445): one OME-NGFF multiscale group per view,
    levels "0", "1", ... of 5-D (t, c, z, y, x) arrays read at the view's (channel, timepoint) indices, mipmap factors
    from the levels' `scale` transformations (zarr.read_multiscales).

Mipmap transforms follow the half-pixel convention of MipmapTransforms.getMipmapTransformDefault for both
(zarr.mipmap_transform_default).  Any other loader raises NotImplementedError.  Host-side plumbing only.
"""
from __future__ import annotations

from . import n5 as bn5
from . import zarr as bzarr


def open_views(data):
    """The view source of a loaded SpimData2."""
    fmt, path = data.image_loader()
    if fmt == "bdv.n5":
        return N5Views(path)
    if fmt == "bdv.multimg.zarr":
        return ZarrViews(path, data.zarr_groups())
    raise NotImplementedError(f"ImageLoader format {fmt}")


class N5Views:
    format = "bdv.n5"

    def __init__(self, root):
        self.store = bn5.N5Store(root)

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
