"""Minimal SpimData2 XML reader / writer (SURVEY.md 8f-2, Appendix B; spim_data 2.3.5 + mvrecon
extensions) -- the fields the two hot paths consume and produce:

  * ViewSetups: id, size, attributes (illumination / channel / tile / angle)   (J/util/ViewUtil.java:107-109,
    grouping at J/SparkPairwiseStitching.java:147-160)
  * ViewRegistrations: ordered <ViewTransform type="affine"> lists; list index 0 is applied LAST
    (J/ClearRegistrations.java:80-99), so model = T0 * T1 * ... * Tn
  * ImageLoader format="bdv.n5" path (J/SparkResaveN5.java:424-433), or format="bdv.multimg.zarr" (AllenOMEZarrLoader,
    :434-445): the container root plus one <zgroup> per view with its group path and (channel, timepoint) indices,
    or format="split.viewerimgloader" (split-images): one of those loaders plus the box of an old setup per new setup,
    or format="spimreconstruction.filemap2" (TIFF stacks): one <FileMapping> of a file, series and channel per view
  * <MissingViews> and the <Attributes> entries of <ViewSetups> (tile names and locations, illuminations)
  * <StitchingResults><PairwiseResult view_setup_a/b tp_a/b> shift (12 doubles), correlation, hash,
    overlap_boundingbox (6 doubles)                                   (J/SparkPairwiseStitching.java:284-301,328-390)
  * <ViewInterestPoints><ViewInterestPointsFile timepoint setup label params>path of the label's group in
    interestpoints.n5 (InterestPointTools.addInterestPoints, J/SparkInterestPointDetection.java:898-903)
  * <BoundingBoxes><BoundingBoxDefinition name>: <min> and <max> (inclusive) integer corners in world coordinates
    (XmlIoBoundingBoxes, recalled; read by Import.getBoundingBox, J/util/Import.java:39-66)

Host-side plumbing only.  Everything else in the file is preserved verbatim on save.
"""
from __future__ import annotations

import copy
import os
import shutil
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field

import numpy as np

SPLIT_LOADER = "split.viewerimgloader"
FILEMAP_LOADER = "spimreconstruction.filemap2"


@dataclass
class ViewSetup:
    id: int
    size: tuple                      # (x, y, z)
    attributes: dict = field(default_factory=dict)   # illumination / channel / tile / angle -> int


def _fmt(values):
    return " ".join(repr(float(v)) for v in values)


class SpimData2:
    def __init__(self, tree: ET.ElementTree, path: str | None = None):
        self.tree = tree
        self.root = tree.getroot()
        self.path = path
        self.setups: dict[int, ViewSetup] = {}
        self.registrations: dict[tuple, list] = {}   # (tp, setup) -> [(name, 3x4 ndarray)], index 0 applied last
        self.timepoints: list[int] = []
        self._parse()

    # ------------------------------------------------------------------ load / save
    @classmethod
    def load(cls, path: str) -> "SpimData2":
        return cls(ET.parse(path), path)

    def _parse(self):
        seq = self.root.find("SequenceDescription")
        for vs in seq.find("ViewSetups").findall("ViewSetup"):
            sid = int(vs.findtext("id"))
            size = tuple(int(v) for v in vs.findtext("size").split())
            attrs = {}
            a = vs.find("attributes")
            if a is not None:
                for ch in a:
                    attrs[ch.tag] = int(ch.text)
            self.setups[sid] = ViewSetup(sid, size, attrs)
        tps = set()
        for vr in self.root.find("ViewRegistrations").findall("ViewRegistration"):
            tp, setup = int(vr.get("timepoint")), int(vr.get("setup"))
            lst = []
            for vt in vr.findall("ViewTransform"):
                m = np.array([float(v) for v in vt.findtext("affine").split()], dtype=np.float64).reshape(3, 4)
                lst.append((vt.findtext("Name") or "", m))
            self.registrations[(tp, setup)] = lst
            tps.add(tp)
        self.timepoints = sorted(tps)

    def _loader_element(self, nested=False):
        il = self.root.find("SequenceDescription").find("ImageLoader")
        return il.find("ImageLoader") if nested else il

    @staticmethod
    def _container_node(il):
        for tag in ("n5", "zarr", "hdf5"):
            if il.find(tag) is not None:
                return il.find(tag)
        return None

    def image_loader(self, nested=False):
        """(format, absolute container path) of the ImageLoader element; ``nested``: of the loader a
        `split.viewerimgloader` wraps."""
        il = self._loader_element(nested)
        fmt = il.get("format")
        node = self._container_node(il)
        p = node.text.strip() if node is not None else None
        if p is not None and node.get("type", "relative") == "relative" and self.path:
            base = self.root.findtext("BasePath") or "."
            p = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(self.path)), base, p))
        return fmt, p

    def zarr_groups(self, nested=False):
        """The views of a `bdv.multimg.zarr` loader: {(tp, setup): (group path, channel index, timepoint index)}.
        Element and attribute names are recalled from XmlIoAllenOMEZarrLoader (PARITY_GAPS R1)."""
        il = self._loader_element(nested)
        out = {}
        zg = il.find("zgroups")
        for g in (zg.findall("zgroup") if zg is not None else []):
            c, t = (int(v) for v in g.get("indicies", "[0, 0]").strip("[] ").split(","))
            out[(int(g.get("tp")), int(g.get("setup")))] = (g.get("path"), c, t)
        return out

    def _loader_path(self, container, xml_path):
        base = os.path.join(os.path.dirname(os.path.abspath(xml_path or self.path)), self.root.findtext("BasePath") or ".")
        return os.path.relpath(os.path.abspath(container), os.path.normpath(base))

    def set_image_loader(self, fmt, container, xml_path=None, zgroups=None):
        """Replace the ImageLoader: ``fmt`` "bdv.n5" (<n5>) or "bdv.multimg.zarr" (<zarr> and <zgroups>, ``zgroups`` =
        {(tp, setup): (group path, channel index, timepoint index)}).  The container path is written relative to the
        BasePath of the XML at ``xml_path`` (default: where it was loaded from)."""
        seq = self.root.find("SequenceDescription")
        old = seq.find("ImageLoader")
        il = ET.Element("ImageLoader", format=fmt, version="1.0")
        tag = "n5" if fmt == "bdv.n5" else "zarr"
        ET.SubElement(il, tag, type="relative").text = self._loader_path(container, xml_path)
        if fmt == "bdv.multimg.zarr":
            zg = ET.SubElement(il, "zgroups")
            for (tp, setup), (gpath, c, t) in sorted(zgroups.items()):
                ET.SubElement(zg, "zgroup", setup=str(setup), tp=str(tp), path=gpath, indicies=f"[{int(c)}, {int(t)}]")
        elif fmt != "bdv.n5":
            raise ValueError(f"ImageLoader format {fmt}")
        seq.insert(list(seq).index(old) if old is not None else 0, il)
        if old is not None:
            seq.remove(old)

    # ------------------------------------------------------------------ TIFF files (the automatic loader)
    def file_mappings(self):
        """The views of a `spimreconstruction.filemap2` loader: {(tp, setup): (absolute file path, series, channel)};
        relative paths resolve against the BasePath.  Element names are recalled from XmlIoFileMapImgLoaderLOCI2
        (PARITY_GAPS T1).  A z-grouped loader (one file per plane) raises NotImplementedError."""
        il = self._loader_element()
        for e in il:
            if e.tag.lower() == "zgrouped" and (e.text or "").strip().lower() == "true":
                raise NotImplementedError(f"ImageLoader {il.get('format')}: ZGrouped (one file per z-plane); "
                                          "only files holding whole stacks are read")
        base = os.path.join(os.path.dirname(os.path.abspath(self.path or ".")), self.root.findtext("BasePath") or ".")
        out = {}
        files = il.find("files")
        for m in (files.findall("FileMapping") if files is not None else []):
            f = m.find("file")
            p = f.text.strip()
            if f.get("type", "relative") == "relative":
                p = os.path.normpath(os.path.join(base, p))
            out[(int(m.get("timepoint")), int(m.get("view_setup")))] = (p, int(m.get("series", 0)),
                                                                        int(m.get("channel", 0)))
        return out

    def set_file_map_loader(self, mappings, xml_path=None):
        """Replace the ImageLoader by a `spimreconstruction.filemap2` one: ``mappings`` = {(tp, setup): (file path,
        series, channel)}, each path written relative to the BasePath of the XML at ``xml_path`` (default: where this
        one was loaded from)."""
        seq = self.root.find("SequenceDescription")
        old = seq.find("ImageLoader")
        il = ET.Element("ImageLoader", format=FILEMAP_LOADER)
        files = ET.SubElement(il, "files")
        for (tp, setup), (path, series, channel) in sorted(mappings.items()):
            m = ET.SubElement(files, "FileMapping", view_setup=str(int(setup)), timepoint=str(int(tp)),
                              series=str(int(series)), channel=str(int(channel)))
            ET.SubElement(m, "file", type="relative").text = self._loader_path(path, xml_path)
        seq.insert(list(seq).index(old) if old is not None else 0, il)
        if old is not None:
            seq.remove(old)

    # ------------------------------------------------------------------ split image loader (split-images)
    def split_setups(self):
        """The sub-views of a `split.viewerimgloader`: {new setup: (old setup, min int64[3], max int64[3])}, the box
        inclusive, in pixels of the old setup; {} for any other loader.  Element names are recalled from
        XmlIoSplitViewerImgLoader (PARITY_GAPS P4)."""
        il = self._loader_element()
        if il.get("format") != SPLIT_LOADER:
            return {}
        out = {}
        for d in il.find("SetupIds").findall("SetupIdDefinition"):
            box = [np.array([int(v) for v in d.findtext(k).split()], dtype=np.int64) for k in ("min", "max")]
            out[int(d.findtext("NewId"))] = (int(d.findtext("OldId")), box[0], box[1])
        return out

    def set_split_image_loader(self, nested, container, definitions, xml_path=None):
        """Replace the ImageLoader by a `split.viewerimgloader` wrapping a copy of ``nested`` (a `bdv.n5` or
        `bdv.multimg.zarr` <ImageLoader> element whose container lies at the absolute path ``container``); a relative
        container path is re-based onto the BasePath of the XML at ``xml_path`` (default: where this one was loaded
        from).  ``definitions``: {new setup: (old setup, min xyz, max xyz)}, old setups being those of the nested
        loader."""
        inner = copy.deepcopy(nested)
        node = self._container_node(inner)
        if node is not None and node.get("type", "relative") == "relative":
            node.text = self._loader_path(container, xml_path)
        seq = self.root.find("SequenceDescription")
        old = seq.find("ImageLoader")
        il = ET.Element("ImageLoader", format=SPLIT_LOADER)
        il.append(inner)
        ids = ET.SubElement(il, "SetupIds")
        for new, (o, mn, mx) in sorted(definitions.items()):
            d = ET.SubElement(ids, "SetupIdDefinition")
            ET.SubElement(d, "NewId").text = str(int(new))
            ET.SubElement(d, "OldId").text = str(int(o))
            ET.SubElement(d, "min").text = " ".join(str(int(v)) for v in mn)
            ET.SubElement(d, "max").text = " ".join(str(int(v)) for v in mx)
        seq.insert(list(seq).index(old) if old is not None else 0, il)
        if old is not None:
            seq.remove(old)

    # ------------------------------------------------------------------ missing views, attribute entries
    def missing_views(self):
        """The (tp, setup) of every <MissingViews><View>."""
        mv = self.root.find("SequenceDescription").find("MissingViews")
        return {(int(v.get("timepoint")), int(v.get("setup"))) for v in (mv.findall("View") if mv is not None else [])}

    def set_missing_views(self, views):
        seq = self.root.find("SequenceDescription")
        mv = seq.find("MissingViews")
        if mv is None:
            mv = ET.SubElement(seq, "MissingViews")
        for v in list(mv):
            mv.remove(v)
        for tp, setup in sorted(views):
            ET.SubElement(mv, "View", timepoint=str(int(tp)), setup=str(int(setup)))

    def attribute_entries(self, name):
        """{id: dict(name=str, location=float64[3] or None)} of <ViewSetups><Attributes name=``name``>; None when the
        element is absent."""
        for a in self.root.find("SequenceDescription").find("ViewSetups").findall("Attributes"):
            if a.get("name") == name:
                out = {}
                for e in a:
                    loc = e.findtext("location")
                    out[int(e.findtext("id"))] = dict(name=e.findtext("name"),
                                                      location=None if loc is None else np.array([float(v) for v in loc.split()]))
                return out
        return None

    def set_attribute_entries(self, name, entries):
        """Rebuild <Attributes name=``name``> from {id: dict(name=, location=)} (entries in id order)."""
        vss = self.root.find("SequenceDescription").find("ViewSetups")
        old = next((a for a in vss.findall("Attributes") if a.get("name") == name), None)
        a = ET.Element("Attributes", name=name)
        for i, e in sorted(entries.items()):
            el = ET.SubElement(a, name.capitalize())
            ET.SubElement(el, "id").text = str(int(i))
            if e.get("name") is not None:
                ET.SubElement(el, "name").text = str(e["name"])
            if e.get("location") is not None:
                ET.SubElement(el, "location").text = _fmt(e["location"])
        if old is not None:
            vss.insert(list(vss).index(old), a)
            vss.remove(old)
        else:
            vss.append(a)

    def save(self, path: str | None = None, backup: bool = True):
        path = path or self.path
        if backup and os.path.exists(path):
            shutil.copyfile(path, path + "~1")   # the reference keeps ~1 backups (J/SparkResaveN5.java:80)
        ET.indent(self.tree, space="  ")
        self.tree.write(path, encoding="UTF-8", xml_declaration=True)

    # ------------------------------------------------------------------ registrations
    def model(self, tp: int, setup: int) -> np.ndarray:
        """ViewRegistration.getModel(): concatenation of the transform list, index 0 applied last."""
        M = np.eye(4)
        for _, m in self.registrations[(tp, setup)]:
            M = M @ np.vstack([m, [0, 0, 0, 1]])
        return M[:3, :].copy()

    def add_registration(self, view, name, M):
        """Preconcatenate the 3 x 4 affine ``M``: a new <ViewTransform> at index 0 of the view's list, applied last."""
        m = np.asarray(M, dtype=np.float64).reshape(3, 4).copy()
        for vr in self.root.find("ViewRegistrations").findall("ViewRegistration"):
            if (int(vr.get("timepoint")), int(vr.get("setup"))) == tuple(view):
                vt = ET.Element("ViewTransform", type="affine")
                ET.SubElement(vt, "Name").text = name
                ET.SubElement(vt, "affine").text = _fmt(m.ravel())
                first = vr.find("ViewTransform")
                vr.insert(list(vr).index(first) if first is not None else len(vr), vt)
                self.registrations[tuple(view)].insert(0, (name, m))
                return
        raise KeyError(f"no ViewRegistration for {view}")

    def remove_first_registration(self, view):
        """Drop the view's <ViewTransform> at index 0 (the one applied last, e.g. the latest solve); returns its
        (name, 3 x 4 affine).  The view must have one."""
        for vr in self.root.find("ViewRegistrations").findall("ViewRegistration"):
            if (int(vr.get("timepoint")), int(vr.get("setup"))) == tuple(view):
                vr.remove(vr.find("ViewTransform"))
                return self.registrations[tuple(view)].pop(0)
        raise KeyError(f"no ViewRegistration for {view}")

    def view_ids(self):
        return sorted(self.registrations)

    def select_views(self, vi=None, angle_ids=None, channel_ids=None, illumination_ids=None, tile_ids=None,
                     timepoint_ids=None):
        """AbstractSelectableViews.loadViewIds / Import.createViewIds (J/abstractcmdline/AbstractSelectableViews.java:
        38-110, J/util/Import.java:79-139): either explicit ViewIds (`-vi 'tp,setup'`, those that exist) OR any
        combination of --angleId / --channelId / --illuminationId / --tileId / --timepointId id lists (None = all);
        both together is an error, an empty selection is an error.  Id lists may be comma-separated strings."""
        attr_filters = (angle_ids, channel_ids, illumination_ids, tile_ids, timepoint_ids)
        if vi is not None and any(f is not None for f in attr_filters):
            raise ValueError("You can only specify ViewIds (-vi) OR angles, channels, illuminations, tiles, timepoints.")

        def ids(x):
            if x is None:
                return None
            if isinstance(x, str):
                return {int(t) for t in x.split(",") if t.strip() != ""}
            return {int(t) for t in x}

        if vi is not None:
            want = []
            for v in vi:
                tp, setup = (int(t) for t in v.split(",")) if isinstance(v, str) else (int(v[0]), int(v[1]))
                want.append((tp, setup))
            out = sorted(set(want) & set(self.view_ids()))
        else:
            a, c, i, ti, tp = (ids(f) for f in attr_filters)
            out = []
            for (t, s) in self.view_ids():
                at = self.setups[s].attributes
                if ((a is None or at.get("angle", 0) in a) and (c is None or at.get("channel", 0) in c) and
                        (i is None or at.get("illumination", 0) in i) and (ti is None or at.get("tile", s) in ti) and
                        (tp is None or t in tp)):
                    out.append((t, s))
        if not out:
            raise ValueError("No views to be processed.")
        return out

    def channels_ordered(self):
        """sd.getAllChannelsOrdered(): the distinct channel ids in ascending order (J/SparkAffineFusion.java:420-421)."""
        return sorted({s.attributes.get("channel", 0) for s in self.setups.values()})

    def views_of(self, channel_index: int, timepoint_index: int, view_ids=None):
        """The views `affine-fusion` fuses into the (channel, timepoint) volume (J/SparkAffineFusion.java:425-440), out
        of ``view_ids`` (the command's view selection; default all)."""
        ch = self.channels_ordered()[channel_index]
        tp = self.timepoints[timepoint_index]
        pool = self.view_ids() if view_ids is None else sorted(view_ids)
        return [v for v in pool if v[0] == tp and self.setups[v[1]].attributes.get("channel", 0) == ch]

    # ------------------------------------------------------------------ pair construction (row a1)
    def stitching_pairs(self):
        """All tile pairs per (timepoint, angle, channel, illumination) whose transformed bounding
        boxes overlap (SpimDataFilteringAndGrouping + filterNonOverlappingPairs,
        J/SparkPairwiseStitching.java:142-176).  Single-view groups (one channel / illumination)."""
        pairs = []
        vids = self.view_ids()
        boxes = {}
        for (tp, s) in vids:
            M = self.model(tp, s)
            dx, dy, dz = self.setups[s].size
            c = np.array([[x, y, z] for x in (0, dx - 1) for y in (0, dy - 1) for z in (0, dz - 1)], dtype=np.float64)
            w = c @ M[:, :3].T + M[:, 3]
            boxes[(tp, s)] = (w.min(axis=0), w.max(axis=0))
        for i, a in enumerate(vids):
            for b in vids[i + 1:]:
                if a[0] != b[0]:
                    continue
                sa, sb = self.setups[a[1]].attributes, self.setups[b[1]].attributes
                if any(sa.get(k, 0) != sb.get(k, 0) for k in ("angle", "channel", "illumination")):
                    continue
                if sa.get("tile", a[1]) == sb.get("tile", b[1]):
                    continue
                lo = np.maximum(boxes[a][0], boxes[b][0])
                hi = np.minimum(boxes[a][1], boxes[b][1])
                if np.all(hi >= lo):
                    pairs.append((a, b))
        return pairs

    def stitching_groups(self, view_ids=None):
        """SpimDataFilteringAndGrouping with the reference's defaults (J/SparkPairwiseStitching.java:141-162): views are
        GROUPED over {channel, illumination}, COMPARED across tiles, per (timepoint, angle).  Returns the overlapping
        pairs of groups: [(groupA, groupB)], a group = ascending list of ViewIds of one tile; non-overlapping
        comparisons are dropped (TransformationTools.filterNonOverlappingPairs, :165).  ``view_ids``: the command's view
        selection (J/SparkPairwiseStitching.java:120-121, default all)."""
        groups = {}
        for (tp, s) in (self.view_ids() if view_ids is None else sorted(view_ids)):
            a = self.setups[s].attributes
            groups.setdefault((tp, a.get("angle", 0), a.get("tile", s)), []).append((tp, s))
        keys = sorted(groups)
        boxes = {}
        for k in keys:
            lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
            for (tp, s) in groups[k]:
                M = self.model(tp, s)
                dx, dy, dz = self.setups[s].size
                c = np.array([[x, y, z] for x in (0, dx - 1) for y in (0, dy - 1) for z in (0, dz - 1)], dtype=np.float64)
                w = c @ M[:, :3].T + M[:, 3]
                lo, hi = np.minimum(lo, w.min(axis=0)), np.maximum(hi, w.max(axis=0))
            boxes[k] = (lo, hi)
        pairs = []
        for i, ka in enumerate(keys):
            for kb in keys[i + 1:]:
                if ka[:2] != kb[:2]:
                    continue
                lo = np.maximum(boxes[ka][0], boxes[kb][0])
                hi = np.minimum(boxes[ka][1], boxes[kb][1])
                if np.all(hi >= lo):
                    pairs.append((sorted(groups[ka]), sorted(groups[kb])))
        return pairs

    # ------------------------------------------------------------------ stitching results (rows a6, f-2)
    @staticmethod
    def transform_hash(reg_a, reg_b) -> float:
        """Stand-in for PairwiseStitchingResult.calculateHash(vrA, vrB): a double derived from both
        views' transform coefficients.  Upstream's exact formula is not recoverable here (PARITY_GAPS
        #22); the Java glue recomputes it with the real method (J/SparkPairwiseStitching.java:287-289),
        `solver` only tests it for equality (J/Solver.java:407-414)."""
        h = 0.0
        for lst in (reg_a, reg_b):
            for i, (_, m) in enumerate(lst):
                h += float(np.sum(m * (np.arange(12).reshape(3, 4) + 1 + 13 * i)))
        return h

    @staticmethod
    def _group_of(pr, side):
        """ViewIds of one side of a <PairwiseResult>: upstream writes comma-separated lists for grouped views."""
        tps = [int(v) for v in pr.get("tp_" + side).split(",")]
        sts = [int(v) for v in pr.get("view_setup_" + side).split(",")]
        if len(tps) == 1 and len(sts) > 1:
            tps = tps * len(sts)
        return tuple(sorted(zip(tps, sts)))

    @staticmethod
    def _as_group(g):
        return tuple(sorted(g)) if isinstance(g[0], (tuple, list)) else (tuple(g),)

    def remove_stitching_results(self, pairs):
        """Drop stored results a->b and b->a for every COMPARED pair, including those that found no shift
        (J/SparkPairwiseStitching.java:323-325)."""
        sr = self.root.find("StitchingResults")
        if sr is None:
            return
        keys = {frozenset((self._as_group(a), self._as_group(b))) for a, b in pairs}
        for pr in list(sr.findall("PairwiseResult")):
            if frozenset((self._group_of(pr, "a"), self._group_of(pr, "b"))) in keys:
                sr.remove(pr)

    def stitching_results(self):
        out = []
        sr = self.root.find("StitchingResults")
        if sr is None:
            return out
        for pr in sr.findall("PairwiseResult"):
            ga, gb = self._group_of(pr, "a"), self._group_of(pr, "b")
            a = ga[0] if len(ga) == 1 else ga
            b = gb[0] if len(gb) == 1 else gb
            shift = np.array([float(v) for v in pr.findtext("shift").split()]).reshape(3, 4)
            bb = [float(v) for v in (pr.findtext("overlap_boundingbox") or "").split()]
            out.append(dict(pair=(a, b), shift=shift, r=float(pr.findtext("correlation")),
                            hash=float(pr.findtext("hash")), bbox=bb))
        return out

    def set_stitching_results(self, results):
        """results: iterable of dict(pair=((tpA,setupA),(tpB,setupB)), shift 3x4, r, hash, bbox_min, bbox_max).
        Existing results for the same pair (either direction) are replaced
        (J/SparkPairwiseStitching.java:328-342)."""
        sr = self.root.find("StitchingResults")
        if sr is None:
            sr = ET.SubElement(self.root, "StitchingResults")
        for res in results:
            ga, gb = self._as_group(res["pair"][0]), self._as_group(res["pair"][1])
            self.remove_stitching_results([(ga, gb)])
            pr = ET.SubElement(sr, "PairwiseResult",
                               view_setup_a=",".join(str(v[1]) for v in ga), view_setup_b=",".join(str(v[1]) for v in gb),
                               tp_a=",".join(str(v[0]) for v in ga), tp_b=",".join(str(v[0]) for v in gb))
            sh = ET.SubElement(pr, "shift", type="affine")
            sh.text = _fmt(np.asarray(res["shift"]).ravel())
            ET.SubElement(pr, "correlation").text = repr(float(res["r"]))
            ET.SubElement(pr, "hash").text = repr(float(res["hash"]))
            ET.SubElement(pr, "overlap_boundingbox").text = _fmt(list(res["bbox_min"]) + list(res["bbox_max"]))

    # ------------------------------------------------------------------ interest points
    def interest_points(self):
        """{(tp, setup): {label: dict(params=..., path=...)}} of <ViewInterestPoints>."""
        out = {}
        vip = self.root.find("ViewInterestPoints")
        if vip is None:
            return out
        for f in vip.findall("ViewInterestPointsFile"):
            key = (int(f.get("timepoint")), int(f.get("setup")))
            out.setdefault(key, {})[f.get("label")] = dict(params=f.get("params"), path=(f.text or "").strip())
        return out

    def set_interest_points(self, label, params, paths):
        """Add or replace the ``label`` entry of every view in ``paths`` ({(tp, setup): path}); other labels are kept.
        Entries stay ordered by (timepoint, setup, label)."""
        vip = self.root.find("ViewInterestPoints")
        if vip is None:
            vip = ET.SubElement(self.root, "ViewInterestPoints")
        entries = {}
        for f in vip.findall("ViewInterestPointsFile"):
            entries[(int(f.get("timepoint")), int(f.get("setup")), f.get("label"))] = f
            vip.remove(f)
        for (tp, setup), path in paths.items():
            f = ET.Element("ViewInterestPointsFile", timepoint=str(tp), setup=str(setup), label=label, params=params)
            f.text = path
            entries[(int(tp), int(setup), label)] = f
        for k in sorted(entries):
            vip.append(entries[k])

    def clear_interest_points(self):
        """Remove every <ViewInterestPointsFile> (all labels of all views); <ViewInterestPoints> stays, empty."""
        vip = self.root.find("ViewInterestPoints")
        for f in (list(vip) if vip is not None else []):
            vip.remove(f)

    # ------------------------------------------------------------------ bounding boxes
    def bounding_boxes(self):
        """{name: (min int64[3], max int64[3])} of <BoundingBoxes>, max inclusive.  When two definitions share a name
        the later one wins, as in Import.getBoundingBox (J/util/Import.java:53-57)."""
        out = {}
        bbs = self.root.find("BoundingBoxes")
        for b in (bbs.findall("BoundingBoxDefinition") if bbs is not None else []):
            out[b.get("name")] = tuple(np.array([int(v) for v in b.findtext(k).split()], dtype=np.int64)
                                       for k in ("min", "max"))
        return out

    def set_bounding_box(self, name, bb_min, bb_max, replace=False):
        """Append a <BoundingBoxDefinition> (earlier ones of the same name stay, and lose to this one on reading;
        ``replace`` removes them instead)."""
        bbs = self.root.find("BoundingBoxes")
        if bbs is None:
            bbs = ET.SubElement(self.root, "BoundingBoxes")
        if replace:
            for b in bbs.findall("BoundingBoxDefinition"):
                if b.get("name") == str(name):
                    bbs.remove(b)
        b = ET.SubElement(bbs, "BoundingBoxDefinition", name=str(name))
        ET.SubElement(b, "min").text = " ".join(str(int(v)) for v in bb_min)
        ET.SubElement(b, "max").text = " ".join(str(int(v)) for v in bb_max)

    # ------------------------------------------------------------------ point spread functions
    def point_spread_functions(self):
        """{(tp, setup): file name relative to `psfs/` next to the XML} of <PointSpreadFunctions> (mvrecon
        XmlIoPointSpreadFunctions, recalled: <PointSpreadFunction timepoint= setup=><file>...</file>)."""
        psfs = self.root.find("PointSpreadFunctions")
        return {(int(p.get("timepoint")), int(p.get("setup"))): (p.findtext("file") or "").strip()
                for p in (psfs.findall("PointSpreadFunction") if psfs is not None else [])}

    def set_point_spread_functions(self, files):
        """Add or replace the <PointSpreadFunction> of every view in ``files`` ({(tp, setup): file name}); the entries
        of other views are kept.  Entries stay ordered by (timepoint, setup)."""
        psfs = self.root.find("PointSpreadFunctions")
        if psfs is None:
            psfs = ET.SubElement(self.root, "PointSpreadFunctions")
        entries = {**self.point_spread_functions(), **{(int(t), int(s)): str(f) for (t, s), f in files.items()}}
        for p in list(psfs):
            psfs.remove(p)
        for (tp, setup), f in sorted(entries.items()):
            p = ET.SubElement(psfs, "PointSpreadFunction", timepoint=str(tp), setup=str(setup))
            ET.SubElement(p, "file").text = f


# ---------------------------------------------------------------------------------------------
def fusion_project(xml_path, dims_xyz, num_channels, num_timepoints, anisotropy_factor=None) -> SpimData2:
    """The BigStitcher project of a fused container (SpimData2Tools.createNewSpimDataForFusion, recalled; the setups
    and timepoints are J/CreateFusionContainer.java:404-434, in-repo): one ViewSetup per channel c (id c, name
    "setup c", size ``dims_xyz``, Tile 0, Channel c, Angle 0, Illumination 0), timepoints 0 .. n-1, and one
    `calibration` ViewTransform per view, diag(1, 1, af) with ``anisotropy_factor`` (identity without), matching the
    voxel size (1, 1, af) or (1, 1, 1) micrometer.  The box minimum is not carried: world = fused pixel grid.  No
    ImageLoader yet (set_image_loader adds it); not saved."""
    af = 1.0 if anisotropy_factor is None else float(anisotropy_factor)
    root = ET.Element("SpimData", version="0.2")
    ET.SubElement(root, "BasePath", type="relative").text = "."
    seq = ET.SubElement(root, "SequenceDescription")
    vss = ET.SubElement(seq, "ViewSetups")
    for c in range(num_channels):
        vs = ET.SubElement(vss, "ViewSetup")
        ET.SubElement(vs, "id").text = str(c)
        ET.SubElement(vs, "name").text = f"setup {c}"
        ET.SubElement(vs, "size").text = " ".join(str(int(v)) for v in dims_xyz)
        vx = ET.SubElement(vs, "voxelSize")
        ET.SubElement(vx, "unit").text = "micrometer"
        ET.SubElement(vx, "size").text = _fmt([1.0, 1.0, af])
        at = ET.SubElement(vs, "attributes")
        for tag, v in (("illumination", 0), ("channel", c), ("tile", 0), ("angle", 0)):
            ET.SubElement(at, tag).text = str(v)
    for tag, ids in (("illumination", [0]), ("channel", range(num_channels)), ("tile", [0]), ("angle", [0])):
        a = ET.SubElement(vss, "Attributes", name=tag)
        for i in ids:
            e = ET.SubElement(a, tag.capitalize())
            ET.SubElement(e, "id").text = str(i)
            ET.SubElement(e, "name").text = f"Channel {i}" if tag == "channel" else str(i)
    tp = ET.SubElement(seq, "Timepoints", type="pattern")
    ET.SubElement(tp, "integerpattern").text = "0" if num_timepoints == 1 else f"0-{num_timepoints - 1}"
    ET.SubElement(seq, "MissingViews")
    vrs = ET.SubElement(root, "ViewRegistrations")
    for t in range(num_timepoints):
        for c in range(num_channels):
            vr = ET.SubElement(vrs, "ViewRegistration", timepoint=str(t), setup=str(c))
            vt = ET.SubElement(vr, "ViewTransform", type="affine")
            ET.SubElement(vt, "Name").text = "calibration"
            ET.SubElement(vt, "affine").text = _fmt([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, af, 0])
    for tag in ("ViewInterestPoints", "BoundingBoxes", "PointSpreadFunctions", "StitchingResults", "IntensityAdjustments"):
        ET.SubElement(root, tag)
    return SpimData2(ET.ElementTree(root), xml_path)


# ---------------------------------------------------------------------------------------------
def write_dataset_xml(path, n5_rel_path, tiles, timepoint=0):
    """Write a fresh SpimData2 project: ``tiles`` = list of dict(setup, size_xyz, tile, translation_xyz
    [, channel, illumination, angle]).  Used by the synthetic end-to-end configs (SURVEY.md 8d config 1/5)."""
    root = ET.Element("SpimData", version="0.2")
    ET.SubElement(root, "BasePath", type="relative").text = "."
    seq = ET.SubElement(root, "SequenceDescription")
    il = ET.SubElement(seq, "ImageLoader", format="bdv.n5", version="1.0")
    ET.SubElement(il, "n5", type="relative").text = n5_rel_path
    vss = ET.SubElement(seq, "ViewSetups")
    for t in tiles:
        vs = ET.SubElement(vss, "ViewSetup")
        ET.SubElement(vs, "id").text = str(t["setup"])
        ET.SubElement(vs, "name").text = str(t["setup"])
        ET.SubElement(vs, "size").text = " ".join(str(int(v)) for v in t["size_xyz"])
        vx = ET.SubElement(vs, "voxelSize")
        ET.SubElement(vx, "unit").text = "px"
        ET.SubElement(vx, "size").text = "1.0 1.0 1.0"
        at = ET.SubElement(vs, "attributes")
        ET.SubElement(at, "illumination").text = str(t.get("illumination", 0))
        ET.SubElement(at, "channel").text = str(t.get("channel", 0))
        ET.SubElement(at, "tile").text = str(t.get("tile", t["setup"]))
        ET.SubElement(at, "angle").text = str(t.get("angle", 0))
    tp = ET.SubElement(seq, "Timepoints", type="pattern")
    ET.SubElement(tp, "integerpattern").text = str(timepoint)
    ET.SubElement(seq, "MissingViews")
    vrs = ET.SubElement(root, "ViewRegistrations")
    for t in tiles:
        vr = ET.SubElement(vrs, "ViewRegistration", timepoint=str(timepoint), setup=str(t["setup"]))
        vt = ET.SubElement(vr, "ViewTransform", type="affine")
        ET.SubElement(vt, "Name").text = "Translation to Regular Grid"
        tx, ty, tz = t["translation_xyz"]
        ET.SubElement(vt, "affine").text = _fmt([1, 0, 0, tx, 0, 1, 0, ty, 0, 0, 1, tz])
        vt = ET.SubElement(vr, "ViewTransform", type="affine")
        ET.SubElement(vt, "Name").text = "calibration"
        ET.SubElement(vt, "affine").text = _fmt([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])
    for tag in ("ViewInterestPoints", "BoundingBoxes", "PointSpreadFunctions", "StitchingResults", "IntensityAdjustments"):
        ET.SubElement(root, tag)
    tree = ET.ElementTree(root)
    ET.indent(tree, space="  ")
    tree.write(path, encoding="UTF-8", xml_declaration=True)
    return path
