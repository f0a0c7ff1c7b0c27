"""nonrigid-fusion --intensityN5Path without a GPU: the coefficient lookup, the check before anything is written, and the
s0 windows handed to intensity_apply and then to the fusion, through a context that records both."""
import os

import numpy as np
import pytest

from bsgpu import commands, intensity as bint, n5 as bn5, native, spimdata
from oracle import intensity_oracle as io
from oracle import nonrigid_oracle as no
from tests import synth
from tests.fake_ctx import FakeContext
from tests.test_nonrigid_cpu import write_correspondences, write_points


class RecordingContext(FakeContext):
    """FakeContext plus the non-rigid entry points: control-point grids from the oracle, fused blocks recorded (their
    views and the dtype of each resident volume) and returned as zeros, intensity_apply recorded and computed by the
    oracle."""

    def __init__(self):
        super().__init__()
        self.applies, self.fused = [], []

    def nonrigid_debug_grid(self, view, block_min_xyz, block_size_xyz, cp_distance=(native.NONRIGID_CP_DISTANCE,) * 3):
        return no.mls_grid(view["target_world_xyz"], view["local_xyz"], view["src_to_world"], block_min_xyz,
                           block_size_xyz, cp_distance)

    def nonrigid_fuse_blocks(self, views, block_mins_xyz, block_sizes_xyz, params=None,
                             cp_distance=(native.NONRIGID_CP_DISTANCE,) * 3, outs=None):
        self.fused.append([(dict(v), self.vols[v["vol_handle"]].dtype) for v in views])
        return [np.zeros(tuple(s)[::-1], dtype=native._out_dtype(params)) for s in block_sizes_xyz]

    def intensity_apply(self, h, full_dims_xyz, level_to_full, coeff_a, coeff_b, window_min_xyz=(0, 0, 0)):
        out = self.volume_upload(io.apply(self.vols[h], window_min_xyz, level_to_full, full_dims_xyz, coeff_a, coeff_b))
        self.applies.append(dict(raw=self.vols[h].copy(), out=out, full_dims=tuple(int(d) for d in full_dims_xyz),
                                 level_to_full=np.asarray(level_to_full), window_min=tuple(int(x) for x in window_min_xyz),
                                 a=np.asarray(coeff_a), b=np.asarray(coeff_b)))
        return out


def scene(tmp_path):
    """Three uint16 views of one field: 0 and 1 overlap by 24 px in x and share 40 corresponding beads, 2 overlaps 0 in y
    and has no points.  Returns (xml, {view: [z, y, x] image}, {view: 3x4 registration})."""
    G = synth.field((20, 76, 110), seed=3, sigma=1.5)
    specs = [(0, (0, 0, 0)), (1, (40, 2, 0)), (2, (8, 30, 0))]
    tiles, imgs = [], {}
    src = bn5.N5Store(str(tmp_path / "dataset.n5"), create=True)
    for s, t in specs:
        img = synth.tile_from(G, (t[2], t[1], t[0]), (20, 40, 64), s + 1)
        imgs[(0, s)] = img
        tiles.append(dict(setup=s, size_xyz=(64, 40, 20), translation_xyz=t))
        bn5.write_bdv_setup(src, s, 0, img, block_size=(32, 32, 16))
    xml = spimdata.write_dataset_xml(str(tmp_path / "dataset.xml"), "dataset.n5", tiles)
    rng = np.random.default_rng(7)
    p = np.column_stack([rng.uniform(40, 63, 40), rng.uniform(2, 39, 40), rng.uniform(0, 19, 40)])
    ips = bn5.N5Store(str(tmp_path / "interestpoints.n5"), create=True)
    a, b = (0, 0), (0, 1)
    write_points(ips, a, "beads", p + rng.uniform(-0.7, 0.7, p.shape))
    write_points(ips, b, "beads", p - (40, 2, 0) + rng.uniform(-0.7, 0.7, p.shape))
    write_correspondences(ips, a, "beads", [(i, b, "beads", i) for i in range(40)])
    write_correspondences(ips, b, "beads", [(i, a, "beads", i) for i in range(40)])
    data = spimdata.SpimData2.load(xml)
    return xml, imgs, {v: data.model(*v) for v in data.view_ids()}


def seeded_coefficients(views, n_cells=(4, 3, 2), seed=12):
    """{view: (a, b)} that vary from cell to cell: a in [0.6, 1.4], b in [-50, 50]."""
    rng = np.random.default_rng(seed)
    shape = tuple(n_cells)[::-1]
    return {v: (rng.uniform(0.6, 1.4, shape), rng.uniform(-50.0, 50.0, shape)) for v in views}


def _run(xml, ctx, out, **kw):
    return commands.nonrigid_fusion(xml, ctx, out, "fused/s0", ["beads"], block_size=(32, 32, 16), blocks_per_call=1,
                                    **kw)


def test_missing_view_raises_before_the_output_exists(tmp_path):
    xml, _, regs = scene(tmp_path)
    cpath = str(tmp_path / "coeff.n5")
    bint.write_coefficients(cpath, "N5", "grp", "intensity", seeded_coefficients([(0, 0), (0, 1)]))
    ctx = RecordingContext()
    out = str(tmp_path / "fused.n5")
    with pytest.raises(ValueError, match=r"setup 2\).*grp/setup2/timepoint0/intensity"):
        _run(xml, ctx, out, intensity_n5_path=cpath, intensity_n5_group="grp")
    assert not os.path.exists(out)
    assert not ctx.applies and not ctx.fused and not ctx.vols
    # the same storage rules as affine-fusion: HDF5 is not built, an unknown ending needs the storage named
    with pytest.raises(NotImplementedError):
        _run(xml, ctx, out, intensity_n5_path=str(tmp_path / "coeff.h5"))
    with pytest.raises(ValueError, match="storage"):
        _run(xml, ctx, out, intensity_n5_path=str(tmp_path / "coeff"))
    assert not os.path.exists(out)
    # a selection without the view reads only what it fuses
    _run(xml, ctx, out, intensity_n5_path=cpath, intensity_n5_group="grp", view_selection=dict(tile_ids=[0, 1]))
    assert ctx.applies and not ctx.vols


@pytest.mark.parametrize("storage, name", [("N5", "coeff.n5"), ("ZARR", "coeff.zarr")])
def test_every_window_is_corrected_at_its_origin(tmp_path, storage, name):
    xml, imgs, regs = scene(tmp_path)
    co = seeded_coefficients(sorted(imgs))
    cpath = str(tmp_path / name)
    bint.write_coefficients(cpath, storage, "", "intensity", co)
    ctx = RecordingContext()
    written = _run(xml, ctx, str(tmp_path / "fused.n5"), data_type="UINT16", min_intensity=0.0, max_intensity=2000.0,
                   intensity_n5_path=cpath)
    assert written and not ctx.vols                       # every raw and corrected window was freed
    applies = {a["out"]: a for a in ctx.applies}
    fused = [fv for call in ctx.fused for fv in call]
    assert len(fused) == len(applies)                     # one correction per staged window, each fused once
    view_of = {tuple(np.asarray(m).reshape(3, 4)[:, 3]): v for v, m in regs.items()}
    origins = set()
    for fv, dt in fused:
        v = view_of[tuple(np.asarray(fv["src_to_world"]).reshape(3, 4)[:, 3])]
        a = applies[fv["vol_handle"]]
        assert dt == np.float32
        assert a["window_min"] == tuple(fv["window_min"]) and a["full_dims"] == tuple(fv["full_dims"]) == (64, 40, 20)
        assert np.array_equal(a["level_to_full"], np.eye(3, 4))
        assert np.array_equal(a["a"], co[v][0]) and np.array_equal(a["b"], co[v][1])
        # the raw window is view v's s0 at window_min
        w, (z, y, x) = a["window_min"], a["raw"].shape
        assert np.array_equal(a["raw"], imgs[v][w[2]:w[2] + z, w[1]:w[1] + y, w[0]:w[0] + x])
        origins.add(w)
    assert len(origins) > 2 and any(o != (0, 0, 0) for o in origins)


def test_without_the_option_nothing_is_corrected(tmp_path):
    xml, imgs, _ = scene(tmp_path)
    ctx = RecordingContext()
    assert _run(xml, ctx, str(tmp_path / "fused.n5"))
    assert not ctx.applies and ctx.fused and not ctx.vols
    assert all(dt == np.uint16 for call in ctx.fused for _, dt in call)
