"""nonrigid-fusion without a GPU: the oracle's known answers (PARITY_GAPS N2-N4), the correspondence reader, the
viewsToFuse / viewsToUse rule, the command's argument checks and the bs_nonrigid_view layout."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy.ndimage import gaussian_filter, map_coordinates

import bsgpu
from bsgpu import commands, n5 as bn5
from oracle import fusion_oracle as fo
from oracle import nonrigid_oracle as no

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------ test writers (N1)
def write_points(store, view, label, loc):
    group = f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}"
    loc = np.asarray(loc, dtype=np.float64).reshape(-1, 3)
    store.set_attributes(group + "/interestpoints", {"pointcloud": "1.0.0", "type": "list", "list version": "1.0.0"})
    store.write_list(group + "/interestpoints/id", np.arange(len(loc), dtype=np.uint64).reshape(-1, 1), 300000, "zstd")
    store.write_list(group + "/interestpoints/loc", loc, 300000, "zstd")


def write_correspondences(store, view, label, rows):
    """rows: [(detection id, (tp, setup), label, corresponding detection id)] as InterestPointsN5 stores them: group
    attributes correspondences = "1.0.0" and idMap {"tp,setup,label": index}, dataset data uint64 {3, M} of
    (detectionId, correspondingDetectionId, idMap index), {0} when empty."""
    group = f"tpId_{view[0]}_viewSetupId_{view[1]}/{label}/correspondences"
    keys = sorted({(pv, pl) for _, pv, pl, _ in rows})
    idmap = {f"{pv[0]},{pv[1]},{pl}": i for i, (pv, pl) in enumerate(keys)}
    store.set_attributes(group, {"correspondences": "1.0.0", "idMap": idmap})
    data = np.array([(a, b, idmap[f"{pv[0]},{pv[1]},{pl}"]) for a, pv, pl, b in rows], dtype=np.uint64).reshape(-1, 3)
    store.write_list(group + "/data", data, 300000, "zstd")


def translation(t):
    return np.array([[1, 0, 0, t[0]], [0, 1, 0, t[1]], [0, 0, 1, t[2]]], dtype=np.float64)


# ------------------------------------------------------------------------------------------ N3 / N4 known answers
def _affine():
    th = np.deg2rad(7.0)
    A = np.array([[np.cos(th), -np.sin(th), 0.05], [np.sin(th), np.cos(th), 0.0], [0.02, 0.0, 1.1]])
    return np.hstack([A, [[12.5], [-3.25], [4.0]]])


def test_grid_of_affine_correspondences_equals_the_map():
    M = _affine()                                        # local pixel -> world
    rng = np.random.default_rng(3)
    loc = rng.uniform(0, 80, (60, 3))
    tgt = loc @ M[:, :3].T + M[:, 3]
    other = np.hstack([np.eye(3) * 1.3, [[1.0], [2.0], [3.0]]])   # a different registration: the fallback is not used
    g = no.mls_grid(tgt, loc, other, (5, -7, 3), (23, 17, 11))
    want = no.control_points((5, -7, 3), (23, 17, 11)) @ fo.invert_affine(M)[:, :3].T + fo.invert_affine(M)[:, 3]
    assert g.shape == (4, 5, 6, 3) and no.grid_dims((23, 17, 11)) == (6, 5, 4)
    assert np.abs(g - want).max() < 1e-9


def test_grid_dims_cover_the_block_plus_one_cell():
    assert no.grid_dims((20, 21, 1)) == (5, 5, 3)
    cp = no.control_points((100, 0, 0), (21, 10, 1))
    assert cp[0, 0, 0].tolist() == [90.0, -10.0, -10.0] and cp[0, 0, -1, 0] == 130.0


def test_control_point_on_a_target_returns_its_local_point():
    rng = np.random.default_rng(4)
    tgt = rng.uniform(0, 50, (12, 3)).round()
    loc = rng.uniform(0, 50, (12, 3))
    tgt[5] = (20.0, 30.0, 10.0)
    r = no.mls(np.array([[20.0, 30.0, 10.0], [20.5, 30.0, 10.0]]), tgt, loc, translation((1, 1, 1)))
    assert np.array_equal(r[0], loc[5]) and not np.array_equal(r[1], loc[5])


def test_fewer_than_four_points_use_the_inverse_registration():
    M = translation((10.0, -4.0, 2.5))
    x = no.control_points((0, 0, 0), (15, 15, 5))
    tgt = np.array([[1.0, 2.0, 3.0], [4.0, 0.0, 1.0], [7.0, 7.0, 0.0]])
    g = no.mls(x, tgt, tgt + 100.0, M)
    assert np.array_equal(g, x - np.array([10.0, -4.0, 2.5]))
    # coplanar points: a singular fit, also the fallback
    cop = np.array([[0.0, 0, 5], [10, 0, 5], [0, 10, 5], [10, 10, 5], [5, 5, 5]])
    assert np.allclose(no.mls(np.array([[3.0, 4.0, 1.0]]), cop, cop * 2, M), [[-7.0, 8.0, -1.5]])


# ------------------------------------------------------------------------------------------ N2 targets on a 3-view chain
def _chain(tmp_path):
    """views a - b - c: a0 <-> b0, b1 <-> c0 (label beads); c1 has a 'nuclei' partner in a (a's nuclei point 0)."""
    store = bn5.N5Store(str(tmp_path / "interestpoints.n5"), create=True)
    a, b, c = (0, 0), (0, 1), (0, 2)
    regs = {a: translation((0, 0, 0)), b: translation((100, 0, 0)), c: translation((200, 0, 0))}
    write_points(store, a, "beads", [[110.0, 5, 5], [1, 1, 1]])
    write_points(store, b, "beads", [[12.0, 5, 5], [95, 7, 3]])
    write_points(store, c, "beads", [[-4.0, 7, 4], [0, 0, 0]])
    write_points(store, a, "nuclei", [[50.0, 50, 50]])
    write_correspondences(store, a, "beads", [(0, b, "beads", 0)])
    write_correspondences(store, b, "beads", [(0, a, "beads", 0), (1, c, "beads", 0)])
    write_correspondences(store, c, "beads", [(0, b, "beads", 1), (1, a, "nuclei", 0)])
    write_correspondences(store, a, "nuclei", [(0, c, "beads", 1)])
    return store, regs, (a, b, c)


def test_targets_average_direct_partners_only(tmp_path):
    store, regs, (a, b, c) = _chain(tmp_path)
    ips = commands._InterestPoints(store, [a, b, c], ["beads"], regs)
    t, l = ips.targets(b, [a, b, c])
    # b0 (world 112) pairs with a0 (world 110): 111; b1 (world 195, 7, 3) pairs with c0 (world 196, 7, 4) -- no chaining
    assert np.allclose(t, [[111.0, 5, 5], [195.5, 7, 3.5]]) and np.allclose(l, [[12.0, 5, 5], [95, 7, 3]])
    t, l = ips.targets(a, [a, b])
    assert np.allclose(t, [[111.0, 5, 5]]) and np.allclose(l, [[110.0, 5, 5]])
    t, _ = ips.targets(a, [a, c])                        # partner outside viewsToUse: no point
    assert t.shape == (0, 3)
    t, l = ips.targets(c, [a, b, c])                     # the nuclei partner does not count for -ip beads
    assert np.allclose(t, [[195.5, 7, 3.5]]) and np.allclose(l, [[-4.0, 7, 4]])
    both = commands._InterestPoints(store, [a, b, c], ["beads", "nuclei"], regs)
    t, l = both.targets(c, [a, b, c])
    assert np.allclose(t, [[195.5, 7, 3.5], [125.0, 25, 25]]) and np.allclose(l, [[-4.0, 7, 4], [0, 0, 0]])
    # the oracle's independent assembly agrees
    pts, corr = {}, {}
    for v in (a, b, c):
        for lab in ("beads", "nuclei"):
            g = f"tpId_0_viewSetupId_{v[1]}/{lab}"
            if "dimensions" in store.get_attributes(g + "/interestpoints/loc"):
                pts[(v, lab)] = (store.read_list(g + "/interestpoints/id").ravel(), store.read_list(g + "/interestpoints/loc"))
                corr[(v, lab)] = store.read_correspondences(g)
    ot, ol = no.target_positions(c, ["beads", "nuclei"], [a, b, c], pts, corr, regs)
    assert np.allclose(ot, t) and np.allclose(ol, l)


def test_correspondence_reader_round_trip(tmp_path):
    store = bn5.N5Store(str(tmp_path / "ip.n5"), create=True)
    rows = [(3, (0, 1), "beads", 7), (0, (2, 4), "nuclei", 1), (3, (0, 1), "beads", 9)]
    write_correspondences(store, (0, 0), "beads", rows)
    a = store.get_attributes("tpId_0_viewSetupId_0/beads/correspondences")
    assert a["correspondences"] == "1.0.0" and set(a["idMap"]) == {"0,1,beads", "2,4,nuclei"}
    d = store.dataset_attributes("tpId_0_viewSetupId_0/beads/correspondences/data")
    assert d["dimensions"] == [3, 3] and d["dataType"] == "uint64"
    assert store.read_correspondences("tpId_0_viewSetupId_0/beads") == rows
    write_correspondences(store, (0, 5), "beads", [])
    assert store.dataset_attributes("tpId_0_viewSetupId_5/beads/correspondences/data")["dimensions"] == [0]
    assert store.read_correspondences("tpId_0_viewSetupId_5/beads") == []
    assert store.read_correspondences("tpId_0_viewSetupId_9/beads") == []


# ------------------------------------------------------------------------------------------ viewsToFuse / viewsToUse
def test_views_to_fuse_and_use_at_50_and_25():
    dims = {(0, s): (10, 10, 10) for s in range(5)}
    # boxes in x: v0 [0, 9]; v1 [59, 68]: 50 from a block ending at 9 -> fused; v2 [60, 69]: 51 away -> not fused;
    # v3 [118, 127]: 50 from v1's box -> used; v4 [119, 128]: 51 from v1 -> not used
    regs = {(0, 0): translation((0, 0, 0)), (0, 1): translation((59, 0, 0)), (0, 2): translation((60, 0, 0)),
            (0, 3): translation((118, 0, 0)), (0, 4): translation((119, 0, 0))}
    fuse, use = commands.nonrigid_views_for_block(dims, regs, (-10, 0, 0), (9, 9, 9), sorted(regs))
    assert fuse == [(0, 0), (0, 1)] and use == [(0, 0), (0, 1), (0, 2), (0, 3)]
    assert (fuse, use) == no.views_for_block(dims, regs, (-10, 0, 0), (9, 9, 9), sorted(regs))


# ------------------------------------------------------------------------------------------ the command's checks
@pytest.mark.parametrize("kw, exc, text", [
    (dict(data_type="UINT16"), ValueError, "minIntensity"),
    (dict(data_type="UINT8", min_intensity=0.0), ValueError, "minIntensity"),
    (dict(interest_points=[]), ValueError, "no interest points"),
    (dict(bdv="0,1"), NotImplementedError, "--bdv"),
    (dict(xml_out="out.xml"), NotImplementedError, "-xo"),
    (dict(bounding_box="roi"), NotImplementedError, "-b"),
    (dict(dry_run=True), NotImplementedError, "--dryRun"),
    (dict(shard=(0, 2)), NotImplementedError, "sharding"),
])
def test_command_rejects(kw, exc, text):
    args = dict(xml_path="missing.xml", ctx=None, out_path="out.n5", n5_dataset="fused/s0", interest_points=["beads"])
    args.update(kw)
    with pytest.raises(exc, match=text):
        commands.nonrigid_fusion(**args)


# ------------------------------------------------------------------------------------------ ABI
def test_nonrigid_view_layout_matches_header(tmp_path):
    n = bsgpu.native
    src = tmp_path / "sz.c"
    src.write_text('''#include <stdio.h>
#include <stddef.h>
#include "bsgpu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\\n", sizeof(bs_nonrigid_view), offsetof(bs_nonrigid_view, n_points),
         offsetof(bs_nonrigid_view, pad), offsetof(bs_nonrigid_view, target_world_xyz), offsetof(bs_nonrigid_view, local_xyz));
  return 0; }''')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    C = n.NonrigidViewC
    assert got == [ctypes.sizeof(C), C.n_points.offset, C.pad.offset, C.target_world_xyz.offset, C.local_xyz.offset]
    assert bsgpu.load_library().bs_version() == 107


# ------------------------------------------------------------------------------------------ recovery of a known warp
def warp_scene(seed=11):
    """Two tiles of one smooth field G, each with half of a known smooth warp in opposite directions, registered by
    their translations only; beads at exact correspondences in the overlap.  Returns (G, tiles, block)."""
    rng = np.random.default_rng(seed)
    G = gaussian_filter(rng.normal(0.0, 1.0, (40, 72, 150)), 3.0)
    G = (1000.0 + 4000.0 * G / G.std()).astype(np.float64)

    def psi(w):                                           # the warp at world points (n, 3)
        return np.stack([1.6 * np.sin(2 * np.pi * w[:, 2] / 40.0) * np.cos(2 * np.pi * w[:, 1] / 90.0),
                         1.2 * np.cos(2 * np.pi * w[:, 2] / 40.0), 0.4 * np.sin(2 * np.pi * w[:, 1] / 70.0)], axis=1)

    size = (88, 64, 32)
    tiles = []
    for s, (t, sign) in enumerate((((4.0, 4.0, 4.0), 1.0), ((56.0, 4.0, 4.0), -1.0))):
        zz, yy, xx = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in size[::-1]], indexing="ij")
        w = np.stack([xx.ravel() + t[0], yy.ravel() + t[1], zz.ravel() + t[2]], axis=1)
        w = w + sign * 0.5 * psi(w)
        img = map_coordinates(G, [w[:, 2], w[:, 1], w[:, 0]], order=3, mode="nearest").reshape(size[::-1])
        tiles.append(dict(t=np.asarray(t), sign=sign, img=img.astype(np.float32), M=translation(t)))
    # beads: true world points in the overlap x in [62, 88]; the local position of each in both tiles
    p = np.stack([rng.uniform(62, 88, 300), rng.uniform(8, 64, 300), rng.uniform(6, 32, 300)], axis=1)
    for tl in tiles:
        l = p - tl["t"]
        for _ in range(30):                               # solve l + t + sign psi(l + t) / 2 = p
            l = p - tl["t"] - tl["sign"] * 0.5 * psi(l + tl["t"])
        tl["loc"] = l
    for tl in tiles:                                      # N2: mean of the two registered world positions
        tl["targets"] = 0.5 * ((tiles[0]["loc"] + tiles[0]["t"]) + (tiles[1]["loc"] + tiles[1]["t"]))
        tl["border"], tl["range"] = fo.adjust_blending(tl["M"])
    return G, tiles, ((64, 12, 10), (20, 44, 16))


def recovery_rms(G, nonrigid, affine, block):
    (bx, by, bz), (sx, sy, sz) = block
    truth = G[bz:bz + sz, by:by + sy, bx:bx + sx]
    return float(np.sqrt(np.mean((nonrigid - truth) ** 2)) / np.sqrt(np.mean((affine - truth) ** 2)))


#: RMS(non-rigid - G) / RMS(affine - G) of the oracle on warp_scene's overlap block, computed once on the CPU
RECOVERY_RATIO = 0.4522


def test_oracle_recovers_the_warp_better_than_affine():
    G, tiles, block = warp_scene()
    nr = no.fuse_block([dict(img=t["img"], src_to_world=t["M"], targets=t["targets"], locals=t["loc"],
                             blend_border=t["border"], blend_range=t["range"]) for t in tiles], *block)
    af = fo.fuse_block([fo.View(t["img"], t["M"], t["border"], t["range"]) for t in tiles], *block, fo.AVG_BLEND)
    ratio = recovery_rms(G, nr, af, block)
    assert abs(ratio - RECOVERY_RATIO) < 0.01 * RECOVERY_RATIO, ratio
