"""detect-interestpoints host logic and oracle pins that need no GPU: ImageJ kernel shape, the median oracle, the
level choice and point transform, block faces, the params string, <ViewInterestPoints> and 2-D N5 lists."""
import numpy as np
import pytest

from oracle import ip_oracle as io


def test_imagej_footprint_point_counts():
    # rows |dy| = 0..r with half widths floor(sqrt(r*r + 1 - dy^2 + 1e-10))
    assert io.imagej_footprint(1).sum() == 9 and io.imagej_footprint(1).all()
    assert io.imagej_footprint(2).sum() == 5 + 2 * (5 + 3) == 21
    assert io.imagej_footprint(3).sum() == 7 + 2 * (7 + 5 + 3) == 37
    # r = 10: half widths 10 10 9 9 9 8 8 7 6 4 1
    assert io.imagej_footprint(10).sum() == 21 + 2 * (21 + 19 + 19 + 19 + 17 + 17 + 15 + 13 + 9 + 3) == 325
    for r in range(1, 33):
        fp = io.imagej_footprint(r)
        assert fp.shape == (2 * r + 1, 2 * r + 1) and fp.sum() % 2 == 1 and np.array_equal(fp, fp[::-1]) \
            and np.array_equal(fp, fp[:, ::-1])


def _brute_median_divide(sl, r):
    fp = io.imagej_footprint(r)
    k = fp.shape[0] // 2
    ext = np.pad(sl.astype(np.float32), k, mode="symmetric")     # mirror-double, also wider than the slice
    out = np.zeros(sl.shape, np.float32)
    for y in range(sl.shape[0]):
        for x in range(sl.shape[1]):
            vals = np.sort(ext[y:y + 2 * k + 1, x:x + 2 * k + 1][fp])
            m = vals[(len(vals) - 1) // 2]
            out[y, x] = np.float32(sl[y, x]) / m if m > 0 else 0.0
    return out


@pytest.mark.parametrize("shape,r", [((6, 7), 1), ((9, 5), 2), ((3, 4), 5), ((1, 2), 3), ((2, 1), 10)])
def test_median_oracle_equals_brute_force_sort(shape, r):
    rng = np.random.default_rng(r)
    sl = rng.normal(1.0, 1.0, shape).astype(np.float32)
    sl[0, 0] = 0.0
    got = io.median_divide(sl[None], r)[0]
    assert np.array_equal(got.view(np.uint32), _brute_median_divide(sl, r).view(np.uint32))


def test_downsample_float_oracle_known_answer():
    v = np.arange(2 * 3 * 5, dtype=np.uint16).reshape(2, 3, 5)
    out = io.downsample_float(v, (2, 1, 2))
    assert out.shape == (1, 3, 2) and out.dtype == np.float32
    assert out[0, 0, 0] == np.float32((0 + 1 + 15 + 16) / 4)
    assert np.array_equal(io.downsample_float(v, (1, 1, 1)), v.astype(np.float32))


def test_interestpoint_level_rule():
    from bsgpu import commands
    lv = [(1, 1, 1), (2, 2, 1), (4, 4, 2), (8, 8, 4)]
    assert commands.interestpoint_level(lv, (2, 2, 1)) == (1, (1, 1, 1))
    assert commands.interestpoint_level(lv, (4, 4, 1)) == (1, (2, 2, 1))
    assert commands.interestpoint_level(lv, (4, 4, 2)) == (2, (1, 1, 1))
    assert commands.interestpoint_level(lv, (16, 16, 1)) == (1, (8, 8, 1))
    assert commands.interestpoint_level(lv, (1, 1, 1)) == (0, (1, 1, 1))
    # non-power-of-two levels are skipped even when they fit; the LAST fitting level wins
    assert commands.interestpoint_level([(1, 1, 1), (3, 3, 1), (2, 2, 1), (6, 6, 1)], (8, 8, 1)) == (2, (4, 4, 1))
    assert commands.interestpoint_level([(1, 1, 1), (1.9, 2.1, 1.0)], (2, 2, 1)) == (1, (1, 1, 1))   # Math.round


def test_interestpoint_transform_hand_example():
    from bsgpu import commands, zarr
    T = commands.interestpoint_transform(zarr.mipmap_transform_default((2, 2, 1)), (2, 2, 1))
    assert np.allclose(T, [[4, 0, 0, 0.5], [0, 4, 0, 0.5], [0, 0, 1, 0]])
    p = T[:, :3] @ np.array([10.0, 20.0, 3.0]) + T[:, 3]
    assert np.allclose(p, (40.5, 80.5, 3.0))
    # the comment's example at J/SparkInterestPointDetection.java:1073-1080
    T = commands.interestpoint_transform([[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 2, 0.5]], (4, 4, 2))
    assert np.allclose(T, [[8, 0, 0, 0.5], [0, 8, 0, 0.5], [0, 0, 4, 0.5]])
    assert np.allclose(io.level_transform([[2, 0, 0, 0.5], [0, 2, 0, 0.5], [0, 0, 2, 0.5]], (4, 4, 2)), T)


@pytest.mark.parametrize("dims,block", [((20, 17, 9), (8, 5, 4)), ((5, 3, 2), (2, 2, 1)), ((2, 9, 9), (4, 4, 4)),
                                        ((33, 10, 7), (512, 512, 128))])
def test_interestpoint_blocks_cover_the_interior_exactly_once(dims, block):
    from bsgpu import commands
    cnt = np.zeros(dims[::-1], int)
    for mn, sz in commands.interestpoint_blocks(dims, block):
        cnt[mn[2]:mn[2] + sz[2], mn[1]:mn[1] + sz[1], mn[0]:mn[0] + sz[0]] += 1
    want = np.zeros(dims[::-1], int)
    want[1:-1, 1:-1, 1:-1] = 1
    assert np.array_equal(cnt, want)


def test_params_string_and_java_doubles():
    from bsgpu import commands
    assert commands.interestpoint_params(1.8, 0.008, False, False, True, 2, 1, 0.0, 2048.0) == (
        "DOG (Spark) s=1.8 t=0.008 overlappingOnly=false min=false max=true downsampleXY=2 downsampleZ=1 "
        "minIntensity=0.0 maxIntensity=2048.0")
    jd = commands.java_double
    assert [jd(v) for v in (0.0, 1.0, 1e-4, 2048.0, 1e7, 1.5e-5, 123456.789, 0.001, -2.5e8, 1e21, 9999999.0)] == [
        "0.0", "1.0", "1.0E-4", "2048.0", "1.0E7", "1.5E-5", "123456.789", "0.001", "-2.5E8", "1.0E21", "9999999.0"]
    assert commands.interestpoint_params(2, 1e-4, True, True, True, 4, 2, 100, 65535).endswith(
        "t=1.0E-4 overlappingOnly=true min=true max=true downsampleXY=4 downsampleZ=2 minIntensity=100.0 "
        "maxIntensity=65535.0")


def test_view_interest_points_round_trip(tmp_path):
    from bsgpu import spimdata
    xml = spimdata.write_dataset_xml(str(tmp_path / "d.xml"), "d.n5", [
        dict(setup=s, size_xyz=(8, 8, 8), tile=s, translation_xyz=(0, 0, 0)) for s in range(2)])
    d = spimdata.SpimData2.load(xml)
    d.set_interest_points("beads", "p1", {(0, 0): "tpId_0_viewSetupId_0/beads", (0, 1): "tpId_0_viewSetupId_1/beads"})
    d.set_interest_points("nuclei", "p2", {(0, 1): "tpId_0_viewSetupId_1/nuclei"})
    d.save(xml)
    d = spimdata.SpimData2.load(xml)
    d.set_interest_points("beads", "p3", {(0, 0): "tpId_0_viewSetupId_0/beads"})      # replace one label of one view
    d.save(xml)
    ips = spimdata.SpimData2.load(xml).interest_points()
    assert ips[(0, 0)] == {"beads": dict(params="p3", path="tpId_0_viewSetupId_0/beads")}
    assert ips[(0, 1)] == {"beads": dict(params="p1", path="tpId_0_viewSetupId_1/beads"),
                           "nuclei": dict(params="p2", path="tpId_0_viewSetupId_1/nuclei")}
    f = spimdata.SpimData2.load(xml).root.find("ViewInterestPoints").findall("ViewInterestPointsFile")
    assert [(e.get("timepoint"), e.get("setup"), e.get("label")) for e in f] == [
        ("0", "0", "beads"), ("0", "1", "beads"), ("0", "1", "nuclei")]


def test_n5_lists_uint64_float64_round_trip(tmp_path):
    from bsgpu import n5 as bn5
    st = bn5.N5Store(str(tmp_path / "ip.n5"), create=True)
    ids = np.arange(7, dtype=np.uint64).reshape(-1, 1) + np.uint64(2 ** 40)
    loc = np.random.default_rng(0).normal(size=(7, 3))
    st.write_list("g/id", ids, 3, "zstd")
    st.write_list("g/loc", loc, 3, "zstd")
    a = st.dataset_attributes("g/loc")
    assert a["dimensions"] == [3, 7] and a["blockSize"] == [3, 3] and a["dataType"] == "float64"
    assert st.dataset_attributes("g/id")["dataType"] == "uint64"
    assert np.array_equal(st.read_list("g/id"), ids) and np.array_equal(st.read_list("g/loc"), loc)
    st.write_list("g/empty", np.zeros((0, 1), np.float32), 3, "zstd")
    assert st.dataset_attributes("g/empty")["dimensions"] == [0] and st.read_list("g/empty").size == 0


def test_unbuilt_flags_raise():
    from bsgpu import commands
    for flag in ("overlapping_only", "only_compare_overlap_tiles", "max_spots_per_overlap"):
        with pytest.raises(NotImplementedError):
            commands.detect_interestpoints("missing.xml", None, "beads", 1.8, 0.008, 0.0, 255.0, **{flag: True})
