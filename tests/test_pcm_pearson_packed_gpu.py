"""GPU: worst-case values for the uint16 slab kernel's packed sums.  k_pearson_u16 forms its products with 2-way
16 x 8-bit dot products into uint32 partials that hold 128 of them between folds into uint64.  Values whose bytes
are all at their maximum are what drive those partials to the bound, and rows longer than 8192 elements are where
the kernel has to fold inside a row.  Every sum must match numpy int64 exactly."""
import numpy as np
import pytest

from tests.test_pcm_pearson_gpu import _dev, _np_sums, _random_boxes, _wrap_candidates

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fill", ["max", "high_bytes"])
def test_bench_shape_near_max_exact(ctx, fill):
    """512^3 crops, all 65535 or uniform in [65280, 65535], with the wrap candidates of a near-zero shift"""
    d, P = (512, 512, 512), (540, 540, 540)
    rng = np.random.default_rng(21)
    if fill == "max":
        a = np.full(d, 65535, dtype=np.uint16)
        b = a.copy()
    else:
        a = rng.integers(65280, 65536, d, dtype=np.uint16)
        b = rng.integers(65280, 65536, d, dtype=np.uint16)
    boxes = np.array(_wrap_candidates((3, 537, 2), P, d, int(0.25 * 512 ** 3)), dtype=np.int32)
    assert len(boxes) >= 1
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))


@pytest.mark.parametrize("width", [
    4096,     # one row per warp, 16 chunks per lane: no fold inside the row
    8192,     # 1024 chunks when the box starts on a 16-byte boundary: exactly at the bound
    8195,     # odd pitch: rows start off 16-byte boundaries, up to 1026 chunks, one fold inside the row
    12000,    # one-row slabs, one fold inside the row
    16384,    # the widest crop accepted, up to 2049 chunks: two folds inside the row
])
def test_all_max_long_rows_exact(ctx, width):
    shape = (3, 4, width)
    rng = np.random.default_rng(width)
    a = np.full(shape, 65535, dtype=np.uint16)
    b = a.copy()
    boxes = _random_boxes(rng, shape[::-1], 12)
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))


@pytest.mark.parametrize("fill", ["max", "random"])
def test_single_element_and_full_box_exact(ctx, fill):
    shape = (6, 9, 1030)
    rng = np.random.default_rng(31)
    if fill == "max":
        a = np.full(shape, 65535, dtype=np.uint16)
        b = a.copy()
    else:
        a = rng.integers(0, 65536, shape, dtype=np.uint16)
        b = rng.integers(0, 65536, shape, dtype=np.uint16)
    dz, dy, dx = shape
    boxes = [[0, 0, 0, 0, 0, 0, dx, dy, dz]]                         # the full box
    for p1 in range(8):                                              # one element, every x offset mod 8 on each side
        for p2 in range(8):
            boxes.append([dx - 1 - p1, int(rng.integers(0, dy)), int(rng.integers(0, dz)),
                          p2, int(rng.integers(0, dy)), int(rng.integers(0, dz)), 1, 1, 1])
    boxes = np.array(boxes, dtype=np.int32)
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))
