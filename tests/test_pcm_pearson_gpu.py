"""GPU: the Pearson sums of explicit candidate boxes (bs_pcm_debug_pearson, the production Pearson launch) against
numpy int64 sums. Integer input must match exactly; float32 within a relative tolerance.

The uint16 slab kernel is reached with 16-byte aligned bases (any row pitch); a base one element off goes to the
generic kernel, as do uint8 and float32."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _np_sums(a, b, boxes, exact=True):
    """a, b: [z, y, x] arrays; boxes (n, 9) {o1 xyz, o2 xyz, sz xyz} -> (n, 5) sums in z-slabs."""
    out = []
    for o1x, o1y, o1z, o2x, o2y, o2z, sx, sy, sz in np.asarray(boxes).tolist():
        s = np.zeros(5, dtype=np.int64 if exact else np.float64)
        for z in range(0, sz, 16):
            nz = min(16, sz - z)
            pa = a[o1z + z:o1z + z + nz, o1y:o1y + sy, o1x:o1x + sx].astype(np.int64 if exact else np.float64)
            pb = b[o2z + z:o2z + z + nz, o2y:o2y + sy, o2x:o2x + sx].astype(np.int64 if exact else np.float64)
            s += [pa.sum(), pb.sum(), (pa * pa).sum(), (pb * pb).sum(), (pa * pb).sum()]
        out.append(s)
    return np.array(out).reshape(-1, 5)


def _random_boxes(rng, dims_xyz, n):
    """boxes with every x-offset parity on either image, shifts up to +-(d - 1), thin and mid-slab boxes"""
    boxes = []
    for i in range(n):
        b = []
        for d in dims_xyz:
            kind = rng.integers(0, 4)
            if kind == 0:                       # extreme shift: a sliver at opposite ends
                sz = min(int(rng.integers(1, 3)), d)
                o1, o2 = (0, d - sz) if rng.integers(0, 2) else (d - sz, 0)
            elif kind == 1:                     # wrap-candidate geometry: one offset zero
                s = int(rng.integers(-(d - 1), d))
                sz = d - abs(s)
                o1, o2 = (s, 0) if s >= 0 else (0, -s)
            else:                               # arbitrary sub-box on both sides
                sz = int(rng.integers(1, d + 1))
                o1, o2 = int(rng.integers(0, d - sz + 1)), int(rng.integers(0, d - sz + 1))
            b.append((o1, o2, sz))
        boxes.append([b[0][0], b[1][0], b[2][0], b[0][1], b[1][1], b[2][1], b[0][2], b[1][2], b[2][2]])
    # every (o1 x, o2 x) parity mod 8 at full width-ish
    for p1 in range(8):
        for p2 in range(0, 8, 3):
            sx = dims_xyz[0] - max(p1, p2)
            boxes.append([p1, 0, 0, p2, 0, 0, sx, dims_xyz[1], dims_xyz[2]])
    return np.array(boxes, dtype=np.int32)


def _dev(x):
    import torch
    t = torch.from_numpy(x.view(np.int16) if x.dtype == np.uint16 else x).cuda()
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("shape", [
    (37, 45, 64),     # 128 B rows
    (37, 45, 70),     # even pitch, not a multiple of 16 B: slabs start mid-chunk
    (29, 33, 71),     # odd pitch, element count not a multiple of 8 (last chunk of the image)
    (3, 5, 1000),     # few rows, wide rows
    (40, 1, 9),       # one row per plane
    (4, 6, 700),      # rows wider than 512: 23-row slabs, slab starts not 16-byte aligned
    (2, 7, 3001),     # 5-row slabs of an odd pitch
])
def test_u16_sums_exact(ctx, shape):
    rng = np.random.default_rng(sum(shape))
    a = rng.integers(0, 65536, shape, dtype=np.uint16)
    b = rng.integers(0, 65536, shape, dtype=np.uint16)
    boxes = _random_boxes(rng, shape[::-1], 40)
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    want = _np_sums(a, b, boxes)
    assert np.array_equal(got.astype(np.int64), want)


def test_u16_max_candidates_exact(ctx):
    shape = (21, 30, 50)
    rng = np.random.default_rng(3)
    a = rng.integers(0, 65536, shape, dtype=np.uint16)
    b = rng.integers(0, 65536, shape, dtype=np.uint16)
    boxes = _random_boxes(rng, shape[::-1], 256 - 24)
    assert len(boxes) == 256
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))


def test_u16_unaligned_base_generic_path(ctx):
    """bases one element past a 16-byte boundary (and an odd pitch) take the generic kernel: same exact sums"""
    import torch
    shape = (19, 23, 41)
    rng = np.random.default_rng(4)
    a = rng.integers(0, 65536, shape, dtype=np.uint16)
    b = rng.integers(0, 65536, shape, dtype=np.uint16)
    n = a.size
    fa = torch.zeros(n + 8, dtype=torch.int16, device="cuda")
    fb = torch.zeros(n + 8, dtype=torch.int16, device="cuda")
    fa[1:n + 1] = torch.from_numpy(a.view(np.int16).ravel()).cuda()
    fb[1:n + 1] = torch.from_numpy(b.view(np.int16).ravel()).cuda()
    ta, tb = fa[1:n + 1].view(shape), fb[1:n + 1].view(shape)
    torch.cuda.synchronize()
    assert ta.data_ptr() % 16 == 2
    boxes = _random_boxes(rng, shape[::-1], 30)
    got = ctx.pcm_debug_pearson(ta, tb, boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))


def test_u8_exact_and_f32_close(ctx):
    shape = (17, 26, 39)
    rng = np.random.default_rng(5)
    boxes = _random_boxes(rng, shape[::-1], 25)
    a8 = rng.integers(0, 256, shape, dtype=np.uint8)
    b8 = rng.integers(0, 256, shape, dtype=np.uint8)
    got = ctx.pcm_debug_pearson(_dev(a8), _dev(b8), boxes)
    assert np.array_equal(got.astype(np.int64), _np_sums(a8, b8, boxes))
    af = rng.random(shape, dtype=np.float32) * 1000
    bf = rng.random(shape, dtype=np.float32) * 1000
    got = ctx.pcm_debug_pearson(_dev(af), _dev(bf), boxes)
    want = _np_sums(af, bf, boxes, exact=False)
    assert np.allclose(got, want, rtol=1e-9, atol=1e-6)


def _wrap_candidates(loc, P, d, min_px):
    """the 2^3 wrap candidates of a PCM peak that overlap by at least min_px voxels (pcm_expand_candidate)"""
    boxes = []
    for i in range(8):
        box, ok, npx = [0] * 9, True, 1
        for ax in range(3):
            s = loc[ax]
            if ((i >> ax) & 1) == 0:
                s = s + P[ax] if s < 0 else s - P[ax]
            n = d[ax]
            if abs(s) >= n:
                ok = False
                continue
            box[ax], box[3 + ax], box[6 + ax] = (s, 0, n - s) if s >= 0 else (0, -s, n + s)
            npx *= box[6 + ax]
        if ok and npx >= min_px:
            boxes.append(box)
    return boxes


def test_bench_shape_wrap_candidates_exact(ctx):
    """512^3 uint16 crops with the wrap candidates of one true peak near shift 0 and 4 noise peaks at seeded PCM
    locations (padded size 540, min overlap 0.25), as the benchmark produces them."""
    d, P = (512, 512, 512), (540, 540, 540)
    rng = np.random.default_rng(11)
    a = rng.integers(0, 65536, d, dtype=np.uint16)
    b = rng.integers(0, 65536, d, dtype=np.uint16)
    peaks = [(3, 537, 2)] + [tuple(int(v) for v in rng.integers(0, 540, 3)) for _ in range(4)]
    boxes = [bx for p in peaks for bx in _wrap_candidates(p, P, d, int(0.25 * 512 ** 3))]
    boxes = np.array(boxes, dtype=np.int32)
    assert len(boxes) >= 5
    got = ctx.pcm_debug_pearson(_dev(a), _dev(b), boxes, dtype=0)
    assert np.array_equal(got.astype(np.int64), _np_sums(a, b, boxes))
