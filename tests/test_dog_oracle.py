"""Known-answer tests of the DoG oracle (next row 8f-4)."""
import numpy as np

from oracle import dog_oracle as do


def _beads(shape=(40, 48, 56), centers=((20.3, 24.6, 17.2), (40.0, 10.0, 30.5), (8.7, 40.1, 8.0)), amp=3000.0, s=1.8, bg=200.0, seed=0):
    z, y, x = np.mgrid[0:shape[0], 0:shape[1], 0:shape[2]].astype(np.float64)
    img = np.full(shape, bg)
    for (cx, cy, cz) in centers:
        img += amp * np.exp(-((x - cx) ** 2 + (y - cy) ** 2 + (z - cz) ** 2) / (2 * s * s))
    img += np.random.default_rng(seed).normal(0, 5, shape)
    return np.clip(np.rint(img), 0, 65535).astype(np.uint16), centers


def test_sigmas_and_kernel():
    sa, sb, kinv = do.compute_sigmas(1.8)
    assert abs(sa - np.sqrt(1.8 ** 2 - 0.25)) < 1e-12 and abs(sb - np.sqrt((1.8 * 2 ** 0.25) ** 2 - 0.25)) < 1e-12
    assert abs(kinv - 1 / (2 ** 0.25 - 1)) < 1e-12
    k = do.gauss_kernel(sa)
    assert len(k) == 2 * (max(2, int(3 * sa + 0.5) + 1) - 1) + 1 and abs(k.sum() - 1) < 1e-6 and np.all(k == k[::-1])


def test_beads_are_found_with_subpixel_accuracy():
    img, centers = _beads()
    pts = do.detect(img, (0, 0, 0), img.shape[::-1], sigma=1.8, threshold=0.004, max_intensity=4000.0)
    assert len(pts) == len(centers)
    for c in centers:
        d = min(np.linalg.norm(np.subtract(p[0], c)) for p in pts)
        assert d < 0.15
    assert all(p[3] for p in pts) and all(p[1] > 0.004 for p in pts)
    # dark blobs are minima
    inv = (4000 - img.astype(np.int64)).clip(0).astype(np.uint16)
    assert len(do.detect(inv, (0, 0, 0), img.shape[::-1], threshold=0.004, max_intensity=4000.0, find_max=False, find_min=True)) == len(centers)


def test_block_grid_invariance():
    """A detection belongs to the block that contains its voxel: the union over a block grid == one whole-image call."""
    img, _ = _beads(seed=3)
    dims = img.shape[::-1]
    whole = do.detect(img, (0, 0, 0), dims, threshold=0.004, max_intensity=4000.0)
    parts = []
    for x0 in (0, 28):
        for y0 in (0, 24):
            parts += do.detect(img, (x0, y0, 0), (28, 24, dims[2]), threshold=0.004, max_intensity=4000.0)
    parts.sort(key=lambda p: (p[2][2], p[2][1], p[2][0]))
    assert [p[2] for p in parts] == [p[2] for p in whole]
    assert np.allclose([p[0] for p in parts], [p[0] for p in whole])


def _mirror_double_index(i, n):
    """Views.extendMirrorDouble, the device's mirror_double: ... c b a | a b c ... with period 2 n."""
    i = np.mod(i, 2 * n)
    return np.where(i < n, i, 2 * n - 1 - i)


def test_symmetric_pad_is_mirror_double_when_the_pad_exceeds_every_axis():
    """dog_reference extends the image with np.pad(mode='symmetric'); that equals mirror_double in N-D even when every
    axis folds over several periods at once."""
    img = np.arange(2 * 3 * 5, dtype=np.float64).reshape(2, 3, 5) ** 1.5
    widths = ((9, 11), (7, 8), (13, 6))
    got = np.pad(img, widths, mode="symmetric")
    idx = [_mirror_double_index(np.arange(-lo, n + hi), n) for (lo, hi), n in zip(widths, img.shape)]
    assert np.array_equal(got, img[np.ix_(*idx)])
    one = np.array([[[7.0]]])
    assert np.array_equal(np.pad(one, 65, mode="symmetric"), np.full((131, 131, 131), 7.0))


def test_dog_reference_agrees_with_the_float32_oracle():
    """The float64 DoG box equals the float32 scipy pipeline within float32 rounding, on an interval touching the near
    faces, an interior one, and a volume smaller than the kernel halo."""
    img, _ = _beads(shape=(20, 24, 28))
    tiny = np.random.default_rng(1).integers(0, 4000, (2, 3, 5)).astype(np.uint16)
    for vol, mn, sz, sigma in [(img, (0, 0, 0), (12, 10, 9), 1.8), (img, (9, 8, 6), (11, 9, 7), 3.5), (tiny, (0, 0, 0), (5, 3, 2), 4.0)]:
        dog, ga, gb = do.dog_reference(vol, mn, sz, sigma, 100.0, 4000.0)
        assert dog.shape == tuple(int(v) + 2 for v in sz[::-1])
        p = 80
        f32 = do.dog_volume(np.pad(vol, p, mode="symmetric"), sigma, 100.0, 4000.0)
        (x0, y0, z0), (nx, ny, nz) = mn, sz
        box = f32[p + z0 - 1:p + z0 + nz + 1, p + y0 - 1:p + y0 + ny + 1, p + x0 - 1:p + x0 + nx + 1]
        sa, sb, kinv = do.compute_sigmas(sigma)
        rb = len(do.gauss_kernel(sb)) // 2
        # float32 accumulation in scipy's passes: the same worst-case form as the device bar
        assert np.all(np.abs(box - dog) <= 3 * 2.0 ** -24 * kinv * (2 * rb + 3) * (ga + gb)), sigma
        assert np.abs(dog).max() > 1e-4


def test_extrema_on_the_oracle_box_is_detect():
    img, _ = _beads(seed=2)
    mn, sz = (6, 5, 4), (30, 28, 26)
    ext = np.pad(img, 65, mode="symmetric")
    dog = do.dog_volume(ext, 1.8, 0.0, 4000.0)[64:-64, 64:-64, 64:-64]
    box = dog[mn[2]:mn[2] + sz[2] + 2, mn[1]:mn[1] + sz[1] + 2, mn[0]:mn[0] + sz[0] + 2]
    for fmax, fmin, loc in [(True, False, True), (False, True, True), (True, True, False)]:
        want = do.detect(img, mn, sz, threshold=0.002, max_intensity=4000.0, find_max=fmax, find_min=fmin, localization=loc)
        got = do.extrema(box, mn, threshold=0.002, find_max=fmax, find_min=fmin, localization=loc)
        assert got == want and len(got) >= 1
