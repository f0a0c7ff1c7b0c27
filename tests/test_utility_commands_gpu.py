"""downsample on the device: the datasets equal, file for decoded file, those of the oracle-backed context for every
type bs_downsample takes, in N5 and Zarr, with levels re-read from the container and kept resident; and the chain
nonrigid-fusion -> downsample gives the chained 2x steps of the fused s0."""
import numpy as np
import pytest

from bsgpu import commands, n5 as bn5
from bsgpu import zarr as bz
from oracle import fusion_oracle as fo
from tests.fake_ctx import FakeContext
from tests.test_nonrigid_gpu import _dataset as _nonrigid_dataset
from tests.test_resave_gpu import _decoded_files
from tests.test_utility_commands_cpu import OUT, STEPS, _storage, _volume, _write_input

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layout", ["n5", "zarr5"])
@pytest.mark.parametrize("dtype", ["uint8", "uint16", "float32"])
@pytest.mark.parametrize("block_scale", [(1, 1, 1), (4, 4, 2)])        # every level re-read / s2 kept resident
def test_device_downsample_equals_fake_context(ctx, tmp_path, layout, dtype, block_scale):
    vol = _volume((203, 151, 37), dtype, seed=11)
    vol[:9, :, :70] = 0                                          # storage blocks that stay unwritten
    files = []
    for name, c in (("dev", ctx), ("fake", FakeContext())):
        root = str(tmp_path / name)
        _write_input(root, layout, vol, (32, 16, 8))
        assert commands.downsample(root, c, "s0", OUT, STEPS, storage=_storage(layout), block_scale=block_scale) == OUT
        files.append(_decoded_files(root))
    assert files[0] == files[1]
    assert sum(k.startswith("s3") for k in files[0]) > 4


@pytest.mark.parametrize("storage, dtype", [("N5", "FLOAT32"), ("ZARR", "UINT16")])
def test_nonrigid_fusion_then_downsample(ctx, tmp_path, storage, dtype):
    xml, _, _ = _nonrigid_dataset(tmp_path)
    out = str(tmp_path / ("fused.n5" if storage == "N5" else "fused.zarr"))
    commands.nonrigid_fusion(xml, ctx, out, "fused/s0", ["beads"], storage=storage, block_size=(32, 32, 16),
                             data_type=dtype, min_intensity=500.0, max_intensity=1600.0)
    commands.downsample(out, ctx, "fused/s0", ["fused/s1", "fused/s2"], "2,2,1; 2,2,2", storage=storage)
    st = bn5.N5Store(out) if storage == "N5" else bz.ZarrStore(out)
    s0 = st.read_volume("fused/s0")
    s1, s2 = st.read_volume("fused/s1"), st.read_volume("fused/s2")
    w1 = fo.downsample2x(s0, (2, 2, 1))
    assert s0.shape == (20, 340, 104) and s1.shape == (20, 170, 52) and s2.shape == (10, 85, 26)
    assert np.array_equal(s1, w1) and np.array_equal(s2, fo.downsample2x(w1, (2, 2, 2)))
    assert s0.any() and not s0[:, 128:192].any() and not s2[:, 32:48].any()     # the slab no view reaches
