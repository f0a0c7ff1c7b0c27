"""The C-ABI library loads on a CPU-only box, exports every symbol include/bsgpu.h declares,
and refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "bsgpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bs_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_all_exported():
    import bsgpu
    lib = bsgpu.load_library()
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/bsgpu.h but not exported"
    assert sorted(bsgpu.native.SYMBOLS) == names


def test_version_and_pure_host_entry_points():
    import bsgpu
    lib = bsgpu.load_library()
    assert lib.bs_version() >= 100
    assert bsgpu.good_fft_size(532, True) == 540
    assert bsgpu.good_fft_size(271) == 288
    p = bsgpu.native.PcmParams()
    lib.bs_pcm_default_params(ctypes.byref(p))
    assert (p.peaks_to_check, p.do_subpixel, p.min_overlap_frac, list(p.extension)) == (5, 1, 0.25, [10, 10, 10])
    f = bsgpu.native.FuseParamsC()
    lib.bs_fuse_default_params(ctypes.byref(f))
    assert (f.fusion_type, f.interpolation, f.out_dtype) == (bsgpu.native.FUSE_AVG_BLEND, 1, bsgpu.native.DTYPE_F32)


def test_struct_layout_matches_header(tmp_path):
    """sizeof/offsetof from the real header (compiled with gcc) == the ctypes mirror."""
    import subprocess
    import bsgpu
    n = bsgpu.native
    src = tmp_path / "sz.c"
    src.write_text('''#include <stdio.h>
#include <stddef.h>
#include "bsgpu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(bs_pcm_params), sizeof(bs_pcm_result), sizeof(bs_view),
         sizeof(bs_fuse_params), offsetof(bs_pcm_result, r), offsetof(bs_pcm_result, pad),
         offsetof(bs_view, blend_border), offsetof(bs_fuse_params, min_intensity));
  return 0; }''')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [ctypes.sizeof(n.PcmParams), ctypes.sizeof(n.PcmResultC), ctypes.sizeof(n.ViewC),
            ctypes.sizeof(n.FuseParamsC), n.PcmResultC.r.offset, n.PcmResultC.pad.offset,
            n.ViewC.blend_border.offset, n.FuseParamsC.min_intensity.offset]
    assert got == want


def test_no_cpu_fallback_without_gpu():
    import torch
    import bsgpu
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(bsgpu.BsError) as e:
        bsgpu.Context(0)
    assert "no CPU fallback" in str(e.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "bigstitcher-spark_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), fn


def test_pcm_switch_list_matches_the_source():
    from tests.pcm_switches import SWITCHES
    src = open(os.path.join(ROOT, "bigstitcher-spark_b200", "csrc", "pcm.cu")).read()
    assert sorted(SWITCHES) == sorted(set(re.findall(r'env_int\("(BS_FFT_\w+)"', src)))
