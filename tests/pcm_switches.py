"""The BS_FFT_* dispatch switches of the PCM passes (csrc/pcm.cu reads them at every launch).

A GPU test that asserts which kernel a pass launches must not inherit a switch from the caller's shell, so each one
clears all of them before setting its own."""

SWITCHES = ("BS_FFT_X_WARP", "BS_FFT_R2C_TMA", "BS_FFT_STATIC", "BS_FFT_YTILE_LOG2", "BS_FFT_ZTILE_LOG2",
            "BS_FFT_X_COL540", "BS_FFT_XY_FUSE", "BS_FFT_XY_KX", "BS_FFT_XY_WINDOW")


def set_switches(monkeypatch, env=None):
    """Clear every switch, then set ``env`` ({name: value})."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        assert k in SWITCHES, k
        monkeypatch.setenv(k, str(v))
