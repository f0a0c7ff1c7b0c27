"""Registration across timepoints on the device: the planted time-lapse of test_timeseries_cpu matched with the device
descriptors (rows identical to the oracle-backed context's) and solved with the device relaxation, and a longer
ALL_TO_ALL_WITH_RANGE run that must not link timepoints beyond the range."""
import numpy as np
import pytest

from bsgpu import commands
from tests.test_match_cpu import MatchFakeContext, read_rows
from tests.test_timeseries_cpu import RUN, P, check_drift, check_rows, match_and_solve, timeseries_scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rtp", ["ALL_TO_ALL", "TO_REFERENCE_TIMEPOINT"])
def test_device_rows_equal_the_oracle_rows_and_the_drift_is_recovered(ctx, tmp_path, rtp):
    (tmp_path / "gpu").mkdir()
    (tmp_path / "fake").mkdir()
    _, truth, drift = timeseries_scene(tmp_path / "gpu")
    timeseries_scene(tmp_path / "fake")
    views = sorted(truth)
    if rtp == "TO_REFERENCE_TIMEPOINT":
        res = match_and_solve(tmp_path / "gpu", ctx, ctx)
        assert res["stats"]["unconnected_views"] == [] and res["stats"]["iterations"] > 20
        check_drift(res["models"], drift, truth, 1)
    else:
        commands.match_interestpoints(str(tmp_path / "gpu" / "dataset.xml"), ctx, ["beads"], registration_tp=rtp, **RUN)
    fake = commands.match_interestpoints(str(tmp_path / "fake" / "dataset.xml"), MatchFakeContext(), ["beads"],
                                         registration_tp=rtp, reference_tp=1, **RUN)
    rows = read_rows(tmp_path / "gpu", views)
    assert rows == read_rows(tmp_path / "fake", views)
    _, cross = check_rows(tmp_path / "gpu", truth, fake)
    assert cross == sum(a[0] != b[0] for a, _, b, _ in fake) > 0


def test_all_to_all_with_range_links_only_timepoints_within_the_range(ctx, tmp_path):
    xml, truth, _ = timeseries_scene(tmp_path, timepoints=4, tile=(400, 300, 80), keep=0.5, seed=11)
    res = commands.match_interestpoints(xml, ctx, ["beads"], registration_tp="ALL_TO_ALL_WITH_RANGE", range_tp=1, **RUN)
    want = [P(a, b) for i, a in enumerate((0, 1, 10, 11, 20, 21, 30, 31))
            for b in (0, 1, 10, 11, 20, 21, 30, 31)[i + 1:] if abs(a // 10 - b // 10) <= 1]
    assert [(a, b) for a, _, b, _ in res] == want and len(want) == 16
    rows, cross = check_rows(tmp_path, truth, res)
    assert cross == 12
    gaps = {abs(v[0] - pv[0]) for v in rows for _, pv, _, _ in rows[v]}
    assert gaps == {0, 1}
    assert all(len(rows[v]) > 0 for v in rows) and np.all([len(p) > 0 for p in res.values()])
