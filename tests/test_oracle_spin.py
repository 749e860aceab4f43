"""The Velodyne front end's oracle (oracle/orc_spin.hpp: the literal reset-order loop and insertion sort) against an independent NumPy
restatement (tests/spin_reference.py: the closed-form flags and a stable sort), bit for bit, on constructed edges."""
import numpy as np
import pytest

import spin_cases as SC
import spin_reference as R
from oracle.spin_oracle import CLOUDS, SpinExtractor

SMALL = sorted(k for k, (sl, raw) in SC.edge_cases().items() if raw.shape[0] <= 7000)


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_numpy_restatement(name, oracle):
    scan_line, raw = SC.edge_cases()[name]
    o = SpinExtractor(scan_line)
    got = o.extract(raw)
    want, info = R.extract(raw, scan_line, voxel_grid=oracle.voxel_grid)
    for k in CLOUDS:
        assert got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    for a, b, k in zip(o.point_info(), info, ("ring", "curvature", "picked", "label")):
        assert np.array_equal(np.asarray(a), np.asarray(b).astype(np.asarray(a).dtype)), k


def test_edges_cover_what_they_claim():
    """The constructed clouds reach the edges they are named for: forward and backward occlusions, the sharp caps, a dropped huge point."""
    cases = SC.edge_cases()
    o = SpinExtractor(16)
    o.extract(cases["sharp_caps_3"][1])
    _, _, _, label = o.point_info()
    assert (label == 2).sum() >= 20 and (label == 1).sum() > 0
    o.extract(cases["nan_inf_near_huge"][1])
    _, curv, _, _ = o.point_info()
    assert np.isinf(curv).any() and not np.isnan(curv).any()
    assert o.counts[0] < cases["nan_inf_near_huge"][1].shape[0]
    o.extract(cases["kept_4"][1])
    assert list(o.counts[1:]) == [0, 0, 0, 0]
