"""The evidence behind the default loss detection of the streaming mapper's recovery (DESIGN.md §4.3.2), as an assertion on the CPU oracle: on a
seeded C3-style stream (matching mode 0) the default max_inlier_threshold lies above the registration score inlier_threshold of every normal scan
and below that of every kidnapped scan registered from the mapper's last pose, and a kidnapped scan's verify fraction at its truth reaches the
default min_verify_fraction where the map covers its view."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import capi  # noqa: E402
from loam_livox_b200 import synthetic as S  # noqa: E402
import recovery_oracle as RO  # noqa: E402


def test_default_bound_separates_normal_from_kidnapped_scans():
    cfg = capi.RecoveryCfg()
    capi.lib().ll_mapper_recovery_default(C.byref(cfg))
    out = RO.measure(72, 0, S.SEED + 7300, kidnaps={56, 64, 71}, back=1.0, yaw_deg=-15.0, aside=-2.0)   # the kidnap of tests/test_gpu_recovery.py
    normal = np.array([x[2] for x in out["normal"]])
    kidnapped = np.array([x[2] for x in out["kidnap"]])
    assert normal.size >= 60 and kidnapped.size == 3
    assert all(x[1] == 1 for x in out["normal"])
    assert normal.max() < cfg.max_inlier_threshold < kidnapped.min(), (normal.max(), kidnapped)
    truth = np.array([v[1] for v in out["verify"]])
    assert truth.max() >= cfg.min_verify_fraction, truth
