"""CPU pins of the oracle's spinning-lidar odometry (tests/spin_mapper_oracle.py, the reference's remapped Velodyne pipeline): its track
against tests/golden/golden_spin.npz, what it feeds the registration (the mapping node's VoxelGrids of the less-sharp and less-flat clouds,
max_t from the full cloud), and its track against the generator's truth -- no GPU."""
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from loam_livox_b200 import synthetic as S  # noqa: E402
import make_golden_spin as G  # noqa: E402
import spin_mapper_oracle as SMO  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "golden_spin.npz")


def test_sweeps_are_the_golden_ones():
    vlp, _ = G.vlp_sweeps()
    hdl, _ = G.hdl_sweeps()
    crc = np.array([zlib.crc32(np.ascontiguousarray(r).tobytes()) for r in vlp + hdl], dtype=np.uint32)
    assert np.array_equal(np.load(GOLD)["sweep_crc"], crc)


@pytest.mark.parametrize("name", [f"track_vlp16_m{m}_w{w}" for m, w in G.CASES] + ["track_hdl64_open"])
def test_oracle_spin_track_reproduces_the_golden_file(oracle, name):
    """Counts and ICP iterations exactly, pose to 1e-9."""
    gold = np.load(GOLD)[name]
    if name == "track_hdl64_open":
        got = G.run(64, 0, 400, G.hdl_sweeps()[0])
    else:
        mode, window = (int(x[1:]) for x in name.split("_")[2:])
        got = G.run(16, mode, window, G.vlp_sweeps()[0])
    assert got.shape == gold.shape
    assert np.array_equal(got[:, :9], gold[:, :9])
    assert np.max(np.abs(got[:, 9:] - gold[:, 9:])) < 1e-9


def test_registration_is_fed_the_remapped_clouds(oracle):
    """corners = VG(less sharp, line leaf), surfaces = VG(less flat, plane leaf), max_t = the largest full-cloud intensity, -10000 when the
    full cloud is empty; no extractor-side VoxelGrid; the frame index counts sweeps."""
    om = G.oracle_mapper(16, 0, 400)
    sweeps, _ = G.vlp_sweeps(4)
    empty = np.full((50, 4), np.nan, np.float32)
    for k, raw in enumerate(sweeps[:2] + [empty] + sweeps[2:]):
        st, q, t, L = om.process_sweep(raw)
        c = om.clouds
        assert L["n_corner"] == oracle.voxel_grid(c["less_sharp"], 0.1).shape[0]
        assert L["n_surf"] == oracle.voxel_grid(c["less_flat"], 0.4).shape[0]
        want = float(max(np.float32(-10000.0), c["full"][:, 3].max())) if c["full"].shape[0] else -10000.0
        assert om.m.last_time_stamp == want
        assert om.m.frame_index == k + 1
    assert om.m.frame_index == 5


def test_oracle_spin_track_stays_near_the_truth(oracle):
    """The VLP-16 room track against the generator's poses, both taken relative to the first sweep.  Measured on this stream: 0.060 m and
    0.049 degrees at most (the first registrations start after mapping_init_accumulate_frames, so the track lags by the motion before them);
    the bound is 0.08 m and 0.2 degrees."""
    gold = np.load(GOLD)["track_vlp16_m0_w400"]
    _, poses = G.vlp_sweeps()
    p0 = poses[0]
    R0 = S.quat_to_mat(p0.q)
    for row, p in zip(gold, poses):
        t_true = R0.T @ (p.t - p0.t)
        q_true = S.quat_mul(np.array([p0.q[0], -p0.q[1], -p0.q[2], -p0.q[3]]), p.q)
        assert np.linalg.norm(row[13:16] - t_true) < 0.08
        assert np.degrees(S.quat_angle(row[9:13], q_true)) < 0.2
