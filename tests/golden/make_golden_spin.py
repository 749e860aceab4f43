"""Regenerates tests/golden/golden_spin.npz: the oracle's spinning-lidar odometry (tests/spin_mapper_oracle.py: the Velodyne feature node's
less-sharp, less-flat and full clouds remapped onto the mapping node) on a 16-sweep VLP-16 stream in the room along synthetic.trajectory
(mapping_init_accumulate_frames 3), in matching_mode 0 with a window of 400 and of 3 clouds (the latter pops) and in matching_mode 1, plus a
6-sweep HDL-64 track in the open scene.  Rows are laid out as in golden_pieces.npz: status, frame index, feature / map / append counts, ICP
iterations and pose; plus a checksum of every generated sweep, so that a change of the generator is told apart from a change of the mapper.
Run: python tests/golden/make_golden_spin.py"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from loam_livox_b200 import synthetic as S  # noqa: E402
from oracle import oracle as O  # noqa: E402
import spin_mapper_oracle as SMO  # noqa: E402

INIT, THREADS = 3, 4
N_VLP, N_HDL = 16, 6
CASES = [(0, 400), (0, 3), (1, 400)]


def vlp_sweeps(n=N_VLP, seed=S.SEED + 700):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    return [S.make_spinning_scan(16, p, seed=seed + k) for k, p in enumerate(poses)], poses


def hdl_sweeps(n=N_HDL, seed=S.SEED + 800):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    return [S.make_spinning_scan(64, p, seed=seed + k, n_azimuth=1000, scene="open") for k, p in enumerate(poses)], poses


def row(st, L, frame_index, q, t):
    icp = L["res"].icp_iterations if L["res"] is not None and L["res"].registered else 0
    app = (L["appended_corner"], L["appended_surf"]) if st else (0, 0)
    return [st, frame_index, L["n_corner"], L["n_surf"], L["map_corner"], L["map_surf"], app[0], app[1], icp] + [float(x) for x in q] + [float(x) for x in t]


def oracle_mapper(scan_line, mode, window, **params):
    return SMO.SpinMapper(scan_line, params=O.default_params(mapping_init_accumulate_frames=INIT, num_threads=THREADS, **params), threads=THREADS,
                          matching_mode=mode, maximum_history_size=window)


def run(scan_line, mode, window, sweeps):
    om = oracle_mapper(scan_line, mode, window)
    rows = []
    for raw in sweeps:
        st, q, t, L = om.process_sweep(raw)
        rows.append(row(st, L, om.m.frame_index, q, t))
    return np.array(rows, dtype=np.float64)


def build():
    vlp, _ = vlp_sweeps()
    hdl, _ = hdl_sweeps()
    out = {"sweep_crc": np.array([zlib.crc32(np.ascontiguousarray(r).tobytes()) for r in vlp + hdl], dtype=np.uint32)}
    for mode, window in CASES:
        out[f"track_vlp16_m{mode}_w{window}"] = run(16, mode, window, vlp)
    out["track_hdl64_open"] = run(64, 0, 400, hdl)
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "golden_spin.npz"), **build())
    print("written")
