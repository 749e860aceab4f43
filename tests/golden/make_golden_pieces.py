"""Regenerates tests/golden/golden_pieces.npz: the oracle's piecewise frame (every piece of a sensor frame registered as a scan of its own, the
shipped odom_mode 1; tests/piecewise_oracle.py) on a 6-frame synthetic sequence (24k-point scans, 3 pieces, mapping_init_accumulate_frames 3),
in matching_mode 0 with a window of 400 and of 3 clouds (the latter pops) and in matching_mode 1, plus a 3-head x 2-piece track (Mid-100 style
frames of 3 x 12k points).  Per published piece: status, frame index, feature / map / append counts, ICP iterations and pose; plus a checksum
of the generated scans so that a change of the generator is told apart from a change of the mapper.  Run: python tests/golden/make_golden_pieces.py"""
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
import piecewise_oracle as PO  # noqa: E402

N_FRAMES, N_PTS, INIT, PIECES = 6, 24000, 3, 3
CASES = [(0, 400), (0, 3), (1, 400)]
HEADS_PIECES = 2


def stamps(k, heads=1):
    return [100.0 + 0.1 * k] * heads


def frames():
    poses = S.trajectory(n_scans=N_FRAMES, n_static=2, speed=1.0)
    return [[S.make_scan(N_PTS, p, seed=S.SEED + 500 + k)] for k, p in enumerate(poses)]


def head_frames():
    poses = S.trajectory(n_scans=N_FRAMES, n_static=2, speed=1.0)
    return [S.make_triple_scan(3 * 12000, p, seed=S.SEED + 600 + 3 * k) for k, p in enumerate(poses)]


def row(st, L, frame_index, q, t):
    icp = L["res"].icp_iterations if L["res"] is not None and L["res"].registered else 0
    app = (L["appended_corner"], L["appended_surf"]) if st else (0, 0)
    return [st, frame_index, L["n_corner"], L["n_surf"], L["map_corner"], L["map_surf"], app[0], app[1], icp] + [float(x) for x in q] + [float(x) for x in t]


def run(mode, window, fr, pieces, threads=4):
    om = O.Mapper(O.default_params(mapping_init_accumulate_frames=INIT, num_threads=threads), threads=threads, matching_mode=mode, maximum_history_size=window)
    rows = []
    for k, heads in enumerate(fr):
        published = PO.process_frame(om, heads, stamps(k, len(heads)), pieces, 1)
        base = om.frame_index - len(published)
        for i, (st, q, t, L) in enumerate(published):
            rows.append(row(st, L, base + i + 1, q, t))
    return np.array(rows, dtype=np.float64)


def build():
    fr, hf = frames(), head_frames()
    out = {"scan_crc": np.array([zlib.crc32(np.ascontiguousarray(h).tobytes()) for f in fr + hf for h in f], dtype=np.uint32)}
    for mode, window in CASES:
        out[f"track_m{mode}_w{window}"] = run(mode, window, fr, PIECES)
    out["track_heads3_p2"] = run(0, 400, hf, HEADS_PIECES)
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "golden_pieces.npz"), **build())
    print("written")
