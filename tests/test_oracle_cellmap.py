"""CPU tests of the oracle's cell map and streaming driver (a14 / config C3) -- oracle only, no GPU.

Reference behaviour being pinned: loam_livox/source/cell_map_keyframe.hpp:556-571 (cell index), :716-758 (revisit), :619-672 (append),
loam_livox/source/laser_mapping.hpp:310-324 (FOV test), :471-516 (mode-1 assembly), :1316-1521 (process_new_scan)."""
import numpy as np

from loam_livox_b200 import synthetic as S


def _cell_keys(p, res=1.0):
    box, half = np.float32(res * 0.5), np.float32(res * 0.25)
    return np.round((p[:, :3].astype(np.float32) - half) / box).astype(np.int64)   # np.round is half-to-even; ties do not occur in the data below


def test_cellmap_counts_and_frame_index(oracle):
    rng = np.random.default_rng(1)
    p = np.zeros((5000, 4), np.float32)
    p[:, :3] = rng.uniform(-6, 6, (5000, 3)).astype(np.float32) + np.float32(0.013)
    cm = oracle.CellMap(1.0, 2000)
    assert cm.frame_idx() == 0
    cm.append_cloud(p[:3000])
    assert cm.frame_idx() == 2                       # set_point_cloud bumps once, append_cloud once more (cell_map_keyframe.hpp:578-617)
    cm.append_cloud(p[3000:])
    assert cm.frame_idx() == 3
    assert cm.points() == 5000
    assert cm.cells() == np.unique(_cell_keys(p), axis=0).shape[0]


def test_cellmap_revisit_replaces_stale_cells(oracle):
    cm = oracle.CellMap(1.0, 3)
    a = np.array([[0.3, 0.3, 0.3, 0]], np.float32)
    b = np.array([[5.3, 0.3, 0.3, 0]], np.float32)
    cm.append_cloud(a)                               # frame 0 -> idx 2
    for _ in range(2):
        cm.append_cloud(b)                           # idx 3, 4: cell of a untouched since frame 0
    assert cm.points() == 3
    cm.append_cloud(a)                               # 4 - 0 >= 3: the stale cell is replaced by a fresh one holding only the new point
    assert cm.points() == 3 and cm.cells() == 2
    cm.append_cloud(a)                               # fresh cell, touched last frame: appended
    assert cm.points() == 4


def test_cellmap_assemble_matches_per_cell_voxelgrid(oracle):
    rng = np.random.default_rng(2)
    p = np.zeros((20000, 4), np.float32)
    p[:, :3] = (rng.normal(0, 4, (20000, 3))).astype(np.float32)
    cm = oracle.CellMap(1.0, 2000)
    cm.append_cloud(p)
    q, t = S.quat_from_euler(0.0, 0.0, 0.4), np.array([0.5, -0.2, 0.1])
    out, nfov = cm.assemble(q, t, 6.0, 45.0, 0.2, replace=False)
    # independent numpy restatement of the selection
    keys = _cell_keys(p)
    uk, inv = np.unique(keys, axis=0, return_inverse=True)
    cen = (uk.astype(np.float32) * np.float32(0.5) + np.float32(0.25))
    d = cen - t.astype(np.float32)
    in_r = (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float64) <= 36.0
    R = S.quat_to_mat(q)
    loc = (cen.astype(np.float64) - t) @ R                                  # R^T (c - t)
    ang = np.degrees(np.arccos(np.clip(np.abs(loc[:, 0]) / np.linalg.norm(loc, axis=1), 0, 1))) * (57.3 / (180 / np.pi))
    in_f = (loc[:, 0] >= 0) & (ang < 45.0)
    sel = in_r & in_f
    assert nfov == int(sel.sum())
    order = np.lexsort((uk[:, 0], uk[:, 1], uk[:, 2]))                       # ascending (k, j, i) = (z, y, x)
    chunks = []
    for ci in order:
        if sel[ci]:
            pts = p[inv.ravel() == ci].copy(); pts[:, 3] = 0
            chunks.append(oracle.voxel_grid(pts, 0.2))
    ref = np.concatenate(chunks)
    assert np.array_equal(out, ref)
    # replace = True: a second assembly sees the down-sampled cells and reproduces the same cloud (VoxelGrid of one point per voxel is exact)
    out1, _ = cm.assemble(q, t, 6.0, 45.0, 0.2, replace=True)
    n_after = cm.points()
    out2, _ = cm.assemble(q, t, 6.0, 45.0, 0.2, replace=True)
    assert np.array_equal(out1, ref) and n_after < 20000 and np.array_equal(out2, out1)


import pytest


@pytest.mark.parametrize("mode,window", [(1, 400), (0, 400), (0, 3)])
def test_streaming_mapper_tracks_trajectory(oracle, mode, window):
    """Oracle end to end on a short C3 sequence: poses relative to the first scan within a few centimetres of ground truth, in matching_mode 1
    (cell map) and 0 (history window of the last `window` feature clouds, laser_mapping.hpp:518-531,1439-1478)."""
    poses = S.trajectory(n_scans=9, n_static=4, speed=1.0)
    p = oracle.default_params(mapping_init_accumulate_frames=3, num_threads=4)
    mp = oracle.Mapper(p, threads=4, matching_mode=mode, maximum_history_size=window)
    R0, t0 = poses[0].R(), poses[0].t
    errs = []
    for k, pose in enumerate(poses):
        raw = S.make_scan(24000, pose, seed=S.SEED + k)
        st, q, t = mp.process_scan(raw, 100.0 + 0.1 * k)
        assert st == 1
        t_true = R0.T @ (pose.t - t0)
        errs.append(np.linalg.norm(t - t_true))
        # the registration sees the frame index BEFORE process_new_scan increments it (laser_mapping.hpp:1349-1350): with
        # mapping_init_accumulate_frames = 3, scans 0..3 are inserted unregistered and scan 4 is the first to run the ICP
        if k <= 3:
            assert mp.last["res"] is None or mp.last["res"].registered == 0
        else:
            assert mp.last["res"].registered == 1
    assert mp.frame_index == 9
    assert max(errs) < 0.05, errs
    assert mp.cells_surf.cells() > 100 and mp.cells_corner.cells() > 10
    assert len(mp.his_surf) == min(9, window) and len(mp.his_corner) == min(9, window)
