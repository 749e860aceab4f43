"""CPU pins of the piecewise frame (laser_feature_extractor.hpp:305-389 publishing every piece, laser_mapping.hpp:1316-1521 registering each):
the slice identity the device front end rests on, the oracle's piecewise track against tests/golden/golden_pieces.npz, and odom_mode 0 -- no GPU."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import piecewise_oracle as PO  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "golden_pieces.npz")


def few_petal_scan(oracle, petals, n=24000, seed=S.SEED):
    """A prefix of a synthetic rosette frame cut so that the extractor keeps exactly `petals` petals."""
    raw = S.make_scan(n, seed=seed)
    ex = oracle.Extractor()
    for m in range(n // 40, n, n // 200):
        if ex.extract(raw[:m], 100.0) == petals:
            return raw[:m].copy()
    raise AssertionError(f"no prefix with {petals} petals")


def inside_range(n, start, end):
    """ex_flags_kernel's / get_features's range test (livox_feature_extractor.hpp:230-236) restated in float32: first and last index kept."""
    fi = np.arange(n, dtype=np.float32)
    keep = ~((fi > np.float32(end) * np.float32(n)) | (fi < np.float32(start) * np.float32(n)))
    idx = np.flatnonzero(keep)
    return (int(idx[0]), int(idx[-1])) if idx.size else (0, -1)


def check_slice_identity(oracle, raw, pieces):
    ex = oracle.Extractor()
    ex.extract(raw, 100.0)
    whole = ex.get_features(0.0, 1.0)
    ts = ex.point_info()["time_stamp"]
    assert np.all(np.diff(ts) > 0)   # the time stamp names the point: the prefix count at index i is the number of earlier time stamps
    start, end = ex.piece_bounds(pieces)
    for i in range(pieces):
        lo, hi = inside_range(raw.shape[0], start[i], end[i])
        piece = ex.get_features(start[i], end[i])
        for cls, (w, p) in enumerate(zip(whole, piece)):
            a = np.searchsorted(w[:, 3], ts[lo], "left") if lo <= hi else 0
            b = np.searchsorted(w[:, 3], ts[hi], "right") if lo <= hi else 0
            assert np.array_equal(w[a:b], p, equal_nan=True), (pieces, i, cls)
    return start, end


@pytest.mark.parametrize("pieces", [1, 2, 3, 5, 16])
def test_pieces_are_slices_of_the_whole_compaction(oracle, pieces):
    """get_features(start_i, end_i) == the slice of get_features(0, 1) between the prefix counts at the first and last index inside the bounds,
    for the corner, surface and full clouds: the invariant the device front end extracts once per head for."""
    for seed in (S.SEED, S.SEED + 7):
        check_slice_identity(oracle, S.make_scan(24000, seed=seed), pieces)


@pytest.mark.parametrize("petals", [6, 7, 8])
def test_pieces_are_slices_when_they_overlap(oracle, petals):
    """Fewer petals than pieces: the bounds clamp (piece_bounds with end_scans < start_scans) and pieces overlap; still slices."""
    raw = few_petal_scan(oracle, petals)
    start, end = check_slice_identity(oracle, raw, 16)
    assert len(set(zip(start.tolist(), end.tolist()))) < 16   # some pieces repeat


@pytest.mark.parametrize("name", ["track_m0_w400", "track_m0_w3", "track_m1_w400", "track_heads3_p2"])
def test_oracle_piecewise_track_reproduces_the_golden_file(oracle, name):
    """The piecewise track of make_golden_pieces.py: counts and ICP iterations exactly, pose to 1e-9."""
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_pieces as G
    gold = np.load(GOLD)
    fr, hf = G.frames(), G.head_frames()
    import zlib
    assert np.array_equal(gold["scan_crc"], np.array([zlib.crc32(np.ascontiguousarray(h).tobytes()) for f in fr + hf for h in f], dtype=np.uint32))
    if name == "track_heads3_p2":
        got = G.run(0, 400, hf, G.HEADS_PIECES)
    else:
        mode, window = int(name[7]), int(name.split("_w")[1])
        got = G.run(mode, window, fr, G.PIECES)
    want = gold[name]
    assert got.shape == want.shape
    assert np.array_equal(got[:, :9], want[:, :9])
    assert np.abs(got[:, 9:] - want[:, 9:]).max() < 1e-9


def test_odom_mode_0_publishes_piece_0_only(oracle):
    """odom_mode 0: one registration per frame, on piece 0's clouds as a staged extractor flow gives them (extract, piece_bounds,
    get_features(start_0, end_0), the two VoxelGrids per class)."""
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=1, num_threads=4), threads=4)
    ex = oracle.Extractor()
    poses = S.trajectory(n_scans=4, n_static=2, speed=1.0)
    for k, pose in enumerate(poses):
        raw = S.make_scan(24000, pose, seed=S.SEED + 40 + k)
        out = PO.process_frame(om, [raw], [100.0 + 0.1 * k], pieces=3, odom_mode=0)
        assert len(out) == 1 and om.frame_index == k + 1
        ex.extract(raw, 100.0 + 0.1 * k)
        start, end = ex.piece_bounds(3)
        c, s, _ = ex.get_features(start[0], end[0])
        c = oracle.voxel_grid(oracle.voxel_grid(c, 0.1), 0.1)
        s = oracle.voxel_grid(oracle.voxel_grid(s, 0.2), 0.4)
        assert (out[0][3]["n_corner"], out[0][3]["n_surf"]) == (c.shape[0], s.shape[0])
    assert om.last["res"] is not None and om.last["res"].registered == 1


def test_no_live_head_publishes_nothing(oracle):
    """Every head with <= 5 petals: nothing is published and the mapper is untouched (laser_feature_extractor.hpp:287)."""
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=1, num_threads=2), threads=2)
    raw = S.make_scan(24000)
    short = raw[: 24000 // 8]
    assert oracle.Extractor().extract(short, 100.0) <= 5
    assert PO.process_frame(om, [short, short], [100.0, 100.0], pieces=2) == []
    assert om.frame_index == 0
    assert len(PO.process_frame(om, [short, raw], [100.1, 100.1], pieces=2)) == 2 and om.frame_index == 2
