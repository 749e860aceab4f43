"""The oracle's piecewise frame: Laser_feature::laserCloudHandler publishing every piece of a sensor frame, and Laser_mapping::process_new_scan
registering each piece as a scan of its own -- composed from the oracle pieces that exist (oracle.Extractor, oracle.voxel_grid and
oracle.Mapper's per-scan step), not from the device path's slices.  Test infrastructure, like oracle/ itself."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O


class _Published:
    """Stands in for the mapper's extractor for one piece: the piece's clouds as the feature node publishes them (before any VoxelGrid)."""

    def __init__(self, c, s, full):
        self.clouds = (c, s, full)

    def extract(self, raw, stamp):
        return 0

    def get_features(self, min_blur=0.0, max_blur=1.0):
        return self.clouds


def frame_pieces(ex, heads, stamps, pieces):
    """laser_feature_extractor.hpp:285-358 with ONE extractor over the heads in turn (Mid-100: 3): a head with <= 5 petals contributes nothing
    (:287); piece i of a head is get_features(start_i, end_i) over the bounds of :313-323; piece i of the frame is the concatenation over the
    contributing heads in head order (:339-358).  Returns ([(corner, surface, full)] per piece, number of contributing heads)."""
    parts = [([], [], []) for _ in range(pieces)]
    live = 0
    for raw, stamp in zip(heads, stamps):
        if ex.extract(raw, stamp) <= 5:          # laserCloudScans.size() <= 5 (:287)
            continue
        live += 1
        start, end = ex.piece_bounds(pieces)
        for i in range(pieces):
            for acc, cloud in zip(parts[i], ex.get_features(start[i], end[i])):
                acc.append(cloud)
    z = np.zeros((0, 4), np.float32)
    return [tuple(np.concatenate(a) if a else z for a in p) for p in parts], live


def process_frame(mapper: O.Mapper, heads, stamps, pieces=3, odom_mode=1):
    """One sensor frame through oracle.Mapper: every published piece (odom_mode 1; 0: piece 0 only, :385-388) goes through the extractor's
    VoxelGrids (:372-380), the mapping node's (laser_mapping.hpp:1367-1373) and the per-scan step of process_new_scan (:1336-1505), exactly
    as oracle.Mapper.process_scan runs them for a whole scan.  Returns one (status, q, t, last) per published piece; [] when no head has
    more than 5 petals (nothing is published, the mapper is untouched)."""
    parts, live = frame_pieces(mapper.ex, heads, stamps, pieces)
    if live == 0:
        return []
    out = []
    ex = mapper.ex
    try:
        for i in range(pieces if odom_mode else 1):
            mapper.ex = _Published(*parts[i])
            st, q, t = mapper.process_scan(None, 0.0)
            out.append((st, q, t, dict(mapper.last)))
    finally:
        mapper.ex = ex
    return out
