"""The oracle's spinning-lidar odometry: the reference's Velodyne feature node with its outputs remapped onto the mapping node's inputs
(/laser_cloud_less_sharp -> /pc2_corners, /laser_cloud_less_flat -> /pc2_surface, /laser_points_2 -> /pc2_full), composed from the oracle
pieces that exist (oracle.spin_oracle.SpinExtractor and oracle.Mapper's per-scan step), not from the device path.  Test infrastructure, like
oracle/ itself.

oracle.Mapper.process_scan runs the Livox feature node's VoxelGrids (laser_feature_extractor.hpp:372-380) before the mapping node's
(laser_mapping.hpp:1367-1373).  The Velodyne branch has none on the less-sharp cloud and has already run its per-ring one on the less-flat
cloud, so the composition builds its mapper with extractor leaves of None, and while a sweep is stepped a VoxelGrid of leaf None passes its
cloud through.  Every other caller of oracle.voxel_grid passes a number and sees no change."""
from __future__ import annotations

import contextlib
import time

import numpy as np

from oracle import oracle as O
from oracle.spin_oracle import SpinExtractor

_voxel_grid = O.voxel_grid


@contextlib.contextmanager
def _no_extractor_voxel_grid():
    O.voxel_grid = lambda cloud, leaf: cloud if leaf is None else _voxel_grid(cloud, leaf)
    try:
        yield
    finally:
        O.voxel_grid = _voxel_grid


class _Published:
    """The mapper's extractor for one sweep: the remapped clouds (corners, surfaces, full) as the feature node publishes them."""

    def __init__(self, c, s, full):
        self.clouds = (c, s, full)

    def extract(self, raw, stamp):
        return 0

    def get_features(self, min_blur=0.0, max_blur=1.0):
        return self.clouds


def mapper(scan_line=16, **kw):
    """(SpinExtractor, oracle.Mapper without extractor VoxelGrids); kw go to oracle.Mapper."""
    return SpinExtractor(scan_line), O.Mapper(extractor_leaf_corner=None, extractor_leaf_surf=None, **kw)


class SpinMapper:
    """process_sweep(raw) -> (status, q, t, last): one sweep through the spin oracle, then oracle.Mapper's step on less sharp -> corners,
    less flat -> surfaces, full -> the time range.  `clouds` holds the sweep's five clouds; `seconds` the CPU time of the last sweep."""

    def __init__(self, scan_line=16, **kw):
        self.front, self.m = mapper(scan_line, **kw)
        self.clouds, self.seconds = None, 0.0

    def process_sweep(self, raw):
        t0 = time.perf_counter()
        self.clouds = self.front.extract(raw)
        ex = self.m.ex
        try:
            self.m.ex = _Published(self.clouds["less_sharp"], self.clouds["less_flat"], self.clouds["full"])
            with _no_extractor_voxel_grid():
                st, q, t = self.m.process_scan(None, 0.0)
        finally:
            self.m.ex = ex
        self.seconds = time.perf_counter() - t0
        return st, q, t, dict(self.m.last)
