"""ctypes binding of oracle/liborcspin.so (orc_spin.hpp) — ORACLE, TEST INFRASTRUCTURE ONLY.

The line-by-line restatement of the reference's Velodyne front end (laser_feature_extractor.hpp:393-825) that the device path is compared
against.  Only tests/ and scripts/ import it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
CLOUDS = ("full", "sharp", "less_sharp", "flat", "less_flat")


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liborcspin.so")
    srcs = [os.path.join(_HERE, f) for f in ("spin_api.cpp", "orc_spin.hpp", "orc_cloud.hpp", "spin.mk")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-f", "spin.mk", "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.orc_spin_create.argtypes = [C.c_int, C.c_float, C.c_float]
        L.orc_spin_create.restype = C.c_void_p
        L.orc_spin_free.argtypes = [C.c_void_p]
        L.orc_spin_extract.argtypes = [C.c_void_p, f32p, C.c_int, i32p]
        L.orc_spin_extract.restype = C.c_double
        L.orc_spin_cloud.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_spin_point_info.argtypes = [C.c_void_p, i32p, f32p, i32p, i32p]
        _LIB = L
    return _LIB


class SpinExtractor:
    """extract(raw [n, 4]) -> dict of the five clouds ([m, 4] float32, push order); point_info() -> (ring, curvature, picked, label)."""

    def __init__(self, scan_line: int = 16, minimum_range: float = 0.1, plane_resolution: float = 0.4):
        self.h = lib().orc_spin_create(scan_line, minimum_range, plane_resolution)
        self.counts = np.zeros(5, np.int32)
        self.seconds = 0.0

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_spin_free(self.h)
            self.h = None

    def extract(self, raw):
        raw = np.ascontiguousarray(raw, dtype=np.float32).reshape(-1, 4)
        self.seconds = lib().orc_spin_extract(self.h, raw, raw.shape[0], self.counts)
        out = {}
        for k, name in enumerate(CLOUDS):
            a = np.zeros((int(self.counts[k]), 4), np.float32)
            lib().orc_spin_cloud(self.h, k, a)
            out[name] = a
        return out

    def point_info(self):
        n = int(self.counts[0])
        ring, curv, picked, label = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        lib().orc_spin_point_info(self.h, ring, curv, picked, label)
        return ring, curv, picked, label
