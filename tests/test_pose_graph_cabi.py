"""Pose graph and re-posed keyframes at the C-ABI without a GPU: exports with the header's parameter counts, null arguments refused, the host
R_aff / T_aff of the re-pose against the oracle, and the C++ mirror (Pose_graph, add_constrain_of_loop, refine_pointclouds) compiling, linking
and running."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

import pose_graph_reference as R
from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_params(name):
    hdr = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"(?:int|void)\s+" + name + r"\(([^;]*)\);", hdr)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n in (("ll_pose_graph_create", 4), ("ll_pose_graph_release", 1), ("ll_pose_graph_optimize", 7), ("ll_pose_graph_step", 11),
                    ("ll_pose_graph_loop_edge", 7), ("ll_keyframes_repose", 10), ("ll_keyframe_affine", 4)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n, name


def test_null_arguments_are_refused():
    L = capi.lib()
    h = C.c_void_p()
    assert L.ll_pose_graph_create(None, 1, 1, C.byref(h)) == capi.LL_ERR_INVALID
    assert L.ll_pose_graph_step(None, None, 0, None, 0, 1.0, None, None, None, None, None) == capi.LL_ERR_INVALID
    assert L.ll_keyframes_repose(None, None, 0, None, 1, None, None, 0.1, None, None) == capi.LL_ERR_INVALID


def test_affine_matches_the_oracle():
    """R_aff / T_aff are the host's; the oracle's re-pose of one point at the origin and of unit points exposes them bit for bit."""
    rng = np.random.default_rng(2)
    L = capi.lib()
    for _ in range(20):
        po = np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3) * 50])
        pp = np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3) * 50])
        a, b = capi.Pose(), capi.Pose()
        a.q_wxyz[:], a.t[:], b.q_wxyz[:], b.t[:] = list(po[:4]), list(po[4:]), list(pp[:4]), list(pp[4:])
        Ra, Ta = np.zeros(9, np.float32), np.zeros(3, np.float32)
        L.ll_keyframe_affine(C.byref(a), C.byref(b), Ra.ctypes.data, Ta.ctypes.data)
        pts = np.array([[0, 0, 0, 1], [1, 0, 0, 1], [0, 1, 0, 1], [0, 0, 1, 1]], np.float32) * np.float32(1000)   # one point per 1 km voxel
        pts[:, 3] = 1
        out, cnt = R.oracle_repose(pts, [4], po, pp, 1.0)
        assert cnt[0] == 4
        assert np.array_equal(out[0, :3], Ta)
        for k in range(3):
            col = (out[1 + k, :3] - Ta) / np.float32(1000)
            assert np.allclose(col, Ra.reshape(3, 3)[:, k], rtol=0, atol=1e-6)


def test_cpp_mirror_compiles_links_and_runs(tmp_path):
    exe = str(tmp_path / "pose_graph_mirror")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pose_graph_mirror.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GPU run" in r.stdout or "no GPU" in r.stdout
