"""CPU checks of the streaming mapper's loop-closure ABI (ll_mapper_loop_closure_default, ll_mapper_set_loop_closure, ll_mapper_loop_read,
ll_mapper_loop_result, ll_mapper_loop_cloud): exported with the header's parameter counts, null arguments refused without a device, the defaults
rosbag_loop.launch runs, the ctypes mirrors laid out as the C structs, and the C++ mirror compiles, links and runs."""
import ctypes as C
import os
import subprocess

import pytest

from loam_livox_b200 import capi
from test_recovery_cabi import _compile, _header_params


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_mapper_loop_closure_default", 1), ("ll_mapper_set_loop_closure", 2), ("ll_mapper_loop_read", 5),
                           ("ll_mapper_loop_result", 7), ("ll_mapper_loop_cloud", 6)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name


def test_defaults_are_the_launch_values():
    L = capi.lib()
    c = capi.LoopClosureCfg()
    L.ll_mapper_loop_closure_default(C.byref(c))
    # performance_precision.yaml (loop_closure/, mapping/surround_pointcloud_resolution, common/if_update_mean_and_cov_incrementally) with
    # rosbag_loop.launch's if_enable_loop_closure 1 and minimum_keyframe_differen 200
    assert (c.scans_of_each_keyframe, c.scans_between_two_keyframe) == (300, 100)
    assert c.loop.minimum_keyframe_differen == 200
    assert c.loop.minimum_similarity_linear == pytest.approx(0.65) and c.loop.minimum_similarity_planar == pytest.approx(0.94)
    assert c.loop.avail_ratio_plane == pytest.approx(0.05) and c.loop.avail_ratio_line == pytest.approx(0.03)   # laser_mapping.hpp:894-895
    assert c.loop.maximum_roi_difference == 5.0 and c.loop.plane_with_line == 0.92
    assert c.map_alignment_resolution == pytest.approx(0.1) and c.map_alignment_maximum_icp_iteration == 5
    assert c.map_alignment_inlier_threshold == pytest.approx(0.20) and c.scene_alignment_maximum_residual_block == 3000
    assert c.surround_pointcloud_resolution == 0.30 and c.incremental_cov == 1
    assert c.reserve_map_points > 0 and c.reserve_history_points > 0 and c.reserve_keyframes > 0
    L.ll_mapper_loop_closure_default(None)   # (no effect, no fault)


def test_null_arguments_are_refused():
    L = capi.lib()
    c = capi.LoopClosureCfg()
    L.ll_mapper_loop_closure_default(C.byref(c))
    assert L.ll_mapper_set_loop_closure(None, C.byref(c)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_set_loop_closure(None, None) == capi.LL_ERR_INVALID
    e, n, d, closed, sz = (capi.LoopEvent * 1)(), C.c_int(), C.c_int(), C.c_int(), C.c_size_t()
    assert L.ll_mapper_loop_read(None, e, 1, C.byref(n), C.byref(d)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_loop_result(None, C.byref(n), C.byref(closed), None, None, 0, None) == capi.LL_ERR_INVALID
    assert L.ll_mapper_loop_cloud(None, 0, None, 0, C.byref(sz), None) == capi.LL_ERR_INVALID


def test_struct_layouts_equal_the_ctypes_mirrors(tmp_path):
    exe = _compile(tmp_path, "loop_closure_layout")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    mirrors = {"ll_loop_closure_cfg": capi.LoopClosureCfg, "ll_loop_event": capi.LoopEvent}
    seen = set()
    for line in r.stdout.splitlines():
        struct, field, value = line.split()
        cls = mirrors[struct]
        if field == "sizeof":
            assert C.sizeof(cls) == int(value), struct
        else:
            assert getattr(cls, field).offset == int(value), (struct, field)
            seen.add((struct, field))
    for struct, cls in mirrors.items():
        assert {f for f, _ in cls._fields_} == {f for s, f in seen if s == struct}, struct


def test_cpp_mirror_loop_closure_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "loop_closure_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
