"""CPU checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/loamlivox_b200.h declares,
its POD structs have the sizes the ctypes mirror assumes, and it refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(ll_[a-z0-9_]+)\s*\(", txt)))


def test_every_declared_symbol_is_exported():
    L = capi.lib()
    names = _declared()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert sorted(capi.EXPORTS) == names, (set(capi.EXPORTS) ^ set(names))


def test_pod_layouts_match_the_header():
    assert C.sizeof(capi.Config) == 7 * 4 + 2 * 4
    assert C.sizeof(capi.RegState) == 10 * 4 + 12 * 8 + (4 + 3 + 4 + 3 + 7) * 8
    assert C.sizeof(capi.RegResult) == 8 * 4 + (4 + 3 + 4 + 3) * 8 + 5 * 8 + 6 * 4
    assert C.sizeof(capi.PipelineCfg) == 7 * 4
    s = capi.default_reg_state()
    assert (s.icp_max_iterations, s.cere_max_iterations, s.cere_prerun_times) == (15, 50, 2)        # performance_precision.yaml:25-26, :91
    assert (s.maximum_dis_line_for_match, s.maximum_dis_plane_for_match, s.huber_a) == (2.0, 50.0, 0.1)   # point_cloud_registration.hpp:64-65,220
    assert (s.inliner_dis, s.inlier_ratio, s.para_max_speed, s.para_max_angular_rate) == (0.02, 0.8, 0.3, 20.0)
    # ll_mapper_config: the defaults written by the library must land in the ctypes fields of the same name (a shifted layout would scramble them)
    m = capi.MapperConfig(); capi.lib().ll_mapper_config_default(C.byref(m))
    assert C.sizeof(capi.MapperConfig) == 13 * 4 + C.sizeof(capi.PipelineCfg) + C.sizeof(capi.RegState) and capi.MapperConfig.reg.offset == 80   # 13 scalars, pipeline, reg state
    assert (m.matching_mode, m.maximum_history_size, m.down_sample_replace, m.threshold_cell_revisit) == (0, 400, 1, 2000)   # performance_precision.yaml:28-29, laser_mapping.hpp:277
    assert (m.reserve_map_points, m.reserve_store_points) == (1 << 22, 1 << 22)
    assert abs(m.line_resolution - 0.1) < 1e-7 and abs(m.plane_resolution - 0.4) < 1e-7 and m.cell_resolution == 1.0 and m.maximum_in_fov_angle == 45.0
    assert (m.pipeline.pieces, m.pipeline.whole_frame) == (3, 1) and abs(m.pipeline.mapping_leaf_surf - 0.4) < 1e-7
    assert (m.reg.icp_max_iterations, m.reg.cere_max_iterations, m.reg.huber_a) == (15, 50, 0.1)
    c = capi.default_config()
    assert abs(c.corner_curvature - 0.1) < 1e-7 and abs(c.surface_curvature - 0.005) < 1e-9 and c.minimum_view_angle == 5.0


def test_no_cpu_fallback():
    """Without a CUDA device the product refuses to construct a context; nothing routes through the oracle or PyTorch."""
    import torch
    if torch.cuda.is_available():
        return
    h = C.c_void_p()
    assert capi.lib().ll_ctx_create(None, 0, C.byref(h)) == capi.LL_ERR_CUDA and not h.value
    src = "".join(open(os.path.join(ROOT, "loam_livox_b200", f)).read() for f in ("capi.py", "registration.py", "distributed.py", "__init__.py"))
    assert "oracle" not in src.replace("no CPU or PyTorch fallback", "")


def test_pose_log_format_matches_reference_printf():
    """ll_format_pose_log is host-only code: the poses.log block of loam_livox/source/laser_mapping.hpp:1506-1511."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import format_pose_log
    r = capi.RegResult()
    r.q_w_curr[:] = [0.9, 0.1, -0.2, 0.3]; r.t_w_curr[:] = [1.5, -2.25, 0.125]
    r.q_w_incre[:] = [1.0, 0.001, 0.002, -0.003]; r.t_w_incre[:] = [0.01, 0.02, -0.03]
    r.final_cost = 12.3456789; r.num_residual_blocks = 4321
    want = "--------------------\n" + "Curr_Q = %f,%f,%f,%f\r\n" % (0.9, 0.1, -0.2, 0.3) + "Curr_T = %f,%f,%f\r\n" % (1.5, -2.25, 0.125) + \
           "Incre_Q = %f,%f,%f,%f\r\n" % (1.0, 0.001, 0.002, -0.003) + "Incre_T = %f,%f,%f\r\n" % (0.01, 0.02, -0.03) + "Cost=%f,blk_size = %d \r\n" % (12.3456789, 4321)
    assert format_pose_log(r) == want


def test_cpp_mirror_compiles_links_and_runs(tmp_path):
    """include/loamlivox_b200.hpp (the reference's class names over the C-ABI) is compiled with g++, linked against the product library and run;
    on a box without a GPU the program must stop at ll_ctx_create with LL_ERR_CUDA (no fallback), on a GPU box it runs a tiny extraction."""
    import os
    import subprocess
    from loam_livox_b200 import capi
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "mirror_smoke")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "mirror_smoke.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
