"""CPU checks of the sequence calls' ABI surface: ll_mapper_process_frames / _scans are exported with the header's signatures, null arguments
are refused without a device, and the C++ mirror's process_new_frames / process_new_scans compile, link and run."""
import ctypes as C
import os
import re
import subprocess

from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_params(name):
    hdr = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"int\s+" + name + r"\(([^;]*)\);", hdr)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_mapper_process_frames", 14), ("ll_mapper_process_scans", 10)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name


def test_null_arguments_are_refused():
    L = capi.lib()
    res, st, n, done = (capi.RegResult * 1)(), (capi.MapperStats * 1)(), (C.c_int * 1)(), C.c_int(-1)
    assert L.ll_mapper_process_frames(None, 1, 1, None, None, capi.LL_FMT_XYZI16, capi.LL_HOST, None, 1, res, st, 1, n, C.byref(done)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_process_scans(None, 1, None, None, capi.LL_FMT_XYZI16, capi.LL_HOST, None, res, st, C.byref(done)) == capi.LL_ERR_INVALID


def test_cpp_mirror_sequences_compile_link_and_run(tmp_path):
    exe = str(tmp_path / "pipeline_mirror")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pipeline_mirror.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
