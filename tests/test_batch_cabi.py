"""CPU checks of the batch registration's ABI surface: ll_register_batch is exported, LL_MAX_BATCH has the same value in the header and the
ctypes binding, null arguments are refused without a device, and the C++ mirror's register_batch compiles, links and runs."""
import ctypes as C
import os
import re
import subprocess

from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_and_max_batch():
    L = capi.lib()
    assert hasattr(L, "ll_register_batch") and "ll_register_batch" in capi.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"#define\s+LL_MAX_BATCH\s+(\d+)", hdr)
    assert m and int(m.group(1)) == capi.LL_MAX_BATCH == 16


def test_null_arguments_are_refused():
    L = capi.lib()
    res, st = (capi.RegResult * 1)(), (C.c_int * 1)()
    assert L.ll_register_batch(None, None, 1, None, None, None, None, capi.LL_FMT_XYZI16, capi.LL_HOST, None, res, st) == capi.LL_ERR_INVALID


def test_cpp_mirror_register_batch_compiles_links_and_runs(tmp_path):
    exe = str(tmp_path / "batch_mirror")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "batch_mirror.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
