"""CPU checks of the mapper recovery's ABI surface (ll_mapper_recovery_default, ll_mapper_set_recovery, ll_mapper_recovery_read,
ll_mapper_recovery_last_inputs): exported with the header's parameter counts, null arguments refused without a device, the ctypes mirrors laid out
as the C structs, and the C++ mirror compiles, links and runs."""
import ctypes as C
import os
import re
import subprocess

from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_params(name):
    hdr = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"(?:int|void)\s+" + name + r"\(([^;]*)\);", hdr)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


def _compile(tmp_path, name):
    exe = str(tmp_path / name)
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_mapper_recovery_default", 1), ("ll_mapper_set_recovery", 2), ("ll_mapper_recovery_read", 5),
                           ("ll_mapper_recovery_last_inputs", 13)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name


def test_null_arguments_are_refused():
    L = capi.lib()
    cfg = capi.RecoveryCfg()
    L.ll_mapper_recovery_default(C.byref(cfg))
    assert cfg.lost_after == 3 and cfg.max_inlier_threshold > 0 and 0 < cfg.min_verify_fraction < 1
    L.ll_mapper_recovery_default(None)   # (no effect, no fault)
    assert L.ll_mapper_set_recovery(None, C.byref(cfg)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_set_recovery(None, None) == capi.LL_ERR_INVALID
    e, n, d = (capi.RecoveryStep * 1)(), C.c_int(), C.c_int()
    assert L.ll_mapper_recovery_read(None, e, 1, C.byref(n), C.byref(d)) == capi.LL_ERR_INVALID
    cnt = (C.c_size_t * 4)()
    assert L.ll_mapper_recovery_last_inputs(None, None, None, None, cnt, None, None, None, None, 0, None, None, 0) == capi.LL_ERR_INVALID


def test_struct_layouts_equal_the_ctypes_mirrors(tmp_path):
    exe = _compile(tmp_path, "recovery_layout")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    mirrors = {"ll_recovery_cfg": capi.RecoveryCfg, "ll_recovery_step": capi.RecoveryStep}
    seen = set()
    for line in r.stdout.splitlines():
        struct, field, value = line.split()
        cls = mirrors[struct]
        if field == "sizeof":
            assert C.sizeof(cls) == int(value), struct
        else:
            assert getattr(cls, field).offset == int(value), (struct, field)
            seen.add((struct, field))
    for struct, cls in mirrors.items():   # every field of the mirror was compared
        assert {f for f, _ in cls._fields_} == {f for s, f in seen if s == struct}, struct


def test_cpp_mirror_recovery_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "recovery_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
