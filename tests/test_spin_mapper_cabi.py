"""CPU checks of the streaming mapper's sweep entry points (ll_mapper_process_sweep / _sweeps): exported with the header's parameter counts,
null arguments and empty sequences refused without a device, the Python mirror present, and the C++ mirror compiles, links and runs."""
import ctypes as C
import subprocess

from loam_livox_b200 import capi
from loam_livox_b200.registration import Laser_mapping
from test_recovery_cabi import _compile, _header_params


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_mapper_process_sweep", 8), ("ll_mapper_process_sweeps", 10)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name
    # the sequence call takes the single call's arguments as arrays, with the count and the completed count around them
    assert L.ll_mapper_process_sweeps.argtypes[-3:-1] == L.ll_mapper_process_sweep.argtypes[-2:]


def test_null_arguments_are_refused():
    L = capi.lib()
    res, stats, done = capi.RegResult(), capi.MapperStats(), C.c_int(7)
    assert L.ll_mapper_process_sweep(None, None, None, 0, capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(res), C.byref(stats)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_process_sweeps(None, None, 1, None, None, capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(res), C.byref(stats), C.byref(done)) == capi.LL_ERR_INVALID
    assert done.value == 0
    assert L.ll_mapper_process_sweeps(None, None, 0, None, None, capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(res), C.byref(stats), None) == capi.LL_ERR_INVALID


def test_python_mirror():
    assert callable(Laser_mapping.process_new_sweep) and callable(Laser_mapping.process_new_sweeps)


def test_cpp_mirror_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "spin_mapper_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GPU run" in r.stdout or "no GPU" in r.stdout
