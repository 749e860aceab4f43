"""CPU checks of the spinning-lidar front end's ABI (ll_spin_*): exported with the header's parameter counts, the defaults of the reference,
null arguments refused without a device, the ctypes mirror laid out as the C struct, and the C++ mirror compiles, links and runs."""
import ctypes as C
import subprocess

from loam_livox_b200 import capi
from test_recovery_cabi import _compile, _header_params


def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_spin_cfg_default", 1), ("ll_spin_create", 3), ("ll_spin_release", 1), ("ll_spin_extract", 6), ("ll_spin_cloud", 6),
                           ("ll_spin_point_info", 7), ("ll_spin_chains", 3)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name


def test_defaults_and_layout():
    c = capi.default_spin_cfg()
    assert (c.scan_line, c.max_points) == (16, 400000)   # laser_feature_extractor.hpp:137, the per-point arrays of :75-78
    assert c.minimum_range == C.c_float(0.1).value and c.plane_resolution == C.c_float(0.4).value
    assert C.sizeof(capi.SpinCfg) == 16 and [f[0] for f in capi.SpinCfg._fields_] == ["scan_line", "minimum_range", "plane_resolution", "max_points"]
    assert (capi.LL_SPIN_FULL, capi.LL_SPIN_SHARP, capi.LL_SPIN_LESS_SHARP, capi.LL_SPIN_FLAT, capi.LL_SPIN_LESS_FLAT) == (0, 1, 2, 3, 4)


def test_null_arguments_are_refused():
    L = capi.lib()
    cfg = capi.default_spin_cfg()
    assert L.ll_spin_create(None, C.byref(cfg), None) == capi.LL_ERR_INVALID
    assert L.ll_spin_extract(None, None, 0, capi.LL_FMT_XYZI16, capi.LL_HOST, None) == capi.LL_ERR_INVALID
    n = C.c_size_t()
    assert L.ll_spin_cloud(None, 0, None, 0, C.byref(n), None) == capi.LL_ERR_INVALID
    assert L.ll_spin_point_info(None, None, None, None, None, 0, C.byref(n)) == capi.LL_ERR_INVALID
    assert L.ll_spin_chains(None, None, None) == capi.LL_ERR_INVALID
    L.ll_spin_release(None)
    L.ll_spin_cfg_default(None)


def test_cpp_mirror_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "spin_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GPU run" in r.stdout or "no GPU" in r.stdout
