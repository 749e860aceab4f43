"""Host-only checks of the loop policy (ll_mapper_set_loop_policy, ll_mapper_loop_edges; DESIGN.md §4.6): the composition's policy
(tests/loop_policy_oracle.py: loops_done, gap_allows; tests/loop_closure_oracle.py: candidate_loop) against a restatement of the reference's
for-loop (laser_mapping.hpp:988-1127) with if_end replaced by the loop count and the gap rule; version-2 loop images through ll_loop_image_info, valid ones reported and every
rule of their LOOP section refused just outside its bound; the C ABI, its ctypes mirrors and the C++ mirror."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

import loop_closure_oracle as LCO
import loop_policy_oracle as LPO
from loam_livox_b200 import capi
from test_loop_image import IMG, accumulated, config, edge, events, image, info, open_kfs, points, pose, scalars, cells, history, summary
from test_recovery_cabi import _compile, _header_params

THR = 0.35


# ---------------------------------------------------------------------------------------------- the policy against the reference's loop
def reference_restated(stream, thr, max_loops, gap):
    """service_loop_detection's for-loop over his (:988-1127) per closed keyframe, `his += 10` / `his += 5` before the loop's own his++, with
    if_end (:990-993, set by a loop) replaced by: stop once max_loops loops closed, and skip a keyframe closer than gap to the last loop's."""
    thr_f, thr2 = float(np.float32(thr)), float(np.float32(thr) * np.float32(2))
    out, n_loops, last = [], 0, None
    for newest, (passes, score) in enumerate(stream):
        if n_loops >= max_loops:
            break
        if last is not None and newest - last < gap:
            continue
        his = 0
        while his < newest:
            if his in passes:   # the gates of :994-1033
                s = score[his]
                if s > thr2:
                    out.append((newest, his, LCO.SKIP10))
                    his += 10
                elif s < thr_f:
                    out.append((newest, his, LCO.ACCEPT))
                    n_loops, last = n_loops + 1, newest
                    break
                else:
                    out.append((newest, his, LCO.SKIP5))
                    his += 5
            his += 1
    return out


def composed(stream, thr, max_loops, gap):
    """The composition's path (LoopPolicyOracle.step / _process): the count and gap rules, then candidate_loop."""
    out, loops = [], []
    for newest, (passes, score) in enumerate(stream):
        if LPO.loops_done(len(loops), max_loops):
            break
        if not LPO.gap_allows(newest, loops, gap):
            continue
        for his, d, _ in LCO.candidate_loop(sorted(passes), lambda h: (score[h], None), thr):
            out.append((newest, his, d))
            if d == LCO.ACCEPT:
                loops.append(newest)
    return out


def test_policy_equals_the_restated_reference_loop():
    rng = np.random.default_rng(7)
    t = np.float32(THR)
    # scores at the threshold and at twice it exactly (float parameter, double score), one ulp around them, and well inside each band
    levels = [float(t), float(t * np.float32(2)), float(np.nextafter(t, np.float32(0))), float(np.nextafter(t * np.float32(2), np.float32(9))),
              float(np.nextafter(t, np.float32(9))), float(np.nextafter(t * np.float32(2), np.float32(0))), 0.05, 0.5, 1.5]
    seen = dict(at_gap=0, below_gap=0, stop_mid=0, at_thr=0, at_thr2=0, loops=0)
    for case in range(4000):
        n = int(rng.integers(2, 48))
        max_loops, gap = int(rng.integers(1, 6)), int(rng.integers(0, 7))
        p_pass, p_accept = rng.uniform(0.05, 0.9), rng.uniform(0.05, 0.8)
        stream = []
        for newest in range(n):
            passes = {h for h in range(newest) if rng.random() < p_pass}
            score = {h: (0.1 if rng.random() < p_accept else levels[int(rng.integers(len(levels)))]) for h in passes}
            stream.append((passes, score))
        want, got = reference_restated(stream, THR, max_loops, gap), composed(stream, THR, max_loops, gap)
        assert got == want, (case, max_loops, gap)
        loops = [k for k, _, d in want if d == LCO.ACCEPT]
        seen["loops"] += len(loops)
        seen["stop_mid"] += len(loops) == max_loops and loops[-1] < n - 1
        seen["at_gap"] += any(b - a == gap for a, b in zip(loops, loops[1:]))
        searched = {k for k, _, _ in want}
        seen["below_gap"] += gap > 0 and any(k - loops[0] == gap - 1 and k not in searched and stream[k][0] for k in range(n)) if loops else 0
        for k, h, _ in want:
            seen["at_thr"] += stream[k][1][h] == levels[0]
            seen["at_thr2"] += stream[k][1][h] == levels[1]
    print(seen)
    assert all(v >= 50 for v in seen.values()), seen


def test_the_default_policy_is_the_reference():
    """max_loops 1, gap 0: the first accepted candidate ends all search, as if_end does."""
    stream = [(set(range(k)), {h: 0.1 for h in range(k)}) for k in range(6)]
    assert composed(stream, THR, 1, 0) == reference_restated(stream, THR, 1, 0) == [(1, 0, LCO.ACCEPT)]
    assert composed(stream, THR, 3, 2) == [(1, 0, LCO.ACCEPT), (3, 0, LCO.ACCEPT), (5, 0, LCO.ACCEPT)]


# ---------------------------------------------------------------------------------------------- version-2 loop images
def parts_k(K=6, closed=True):
    """A valid version-1 image's sections with K closed keyframes and three open ones."""
    infos = b"".join(bytes(info()) for _ in range(K))
    return [config(), scalars(closed=int(closed), n_keyframes=K), cells(), history(), open_kfs(), infos, b"".join(pose(0.3 * k) for k in range(K)),
            b"".join(edge(k - 1, k) for k in range(1, K)), np.zeros(K * IMG, "<f4").tobytes(), points(5 * K, 5),
            accumulated(tuple(3 * (k + 1) for k in range(K + 2))), b"", events()]


def loop2(max_loops=3, gap=2, loops=((2, 0), (4, 1)), n_opt=None, pad=0, opt=None) -> bytes:
    n_opt = (max(loops[-1]) + 1 if loops else 0) if n_opt is None else n_opt
    opt = b"".join(pose(0.3 * k + 0.01) for k in range(n_opt)) if opt is None else opt
    return struct.pack("<iiii", max_loops, gap, len(loops), pad) + b"".join(edge(a, b) for a, b in loops) + opt


def v2(loop=None, closed=None, K=6, **kw):
    p = parts_k(K)
    p[11] = loop2(**kw) if loop is None else loop
    n_loops = struct.unpack_from("<i", p[11], 8)[0] if len(p[11]) >= 12 else 0
    p[1] = scalars(closed=int(n_loops > 0) if closed is None else closed, n_keyframes=K)
    return image(p, version=capi.LL_LOOP_IMAGE_VERSION_POLICY)


def status(img):
    return summary(img)[0]


def test_valid_version_2_images_are_accepted_and_reported():
    st, got = summary(v2())
    assert st == capi.LL_OK and (got.version, got.closed, got.keyframes) == (2, 1, 6)
    st, got = summary(v2(loops=()))   # no loop yet: the policy, n_loops 0 and nothing else
    assert st == capi.LL_OK and (got.version, got.closed) == (2, 0)
    assert status(v2(max_loops=capi.LL_MAX_LOOPS)) == capi.LL_OK
    assert status(v2(max_loops=2)) == capi.LL_OK                          # n_loops = max_loops
    assert status(v2(loops=((0, 2), (1, 4)))) == capi.LL_OK                # the newest id either way round
    assert status(v2(loops=((1, 0), (5, 3)), gap=4)) == capi.LL_OK        # newest - L exactly the gap
    assert status(v2(loops=((1, 0), (2, 0), (3, 1)), gap=0)) == capi.LL_OK
    p = parts_k()
    p[1] = scalars(closed=0, n_keyframes=6)
    assert status(image(p)) == capi.LL_OK                                  # the same parts as version 1
    from loam_livox_b200.registration import loop_image_info
    assert loop_image_info(v2())["version"] == 2


def test_version_2_refusals():
    bad = {
        "max_loops 1 (the default writes version 1)": v2(max_loops=1, loops=((2, 0),)),
        "max_loops 0": v2(max_loops=0, loops=()),
        "max_loops above LL_MAX_LOOPS": v2(max_loops=capi.LL_MAX_LOOPS + 1),
        "negative gap": v2(gap=-1),
        "n_loops above max_loops": v2(max_loops=2, loops=((1, 0), (3, 0), (5, 0)), gap=0),
        "edge id = n_keyframes": v2(loops=((2, 0), (6, 1))),
        "negative edge id": v2(loops=((2, -1), (4, 1))),
        "equal ids": v2(loops=((2, 0), (4, 4))),
        "newest decreasing": v2(loops=((4, 1), (2, 0))),
        "newest repeated": v2(loops=((4, 1), (4, 0)), gap=0),
        "gap broken": v2(loops=((1, 0), (5, 3)), gap=5),
        "pad not zero": v2(pad=1),
        "closed 0 with loops": v2(closed=0),
        "closed 1 without loops": v2(loops=(), closed=1),
        "one optimized pose short": v2(n_opt=4),
        "one optimized pose long": v2(n_opt=6),
        "trailing bytes": v2(loop=loop2() + b"\0" * 8),
        "shorter than its count": v2(loop=loop2()[:12]),
        "empty": v2(loop=b"", closed=0),
        "non-finite optimized pose": v2(opt=b"".join(pose(0.3 * k) for k in range(4)) + pose(float("nan"))),
    }
    nan_edge = bytearray(loop2())
    nan_edge[16 + 8 + 32:16 + 8 + 40] = struct.pack("<d", float("inf"))   # the first edge's t.x
    bad["non-finite edge"] = v2(loop=bytes(nan_edge))
    for name, img in bad.items():
        assert status(img) == capi.LL_ERR_INVALID, name
    # a version-1 image cannot hold a version-2 LOOP section
    p = parts_k()
    p[11] = loop2()
    assert status(image(p)) == capi.LL_ERR_INVALID


# ---------------------------------------------------------------------------------------------- ABI
def test_symbols_signatures_and_default():
    L = capi.lib()
    for name, n_params in (("ll_mapper_loop_policy_default", 1), ("ll_mapper_set_loop_policy", 2), ("ll_mapper_loop_edges", 4)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name
    p = capi.LoopPolicy(max_loops=7, min_keyframes_between_loops=9)
    L.ll_mapper_loop_policy_default(C.byref(p))
    assert (p.max_loops, p.min_keyframes_between_loops) == (1, 0)
    L.ll_mapper_loop_policy_default(None)
    n = C.c_int()
    assert L.ll_mapper_set_loop_policy(None, C.byref(p)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_set_loop_policy(None, None) == capi.LL_ERR_INVALID
    assert L.ll_mapper_loop_edges(None, None, 0, C.byref(n)) == capi.LL_ERR_INVALID
    assert capi.LL_MAX_LOOPS == capi.LL_PG_MAX_BORDER // 2 == 32


def test_struct_layout_equals_the_ctypes_mirror(tmp_path):
    exe = _compile(tmp_path, "loop_policy_mirror")
    r = subprocess.run([exe, "layout"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    seen = set()
    for line in r.stdout.splitlines():
        name, field, value = line.split()
        if name == "const":
            assert getattr(capi, field) == int(value), field
        elif field == "sizeof":
            assert C.sizeof(capi.LoopPolicy) == int(value) == 8
        else:
            assert getattr(capi.LoopPolicy, field).offset == int(value), field
            seen.add(field)
    assert seen == {f for f, _ in capi.LoopPolicy._fields_}


def test_cpp_mirror_loop_policy_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "loop_policy_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)


@pytest.mark.parametrize("name", ["set_loop_policy", "loop_edges"])
def test_python_mirrors_exist(name):
    from loam_livox_b200.registration import Laser_mapping
    assert callable(getattr(Laser_mapping, name))
