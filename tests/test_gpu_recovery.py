"""Tracking-loss recovery inside the streaming mapper (ll_mapper_set_recovery, ll_mapper_recovery_read, ll_mapper_recovery_last_inputs;
DESIGN.md §4.3.2): recovery on but idle changes nothing, a kidnapped sensor is held back, found and tracked again through the single and the
sequence calls, every attempt is ll_relocalize_field of its own inputs, held-back steps freeze the map, a view the map does not cover never
moves the pose, and bad configurations are refused without a change."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu

N = 24000
STAT_INTS = ("n_corner", "n_surf", "map_corner", "map_surf", "cells_in_fov_corner", "cells_in_fov_surf", "appended_corner", "appended_surf")
K_JUMP = 160   # the kidnap: 1 m back, 2 m to the side, 15 deg to the right (a view the map covers; tests/recovery_oracle.py)
KIDNAP = (np.array([-1.0, -2.0, 0.0]), -15.0)


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=60000, max_features=60000) for _ in range(3)]
    yield cs
    for c in cs:
        c.close()


def _mapper(ctx, mode, p0, pieces=3, **reg):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    st = capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t, **reg)
    return Laser_mapping(ctx, reg=st, pipeline=pipe, matching_mode=mode, maximum_history_size=400)


def _moved(p, offset, yaw_deg):
    return S.Pose(S.quat_mul(p.q, S.quat_from_euler(0.0, 0.0, np.radians(yaw_deg))), p.t + offset)


def _stream(n, seed, jump=None, turn=None):
    """C3-style poses; from scan jump on the sensor is kidnapped (KIDNAP applied to the rest of the path); scans in `turn` (a range) look the
    other way (yaw + 180 deg, a view the map does not cover)."""
    poses = S.trajectory(n_scans=n, n_static=4, speed=1.0)
    if jump is not None:
        poses = poses[:jump] + [_moved(p, *KIDNAP) for p in poses[jump:]]
    if turn is not None:
        poses = [_moved(p, np.zeros(3), 180.0) if k in turn else p for k, p in enumerate(poses)]
    return poses, [S.make_scan(N, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(n)]


def _b(x):
    return np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()


def _entry(res):
    from loam_livox_b200 import capi
    return tuple(_b(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms"))


def _stats(st):
    return tuple(getattr(st, f) for f in STAT_INTS)


def _log_key(e):
    from loam_livox_b200 import capi
    return tuple(_b(getattr(e, f)) for f, _ in capi.RecoveryStep._fields_ if not f.startswith("ms_"))


def _section(img, k):
    off, length = struct.unpack_from("<QQ", img, 24 + 16 * k)
    return img[off:off + length]


def _map_sections(img):
    from loam_livox_b200 import capi
    return tuple(_section(img, k) for k in (capi.LL_IMAGE_HISTORY_CORNER, capi.LL_IMAGE_HISTORY_SURF, capi.LL_IMAGE_CELLS_CORNER, capi.LL_IMAGE_CELLS_SURF))


def _err(q, t, p):
    return np.linalg.norm(t - p.t), np.degrees(S.quat_angle(q, p.q))


# ---------------------------------------------------------------------------------------------- 1. off and idle change nothing
@pytest.mark.parametrize("mode", [0, 1])
def test_idle_recovery_changes_nothing(ctxs, mode):
    from loam_livox_b200 import capi
    poses, raws, stamps = _stream(200, S.SEED + 2100)
    a, b = _mapper(ctxs[0], mode, poses[0]), _mapper(ctxs[1], mode, poses[0])
    b.set_recovery()
    l0, l1 = ctxs[0].launches(), ctxs[1].launches()
    for lo in range(0, 200, 50):   # the sequence call in chunks of 50 scans, saving the image between them
        ra = a.process_new_scans(raws[lo:lo + 50], stamps[lo:lo + 50])
        rb = b.process_new_scans(raws[lo:lo + 50], stamps[lo:lo + 50])
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
        assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]
        assert a.save() == b.save()
    qa, ta, fa = a.pose()
    qb, tb, fb = b.pose()
    assert qa.tobytes() == qb.tobytes() and ta.tobytes() == tb.tobytes() and fa == fb
    assert ctxs[0].launches() - l0 == ctxs[1].launches() - l1
    log, dropped = b.recovery_log()
    assert dropped == 0 and len(log) == 200   # one entry per step (the first ones do not register: no map, then the :199 gate)
    assert all(e.bad == capi.LL_BAD_NONE and e.attempted == 0 and e.appended == 1 and e.state_after == capi.LL_TRACKING for e in log)
    assert [e.frame_index for e in log] == list(range(200))
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- 2, 3, 6. kidnap
def _identity(ctx, lm, e):
    """The attempt behind log entry e is ll_relocalize_field of the hook's inputs on a fresh context against the mapper's whole map."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import RelocField
    inp = lm.recovery_last_inputs()
    cfg = lm.recovery_cfg
    m = lm.whole_map()
    f = RelocField(ctx, m, cfg.res, cfg.trunc, cfg.max_hypotheses)
    K = inp["coarse"].max_candidates
    cand, res, status = (capi.RelocFieldCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    p = [np.ascontiguousarray(inp[k]) for k in ("score_corner", "score_surf", "corner", "surf")]
    assert [x.shape[0] for x in p] == [e.n_score[0], e.n_score[1], p[2].shape[0], p[3].shape[0]]
    ctx.check(ctx._lib.ll_relocalize_field(ctx.h, m.h, f.h, p[0].ctypes.data, p[0].shape[0], p[1].ctypes.data, p[1].shape[0], p[2].ctypes.data, p[2].shape[0],
                                           p[3].ctypes.data, p[3].shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(inp["coarse"]), C.byref(inp["fine"]),
                                           C.byref(inp["tmpl"]), cand, res, status, C.byref(n), C.byref(best)))
    assert (n.value, best.value) == (e.n_cand, e.best)
    assert [inp["coarse"].nt[i] for i in range(3)] == list(e.nt) and inp["coarse"].n_rot == e.n_yaw
    if best.value >= 0:
        r = res[best.value]
        T2 = cfg.trunc * cfg.trunc
        assert np.array(r.q_w_curr).tobytes() == np.array(e.q_wxyz).tobytes() and np.array(r.t_w_curr).tobytes() == np.array(e.t).tobytes()
        assert _b(r.inlier_threshold) == _b(e.inlier_threshold)
        assert cand[best.value].verify_score / (T2 * (e.n_score[0] + e.n_score[1])) == e.verify_fraction
    f.close(); m.release()


def _check_kidnap(log, results, poses, ref, lm_pose_after, label):
    """log: the entries from the jump on; results: (RegResult, stats) per step from the jump on; ref: the never-jumped mapper's poses."""
    from loam_livox_b200 import capi
    lost_after = 3
    first_bad = next(i for i, e in enumerate(log) if e.bad != capi.LL_BAD_NONE)
    assert first_bad == 0, label   # the jump itself is the first bad step
    lost_at = next(i for i, e in enumerate(log) if e.state_after == capi.LL_LOST)
    assert lost_at == lost_after - 1, label   # declared within lost_after steps
    adopted = [i for i, e in enumerate(log) if e.adopted]
    assert adopted and adopted[0] <= lost_at + 2, (label, [(e.bad, e.attempted, e.attempt_status, e.n_cand, e.best, e.verify_fraction, e.inlier_threshold) for e in log[:8]])
    rec = adopted[0]
    for i in range(rec + 1):   # nothing appended from the first bad step to the recovering one
        assert log[i].appended == 0 and results[i][1].appended_corner == 0 and results[i][1].appended_surf == 0, (label, i)
    for i in range(rec + 1, len(log)):   # tracked again: every later step good and appended, within 0.05 m / 0.5 deg beyond the reference's drift
        e = log[i]
        assert e.bad == capi.LL_BAD_NONE and e.appended == 1 and results[i][0].status == 1, (label, i)
        q, t = np.array(results[i][0].q_w_curr), np.array(results[i][0].t_w_curr)
        e_t, e_r = _err(q, t, poses[i])
        f_t, f_r = ref[i]
        assert e_t < f_t + 0.05 and e_r < f_r + 0.5, (label, i, e_t, f_t, e_r, f_r)
    return rec


@pytest.fixture(scope="module")
def kidnap_data():
    n = K_JUMP + 12
    seed = S.SEED + 2300
    poses, raws, stamps = _stream(n, seed, jump=K_JUMP)
    ref_poses, ref_raws, _ = _stream(n, seed)
    return poses, raws, stamps, ref_poses, ref_raws


@pytest.fixture(scope="module")
def kidnap_ref(ctxs, kidnap_data):
    """Per mode, the error of a mapper that never jumped at every scan from the jump on."""
    poses, _, stamps, ref_poses, ref_raws = kidnap_data
    out = {}
    for mode in (0, 1):
        lm = _mapper(ctxs[2], mode, poses[0])
        rs = lm.process_new_scans(ref_raws, stamps)
        out[mode] = [_err(np.array(r.q_w_curr), np.array(r.t_w_curr), ref_poses[k]) for k, (r, _) in enumerate(rs)][K_JUMP:]
        lm.close()
    return out


@pytest.mark.parametrize("mode", [0, 1])
def test_kidnap_scans(ctxs, kidnap_data, kidnap_ref, mode):
    poses, raws, stamps, _, _ = kidnap_data
    n = len(raws)
    a, b = _mapper(ctxs[0], mode, poses[0]), _mapper(ctxs[1], mode, poses[0])
    a.recovery_cfg = a.set_recovery()
    b.set_recovery()
    # one by one, checking every attempt against the public call on a fresh context (the mapper is unchanged by the attempt)
    ra, la = [], []
    for k in range(n):
        ra.append(a.process_new_scan(raws[k], stamps[k]))
        log, _ = a.recovery_log()
        la += log
        if k >= K_JUMP and log and log[-1].attempted:
            assert log[-1].attempt_status == 0
            _identity(ctxs[2], a, log[-1])
    # the same through the sequence call, in two calls split inside the loss
    rb = b.process_new_scans(raws[:K_JUMP + 2], stamps[:K_JUMP + 2]) + b.process_new_scans(raws[K_JUMP + 2:], stamps[K_JUMP + 2:])
    lb, dropped = b.recovery_log()
    assert dropped == 0 and len(la) == len(lb) == n
    assert [_log_key(e) for e in la] == [_log_key(e) for e in lb]
    assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb] and [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]
    assert a.save() == b.save()
    off = K_JUMP   # log index of the jump
    rec = _check_kidnap(la[off:], ra[K_JUMP:], poses[K_JUMP:], kidnap_ref[mode], a.pose(), f"mode {mode}")
    assert la[off + rec].frame_index == K_JUMP + rec   # (the registration's frame index)
    a.close(); b.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_kidnap_frames(ctxs, kidnap_data, kidnap_ref, mode):
    """The same stream as one-head frames of one piece each (odom_mode 1): process_new_frame and process_new_frames."""
    poses, raws, stamps, _, _ = kidnap_data
    n = len(raws)
    a, b = _mapper(ctxs[0], mode, poses[0], pieces=1), _mapper(ctxs[1], mode, poses[0], pieces=1)
    a.set_recovery(); b.set_recovery()
    ra = [a.process_new_frame([raws[k]], [stamps[k]], odom_mode=1) for k in range(n)]
    rb = b.process_new_frames([[r] for r in raws], [[t] for t in stamps], odom_mode=1)
    assert all(len(x) == 1 for x in ra) and all(len(x) == 1 for x in rb)
    la, _ = a.recovery_log()
    lb, _ = b.recovery_log()
    assert [_log_key(e) for e in la] == [_log_key(e) for e in lb]
    assert [_entry(x[0][0]) for x in ra] == [_entry(x[0][0]) for x in rb] and a.save() == b.save()
    off = len(la) - (n - K_JUMP)
    _check_kidnap(la[off:], [x[0] for x in ra[K_JUMP:]], poses[K_JUMP:], kidnap_ref[mode], a.pose(), f"frames mode {mode}")
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- 4. held-back steps
@pytest.mark.parametrize("mode", [0, 1])
def test_every_step_held_back(ctxs, mode):
    from loam_livox_b200 import capi
    poses, raws, stamps = _stream(20, S.SEED + 2500)
    lm = _mapper(ctxs[0], mode, poses[0])
    for k in range(10):
        lm.process_new_scan(raws[k], stamps[k])
    lm.set_recovery(max_inlier_threshold=0.0)
    q0, t0, _ = lm.pose()
    his0 = _map_sections(lm.save())[:2]
    for k in range(10, 20):
        r, st = lm.process_new_scan(raws[k], stamps[k])
        assert r.registered == 1 and st.appended_corner == 0 and st.appended_surf == 0
        sec = _map_sections(lm.save())
        if k == 10:   # (in mode 1 the first step's refresh, of scan 9's append, stamps the cells it visits)
            sec0 = sec
        assert sec[:2] == his0 and sec == sec0, k
        q, t, _ = lm.pose()
        assert q.tobytes() == q0.tobytes() and t.tobytes() == t0.tobytes(), k
    log, _ = lm.recovery_log()
    assert len(log) == 10 and all(e.bad != capi.LL_BAD_NONE and e.appended == 0 and e.adopted == 0 for e in log)
    assert [e.attempted for e in log] == [0, 0] + [1] * 8 and [e.state_after for e in log] == [1, 1] + [2] * 8
    assert all(e.attempt_status == 0 for e in log[2:])
    lm.close()


# ---------------------------------------------------------------------------------------------- 5. no way back
@pytest.mark.parametrize("mode", [0, 1])
def test_no_way_back_then_the_mapped_place(ctxs, mode):
    from loam_livox_b200 import capi
    k0, n_turn = 60, 6
    poses, raws, stamps = _stream(k0 + n_turn + 8, S.SEED + 2700, turn=range(k0, k0 + n_turn))
    n = len(raws)
    a, b = _mapper(ctxs[0], mode, poses[0]), _mapper(ctxs[1], mode, poses[0])
    a.set_recovery(); b.set_recovery()
    ra = []
    for k in range(n):
        if k == k0:
            q0, t0, _ = a.pose()
            his0 = _map_sections(a.save())[:2]
        ra.append(a.process_new_scan(raws[k], stamps[k]))
        if k0 <= k < k0 + n_turn:
            q, t, _ = a.pose()
            sec = _map_sections(a.save())
            if k == k0:   # (in mode 1 the first step's refresh stamps the cells it visits)
                sec0 = sec
            assert q.tobytes() == q0.tobytes() and t.tobytes() == t0.tobytes() and sec[:2] == his0 and sec == sec0, k
    rb = b.process_new_scans(raws, stamps)
    la, _ = a.recovery_log()
    lb, _ = b.recovery_log()
    assert [_log_key(e) for e in la] == [_log_key(e) for e in lb] and [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
    turned = la[k0:k0 + n_turn]
    assert all(e.bad != capi.LL_BAD_NONE and e.appended == 0 and e.adopted == 0 for e in turned)
    assert sum(e.attempted for e in turned) == n_turn - 2 and all(e.attempt_status == 0 for e in turned if e.attempted)
    after = la[k0 + n_turn:]
    assert after[0].state_before == capi.LL_LOST and all(e.bad == capi.LL_BAD_NONE and e.appended == 1 and e.state_after == capi.LL_TRACKING for e in after)
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- 7. validation
def test_bad_configurations_are_refused(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import LoamLivoxError
    L = ctxs[0]._lib
    poses, raws, stamps = _stream(14, S.SEED + 2900)
    a, b = _mapper(ctxs[0], 0, poses[0]), _mapper(ctxs[1], 0, poses[0])
    bad = {"max_inlier_threshold": [-1.0, float("nan"), float("inf")], "lost_after": [0], "trunc": [0, 16], "res": [0.0, -0.2, float("nan")],
           "score_leaf": [0.0], "yaw_step_deg": [0.0, 361.0], "t_step": [0.0, float("inf")], "window_base": [-1.0], "window_growth": [float("nan")],
           "max_candidates": [0, 17], "max_hypotheses": [0, (1 << 24) + 1, 100], "fine_yaw_step_deg": [0.0], "fine_t_step": [-0.1],
           "fine_t_half": [-1.0], "min_verify_fraction": [-0.1, 1.5], "reserve_field_voxels": [-1, (1 << 30) + 1], "reserve_whole_map_points": [-1]}
    for k in range(7):
        a.process_new_scan(raws[k], stamps[k]); b.process_new_scan(raws[k], stamps[k])
    for field, values in bad.items():
        for v in values:
            cfg = capi.RecoveryCfg()
            L.ll_mapper_recovery_default(C.byref(cfg))
            setattr(cfg, field, v)
            assert L.ll_mapper_set_recovery(a.h, C.byref(cfg)) == capi.LL_ERR_INVALID, (field, v)
            with pytest.raises(LoamLivoxError):
                a.set_recovery(**{field: v})
    cfg = capi.RecoveryCfg()
    L.ll_mapper_recovery_default(C.byref(cfg))
    assert L.ll_mapper_set_recovery(None, C.byref(cfg)) == capi.LL_ERR_INVALID
    for k in range(7, 14):   # unchanged and usable: recovery still off, the same steps as the untouched mapper
        ra, sa = a.process_new_scan(raws[k], stamps[k])
        rb, sb = b.process_new_scan(raws[k], stamps[k])
        assert _entry(ra) == _entry(rb) and _stats(sa) == _stats(sb)
    assert a.recovery_log() == ([], 0) and a.save() == b.save()
    a.close(); b.close()
