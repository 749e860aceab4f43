"""GPU tests of the solver kernel (lm_solve_kernel, csrc/solve.cu) over caller-given residual blocks (ll_set_blocks), against the
extended-precision reference of tests/solver_reference.py and the oracle.

Bar for the normal equations, the cost and the L1 norms: |gpu - ref| <= K u S per entry, u = 2^-53, S the reference's a-priori rounding scale,
K = 256.  K bounds the depth of the fp64 rounding chain between the exact value and any output entry, in units of u S:
  - per block, the closed form (fast path) or the chain rule (*_mb path): two cross products of the rotation, the staging rotation into the
    last pose's frame, d = y + t - a', the projection, G, the Huber weight (sqrt, divide) and the products of the sum terms: about 30 dependent
    roundings, each bounded by u times a magnitude S covers;
  - per thread, the serial sum over at most 12 tiles (14 on the deblur path);
  - the warp's transposing butterfly: 5 levels;
  - the CTA: 8 warps summed in order;
  - the grid: each of 8 groups sums its rows in 4 chains of at most 5 (132 rows), 2 combines, then 8 groups in order.
That is at most about 30 + 14 + 5 + 8 + 5 + 2 + 8 = 72 < K / 3: the bar holds with a factor of 3 to spare and is not fitted to observed errors.
The oracle is held to the same bar where it is checked; its formula (world frame) rounds differently, which is why both are compared with the
reference instead of with each other at 1e-9.
"""
import ctypes as C

import numpy as np
import pytest

import solver_reference as R
from loam_livox_b200 import capi

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not R.EXTENDED, reason="long double is plain double on this platform")]

K = 256
U = R.EPS64
BOUND = float(np.float32(0.3))   # fill_state: bound = (double)(float)para_max_speed


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _reg(ctx, ql=(1, 0, 0, 0), tl=(0, 0, 0), deblur=False, **kw):
    from loam_livox_b200.registration import Point_cloud_registration
    st = dict(q_w_last=list(ql), t_w_last=list(tl), q_w_curr=list(ql), t_w_curr=list(tl), if_motion_deblur=int(deblur), minimum_pt_time_stamp=0.0,
              maximum_pt_time_stamp=1.0)
    st.update(kw)
    return Point_cloud_registration(ctx, **st)


def _stage(reg, B, holes=None):
    """Blocks B (oracle layout) into the library's slots: type + 1, 0 where `holes`; intensity = blur factor (refine_blur over [0, 1] is exact)."""
    typ = B[:, 0].astype(np.int32) + 1
    if holes is not None:
        typ[holes] = 0
    p = np.zeros((B.shape[0], 4), np.float32)
    p[:, :3] = B[:, 1:4]
    p[:, 3] = np.where(np.isnan(B[:, 10]), 0.0, B[:, 10])
    reg.set_blocks(typ, p, B[:, 4:7], B[:, 7:10])
    return typ


def _within(got, ref, key, skey):
    err = np.abs(np.asarray(got, np.longdouble) - ref[key])
    ratio = np.where(err > 0, err / np.maximum(U * ref[skey], np.finfo(np.longdouble).tiny), 0)   # S = 0 (a zero-residual gradient) allows no error
    return bool(np.all(err <= K * U * ref[skey])), float(np.max(ratio))


def _check_ne(reg, x, ref):
    H, g, cost = reg.normal_equations(x)
    bad = {}
    for name, got, key, sk in (("H", H, "H", "S_H"), ("g", g, "g", "S_g"), ("cost", cost, "cost", "S_cost")):
        ok, worst = _within(got, ref, key, sk)
        if not ok:
            bad[name] = worst
    return (H, g, cost), bad


def _tiled(Bu, M, rng, hole_frac=0.1):
    """M slots cycling through the distinct blocks Bu, random type-0 holes; returns (B, holes, multiplicity of each distinct block)."""
    idx = np.arange(M) % Bu.shape[0]
    holes = rng.random(M) < hole_frac if M > 2 else np.zeros(M, bool)
    mult = np.bincount(idx[~holes], minlength=Bu.shape[0])
    return Bu[idx], holes, mult


# ---------------------------------------------------------------------------------------------- A. slot counts
SIZES = [1, 2, 31, 32, 33, 4223, 4224, 4225, 33791, 33792, 33793, 67585, 200000]


@pytest.mark.parametrize("M", SIZES)
def test_slot_counts_against_the_reference(ctx, M):
    """One tile per CTA up to 132 x 256 slots, then 2..8 tiles; 32-slot tiles on grids smaller than the SM count; lines only, planes only and
    alternating types, each with random holes."""
    kinds = ["line", "plane", "mix"]
    rng = np.random.default_rng(M)
    ql, tl = R.quat_axis_angle((0.3, 0.4, -0.5), 0.6), (4.0, -3.0, 2.0)
    x = np.array([0.01, -0.012, 0.008, 1.0, 0.04, -0.03, 0.02])
    x[:4] /= np.linalg.norm(x[:4])
    for kind in kinds:
        Bu = R.make_blocks(min(M, 2048), rng, kind, ql, tl)
        B, holes, mult = _tiled(Bu, M, rng)
        if mult.sum() == 0:
            continue
        ref = R.normal_equations(Bu, ql, tl, x, 0.1, mult=mult)
        reg = _reg(ctx, ql, tl)
        _stage(reg, B, holes)
        out, bad = _check_ne(reg, x, ref)
        assert not bad, (kind, bad)
        again = reg.normal_equations(x)
        assert all(np.array_equal(a, b) for a, b in zip(out, again)), "two calls differ"


def test_empty_warp_tile_and_cta(ctx):
    """Holes that empty a whole warp, a whole tile and every tile of one CTA (M = 67585: 265 tiles of 256 slots on 132 CTAs, 3 tiles per CTA)."""
    M, sms = 67585, _sms()
    tile = min(256, ((-(-M // sms)) + 31) // 32 * 32)
    tiles = -(-M // tile)
    grid = min(tiles, sms)
    rng = np.random.default_rng(3)
    Bu = R.make_blocks(2048, rng, "mix")
    B, _, _ = _tiled(Bu, M, rng, 0.0)
    holes = np.zeros(M, bool)
    holes[32:64] = True                                  # a warp of tile 0
    holes[5 * tile:6 * tile] = True                      # tile 5
    for t in range(7, tiles, grid):                      # every tile of CTA 7
        holes[t * tile:(t + 1) * tile] = True
    mult = np.bincount((np.arange(M) % 2048)[~holes], minlength=2048)
    x = np.array([0.0, 0.0, 0.0, 1.0, 0.01, 0.0, 0.0])
    ref = R.normal_equations(Bu, (1, 0, 0, 0), (0, 0, 0), x, 0.1, mult=mult)
    reg = _reg(ctx)
    _stage(reg, B, holes)
    _, bad = _check_ne(reg, x, ref)
    assert not bad, bad


@pytest.mark.parametrize("deblur", [False, True])
def test_capacity_edge_and_one_slot_past_it(oracle, deblur):
    """The largest slot count the shared memory holds (12 tiles x 256 x 64 B, or 14 x 256 x 56 B on the deblur path, per SM) evaluates within the
    bar, two contexts give the same bits; one slot more is LL_ERR_CAPACITY from ll_set_blocks and ll_register before anything is enqueued, and the
    context then registers exactly as a fresh one."""
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context, Map
    sms = _sms()
    per = 204800 // (256 * (56 if deblur else 64))
    Mmax = sms * 256 * per
    rng = np.random.default_rng(11)
    Bu = R.make_blocks(4096, rng, "mix", blur=np.linspace(-0.2, 1.0, 4096) if deblur else None)
    B, holes, mult = _tiled(Bu, Mmax, rng)
    x = np.array([0.0, 0.01, 0.0, 1.0, 0.02, 0.0, -0.01])
    x[:4] /= np.linalg.norm(x[:4])
    ref = R.normal_equations(Bu, (1, 0, 0, 0), (0, 0, 0), x, 0.1, mult=mult)
    outs = []
    for _ in range(2):
        c = Context(0, max_scan_points=480000, max_features=480000)
        reg = _reg(c, deblur=deblur)
        _stage(reg, B, holes)
        out, bad = _check_ne(reg, x, ref)
        assert not bad, bad
        outs.append(out)
        if len(outs) == 1:
            c.close()
    assert all(np.array_equal(a, b) for a, b in zip(*outs))
    # one slot past the limit
    B1 = np.concatenate([B, B[:1]])
    p = np.zeros((Mmax + 1, 4), np.float32)
    p[:, :3] = B1[:, 1:4]
    typ = B1[:, 0].astype(np.int32) + 1
    a3 = np.ascontiguousarray(B1[:, 4:7], np.float32)
    v3 = np.ascontiguousarray(B1[:, 7:10])
    assert c._lib.ll_set_blocks(c.h, C.byref(reg.state), Mmax + 1, typ.ctypes.data, p.ctypes.data, a3.ctypes.data, v3.ctypes.data) == capi.LL_ERR_CAPACITY
    mc, ms = S.make_map(500, 4500)
    pose = S.default_pose()
    fc, fs = S.make_features(200, Mmax + 1 - 200, pose)
    m = Map(c, mc, ms)
    st = capi.default_reg_state(q_w_last=pose.q, t_w_last=pose.t, q_w_curr=pose.q, t_w_curr=pose.t, if_motion_deblur=int(deblur))
    res = capi.RegResult()
    assert c._lib.ll_register(c.h, m.h, fc.ctypes.data, fc.shape[0], fs.ctypes.data, fs.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(st),
                              C.byref(res)) == capi.LL_ERR_CAPACITY
    # the same context registers as a fresh one afterwards
    fc2, fs2 = fc[:150], fs[:1500]
    guess = S.perturb_pose(pose, np.random.default_rng(2))
    st2 = capi.default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t, if_motion_deblur=int(deblur))

    def run(cc, mm):
        r = capi.RegResult()
        cc.check(cc._lib.ll_register(cc.h, mm.h, fc2.ctypes.data, fc2.shape[0], fs2.ctypes.data, fs2.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST,
                                     C.byref(st2), C.byref(r)))
        return (r.status, r.icp_iterations, r.num_residual_blocks, tuple(r.q_w_curr), tuple(r.t_w_curr), r.final_cost)
    got = run(c, m)
    m.release()
    c.close()
    f = Context(0, max_scan_points=50000, max_features=50000)
    fm = Map(f, mc, ms)
    assert run(f, fm) == got
    fm.release()
    f.close()


# ---------------------------------------------------------------------------------------------- B. geometry of the closed form
POSES = {
    "identity": ((1, 0, 0, 0), (0, 0, 0)),
    "rot90x": (R.quat_axis_angle((1, 0, 0), np.pi / 2), (1, 2, 3)),
    "rot90y": (R.quat_axis_angle((0, 1, 0), np.pi / 2), (1, 2, 3)),
    "rot90z": (R.quat_axis_angle((0, 0, 1), np.pi / 2), (1, 2, 3)),
    "rot180": (R.quat_axis_angle((0.6, 0, 0.8), np.pi), (-3, 1, 2)),
    "neg_q": (-R.quat_axis_angle((0.2, 1, -0.4), 0.7), (1, 2, 3)),
}


@pytest.mark.parametrize("pose", list(POSES))
@pytest.mark.parametrize("far", [0.0, 1e3, 1e4, 1e5])
def test_geometry_against_the_reference(ctx, oracle, pose, far):
    """Last poses at 90 deg about each axis, 180 deg (w = 0), given as -q; t_last and anchors up to 1e5 m from the origin with features to 200 m;
    directions / normals of length 0.5, 1 and 2; trial points x and -x (the same rotation: the same normal equations)."""
    ql, tl = POSES[pose]
    tl = np.asarray(tl, np.float64) + far * np.array([1.0, -0.7, 0.3])
    rng = np.random.default_rng(int(far) + len(pose))
    B = np.concatenate([R.make_blocks(1500, rng, "mix", ql, tl, radius=200.0 if far else 30.0, vnorm=vn) for vn in (0.5, 1.0, 2.0)])
    reg = _reg(ctx, ql, tl)
    _stage(reg, B)
    x = np.array([0.02, -0.01, 0.015, 1.0, 0.05, -0.04, 0.03])
    x[:4] /= np.linalg.norm(x[:4])
    ref = R.normal_equations(B, ql, tl, x, 0.1)
    for xs in (x, np.concatenate([-x[:4], x[4:]])):
        _, bad = _check_ne(reg, xs, ref)
        assert not bad, (xs[3], bad)
    oc, og, oH = oracle.evaluate(B, ql, tl, x)
    worst = {k: _within(v, ref, kk, sk)[1] for k, v, kk, sk in (("H", oH, "H", "S_H"), ("g", og, "g", "S_g"), ("cost", oc, "cost", "S_cost"))}
    if max(worst.values()) > K:
        print(f"oracle outside its bar at {pose} / {far:g} m: {worst}")   # reported, not a library defect


# ---------------------------------------------------------------------------------------------- C. loss edges
def test_huber_boundary_tail_zero_and_huge_residuals(ctx):
    """huber_a = 0.125: |r|^2 == a^2 exactly, one ulp above and below; blocks that are all in the tail; exactly zero residuals; 1e6 m."""
    from test_solver_reference import huber_boundary_blocks, zero_residual_blocks
    rng = np.random.default_rng(5)
    Bb, shifts = huber_boundary_blocks(512)
    sets = [(Bb, np.array([0, 0, 0, 1.0, 0, 0, dz])) for dz in shifts]
    sets.append((R.make_blocks(3000, rng, "mix", offset=(0.5, 5.0)), np.array([0, 0, 0, 1.0, 0.01, 0, 0])))
    sets.append((zero_residual_blocks(600), np.array([0, 0, 0, 1.0, 0, 0, 0])))
    sets.append((R.make_blocks(600, rng, "mix", offset=(1e6, 1e6)), np.array([0, 0, 0, 1.0, 0, 0, 0])))
    for i, (B, x) in enumerate(sets):
        reg = _reg(ctx, huber_a=0.125)
        _stage(reg, B)
        ref = R.normal_equations(B, (1, 0, 0, 0), (0, 0, 0), x, 0.125)
        _, bad = _check_ne(reg, x, ref)
        assert not bad, (i, bad)


# ---------------------------------------------------------------------------------------------- D. the fused ICP iteration
def _fused_case(name, rng):
    if name == "perfect":
        return R.make_blocks(5000, rng, "mix", offset=(0.0, 0.0)), None
    if name == "duplicates":
        Bu = R.make_blocks(3000, rng, "mix")
        return Bu[np.arange(12000) % 3000], None
    if name == "multi_tile":
        return R.make_blocks(40000, rng, "mix", offset=(0.0, 0.4)), None
    return R.make_blocks(2000, rng, "mix", offset=(0.0, 0.4)), None


@pytest.mark.parametrize("name", ["noisy", "perfect", "duplicates", "multi_tile"])
def test_fused_iteration(ctx, oracle, name):
    """ll_solve_fused: the per-slot L1 norms (prerun 0: at the start point) within the reference bar; threshold and distinct count equal to the
    np.unique order statistic of the kernel's own L1 vector, the kept count to count(l1 <= threshold), exactly; with prerun 2 the iterations, kept
    count and x equal the composition of the oracle's pieces."""
    rng = np.random.default_rng(len(name))
    B, _ = _fused_case(name, rng)
    M = B.shape[0]
    holes = np.zeros(M, bool)
    holes[7::97] = True
    ql, tl = R.quat_axis_angle((1, 2, 3), 0.4), (2.0, 1.0, -1.0)
    # the blocks were made around the identity increment; move the start point off it
    x0 = np.array([0.004, -0.003, 0.002, 1.0, 0.03, -0.02, 0.01])
    x0[:4] /= np.linalg.norm(x0[:4])
    reg = _reg(ctx, ql, tl)
    _stage(reg, B, holes)
    Bv = B[~holes]
    ratio, dis = 0.8, 0.02
    # L1 norms at the start point against the reference
    x, thr, nd, nk, l1, its = reg.solve_fused(x0, 0, 50)
    ref = R.normal_equations(Bv, ql, tl, x0, 0.1)
    assert np.all(np.isinf(l1[holes])) and its[0] == 0
    err = np.abs(l1[~holes].astype(np.longdouble) - ref["l1"])
    assert np.all(err <= K * U * ref["S_l1"]), float(np.max(err / (U * ref["S_l1"])))
    for prerun in (0, 2):
        x, thr, nd, nk, l1, its = reg.solve_fused(x0, prerun, 50)
        u = np.unique(l1[np.isfinite(l1)])
        assert nd == len(u) and thr == max(dis, u[min(int(ratio * len(u)), len(u) - 1)])
        assert nk == int(np.sum(l1 <= thr))
        x1, s1 = oracle.solve(Bv, ql, tl, x0, prerun, bound=BOUND)
        _, _, _, r, _ = oracle.evaluate(Bv, ql, tl, x1, want_full=True)
        ol1 = np.abs(r).reshape(-1, 3).sum(1)
        ou = np.unique(ol1)
        othr = max(dis, ou[min(int(ratio * len(ou)), len(ou) - 1)])
        keep = ol1 <= othr
        x2, s2 = oracle.solve(Bv[keep], ql, tl, x1, 50, bound=BOUND)
        assert its == (int(s1["iterations"]), int(s2["iterations"])), (its, s1, s2)
        assert nk == int(keep.sum()) and abs(thr - othr) <= 1e-9 * othr
        assert np.allclose(x, x2, rtol=0, atol=1e-9), np.abs(x - x2).max()
    if name == "perfect":   # every L1 norm exactly 0: the threshold is inliner_dis and every block stays
        from test_solver_reference import zero_residual_blocks
        Z = zero_residual_blocks(3000)
        reg = _reg(ctx)
        _stage(reg, Z, holes[:3000])
        x, thr, nd, nk, l1, its = reg.solve_fused(np.array([0, 0, 0, 1.0, 0, 0, 0]), 2, 50)
        assert np.all(l1[~holes[:3000]] == 0) and (thr, nd, nk) == (dis, 1, 3000 - holes[:3000].sum())


# ---------------------------------------------------------------------------------------------- E. LM edges
def _lm_cases(rng):
    ql, tl = R.quat_axis_angle((0, 0, 1), 0.3), (1.0, 2.0, 0.0)
    same_n = R.make_blocks(500, rng, "plane", ql, tl)
    same_n[:, 7:10] = [0.0, 0.6, 0.8]
    par = R.make_blocks(500, rng, "line", ql, tl)
    par[:, 7:10] = [0.48, 0.6, 0.64]
    one = R.make_blocks(1, rng, "plane", ql, tl)
    zero = R.make_blocks(400, rng, "mix", ql, tl, offset=(0.0, 0.0))
    zero[:, 4:7] = zero[:, 1:4]
    zero_ql, zero_tl = (1, 0, 0, 0), (0, 0, 0)
    bnd = R.make_blocks(800, rng, "mix", ql, tl, true_x=[0, 0, 0, 1, 0.05, 0.0, -0.05], offset=(0.0, 0.02))
    return [("bound", bnd, ql, tl, 0.005, (50,)), ("one_normal", same_n, ql, tl, 0.3, (50,)), ("parallel_lines", par, ql, tl, 0.3, (50,)),
            ("one_block", one, ql, tl, 0.3, (50,)), ("zero_residual", zero, zero_ql, zero_tl, 0.3, (50,)),
            ("max_iter", R.make_blocks(800, rng, "mix", ql, tl, true_x=[0.01, 0, 0, 1, 0.1, 0, 0]), ql, tl, 0.3, (1, 2))]


@pytest.mark.parametrize("case", range(6))
def test_lm_edges_against_the_oracle(ctx, oracle, case):
    name, B, ql, tl, speed, iters = _lm_cases(np.random.default_rng(17))[case]
    reg = _reg(ctx, ql, tl, para_max_speed=speed)
    _stage(reg, B)
    bound = float(np.float32(speed))
    x0 = [0, 0, 0, 1, 0, 0, 0]
    # a cost that converged to the rounding floor of r (one block: |r| ~ 1e-11 m) has no relative accuracy: its absolute floor is
    # |r| times the rounding of d = pt_tr - a, K u (|a| + |t_last| + |p|) per block
    A = np.max(np.linalg.norm(B[:, 4:7], axis=1) + np.linalg.norm(tl) + np.linalg.norm(B[:, 1:4], axis=1) + 1.0)
    for it in iters:
        xg, ic, fc, n = reg.solve(x0, it)
        xo, so = oracle.solve(B, ql, tl, x0, it, bound=bound)
        assert n == int(so["iterations"]), (name, n, so)
        for got, want in ((ic, so["initial_cost"]), (fc, so["final_cost"])):
            assert abs(got - want) <= 1e-10 * abs(want) + K * U * A * np.sqrt(2 * abs(want) * B.shape[0]), (name, got, want)
        assert np.allclose(xg, xo, rtol=0, atol=1e-9), (name, np.abs(xg - xo).max())
        if name == "bound":
            assert np.max(np.abs(xg[4:])) == bound   # the bound is active


# ---------------------------------------------------------------------------------------------- F. deblur: Eigen's slerp at its lerp switch
def _slerp_x(w, sign=1.0):
    u = np.array([0.3, -0.5, 0.8])
    u = u / np.linalg.norm(u) * np.sqrt(max(0.0, 1.0 - w * w))
    return np.concatenate([u, [w], [0.02, -0.01, 0.03]]) * np.array([sign] * 4 + [1] * 3)


W_CASES = [("w1", 1.0), ("1-2^-53", 1 - 2.0 ** -53), ("lerp 1-2^-52", 1 - 2.0 ** -52), ("slerp 1-3*2^-53", 1 - 3 * 2.0 ** -53),
           ("rot1e-7", np.cos(0.5e-7)), ("rot1e-6", np.cos(0.5e-6)), ("rot0.05", np.cos(0.025))]


@pytest.mark.parametrize("wc", W_CASES, ids=[w[0] for w in W_CASES])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_deblur_slerp_edges(ctx, oracle, wc, sign):
    """*_mb functors with |w| = 1, 1 - 2^-53, 1 - 2^-52 (lerp), 1 - 3 2^-53 (slerp), rotations of 1e-7 and 1e-6 rad, w < 0, blur factors 0, 1,
    negative and in between.  GPU against the oracle, within K u S plus K times the spread between the reference evaluated in fp64 and in
    extended precision (the conditioning of the formula itself in that band)."""
    name, w = wc
    x = _slerp_x(w, sign)
    ql, tl = R.quat_axis_angle((1, 0, 1), 0.3), (1.0, -1.0, 0.5)
    rng = np.random.default_rng(23)
    blur = np.concatenate([[0.0, 1.0, -0.25], np.linspace(-0.1, 0.95, 509)])
    B = R.make_blocks(512, rng, "mix", ql, tl, blur=blur)
    reg = _reg(ctx, ql, tl, deblur=True)
    _stage(reg, B)
    ref = R.normal_equations(B, ql, tl, x, 0.1)
    r64 = R.normal_equations(B, ql, tl, x, 0.1, h=1e-150, dtype=np.complex128)
    H, g, cost = reg.normal_equations(x)
    oc, og, oH = oracle.evaluate(B, ql, tl, x)
    report = {}
    for nm, gv, ov, key, sk in (("H", H, oH, "H", "S_H"), ("g", g, og, "g", "S_g"), ("cost", cost, oc, "cost", "S_cost")):
        spread = np.abs(np.asarray(r64[key], np.longdouble) - ref[key])
        bar = K * (U * ref[sk] + spread)
        assert np.all(np.abs(np.asarray(gv, np.longdouble) - np.asarray(ov, np.longdouble)) <= bar), (nm, name)
        report[nm] = (float(np.max(np.abs(gv - ref[key]) / np.abs(ref[key]).max())), float(np.max(np.abs(ov - ref[key]) / np.abs(ref[key]).max())))
    print(f"{name} sign {sign:+g}: max |gpu - ref| / max|ref|, |oracle - ref| / max|ref|: {report}")
