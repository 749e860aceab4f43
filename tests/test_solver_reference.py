"""CPU pins of the extended-precision solver reference (tests/solver_reference.py) before any GPU test relies on it: the reference equals the
oracle's Jets (oracle.evaluate) within the rounding bar K u S of tests/test_gpu_solver.py, and its complex-step Jacobians equal central
differences, on random blocks, on the committed golden blocks and on every geometry and loss edge the GPU tests use."""
import os

import numpy as np
import pytest

import solver_reference as R

pytestmark = pytest.mark.skipif(not R.EXTENDED, reason="long double is plain double on this platform")

K = 256   # the GPU tests' constant; justified in tests/test_gpu_solver.py
U = R.EPS64
GOLD = os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz")


def _x(rot, axis=(0.3, -0.5, 0.8), t=(0.05, -0.04, 0.03), neg=False):
    q = R.quat_axis_angle(axis, rot)
    x = np.array([q[1], q[2], q[3], q[0], *t])
    if neg:
        x[:4] = -x[:4]
    return x


# (name, q_last, t_last, trial x, block kwargs): the geometry and loss edges of tests/test_gpu_solver.py
CASES = [
    ("identity", (1, 0, 0, 0), (0, 0, 0), _x(0.02), {}),
    ("rot90x", R.quat_axis_angle((1, 0, 0), np.pi / 2), (0, 0, 0), _x(0.02), {}),
    ("rot180", R.quat_axis_angle((0.6, 0, 0.8), np.pi), (3, -2, 1), _x(0.02), {}),
    ("neg_last", -R.quat_axis_angle((0.2, 1, -0.4), 0.7), (1, 2, 3), _x(0.02), {}),
    ("neg_trial", R.quat_axis_angle((0.2, 1, -0.4), 0.7), (1, 2, 3), _x(0.02, neg=True), {}),
    ("far1e5", R.quat_axis_angle((0, 0, 1), 2.0), (1e5, -7e4, 3e4), _x(0.01), dict(radius=200.0)),
    ("vnorm05", (1, 0, 0, 0), (10, 0, 0), _x(0.02), dict(vnorm=0.5)),
    ("vnorm2", R.quat_axis_angle((1, 1, 0), 1.0), (10, 0, 0), _x(0.02), dict(vnorm=2.0)),
    ("tail", (1, 0, 0, 0), (0, 0, 0), _x(0.0), dict(offset=(0.5, 5.0))),
    ("far_res", (1, 0, 0, 0), (0, 0, 0), _x(0.0), dict(offset=(1e6, 1e6))),
    ("deblur", R.quat_axis_angle((0, 1, 0), 0.5), (5, 5, 5), _x(0.05), dict(blur=np.linspace(-0.3, 1.0, 64))),
    ("deblur_neg", R.quat_axis_angle((0, 1, 0), 0.5), (5, 5, 5), _x(0.05, neg=True), dict(blur=np.linspace(-0.3, 1.0, 64))),
]


def _check_vs_oracle(oracle, B, ql, tl, x, a):
    ref = R.normal_equations(B, ql, tl, x, a)
    oc, og, oH = oracle.evaluate(B, ql, tl, x, huber_a=a)
    bad = []
    for name, got, want, S in (("H", oH, ref["H"], ref["S_H"]), ("g", og, ref["g"], ref["S_g"]), ("cost", oc, ref["cost"], ref["S_cost"])):
        err = np.abs(np.asarray(got, np.longdouble) - want)
        if not np.all(err <= K * U * S):
            bad.append((name, float(np.max(err / (U * S)))))
    return ref, bad


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_reference_matches_the_oracle_and_central_differences(oracle, case):
    name, ql, tl, x, kw = case
    rng = np.random.default_rng(len(name))
    B = R.make_blocks(64, rng, "mix", ql, tl, **kw)
    a = 0.125 if name in ("tail", "far_res") else 0.1
    ref, bad = _check_vs_oracle(oracle, B, ql, tl, x, a)
    assert not bad, bad
    # complex step against central differences of the same long-double expression (h = 1e-7 in the tangent space)
    h = 1e-7
    for c in range(6):
        dp, dm = [0.0] * 6, [0.0] * 6
        dp[c], dm[c] = h, -h
        rp = R.residuals(B, ql, tl, *R.plus(x, dp, R.LD), R.LD)[0]
        rm = R.residuals(B, ql, tl, *R.plus(x, dm, R.LD), R.LD)[0]
        cd = (rp - rm) / (2 * R.LD(h))
        scale = np.maximum(1.0, np.abs(ref["J"][:, :, c]))
        assert np.all(np.abs(cd - ref["J"][:, :, c]) <= 1e-7 * scale * (1 + np.abs(B[:, 1:4]).max())), (name, c)


def test_reference_matches_the_golden_evaluation(oracle):
    """The committed golden blocks (golden_small: features, map and guess) and the normal equations stored with them."""
    g = np.load(GOLD)
    p = oracle.default_params(q_w_last=g["guess_q"], t_w_last=g["guess_t"], q_w_curr=g["guess_q"], t_w_curr=g["guess_t"])
    B, _, _, _ = oracle.build_blocks(g["map_corner"], oracle.KdTree(g["map_corner"]), g["map_surf"], oracle.KdTree(g["map_surf"]),
                                     g["feat_corner"], g["feat_surf"], p)
    assert B.shape[0] == int(g["n_blocks"])
    ref, bad = _check_vs_oracle(oracle, B, g["guess_q"], g["guess_t"], g["eval_x"], 0.1)
    assert not bad, bad
    for got, want, S in ((g["eval_H"], ref["H"], ref["S_H"]), (g["eval_g"], ref["g"], ref["S_g"]), (g["eval_cost"], ref["cost"], ref["S_cost"])):
        assert np.all(np.abs(np.asarray(got, np.longdouble) - want) <= K * U * S)


def huber_boundary_blocks(n=32):
    """Plane blocks whose residual at identity is exactly huber_a = 0.125 (|r|^2 == a^2, representable), and the trial translations that move it
    one ulp above (2^-55) and one below (-2^-56)."""
    B = np.zeros((n, 11))
    B[:, 0] = 1
    B[:, 1:4] = np.arange(3 * n).reshape(n, 3) % 7 - 3.0     # features at small integers
    B[:, 4:7] = B[:, 1:4]
    B[:, 6] -= 0.125                                          # anchor 0.125 below the feature along z
    B[:, 9] = 1.0                                             # normal e_z
    B[:, 10] = np.nan
    return B, (0.0, 2.0 ** -55, -(2.0 ** -56))


def zero_residual_blocks(n=32):
    """Axis-aligned lines and planes through their features: r = 0 exactly at identity."""
    B = np.zeros((n, 11))
    B[:, 0] = np.arange(n) % 2
    B[:, 1:4] = (np.arange(3 * n).reshape(n, 3) % 11 - 5.0) * 0.5
    B[:, 4:7] = B[:, 1:4]
    B[np.arange(n), 7 + np.arange(n) % 3] = 1.0
    B[:, 10] = np.nan
    return B


def test_reference_at_the_huber_boundary_and_zero_residuals(oracle):
    B, shifts = huber_boundary_blocks()
    for dz in shifts:
        x = np.array([0, 0, 0, 1, 0, 0, dz])
        ref, bad = _check_vs_oracle(oracle, B, (1, 0, 0, 0), (0, 0, 0), x, 0.125)
        assert not bad, (dz, bad)
        sq = (ref["r"] ** 2).sum(1)
        assert np.all(sq == R.LD(0.125) ** 2) if dz == 0 else np.all((sq > R.LD(0.125) ** 2) == (dz > 0))
    Z = zero_residual_blocks()
    ref, bad = _check_vs_oracle(oracle, Z, (1, 0, 0, 0), (0, 0, 0), np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.125)
    assert not bad and ref["cost"] == 0 and np.all(ref["r"] == 0) and np.any(ref["H"] != 0)
