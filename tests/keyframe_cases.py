"""Constructed inputs of the keyframe kernels (ll_keyframe_append / ll_keyframe_analyze / ll_loop_search): point sets that sit on their edges,
shared by the oracle and device tests.  Every cloud is for a map of resolution 1.0 (cells 0.5 wide, cell i spans [0.5 i, 0.5 i + 0.5))."""
import numpy as np

BOX, HALF = np.float32(0.5), np.float32(0.25)
STEP = np.pi / 60
f32 = np.float32


def centre(i, j, k):
    return np.array([i * BOX + HALF, j * BOX + HALF, k * BOX + HALF], np.float32)


def cell_of(pts):
    """The cell indices (i, j, k) of every point, as the map computes them: round((p - half) / box) in float."""
    p = np.asarray(pts, np.float32)[:, :3]
    return np.round(((p - HALF) / BOX).astype(np.float32)).astype(np.int64)


def six_axes(c, x, y, z, reps=(1, 1, 1), centre_pts=0):
    """Pairs +-x, +-y, +-z about c (repeated reps times per axis) and centre_pts copies of c: the mean is c and the covariance diagonal, both
    exact when the offsets are dyadic."""
    c = np.asarray(c, np.float32)
    out = []
    for a, (d, r) in enumerate(zip((x, y, z), reps)):
        e = np.zeros(3, np.float32)
        e[a] = d
        out += [c + e, c - e] * r
    out += [c] * centre_pts
    return np.array(out, np.float32)


def line_cell(c, q, cross=0.03):
    """Nine points along the unit direction q through c, with a small symmetric cross (a collinear set can type as PLANE from rounding noise)."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q)
    e1 = np.cross(q, [1.0, 0, 0] if abs(q[0]) < 0.9 else [0, 1.0, 0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(q, e1)
    offs = [t * q for t in (-0.16, -0.08, 0.0, 0.08, 0.16)] + [cross * e1, -cross * e1, cross * e2, -cross * e2]
    return (np.asarray(c, np.float64) + np.array(offs)).astype(np.float32)


def axis_line(c, axis, n=9):
    """n points exactly on an axis-aligned line through c at dyadic steps, with a dyadic symmetric cross."""
    c = np.asarray(c, np.float32)
    e = np.zeros(3, np.float32)
    e[axis] = 1
    p = [c + f32(t) * e for t in (-0.1875, -0.125, -0.0625, 0.0, 0.0625, 0.125, 0.1875)][: n - 4]
    for b in range(3):
        if b != axis:
            d = np.zeros(3, np.float32)
            d[b] = f32(1 / 128)
            p += [c + d, c - d]
    return np.array(p, np.float32)


def axis_plane(c, normal):
    """A 3 x 3 dyadic grid in the plane through c with the given axis as its normal: the covariance is exactly diagonal, the normal exactly an axis."""
    c = np.asarray(c, np.float32)
    a, b = [x for x in range(3) if x != normal]
    out = []
    for u in (-0.125, 0.0, 0.125):
        for v in (-0.125, 0.0, 0.125):
            p = c.copy()
            p[a] += f32(u)
            p[b] += f32(v)
            out.append(p)
    return np.array(out, np.float32)


def pixel_direction(pi, ti, basis="z"):
    """A unit direction whose image bin is (pi, ti), aimed at the pixel's centre.  basis "z": a keyframe without plane cells or with +z plane
    normals (image frame x' = q_z, y' = q_y, z' = -q_x); "y": +y plane normals (x' = q_y, y' = q_z, z' = q_x)."""
    ph, th = (pi + 0.5) * STEP - np.pi / 2, (ti + 0.5) * STEP - np.pi / 2
    x, y, z = np.cos(th) * np.cos(ph), np.cos(th) * np.sin(ph), np.sin(th)
    return np.array([-z, y, x]) if basis == "z" else np.array([z, x, y])


def _slot(n, block=0):
    """n distinct cells packed in a cube about the origin (negative indices included), or in cube `block` of a 7 x 7 x 7 lattice of 4-cell
    cubes: near the origin the float batch covariance keeps the small cross of a line cell above its rounding noise."""
    idx = np.arange(n)
    if block:
        o = np.array([block % 7 - 3, (block // 7) % 7 - 3, block // 49 - 3]) * 4
        return np.c_[idx % 4, (idx // 4) % 4, idx // 16] + o
    s = max(1, int(np.ceil(n ** (1 / 3))))
    return np.c_[idx % s, (idx // s) % s, idx // (s * s)] - s // 2


# ---- cell statistics and typing ------------------------------------------------------------------------------------------------------------
def cell_cases():
    """name -> list of (cell (i, j, k), points in append order, what it reaches).  One keyframe takes all the cells of a case in one append."""
    rng = np.random.default_rng(17)
    cases = {}
    # 1 to 8 points per cell: a noisy plane, so the type and vector follow every covariance entry (incremental: 5 and 6 points keep the 4-point
    # covariance, the 7th starts the recurrence)
    cs = []
    for n in range(1, 9):
        for rep in range(3):
            c = centre(n, rep, 0)
            p = c + np.c_[rng.uniform(-0.2, 0.2, (n, 2)), rng.normal(0, 0.01, n)]
            cs.append(((n, rep, 0), p.astype(np.float32), f"{n} points"))
    cases["points_1_to_8"] = cs
    # the one-third rule exactly at both boundaries: 17 points with an exact mean and an exactly diagonal covariance (divided by 16), w1 = 3 w0
    # (not PLANE: LINE) and w2 = 3 w1 (not LINE: SPHERE)
    u = f32(1 / 16)
    cs = [((0, 0, 1), six_axes(centre(0, 0, 1), f32(0.21875), u, u, reps=(1, 3, 1), centre_pts=7), "plane tie"),
          ((0, 1, 1), six_axes(centre(0, 1, 1), u, u, f32(0.75) * u, reps=(3, 1, 1), centre_pts=7), "line tie")]
    # one float of a coordinate either side of each boundary: six points on the axes, the flip found by the oracle on the exact coordinates
    for s, (axis, side) in enumerate([(2, "below"), (2, "above"), (1, "below"), (1, "above")]):
        c = centre(s, 2, 1)
        e = one_third_flip(c, axis)[side == "above"]
        cs.append(((s, 2, 1), six_axes(c, *e), f"{'plane' if axis == 2 else 'line'} flip {side}"))
    cases["one_third"] = cs
    # identical points: a covariance of pure rounding noise (all zero; rank 1 with three equal entries; a negative eigenvalue)
    cases["identical_points"] = [((0, 0, 0), np.full((5, 3), 0.3, np.float32), "5 x 0.3: zero covariance"),
                                 ((1, 1, 1), np.full((7, 3), 0.7, np.float32), "7 x 0.7: rank 1, three equal entries"),
                                 ((246, 246, 246), np.full((5, 3), 123.456, np.float32), "5 x 123.456: a negative eigenvalue")]
    # exactly axis-aligned lines and planes (Jacobi exits at once, the vector is exactly an axis); lines along (1, +-1, 0) / sqrt 2 (first of equals)
    cs = [((a, 0, 2), axis_line(centre(a, 0, 2), a), f"line axis {a}") for a in range(3)]
    cs += [((a, 1, 2), axis_plane(centre(a, 1, 2), a), f"plane axis {a}") for a in range(3)]
    c = centre(0, 2, 2)
    cs.append(((0, 2, 2), (c + np.outer(np.arange(-3, 4) * f32(0.03125), [1, 1, 0])).astype(np.float32), "line (1, 1, 0)"))
    c = centre(1, 2, 2)
    cs.append(((1, 2, 2), (c + np.outer(np.arange(-3, 4) * f32(0.03125), [1, -1, 0])).astype(np.float32), "line (1, -1, 0)"))
    cases["axis_aligned"] = cs
    # the 0.75 box centre gate: a plane patch whose mean lies at distance 0.375 exactly, and one float either side (gate_offsets)
    cs = []
    for s, w in enumerate(("below", "at", "above")):   # the search runs on each cell's own coordinates
        c = centre(s, 0, 3)
        d, zs = gate_offsets(c)
        cs.append(((s, 0, 3), gate_patch(c, d, zs[s]), f"gate {w}"))
    cases["centre_gate"] = cs
    # far cells and negative indices: the float batch covariance is all cancellation
    cs = []
    for s, x0 in enumerate((-1e5, -3e4, -1e4, 1e4, 3e4, 1e5)):
        for t in range(8):
            i = int(np.floor(x0 / 0.5)) + t
            c = centre(i, -7 - t, -3)
            kind = t % 3
            if kind == 0:
                p = c + np.c_[rng.uniform(-0.2, 0.2, (30, 2)), rng.normal(0, 0.005, 30)]
            elif kind == 1:
                p = c + np.c_[rng.uniform(-0.2, 0.2, 30), rng.normal(0, 0.005, (30, 2))]
            else:
                p = c + rng.normal(0, 0.08, (30, 3))
            cs.append(((i, -7 - t, -3), np.clip(p, c - 0.24, c + 0.24).astype(np.float32), "far"))
    cases["far_cells"] = cs
    # one cell of 100 000 points: a long serial float sum
    c = centre(-5, 4, 0)
    p = c + np.c_[rng.uniform(-0.2, 0.2, (100000, 2)), rng.normal(0, 0.01, 100000)]
    cases["big_cell"] = [((-5, 4, 0), p.astype(np.float32), "100000 points")]
    return cases


def one_third_flip(c, axis):
    """The extents (x, y, z) of a six-point cell about c either side of where the oracle's type flips, one float of `axis` apart: the plane rule
    (axis 2: l1 / 3 vs l0) or the line rule (axis 1: l2 / 3 vs l1)."""
    import keyframe_reference as K
    e = [f32(0.2), f32(0.1), f32(np.sqrt((f32(0.004) / 3) * 5 / 2))] if axis == 2 else [f32(0.2), f32(0.2 / np.sqrt(3)), f32(0.08)]
    for _ in range(300):
        e[axis] = np.nextafter(e[axis], f32(0), dtype=np.float32)
    t0 = K.cell_type(six_axes(c, *e), c)[0]
    for _ in range(600):
        up = list(e)
        up[axis] = np.nextafter(e[axis], f32(1), dtype=np.float32)
        if K.cell_type(six_axes(c, *up), c)[0] != t0:
            return e, up
        e = up
    raise AssertionError("no flip within 300 floats")


def gate_patch(c, d, z):
    """Eight points of a plane patch at height z whose x, y mean is c + d exactly."""
    q = [(c[0] + d + a, c[1] + d + b, z) for a in (-1 / 64, 1 / 64) for b in (-1 / 64, 1 / 64)] * 2
    return np.array(q, np.float32)


def gate_distance(c, d, z):
    """The float distance the gate tests: |centre - mean| with the oracle's mean of gate_patch(c, d, z)."""
    import keyframe_reference as K
    m = K.cell_type(gate_patch(c, d, z), c)[2]
    e = (c - m).astype(np.float32)
    return np.sqrt(f32(e[0] * e[0] + f32(e[1] * e[1] + e[2] * e[2])))


def gate_offsets(c):
    """(d, [z below, z at, z above]): heights putting the mean of gate_patch at float distance 0.375 from c exactly, and the nearest heights
    either side that do not."""
    for d in (f32(7 / 32), f32(27 / 128), f32(29 / 128), f32(55 / 256), f32(53 / 256), f32(57 / 256)):
        z0 = f32(c[2] + np.sqrt(0.375 ** 2 - 2 * float(d) ** 2))
        for k in range(-40, 41):
            z = z0
            for _ in range(abs(k)):
                z = np.nextafter(z, f32(np.sign(k)), dtype=np.float32)
            if gate_distance(c, d, z) == f32(0.375):
                lo, hi = z, z
                while gate_distance(c, d, lo) == f32(0.375):
                    lo = np.nextafter(lo, f32(-np.inf), dtype=np.float32)
                while gate_distance(c, d, hi) == f32(0.375):
                    hi = np.nextafter(hi, f32(np.inf), dtype=np.float32)
                return d, [lo, z, hi]
    raise AssertionError("no height puts the mean at 0.375 exactly")


def cells_cloud(cells):
    return np.vstack([p for _, p, _ in cells]).astype(np.float32)


# ---- keyframe sizes and growth -------------------------------------------------------------------------------------------------------------
def size_cloud(n_cells, seed=0):
    """One append of n_cells distinct cells: every 7th a noisy plane, every 11th a noisy line (9 points), the rest 1 to 3 points."""
    rng = np.random.default_rng(seed)
    ijk = _slot(n_cells)
    out = []
    for r, (i, j, k) in enumerate(ijk):
        c = centre(i, j, k)
        if r % 7 == 0:
            p = c + np.c_[rng.uniform(-0.2, 0.2, (9, 2)), rng.normal(0, 0.005, 9)]
        elif r % 11 == 0:
            p = c + np.c_[rng.normal(0, 0.005, (9, 2)), rng.uniform(-0.2, 0.2, 9)]
        else:
            p = c + rng.uniform(-0.2, 0.2, (1 + r % 3, 3))
        out.append(p)
    return np.vstack(out).astype(np.float32)


SIZES = (1, 2, 3, 128, 129, 4096, 4097, 65536, 65537)


def growth_appends(seed=1):
    """[(cloud, open keyframes)]: keyframe 0 grows past 4096 cells over five appends, keyframe 1 is open from the third on; a revisited cell is
    held in both incarnations (revisit threshold 2)."""
    rng = np.random.default_rng(seed)
    out = []
    for a in range(5):
        ijk = _slot(1100) + [0, 0, 20 * (a + 1)]
        p = np.vstack([centre(i, j, k) + np.c_[rng.uniform(-0.2, 0.2, (4, 2)), rng.normal(0, 0.004 * (1 + a), 4)] for i, j, k in ijk])
        rv = centre(0, 0, 0) + np.c_[rng.uniform(-0.2, 0.2, (8, 2)), rng.normal(0, 0.01, 8)]   # the same cell in every append
        out.append((np.vstack([rv, p]).astype(np.float32), [0] if a < 2 else [0, 1]))
    return out


# ---- direction bins ------------------------------------------------------------------------------------------------------------------------
def direction_cases():
    """name -> (cloud, designed line count image [60, 60], designed plane count image [60, 60]).  Line cells aimed at pixel centres (or along
    axes, which land on the clamps), plane cells with axis normals fixing the image basis."""
    cases = {}

    def build(pixels, planes=0, basis="z", extra=()):
        cl, cp = np.zeros((60, 60), np.float32), np.zeros((60, 60), np.float32)
        pts, n = [], 0
        slots = _slot(len(pixels) + planes + len(extra))
        for (pi, ti) in pixels:
            pts.append(line_cell(centre(*slots[n]), pixel_direction(pi, ti, basis)))
            cl[pi, ti] += 1
            n += 1
        for q, px in extra:
            pts.append(q(centre(*slots[n])))
            cl[px] += 1
            n += 1
        for _ in range(planes):
            pts.append(axis_plane(centre(*slots[n]), 2 if basis == "z" else 1))
            cp[30, 30] += 1
            n += 1
        return np.vstack(pts).astype(np.float32), cl, cp

    # axis lines with the identity basis: x -> asin(-1) (theta / step = -1, clamped to 0) at phi = pi / 2 exactly (bin 30); y -> phi / step just
    # above 60 (clamped to 59); z -> the centre pixel; with +y plane normals an x line reaches asin(+1) (60.0000008, clamped to 59)
    ax = [(lambda c, a=a: axis_line(c, a), px) for a, px in ((0, (30, 0)), (1, (59, 30)), (2, (30, 30)))]
    cases["clamps_identity_basis"] = build([], extra=ax)
    cases["clamps_z_normals"] = build([], planes=3, extra=ax)
    cases["clamps_y_normals"] = build([], planes=2, basis="y", extra=[(lambda c: axis_line(c, 0), (30, 59))])
    corners = [(0, 0), (0, 59), (59, 0), (59, 59)]
    edges = [(0, t) for t in range(1, 59, 7)] + [(59, t) for t in range(2, 59, 7)] + [(p, 0) for p in range(3, 59, 7)] + [(p, 59) for p in range(4, 59, 7)]
    cases["corners_and_edges"] = build(corners + edges, planes=1)
    cases["full_image"] = build([(p, t) for p in range(60) for t in range(60)] + [(p, (7 * p) % 60) for p in range(60)])
    cases["single_large_count"] = build([(17, 42)] * 1000)
    return cases


# ---- ROI ----------------------------------------------------------------------------------------------------------------------------------
def roi_cases():
    """name -> cloud of one point per cell (a first append takes every touched cell)."""
    cases = {"one_cell": centre(3, -4, 5)[None]}
    cases["cube_corners"] = np.array([centre(i, j, k) for i in (0, 1) for j in (4, 5) for k in (-1, 0)], np.float32)   # all at one distance: u = 1
    cases["duplicate_distances"] = np.array([centre(i, 0, 0) for i in range(-6, 6)] + [centre(0, j, 0) for j in range(-6, 6)], np.float32)
    for n in (2, 3, 6, 10, 11, 12, 20, 21, 22, 101):   # u - 1 = n - 1: (u - 1) 0.9f onto an integer (10, 20, 100) or not
        cases[f"distinct_{n}"] = np.array([centre(i * i, 2 * i, 0) for i in range(n)], np.float32)
    return cases


# ---- blur and search ----------------------------------------------------------------------------------------------------------------------
def pattern_cloud(line_px, planes, block):
    """A keyframe cloud whose line count image holds line_px ({(pi, ti): count}) and whose plane image holds `planes` at (30, 30) (+z normals),
    in the cells of lattice cube `block` (1 to 342)."""
    pixels = [px for px, n in line_px.items() for _ in range(int(n))]
    slots = _slot(len(pixels) + planes, block)
    pts = [line_cell(centre(*slots[r]), pixel_direction(*px)) for r, px in enumerate(pixels)]
    pts += [axis_plane(centre(*slots[len(pixels) + r]), 2) for r in range(planes)]
    return np.vstack(pts).astype(np.float32) if pts else np.zeros((0, 3), np.float32)


def roll(px, dp, dt):
    return {((p + dp) % 60, (t + dt) % 60): n for (p, t), n in px.items()}


def search_cases():
    """name -> list of (line pixels, plane cells) per keyframe, the newest last."""
    rng = np.random.default_rng(23)
    base = {}
    for _ in range(40):
        px = (int(rng.integers(60)), int(rng.integers(60)))
        base[px] = base.get(px, 0) + int(rng.integers(1, 4))
    base[(0, 0)], base[(59, 59)], base[(0, 59)] = 2, 1, 3
    cases = {"newest_1": [(base, 3), (base, 3)]}
    shifts = [(30, 0), (-30, 0), (0, 30), (0, -30), (30, 30), (-30, -30), (30, -30), (31, 0), (0, 31), (31, 31), (1, 0), (-29, 17)]
    cases["cyclic_shifts"] = [(roll(base, *s), 2) for s in shifts] + [({**base, (10, 10): base.get((10, 10), 0) + 1}, 2), (base, 2)]
    # all-zero line images (no line cell) as the template and as the image; one-pixel images
    cases["zero_and_one_pixel"] = [({}, 2), ({(5, 6): 1}, 0), ({(40, 2): 4}, 1), ({}, 0), ({(5, 6): 2}, 1), ({}, 1)]
    many = []
    for k in range(301):
        px = {(int(rng.integers(60)), int(rng.integers(60))): 1 for _ in range(int(rng.integers(0, 6)))}
        many.append((px, int(rng.integers(0, 3))))
    many[-1] = (roll(many[0][0], 30, 30), many[0][1])
    cases["newest_300"] = many
    return cases
