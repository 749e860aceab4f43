"""The evidence behind the streaming mapper's loss detection (ll_mapper_set_recovery, DESIGN.md §4.3.2), on the CPU oracle: the registration score
inlier_threshold (point_cloud_registration.hpp:559) of every registered scan of a normal C3-style stream, the same score of kidnapped scans registered
from the mapper's last pose, and the verify fraction (the class-aware field score over its maximum, tests/reloc_field_reference.py) of a kidnapped
scan at its truth and at the pillar-pitch aliases.

    python tests/recovery_oracle.py --scans 210 --mode 0      # the table of DESIGN.md §4.3.2
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from loam_livox_b200 import synthetic as S  # noqa: E402
from oracle import oracle as O  # noqa: E402

N_POINTS = 24000
PITCH = 4.0   # the synthetic room repeats itself every 4 m in x (the pillar pitch)


def stream(n, seed):
    """A C3-style stream: 4 static scans, then forward motion at 0.03 m per scan with a sinusoidal yaw."""
    poses = S.trajectory(n_scans=n, n_static=4, speed=1.0)
    return poses, [S.make_scan(N_POINTS, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(n)]


def kidnap_pose(pose, back=2.6, yaw_deg=18.0, aside=0.0):
    """The sensor moved `back` metres back along x and `aside` metres along y, and turned by yaw_deg."""
    return S.Pose(S.quat_mul(pose.q, S.quat_from_euler(0.0, 0.0, np.radians(yaw_deg))), pose.t + np.array([-back, aside, 0.0]))


def mapper(mode, p0, init=3):
    p = O.default_params(mapping_init_accumulate_frames=init, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return O.Mapper(params=p, matching_mode=mode)


def refresh(m):
    """The match-map refresh process_scan runs first when the map is dirty (oracle.Mapper.process_scan), run ahead: the next process_scan then
    finds the map clean and registers against the same map."""
    if not m.dirty:
        return
    if m.matching_mode == 0:
        mc, ms = np.concatenate(m.his_corner), np.concatenate(m.his_surf)
    else:
        mc, _ = m.cells_corner.assemble(m.q, m.t, m.search_range, m.fov_angle, m.line_resolution, m.replace)
        ms, _ = m.cells_surf.assemble(m.q, m.t, m.search_range, m.fov_angle, m.plane_resolution, m.replace)
    m.map_c, m.map_s = O.voxel_grid(mc, m.line_resolution), O.voxel_grid(ms, m.plane_resolution)
    m.tree_c, m.tree_s = O.KdTree(m.map_c), O.KdTree(m.map_s)
    m.dirty = False


def features(m, raw, stamp):
    ex = O.Extractor()
    ex.extract(raw, stamp)
    c, s, _ = ex.get_features(0.0, 1.0)
    return O.voxel_grid(O.voxel_grid(c, m.leaf_c), m.line_resolution), O.voxel_grid(O.voxel_grid(s, m.leaf_s), m.plane_resolution)


def register_from_last_pose(m, c, s):
    """What the mapper's next step would register for features (c, s), without changing the mapper."""
    refresh(m)
    p = O.RegParams.from_buffer_copy(m.params)
    p.current_frame_index = m.frame_index
    p.rng_seed = m.params.rng_seed + m.frame_index
    p.q_w_last[:] = list(m.q); p.q_w_curr[:] = list(m.q)
    p.t_w_last[:] = list(m.t); p.t_w_curr[:] = list(m.t)
    p.para_buffer_incremental[:] = [0, 0, 0, 1, 0, 0, 0]
    return O.register(m.map_c, m.tree_c, m.map_s, m.tree_s, c, s, p)


def whole_map(m):
    """ll_mapper_whole_map of matching mode 0: the VoxelGrid of the history window (the oracle keeps the window in mode 1 too, and on a stream
    shorter than the window it holds every appended point, as the cell maps do)."""
    c, s = np.concatenate(m.his_corner), np.concatenate(m.his_surf)
    return O.voxel_grid(c, m.line_resolution), O.voxel_grid(s, m.plane_resolution)


def verify_fraction(field, res, T, sc, ss, q, t):
    import reloc_field_reference as F
    dims, lo, d2 = field
    v = int(F.field_scores(d2, dims, lo, res, T, [sc, ss], np.asarray(q, np.float64)[None], np.asarray(t, np.float64), (0.0, 0.0, 0.0), (1, 1, 1))[0])
    return v / float(T * T * (sc.shape[0] + ss.shape[0]))


def measure(n_scans, mode, seed, kidnaps, res=0.2, T=2, score_leaf=0.5, back=2.6, yaw_deg=18.0, aside=0.0, want_verify=True):
    """{"normal": inlier_threshold of every registered scan, "kidnap": [(k, status, inlier_threshold)], "verify": [(k, truth, x - 4, x + 4)]}."""
    import reloc_field_reference as F
    poses, raws, stamps = stream(n_scans, seed)
    m = mapper(mode, poses[0])
    normal, kid, ver = [], [], []
    for k in range(n_scans):
        if k in kidnaps and m.map_c is not None:
            pk = kidnap_pose(poses[k], back, yaw_deg, aside)
            c, s = features(m, S.make_scan(N_POINTS, pk, seed=seed + 100000 + k), stamps[k])
            st, r = register_from_last_pose(m, c, s)
            kid.append((k, int(st), float(r.inlier_threshold)))
            if want_verify:
                wc, ws = whole_map(m)
                fld = F.field([wc, ws], res, T)
                sc, ss = O.voxel_grid(c, score_leaf), O.voxel_grid(s, score_leaf)
                row = [k]
                for dx in (0.0, -PITCH, PITCH):
                    row.append(verify_fraction(fld, res, T, sc, ss, pk.q, pk.t + np.array([dx, 0.0, 0.0])))
                ver.append(tuple(row))
        st, _, _ = m.process_scan(raws[k], stamps[k])
        r = m.last.get("res")
        if r is not None and r.registered:
            normal.append((k, int(st), float(r.inlier_threshold)))
    return {"normal": normal, "kidnap": kid, "verify": ver}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=210)
    ap.add_argument("--mode", type=int, default=0)
    ap.add_argument("--seed", type=int, default=S.SEED + 7000)
    ap.add_argument("--every", type=int, default=10)
    a = ap.parse_args()
    kid = set(range(100, a.scans, a.every))   # (from scan 100 on the place 2.6 m back lies on the path)
    out = measure(a.scans, a.mode, a.seed, kid)
    th = np.array([x[2] for x in out["normal"]])
    rej = sum(1 for x in out["normal"] if x[1] == 0)
    print(f"mode {a.mode}: {th.size} registered normal scans, {rej} rejected; inlier_threshold min {th.min():.4f} median {np.median(th):.4f} "
          f"p99 {np.quantile(th, 0.99):.4f} max {th.max():.4f}")
    kt = np.array([x[2] for x in out["kidnap"]])
    print(f"mode {a.mode}: {kt.size} kidnapped scans, {sum(1 for x in out['kidnap'] if x[1] == 0)} rejected; inlier_threshold min {kt.min():.4f} "
          f"median {np.median(kt):.4f} max {kt.max():.4f}")
    for row in out["kidnap"]:
        print("  kidnap", row)
    v = np.array([x[1:] for x in out["verify"]])
    print(f"verify fraction: truth min {v[:, 0].min():.3f} median {np.median(v[:, 0]):.3f}; x-4 max {v[:, 1].max():.3f}; x+4 max {v[:, 2].max():.3f}")
    for row in out["verify"]:
        print("  verify", tuple(round(x, 4) if isinstance(x, float) else x for x in row))


if __name__ == "__main__":
    main()
