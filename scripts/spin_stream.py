"""Streaming mapper on spinning-lidar sweeps (ll_mapper_process_sweep / _sweeps): VLP-16 sweeps in the room and HDL-64 sweeps in the open
scene along synthetic.trajectory.  Per stream: wall-clock ms per sweep of the single calls and of one sequence call (each on a fresh mapper,
after a warm-up stream of the same shape), the mean ms_front_end / ms_register / ms_append of the stats, whether both arms agree, and the oracle
composition's CPU time per sweep (tests/spin_mapper_oracle.py, on the first sweeps).  The card's name and power limit are read in the same run.
One JSON line per stream, then a summary line; with --out the lines also go to that file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from loam_livox_b200 import capi, synthetic as S  # noqa: E402
from loam_livox_b200.registration import Context, Laser_feature, Laser_mapping  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def sweeps(scan_line, n, seed):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0, zero_mean_yaw=True)
    if scan_line == 16:
        return [S.make_spinning_scan(16, p, seed=seed + k) for k, p in enumerate(poses)]
    return [S.make_spinning_scan(64, p, seed=seed + k, n_azimuth=2080, scene="open") for k, p in enumerate(poses)]


def mapper(ctx):
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=3))


def run(ctx, front, raws, sequence):
    gm = mapper(ctx)
    t0 = time.perf_counter()
    out = gm.process_new_sweeps(front, raws) if sequence else [gm.process_new_sweep(front, r) for r in raws]
    ms = (time.perf_counter() - t0) * 1e3 / len(raws)
    pose = gm.pose()
    gm.close()
    return ms, out, pose


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--oracle-sweeps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []

    def emit(d):
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)

    ctx = Context(0, max_scan_points=1000, max_features=100000)
    for scan_line, name in ((16, "vlp16_room"), (64, "hdl64_open")):
        front = Laser_feature(ctx, scan_line)
        raws = sweeps(scan_line, a.sweeps, S.SEED + 3000)
        run(ctx, front, raws[:a.warmup], False)
        run(ctx, front, raws[:a.warmup], True)
        ms_single, out_s, pose_s = run(ctx, front, raws, False)
        ms_seq, out_q, pose_q = run(ctx, front, raws, True)
        same = pose_s[0].tobytes() == pose_q[0].tobytes() and pose_s[1].tobytes() == pose_q[1].tobytes() and \
            all(r.icp_iterations == q.icp_iterations and s.n_corner == t.n_corner and s.n_surf == t.n_surf for (r, s), (q, t) in zip(out_s, out_q))
        mean = lambda out, f: float(np.mean([getattr(s, f) for _, s in out]))  # noqa: E731
        import spin_mapper_oracle as SMO
        om = SMO.SpinMapper(scan_line, threads=1)
        secs = []
        for r in raws[:a.oracle_sweeps]:
            om.process_sweep(r)
            secs.append(om.seconds)
        emit(dict(stream=name, sweeps=len(raws), points_per_sweep=int(raws[0].shape[0]), features_last=[out_s[-1][1].n_corner, out_s[-1][1].n_surf],
                  ms_per_sweep_single=round(ms_single, 3), ms_per_sweep_sequence=round(ms_seq, 3),
                  single=dict(ms_front_end=round(mean(out_s, "ms_front_end"), 3), ms_register=round(mean(out_s, "ms_register"), 3),
                              ms_append=round(mean(out_s, "ms_append"), 3)),
                  sequence=dict(ms_front_end=round(mean(out_q, "ms_front_end"), 3), ms_register=round(mean(out_q, "ms_register"), 3),
                                ms_append=round(mean(out_q, "ms_append"), 3)),
                  sequence_equals_single=bool(same), final_t=[round(float(x), 4) for x in pose_s[1]],
                  oracle_ms_per_sweep_one_thread=round(1e3 * float(np.mean(secs)), 2), oracle_sweeps=len(secs)))
        front.close()
    emit(dict(card=card(), note="host-input XYZI16 sweeps; wall clock around calls that end in a device synchronisation"))
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
