"""Times ll_keyframe_append, ll_keyframe_analyze and ll_loop_search against the keyframe oracle on one CPU thread, and the search against
the keyframe count.  Host clock around calls that end in a device synchronise; prints one JSON line (with the card and its power limit)."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import keyframe_reference as K  # noqa: E402
from loam_livox_b200 import capi  # noqa: E402
from loam_livox_b200.registration import Context, Keyframe, Points_cloud_map, loop_search  # noqa: E402
from test_gpu_keyframe import _scene  # noqa: E402


def main():
    ctx = Context(0, max_scan_points=200000, max_features=20000)
    g, o = Points_cloud_map(ctx, 1.0, 2147483647, 0), K.OracleMap(1.0)
    kfs, oks, t_app, t_oapp, t_an, t_oan = [], [], [], [], [], []
    n_kf, per = 300, 5000
    for k in range(n_kf):
        ang = 2 * np.pi * k / n_kf
        c = _scene(k, per, shift=(3 * np.cos(ang), 3 * np.sin(ang)))
        kf, ko = Keyframe(ctx), o.new_keyframe()
        t0 = time.perf_counter(); Keyframe.append(ctx, g, c, [kf]); t_app.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); kf.analyze(g); t_an.append(time.perf_counter() - t0)
        if k < 5:
            t0 = time.perf_counter(); o.append(c, [ko]); t_oapp.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); o.analyze(ko); t_oan.append(time.perf_counter() - t0)
        kfs.append(kf)
    search = {}
    for n in (10, 100, 300):
        loop_search(ctx, kfs[:n])
        ts = []
        for _ in range(5):
            t0 = time.perf_counter(); loop_search(ctx, kfs[:n]); ts.append(time.perf_counter() - t0)
        search[n] = float(np.median(ts)) * 1e3
    imgs = np.stack([np.stack([kf.images()[3], kf.images()[2]]) for kf in kfs[:11]])
    t0 = time.perf_counter()
    K.oracle_search(np.zeros(11, np.int64), np.zeros(11, np.float32), np.zeros(11, np.float32), np.zeros(11, np.float32), imgs, 10)
    oracle_pair_ms = (time.perf_counter() - t0) * 1e3 / 10
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    stored = g.stats()[1]
    print(json.dumps({"gpu": gpu, "keyframes": n_kf, "points_per_append": int(len(c)), "stored_points_at_end": stored,
                      "append_ms_median": float(np.median(t_app)) * 1e3, "analyze_ms_median_first5": float(np.median(t_an[:5])) * 1e3,
                      "analyze_ms_median_last5": float(np.median(t_an[-5:])) * 1e3,
                      "oracle_append_ms_median": float(np.median(t_oapp)) * 1e3, "oracle_analyze_ms_median": float(np.median(t_oan)) * 1e3,
                      "search_ms_by_keyframes": search, "oracle_search_ms_per_pair": oracle_pair_ms, "launches": ctx.launches()}))
    ctx.close()


if __name__ == "__main__":
    main()
