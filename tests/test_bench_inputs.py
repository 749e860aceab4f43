"""bench.py's inputs, validated without a GPU: every rank's scans (make_inputs(r), r = 0..7, the seeds `--gpus 8` uses) go through the oracle.
Round 1's N = 4 / 8 scaling runs died on a distance-to-truth assert for two of these seeds; the bar is GPU-vs-oracle parity (bench.py asserts that on
the GPU box), and what must hold for the inputs themselves is only that the reference algorithm accepts them: registered, accepted, a bounded distance
to the injected pose (the ICP loop stops on its own 1 cm increment test, point_cloud_registration.hpp:521-526, so a few centimetres remain on some)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_all_rank_inputs_register_on_the_oracle(oracle):
    import bench
    from loam_livox_b200 import synthetic as S
    maps = S.make_map(bench.N_MAP_CORNER, bench.N_MAP_SURF)
    trees = (oracle.KdTree(maps[0]), oracle.KdTree(maps[1]))
    ex = oracle.Extractor()
    threads = min(8, bench.host_threads())
    worst = 0.0
    for rank in range(8):
        mc, ms, scans, guesses, truths = bench.make_inputs(rank, "c2", maps=maps)
        assert len(scans) == bench.N_DISTINCT_SCANS
        for k in range(len(scans)):
            st, res, nc, ns = bench.oracle_step(oracle, ex, trees, mc, ms, scans[k], guesses[k], threads)
            err = float(np.linalg.norm(np.array(res.t_w_curr) - truths[k].t))
            assert st == 1 and res.registered == 1 and 1 <= res.icp_iterations <= 15, (rank, k, st)
            assert nc > 300 and ns > 20000, (rank, k, nc, ns)
            assert err < 0.15, (rank, k, err)
            worst = max(worst, err)
    assert worst < 0.15


def test_host_threads_ignores_omp_env(monkeypatch):
    """torchrun exports OMP_NUM_THREADS=1; the CPU arm must still see the host's cores (round 1's multi-GPU CPU arms ran on one thread)."""
    import bench
    monkeypatch.setenv("OMP_NUM_THREADS", "1")
    assert bench.host_threads() == len(os.sched_getaffinity(0))


def test_reference_arm_contract(tmp_path):
    """`bench.py --impl reference` as torchrun launches it: rank 0 prints ONE JSON line with impl / metric / config / cpu_baseline / e2e, honours the
    requested steps and uses the host's cores although torchrun-style OMP_NUM_THREADS=1 is exported; other ranks exit 0 silently."""
    import json
    import subprocess
    env = dict(os.environ, OMP_NUM_THREADS="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "3", "--warmup", "3"], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "scans_per_sec" and d["unit"] == "scans/s" and d["higher_is_better"] is True
    assert d["steps"] == 3 and d["n_gpus"] == 2 and d["value"] > 0 and d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and "host threads" in d["cpu_baseline"]["sample"]
    assert d["config"]["workload"].startswith("C2:") and d["config"]["pipeline"]["mapping_leaf_surf"] == 0.02
    env["RANK"] = "1"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "3"], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0 and not r.stdout.strip()
