"""CPU checks of the loop-closure oracle composition (tests/loop_closure_oracle.py): its keyframe schedule against a restatement of
laser_mapping.hpp:1523-1564 and its candidate loop against a restatement of service_loop_detection's for-loop (:988-1127) on constructed
decisions, scores exactly at the threshold and at twice it included."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import loop_closure_oracle as LCO  # noqa: E402


def _reference_schedule(n_frames, each, between):
    """:1523-1564 as written: a list of keyframes with m_accumulate_frames, front closed at `each`, back opened from at `between`."""
    updating, closed, opened = [{"id": 0, "acc": 0}], [], []
    next_id = 1
    for f in range(n_frames):
        for kf in updating:                       # add_cells ... m_accumulate_frames++ (:1527-1533)
            kf["acc"] += 1
        if updating[0]["acc"] >= each:            # :1536
            closed.append((f, updating.pop(0)["id"]))
        if updating[-1]["acc"] >= between:        # :1546
            opened.append((f, updating[-1]["id"]))
            updating.append({"id": next_id, "acc": 0})
            next_id += 1
    return closed, opened


@pytest.mark.parametrize("each,between", [(300, 100), (6, 2), (6, 5), (6, 1), (3, 2), (2, 1), (7, 3)])
def test_schedule_equals_the_reference_bookkeeping(each, between):
    s = LCO.Schedule(each, between)
    closed, opened = [], []
    for f in range(1000):
        c, b = s.step()
        if c is not None:
            closed.append((f, c))
        if b is not None:
            opened.append((f, b))
    assert (closed, opened) == _reference_schedule(1000, each, between)
    # every keyframe takes its accumulated cloud before it closes
    first_open = {k: f for f, k in opened}
    assert all(first_open[k] < f for f, k in closed)


def _reference_loop(n_kf, passes, score, thr):
    """The for-loop of :988-1127 over his = 0 .. n - 2: the gates (`passes`), the alignment, `his += 10; continue` above twice the threshold,
    the loop below it, `his += 5` otherwise (then the for's own his++)."""
    out, his = [], 0
    thr32 = np.float32(thr)
    while his < n_kf - 1:
        if his in passes:
            s = score(his)
            if s > float(thr32 * np.float32(2)):
                out.append((his, LCO.SKIP10)); his += 10; his += 1; continue
            if s < float(thr32):
                out.append((his, LCO.ACCEPT)); break
            out.append((his, LCO.SKIP5)); his += 5
        his += 1
    return out


def test_candidate_loop_equals_the_reference_loop():
    rng = np.random.default_rng(7)
    thr = 0.35
    edge = [float(np.float32(thr)), float(np.float32(thr) * np.float32(2))]
    for trial in range(3000):
        n = int(rng.integers(2, 80))
        passes = sorted(set(rng.choice(n - 1, size=int(rng.integers(0, n)), replace=True).tolist())) if n > 1 else []
        table = {h: (edge[int(rng.integers(2))] if rng.random() < 0.3 else float(rng.uniform(0.0, 1.2))) for h in range(n)}
        got = [(h, d) for h, d, _ in LCO.candidate_loop(passes, lambda h: (table[h], None), thr)]
        assert got == _reference_loop(n, set(passes), lambda h: table[h], thr), (trial, passes, table)


def test_candidate_loop_edges():
    thr = 0.35
    t, t2 = float(np.float32(thr)), float(np.float32(thr) * np.float32(2))
    run = lambda cands, scores: [(h, d) for h, d, _ in LCO.candidate_loop(cands, lambda h: (scores[h], None), thr)]
    # exactly twice the threshold is not above it: his += 5; exactly the threshold is not below it: his += 5
    assert run([0, 5, 6], {0: t2, 5: 0.9, 6: 0.1}) == [(0, LCO.SKIP5), (6, LCO.ACCEPT)]
    assert run([0, 5, 6], {0: t, 5: 0.9, 6: 0.1}) == [(0, LCO.SKIP5), (6, LCO.ACCEPT)]
    # one float above twice the threshold: his += 10 (10 more skipped, the 11th is aligned)
    above = float(np.nextafter(np.float64(t2), 2.0))
    assert run([0, 10, 11], {0: above, 10: 0.1, 11: 0.1}) == [(0, LCO.SKIP10), (11, LCO.ACCEPT)]
    # just below the threshold: a loop, nothing after it
    below = float(np.nextafter(np.float64(t), 0.0))
    assert run([3, 4], {3: below, 4: 0.1}) == [(3, LCO.ACCEPT)]
