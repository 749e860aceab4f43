"""ll_frame_to_pose repeated and interleaved on one context: the same frame three times from a reset extractor returns the same features,
result and launch count, and ll_frame_to_pose, ll_mapper_process_frame and ll_scan_to_pose in turn (the front-end graphs of the scan and of
the mapper's frame captured and replayed in between the other calls) each match the oracle.  Any change to how these entry points share the
context's front-end arenas, graphs and extractor has to keep both."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import piecewise_oracle as PO  # noqa: E402
import test_gpu_front_end as FE  # noqa: E402

SELECTIONS = [dict(whole=1), dict(whole=0, use_piece=1)]


@pytest.fixture(scope="module")
def fctx():
    """A context of its own, so that the first call of every shape here runs eagerly."""
    from loam_livox_b200.registration import Context
    c = Context(0, max_scan_points=60000, max_features=60000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def fmap(fctx):
    from loam_livox_b200.registration import Map
    m = Map(fctx, *S.make_map(5000, 45000))
    yield m
    m.release()


def frame(k):
    return S.make_triple_scan(36000, S.default_pose(), seed=S.SEED + 5000 + k)


@pytest.mark.gpu
@pytest.mark.parametrize("sel", SELECTIONS, ids=["whole", "piece1of3"])
def test_same_frame_three_times(fctx, fmap, oracle, sel):
    """Three calls on the same heads from a reset extractor: identical features, counts, result and ll_launch_count delta, and the oracle's
    features."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import frame_to_pose
    pc = FE.pipe(**sel)
    heads, stamps = frame(0 if sel["whole"] else 1), [100.0, 100.01, 100.02]
    guess = S.perturb_pose(S.default_pose(), np.random.default_rng(5), dt=0.05, dang_deg=1.0)
    runs = []
    for _ in range(3):
        fctx._lib.ll_extract_reset(fctx.h)
        l0 = fctx.launches()
        res, nc, ns = frame_to_pose(fctx, fmap, heads, stamps, pc, capi.default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t))
        got = FE.features(fctx)
        runs.append((fctx.launches() - l0, nc, ns, res.status, res.registered, res.icp_iterations, tuple(res.q_w_curr), tuple(res.t_w_curr), res.final_cost,
                     got[0].tobytes(), got[1].tobytes()))
    assert runs[0][4] == 1 and runs[0][0] > 0
    assert runs[1] == runs[0] and runs[2] == runs[0]
    c, s = FE.want_frame(oracle, oracle.Extractor(), heads, stamps, pc)
    assert (runs[0][1], runs[0][2]) == (c.shape[0], s.shape[0]) and runs[0][9] == c.tobytes() and runs[0][10] == s.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("sel", SELECTIONS, ids=["whole", "piece1of3"])
def test_interleaved_with_mapper_frames_and_scans(fctx, fmap, oracle, sel):
    """Four rounds of one shape each: ll_frame_to_pose, ll_mapper_process_frame (3 pieces) and ll_scan_to_pose on one context, every call against
    the oracle, which follows the same extractor bookkeeping (the mapper's creation reset the context's extractor)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    gm = Laser_mapping(fctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=2), pipeline=FE.pipe(whole=0))
    ex = oracle.Extractor()
    registered = 0
    try:
        for k in range(4):
            t = 100.0 + k
            heads = frame(10 + k)
            FE.check_frame(fctx, oracle, fmap, ex, heads, [t, t + 0.01, t + 0.02], FE.pipe(**sel))
            stamps = [t + 0.3] * 3
            parts, live = PO.frame_pieces(ex, heads, stamps, 3)
            got = gm.process_new_frame(heads, stamps)
            assert live == 3 and len(got) == 3, k
            last = None
            for (res, st), (c, s, _) in zip(got, parts):
                c, s = FE.voxel_chains(oracle, c, s)
                assert (st.n_corner, st.n_surf) == (c.shape[0], s.shape[0]), k
                last = (c, s) if res.registered else last
            if last is not None:   # the features a mapper registers are the context's last ones
                registered += 1
                f = FE.features(fctx)
                assert f[0].tobytes() == last[0].tobytes() and f[1].tobytes() == last[1].tobytes(), k
            FE.check_scan(fctx, oracle, fmap, ex, FE.scan(20 + k, 20000), t + 0.6, FE.pipe(whole=0))
    finally:
        gm.close()
    assert registered >= 2
