"""The loop-closure oracle composition (tests/loop_closure_oracle.py) under a loop policy (ll_mapper_set_loop_policy; DESIGN.md §4.6): loops after
the first, a gap after each loop, and one pose graph over every loop edge.

The policy's two rules (loops_done, gap_allows) are plain Python beside candidate_loop, so that a CPU test pins them against a restatement of the
reference's for-loop (laser_mapping.hpp:988-1127) with if_end replaced by them.  LoopPolicyOracle keeps the composition's schedule, history, full
map, accumulated clouds and search, and changes only what a closed keyframe does: the gap rule before the search, and the alignment of both
keyframes' typed clouds as their analyses left them (what the device aligns; the second pass of a multi-loop stream refills the first pass's
cells, so reading the live cells would blur the parity, DESIGN.md §4.6 deviation (xx))."""
import numpy as np

import keyframe_reference as K
import loop_closure_oracle as LCO
import pose_graph_reference as R
from oracle import oracle as O


def loops_done(n_loops, max_loops):
    """The count rule that replaces the reference's if_end (:990-993): after max_loops loops all loop-closure work stops."""
    return n_loops >= max_loops


def gap_allows(newest, loop_newests, gap):
    """The gap rule: a keyframe is searched unless a loop has closed and newest - L < gap, L the newest keyframe of the last loop."""
    return not loop_newests or newest - loop_newests[-1] >= gap


class LoopPolicyOracle(LCO.LoopClosureOracle):
    """LoopClosureOracle with max_loops and min_keyframes_between_loops.  loops: [(newest, his, result)] in closing order; n_candidates: each
    keyframe's candidate count (0: not searched); loop: the max_loops-th loop once all work has stopped (the composition's stop condition)."""

    def __init__(self, *args, max_loops=1, min_keyframes_between_loops=0):
        super().__init__(*args)
        self.max_loops, self.gap = max_loops, min_keyframes_between_loops
        self.loops, self.n_candidates, self.frozen = [], [], []

    def _process(self, k, frame_index):
        h = self.handle[k]
        self.map.analyze(h)
        self.infos.append(dict(self.map.info(h), all_points=self.map.cloud(h, -1).shape[0]))
        self.frozen.append((self.map.cloud(h, 1), self.map.cloud(h, 2)))
        self.kfs.append(h)
        self.poses.append(np.concatenate([self.q_w, self.t_w]))
        self.ending.append(frame_index)
        newest = len(self.kfs) - 1
        if not gap_allows(newest, [n for n, _, _ in self.loops], self.gap):
            self.last_candidates = []
            self.n_candidates.append(0)
            return
        infos = [self.map.info(x) for x in self.kfs]
        imgs = np.stack([np.stack([self.map.images(x)[3], self.map.images(x)[2]]) for x in self.kfs])
        _, cand = K.oracle_search(np.array([i["cells"] for i in infos], np.int64), np.array([i["roi_range"] for i in infos], np.float32),
                                  np.array([i["ratio_plane"] for i in infos], np.float32), np.array([i["ratio_line"] for i in infos], np.float32),
                                  imgs, newest, self.loop_cfg)
        self.last_candidates = cand
        self.n_candidates.append(len(cand))

        def align(his):
            t0 = (infos[newest]["center"] - infos[his]["center"]).astype(np.float32).astype(np.float64)
            res, _ = O.scene_align(*self.frozen[newest], *self.frozen[his], t_init=t0, accepted_threshold=self.thr, **self.align_kw)
            return res.inlier_threshold, res

        for his, d, res in LCO.candidate_loop(cand, align, self.thr):
            self.decisions.append((newest, his, d, res))
            if d == LCO.ACCEPT:
                self.loops.append((newest, his, res))
        if loops_done(len(self.loops), self.max_loops):
            self.loop = self.loops[-1]

    def optimize_loops(self, loop_edges):
        """oracle_optimize of the keyframes up to the newest of the last loop edge, on their odometry edges plus every loop edge
        [((begin, end), [q, t])], from the odometry poses."""
        n = max(loop_edges[-1][0]) + 1
        P = np.array(self.poses[:n])
        E = [(k - 1, k, LCO.odometry_edge(P[k - 1], P[k])) for k in range(1, n)] + [(a, b, m) for (a, b), m in loop_edges]
        ids = np.array([[a, b] for a, b, _ in E], np.int32)
        meas = np.array([m for _, _, m in E], np.float64)
        return R.oracle_optimize(P, ids, meas)[0]

    def refined_upto(self, poses_opt, n):
        """The re-posed accumulated clouds (Mapping_refine::refine_pointcloud, leaf 0.2) of keyframes 0 .. n - 1: a list of [m, 4]."""
        clouds = [self.acc[k] for k in range(n)]
        seg_end = np.cumsum([c.shape[0] for c in clouds]).astype(np.int64)
        pts, cnt = R.oracle_repose(np.concatenate(clouds) if seg_end[-1] else np.zeros((0, 4), np.float32), seg_end, np.array(self.poses[:n]),
                                   np.asarray(poses_opt)[:n], 0.2)
        ends = np.concatenate([[0], np.cumsum(cnt)])
        return [pts[ends[k]:ends[k + 1]] for k in range(n)]
