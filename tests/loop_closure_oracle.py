"""The streaming mapper's loop closure composed from the oracles (DESIGN.md §4.6): Laser_mapping::process_new_scan's keyframe block
(laser_mapping.hpp:1442, 1446-1459, 1480-1487, 1523-1564) and service_loop_detection (:874-1127), driven by the device's registration poses.

Pieces: the oracle extractor's full cloud, orc_transform, the full history, the oracle VoxelGrid, the keyframe oracle (keyframe_reference.py:
the full map, add_cells, analyze, the search), O.scene_align, and the pose-graph oracle (pose_graph_reference.py: the loop edge, the solve,
the re-pose).  The schedule (Schedule) and the candidate loop (candidate_loop) are plain Python, so that a CPU test pins them against a
restatement of the reference's own loops."""
import numpy as np

import keyframe_reference as K
import pose_graph_reference as R
from oracle import oracle as O

SKIP10, SKIP5, ACCEPT = 0, 1, 2   # ll_loop_event::decision


class Schedule:
    """m_keyframe_of_updating_list's bookkeeping (:1534-1563): step() after each appended frame returns (closed, opened): the index of the keyframe
    closed by this frame (or None) and whether a keyframe was opened (the back keyframe then takes the history as its accumulated cloud)."""

    def __init__(self, each, between):
        self.each, self.between = each, between
        self.open = [[0, 0]]   # [keyframe index, accumulate_frames], front first
        self.created = 1

    def step(self):
        for o in self.open:
            o[1] += 1
        closed = None
        if self.open[0][1] >= self.each:
            closed = self.open.pop(0)[0]
        back = self.open[-1][0] if self.open[-1][1] >= self.between else None
        if back is not None:
            self.open.append([self.created, 0])
            self.created += 1
        return closed, back


def candidate_loop(candidates, align, thr):
    """The candidates (his ascending) through the alignment with the skips of :1048-1052 and :1113-1116: returns [(his, decision, result)], the
    last one ACCEPT when a loop closes.  align(his) -> (inlier_threshold, result); thr is the float threshold (compared in double)."""
    out, skip_to = [], -1
    thr2 = float(np.float32(thr) * np.float32(2))
    for his in candidates:
        if his <= skip_to:
            continue
        score, res = align(his)
        if score > thr2:
            out.append((his, SKIP10, res)); skip_to = his + 10
        elif not score < float(np.float32(thr)):
            out.append((his, SKIP5, res)); skip_to = his + 5
        else:
            out.append((his, ACCEPT, res))
            break
    return out


def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def qinv(q):
    return np.array([q[0], -q[1], -q[2], -q[3]]) / float(np.dot(q, q))


def qrot(q, v):
    return qmul(qmul(q, np.concatenate([[0.0], v])), qinv(q))[1:]


def odometry_edge(prev, cur):
    """(:952-958) as [q w x y z, t]: q_prev^-1 q_cur, q_prev^-1 (t_cur - t_prev)."""
    qi = qinv(prev[:4])
    return np.concatenate([qmul(qi, cur[:4]), qrot(qi, cur[4:] - prev[4:])])


class LoopClosureOracle:
    def __init__(self, each, between, loop_cfg, thr, align_kw, surround_res, cell_res, revisit, incremental, max_history, q0, t0):
        self.sched = Schedule(each, between)
        self.map = K.OracleMap(cell_res, revisit, incremental)
        self.handle = {0: self.map.new_keyframe()}
        self.loop_cfg, self.thr, self.align_kw, self.surround_res, self.max_history = loop_cfg, thr, align_kw, surround_res, max_history
        self.full_history, self.n_feature_history = [], 0
        self.last_his_q, self.last_his_t = np.array([1.0, 0, 0, 0]), np.zeros(3)
        self.q_w, self.t_w = np.asarray(q0, np.float64), np.asarray(t0, np.float64)   # the pose adopted from the previous step
        self.acc = {}                          # keyframe index -> accumulated cloud, down-sampled
        self.kfs, self.poses, self.ending, self.infos = [], [], [], []   # infos: as analyze left them (a later keyframe's analyze re-types
        #                                                                    the cells they share, so a later read differs)
        self.decisions, self.loop = [], None   # [(newest, his, decision, result)]; (newest, his, result) once closed

    def step(self, full_local, q, t, frame_index):
        """One appended step: full_local the step's full cloud (scan frame), (q, t) its registration pose (adopted)."""
        if self.loop is not None:
            return
        w = O.transform(full_local, q, t)
        # the feature history's push condition (:1446-1459) with the pose adopted from the previous step; the full history follows it
        dot = min(abs(float(np.dot(self.q_w, self.last_his_q))), 1.0)
        r_diff, t_diff = 2.0 * np.arccos(dot) * 57.3, float(np.linalg.norm(self.t_w - self.last_his_t))
        if self.n_feature_history < self.max_history or t_diff > 0.0 or r_diff > 0.0:
            self.last_his_q, self.last_his_t = self.q_w.copy(), self.t_w.copy()
            self.n_feature_history += 1
            self.full_history.append(w)
        self.n_feature_history = min(self.n_feature_history, self.max_history)
        if len(self.full_history) > self.max_history:
            self.full_history.pop(0)
        self.q_w, self.t_w = np.asarray(q, np.float64), np.asarray(t, np.float64)
        self.map.append(w, [self.handle[k] for k, _ in self.sched.open])
        closed, back = self.sched.step()
        if back is not None:
            h = np.concatenate(self.full_history) if self.full_history else np.zeros((0, 4), np.float32)
            self.acc[back] = O.voxel_grid(h, np.float32(self.surround_res)) if h.shape[0] else h
            self.full_history = []
            self.handle[self.sched.created - 1] = self.map.new_keyframe()
        if closed is not None:
            self._process(closed, frame_index)

    def _process(self, k, frame_index):
        h = self.handle[k]
        self.map.analyze(h)
        self.infos.append(dict(self.map.info(h), all_points=self.map.cloud(h, -1).shape[0]))
        self.kfs.append(h)
        self.poses.append(np.concatenate([self.q_w, self.t_w]))
        self.ending.append(frame_index)
        newest = len(self.kfs) - 1
        infos = [self.map.info(x) for x in self.kfs]
        imgs = np.stack([np.stack([self.map.images(x)[3], self.map.images(x)[2]]) for x in self.kfs])
        _, cand = K.oracle_search(np.array([i["cells"] for i in infos], np.int64), np.array([i["roi_range"] for i in infos], np.float32),
                                  np.array([i["ratio_plane"] for i in infos], np.float32), np.array([i["ratio_line"] for i in infos], np.float32),
                                  imgs, newest, self.loop_cfg)
        self.last_candidates = cand

        def align(his):
            t0 = (infos[newest]["center"] - infos[his]["center"]).astype(np.float32).astype(np.float64)
            c = lambda x, w: self.map.cloud(self.kfs[x], w)
            res, _ = O.scene_align(c(newest, 1), c(newest, 2), c(his, 1), c(his, 2), t_init=t0, accepted_threshold=self.thr, **self.align_kw)
            return res.inlier_threshold, res

        for his, d, res in candidate_loop(cand, align, self.thr):
            self.decisions.append((newest, his, d, res))
            if d == ACCEPT:
                self.loop = (newest, his, res)

    def odometry_edges(self):
        P = np.array(self.poses)
        return [(k - 1, k, odometry_edge(P[k - 1], P[k])) for k in range(1, len(P))]

    def optimize(self, loop_edge_ids, loop_edge_meas):
        """oracle_optimize on the odometry edges plus the given loop edge (ids (begin, end), [q, t])."""
        E = self.odometry_edges()
        ids = np.array([[a, b] for a, b, _ in E] + [list(loop_edge_ids)], np.int32)
        meas = np.array([m for _, _, m in E] + [loop_edge_meas], np.float64)
        return R.oracle_optimize(np.array(self.poses), ids, meas)[0]

    def refined(self, poses_opt):
        """The re-posed accumulated clouds (Mapping_refine::refine_pointcloud, leaf 0.2) of every keyframe: a list of [m, 4]."""
        n = len(self.kfs)
        clouds = [self.acc[k] for k in range(n)]
        seg_end = np.cumsum([c.shape[0] for c in clouds]).astype(np.int64)
        pts, cnt = R.oracle_repose(np.concatenate(clouds) if seg_end[-1] else np.zeros((0, 4), np.float32), seg_end, np.array(self.poses),
                                   np.asarray(poses_opt), 0.2)
        ends = np.concatenate([[0], np.cumsum(cnt)])
        return [pts[ends[k]:ends[k + 1]] for k in range(n)]
