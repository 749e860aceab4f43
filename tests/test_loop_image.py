"""Host-only checks of the loop image (include/loamlivox_b200.h, "loop image"): a small NumPy writer of the documented layout builds valid
images that ll_loop_image_info accepts and reports; the validator refuses every structural and content rule just outside its bound and accepts
it just inside, before any device is involved; the ctypes mirrors have the C layout; the entry points are exported with the header's
parameter counts; and the C++ mirror's loop_save / loop_load compiles, links and runs (without a GPU it stops at the context)."""
import ctypes as C
import functools
import struct
import subprocess

import numpy as np
import pytest

import image_writer
from image_writer import CELL, CELL_POINT, key
from loam_livox_b200 import capi
from test_recovery_cabi import _compile, _header_params

HEADER = 24 + 16 * capi.LL_LOOP_IMAGE_SECTIONS   # ll_loop_image_header
IMG = 4 * 3600   # floats of one keyframe's four images


# ---------------------------------------------------------------------------------------------- writer of the documented layout
def config(**kw) -> bytes:
    c = capi.LoopClosureCfg()
    capi.lib().ll_mapper_loop_closure_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return bytes(c)


def scalars(frame_index=12, mode=0, revisit=2000, history=400, pieces=3, cell_res=1.0, stamp=100.5, q=(1.0, 0, 0, 0), t=(0.5, 0.0, 0.0), closed=0,
            stopped=0, n_keyframes=2, n_open=3, n_events=2, n_dropped=0) -> bytes:
    return struct.pack("<5if8d6i", frame_index, mode, revisit, history, pieces, cell_res, stamp, *q, *t, closed, stopped, n_keyframes, n_open, n_events, n_dropped)


def cells(frame_idx=12, n_out_of_range=0, keys=None, stamps=None, cur=(0, 1, 0, 2, 0), ranks=(0, 1, 1, 2, 3, 3, 3, 4, 0), ords=(0, 1, 0, 0, 2, 1, 2, 0, 0),
          pts=None) -> bytes:
    n = len(cur)
    c = np.zeros(n, CELL)
    c["key"] = sorted(key(k, -k, 2 * k) for k in range(n)) if keys is None else keys
    c["create_frame"], c["last_update"] = (np.arange(n) % frame_idx, np.minimum(np.arange(n) % frame_idx + 1, frame_idx)) if stamps is None else stamps
    p = np.zeros(len(ranks), CELL_POINT)
    xyz = np.random.default_rng(1).uniform(-20, 20, (len(ranks), 3)).astype("<f4") if pts is None else pts
    p["x"], p["y"], p["z"], p["cell"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], ranks
    return (struct.pack("<iiqq", frame_idx, n_out_of_range, n, len(ranks)) + c.tobytes() + p.tobytes() + np.asarray(cur, "<i4").tobytes()
            + np.asarray(ords, "<i4").tobytes())


def history(sizes=(3, 2), seed=2) -> bytes:
    return image_writer.history(sizes, np.random.default_rng(seed).uniform(-9, 9, (int(sum(sizes)), 4)).astype("<f4"))


def open_kfs(kfs=((4, 4, [(0, 0), (1, 0), (1, 1)]), (2, 2, [(3, 2)]), (0, 0, []))) -> bytes:
    head = b"".join(struct.pack("<iiq", f, a, len(r)) for f, a, r in kfs)
    return head + b"".join(struct.pack("<ii", c, i) for _, _, r in kfs for c, i in r)


def info(cells=3, line_cells=1, plane_cells=1, accumulate_frames=6, line_points=2, plane_points=3, all_points=7, roi=4.0):
    x = capi.KeyframeInfo(cells=cells, line_cells=line_cells, plane_cells=plane_cells, accumulate_frames=accumulate_frames, roi_range=roi,
                          ratio_nonzero_line=0.1, ratio_nonzero_plane=0.2, line_points=line_points, plane_points=plane_points, all_points=all_points)
    x.center[:] = [1.0, 2.0, 0.5]
    return x


def pose(x=0.0, q=(1.0, 0.0, 0.0, 0.0)):
    p = capi.Pose()
    p.q_wxyz[:], p.t[:] = q, [x, 0.0, 0.0]
    return bytes(p)


def edge(a, b):
    e = capi.PgEdge(id_begin=a, id_end=b)
    e.q_wxyz[:] = [1.0, 0.0, 0.0, 0.0]
    e.t[:] = [0.3, 0.0, 0.0]
    for k in range(6):
        e.information[7 * k] = 1.0
    return bytes(e)


def points(n, seed):
    return np.random.default_rng(seed).uniform(-9, 9, (n, 4)).astype("<f4").tobytes()


def accumulated(ends=(5, 5, 9, 12)) -> bytes:
    return struct.pack("<q", len(ends)) + np.asarray(ends, "<i8").tobytes() + points(ends[-1] if ends else 0, 7)


def events(kinds=(capi.LL_LOOP_KEYFRAME, capi.LL_LOOP_ALIGNMENT)) -> bytes:
    return b"".join(bytes(capi.LoopEvent(kind=k, keyframe=1)) for k in kinds)


def parts(closed=False):
    """The thirteen sections of a valid image, in index order: two closed keyframes, three open ones (the last without an append)."""
    infos = [info(), info(cells=2, line_points=1, plane_points=0, all_points=4)]
    loop = (edge(0, 1) + pose(0.0) + pose(0.31)) if closed else b""
    return [config(), scalars(closed=int(closed)), cells(), history(), open_kfs(), b"".join(bytes(x) for x in infos), pose(0.0) + pose(0.3), edge(0, 1),
            np.zeros(2 * IMG, "<f4").tobytes(), points(2 + 3 + 1, 5), accumulated(), loop, events()]


image = functools.partial(image_writer.image, magic=b"LLLOOPIM", config_bytes=C.sizeof(capi.LoopClosureCfg))


def summary(img):
    out = capi.LoopImageSummary()
    buf = np.frombuffer(img, np.uint8) if len(img) else np.zeros(1, np.uint8)
    return capi.lib().ll_loop_image_info(buf.ctypes.data, len(img), C.byref(out)), out


def status(img):
    return summary(img)[0]


def with_part(k, data, closed=False):
    p = parts(closed)
    p[k] = data
    return image(p)


# ---------------------------------------------------------------------------------------------- valid images
def test_valid_images_are_accepted_and_reported():
    st, got = summary(image(parts()))
    assert st == capi.LL_OK
    assert (got.version, got.frame_index, got.matching_mode, got.closed, got.stopped) == (1, 12, 0, 0, 0)
    assert (got.keyframes, got.open_keyframes, got.events, got.dropped) == (2, 3, 2, 0)
    assert (got.cells, got.cell_points, got.history_points, got.cloud_points, got.accumulated_points) == (5, 9, 5, 6, 12)
    # ordinals (0, 1, 0, 0, 2, 1, 2, 0, 0) against their cells' current ones (0, 1, 1, 0, 2, 2, 2, 0, 0): two replaced
    assert got.replaced_points == 2 and got.max_incarnation == 2
    assert got.bytes == len(image(parts()))
    st, got = summary(image(parts(closed=True)))
    assert st == capi.LL_OK and got.closed == 1
    # sections need not be in index order
    p = parts()
    order = list(range(capi.LL_LOOP_IMAGE_SECTIONS))[::-1]
    offs, off = {}, HEADER
    for k in order:
        offs[k] = off
        off += len(p[k])
    head = struct.pack("<8sIIQ", b"LLLOOPIM", 1, C.sizeof(capi.LoopClosureCfg), off) + b"".join(struct.pack("<QQ", offs[k], len(p[k])) for k in range(len(p)))
    assert status(head + b"".join(p[k] for k in order)) == capi.LL_OK


def test_python_wrapper_reports_and_refuses():
    from loam_livox_b200.registration import LoamLivoxError, loop_image_info
    assert loop_image_info(image(parts()))["keyframes"] == 2
    with pytest.raises(LoamLivoxError):
        loop_image_info(image(parts())[:-1])


# ---------------------------------------------------------------------------------------------- structure
def test_structure_is_checked():
    good = image(parts())
    assert status(b"") == status(good[:HEADER - 1]) == capi.LL_ERR_INVALID
    assert status(image(parts(), magic=b"LLMAPIMG")) == capi.LL_ERR_INVALID
    assert status(image(parts(), version=2)) == capi.LL_ERR_INVALID
    assert status(image(parts(), config_bytes=C.sizeof(capi.LoopClosureCfg) + 8)) == capi.LL_ERR_INVALID
    assert status(image(parts(), total=len(good) + 1)) == capi.LL_ERR_INVALID
    assert status(good + b"\0") == capi.LL_ERR_INVALID
    assert status(image(parts(), offsets={3: len(good) - 4})) == capi.LL_ERR_INVALID        # outside the image
    assert status(image(parts(), offsets={3: HEADER - 8})) == capi.LL_ERR_INVALID           # inside the header
    p = parts()
    assert status(image(p, offsets={3: HEADER + len(p[0]) + len(p[1]) + 8})) == capi.LL_ERR_INVALID   # overlapping its neighbour


# ---------------------------------------------------------------------------------------------- content, each rule on both sides of its bound
def test_config_and_scalars():
    assert status(with_part(0, config(scans_of_each_keyframe=6, scans_between_two_keyframe=5))) == capi.LL_OK
    assert status(with_part(0, config(scans_of_each_keyframe=6, scans_between_two_keyframe=6))) == capi.LL_ERR_INVALID
    assert status(with_part(0, config()[:-8])) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(stamp=float("nan")))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(t=(0.0, float("inf"), 0.0)))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(mode=2))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(pieces=0))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(stopped=1))) == capi.LL_OK
    assert status(with_part(1, scalars(stopped=2))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(n_dropped=-1))) == capi.LL_ERR_INVALID
    assert status(with_part(1, scalars(cell_res=0.0))) == capi.LL_ERR_INVALID


def test_cell_map():
    assert status(with_part(2, cells(keys=[key(0, 0, k) for k in range(5)]))) == capi.LL_OK
    assert status(with_part(2, cells(keys=[key(0, 0, 0)] * 2 + [key(0, 0, k) for k in range(2, 5)]))) == capi.LL_ERR_INVALID   # not strictly ascending
    assert status(with_part(2, cells(keys=[key(0, 0, k) for k in range(4)] + [1 << 63]))) == capi.LL_ERR_INVALID            # bit 63
    assert status(with_part(2, cells(stamps=([0, 1, 2, 3, 12], [1, 2, 3, 4, 12])))) == capi.LL_OK                           # stamp = frame index
    assert status(with_part(2, cells(stamps=([0, 1, 2, 3, 13], [1, 2, 3, 4, 12])))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(cur=(0, 1, 0, 2, -1)))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(ranks=(0, 1, 1, 2, 3, 3, 3, 4, 4)))) == capi.LL_OK                                     # rank = cells - 1
    assert status(with_part(2, cells(ranks=(0, 1, 1, 2, 3, 3, 3, 4, 5)))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(ords=(0, 1, 0, 0, 2, 1, 2, 0, -1)))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(ords=(0, 1, 0, 0, 2, 1, 2, 0, 1)))) == capi.LL_ERR_INVALID                              # above the cell's current
    bad = np.zeros((9, 3), "<f4")
    bad[4, 1] = np.inf
    assert status(with_part(2, cells(pts=bad))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells()[:-4])) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(n_out_of_range=-1))) == capi.LL_ERR_INVALID


def test_history():
    assert status(with_part(3, history(sizes=()))) == capi.LL_OK
    h = bytearray(history())
    h[16:20] = struct.pack("<i", 4)   # sizes no longer sum to the points
    assert status(with_part(3, bytes(h))) == capi.LL_ERR_INVALID


def test_open_keyframes():
    assert status(with_part(4, open_kfs(((4, 4, [(4, 0)]), (2, 2, [(3, 2)]), (0, 0, []))))) == capi.LL_OK   # the last cell, its only incarnation
    for bad in (((4, 4, [(5, 0)]), (2, 2, []), (0, 0, [])),            # no such cell
                ((4, 4, [(1, 2)]), (2, 2, []), (0, 0, [])),            # incarnation above the cell's current
                ((4, 4, [(1, 1), (1, 0)]), (2, 2, []), (0, 0, [])),    # not ascending
                ((4, 4, [(1, 1), (1, 1)]), (2, 2, []), (0, 0, [])),    # repeated
                ((4, 4, []), (2, 2, []), (0, 0, [(0, 0)])),            # cells without an append
                ((-1, 4, []), (2, 2, []), (0, 0, []))):
        assert status(with_part(4, open_kfs(bad))) == capi.LL_ERR_INVALID, bad
    assert status(with_part(4, open_kfs()[:-8])) == capi.LL_ERR_INVALID


def test_closed_keyframes_and_accumulated_clouds():
    p = parts()
    # edges = keyframes - 1
    assert status(with_part(7, b"")) == capi.LL_ERR_INVALID
    assert status(with_part(7, edge(0, 1) + edge(1, 2))) == capi.LL_ERR_INVALID
    assert status(with_part(7, edge(1, 0))) == capi.LL_ERR_INVALID
    assert status(with_part(6, pose(0.0) + pose(float("nan")))) == capi.LL_ERR_INVALID
    assert status(with_part(5, bytes(info()) + bytes(info(line_points=3, plane_points=4, all_points=7)))) == capi.LL_ERR_INVALID   # clouds now 12
    assert status(with_part(5, bytes(info()) + bytes(info(line_points=4, plane_points=4, all_points=7)))) == capi.LL_ERR_INVALID   # > all_points
    assert status(with_part(8, p[8][:-4])) == capi.LL_ERR_INVALID
    # accumulated: one per closed keyframe and per open one but the newest; ends non-decreasing
    assert status(with_part(10, accumulated((0, 0, 0, 0)))) == capi.LL_OK
    assert status(with_part(10, accumulated((5, 4, 9, 12)))) == capi.LL_ERR_INVALID
    assert status(with_part(10, accumulated((5, 5, 12)))) == capi.LL_ERR_INVALID
    acc = bytearray(accumulated())
    acc[-4 * 4:-4 * 4 + 4] = struct.pack("<f", np.nan)
    assert status(with_part(10, bytes(acc))) == capi.LL_ERR_INVALID


def test_the_loop_and_the_events():
    # closed: two keyframes at least, the edge's ids in range; unclosed: no loop section
    assert status(with_part(11, edge(0, 1) + pose(0.0) + pose(0.3))) == capi.LL_ERR_INVALID
    assert status(with_part(11, edge(0, 2) + pose(0.0) + pose(0.3), closed=True)) == capi.LL_ERR_INVALID
    assert status(with_part(11, edge(1, 0) + pose(0.0) + pose(0.3), closed=True)) == capi.LL_OK
    assert status(with_part(11, edge(0, 1) + pose(0.0), closed=True)) == capi.LL_ERR_INVALID
    one = parts(closed=True)
    one[1] = scalars(closed=1, n_keyframes=1, n_open=4)
    one[5], one[6], one[7], one[8], one[9] = bytes(info()), pose(0.0), b"", np.zeros(IMG, "<f4").tobytes(), points(5, 5)
    one[11] = edge(0, 0) + pose(0.0)
    assert status(image(one)) == capi.LL_ERR_INVALID   # a closed image with one keyframe
    one[1] = scalars(closed=0, n_keyframes=1, n_open=4)
    one[4] = open_kfs(((4, 4, []), (3, 3, []), (2, 2, []), (0, 0, [])))
    one[11] = b""
    assert status(image(one)) == capi.LL_OK
    # at most LL_LOOP_LOG events, of known kinds
    p = parts()
    p[1], p[12] = scalars(n_events=capi.LL_LOOP_LOG), events([0] * capi.LL_LOOP_LOG)
    assert status(image(p)) == capi.LL_OK
    p[1], p[12] = scalars(n_events=capi.LL_LOOP_LOG + 1), events([0] * (capi.LL_LOOP_LOG + 1))
    assert status(image(p)) == capi.LL_ERR_INVALID
    assert status(with_part(12, events((0, 4)))) == capi.LL_ERR_INVALID
    timed = capi.LoopEvent(kind=capi.LL_LOOP_CLOSED, keyframe=1)
    timed.summary.cycles_total = 1   # timing counters are saved as 0
    assert status(with_part(12, events((0,)) + bytes(timed))) == capi.LL_ERR_INVALID
    timed.summary.cycles_total = 0
    assert status(with_part(12, events((0,)) + bytes(timed))) == capi.LL_OK


def test_a_full_table_is_reported_not_refused():
    """More cells than half the table of the image's max_cells: a mapper loaded with a larger max_cells saves such images, so the host check
    reports the count; ll_mapper_loop_load refuses it (LL_ERR_CAPACITY) unless its cfg's max_cells holds them."""
    n = 2049   # more than half of the smallest table (4096 slots, max_cells <= 2048)
    p = parts()
    p[0] = config(max_cells=2048)
    p[2] = cells(keys=[key(0, 0, k) for k in range(n)], stamps=(np.zeros(n, int), np.zeros(n, int)), cur=[0] * n, ranks=(), ords=(), pts=np.zeros((0, 3), "<f4"))
    p[4] = open_kfs(((4, 4, []), (2, 2, []), (0, 0, [])))
    st, got = summary(image(p))
    assert st == capi.LL_OK and got.cells == n
    from loam_livox_b200.registration import loop_image_info
    assert loop_image_info(image(p))["cells"] == n


def test_max_cells_above_2_29_is_refused():
    assert status(with_part(0, config(max_cells=2**29))) == capi.LL_OK
    assert status(with_part(0, config(max_cells=2**29 + 1))) == capi.LL_ERR_INVALID   # ll_cellmap_create refuses it


def test_config_padding_must_be_zero():
    fields = capi.LoopClosureCfg._fields_
    ends = [getattr(capi.LoopClosureCfg, f).offset + C.sizeof(t) for f, t in fields]
    starts = [getattr(capi.LoopClosureCfg, f).offset for f, _ in fields[1:]] + [C.sizeof(capi.LoopClosureCfg)]
    gaps = [e for e, s in zip(ends, starts) if s > e]
    assert gaps   # the struct has padding (after max_cells and after reserve_keyframes)
    for g in gaps:
        c = bytearray(config())
        c[g] = 1
        assert status(with_part(0, bytes(c))) == capi.LL_ERR_INVALID, g


def test_incarnation_and_history_bounds():
    # a cell's current ordinal is at most current_frame_idx (one revisit per cell and append)
    assert status(with_part(2, cells(cur=(0, 1, 0, 12, 0), ords=(0, 1, 0, 0, 12, 1, 2, 0, 0)))) == capi.LL_OK
    assert status(with_part(2, cells(cur=(0, 1, 0, 13, 0), ords=(0, 1, 0, 0, 13, 1, 2, 0, 0)))) == capi.LL_ERR_INVALID
    assert status(with_part(2, cells(cur=(0, 1, 0, 2**31 - 1, 0), ords=(0, 1, 0, 0, 2, 1, 2, 0, 0)))) == capi.LL_ERR_INVALID
    # history segments at most the stamp's maximum_history_size (two segments in parts())
    assert status(with_part(1, scalars(history=2))) == capi.LL_OK
    assert status(with_part(1, scalars(history=1))) == capi.LL_ERR_INVALID


# ---------------------------------------------------------------------------------------------- ABI
def test_symbols_and_signatures():
    L = capi.lib()
    for name, n_params in (("ll_mapper_loop_save", 4), ("ll_mapper_loop_load", 4), ("ll_loop_image_info", 3)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name
    n = C.c_size_t()
    assert L.ll_mapper_loop_save(None, None, 0, C.byref(n)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_loop_load(None, None, 0, None) == capi.LL_ERR_INVALID
    assert L.ll_loop_image_info(None, 0, None) == capi.LL_ERR_INVALID


def test_struct_layouts_equal_the_ctypes_mirrors(tmp_path):
    exe = _compile(tmp_path, "loop_image_mirror")
    r = subprocess.run([exe, "layout"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    mirrors = {"ll_loop_image_scalars": capi.LoopImageScalars, "ll_loop_image_summary": capi.LoopImageSummary}
    sizes = {"ll_loop_image_header": HEADER, "ll_loop_image_scalars": 112, "ll_loop_image_summary": 96, "ll_loop_image_open": 16, "ll_loop_image_ref": 8,
             "ll_keyframe_info": C.sizeof(capi.KeyframeInfo), "ll_pose": C.sizeof(capi.Pose), "ll_pg_edge": C.sizeof(capi.PgEdge)}
    seen = set()
    for line in r.stdout.splitlines():
        name, field, value = line.split()
        if field == "sizeof":
            assert sizes[name] == int(value), name
            if name in mirrors:
                assert C.sizeof(mirrors[name]) == int(value), name
        else:
            assert getattr(mirrors[name], field).offset == int(value), (name, field)
            seen.add((name, field))
    for name, cls in mirrors.items():
        assert {f for f, _ in cls._fields_} == {f for s, f in seen if s == name}, name
    assert len(scalars()) == 112


def test_cpp_mirror_loop_image_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "loop_image_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
