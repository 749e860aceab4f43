"""Host-only checks of the mapper image (include/loamlivox_b200.h, "checkpoint"): a small NumPy writer of the documented layout builds valid
images that ll_mapper_image_info accepts and reports; the validator refuses every kind of corruption before any device is involved; the
ctypes struct has the header's size; and the C++ mirror's save / load compiles, links and runs (without a GPU it stops at the context)."""
import ctypes as C
import functools
import os
import struct
import subprocess

import numpy as np
import pytest

import image_writer
from image_writer import CELL, CELL_POINT, key
from loam_livox_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = 8 + 4 + 4 + 8 + 16 * capi.LL_IMAGE_SECTIONS   # ll_mapper_image_header


# ---------------------------------------------------------------------------------------------- writer of the documented layout
def config(**kw) -> bytes:
    c = capi.MapperConfig()
    capi.lib().ll_mapper_config_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return bytes(c)


def scalars(frame_index=6, map_dirty=1, have_map=1, snap_n=(2, 3), fov=(4, 5), reserved=0, q=(1.0, 0, 0, 0), t=(0.5, -0.25, 0.0),
            last_time_stamp=0.1, times=(100.0, 0.5, 0.6)) -> bytes:
    return struct.pack("<8i18d", frame_index, map_dirty, have_map, *snap_n, *fov, reserved, last_time_stamp, *q, *t, *q, *t, *times)


def points(n, seed):
    return np.random.default_rng(seed).uniform(-20, 20, (n, 4)).astype("<f4")


def history(sizes, seed) -> bytes:
    return image_writer.history(sizes, points(int(sum(sizes)), seed))


def snapshot(n, seed) -> bytes:
    return struct.pack("<q", n) + points(n, seed).tobytes()


def cellmap(frame_idx=6, n_out_of_range=0, n_cells=5, n_points=9, seed=0, cells=None, pts=None) -> bytes:
    if cells is None:
        cells = np.zeros(n_cells, CELL)
        cells["key"] = sorted(key(k, -k, 2 * k) for k in range(n_cells))
        cells["create_frame"] = np.arange(n_cells) % max(frame_idx, 1)
        cells["last_update"] = np.minimum(cells["create_frame"] + 1, frame_idx)
    if pts is None:
        pts = np.zeros(n_points, CELL_POINT)
        p = points(n_points, seed + 1)
        pts["x"], pts["y"], pts["z"] = p[:, 0], p[:, 1], p[:, 2]
        pts["cell"] = np.arange(n_points) % max(len(cells), 1)
    return struct.pack("<iiqq", frame_idx, n_out_of_range, len(cells), len(pts)) + cells.tobytes() + pts.tobytes()


def parts(**cfg):
    """The eight sections of a valid image, in index order: a mode-1 mapper after six scans."""
    return [config(**({"matching_mode": 1} | cfg)), scalars(), history([3, 0, 2], 1), history([4, 1, 1], 2), snapshot(2, 3), snapshot(3, 4),
            cellmap(seed=5), cellmap(n_cells=7, n_points=4, seed=6)]


image = functools.partial(image_writer.image, magic=b"LLMAPIMG", config_bytes=C.sizeof(capi.MapperConfig))


def info(img):
    out = capi.ImageInfo()
    buf = np.frombuffer(img, np.uint8) if len(img) else np.zeros(1, np.uint8)
    return capi.lib().ll_mapper_image_info(buf.ctypes.data, len(img), C.byref(out)), out


def status(img):
    return info(img)[0]


# ---------------------------------------------------------------------------------------------- valid images
def test_struct_sizes_match_the_header():
    assert C.sizeof(capi.ImageInfo) == 112
    assert HEADER == 152 and len(scalars()) == 176 and CELL.itemsize == CELL_POINT.itemsize == 16


def test_valid_images_are_accepted_and_reported():
    st, got = info(image(parts()))
    assert st == capi.LL_OK
    assert (got.version, got.matching_mode, got.frame_index, got.have_map, got.map_dirty) == (1, 1, 6, 1, 1)
    assert list(got.history_segments) == [3, 3] and list(got.history_points) == [5, 6] and list(got.snapshot_points) == [2, 3]
    assert list(got.cells) == [5, 7] and list(got.cell_points) == [9, 4] and list(got.cell_frame_idx) == [6, 6]
    assert got.bytes == len(image(parts()))
    # a fresh mapper: nothing in it
    fresh = [config(), scalars(frame_index=0, map_dirty=0, have_map=0, snap_n=(0, 0), fov=(0, 0), times=(-1.0, 0.0, 0.0)), history([], 0), history([], 0),
             snapshot(0, 0), snapshot(0, 0), cellmap(0, n_cells=0, n_points=0), cellmap(0, n_cells=0, n_points=0)]
    st, got = info(image(fresh))
    assert st == capi.LL_OK and list(got.cells) == [0, 0] and got.have_map == 0
    # no index: empty snapshot sections while snap_n keeps the counts the next stats report
    p = parts()
    p[1], p[4], p[5] = scalars(have_map=0, snap_n=(7, 0)), snapshot(0, 0), snapshot(0, 0)
    assert status(image(p)) == capi.LL_OK
    # sections need not be in index order
    p = parts()
    order = [0, 1, 7, 6, 5, 4, 3, 2]
    offs, off = {}, HEADER
    for k in order:
        offs[k] = off
        off += len(p[k])
    img = image(p, offsets=offs)
    body = b"".join(p[k] for k in order)
    assert status(img[:HEADER] + body) == capi.LL_OK
    from loam_livox_b200.registration import image_config, image_info
    assert image_info(image(parts()))["cells"] == [5, 7] and image_config(image(parts())).matching_mode == 1


def test_too_many_cells_for_the_table_is_a_capacity_error():
    p = parts(max_cells=2048)   # table of 4096 slots: at most 2048 cells
    assert status(image(p)) == capi.LL_OK
    p[6] = cellmap(n_cells=2049, n_points=3)
    assert status(image(p)) == capi.LL_ERR_CAPACITY


# ---------------------------------------------------------------------------------------------- refusals
def test_truncations_are_refused():
    img = image(parts())
    cuts = {0, 8, HEADER - 1, HEADER, len(img) - 1}
    off = HEADER
    for s in parts():
        cuts |= {off, off + len(s) - 1}
        off += len(s)
    for cut in sorted(cuts):
        assert status(img[:cut]) == capi.LL_ERR_INVALID, cut
    assert status(img + b"\0") == capi.LL_ERR_INVALID


def test_header_corruptions_are_refused():
    p = parts()
    assert status(image(p, magic=b"LLMAPIMH")) == capi.LL_ERR_INVALID
    assert status(image(p, version=2)) == capi.LL_ERR_INVALID
    assert status(image(p, config_bytes=C.sizeof(capi.MapperConfig) - 8)) == capi.LL_ERR_INVALID
    assert status(image(p, total=len(image(p)) + 16)) == capi.LL_ERR_INVALID


def test_overlapping_or_out_of_range_sections_are_refused():
    p = parts()
    n = len(image(p))
    off3 = HEADER + sum(len(s) for s in p[:3])
    for offsets in ({3: off3 - 1}, {3: off3 - 16}, {4: HEADER}, {0: 0}, {0: HEADER - 1}, {7: n - len(p[7]) + 1}, {7: n}, {6: 1 << 62}):
        assert status(image(p, offsets=offsets)) == capi.LL_ERR_INVALID, offsets


def patched(section, at, fmt, value):
    p = parts()
    b = bytearray(p[section])
    struct.pack_into(fmt, b, at, value)
    p[section] = bytes(b)
    return image(p)


def test_counts_that_disagree_are_refused():
    H, S, M = capi.LL_IMAGE_HISTORY_CORNER, capi.LL_IMAGE_SNAPSHOT_SURF, capi.LL_IMAGE_CELLS_SURF
    for sec, at, fmt, value in ((H, 0, "<q", 4), (H, 0, "<q", -1), (H, 8, "<q", 6), (H, 8, "<q", 1 << 61), (S, 0, "<q", 2), (S, 0, "<q", 4),
                                (M, 8, "<q", 8), (M, 16, "<q", 3), (M, 16, "<q", -1)):
        assert status(patched(sec, at, fmt, value)) == capi.LL_ERR_INVALID, (sec, at, value)
    # segment sizes that do not sum to the window's points (same length), or a negative one
    assert status(patched(H, 16, "<i", 4)) == capi.LL_ERR_INVALID
    assert status(patched(H, 16, "<i", -1)) == capi.LL_ERR_INVALID
    # snapshot count != snap_n, or points while there is no index
    p = parts()
    p[1] = scalars(snap_n=(2, 4))
    assert status(image(p)) == capi.LL_ERR_INVALID
    p = parts()
    p[1] = scalars(have_map=0)
    assert status(image(p)) == capi.LL_ERR_INVALID
    # scalars out of range
    for kw in (dict(map_dirty=2), dict(have_map=-1), dict(reserved=1), dict(frame_index=-1), dict(fov=(-1, 0))):
        p = parts()
        p[1] = scalars(**kw)
        assert status(image(p)) == capi.LL_ERR_INVALID, kw


def cells_with(mutate):
    c = np.frombuffer(parts()[6][24:24 + 5 * 16], CELL).copy()
    pts = np.frombuffer(parts()[6][24 + 5 * 16:], CELL_POINT).copy()
    mutate(c, pts)
    p = parts()
    p[6] = cellmap(cells=c, pts=pts)
    return image(p)


def test_bad_cell_lists_are_refused():
    assert status(cells_with(lambda c, p: None)) == capi.LL_OK
    def swap(c, p):
        c["key"][[1, 2]] = c["key"][[2, 1]]
    def dup(c, p):
        c["key"][3] = c["key"][2]
    def bit63(c, p):
        c["key"][4] |= np.uint64(1 << 63)
    def rank(c, p):
        p["cell"][0] = 5
    def rank_neg(c, p):
        p["cell"][0] = -1
    def create(c, p):
        c["create_frame"][1] = 7
    def last(c, p):
        c["last_update"][0] = 7
    def stamp_neg(c, p):
        c["create_frame"][2] = -1
    def nan_point(c, p):
        p["y"][3] = np.nan
    for f in (swap, dup, bit63, rank, rank_neg, create, last, stamp_neg, nan_point):
        assert status(cells_with(f)) == capi.LL_ERR_INVALID, f.__name__


def test_non_finite_values_are_refused():
    H, S = capi.LL_IMAGE_HISTORY_SURF, capi.LL_IMAGE_SNAPSHOT_CORNER
    assert status(patched(H, 16 + 3 * 4 + 16 * 2 + 4, "<f", np.inf)) == capi.LL_ERR_INVALID    # a history point's y
    assert status(patched(S, 8 + 16 + 8, "<f", np.nan)) == capi.LL_ERR_INVALID                   # a snapshot point's z
    for kw in (dict(q=(np.nan, 0, 0, 0)), dict(t=(0, np.inf, 0)), dict(last_time_stamp=np.nan), dict(times=(100.0, np.inf, 0.0))):
        p = parts()
        p[1] = scalars(**kw)
        assert status(image(p)) == capi.LL_ERR_INVALID, kw


def test_bad_configs_are_refused():
    for kw in (dict(matching_mode=2), dict(matching_mode=-1), dict(cell_resolution=0.0), dict(threshold_cell_revisit=0)):
        assert status(image(parts(**kw))) == capi.LL_ERR_INVALID, kw
    p = parts()
    p[0] = p[0][:-8]
    assert status(image(p)) == capi.LL_ERR_INVALID


def test_max_cells_above_2_29_is_refused():
    assert status(image(parts(max_cells=2**29))) == capi.LL_OK
    assert status(image(parts(max_cells=2**29 + 1))) == capi.LL_ERR_INVALID   # ll_cellmap_create refuses it


def test_null_arguments_are_refused():
    L = capi.lib()
    out = capi.ImageInfo()
    img = np.frombuffer(image(parts()), np.uint8)
    assert L.ll_mapper_image_info(None, 0, C.byref(out)) == capi.LL_ERR_INVALID
    assert L.ll_mapper_image_info(img.ctypes.data, img.shape[0], None) == capi.LL_ERR_INVALID
    n = C.c_size_t()
    assert L.ll_mapper_save(None, None, 0, C.byref(n)) == capi.LL_ERR_INVALID
    h = C.c_void_p()
    assert L.ll_mapper_load(None, img.ctypes.data, img.shape[0], None, C.byref(h)) == capi.LL_ERR_INVALID and not h.value


def test_cpp_mirror_save_load_compiles_links_and_runs(tmp_path):
    exe = str(tmp_path / "checkpoint_mirror")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "checkpoint_mirror.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)


@pytest.mark.parametrize("section", range(8))
def test_every_section_length_off_by_sixteen_is_refused(section):
    p = parts()
    p[section] = p[section] + bytes(16)
    assert status(image(p)) == capi.LL_ERR_INVALID
