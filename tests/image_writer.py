"""The parts of a NumPy writer of the documented byte-image layout (include/loamlivox_b200.h) that the mapper image and the loop image share: the
header with its (offset, length) pairs, the history section, the cell and cell-point records and the packed cell key."""
import struct

import numpy as np

CELL = np.dtype([("key", "<u8"), ("create_frame", "<i4"), ("last_update", "<i4")])   # ll_image_cell
CELL_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("cell", "<i4")])    # ll_image_cell_point
BIAS = 1 << 20


def key(k, j, i):
    return ((k + BIAS) << 42) | ((j + BIAS) << 21) | (i + BIAS)


def history(sizes, pts) -> bytes:
    """A history section: the segment sizes, then the (n, 4) float32 points they sum to."""
    return struct.pack("<qq", len(sizes), int(sum(sizes))) + np.asarray(sizes, "<i4").tobytes() + pts.tobytes()


def image(sections, magic, config_bytes, version=1, total=None, offsets=None) -> bytes:
    """Header + the sections back to back in index order (offsets: per-section overrides)."""
    offs, off = [], 24 + 16 * len(sections)
    for s in sections:
        offs.append(off)
        off += len(s)
    for k, o in (offsets or {}).items():
        offs[k] = o
    head = struct.pack("<8sIIQ", magic, version, config_bytes, off if total is None else total)
    head += b"".join(struct.pack("<QQ", o, len(s)) for o, s in zip(offs, sections))
    return head + b"".join(sections)
