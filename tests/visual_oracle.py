"""ctypes binding of the CPU oracle of Image.diff, applyColormap, flipLeftRight / flipTopBottom and invert (oracle/zo_visual.cpp ->
oracle/libzo_visual.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile;
__graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).
"""
from __future__ import annotations

import ctypes as C
import functools
import json
from pathlib import Path

import numpy as np

from oracle_lib import OracleStatus, ZoImage, load, pixfmt_of
from oracle_lib import as_image as _as_image

TABLES = Path(__file__).resolve().parent / "golden" / "colormap_tables.json"
JET, HEAT, TURBO, VIRIDIS, INFERNO = 0, 1, 2, 3, 4
MAPS = ("jet", "heat", "turbo", "viridis", "inferno")
STATS_FIELDS = ("n", "diff_count", "sum", "mean", "variance", "min", "max")


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_visual.so")
    vp, i, f, d = C.c_void_p, C.c_int, C.c_float, C.c_double
    L.zo_diff.argtypes = [vp, vp, vp, i, f, f, i, i, vp]
    L.zo_colormap_lut.argtypes = [i, vp]
    L.zo_apply_colormap.argtypes = [vp, i, vp, i, d, i, d, vp]
    for name in ("zo_flip_left_right", "zo_flip_top_bottom", "zo_invert"):
        getattr(L, name).argtypes = [vp, i]
    for name in ("zo_diff", "zo_colormap_lut", "zo_apply_colormap", "zo_flip_left_right", "zo_flip_top_bottom", "zo_invert"):
        getattr(L, name).restype = C.c_int
    return L


def as_image(a: np.ndarray):
    """oracle_lib.as_image, plus empty images (numpy gives them all-zero strides)."""
    return ZoImage(None, a.shape[0], a.shape[1], a.shape[1]) if a.size == 0 else _as_image(a)


def _check(rc, what):
    if rc != 0:
        raise OracleStatus(rc, what)


def diff(a: np.ndarray, b: np.ndarray, threshold=0.0, scale=1.0, binary=False, force_opaque=False, out=None):
    """diff.compute (diff.zig:27-203): (out, stats) with stats a dict of STATS_FIELDS (n and diff_count as int).  out may be a or b."""
    out = np.zeros_like(a) if out is None else out
    st = np.zeros(7, np.float64)
    _check(lib().zo_diff(C.byref(as_image(a)), C.byref(as_image(b)), C.byref(as_image(out)), pixfmt_of(a), float(threshold), float(scale),
                         int(bool(binary)), int(bool(force_opaque)), st.ctypes.data), "diff")
    stats = dict(zip(STATS_FIELDS, st.tolist()))
    stats["n"], stats["diff_count"] = int(stats["n"]), int(stats["diff_count"])
    return out, stats


def colormap_lut(cmap: int) -> np.ndarray:
    """The (256, 3) table of jet / heat / turbo (colormaps.zig:92-190); viridis / inferno from the data fixture."""
    if cmap in (VIRIDIS, INFERNO):
        return np.asarray(json.loads(TABLES.read_text())[MAPS[cmap]], np.uint8)
    lut = np.zeros((256, 3), np.uint8)
    _check(lib().zo_colormap_lut(int(cmap), lut.ctypes.data), "colormap_lut")
    return lut


def apply_colormap(src: np.ndarray, lut, min=None, max=None) -> np.ndarray:
    """Image.applyColormap (image.zig:1190-1247) with a (256, 3) table: the (rows, cols, 3) uint8 result."""
    lut = np.ascontiguousarray(lut, np.uint8)
    out = np.zeros(src.shape[:2] + (3,), np.uint8)
    _check(lib().zo_apply_colormap(C.byref(as_image(src)), pixfmt_of(src), lut.ctypes.data, int(min is not None),
                                   0.0 if min is None else float(min), int(max is not None), 0.0 if max is None else float(max),
                                   C.byref(as_image(out))), "apply_colormap")
    return out


def _in_place(fn, img: np.ndarray, what) -> np.ndarray:
    _check(fn(C.byref(as_image(img)), pixfmt_of(img)), what)
    return img


def flip_left_right(img: np.ndarray) -> np.ndarray:
    return _in_place(lib().zo_flip_left_right, img, "flip_left_right")


def flip_top_bottom(img: np.ndarray) -> np.ndarray:
    return _in_place(lib().zo_flip_top_bottom, img, "flip_top_bottom")


def invert(img: np.ndarray) -> np.ndarray:
    """In place; an f32 image raises OracleStatus 3 (a compile error in the reference)."""
    return _in_place(lib().zo_invert, img, "invert")
