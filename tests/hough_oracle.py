"""ctypes binding of the CPU oracle of HoughTransform (oracle/zo_hough.cpp -> oracle/libzo_hough.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile;
__graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from oracle_lib import OracleStatus, ZoImage, as_image, load


class ZoHoughLine(C.Structure):
    _fields_ = [("angle", C.c_float), ("radius", C.c_float), ("score", C.c_uint32), ("p1x", C.c_float), ("p1y", C.c_float),
                ("p2x", C.c_float), ("p2y", C.c_float)]


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_hough.so")
    img = C.POINTER(ZoImage)
    u32 = C.c_uint32
    L.zo_hough_tables.argtypes = [u32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.zo_hough_compute.argtypes = [u32, img, u32, u32, u32, u32, img]
    L.zo_hough_find_lines.argtypes = [u32, img, u32, C.c_float, C.c_float, C.POINTER(ZoHoughLine), u32, C.POINTER(u32)]
    return L


def tables(size):
    """HoughTransform.init (hough.zig:38-66) -> (cos_table, sin_table) as int32 arrays."""
    cos_t, sin_t = np.zeros(max(size, 0), np.int32), np.zeros(max(size, 0), np.int32)
    rc = lib().zo_hough_tables(int(size), cos_t.ctypes.data_as(C.POINTER(C.c_int32)), sin_t.ctypes.data_as(C.POINTER(C.c_int32)))
    if rc != 0:
        raise OracleStatus(rc, "hough_tables")
    return cos_t, sin_t


def compute(size, edges, box, accumulator):
    """HoughTransform.compute (hough.zig:75-139): adds into `accumulator` (uint32, size x size, may be a strided view)."""
    assert edges.dtype == np.uint8 and accumulator.dtype == np.uint32
    l, t, r, b = box
    rc = lib().zo_hough_compute(int(size), as_image(edges), int(l), int(t), int(r), int(b), as_image(accumulator))
    if rc != 0:
        raise OracleStatus(rc, "hough_compute")
    return accumulator


def find_lines(size, accumulator, threshold, angle_nms, radius_nms):
    """HoughTransform.findLines (hough.zig:142-204) -> list of (angle, radius, score, p1x, p1y, p2x, p2y) with f32 values."""
    acc = np.ascontiguousarray(accumulator, dtype=np.uint32) if accumulator.dtype != np.uint32 else accumulator
    n = C.c_uint32(0)
    rc = lib().zo_hough_find_lines(int(size), as_image(acc), int(threshold), C.c_float(angle_nms), C.c_float(radius_nms), None, 0, C.byref(n))
    if rc != 0:
        raise OracleStatus(rc, "hough_find_lines")
    out = (ZoHoughLine * max(n.value, 1))()
    lib().zo_hough_find_lines(int(size), as_image(acc), int(threshold), C.c_float(angle_nms), C.c_float(radius_nms), out, n.value, C.byref(n))
    return [(o.angle, o.radius, int(o.score), o.p1x, o.p1y, o.p2x, o.p2y) for o in out[:n.value]]
