"""ctypes binding of the CPU oracle of Image.floodFill (oracle/zo_flood_fill.cpp -> oracle/libzo_flood_fill.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by
oracle/Makefile; __graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from oracle_lib import OracleStatus, as_image, load

SEED, NEIGHBOR = 0, 1
OUT_OF_BOUNDS = 27


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_flood_fill.so")
    L.zo_flood_fill.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_void_p, C.c_double, C.c_int, C.c_int]
    L.zo_flood_fill.restype = C.c_int
    return L


def pixfmt_of(img: np.ndarray) -> int:
    ch = img.shape[2] if img.ndim == 3 else 1
    return {(np.uint8, 1): 0, (np.float32, 1): 1, (np.uint8, 3): 2, (np.uint8, 4): 3, (np.float32, 4): 4}[(img.dtype.type, ch)]


def fill_pixel(img: np.ndarray, fill_value) -> np.ndarray:
    """fill_value (a scalar, or a tuple of channels) as one packed pixel of img's type."""
    ch = img.shape[2] if img.ndim == 3 else 1
    px = np.asarray(fill_value, np.float64).astype(img.dtype).reshape(-1)
    assert px.size == ch, (fill_value, img.shape)
    return px


def flood_fill(img: np.ndarray, start_row, start_col, fill_value, threshold=0.0, connectivity=4, mode=SEED) -> np.ndarray:
    """Image.floodFill (flood_fill.zig:59-131) in place on `img` (may be a row-strided view); returns img.  OutOfBounds raises
    OracleStatus with status 27."""
    px = fill_pixel(img, fill_value)
    rc = lib().zo_flood_fill(C.byref(as_image(img)), pixfmt_of(img), int(start_row), int(start_col), px.ctypes.data, float(threshold),
                             int(connectivity), int(mode))
    if rc != 0:
        raise OracleStatus(rc, "flood_fill")
    return img
