"""ctypes binding of the CPU oracle of the 8-bit histogram family and binary morphology (oracle/zo_binary.cpp -> oracle/libzo_binary.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile
(the main oracle's flags: -ffp-contract=off, no fast math); __graft_entry__.build() runs it and lib() repeats it (make rebuilds only when the
source is newer).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from oracle_lib import OracleStatus, ZoImage, as_image, load, pixfmt_of

MORPH = {"dilate": 0, "erode": 1, "open": 2, "close": 3}


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_binary.so")
    P = C.POINTER
    img = P(ZoImage)
    u8p = P(C.c_uint8)
    L.zo_histogram.argtypes = [img, C.c_int, P(C.c_uint32)]
    L.zo_autocontrast.argtypes = [img, C.c_int, C.c_float]
    L.zo_equalize.argtypes = [img, C.c_int]
    L.zo_threshold_otsu.argtypes = [img, img, u8p]
    L.zo_threshold_adaptive_mean.argtypes = [img, img, C.c_uint32, C.c_float]
    L.zo_morph_binary.argtypes = [img, img, u8p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int]
    return L


def _check(rc, what):
    if rc != 0:
        raise OracleStatus(rc, what)


def histogram(src):
    """Image.histogram (image.zig:1161-1185) -> (channels, 256) uint32."""
    ch = 1 if src.ndim == 2 else src.shape[2]
    counts = np.zeros((ch, 256), np.uint32)
    _check(lib().zo_histogram(as_image(src), pixfmt_of(src), counts.ctypes.data_as(C.POINTER(C.c_uint32))), "histogram")
    return counts


def autocontrast(src, cutoff=0.0):
    """Image.autocontrast (enhancement.zig:11-80) on a copy of src."""
    out = np.ascontiguousarray(src).copy()
    _check(lib().zo_autocontrast(as_image(out), pixfmt_of(out), C.c_float(cutoff)), "autocontrast")
    return out


def equalize(src):
    """Image.equalize (enhancement.zig:84-252) on a copy of src (64-bit numerator)."""
    out = np.ascontiguousarray(src).copy()
    _check(lib().zo_equalize(as_image(out), pixfmt_of(out)), "equalize")
    return out


def threshold_otsu(src, out=None):
    """Image(u8).thresholdOtsu (binary.zig:38-84) -> (out, threshold)."""
    out = np.zeros_like(src) if out is None else out
    t = C.c_uint8(0)
    _check(lib().zo_threshold_otsu(as_image(src), as_image(out), C.byref(t)), "threshold_otsu")
    return out, int(t.value)


def threshold_adaptive_mean(src, radius, c, out=None):
    """Image(u8).thresholdAdaptiveMean (binary.zig:86-119)."""
    out = np.zeros_like(src) if out is None else out
    _check(lib().zo_threshold_adaptive_mean(as_image(src), as_image(out), radius, C.c_float(c)), "threshold_adaptive_mean")
    return out


def morph_binary(src, kernel, iterations, op, out=None):
    """dilate / erode / open / close (binary.zig:121-280); op is a MORPH key, kernel a 2-D uint8 array."""
    k = np.ascontiguousarray(kernel, dtype=np.uint8)
    out = np.zeros_like(src) if out is None else out
    _check(lib().zo_morph_binary(as_image(src), as_image(out), k.ctypes.data_as(C.POINTER(C.c_uint8)), k.shape[0], k.shape[1], iterations,
                                 MORPH[op]), "morph_binary")
    return out
