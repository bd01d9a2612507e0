"""ctypes binding of the CPU oracle of colour quantization and dithering (oracle/zo_quantize.cpp -> oracle/libzo_quantize.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile;
__graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).  Images of a type other than Rgb(u8)
are converted with the main oracle's convertColor (oracle_lib.convert) first, as medianCut and the index lookup do per pixel.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import oracle_lib
from oracle_lib import OracleStatus, as_image, load

FIXED_6X7X6, FIXED_VGA16, FIXED_WEB216, ADAPTIVE = 0, 1, 2, 3
NONE, FLOYD_STEINBERG, ATKINSON, ORDERED, AUTO = 0, 1, 2, 3, 4
NO_PALETTE_COLORS = 28


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_quantize.so")
    vp, u32 = C.c_void_p, C.c_uint32
    L.zo_median_cut.argtypes = [vp, C.c_uint16, vp, u32, C.POINTER(u32)]
    L.zo_build_palette.argtypes = [vp, C.c_int, C.c_uint16, vp, C.POINTER(u32)]
    L.zo_color_lut.argtypes = [vp, u32, vp]
    L.zo_dither.argtypes = [vp, vp, u32, vp, C.c_int]
    L.zo_palette_lookup.argtypes = [vp, vp, vp]
    L.zo_heap_sort_u8.argtypes = [vp, u32]
    L.zo_heap_sort_u8.restype = None
    for name in ("zo_median_cut", "zo_build_palette", "zo_color_lut", "zo_dither", "zo_palette_lookup"):
        getattr(L, name).restype = C.c_int
    return L


def as_rgb8(img: np.ndarray) -> np.ndarray:
    """convertColor(Rgb, px) over the image (a view is kept as it is when it already is Rgb(u8))."""
    if img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3:
        return img
    return oracle_lib.convert(np.ascontiguousarray(img), 2)


def _check(rc, what):
    if rc != 0:
        raise OracleStatus(rc, what)


def median_cut(img: np.ndarray, max_colors=256, cap=256) -> np.ndarray:
    """medianCut (quantize.zig:175-412): the (n, 3) palette.  NoPaletteColors raises OracleStatus with status 28."""
    src = as_rgb8(img)
    out = np.zeros((max(int(cap), 1), 3), np.uint8)
    n = C.c_uint32(0)
    _check(lib().zo_median_cut(C.byref(as_image(src)), int(max_colors), out.ctypes.data, int(cap), C.byref(n)), "median_cut")
    return out[:n.value].copy()


def build_palette(img, mode, max_colors=256) -> np.ndarray:
    src = as_rgb8(img) if img is not None else None
    out = np.zeros((256, 3), np.uint8)
    n = C.c_uint32(0)
    _check(lib().zo_build_palette(C.byref(as_image(src)) if src is not None else None, int(mode), int(max_colors), out.ctypes.data,
                                  C.byref(n)), "build_palette")
    return out[:n.value].copy()


def color_lut(palette) -> np.ndarray:
    p = np.ascontiguousarray(np.asarray(palette, np.uint8).reshape(-1, 3))
    lut = np.zeros(32768, np.uint8)
    _check(lib().zo_color_lut(p.ctypes.data, p.shape[0], lut.ctypes.data), "color_lut")
    return lut


def dither(img: np.ndarray, palette, lut: np.ndarray, mode) -> np.ndarray:
    """dither.apply (dither.zig:34-41) in place on an Rgb(u8) image (may be a row-strided view); returns img."""
    p = np.ascontiguousarray(np.asarray(palette, np.uint8).reshape(-1, 3))
    _check(lib().zo_dither(C.byref(as_image(img)), p.ctypes.data, p.shape[0], np.ascontiguousarray(lut).ctypes.data, int(mode)), "dither")
    return img


def palette_lookup(img: np.ndarray, lut: np.ndarray) -> np.ndarray:
    src = as_rgb8(img)
    out = np.zeros(src.shape[:2], np.uint8)
    _check(lib().zo_palette_lookup(C.byref(as_image(src)), np.ascontiguousarray(lut).ctypes.data, C.byref(as_image(out))), "palette_lookup")
    return out


def heap_sort_u8(values) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(values, np.uint8)).copy()
    lib().zo_heap_sort_u8(a.ctypes.data, a.size)
    return a
