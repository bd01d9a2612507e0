"""ctypes binding of the CPU oracle of Image.shenCastan (oracle/zo_shen_castan.cpp -> oracle/libzo_shen_castan.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by
oracle/Makefile against the main oracle (its summed-area tables are zo_integral_plane's); __graft_entry__.build() runs it and lib()
repeats it (make rebuilds only when a source is newer).
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass

import numpy as np

import oracle_lib
from oracle_lib import OracleStatus, as_image, load, pixfmt_of


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_shen_castan.so")
    img = C.POINTER(oracle_lib.ZoImage)
    L.zo_shen_castan.argtypes = [img, img, C.c_int, C.c_float, C.c_uint64, C.c_float, C.c_float, C.c_int, C.c_int,
                                 C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint64)]
    return L


@dataclass(frozen=True)
class Options:
    """The reference's ShenCastan options (ShenCastan.zig:9-37)."""
    smooth: float = 0.9
    window_size: int = 7
    high_ratio: float = 0.99
    low_rel: float = 0.5
    hysteresis: bool = True
    use_nms: bool = False


# ShenCastan.zig:51-99
PRESETS = {
    "default": Options(),
    "low_noise": Options(smooth=0.95, high_ratio=0.98),
    "high_noise": Options(smooth=0.7, window_size=11),
    "heavy_smooth": Options(smooth=0.5, window_size=9, high_ratio=0.95),
    "sensitive": Options(high_ratio=0.97, low_rel=0.4),
    "thin": Options(use_nms=True),
    "strong_only": Options(hysteresis=False),
}


def shen_castan_ex(src, opts: Options = Options(), out=None):
    """Image.shenCastan (image.zig:1015-1027, edges.zig:83-198) -> (edge map, t_high, t_low, candidate count)."""
    out = np.zeros(src.shape[:2], np.uint8) if out is None else out
    th, tl, cand = C.c_float(), C.c_float(), C.c_uint64()
    rc = lib().zo_shen_castan(as_image(src), as_image(out), pixfmt_of(src), C.c_float(opts.smooth), int(opts.window_size),
                              C.c_float(opts.high_ratio), C.c_float(opts.low_rel), int(bool(opts.hysteresis)), int(bool(opts.use_nms)),
                              C.byref(th), C.byref(tl), C.byref(cand))
    if rc != 0:
        raise OracleStatus(rc, "shen_castan")
    return out, th.value, tl.value, cand.value


def shen_castan(src, opts: Options = Options(), out=None):
    return shen_castan_ex(src, opts, out)[0]
