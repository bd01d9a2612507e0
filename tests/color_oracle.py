"""ctypes binding of the CPU oracle of convertColor between the 33 colour formats (oracle/zo_color.cpp -> oracle/libzo_color.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile;
__graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).
A format is a (space, component) pair of ints in the C ABI's numbering (zignal_b200.ColorSpace / Component).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from oracle_lib import load

NP = {0: np.uint8, 1: np.float32, 2: np.float64}


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_color.so")
    i, vp = C.c_int, C.c_void_p
    L.zo_color_valid.argtypes = [i, i]
    L.zo_color_path.argtypes = [i, i, i, i, C.POINTER(C.c_uint32)]
    L.zo_convert_color.argtypes = [vp, i, i, vp, i, i, C.c_size_t]
    return L


def channels(space: int) -> int:
    return 4 if space == 9 else 1 if space in (0, 13) else 3


def valid(space: int, component: int) -> bool:
    return bool(lib().zo_color_valid(int(space), int(component)))


def path(src, dst) -> list:
    """The spaces convertColor visits after the source's (empty for a scalar <-> scalar or same-space pair)."""
    h = C.c_uint32()
    n = lib().zo_color_path(int(src[0]), int(src[1]), int(dst[0]), int(dst[1]), C.byref(h))
    assert n >= 0, (src, dst)
    return [(h.value >> (4 * k)) & 15 for k in range(n)]


def convert(a: np.ndarray, src, dst) -> np.ndarray:
    """convertColor(dst, px) for every pixel of a, an array of shape (..., channels) (no channel axis for one channel)."""
    ss, sc = int(src[0]), int(src[1])
    ds, dc = int(dst[0]), int(dst[1])
    a = np.ascontiguousarray(a, dtype=NP[sc])
    ns, nd = channels(ss), channels(ds)
    lead = a.shape if ns == 1 else a.shape[:-1]
    assert ns == 1 or a.shape[-1] == ns
    out = np.empty(lead + ((nd,) if nd > 1 else ()), NP[dc])
    n = int(np.prod(lead))
    rc = lib().zo_convert_color(a.ctypes.data, ss, sc, out.ctypes.data, ds, dc, n)
    if rc:
        raise ValueError(f"invalid format pair {src} -> {dst}")
    return out
