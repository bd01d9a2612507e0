"""ctypes binding of the CPU oracle of Matrix.lu, LuResult.solve, det, inv and chol (oracle/zo_linsolve.cpp -> oracle/libzo_linsolve.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by
oracle/Makefile; __graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).
Each function returns (status, result...) with status 0, 32 (Singular) or 33 (NotPositiveDefinite); matrices are numpy arrays.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from oracle_lib import load

SINGULAR, NOT_POSITIVE_DEFINITE = 32, 33


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_linsolve.so")
    vp, i = C.c_void_p, C.c_int
    for s in ("f32", "f64"):
        getattr(L, f"zo_lu_{s}").argtypes = [vp, i, vp, vp, vp, vp]
        getattr(L, f"zo_lu_solve_{s}").argtypes = [vp, vp, vp, i, vp, i, vp]
        for name in ("det", "inv", "chol"):
            getattr(L, f"zo_{name}_{s}").argtypes = [vp, i, vp]
        for name in ("lu", "lu_solve", "det", "inv", "chol"):
            getattr(L, f"zo_{name}_{s}").restype = i
    return L


def _fn(name, a):
    return getattr(lib(), f"zo_{name}_{'f64' if a.dtype == np.float64 else 'f32'}")


def _sq(a):
    a = np.ascontiguousarray(a)
    assert a.ndim == 2 and a.shape[0] == a.shape[1] and a.dtype in (np.float32, np.float64)
    return a


def lu(a):
    """-> (l, u, p, sign)"""
    a = _sq(a)
    n = a.shape[0]
    l, u = np.zeros_like(a), np.zeros_like(a)
    p = np.zeros(n, np.uint32)
    sign = np.zeros(1, a.dtype)
    _fn("lu", a)(a.ctypes.data, n, l.ctypes.data, u.ctypes.data, p.ctypes.data, sign.ctypes.data)
    return l, u, p, sign[0]


def lu_solve(l, u, p, b):
    """-> (status, x)"""
    b = np.ascontiguousarray(b, dtype=l.dtype)
    x = np.zeros_like(b)
    p = np.ascontiguousarray(p, np.uint32)
    st = _fn("lu_solve", l)(l.ctypes.data, u.ctypes.data, p.ctypes.data, l.shape[0], b.ctypes.data, b.shape[1], x.ctypes.data)
    return st, x


def solve(a, b):
    """Matrix.solve: -> (status, x)"""
    l, u, p, _ = lu(a)
    return lu_solve(l, u, p, b)


def det(a):
    a = _sq(a)
    assert a.shape[0] > 0
    out = np.zeros(1, a.dtype)
    _fn("det", a)(a.ctypes.data, a.shape[0], out.ctypes.data)
    return out[0]


def inv(a):
    """-> (status, inverse)"""
    a = _sq(a)
    assert a.shape[0] > 0
    out = np.zeros_like(a)
    return _fn("inv", a)(a.ctypes.data, a.shape[0], out.ctypes.data), out


def chol(a):
    """-> (status, l)"""
    a = _sq(a)
    out = np.zeros_like(a)
    return _fn("chol", a)(a.ctypes.data, a.shape[0], out.ctypes.data), out
