"""Matrix.lu, LuResult.solve, solve, det, inv and chol without a GPU: the CPU oracle (oracle/zo_linsolve.cpp) against the reference's
own tests (src/matrix/test_ops_decomposition.zig, test_ops_determinant.zig, test_ops_inverse.zig), hand-derived closed forms, mpmath and
LAPACK; the two new status names; and the argument errors every device entry point returns before touching a device."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.linalg

import linsolve_oracle as lo

ROOT = Path(__file__).resolve().parent.parent
F64 = np.float64


def m(*rows, dtype=F64):
    return np.array(rows, dtype=dtype)


KAT_LU = m([2, 1, 1], [4, 3, 3], [8, 7, 9])
KAT_SPD = m([4, 2, 2], [2, 5, 3], [2, 3, 6])
KAT_DET3 = m([1, 2, 3], [0, 1, 4], [5, 6, 0])
KAT_4 = m([5, 1, 0, 2], [1, 4, 1, 1], [0, 1, 3, 0], [2, 1, 0, 4])
SING4_DET = m([1, 2, 3, 4], [2, 4, 6, 8], [3, 5, 7, 9], [4, 6, 8, 10])
SING4_INV = m([1, 2, 3, 4], [5, 6, 7, 8], [6, 8, 10, 12], [9, 10, 11, 12])


# ---- the reference's tests, on the oracle ----

def test_lu_kat():
    l, u, p, sign = lo.lu(KAT_LU)
    assert np.array_equal(np.diag(l), np.ones(3)) and np.all(np.triu(l, 1) == 0) and np.all(np.tril(u, -1) == 0)
    assert np.max(np.abs(KAT_LU[p] - l @ u)) < 1e-10
    assert sign in (1.0, -1.0)


def test_cholesky_kat():
    st, l = lo.chol(KAT_SPD)
    assert st == 0
    assert np.max(np.abs(l - m([2, 0, 0], [1, 2, 0], [1, 1, 2]))) < 1e-10
    assert np.max(np.abs(l @ l.T - KAT_SPD)) < 1e-10
    assert lo.chol(m([1, 2], [2, 1]))[0] == lo.NOT_POSITIVE_DEFINITE


def test_solve_kats():
    st, x = lo.solve(KAT_LU, m([7], [19], [49]))
    assert st == 0 and np.max(np.abs(x[:, 0] - [1, 2, 3])) < 1e-12
    a = m([3, 2], [1, 4])
    st, x = lo.solve(a, np.eye(2))
    assert st == 0 and np.max(np.abs(a @ x - np.eye(2))) < 1e-12
    assert lo.solve(m([1, 2], [2, 4]), m([1], [2]))[0] == lo.SINGULAR


def test_det_kats():
    assert lo.det(m([5])) == 5.0
    assert lo.det(m([4, 7], [2, 6])) == 10.0
    assert lo.det(KAT_DET3) == 1.0
    assert abs(lo.det(KAT_4)) > 1e-10
    assert abs(lo.det(SING4_DET)) < 1e-10
    assert lo.det(np.eye(5)) == 1.0


def test_inverse_kats():
    for a in (m([4, 7], [2, 6]), KAT_DET3, KAT_4, np.array([[10.0 if i == j else (i + j) * 0.5 for j in range(5)] for i in range(5)])):
        st, ai = lo.inv(a)
        assert st == 0 and np.max(np.abs(a @ ai - np.eye(len(a)))) < 1e-10
    assert lo.inv(m([1, 2], [2, 4]))[0] == lo.SINGULAR
    assert lo.inv(SING4_INV)[0] == lo.SINGULAR


# ---- the n <= 3 closed forms, bit for bit against hand-derived expressions ----

@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_closed_forms_bitwise(dtype):
    rng = np.random.default_rng(3)
    for _ in range(50):
        a = rng.standard_normal((3, 3)).astype(dtype)
        x = [[dtype(v) for v in row] for row in a]
        d3 = (x[0][0] * x[1][1] * x[2][2] + x[0][1] * x[1][2] * x[2][0] + x[0][2] * x[1][0] * x[2][1] - x[0][2] * x[1][1] * x[2][0]
              - x[0][1] * x[1][0] * x[2][2] - x[0][0] * x[1][2] * x[2][1])
        assert lo.det(a) == d3
        c00 = x[1][1] * x[2][2] - x[1][2] * x[2][1]
        c01 = x[0][2] * x[2][1] - x[0][1] * x[2][2]
        c02 = x[0][1] * x[1][2] - x[0][2] * x[1][1]
        d = x[0][0] * c00 + x[1][0] * c01 + x[2][0] * c02
        want = np.array([c00 / d, c01 / d, c02 / d,
                         (x[1][2] * x[2][0] - x[1][0] * x[2][2]) / d, (x[0][0] * x[2][2] - x[0][2] * x[2][0]) / d,
                         (x[0][2] * x[1][0] - x[0][0] * x[1][2]) / d,
                         (x[1][0] * x[2][1] - x[1][1] * x[2][0]) / d, (x[0][1] * x[2][0] - x[0][0] * x[2][1]) / d,
                         (x[0][0] * x[1][1] - x[0][1] * x[1][0]) / d], dtype).reshape(3, 3)
        st, got = lo.inv(a)
        assert st == 0 and np.array_equal(got.view(np.uint8), want.view(np.uint8))
        b = a[:2, :2]
        d2 = x[0][0] * x[1][1] - x[0][1] * x[1][0]
        assert lo.det(b) == d2
        st, got = lo.inv(b)
        want = np.array([x[1][1] / d2, -x[0][1] / d2, -x[1][0] / d2, x[0][0] / d2], dtype).reshape(2, 2)
        assert st == 0 and np.array_equal(got.view(np.uint8), want.view(np.uint8))
        st, got = lo.inv(a[:1, :1])
        assert st == 0 and got[0, 0] == dtype(1) / x[0][0]


# ---- the oracle against mpmath (40 digits) and LAPACK ----

def test_oracle_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    rng = np.random.default_rng(5)
    with mpmath.workdps(40):
        for n in (4, 9, 17, 33, 64):
            a = rng.standard_normal((n, n))
            b = rng.standard_normal((n, 1))
            st, x = lo.solve(a, b)
            exact = mpmath.lu_solve(mpmath.matrix(a.tolist()), mpmath.matrix(b.tolist()))
            ex = np.array([float(v) for v in exact])
            kappa = np.linalg.cond(a)
            assert st == 0 and np.max(np.abs(x[:, 0] - ex)) <= 64 * n * kappa * 2.0 ** -52 * np.max(np.abs(ex))
            d = float(mpmath.det(mpmath.matrix(a.tolist())))
            assert abs(lo.det(a) - d) <= 64 * n * kappa * 2.0 ** -52 * abs(d)


@pytest.mark.parametrize("n", [4, 31, 64, 129])
def test_oracle_against_lapack(n):
    rng = np.random.default_rng(n)
    a = rng.standard_normal((n, n))
    l, u, p, sign = lo.lu(a)
    lu_, piv = scipy.linalg.lu_factor(a)
    perm = np.arange(n)
    for k, q in enumerate(piv):
        perm[[k, q]] = perm[[q, k]]
    assert np.array_equal(p, perm)
    assert sign == (-1.0) ** int(np.sum(piv != np.arange(n)))
    assert np.max(np.abs(np.triu(lu_) - u)) <= 1e-12 * n * np.max(np.abs(u))
    eps = 2.0 ** -52
    st, ai = lo.inv(a)
    assert st == 0 and np.linalg.norm(ai - np.linalg.inv(a)) <= 100 * n * eps * np.linalg.cond(a) * np.linalg.norm(ai)
    spd = a @ a.T + n * np.eye(n)
    st, lc = lo.chol(spd)
    assert st == 0 and np.max(np.abs(lc - np.linalg.cholesky(spd))) <= 100 * n * eps * np.max(np.abs(lc))
    assert abs(lo.det(a) - np.linalg.det(a)) <= 100 * n * eps * np.linalg.cond(a) * abs(np.linalg.det(a))


# ---- the library: status names and argument errors without a device ----

def test_status_names():
    import zignal_b200 as zb
    assert zb.lib().zb_status_name(32).decode() == "Singular"
    assert zb.lib().zb_status_name(33).decode() == "NotPositiveDefinite"


ARG_ERRORS = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from zignal_b200 import _ffi
L = _ffi.lib()
buf = (C.c_double * 16)()
fbuf = (C.c_float * 16)()
pm = (C.c_uint32 * 4)()
d, f = C.cast(buf, C.POINTER(C.c_double)), C.cast(fbuf, C.POINTER(C.c_float))
sd, sf = C.c_double(0), C.c_float(0)
out = {}
for s, p, sc in (("f64", d, sd), ("f32", f, sf)):
    lu, lus, det, inv, chol = (getattr(L, f"zb_{x}_{s}") for x in ("lu", "lu_solve", "det", "inv", "chol"))
    out[s] = [
        lu(p, 2, 3, p, pm, C.byref(sc), None), lu(None, 2, 2, p, pm, C.byref(sc), None), lu(p, 2, 2, p, None, C.byref(sc), None),
        lus(p, pm, 2, p, 3, 1, p, None), lus(p, pm, 0, p, 0, 1, p, None), lus(None, pm, 2, p, 2, 1, p, None),
        det(p, 2, 3, C.byref(sc), None), det(p, 0, 0, C.byref(sc), None), det(None, 2, 2, C.byref(sc), None),
        inv(p, 3, 2, p, None), inv(p, 0, 0, p, None), inv(p, 2, 2, None, None),
        chol(p, 1, 2, p, None), chol(None, 2, 2, p, None),
    ]
print(json.dumps(out))
"""


def test_argument_errors_need_no_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", ARG_ERRORS, str(ROOT)], capture_output=True, text=True, env=env, timeout=120)
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    want = [18, 5, 5, 1, 32, 5, 18, 1, 5, 18, 1, 5, 18, 5]
    assert got == {"f64": want, "f32": want}
