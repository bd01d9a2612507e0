"""Matrix.lu, LuResult.solve, solve, det, inv and chol on the H100 (csrc/zb_linsolve.cu) against the CPU oracle
(oracle/zo_linsolve.cpp): the reference's bits up to 64 x 64 (one panel), agreement to rounding above, residuals at large n, the
Singular / NotPositiveDefinite statuses, NaN / inf entries, and the same bits from run to run, on other streams and threads."""
import threading

import numpy as np
import pytest
import torch

import linsolve_oracle as lo
from zignal_b200 import matrix as zm
from zignal_b200._ffi import ZignalError

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
SMALL = [1, 2, 3, 4, 5, 31, 63, 64]
LARGE = [65, 127, 128, 129, 200, 513, 1000]


def same(a, b):
    """Bit-identical, except that any NaN equals any NaN (the device and the host spell the default NaN differently)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(u), b[~nb].view(u))


def status(fn, *args):
    try:
        return 0, fn(*args)
    except ZignalError as e:
        return e.status, None


def check_all_bitwise(a):
    """Every output of every operation on a equals the oracle's bits (statuses included)."""
    n = a.shape[0]
    r = zm.lu(a)
    l, u, p, sign = lo.lu(a)
    assert same(r.l, l) and same(r.u, u) and np.array_equal(r.p, p) and r.sign == sign
    assert same(np.asarray(zm.det(a), a.dtype), lo.det(a))
    b = np.random.default_rng(n).standard_normal((n, 3)).astype(a.dtype)
    st, x = status(r.solve, b)
    ost, ox = lo.lu_solve(l, u, p, b)
    assert st == ost and (st != 0 or same(x, ox))
    st, x = status(zm.inv, a)
    ost, ox = lo.inv(a)
    assert st == ost and (st != 0 or same(x, ox))
    st, x = status(zm.chol, a)
    ost, ox = lo.chol(a)
    assert st == ost and (st != 0 or same(x, ox))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SMALL)
def test_bit_identical_up_to_one_panel(n, dtype):
    rng = np.random.default_rng(100 + n)
    a = rng.standard_normal((n, n)).astype(dtype)
    check_all_bitwise(a)
    spd = (a @ a.T + n * np.eye(n)).astype(dtype)
    check_all_bitwise(spd)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rank_deficient_integer_statuses(dtype):
    rng = np.random.default_rng(7)
    for _ in range(200):
        n = int(rng.integers(4, 9))
        r = int(rng.integers(1, n))
        a = (rng.integers(-4, 5, (n, r)) @ rng.integers(-4, 5, (r, n))).astype(dtype)
        b = rng.integers(-9, 10, (n, 2)).astype(dtype)
        st, x = status(zm.inv, a)
        ost, ox = lo.inv(a)
        assert st == ost and (st != 0 or same(x, ox))
        st, x = status(zm.solve, a, b)
        ost, ox = lo.solve(a, b)
        assert st == ost and (st != 0 or same(x, ox))
        assert same(np.asarray(zm.det(a), dtype), lo.det(a))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [4, 5, 31, 64])
def test_nonfinite_entries(n, dtype):
    rng = np.random.default_rng(11 + n)
    for trial in range(12):
        a = rng.standard_normal((n, n)).astype(dtype)
        for _ in range(1 + trial % 3):
            a[rng.integers(n), rng.integers(n)] = [np.nan, np.inf, -np.inf][int(rng.integers(3))]
        if trial % 4 == 0:
            a[0, 0] = np.nan   # a NaN on the diagonal stays the pivot
        check_all_bitwise(a)
    spd = np.eye(n, dtype=dtype) * 4
    spd[n - 1, 0] = np.nan   # a NaN sum passes the positivity test
    st, l = status(zm.chol, spd)
    ost, ol = lo.chol(spd)
    assert st == ost == 0 and same(l, ol)


def residuals(a, dtype):
    n = a.shape[0]
    eps = float(np.finfo(dtype).eps)
    ta = torch.from_numpy(a).cuda()
    lu, perm, sign = zm.lu_device(ta)
    L = torch.tril(lu, -1) + torch.eye(n, dtype=lu.dtype, device="cuda")
    U = torch.triu(lu)
    pa = ta[perm.long()]
    r_lu = float(torch.linalg.norm(pa.double() - (L.double() @ U.double())) / (torch.linalg.norm(ta.double()) * n * eps))
    return lu, perm, sign, r_lu


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", LARGE)
def test_blocked_agrees_to_rounding(n, dtype):
    rng = np.random.default_rng(200 + n)
    a = rng.standard_normal((n, n)).astype(dtype)
    eps = float(np.finfo(dtype).eps)
    lu, perm, sign, r_lu = residuals(a, dtype)
    l, u, p, osign = lo.lu(a)
    assert np.array_equal(perm.cpu().numpy().view(np.uint32), p) and sign == osign
    assert r_lu < 1.0, r_lu
    # det of a matrix whose singular values lie near 1, so that the product of the pivots neither overflows nor underflows
    w = (np.eye(n) + 0.5 * rng.standard_normal((n, n)) / np.sqrt(n)).astype(dtype)
    kappa = np.linalg.cond(w.astype(np.float64))
    d, od = zm.det(w), lo.det(w)
    assert np.isfinite(od) and abs(d - od) <= n * eps * kappa * abs(od), (d, od)
    b = rng.standard_normal((n, 2)).astype(dtype)
    x = zm.solve(a, b).astype(np.float64)
    a64 = a.astype(np.float64)
    back = np.linalg.norm(a64 @ x - b, np.inf) / (np.linalg.norm(a64, np.inf) * np.linalg.norm(x, np.inf) + np.linalg.norm(b, np.inf))
    assert back < n * eps, back
    ai = zm.inv(a).astype(np.float64)
    assert np.linalg.norm(a64 @ ai - np.eye(n)) / np.linalg.norm(np.linalg.inv(a64)) < 4 * n * eps * np.linalg.norm(a64)
    spd = (a64 @ a64.T / n + np.eye(n)).astype(dtype)
    lc = zm.chol(spd).astype(np.float64)
    assert np.all(np.triu(lc, 1) == 0)
    assert np.linalg.norm(spd - lc @ lc.T) / (np.linalg.norm(spd.astype(np.float64)) * n * eps) < 1.0


@pytest.mark.parametrize("dtype,n", [(np.float64, 8192), (np.float32, 4096)])
def test_large_residuals(dtype, n):
    torch.manual_seed(0)
    eps = float(np.finfo(dtype).eps)
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    ta = torch.randn(n, n, dtype=tdt, device="cuda")
    lu, perm, sign = zm.lu_device(ta)
    L = torch.tril(lu, -1) + torch.eye(n, dtype=tdt, device="cuda")
    r = torch.linalg.norm(ta[perm.long()].double() - L.double() @ torch.triu(lu).double()) / (torch.linalg.norm(ta.double()) * n * eps)
    assert float(r) < 1.0, float(r)
    b = torch.randn(n, 1, dtype=tdt, device="cuda")
    x = zm.lu_solve_device(lu, perm, b)
    ad, xd, bd = ta.double(), x.double(), b.double()
    back = torch.linalg.norm(ad @ xd - bd, float("inf")) / (torch.linalg.norm(ad, float("inf")) * torch.linalg.norm(xd, float("inf")))
    assert float(back) < n * eps, float(back)
    spd = (ta @ ta.T) / n + torch.eye(n, dtype=tdt, device="cuda")
    from zignal_b200.matrix import _fns, _ptr, _stream
    fn, ct = _fns(tdt, "chol")
    lc = torch.empty_like(spd)
    from zignal_b200._ffi import check
    check(fn(_ptr(spd, ct), n, n, _ptr(lc, ct), _stream(spd)))
    r = torch.linalg.norm(spd.double() - lc.double() @ lc.double().T) / (torch.linalg.norm(spd.double()) * n * eps)
    assert float(r) < 1.0, float(r)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [5, 64, 1000])
def test_zero_column(n, dtype):
    rng = np.random.default_rng(n)
    a = (np.eye(n) + 0.5 * rng.standard_normal((n, n)) / np.sqrt(n)).astype(dtype)   # the pivots' product stays finite
    a[:, n // 2] = 0
    b = rng.standard_normal((n, 1)).astype(dtype)
    assert status(zm.inv, a)[0] == 32
    assert status(zm.solve, a, b)[0] == 32
    r = zm.lu(a)
    assert np.all(r.l[n // 2 + 1:, n // 2] == 0)
    assert zm.det(a) == 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [2, 64, 300])
def test_indefinite(n, dtype):
    a = np.eye(n, dtype=dtype)
    a[n - 1, n - 1] = -1
    assert status(zm.chol, a)[0] == 33
    assert lo.chol(a)[0] == 33


def test_errors():
    with pytest.raises(ZignalError) as e:
        zm.inv(np.zeros((0, 0)))
    assert e.value.status == 1
    with pytest.raises(ZignalError) as e:
        zm.lu(np.zeros((3, 4)))
    assert e.value.status == 18


@pytest.mark.parametrize("n", [64, 300])
def test_in_place_and_deterministic(n):
    rng = np.random.default_rng(n)
    a = torch.from_numpy(rng.standard_normal((n, n))).cuda()
    lu1, p1, s1 = zm.lu_device(a)
    lu2, p2, s2 = zm.lu_device(a)
    assert torch.equal(lu1, lu2) and torch.equal(p1, p2) and s1 == s2
    # in place: lu == a
    from zignal_b200._ffi import check, lib
    import ctypes as C
    w = a.clone()
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    sign = C.c_double(0)
    check(lib().zb_lu_f64(zm._ptr(w, C.c_double), n, n, zm._ptr(w, C.c_double), zm._ptr(perm, C.c_uint32), C.byref(sign),
                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(w, lu1) and torch.equal(perm, p1)
    spd = a @ a.T / n + torch.eye(n, dtype=a.dtype, device="cuda")
    want = torch.from_numpy(zm.chol(spd.cpu().numpy())).cuda()
    check(lib().zb_chol_f64(zm._ptr(spd, C.c_double), n, n, zm._ptr(spd, C.c_double), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(spd, want)
    # a non-blocking stream, and two host threads
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        lu3, p3, _ = zm.lu_device(a)
    s.synchronize()
    assert torch.equal(lu3, lu1) and torch.equal(p3, p1)
    out = [None, None]

    def run(i):
        with torch.cuda.stream(torch.cuda.Stream()):
            r = zm.lu_device(a)
            torch.cuda.current_stream().synchronize()
            out[i] = r

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for r in out:
        assert torch.equal(r[0], lu1) and torch.equal(r[1], p1)
