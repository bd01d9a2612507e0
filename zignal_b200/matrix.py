"""Host-side mirror of zignal's Matrix(T) operations on the hot path: `gemm` (reference
src/matrix/Matrix.zig:696-822) runs on the device through the C ABI; `svd` (Matrix.zig:1570, svd.zig:80-496) and `eigh`
(matrix/eigen.zig:34) are parallel-ordering Jacobi methods (csrc/zb_jacobi.cu: a persistent cooperative kernel for 24 columns
and more, the same algorithm on the host below that).  `lu` / `LuResult.solve`, `solve`, `det`, `inv` and `chol` (Matrix.zig:67-85,
376-441, 511-583, 1156-1365) are blocked factorisations on the device (csrc/zb_linsolve.cu), the reference's bits up to 64 x 64."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._ffi import ZignalError, check, lib


def _torch():
    import torch
    return torch


def _ptr(t, ctype):
    return C.cast(t.data_ptr(), C.POINTER(ctype))


def gemm_device(a, b, trans_a=False, trans_b=False, alpha=1.0, beta=0.0, c=None):
    """C = alpha * op(A) * op(B) + beta * C on CUDA tensors (row-major, contiguous); returns a new CUDA tensor."""
    import torch
    assert a.is_cuda and b.is_cuda and a.dtype == b.dtype and a.is_contiguous() and b.is_contiguous()
    ar, ac = a.shape
    br, bc = b.shape
    m = ac if trans_a else ar
    n = br if trans_b else bc
    out = torch.empty((m, n), dtype=a.dtype, device=a.device)
    stream = torch.cuda.current_stream().cuda_stream
    if a.dtype == torch.float32:
        cp = _ptr(c, C.c_float) if c is not None else None
        check(lib().zb_gemm_f32(_ptr(a, C.c_float), ar, ac, int(trans_a), _ptr(b, C.c_float), br, bc, int(trans_b), C.c_float(alpha),
                                C.c_float(beta), cp, _ptr(out, C.c_float), stream))
    elif a.dtype == torch.float64:
        cp = _ptr(c, C.c_double) if c is not None else None
        check(lib().zb_gemm_f64(_ptr(a, C.c_double), ar, ac, int(trans_a), _ptr(b, C.c_double), br, bc, int(trans_b), C.c_double(alpha),
                                C.c_double(beta), cp, _ptr(out, C.c_double), stream))
    else:
        raise TypeError("gemm supports f32 and f64")
    return out


def center_columns(x, mean, compute_mean: bool, centered):
    """Pca centering on CUDA tensors: (optionally) mean[j] = column mean of x, centered = x - mean."""
    import torch
    n, dim = x.shape
    stream = torch.cuda.current_stream().cuda_stream
    if x.dtype == torch.float32:
        check(lib().zb_center_columns_f32(_ptr(x, C.c_float), n, dim, _ptr(mean, C.c_float), int(compute_mean), _ptr(centered, C.c_float), stream))
    else:
        check(lib().zb_center_columns_f64(_ptr(x, C.c_double), n, dim, _ptr(mean, C.c_double), int(compute_mean), _ptr(centered, C.c_double), stream))


def gemm(a: np.ndarray, b: np.ndarray, trans_a=False, trans_b=False, alpha=1.0, beta=0.0, c=None) -> np.ndarray:
    """numpy in / numpy out convenience wrapper around `gemm_device`."""
    import torch
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, dtype=a.dtype)
    ta = torch.from_numpy(a).cuda()
    tb = torch.from_numpy(b).cuda()
    tc = torch.from_numpy(np.ascontiguousarray(c, dtype=a.dtype)).cuda() if c is not None else None
    return gemm_device(ta, tb, trans_a, trans_b, alpha, beta, tc).cpu().numpy()


_MODES = {"no_u": 0, "skinny_u": 1, "full_u": 2}


def svd(a: np.ndarray, mode: str = "full_u", with_v: bool = False):
    """Matrix.svd(allocator, .{ .with_v, .mode }) -> (u, s, v, converged).  rows >= cols required (svd.zig:86)."""
    a = np.ascontiguousarray(a)
    m, n = a.shape
    if m < n:
        raise ZignalError(1, "DimensionMismatch")
    u = np.zeros((m, m if mode == "full_u" else n), a.dtype) if mode != "no_u" else np.zeros((0, 0), a.dtype)
    s = np.zeros(n, a.dtype)
    v = np.zeros((n, n), a.dtype) if with_v else np.zeros((0, 0), a.dtype)
    conv = C.c_uint64(0)
    if a.dtype == np.float64:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_double)) if x.size else None
        check(lib().zb_svd_f64(P(a), m, n, _MODES[mode], int(with_v), P(u), P(s), P(v), C.byref(conv)))
    elif a.dtype == np.float32:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_float)) if x.size else None
        check(lib().zb_svd_f32(P(a), m, n, _MODES[mode], int(with_v), P(u), P(s), P(v), C.byref(conv)))
    else:
        raise TypeError("svd supports f32 and f64")
    return u, s, v, conv.value


def svd_device(a, with_u: bool = True, with_v: bool = False):
    """The same decomposition for a CUDA tensor (m x n, m >= n, f32 / f64) that stays on the device (zb_svd_dev_*):
    -> (u: m x n or None, s: n descending, v: n x n or None, converged) as CUDA tensors."""
    torch = _torch()
    assert a.is_cuda and a.is_contiguous() and a.dim() == 2
    m, n = a.shape
    if m < n:
        raise ZignalError(1, "DimensionMismatch")
    u = torch.empty((m, n), dtype=a.dtype, device=a.device) if with_u else None
    s = torch.empty(n, dtype=a.dtype, device=a.device)
    v = torch.empty((n, n), dtype=a.dtype, device=a.device) if with_v else None
    conv = C.c_uint64(0)
    ct = C.c_double if a.dtype == torch.float64 else C.c_float
    fn = lib().zb_svd_dev_f64 if a.dtype == torch.float64 else lib().zb_svd_dev_f32
    with torch.cuda.device(a.device):
        check(fn(_ptr(a, ct), m, n, _ptr(u, ct) if u is not None else None, _ptr(s, ct), _ptr(v, ct) if v is not None else None,
                 C.byref(conv), torch.cuda.current_stream(a.device).cuda_stream))
    return u, s, v, conv.value


def eigh(a: np.ndarray):
    """Matrix.eigh(allocator) (matrix/eigen.zig:34-136) -> (values ascending, vectors with eigenvectors as columns)."""
    a = np.ascontiguousarray(a)
    if a.ndim != 2:
        raise ZignalError(18, "NotSquare")
    rows, cols = a.shape
    values = np.zeros(rows, a.dtype)
    vectors = np.zeros((rows, rows), a.dtype)
    if a.dtype == np.float64:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
        check(lib().zb_eigh_f64(P(a), rows, cols, P(values), P(vectors)))
    elif a.dtype == np.float32:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))
        check(lib().zb_eigh_f32(P(a), rows, cols, P(values), P(vectors)))
    else:
        raise TypeError("eigh supports f32 and f64")
    return values, vectors


# ---- dense linear systems (csrc/zb_linsolve.cu) ----

def _fns(dtype, name):
    torch = _torch()
    if dtype in (np.float64, torch.float64):
        return getattr(lib(), f"zb_{name}_f64"), C.c_double
    if dtype in (np.float32, torch.float32):
        return getattr(lib(), f"zb_{name}_f32"), C.c_float
    raise TypeError(f"{name} supports f32 and f64")


def _stream(t):
    return _torch().cuda.current_stream(t.device).cuda_stream


def lu_device(a):
    """Packed LU of a square CUDA tensor (zb_lu_*): -> (lu, perm, sign).  lu's strict lower triangle is L (unit diagonal implied), its
    upper triangle U; perm (int32, the u32 bits) maps row i of PA to row perm[i] of A; sign = +1 / -1."""
    torch = _torch()
    assert a.is_cuda and a.is_contiguous() and a.dim() == 2
    fn, ct = _fns(a.dtype, "lu")
    rows, cols = a.shape
    lu = torch.empty_like(a)
    perm = torch.empty(rows, dtype=torch.int32, device=a.device)
    sign = ct(0)
    with torch.cuda.device(a.device):
        check(fn(_ptr(a, ct), rows, cols, _ptr(lu, ct), _ptr(perm, C.c_uint32), C.byref(sign), _stream(a)))
    return lu, perm, sign.value


def lu_solve_device(lu, perm, b):
    """x with A x = b from lu_device's (lu, perm) (zb_lu_solve_*); b is n x k (CUDA)."""
    torch = _torch()
    assert lu.is_cuda and lu.is_contiguous() and b.is_cuda and b.dtype == lu.dtype and b.dim() == 2
    b = b.contiguous()
    fn, ct = _fns(lu.dtype, "lu_solve")
    n = lu.shape[0]
    x = torch.empty((n, b.shape[1]), dtype=b.dtype, device=b.device)
    with torch.cuda.device(lu.device):
        check(fn(_ptr(lu, ct), _ptr(perm, C.c_uint32), n, _ptr(b, ct), b.shape[0], b.shape[1], _ptr(x, ct), _stream(lu)))
    return x


def _dev(a: np.ndarray):
    torch = _torch()
    a = np.ascontiguousarray(a)
    if a.ndim != 2:
        raise ZignalError(18, "NotSquare")
    return torch.from_numpy(a).cuda()


class LuResult:
    """Matrix.LuResult (Matrix.zig:1157-1222): l unit lower, u upper, p (row i of PA is row p[i] of A), sign = +1 / -1."""

    def __init__(self, lu, perm, sign):
        self._lu, self._perm = lu, perm
        packed = lu.cpu().numpy()
        self.l = np.tril(packed, -1)   # np.where-based: a factor of -0.0 keeps its sign
        np.fill_diagonal(self.l, 1)
        self.u = np.triu(packed)
        self.p = perm.cpu().numpy().view(np.uint32)
        self.sign = sign

    def solve(self, b: np.ndarray) -> np.ndarray:
        """LuResult.solve(b), b: n x k."""
        b = np.ascontiguousarray(b, dtype=self.l.dtype)
        if b.ndim != 2:
            raise ZignalError(1, "DimensionMismatch")
        return lu_solve_device(self._lu, self._perm, _torch().from_numpy(b).to(self._lu.device)).cpu().numpy()


def lu(a: np.ndarray) -> LuResult:
    """Matrix.lu() (Matrix.zig:1226-1316)."""
    return LuResult(*lu_device(_dev(a)))


def solve(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Matrix.solve(b) (Matrix.zig:435-441): NotSquare, then DimensionMismatch, then lu and LuResult.solve."""
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, dtype=a.dtype)
    if a.ndim != 2 or a.shape[0] != a.shape[1]:
        raise ZignalError(18, "NotSquare")
    if b.ndim != 2 or b.shape[0] != a.shape[0]:
        raise ZignalError(1, "DimensionMismatch")
    return lu(a).solve(b)


def _host_scalar(name, a):
    t = _dev(a)
    fn, ct = _fns(t.dtype, name)
    out = ct(0)
    with _torch().cuda.device(t.device):
        check(fn(_ptr(t, ct), t.shape[0], t.shape[1], C.byref(out), _stream(t)))
    return out.value


def _square_op(name, a, shape):
    t = _dev(a)
    fn, ct = _fns(t.dtype, name)
    out = _torch().empty(shape(t), dtype=t.dtype, device=t.device)
    with _torch().cuda.device(t.device):
        check(fn(_ptr(t, ct), t.shape[0], t.shape[1], _ptr(out, ct), _stream(t)))
    return out.cpu().numpy()


def det(a: np.ndarray):
    """Matrix.det() (Matrix.zig:1336-1365)."""
    return _host_scalar("det", a)


def inv(a: np.ndarray) -> np.ndarray:
    """Matrix.inv() (Matrix.zig:376-427, 511-583); a 0 x 0 matrix raises DimensionMismatch."""
    return _square_op("inv", a, lambda t: (t.shape[0], t.shape[0]))


def chol(a: np.ndarray) -> np.ndarray:
    """Matrix.chol() (Matrix.zig:1320-1332): L with A = L L^T from A's lower triangle."""
    return _square_op("chol", a, lambda t: (t.shape[0], t.shape[0]))
