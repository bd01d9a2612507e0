"""ctypes binding of the CPU oracle (oracle/libzignal_oracle.so) for the test-suite and bench.py.

TEST INFRASTRUCTURE ONLY: nothing under zignal_b200/ may import this module (the product path must
fail loudly without its CUDA library; it never falls back to the oracle).
"""
from __future__ import annotations

import ctypes as C
import functools
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE_DIR = ROOT / "oracle"

# enums (oracle/zignal_oracle.h)
BORDER = {"zero": 0, "replicate": 1, "mirror": 2, "wrap": 3}
INTERP = {"nearest": 0, "bilinear": 1, "bicubic": 2, "catmull_rom": 3, "mitchell": 4, "lanczos": 5}
PIX_U8, PIX_F32, PIX_RGB8, PIX_RGBA8, PIX_RGBAF32 = 0, 1, 2, 3, 4
XFORM = {"similarity": 0, "affine": 1, "projective": 2}
SVD_NO_U, SVD_SKINNY_U, SVD_FULL_U = 0, 1, 2


class ZoImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("rows", C.c_uint32), ("cols", C.c_uint32), ("stride", C.c_uint64)]


def load(name: str) -> C.CDLL:
    """oracle/<name> (e.g. "libzo_hough.so"), after `make -C oracle <name>` has rebuilt it if a source is newer.  Where make fails
    (no make, or a read-only tree) a library built earlier by __graft_entry__.build() is used as it is."""
    path = ORACLE_DIR / name
    try:
        subprocess.run(["make", "-C", str(ORACLE_DIR), "-j8", name], check=True, capture_output=True, text=True)
    except (OSError, subprocess.CalledProcessError) as e:
        if not path.exists():
            raise RuntimeError(f"cannot build oracle/{name}: {getattr(e, 'stderr', None) or e}") from e
    return C.CDLL(str(path))


@functools.cache
def lib() -> C.CDLL:
    L = load("libzignal_oracle.so")
    _declare(L)
    return L


def _declare(L):
    P = C.POINTER
    img = P(ZoImage)
    fp, dp = P(C.c_float), P(C.c_double)
    L.zo_set_threads.argtypes = [C.c_int]
    L.zo_get_threads.restype = C.c_int
    L.zo_hw_threads.restype = C.c_int
    L.zo_resolve_index.argtypes = [C.c_int64, C.c_int64, C.c_int]
    L.zo_resolve_index.restype = C.c_int64
    L.zo_clamp_u8_f32.argtypes = [C.c_float]
    L.zo_clamp_u8_f32.restype = C.c_uint8
    L.zo_div_clamp_u8.argtypes = [C.c_int64, C.c_int64]
    L.zo_div_clamp_u8.restype = C.c_uint8
    L.zo_gaussian_taps.argtypes = [C.c_float, fp, C.c_int]
    L.zo_conv_separable.argtypes = [img, img, C.c_int, fp, C.c_int, fp, C.c_int, C.c_int]
    L.zo_convolve.argtypes = [img, img, C.c_int, fp, C.c_int, C.c_int, C.c_int]
    L.zo_gaussian_blur.argtypes = [img, img, C.c_int, C.c_float]
    L.zo_integral_plane.argtypes = [img, C.c_int, fp]
    L.zo_box_blur.argtypes = [img, img, C.c_int, C.c_uint32]
    L.zo_sharpen.argtypes = [img, img, C.c_int, C.c_uint32]
    L.zo_sobel.argtypes = [img, img, C.c_int]
    L.zo_order_blur.argtypes = [img, img, C.c_int, C.c_uint32, C.c_int, C.c_double, C.c_int]
    for fn in (L.zo_psnr, L.zo_ssim, L.zo_mean_pixel_error):
        fn.argtypes = [img, img, C.c_int, C.POINTER(C.c_double)]
    L.zo_motion_blur_line.argtypes = [img, img, C.c_int, C.c_float, C.c_float, C.c_uint32]
    L.zo_motion_blur_radial.argtypes = [img, img, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int]
    L.zo_convert.argtypes = [img, C.c_int, img, C.c_int]
    L.zo_canny.argtypes = [img, img, C.c_int, C.c_float, C.c_float, C.c_float]
    L.zo_interpolate.argtypes = [img, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p]
    L.zo_resize.argtypes = [img, img, C.c_int, C.c_int, C.c_float, C.c_float]
    L.zo_rotate_bounds.argtypes = [C.c_uint32, C.c_uint32, C.c_float, P(C.c_uint32), P(C.c_uint32)]
    L.zo_rotate_bounds.restype = None
    L.zo_rotate_class.argtypes = [C.c_float]
    L.zo_rotate_into.argtypes = [img, img, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float, C.c_int]
    L.zo_warp.argtypes = [img, img, C.c_int, C.c_int, fp, C.c_int, C.c_float, C.c_float]
    L.zo_extract.argtypes = [img, img, C.c_int] + [C.c_float] * 7 + [C.c_int, C.c_float, C.c_float, C.c_int]
    L.zo_insert.argtypes = [img, img, C.c_int] + [C.c_float] * 7 + [C.c_int, C.c_float, C.c_float]
    L.zo_insert_blend.argtypes = [img, img, C.c_int] + [C.c_float] * 7 + [C.c_int, C.c_float, C.c_float, C.c_int]
    L.zo_blend_rgba8.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_char_p]
    L.zo_blend_rgba8.restype = None
    L.zo_svd_f64.argtypes = [dp, C.c_uint32, C.c_uint32, C.c_int, C.c_int, dp, dp, dp]
    L.zo_svd_f64.restype = C.c_int64
    L.zo_svd_f32.argtypes = [fp, C.c_uint32, C.c_uint32, C.c_int, C.c_int, fp, fp, fp]
    L.zo_svd_f32.restype = C.c_int64
    L.zo_gemm_f32.argtypes = [fp, C.c_uint32, C.c_uint32, C.c_int, fp, C.c_uint32, C.c_uint32, C.c_int,
                              C.c_float, C.c_float, fp, fp, C.c_int]
    L.zo_gemm_f64.argtypes = [dp, C.c_uint32, C.c_uint32, C.c_int, dp, C.c_uint32, C.c_uint32, C.c_int,
                              C.c_double, C.c_double, dp, dp, C.c_int]
    L.zo_fdm_stats.argtypes = [img, C.c_int, C.c_int, dp, dp, P(C.c_int)]
    L.zo_fdm_match.argtypes = [img, img, C.c_int]
    L.zo_fdm_apply.argtypes = [img, C.c_int, dp, dp]
    L.zo_pca_fit_f64.argtypes = [dp, C.c_uint32, C.c_uint32, C.c_uint32, dp, dp, dp]
    L.zo_pca_fit_f32.argtypes = [fp, C.c_uint32, C.c_uint32, C.c_uint32, fp, fp, fp]
    L.zo_pca_transform_f64.argtypes = [dp, C.c_uint32, C.c_uint32, C.c_uint32, dp, dp, dp]
    L.zo_pca_transform_f32.argtypes = [fp, C.c_uint32, C.c_uint32, C.c_uint32, fp, fp, fp]


# ---------------------------------------------------------------------------------------------
# numpy <-> zo_image
# ---------------------------------------------------------------------------------------------
def pixfmt_of(a: np.ndarray) -> int:
    if a.dtype == np.uint8:
        if a.ndim == 2:
            return PIX_U8
        if a.ndim == 3 and a.shape[2] == 3:
            return PIX_RGB8
        if a.ndim == 3 and a.shape[2] == 4:
            return PIX_RGBA8
    if a.dtype == np.float32:
        if a.ndim == 2:
            return PIX_F32
        if a.ndim == 3 and a.shape[2] == 4:
            return PIX_RGBAF32
    raise TypeError(f"unsupported image array {a.dtype} {a.shape}")


def as_image(a: np.ndarray) -> ZoImage:
    """View a (rows, cols[, ch]) array whose rows may be strided (a crop of a bigger array) as zo_image."""
    px_bytes = a.dtype.itemsize * (a.shape[2] if a.ndim == 3 else 1)
    if a.ndim == 3:
        assert a.strides[2] == a.dtype.itemsize and a.strides[1] == px_bytes, "pixels must be packed"
    else:
        assert a.shape[1] <= 1 or a.strides[1] == a.dtype.itemsize
    row_stride = a.strides[0] if a.shape[0] > 1 else a.shape[1] * px_bytes
    assert row_stride % px_bytes == 0
    return ZoImage(a.ctypes.data, a.shape[0], a.shape[1], row_stride // px_bytes)


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class OracleStatus(RuntimeError):
    def __init__(self, status, what):
        self.status = status
        super().__init__(f"oracle {what} failed with status {status}")


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"oracle {what} failed with status {rc}")


def resolve_index(idx, length, border):
    r = lib().zo_resolve_index(idx, length, BORDER[border])
    return None if r < 0 else r


def gaussian_taps(sigma: float) -> np.ndarray:
    buf = np.zeros(4096, dtype=np.float32)
    n = lib().zo_gaussian_taps(C.c_float(sigma), _fptr(buf), buf.size)
    if n < 0:
        raise ValueError("invalid sigma")
    return buf[:n].copy()


def conv_separable(src, kx, ky, border="mirror", out=None):
    kx = np.ascontiguousarray(kx, dtype=np.float32)
    ky = np.ascontiguousarray(ky, dtype=np.float32)
    dst = np.empty_like(src) if out is None else out
    s, d = as_image(src), as_image(dst)
    _check(lib().zo_conv_separable(s, d, pixfmt_of(src), _fptr(kx), kx.size, _fptr(ky), ky.size, BORDER[border]), "conv_separable")
    return dst


def convolve(src, kernel, border="mirror", out=None):
    k = np.ascontiguousarray(kernel, dtype=np.float32)
    assert k.ndim == 2
    dst = np.empty_like(src) if out is None else out
    s, d = as_image(src), as_image(dst)
    _check(lib().zo_convolve(s, d, pixfmt_of(src), _fptr(k), k.shape[0], k.shape[1], BORDER[border]), "convolve")
    return dst


def gaussian_blur(src, sigma, out=None):
    dst = np.empty_like(src) if out is None else out
    s, d = as_image(src), as_image(dst)
    rc = lib().zo_gaussian_blur(s, d, pixfmt_of(src), C.c_float(sigma))
    if rc == 2:
        raise ValueError("InvalidSigma")
    _check(rc, "gaussian_blur")
    return dst


def integral_plane(src):
    sat = np.empty(src.shape[:2], dtype=np.float32)
    s = as_image(src)
    _check(lib().zo_integral_plane(s, pixfmt_of(src), _fptr(sat)), "integral_plane")
    return sat


def box_blur(src, radius, out=None):
    dst = np.empty_like(src) if out is None else out
    s, d = as_image(src), as_image(dst)
    _check(lib().zo_box_blur(s, d, pixfmt_of(src), radius), "box_blur")
    return dst


def sharpen(src, radius, out=None):
    dst = np.empty_like(src) if out is None else out
    s, d = as_image(src), as_image(dst)
    _check(lib().zo_sharpen(s, d, pixfmt_of(src), radius), "sharpen")
    return dst


def interpolate(src, x, y, method="bilinear", border="mirror", b=1.0 / 3.0, c=1.0 / 3.0):
    fmt = pixfmt_of(src)
    shape = () if src.ndim == 2 else (src.shape[2],)
    out = np.zeros(shape, dtype=src.dtype)
    s = as_image(src)
    ok = lib().zo_interpolate(s, fmt, C.c_float(x), C.c_float(y), INTERP[method], C.c_float(b), C.c_float(c), BORDER[border],
                              out.ctypes.data)
    return out if ok else None


def resize(src, out_shape, method="bilinear", b=1.0 / 3.0, c=1.0 / 3.0, out=None):
    if out is None:
        shp = (out_shape[0], out_shape[1]) + tuple(src.shape[2:])
        out = np.zeros(shp, dtype=src.dtype)
    s, d = as_image(src), as_image(out)
    _check(lib().zo_resize(s, d, pixfmt_of(src), INTERP[method], C.c_float(b), C.c_float(c)), "resize")
    return out


def rotate_bounds(rows, cols, angle):
    r, c = C.c_uint32(), C.c_uint32()
    lib().zo_rotate_bounds(rows, cols, C.c_float(angle), C.byref(r), C.byref(c))
    return r.value, c.value


def rotate_class(angle):
    return lib().zo_rotate_class(C.c_float(angle))


def rotate_into(src, out, angle, method="bilinear", border="zero", cos_sin=None, b=1.0 / 3.0, c=1.0 / 3.0):
    a32 = np.float32(angle)
    if cos_sin is None:
        cos_sin = (np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32))
    s, d = as_image(src), as_image(out)
    _check(lib().zo_rotate_into(s, d, pixfmt_of(src), C.c_float(a32), C.c_float(cos_sin[0]), C.c_float(cos_sin[1]),
                                INTERP[method], C.c_float(b), C.c_float(c), BORDER[border]), "rotate_into")
    return out


def sobel(src):
    out = np.zeros(src.shape[:2], np.uint8)
    s, d = as_image(src), as_image(out)
    _check(lib().zo_sobel(s, d, pixfmt_of(src)), "sobel")
    return out


ORDER_MODE = {"percentile": 0, "midpoint": 1, "alpha_trimmed": 2}


def order_blur(src, radius, mode="percentile", param=0.5, border="mirror", out=None):
    """percentileBlur / midpointBlur / alphaTrimmedMeanBlur; medianBlur = ("percentile", 0.5, "mirror")."""
    out = np.zeros_like(src) if out is None else out
    s, d = as_image(src), as_image(out)
    rc = lib().zo_order_blur(s, d, pixfmt_of(src), radius, ORDER_MODE[mode], C.c_double(param), BORDER[border])
    if rc != 0:
        raise OracleStatus(rc, "order_blur")
    return out


def _metric(fn, what, a, b):
    out = C.c_double(0.0)
    rc = fn(as_image(a), as_image(b), pixfmt_of(a), C.byref(out))
    if rc != 0:
        raise OracleStatus(rc, what)
    return out.value


def psnr(a, b):
    return _metric(lib().zo_psnr, "psnr", a, b)


def ssim(a, b):
    return _metric(lib().zo_ssim, "ssim", a, b)


def mean_pixel_error(a, b):
    return _metric(lib().zo_mean_pixel_error, "mean_pixel_error", a, b)


def motion_blur_linear(src, angle, distance, cos_sin=None):
    """MotionBlurOps.linear (motion_blur.zig:65-250): copy, the two convolveSeparable branches, or the diagonal line integral."""
    a32 = np.float32(angle)
    if cos_sin is None:
        cos_sin = (np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32))
    if distance == 0:
        return src.copy()
    kernel = np.full(distance, np.float32(1.0) / np.float32(distance), dtype=np.float32)
    identity = np.ones(1, np.float32)
    if abs(float(cos_sin[1])) < 0.001:
        return conv_separable(src, kernel, identity, "replicate")
    if abs(float(cos_sin[0])) < 0.001:
        return conv_separable(src, identity, kernel, "replicate")
    out = np.zeros_like(src)
    _check(lib().zo_motion_blur_line(as_image(src), as_image(out), pixfmt_of(src), C.c_float(cos_sin[0]), C.c_float(cos_sin[1]), distance),
           "motion_blur_line")
    return out


def motion_blur_radial(src, center_x, center_y, strength, spin=False):
    out = np.zeros_like(src)
    _check(lib().zo_motion_blur_radial(as_image(src), as_image(out), pixfmt_of(src), C.c_float(center_x), C.c_float(center_y),
                                       C.c_float(strength), int(bool(spin))), "motion_blur_radial")
    return out


_FMT_SHAPE = {0: ((), np.uint8), 1: ((), np.float32), 2: ((3,), np.uint8), 3: ((4,), np.uint8), 4: ((4,), np.float32)}


def convert(src, dst_pixfmt):
    """Image.convert (image.zig:396-421); dst_pixfmt is a ZO_PIX_* value (0 u8, 1 f32, 2 rgb8, 3 rgba8, 4 rgbaf32)."""
    tail, dtype = _FMT_SHAPE[int(dst_pixfmt)]
    out = np.zeros(src.shape[:2] + tail, dtype)
    _check(lib().zo_convert(as_image(src), pixfmt_of(src), as_image(out), int(dst_pixfmt)), "convert")
    return out


def canny(src, sigma, low, high):
    out = np.zeros(src.shape[:2], np.uint8)
    s, d = as_image(src), as_image(out)
    rc = lib().zo_canny(s, d, pixfmt_of(src), C.c_float(sigma), C.c_float(low), C.c_float(high))
    if rc != 0:
        raise OracleStatus(rc, "canny")
    return out


def extract(src, out, rect, angle=0.0, method="bilinear", border="zero", cos_sin=None, b=1.0 / 3.0, c=1.0 / 3.0):
    """rect = (l, t, r, b) in source coordinates (transforms.zig:232-283)."""
    a32 = np.float32(angle)
    if cos_sin is None:
        cos_sin = (np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32))
    s, d = as_image(src), as_image(out)
    _check(lib().zo_extract(s, d, pixfmt_of(src), C.c_float(rect[0]), C.c_float(rect[1]), C.c_float(rect[2]), C.c_float(rect[3]), C.c_float(a32),
                            C.c_float(cos_sin[0]), C.c_float(cos_sin[1]), INTERP[method], C.c_float(b), C.c_float(c), BORDER[border]), "extract")
    return out


BLEND = {name: i for i, name in enumerate(["none", "normal", "multiply", "screen", "overlay", "soft_light", "hard_light", "color_dodge",
                                            "color_burn", "darken", "lighten", "difference", "exclusion"])}


def blend_rgba8(base, overlay, mode):
    """blendColors(u8, base, overlay, mode) (blending.zig:26-156) on 4-tuples."""
    out = C.create_string_buffer(4)
    lib().zo_blend_rgba8(bytes(bytearray(base)), bytes(bytearray(overlay)), BLEND[mode], out)
    return tuple(out.raw)


def insert(dest, source, rect, angle=0.0, method="bilinear", cos_sin=None, b=1.0 / 3.0, c=1.0 / 3.0, blend="none"):
    """dest.insert(source, rect, angle, method, blend) (transforms.zig:293-376); returns the modified copy of dest."""
    a32 = np.float32(angle)
    if cos_sin is None:
        cos_sin = (np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32))
    out = np.ascontiguousarray(dest).copy()
    d, s = as_image(out), as_image(source)
    _check(lib().zo_insert_blend(d, s, pixfmt_of(out), C.c_float(rect[0]), C.c_float(rect[1]), C.c_float(rect[2]), C.c_float(rect[3]),
                                 C.c_float(a32), C.c_float(cos_sin[0]), C.c_float(cos_sin[1]), INTERP[method], C.c_float(b), C.c_float(c),
                                 BLEND[blend]), "insert")
    return out


def rotate(src, angle, method="bilinear", border="zero", cos_sin=None):
    rows, cols = rotate_bounds(src.shape[0], src.shape[1], angle)
    out = np.zeros((rows, cols) + tuple(src.shape[2:]), dtype=src.dtype)
    return rotate_into(src, out, angle, method, border, cos_sin)


def warp(src, out, kind, m, method="bilinear", b=1.0 / 3.0, c=1.0 / 3.0):
    m = np.ascontiguousarray(m, dtype=np.float32).ravel()
    assert m.size == (9 if kind == "projective" else 6)
    s, d = as_image(src), as_image(out)
    _check(lib().zo_warp(s, d, pixfmt_of(src), XFORM[kind], _fptr(m), INTERP[method], C.c_float(b), C.c_float(c)), "warp")
    return out


def svd(a, mode="skinny_u", with_v=True):
    a = np.ascontiguousarray(a)
    m, n = a.shape
    modes = {"no_u": SVD_NO_U, "skinny_u": SVD_SKINNY_U, "full_u": SVD_FULL_U}
    ucols = m if mode == "full_u" else n
    u = np.zeros((m, ucols), dtype=a.dtype)
    s = np.zeros(n, dtype=a.dtype)
    v = np.zeros((n, n), dtype=a.dtype)
    if a.dtype == np.float64:
        rc = lib().zo_svd_f64(_dptr(a), m, n, modes[mode], int(with_v), _dptr(u), _dptr(s), _dptr(v))
    else:
        rc = lib().zo_svd_f32(_fptr(a), m, n, modes[mode], int(with_v), _fptr(u), _fptr(s), _fptr(v))
    return u, s, v, rc


def eigh(a):
    """Matrix.eigh (eigen.zig:34-136) -> (values ascending, vectors as columns); raises OracleStatus (18 NotSquare, 19 NotSymmetric, 20 NotFinite)."""
    a = np.ascontiguousarray(a)
    rows, cols = a.shape
    values = np.zeros(rows, a.dtype)
    vectors = np.zeros((rows, rows), a.dtype)
    if a.dtype == np.float64:
        rc = lib().zo_eigh_f64(_dptr(a), rows, cols, _dptr(values), _dptr(vectors))
    else:
        rc = lib().zo_eigh_f32(_fptr(a), rows, cols, _fptr(values), _fptr(vectors))
    if rc != 0:
        raise OracleStatus(rc, "eigh")
    return values, vectors


def gemm(a, b, trans_a=False, trans_b=False, alpha=1.0, beta=0.0, c=None, vec_len=0):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, dtype=a.dtype)
    ar, ac = a.shape
    br, bc = b.shape
    out_r = ac if trans_a else ar
    out_c = br if trans_b else bc
    out = np.zeros((out_r, out_c), dtype=a.dtype)
    if a.dtype == np.float64:
        cp = _dptr(np.ascontiguousarray(c, dtype=a.dtype)) if c is not None else None
        rc = lib().zo_gemm_f64(_dptr(a), ar, ac, int(trans_a), _dptr(b), br, bc, int(trans_b), alpha, beta, cp, _dptr(out), vec_len)
    else:
        cp = _fptr(np.ascontiguousarray(c, dtype=a.dtype)) if c is not None else None
        rc = lib().zo_gemm_f32(_fptr(a), ar, ac, int(trans_a), _fptr(b), br, bc, int(trans_b), alpha, beta, cp, _fptr(out), vec_len)
    if rc == 1:
        raise ValueError("DimensionMismatch")
    _check(rc, "gemm")
    return out


def fdm_stats(img, as_luma=False):
    mean = np.zeros(3)
    cov = np.zeros(9)
    g = C.c_int()
    im = as_image(img)
    _check(lib().zo_fdm_stats(im, pixfmt_of(img), int(as_luma), _dptr(mean), _dptr(cov), C.byref(g)), "fdm_stats")
    return mean, cov.reshape(3, 3), bool(g.value)


def fdm_match(source, target):
    """Returns the matched copy of `source` (the oracle works in place on the copy)."""
    out = np.ascontiguousarray(source).copy()
    tgt = np.ascontiguousarray(target)
    s, t = as_image(out), as_image(tgt)
    _check(lib().zo_fdm_match(s, t, pixfmt_of(out)), "fdm_match")
    return out


def fdm_apply(source, w, bias):
    out = np.ascontiguousarray(source).copy()
    w = np.ascontiguousarray(w, dtype=np.float64)
    bias = np.ascontiguousarray(bias, dtype=np.float64)
    s = as_image(out)
    _check(lib().zo_fdm_apply(s, pixfmt_of(out), _dptr(w), _dptr(bias)), "fdm_apply")
    return out


def pca_fit(data, k=None):
    data = np.ascontiguousarray(data)
    n, dim = data.shape
    kmax = min(n - 1, dim)
    k = kmax if k is None else min(k, kmax)
    mean = np.zeros(dim, dtype=data.dtype)
    comps = np.zeros((dim, k), dtype=data.dtype)
    eig = np.zeros(k, dtype=data.dtype)
    if data.dtype == np.float64:
        rc = lib().zo_pca_fit_f64(_dptr(data), n, dim, k, _dptr(mean), _dptr(comps), _dptr(eig))
    else:
        rc = lib().zo_pca_fit_f32(_fptr(data), n, dim, k, _fptr(mean), _fptr(comps), _fptr(eig))
    _check(rc, "pca_fit")
    return mean, comps, eig


def pca_transform(data, mean, comps):
    data = np.ascontiguousarray(data)
    n, dim = data.shape
    k = comps.shape[1]
    out = np.zeros((n, k), dtype=data.dtype)
    comps = np.ascontiguousarray(comps)
    if data.dtype == np.float64:
        rc = lib().zo_pca_transform_f64(_dptr(data), n, dim, k, _dptr(mean), _dptr(comps), _dptr(out))
    else:
        rc = lib().zo_pca_transform_f32(_fptr(data), n, dim, k, _fptr(mean), _fptr(comps), _fptr(out))
    _check(rc, "pca_transform")
    return out


def parallel_fill_f32(a: np.ndarray, seed: int):
    """First-touch `a` (a C-contiguous f32 plane, e.g. from np.empty) with uniform [0, 1) values, rows split across the oracle's
    threads like its convolution loops -- NUMA placement for the CPU arm of bench.py."""
    assert a.dtype == np.float32 and a.ndim == 2 and a.flags.c_contiguous
    fn = lib().zo_parallel_fill_f32
    fn.argtypes = [C.POINTER(C.c_float), C.c_uint64, C.c_uint64, C.c_uint64]
    fn.restype = None
    fn(_fptr(a), a.shape[0], a.shape[1], int(seed))
    return a


def set_threads(n: int):
    lib().zo_set_threads(n)


def hw_threads() -> int:
    return lib().zo_hw_threads()
