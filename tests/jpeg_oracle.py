"""ctypes binding of the CPU oracle of the baseline JPEG encoder (oracle/zo_jpeg.cpp -> oracle/libzo_jpeg.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by oracle/Makefile;
__graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).

jpeg.encode (codecs/jpeg.zig:307-325) encodes Image(u8) as grayscale and Image(Rgb(u8)) as colour; every other pixel type is converted
with image.convert(Rgb) first.  encode() and coefficients() do that conversion with the main oracle's Image.convert (oracle_lib.convert).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import oracle_lib
from oracle_lib import OracleStatus, load, pixfmt_of
from oracle_lib import as_image

YUV444, YUV422, YUV420 = 0, 1, 2
PIX_U8, PIX_RGB8 = 0, 2
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63])


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_jpeg.so")
    vp, i, u64 = C.c_void_p, C.c_int, C.c_uint64
    L.zo_jpeg_encode.argtypes = [vp, i, i, i, i, vp, C.c_int64, vp, u64, C.POINTER(u64)]
    L.zo_jpeg_coefficients.argtypes = [vp, i, i, i, vp, u64, C.POINTER(u64)]
    L.zo_jpeg_encode.restype = L.zo_jpeg_coefficients.restype = C.c_int
    return L


def encodable(img: np.ndarray) -> np.ndarray:
    """The image jpeg.encode actually encodes: u8 and Rgb(u8) as they are, anything else through Image.convert(Rgb)."""
    fmt = pixfmt_of(img)
    if fmt in (PIX_U8, PIX_RGB8) or img.size == 0:
        return img
    return oracle_lib.convert(img, PIX_RGB8)


def _img(a: np.ndarray):
    return oracle_lib.ZoImage(None, a.shape[0], a.shape[1], a.shape[1]) if a.size == 0 else as_image(a)


def encode(img: np.ndarray, quality: int = 90, subsampling: int = YUV420, density_dpi: int = 72, comment: bytes | None = None) -> bytes:
    """jpeg.encode(T, allocator, image, .{quality, subsampling, density_dpi, comment}) -> the file's bytes.  Raises OracleStatus with
    29 (InvalidImageDimensions), 30 (ImageTooLarge) or 5 (comment over 65533 bytes, subsampling > 2)."""
    src = encodable(img)
    zi = _img(src)
    n = C.c_uint64()
    cbuf = None if comment is None else (C.c_uint8 * max(1, len(comment))).from_buffer_copy(comment or b"\0")
    clen = -1 if comment is None else len(comment)
    args = (C.byref(zi), pixfmt_of(src) if src.size else PIX_U8, int(quality), int(subsampling), int(density_dpi), cbuf, clen)
    rc = lib().zo_jpeg_encode(*args, None, 0, C.byref(n))
    if rc not in (0, 6):
        raise OracleStatus(rc, "jpeg_encode")
    out = np.zeros(n.value, np.uint8)
    rc = lib().zo_jpeg_encode(*args, out.ctypes.data, n.value, C.byref(n))
    if rc != 0:
        raise OracleStatus(rc, "jpeg_encode")
    return out.tobytes()


def coefficients(img: np.ndarray, quality: int = 90, subsampling: int = YUV420) -> np.ndarray:
    """The quantised coefficients of every block in scan order, natural (row-major) order inside a block: (n_blocks, 64) int32."""
    src = encodable(img)
    zi = _img(src)
    n = C.c_uint64()
    fmt = pixfmt_of(src)
    rc = lib().zo_jpeg_coefficients(C.byref(zi), fmt, int(quality), int(subsampling), None, 0, C.byref(n))
    if rc not in (0, 6):
        raise OracleStatus(rc, "jpeg_coefficients")
    out = np.zeros((n.value, 64), np.int32)
    rc = lib().zo_jpeg_coefficients(C.byref(zi), fmt, int(quality), int(subsampling), out.ctypes.data, n.value, C.byref(n))
    if rc != 0:
        raise OracleStatus(rc, "jpeg_coefficients")
    return out
