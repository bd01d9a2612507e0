"""ctypes binding of the CPU oracle of the baseline JPEG decoder (oracle/zo_jpeg_decode.cpp -> oracle/libzo_jpeg_decode.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: nothing under zignal_b200/ may import it.  The library is built on its own by
oracle/Makefile; __graft_entry__.build() runs it and lib() repeats it (make rebuilds only when a source is newer).

decode() is jpeg.loadFromBytes(T, ...) (codecs/jpeg.zig:2825-2851): the native image (u8 or Rgb(u8)) comes from the oracle, and any
other T goes through the main oracle's Image.convert (oracle_lib.convert), as loadFromBytes does.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import oracle_lib
from oracle_lib import OracleStatus, load

PIX_U8, PIX_F32, PIX_RGB8, PIX_RGBA8, PIX_RGBAF32 = 0, 1, 2, 3, 4
UNSUPPORTED, OUT_OF_MEMORY, IMAGE_TOO_LARGE, INVALID_JPEG = 3, 6, 30, 31


class Limits(C.Structure):
    """jpeg.DecodeLimits (codecs/jpeg.zig:19-33), its defaults; 0 disables a limit."""
    _fields_ = [("max_jpeg_bytes", C.c_uint64), ("max_marker_bytes", C.c_uint64), ("max_width", C.c_uint32), ("max_height", C.c_uint32),
                ("max_pixels", C.c_uint64), ("max_blocks", C.c_uint64), ("max_scans", C.c_uint64)]

    def __init__(self, **kw):
        d = dict(max_jpeg_bytes=100 << 20, max_marker_bytes=100 << 20, max_width=8192, max_height=8192, max_pixels=67108864,
                 max_blocks=1048576, max_scans=64)
        d.update(kw)
        super().__init__(**d)


class Header(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("frame_type", C.c_int32), ("num_components", C.c_int32),
                ("precision", C.c_int32), ("subsampling", C.c_int32)]


class DecodeError(OracleStatus):
    """An oracle refusal: status (3 Unsupported, 30 ImageTooLarge, 31 InvalidJpeg) and the reference's error name."""

    def __init__(self, status: int, name: str):
        super().__init__(status, "jpeg_decode")
        self.status, self.name = status, name

    def __str__(self):
        return f"jpeg_decode: {self.name} (status {self.status})"


@functools.cache
def lib() -> C.CDLL:
    L = load("libzo_jpeg_decode.so")
    vp, i, u64, cp = C.c_void_p, C.c_int, C.c_uint64, C.c_char_p
    L.zo_jpeg_info.argtypes = [vp, u64, vp, C.POINTER(Header), cp, i]
    L.zo_jpeg_decode.argtypes = [vp, u64, vp, i, vp, u64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_int), cp, i]
    L.zo_jpeg_decode_coefficients.argtypes = [vp, u64, vp, i, vp, u64, C.POINTER(u64), vp, cp, i]
    L.zo_jpeg_info.restype = L.zo_jpeg_decode.restype = L.zo_jpeg_decode_coefficients.restype = C.c_int
    return L


def _buf(data: bytes):
    return (C.c_uint8 * max(1, len(data))).from_buffer_copy(bytes(data) or b"\0")


def _lim(limits):
    return None if limits is None else C.byref(limits)


def info(data: bytes, limits: Limits | None = None) -> Header:
    h, err = Header(), C.create_string_buffer(64)
    rc = lib().zo_jpeg_info(_buf(data), len(data), _lim(limits), C.byref(h), err, 64)
    if rc:
        raise DecodeError(rc, err.value.decode())
    return h


def native(data: bytes, limits: Limits | None = None, literal_flush: bool = False) -> np.ndarray:
    """decode -> toNativeImage: (rows, cols) u8 for one component, (rows, cols, 3) u8 for three."""
    rows, cols, ch, err = C.c_uint32(), C.c_uint32(), C.c_int(), C.create_string_buffer(64)
    b = _buf(data)
    args = (b, len(data), _lim(limits), int(literal_flush))
    rc = lib().zo_jpeg_decode(*args, None, 0, C.byref(rows), C.byref(cols), C.byref(ch), err, 64)
    if rc != OUT_OF_MEMORY:
        raise DecodeError(rc, err.value.decode())
    shape = (rows.value, cols.value) + ((3,) if ch.value == 3 else ())
    out = np.zeros(shape, np.uint8)
    rc = lib().zo_jpeg_decode(*args, out.ctypes.data, out.size, C.byref(rows), C.byref(cols), C.byref(ch), err, 64)
    if rc:
        raise DecodeError(rc, err.value.decode())
    return out


def decode(data: bytes, pixfmt: int | None = None, limits: Limits | None = None) -> np.ndarray:
    """jpeg.loadFromBytes(T, allocator, data, limits); pixfmt None is the native type."""
    img = native(data, limits)
    fmt = PIX_U8 if img.ndim == 2 else PIX_RGB8
    if pixfmt is None or pixfmt == fmt:
        return img
    return oracle_lib.convert(img, pixfmt)


def coefficients(data: bytes, limits: Limits | None = None, literal_flush: bool = False):
    """The block storage after performBlockScan: (bwa * bha, ncomp, 64) int32 in natural order, and (bw, bh, bwa, bha, ncomp)."""
    n, geo, err = C.c_uint64(), (C.c_uint32 * 5)(), C.create_string_buffer(64)
    b = _buf(data)
    args = (b, len(data), _lim(limits), int(literal_flush))
    rc = lib().zo_jpeg_decode_coefficients(*args, None, 0, C.byref(n), geo, err, 64)
    if rc != OUT_OF_MEMORY:
        raise DecodeError(rc, err.value.decode())
    out = np.zeros((n.value, geo[4], 64), np.int32)
    rc = lib().zo_jpeg_decode_coefficients(*args, out.ctypes.data, n.value, C.byref(n), geo, err, 64)
    if rc:
        raise DecodeError(rc, err.value.decode())
    return out, tuple(geo)
