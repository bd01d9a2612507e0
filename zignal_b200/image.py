"""Host-side mirror of zignal's `Image(T)` for the hot path (reference src/image.zig:97-1249).

Same method names, argument meaning and error behaviour as the reference's Zig API (snake_case as in
the reference's own Python binding, bindings/python/src/image/*.zig); every method body is a call
through the C ABI in include/zignal_b200.h.  Pixel storage lives in device memory (a torch CUDA
tensor is used purely as the owner of that memory and of the stream); `Image.from_numpy` /
`to_numpy` move data across PCIe, and the module-level `host_*` functions are the literal drop-in
for host-resident `Image.data` (H2D + op + D2H inside one C call).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from enum import IntEnum
from typing import Optional, Tuple

import numpy as np

from . import _ffi
from ._ffi import ZbImage, check, lib


class PixFmt(IntEnum):
    U8 = 0        # Image(u8)
    F32 = 1       # Image(f32)
    RGB8 = 2      # Image(Rgb(u8))
    RGBA8 = 3     # Image(Rgba(u8))
    RGBAF32 = 4   # Image(Rgba(f32))


class BorderMode(IntEnum):  # reference border.zig:10-19
    ZERO = 0
    REPLICATE = 1
    MIRROR = 2
    WRAP = 3


class Blending(IntEnum):  # reference blending.zig:8-22
    NONE = 0
    NORMAL = 1
    MULTIPLY = 2
    SCREEN = 3
    OVERLAY = 4
    SOFT_LIGHT = 5
    HARD_LIGHT = 6
    COLOR_DODGE = 7
    COLOR_BURN = 8
    DARKEN = 9
    LIGHTEN = 10
    DIFFERENCE = 11
    EXCLUSION = 12


class Interpolation(IntEnum):  # reference interpolation.zig:53-68
    NEAREST = 0
    BILINEAR = 1
    BICUBIC = 2
    CATMULL_ROM = 3
    MITCHELL = 4
    LANCZOS = 5


class Connectivity(IntEnum):  # reference image/flood_fill.zig:6-9 (tag value = neighbour count)
    FOUR = 4
    EIGHT = 8


class FloodFillMode(IntEnum):  # reference image/flood_fill.zig:11-16 (ThresholdMode)
    SEED = 0       # compare each candidate against the seed pixel
    NEIGHBOR = 1   # compare each candidate against the neighbour it spread from


class Colormap(IntEnum):  # reference image/colormaps.zig:21-31 (union tag order)
    JET = 0
    HEAT = 1
    TURBO = 2
    VIRIDIS = 3   # a data table in the reference: pass its 256 x 3 bytes to Image.apply_colormap
    INFERNO = 4   # likewise


class JpegSubsampling(IntEnum):  # reference codecs/jpeg.zig:262-282 (Subsampling, enum order)
    YUV444 = 0
    YUV422 = 1
    YUV420 = 2


def _jpeg_options(quality: int, subsampling, density_dpi: int, comment: Optional[bytes]):
    """zb_jpeg_options plus the buffer that keeps the comment alive for the call."""
    if not 0 <= int(quality) <= 255 or not 0 <= int(density_dpi) <= 65535:
        raise ValueError("quality is a u8 and density_dpi a u16, as in jpeg.EncodeOptions")
    buf = None
    if comment is not None:
        comment = bytes(comment)
        buf = C.create_string_buffer(comment, len(comment) or 1)
    opts = _ffi.ZbJpegOptions(int(quality), int(subsampling), int(density_dpi), C.cast(buf, C.c_void_p) if buf is not None else None,
                              0 if comment is None else len(comment))
    return opts, buf


def jpeg_encode_bound(rows: int, cols: int, pixfmt, quality: int = 90, subsampling=2, density_dpi: int = 72,
                      comment: Optional[bytes] = None) -> int:
    """zb_jpeg_encode_bound: a byte capacity that always holds Image.encode_jpeg's output (no device work)."""
    opts, _keep = _jpeg_options(quality, subsampling, density_dpi, comment)
    n = C.c_uint64()
    check(lib().zb_jpeg_encode_bound(int(rows), int(cols), int(pixfmt), C.byref(opts), C.byref(n)))
    return n.value


@dataclass
class JpegLimits:  # reference codecs/jpeg.zig:19-33 (DecodeLimits, with its defaults; 0 disables a limit)
    max_jpeg_bytes: int = 100 * 1024 * 1024
    max_marker_bytes: int = 100 * 1024 * 1024
    max_width: int = 8192
    max_height: int = 8192
    max_pixels: int = 67_108_864
    max_blocks: int = 1_048_576
    max_scans: int = 64

    def _c(self):
        return _ffi.ZbJpegLimits(self.max_jpeg_bytes, self.max_marker_bytes, self.max_width, self.max_height, self.max_pixels,
                                 self.max_blocks, self.max_scans)


@dataclass(frozen=True)
class JpegHeader:  # reference codecs/jpeg.zig:61-73 (Header); subsampling None for grayscale or another layout
    width: int
    height: int
    progressive: bool
    num_components: int
    precision: int
    subsampling: Optional[JpegSubsampling]


def jpeg_info(data: bytes, limits: Optional[JpegLimits] = None) -> JpegHeader:
    """jpeg.getInfo (codecs/jpeg.zig:77-180): the first SOF's header, read on the host (progressive files included)."""
    h = _ffi.ZbJpegHeader()
    buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(bytes(data) or b"\0")
    check(lib().zb_jpeg_info(buf, len(data), None if limits is None else C.byref(limits._c()), C.byref(h)))
    return JpegHeader(int(h.width), int(h.height), bool(h.progressive), int(h.num_components), int(h.precision),
                      None if h.subsampling < 0 else JpegSubsampling(h.subsampling))


@dataclass(frozen=True)
class DiffStats:
    """RunningStats(f64, .summary) of Image.diff's samples, with the accessor names of the reference's Python RunningStats."""
    count: int
    sum: float
    mean: float
    variance: float
    min: float
    max: float

    @property
    def std_dev(self) -> float:
        return math.sqrt(self.variance)


@dataclass(frozen=True)
class DiffResult:  # reference image/diff.zig:19-22
    stats: DiffStats
    diff_count: int


def colormap_lut(cmap: Colormap) -> np.ndarray:
    """The (256, 3) uint8 table of jet / heat / turbo (colormaps.zig:92-190); viridis / inferno raise ZignalError Unsupported."""
    lut = np.zeros((256, 3), np.uint8)
    check(lib().zb_colormap_lut(int(Colormap(cmap)), lut.ctypes.data_as(C.c_void_p)))
    return lut


_CH = {PixFmt.U8: 1, PixFmt.F32: 1, PixFmt.RGB8: 3, PixFmt.RGBA8: 4, PixFmt.RGBAF32: 4}
_NP = {PixFmt.U8: np.uint8, PixFmt.F32: np.float32, PixFmt.RGB8: np.uint8, PixFmt.RGBA8: np.uint8, PixFmt.RGBAF32: np.float32}


def pixfmt_of_array(a) -> PixFmt:
    dt = np.dtype(str(a.dtype).replace("torch.", ""))
    nd = a.ndim
    ch = a.shape[2] if nd == 3 else 1
    if dt == np.uint8 and nd == 2:
        return PixFmt.U8
    if dt == np.uint8 and ch == 3:
        return PixFmt.RGB8
    if dt == np.uint8 and ch == 4:
        return PixFmt.RGBA8
    if dt == np.float32 and nd == 2:
        return PixFmt.F32
    if dt == np.float32 and ch == 4:
        return PixFmt.RGBAF32
    raise TypeError(f"unsupported pixel array: dtype={a.dtype} shape={tuple(a.shape)}")


def _np_image(a: np.ndarray) -> ZbImage:
    """zb_image over a (possibly row-strided) numpy array."""
    px_bytes = a.dtype.itemsize * (a.shape[2] if a.ndim == 3 else 1)
    if a.ndim == 3:
        assert a.strides[2] == a.dtype.itemsize and a.strides[1] == px_bytes, "pixels must be packed"
    elif a.shape[1] > 1:
        assert a.strides[1] == a.dtype.itemsize
    row = a.strides[0] if a.shape[0] > 1 else a.shape[1] * px_bytes
    assert row % px_bytes == 0
    return ZbImage(a.ctypes.data, a.shape[0], a.shape[1], row // px_bytes)


def _fptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _mitchell(method, b, c):
    return int(method), C.c_float(b), C.c_float(c)


def _torch():
    import torch
    return torch


def current_stream() -> int:
    torch = _torch()
    return torch.cuda.current_stream().cuda_stream


@dataclass
class Rectangle:  # reference geometry/Rectangle.zig: l, t, r, b (exclusive r, b)
    l: int
    t: int
    r: int
    b: int


class Image:
    """Device-resident mirror of zignal's Image(T) {rows, cols, data, stride} (image.zig:97-102)."""

    def __init__(self, tensor, pixfmt: PixFmt, rows: int, cols: int, stride: int, offset_px: int = 0):
        self._t = tensor          # torch tensor that owns the storage (flat, channel elements)
        self.pixfmt = PixFmt(pixfmt)
        self.rows, self.cols, self.stride = int(rows), int(cols), int(stride)
        self._off = int(offset_px)

    # ---- construction (image.zig:124-184) -------------------------------------------------------
    @classmethod
    def init(cls, rows: int, cols: int, pixfmt: PixFmt, device=None) -> "Image":
        torch = _torch()
        lib()  # fail loudly if the CUDA library is missing
        dt = torch.uint8 if _NP[PixFmt(pixfmt)] == np.uint8 else torch.float32
        t = torch.empty(int(rows) * int(cols) * _CH[PixFmt(pixfmt)], dtype=dt, device=device or "cuda")
        return cls(t, pixfmt, rows, cols, cols)

    @classmethod
    def init_like(cls, other: "Image") -> "Image":
        return cls.init(other.rows, other.cols, other.pixfmt, other._t.device)

    @classmethod
    def from_numpy(cls, a: np.ndarray, device=None) -> "Image":
        torch = _torch()
        lib()
        fmt = pixfmt_of_array(a)
        t = torch.from_numpy(np.ascontiguousarray(a)).to(device or "cuda").reshape(-1)
        return cls(t, fmt, a.shape[0], a.shape[1], a.shape[1])

    @classmethod
    def from_tensor(cls, t) -> "Image":
        """Wrap a contiguous CUDA tensor of shape (rows, cols[, ch]) without copying."""
        fmt = pixfmt_of_array(t)
        assert t.is_cuda and t.is_contiguous()
        return cls(t.reshape(-1), fmt, t.shape[0], t.shape[1], t.shape[1])

    def to_numpy(self) -> np.ndarray:
        ch = _CH[self.pixfmt]
        full = self._t.cpu().numpy()
        if self.rows == 0 or self.cols == 0:
            return np.zeros((self.rows, self.cols) + ((ch,) if ch > 1 else ()), _NP[self.pixfmt])
        idx = (self._off + np.arange(self.rows)[:, None] * self.stride + np.arange(self.cols)[None, :])
        if ch == 1:
            return full[idx]
        return full.reshape(-1, ch)[idx]

    def tensor(self):
        """The (rows, cols[, ch]) CUDA tensor of a contiguous, non-view image."""
        assert self.is_contiguous() and self._off == 0
        ch = _CH[self.pixfmt]
        return self._t.view(self.rows, self.cols, ch) if ch > 1 else self._t.view(self.rows, self.cols)

    # ---- views (image.zig:332-357) --------------------------------------------------------------
    def view(self, rect: Rectangle) -> "Image":
        l, t = max(0, rect.l), max(0, rect.t)
        r, b = min(self.cols, rect.r), min(self.rows, rect.b)
        if r <= l or b <= t:
            return Image(self._t, self.pixfmt, 0, 0, 0, 0)
        return Image(self._t, self.pixfmt, b - t, r - l, self.stride, self._off + t * self.stride + l)

    def is_contiguous(self) -> bool:
        return self.cols == self.stride

    def has_same_shape(self, other) -> bool:
        return self.rows == other.rows and self.cols == other.cols

    def get_center(self) -> Tuple[float, float]:  # image.zig:322-327
        return (np.float32(self.cols) / np.float32(2), np.float32(self.rows) / np.float32(2))

    def _zb(self) -> ZbImage:
        esz = self._t.element_size() * _CH[self.pixfmt]
        return ZbImage(self._t.data_ptr() + self._off * esz, self.rows, self.cols, self.stride)

    def copy(self, dst: "Image") -> None:  # image.zig:375-392
        assert self.has_same_shape(dst)
        self._peer(dst, what="dst")
        a, d = self._zb(), dst._zb()
        self._run(lib().zb_copy, a, d, int(self.pixfmt))

    def dupe(self) -> "Image":  # image.zig:367-371
        out = Image.init_like(self)
        self.copy(out)
        return out

    def _peer(self, other: "Image", fmt: Optional[PixFmt] = None, what: str = "out") -> "Image":
        """Zig's Image(T) typing makes a mismatched `out` a compile error; the C ABI takes one pixfmt for both buffers, so the
        mirror checks it here: same pixel type (or the op's fixed result type) and same CUDA device as self."""
        fmt = self.pixfmt if fmt is None else PixFmt(fmt)
        if not isinstance(other, Image):
            raise TypeError(f"{what} must be an Image")
        if other.pixfmt != fmt:
            raise TypeError(f"{what} must be an Image of pixel type {fmt.name}, got {other.pixfmt.name}")
        if other._t.device != self._t.device:
            raise ValueError(f"{what} lives on {other._t.device}, self on {self._t.device}")
        return other

    def _run(self, fn, *args) -> None:
        """Call a stream-taking entry point on self's device and on that device's current stream (not the stream of whatever
        device happens to be current)."""
        torch = _torch()
        dev = self._t.device
        with torch.cuda.device(dev):
            check(fn(*args, torch.cuda.current_stream(dev).cuda_stream))

    def _out(self, out: Optional["Image"], fmt: Optional[PixFmt] = None) -> "Image":
        if out is None:
            return Image.init(self.rows, self.cols, self.pixfmt if fmt is None else fmt, self._t.device)
        return self._peer(out, fmt)

    # ---- filters (image.zig:635-648, 785-799, 917-994) --------------------------------------------
    def box_blur(self, radius: int, out: Optional["Image"] = None) -> "Image":
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_box_blur, a, d, int(self.pixfmt), int(radius))
        return out

    def sharpen(self, radius: int, out: Optional["Image"] = None) -> "Image":
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_sharpen, a, d, int(self.pixfmt), int(radius))
        return out

    def convolve(self, kernel, border: BorderMode = BorderMode.MIRROR, out: Optional["Image"] = None) -> "Image":
        k = np.ascontiguousarray(kernel, dtype=np.float32)
        if k.ndim != 2:
            raise ValueError("Kernel must be a 2D array")  # convolution.zig:200
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_convolve, a, d, int(self.pixfmt), _fptr(k), k.shape[0], k.shape[1], int(border))
        return out

    def convolve_separable(self, kernel_x, kernel_y, border: BorderMode = BorderMode.MIRROR,
                           out: Optional["Image"] = None) -> "Image":
        kx = np.ascontiguousarray(kernel_x, dtype=np.float32)
        ky = np.ascontiguousarray(kernel_y, dtype=np.float32)
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_conv_separable, a, d, int(self.pixfmt), _fptr(kx), kx.size, _fptr(ky), ky.size, int(border))
        return out

    def gaussian_blur(self, sigma: float, out: Optional["Image"] = None) -> "Image":
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_gaussian_blur, a, d, int(self.pixfmt), C.c_float(sigma))
        return out

    # ---- resampling (image.zig:523-541) -----------------------------------------------------------
    def resize(self, out: "Image", method: Interpolation = Interpolation.BILINEAR, b: float = 1 / 3, c: float = 1 / 3) -> "Image":
        self._peer(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_resize, a, d, int(self.pixfmt), int(method), C.c_float(b), C.c_float(c))
        return out

    def scale(self, factor: float, method: Interpolation = Interpolation.BILINEAR) -> "Image":
        if factor <= 0:
            raise _ffi.ZignalError(8, "InvalidScaleFactor")       # image.zig:531
        new_rows = int(_round_half_away(np.float32(self.rows) * np.float32(factor)))
        new_cols = int(_round_half_away(np.float32(self.cols) * np.float32(factor)))
        if new_rows == 0 or new_cols == 0:
            raise _ffi.ZignalError(9, "InvalidDimensions")        # image.zig:536
        return self.resize(Image.init(new_rows, new_cols, self.pixfmt, self._t.device), method)

    # ---- geometry (image.zig:558-623) -------------------------------------------------------------
    def rotate_bounds(self, angle: float) -> Tuple[int, int]:
        r, c = C.c_uint32(), C.c_uint32()
        check(lib().zb_rotate_bounds(self.rows, self.cols, C.c_float(angle), C.byref(r), C.byref(c)))
        return r.value, c.value

    def rotate_into(self, out: "Image", angle: float, method: Interpolation = Interpolation.BILINEAR,
                    border: BorderMode = BorderMode.ZERO, cos_sin=None, b: float = 1 / 3, c: float = 1 / 3) -> "Image":
        self._peer(out)
        a, d = self._zb(), out._zb()
        if cos_sin is None:
            self._run(lib().zb_rotate_into, a, d, int(self.pixfmt), C.c_float(angle), int(method), C.c_float(b), C.c_float(c), int(border))
        else:
            self._run(lib().zb_rotate_into_cs, a, d, int(self.pixfmt), C.c_float(angle), C.c_float(cos_sin[0]), C.c_float(cos_sin[1]),
                                          int(method), C.c_float(b), C.c_float(c), int(border))
        return out

    def rotate(self, angle: float, method: Interpolation = Interpolation.BILINEAR, border: BorderMode = BorderMode.ZERO,
               cos_sin=None) -> "Image":
        rows, cols = self.rotate_bounds(angle)
        out = Image.init(rows, cols, self.pixfmt, self._t.device)
        return self.rotate_into(out, angle, method, border, cos_sin)

    def sobel(self, out: Optional["Image"] = None) -> "Image":
        """Image.sobel (image.zig:999-1009): gradient magnitude into an Image(u8) of the same shape."""
        out = self._out(out, PixFmt.U8)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_sobel, a, d, int(self.pixfmt))
        return out

    def convert(self, target: PixFmt, out: Optional["Image"] = None) -> "Image":
        """Image.convert(allocator, TargetType) / convertInto (image.zig:396-421): per-pixel convertColor into another pixel type."""
        target = PixFmt(target)
        out = self._out(out, target)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_convert, a, int(self.pixfmt), d, int(target))
        return out

    # ---- quality metrics (image.zig:1105-1147, metrics.zig) ----
    def _metric(self, fn, other: "Image") -> float:
        self._peer(other, what="other")  # Image(T).psnr(other: Image(T))
        out = C.c_double(0.0)
        a, b = self._zb(), other._zb()
        self._run(fn, a, b, int(self.pixfmt), C.byref(out))
        return out.value

    def psnr(self, other: "Image") -> float:
        """Image.psnr (image.zig:1105, metrics.zig:10-54): dB, inf for identical images."""
        return self._metric(lib().zb_psnr, other)

    def ssim(self, other: "Image") -> float:
        """Image.ssim (image.zig:1126, metrics.zig:56-114): mean SSIM over the interior, 11x11 Gaussian window (sigma 1.5)."""
        return self._metric(lib().zb_ssim, other)

    def mean_pixel_error(self, other: "Image") -> float:
        """Image.meanPixelError (image.zig:1145, metrics.zig:116-165): mean absolute component difference / component range."""
        return self._metric(lib().zb_mean_pixel_error, other)

    # ---- order-statistic filters (image.zig:650-790, order_statistic_blur.zig) ----
    def _order(self, radius: int, mode: int, param: float, border: BorderMode, out: Optional["Image"]) -> "Image":
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_order_blur, a, d, int(self.pixfmt), int(radius), mode, C.c_double(param), int(border))
        return out

    def percentile_blur(self, radius: int, percentile: float, border: BorderMode = BorderMode.MIRROR, out: Optional["Image"] = None) -> "Image":
        """Image.percentileBlur (image.zig:672-684)."""
        return self._order(radius, 0, percentile, border, out)

    def median_blur(self, radius: int, out: Optional["Image"] = None) -> "Image":
        """Image.medianBlur (image.zig:650-658): percentile 0.5 with .mirror (order_statistic_blur.zig:28)."""
        return self._order(radius, 0, 0.5, BorderMode.MIRROR, out)

    def min_blur(self, radius: int, border: BorderMode = BorderMode.MIRROR, out: Optional["Image"] = None) -> "Image":
        """Image.minBlur (image.zig:696-707): erosion."""
        return self._order(radius, 0, 0.0, border, out)

    def max_blur(self, radius: int, border: BorderMode = BorderMode.MIRROR, out: Optional["Image"] = None) -> "Image":
        """Image.maxBlur (image.zig:719-730): dilation."""
        return self._order(radius, 0, 1.0, border, out)

    def midpoint_blur(self, radius: int, border: BorderMode = BorderMode.MIRROR, out: Optional["Image"] = None) -> "Image":
        """Image.midpointBlur (image.zig:742-753)."""
        return self._order(radius, 1, 0.0, border, out)

    def alpha_trimmed_mean_blur(self, radius: int, trim_fraction: float, border: BorderMode = BorderMode.MIRROR,
                                out: Optional["Image"] = None) -> "Image":
        """Image.alphaTrimmedMeanBlur (image.zig:767-779)."""
        return self._order(radius, 2, trim_fraction, border, out)

    def canny(self, sigma: float, low_threshold: float, high_threshold: float, out: Optional["Image"] = None) -> "Image":
        """Image.canny (image.zig:1041-1063, edges.zig:212-274): binary (0 / 255) edge map into an Image(u8) of the same shape."""
        out = self._out(out, PixFmt.U8)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_canny, a, d, int(self.pixfmt), C.c_float(sigma), C.c_float(low_threshold), C.c_float(high_threshold))
        return out

    def shen_castan(self, smooth: float = 0.9, window_size: int = 7, high_ratio: float = 0.99, low_rel: float = 0.5,
                    hysteresis: bool = True, use_nms: bool = False, out: Optional["Image"] = None) -> "Image":
        """Image.shenCastan (image.zig:1015-1027, edges.zig:83-198): binary (0 / 255) edge map into an Image(u8) of the same shape.
        The defaults are ShenCastan's (ShenCastan.zig:9-32); `ShenCastan.<preset>.apply(img)` runs one of the reference's presets."""
        out = self._out(out, PixFmt.U8)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_shen_castan, a, d, int(self.pixfmt), C.c_float(smooth), int(window_size), C.c_float(high_ratio), C.c_float(low_rel),
                  int(bool(hysteresis)), int(bool(use_nms)))
        return out

    # ---- histogram-based and binary operations on 8-bit images (image.zig:804-914, 1161-1185) ----
    def histogram(self) -> np.ndarray:
        """Image.histogram (image.zig:1161-1185): (channels, 256) uint32 counts; RGBA8 counts alpha too."""
        counts = np.zeros((_CH[self.pixfmt], 256), np.uint32)
        a = self._zb()
        self._run(lib().zb_histogram, a, int(self.pixfmt), counts.ctypes.data_as(C.POINTER(C.c_uint32)))
        return counts

    def autocontrast(self, cutoff: float = 0.0) -> "Image":
        """Image.autocontrast (image.zig:804, enhancement.zig:11-80): in place; RGBA alpha is left untouched."""
        a = self._zb()
        self._run(lib().zb_autocontrast, a, int(self.pixfmt), C.c_float(cutoff))
        return self

    def equalize(self) -> "Image":
        """Image.equalize (image.zig:824, enhancement.zig:84-252): in place, every channel (RGBA alpha too)."""
        a = self._zb()
        self._run(lib().zb_equalize, a, int(self.pixfmt))
        return self

    def flood_fill(self, start_row: int, start_col: int, fill_value, threshold: float = 0.0,
                   connectivity: Connectivity = Connectivity.FOUR, mode: FloodFillMode = FloodFillMode.SEED) -> "Image":
        """Image.floodFill (image.zig:831-840, image/flood_fill.zig:59-131): in place, returns self.  fill_value is a scalar for U8 / F32 and
        a tuple of 3 (RGB8) or 4 (RGBA8, RGBAF32) channels.  A seed outside the image raises ZignalError OutOfBounds."""
        ch = _CH[self.pixfmt]
        v = np.atleast_1d(np.asarray(fill_value, dtype=np.float64))
        if v.ndim != 1 or v.size != ch:
            raise ValueError(f"fill_value must have {ch} channel(s) for {self.pixfmt.name}, got {fill_value!r}")
        if _NP[self.pixfmt] == np.uint8 and not np.all((v >= 0) & (v <= 255) & (v == np.floor(v))):
            raise ValueError(f"fill_value {fill_value!r} is not a u8 pixel")
        px = v.astype(_NP[self.pixfmt])
        a = self._zb()
        self._run(lib().zb_flood_fill, a, int(self.pixfmt), int(start_row), int(start_col), px.ctypes.data_as(C.c_void_p),
                  C.c_double(threshold), int(Connectivity(connectivity)), int(FloodFillMode(mode)))
        return self

    def dither(self, lut, mode) -> "Image":
        """dither.apply (dither.zig:34-331) in place on an Rgb(u8) image or view with lut.palette and lut (a quantize.ColorLookupTable);
        `mode` a quantize.DitherMode (NONE and AUTO do nothing).  Returns self."""
        pal = lut.palette
        a = self._zb()
        self._run(lib().zb_dither, a, int(self.pixfmt), pal.ctypes.data_as(C.c_void_p), pal.shape[0], lut.table.data_ptr(), int(mode))
        return self

    def palette_indices(self, lut, out: Optional["Image"] = None) -> "Image":
        """ColorLookupTable.lookup(convertColor(Rgb, px)) per pixel (quantize.zig:163-168) into a u8 index image; any pixel type."""
        out = self._out(out, PixFmt.U8)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_palette_lookup, a, int(self.pixfmt), lut.table.data_ptr(), d)
        return out

    # ---- visualisation (image.zig:480-511, 1139, 1190-1247) ----
    def diff(self, other: "Image", out: Optional["Image"] = None, threshold: float = 0.0, scale: float = 1.0, binary: bool = False,
             force_opaque: bool = False) -> Tuple["Image", DiffResult]:
        """Image.diff (image.zig:1139, diff.zig:27-203): (out, DiffResult).  out may be self or other."""
        self._peer(other, what="other")
        out = self._out(out)
        st = _ffi.ZbDiffStats()
        a, b, d = self._zb(), other._zb(), out._zb()
        self._run(lib().zb_diff, a, b, d, int(self.pixfmt), C.c_float(threshold), C.c_float(scale), int(bool(binary)), int(bool(force_opaque)),
                  C.byref(st))
        stats = DiffStats(int(st.n), st.sum, st.mean, st.variance, st.min, st.max)
        return out, DiffResult(stats, int(st.diff_count))

    def encode_jpeg(self, quality: int = 90, subsampling: "JpegSubsampling" = JpegSubsampling.YUV420, density_dpi: int = 72,
                    comment: Optional[bytes] = None) -> bytes:
        """jpeg.encode(T, allocator, image, options) (codecs/jpeg.zig:307-325): the baseline JPEG file as bytes, byte-identical to
        zignal's encoder.  U8 images are grayscale JPEGs; every other pixel type is encoded as Rgb(u8) (Image.convert(Rgb) first).  The
        defaults are jpeg.save's, so Image.save("x.jpg") is open(...).write(img.encode_jpeg()).  Errors: InvalidImageDimensions (an
        empty image), ImageTooLarge (rows or cols above 65535)."""
        opts, _keep = _jpeg_options(quality, subsampling, density_dpi, comment)
        src = self._zb()
        n = C.c_uint64()
        # the raw pixel bytes plus the header hold almost every image; a larger stream reports its exact size and is fetched again
        cap = self.rows * self.cols * _CH[self.pixfmt] * self._t.element_size() + 1024 + (0 if comment is None else len(comment))
        for attempt in range(2):
            out = (C.c_uint8 * max(1, cap))()
            torch = _torch()
            dev = self._t.device
            with torch.cuda.device(dev):
                rc = lib().zb_jpeg_encode(src, int(self.pixfmt), C.byref(opts), out, cap, C.byref(n),
                                          torch.cuda.current_stream(dev).cuda_stream)
            if rc == 6 and attempt == 0 and n.value > cap:
                cap = n.value
                continue
            check(rc)
            return bytes(memoryview(out)[:n.value])
        raise AssertionError("unreachable")

    @classmethod
    def decode_jpeg(cls, data: bytes, pixfmt: Optional[PixFmt] = None, limits: Optional[JpegLimits] = None, device=None,
                    out: Optional["Image"] = None) -> "Image":
        """jpeg.loadFromBytes(T, allocator, data, limits) (codecs/jpeg.zig:2825-2851) for baseline JPEGs, decoded on the device (entropy
        decoding included) and equal pixel for pixel to zignal's decoder.  pixfmt None means the file's native type (U8 for one
        component, RGB8 for three).  out: an existing device image (a view is fine) of the file's size to decode into.  Progressive
        files raise Unsupported; malformed ones InvalidJpeg; files over the limits ImageTooLarge."""
        if out is None:
            hdr = jpeg_info(data, limits)
            if pixfmt is None:
                pixfmt = PixFmt.U8 if hdr.num_components == 1 else PixFmt.RGB8
            out = cls.init(hdr.height, hdr.width, PixFmt(pixfmt), device)
        elif pixfmt is not None and PixFmt(pixfmt) != out.pixfmt:
            raise TypeError("out's pixel type differs from pixfmt")
        buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(bytes(data) or b"\0")
        lim = None if limits is None else C.byref(limits._c())
        out._run(lib().zb_jpeg_decode, buf, len(data), lim, out._zb(), int(out.pixfmt))
        return out

    @classmethod
    def decode_jpeg_batch(cls, datas, pixfmt=None, limits: Optional[JpegLimits] = None, device=None) -> list:
        """decode_jpeg for many files in one call (zb_jpeg_decode_batch): the files' scans go to the device together and every stage
        runs once for the batch.  pixfmt: None (each file's native type), one PixFmt, or one per file.  Returns, in order, an Image or
        the ZignalError that decode_jpeg would have raised for each file, so one bad file does not cost the others."""
        datas = [bytes(d) for d in datas]
        n = len(datas)
        fmts = list(pixfmt) if isinstance(pixfmt, (list, tuple)) else [pixfmt] * n
        if len(fmts) != n:
            raise ValueError(f"{len(fmts)} pixel formats for {n} files")
        out: list = [None] * n
        sent = []   # (index, image) of the files whose header jpeg_info reads
        for k, (d, fmt) in enumerate(zip(datas, fmts)):
            try:
                hdr = jpeg_info(d, limits)
            except _ffi.ZignalError as e:
                out[k] = e
                continue
            if fmt is None:
                fmt = PixFmt.U8 if hdr.num_components == 1 else PixFmt.RGB8
            sent.append((k, cls.init(hdr.height, hdr.width, PixFmt(fmt), device)))
        if not sent:
            return out
        m = len(sent)
        bufs = [(C.c_uint8 * max(1, len(datas[k]))).from_buffer_copy(datas[k] or b"\0") for k, _ in sent]
        ptrs = (C.c_void_p * m)(*[C.addressof(b) for b in bufs])
        lens = (C.c_uint64 * m)(*[len(datas[k]) for k, _ in sent])
        dsts = (ZbImage * m)(*[img._zb() for _, img in sent])
        fmt_arr = (C.c_int * m)(*[int(img.pixfmt) for _, img in sent])
        status = (C.c_int * m)()
        lim = None if limits is None else C.byref(limits._c())
        sent[0][1]._run(lib().zb_jpeg_decode_batch, m, ptrs, lens, lim, dsts, fmt_arr, status)
        for (k, img), st in zip(sent, status):
            try:
                check(st)
                out[k] = img
            except _ffi.ZignalError as e:
                out[k] = e
        return out

    def apply_colormap(self, map_or_lut, min: Optional[float] = None, max: Optional[float] = None) -> "Image":
        """Image.applyColormap (image.zig:1190-1247): a new RGB8 image.  map_or_lut: a Colormap (jet / heat / turbo) or a (256, 3) uint8
        table (viridis / inferno come as data, e.g. zignal's colormaps.viridis(i, 0, 255) for i in 0..255).  A bound left None comes from
        the image's pixels."""
        if isinstance(map_or_lut, (int, Colormap)):
            lut = colormap_lut(map_or_lut)
        else:
            lut = np.ascontiguousarray(map_or_lut, dtype=np.uint8)
            if lut.shape != (256, 3):
                raise ValueError(f"a colormap table is 256 x 3 bytes, got shape {lut.shape}")
        out = Image.init(self.rows, self.cols, PixFmt.RGB8, self._t.device)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_apply_colormap, a, int(self.pixfmt), lut.ctypes.data_as(C.c_void_p), int(min is not None),
                  C.c_double(0.0 if min is None else min), int(max is not None), C.c_double(0.0 if max is None else max), d)
        return out

    def flip_left_right(self) -> "Image":
        """Image.flipLeftRight (image.zig:480-483, transforms.zig:28-33): in place, returns self."""
        a = self._zb()
        self._run(lib().zb_flip_left_right, a, int(self.pixfmt))
        return self

    def flip_top_bottom(self) -> "Image":
        """Image.flipTopBottom (image.zig:485-488, transforms.zig:36-44): in place, returns self."""
        a = self._zb()
        self._run(lib().zb_flip_top_bottom, a, int(self.pixfmt))
        return self

    def invert(self) -> "Image":
        """Image.invert (image.zig:494-511): in place, returns self; Rgba alpha is kept; F32 raises ZignalError Unsupported."""
        a = self._zb()
        self._run(lib().zb_invert, a, int(self.pixfmt))
        return self

    def threshold_otsu(self, out: Optional["Image"] = None) -> Tuple["Image", int]:
        """Image(u8).thresholdOtsu (image.zig:845, binary.zig:38-84): (out, threshold); out = src > threshold ? 255 : 0."""
        self._require_u8()
        out = self._out(out)
        t = C.c_uint8(0)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_threshold_otsu, a, d, C.byref(t))
        return out, int(t.value)

    def threshold_adaptive_mean(self, radius: int, c: float, out: Optional["Image"] = None) -> "Image":
        """Image(u8).thresholdAdaptiveMean (image.zig:858, binary.zig:86-119): src > mean of the clipped (2r+1)^2 window - c ? 255 : 0."""
        self._require_u8()
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_threshold_adaptive_mean, a, d, int(radius), C.c_float(c))
        return out

    def _morph(self, op: int, kernel, iterations: int, out: Optional["Image"]) -> "Image":
        self._require_u8()
        k = np.ascontiguousarray(kernel, dtype=np.uint8)
        if k.ndim != 2:
            raise ValueError("kernel must be a 2D array")
        out = self._out(out)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_morph_binary, a, d, k.ctypes.data_as(C.POINTER(C.c_uint8)), k.shape[0], k.shape[1], int(iterations), op)
        return out

    def dilate_binary(self, kernel, iterations: int = 1, out: Optional["Image"] = None) -> "Image":
        """Image(u8).dilateBinary (image.zig:870, binary.zig:121-280); kernel: 2-D uint8 array, odd x odd, non-zero = on."""
        return self._morph(0, kernel, iterations, out)

    def erode_binary(self, kernel, iterations: int = 1, out: Optional["Image"] = None) -> "Image":
        """Image(u8).erodeBinary (image.zig:881)."""
        return self._morph(1, kernel, iterations, out)

    def open_binary(self, kernel, iterations: int = 1, out: Optional["Image"] = None) -> "Image":
        """Image(u8).openBinary (image.zig:892): erode^n then dilate^n."""
        return self._morph(2, kernel, iterations, out)

    def close_binary(self, kernel, iterations: int = 1, out: Optional["Image"] = None) -> "Image":
        """Image(u8).closeBinary (image.zig:903): dilate^n then erode^n."""
        return self._morph(3, kernel, iterations, out)

    def _require_u8(self) -> None:
        if self.pixfmt != PixFmt.U8:   # a compile error for Image(T != u8) in the reference (image.zig:846,859,871)
            raise _ffi.ZignalError(3, "Unsupported", f"only Image(u8), got {self.pixfmt.name}")

    def extract(self, out: "Image", rect, angle: float = 0.0, method: Interpolation = Interpolation.BILINEAR,
                border: BorderMode = BorderMode.ZERO, b: float = 1 / 3, c: float = 1 / 3) -> "Image":
        """Image.extract (transforms.zig:232-283): rect = (l, t, r, b) floats in source coordinates, rotated by `angle` CCW."""
        self._peer(out)
        a32 = np.float32(angle)
        cos_a, sin_a = np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32)
        a, d = self._zb(), out._zb()
        self._run(lib().zb_extract, a, d, int(self.pixfmt), C.c_float(rect[0]), C.c_float(rect[1]), C.c_float(rect[2]), C.c_float(rect[3]),
                               C.c_float(a32), C.c_float(cos_a), C.c_float(sin_a), int(method), C.c_float(b), C.c_float(c), int(border))
        return out

    def insert(self, source: "Image", rect, angle: float = 0.0, method: Interpolation = Interpolation.BILINEAR,
               b: float = 1 / 3, c: float = 1 / 3, blend: "Blending" = Blending.NONE) -> "Image":
        """Image.insert(source, rect, angle, method, blend_mode) (transforms.zig:293-376): modifies self in place.  Rgba(u8) samples are
        composited under a blend mode (blending.zig:26-156); other pixel types are assigned (image.zig:67-95)."""
        a32 = np.float32(angle)
        cos_a, sin_a = np.cos(a32, dtype=np.float32), np.sin(a32, dtype=np.float32)
        self._peer(source, fmt=source.pixfmt, what="source")          # `source: anytype`: any pixel type, same device
        d, s = self._zb(), source._zb()
        self._run(lib().zb_insert_from, d, int(self.pixfmt), s, int(source.pixfmt), C.c_float(rect[0]), C.c_float(rect[1]), C.c_float(rect[2]),
                  C.c_float(rect[3]), C.c_float(a32), C.c_float(cos_a), C.c_float(sin_a), int(method), C.c_float(b), C.c_float(c), int(blend))
        return self

    def crop(self, rect) -> "Image":
        """Image.crop (transforms.zig:216-222): round(height) x round(width) chip, out-of-bounds pixels zero."""
        def rnd(v):  # @round on f32, half away from zero
            v = np.float32(v)
            return int(np.sign(v) * np.floor(np.abs(np.float64(v)) + 0.5))
        l, t, r, b = (np.float32(v) for v in rect)
        rows, cols = rnd(np.float32(0) if t >= b else b - t), rnd(np.float32(0) if l >= r else r - l)   # Rectangle.height / width
        chip = Image.init(max(rows, 0), max(cols, 0), self.pixfmt, device=self._t.device)
        return self.extract(chip, rect, 0.0, Interpolation.NEAREST, BorderMode.ZERO)

    def warp(self, out: "Image", transform, method: Interpolation = Interpolation.BILINEAR, b: float = 1 / 3, c: float = 1 / 3) -> "Image":
        self._peer(out)
        kind, m = transform.as_f32()
        a, d = self._zb(), out._zb()
        self._run(lib().zb_warp, a, d, int(self.pixfmt), kind, _fptr(m), int(method), C.c_float(b), C.c_float(c))
        return out


@dataclass(frozen=True)
class ShenCastan:
    """Options of Image.shen_castan (the reference's ShenCastan, ShenCastan.zig:9-37) and its presets (:51-99) as class attributes:
    ShenCastan.default, low_noise, high_noise, heavy_smooth, sensitive, thin, strong_only."""
    smooth: float = 0.9          # ISEF smoothing factor, 0 < smooth < 1
    window_size: int = 7         # odd, >= 3: window of the local gradient statistics
    high_ratio: float = 0.99     # percentile of the high threshold, 0 < high_ratio < 1
    low_rel: float = 0.5         # low threshold as a fraction of the high one, 0 < low_rel < 1
    hysteresis: bool = True      # link weak edges to strong ones
    use_nms: bool = False        # non-maximum suppression instead of forward-neighbour thinning

    def apply(self, img: Image, out: Optional[Image] = None) -> Image:
        return img.shen_castan(self.smooth, self.window_size, self.high_ratio, self.low_rel, self.hysteresis, self.use_nms, out=out)


ShenCastan.default = ShenCastan()
ShenCastan.low_noise = ShenCastan(smooth=0.95, high_ratio=0.98)
ShenCastan.high_noise = ShenCastan(smooth=0.7, window_size=11)
ShenCastan.heavy_smooth = ShenCastan(smooth=0.5, window_size=9, high_ratio=0.95)
ShenCastan.sensitive = ShenCastan(high_ratio=0.97, low_rel=0.4)
ShenCastan.thin = ShenCastan(use_nms=True)
ShenCastan.strong_only = ShenCastan(hysteresis=False)
ShenCastan.PRESETS = ("default", "low_noise", "high_noise", "heavy_smooth", "sensitive", "thin", "strong_only")


def _round_half_away(v) -> float:
    v = float(v)
    return math.floor(abs(v) + 0.5) * (1 if v >= 0 else -1)


# ---------------------------------------------------------------------------------------------------
# Host-resident drop-ins: numpy in, numpy out; H2D + kernel + D2H happen inside one C-ABI call.
# ---------------------------------------------------------------------------------------------------
def _host_call(fn_name, src: np.ndarray, out: np.ndarray, *args):
    a, d = _np_image(src), _np_image(out)
    check(getattr(lib(), fn_name)(a, d, int(pixfmt_of_array(src)), *args))
    return out


def host_gaussian_blur(src: np.ndarray, sigma: float, out: Optional[np.ndarray] = None) -> np.ndarray:
    out = np.empty_like(src) if out is None else out
    return _host_call("zb_host_gaussian_blur", src, out, C.c_float(sigma))


def host_conv_separable(src, kx, ky, border=BorderMode.MIRROR, out=None) -> np.ndarray:
    out = np.empty_like(src) if out is None else out
    kx = np.ascontiguousarray(kx, dtype=np.float32)
    ky = np.ascontiguousarray(ky, dtype=np.float32)
    return _host_call("zb_host_conv_separable", src, out, _fptr(kx), kx.size, _fptr(ky), ky.size, int(border))


def host_convolve(src, kernel, border=BorderMode.MIRROR, out=None) -> np.ndarray:
    out = np.empty_like(src) if out is None else out
    k = np.ascontiguousarray(kernel, dtype=np.float32)
    return _host_call("zb_host_convolve", src, out, _fptr(k), k.shape[0], k.shape[1], int(border))


def host_box_blur(src, radius, out=None) -> np.ndarray:
    out = np.empty_like(src) if out is None else out
    return _host_call("zb_host_box_blur", src, out, int(radius))


def host_sharpen(src, radius, out=None) -> np.ndarray:
    out = np.empty_like(src) if out is None else out
    return _host_call("zb_host_sharpen", src, out, int(radius))


def host_resize(src, out_shape, method=Interpolation.BILINEAR, b=1 / 3, c=1 / 3, out=None) -> np.ndarray:
    if out is None:
        out = np.zeros((out_shape[0], out_shape[1]) + tuple(src.shape[2:]), dtype=src.dtype)
    return _host_call("zb_host_resize", src, out, int(method), C.c_float(b), C.c_float(c))


def host_rotate(src, angle, method=Interpolation.BILINEAR, border=BorderMode.ZERO) -> np.ndarray:
    r, c = C.c_uint32(), C.c_uint32()
    check(lib().zb_rotate_bounds(src.shape[0], src.shape[1], C.c_float(angle), C.byref(r), C.byref(c)))
    out = np.zeros((r.value, c.value) + tuple(src.shape[2:]), dtype=src.dtype)
    return _host_call("zb_host_rotate_into", src, out, C.c_float(angle), int(method), C.c_float(1 / 3), C.c_float(1 / 3), int(border))


def host_warp(src, out, transform, method=Interpolation.BILINEAR) -> np.ndarray:
    kind, m = transform.as_f32()
    return _host_call("zb_host_warp", src, out, kind, _fptr(m), int(method), C.c_float(1 / 3), C.c_float(1 / 3))


def gaussian_taps(sigma: float) -> np.ndarray:
    """Host math of gaussianBlur (image.zig:972-990)."""
    n = C.c_int()
    buf = np.zeros(8192, np.float32)
    check(lib().zb_gaussian_taps(C.c_float(sigma), _fptr(buf), buf.size, C.byref(n)))
    return buf[: n.value].copy()
