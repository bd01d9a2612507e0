"""zignal_b200 -- H100 (sm_90a) implementation of zignal's per-pixel image hot path behind a C ABI.

`zignal_b200.lib/libzignal_b200.so` is the product; this package is the thin host-side mirror of the
reference's Image(T)/Matrix API over that ABI (see include/zignal_b200.h and INTEGRATION.md).
"""
from ._ffi import LibraryMissing, ZignalError, ZbImage, declared_symbols, lib  # noqa: F401
from .image import (Blending, BorderMode, ColorFormat, Colormap, ColorSpace, Component, Connectivity, DiffResult, DiffStats, FloodFillMode, Image, Interpolation, JpegHeader, JpegLimits, JpegSubsampling, PixFmt, Rectangle, ShenCastan,  # noqa: F401
                    colormap_lut, gaussian_taps, host_box_blur, jpeg_encode_bound, jpeg_info,
                    host_conv_separable, host_convolve, host_gaussian_blur, host_resize, host_rotate, host_sharpen,
                    host_warp)
from .hough import HoughTransform, Line  # noqa: F401
from .quantize import ColorLookupTable, DitherMode, PaletteMode, build_palette, median_cut  # noqa: F401

from . import fdm, matrix, pca  # noqa: F401,E402

decode_jpeg_batch = Image.decode_jpeg_batch

__version__ = "0.1.0"
