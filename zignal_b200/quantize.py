"""Colour quantization (reference src/image/quantize.zig) and the palette side of dithering (src/image/dither.zig) on the GPU.

`median_cut` / `build_palette` return a host palette, an (n, 3) uint8 array, as the reference's functions fill a `[]Rgb`; they wait for the
device.  `ColorLookupTable` holds the 32x32x32 nearest-colour table on the device, together with the palette it was built from.
`Image.dither` and `Image.palette_indices` (image.py) take one.
"""
from __future__ import annotations

import ctypes as C
from enum import IntEnum

import numpy as np

from ._ffi import check, lib
from .image import Image, _torch

LUT_SIZE = 32768


class PaletteMode(IntEnum):  # reference quantize.zig:476-487 (tag order); ADAPTIVE takes max_colors
    FIXED_6X7X6 = 0
    FIXED_VGA16 = 1
    FIXED_WEB216 = 2
    ADAPTIVE = 3


class DitherMode(IntEnum):  # reference dither.zig:18-30 (tag order); AUTO is left to the caller to resolve, so apply() ignores it
    NONE = 0
    FLOYD_STEINBERG = 1
    ATKINSON = 2
    ORDERED = 3
    AUTO = 4


def _palette_array(palette) -> np.ndarray:
    p = np.ascontiguousarray(np.asarray(palette, dtype=np.uint8).reshape(-1, 3))
    if not 1 <= p.shape[0] <= 256:
        raise ValueError(f"a palette has 1 to 256 colours, got {p.shape[0]}")
    return p


def _stream(image: Image):
    torch = _torch()
    return torch.cuda.current_stream(image._t.device).cuda_stream


def median_cut(image: Image, max_colors: int = 256, cap: int = 256) -> np.ndarray:
    """medianCut (quantize.zig:175-412) over a device image of any pixel type: at most min(max_colors, cap) colours.  No colour
    (empty image, max_colors == 0, cap == 0) raises ZignalError NoPaletteColors."""
    torch = _torch()
    out = np.zeros((max(int(cap), 1), 3), np.uint8)
    n = C.c_uint32(0)
    with torch.cuda.device(image._t.device):
        check(lib().zb_median_cut(image._zb(), int(image.pixfmt), int(max_colors), out.ctypes.data_as(C.c_void_p), int(cap), C.byref(n),
                                  _stream(image)))
    return out[:n.value].copy()


def build_palette(image: Image, mode: PaletteMode, max_colors: int = 256) -> np.ndarray:
    """buildPalette (quantize.zig:502-527): a fixed palette, or median cut falling back to the fixed 6x7x6 one as the reference does."""
    torch = _torch()
    out = np.zeros((256, 3), np.uint8)
    n = C.c_uint32(0)
    with torch.cuda.device(image._t.device):
        check(lib().zb_build_palette(image._zb(), int(image.pixfmt), int(PaletteMode(mode)), int(max_colors),
                                     out.ctypes.data_as(C.c_void_p), C.byref(n), _stream(image)))
    return out[:n.value].copy()


class ColorLookupTable:
    """ColorLookupTable.init(palette) (quantize.zig:66-159) on the device: `table` is a CUDA uint8 tensor of 32768 entries,
    table[r5 << 10 | g5 << 5 | b5] = the palette index nearest to the 5-bit colour (smallest index on ties)."""

    def __init__(self, palette, device=None):
        torch = _torch()
        self.palette = _palette_array(palette)
        dev = torch.device(device or "cuda")
        self.table = torch.empty(LUT_SIZE, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(lib().zb_color_lut(self.palette.ctypes.data_as(C.c_void_p), self.palette.shape[0], self.table.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream))

    def to_numpy(self) -> np.ndarray:
        return self.table.cpu().numpy()
