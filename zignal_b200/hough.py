"""Host-side mirror of zignal's HoughTransform (reference src/image/hough.zig:10-257): line detection on a binary edge map.

`compute` votes on the GPU into a caller-owned accumulator, a 2-D CUDA int32 / uint32 tensor of size x size (a view with unit column
stride is fine); like the reference it ADDS to the accumulator, so zero it first.  `find_lines` finds the peaks on the GPU and runs the
sort, the non-maximum suppression and the line geometry on the host, as the reference does.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Tuple

from ._ffi import ZbHoughLine, ZbImage, check, lib
from .image import Image, PixFmt, Rectangle, _torch


@dataclass(frozen=True)
class Line:
    """HoughTransform.Line (hough.zig:13-25): angle in degrees (0 horizontal, +-90 vertical), radius from the centre of the Hough box,
    score (votes), and the end points of the segment clipped to [0, size]^2 in box coordinates."""
    angle: float
    radius: float
    score: int
    p1: Tuple[float, float]
    p2: Tuple[float, float]


def _acc_image(acc) -> ZbImage:
    torch = _torch()
    if not (isinstance(acc, torch.Tensor) and acc.is_cuda and acc.dtype in (torch.int32, torch.uint32) and acc.dim() == 2):
        raise TypeError("accumulator must be a 2-D CUDA int32 or uint32 tensor")
    rows, cols = acc.shape
    if cols > 1 and acc.stride(1) != 1:
        raise ValueError("accumulator columns must be contiguous (unit column stride)")
    stride = acc.stride(0) if rows > 1 else cols
    return ZbImage(acc.data_ptr(), rows, cols, stride)


class HoughTransform:
    """HoughTransform.init(allocator, size) (hough.zig:38-66): a size x size Hough space.  size <= 1 raises InvalidArgument, size > 32768
    raises Unsupported (the reference's i32 arithmetic overflows there)."""

    def __init__(self, size: int):
        h = C.c_void_p()
        check(lib().zb_hough_create(int(size), None, None, C.byref(h)))
        self._h = h
        self.size = int(size)
        self.even_size = self.size - self.size % 2

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib().zb_hough_destroy(h)
            self._h = None

    def deinit(self) -> None:
        self.__del__()

    def compute(self, edges: Image, box: Rectangle, accumulator) -> None:
        """HoughTransform.compute (hough.zig:75-139): every non-zero pixel of `edges` (an Image(u8)) inside box ∩ image adds one vote per
        angle column to `accumulator`.  box must be size x size and so must the accumulator (DimensionMismatch otherwise)."""
        if not isinstance(edges, Image) or edges.pixfmt != PixFmt.U8:
            raise TypeError("edges must be an Image of pixel type U8")
        acc = _acc_image(accumulator)
        if accumulator.device != edges._t.device:
            raise ValueError(f"accumulator lives on {accumulator.device}, edges on {edges._t.device}")
        e = edges._zb()
        edges._run(lib().zb_hough_compute, self._h, e, int(box.l), int(box.t), int(box.r), int(box.b), acc)

    def find_lines(self, accumulator, threshold: int, angle_nms_thresh: float, radius_nms_thresh: float) -> List[Line]:
        """HoughTransform.findLines (hough.zig:142-204): local maxima with at least `threshold` votes, strongest first, after greedy
        non-maximum suppression (lines closer than both thresholds to a kept one, including the wrap-around at +-90 degrees, are
        dropped)."""
        torch = _torch()
        acc = _acc_image(accumulator)
        dev = accumulator.device
        cap, n = 1024, C.c_uint32(0)
        while True:
            out = (ZbHoughLine * cap)()
            with torch.cuda.device(dev):
                check(lib().zb_hough_find_lines(self._h, acc, int(threshold), C.c_float(angle_nms_thresh), C.c_float(radius_nms_thresh), out,
                                                cap, C.byref(n), torch.cuda.current_stream(dev).cuda_stream))
            if n.value <= cap:
                break
            cap = n.value
        return [Line(o.angle, o.radius, int(o.score), (o.p1x, o.p1y), (o.p2x, o.p2y)) for o in out[:n.value]]
