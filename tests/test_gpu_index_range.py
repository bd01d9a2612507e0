"""Every device entry point that takes a zb_image, on images past the 32-bit index range.

zb_image holds rows and cols as u32 and the stride as u64, so a 1 x 2,200,000,000 gray image is a valid argument, and on an 80 GB
H100 an ordinary allocation.  The kernels index rows, and channel elements or bytes within a row, with int (offsets from the start
are 64-bit), so the entry points that run them refuse an image with 2^31 rows or more, or a row of 2^31 bytes or more, with
Unsupported before any allocation or launch.  Copies and fills move the bytes whatever the shape, and the histogram family counts in
64-bit offsets.
Images whose dimensions are small but whose byte and element offsets pass 2^31 and 2^32 (B4, BF, V) must give the reference's result.

Shape classes (per image):
  W1  1 x (2^31 + 80) u8            cols > INT_MAX                                  2 GiB
  W4  1 x (2^29 + 24) Rgba u8       cols x 4 > INT_MAX, cols < 2^31                 2 GiB
  T1  (2^31 + 80) x 1 u8            rows > INT_MAX                                  2 GiB
  B4  33,000 x 33,000 Rgba u8       more than 2^32 bytes and channel elements      4.4 GB
  BF  23,200 x 23,200 Rgba f32      float element offsets > 2^31                    8.6 GB
  V   a 400 x 32,986 view of a B4 image, starting past byte 2^32, stride 33,000

ENTRY_POINTS has one row per zb_* function of include/zignal_b200.h with a zb_image parameter; a CPU test fails when the header and
the table disagree.  Each cell is "result" (bit-exact with the oracle or with the torch operation), "Unsupported" (refused, output
untouched), the reference's own error for that shape, or "-" (not run); every row with a "-" says why in its `why`, and the CPU
test checks that.  A sentinel fills every output first, so an ok status with an unwritten or partly written output fails.

The samplers (resize, rotate, warp, extract) take NEAREST samples of a random image at positions that span it, up to the last row
(past byte 2^32), and every output pixel is compared with the source pixel it must pick: resize through the host tables' expression
(d + 0.5) * ratio - 0.5 in f32, rotate with cos 0 / sin 1 (a 90-degree turn in exact f32 arithmetic), warp and extract with integer
(or within 0.01 of integer) positions.  Metrics, reductions and fills use inputs with a closed-form answer.

Local filters run on a constant background with random patches at pixel 0, on both sides of 2^31 (and 2^32) elements and bytes, and
at the last pixel; each patch's neighbourhood is compared with the oracle on a crop with the same background and enough margin, and
everything else with one device comparison against the filter of the background.

The guards themselves are checked with data-less descriptors in a child process that sees no device, so a guard that regressed
shows as a status mismatch and never as a launch (test_index_range_guards_without_a_device).

Box blur and sharpen sum through the reference's f32 summed-area table of the whole image, which is exact only while its sums stay
below 2^24; they run on a zero background with the patches in separate rows, where a crop's table gives the same window sums.

Memory: the largest test (BF box blur, in place, with its f32 summed-area table) needs about 18 GB; a test skips, naming what it
needs, when torch.cuda.mem_get_info() reports less free memory.  Cost: the GPU tests of this file (70) ran in 75 s on one H100 80GB
HBM3 at a 700 W power limit, most of it in the two 2 GiB host-pointer refusal sweeps.
"""
import ctypes as C
import math
import re
from pathlib import Path

import numpy as np
import pytest

import zignal_b200 as zb
from zignal_b200.image import ZbImage

HEADER = Path(__file__).resolve().parent.parent / "include" / "zignal_b200.h"
CLASSES = ("W1", "W4", "T1", "B4", "BF", "V")
R, U, N = "result", "Unsupported", "-"
UNSUPPORTED = 3


def _row(W1=N, W4=N, T1=N, B4=N, BF=N, V=N, why=""):
    """One table row; `why` says why each "-" cell is not run (required when there is one)."""
    return {"W1": W1, "W4": W4, "T1": T1, "B4": B4, "BF": BF, "V": V, "why": why}


_GRAY = "W4 / B4 / BF / V are Rgba images: the entry point takes U8 only"
_VIEWS = "V: views of the B4 buffer are run through the samplers, the separable / box / Sobel / Canny filters, convert, flips and copy"
_NO_RGBAF32 = ("BF: not run here; float element offsets past 2^31 are run through the separable, Gaussian, box, convert and copy "
               "BF cases")
_HOST = "host-pointer twins: refused before staging (W1 / T1); their device kernels are the device entry points' own"

ENTRY_POINTS = {
    "zb_set_border_zero": _row(R, N, R, R, why="W4 / BF / V: the same linear and 2-D spans as W1 / T1 / B4"),
    "zb_upload": _row(R, why="one copy routine (zb_copy) for every class; this one reads host memory"),
    "zb_download": _row(R, why="one copy routine (zb_copy) for every class; this one writes host memory"),
    "zb_copy": _row(R, R, R, R, R, R),
    "zb_conv_separable": _row(U, U, U, R, R, R),
    "zb_conv_separable_rows": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_convolve": _row(U, U, U, R, why="BF: no Rgba(f32) form (convolution.zig:295); " + _VIEWS),
    "zb_gaussian_blur": _row(U, U, U, R, R, R),
    "zb_box_blur": _row(U, U, U, R, R, R),
    "zb_sharpen": _row(U, U, U, R, why="BF: the summed-area table of box_blur BF; " + _VIEWS),
    "zb_integral_plane": _row(U, N, U, why=_GRAY + " or F32"),
    "zb_resize": _row(U, U, U, R, why=_NO_RGBAF32, V=R),
    "zb_rotate_into": _row(U, U, U, R, why="B4: the orthogonal kernel (180 degrees); the gather kernel runs through zb_rotate_into_cs; " + _NO_RGBAF32 + "; " + _VIEWS),
    "zb_rotate_into_cs": _row(U, U, U, R, V=R, why=_NO_RGBAF32),
    "zb_rotate_into_batch": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_warp": _row(U, U, U, R, V=R, why=_NO_RGBAF32),
    "zb_sobel": _row(U, U, U, R, N, R, why="BF: no Rgba(f32) form"),
    "zb_canny": _row(U, U, U, N, N, R, why="B4: its f32 planes (5 x 4.4 GB) pass the memory budget, V runs the same kernels; BF: no Rgba(f32) form"),
    "zb_shen_castan": _row(U, U, U, why="B4 / BF / V: the high threshold comes from the whole image's histogram, so no crop has the same answer, "
                                         "and its three f32 summed-area tables are exact only below 2^24"),
    "zb_order_blur": _row(U, U, U, R, why="BF: 8-bit only; " + _VIEWS),
    "zb_motion_blur_linear": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_motion_blur_radial": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_histogram": _row(R, R, R, R, why="BF: 8-bit only; " + _VIEWS),
    "zb_autocontrast": _row(R, N, R, why="W4 / B4 / V: the histogram walk of zb_histogram and the LUT map of W1 / T1; BF: 8-bit only"),
    "zb_equalize": _row(R, N, R, why="W4 / B4 / V: the histogram walk of zb_histogram and the LUT map of W1 / T1; BF: 8-bit only"),
    "zb_threshold_otsu": _row(R, N, R, why=_GRAY),
    "zb_threshold_adaptive_mean": _row(U, N, U, why=_GRAY),
    "zb_morph_binary": _row(U, N, U, why=_GRAY),
    "zb_hough_compute": _row(U, N, U, why=_GRAY),
    "zb_hough_find_lines": _row(why="the accumulator is at most 32,768 x 32,768 u32 (the handle's size); no pixel format"),
    "zb_flood_fill": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_median_cut": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_build_palette": _row(U, U, U, why="B4 / BF / V: the adaptive mode is zb_median_cut"),
    "zb_dither": _row(why="Rgb(u8) only, no class is Rgb; the guard is checked with a 1 x 716,000,000 Rgb descriptor"),
    "zb_palette_lookup": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_convert": _row(U, U, U, R, R, R),
    "zb_psnr": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_ssim": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_mean_pixel_error": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_diff": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_apply_colormap": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_flip_left_right": _row(U, U, U, R, N, R, why="BF: bytes moved whatever the pixel type"),
    "zb_flip_top_bottom": _row(U, U, U, R, why="BF: bytes moved whatever the pixel type; " + _VIEWS),
    "zb_invert": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_extract": _row(U, U, U, R, V=R, why=_NO_RGBAF32),
    "zb_insert": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_insert_blend": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_insert_from": _row(U, U, U, R, why=_NO_RGBAF32 + "; " + _VIEWS),
    "zb_jpeg_encode": _row("ImageTooLarge", "ImageTooLarge", "ImageTooLarge",
                           why="codecs/jpeg.zig:312-314 refuses sides above 65,535; B4 / BF / V: not run (the codec's own limits are tested "
                               "in test_gpu_jpeg.py)"),
    "zb_jpeg_decode": _row(why="the destination's shape is the file's: at most 65,535 per side"),
    "zb_jpeg_decode_batch": _row(why="the destination's shape is the file's: at most 65,535 per side"),
    "zb_fdm_set_target": _row(why="not run: contiguous images, 64-bit pixel counts (zb_fdm.cu moments_kernel / fdm_map_kernel)"),
    "zb_fdm_set_source": _row(why="not run: stores the descriptor only"),
    "zb_fdm_match": _row(why="not run: zb_fdm_set_target + zb_fdm_update"),
    "zb_fdm_moments": _row(why="not run: contiguous images, 64-bit pixel counts"),
    "zb_shard_image_create": _row(why="multi-GPU: needs more than one GPU"),
    "zb_shard_image_block": _row(why="multi-GPU: needs more than one GPU"),
    "zb_shard_view": _row(why="multi-GPU: needs more than one GPU"),
    "zb_shard_fdm_set_target": _row(why="multi-GPU: needs more than one GPU"),
    "zb_host_conv_separable": _row(U, N, U, why=_HOST),
    "zb_host_convolve": _row(U, N, U, why=_HOST),
    "zb_host_gaussian_blur": _row(U, N, U, why=_HOST),
    "zb_host_box_blur": _row(U, N, U, why=_HOST),
    "zb_host_sharpen": _row(U, N, U, why=_HOST),
    "zb_host_resize": _row(U, N, U, why=_HOST),
    "zb_host_rotate_into": _row(U, N, U, why=_HOST),
    "zb_host_warp": _row(U, N, U, why=_HOST),
    "zb_host_fdm_match": _row(why="not run: fdm (64-bit pixel counts) behind the host stage"),
}

W1_COLS = (1 << 31) + 80
W4_COLS = (1 << 29) + 24
T1_ROWS = (1 << 31) + 80
B4_SIDE = 33_000
BF_SIDE = 23_200
V_ROWS, V_COL0 = (32_600, 33_000), 7            # view rows [32,600, 33,000), cols [7, 32,993) of a B4 buffer
CLASS_SHAPE = {"W1": (1, W1_COLS, zb.PixFmt.U8), "W4": (1, W4_COLS, zb.PixFmt.RGBA8), "T1": (T1_ROWS, 1, zb.PixFmt.U8)}


def _header_image_functions():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return {m[1] for m in re.finditer(r"\b(zb_\w+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S) if "zb_image" in m[2]}


def test_entry_point_table_matches_header():
    CALL = _call_table()
    found = _header_image_functions()
    assert found == set(ENTRY_POINTS), (sorted(found - set(ENTRY_POINTS)), sorted(set(ENTRY_POINTS) - found))
    for name, row in ENTRY_POINTS.items():
        assert set(row) == set(CLASSES) | {"why"}, name
        assert row["why"] or N not in (row[c] for c in CLASSES), (name, "a cell is not run and the row gives no reason")
        for cls in CLASSES:
            want = row[cls]
            assert want in (R, U, N) or want == "ImageTooLarge", (name, cls, want)
            if want == U or want == "ImageTooLarge":
                assert name in CALL, (name, cls)
            if want == R:
                assert (name, cls) in RESULT_TESTS, (name, cls)


# ---- one call per entry point, with fixed arguments, for the refusal tests --------------------------------------------------------

_f = C.c_float
_K3 = (C.c_float * 3)(0.25, 0.5, 0.25)
_K9 = (C.c_float * 9)(*([1 / 9] * 9))
_M6 = (C.c_float * 6)(0.5, 0.0, 0.0, 0.5, 1.0, 0.0)
_MORPH = (C.c_uint8 * 9)(*([1] * 9))
_PAL = (C.c_uint8 * 768)()
_LUT768 = (C.c_uint8 * 768)()
_COUNTS = (C.c_uint32 * 1024)()
_FILL = (C.c_uint8 * 16)()


def _call_table():
    L = zb.lib()
    n, d = C.c_uint32(), C.c_double()
    jl = C.c_uint64()
    opts, _ = zb.image._jpeg_options(90, 2, 72, None)

    def hough(s, dd, fmt, ext):
        h = C.c_void_p()
        assert L.zb_hough_create(64, None, None, C.byref(h)) == 0
        acc = ZbImage(ext.get("acc"), 64, 64, 64)
        try:
            return L.zb_hough_compute(h, s, 0, 0, 64, 64, acc, None)
        finally:
            L.zb_hough_destroy(h)

    return {
        "zb_conv_separable": lambda s, dd, fmt, ext: L.zb_conv_separable(s, dd, fmt, _K3, 3, _K3, 3, 2, None),
        "zb_conv_separable_rows": lambda s, dd, fmt, ext: L.zb_conv_separable_rows(s, dd, fmt, _K3, 3, _K3, 3, 2, 0, 0, None),
        "zb_convolve": lambda s, dd, fmt, ext: L.zb_convolve(s, dd, fmt, _K9, 3, 3, 2, None),
        "zb_gaussian_blur": lambda s, dd, fmt, ext: L.zb_gaussian_blur(s, dd, fmt, _f(1.0), None),
        "zb_box_blur": lambda s, dd, fmt, ext: L.zb_box_blur(s, dd, fmt, 2, None),
        "zb_sharpen": lambda s, dd, fmt, ext: L.zb_sharpen(s, dd, fmt, 2, None),
        "zb_integral_plane": lambda s, dd, fmt, ext: L.zb_integral_plane(s, fmt, C.cast(ext.get("sat"), C.POINTER(C.c_float)), None),
        "zb_resize": lambda s, dd, fmt, ext: L.zb_resize(s, ext["small"], fmt, 1, _f(0), _f(0), None),
        "zb_rotate_into": lambda s, dd, fmt, ext: L.zb_rotate_into(s, dd, fmt, _f(0.3), 1, _f(0), _f(0), 1, None),
        "zb_rotate_into_cs": lambda s, dd, fmt, ext: L.zb_rotate_into_cs(s, dd, fmt, _f(0.3), _f(np.cos(0.3)), _f(np.sin(0.3)), 1, _f(0),
                                                                         _f(0), 1, None),
        "zb_rotate_into_batch": lambda s, dd, fmt, ext: L.zb_rotate_into_batch(s, 0, dd, 0, 1, fmt, _f(0.3), _f(np.cos(0.3)),
                                                                               _f(np.sin(0.3)), 1, _f(0), _f(0), 1, None),
        "zb_warp": lambda s, dd, fmt, ext: L.zb_warp(s, dd, fmt, 1, _M6, 1, _f(0), _f(0), None),
        "zb_sobel": lambda s, dd, fmt, ext: L.zb_sobel(s, ext["dst_u8"], fmt, None),
        "zb_canny": lambda s, dd, fmt, ext: L.zb_canny(s, ext["dst_u8"], fmt, _f(1.0), _f(20.0), _f(60.0), None),
        "zb_shen_castan": lambda s, dd, fmt, ext: L.zb_shen_castan(s, ext["dst_u8"], fmt, _f(0.9), 7, _f(0.99), _f(0.5), 1, 0, None),
        "zb_order_blur": lambda s, dd, fmt, ext: L.zb_order_blur(s, dd, fmt, 1, 0, 0.5, 2, None),
        "zb_motion_blur_linear": lambda s, dd, fmt, ext: L.zb_motion_blur_linear(s, dd, fmt, _f(0.7), _f(np.cos(0.7)), _f(np.sin(0.7)), 5,
                                                                                 None),
        "zb_motion_blur_radial": lambda s, dd, fmt, ext: L.zb_motion_blur_radial(s, dd, fmt, _f(0.5), _f(0.5), _f(0.3), 0, None),
        "zb_threshold_adaptive_mean": lambda s, dd, fmt, ext: L.zb_threshold_adaptive_mean(s, dd, 2, _f(1.0), None),
        "zb_morph_binary": lambda s, dd, fmt, ext: L.zb_morph_binary(s, dd, _MORPH, 3, 3, 1, 0, None),
        "zb_hough_compute": hough,
        "zb_flood_fill": lambda s, dd, fmt, ext: L.zb_flood_fill(s, fmt, 0, 0, _FILL, 10.0, 4, 0, None),
        "zb_median_cut": lambda s, dd, fmt, ext: L.zb_median_cut(s, fmt, 16, _PAL, 256, C.byref(n), None),
        "zb_build_palette": lambda s, dd, fmt, ext: L.zb_build_palette(s, fmt, 3, 16, _PAL, C.byref(n), None),
        "zb_palette_lookup": lambda s, dd, fmt, ext: L.zb_palette_lookup(s, fmt, ext.get("lut"), ext["dst_u8"], None),
        "zb_convert": lambda s, dd, fmt, ext: L.zb_convert(s, fmt, ext["dst_f32"], 1, None),
        "zb_psnr": lambda s, dd, fmt, ext: L.zb_psnr(s, dd, fmt, C.byref(d), None),
        "zb_ssim": lambda s, dd, fmt, ext: L.zb_ssim(s, dd, fmt, C.byref(d), None),
        "zb_mean_pixel_error": lambda s, dd, fmt, ext: L.zb_mean_pixel_error(s, dd, fmt, C.byref(d), None),
        "zb_diff": lambda s, dd, fmt, ext: L.zb_diff(s, s, dd, fmt, _f(0), _f(1), 0, 0, None, None),
        "zb_apply_colormap": lambda s, dd, fmt, ext: L.zb_apply_colormap(s, fmt, _LUT768, 0, 0.0, 0, 0.0, ext["dst_rgb8"], None),
        "zb_flip_left_right": lambda s, dd, fmt, ext: L.zb_flip_left_right(s, fmt, None),
        "zb_flip_top_bottom": lambda s, dd, fmt, ext: L.zb_flip_top_bottom(s, fmt, None),
        "zb_invert": lambda s, dd, fmt, ext: L.zb_invert(s, fmt, None),
        "zb_extract": lambda s, dd, fmt, ext: L.zb_extract(s, dd, fmt, _f(0), _f(0), _f(4), _f(1), _f(0), _f(1), _f(0), 1, _f(0), _f(0), 2,
                                                           None),
        "zb_insert": lambda s, dd, fmt, ext: L.zb_insert(s, ext["small"], fmt, _f(0), _f(0), _f(4), _f(1), _f(0), _f(1), _f(0), 1, _f(0),
                                                         _f(0), None),
        "zb_insert_blend": lambda s, dd, fmt, ext: L.zb_insert_blend(s, ext["small"], fmt, _f(0), _f(0), _f(4), _f(1), _f(0), _f(1), _f(0),
                                                                     1, _f(0), _f(0), 1, None),
        "zb_insert_from": lambda s, dd, fmt, ext: L.zb_insert_from(s, fmt, ext["small_f32"], 1, _f(0), _f(0), _f(4), _f(1), _f(0), _f(1),
                                                                   _f(0), 1, _f(0), _f(0), 0, None),
        "zb_jpeg_encode": lambda s, dd, fmt, ext: L.zb_jpeg_encode(s, fmt, C.byref(opts), None, 0, C.byref(jl), None),
        "zb_host_conv_separable": lambda s, dd, fmt, ext: L.zb_host_conv_separable(s, dd, fmt, _K3, 3, _K3, 3, 2),
        "zb_host_convolve": lambda s, dd, fmt, ext: L.zb_host_convolve(s, dd, fmt, _K9, 3, 3, 2),
        "zb_host_gaussian_blur": lambda s, dd, fmt, ext: L.zb_host_gaussian_blur(s, dd, fmt, _f(1.0)),
        "zb_host_box_blur": lambda s, dd, fmt, ext: L.zb_host_box_blur(s, dd, fmt, 2),
        "zb_host_sharpen": lambda s, dd, fmt, ext: L.zb_host_sharpen(s, dd, fmt, 2),
        "zb_host_resize": lambda s, dd, fmt, ext: L.zb_host_resize(s, ext["small"], fmt, 1, _f(0), _f(0)),
        "zb_host_rotate_into": lambda s, dd, fmt, ext: L.zb_host_rotate_into(s, dd, fmt, _f(0.3), 1, _f(0), _f(0), 1),
        "zb_host_warp": lambda s, dd, fmt, ext: L.zb_host_warp(s, dd, fmt, 1, _M6, 1, _f(0), _f(0)),
    }


EXPECTED_STATUS = {U: UNSUPPORTED, "ImageTooLarge": 30}


def _refusals(cls):
    return [name for name, row in ENTRY_POINTS.items() if row[cls] in EXPECTED_STATUS]


def _guard_statuses():
    """(name, class, got, want) for every refusal cell, on data-less descriptors, plus the guards no class reaches: dither (Rgb only)
    and a row of 2^31 bytes or more in Rgba(f32) whose cols x channels is still below 2^31."""
    table = _call_table()
    L = zb.lib()
    fake = 1 << 40      # never dereferenced: the guard returns first, and the calls run where no device is visible
    out = []
    for cls in ("W1", "W4", "T1"):
        rows, cols, fmt = CLASS_SHAPE[cls]
        for name in _refusals(cls):
            s, dd = ZbImage(fake, rows, cols, cols), ZbImage(fake << 1, rows, cols, cols)   # apart: row windows refuse overlaps first
            ext = {"small": ZbImage(fake, 4, 4, 4), "small_f32": ZbImage(fake, 4, 4, 4), "dst_u8": ZbImage(fake << 1, rows, cols, cols),
                   "dst_f32": ZbImage(fake << 1, rows, cols, cols), "dst_rgb8": ZbImage(fake << 1, rows, cols, cols), "lut": fake,
                   "sat": fake, "acc": fake}
            out.append((name, cls, table[name](s, dd, int(fmt), ext), EXPECTED_STATUS[ENTRY_POINTS[name][cls]]))
    rgb = ZbImage(fake, 1, 716_000_000, 716_000_000)                                   # 2,148,000,000 bytes
    out.append(("zb_dither", "1 x 716,000,000 Rgb", L.zb_dither(rgb, int(zb.PixFmt.RGB8), _PAL, 16, fake, 3, None), UNSUPPORTED))
    out.append(("zb_dither NONE", "1 x 716,000,000 Rgb", L.zb_dither(rgb, int(zb.PixFmt.RGB8), _PAL, 16, fake, 0, None), 0))
    wf = (1 << 27) + 8                                                                 # 16 B pixels: 2^31 + 128 bytes, 2^29 + 32 floats
    s, dd = ZbImage(fake, 1, wf, wf), ZbImage(fake << 1, 1, wf, wf)
    f4 = int(zb.PixFmt.RGBAF32)
    out.append(("zb_conv_separable", "1 x (2^27 + 8) Rgba(f32)", table["zb_conv_separable"](s, dd, f4, {}), UNSUPPORTED))
    out.append(("zb_resize", "1 x (2^27 + 8) Rgba(f32)", L.zb_resize(ZbImage(fake, 0, 0, 0), dd, f4, 1, _f(0), _f(0), None), UNSUPPORTED))
    out.append(("zb_extract", "1 x (2^27 + 8) Rgba(f32)", table["zb_extract"](ZbImage(fake, 0, 0, 0), dd, f4, {}), UNSUPPORTED))
    return out


def test_index_range_guards_without_a_device():
    """The refusals are decided before any device work.  The calls run in a child process that sees no device, so a guard that
    regressed fails with a status mismatch and can never launch a kernel."""
    import json
    import os
    import subprocess
    import sys
    here = Path(__file__).resolve().parent
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="",
               PYTHONPATH=os.pathsep.join([str(here.parent), str(here), os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_index_range as t; print(json.dumps(t._guard_statuses()))"
    res = subprocess.run([sys.executable, "-s", "-c", code], cwd=here, env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr[-2000:]
    rows = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(rows) > 100
    bad = [r for r in rows if r[2] != r[3]]
    assert not bad, bad


# ---- device helpers ---------------------------------------------------------------------------------------------------------------

GiB = 1 << 30
_CHUNK = 1 << 28      # elements per chunk of the device comparisons (keeps their temporaries small)


@pytest.fixture
def torch_dev():
    import torch
    assert torch.cuda.is_available()
    yield torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _need(torch, nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")


def _all_equal(t, value):
    """Every element of the (possibly strided) tensor t equals value; compared in chunks of rows."""
    if t.dim() == 1:
        t = t.view(1, -1)
    per = max(1, _CHUNK // max(1, t[0].numel()))
    for r in range(0, t.shape[0], per):
        part = t[r:r + per]
        if part.dim() >= 2 and part.shape[0] == 1 and part[0].numel() > _CHUNK:
            flat = part.reshape(-1)
            for k in range(0, flat.numel(), _CHUNK):
                if not bool((flat[k:k + _CHUNK] == value).all()):
                    return False
        elif not bool((part == value).all()):
            return False
    return True


def _zbi(t, rows, cols, stride=None):
    return ZbImage(t.data_ptr(), rows, cols, cols if stride is None else stride)


# ---- W1 / W4 / T1: refusals -------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("cls", ["W1", "W4", "T1"])
def test_wide_and_tall_refusals_leave_every_buffer_untouched(torch_dev, cls):
    torch = torch_dev
    rows, cols, fmt = CLASS_SHAPE[cls]
    ch = 4 if fmt == zb.PixFmt.RGBA8 else 1
    n_px = rows * cols
    _need(torch, n_px * ch + n_px * 4 + 64 * 1024 * 1024)
    src = torch.full((n_px * ch,), 0x3C, dtype=torch.uint8, device="cuda")
    dst = torch.full((n_px * 4,), 0xA5, dtype=torch.uint8, device="cuda")   # room for an f32 plane of the shape
    small = torch.full((4 * 4 * ch,), 0x11, dtype=torch.uint8, device="cuda")
    small_f32 = torch.full((16,), 0.5, dtype=torch.float32, device="cuda")
    lut = torch.zeros(32768, dtype=torch.uint8, device="cuda")
    acc = torch.zeros(64 * 64, dtype=torch.int32, device="cuda")
    table = _call_table()
    host_src = host_dst = None
    for name in _refusals(cls):
        if name.startswith("zb_host_"):
            if host_src is None:
                host_src = np.full(n_px * ch, 0x3C, np.uint8)
                host_dst = np.full(n_px * ch, 0xA5, np.uint8)
            s, d = ZbImage(host_src.ctypes.data, rows, cols, cols), ZbImage(host_dst.ctypes.data, rows, cols, cols)
            small_h = np.full(16 * ch, 0x11, np.uint8)
            ext = {"small": ZbImage(small_h.ctypes.data, 4, 4, 4)}
        else:
            s, d = _zbi(src, rows, cols), _zbi(dst, rows, cols)
            ext = {"small": _zbi(small, 4, 4), "small_f32": _zbi(small_f32, 4, 4), "dst_u8": d, "dst_f32": d, "dst_rgb8": d,
                   "lut": lut.data_ptr(), "sat": dst.data_ptr(), "acc": acc.data_ptr()}
        got = table[name](s, d, int(fmt), ext)
        torch.cuda.synchronize()
        assert got == EXPECTED_STATUS[ENTRY_POINTS[name][cls]], (name, cls, got)
        assert _all_equal(src, 0x3C) and _all_equal(dst, 0xA5), (name, cls, "written")
        assert _all_equal(small, 0x11) and _all_equal(acc, 0), (name, cls, "written")
        if host_src is not None:
            assert (host_src == 0x3C).all() and (host_dst == 0xA5).all(), (name, cls, "host buffer written")


# ---- W1 / W4 / T1: results --------------------------------------------------------------------------------------------------------

def _marked(torch, n, seed):
    """A device u8 vector of n bytes: 0x3C everywhere, distinct bytes at 0, around 2^31 and at the end."""
    t = torch.full((n,), 0x3C, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(seed)
    spots = {}
    for p in (0, 1, (1 << 31) - 2, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, n - 2, n - 1):
        if 0 <= p < n:
            spots[p] = int(rng.integers(0, 256))
            t[p] = spots[p]
    return t, spots


def _copy_family(torch, cls):
    rows, cols, fmt = CLASS_SHAPE[cls]
    ch = 4 if fmt == zb.PixFmt.RGBA8 else 1
    n = rows * cols * ch
    _need(torch, 2 * n + GiB)
    L = zb.lib()
    src, spots = _marked(torch, n, 1)
    dst = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
    assert L.zb_copy(_zbi(src, rows, cols), _zbi(dst, rows, cols), int(fmt), None) == 0
    assert torch.equal(src, dst)
    return L, rows, cols, fmt, src, dst, spots


def _test_copy(torch, cls):
    _copy_family(torch, cls)


def _test_set_border_zero(torch, cls):
    L, rows, cols, fmt, src, dst, spots = _copy_family(torch, cls)
    n = dst.numel()
    if cls == "W1":     # keep columns [5, cols - 7): zero 5 on the left, 7 on the right
        assert L.zb_set_border_zero(_zbi(dst, rows, cols), int(fmt), 5, 0, cols - 7, 1, None) == 0
        want = src.clone()
        want[:5] = 0
        want[n - 7:] = 0
    else:               # T1: keep rows [3, rows - 9)
        assert L.zb_set_border_zero(_zbi(dst, rows, cols), int(fmt), 0, 3, 1, rows - 9, None) == 0
        want = src.clone()
        want[:3] = 0
        want[n - 9:] = 0
    assert torch.equal(dst, want)


def _test_upload_download(torch, cls):
    rows, cols, fmt = CLASS_SHAPE[cls]
    n = rows * cols
    _need(torch, n + GiB)
    L = zb.lib()
    host = np.full(n, 0x3C, np.uint8)
    for p, v in ((0, 7), ((1 << 31) - 1, 8), (1 << 31, 9), (n - 1, 10)):
        host[p] = v
    dev = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
    assert L.zb_upload(ZbImage(host.ctypes.data, rows, cols, cols), _zbi(dev, rows, cols), int(fmt), None) == 0
    torch.cuda.synchronize()
    for p in (0, (1 << 31) - 1, 1 << 31, n - 1):
        assert int(dev[p]) == host[p], p
    assert int((dev != 0x3C).sum()) == 4
    back = np.full(n, 0xA5, np.uint8)
    assert L.zb_download(_zbi(dev, rows, cols), ZbImage(back.ctypes.data, rows, cols, cols), int(fmt), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(back, host)


def _test_histogram(torch, cls):
    rows, cols, fmt = CLASS_SHAPE[cls]
    ch = 4 if fmt == zb.PixFmt.RGBA8 else 1
    n = rows * cols * ch
    _need(torch, n + GiB)
    src, spots = _marked(torch, n, 2)
    counts = (C.c_uint32 * 1024)()
    assert zb.lib().zb_histogram(_zbi(src, rows, cols), int(fmt), counts, None) == 0
    want = np.zeros((ch, 256), np.int64)
    want[:, 0x3C] = n // ch
    for p, v in spots.items():
        want[p % ch, 0x3C] -= 1
        want[p % ch, v] += 1
    assert np.array_equal(np.array(counts[:ch * 256], np.int64).reshape(ch, 256), want)


def _test_enhance(torch, cls, mode):
    """equalize / autocontrast in place (histogram, then the LUT map of every byte) against their LUTs computed here from the counts:
    enhancement.zig:84-252 with the 64-bit numerator, and :11-80 with cutoff 0 (min / max of the values present)."""
    rows, cols, fmt = CLASS_SHAPE[cls]
    n = rows * cols
    _need(torch, 2 * n + GiB)
    src, spots = _marked(torch, n, 3)
    counts = np.zeros(256, np.int64)
    counts[0x3C] = n - len(spots)
    for v in spots.values():
        counts[v] += 1
    orig = src.clone()
    L = zb.lib()
    if mode == "equalize":
        assert L.zb_equalize(_zbi(src, rows, cols), int(fmt), None) == 0
        cdf = np.cumsum(counts)
        cmin = int(cdf[np.nonzero(cdf)[0][0]])
        lut = np.where(cdf >= cmin, (cdf - cmin) * 255 // (n - cmin), 0)
    else:
        assert L.zb_autocontrast(_zbi(src, rows, cols), int(fmt), _f(0.0), None) == 0
        present = np.nonzero(counts)[0]
        mn, mx = int(present[0]), int(present[-1])
        v = np.clip(np.arange(256), mn, mx)
        norm = (v - mn).astype(np.float32) / np.float32(max(mx - mn, 1))
        lut = np.floor((norm * np.float32(255)).astype(np.float64) + 0.5)
    torch.cuda.synchronize()
    lut_t = torch.from_numpy(lut.astype(np.uint8)).to("cuda")
    for k in range(0, n, _CHUNK):
        assert torch_equal(src[k:k + _CHUNK], lut_t[orig[k:k + _CHUNK].long()]), (mode, k)


def _test_otsu(torch, cls):
    """Two values, 0x3C and 200: every threshold in [0x3C, 200) separates them, so dst is 255 exactly at the 200s."""
    rows, cols, fmt = CLASS_SHAPE[cls]
    n = rows * cols
    _need(torch, 2 * n + GiB)
    src = torch.full((n,), 0x3C, dtype=torch.uint8, device="cuda")
    spots = [0, (1 << 31) - 1, 1 << 31, n - 1]
    for q in spots:
        src[q] = 200
    dst = torch.full_like(src, 0xA5)
    t = C.c_uint8(0)
    assert zb.lib().zb_threshold_otsu(_zbi(src, rows, cols), _zbi(dst, rows, cols), C.byref(t), None) == 0
    torch.cuda.synchronize()
    assert 0x3C <= t.value < 200
    for q in spots:
        assert int(dst[q]) == 255
        dst[q] = 0
    assert _all_equal(dst, 0)


# ---- B4 / BF / V: local filters against the oracle on crops ----------------------------------------------------------------------

def _geometry(cls):
    """(buffer rows, buffer cols, view top, view left, view rows, view cols, pixfmt, patch centres in view coordinates)."""
    if cls == "B4":
        n = B4_SIDE * B4_SIDE
        cen = [divmod(p, B4_SIDE) for p in (0, 1 << 29, 1 << 30, n - 1)]                      # 2^31 / 2^32 elements and bytes
        return B4_SIDE, B4_SIDE, 0, 0, B4_SIDE, B4_SIDE, zb.PixFmt.RGBA8, cen
    if cls == "BF":
        n = BF_SIDE * BF_SIDE
        cen = [divmod(p, BF_SIDE) for p in (0, 1 << 27, 1 << 28, 1 << 29, n - 1)]             # bytes 2^31, 2^32; elements 2^31
        return BF_SIDE, BF_SIDE, 0, 0, BF_SIDE, BF_SIDE, zb.PixFmt.RGBAF32, cen
    vr, vc = V_ROWS[1] - V_ROWS[0], B4_SIDE - 2 * V_COL0
    return B4_SIDE, B4_SIDE, V_ROWS[0], V_COL0, vr, vc, zb.PixFmt.RGBA8, [(0, 0), (vr // 2, vc // 2), (vr - 1, vc - 1)]


def _run_local(torch, cls, call, oracle, reach, bg, out_fmt=None, in_place=False, float_patch=False):
    """call(src_image, dst_image) on a constant-`bg` image with random 5 x 5 patches; see the module docstring."""
    import oracle_lib  # noqa: F401  (the oracle library must be built)
    brows, bcols, top, left, rows, cols, fmt, centres = _geometry(cls)
    out_fmt = fmt if out_fmt is None else out_fmt
    flt = fmt == zb.PixFmt.RGBAF32
    dt = torch.float32 if flt else torch.uint8
    odt = torch.float32 if out_fmt in (zb.PixFmt.F32, zb.PixFmt.RGBAF32) else torch.uint8
    och = {zb.PixFmt.U8: 1, zb.PixFmt.F32: 1, zb.PixFmt.RGB8: 3}.get(out_fmt, 4)
    esz = 4 if flt else 1
    _need(torch, brows * bcols * 4 * esz * (1 if in_place else 2) + (brows * bcols * 16 if flt and in_place else 0) + GiB)
    sentinel = -7.5 if odt == torch.float32 else 0xA5
    sbuf = torch.full((brows, bcols, 4), bg, dtype=dt, device="cuda")
    src = sbuf[top:top + rows, left:left + cols]
    rng = np.random.default_rng(CLASSES.index(cls))
    for r, c in centres:
        r0, r1, c0, c1 = max(0, r - 2), min(rows, r + 3), max(0, c - 2), min(cols, c + 3)
        if float_patch:
            vals = rng.integers(0, 16, (r1 - r0, c1 - c0, 4)).astype(np.float32) / 16
        else:
            vals = rng.integers(0, 256, (r1 - r0, c1 - c0, 4)).astype(np.uint8)
        src[r0:r1, c0:c1] = torch.from_numpy(vals).to("cuda")
    windows = []
    for r, c in centres:        # compared window W and the crop (W plus reach) the oracle sees, clipped to the view
        w = (max(0, r - 2 - reach), min(rows, r + 3 + reach), max(0, c - 2 - reach), min(cols, c + 3 + reach))
        k = (max(0, w[0] - reach), min(rows, w[1] + reach), max(0, w[2] - reach), min(cols, w[3] + reach))
        windows.append((w, k, src[k[0]:k[1], k[2]:k[3]].cpu().numpy()))
    if in_place:
        dbuf, dst = sbuf, src
    else:
        dbuf = torch.full((brows, bcols, och) if och > 1 else (brows, bcols), sentinel, dtype=odt, device="cuda")
        dst = dbuf[top:top + rows, left:left + cols]
    si = zb.Image(sbuf.view(-1), fmt, rows, cols, bcols, top * bcols + left)
    di = zb.Image(dbuf.view(-1), out_fmt, rows, cols, bcols, top * bcols + left)
    call(si, di)
    torch.cuda.synchronize()
    side = 4 * reach + 9
    bg_img = np.full((side, side, 4), bg, np.float32 if flt else np.uint8)
    bg_out = oracle(bg_img)[side // 2, side // 2]
    for (w, k, crop) in windows:
        want = oracle(crop)[w[0] - k[0]:w[1] - k[0], w[2] - k[2]:w[3] - k[2]]
        got = dst[w[0]:w[1], w[2]:w[3]].cpu().numpy()
        assert np.array_equal(got, want), (cls, w, np.argwhere(got != want)[:4].tolist())
        dst[w[0]:w[1], w[2]:w[3]] = torch.from_numpy(np.broadcast_to(bg_out, got.shape).copy()).to("cuda")
    bg_t = torch.from_numpy(np.asarray(bg_out).reshape(-1)).to("cuda")
    per = max(1, _CHUNK // (cols * och))
    for r in range(0, rows, per):
        part = dst[r:r + per]
        assert bool((part == (bg_t if och > 1 else bg_t[0])).all()), (cls, "rows", r, r + per)
    if cls == "V":      # nothing outside the view was written
        dst[:] = sentinel
        assert _all_equal(dbuf, sentinel)


def _exact_f32(fn):
    def run(si, di):
        L = zb.lib()
        L.zb_set_exact_f32(1)
        try:
            fn(si, di)
        finally:
            L.zb_set_exact_f32(0)
    return run


def _local_case(name, cls, torch):
    import oracle_lib as zo
    K3 = np.array([0.25, 0.5, 0.25], np.float32)
    K33 = np.array([[1, 2, 1], [0, 3, -1], [1, -2, 2]], np.float32) / 7
    M = zb.BorderMode.MIRROR
    flt = cls == "BF"
    bg = 0.0 if flt else 77
    cases = {
        "zb_conv_separable": (_exact_f32(lambda s, d: s.convolve_separable(K3, K3, M, out=d)),
                              lambda a: zo.conv_separable(a, K3, K3, "mirror"), 1, {}),
        "zb_gaussian_blur": (_exact_f32(lambda s, d: s.gaussian_blur(1.0, out=d)), lambda a: zo.gaussian_blur(a, 1.0), 3, {}),
        "zb_convolve": (lambda s, d: s.convolve(K33, M, out=d), lambda a: zo.convolve(a, K33, "mirror"), 1, {}),
        # the reference sums through an f32 summed-area table of the whole image, exact only while its sums stay below 2^24: a zero
        # background with the patches in separate rows keeps them there, so a crop's table gives the same window sums
        "zb_box_blur": (lambda s, d: s.box_blur(2, out=d), lambda a: zo.box_blur(a, 2), 2, {"in_place": flt, "bg": 0}),
        "zb_sharpen": (lambda s, d: s.sharpen(2, out=d), lambda a: zo.sharpen(a, 2), 2, {"bg": 0}),
        "zb_order_blur": (lambda s, d: s.median_blur(1, out=d), lambda a: zo.order_blur(a, 1, "percentile", 0.5, "mirror"), 1, {}),
        "zb_sobel": (lambda s, d: s.sobel(out=d), zo.sobel, 1, {"out_fmt": zb.PixFmt.U8}),
        "zb_canny": (lambda s, d: s.canny(1.0, 20.0, 60.0, out=d), lambda a: zo.canny(a, 1.0, 20.0, 60.0), 8, {"out_fmt": zb.PixFmt.U8}),
        # cos / sin cross the ABI as data: 0.5 / 0.75 make every sample position c + t cos, r + t sin exact in f32 at any column, so
        # a crop samples at the same fractions as the whole image (with a rounded cos / sin they differ in the last bits far out)
        "zb_motion_blur_linear": (_motion, lambda a: zo.motion_blur_linear(a, 0.0, 5, cos_sin=(np.float32(0.5), np.float32(0.75))), 6, {}),
        "zb_convert": ((lambda s, d: s.convert(zb.PixFmt.RGBA8, out=d)) if flt else (lambda s, d: s.convert(zb.PixFmt.U8, out=d)),
                       (lambda a: zo.convert(a, zo.PIX_RGBA8)) if flt else (lambda a: zo.convert(a, zo.PIX_U8)), 0,
                       {"out_fmt": zb.PixFmt.RGBA8 if flt else zb.PixFmt.U8}),
    }
    call, oracle, reach, kw = cases[name]
    kw = dict(kw)
    _run_local(torch, cls, call, oracle, reach, kw.pop("bg", bg), float_patch=flt, **kw)


def _motion(s, d):
    assert 0 == (zb.lib().zb_motion_blur_linear(s._zb(), d._zb(), int(s.pixfmt), _f(0.0), _f(0.5), _f(0.75), 5, None))


# ---- B4 / V: operations checked against torch -------------------------------------------------------------------------------------

def _b4(torch, cls, extra=1):
    brows, bcols, top, left, rows, cols, fmt, centres = _geometry(cls)
    _need(torch, brows * bcols * 4 * (1 + extra) + GiB)
    g = torch.Generator(device="cuda").manual_seed(5)
    buf = torch.randint(0, 256, (brows, bcols, 4), dtype=torch.uint8, device="cuda", generator=g)
    view = buf[top:top + rows, left:left + cols]
    img = zb.Image(buf.view(-1), fmt, rows, cols, bcols, top * bcols + left)
    return buf, view, img


def _equal_rows(a, b):
    per = max(1, _CHUNK // a[0].numel())
    return all(torch_equal(a[r:r + per], b[r:r + per]) for r in range(0, a.shape[0], per))


def torch_equal(a, b):
    return bool((a == b).all())


def _torch_case(name, cls, torch):
    M = zb.BorderMode
    if name == "zb_copy":
        if cls == "BF":
            _need(torch, 2 * BF_SIDE * BF_SIDE * 16 + GiB)
            a = torch.rand((BF_SIDE, BF_SIDE, 4), device="cuda")
            b = torch.full_like(a, -7.5)
            zb.Image(a.view(-1), zb.PixFmt.RGBAF32, BF_SIDE, BF_SIDE, BF_SIDE).copy(zb.Image(b.view(-1), zb.PixFmt.RGBAF32, BF_SIDE, BF_SIDE, BF_SIDE))
            assert _equal_rows(a, b)
            return
        buf, view, img = _b4(torch, cls)
        out = torch.full_like(buf, 0xA5)
        oimg = zb.Image(out.view(-1), img.pixfmt, img.rows, img.cols, img.stride, img._off)
        img.copy(oimg)
        brows, bcols, top, left, rows, cols, fmt, _ = _geometry(cls)
        assert _equal_rows(out[top:top + rows, left:left + cols], view)
        out[top:top + rows, left:left + cols] = 0xA5
        assert _all_equal(out, 0xA5)
        return
    buf, view, img = _b4(torch, cls)
    if name == "zb_set_border_zero":
        want = view.clone()
        L = zb.lib()
        l, t, r, b = 1000, 2000, B4_SIDE - 3, B4_SIDE - 5
        assert L.zb_set_border_zero(img._zb(), int(img.pixfmt), l, t, r, b, None) == 0
        want[:t] = 0; want[b:] = 0; want[:, :l] = 0; want[:, r:] = 0
        assert _equal_rows(view, want)
    elif name == "zb_flip_left_right":
        want = view.flip(1)
        img.flip_left_right()
        assert _equal_rows(view, want)
    elif name == "zb_flip_top_bottom":
        want = view.flip(0)
        img.flip_top_bottom()
        assert _equal_rows(view, want)
    elif name == "zb_invert":
        want = view.clone()
        want[..., :3] = 255 - want[..., :3]
        img.invert()
        assert _equal_rows(view, want)
    elif name == "zb_diff":
        _need(torch, 3 * B4_SIDE * B4_SIDE * 4 + 2 * GiB)
        other = view.clone()
        other[B4_SIDE // 2:] = 255 - other[B4_SIDE // 2:]
        oimg = zb.Image(other.view(-1), img.pixfmt, img.rows, img.cols, img.cols)
        out = torch.full_like(other, 0xA5)
        img.diff(oimg, out=zb.Image(out.view(-1), img.pixfmt, img.rows, img.cols, img.cols))
        per = max(1, _CHUNK // view[0].numel())
        for r in range(0, view.shape[0], per):
            want = (view[r:r + per].to(torch.int16) - other[r:r + per].to(torch.int16)).abs().to(torch.uint8)
            assert torch_equal(out[r:r + per], want), r
    elif name in ("zb_psnr", "zb_mean_pixel_error"):
        view.fill_(100)
        other = torch.full_like(view, 100)
        other[(1 << 29) // B4_SIDE, (1 << 29) % B4_SIDE] = torch.tensor([100, 103, 96, 101], dtype=torch.uint8)
        other[-1, -1, 2] = 0
        oimg = zb.Image(other.view(-1), img.pixfmt, img.rows, img.cols, img.cols)
        n = B4_SIDE * B4_SIDE * 4
        if name == "zb_psnr":
            mse = (9 + 16 + 1 + 100 * 100) / n
            assert img.psnr(oimg) == 20.0 * math.log10(255.0) - 10.0 * math.log10(mse)
        else:
            assert img.mean_pixel_error(oimg) == ((3 + 4 + 1 + 100) / n) / 255.0
    elif name == "zb_histogram":
        view.fill_(9)
        view[(1 << 30) // B4_SIDE, (1 << 30) % B4_SIDE] = torch.tensor([1, 2, 3, 4], dtype=torch.uint8)
        h = img.histogram()
        want = np.zeros((4, 256), np.int64)
        want[:, 9] = B4_SIDE * B4_SIDE - 1
        want[[0, 1, 2, 3], [1, 2, 3, 4]] = 1
        assert np.array_equal(np.asarray(h, np.int64).reshape(4, 256), want)
    elif name in ("zb_resize", "zb_rotate_into", "zb_rotate_into_cs", "zb_rotate_into_batch", "zb_warp", "zb_extract"):
        _sampler_case(torch, name, cls, view, img)
    elif name == "zb_insert":
        src = torch.randint(0, 256, (300, 500, 4), dtype=torch.uint8, device="cuda")
        r0, c0 = B4_SIDE - 300, B4_SIDE - 500
        above, left = view[r0 - 3:r0].clone(), view[r0:, c0 - 3:c0].clone()
        img.insert(zb.Image(src.view(-1), img.pixfmt, 300, 500, 500), (c0, r0, B4_SIDE, B4_SIDE), 0.0, zb.Interpolation.NEAREST)
        assert torch_equal(view[r0:, c0:], src)
        assert torch_equal(view[r0 - 3:r0], above) and torch_equal(view[r0:, c0 - 3:c0], left)   # nothing outside the rectangle
    elif name == "zb_insert_blend":      # an opaque source with the normal blend: dest = source (blending.zig:26-156, alpha 1)
        src = torch.randint(0, 256, (300, 500, 4), dtype=torch.uint8, device="cuda")
        src[..., 3] = 255
        r0, c0 = B4_SIDE - 300, B4_SIDE - 500
        assert zb.lib().zb_insert_blend(img._zb(), _zbi(src, 300, 500), int(img.pixfmt), _f(c0), _f(r0), _f(B4_SIDE), _f(B4_SIDE), _f(0),
                                        _f(1), _f(0), int(zb.Interpolation.NEAREST), _f(0), _f(0), int(zb.Blending.NORMAL), None) == 0
        torch.cuda.synchronize()
        assert torch_equal(view[r0:, c0:], src)
    elif name == "zb_insert_from":       # a gray u8 source into the Rgba(u8) image: (v, v, v, 255) (color.zig:355)
        src = torch.randint(0, 256, (300, 500), dtype=torch.uint8, device="cuda")
        r0, c0 = B4_SIDE - 300, B4_SIDE - 500
        assert zb.lib().zb_insert_from(img._zb(), int(img.pixfmt), _zbi(src, 300, 500), int(zb.PixFmt.U8), _f(c0), _f(r0), _f(B4_SIDE),
                                       _f(B4_SIDE), _f(0), _f(1), _f(0), int(zb.Interpolation.NEAREST), _f(0), _f(0), 0, None) == 0
        torch.cuda.synchronize()
        want = torch.stack([src, src, src, torch.full_like(src, 255)], dim=-1)
        assert torch_equal(view[r0:, c0:], want)
    elif name == "zb_ssim":              # an image against an exact copy: every window gives 1, so the mean is exactly 1
        _need(torch, 3 * B4_SIDE * B4_SIDE * 4 + GiB)
        other = view.clone()
        assert img.ssim(zb.Image(other.view(-1), img.pixfmt, img.rows, img.cols, img.cols)) == 1.0
        other[(1 << 30) // B4_SIDE, (1 << 30) % B4_SIDE] ^= 0x80   # one changed pixel past 2^32 bytes must lower it
        assert img.ssim(zb.Image(other.view(-1), img.pixfmt, img.rows, img.cols, img.cols)) < 1.0
    elif name == "zb_apply_colormap":    # black with white pixels: the scanned range is [0, 1], black -> lut[0], white -> lut[255]
        _need(torch, B4_SIDE * B4_SIDE * 7 + GiB)
        view.fill_(0)
        spots = [divmod(p, B4_SIDE) for p in (1 << 29, 1 << 30, B4_SIDE * B4_SIDE - 1)]
        for r, c in spots:
            view[r, c] = 255
        lut = zb.image.colormap_lut(zb.Colormap.JET)
        out = torch.full((B4_SIDE, B4_SIDE, 3), 0xA5, dtype=torch.uint8, device="cuda")
        lut_c = (C.c_uint8 * 768)(*lut.reshape(-1).tolist())
        assert zb.lib().zb_apply_colormap(img._zb(), int(img.pixfmt), lut_c, 0, 0.0, 0, 0.0, _zbi(out, B4_SIDE, B4_SIDE), None) == 0
        torch.cuda.synchronize()
        lo, hi = torch.from_numpy(lut[0].copy()).to("cuda"), torch.from_numpy(lut[255].copy()).to("cuda")
        for r, c in spots:
            assert torch_equal(out[r, c], hi), (r, c)
            out[r, c] = lo
        assert all(torch_equal(out[r:r + 2048], lo) for r in range(0, B4_SIDE, 2048))
    elif name == "zb_palette_lookup":    # dst = lut[key(convertColor(Rgb, px))], the key computed here per pixel
        out = torch.full((B4_SIDE, B4_SIDE), 0xA5, dtype=torch.uint8, device="cuda")
        lut = (torch.arange(32768, device="cuda") * 7 % 251).to(torch.uint8)
        assert zb.lib().zb_palette_lookup(img._zb(), int(img.pixfmt), lut.data_ptr(), _zbi(out, B4_SIDE, B4_SIDE), None) == 0
        torch.cuda.synchronize()
        for r in range(0, B4_SIDE, 2048):
            v = view[r:r + 2048].to(torch.int64)
            key = (v[..., 0] >> 3) << 10 | (v[..., 1] >> 3) << 5 | (v[..., 2] >> 3)
            assert torch_equal(out[r:r + 2048], lut[key]), r
    elif name == "zb_median_cut":        # three colours, first touched in this order: the palette of the same three on a tiny image
        import quantize_oracle as qo
        cols = [(40, 80, 120, 255), (200, 16, 8, 255), (8, 248, 96, 255)]
        view[:] = torch.tensor(cols[0], dtype=torch.uint8, device="cuda")
        r, c = divmod(1 << 30, B4_SIDE)
        view[r, c] = torch.tensor(cols[1], dtype=torch.uint8, device="cuda")
        view[-1, -1] = torch.tensor(cols[2], dtype=torch.uint8, device="cuda")
        got = zb.median_cut(img, 16)
        tiny = np.array([[cols[0], cols[0], cols[1], cols[2]]], np.uint8)
        assert np.array_equal(got, qo.median_cut(tiny, 16))
    elif name == "zb_flood_fill":        # a uniform image with a 5 x 5 block of another value past 2^32 bytes: all but the block fills
        view.fill_(50)
        r, c = divmod(1 << 30, B4_SIDE)
        view[r - 2:r + 3, c - 2:c + 3] = 200
        fill = (C.c_uint8 * 4)(9, 8, 7, 6)
        assert zb.lib().zb_flood_fill(img._zb(), int(img.pixfmt), 0, 0, fill, 0.0, 4, 0, None) == 0
        torch.cuda.synchronize()
        assert _all_equal(view[r - 2:r + 3, c - 2:c + 3], 200)
        view[r - 2:r + 3, c - 2:c + 3] = torch.tensor([9, 8, 7, 6], dtype=torch.uint8, device="cuda")
        want = torch.tensor([9, 8, 7, 6], dtype=torch.uint8, device="cuda")
        assert all(torch_equal(view[q:q + 2048], want) for q in range(0, B4_SIDE, 2048))
    elif name == "zb_motion_blur_radial":   # a uniform image: every sample is the same value
        view.fill_(77)
        out = torch.full_like(buf, 0xA5)
        from zignal_b200.compose import motion_blur_radial
        motion_blur_radial(img, zb.Image(out.view(-1), img.pixfmt, img.rows, img.cols, img.cols), 0.5, 0.999, 0.3)
        assert _all_equal(out, 77)
    elif name == "zb_conv_separable_rows":   # rows [16,200, 16,300) and the last 100 rows against the whole call
        _need(torch, 3 * B4_SIDE * B4_SIDE * 4 + GiB)
        k = (C.c_float * 3)(0.25, 0.5, 0.25)
        full = torch.full_like(buf, 0xA5)
        part = torch.full_like(buf, 0xA5)
        L = zb.lib()
        assert L.zb_conv_separable(img._zb(), _zbi(full, B4_SIDE, B4_SIDE), int(img.pixfmt), k, 3, k, 3, 2, None) == 0
        for r0, r1 in ((16_200, 16_300), (B4_SIDE - 100, 0)):
            assert L.zb_conv_separable_rows(img._zb(), _zbi(part, B4_SIDE, B4_SIDE), int(img.pixfmt), k, 3, k, 3, 2, r0, r1, None) == 0
        torch.cuda.synchronize()
        assert torch_equal(part[16_200:16_300], full[16_200:16_300]) and torch_equal(part[-100:], full[-100:])
        part[16_200:16_300] = 0xA5
        part[-100:] = 0xA5
        assert _all_equal(part, 0xA5)
    else:
        raise AssertionError(name)


def _nearest_index(src_n, dst_n):
    """Source index of each destination index for NEAREST resize, as the host tables of zb_resize.cu compute it: s = (d + 0.5) * ratio
    - 0.5 in f32, rounded half away from zero, clamped to the last index."""
    f = np.float32
    ratio = f(src_n) / f(dst_n)
    s = (np.arange(dst_n, dtype=f) + f(0.5)) * ratio - f(0.5)
    return np.minimum(np.floor(s.astype(np.float64) + 0.5), src_n - 1).astype(np.int64)


def _gather(torch, view, ri, ci):
    ri, ci = torch.from_numpy(ri).to("cuda"), torch.from_numpy(ci).to("cuda")
    return view.index_select(0, ri).index_select(1, ci)


def _sampler_case(torch, name, cls, view, img):
    """NEAREST samples of a random image at positions that span it (past row 32,537, i.e. byte 2^32, up to the last row), compared
    pixel for pixel with the source pixels the sampler must pick."""
    rows, cols = img.rows, img.cols
    L = zb.lib()
    NEAREST = int(zb.Interpolation.NEAREST)
    if name in ("zb_rotate_into_cs", "zb_rotate_into_batch"):
        # cos 0, sin 1 with a non-orthogonal angle: the gather kernel turns by 90 degrees with exact f32 coordinates.  With the centre
        # (cols / 2, rows / 2) and dst of src's shape, dst(y, x) = src(x - cx + cy, cx + cy - y) where that is inside, else zero.
        out = torch.full_like(view if view.is_contiguous() else view.contiguous(), 0xA5)
        oimg = zb.Image(out.view(-1), img.pixfmt, rows, cols, cols)
        args = (int(img.pixfmt), _f(0.3), _f(0.0), _f(1.0), NEAREST, _f(0), _f(0), int(zb.BorderMode.ZERO), None)
        if name == "zb_rotate_into_cs":
            assert L.zb_rotate_into_cs(img._zb(), oimg._zb(), *args) == 0
        else:
            assert L.zb_rotate_into_batch(img._zb(), 0, oimg._zb(), 0, 1, *args) == 0
        torch.cuda.synchronize()
        cx, cy = cols // 2, rows // 2
        assert cols % 2 == 0 and rows % 2 == 0
        x0, x1 = max(0, cx - cy), min(cols, rows + cx - cy)       # columns whose source row x - cx + cy is inside
        for y0 in range(0, rows, 256):
            y = np.arange(y0, min(rows, y0 + 256))
            sc = cx + cy - y
            ok = (sc >= 0) & (sc < cols)
            got = out[y0:y0 + len(y)]
            if ok.any():
                want = _gather(torch, view, np.arange(x0, x1) - cx + cy, sc[ok]).transpose(0, 1)   # (rows of y, x0..x1)
                assert torch_equal(got[torch.from_numpy(np.nonzero(ok)[0]).to("cuda"), x0:x1], want), y0
                got[torch.from_numpy(np.nonzero(ok)[0]).to("cuda"), x0:x1] = 0
            assert torch_equal(got, 0), y0
        return
    if name == "zb_rotate_into":         # 180 degrees: the orthogonal kernel, over the whole image
        out = torch.full_like(view, 0xA5)
        img.rotate_into(zb.Image(out.view(-1), img.pixfmt, rows, cols, cols), float(np.float32(np.pi)), zb.Interpolation.NEAREST)
        assert zb.lib().zb_last_kernel().decode() == "rotate_orthogonal"
        assert _equal_rows(out, view.flip(0).flip(1))
        return
    if name == "zb_resize":
        dr, dc = (1000, 1000) if cls == "B4" else (173, 1001)
        ri, ci = _nearest_index(rows, dr), _nearest_index(cols, dc)
        out = torch.full((dr, dc, 4), 0xA5, dtype=torch.uint8, device="cuda")
        img.resize(zb.Image(out.view(-1), img.pixfmt, dr, dc, dc), zb.Interpolation.NEAREST)
    elif name == "zb_warp":              # affine x' = 33 x + 32 (B4) / 33 x + 5 (V), y' = 33 y + 32 (B4) / y (V): integer positions
        if cls == "B4":
            dr, dc, m = 1000, 1000, (33.0, 0.0, 0.0, 33.0, 32.0, 32.0)
            ri, ci = 33 * np.arange(dr) + 32, 33 * np.arange(dc) + 32
        else:
            dr, dc, m = rows, 999, (33.0, 0.0, 0.0, 1.0, 5.0, 0.0)
            ri, ci = np.arange(dr), 33 * np.arange(dc) + 5
        out = torch.full((dr, dc, 4), 0xA5, dtype=torch.uint8, device="cuda")
        mm = (C.c_float * 6)(*m)
        assert L.zb_warp(img._zb(), _zbi(out, dr, dc), int(img.pixfmt), 1, mm, NEAREST, _f(0), _f(0), None) == 0
        torch.cuda.synchronize()
    else:                                # zb_extract: the gather path (rect size != dst size); positions within 0.01 of integers
        if cls == "B4":
            dr, dc, rect = 1000, 1000, (32.0, 32.0, 32.0 + 33 * 999, 32.0 + 33 * 999)
            ri, ci = 33 * np.arange(dr) + 32, 33 * np.arange(dc) + 32
        else:
            dr, dc, rect = rows, 1000, (5.0, 0.0, 5.0 + 33 * 999, float(rows - 1))
            ri, ci = np.arange(dr), 33 * np.arange(dc) + 5
        out = torch.full((dr, dc, 4), 0xA5, dtype=torch.uint8, device="cuda")
        img.extract(zb.Image(out.view(-1), img.pixfmt, dr, dc, dc), rect, 0.0, zb.Interpolation.NEAREST, zb.BorderMode.ZERO)
        assert zb.lib().zb_last_kernel().decode() == "extract_gather"
    assert ri.max() >= (32_537 if cls == "B4" else rows - 2) and ci.max() > cols - 100   # the samples reach the far end
    assert torch_equal(out, _gather(torch, view, ri, ci)), name


RESULT_TESTS = {}
for _name, _row_ in ENTRY_POINTS.items():
    for _cls in CLASSES:
        if _row_[_cls] != R:
            continue
        if _cls in ("W1", "W4", "T1"):
            RESULT_TESTS[(_name, _cls)] = {"zb_copy": _test_copy, "zb_set_border_zero": _test_set_border_zero,
                                           "zb_upload": _test_upload_download, "zb_download": _test_upload_download,
                                           "zb_histogram": _test_histogram, "zb_autocontrast": lambda torch, cls: _test_enhance(torch, cls, "autocontrast"),
                                           "zb_equalize": lambda torch, cls: _test_enhance(torch, cls, "equalize"), "zb_threshold_otsu": _test_otsu}[_name]
        elif _name in ("zb_conv_separable", "zb_gaussian_blur", "zb_convolve", "zb_box_blur", "zb_sharpen", "zb_order_blur", "zb_sobel",
                       "zb_canny", "zb_motion_blur_linear", "zb_convert"):
            RESULT_TESTS[(_name, _cls)] = lambda torch, cls, n=_name: _local_case(n, cls, torch)
        else:
            RESULT_TESTS[(_name, _cls)] = lambda torch, cls, n=_name: _torch_case(n, cls, torch)


@pytest.mark.gpu
@pytest.mark.parametrize("name,cls", sorted(RESULT_TESTS), ids=[f"{n}-{c}" for n, c in sorted(RESULT_TESTS)])
def test_result_past_the_32_bit_range(torch_dev, name, cls):
    RESULT_TESTS[(name, cls)](torch_dev, cls)
