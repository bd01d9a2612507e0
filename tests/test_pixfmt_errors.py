"""The status every entry point with a pixel-format parameter returns for a format it does not accept (including the values 5, -1
and 99, which name no format), with small non-empty images and otherwise valid arguments.  Runs without a GPU: every call listed
here is refused on the host, before any device work, so no pointer in it is ever read.  Calls whose format is accepted reach the
device and are not made here."""
import ctypes as C
import re
from pathlib import Path

import pytest

import zignal_b200 as zb
from zignal_b200 import _ffi

HEADER = Path(__file__).resolve().parent.parent / "include" / "zignal_b200.h"
RGBA8 = 3

# function -> {pixel format: status}; for the two-format calls the key is (source or self format, other format).  3 is Unsupported;
# the SSIM of a 4 x 4 image is ImageTooSmall (17) and 16 zero bytes are no JPEG (31) whatever the format.
EXPECTED = {
    "zb_apply_colormap": {5: 3, -1: 3, 99: 3},
    "zb_autocontrast": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_box_blur": {5: 3, -1: 3, 99: 3},
    "zb_build_palette": {5: 3, -1: 3, 99: 3},
    "zb_canny": {4: 3, 5: 3, -1: 3, 99: 3},
    "zb_conv_separable": {5: 3, -1: 3, 99: 3},
    "zb_conv_separable_rows": {5: 3, -1: 3, 99: 3},
    "zb_convert": {
        (0, 5): 3, (0, -1): 3, (0, 99): 3, (1, 5): 3, (1, -1): 3, (1, 99): 3, (2, 5): 3, (2, -1): 3, (2, 99): 3, (3, 5): 3, (3, -1): 3,
        (3, 99): 3, (4, 5): 3, (4, -1): 3, (4, 99): 3, (5, 0): 3, (5, 1): 3, (5, 2): 3, (5, 3): 3, (5, 4): 3, (5, 5): 3, (5, -1): 3,
        (5, 99): 3, (-1, 0): 3, (-1, 1): 3, (-1, 2): 3, (-1, 3): 3, (-1, 4): 3, (-1, 5): 3, (-1, -1): 3, (-1, 99): 3, (99, 0): 3,
        (99, 1): 3, (99, 2): 3, (99, 3): 3, (99, 4): 3, (99, 5): 3, (99, -1): 3, (99, 99): 3,
    },
    "zb_convolve": {5: 3, -1: 3, 99: 3},
    "zb_copy": {5: 3, -1: 3, 99: 3},
    "zb_diff": {5: 3, -1: 3, 99: 3},
    "zb_dither": {0: 3, 1: 3, 3: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_download": {5: 3, -1: 3, 99: 3},
    "zb_equalize": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_extract": {5: 3, -1: 3, 99: 3},
    "zb_fdm_create": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_fdm_moments": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_flip_left_right": {5: 3, -1: 3, 99: 3},
    "zb_flip_top_bottom": {5: 3, -1: 3, 99: 3},
    "zb_flood_fill": {5: 3, -1: 3, 99: 3},
    "zb_gaussian_blur": {5: 3, -1: 3, 99: 3},
    "zb_histogram": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_host_conv_separable": {5: 3, -1: 3, 99: 3},
    "zb_host_convolve": {5: 3, -1: 3, 99: 3},
    "zb_host_fdm_match": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_host_gaussian_blur": {5: 3, -1: 3, 99: 3},
    "zb_insert": {5: 3, -1: 3, 99: 3},
    "zb_insert_blend": {5: 3, -1: 3, 99: 3},
    "zb_insert_from": {
        (0, 5): 3, (0, -1): 3, (0, 99): 3, (1, 5): 3, (1, -1): 3, (1, 99): 3, (2, 5): 3, (2, -1): 3, (2, 99): 3, (3, 5): 3, (3, -1): 3,
        (3, 99): 3, (4, 5): 3, (4, -1): 3, (4, 99): 3, (5, 0): 3, (5, 1): 3, (5, 2): 3, (5, 3): 3, (5, 4): 3, (5, 5): 3, (5, -1): 3,
        (5, 99): 3, (-1, 0): 3, (-1, 1): 3, (-1, 2): 3, (-1, 3): 3, (-1, 4): 3, (-1, 5): 3, (-1, -1): 3, (-1, 99): 3, (99, 0): 3,
        (99, 1): 3, (99, 2): 3, (99, 3): 3, (99, 4): 3, (99, 5): 3, (99, -1): 3, (99, 99): 3,
    },
    "zb_invert": {1: 3, 5: 3, -1: 3, 99: 3},
    "zb_jpeg_decode": {0: 31, 1: 31, 2: 31, 3: 31, 4: 31, 5: 3, -1: 3, 99: 3},
    "zb_jpeg_decode_batch": {0: 31, 1: 31, 2: 31, 3: 31, 4: 31, 5: 3, -1: 3, 99: 3},
    "zb_jpeg_encode": {5: 3, -1: 3, 99: 3},
    "zb_jpeg_encode_bound": {5: 3, -1: 3, 99: 3},
    "zb_mean_pixel_error": {5: 3, -1: 3, 99: 3},
    "zb_median_cut": {5: 3, -1: 3, 99: 3},
    "zb_motion_blur_linear": {5: 3, -1: 3, 99: 3},
    "zb_motion_blur_radial": {5: 3, -1: 3, 99: 3},
    "zb_order_blur": {1: 3, 4: 3, 5: 3, -1: 3, 99: 3},
    "zb_palette_lookup": {5: 3, -1: 3, 99: 3},
    "zb_psnr": {5: 3, -1: 3, 99: 3},
    "zb_resize": {5: 3, -1: 3, 99: 3},
    "zb_rotate_into": {5: 3, -1: 3, 99: 3},
    "zb_rotate_into_batch": {5: 3, -1: 3, 99: 3},
    "zb_rotate_into_cs": {5: 3, -1: 3, 99: 3},
    "zb_set_border_zero": {5: 3, -1: 3, 99: 3},
    "zb_sharpen": {5: 3, -1: 3, 99: 3},
    "zb_shen_castan": {4: 3, 5: 3, -1: 3, 99: 3},
    "zb_sobel": {4: 3, 5: 3, -1: 3, 99: 3},
    "zb_ssim": {0: 17, 1: 17, 2: 17, 3: 17, 4: 17, 5: 3, -1: 3, 99: 3},
    "zb_upload": {5: 3, -1: 3, 99: 3},
    "zb_warp": {5: 3, -1: 3, 99: 3},
}

# Entry points that look at the pixel format only after they have reached the device (or, for the shard image, need a communicator
# that only the device can make): their format errors are not reachable without a GPU.
NOT_REACHABLE = {"zb_shard_image_create", "zb_integral_plane", "zb_host_box_blur", "zb_host_sharpen", "zb_host_resize",
                 "zb_host_rotate_into", "zb_host_warp"}


def _header_signatures():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    out = {}
    for m in re.finditer(r"\b(zb_\w+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S):
        params = [p.strip() for p in m[2].split(",")]
        names = [re.findall(r"\w+", p)[-1] for p in params if p and p != "void"]
        if any("pixfmt" in n for n in names):
            out[m[1]] = names
    return out


class _Args:
    """Buffers that outlive a call: host memory, never dereferenced by a call the parent refuses on the host."""

    def __init__(self):
        self.keep = []

    def buf(self, nbytes, ctype=C.c_uint8):
        a = (ctype * nbytes)()
        self.keep.append(a)
        return a

    def image(self, rows=4, cols=4):
        data = self.buf(rows * cols * 16)
        img = _ffi.ZbImage(C.cast(data, C.c_void_p), rows, cols, cols)
        self.keep.append(img)
        return C.pointer(img)


def _value(name, ctype, fmt, other, args):
    """An argument for parameter `name` of type `ctype`: the format under test for a pixel-format parameter, a valid value otherwise."""
    if name in ("pixfmt", "src_pixfmt", "source_pixfmt"):
        return fmt
    if name in ("dst_pixfmt", "self_pixfmt"):
        return other
    if name == "mode" and ctype is C.c_int and args.fn == "zb_build_palette":
        return 3   # ZB_PALETTE_ADAPTIVE: the fixed palettes ignore the image
    if ctype is C.POINTER(_ffi.ZbImage):
        return args.image()
    if ctype is C.POINTER(_ffi.ZbJpegOptions):
        o = _ffi.ZbJpegOptions()
        o.quality = 90
        args.keep.append(o)
        return C.pointer(o)
    if ctype is C.POINTER(_ffi.ZbJpegLimits):
        return None
    if ctype is C.POINTER(_ffi.ZbDiffStats):
        return None
    if ctype is C.POINTER(C.c_float):
        k = args.buf(16, C.c_float)
        for i in range(16):
            k[i] = 1.0 / 9.0
        return k
    if ctype is C.POINTER(C.c_double):
        return args.buf(16, C.c_double)
    if ctype in (C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.c_void_p,
                 C.POINTER(C.c_void_p)) or (isinstance(ctype, type) and issubclass(ctype, C._Pointer)):
        if name in ("s", "stream", "s_"):
            return None
        return C.cast(args.buf(1 << 17), ctype)
    ints = {"nx": 3, "ny": 3, "kh": 3, "kw": 3, "radius": 1, "method": 1, "border": 1, "xform_kind": 0, "mode": 0, "spin": 0,
            "connectivity": 4, "max_colors": 4, "cap": 256, "n": 4, "distance": 2, "window_size": 5, "hysteresis": 1,
            "use_nms": 1, "blend_mode": 0, "as_luma": 0, "rows": 4, "cols": 4, "halo_cap": 1, "len": 16, "has_min": 0,
            "has_max": 0, "binary": 0, "force_opaque": 0, "start_row": 0, "start_col": 0, "l": 0, "t": 0, "r": 0, "b": 0,
            "map": 0}
    floats = {"sigma": 1.0, "angle": 0.0, "cos_a": 1.0, "sin_a": 0.0, "mitchell_b": 1 / 3, "mitchell_c": 1 / 3, "low_threshold": 0.1,
              "high_threshold": 0.3, "smooth": 0.9, "high_ratio": 0.99, "low_rel": 0.5, "rect_l": 0.0, "rect_t": 0.0, "rect_r": 2.0,
              "rect_b": 2.0, "center_x": 0.5, "center_y": 0.5, "strength": 0.5, "threshold": 0.5, "scale": 1.0, "cutoff": 0.1,
              "param": 0.5, "min": 0.0, "max": 1.0}
    if ctype in (C.c_float, C.c_double):
        return floats.get(name, 0.5)
    return ints.get(name, 1)


def call(name, fmt, other=RGBA8):
    L = zb.lib()
    fn = getattr(L, name)
    names = _header_signatures()[name]
    args = _Args()
    args.fn = name
    if name == "zb_jpeg_decode_batch":   # (n, data, len, limits, dst, pixfmt[], status[], s)
        data = args.buf(16)
        datas = (C.POINTER(C.c_uint8) * 1)(C.cast(data, C.POINTER(C.c_uint8)))
        lens = (C.c_uint64 * 1)(16)
        fmts = (C.c_int * 1)(fmt)
        status = (C.c_int * 1)(0)
        rc = fn(1, datas, lens, None, args.image(), fmts, status, None)
        return rc or status[0]
    return fn(*[_value(n, t, fmt, other, args) for n, t in zip(names, fn.argtypes)])


def test_table_covers_every_pixel_format_entry_point():
    assert set(EXPECTED) | NOT_REACHABLE == set(_header_signatures())


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_unaccepted_pixel_formats_are_refused(name):
    for key, want in EXPECTED[name].items():
        got = call(name, *key) if isinstance(key, tuple) else call(name, key)
        assert got == want, (name, key, got, want)
