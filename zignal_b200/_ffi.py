"""ctypes binding of libzignal_b200.so (the C ABI declared in include/zignal_b200.h).

The product path fails loudly when the CUDA library is missing: there is no CPU fallback and this
package never imports anything under oracle/.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
LIB_PATH = PKG / "lib" / "libzignal_b200.so"
HEADER = ROOT / "include" / "zignal_b200.h"


class ZbImage(C.Structure):
    """zb_image: mirror of zignal's Image(T) {rows, cols, data, stride} (reference image.zig:97-102)."""
    _fields_ = [("data", C.c_void_p), ("rows", C.c_uint32), ("cols", C.c_uint32), ("stride", C.c_uint64)]


class ZbHoughLine(C.Structure):
    """zb_hough_line: HoughTransform.Line (reference image/hough.zig:13-25) with the points flattened."""
    _fields_ = [("angle", C.c_float), ("radius", C.c_float), ("score", C.c_uint32), ("p1x", C.c_float), ("p1y", C.c_float),
                ("p2x", C.c_float), ("p2y", C.c_float)]


class ZbDiffStats(C.Structure):
    """zb_diff_stats: DiffResult (reference image/diff.zig:19-22) with RunningStats(f64, .summary) flattened."""
    _fields_ = [("n", C.c_uint64), ("diff_count", C.c_uint64), ("sum", C.c_double), ("mean", C.c_double), ("variance", C.c_double),
                ("min", C.c_double), ("max", C.c_double)]


class ZbJpegOptions(C.Structure):
    """zb_jpeg_options: jpeg.EncodeOptions (reference codecs/jpeg.zig:284-290); comment NULL = no COM segment."""
    _fields_ = [("quality", C.c_uint8), ("subsampling", C.c_uint8), ("density_dpi", C.c_uint16), ("comment", C.c_void_p),
                ("comment_len", C.c_uint32)]


class ZbJpegLimits(C.Structure):
    """zb_jpeg_limits: jpeg.DecodeLimits (reference codecs/jpeg.zig:19-33); 0 disables a limit."""
    _fields_ = [("max_jpeg_bytes", C.c_uint64), ("max_marker_bytes", C.c_uint64), ("max_width", C.c_uint32), ("max_height", C.c_uint32),
                ("max_pixels", C.c_uint64), ("max_blocks", C.c_uint64), ("max_scans", C.c_uint64)]


class ZbJpegHeader(C.Structure):
    """zb_jpeg_header: jpeg.Header (reference codecs/jpeg.zig:61-73)."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("progressive", C.c_int32), ("num_components", C.c_int32),
                ("precision", C.c_int32), ("subsampling", C.c_int32)]


class ZignalError(RuntimeError):
    def __init__(self, status: int, name: str, detail: str = ""):
        self.status = status
        self.name = name
        super().__init__(f"{name} (status {status})" + (f": {detail}" if detail else ""))


class LibraryMissing(ImportError):
    pass


def declared_symbols() -> list[str]:
    """Every function the public header declares (used by the export test)."""
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(zb_[a-z0-9_]+)\s*\(", text)))


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise LibraryMissing(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  zignal_b200 has no CPU fallback.")
        _lib = C.CDLL(str(LIB_PATH))
        _declare(_lib)
    return _lib


def _declare(L):
    P = C.POINTER
    img = P(ZbImage)
    fp, dp = P(C.c_float), P(C.c_double)
    vp = C.c_void_p
    u32, u64, i = C.c_uint32, C.c_uint64, C.c_int
    f = C.c_float
    sig = {
        "zb_version": ([], i),
        "zb_status_name": ([i], C.c_char_p),
        "zb_last_error": ([], C.c_char_p),
        "zb_last_kernel": ([], C.c_char_p),
        "zb_last_sweeps": ([], i),
        "zb_device_count": ([P(i)], i),
        "zb_set_device": ([i], i),
        "zb_get_device": ([P(i)], i),
        "zb_sm_count": ([P(i)], i),
        "zb_stream_create": ([P(vp)], i),
        "zb_stream_destroy": ([vp], i),
        "zb_stream_synchronize": ([vp], i),
        "zb_malloc": ([P(vp), C.c_size_t, vp], i),
        "zb_free": ([vp, vp], i),
        "zb_malloc_host": ([P(vp), C.c_size_t], i),
        "zb_free_host": ([vp], i),
        "zb_upload": ([img, img, i, vp], i),
        "zb_download": ([img, img, i, vp], i),
        "zb_copy": ([img, img, i, vp], i),
        "zb_kernel_launch_count": ([], u64),
        "zb_gaussian_taps": ([f, fp, i, P(i)], i),
        "zb_sobel": ([img, img, i, vp], i),
        "zb_canny": ([img, img, i, f, f, f, vp], i),
        "zb_shen_castan": ([img, img, i, f, u64, f, f, i, i, vp], i),
        "zb_motion_blur_linear": ([img, img, i, f, f, f, u32, vp], i),
        "zb_motion_blur_radial": ([img, img, i, f, f, f, i, vp], i),
        "zb_eigh_f64": ([P(C.c_double), u32, u32, P(C.c_double), P(C.c_double)], i),
        "zb_eigh_f32": ([P(f), u32, u32, P(f), P(f)], i),
        "zb_convert": ([img, i, img, i, vp], i),
        "zb_psnr": ([img, img, i, P(C.c_double), vp], i),
        "zb_ssim": ([img, img, i, P(C.c_double), vp], i),
        "zb_mean_pixel_error": ([img, img, i, P(C.c_double), vp], i),
        "zb_order_blur": ([img, img, i, u32, i, C.c_double, i, vp], i),
        "zb_histogram": ([img, i, P(u32), vp], i),
        "zb_autocontrast": ([img, i, f, vp], i),
        "zb_equalize": ([img, i, vp], i),
        "zb_threshold_otsu": ([img, img, P(C.c_uint8), vp], i),
        "zb_threshold_adaptive_mean": ([img, img, u32, f, vp], i),
        "zb_morph_binary": ([img, img, P(C.c_uint8), u32, u32, u32, i, vp], i),
        "zb_flood_fill": ([img, i, u32, u32, vp, C.c_double, i, i, vp], i),
        "zb_median_cut": ([img, i, C.c_uint16, vp, u32, P(u32), vp], i),
        "zb_build_palette": ([img, i, i, C.c_uint16, vp, P(u32), vp], i),
        "zb_color_lut": ([vp, u32, vp, vp], i),
        "zb_dither": ([img, i, vp, u32, vp, i, vp], i),
        "zb_palette_lookup": ([img, i, vp, img, vp], i),
        "zb_diff": ([img, img, img, i, f, f, i, i, P(ZbDiffStats), vp], i),
        "zb_colormap_lut": ([i, vp], i),
        "zb_apply_colormap": ([img, i, vp, i, C.c_double, i, C.c_double, img, vp], i),
        "zb_jpeg_encode_bound": ([u32, u32, i, P(ZbJpegOptions), P(u64)], i),
        "zb_jpeg_encode": ([img, i, P(ZbJpegOptions), vp, u64, P(u64), vp], i),
        "zb_jpeg_info": ([vp, u64, P(ZbJpegLimits), P(ZbJpegHeader)], i),
        "zb_jpeg_decode": ([vp, u64, P(ZbJpegLimits), img, i, vp], i),
        "zb_jpeg_decode_batch": ([u32, vp, vp, P(ZbJpegLimits), vp, vp, vp, vp], i),
        "zb_flip_left_right": ([img, i, vp], i),
        "zb_flip_top_bottom": ([img, i, vp], i),
        "zb_invert": ([img, i, vp], i),
        "zb_insert": ([img, img, i, f, f, f, f, f, f, f, i, f, f, vp], i),
        "zb_insert_blend": ([img, img, i, f, f, f, f, f, f, f, i, f, f, i, vp], i),
        "zb_insert_from": ([img, i, img, i, f, f, f, f, f, f, f, i, f, f, i, vp], i),
        "zb_extract": ([img, img, i, f, f, f, f, f, f, f, i, f, f, i, vp], i),
        "zb_set_border_zero": ([img, i, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp], i),
        "zb_conv_separable": ([img, img, i, fp, i, fp, i, i, vp], i),
        "zb_conv_separable_rows": ([img, img, i, fp, i, fp, i, i, C.c_uint32, C.c_uint32, vp], i),
        "zb_convolve": ([img, img, i, fp, i, i, i, vp], i),
        "zb_gaussian_blur": ([img, img, i, f, vp], i),
        "zb_box_blur": ([img, img, i, u32, vp], i),
        "zb_sharpen": ([img, img, i, u32, vp], i),
        "zb_integral_plane": ([img, i, fp, vp], i),
        "zb_resize": ([img, img, i, i, f, f, vp], i),
        "zb_rotate_bounds": ([u32, u32, f, P(u32), P(u32)], i),
        "zb_rotate_into": ([img, img, i, f, i, f, f, i, vp], i),
        "zb_rotate_into_cs": ([img, img, i, f, f, f, i, f, f, i, vp], i),
        "zb_rotate_into_batch": ([img, u64, img, u64, u32, i, f, f, f, i, f, f, i, vp], i),
        "zb_warp": ([img, img, i, i, fp, i, f, f, vp], i),
        "zb_gemm_f32": ([fp, u32, u32, i, fp, u32, u32, i, f, f, fp, fp, vp], i),
        "zb_gemm_f64": ([dp, u32, u32, i, dp, u32, u32, i, C.c_double, C.c_double, dp, dp, vp], i),
        "zb_center_columns_f32": ([fp, u32, u32, fp, i, fp, vp], i),
        "zb_center_columns_f64": ([dp, u32, u32, dp, i, dp, vp], i),
        "zb_svd_f64": ([dp, u32, u32, i, i, dp, dp, dp, P(u64)], i),
        "zb_svd_f32": ([fp, u32, u32, i, i, fp, fp, fp, P(u64)], i),
        "zb_svd_dev_f64": ([dp, u32, u32, dp, dp, dp, P(u64), vp], i),
        "zb_svd_dev_f32": ([fp, u32, u32, fp, fp, fp, P(u64), vp], i),
        "zb_hough_create": ([u32, P(C.c_int32), P(C.c_int32), P(vp)], i),
        "zb_hough_destroy": ([vp], i),
        "zb_hough_compute": ([vp, img, u32, u32, u32, u32, img, vp], i),
        "zb_hough_find_lines": ([vp, img, u32, f, f, P(ZbHoughLine), u32, P(u32), vp], i),
        "zb_fdm_create": ([P(vp), i], i),
        "zb_fdm_destroy": ([vp], i),
        "zb_fdm_set_target": ([vp, img, vp], i),
        "zb_fdm_set_source": ([vp, img], i),
        "zb_fdm_update": ([vp, vp], i),
        "zb_fdm_status": ([vp, vp], i),
        "zb_fdm_match": ([vp, img, img, vp], i),
        "zb_fdm_moments": ([img, i, i, P(u64), vp], i),
        "zb_fdm_set_target_moments": ([vp, P(u64)], i),
        "zb_fdm_update_with_moments": ([vp, P(u64), vp], i),
        "zb_host_conv_separable": ([img, img, i, fp, i, fp, i, i], i),
        "zb_host_convolve": ([img, img, i, fp, i, i, i], i),
        "zb_host_gaussian_blur": ([img, img, i, f], i),
        "zb_host_box_blur": ([img, img, i, u32], i),
        "zb_host_sharpen": ([img, img, i, u32], i),
        "zb_host_resize": ([img, img, i, i, f, f], i),
        "zb_host_rotate_into": ([img, img, i, f, i, f, f, i], i),
        "zb_host_warp": ([img, img, i, i, fp, i, f, f], i),
        "zb_host_fdm_match": ([img, img, i], i),
        "zb_shard_unique_id": ([P(C.c_uint8)], i),
        "zb_shard_comm_create": ([P(vp), i, i, P(C.c_uint8)], i),
        "zb_shard_comm_destroy": ([vp], i),
        "zb_shard_comm_info": ([vp, P(i), P(i), P(i)], i),
        "zb_shard_status": ([vp, vp], i),
        "zb_shard_alloc": ([vp, C.c_size_t, P(vp)], i),
        "zb_shard_free": ([vp, vp], i),
        "zb_shard_image_create": ([vp, img, u32, i, P(vp)], i),
        "zb_shard_image_destroy": ([vp], i),
        "zb_shard_image_block": ([vp, img], i),
        "zb_shard_split": ([u32, i, i, P(u32), P(u32)], i),
        "zb_shard_halo_exchange": ([vp, vp, u32, i, vp], i),
        "zb_shard_view": ([vp, u32, i, img, P(u32)], i),
        "zb_shard_conv_separable": ([vp, vp, vp, fp, i, fp, i, i, vp], i),
        "zb_shard_gaussian_blur": ([vp, vp, vp, f, vp], i),
        "zb_shard_allreduce": ([vp, vp, C.c_size_t, i, vp], i),
        "zb_shard_fdm_set_target": ([vp, vp, img, vp], i),
        "zb_shard_fdm_update": ([vp, vp, vp], i),
        "zb_shard_tune_path": ([i], i),
        "zb_shard_debug_times": ([vp, vp, vp], i),
        "zb_set_exact_f32": ([i], i),
        "zb_set_force_generic": ([i], i),
        "zb_tune": ([C.c_char_p, i], i),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name, None)
        if fn is None:
            continue  # the export test reports missing symbols; calling one raises AttributeError
        fn.argtypes = args
        fn.restype = res


def check(status: int):
    if status != 0:
        L = lib()
        name = L.zb_status_name(status).decode()
        detail = L.zb_last_error().decode() if status == 7 else ""
        raise ZignalError(status, name, detail)
