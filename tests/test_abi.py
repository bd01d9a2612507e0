"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol the public
header declares, and its host-side entry points (no device work) agree with the oracle."""
import ctypes as C
import re

import numpy as np
import pytest

import oracle_lib as zo
import zignal_b200 as zb
from zignal_b200 import _ffi


def test_library_loads_and_exports_every_declared_symbol():
    L = zb.lib()
    names = zb.declared_symbols()
    assert len(names) >= 50
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, f"header declares symbols the library does not export: {missing}"
    assert L.zb_version() == 1


def test_enums_match_between_product_header_and_oracle_header():
    prod = (_ffi.ROOT / "include" / "zignal_b200.h").read_text()
    orac = (_ffi.ROOT / "oracle" / "zignal_oracle.h").read_text()
    for suffix in ("BORDER_ZERO", "BORDER_REPLICATE", "BORDER_MIRROR", "BORDER_WRAP", "INTERP_NEAREST", "INTERP_BILINEAR",
                   "INTERP_BICUBIC", "INTERP_CATMULL_ROM", "INTERP_MITCHELL", "INTERP_LANCZOS", "PIX_U8", "PIX_F32", "PIX_RGB8",
                   "PIX_RGBA8", "PIX_RGBAF32", "XFORM_SIMILARITY", "XFORM_AFFINE", "XFORM_PROJECTIVE", "SVD_NO_U", "SVD_SKINNY_U",
                   "SVD_FULL_U"):
        a = re.search(rf"ZB_{suffix}\s*=\s*(\d+)", prod)
        b = re.search(rf"ZO_{suffix}\s*=\s*(\d+)", orac)
        assert a and b and a.group(1) == b.group(1), suffix


def test_status_names_follow_zig_error_names():
    L = zb.lib()
    want = {0: "Ok", 1: "DimensionMismatch", 2: "InvalidSigma", 4: "NotConverged", 6: "OutOfMemory", 7: "DeviceFailure",
            8: "InvalidScaleFactor", 9: "InvalidDimensions", 10: "NoTargetSet", 11: "NoSourceSet"}
    for k, v in want.items():
        assert L.zb_status_name(k).decode() == v


def test_product_does_not_import_the_oracle():
    pkg = _ffi.PKG
    for path in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.h")) + list(pkg.rglob("*.cuh")) + list(pkg.rglob("*.hpp")):
        text = path.read_text()
        assert "oracle_lib" not in text and "zignal_oracle" not in text and "libzignal_oracle" not in text, path


def test_gaussian_taps_match_oracle_bit_for_bit():
    for sigma in (0.5, 1.0, 1.4, 2.0, 2.25, 3.3, 7.0):
        assert np.array_equal(zb.gaussian_taps(sigma), zo.gaussian_taps(sigma)), sigma
    assert zb.gaussian_taps(0.0).size == 0
    n = C.c_int()
    assert zb.lib().zb_gaussian_taps(C.c_float(-1.0), None, 0, C.byref(n)) == 2  # InvalidSigma
    for bad in (float("inf"), float("nan")):     # image.zig:973 would panic on the usize cast; an error code here, no huge allocation
        assert zb.lib().zb_gaussian_taps(C.c_float(bad), None, 0, C.byref(n)) == 2, bad
    assert zb.lib().zb_gaussian_taps(C.c_float(1e30), None, 0, C.byref(n)) != 0


def test_rotate_bounds_match_oracle():
    L = zb.lib()
    rng = np.random.default_rng(0)
    angles = [0.0, np.pi / 2, np.pi, 3 * np.pi / 2, 2 * np.pi, np.pi / 4, -0.3, 1e-7, 7.0] + list(rng.uniform(-10, 10, 20))
    for a in angles:
        for (r, c) in [(3, 4), (1080, 1920), (17, 1)]:
            orr, occ = C.c_uint32(), C.c_uint32()
            assert L.zb_rotate_bounds(r, c, C.c_float(a), C.byref(orr), C.byref(occ)) == 0
            assert (orr.value, occ.value) == zo.rotate_bounds(r, c, np.float32(a)), (a, r, c)
    orr, occ = C.c_uint32(), C.c_uint32()
    L.zb_rotate_bounds(1080, 1920, C.c_float(np.float32(np.pi / 4)), C.byref(orr), C.byref(occ))
    assert (orr.value, occ.value) == (2122, 2122)


def _svd_prod(a, mode, with_v):
    a = np.ascontiguousarray(a)
    m, n = a.shape
    modes = {"no_u": 0, "skinny_u": 1, "full_u": 2}
    u = np.zeros((m, m if mode == "full_u" else n), a.dtype)
    s = np.zeros(n, a.dtype)
    v = np.zeros((n, n), a.dtype)
    conv = C.c_uint64(99)
    if a.dtype == np.float64:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
        rc = zb.lib().zb_svd_f64(P(a), m, n, modes[mode], int(with_v), P(u), P(s), P(v), C.byref(conv))
    else:
        P = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))
        rc = zb.lib().zb_svd_f32(P(a), m, n, modes[mode], int(with_v), P(u), P(s), P(v), C.byref(conv))
    assert rc == 0
    return u, s, v, conv.value


def _check_svd_against_oracle(a, u, s, v, mode):
    """The reference's own criterion for two SVD implementations (test_svd_comparison.zig:51-72, svd.zig:498-636): singular values
    agree to sqrt(eps) (here: far tighter), factors orthonormal, A = U S V^T; vectors are compared as subspaces up to sign."""
    dtype = a.dtype
    m, n = a.shape
    eps = np.finfo(dtype).eps
    _, so, vo, rco = zo.svd(a, mode, True)
    assert rco == 0
    scale = max(float(so[0]), 1e-300) if so.size else 1.0
    assert np.all(np.diff(s) <= 0) and np.all(s >= 0)                                    # descending, non-negative (svd.zig:520-530)
    assert np.max(np.abs(s.astype(np.float64) - so.astype(np.float64))) <= 16 * eps * max(m, n, 4) * scale   # both routines: O(n eps |A|)
    assert np.max(np.abs(s - so)) <= np.sqrt(eps) * scale                                # the reference's stated tolerance
    tol = 200 * eps * max(m, n)
    assert np.allclose(v.T.astype(np.float64) @ v.astype(np.float64), np.eye(n), atol=tol)
    if mode != "no_u":
        u64 = u.astype(np.float64)
        assert np.allclose(u64.T @ u64, np.eye(u.shape[1]), atol=tol)
        assert np.allclose(u64[:, :n] @ np.diag(s.astype(np.float64)) @ v.T.astype(np.float64), a, atol=tol * scale)
    # well separated singular values: the right vectors agree with the oracle's up to sign
    gaps = np.abs(np.diff(np.concatenate([so.astype(np.float64), [0.0]])))
    for i in range(n):
        left = so[i - 1] - so[i] if i > 0 else np.inf
        if min(left, gaps[i]) > 1e-2 * scale:
            d = abs(float(v[:, i].astype(np.float64) @ vo[:, i].astype(np.float64)))
            assert abs(d - 1.0) <= (1e-9 if dtype == np.float64 else 2e-3), (i, d)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(3, 3), (5, 4), (9, 9), (23, 17), (2, 2), (1, 1)])
@pytest.mark.parametrize("mode", ["no_u", "skinny_u", "full_u"])
def test_host_svd_agrees_with_the_oracle_by_the_references_criterion(dtype, shape, mode):
    """Matrices of fewer than 24 columns are decomposed on the host (no GPU needed); larger ones are in tests/test_gpu_linalg.py."""
    rng = np.random.default_rng(abs(hash((shape, mode))) % 2**32)
    a = rng.standard_normal(shape).astype(dtype)
    u, s, v, conv = _svd_prod(a, mode, True)
    assert conv == 0
    _check_svd_against_oracle(a, u, s, v, mode)


def test_host_svd_rank_deficient_and_wikipedia():
    a = np.array([[1, 0, 0, 0], [0, 0, 0, 2], [0, 3, 0, 0], [0, 0, 0, 0], [2, 0, 0, 0]], np.float64)
    u, s, v, conv = _svd_prod(a, "full_u", True)
    assert conv == 0 and np.allclose(s, [3, np.sqrt(5), 2, 0], atol=1e-12)
    assert u.shape == (5, 5) and np.allclose(u.T @ u, np.eye(5), atol=1e-12)      # full U completed to an orthonormal basis
    assert np.allclose(u[:, :4] @ np.diag(s) @ v.T, a, atol=1e-12)
    a = np.array([[1, 2, 3], [2, 4, 6], [1, 2, 3]], np.float64)
    _, s, _, _ = _svd_prod(a, "full_u", True)
    assert np.count_nonzero(s < np.sqrt(np.finfo(float).eps)) == 2
    assert zb.lib().zb_svd_f64(None, 2, 3, 1, 0, None, None, None, None) != 0


def test_argument_errors_are_reported_before_touching_the_device():
    L = zb.lib()
    a = np.zeros((4, 4), np.uint8)
    b = np.zeros((4, 5), np.uint8)
    ia, ib = zb.image._np_image(a), zb.image._np_image(b)
    k = np.ones(3, np.float32) / 3
    fp = k.ctypes.data_as(C.POINTER(C.c_float))
    assert L.zb_conv_separable(ia, ib, 0, fp, 3, fp, 3, 2, None) == 1      # DimensionMismatch (image.zig:947)
    assert L.zb_gaussian_blur(ia, ib, 0, C.c_float(1.0), None) == 1          # image.zig:962
    assert L.zb_gaussian_blur(ia, ia, 0, C.c_float(-1.0), None) == 2         # InvalidSigma (image.zig:970)
    assert L.zb_box_blur(ia, ib, 0, 1, None) == 1                            # image.zig:636
    assert L.zb_sharpen(ia, ib, 0, 1, None) == 1                             # image.zig:786
    assert L.zb_convolve(ia, ib, 0, fp, 1, 3, 0, None) == 1                  # image.zig:927
    assert L.zb_conv_separable(ia, ia, 99, fp, 3, fp, 3, 2, None) == 3       # unsupported pixel type
    f = C.c_void_p()
    assert L.zb_fdm_create(C.byref(f), 1) == 3                               # fdm.zig:20: only u8 / Rgb / Rgba
    assert L.zb_fdm_create(C.byref(f), 2) == 0
    assert L.zb_fdm_update(f, None) == 10                                    # NoTargetSet (fdm.zig:142, :583-604)
    assert L.zb_fdm_destroy(f) == 0
    assert L.zb_tune(b"conv.band_rows", 7) == 5                             # out of range (>= 64)
    assert L.zb_tune(b"conv.stages", 2) == 5                                 # removed knobs are unknown keys
    assert L.zb_tune(b"conv.variant", 0) == 5


def test_scale_shapes_and_errors_host_logic():
    # tests/resize.zig:258-298: factors .5 / 2 / 1.5 on 100x100 -> 50 / 200 / 150; errors for <= 0 and zero-size
    img = zb.Image(None, zb.PixFmt.U8, 100, 100, 100)
    from zignal_b200.image import _round_half_away
    for f, n in [(0.5, 50), (2.0, 200), (1.5, 150)]:
        assert int(_round_half_away(np.float32(100) * np.float32(f))) == n
    with pytest.raises(zb.ZignalError) as e:
        img.scale(0.0)
    assert e.value.name == "InvalidScaleFactor"
    with pytest.raises(zb.ZignalError) as e:
        img.scale(0.001)
    assert e.value.name == "InvalidDimensions"


def test_public_header_is_valid_c99(tmp_path):
    """The boundary is a C ABI: include/zignal_b200.h must compile as plain C (what cgo / Zig's translate-c / a C caller would consume)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    src = tmp_path / "hdr.c"
    src.write_text('#include "zignal_b200.h"\nint main(void) { return ZB_BLEND_EXCLUSION + ZB_ORDER_ALPHA_TRIMMED + ZB_ERR_NOT_FINITE + ZB_PIX_RGBAF32; }\n')
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", str(_ffi.HEADER.parent), str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]


def test_8f_status_names_and_argument_errors_before_the_device():
    """Error behaviour of the 8(f) entry points that is decided on the host (reference error names; no kernel is launched)."""
    L = zb.lib()
    names = {14: "InvalidThreshold", 15: "InvalidPercentile", 16: "InvalidTrim", 17: "ImageTooSmall", 18: "NotSquare", 19: "NotSymmetric",
             20: "NotFinite", 12: "InsufficientData", 13: "InvalidComponents"}
    for k, v in names.items():
        assert L.zb_status_name(k).decode() == v
    a = np.zeros((12, 12), np.uint8)
    b = np.zeros((12, 13), np.uint8)
    ia, ib = zb.image._np_image(a), zb.image._np_image(b)
    f32 = C.c_float
    assert L.zb_canny(ia, ia, 0, f32(float("nan")), f32(1), f32(2), None) == 5       # InvalidParameter (edges.zig:221)
    assert L.zb_canny(ia, ia, 0, f32(-1.0), f32(1), f32(2), None) == 2                # InvalidSigma (:224)
    assert L.zb_canny(ia, ia, 0, f32(1.0), f32(3), f32(2), None) == 14               # InvalidThreshold (:226)
    assert L.zb_canny(ia, ib, 0, f32(1.0), f32(1), f32(2), None) == 1                # DimensionMismatch
    assert L.zb_canny(ia, ia, 4, f32(1.0), f32(1), f32(2), None) == 3                # Rgba(f32) is not a canny input here
    assert L.zb_order_blur(ia, ib, 0, 1, 0, C.c_double(0.5), 2, None) == 1           # image.zig:679
    assert L.zb_order_blur(ia, ia, 0, 1, 2, C.c_double(0.5), 2, None) == 16          # InvalidTrim (order_statistic_blur.zig:160)
    assert L.zb_order_blur(ia, ia, 0, 1, 0, C.c_double(1.5), 2, None) == 15          # InvalidPercentile (:48)
    assert L.zb_order_blur(ia, ia, 1, 1, 0, C.c_double(0.5), 2, None) == 3           # UnsupportedPixelType (:66)
    assert L.zb_order_blur(ia, ia, 0, 5000, 0, C.c_double(0.5), 2, None) == 3        # a window no SM's shared memory can hold
    assert L.zb_order_blur(ia, ia, 0, 1, 7, C.c_double(0.5), 2, None) == 5           # unknown mode
    out = C.c_double(0.0)
    assert L.zb_psnr(ia, ib, 0, C.byref(out), None) == 1                             # metrics.zig:11
    small = zb.image._np_image(np.zeros((10, 30), np.uint8))
    assert L.zb_ssim(small, small, 0, C.byref(out), None) == 17                      # ImageTooSmall (metrics.zig:60)
    assert L.zb_ssim(ia, ia, 9, C.byref(out), None) == 3
    assert L.zb_convert(ia, 0, ib, 1, None) == 1                                     # image.zig:397
    assert L.zb_convert(ia, 0, ia, 9, None) == 3
    assert L.zb_motion_blur_linear(ia, ib, 0, f32(0.5), f32(0.8), f32(0.5), 3, None) == 1
    assert L.zb_motion_blur_radial(ia, ib, 0, f32(0.5), f32(0.5), f32(0.5), 0, None) == 1
    assert L.zb_insert_blend(ia, ia, 0, f32(0), f32(0), f32(1), f32(1), f32(0), f32(1), f32(0), 0, f32(0), f32(0), 13, None) == 5   # unknown blend mode
