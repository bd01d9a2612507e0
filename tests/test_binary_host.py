"""CPU checks of the 8-bit histogram family and binary morphology: the oracle (oracle/zo_binary.cpp, bound in tests/binary_oracle.py) against the reference's own tests
(image/tests/binary.zig, image/histogram.zig:665-845), autocontrast / equalize against an independent numpy restatement (the reference
has no tests for them), and the error behaviour of the new C-ABI entry points that is decided before any device work."""
import ctypes as C

import numpy as np
import pytest

import binary_oracle as zo
import zignal_b200 as zb

BOX3 = np.ones((3, 3), np.uint8)


# ---- image/tests/binary.zig ----------------------------------------------------------------------------------------------------------
def test_kat_threshold_otsu_binarizes_bimodal_image():   # binary.zig tests:7-24
    img = np.array([[10, 10, 10, 10], [200, 200, 200, 200]], np.uint8)
    out, t = zo.threshold_otsu(img)
    assert 5 <= t <= 50
    assert np.array_equal(out, np.array([[0] * 4, [255] * 4], np.uint8))


def test_kat_adaptive_mean_threshold_isolates_bright_center():   # :26-45
    img = np.array([[50, 50, 50], [50, 200, 50], [50, 50, 50]], np.uint8)
    out = zo.threshold_adaptive_mean(img, 1, 10.0)
    want = np.zeros((3, 3), np.uint8)
    want[1, 1] = 255
    assert np.array_equal(out, want)


def test_kat_adaptive_mean_threshold_rejects_zero_radius():   # :47-58
    img = np.array([[10, 20], [30, 40]], np.uint8)
    with pytest.raises(zo.OracleStatus) as e:
        zo.threshold_adaptive_mean(img, 0, 0.0)
    assert e.value.status == 22


def test_kat_binary_dilation_expands_single_pixel():   # :60-88
    img = np.zeros((5, 5), np.uint8)
    img[2, 2] = 255
    out = zo.morph_binary(img, BOX3, 1, "dilate")
    want = np.zeros((5, 5), np.uint8)
    want[1:4, 1:4] = 255
    assert np.array_equal(out, want)


def test_kat_binary_open_removes_isolated_noise_in_place():   # :90-114 (image.openBinary(image, ...))
    img = np.zeros((5, 5), np.uint8)
    img[1, 1:5] = 255
    img[2:4, 1:4] = 255
    zo.morph_binary(img, BOX3, 1, "open", out=img)
    want = np.zeros((5, 5), np.uint8)
    want[1:4, 1:4] = 255
    assert np.array_equal(img, want)


def test_kat_binary_close_fills_holes_in_place():   # :116-140
    img = np.zeros((5, 5), np.uint8)
    img[1:4, 1:4] = 255
    img[2, 2] = 0
    zo.morph_binary(img, BOX3, 1, "close", out=img)
    want = np.zeros((5, 5), np.uint8)
    want[1:4, 1:4] = 255
    assert np.array_equal(img, want)


def test_kat_binary_erosion_shrinks_block_across_iterations():   # :142-167
    img = np.full((5, 5), 255, np.uint8)
    out = zo.morph_binary(img, BOX3, 2, "erode")
    want = np.zeros((5, 5), np.uint8)
    want[2, 2] = 255
    assert np.array_equal(out, want)


# ---- image/histogram.zig:665-845 -----------------------------------------------------------------------------------------------------
def test_kat_histogram_u8_grayscale_basic():   # :665-703
    img = np.array([0, 128, 255, 128, 128, 255, 0, 0, 255], np.uint8).reshape(3, 3)
    h = zo.histogram(img)[0]
    assert h[0] == 3 and h[128] == 3 and h[255] == 3 and h.sum() == 9 and h.max() == 3


def test_kat_histogram_rgb_color():   # :705-739
    img = np.array([[[255, 0, 0], [0, 255, 0]], [[0, 0, 255], [128, 128, 128]]], np.uint8)
    h = zo.histogram(img)
    for k in range(3):
        assert (h[k, 0], h[k, 128], h[k, 255]) == (2, 1, 1)
    assert h[0].sum() == 4 and h.max() == 2


def test_kat_histogram_rgba_with_alpha():   # :741-766
    img = np.array([[[255, 0, 0, 255], [0, 255, 0, 128]], [[0, 0, 255, 64], [128, 128, 128, 0]]], np.uint8)
    h = zo.histogram(img)
    assert (h[3, 0], h[3, 64], h[3, 128], h[3, 255]) == (1, 1, 1, 1)
    assert h[0].sum() == 4


def test_kat_histogram_empty_image():   # :768-786
    h = zo.histogram(np.zeros((0, 0), np.uint8))
    assert h.shape == (1, 256) and not h.any()


def test_kat_histogram_single_pixel():   # :788-801
    h = zo.histogram(np.array([[42]], np.uint8))[0]
    assert h[42] == 1 and h.sum() == 1


def test_kat_histogram_uniform_color():   # :803-845
    h = zo.histogram(np.full((10, 10, 3), 100, np.uint8))
    for k in range(3):
        assert h[k, 100] == 100 and h[k].sum() == 100


def test_histogram_counts_only_the_view():
    big = np.full((6, 9), 7, np.uint8)
    big[1:4, 2:7] = np.arange(15, dtype=np.uint8).reshape(3, 5)
    h = zo.histogram(big[1:4, 2:7])[0]
    assert np.array_equal(h[:15], np.ones(15, np.uint32)) and h.sum() == 15


# ---- autocontrast / equalize: an independent numpy restatement of enhancement.zig ------------------------------------------------------
def _np_cutoffs(hist, cutoff_pixels):
    if cutoff_pixels == 0:
        nz = np.nonzero(hist)[0]
        mn = int(nz[0]) if nz.size else 0
        nz_hi = nz[nz > 0]
        mx = int(nz_hi[-1]) if nz_hi.size else 0        # bin 0 is never visited from the top (histogram.zig:148)
        return mn, mx
    cum = np.cumsum(hist.astype(np.int64))
    above = np.nonzero(cum > cutoff_pixels)[0]
    mn = int(above[0]) if above.size else 255
    suffix = np.cumsum(hist[::-1].astype(np.int64))[::-1]  # suffix[i] = sum(hist[i:])
    above = [i for i in range(255, 0, -1) if suffix[i] > cutoff_pixels]
    mx = above[0] if above else 0
    return mn, mx


def np_autocontrast(img, cutoff):
    out = img.copy()
    planes = out[..., None] if out.ndim == 2 else out
    total = img.shape[0] * img.shape[1]
    cutoff_pixels = int(np.trunc(np.float32(total) * np.float32(cutoff)))
    for k in range(min(planes.shape[2], 3)):
        hist = np.bincount(planes[..., k].ravel(), minlength=256)
        mn, mx = _np_cutoffs(hist, cutoff_pixels)
        v = np.arange(256)
        clamped = np.maximum(mn, np.minimum(mx, v))
        rng = np.float32(mx - mn if mx > mn else 1)
        norm = (clamped - mn).astype(np.float32) / rng
        scaled = norm * np.float32(255.0)
        lut = np.floor(scaled.astype(np.float64) + 0.5).astype(np.uint8)   # non-negative: half away == floor(x + .5)
        planes[..., k] = lut[planes[..., k]]
    return out


def np_equalize(img):
    out = img.copy()
    planes = out[..., None] if out.ndim == 2 else out
    total = img.shape[0] * img.shape[1]
    for k in range(planes.shape[2]):
        cdf = np.cumsum(np.bincount(planes[..., k].ravel(), minlength=256)).astype(np.int64)
        nz = cdf[cdf > 0]
        cdf_min = int(nz[0]) if nz.size else 0
        den = total - cdf_min
        if den == 0:
            lut = np.arange(256)
        else:
            lut = np.where(cdf >= cdf_min, (cdf - cdf_min) * 255 // den, 0)
        planes[..., k] = lut.astype(np.uint8)[planes[..., k]]
    return out


def _images():
    rng = np.random.default_rng(7)
    yield np.full((9, 13), 77, np.uint8)                                      # constant
    two = np.full((8, 10), 40, np.uint8)
    two[:, 5:] = 180
    yield two                                                                 # two values
    yield np.zeros((5, 6), np.uint8)                                          # only bin 0
    yield rng.integers(0, 256, (17, 23), dtype=np.uint8)
    yield (np.add.outer(np.arange(31), np.arange(29)) * 3 % 256).astype(np.uint8)
    yield rng.integers(30, 90, (11, 14, 3), dtype=np.uint8)
    yield rng.integers(0, 256, (12, 7, 4), dtype=np.uint8)


@pytest.mark.parametrize("cutoff", [0.0, 0.01, 0.2, 0.49])
def test_autocontrast_matches_numpy_restatement(cutoff):
    for img in _images():
        got = zo.autocontrast(img, cutoff)
        assert np.array_equal(got, np_autocontrast(img, cutoff)), (img.shape, cutoff)
        if img.ndim == 3 and img.shape[2] == 4:
            assert np.array_equal(got[..., 3], img[..., 3])                   # alpha untouched


def test_autocontrast_rejects_invalid_cutoff():
    img = np.zeros((3, 3), np.uint8)
    for bad in (0.5, -0.1, 0.75):
        with pytest.raises(zo.OracleStatus) as e:
            zo.autocontrast(img, bad)
        assert e.value.status == 21


def test_equalize_matches_numpy_restatement():
    for img in _images():
        got = zo.equalize(img)
        assert np.array_equal(got, np_equalize(img)), img.shape
    rgba = np.random.default_rng(3).integers(0, 256, (6, 9, 4), dtype=np.uint8)
    rgba[..., 3] = np.random.default_rng(4).integers(100, 140, (6, 9))
    assert not np.array_equal(zo.equalize(rgba)[..., 3], rgba[..., 3])       # alpha is equalized too
    assert np.array_equal(zo.autocontrast(rgba, 0.0)[..., 3], rgba[..., 3])


def test_equalize_uses_the_64_bit_numerator_above_the_u32_limit():
    # total - cdf_min > 16,843,009: (cdf - cdf_min) * 255 no longer fits u32; the oracle and the restatement use the exact product
    img = np.zeros((4200, 4200), np.uint8)
    img[:, 2100:] = np.arange(2100, dtype=np.uint32)[None, :].astype(np.uint8)
    img[:10] = 3
    got = zo.equalize(img)
    assert np.array_equal(got, np_equalize(img))


# ---- C-ABI errors decided on the host (no kernel is launched) ---------------------------------------------------------------------
def test_binary_status_names_and_argument_errors_before_the_device():
    L = zb.lib()
    for k, v in {21: "InvalidCutoff", 22: "InvalidRadius", 23: "InvalidKernelSize"}.items():
        assert L.zb_status_name(k).decode() == v
    a = np.zeros((12, 12), np.uint8)
    b = np.zeros((12, 13), np.uint8)
    ia, ib = zb.image._np_image(a), zb.image._np_image(b)
    empty = zb.image.ZbImage(None, 0, 4, 4)
    counts = (C.c_uint32 * 1024)()
    f32 = C.c_float
    assert L.zb_histogram(ia, 1, counts, None) == 3                                  # F32: not a histogram type (image.zig:1181)
    assert L.zb_histogram(ia, 4, counts, None) == 3
    counts[5] = 9
    assert L.zb_histogram(empty, 0, counts, None) == 0 and counts[5] == 0             # empty: all zero counts
    assert L.zb_autocontrast(ia, 1, f32(0.1), None) == 3                             # unsupported type before the cutoff check
    assert L.zb_autocontrast(ia, 0, f32(0.5), None) == 21                            # InvalidCutoff (enhancement.zig:16)
    assert L.zb_autocontrast(ia, 0, f32(-0.1), None) == 21
    assert L.zb_autocontrast(ia, 2, f32(float("nan")), None) == 21
    assert L.zb_autocontrast(empty, 0, f32(0.2), None) == 0
    assert L.zb_equalize(ia, 4, None) == 3
    assert L.zb_equalize(empty, 3, None) == 0
    huge = zb.image.ZbImage(None, 1 << 16, 1 << 16, 1 << 16)                          # 2^32 pixels: u32 counts would wrap
    assert L.zb_histogram(huge, 0, counts, None) == 3
    assert L.zb_equalize(huge, 0, None) == 3
    t = C.c_uint8(9)
    assert L.zb_threshold_otsu(ia, ib, C.byref(t), None) == 1                        # DimensionMismatch first (image.zig:849)
    assert L.zb_threshold_otsu(empty, empty, C.byref(t), None) == 0 and t.value == 0
    assert L.zb_threshold_adaptive_mean(ia, ib, 0, f32(1), None) == 1                # DimensionMismatch before InvalidRadius
    assert L.zb_threshold_adaptive_mean(ia, ia, 0, f32(1), None) == 22               # InvalidRadius (binary.zig:93)
    assert L.zb_threshold_adaptive_mean(empty, empty, 0, f32(1), None) == 22
    assert L.zb_threshold_adaptive_mean(empty, empty, 3, f32(1), None) == 0
    k = (C.c_uint8 * 9)(*([1] * 9))
    assert L.zb_morph_binary(ia, ib, k, 2, 3, 1, 0, None) == 23                      # even size: Kernel.init comes first
    assert L.zb_morph_binary(ia, ia, k, 3, 0, 1, 1, None) == 23                      # zero size
    assert L.zb_morph_binary(ia, ib, k, 3, 3, 1, 2, None) == 1                       # DimensionMismatch
    assert L.zb_morph_binary(ia, ia, k, 3, 3, 1, 7, None) == 5                       # unknown op
    assert L.zb_morph_binary(empty, empty, k, 3, 3, 2, 3, None) == 0
    big = (C.c_uint8 * (65 * 65))(*([1] * (65 * 65)))
    assert L.zb_morph_binary(ia, ia, big, 65, 65, 1, 0, None) == 3                   # beyond the shared-memory tile's halo


def test_python_mirror_rejects_non_u8_threshold_and_morphology():
    img = zb.Image(None, zb.PixFmt.RGB8, 4, 4, 4)
    for call in (lambda: img.threshold_otsu(), lambda: img.threshold_adaptive_mean(2, 1.0), lambda: img.dilate_binary(BOX3)):
        with pytest.raises(zb.ZignalError) as e:
            call()
        assert e.value.name == "Unsupported"


def test_oracle_error_order():
    a = np.zeros((4, 4), np.uint8)
    with pytest.raises(zo.OracleStatus) as e:
        zo.morph_binary(a, np.ones((2, 3), np.uint8), 1, "dilate", out=np.zeros((4, 5), np.uint8))
    assert e.value.status == 23
    with pytest.raises(zo.OracleStatus) as e:
        zo.threshold_adaptive_mean(a, 0, 1.0, out=np.zeros((4, 5), np.uint8))
    assert e.value.status == 1
    with pytest.raises(zo.OracleStatus) as e:
        zo.histogram(np.zeros((3, 3), np.float32))
    assert e.value.status == 3


def test_oracle_reproduces_binary_fixtures():
    """tests/golden/golden_binary.json (make_golden_binary.py): equalize, autocontrast, Otsu, the QR detector's adaptive threshold,
    open and close."""
    import json
    from pathlib import Path

    from golden_binary import CASES
    from gpu_utils import sha
    g = json.loads((Path(__file__).resolve().parent / "golden" / "golden_binary.json").read_text())
    assert set(g["cases"]) == set(CASES)
    for name, (build, oracle, _device) in CASES.items():
        img = build()
        assert sha(img) == g["cases"][name]["input_sha256"], name
        res = oracle(img)
        assert list(res.shape) == g["cases"][name]["shape"] and sha(res) == g["cases"][name]["output_sha256"], name
