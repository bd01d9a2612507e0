"""The [0, 1] clamp of float -> 8-bit conversions in the CPU oracle, against values derived by hand from the reference's definitions
(no GPU).  The reference clamps with std.math.clamp(v, 0, 1) = @max(0, @min(v, 1)), and Zig's @min / @max return the non-NaN
operand, so NaN clamps to 1: 255 in u8.  Then:
  * a float scalar to u8 is @round(clamp(v, 0, 1) * 255) in f64 (color.zig:114-118): Image.convert, and the gray plane of Canny and
    Shen-Castan on Image(f32) (as(f32, convertColor(u8, v)));
  * a float component to u8 is @round(255 * clamp(v, 0, 1)) in f32 (color.zig:376-379, 496-501, 553);
  * Rgba(f32) to a scalar is the luma clamp(0.2126 r + 0.7152 g + 0.0722 b, 0, 1) in f32 (color.zig:1043-1045), then the rule above.
@round rounds half away from zero, so the ties (k + 1/2) / 255 are included."""
import numpy as np
import pytest

import oracle_lib as zo
import shen_castan_oracle as sco

F32 = np.float32
NAN_NEG = np.array([0xFFC00000], np.uint32).view(F32)[0]           # quiet NaN with the sign bit set
SPECIAL = np.array([np.nan, NAN_NEG, np.inf, -np.inf, 0.0, -0.0, np.nextafter(F32(1), F32(2)), -np.nextafter(F32(0), F32(1)),
                    np.nextafter(F32(0), F32(1)), np.finfo(F32).max, -np.finfo(F32).max, 1e30, 1.0, 0.5], F32)
TIES = ((np.arange(255) + 0.5) / 255).astype(F32)


def _round_half_away(x):
    x = np.asarray(x, np.float64)
    return np.sign(x) * np.floor(np.abs(x) + 0.5)


def _clamp01(v):
    """@max(0, @min(v, 1)) with Zig's NaN rule, elementwise in v's own type.  The reference's @max leaves the sign of a zero open;
    the project pins +0 for -0 (and for every value <= 0)."""
    v = np.asarray(v)
    t = v.dtype.type
    return np.where(np.isnan(v), t(1), np.where(v > 0, np.minimum(v, t(1)), t(0)))


def _scalar_to_u8(v):
    """convertColor(u8, f32 v): through f64."""
    return _round_half_away(_clamp01(np.asarray(v, np.float64)) * 255.0).astype(np.uint8)


def _component_to_u8(v):
    """Gray / Rgb / Rgba(f32).as(u8): 255 * clamp(v) rounded to f32, then @round."""
    prod = (F32(255) * _clamp01(np.asarray(v, F32))).astype(F32)
    return _round_half_away(prod).astype(np.uint8)


def _values():
    return np.concatenate([SPECIAL, TIES])


def test_hand_rule_on_named_values():
    """The derivation helpers themselves, on the values the issue of NaN is about."""
    got = _scalar_to_u8(SPECIAL[:8])
    assert got.tolist() == [255, 255, 255, 0, 0, 0, 255, 0]
    assert _component_to_u8(SPECIAL[:8]).tolist() == [255, 255, 255, 0, 0, 0, 255, 0]
    assert _scalar_to_u8(np.array([0.5], F32)).tolist() == [128]          # 127.5 rounds away from zero


def test_convert_f32_to_u8():
    v = _values().reshape(1, -1)
    got = zo.convert(v, zo.PIX_U8)
    assert np.array_equal(got, _scalar_to_u8(v)), np.nonzero(got != _scalar_to_u8(v))


@pytest.mark.parametrize("dst", [zo.PIX_RGB8, zo.PIX_RGBA8])
def test_convert_f32_to_colour(dst):
    """Gray(f32).as(u8).to(rgb[a]): the f32 component rule, alpha 255."""
    v = _values().reshape(1, -1)
    got = zo.convert(v, dst)
    y = _component_to_u8(v)
    assert np.array_equal(got[..., 0], y) and np.array_equal(got[..., 1], y) and np.array_equal(got[..., 2], y)
    if dst == zo.PIX_RGBA8:
        assert (got[..., 3] == 255).all()


@pytest.mark.parametrize("dst", [zo.PIX_RGB8, zo.PIX_RGBA8])
def test_convert_rgbaf32_to_colour(dst):
    """Rgba(f32).to(space).as(u8): every component, alpha included, by the f32 component rule; the special values sit in every
    channel position."""
    v = _values()
    img = np.stack([np.roll(v, k) for k in range(4)], axis=-1).reshape(1, -1, 4)
    got = zo.convert(img, dst)
    want = _component_to_u8(img)
    n = 4 if dst == zo.PIX_RGBA8 else 3
    assert np.array_equal(got, want[..., :n])


def _luma_f32(r, g, b):
    r, g, b = (np.asarray(x, F32) for x in (r, g, b))
    with np.errstate(invalid="ignore", over="ignore"):
        return ((F32(0.2126) * r + F32(0.7152) * g).astype(F32) + F32(0.0722) * b).astype(F32)


def test_convert_rgbaf32_luma():
    """Rgba(f32) -> u8 / f32: the clamped f32 luma.  (Inf, -Inf, 0) sums to NaN, which clamps to 1.0 (255)."""
    px = np.array([[np.inf, -np.inf, 0, 1], [np.nan, 0, 0, 1], [-np.inf, 0, 0, 1], [np.inf, 0, 0, 1], [0, np.nan, np.inf, 0],
                   [1, 1, 1, 1], [-0.0, -0.0, -0.0, 1], [2, -1, 0.5, 0], [np.finfo(F32).max, np.finfo(F32).max, 0, 1]], F32)
    img = px.reshape(1, -1, 4)
    y = _clamp01(_luma_f32(px[:, 0], px[:, 1], px[:, 2]))
    assert y[0] == 1.0 and not np.signbit(y[6])                             # NaN -> 1, -0 -> +0
    got_f = zo.convert(img, zo.PIX_F32)[0]
    assert np.array_equal(got_f.view(np.uint32), y.astype(F32).view(np.uint32)), (got_f, y)
    got_u = zo.convert(img, zo.PIX_U8)[0]
    assert got_u[0] == 255
    assert np.array_equal(got_u, _component_to_u8(y))


def _nan_image(rng, rows, cols):
    img = rng.random((rows, cols), dtype=F32)
    img[rng.random((rows, cols)) < 0.05] = np.nan
    img[5, :] = np.nan                                                      # a whole row
    img[:, 7] = np.inf
    img[rows - 9, 3:20] = -np.inf
    img[0, 0] = img[rows - 1, cols - 1] = NAN_NEG
    img[20:24, 30:34] = 1.5
    img[30, 10:20] = -0.0
    return img


def test_canny_f32_equals_canny_of_clamped_u8():
    """Canny on Image(f32) reads as(f32, convertColor(u8, v)): the same edges as Canny on the u8 image the scalar rule gives."""
    img = _nan_image(np.random.default_rng(5), 64, 80)
    gray = _scalar_to_u8(img)
    for sigma, lo, hi in ((1.0, 20.0, 60.0), (0.0, 10.0, 40.0)):
        assert np.array_equal(zo.canny(img, sigma, lo, hi), zo.canny(gray, sigma, lo, hi)), sigma


def test_shen_castan_f32_equals_shen_castan_of_clamped_u8():
    img = _nan_image(np.random.default_rng(6), 64, 80)
    gray = _scalar_to_u8(img)
    for o in (sco.Options(), sco.Options(use_nms=True)):
        assert np.array_equal(sco.shen_castan(img, o), sco.shen_castan(gray, o)), o
