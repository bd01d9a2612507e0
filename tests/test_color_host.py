"""CPU checks of the colour-format conversions: the oracle (oracle/zo_color.cpp) against the reference's own colour tests and an
independent numpy restatement, its agreement with the five-format oracle (zo_convert) on the 25 old pairs, and the argument and format
refusals of zb_convert_color and of the Image mirror, all reached without a device."""
import ctypes as C

import numpy as np
import pytest
import torch

import color_oracle as co
import oracle_lib as zo
import zignal_b200 as zb
from zignal_b200 import ColorFormat, ColorSpace as S, Component as K, PixFmt
from zignal_b200._ffi import ZbColorImage

RGB8, F64 = (int(S.RGB), 0), 2


def ulps(a, b):
    return abs(int(np.float64(a).view(np.int64)) - int(np.float64(b).view(np.int64)))


# Every testRoundTripConversion of color.zig ("primary", "secondary", "complementary", "neutral", "pastel" and "vivid colors",
# :1641-1725): Rgb(u8) -> X(f64), and the reference's X(f64) back to Rgb(u8).  The last column is the oracle's measured distance in
# ulp per component, held here.  Every Hsl, Hsv and L* value is bit-identical.  The misses are all in a* and b*: 500 (fx - fy) and
# 200 (fy - fz) turn one ulp of a cube root into several.  They stay the same whether the cube root is the oracle's restatement of
# std.math.pow, the host's pow, exp(y log x) or a correctly rounded cbrt, and with fused or unfused sums; for green the cube root's
# argument 35.76 / 95.047 is computed exactly as the reference computes it (gamma of 1.0 is 1.0).  So the reference's own pow(t, 1/3),
# built on Zig's compiler-rt exp and log, rounds those arguments differently from every correctly rounded restatement.
ROUND_TRIP_KATS = [
    ("red", (255, 0, 0), S.HSL, (0.0, 100.0, 50.0), (0, 0, 0)),
    ("red", (255, 0, 0), S.HSV, (0.0, 100.0, 100.0), (0, 0, 0)),
    ("red", (255, 0, 0), S.LAB, (53.23288178584245, 80.10930952982204, 67.22006831026425), (0, 0, 0)),
    ("green", (0, 255, 0), S.HSL, (120.0, 100.0, 50.0), (0, 0, 0)),
    ("green", (0, 255, 0), S.HSV, (120.0, 100.0, 100.0), (0, 0, 0)),
    ("green", (0, 255, 0), S.LAB, (87.73703347354422, -86.1846364976253, 83.18116474777855), (0, 4, 1)),
    ("blue", (0, 0, 255), S.HSL, (240.0, 100.0, 50.0), (0, 0, 0)),
    ("blue", (0, 0, 255), S.HSV, (240.0, 100.0, 100.0), (0, 0, 0)),
    ("blue", (0, 0, 255), S.LAB, (32.302586667249486, 79.19666178930935, -107.86368104495168), (0, 0, 0)),
    ("cyan", (0, 255, 255), S.HSL, (180.0, 100.0, 50.0), (0, 0, 0)),
    ("cyan", (0, 255, 255), S.HSV, (180.0, 100.0, 100.0), (0, 0, 0)),
    ("cyan", (0, 255, 255), S.LAB, (91.11652110946342, -48.079618466228716, -14.138127754846131), (0, 0, 0)),
    ("magenta", (255, 0, 255), S.HSL, (300.0, 100.0, 50.0), (0, 0, 0)),
    ("magenta", (255, 0, 255), S.HSV, (300.0, 100.0, 100.0), (0, 0, 0)),
    ("magenta", (255, 0, 255), S.LAB, (60.319933664076004, 98.25421868616108, -60.84298422386232), (0, 0, 0)),
    ("yellow", (255, 255, 0), S.HSL, (60.0, 100.0, 50.0), (0, 0, 0)),
    ("yellow", (255, 255, 0), S.HSV, (60.0, 100.0, 100.0), (0, 0, 0)),
    ("yellow", (255, 255, 0), S.LAB, (97.13824698129729, -21.555908334832285, 94.48248544644461), (0, 0, 0)),
    ("orange", (255, 136, 0), S.HSL, (32.0, 100.0, 50.0), (0, 0, 0)),
    ("orange", (255, 136, 0), S.HSV, (32.0, 100.0, 100.0), (0, 0, 0)),
    ("orange", (255, 136, 0), S.LAB, (68.65577208167872, 38.85052375564019, 74.99022544139406), (0, 7, 2)),
    ("purple", (128, 0, 128), S.HSL, (300.0, 100.0, 25.098039215686274), (0, 0, 0)),
    ("purple", (128, 0, 128), S.HSV, (300.0, 100.0, 50.19607843137255), (0, 0, 0)),
    ("purple", (128, 0, 128), S.LAB, (29.782100092098077, 58.93983731904206, -36.49792996282386), (0, 0, 0)),
    ("white", (255, 255, 255), S.HSL, (0.0, 0.0, 100.0), (0, 0, 0)),
    ("white", (255, 255, 255), S.HSV, (0.0, 0.0, 100.0), (0, 0, 0)),
    ("white", (255, 255, 255), S.LAB, (100.0, 0.00526049995830391, -0.010408184525267927), (0, 0, 0)),
    ("gray", (128, 128, 128), S.HSL, (0.0, 0.0, 50.19607843137255), (0, 0, 0)),
    ("gray", (128, 128, 128), S.HSV, (0.0, 0.0, 50.19607843137255), (0, 0, 0)),
    ("gray", (128, 128, 128), S.LAB, (53.58501345216902, 0.003155620347972121, -0.006243566036268078), (0, 0, 0)),
    ("black", (0, 0, 0), S.HSL, (0.0, 0.0, 0.0), (0, 0, 0)),
    ("black", (0, 0, 0), S.HSV, (0.0, 0.0, 0.0), (0, 0, 0)),
    ("black", (0, 0, 0), S.LAB, (0.0, 0.0, 0.0), (0, 0, 0)),
    ("pale_pink", (255, 211, 186), S.HSL, (21.739130434782602, 100.0, 86.47058823529412), (0, 0, 0)),
    ("pale_pink", (255, 211, 186), S.HSV, (21.739130434782602, 27.058823529411768, 100.0), (0, 0, 0)),
    ("pale_pink", (255, 211, 186), S.LAB, (87.67593388241974, 11.843797404960165, 18.16236917854479), (0, 0, 0)),
    ("mint_green", (150, 250, 150), S.HSL, (120.0, 90.90909090909089, 78.43137254901961), (0, 0, 0)),
    ("mint_green", (150, 250, 150), S.HSV, (120.0, 40.0, 98.0392156862745), (0, 0, 0)),
    ("mint_green", (150, 250, 150), S.LAB, (90.34795996024553, -48.75545372512652, 38.96689290268498), (0, 0, 0)),
    ("sky_blue", (138, 209, 237), S.HSL, (196.96969696969697, 73.33333333333336, 73.52941176470588), (0, 0, 0)),
    ("sky_blue", (138, 209, 237), S.HSV, (196.96969696969697, 41.77215189873419, 92.94117647058823), (0, 0, 0)),
    ("sky_blue", (138, 209, 237), S.LAB, (80.24627015828005, -15.11865203941365, -20.767024460106565), (0, 32, 6)),
    ("hot_pink", (255, 102, 179), S.HSL, (329.80392156862746, 99.99999999999997, 70.0), (0, 0, 0)),
    ("hot_pink", (255, 102, 179), S.HSV, (329.80392156862746, 60.0, 100.0), (0, 0, 0)),
    ("hot_pink", (255, 102, 179), S.LAB, (64.9763931162809, 65.40669278373645, -10.847761988977656), (0, 4, 0)),
    ("lime_green", (49, 204, 49), S.HSL, (120.0, 61.26482213438735, 49.6078431372549), (0, 0, 0)),
    ("lime_green", (49, 204, 49), S.HSV, (120.0, 75.98039215686275, 80.0), (0, 0, 0)),
    ("lime_green", (49, 204, 49), S.LAB, (72.26888334336961, -67.03378336285304, 61.425460443480894), (0, 0, 0)),
    ("electric_blue", (128, 223, 255), S.HSL, (195.11811023622047, 100.0, 75.09803921568627), (0, 0, 0)),
    ("electric_blue", (128, 223, 255), S.HSV, (195.11811023622047, 49.80392156862745, 100.0), (0, 0, 0)),
    ("electric_blue", (128, 223, 255), S.LAB, (84.26919487615707, -19.773688316136685, -24.252061008370738), (0, 16, 0)),
]


@pytest.mark.parametrize("name, rgb, space, want, max_ulps", ROUND_TRIP_KATS, ids=[f"{k[0]}-{k[2].name}" for k in ROUND_TRIP_KATS])
def test_oracle_reproduces_the_reference_round_trips(name, rgb, space, want, max_ulps):
    got = co.convert(np.array([rgb], np.uint8), RGB8, (int(space), F64))[0]
    assert tuple(ulps(g, w) for g, w in zip(got, want)) == max_ulps
    back = co.convert(np.array([want]), (int(space), F64), RGB8)[0]
    assert tuple(back) == rgb


def test_oracle_grayscale_cases():
    # "convert grayscale" (color.zig:1556-1562)
    g = lambda a, src: int(co.convert(np.array([a], dtype=co.NP[src[1]]), src, (int(S.GRAY), 0))[0])
    assert g((128, 128, 128), RGB8) == 128
    assert g((255, 0, 0), RGB8) == 54
    assert g((0.0, 100.0, 50.0), (int(S.HSL), F64)) == 54
    assert g((0.0, 100.0, 50.0), (int(S.HSV), F64)) == 27
    assert g((50.0, 0.0, 0.0), (int(S.LAB), F64)) == 119


def test_oracle_scalar_rules():
    # u8 -> float is v / 255 in the destination type; float -> u8 goes through f64 (color.zig:113-118)
    v = np.arange(256, dtype=np.uint8)
    assert np.array_equal(co.convert(v, (13, 0), (13, 1)), v.astype(np.float32) / np.float32(255))
    f = np.array([0.5 / 255, 1.5 / 255, 0.5, 254.5 / 255, -1.0, 2.0, np.nan], np.float32)
    want = np.round(np.clip(f.astype(np.float64), 0, 1) * 255)
    want[-1] = 255
    assert np.array_equal(co.convert(f, (13, 1), (13, 0)), want.astype(np.uint8))
    # Rgb(u8) -> f32 takes the fixed-point luma, then / 255; Rgb(u8) -> Gray(f32) the clamped float luma
    px = np.array([[200, 100, 50]], np.uint8)
    assert co.convert(px, RGB8, (13, 1))[0] == np.float32(co.convert(px, RGB8, (13, 0))[0]) / np.float32(255)
    f = px.astype(np.float32) / np.float32(255)
    y = np.float32(0.2126) * f[0, 0] + np.float32(0.7152) * f[0, 1] + np.float32(0.0722) * f[0, 2]
    assert co.convert(px, RGB8, (int(S.GRAY), 1))[0] == y


def test_reference_scalar_colors():
    # "scalar colors" (color.zig:1571-1583)
    assert tuple(co.convert(np.array([128], np.uint8), (13, 0), RGB8)[0]) == (128, 128, 128)
    assert tuple(co.convert(np.array([0.5]), (13, 2), RGB8)[0]) == (128, 128, 128)
    assert abs(co.convert(np.array([128], np.uint8), (13, 0), (13, 2))[0] - 128.0 / 255.0) <= 1e-7
    assert co.convert(np.array([0.5]), (13, 2), (13, 0))[0] == 128
    assert co.convert(np.array([0.25], np.float32), (13, 1), (13, 2))[0] == 0.25


def test_reference_color_space_convert():
    # "ColorSpace.convert" (color.zig:1787-1798), in f32
    red_hsv = np.array([[0.0, 100.0, 100.0]], np.float32)
    assert tuple(co.convert(red_hsv, (int(S.HSV), 1), RGB8)[0]) == (255, 0, 0)
    assert co.convert(red_hsv, (int(S.HSV), 1), (int(S.RGB), 1))[0].tolist() == [1.0, 0.0, 0.0]
    assert co.convert(np.array([[255, 0, 0]], np.uint8), RGB8, (int(S.HSV), 1))[0].tolist() == [0.0, 100.0, 100.0]


def test_reference_clamping():
    # "clamping out-of-range inputs" (color.zig:1854-1865)
    assert co.convert(np.array([-0.5], np.float32), (13, 1), (13, 0))[0] == 0
    assert co.convert(np.array([1.5], np.float32), (13, 1), (13, 0))[0] == 255
    assert tuple(co.convert(np.array([[1.2, -0.2, 0.5]], np.float32), (int(S.RGB), 1), RGB8)[0]) == (255, 0, 128)


def test_oracle_ycbcr_rules():
    # integer BT.601 for u8 (color.zig:987-1018, 1057-1067); (cb - 128) / 255 and + 0.5 at the float boundary (:955-975)
    px = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [128, 128, 128]], np.uint8)
    y = co.convert(px, RGB8, (int(S.YCBCR), 0))
    r, g, b = px.astype(np.int64).T
    want = np.stack([(19595 * r + 38470 * g + 7471 * b + 32768) >> 16,
                     ((-11059 * r - 21710 * g + 32768 * b + 32768) >> 16) + 128,
                     ((32768 * r - 27439 * g - 5329 * b + 32768) >> 16) + 128], -1).clip(0, 255)
    assert np.array_equal(y, want)
    f = co.convert(y, (int(S.YCBCR), 0), (int(S.YCBCR), 1))
    assert np.array_equal(f[:, 1], (y[:, 1].astype(np.float32) - np.float32(128)) / np.float32(255))
    # the two rules are not inverses: (cb - 128) / 255 + 0.5 can land below a half-integer, so the way back may lose one step
    assert np.abs(co.convert(f, (int(S.YCBCR), 1), (int(S.YCBCR), 0)).astype(int) - y).max() <= 1


def test_oracle_hue_mod_and_clamping():
    # @mod on a negative hue: a tiny negative value gives 0, not 360; Hsv hue and saturation clamp before the sectors
    hsv = np.array([[-1e-7, 50.0, 50.0], [-1e30, 50.0, 50.0], [720.0, 150.0, 150.0]])
    rgb = co.convert(hsv, (int(S.HSV), F64), (int(S.RGB), F64))
    assert np.all((rgb >= 0) & (rgb <= 1))
    h = co.convert(np.array([[1.0, 1.0, 1.0 - 1e-17]]), (int(S.RGB), F64), (int(S.HSV), F64))[0, 0]
    assert 0.0 <= h < 360.0


def test_random_colors_round_trip_over_the_cube():
    # "100 random colors" run over a strided pass of the whole cube: Rgb(u8) -> X(f64) -> Rgb(u8) gives the colour back
    v = np.arange(0, 1 << 24, 997, dtype=np.uint32)
    rgb = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8)
    for space in (S.HSL, S.HSV, S.XYZ, S.LAB, S.LCH, S.LMS, S.OKLAB, S.OKLCH, S.XYB, S.YCBCR):
        mid = co.convert(rgb, RGB8, (int(space), F64))
        assert np.array_equal(co.convert(mid, (int(space), F64), RGB8), rgb), space.name


def np_rgb_to_hsv(rgb):
    """Independent numpy restatement of rgbToHsv (color.zig:1087-1108) in the array's dtype."""
    t = rgb.dtype.type
    r, g, b = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    mx, mn = np.maximum(r, np.maximum(g, b)), np.minimum(r, np.minimum(g, b))
    d = mx - mn
    with np.errstate(divide="ignore", invalid="ignore"):
        h = np.where(mx == r, (g - b) / d * t(60), np.where(mx == g, t(120) + (b - r) / d * t(60), t(240) + (r - g) / d * t(60)))
        h = np.where(d == 0, t(0), h)
        m = np.fmod(h, t(360))
        h = np.where(h < 0, np.fmod(m + t(360), t(360)), m)
        s = np.where(mx == 0, t(0), (d / mx) * t(100))
    return np.stack([h, s, mx * t(100)], -1)


def np_rgb_to_xyz(rgb):
    """Independent numpy restatement of rgbToXyz (color.zig:1252-1272) with the host's pow."""
    t = rgb.dtype.type
    lin = np.where(rgb > t(0.04045), ((rgb + t(0.055)) / t(1.055)) ** t(2.4), rgb / t(12.92))
    r, g, b = lin[:, 0], lin[:, 1], lin[:, 2]
    return np.stack([(r * t(0.4124) + g * t(0.3576) + b * t(0.1805)) * t(100), (r * t(0.2126) + g * t(0.7152) + b * t(0.0722)) * t(100),
                     (r * t(0.0193) + g * t(0.1192) + b * t(0.9505)) * t(100)], -1)


@pytest.mark.parametrize("dtype, comp", [(np.float32, 1), (np.float64, 2)])
def test_oracle_against_numpy_restatement(dtype, comp):
    rgb = np.random.default_rng(1).uniform(-0.05, 1.05, (4000, 3)).astype(dtype)
    assert np.array_equal(co.convert(rgb, (int(S.RGB), comp), (int(S.HSV), comp)), np_rgb_to_hsv(rgb))   # bit for bit
    got = co.convert(rgb, (int(S.RGB), comp), (int(S.XYZ), comp))
    tol = 1e-5 if dtype == np.float32 else 1e-12
    assert np.max(np.abs(got - np_rgb_to_xyz(rgb))) <= tol * 100


def np_forward(space, v):
    """Independent numpy restatements of the Xyz-hub edges (color.zig:1275-1480), one column per component, in v's dtype; the
    transcendentals come from numpy (** for pow, np.cbrt, np.arctan2, np.cos, np.sin)."""
    t = v.dtype.type
    a, b, c = v[:, 0], v[:, 1], v[:, 2]
    if space == "xyz->lab":
        f = lambda u: np.where(u > t(0.008856), u ** t(1.0 / 3.0), t(7.787) * u + t(16.0 / 116.0))
        fx, fy, fz = f(a / t(95.047)), f(b / t(100.0)), f(c / t(108.883))
        return np.stack([np.maximum(t(0), t(116.0) * fy - t(16.0)), t(500.0) * (fx - fy), t(200.0) * (fy - fz)], -1)
    if space == "lab->xyz":
        fy = ((a + t(16.0)) / t(116.0)).astype(np.float64)
        fx = (b / t(500.0)).astype(np.float64) + fy
        fz = fy - (c / t(200.0)).astype(np.float64)
        g = lambda u: np.where(u * u * u > 0.008856, u * u * u, (u - 16.0 / 116.0) / 7.787)
        return np.stack([g(fx) * 95.047, g(fy) * 100.0, g(fz) * 108.883], -1).astype(v.dtype)
    if space in ("lab->lch", "oklab->oklch"):
        h = np.arctan2(c, b) * t(57.295779513082320876798154814105170332405472466564321549160243861)
        m = np.fmod(h, t(360.0))
        return np.stack([a, np.sqrt(b * b + c * c), np.where(h < 0, np.fmod(m + t(360.0), t(360.0)), m)], -1)
    if space in ("lch->lab", "oklch->oklab"):
        r = c * t(0.017453292519943295769236907684886127134428718885417254560971914)
        return np.stack([a, b * np.cos(r), b * np.sin(r)], -1)
    if space == "xyz->lms":
        return np.stack([(t(0.8951) * a + t(0.2664) * b - t(0.1614) * c) / t(100), (t(-0.7502) * a + t(1.7135) * b + t(0.0367) * c) / t(100),
                         (t(0.0389) * a - t(0.0685) * b + t(1.0296) * c) / t(100)], -1)
    if space == "lms->xyz":
        return np.stack([t(100) * (t(0.9869929) * a - t(0.1470543) * b + t(0.1599627) * c),
                         t(100) * (t(0.4323053) * a + t(0.5183603) * b + t(0.0492912) * c),
                         t(100) * (t(-0.0085287) * a + t(0.0400428) * b + t(0.9684867) * c)], -1)
    if space == "xyz->oklab":
        x, y, z = a / t(100.0), b / t(100.0), c / t(100.0)
        l_ = np.cbrt(t(0.8189330101) * x + t(0.3618667424) * y - t(0.1288597137) * z)
        m_ = np.cbrt(t(0.0329845436) * x + t(0.9293118715) * y + t(0.0361456387) * z)
        s_ = np.cbrt(t(0.0482003018) * x + t(0.2643662691) * y + t(0.6338517070) * z)
        return np.stack([t(0.2104542553) * l_ + t(0.7936177850) * m_ - t(0.0040720468) * s_,
                         t(1.9779984951) * l_ - t(2.4285922050) * m_ + t(0.4505937099) * s_,
                         t(0.0259040371) * l_ + t(0.7827717662) * m_ - t(0.8086757660) * s_], -1)
    if space == "oklab->xyz":
        l_ = a + t(0.3963377774) * b + t(0.2158037573) * c
        m_ = a - t(0.1055613458) * b - t(0.0638541728) * c
        s_ = a - t(0.0894841775) * b - t(1.2914855480) * c
        l3, m3, s3 = l_ * l_ * l_, m_ * m_ * m_, s_ * s_ * s_
        return np.stack([t(100.0) * (t(1.2270138511) * l3 - t(0.5577999807) * m3 + t(0.2812561490) * s3),
                         t(100.0) * (t(-0.0405801784) * l3 + t(1.1122568696) * m3 - t(0.0716766787) * s3),
                         t(100.0) * (t(-0.0763812845) * l3 - t(0.4214819784) * m3 + t(1.5861632204) * s3)], -1)
    r = (a * t(3.2406) + b * t(-1.5372) + c * t(-0.4986)) / t(100)
    g = (a * t(-0.9689) + b * t(1.8758) + c * t(0.0415)) / t(100)
    bl = (a * t(0.0557) + b * t(-0.2040) + c * t(1.0570)) / t(100)
    if space == "xyz->rgb":
        with np.errstate(invalid="ignore"):   # ** of the negative values np.where discards
            gam = lambda u: np.clip(np.where(u > t(0.0031308), t(1.055) * u ** t(1.0 / 2.4) - t(0.055), u * t(12.92)), t(0), t(1))
            return np.stack([gam(r), gam(g), gam(bl)], -1)
    bias = t(0.00379307325527544933)
    l_ = np.cbrt(np.maximum(t(0), t(0.30) * r + t(0.622) * g + t(0.078) * bl + bias)) - t(0.15595420054924863)
    m_ = np.cbrt(np.maximum(t(0), t(0.23) * r + t(0.692) * g + t(0.078) * bl + bias)) - t(0.15595420054924863)
    s_ = np.cbrt(np.maximum(t(0), t(0.24342268924547819) * r + t(0.20476744424496821) * g + t(0.5518098665095536) * bl + bias)) \
        - t(0.15595420054924863)
    return np.stack([t(0.5) * (l_ - m_), t(0.5) * (l_ + m_), s_], -1)   # xyz->xyb


# (edge, source space, destination space, input ranges, bit for bit?)
EDGES = [("xyz->lab", S.XYZ, S.LAB, [(0, 95), (0, 100), (0, 108)], False), ("lab->xyz", S.LAB, S.XYZ, [(0, 100), (-100, 100)] + [(-100, 100)], True),
         ("lab->lch", S.LAB, S.LCH, [(0, 100), (-100, 100), (-100, 100)], False), ("lch->lab", S.LCH, S.LAB, [(0, 100), (0, 120), (0, 360)], False),
         ("xyz->lms", S.XYZ, S.LMS, [(0, 95), (0, 100), (0, 108)], True), ("lms->xyz", S.LMS, S.XYZ, [(0, 1)] * 3, True),
         ("xyz->oklab", S.XYZ, S.OKLAB, [(0, 95), (0, 100), (0, 108)], False), ("oklab->xyz", S.OKLAB, S.XYZ, [(0, 1), (-0.3, 0.3), (-0.3, 0.3)], True),
         ("oklab->oklch", S.OKLAB, S.OKLCH, [(0, 1), (-0.3, 0.3), (-0.3, 0.3)], False),
         ("oklch->oklab", S.OKLCH, S.OKLAB, [(0, 1), (0, 0.3), (0, 360)], False),
         ("xyz->rgb", S.XYZ, S.RGB, [(0, 95), (0, 100), (0, 108)], False), ("xyz->xyb", S.XYZ, S.XYB, [(0, 95), (0, 100), (0, 108)], False)]


@pytest.mark.parametrize("dtype, comp", [(np.float32, 1), (np.float64, 2)], ids=["f32", "f64"])
@pytest.mark.parametrize("edge, src, dst, ranges, bitwise", EDGES, ids=[e[0] for e in EDGES])
def test_oracle_edges_against_numpy_restatement(edge, src, dst, ranges, bitwise, dtype, comp):
    rng = np.random.default_rng(5)
    v = np.stack([rng.uniform(lo, hi, 5000) for lo, hi in ranges], -1).astype(dtype)
    got = co.convert(v, (int(src), comp), (int(dst), comp))
    want = np_forward(edge, v)
    if bitwise:
        assert np.array_equal(got, want)
        return
    span = {S.LAB: (100, 256, 256), S.LCH: (100, 150, 360), S.OKLAB: (1, 1, 1), S.OKLCH: (1, 1, 360), S.RGB: (1, 1, 1), S.XYB: (1, 1, 1)}[dst]
    tol = 1e-4 if dtype == np.float32 else 1e-12
    for k in range(3):
        d = np.abs(got[:, k].astype(np.float64) - want[:, k].astype(np.float64))
        if k == 2 and dst in (S.LCH, S.OKLCH):   # hue modulo 360, where the chroma is at least 1 % of its span
            d = np.minimum(d % 360, 360 - d % 360)[want[:, 1] >= 0.01 * span[1]]
        assert d.max() <= tol * span[k], (edge, k, d.max())


OLD = {PixFmt.U8: ((13, 0), np.uint8, 1), PixFmt.F32: ((13, 1), np.float32, 1), PixFmt.RGB8: ((8, 0), np.uint8, 3),
       PixFmt.RGBA8: ((9, 0), np.uint8, 4), PixFmt.RGBAF32: ((9, 1), np.float32, 4)}


@pytest.mark.parametrize("src", list(OLD), ids=lambda p: p.name)
def test_oracle_agrees_with_the_five_format_oracle(src):
    (fmt, dt, ch) = OLD[src]
    rng = np.random.default_rng(int(src))
    shape = (23, 31) + ((ch,) if ch > 1 else ())
    a = rng.integers(0, 256, shape).astype(dt) if dt == np.uint8 else rng.uniform(-0.1, 1.1, shape).astype(dt)
    if dt != np.uint8:
        a.reshape(-1)[:6] = [np.nan, np.inf, -np.inf, -0.0, 0.5 / 255, 1e-40]
    for dst, (dfmt, _, _) in OLD.items():
        if dst == src:
            continue
        want = zo.convert(a, dst)
        got = co.convert(a, fmt, dfmt)
        assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), (src.name, dst.name)


def test_the_33_formats():
    fmts = ColorFormat.all()
    assert len(fmts) == 33 and len(set(fmts)) == 33
    for s in range(14):
        for c in range(3):
            assert co.valid(s, c) == ColorFormat(S(s), K(c)).valid
    assert not co.valid(14, 1) and not co.valid(3, 3) and not co.valid(-1, 0)


# ---- refusals of zb_convert_color, all decided before any device work ----

def call(src, dst):
    return zb.lib().zb_convert_color(C.byref(src) if src is not None else None, C.byref(dst) if dst is not None else None, None)


def cimg(space, comp, rows=4, cols=4, data=1 << 20, stride=None):
    return ZbColorImage(data, rows, cols, cols if stride is None else stride, int(space), int(comp))


def test_null_arguments():
    a = cimg(S.RGB, 0)
    assert call(None, a) == 5 and call(a, None) == 5


@pytest.mark.parametrize("space, comp", [(S.LAB, 0), (S.HSV, 0), (S.XYB, 0), (14, 1), (-1, 1), (S.RGB, 3), (S.RGB, -1)])
def test_invalid_formats_are_unsupported(space, comp):
    good = cimg(S.RGB, 1, data=1 << 30)
    bad = cimg(space, comp, data=1 << 20)
    assert call(bad, good) == 3 and call(good, bad) == 3


def test_every_invalid_pair_is_refused():
    good = [(s, c) for s in range(14) for c in range(3) if co.valid(s, c)]
    bad = [(s, c) for s in range(-1, 15) for c in range(-1, 4) if not co.valid(s, c)]
    for s in good:
        for b in bad:
            assert call(cimg(*s, data=1 << 20), cimg(*b, data=1 << 30)) == 3
            assert call(cimg(*b, data=1 << 20), cimg(*s, data=1 << 30)) == 3


def test_shape_alignment_and_overlap():
    assert call(cimg(S.RGB, 0, 4, 4), cimg(S.LAB, 1, 4, 5, data=1 << 30)) == 1
    assert call(cimg(S.RGB, 0, 4, 4), cimg(S.LAB, 1, 5, 4, data=1 << 30)) == 1
    # a data pointer not aligned to its component: InvalidArgument
    assert call(cimg(S.RGB, 1, data=(1 << 20) + 2), cimg(S.LAB, 1, data=1 << 30)) == 5
    assert call(cimg(S.RGB, 0, data=(1 << 20) + 1), cimg(S.LAB, 2, data=(1 << 30) + 4)) == 5
    # overlapping views with different pixel sizes, or shifted views of one buffer: InvalidArgument
    assert call(cimg(S.RGB, 1), cimg(S.LAB, 2, data=(1 << 20) + 8)) == 5
    assert call(cimg(S.RGB, 1), cimg(S.LAB, 1, data=(1 << 20) + 12)) == 5


@pytest.mark.parametrize("cls, rows, cols, src, dst", [
    ("W1", 1, (1 << 31) + 80, (S.GRAY, 0), (S.GRAY, 1)),      # a row of 2^31 px
    ("W4", 1, (1 << 29) + 80, (S.RGBA, 0), (S.LAB, 1)),       # a row of 2^31 bytes
    ("T1", (1 << 31) + 80, 1, (S.RGB, 0), (S.YCBCR, 0))])     # 2^31 rows
def test_index_range_is_refused(cls, rows, cols, src, dst):
    a = ZbColorImage(1 << 20, rows, cols, cols, int(src[0]), src[1])
    b = ZbColorImage(1 << 50, rows, cols, cols, int(dst[0]), dst[1])
    assert call(a, b) == 3, cls


# ---- the Image mirror refuses every other method on an image of a new format ----

def host_image(fmt):
    return zb.Image(torch.zeros(16 * fmt.channels, dtype=getattr(torch, np.dtype(fmt.dtype).name)), fmt, 4, 4, 4)


@pytest.mark.parametrize("fmt", [f for f in ColorFormat.all() if f not in (ColorFormat(S.SCALAR, K.U8), ColorFormat(S.SCALAR, K.F32),
                                                                          ColorFormat(S.RGB, K.U8), ColorFormat(S.RGBA, K.U8),
                                                                          ColorFormat(S.RGBA, K.F32))], ids=lambda f: f.name)
def test_other_methods_refuse_new_formats(fmt):
    img = host_image(fmt)
    assert img.format == fmt
    with pytest.raises(TypeError):
        img.pixfmt
    calls = [lambda: img.gaussian_blur(1.0), lambda: img.box_blur(1), lambda: img.sobel(), lambda: img.histogram(), lambda: img.invert(),
             lambda: img.flip_left_right(), lambda: img.dupe(), lambda: img.apply_colormap(zb.Colormap(0)), lambda: img.psnr(img),
             lambda: img.resize(img), lambda: img.copy(img), lambda: img.encode_jpeg(), lambda: img.median_blur(1),
             lambda: img.canny(1.0, 0.1, 0.2), lambda: img.threshold_otsu(), lambda: img.diff(img)]
    for f in calls:
        with pytest.raises(TypeError):
            f()
    v = img.view(zb.Rectangle(1, 1, 3, 3))
    assert v.format == fmt and (v.rows, v.cols) == (2, 2)
    assert v.to_numpy().shape == (2, 2) + ((fmt.channels,) if fmt.channels > 1 else ())


def test_invalid_format_and_mismatched_arrays():
    with pytest.raises(TypeError):
        zb.Image(torch.zeros(48, dtype=torch.uint8), ColorFormat(S.LAB, K.U8), 4, 4, 4)
    with pytest.raises(TypeError):
        zb.Image.from_numpy(np.zeros((4, 4, 3), np.float32), format=ColorFormat(S.LAB, K.F64))
    with pytest.raises(TypeError):
        zb.Image.from_numpy(np.zeros((4, 4, 4), np.float32), format=ColorFormat(S.LAB, K.F32))
