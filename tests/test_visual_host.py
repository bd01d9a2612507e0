"""CPU tests of Image.diff, applyColormap, the flips and invert: the reference's own tests as known answers, the oracle against an
independent numpy restatement over every option combination, the turbo table's summation order, and the C ABI's argument errors
(decided before any device work, so no GPU is needed)."""
import ctypes as C
import json
import math
from fractions import Fraction

import numpy as np
import pytest

import visual_oracle as zo
from golden_visual import FORMATS, PIX, near_pair, random_image

F32_MAX = np.finfo(np.float64).max


# ---- independent restatement -----------------------------------------------------------------------------------------------------------

def round_half_away(x):
    x = np.asarray(x, np.float64)
    return np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5))


def np_diff(a, b, threshold, scale, binary, force_opaque):
    """diff.zig restated over whole arrays: (out, samples, diff_count)."""
    flt = a.dtype == np.float32
    a3, b3 = (a, b) if a.ndim == 3 else (a[..., None], b[..., None])
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.abs(a3 - b3) if flt else np.abs(a3.astype(np.int16) - b3).astype(np.float32)
        differs = (d > np.float32(threshold)).any(axis=2)
        maxv = 1.0 if flt else 255
        if binary:
            v = np.broadcast_to(np.where(differs[..., None], maxv, 0), d.shape).astype(a.dtype)
        else:
            s = (d * np.float32(scale)).astype(np.float32)
            v = s if flt else np.where(np.isnan(s), 255, np.clip(round_half_away(s), 0, 255)).astype(np.uint8)
        v = np.array(v)
        ch = v.shape[2]
        if ch == 1:
            samples = v[..., 0].astype(np.float64)
        else:
            used = v[..., :3] if (force_opaque and ch == 4) else v
            samples = np.fmax(0.0, np.fmax.reduce(used.astype(np.float64), axis=2))
        if force_opaque and ch == 4:
            v[..., 3] = maxv
    out = v if a.ndim == 3 else v[..., 0]
    return out, samples.reshape(-1), int(differs.sum())


def exact_stats(samples):
    """Exact sum, mean and variance of finite samples (Fractions)."""
    fr = [Fraction(float(x)) for x in samples]
    n = len(fr)
    s = sum(fr)
    mean = s / n if n else Fraction(0)
    var = sum((x - mean) ** 2 for x in fr) / (n - 1) if n > 1 else Fraction(0)
    return s, mean, var


def scalar_values(img):
    """meta.as(f64, px) / convertColor(f64, px) (image.zig:1217)."""
    if img.ndim == 2:
        return img.astype(np.float64)
    if img.dtype == np.uint8:
        r, g, b = (img[..., k].astype(np.int64) for k in range(3))
        y = np.clip((13933 * r + 46871 * g + 4732 * b + 32768) >> 16, 0, 255)
        return y.astype(np.float64) / 255.0
    r, g, b = (img[..., k] for k in range(3))
    with np.errstate(invalid="ignore", over="ignore"):
        l = (np.float32(0.2126) * r + np.float32(0.7152) * g) + np.float32(0.0722) * b
    return np.fmax(np.float32(0), np.fmin(l, np.float32(1))).astype(np.float64)


def np_colormap(img, lut, mn=None, mx=None):
    v = scalar_values(img)
    if mn is None or mx is None:
        if v.size == 0:
            lo, hi = 0.0, 1.0
        else:
            lo, hi = np.fmin(F32_MAX, np.fmin.reduce(v, axis=None)), np.fmax(-F32_MAX, np.fmax.reduce(v, axis=None))
        mn = lo if mn is None else mn
        mx = hi if mx is None else mx
    if mx <= mn:
        mx = mn + 1.0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        bad = np.isnan(v) | math.isnan(mn) | math.isnan(mx) | (mx <= mn)
        t = np.where(bad, 0.0, np.fmax(0.0, np.fmin((v - mn) / (mx - mn), 1.0)))
    idx = round_half_away(t * 255.0).astype(np.int64)
    return np.asarray(lut, np.uint8)[idx]


def np_invert(img):
    if img.dtype == np.uint8:
        out = 255 - img
        if img.ndim == 3 and img.shape[2] == 4:
            out[..., 3] = img[..., 3]
        return out
    out = (np.float32(1) - img).astype(np.float32)
    out[..., 3] = img[..., 3]
    return out


def same_bits(x, y):
    """Bit-identical arrays, except that a NaN matches any NaN: the sign and payload a NaN carries out of an arithmetic operation are
    the hardware's (x86 and CUDA differ) and no zignal result depends on them."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    if x.dtype != y.dtype or x.shape != y.shape:
        return False
    if x.dtype.kind == "f":
        nx, ny = np.isnan(x), np.isnan(y)
        if not np.array_equal(nx, ny):
            return False
        x, y = np.where(nx, 0, x).astype(x.dtype), np.where(ny, 0, y).astype(y.dtype)
    return np.array_equal(x.view(np.uint8), y.view(np.uint8))


# ---- the reference's own tests -----------------------------------------------------------------------------------------------------

def test_invert_kat():                                                   # image/tests/filters.zig:16-48
    gray = np.array([[0, 255], [100, 128]], np.uint8)
    assert zo.invert(gray).tolist() == [[255, 0], [155, 127]]
    rgb = np.array([[[0, 128, 255]]], np.uint8)
    assert zo.invert(rgb).tolist() == [[[255, 127, 0]]]
    rgba = np.array([[[0, 128, 255, 64]]], np.uint8)
    assert zo.invert(rgba).tolist() == [[[255, 127, 0, 64]]]


def test_flip_kats():                                                    # image/tests/transforms.zig:427-456
    img = np.array([[1, 2, 3], [4, 5, 6]], np.uint8)
    assert zo.flip_left_right(img).tolist() == [[3, 2, 1], [6, 5, 4]]
    img = np.array([[1, 2], [3, 4], [5, 6]], np.uint8)
    assert zo.flip_top_bottom(img).tolist() == [[5, 6], [3, 4], [1, 2]]


def test_colormaps_kat():                                                # image/colormaps.zig:711-812
    gradient = np.arange(256, dtype=np.uint8)[None, :]
    jet = zo.apply_colormap(gradient, zo.colormap_lut(zo.JET))
    assert jet[0, 0].tolist() == [0, 0, 128] and jet[0, 128, 1] == 255 and jet[0, 255].tolist() == [128, 0, 0]
    heat = zo.apply_colormap(gradient, zo.colormap_lut(zo.HEAT))
    assert heat[0, 0].tolist() == [0, 0, 0] and heat[0, 255].tolist() == [255, 255, 255]
    turbo = zo.apply_colormap(gradient, zo.colormap_lut(zo.TURBO))
    assert np.all(np.abs(turbo[0, 0].astype(int) - [35, 23, 27]) <= 1)
    assert np.all(np.abs(turbo[0, 255].astype(int) - [144, 13, 0]) <= 2)
    viridis = zo.apply_colormap(gradient, zo.colormap_lut(zo.VIRIDIS))
    assert viridis[0, 0].tolist() == [68, 1, 84] and viridis[0, 255].tolist() == [253, 231, 37]
    inferno = zo.apply_colormap(gradient, zo.colormap_lut(zo.INFERNO))
    assert inferno[0, 0].tolist() == [0, 0, 4] and inferno[0, 255].tolist() == [252, 255, 164]
    clamped = zo.apply_colormap(gradient, zo.colormap_lut(zo.JET), 0.0, 128.0 / 255.0)
    assert clamped[0, 128].tolist() == [128, 0, 0] and clamped[0, 255].tolist() == [128, 0, 0]


def test_colormap_nan_safety():                                          # colormaps.zig:814-823: index 0 for a NaN value
    img = np.array([[np.nan, 0.5]], np.float32)
    for m in range(5):
        lut = zo.colormap_lut(m)
        out = zo.apply_colormap(img, lut, 0.0, 1.0)
        assert out[0, 0].tolist() == lut[0].tolist()


def test_colormap_on_view():                                             # colormaps.zig:825-847: the range comes from the view only
    img = np.zeros((10, 10), np.uint8)
    img[0, 0] = 255
    v = img[4:6, 4:6]
    v[...] = 128
    vis = zo.apply_colormap(v, zo.colormap_lut(zo.JET))
    assert vis[0, 0].tolist() == [0, 0, 128]


def test_cli_call():                                                     # cli/diff.zig:86-104: Rgba(u8), force_opaque, integer threshold
    a, b = near_pair("rgba8", 40, 50, 3)
    out, st = zo.diff(a, b, threshold=2.0, scale=1.0, binary=False, force_opaque=True)
    assert np.all(out[..., 3] == 255)
    assert st["max"] == np.abs(a[..., :3].astype(int) - b[..., :3]).max()
    assert st["diff_count"] == int((np.abs(a.astype(int) - b) > 2).any(axis=2).sum())


# ---- the oracle against the restatement ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("force_opaque", [False, True])
@pytest.mark.parametrize("threshold,scale", [(0.0, 1.0), (2.0, 1.0), (0.125, 3.5), (1.0, -2.0), (0.0, 1e30), (0.0, float("nan")),
                                             (float("nan"), 1.0), (-1.0, 0.5)])
def test_diff_oracle_matches_numpy(fmt, binary, force_opaque, threshold, scale):
    a, b = near_pair(fmt, 23, 37, 100 + PIX[fmt])
    out, st = zo.diff(a, b, threshold, scale, binary, force_opaque)
    want, samples, count = np_diff(a, b, threshold, scale, binary, force_opaque)
    assert same_bits(out, want)
    assert st["n"] == samples.size and st["diff_count"] == count
    finite = samples[np.isfinite(samples)]
    if finite.size == samples.size:
        s, mean, var = exact_stats(samples)
        assert st["min"] == samples.min() and st["max"] == samples.max()
        assert st["sum"] == pytest.approx(float(s), rel=1e-12, abs=1e-300)
        assert st["mean"] == pytest.approx(float(mean), rel=1e-9, abs=1e-300)
        assert st["variance"] == pytest.approx(float(var), rel=1e-9, abs=1e-300)
        if a.dtype == np.uint8:
            assert st["sum"] == float(s)                                  # integer samples: the f64 sum is exact


def test_diff_threshold_at_a_difference_value():
    a = np.array([[10, 10, 10]], np.uint8)
    b = np.array([[12, 13, 10]], np.uint8)
    out, st = zo.diff(a, b, threshold=2.0, binary=True)
    assert out.tolist() == [[0, 255, 0]] and st["diff_count"] == 1


def test_diff_f32_specials():
    a = random_image("f32", 16, 16, 7, specials=True)
    b = random_image("f32", 16, 16, 8, specials=True)
    out, st = zo.diff(a, b, 0.1, 2.0)
    want, samples, count = np_diff(a, b, 0.1, 2.0, False, False)
    assert same_bits(out, want) and st["diff_count"] == count
    assert math.isnan(st["sum"]) and math.isnan(st["mean"])               # a NaN sample enters the sum and the moments ...
    assert st["min"] == np.fmin.reduce(samples) and st["max"] == np.fmax.reduce(samples)   # ... but not the extrema


def test_diff_rgba_nan_channel_never_enters_sample():
    a = np.array([[[np.nan, 0.5, 0.0, 1.0]]], np.float32)
    b = np.zeros((1, 1, 4), np.float32)
    out, st = zo.diff(a, b)
    assert math.isnan(out[0, 0, 0]) and st["max"] == 1.0 and st["sum"] == 1.0


def test_diff_alpha_counts_under_force_opaque():
    a = np.array([[[5, 5, 5, 0]]], np.uint8)
    b = np.array([[[5, 5, 5, 200]]], np.uint8)
    out, st = zo.diff(a, b, threshold=10.0, binary=True, force_opaque=True)
    assert out.tolist() == [[[255, 255, 255, 255]]] and st["diff_count"] == 1 and st["max"] == 255


def test_diff_empty_and_single():
    e = np.zeros((0, 5), np.uint8)
    _, st = zo.diff(e, e)
    assert st == {"n": 0, "diff_count": 0, "sum": 0.0, "mean": 0.0, "variance": 0.0, "min": 0.0, "max": 0.0}
    _, st = zo.diff(np.array([[3]], np.uint8), np.array([[7]], np.uint8))
    assert st["n"] == 1 and st["variance"] == 0.0 and st["mean"] == 4.0


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("cmap", range(5))
@pytest.mark.parametrize("rng_", [(None, None), (0.1, None), (None, 0.7), (0.25, 0.75), (0.9, 0.1), (float("nan"), 1.0),
                                  (0.0, float("nan")), (-1e300, 1e300), (5.0, 5.0)])
def test_colormap_oracle_matches_numpy(fmt, cmap, rng_):
    img = random_image(fmt, 19, 29, 200 + PIX[fmt], specials=True)
    lut = zo.colormap_lut(cmap)
    assert np.array_equal(zo.apply_colormap(img, lut, *rng_), np_colormap(img, lut, *rng_))


@pytest.mark.parametrize("fmt", FORMATS)
def test_colormap_constant_empty_and_all_nan(fmt):
    lut = zo.colormap_lut(zo.TURBO)
    const = np.ascontiguousarray(np.broadcast_to(random_image(fmt, 1, 1, 5), (4, 6) + random_image(fmt, 1, 1, 5).shape[2:]))
    assert np.array_equal(zo.apply_colormap(const, lut), np_colormap(const, lut))
    assert zo.apply_colormap(random_image(fmt, 0, 3, 1), lut).shape == (0, 3, 3)
    if fmt == "f32":
        nan = np.full((3, 3), np.nan, np.float32)
        assert np.array_equal(zo.apply_colormap(nan, lut), np_colormap(nan, lut))
        inf = np.full((2, 2), np.inf, np.float32)                      # min stays floatMax: (inf - max) / (inf - max) is NaN -> 1
        assert np.array_equal(zo.apply_colormap(inf, lut), np.broadcast_to(lut[255], (2, 2, 3)))


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("shape", [(1, 1), (1, 8), (7, 1), (5, 6), (6, 7)])
def test_flips_and_invert_match_numpy(fmt, shape):
    img = random_image(fmt, *shape, seed=shape[0] * 10 + shape[1], specials=True)
    assert same_bits(zo.flip_left_right(img.copy()), img[:, ::-1])
    assert same_bits(zo.flip_top_bottom(img.copy()), img[::-1])
    if fmt == "f32":
        with pytest.raises(Exception):
            zo.invert(img.copy())
    else:
        assert same_bits(zo.invert(img.copy()), np_invert(img))


def test_flip_on_view_leaves_the_rest():
    base = np.arange(8 * 9, dtype=np.uint8).reshape(8, 9)
    img = base.copy()
    zo.flip_left_right(img[2:5, 1:8])
    want = base.copy()
    want[2:5, 1:8] = base[2:5, 1:8][:, ::-1]
    assert np.array_equal(img, want)


# ---- LUT data ------------------------------------------------------------------------------------------------------------------------

_TURBO = ((0.13572138, 4.61539260, -42.66032258, 132.13108234, -152.94239396, 59.28637943),
          (0.09140261, 2.19418839, 4.84296658, -14.18503333, 4.27729857, 2.82956604),
          (0.10667330, 12.64194608, -60.58204836, 110.36276771, -89.90310912, 27.34824973))


def _turbo_table(order):
    out = np.zeros((256, 3), np.uint8)
    for i in range(256):
        t = i / 255.0
        t2 = t * t
        t3 = t2 * t
        t4 = t3 * t
        t5 = t4 * t
        v = (1.0, t, t2, t3, t4, t5)
        for ch in range(3):
            p = [v[k] * _TURBO[ch][k] for k in range(6)]
            if order == "left":
                acc = p[0]
                for x in p[1:]:
                    acc = acc + x
            elif order == "pairwise":
                acc = ((p[0] + p[1]) + (p[2] + p[3])) + (p[4] + p[5])
            else:                                                        # halves, as a vector reduction folds lanes
                q = [p[0] + p[3], p[1] + p[4], p[2] + p[5]]
                acc = (q[0] + q[1]) + q[2]
            c = max(0.0, min(acc, 1.0))
            out[i, ch] = int(math.floor(c * 255.0 + 0.5))
    return out


def test_turbo_summation_order_does_not_matter():
    """@reduce(.Add)'s order is the compiler's; every plausible order gives the same 768 bytes, so the table is the reference's."""
    left = _turbo_table("left")
    assert np.array_equal(left, _turbo_table("pairwise"))
    assert np.array_equal(left, _turbo_table("halves"))
    assert np.array_equal(left, zo.colormap_lut(zo.TURBO))


def test_library_luts_equal_the_oracle():
    import zignal_b200 as zb
    for m in (zo.JET, zo.HEAT, zo.TURBO):
        assert np.array_equal(zb.colormap_lut(m), zo.colormap_lut(m))
    for m in (zo.VIRIDIS, zo.INFERNO):
        with pytest.raises(zb.ZignalError) as e:
            zb.colormap_lut(m)
        assert e.value.status == 3


def test_viridis_inferno_fixture_is_256_rgb():
    t = json.loads(zo.TABLES.read_text())
    for name in ("viridis", "inferno"):
        a = np.asarray(t[name])
        assert a.shape == (256, 3) and a.min() >= 0 and a.max() <= 255


# ---- ABI argument errors, before any device work -------------------------------------------------------------------------------------

def test_abi_argument_errors():
    import zignal_b200 as zb
    L = zb.lib()
    good = zb.ZbImage(1, 4, 4, 4)
    other = zb.ZbImage(1, 4, 5, 5)
    st = zb._ffi.ZbDiffStats()
    lut = (C.c_uint8 * 768)()
    assert L.zb_diff(None, good, good, 0, 0.0, 1.0, 0, 0, None, None) == 5
    assert L.zb_diff(good, good, None, 0, 0.0, 1.0, 0, 0, None, None) == 5
    assert L.zb_diff(good, good, good, 9, 0.0, 1.0, 0, 0, C.byref(st), None) == 3
    assert L.zb_diff(good, other, good, 0, 0.0, 1.0, 0, 0, C.byref(st), None) == 1
    assert L.zb_diff(good, good, other, 3, 0.0, 1.0, 0, 0, None, None) == 1
    assert L.zb_colormap_lut(0, None) == 5 and L.zb_colormap_lut(5, lut) == 5 and L.zb_colormap_lut(-1, lut) == 5
    assert L.zb_colormap_lut(3, lut) == 3 and L.zb_colormap_lut(4, lut) == 3
    assert L.zb_apply_colormap(good, 0, None, 0, 0.0, 0, 0.0, good, None) == 5
    assert L.zb_apply_colormap(None, 0, lut, 0, 0.0, 0, 0.0, good, None) == 5
    assert L.zb_apply_colormap(good, 7, lut, 0, 0.0, 0, 0.0, good, None) == 3
    assert L.zb_apply_colormap(good, 1, lut, 0, 0.0, 0, 0.0, other, None) == 1
    for fn in (L.zb_flip_left_right, L.zb_flip_top_bottom, L.zb_invert):
        assert fn(None, 0, None) == 5
        assert fn(good, 5, None) == 3
    assert L.zb_invert(good, 1, None) == 3                               # Image(f32) has no invert
    empty = zb.ZbImage(None, 0, 7, 7)
    assert L.zb_diff(empty, empty, empty, 2, 0.0, 1.0, 0, 0, C.byref(st), None) == 0 and st.n == 0 and st.max == 0.0
    assert L.zb_apply_colormap(empty, 0, lut, 0, 0.0, 0, 0.0, empty, None) == 0
    assert L.zb_invert(empty, 0, None) == 0 and L.zb_flip_left_right(empty, 4, None) == 0
