"""Image.convert between the 33 colour formats on the H100 (csrc/zb_color.cu) against the CPU oracle (oracle/zo_color.cpp): every pair
on seeded images (odd sizes, views, in place), the exactness contract of DESIGN.md §4.11, round trips over all 2^24 Rgb(u8) colours,
non-finite and out-of-range inputs, images past the 32-bit index range, and the same bits on other streams and threads."""
import threading

import numpy as np
import pytest
import torch

import color_oracle as co
import zignal_b200 as zb
from zignal_b200 import ColorFormat, ColorSpace as S, Component as K

pytestmark = pytest.mark.gpu

FORMATS = ColorFormat.all()
# edges of the `to` switches that call pow / cbrt / atan2 / sin / cos
TRANSCENDENTAL = {(S.RGB, S.XYZ), (S.RGB, S.XYB), (S.XYZ, S.RGB), (S.XYB, S.RGB), (S.XYZ, S.LAB), (S.XYZ, S.OKLAB), (S.XYZ, S.XYB),
                  (S.LAB, S.LCH), (S.LCH, S.LAB), (S.OKLAB, S.OKLCH), (S.OKLCH, S.OKLAB)}
# Bounds relative to each component's span.  f32: 1e-4, not 1e-5: a* = 500 (fx - fy) turns one ulp of fx into 3e-5, and an Hsv / Hsl
# saturation divides the RGB error by max(r, g, b), so dark colours reach 1.5e-5 of the span.
TOL = {K.F32: 1e-4, K.F64: 1e-12}
SPAN = {S.SCALAR: (1,), S.GRAY: (1,), S.RGB: (1, 1, 1), S.RGBA: (1, 1, 1, 1), S.YCBCR: (1, 1, 1), S.HSL: (360, 100, 100),
        S.HSV: (360, 100, 100), S.XYZ: (100, 100, 100), S.LAB: (100, 256, 256), S.LCH: (100, 150, 360), S.LMS: (1, 1, 1),
        S.OKLAB: (1, 1, 1), S.OKLCH: (1, 1, 360), S.XYB: (1, 1, 1)}
HUE = {S.HSL: (0, 1), S.HSV: (0, 1), S.LCH: (2, 1), S.OKLCH: (2, 1)}       # hue component, component of its chroma / saturation
CHROMA_MIN = {S.HSL: 1.0, S.HSV: 1.0, S.LCH: 1.5, S.OKLCH: 0.004}           # 1 % of the range of that component


def fmt_id(f):
    return f.name


def key(f):
    return (int(f.space), int(f.component))


def in_space(f):
    return S.GRAY if f.space == S.SCALAR else f.space


def exact(src, dst):
    """True when convertColor's path from src to dst calls no transcendental function."""
    s = in_space(src)
    for t in co.path(key(src), key(dst)):
        if (s, t) in TRANSCENDENTAL:
            return False
        s = t
    return True


def compute_component(src, dst):
    if src.space == S.SCALAR and dst.space == S.SCALAR:
        return dst.component if src.component == K.U8 else K.F64 if dst.component == K.U8 else dst.component
    if src.space == S.SCALAR:
        return dst.component
    if dst.space == S.SCALAR:
        return src.component
    return dst.component if dst.component != K.U8 else src.component


RANGES = {S.SCALAR: [(-0.05, 1.05)], S.GRAY: [(-0.05, 1.05)], S.RGB: [(-0.05, 1.05)] * 3, S.RGBA: [(-0.05, 1.05)] * 4,
          S.YCBCR: [(0, 1), (-0.5, 0.5), (-0.5, 0.5)], S.HSL: [(-30, 390), (0, 100), (0, 100)], S.HSV: [(-30, 390), (0, 100), (0, 100)],
          S.XYZ: [(0, 95), (0, 100), (0, 108)], S.LAB: [(0, 100), (-100, 100), (-100, 100)], S.LCH: [(0, 100), (0, 120), (0, 360)],
          S.LMS: [(0, 1)] * 3, S.OKLAB: [(0, 1), (-0.3, 0.3), (-0.3, 0.3)], S.OKLCH: [(0, 1), (0, 0.3), (0, 360)],
          S.XYB: [(-0.02, 0.02), (0, 0.8), (0, 0.8)]}


def sample(f, rows, cols, seed):
    rng = np.random.default_rng(seed)
    ch = f.channels
    if f.component == K.U8:
        a = rng.integers(0, 256, (rows, cols, ch), dtype=np.uint8)
    else:
        a = np.stack([rng.uniform(lo, hi, (rows, cols)) for lo, hi in RANGES[f.space]], axis=-1).astype(f.dtype)
    return a[..., 0] if ch == 1 else a


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == np.uint8:
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(u), b[~nb].view(u))


HALF_TOL = {K.F32: 1e-3, K.F64: 1e-9}


def before_rounding(a, src, dst):
    """The oracle's u8 output before @round, for a pair whose computation is in the source's float type: 255 * clamp(v, 0, 1) of
    the destination's space in that type (Gray for a scalar destination; cb and cr + 0.5 for Ycbcr, color.zig:968-972)."""
    space = S.GRAY if dst.space == S.SCALAR else dst.space
    v = co.convert(a, key(src), (int(space), int(src.component))).astype(np.float64)
    v = v.reshape(v.shape[:2] + (-1,))
    if space == S.YCBCR:
        v[..., 1:] += 0.5
    return 255.0 * np.clip(np.nan_to_num(v, nan=1.0), 0.0, 1.0)


def check(got, want, src, dst, what="", a=None):
    """The exactness contract: bits on transcendental-free paths; otherwise floats within TOL of the component's span, hues
    modulo 360 where their chroma / saturation is at least 1 % of its range, and u8 equal except where the oracle's value before
    rounding lies within 1e-3 (f32) / 1e-9 (f64) of a half-integer, where 1 off is allowed.  `a` is the source array (needed for
    u8 outputs).  Returns the number of u8 values off by 1."""
    if exact(src, dst):
        assert same_bits(got, want), f"{src.name} -> {dst.name}{what}: not bit-identical"
        return 0
    got = got.reshape(want.shape[:2] + (-1,))
    want = want.reshape(want.shape[:2] + (-1,))
    if dst.component == K.U8:
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        pre = before_rounding(a, src, dst)
        near_half = np.abs(pre - np.floor(pre) - 0.5) <= HALF_TOL[compute_component(src, dst)]
        assert d.max(initial=0) <= 1, f"{src.name} -> {dst.name}{what}: u8 off by {d.max()}"
        assert not np.any((d == 1) & ~near_half), f"{src.name} -> {dst.name}{what}: u8 off by 1 away from a half-integer"
        return int((d == 1).sum())
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{src.name} -> {dst.name}{what}: NaN positions differ"
    tol = TOL[compute_component(src, dst)]
    for k in range(want.shape[-1]):
        g, w = got[..., k].astype(np.float64), want[..., k].astype(np.float64)
        ok = np.isfinite(w)
        assert np.array_equal(g[~ok & ~np.isnan(w)], w[~ok & ~np.isnan(w)]), f"{src.name} -> {dst.name}{what}: infinities differ"
        if dst.space in HUE and k == HUE[dst.space][0]:
            mask = ok & (want[..., HUE[dst.space][1]] >= CHROMA_MIN[dst.space])
            d = np.abs(g - w) % 360.0
            d = np.minimum(d, 360.0 - d)
            rng = 360.0
        else:
            mask = ok
            d = np.abs(g - w)
            rng = SPAN[dst.space][k]
        worst = float(d[mask].max(initial=0.0))
        assert worst <= tol * rng, f"{src.name} -> {dst.name}{what}: component {k} off by {worst:.3g} (allowed {tol * rng:.3g})"
    return 0


def to_dev(a, f):
    return zb.Image.from_numpy(a, format=f)


@pytest.mark.parametrize("src", FORMATS, ids=fmt_id)
def test_every_pair_matches_the_oracle(src):
    rows, cols = 37, 53
    a = sample(src, rows, cols, seed=int(src.space) * 3 + int(src.component))
    img = to_dev(a, src)
    ones = 0
    for dst in FORMATS:
        if dst == src:
            continue
        got = img.convert(dst).to_numpy()
        want = co.convert(a, key(src), key(dst))
        ones += check(got, want, src, dst, a=a)
    print(f"{src.name}: {ones} u8 values within 1 of the oracle")


@pytest.mark.parametrize("src", [ColorFormat(S.RGB, K.U8), ColorFormat(S.LAB, K.F32), ColorFormat(S.HSV, K.F64),
                                 ColorFormat(S.RGBA, K.F32)], ids=fmt_id)
def test_views_and_in_place(src):
    big = sample(src, 41, 67, seed=7)
    img = to_dev(big, src)
    view = img.view(zb.Rectangle(5, 3, 60, 38))
    sub = big[3:38, 5:60]
    for dst in FORMATS:
        if dst == src:
            continue
        out_big = zb.Image.init(41, 67, dst)
        before = out_big.to_numpy()
        out = out_big.view(zb.Rectangle(2, 4, 57, 39))
        view.convert(dst, out=out)
        after = out_big.to_numpy()
        check(after[4:39, 2:57], co.convert(sub, key(src), key(dst)), src, dst, " (view)", a=sub)
        outside = np.ones(after.shape[:2], bool)
        outside[4:39, 2:57] = False
        assert same_bits(after[outside], before[outside]), f"{src.name} -> {dst.name}: wrote outside the view"
        if dst.component == src.component and dst.channels == src.channels:
            inplace = to_dev(big, src)
            v = inplace.view(zb.Rectangle(5, 3, 60, 38))
            w = zb.Image(v._t, dst, v.rows, v.cols, v.stride, v._off)
            v.convert(dst, out=w)
            check(w.to_numpy(), co.convert(sub, key(src), key(dst)), src, dst, " (in place)", a=sub)


def all_colors():
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)


@pytest.mark.parametrize("component", [K.F32, K.F64], ids=["f32", "f64"])
def test_round_trip_of_all_rgb_colors(component):
    rgb = all_colors()
    img = to_dev(rgb, ColorFormat(S.RGB, K.U8))
    src = ColorFormat(S.RGB, K.U8)
    for space in S:
        if space in (S.SCALAR, S.GRAY, S.RGB, S.RGBA):
            continue
        mid = ColorFormat(space, component)
        back = img.convert(mid).convert(src).to_numpy()
        want = co.convert(co.convert(rgb, key(src), key(mid)), key(mid), key(src))
        lost_oracle = int(np.any(want != rgb, axis=-1).sum())
        lost = int(np.any(back != rgb, axis=-1).sum())
        print(f"Rgb(u8) -> {mid.name} -> Rgb(u8): device loses {lost}, oracle {lost_oracle} of 2^24 colours")
        if lost_oracle == 0:
            assert lost == 0, mid.name
        else:
            assert np.abs(back.astype(int) - want.astype(int)).max() <= 1, mid.name


def test_ycbcr_u8_round_trip_within_one():
    rgb = all_colors()
    img = to_dev(rgb, ColorFormat(S.RGB, K.U8))
    back = img.convert(ColorFormat(S.YCBCR, K.U8)).convert(ColorFormat(S.RGB, K.U8)).to_numpy()
    assert np.abs(back.astype(int) - rgb.astype(int)).max() <= 1


SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, 5e-324, 1e30, -1e30, 2.0, -1.0, 360.0, -360.0, 1e-7, -1e-7,
                    100.0, 0.5, 1.0, 255.0])


@pytest.mark.parametrize("src", [f for f in FORMATS if f.component != K.U8], ids=fmt_id)
def test_special_values(src):
    vals = SPECIAL.astype(src.dtype)
    n = len(vals)
    rng = np.random.default_rng(11)
    ch = src.channels
    # every special value in every channel against ordinary values in the others, and a few all-special pixels
    base = sample(src, n * ch + 16, 1, seed=3).reshape(n * ch + 16, ch) if ch > 1 else sample(src, n + 16, 1, seed=3).reshape(-1, 1)
    for c in range(ch):
        base[c * n:(c + 1) * n, c] = vals
    base[-16:] = rng.choice(vals, (16, ch))
    a = base.reshape(1, -1, ch) if ch > 1 else base.reshape(1, -1)
    img = to_dev(np.ascontiguousarray(a), src)
    for dst in FORMATS:
        if dst == src:
            continue
        got = img.convert(dst).to_numpy()
        want = co.convert(a, key(src), key(dst))
        if exact(src, dst) or dst.component == K.U8:
            check(got, want, src, dst, " (special values)", a=a)
            continue
        # transcendental paths: NaN and infinities where the oracle has them; the contract on the pixels whose inputs lie in the
        # space's range (out of it, a grey of 255 has an Oklch hue made of rounding noise, and huge values cancel in the matrices)
        g, w = got.reshape(-1, dst.channels).astype(np.float64), want.reshape(-1, dst.channels).astype(np.float64)
        assert np.array_equal(np.isnan(g), np.isnan(w)), f"{src.name} -> {dst.name}: NaN positions differ"
        inf = np.isinf(w)
        assert np.array_equal(g[inf], w[inf]), f"{src.name} -> {dst.name}: infinities differ"
        lo = np.array([a - 0.1 * (b - a) for a, b in RANGES[src.space]])
        hi = np.array([b + 0.1 * (b - a) for a, b in RANGES[src.space]])
        ordinary = np.all(np.isfinite(base) & (base >= lo) & (base <= hi), axis=-1)
        check(got.reshape(1, -1, *got.shape[2:])[:, ordinary], want.reshape(1, -1, *want.shape[2:])[:, ordinary], src, dst,
              " (special values)")


@pytest.mark.parametrize("src, dst", [(ColorFormat(S.RGB, K.U8), ColorFormat(S.YCBCR, K.U8)),
                                      (ColorFormat(S.GRAY, K.F32), ColorFormat(S.LAB, K.F32))], ids=["rgb8-ycbcr8", "grayf32-labf32"])
def test_past_the_32_bit_range(src, dst):
    """2^15 x (2^16 + 5) pixels: pixel indices past 2^31 and byte offsets past 2^32 on both sides; the last two rows against the
    oracle."""
    rows, cols = 1 << 15, (1 << 16) + 5
    torch.cuda.empty_cache()
    img = zb.Image.init(rows, cols, src)
    tail = sample(src, 2, cols, seed=5)
    t = img._t.view(rows, -1)
    t[-2:] = torch.from_numpy(tail.reshape(2, -1)).cuda()
    out = img.convert(dst)
    got = out._t.view(rows, -1)[-2:].cpu().numpy()
    want = co.convert(tail, key(src), key(dst))
    check(got.view(want.dtype).reshape(want.shape), want, src, dst, " (far corner)", a=tail)
    del img, out, t
    torch.cuda.empty_cache()


def test_same_bits_on_streams_and_threads():
    src, dst = ColorFormat(S.RGB, K.U8), ColorFormat(S.OKLCH, K.F32)
    a = sample(src, 512, 777, seed=9)
    img = to_dev(a, src)
    ref = img.convert(dst).to_numpy()
    results, errors = [None] * 4, []

    def work(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                out = None
                for _ in range(3):
                    out = img.convert(dst)
                s.synchronize()
                results[k] = out.to_numpy()
        except Exception as e:   # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for r in results:
        assert same_bits(r, ref)
