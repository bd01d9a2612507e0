"""CPU checks of Image.shenCastan: the oracle (oracle/zo_shen_castan.cpp, bound in tests/shen_castan_oracle.py) against the reference's own
tests (image/tests/shen_castan.zig), against an independent numpy restatement of edges.zig bit for bit, and against its golden fixtures;
plus the error behaviour of zb_shen_castan that is decided before any device work, and the presets of the three host mirrors."""
import ctypes as C
import json
import re
import shutil
import subprocess
import textwrap
from pathlib import Path

import numpy as np
import pytest
from scipy import ndimage

import shen_castan_oracle as zo
import zignal_b200 as zb
from golden_shen_castan import CASES, oracle, smooth_noise
from gpu_utils import sha

ROOT = Path(__file__).resolve().parents[1]
F = np.float32


def _count(e):
    return int((e > 0).sum())


# ---- image/tests/shen_castan.zig ---------------------------------------------------------------------------------------------------
def test_kat_basic_square():   # shen_castan.zig:10-58
    img = np.tile((np.arange(50) * 2).astype(np.uint8), (50, 1))
    img[15:35, 15:35] = 200
    e = zo.shen_castan(img, zo.Options(smooth=0.8, window_size=7, high_ratio=0.9, low_rel=0.3))
    assert 0 < _count(e) < 500


def test_kat_parameter_validation():   # :60-87
    img = np.zeros((10, 10), np.uint8)
    cases = [(dict(smooth=0.0), 24), (dict(smooth=1.0), 24), (dict(smooth=-0.5), 24), (dict(high_ratio=0.0), 14), (dict(high_ratio=1.0), 14),
             (dict(low_rel=0.0), 14), (dict(window_size=6), 25), (dict(window_size=1), 26)]
    for kw, status in cases:
        with pytest.raises(zo.OracleStatus) as e:
            zo.shen_castan(img, zo.Options(**kw))
        assert e.value.status == status, kw


def test_kat_gradient_image():   # :89-128
    img = np.zeros((50, 50), np.uint8)
    img[:, :25] = np.minimum(np.arange(25) * 10, 200)
    img[:, 25:] = 240
    e = zo.shen_castan(img, zo.Options(smooth=0.85, window_size=7, high_ratio=0.8, low_rel=0.3))
    assert e[10:40, 24:27].any()


def test_kat_different_b_parameters():   # :130-177
    r, c = np.mgrid[0:40, 0:40]
    dist = np.sqrt((r.astype(F) - F(20)) ** 2 + (c.astype(F) - F(20)) ** 2)
    img = np.where(dist <= 10, 200, 50 + (r + c) // 2).astype(np.uint8)
    assert _count(zo.shen_castan(img, zo.Options(smooth=0.7, window_size=7, high_ratio=0.9))) > 0
    assert _count(zo.shen_castan(img, zo.Options(smooth=0.9, window_size=7, high_ratio=0.9))) > 0


def test_kat_rgb():   # :179-219
    img = np.zeros((30, 30, 3), np.uint8)
    img[:, :, 2] = np.minimum(100 + np.arange(30) * 3, 255)[:, None]
    img[10:20, 10:20] = (200, 50, 50)
    assert _count(zo.shen_castan(img, zo.Options(smooth=0.8, window_size=7, high_ratio=0.9))) > 0


def test_kat_threshold_monotonicity():   # :221-262
    img = np.zeros((40, 40), np.uint8)
    img[:20, :20] = 255
    img[20:, 20:] = 255
    low = _count(zo.shen_castan(img, zo.Options(smooth=0.8, window_size=7, high_ratio=0.95, low_rel=0.5)))
    high = _count(zo.shen_castan(img, zo.Options(smooth=0.8, window_size=7, high_ratio=0.999, low_rel=0.5)))
    assert high <= low and low > 0


def test_kat_diagonal_edge():   # :264-300
    r, c = np.mgrid[0:30, 0:30]
    img = np.where(r > c + 2, 200, np.where(r + 2 < c, 50, np.clip(125 + (r - c) * 10, 50, 200))).astype(np.uint8)
    e = zo.shen_castan(img, zo.Options(smooth=0.8, window_size=7, high_ratio=0.9))
    i = np.arange(5, 25)
    assert (e[i, i] > 0).any() or (e[i, i - 1] > 0).any() or (e[i - 1, i] > 0).any()


def test_kat_window_size_effect():   # :302-339
    r, c = np.mgrid[0:50, 0:50]
    base = np.where((r >= 15) & (r < 35) & (c >= 15) & (c < 35), 200, 50)
    img = (base + (r * 7 + c * 13) % 20).astype(np.uint8)
    assert _count(zo.shen_castan(img, zo.Options(smooth=0.8, window_size=3, high_ratio=0.9))) > 0
    assert _count(zo.shen_castan(img, zo.Options(smooth=0.8, window_size=11, high_ratio=0.9))) > 0


# ---- an independent numpy restatement of edges.zig ---------------------------------------------------------------------------------
def _round_half_away(x):   # non-negative inputs; exact: x - floor(x) is representable
    fl = np.floor(x)
    return np.where(x - fl >= 0.5, fl + 1, fl)


def np_gray(img):   # as(f32, convertColor(u8, px)), color.zig:114-118, 1031-1041
    if img.dtype == np.float32:
        return _round_half_away(np.clip(img.astype(np.float64), 0.0, 1.0) * 255.0).astype(F)
    if img.ndim == 2:
        return img.astype(F)
    p = img.astype(np.int64)
    return np.clip((13933 * p[..., 0] + 46871 * p[..., 1] + 4732 * p[..., 2] + 32768) >> 16, 0, 255).astype(F)


def np_isef_rows(x, b):   # isefFilter1D (edges.zig:283-306) on every row at once; sequential along the row
    a = F(1.0) - b
    n = x.shape[1]
    temp = np.empty_like(x)
    temp[:, 0] = b * x[:, 0]
    for i in range(1, n):
        temp[:, i] = b * x[:, i] + a * temp[:, i - 1]
    y = np.empty_like(x)
    y[:, n - 1] = temp[:, n - 1]
    for i in range(n - 2, -1, -1):
        y[:, i] = b * temp[:, i] + a * y[:, i + 1]
    return y


def np_zero_crossings(bli, use_forward):   # edges.zig:356-414
    rows, cols = bli.shape
    p = np.pad(bli.astype(np.int16), 1, constant_values=-1)   # -1: out of bounds, never compared
    ctr = p[1:-1, 1:-1]

    def differs(dr, dc):
        nb = p[1 + dr:1 + dr + rows, 1 + dc:1 + dc + cols]
        return (nb >= 0) & (nb != ctr)

    if use_forward:
        return differs(0, 1) | differs(1, 0) | differs(1, 1) | differs(1, -1)
    four = differs(0, -1) | differs(0, 1) | differs(-1, 0) | differs(1, 0)
    if rows >= 3 and cols >= 3:
        interior = np.zeros_like(four)
        interior[1:-1, 1:-1] = True
        return four & interior
    return four


def np_sat(plane):   # integral.zig:41-78: sequential row sums, then row r-1 added into row r
    return np.cumsum(np.cumsum(plane, axis=1, dtype=F), axis=0, dtype=F)


def np_shen_castan(img, o):
    gray = np_gray(img)
    rows, cols = gray.shape
    b = F(o.smooth)
    smoothed = np_isef_rows(np_isef_rows(gray, b).T.copy(), b).T
    bli = ((smoothed - gray) >= 0).astype(np.uint8)
    edges = np_zero_crossings(bli, not o.use_nms)
    # computeAdaptiveGradients, :417-495
    half = o.window_size // 2
    padded = [np.pad(np_sat(p), ((1, 0), (1, 0))) for p in (gray, bli.astype(F), gray * bli.astype(F))]
    r = np.arange(rows)[:, None]
    c = np.arange(cols)[None, :]
    r1, r2 = np.maximum(r - half, 0), np.minimum(r + half, rows - 1)
    c1, c2 = np.maximum(c - half, 0), np.minimum(c + half, cols - 1)

    def box(P):   # ((D - left) - top) + corner; the zero row / column of P stands for the "else 0" branches
        return ((P[r2 + 1, c2 + 1] - P[r2 + 1, c1]) - P[r1, c2 + 1]) + P[r1, c1]

    area = ((r2 - r1 + 1) * (c2 - c1 + 1)).astype(F)
    s_gray, count1, sum1 = box(padded[0]), box(padded[1]), box(padded[2])
    count0 = area - count1
    ok = edges & (count0 > 0) & (count1 > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = np.abs(sum1 / count1 - (s_gray - sum1) / count0)
    grad = np.where(ok, g, F(0)).astype(F)
    # thresholds, :139-170
    hist = np.bincount(_round_half_away(np.clip(grad[edges], 0, 255)).astype(np.int64), minlength=256)
    total = int(edges.sum())
    if total == 0:
        return np.zeros((rows, cols), np.uint8), 0.0, 0.0, hist, 0
    target = int(np.floor(F(total) * F(o.high_ratio)))
    cum, idx = 0, 0
    while idx < 256 and cum < target:
        cum += int(hist[idx])
        idx += 1
    t_high = F(min(idx, 255))
    t_low = F(o.low_rel) * t_high
    keep = edges
    if o.use_nms:   # :582-656
        keep = np.zeros_like(edges)
        if rows >= 3 and cols >= 3:
            s = smoothed
            gx = F(0.5) * (s[1:-1, 2:] - s[1:-1, :-2])
            gy = F(0.5) * (s[2:, 1:-1] - s[:-2, 1:-1])
            ax, ay = np.abs(gx), np.abs(gy)
            K = F(0.414213562)
            d0, d90, d45 = ay <= K * ax, ax <= K * ay, gx * gy > 0
            dr = np.where(d0, 0, -1)
            dc = np.where(d0, -1, np.where(d90, 0, np.where(d45, 1, -1)))
            rr, cc = np.mgrid[1:rows - 1, 1:cols - 1]
            m = grad[1:-1, 1:-1]
            n1, n2 = grad[rr + dr, cc + dc], grad[rr - dr, cc - dc]
            keep[1:-1, 1:-1] = edges[1:-1, 1:-1] & (m >= n1) & (m >= n2)
    seeds = keep & (grad >= t_high)
    if not o.hysteresis:
        return np.where(seeds, 255, 0).astype(np.uint8), t_high, t_low, hist, target
    weak = keep & (grad >= t_low)   # :499-575: components of the candidates, 8-connected, that hold a seed
    labels, _ = ndimage.label(weak, structure=np.ones((3, 3), int))
    grown = np.isin(labels, np.unique(labels[seeds])) & weak
    return np.where(grown | seeds, 255, 0).astype(np.uint8), t_high, t_low, hist, target


def _agree(img, o):
    want, th, tl, _hist, _target = np_shen_castan(img, o)
    got, oth, otl, _cand = zo.shen_castan_ex(img, o)
    assert np.array_equal(got, want), (o, img.shape, int((got != want).sum()))
    assert F(oth) == th and F(otl) == tl, (o, oth, th)


@pytest.mark.parametrize("preset", list(zo.PRESETS))
def test_numpy_restatement_matches_oracle_on_every_preset(preset):
    for fmt, img in {"u8": smooth_noise(1, 37, 53, sigma=15), "rgb8": smooth_noise(2, 29, 41, 3), "rgba8": smooth_noise(3, 23, 31, 4),
                     "f32": smooth_noise(4, 31, 27).astype(F) / F(255)}.items():
        _agree(img, zo.PRESETS[preset])


@pytest.mark.parametrize("shape", [(1, 1), (1, 40), (2, 40), (40, 1), (40, 2), (3, 3), (2, 2), (17, 23), (33, 65)])
def test_numpy_restatement_matches_oracle_on_thin_shapes_windows_and_switches(shape):
    img = smooth_noise(shape[0] * 100 + shape[1], *shape, sigma=25)
    for window in (3, 7, 11, 2 * max(shape) + 3):
        for use_nms in (False, True):
            for hysteresis in (False, True):
                _agree(img, zo.Options(window_size=window, use_nms=use_nms, hysteresis=hysteresis, high_ratio=0.85, low_rel=0.4))


def test_target_on_a_bin_boundary_takes_the_next_bin():
    """When the cumulative count reaches `target` exactly at bin k, the loop still increments idx: t_high = k + 1 (edges.zig:165-169)."""
    found = 0
    for seed in range(60):
        img = smooth_noise(500 + seed, 21, 26, sigma=20)
        o = zo.Options(high_ratio=0.75, use_nms=bool(seed % 2))
        want, th, _tl, hist, target = np_shen_castan(img, o)
        cum = np.cumsum(hist)
        if target > 0 and target in cum:
            k = int(np.argmax(cum >= target))
            assert cum[k] == target and th == F(min(k + 1, 255))
            _agree(img, o)
            found += 1
    assert found >= 3


def test_oracle_matches_golden_fixtures():
    g = json.loads((ROOT / "tests" / "golden" / "golden_shen_castan.json").read_text())
    assert set(g["cases"]) == set(CASES)
    for name, (build, preset) in CASES.items():
        img = build()
        assert sha(img) == g["cases"][name]["input_sha256"], name
        res = oracle(name, img)
        assert g["cases"][name]["preset"] == preset
        assert list(res.shape) == g["cases"][name]["shape"] and sha(res) == g["cases"][name]["output_sha256"], name


def test_oracle_error_order_and_unsupported_format():
    a = np.zeros((4, 4), np.uint8)
    with pytest.raises(zo.OracleStatus) as e:   # DimensionMismatch before validate
        zo.shen_castan(a, zo.Options(smooth=2.0), out=np.zeros((4, 5), np.uint8))
    assert e.value.status == 1
    with pytest.raises(zo.OracleStatus) as e:
        zo.shen_castan(np.zeros((4, 4, 4), np.float32))
    assert e.value.status == 3


# ---- C ABI: errors decided on the host (no kernel is launched) ---------------------------------------------------------------------
def test_status_names_and_argument_errors_before_the_device():
    L = zb.lib()
    for k, v in {24: "InvalidBParameter", 25: "WindowSizeMustBeOdd", 26: "WindowSizeTooSmall"}.items():
        assert L.zb_status_name(k).decode() == v
    a, b = np.zeros((12, 12), np.uint8), np.zeros((12, 13), np.uint8)
    ia, ib = zb.image._np_image(a), zb.image._np_image(b)
    empty = zb.image.ZbImage(None, 0, 4, 4)
    f = C.c_float

    def sc(src, dst, fmt=0, smooth=0.9, window=7, hr=0.99, lr=0.5):
        return L.zb_shen_castan(src, dst, fmt, f(smooth), window, f(hr), f(lr), 1, 0, None)

    assert L.zb_shen_castan(None, ia, 0, f(0.9), 7, f(0.99), f(0.5), 1, 0, None) == 5   # NULL
    assert sc(ia, ib, fmt=4, smooth=2.0) == 3                                            # Rgba(f32): unsupported, first of the checks
    assert sc(ia, ib, fmt=9) == 3
    assert sc(ia, ib, smooth=2.0, window=0) == 1                                         # DimensionMismatch before validate (image.zig:1023)
    for smooth in (0.0, 1.0, -0.5, float("nan"), float("inf")):
        assert sc(ia, ia, smooth=smooth, window=0, hr=0.0) == 24                         # InvalidBParameter first (ShenCastan.zig:40)
    assert sc(ia, ia, window=0, hr=0.0) == 25                                            # window 0 is even
    assert sc(ia, ia, window=6) == 25
    assert sc(ia, ia, window=2 ** 64 - 2) == 25
    assert sc(ia, ia, window=1, hr=0.0) == 26                                            # WindowSizeTooSmall before the thresholds
    for hr in (0.0, 1.0, float("nan")):
        assert sc(ia, ia, hr=hr, lr=5.0) == 14
    for lr in (0.0, 1.0, -1.0, float("nan")):
        assert sc(ia, ia, lr=lr) == 14
    assert sc(empty, empty) == 0                                                         # empty: ok, no device work
    assert sc(empty, empty, fmt=3, window=2 ** 64 - 1) == 0
    assert sc(empty, empty, window=4) == 25


def test_python_mirror_presets_match_the_reference():
    for name, want in zo.PRESETS.items():
        got = getattr(zb.ShenCastan, name)
        assert (got.smooth, got.window_size, got.high_ratio, got.low_rel, got.hysteresis, got.use_nms) == \
               (want.smooth, want.window_size, want.high_ratio, want.low_rel, want.hysteresis, want.use_nms), name
    assert tuple(zo.PRESETS) == zb.ShenCastan.PRESETS


def test_zig_shim_has_shen_castan_with_the_reference_presets():
    z = (ROOT / "zig" / "zignal_b200.zig").read_text()
    assert re.search(r"pub fn shenCastan\(self: Image, out: anytype, _: Allocator, opts: ShenCastan\)", z)
    for name in ("InvalidBParameter", "WindowSizeMustBeOdd", "WindowSizeTooSmall"):
        assert name in z.split("pub const Error")[1].split("\n")[0]
    for name in zo.PRESETS:
        assert re.search(rf"pub const {name}: ShenCastan = ", z), name


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")
def test_cpp_mirror_shen_castan_compiles_for_every_pixel_type(tmp_path):
    lib_dir = ROOT / "zignal_b200" / "lib"
    program = textwrap.dedent(r"""
        #include <cstdio>
        #include "zignal_b200/host/zignal.hpp"
        using namespace zignal;
        template <typename T> void instantiate() {
            DeviceImage<T> d;
            DeviceImage<uint8_t> e;
            d.shenCastan(e, ShenCastan{}); d.shenCastan(e, ShenCastan::thin()); d.shenCastan(e, ShenCastan::heavy_smooth());
        }
        template void instantiate<uint8_t>();
        template void instantiate<float>();
        template void instantiate<Rgb8>();
        template void instantiate<Rgba8>();
        int main() {
            DeviceImage<uint8_t> a{0, 4, nullptr, 4, nullptr}, b{0, 4, nullptr, 4, nullptr};
            ShenCastan o = ShenCastan::sensitive();
            o.window_size = 4;
            try { a.shenCastan(b, o); } catch (const Error& err) { std::printf("%d %s\n", err.status, err.what()); }
            a.shenCastan(b, ShenCastan::strong_only());
            std::printf("ok %zu %.2f\n", ShenCastan::high_noise().window_size, ShenCastan::low_noise().smooth);
            return 0;
        }
    """)
    src = tmp_path / "sc.cpp"
    src.write_text(program)
    exe = tmp_path / "sc"
    gxx = "/usr/bin/g++" if Path("/usr/bin/g++").exists() else "g++"
    res = subprocess.run([gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT), str(src), "-o", str(exe), "-L", str(lib_dir),
                          "-lzignal_b200", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.splitlines() == ["25 zignal error.WindowSizeMustBeOdd", "ok 11 0.95"]
