"""Image.diff, applyColormap, the flips and invert on the GPU, bit-identical to the oracle (oracle/zo_visual.cpp, bound in
tests/visual_oracle.py): every pixel format with scaled and binary output, with and without force_opaque, thresholds exactly at a
difference value, negative / huge / NaN scales and NaN / inf inputs; the diff statistics against exact values; applyColormap with auto,
partial, explicit and NaN ranges and every map; flips at odd and even sizes; 1 x 1, 1 x N, N x 1, unaligned widths, views with sentinels,
`out` aliasing an input, 8192^2 and a 600,000-row image; a non-blocking stream, two host threads and the golden fixtures."""
import ctypes as C
import json
import math
import threading
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import visual_oracle as zo
from golden_visual import CASES, FORMATS, PIX, case_inputs, near_pair, random_image
from gpu_utils import sha
from test_visual_host import np_diff, same_bits

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_visual.json"
DIFF_OPTS = [(0.0, 1.0), (2.0, 1.0), (0.25, 3.0), (1.0, -2.0), (0.0, 1e30), (0.0, float("nan")), (0.125, 0.5)]


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def gpu_diff(zb, a, b, **prm):
    out, res = zb.Image.from_numpy(a).diff(zb.Image.from_numpy(b), **prm)
    return out.to_numpy(), res


def check_stats(res, want, samples=None):
    """n / diff_count / min / max equal to the oracle; 8-bit sum exact and mean / variance the exactly rounded rationals, within 1e-9
    of the oracle's Welford; float sum / mean within 1e-12 and variance within 1e-9 of the exact values."""
    st = res.stats
    assert (st.count, res.diff_count) == (want["n"], want["diff_count"])
    assert st.min == want["min"] and st.max == want["max"]             # == rather than bits: the sign of a zero extreme is free
    if samples is None or not np.all(np.isfinite(samples)):
        return
    n = samples.size
    if want.get("int", False):
        s = int(samples.astype(np.int64).sum())
        q = int((samples.astype(np.int64) ** 2).sum())
        assert st.sum == want["sum"] == float(s)
        assert st.mean == float(Fraction(s, n))
        assert st.variance == (float(Fraction(n * q - s * s, n * (n - 1))) if n > 1 else 0.0)
        assert st.mean == pytest.approx(want["mean"], rel=1e-9, abs=1e-300)
        assert st.variance == pytest.approx(want["variance"], rel=1e-9, abs=1e-300)
    else:
        fs = math.fsum(samples.tolist())
        mean = fs / n
        var = math.fsum(((samples - mean) ** 2).tolist()) / (n - 1) if n > 1 else 0.0
        assert st.sum == pytest.approx(fs, rel=1e-12, abs=1e-300)
        assert st.mean == pytest.approx(mean, rel=1e-12, abs=1e-300)
        assert st.variance == pytest.approx(var, rel=1e-9, abs=1e-300)


def full_check(zb, a, b, **prm):
    got, res = gpu_diff(zb, a, b, **prm)
    want, wst = zo.diff(a, b, **prm)
    assert same_bits(got, want), prm
    _, samples, _ = np_diff(a, b, prm.get("threshold", 0.0), prm.get("scale", 1.0), prm.get("binary", False), prm.get("force_opaque", False))
    wst["int"] = a.dtype == np.uint8
    check_stats(res, wst, samples)
    return res


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("force_opaque", [False, True])
@pytest.mark.parametrize("threshold,scale", DIFF_OPTS)
def test_diff_matches_oracle(zb, fmt, binary, force_opaque, threshold, scale):
    a, b = near_pair(fmt, 37, 53, 300)
    full_check(zb, a, b, threshold=threshold, scale=scale, binary=binary, force_opaque=force_opaque)


@pytest.mark.parametrize("fmt", ["f32", "rgbaf32"])
@pytest.mark.parametrize("binary", [False, True])
def test_diff_float_specials(zb, fmt, binary):
    a, b = random_image(fmt, 45, 67, 1, specials=True), random_image(fmt, 45, 67, 2, specials=True)
    got, res = gpu_diff(zb, a, b, threshold=0.1, scale=2.0, binary=binary)
    want, wst = zo.diff(a, b, 0.1, 2.0, binary)
    assert same_bits(got, want)
    assert (res.stats.count, res.diff_count, res.stats.min, res.stats.max) == (wst["n"], wst["diff_count"], wst["min"], wst["max"])
    for k in ("sum", "mean", "variance"):
        assert math.isnan(getattr(res.stats, k)) == math.isnan(wst[k]) or math.isinf(wst[k]), k


@pytest.mark.parametrize("shape", [(1, 1), (1, 7), (1, 6145), (9, 1), (3, 17), (13, 4097), (5, 6147), (257, 3)])
@pytest.mark.parametrize("fmt", FORMATS)
def test_diff_shapes(zb, shape, fmt):
    a, b = near_pair(fmt, *shape, seed=shape[1])
    full_check(zb, a, b, threshold=1.0, scale=7.0)


@pytest.mark.parametrize("fmt", ["u8", "rgb8", "rgba8"])
def test_diff_stats_8bit_large(zb, fmt):
    a, b = random_image(fmt, 1031, 2053, 3), random_image(fmt, 1031, 2053, 4)
    full_check(zb, a, b, scale=1.0, force_opaque=fmt == "rgba8")


def test_diff_float_near_constant_has_no_cancellation(zb):
    rng = np.random.default_rng(5)
    a = np.full((1024, 1536), 4096.0, np.float32)
    b = (np.float32(3072.0) + rng.integers(-8, 9, a.shape).astype(np.float32) * np.float32(2.0 ** -12)).astype(np.float32)
    res = full_check(zb, a, b)
    assert res.stats.variance > 0
    got2 = gpu_diff(zb, a, b)[1]
    assert got2 == res                                                   # repeat call, same bits


def test_diff_repeat_identical_bits(zb):
    a, b = near_pair("rgbaf32", 777, 1111, 9)
    first = gpu_diff(zb, a, b, scale=1.5)[1]
    for _ in range(3):
        assert gpu_diff(zb, a, b, scale=1.5)[1] == first


def test_diff_out_aliases_an_input(zb):
    for fmt in FORMATS:
        a, b = near_pair(fmt, 63, 129, 11)
        want, wst = zo.diff(a, b, threshold=1.0, scale=5.0)
        da, db = zb.Image.from_numpy(a), zb.Image.from_numpy(b)
        _, res = da.diff(db, out=da, threshold=1.0, scale=5.0)
        assert same_bits(da.to_numpy(), want) and res.diff_count == wst["diff_count"]
        da = zb.Image.from_numpy(a)
        da.diff(db, out=db, threshold=1.0, scale=5.0)
        assert same_bits(db.to_numpy(), want)


def test_diff_without_stats_only_enqueues(zb, torch):
    a, b = near_pair("rgb8", 100, 333, 12)
    da, db, do = zb.Image.from_numpy(a), zb.Image.from_numpy(b), zb.Image.from_numpy(np.zeros_like(a))
    L = zb.lib()
    x, y, o = da._zb(), db._zb(), do._zb()
    assert L.zb_diff(x, y, o, int(da.pixfmt), C.c_float(0.0), C.c_float(9.0), 0, 0, None, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert same_bits(do.to_numpy(), zo.diff(a, b, scale=9.0)[0])


def _sentinel_view(zb, img, fill):
    """A device image holding img at (13, 37) inside a frame of `fill`: (whole numpy array, device image, device view, slice)."""
    rows, cols = img.shape[:2]
    big = np.full((rows + 29, cols + 71) + img.shape[2:], fill, img.dtype)
    sl = (slice(13, 13 + rows), slice(37, 37 + cols))
    big[sl] = img
    dev = zb.Image.from_numpy(big)
    return big, dev, dev.view(zb.Rectangle(37, 13, 37 + cols, 13 + rows)), sl


@pytest.mark.parametrize("fmt", FORMATS)
def test_views_with_sentinels(zb, fmt):
    fill = 0xA5 if fmt in ("u8", "rgb8", "rgba8") else -7.5
    a, b = near_pair(fmt, 41, 203, 21)
    ba, _, va, sl = _sentinel_view(zb, a, fill)
    bb, _, vb, _ = _sentinel_view(zb, b, fill)
    bo, do, vo, _ = _sentinel_view(zb, np.zeros_like(a), fill)
    va.diff(vb, out=vo, threshold=1.0, scale=3.0, force_opaque=True)
    want = bo.copy()
    want[sl] = zo.diff(a, b, threshold=1.0, scale=3.0, force_opaque=True)[0]
    assert same_bits(do.to_numpy(), want)
    for op, ref in (("flip_left_right", zo.flip_left_right), ("flip_top_bottom", zo.flip_top_bottom), ("invert", zo.invert)):
        if op == "invert" and fmt == "f32":
            continue
        big, dev, v, sl = _sentinel_view(zb, a, fill)
        getattr(v, op)()
        want = big.copy()
        ref(want[sl])
        assert same_bits(dev.to_numpy(), want), op
    big, dev, v, sl = _sentinel_view(zb, a, fill)
    lut = zo.colormap_lut(zo.JET)
    assert np.array_equal(v.apply_colormap(zb.Colormap.JET).to_numpy(), zo.apply_colormap(np.ascontiguousarray(big[sl]), lut))


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("out_col", [41, 54])
def test_diff_views_at_different_alignments(zb, fmt, out_col):
    """a, b and out at columns 37, 38 and out_col of frames 368 pixels wide (a row pitch that is a multiple of 16 bytes), so on every
    row out agrees modulo 16 bytes with b but not with a (out_col 54 = 38 + 16), or with neither (41; for U8, F32, Rgb and Rgba(u8)):
    the staged output is written from b's buffer, or byte by byte."""
    fill = 0x5A if fmt in ("u8", "rgb8", "rgba8") else 3.25
    a, b = near_pair(fmt, 23, 301, 61)
    rows, cols = a.shape[:2]

    def framed(img, col):
        big = np.full((rows + 9, 368) + img.shape[2:], fill, img.dtype)
        sl = (slice(4, 4 + rows), slice(col, col + cols))
        big[sl] = img
        dev = zb.Image.from_numpy(big)
        return big, dev, dev.view(zb.Rectangle(col, 4, col + cols, 4 + rows)), sl

    _, _, va, _ = framed(a, 37)
    _, _, vb, _ = framed(b, 38)
    bo, do, vo, sl = framed(np.zeros_like(a), out_col)
    _, res = va.diff(vb, out=vo, threshold=1.0, scale=3.0)
    want = bo.copy()
    out, wst = zo.diff(a, b, threshold=1.0, scale=3.0)
    want[sl] = out
    assert same_bits(do.to_numpy(), want)
    assert res.diff_count == wst["diff_count"] and res.stats.max == wst["max"]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("cmap", range(5))
@pytest.mark.parametrize("rng_", [(None, None), (0.1, None), (None, 100.0), (0.25, 0.75), (0.9, 0.1), (float("nan"), 1.0), (0.0, float("nan"))])
def test_colormap_matches_oracle(zb, fmt, cmap, rng_):
    img = random_image(fmt, 53, 211, 400 + cmap, specials=True)
    lut = zo.colormap_lut(cmap)
    got = zb.Image.from_numpy(img).apply_colormap(lut if cmap >= zo.VIRIDIS else zb.Colormap(cmap), *rng_).to_numpy()
    assert np.array_equal(got, zo.apply_colormap(img, lut, *rng_))


@pytest.mark.parametrize("fmt", FORMATS)
def test_colormap_constant_empty_and_odd_shapes(zb, fmt):
    lut = zo.colormap_lut(zo.TURBO)
    px = random_image(fmt, 1, 1, 5)
    for shape in ((1, 1), (1, 4099), (3001, 1), (5, 6147), (0, 4)):
        img = np.repeat(np.repeat(px, shape[0], axis=0), shape[1], axis=1)
        got = zb.Image.from_numpy(img).apply_colormap(zb.Colormap.TURBO).to_numpy() if img.size else None
        if img.size:
            assert np.array_equal(got, zo.apply_colormap(img, lut)), shape
        img = random_image(fmt, *shape, seed=shape[1])
        if img.size:
            assert np.array_equal(zb.Image.from_numpy(img).apply_colormap(zb.Colormap.TURBO).to_numpy(), zo.apply_colormap(img, lut)), shape
    e = zb.Image.init(0, 4, zb.PixFmt(PIX[fmt]))
    assert e.apply_colormap(zb.Colormap.JET).rows == 0


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("shape", [(1, 1), (1, 2), (2, 1), (1, 6145), (7, 12289), (8, 3072), (3, 3), (4, 4), (31, 4), (600000, 3)])
def test_flips_and_invert(zb, fmt, shape):
    img = random_image(fmt, *shape, seed=shape[0] + shape[1], specials=True)
    assert same_bits(zb.Image.from_numpy(img).flip_left_right().to_numpy(), img[:, ::-1])
    assert same_bits(zb.Image.from_numpy(img).flip_top_bottom().to_numpy(), img[::-1])
    if fmt == "f32":
        with pytest.raises(zb.ZignalError) as e:
            zb.Image.from_numpy(img).invert()
        assert e.value.status == 3
    else:
        assert same_bits(zb.Image.from_numpy(img).invert().to_numpy(), zo.invert(img.copy()))


def test_tall_image_diff_and_colormap(zb):
    a, b = near_pair("u8", 600000, 5, 31)
    full_check(zb, a, b, threshold=1.0, scale=2.0)
    assert np.array_equal(zb.Image.from_numpy(a).apply_colormap(zb.Colormap.HEAT).to_numpy(), zo.apply_colormap(a, zo.colormap_lut(zo.HEAT)))


def test_8192_squared(zb):
    a, b = near_pair("rgba8", 8192, 8192, 41)
    got, res = gpu_diff(zb, a, b, threshold=2.0, scale=1.0, force_opaque=True)       # the CLI's call
    want, wst = zo.diff(a, b, threshold=2.0, scale=1.0, force_opaque=True)
    assert same_bits(got, want)
    _, samples, _ = np_diff(a, b, 2.0, 1.0, False, True)
    wst["int"] = True
    check_stats(res, wst, samples)
    f = random_image("f32", 8192, 8192, 42)
    assert np.array_equal(zb.Image.from_numpy(f).apply_colormap(zb.Colormap.TURBO).to_numpy(), zo.apply_colormap(f, zo.colormap_lut(zo.TURBO)))
    assert same_bits(zb.Image.from_numpy(a).flip_left_right().flip_top_bottom().invert().to_numpy(),
                     zo.invert(np.ascontiguousarray(a[::-1, ::-1])))


def test_cli_call(zb):
    """cli/diff.zig:86-104: Rgba(u8), force_opaque, an integer threshold; it reports stats.max() and diff_count."""
    a, b = near_pair("rgba8", 480, 640, 51)
    for binary in (False, True):
        res = full_check(zb, a, b, threshold=float(2), scale=1.0, binary=binary, force_opaque=True)
        assert int(res.stats.max) == (255 if binary else np.abs(a[..., :3].astype(int) - b[..., :3]).max())


def test_non_blocking_stream_and_two_threads(zb, torch):
    cases = {seed: near_pair("rgba8", 1031, 1537, seed) for seed in (1, 2)}
    wants = {seed: zo.diff(*cases[seed], threshold=1.0, scale=4.0) for seed in cases}
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got, res = gpu_diff(zb, *cases[1], threshold=1.0, scale=4.0)
        assert same_bits(got, wants[1][0]) and res.diff_count == wants[1][1]["diff_count"]
    results, errors = {}, []
    start = threading.Barrier(2)

    def work(seed):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                da, db = (zb.Image.from_numpy(x) for x in cases[seed])
                st.synchronize()
                start.wait()
                out, res = da.diff(db, threshold=1.0, scale=4.0)
                cm = da.apply_colormap(zb.Colormap.JET)
                da.flip_left_right().invert()
                st.synchronize()
                results[seed] = (out.to_numpy(), res, cm.to_numpy(), da.to_numpy())
        except BaseException as e:   # noqa: B902 -- reported by the main thread
            errors.append((seed, repr(e)))
            start.abort()

    threads = [threading.Thread(target=work, args=(seed,)) for seed in (1, 2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for seed in (1, 2):
        out, res, cm, inv = results[seed]
        a = cases[seed][0]
        assert same_bits(out, wants[seed][0]) and res.diff_count == wants[seed][1]["diff_count"]
        assert np.array_equal(cm, zo.apply_colormap(a, zo.colormap_lut(zo.JET)))
        assert same_bits(inv, zo.invert(np.ascontiguousarray(a[:, ::-1])))


def test_golden(zb):
    g = json.loads(GOLDEN.read_text())["cases"]
    assert set(g) == set(CASES)
    for name, (op, fmt, rows, cols, seed, prm) in CASES.items():
        inputs = case_inputs(name)
        assert [sha(x) for x in inputs] == g[name]["input_sha256"], name
        dev = zb.Image.from_numpy(inputs[0])
        if op == "diff":
            out, res = dev.diff(zb.Image.from_numpy(inputs[1]), **prm)
            st = g[name]["stats"]
            assert res.diff_count == st["diff_count"] and res.stats.count == st["n"]
            assert res.stats.sum == float.fromhex(st["sum"]) and res.stats.max == float.fromhex(st["max"])
            assert res.stats.min == float.fromhex(st["min"])
            out = out.to_numpy()
        elif op == "colormap":
            m = prm["map"]
            out = dev.apply_colormap(zo.colormap_lut(m) if m >= zo.VIRIDIS else zb.Colormap(m), prm["min"], prm["max"]).to_numpy()
        else:
            out = getattr(dev, {"flip_lr": "flip_left_right", "flip_tb": "flip_top_bottom", "invert": "invert"}[op])().to_numpy()
        assert sha(out) == g[name]["output_sha256"], name
