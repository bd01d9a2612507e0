"""Image.shenCastan on the GPU, bit-exact against the oracle (oracle/zo_shen_castan.cpp, bound in tests/shen_castan_oracle.py): the four
pixel formats, the reference's seven presets and both switches, thin and ragged shapes, strided source and destination views guarded by
sentinel bytes, in-place U8, a constant image, subnormal ISEF tails, long contours across many hysteresis tiles, windows larger than the
image, a 4200 x 4200 image (summed-area tables beyond 2^24), a 1080p RGB frame and the golden fixtures."""
import json
from pathlib import Path

import numpy as np
import pytest

import shen_castan_oracle as zo
from golden_shen_castan import CASES, device, smooth_noise
from gpu_utils import sha

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    return zb


def _run(zb, img, o, out=None):
    return zb.Image.from_numpy(img).shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms, out=out)


def _check(zb, img, o, what=""):
    got = _run(zb, img, o).to_numpy()
    assert zb.lib().zb_last_kernel().decode() == "shen_castan"
    want = zo.shen_castan(img, o)
    assert np.array_equal(got, want), (what, o, int((got != want).sum()))
    return want


def _formats(seed, rows, cols):
    g = smooth_noise(seed, rows, cols)
    return {"u8": g, "f32": g.astype(np.float32) / np.float32(255.0), "rgb8": smooth_noise(seed, rows, cols, 3),
            "rgba8": smooth_noise(seed, rows, cols, 4)}


@pytest.mark.parametrize("preset", list(zo.PRESETS))
@pytest.mark.parametrize("fmt", ["u8", "f32", "rgb8", "rgba8"])
def test_presets_and_formats_match_oracle(zb, preset, fmt):
    img = _formats(7, 97, 131)[fmt]
    _check(zb, img, zo.PRESETS[preset], fmt)


@pytest.mark.parametrize("shape", [(1, 1), (1, 77), (2, 95), (77, 1), (95, 2), (3, 3), (31, 33), (64, 64), (65, 130), (129, 47)])
@pytest.mark.parametrize("use_nms", [False, True])
@pytest.mark.parametrize("hysteresis", [False, True])
def test_thin_and_ragged_shapes(zb, shape, use_nms, hysteresis):
    img = smooth_noise(shape[0] * 7 + shape[1], *shape, sigma=30.0)
    for window in (3, 7, 11, 2 * max(shape) + 1):
        _check(zb, img, zo.Options(window_size=window, hysteresis=hysteresis, use_nms=use_nms, high_ratio=0.8), (shape, window))


def test_strided_views_with_sentinels_and_in_place(zb):
    for fmt, img in _formats(11, 70, 91).items():
        t, l = 3, 5
        base = np.full((img.shape[0] + t + 2, img.shape[1] + l + 7) + img.shape[2:], 0 if fmt == "f32" else SENTINEL, img.dtype)
        base[t:t + img.shape[0], l:l + img.shape[1]] = img
        src_dev = zb.Image.from_numpy(base)
        view = src_dev.view(zb.Rectangle(l, t, l + img.shape[1], t + img.shape[0]))
        obase = np.full((img.shape[0] + 4, img.shape[1] + 9), SENTINEL, np.uint8)
        out_dev = zb.Image.from_numpy(obase)
        oview = out_dev.view(zb.Rectangle(2, 1, 2 + img.shape[1], 1 + img.shape[0]))
        for o in (zo.PRESETS["default"], zo.PRESETS["thin"], zo.PRESETS["strong_only"]):
            view.shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms, out=oview)
            got = out_dev.to_numpy()
            assert np.array_equal(got[1:1 + img.shape[0], 2:2 + img.shape[1]], zo.shen_castan(img, o)), (fmt, o)
            m = np.ones(got.shape, bool)
            m[1:1 + img.shape[0], 2:2 + img.shape[1]] = False
            assert (got[m] == SENTINEL).all(), fmt
    img = smooth_noise(12, 83, 120)
    for o in (zo.PRESETS["sensitive"], zo.PRESETS["thin"], zo.PRESETS["strong_only"]):
        dev = zb.Image.from_numpy(img)
        dev.shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms, out=dev)   # in place
        assert np.array_equal(dev.to_numpy(), zo.shen_castan(img, o)), o


def test_constant_image_clears_garbage(zb):
    img = np.full((67, 45), 93, np.uint8)
    for o in zo.PRESETS.values():
        out = zb.Image.from_numpy(np.full((67, 45), 7, np.uint8))
        _run(zb, img, o, out=out)
        assert not out.to_numpy().any()
        assert not zo.shen_castan(img, o).any()


def test_bright_dot_subnormal_tails(zb):
    img = np.zeros((150, 170), np.uint8)
    img[75, 80] = 255
    img[20:23, 140:143] = 200
    for smooth in (0.9, 0.5, 0.3):
        for use_nms in (False, True):
            _check(zb, img, zo.Options(smooth=smooth, use_nms=use_nms, high_ratio=0.5), (smooth, use_nms))
    f = img.astype(np.float32) / np.float32(255.0)
    _check(zb, f, zo.Options(smooth=0.95, high_ratio=0.6), "f32 dot")


def test_long_contours_cross_many_hysteresis_tiles(zb):
    rows, cols = 700, 900
    yy, xx = np.mgrid[0:rows, 0:cols]
    rng = np.random.default_rng(21)
    img = (100 + 60 * (np.sin(xx / 41.0 + yy / 67.0) > 0) + 40 * (((xx - 450) ** 2 + (yy - 350) ** 2) < 300 ** 2)).astype(np.float64)
    img = np.clip(img + rng.normal(0, 8, img.shape), 0, 255).astype(np.uint8)
    for o in (zo.Options(), zo.Options(low_rel=0.1, high_ratio=0.999), zo.PRESETS["thin"], zo.PRESETS["sensitive"]):
        want = _check(zb, img, o)
        assert want.any()


def test_window_larger_than_the_image(zb):
    img = smooth_noise(31, 40, 57, sigma=20.0)
    for window in (81, 115, 1001, 2 ** 40 + 1):
        for use_nms in (False, True):
            _check(zb, img, zo.Options(window_size=window, use_nms=use_nms, high_ratio=0.9), window)


def test_1080p_rgb_frame(zb):
    img = smooth_noise(41, 1080, 1920, 3)
    for o in (zo.PRESETS["default"], zo.PRESETS["heavy_smooth"], zo.PRESETS["thin"]):
        _check(zb, img, o)


def test_golden_fixtures_including_4200_squared(zb):
    g = json.loads((Path(__file__).resolve().parent / "golden" / "golden_shen_castan.json").read_text())
    assert set(g["cases"]) == set(CASES)
    for name, (build, _preset) in CASES.items():
        img = build()
        assert sha(img) == g["cases"][name]["input_sha256"], name
        got = device(zb, name, img)
        assert sha(got) == g["cases"][name]["output_sha256"], name


def test_presets_of_the_python_mirror(zb):
    img = smooth_noise(51, 60, 80)
    for name in zb.ShenCastan.PRESETS:
        got = getattr(zb.ShenCastan, name).apply(zb.Image.from_numpy(img)).to_numpy()
        assert np.array_equal(got, zo.shen_castan(img, zo.PRESETS[name])), name
    with pytest.raises(zb.ZignalError) as e:
        zb.Image.from_numpy(img).shen_castan(window_size=6)
    assert e.value.name == "WindowSizeMustBeOdd"
