"""Colour quantization and dithering on the GPU, bit-identical to the oracle (oracle/zo_quantize.cpp, bound in tests/quantize_oracle.py):
median cut over every pixel format with max_colors from 0 to 256 and caps below it, an image touching all 32768 bins in shuffled order,
the LUT for fixed, random, tiny and duplicate-laden palettes, every dither mode from 1 x 1 through odd sizes, warp and band boundaries
+-1, 4096^2 and 8192^2, a 70,000 x 3 tall and a 3 x 70,000 wide image, saturated noise under VGA16, strided views guarded by sentinels,
back-to-back calls on one stream, a non-blocking stream and two host threads, the GIF chain on a 1080p frame and the golden fixtures."""
import json
import threading
from pathlib import Path

import numpy as np
import pytest

import quantize_oracle as zo
from golden_quantize import CASES, DITHER_MODES, FORMATS, all_bins_shuffled, palette, random_image, random_palette, smooth_rgb
from gpu_utils import sha

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_quantize.json"
KERNEL = {zo.FLOYD_STEINBERG: "dither_floyd_steinberg", zo.ATKINSON: "dither_atkinson", zo.ORDERED: "dither_ordered"}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def _dither(zb, img, pal, mode):
    lut = zb.ColorLookupTable(pal)
    dev = zb.Image.from_numpy(img)
    assert dev.dither(lut, zb.DitherMode(mode)) is dev
    if mode in KERNEL:
        assert zb.lib().zb_last_kernel().decode() == KERNEL[mode]
    return dev.to_numpy()


def _check_dither(zb, img, pal, mode, what=""):
    got = _dither(zb, img, pal, mode)
    want = zo.dither(img.copy(), pal, zo.color_lut(pal), mode)
    if sha(got) != sha(want):
        bad = (got != want).any(axis=2)
        pytest.fail(f"{what} {img.shape} mode {mode} n {len(pal)}: {int(bad.sum())} pixels differ, first at {np.argwhere(bad)[:3].tolist()}")


def test_reference_tests(zb):
    # sixel: a 4x4 eight-colour image, adaptive with max_colors 4 -> at most 4 entries
    cols8 = np.array([[0, 0, 0], [255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [255, 0, 255], [0, 255, 255], [255, 255, 255]], np.uint8)
    img = cols8[np.arange(16) % 8].reshape(4, 4, 3)
    got = zb.build_palette(zb.Image.from_numpy(img), zb.PaletteMode.ADAPTIVE, 4)
    assert 1 <= len(got) <= 4 and np.array_equal(got, zo.build_palette(img, zo.ADAPTIVE, 4))
    # the fixed 6x7x6 mapping of black, white and red
    pal = zb.build_palette(zb.Image.from_numpy(img), zb.PaletteMode.FIXED_6X7X6)
    lut = zb.ColorLookupTable(pal)
    px = np.array([[[0, 0, 0], [255, 255, 255], [255, 0, 0]]], np.uint8)
    idx = zb.Image.from_numpy(px).palette_indices(lut).to_numpy()
    assert [tuple(pal[i]) for i in idx[0]] == [(0, 0, 0), (255, 255, 255), (255, 0, 0)]
    # a single-colour 4x4 -> one entry, the colour of its 5-bit bin (r5 << 3 | r5 >> 2, ...)
    one = np.full((4, 4, 3), (10, 20, 30), np.uint8)
    assert zb.median_cut(zb.Image.from_numpy(one), 16).tolist() == [[8, 16, 24]]
    # GIF: 16x16 gradient; 8x8 / 8-colour Floyd-Steinberg
    rr, cc = np.mgrid[0:16, 0:16]
    grad = np.stack([rr * 16, cc * 16, (rr + cc) * 8], axis=2).astype(np.uint8)
    assert np.array_equal(zb.median_cut(zb.Image.from_numpy(grad), 256), zo.median_cut(grad, 256))
    small = grad[:8, :8].copy()
    pal8 = zo.median_cut(small, 8)
    _check_dither(zb, small, pal8, zo.FLOYD_STEINBERG)


@pytest.mark.parametrize("fmt", FORMATS)
def test_median_cut_formats(zb, fmt):
    img = random_image(fmt, 67, 131, 3)
    dev = zb.Image.from_numpy(img)
    for max_colors in (0, 1, 2, 3, 7, 16, 100, 255, 256):
        for cap in sorted({256, max_colors, max(max_colors - 1, 0), 1}):
            try:
                want = zo.median_cut(img, max_colors, cap)
            except zo.OracleStatus as e:
                assert e.status == zo.NO_PALETTE_COLORS
                with pytest.raises(zb.ZignalError) as ge:
                    zb.median_cut(dev, max_colors, cap)
                assert ge.value.name == "NoPaletteColors"
                continue
            got = zb.median_cut(dev, max_colors, cap)
            assert np.array_equal(got, want), (fmt, max_colors, cap)
        assert zb.lib().zb_last_kernel().decode() == "median_cut_histogram"
    for mode in (zo.FIXED_6X7X6, zo.FIXED_VGA16, zo.FIXED_WEB216, zo.ADAPTIVE):
        assert np.array_equal(zb.build_palette(dev, zb.PaletteMode(mode), 200), zo.build_palette(img, mode, 200))


def test_all_bins_shuffled_and_large_median_cut(zb):
    img = all_bins_shuffled(11)
    for k in (2, 17, 256):
        assert np.array_equal(zb.median_cut(zb.Image.from_numpy(img), k), zo.median_cut(img, k))
    big = smooth_rgb(8192, 8192, 5)
    assert np.array_equal(zb.median_cut(zb.Image.from_numpy(big), 256), zo.median_cut(big, 256))


def test_lut(zb):
    pals = [palette("6x7x6"), palette("vga16"), palette("web216")] + [random_palette(n, n) for n in (1, 2, 15, 16, 17, 33, 255, 256)]
    dup = random_palette(40, 9)
    dup[20:] = dup[:20]                                            # duplicates: the lower index wins
    pals.append(dup)
    pals.append(np.zeros((256, 3), np.uint8))
    for p in pals:
        lut = zb.ColorLookupTable(p)
        assert zb.lib().zb_last_kernel().decode() == "color_lut"
        assert np.array_equal(lut.to_numpy(), zo.color_lut(p)), len(p)


SIZES = [(1, 1), (1, 2), (2, 1), (2, 2), (1, 9), (9, 1), (3, 5), (31, 31), (32, 32), (33, 33), (31, 65), (63, 64), (64, 63), (65, 97),
         (95, 31), (96, 3), (97, 200), (127, 129), (128, 1), (129, 130), (255, 257), (300, 77)]


@pytest.mark.parametrize("mode", DITHER_MODES)
def test_dither_sizes(zb, mode):
    for k, (rows, cols) in enumerate(SIZES):
        img = smooth_rgb(rows, cols, k) if k % 2 else random_image("rgb8", rows, cols, k)
        for kind in ("vga16", "random2", "6x7x6", "random256"):
            _check_dither(zb, img, palette(kind), mode, kind)
    # palettes of 1 entry, and with duplicates
    img = smooth_rgb(70, 90, 1)
    _check_dither(zb, img, random_palette(1, 4), mode)
    dup = random_palette(30, 5)
    dup[15:] = dup[:15]
    _check_dither(zb, img, dup, mode)


@pytest.mark.parametrize("mode", [zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED])
def test_dither_large(zb, mode):
    for n in (4096, 8192):
        img = smooth_rgb(n, n, n)
        pal = zo.median_cut(img, 64)
        _check_dither(zb, img, pal, mode, f"{n}^2")


@pytest.mark.parametrize("mode", [zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED])
def test_tall_and_wide(zb, mode):
    for shape in ((70000, 3), (3, 70000)):
        img = smooth_rgb(*shape, 3)
        _check_dither(zb, img, palette("web216"), mode, str(shape))


def test_saturated_noise_vga16(zb):
    rng = np.random.default_rng(12)
    img = np.where(rng.random((517, 611, 3)) < 0.5, 0, 255).astype(np.uint8)
    img[rng.random((517, 611)) < 0.3] = (255, 255, 255)
    for mode in (zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED):
        _check_dither(zb, img, palette("vga16"), mode)


def test_palette_lookup_formats(zb):
    pal = random_palette(77, 3)
    lut = zb.ColorLookupTable(pal)
    want_lut = zo.color_lut(pal)
    for fmt in FORMATS:
        for shape in ((1, 1), (33, 257), (1000, 999)):
            img = random_image(fmt, *shape, 7)
            got = zb.Image.from_numpy(img).palette_indices(lut).to_numpy()
            assert zb.lib().zb_last_kernel().decode() == "palette_lookup"
            assert np.array_equal(got, zo.palette_lookup(img, want_lut)), (fmt, shape)


def test_strided_views_with_sentinels(zb, torch):
    base = smooth_rgb(300, 400, 21)
    l, t, r, b = 37, 13, 37 + 255, 13 + 201
    pal = palette("vga16")
    lut = zb.ColorLookupTable(pal)
    for mode in (zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED):
        big = np.full_like(base, 0xA5)
        big[t:b, l:r] = base[t:b, l:r]
        dev = zb.Image.from_numpy(big)
        dev.view(zb.Rectangle(l, t, r, b)).dither(lut, zb.DitherMode(mode))
        expect = big.copy()
        zo.dither(expect[t:b, l:r], pal, zo.color_lut(pal), mode)
        assert sha(dev.to_numpy()) == sha(expect), mode
    big = base.copy()
    v = zb.Image.from_numpy(big).view(zb.Rectangle(l, t, r, b))
    assert np.array_equal(v.palette_indices(lut).to_numpy(), zo.palette_lookup(np.ascontiguousarray(big[t:b, l:r]), zo.color_lut(pal)))
    assert np.array_equal(zb.median_cut(v, 50), zo.median_cut(big[t:b, l:r], 50))


def test_back_to_back_on_one_stream(zb, torch):
    pal = palette("web216")
    lut = zb.ColorLookupTable(pal)
    imgs = [smooth_rgb(200 + 31 * k, 300 - 17 * k, k) for k in range(4)]
    devs = [zb.Image.from_numpy(i) for i in imgs]
    for _ in range(2):                                             # the second round dithers the dithered images
        for d in devs:
            d.dither(lut, zb.DitherMode.ATKINSON)
            d.dither(lut, zb.DitherMode.FLOYD_STEINBERG)
    want_lut = zo.color_lut(pal)
    for img, d in zip(imgs, devs):
        w = img.copy()
        for _ in range(2):
            zo.dither(w, pal, want_lut, zo.ATKINSON)
            zo.dither(w, pal, want_lut, zo.FLOYD_STEINBERG)
        assert sha(d.to_numpy()) == sha(w)


def test_non_blocking_stream_and_two_threads(zb, torch):
    def case(seed):
        img = smooth_rgb(1031, 1537, seed)
        pal = zo.median_cut(img, 32)
        return img, pal, zo.dither(img.copy(), pal, zo.color_lut(pal), zo.FLOYD_STEINBERG)

    cases = {seed: case(seed) for seed in (1, 2)}
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        img, pal, want = cases[1]
        dev = zb.Image.from_numpy(img)
        lut = zb.ColorLookupTable(pal)
        dev.dither(lut, zb.DitherMode.FLOYD_STEINBERG)
        s.synchronize()
        assert sha(dev.to_numpy()) == sha(want)
    results, errors = {}, []
    start = threading.Barrier(2)

    def work(seed):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                img, pal, _ = cases[seed]
                dev = zb.Image.from_numpy(img)
                lut = zb.ColorLookupTable(pal)
                st.synchronize()
                start.wait()
                dev.dither(lut, zb.DitherMode.FLOYD_STEINBERG)
                st.synchronize()
                results[seed] = dev.to_numpy()
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
        assert sha(results[seed]) == sha(cases[seed][2]), seed


def test_gif_chain_1080p(zb):
    frame = random_image("rgbaf32", 1080, 1920, 5)
    dev = zb.Image.from_numpy(frame)
    rgb = dev.convert(zb.PixFmt.RGB8)
    pal = zb.median_cut(rgb, 256)
    lut = zb.ColorLookupTable(pal)
    rgb.dither(lut, zb.DitherMode.FLOYD_STEINBERG)
    idx = rgb.palette_indices(lut).to_numpy()
    want_rgb = zo.as_rgb8(frame)
    want_pal = zo.median_cut(want_rgb, 256)
    want_lut = zo.color_lut(want_pal)
    want_img = zo.dither(want_rgb.copy(), want_pal, want_lut, zo.FLOYD_STEINBERG)
    assert np.array_equal(pal, want_pal)
    assert np.array_equal(lut.to_numpy(), want_lut)
    assert sha(rgb.to_numpy()) == sha(want_img)
    assert sha(idx) == sha(zo.palette_lookup(want_img, want_lut))


def test_argument_errors(zb, torch):
    L = zb.lib()
    img = zb.Image.from_numpy(smooth_rgb(8, 8))
    a = img._zb()
    pal = np.zeros((4, 3), np.uint8)
    lut = torch.zeros(32768, dtype=torch.uint8, device="cuda")
    p = pal.ctypes.data
    assert L.zb_dither(a, int(zb.PixFmt.RGBA8), p, 4, lut.data_ptr(), 1, None) == 3
    assert L.zb_dither(a, int(zb.PixFmt.RGB8), p, 0, lut.data_ptr(), 1, None) == 5
    assert L.zb_dither(a, int(zb.PixFmt.RGB8), p, 257, lut.data_ptr(), 1, None) == 5
    assert L.zb_dither(a, int(zb.PixFmt.RGB8), p, 4, lut.data_ptr(), 5, None) == 5
    assert L.zb_dither(a, int(zb.PixFmt.RGB8), None, 4, lut.data_ptr(), 1, None) == 5
    assert L.zb_color_lut(p, 0, lut.data_ptr(), None) == 5
    assert L.zb_color_lut(p, 257, lut.data_ptr(), None) == 5
    out = zb.Image.init(8, 9, zb.PixFmt.U8)
    assert L.zb_palette_lookup(a, int(zb.PixFmt.RGB8), lut.data_ptr(), out._zb(), None) == 1
    with pytest.raises(zb.ZignalError) as e:
        zb.median_cut(img, 0)
    assert e.value.status == 28 and e.value.name == "NoPaletteColors"
    assert len(zb.build_palette(img, zb.PaletteMode.ADAPTIVE, 0)) == 252   # the reference's fallback


def test_golden_fixtures(zb):
    gold = json.loads(GOLDEN.read_text())["cases"]
    for name, (builder, kind, mode) in CASES.items():
        img = builder()
        g = gold[name]
        assert sha(img) == g["input_sha256"], name
        dev = zb.Image.from_numpy(img)
        if kind.startswith("adaptive"):
            pal = zb.build_palette(dev, zb.PaletteMode.ADAPTIVE, int(kind[8:]))
        else:
            pal = palette(kind)
        assert sha(pal) == g["palette_sha256"], name
        lut = zb.ColorLookupTable(pal)
        assert sha(lut.to_numpy()) == g["lut_sha256"], name
        assert sha(dev.palette_indices(lut).to_numpy()) == g["indices_sha256"], name
        assert sha(dev.dither(lut, zb.DitherMode(mode)).to_numpy()) == g["dithered_sha256"], name
