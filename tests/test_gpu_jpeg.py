"""jpeg.encode on the GPU (zb_jpeg_encode), byte-identical to the oracle (oracle/zo_jpeg.cpp, bound in tests/jpeg_oracle.py): every pixel
format x subsampling x quality, sizes from 1 x 1 to 16384^2 with +-1 around the kernels' tile sizes, the 65535 limits and the 65536
errors, constant / noise / DC-ramp / checkerboard / trailing-ZRL content, strided views, a capacity one byte short, the golden fixtures,
back-to-back calls, a non-blocking stream and two host threads.  Every case also checks the kernel variant the call reports."""
import ctypes as C
import hashlib
import json
import threading
from pathlib import Path

import numpy as np
import pytest

import jpeg_oracle as jo
from golden_jpeg import CASES, FORMATS, case_input, case_options, make, noise, smooth

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_jpeg.json"
SUB_NAME = {0: "444", 1: "422", 2: "420"}
FMT_NAME = {0: "u8", 1: "f32", 2: "rgb8", 3: "rgba8", 4: "rgbaf32"}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def kernel_for(pix, sub):
    return "jpeg_gray_u8" if pix == 0 else f"jpeg_{SUB_NAME[sub]}_{FMT_NAME[pix]}"


def encode_both(zb, img, quality=90, subsampling=2, density_dpi=72, comment=None):
    dev = zb.Image.from_numpy(img)
    got = dev.encode_jpeg(quality, subsampling, density_dpi, comment)
    assert zb.lib().zb_last_kernel().decode() == kernel_for(int(dev.pixfmt), subsampling)
    want = jo.encode(img, quality, subsampling, density_dpi, comment)
    return got, want


def assert_same(got: bytes, want: bytes):
    if got != want:
        n = min(len(got), len(want))
        first = next((i for i in range(n) if got[i] != want[i]), n)
        pytest.fail(f"bytes differ: len {len(got)} vs {len(want)}, first difference at byte {first}")


# grayscale ignores the subsampling, so u8 runs once per quality
FMT_SUB = [("u8", 2)] + [(f, s) for f in FORMATS[1:] for s in (0, 1, 2)]


@pytest.mark.parametrize("fmt,sub", FMT_SUB)
@pytest.mark.parametrize("quality", [1, 50, 90, 100])
def test_formats_subsamplings_qualities(zb, fmt, sub, quality):
    img = smooth(fmt, 37, 53, 11) if quality != 100 else noise(fmt, 37, 53, 12)
    assert_same(*encode_both(zb, img, quality, sub))


# 1 x 1 .. 37 x 53, 1080p; MCUs per CTA are 32 / 10 / 8 / 5 (gray / 444 / 422 / 420), the scan tile is 2048 blocks and a stuffing
# thread takes 16 bytes, so widths of k MCU-per-CTA groups +-1 pixel and block counts around 2048 are the edges.
SIZES = [(1, 1), (1, 7), (7, 1), (1, 300), (300, 1), (7, 9), (8, 8), (9, 8), (15, 17), (16, 16), (17, 33), (37, 53),
         (8, 8 * 32 - 1), (8, 8 * 32), (8, 8 * 32 + 1), (16, 16 * 5 - 1), (16, 16 * 5 + 1), (8, 8 * 10 + 1), (16, 16 * 8 + 1),
         (8, 8 * 2047), (8, 8 * 2048), (8, 8 * 2048 + 1), (16, 8 * 2048 + 8), (1080, 1920)]


@pytest.mark.parametrize("shape", SIZES, ids=[f"{r}x{c}" for r, c in SIZES])
@pytest.mark.parametrize("fmt,sub", [("u8", 0), ("rgb8", 0), ("rgb8", 1), ("rgb8", 2), ("rgba8", 2)])
def test_sizes(zb, shape, fmt, sub):
    img = noise(fmt, *shape, seed=shape[0] * 7 + shape[1])
    assert_same(*encode_both(zb, img, 90, sub))


@pytest.mark.parametrize("fmt,sub,quality,kind", [("u8", 0, 90, "smooth"), ("rgb8", 2, 90, "smooth"), ("rgb8", 0, 100, "noise"),
                                                   ("f32", 1, 75, "smooth")])
def test_4096(zb, fmt, sub, quality, kind):
    img = make(kind, fmt, 4096, 4096, 21)
    assert_same(*encode_both(zb, img, quality, sub))


def test_8192_rgb8_save_default_and_q100_444(zb):
    img = smooth("rgb8", 8192, 8192, 22)
    assert_same(*encode_both(zb, img, 90, 2))
    img = noise("rgb8", 8192, 8192, 23)   # 3 M blocks: more than 1024 scan tiles
    assert_same(*encode_both(zb, img, 100, 0))


def test_16384_noise_q100_444_passes_2_pow_32_bits(zb):
    img = noise("rgb8", 16384, 16384, 24)
    dev = zb.Image.from_numpy(img)
    got = dev.encode_jpeg(100, 0)
    assert zb.lib().zb_last_kernel().decode() == "jpeg_444_rgb8"
    want = jo.encode(img, 100, 0)
    assert len(got) == len(want) and len(want) * 8 > 2 ** 32
    assert hashlib.sha256(got).hexdigest() == hashlib.sha256(want).hexdigest()


@pytest.mark.parametrize("shape", [(65535, 8), (8, 65535)])
@pytest.mark.parametrize("fmt,sub", [("u8", 0), ("rgb8", 2)])
def test_largest_dimension(zb, shape, fmt, sub):
    assert_same(*encode_both(zb, noise(fmt, *shape, seed=31), 85, sub))


@pytest.mark.parametrize("shape", [(65536, 8), (8, 65536), (0, 8), (8, 0)])
def test_dimension_errors(zb, torch, shape):
    t = torch.zeros(max(1, shape[0] * shape[1]) * 3, dtype=torch.uint8, device="cuda")
    img = zb.Image(t, zb.PixFmt.RGB8, shape[0], shape[1], max(1, shape[1]))
    want = "ImageTooLarge" if max(shape) > 65535 else "InvalidImageDimensions"
    with pytest.raises(zb.ZignalError, match=want):
        img.encode_jpeg()


@pytest.mark.parametrize("kind,fmt,sub,quality", [("const0", "rgb8", 2, 90), ("const255", "rgb8", 0, 100), ("const0", "u8", 0, 100),
                                                  ("const255", "rgbaf32", 1, 50), ("dc_ramp", "rgb8", 0, 100),
                                                  ("dc_ramp", "rgb8", 2, 100), ("checker", "rgb8", 0, 100), ("checker", "rgb8", 2, 100),
                                                  ("trailing", "u8", 0, 50), ("trailing", "u8", 0, 90)])
def test_content(zb, kind, fmt, sub, quality):
    img = make(kind, fmt, 128, 128, 41)
    if kind == "trailing":
        zz = jo.coefficients(img, quality, sub)[:, jo.ZIGZAG]
        last = {int(np.nonzero(r)[0].max()) for r in zz if np.any(r)}
        assert {15, 31, 47, 63} <= last
    if kind == "dc_ramp":
        assert np.abs(np.diff(jo.coefficients(img, quality, sub)[:, 0])).max() >= 1024   # category 11
    assert_same(*encode_both(zb, img, quality, sub))


@pytest.mark.parametrize("fmt", FORMATS)
def test_strided_view(zb, fmt):
    big = smooth(fmt, 70, 90, 51)
    dev = zb.Image.from_numpy(big).view(zb.Rectangle(5, 3, 5 + 61, 3 + 43))
    got = dev.encode_jpeg(85, 1)
    want = jo.encode(np.ascontiguousarray(big[3:46, 5:66]), 85, 1)
    assert_same(got, want)


def test_capacity_one_byte_short(zb, torch):
    img = smooth("rgb8", 40, 56, 61)
    want = jo.encode(img, 90, 2)
    dev = zb.Image.from_numpy(img)
    opts = zb._ffi.ZbJpegOptions(90, 2, 72, None, 0)
    buf = (C.c_uint8 * len(want))(*([0xAB] * len(want)))
    n = C.c_uint64(0)
    s = torch.cuda.current_stream().cuda_stream
    rc = zb.lib().zb_jpeg_encode(dev._zb(), int(dev.pixfmt), C.byref(opts), buf, len(want) - 1, C.byref(n), s)
    assert rc == 6 and n.value == len(want)
    assert bytes(buf) == b"\xab" * len(want)
    rc = zb.lib().zb_jpeg_encode(dev._zb(), int(dev.pixfmt), C.byref(opts), buf, len(want), C.byref(n), s)
    assert rc == 0 and n.value == len(want) and bytes(buf) == want
    bound = zb.jpeg_encode_bound(40, 56, zb.PixFmt.RGB8)
    assert bound >= len(want)


def test_small_capacity_retry_in_python(zb):
    # noise at q100 4:4:4 outgrows the raw pixel bytes, so the mirror's first attempt reports the size and the second fetches it
    img = noise("u8", 64, 64, 62)
    got, want = encode_both(zb, img, 100, 0)
    assert len(want) > img.size
    assert_same(got, want)


def test_header_options(zb):
    img = smooth("rgb8", 20, 30, 71)
    for comment in (None, b"", b"x" * 65533):
        assert_same(*encode_both(zb, img, 90, 2, 300, comment))
    with pytest.raises(zb.ZignalError, match="InvalidArgument"):
        zb.Image.from_numpy(img).encode_jpeg(comment=b"x" * 65534)
    with pytest.raises(zb.ZignalError, match="InvalidArgument"):
        zb.Image.from_numpy(img).encode_jpeg(subsampling=3)


def test_golden_fixtures(zb):
    gold = json.loads(GOLDEN.read_text())["cases"]
    assert set(gold) == set(CASES)
    for name in CASES:
        img = case_input(name)
        got = zb.Image.from_numpy(img).encode_jpeg(**case_options(name))
        assert hashlib.sha256(got).hexdigest() == gold[name]["sha256"] and len(got) == gold[name]["len"], name


def test_back_to_back_and_streams(zb, torch):
    imgs = [smooth("rgb8", 48 + 8 * k, 64 + 16 * k, 80 + k) for k in range(4)]
    want = [jo.encode(a, 85, 2) for a in imgs]
    devs = [zb.Image.from_numpy(a) for a in imgs]
    assert [d.encode_jpeg(85, 2) for d in devs] == want
    s = torch.cuda.Stream()   # non-blocking with respect to the legacy default stream
    with torch.cuda.stream(s):
        got = [d.encode_jpeg(85, 2) for d in devs]
    assert got == want
    results = {}

    def worker(k):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            results[k] = [devs[i].encode_jpeg(85, 2) for i in range(4) for _ in range(3)]

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for k in range(2):
        assert results[k] == [want[i] for i in range(4) for _ in range(3)]
