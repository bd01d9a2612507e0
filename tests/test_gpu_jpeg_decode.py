"""jpeg.loadFromBytes on the GPU (zb_jpeg_decode), equal pixel for pixel to the oracle (oracle/zo_jpeg_decode.cpp, bound in
tests/jpeg_decode_oracle.py): zignal-encoder streams of every input format x subsampling x quality decoded to every pixel format,
sizes from 1 x 1 to 8192^2 around the subsequence and tile sizes, the stored fixtures (liza.jpg, Pillow streams with restart
intervals, optimised tables, gray, q100), hand-built streams (4:1:1, gray with id 1 (walked block by block) and id != 1 with 2 x 2 sampling, restart
intervals, FF bytes before an RST (which end the scan), tables whose codes all have one length, the decoding details and error
classes of jpeg_streams.semantic_cases), truncation at many byte positions, corrupted streams, the 65535 limits, a
16384^2 stream past 2^32 bits, strided and wrongly shaped destinations, back-to-back calls, a non-blocking stream and two host
threads.  Every decode also checks the kernel variant the call reports."""
import threading
from pathlib import Path

import numpy as np
import pytest

import jpeg_decode_oracle as jd
import jpeg_oracle as jo
import jpeg_streams as js

pytestmark = pytest.mark.gpu

FIX = Path(__file__).resolve().parent / "golden" / "jpeg_decode"
FMT_NAME = {0: "u8", 1: "f32", 2: "rgb8", 3: "rgba8", 4: "rgbaf32"}
LAYOUT = {(1, 1): "444", (2, 1): "422", (4, 1): "411", (2, 2): "420"}
BIG = jd.Limits(max_jpeg_bytes=0, max_marker_bytes=0, max_width=0, max_height=0, max_pixels=0, max_blocks=0, max_scans=0)


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def zb_limits(zb, lim):
    if lim is None:
        return None
    return zb.JpegLimits(*[getattr(lim, f) for f, _ in jd.Limits._fields_])


def expected_kernel(data, pixfmt):
    h = jd.info(data)
    if h.num_components == 1:
        lay = "gray"
    else:
        # the colour stage follows the luma sampling factors of the SOF
        i = data.index(b"\xFF\xC0")
        f = data[i + 2 + 2 + 6 + 1]
        lay = LAYOUT[(f >> 4, f & 15)]
    return f"jpeg_dec_{lay}_{FMT_NAME[pixfmt]}"


def decode_both(zb, data, pixfmt=None, limits=None, check_kernel=True):
    """(device result as numpy, oracle result), or the two statuses when either refuses."""
    try:
        want = jd.decode(data, pixfmt, limits)
        wrc = 0
    except jd.DecodeError as e:
        want, wrc = None, e.status
    try:
        got = zb.Image.decode_jpeg(data, pixfmt, zb_limits(zb, limits)).to_numpy()
        grc = 0
    except zb.ZignalError as e:
        got, grc = None, e.status
    assert grc == wrc, (grc, wrc)
    if wrc == 0 and check_kernel:
        fmt = pixfmt if pixfmt is not None else (0 if want.ndim == 2 else 2)
        assert zb.lib().zb_last_kernel().decode() == expected_kernel(data, fmt)
    return got, want


def assert_equal(got, want):
    if want is None:
        assert got is None
        return
    assert got.shape == want.shape and got.dtype == want.dtype
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"{len(bad)} elements differ, first at {bad[0].tolist()}: got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def content(rng, rows, cols, fmt):
    y, x = np.mgrid[0:rows, 0:cols]
    base = np.stack([(x * 7 + y * 3) % 256, (y * 5) % 256, ((x ^ y) * 3) % 256], -1)
    img = np.clip(base + rng.integers(-25, 26, base.shape), 0, 255).astype(np.uint8)
    if fmt == 0:
        return img[..., 0].copy()
    if fmt == 1:
        return (img[..., 0] / 255.0).astype(np.float32)
    if fmt == 2:
        return img
    if fmt == 3:
        return np.concatenate([img, np.full((rows, cols, 1), 200, np.uint8)], -1)
    return np.concatenate([img / 255.0, np.ones((rows, cols, 1))], -1).astype(np.float32)


@pytest.mark.parametrize("src_fmt", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("sub", [0, 1, 2])
@pytest.mark.parametrize("quality", [1, 50, 90, 100])
def test_encoder_streams_every_format(zb, src_fmt, sub, quality):
    rng = np.random.default_rng(src_fmt * 100 + sub * 10 + quality)
    img = content(rng, 45, 67, src_fmt)
    data = zb.Image.from_numpy(img).encode_jpeg(quality, sub)
    for out in (None, 0, 1, 2, 3, 4):
        assert_equal(*decode_both(zb, data, out))


@pytest.mark.parametrize("shape", [(1, 1), (1, 2), (2, 1), (7, 9), (8, 8), (9, 8), (16, 16), (17, 33), (1, 300), (300, 1), (63, 65),
                                   (255, 257), (128, 1024), (362, 362), (720, 1280), (1080, 1920), (2049, 17),
                                   # one reconstruction CTA is 80 px wide at 4:4:4 and 4:2:0 (10 and 5 MCUs): +-1 pixel and +-1 tile
                                   (16, 79), (16, 80), (16, 81), (16, 159), (16, 160), (16, 161)])
@pytest.mark.parametrize("sub", [0, 2])
def test_sizes(zb, shape, sub):
    rng = np.random.default_rng(shape[0] * 7 + shape[1])
    img = content(rng, shape[0], shape[1], 2)
    data = jo.encode(img, 90, sub)
    assert_equal(*decode_both(zb, data, 2))


@pytest.mark.parametrize("name", sorted(p.name for p in FIX.glob("*.jpg")))
@pytest.mark.parametrize("pixfmt", [None, 0, 1, 3, 4])
def test_fixtures(zb, name, pixfmt):
    assert_equal(*decode_both(zb, (FIX / name).read_bytes(), pixfmt))


def test_liza_and_8192_encoder_output(zb):
    assert_equal(*decode_both(zb, (FIX / "liza.jpg").read_bytes()))
    rng = np.random.default_rng(8192)
    img = content(rng, 8192, 8192, 2)
    data = zb.Image.from_numpy(img).encode_jpeg(90, 2)
    assert_equal(*decode_both(zb, data, 2))


def _synthetic(kind, rng):
    q = {0: np.full(64, 3), 1: np.full(64, 5)}
    if kind == "411":
        comps = [(1, 4, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
        scan = [(1, 0, 0), (2, 0, 0), (3, 0, 0)]
        w, h = 75, 21
        n = ((w + 31) // 32) * ((h + 7) // 8)
        return js.write(w, h, comps, scan, js.random_mcus(rng, n, [0, 0, 0, 0, 1, 2]), q)
    if kind == "gray_id7_2x2":
        comps = [(7, 2, 2, 0)]
        w, h = 37, 29
        n = ((w + 15) // 16) * ((h + 15) // 16)
        return js.write(w, h, comps, [(7, 0, 0)], js.random_mcus(rng, n, [0, 0, 0, 0]), q)
    if kind == "gray_id1_2x2":
        comps = [(1, 2, 2, 0)]
        w, h = 37, 29
        n = ((w + 7) // 8) * ((h + 7) // 8)
        return js.write(w, h, comps, [(1, 0, 0)], js.random_mcus(rng, n, [0]), q)
    if kind in ("dri_ff_ends_scan", "dri"):
        comps = [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
        w, h = 90, 70
        n = ((w + 15) // 16) * ((h + 15) // 16)
        return js.write(w, h, comps, [(1, 0, 0), (2, 0, 0), (3, 0, 0)], js.random_mcus(rng, n, [0, 0, 0, 0, 1, 2]), q, restart=3,
                        fill_ff_before_rst=2 if kind == "dri_ff_ends_scan" else 0)
    if kind == "flat_tables":
        comps = [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
        w, h = 640, 480
        n = (w // 8) * (h // 8)
        tabs_dc = {0: (js.FLAT_DC_BITS, js.DC_VALS)}
        tabs_ac = {0: (js.FLAT_AC_BITS, js.AC_VALS)}
        return js.write(w, h, comps, [(1, 0, 0), (2, 0, 0), (3, 0, 0)], js.random_mcus(rng, n, [0, 1, 2]), q, tabs_dc, tabs_ac)
    raise KeyError(kind)


@pytest.mark.parametrize("kind", ["411", "gray_id7_2x2", "gray_id1_2x2", "dri", "dri_ff_ends_scan", "flat_tables"])
@pytest.mark.parametrize("pixfmt", [None, 4])
def test_hand_built_streams(zb, kind, pixfmt):
    data = _synthetic(kind, np.random.default_rng(len(kind)))
    got, want = decode_both(zb, data, pixfmt)
    assert want is not None
    assert_equal(got, want)
    if kind == "dri_ff_ends_scan":
        # an FF followed by FF ends the scan (findScanEnd): the decode is a truncation at the first fill, so everything after the
        # first restart interval stays zero and the image differs from the same stream without the fill bytes
        plain = zb.Image.decode_jpeg(_synthetic("dri", np.random.default_rng(len(kind))), pixfmt).to_numpy()
        assert not np.array_equal(got, plain)


@pytest.mark.parametrize("name", list(js.semantic_cases()))
def test_decoding_details_and_error_classes(zb, name):
    """Run to k = 64 without magnitude bits, the ZRL clip, InvalidDCCoefficient, InvalidACCoefficient, InvalidHuffmanCode and
    MissingHuffmanTable, each also behind an end of data that comes first (then the call succeeds), and a second scan that is
    ignored: the device's status and pixels equal the oracle's."""
    data, status, _ = js.semantic_cases()[name]
    got, want = decode_both(zb, data, 2)
    assert (want is None) == bool(status)
    assert_equal(got, want)
    if status:
        with pytest.raises(zb.ZignalError) as e:
            zb.Image.decode_jpeg(data)
        assert e.value.status == status


def _positions(n, rng, data):
    pos = set(range(0, min(n, 700), 37)) | set(rng.integers(0, n, 40).tolist()) | {n - 1, n - 2, n - 3}
    start = data.index(b"\xFF\xDA") + 2 + int.from_bytes(data[data.index(b"\xFF\xDA") + 2:][:2], "big")
    for m in range(1, 5):   # ends of the scan around whole 512-bit subsequences
        pos |= {start + 64 * m - 1, start + 64 * m, start + 64 * m + 1}
    for i in range(len(data) - 1):   # inside an FF 00 pair and right after an RST
        if data[i] == 0xFF and data[i + 1] == 0x00 and len(pos) < 70:
            pos.add(i + 1)
        if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7 and len(pos) < 80:
            pos |= {i + 1, i + 2, i + 3}
    return sorted(p for p in pos if 0 < p <= n)


@pytest.mark.parametrize("name", ["pillow_restart4_420.jpg", "enc420", "enc_gray"])
def test_truncation(zb, name):
    rng = np.random.default_rng(5)
    if name == "enc420":
        data = jo.encode(content(rng, 61, 83, 2), 80, 2)
    elif name == "enc_gray":
        data = jo.encode(content(rng, 61, 83, 0), 80)
    else:
        data = (FIX / name).read_bytes()
    for cut in _positions(len(data), rng, data):
        assert_equal(*decode_both(zb, data[:cut], 2, check_kernel=False))


def test_corrupted_streams(zb):
    """Random byte changes inside the scan: the device gives the oracle's status, and its pixels when both decode."""
    rng = np.random.default_rng(11)
    base = [jo.encode(content(rng, 50, 70, 2), 75, 2), (FIX / "pillow_restart4_420.jpg").read_bytes(),
            (FIX / "pillow_optimize_422.jpg").read_bytes()]
    statuses = set()
    for data in base:
        start = data.index(b"\xFF\xDA") + 14
        for _ in range(25):
            b = bytearray(data)
            for i in rng.integers(start, len(b) - 2, 3):
                b[i] = int(rng.integers(0, 256))
            got, want = decode_both(zb, bytes(b), 2, check_kernel=False)
            statuses.add(want is None)
            assert_equal(got, want)
    assert statuses == {True, False}


def test_header_errors(zb):
    data = jo.encode(content(np.random.default_rng(1), 20, 20, 2), 90, 2)
    cases = {
        "no_soi": data[2:],
        "sof1": data.replace(b"\xFF\xC0", b"\xFF\xC1", 1),
        "progressive": data.replace(b"\xFF\xC0", b"\xFF\xC2", 1),
        "dac": data[:2] + b"\xFF\xCC\x00\x04\x00\x00" + data[2:],
        "no_sos": data[:data.index(b"\xFF\xDA")] + b"\xFF\xD9",
        "too_wide": data,
    }
    want = {"no_soi": 31, "sof1": 3, "progressive": 3, "dac": 3, "no_sos": 31, "too_wide": 30}
    for k, d in cases.items():
        lim = jd.Limits(max_width=19) if k == "too_wide" else None
        got, ref = decode_both(zb, d, 2, lim)
        assert got is None and ref is None
        with pytest.raises(zb.ZignalError) as e:
            zb.Image.decode_jpeg(d, 2, zb_limits(zb, lim))
        assert e.value.status == want[k], k


@pytest.mark.parametrize("shape", [(65535, 8), (8, 65535)])
def test_65535_limits(zb, shape):
    img = content(np.random.default_rng(3), shape[0], shape[1], 2)
    data = jo.encode(img, 90, 2)
    assert_equal(*decode_both(zb, data, 2, BIG))


def test_16384_noise_past_2_32_bits(zb, torch):
    rng = np.random.default_rng(16384)
    img = rng.integers(0, 256, (16384, 16384, 3), dtype=np.uint8)
    data = zb.Image.from_numpy(img).encode_jpeg(100, 0)
    del img
    start = data.index(b"\xFF\xDA")
    assert (len(data) - start) * 8 > 2 ** 32
    got = zb.Image.decode_jpeg(data, 2, zb_limits(zb, BIG))
    assert zb.lib().zb_last_kernel().decode() == "jpeg_dec_444_rgb8"
    want = jd.decode(data, 2, BIG)
    assert_equal(got.to_numpy(), want)


def test_strided_destination_and_wrong_shape(zb, torch):
    data = (FIX / "pillow_optimize_422.jpg").read_bytes()
    h = zb.jpeg_info(data)
    big = zb.Image.from_numpy(np.full((h.height + 10, h.width + 13, 4), 7, np.uint8))
    view = big.view(zb.Rectangle(5, 3, 5 + h.width, 3 + h.height))
    zb.Image.decode_jpeg(data, out=view)
    full = big.to_numpy()
    want = jd.decode(data, 3)
    assert_equal(full[3:3 + h.height, 5:5 + h.width], want)
    mask = np.ones(full.shape[:2], bool)
    mask[3:3 + h.height, 5:5 + h.width] = False
    assert (full[mask] == 7).all()
    wrong = zb.Image.init(h.height, h.width + 1, 2)
    with pytest.raises(zb.ZignalError) as e:
        zb.Image.decode_jpeg(data, out=wrong)
    assert e.value.status == 1


def test_streams_and_threads(zb, torch):
    a = (FIX / "liza.jpg").read_bytes()
    b = (FIX / "pillow_restart4_420.jpg").read_bytes()
    wa, wb = jd.decode(a), jd.decode(b)
    for _ in range(3):   # back to back
        assert_equal(zb.Image.decode_jpeg(a).to_numpy(), wa)
        assert_equal(zb.Image.decode_jpeg(b).to_numpy(), wb)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = zb.Image.decode_jpeg(a)
    s.synchronize()
    assert_equal(got.to_numpy(), wa)
    errs = []

    def run(data, want):
        try:
            for _ in range(4):
                assert_equal(zb.Image.decode_jpeg(data).to_numpy(), want)
        except Exception as e:   # reported below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(a, wa)), threading.Thread(target=run, args=(b, wb))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_golden_hashes(zb):
    """The device's pixels for every stored stream and pixel format hash to the values tests/golden/make_golden_jpeg_decode.py
    recorded from the oracle."""
    import hashlib
    import json
    want = json.loads((FIX.parent / "golden_jpeg_decode.json").read_text())
    assert len(want) == 5 * len(list(FIX.glob("*.jpg")))
    for key, digest in want.items():
        name, fmt = key.split(":")
        got = zb.Image.decode_jpeg((FIX / name).read_bytes(), list(FMT_NAME.values()).index(fmt)).to_numpy()
        assert hashlib.sha256(got.tobytes()).hexdigest() == digest, key
