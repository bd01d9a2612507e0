"""Histogram, autocontrast, equalize, Otsu and adaptive-mean thresholds and binary morphology on the GPU, bit-exact against the oracle
(oracle/zo_binary.cpp, bound in tests/binary_oracle.py): every 8-bit format, 1 x N / N x 1 / ragged shapes, strided views with sentinel bytes around them, constant,
two-value, random and smooth content, the empty image, in-place calls, and both box-sum paths of the adaptive threshold."""
import numpy as np
import pytest

import binary_oracle as zo

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    return zb


def _content(kind, shape, rng):
    if kind == "constant":
        return np.full(shape, 77, np.uint8)
    if kind == "two":
        a = np.full(shape, 40, np.uint8)
        a[:, shape[1] // 2:] = 190
        return a
    if kind == "random":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    r = np.arange(shape[0])[:, None] * 3
    c = np.arange(shape[1])[None, :] * 2
    smooth = ((r + c) // 5 % 256).astype(np.uint8)   # smooth ramps
    return np.broadcast_to(smooth[..., None] if len(shape) == 3 else smooth, shape).copy()


SHAPES = [(1, 1000), (1000, 1), (7, 13), (33, 47), (64, 70), (257, 301)]
KINDS = ["constant", "two", "random", "smooth"]
FORMATS = {"u8": (), "rgb8": (3,), "rgba8": (4,)}


def _view(zb, img, pad=(3, 5)):
    """A device view of `img` inside a bigger buffer filled with SENTINEL (rows / cols offset by pad, ragged stride)."""
    t, l = pad
    base = np.full((img.shape[0] + t + 2, img.shape[1] + l + 3) + img.shape[2:], SENTINEL, np.uint8)
    base[t:t + img.shape[0], l:l + img.shape[1]] = img
    dev = zb.Image.from_numpy(base)
    return dev, dev.view(zb.Rectangle(l, t, l + img.shape[1], t + img.shape[0])), base, (t, l)


def _outside(a, img_shape, pad):
    t, l = pad
    m = np.ones(a.shape[:2], bool)
    m[t:t + img_shape[0], l:l + img_shape[1]] = False
    return a[m]


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("shape", SHAPES)
def test_histogram_equalize_autocontrast_match_oracle(zb, fmt, shape):
    rng = np.random.default_rng(shape[0] * 31 + shape[1])
    for kind in KINDS:
        img = _content(kind, shape + FORMATS[fmt], rng)
        dev = zb.Image.from_numpy(img)
        assert np.array_equal(dev.histogram(), zo.histogram(img)), kind
        assert np.array_equal(zb.Image.from_numpy(img).equalize().to_numpy(), zo.equalize(img)), kind
        for cutoff in (0.0, 0.02, 0.2, 0.49):
            assert np.array_equal(zb.Image.from_numpy(img).autocontrast(cutoff).to_numpy(), zo.autocontrast(img, cutoff)), (kind, cutoff)
        # strided view with sentinel bytes around it: only the view is counted and rewritten
        base_dev, v, base, pad = _view(zb, img)
        assert np.array_equal(v.histogram(), zo.histogram(img)), kind
        v.equalize()
        got = base_dev.to_numpy()
        t, l = pad
        assert np.array_equal(got[t:t + shape[0], l:l + shape[1]], zo.equalize(img)), kind
        assert (_outside(got, shape, pad) == SENTINEL).all()
        v.autocontrast(0.02)
        got2 = base_dev.to_numpy()
        assert np.array_equal(got2[t:t + shape[0], l:l + shape[1]], zo.autocontrast(zo.equalize(img), 0.02)), kind
        assert (_outside(got2, shape, pad) == SENTINEL).all()


def test_histogram_family_on_the_empty_image(zb):
    for ch in ((), (3,), (4,)):
        e = zb.Image.init(0, 5, zb.image.pixfmt_of_array(np.zeros((1, 1) + ch, np.uint8)))
        assert not e.histogram().any()
        e.equalize()
        e.autocontrast(0.1)
    e = zb.Image.init(0, 0, zb.PixFmt.U8)
    out, t = e.threshold_otsu()
    assert t == 0
    e.threshold_adaptive_mean(3, 1.0)
    e.open_binary(np.ones((3, 3), np.uint8), 2)


def test_histogram_constant_and_large_images(zb):
    """Uniform 16-byte chunks take the grouped path (one shared-memory add per group of lanes): a constant image must still count right,
    also where rows are not 16-byte aligned."""
    import torch
    for shape in [(4096, 4096, 4), (2048, 1001, 3), (3001, 2049)]:
        t = torch.full(shape, 201, dtype=torch.uint8, device="cuda")
        h = zb.Image.from_tensor(t).histogram()
        n = shape[0] * shape[1]
        assert (h[:, 201] == n).all() and h.sum() == n * h.shape[0]
        g = torch.Generator(device="cuda").manual_seed(shape[1])
        r = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=g)
        r[: shape[0] // 2] = 9   # half constant, half random
        host = r.cpu().numpy()
        assert np.array_equal(zb.Image.from_tensor(r).histogram(), zo.histogram(host))


def test_equalize_above_the_u32_limit_uses_the_64_bit_numerator(zb):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (4200, 4200), dtype=np.uint8)   # total - cdf_min > 16,843,009
    got = zb.Image.from_numpy(img).equalize().to_numpy()
    want = zo.equalize(img)
    assert np.array_equal(got, want)
    cdf = np.cumsum(np.bincount(img.ravel(), minlength=256)).astype(np.int64)
    cdf_min = int(cdf[cdf > 0][0])
    lut = ((cdf - cdf_min) * 255 // (img.size - cdf_min)).astype(np.uint8)
    assert np.array_equal(got, lut[img])


@pytest.mark.parametrize("shape", SHAPES)
def test_threshold_otsu_matches_oracle(zb, shape):
    rng = np.random.default_rng(shape[0] + 7 * shape[1])
    for kind in KINDS:
        img = _content(kind, shape, rng)
        want, wt = zo.threshold_otsu(img)
        out, t = zb.Image.from_numpy(img).threshold_otsu()
        assert t == wt and np.array_equal(out.to_numpy(), want), kind
        base_dev, v, base, pad = _view(zb, img)
        _, t2 = v.threshold_otsu(out=v)                          # in place on a strided view
        got = base_dev.to_numpy()
        ti, li = pad
        assert t2 == wt and np.array_equal(got[ti:ti + shape[0], li:li + shape[1]], want), kind
        assert (_outside(got, shape, pad) == SENTINEL).all()


def test_threshold_otsu_shifted_overlap(zb):
    rng = np.random.default_rng(11)
    base = rng.integers(0, 256, (40, 50), dtype=np.uint8)
    dev = zb.Image.from_numpy(base)
    src = dev.view(zb.Rectangle(0, 0, 50, 30))
    dst = dev.view(zb.Rectangle(0, 5, 50, 35))
    want, wt = zo.threshold_otsu(base[:30].copy())
    _, t = src.threshold_otsu(out=dst)
    assert t == wt and np.array_equal(dev.to_numpy()[5:35], want)


@pytest.mark.parametrize("radius", [1, 2, 15, 16, 67])
@pytest.mark.parametrize("c", [4.0, -3.5, 0.25])
def test_threshold_adaptive_mean_fused_generic_and_in_place(zb, radius, c):
    L = zb.lib()
    rng = np.random.default_rng(radius * 13 + int(c * 4) + 100)
    img = rng.integers(0, 64, (300, 704), dtype=np.uint8) | 0xC0     # bright: SAT values pass 2^24 (4-byte rows: the fused path applies)
    want = zo.threshold_adaptive_mean(img, radius, c)
    dev = zb.Image.from_numpy(img)
    got = dev.threshold_adaptive_mean(radius, c)
    assert L.zb_last_kernel().decode() == ("box_fused_threshold" if radius <= 15 else "sat_threshold")
    assert np.array_equal(got.to_numpy(), want)
    L.zb_set_force_generic(1)
    try:
        got = dev.threshold_adaptive_mean(radius, c)
        assert L.zb_last_kernel().decode() == "sat_threshold"
    finally:
        L.zb_set_force_generic(0)
    assert np.array_equal(got.to_numpy(), want)
    dev.threshold_adaptive_mean(radius, c, out=dev)                 # in place
    assert np.array_equal(dev.to_numpy(), want)
    for shape in [(1, 900), (900, 1), (37, 45)]:                    # thin and ragged shapes, strided views
        small = rng.integers(0, 256, shape, dtype=np.uint8)
        want = zo.threshold_adaptive_mean(small, radius, c)
        base_dev, v, base, pad = _view(zb, small)
        out = zb.Image.from_numpy(np.full(base.shape, SENTINEL, np.uint8))
        ov = out.view(zb.Rectangle(pad[1], pad[0], pad[1] + shape[1], pad[0] + shape[0]))
        v.threshold_adaptive_mean(radius, c, out=ov)
        got = out.to_numpy()
        assert np.array_equal(got[pad[0]:pad[0] + shape[0], pad[1]:pad[1] + shape[1]], want), shape
        assert (_outside(got, shape, pad) == SENTINEL).all()


def test_threshold_adaptive_mean_qr_detector_call(zb):
    rng = np.random.default_rng(67)
    img = _content("smooth", (1080, 1920), rng) ^ rng.integers(0, 32, (1080, 1920), dtype=np.uint8)
    radius = max(min(1080, 1920) // 16, 8)   # qrcode/detector.zig:74
    got = zb.Image.from_numpy(img).threshold_adaptive_mean(radius, 4.0).to_numpy()
    assert np.array_equal(got, zo.threshold_adaptive_mean(img, radius, 4.0))


def _disc(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return (x * x + y * y <= r * r).astype(np.uint8)


KERNELS = {
    "1x1": np.ones((1, 1), np.uint8),
    "3x3": np.ones((3, 3), np.uint8),
    "cross": np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], np.uint8),
    "asym3x5": np.array([[1, 0, 0, 0, 0], [0, 0, 1, 0, 7], [0, 1, 0, 0, 1]], np.uint8),   # holes, not symmetric: shows the unreflected offsets
    "zero": np.zeros((3, 3), np.uint8),
    "1x31": np.ones((1, 31), np.uint8),
    "31x1": np.ones((31, 1), np.uint8),
    "disc15": _disc(7),
}
OPS = {"dilate": "dilate_binary", "erode": "erode_binary", "open": "open_binary", "close": "close_binary"}


@pytest.mark.parametrize("kname", list(KERNELS))
@pytest.mark.parametrize("op", list(OPS))
def test_morphology_matches_oracle(zb, kname, op):
    k = KERNELS[kname]
    rng = np.random.default_rng(len(kname) * 7 + len(op))
    for shape in [(150, 37), (29, 203), (64, 96)]:
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        img[rng.random(shape) < 0.55] = 0                     # non-binary input with mixed density
        for it in (0, 1, 2, 5):
            want = zo.morph_binary(img, k, it, op)
            dev = zb.Image.from_numpy(img)
            got = getattr(dev, OPS[op])(k, it)
            assert np.array_equal(got.to_numpy(), want), (shape, it)
            getattr(dev, OPS[op])(k, it, out=dev)             # in place
            assert np.array_equal(dev.to_numpy(), want), (shape, it, "in place")
        base_dev, v, base, pad = _view(zb, img)              # strided view, in place, sentinel bytes around it
        getattr(v, OPS[op])(k, 2, out=v)
        got = base_dev.to_numpy()
        assert np.array_equal(got[pad[0]:pad[0] + shape[0], pad[1]:pad[1] + shape[1]], zo.morph_binary(img, k, 2, op)), shape
        assert (_outside(got, shape, pad) == SENTINEL).all()


def test_morphology_thin_and_large_images(zb):
    rng = np.random.default_rng(3)
    for shape in [(1, 333), (333, 1), (1000, 1100)]:
        img = (rng.random(shape) < 0.5).astype(np.uint8) * 255
        for op in OPS:
            k = KERNELS["cross"] if shape[0] > 1 else KERNELS["1x31"]
            want = zo.morph_binary(img, k, 2, op)
            got = getattr(zb.Image.from_numpy(img), OPS[op])(k, 2).to_numpy()
            assert np.array_equal(got, want), (shape, op)


def test_morphology_reference_kats(zb):
    box = np.ones((3, 3), np.uint8)
    img = np.zeros((5, 5), np.uint8)
    img[2, 2] = 255
    want = np.zeros((5, 5), np.uint8)
    want[1:4, 1:4] = 255
    assert np.array_equal(zb.Image.from_numpy(img).dilate_binary(box).to_numpy(), want)     # binary.zig tests:60-88
    ring = np.zeros((5, 5), np.uint8)
    ring[1:4, 1:4] = 255
    ring[2, 2] = 0
    dev = zb.Image.from_numpy(ring)
    dev.close_binary(box, out=dev)                                                          # :116-140 (in place)
    assert np.array_equal(dev.to_numpy(), want)
    full = zb.Image.from_numpy(np.full((5, 5), 255, np.uint8)).erode_binary(box, 2).to_numpy()   # :142-167
    assert full[2, 2] == 255 and full.sum() == 255
    with pytest.raises(zb.ZignalError) as e:
        zb.Image.from_numpy(img).dilate_binary(np.ones((2, 3), np.uint8))
    assert e.value.name == "InvalidKernelSize"


def test_binary_fixtures(zb):
    """The device results hash to tests/golden/golden_binary.json."""
    import json
    from pathlib import Path

    from golden_binary import CASES
    from gpu_utils import sha
    g = json.loads((Path(__file__).resolve().parent / "golden" / "golden_binary.json").read_text())
    for name, (build, _oracle, device) in CASES.items():
        res = device(zb, build())
        assert list(res.shape) == g["cases"][name]["shape"] and str(res.dtype) == g["cases"][name]["dtype"], name
        assert sha(res) == g["cases"][name]["output_sha256"], name
