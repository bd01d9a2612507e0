"""HoughTransform on the GPU, bit-exact against the oracle (oracle/zo_hough.cpp, bound in tests/hough_oracle.py): the accumulator must equal
the oracle's cell for cell and find_lines must return identical lines, over odd and even sizes up to 4096, boxes inside, partly and fully
outside the image, random edge values 1..255, prior accumulator contents, strided edge and accumulator views guarded by sentinels, an empty
and an all-255 box, the size = 32768 limit, a canny -> compute -> find_lines chain on a 1080p frame, a capacity below the line count and the
golden fixtures.

The vote kernel counts in u32 shared-memory counters, so no counter bound below the reference's own u32 applies; the all-255 box is the
densest per-cell count (about 2 size votes in a cell along a line)."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

import hough_oracle as zo
from golden_hough import CASES, device, edges, lines_array
from gpu_utils import sha

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_hough.json"
SENTINEL = -0x5A5A5A5B   # 0xA5A5A5A5 as int32


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def _lines(lines):
    return [(l.angle, l.radius, l.score, l.p1[0], l.p1[1], l.p2[0], l.p2[1]) for l in lines]


def _check(zb, torch, size, img, box, prior=None, thresholds=(), nms=(4.0, 3.0), dtype=None):
    """compute on the device and in the oracle from the same prior; then find_lines at each threshold."""
    dtype = dtype or torch.int32
    prior = np.zeros((size, size), np.uint32) if prior is None else prior
    acc = torch.from_numpy(prior.view(np.int32)).cuda()
    if dtype != torch.int32:
        acc = acc.view(dtype)
    h = zb.HoughTransform(size)
    h.compute(zb.Image.from_numpy(img), zb.Rectangle(*box), acc)
    assert zb.lib().zb_last_kernel().decode() == "hough_vote" or not _intersects(img, box)
    got = acc.view(torch.int32).cpu().numpy().view(np.uint32)
    want = zo.compute(size, img, box, prior.copy())
    assert np.array_equal(got, want), (size, box, int((got != want).sum()))
    for th in thresholds:
        assert _lines(h.find_lines(acc, th, *nms)) == zo.find_lines(size, want, th, *nms), (size, box, th)
    return want


def _intersects(img, box):
    l, t, r, b = box
    return l < min(r, img.shape[1]) and t < min(b, img.shape[0])


def _random(seed, rows, cols, density):
    rng = np.random.default_rng(seed)
    img = rng.integers(1, 256, (rows, cols), dtype=np.uint8)
    img[rng.random((rows, cols)) >= density] = 0
    return img


@pytest.mark.parametrize("size", [2, 3, 4, 5, 31, 33, 300, 1024, 1025, 4096])
@pytest.mark.parametrize("where", ["inside", "partly_outside", "fully_outside"])
def test_sizes_and_boxes(zb, torch, size, where):
    rows, cols = size + 11, size + 17
    img = _random(size + len(where), rows, cols, 0.3 if size < 300 else (0.02 if size < 4096 else 0.002))
    box = {"inside": (2, 3, 2 + size, 3 + size), "partly_outside": (cols // 2, rows // 3, cols // 2 + size, rows // 3 + size),
           "fully_outside": (cols, 0, cols + size, size)}[where]
    prior = np.random.default_rng(size).integers(0, 500, (size, size), dtype=np.uint32)
    acc = _check(zb, torch, size, img, box, prior)
    votes = acc.astype(np.int64) - prior
    ths = (int(acc.max()) - 5, int(votes.max()) // 2 + 500) if size <= 1025 else (int(acc.max()) - 40,)
    for th in ths:
        h = zb.HoughTransform(size)
        t_acc = torch.from_numpy(acc.view(np.int32)).cuda()
        assert _lines(h.find_lines(t_acc, th, 4.0, 3.0)) == zo.find_lines(size, acc, th, 4.0, 3.0), th


def test_uint32_accumulator_and_plateaus(zb, torch):
    size = 33
    img = _random(3, 40, 40, 0.3)
    _check(zb, torch, size, img, (0, 0, size, size), thresholds=(0, 5, 30), dtype=torch.uint32)


def test_strided_views_with_sentinels(zb, torch):
    size = 301
    img_big = _random(21, 420, 500, 0.03)
    view = img_big[13:380, 29:450]                      # the edge map: a strided view
    dev_big = zb.Image.from_numpy(img_big)
    dev_view = dev_big.view(zb.Rectangle(29, 13, 450, 380))
    box = (40, 60, 40 + size, 60 + size)                # partly outside the view
    prior = np.random.default_rng(1).integers(0, 1000, (size, size), dtype=np.uint32)
    big = torch.full((size + 6, size + 40), SENTINEL, dtype=torch.int32, device="cuda")
    acc = big[3:3 + size, 17:17 + size]
    acc.copy_(torch.from_numpy(prior.view(np.int32)).cuda())
    h = zb.HoughTransform(size)
    h.compute(dev_view, zb.Rectangle(*box), acc)
    want = zo.compute(size, view, box, prior.copy())
    assert np.array_equal(acc.cpu().numpy().view(np.uint32), want)
    b = big.cpu().numpy()
    assert (b[:3] == SENTINEL).all() and (b[3 + size:] == SENTINEL).all()
    assert (b[:, :17] == SENTINEL).all() and (b[:, 17 + size:] == SENTINEL).all()
    assert np.array_equal(dev_big.to_numpy(), img_big)   # compute does not write the edge map
    th = int(want.max()) - 20
    assert _lines(h.find_lines(acc, th, 3.0, 3.0)) == zo.find_lines(size, np.ascontiguousarray(want), th, 3.0, 3.0)


def test_empty_and_all_255_boxes(zb, torch):
    size = 300
    _check(zb, torch, size, np.zeros((400, 400), np.uint8), (50, 50, 350, 350), thresholds=(0, 1))
    for size in (300, 1024):
        full = np.full((size + 8, size + 8), 255, np.uint8)
        acc = _check(zb, torch, size, full, (4, 4, 4 + size, 4 + size), thresholds=())
        assert acc.max() >= size   # the densest cells: about 2 size votes along a line
        th = int(acc.max()) * 3 // 4
        h = zb.HoughTransform(size)
        assert _lines(h.find_lines(torch.from_numpy(acc.view(np.int32)).cuda(), th, 2.0, 2.0)) == zo.find_lines(size, acc, th, 2.0, 2.0)


def test_size_32768_on_a_sparse_map(zb, torch):
    size = 32768
    img = _random(5, 900, 1100, 0.0001)
    img[450, 100:1000] = 255                            # one horizontal run, so find_lines has a clear peak
    acc = torch.zeros((size, size), dtype=torch.int32, device="cuda")
    h = zb.HoughTransform(size)
    h.compute(zb.Image.from_numpy(img), zb.Rectangle(0, 0, size, size), acc)
    # expected votes from the oracle's tables (the restatement checked against the oracle in tests/test_hough_host.py)
    cos_t, sin_t = (t.astype(np.int64) for t in zo.tables(size))
    ys, xs = np.nonzero(img)
    x_val, y_val = 2 * xs.astype(np.int64) - (size - 1), 2 * ys.astype(np.int64) - (size - 1)
    rho = x_val[:, None] * cos_t[None, :] + y_val[:, None] * sin_t[None, :]
    assert np.abs(rho).max() < 2 ** 31
    rr = ((rho >> 1) + (2 * 16384 * size)) >> 16
    ok = (rr >= 0) & (rr < size)
    cells = (rr * size + np.arange(size)[None, :])[ok]
    uniq, counts = np.unique(cells, return_counts=True)
    nz = torch.nonzero(acc.view(-1)).view(-1)
    assert np.array_equal(nz.cpu().numpy(), uniq)
    assert np.array_equal(acc.view(-1)[nz].cpu().numpy(), counts)
    lines = h.find_lines(acc, 700, 5.0, 5.0)
    assert lines and lines[0].score == int(counts.max()) and abs(lines[0].angle) < 1.0
    del acc
    torch.cuda.empty_cache()


def test_canny_chain_1080p(zb, torch):
    from golden_shen_castan import smooth_noise
    frame = smooth_noise(31, 1080, 1920, 3)
    edges_dev = zb.Image.from_numpy(frame).canny(1.4, 20.0, 60.0)
    size = 1080
    box = zb.Rectangle(420, 0, 420 + size, size)
    acc = torch.zeros((size, size), dtype=torch.int32, device="cuda")
    h = zb.HoughTransform(size)
    h.compute(edges_dev, box, acc)
    acc_np = acc.cpu().numpy().view(np.uint32)
    edges_np = edges_dev.to_numpy()
    want = zo.compute(size, edges_np, (420, 0, 420 + size, size), np.zeros((size, size), np.uint32))
    assert np.array_equal(acc_np, want)
    th = max(1, int(want.max()) // 2)
    lines = _lines(h.find_lines(acc, th, 5.0, 5.0))
    assert lines == zo.find_lines(size, want, th, 5.0, 5.0) and len(lines) > 0


def test_cap_smaller_than_n(zb, torch):
    size = 256
    img = _random(9, 300, 300, 0.05)
    acc_np = _check(zb, torch, size, img, (0, 0, size, size))
    want = zo.find_lines(size, acc_np, 1, 2.0, 2.0)
    assert len(want) > 5
    acc = torch.from_numpy(acc_np.view(np.int32)).cuda()
    h = zb.HoughTransform(size)
    L = zb.lib()
    out = (zb._ffi.ZbHoughLine * 3)()
    n = C.c_uint32(0)
    a = zb.ZbImage(acc.data_ptr(), size, size, size)
    assert L.zb_hough_find_lines(h._h, a, 1, C.c_float(2.0), C.c_float(2.0), out, 3, C.byref(n), torch.cuda.current_stream().cuda_stream) == 0
    assert n.value == len(want)
    assert [(o.angle, o.radius, o.score, o.p1x, o.p1y, o.p2x, o.p2y) for o in out] == want[:3]


@pytest.mark.parametrize("name", list(CASES))
def test_golden_fixtures(zb, torch, name):
    want = json.loads(GOLDEN.read_text())["cases"][name]
    img = edges(name)
    acc, lines = device(zb, torch, name, img)
    assert zb.lib().zb_last_kernel().decode() == "hough_vote"
    assert sha(acc) == want["accumulator_sha256"]
    assert len(lines) == want["lines"] and sha(lines_array(lines)) == want["lines_sha256"]
