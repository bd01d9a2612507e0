"""Image.floodFill on the GPU, bit-identical to the oracle (oracle/zo_flood_fill.cpp, bound in tests/flood_fill_oracle.py) pixel for pixel:
the reference's four tests through the ABI; all five pixel formats x both modes x both connectivities on random images of odd sizes from
1 x 1 to 4096^2; adversarial topologies (a uniform image, a one-pixel-wide spiral, a checkerboard and crossing diagonals under
8-connectivity through tile corners, noise at the site-percolation threshold, seed-only fills, a fill value equal to the region's value);
strided views guarded by sentinels; more than 65,535 row tiles; an out-of-bounds seed; a non-blocking stream and two host threads with a
stream each; the golden fixtures."""
import json
import threading
from pathlib import Path

import numpy as np
import pytest

import flood_fill_oracle as zo
from golden_flood_fill import CASES, FORMATS, PERCOLATION, checkerboard, diagonals, image, percolation, random_image, special_floats, spiral
from gpu_utils import sha

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_flood_fill.json"
FILLS = {"u8": 42, "f32": -7.25, "rgb8": (1, 2, 3), "rgba8": (9, 8, 7, 6), "rgbaf32": (0.5, -0.5, 2.0, 3.0)}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def _device(zb, img, r, c, fill, th, conn, mode):
    dev = zb.Image.from_numpy(img)
    out = dev.flood_fill(r, c, fill, th, zb.Connectivity(conn), zb.FloodFillMode(mode))
    assert out is dev
    assert zb.lib().zb_last_kernel().decode() == "flood_fill"
    return dev.to_numpy()


def _check(zb, img, r, c, fill, th=0.0, conn=4, mode=zo.SEED):
    got = _device(zb, img, r, c, fill, th, conn, mode)
    want = zo.flood_fill(img.copy(), r, c, fill, th, conn, mode)
    if sha(got) != sha(want):
        bad = (got.view(np.uint8) != want.view(np.uint8)).reshape(img.shape[0], img.shape[1], -1).any(axis=2)
        pytest.fail(f"{img.shape} {img.dtype} seed ({r}, {c}) th {th} conn {conn} mode {mode}: {int(bad.sum())} pixels differ, "
                    f"first at {np.argwhere(bad)[:3].tolist()}")
    return got


def test_reference_tests(zb):
    img = np.zeros((5, 5), np.uint8)
    for r, c in ((0, 1), (1, 2), (2, 0), (2, 1), (2, 2), (2, 3), (2, 4), (3, 2), (4, 2)):
        img[r, c] = 5
    assert _check(zb, img, 2, 2, 9, 0.0, 4)[0, 1] == 5
    assert _check(zb, img, 2, 2, 9, 0.0, 8)[0, 1] == 9
    grad = np.arange(5, dtype=np.uint8).reshape(1, 5)
    assert _check(zb, grad, 0, 0, 9, 1.0, 4, zo.SEED).tolist() == [[9, 9, 2, 3, 4]]
    assert _check(zb, grad, 0, 0, 9, 1.0, 4, zo.NEIGHBOR).tolist() == [[9, 9, 9, 9, 9]]
    rgb = np.array([[[100, 100, 100], [100, 100, 103], [100, 100, 107]]], np.uint8)
    assert _check(zb, rgb, 0, 0, (255, 0, 0), 4.0)[0, 2].tolist() == [100, 100, 107]
    assert _check(zb, rgb, 0, 0, (255, 0, 0), 8.0)[0, 2].tolist() == [255, 0, 0]
    dev = zb.Image.from_numpy(np.zeros((3, 3), np.uint8))
    with pytest.raises(zb.ZignalError) as e:
        dev.flood_fill(3, 3, 9, 1.0)
    assert e.value.name == "OutOfBounds"


SHAPES = [(1, 1), (1, 777), (613, 1), (17, 33), (33, 65), (127, 255), (1000, 999)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("conn", [4, 8])
@pytest.mark.parametrize("mode", [zo.SEED, zo.NEIGHBOR], ids=["seed", "neighbor"])
def test_random_images(zb, fmt, conn, mode):
    scale = 1.0 if fmt in ("f32", "rgbaf32") else 255.0
    for k, (rows, cols) in enumerate(SHAPES):
        rng = np.random.default_rng(k)
        img = random_image(fmt, rows, cols, 10 * k + conn + mode, levels=2 + k % 3)
        if fmt in ("f32", "rgbaf32") and k % 2:
            img = special_floats(rows, cols, k, channels=4 if fmt == "rgbaf32" else None)
        for th in (0.0, 0.6 * scale, 1.5 * scale):
            _check(zb, img, int(rng.integers(0, rows)), int(rng.integers(0, cols)), FILLS[fmt], th, conn, mode)


@pytest.mark.parametrize("fmt", FORMATS)
def test_4096_square(zb, fmt):
    img = random_image(fmt, 4096, 4096, 99, levels=2)
    th = 0.0 if fmt == "u8" else (1.0 if fmt in ("f32", "rgbaf32") else 255.0)
    _check(zb, img, 2048, 1000, FILLS[fmt], th, 8 if fmt in ("u8", "rgb8") else 4, zo.SEED if fmt != "rgba8" else zo.NEIGHBOR)


def test_uniform_image_is_one_component(zb):
    for shape in ((4096, 4096), (1999, 3001)):
        img = np.full(shape, 17, np.uint8)
        got = _check(zb, img, shape[0] - 1, shape[1] // 2, 200, 0.0, 4)
        assert (got == 200).all()
    img = np.full((777, 1025, 4), 0.25, np.float32)
    assert (_check(zb, img, 0, 0, (1.0, 2.0, 3.0, 4.0), 0.0, 8, zo.NEIGHBOR)[..., 3] == 4.0).all()


def test_spiral_maze(zb):
    for n in (509, 2048, 4096):
        img = spiral(n)
        for conn in (4, 8):
            got = _check(zb, img, 0, 0, 100, 0.0, conn)
            if conn == 4:
                assert (got == 100).sum() == (img == 255).sum()
    _check(zb, spiral(1023), 511, 511, 3, 0.0, 4, zo.NEIGHBOR)   # from the centre of the maze outwards


def test_diagonal_connections_across_tile_corners(zb):
    for offset in (0, 1):
        _check(zb, checkerboard(161, 259, offset), 0, 1 - offset, 7, 0.0, 8)
        _check(zb, checkerboard(161, 259, offset), 0, 1 - offset, 7, 0.0, 8, zo.NEIGHBOR)
        _check(zb, checkerboard(64, 96, offset), 16, 32 - offset, 7, 0.0, 4)
    img = diagonals(257, 257)
    got = _check(zb, img, 0, 0, 9, 0.0, 8)
    assert (got == 9).sum() == (img == 255).sum()               # both diagonals, joined at the centre
    _check(zb, diagonals(300, 450), 0, 449, 9, 0.0, 8)
    _check(zb, diagonals(300, 450), 0, 449, 9, 0.0, 4)


def test_percolation_noise(zb):
    for conn in (4, 8):
        for k, n in enumerate((1000, 4096)):
            img = percolation(n, n, PERCOLATION[conn], 50 + k)
            _check(zb, img, n // 2, n // 2, 1, 0.0, conn)
            _check(zb, img, n // 2, n // 2, 1, 0.0, conn, zo.NEIGHBOR)


def test_seed_only_fills(zb):
    img = random_image("f32", 100, 130, 3)
    for th in (-1.0, float("nan"), -np.inf):
        for mode in (zo.SEED, zo.NEIGHBOR):
            got = _check(zb, img, 50, 60, 5.0, th, 8, mode)
            assert (got == 5.0).sum() == 1
    nan_img = np.full((64, 70), np.nan, np.float32)
    got = _check(zb, nan_img, 10, 10, 1.0, np.inf, 8)
    assert (got == 1.0).sum() == 1
    inf_img = np.full((40, 50, 4), np.inf, np.float32)            # inf - inf is NaN: no neighbour is within any threshold
    _check(zb, inf_img, 3, 4, (0.0, 0.0, 0.0, 0.0), np.inf, 4, zo.NEIGHBOR)


def test_fill_value_equal_to_region_value(zb):
    img = random_image("u8", 300, 301, 8, levels=2)
    got = _check(zb, img, 150, 150, int(img[150, 150]), 0.0, 4)
    assert np.array_equal(got, img)
    rgb = random_image("rgb8", 90, 91, 9, levels=2)
    _check(zb, rgb, 45, 45, tuple(int(x) for x in rgb[45, 45]), 0.0, 8, zo.NEIGHBOR)


def test_strided_views_with_sentinels(zb, torch):
    for fmt, sentinel in (("u8", 0xA5), ("rgb8", 0xA5), ("rgbaf32", -123.5), ("f32", np.nan)):
        base = random_image(fmt, 300, 400, 21, levels=2)
        l, t, r, b = 37, 13, 37 + 255, 13 + 201
        big = np.full_like(base, sentinel)                          # sentinels everywhere outside the view
        big[t:b, l:r] = base[t:b, l:r]
        dev = zb.Image.from_numpy(big)
        v = dev.view(zb.Rectangle(l, t, r, b))
        th = 0.0 if fmt in ("u8", "rgb8") else 1.0
        v.flood_fill(100, 50, FILLS[fmt], th, zb.Connectivity.EIGHT, zb.FloodFillMode.SEED)
        got = dev.to_numpy()
        expect = big.copy()
        zo.flood_fill(expect[t:b, l:r], 100, 50, FILLS[fmt], th, 8, zo.SEED)
        assert sha(got) == sha(expect), fmt


def test_more_than_65535_row_tiles(zb):
    rows = 65536 * 16 + 37                                          # 65,539 row tiles of 16 rows
    img = np.zeros((rows, 3), np.uint8)
    img[:, 1] = 255                                                 # one column from top to bottom
    img[rows // 3, 1] = 0                                           # cut once
    got = _check(zb, img, rows - 1, 1, 9, 0.0, 4)
    assert (got[:, 1] == 9).sum() == rows - rows // 3 - 1
    _check(zb, img, 0, 0, 9, 0.0, 8)


def test_out_of_bounds_leaves_the_image_untouched(zb, torch):
    img = random_image("rgba8", 40, 50, 2)
    dev = zb.Image.from_numpy(img)
    for r, c in ((40, 0), (0, 50), (2**32 - 1, 3)):
        with pytest.raises(zb.ZignalError) as e:
            dev.flood_fill(r, c, (1, 2, 3, 4))
        assert e.value.status == 27
    torch.cuda.synchronize()
    assert np.array_equal(dev.to_numpy(), img)


def _stream_case(zb, torch, seed):
    img = percolation(1024, 1536, PERCOLATION[8], seed)
    dev = zb.Image.from_numpy(img)
    torch.cuda.current_stream().synchronize()
    dev.flood_fill(512, 768, 3, 0.0, zb.Connectivity.EIGHT, zb.FloodFillMode.SEED)
    return img, dev


def test_non_blocking_stream_and_two_threads(zb, torch):
    want = {}
    for seed in (1, 2):
        img, dev = _stream_case(zb, torch, seed)
        want[seed] = dev.to_numpy()
        assert sha(want[seed]) == sha(zo.flood_fill(img.copy(), 512, 768, 3, 0.0, 8, zo.SEED))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _, dev = _stream_case(zb, torch, 1)
        s.synchronize()
        assert sha(dev.to_numpy()) == sha(want[1])
    results, errors = {}, []
    start = threading.Barrier(2)

    def work(seed):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                img = percolation(1024, 1536, PERCOLATION[8], seed)
                dev = zb.Image.from_numpy(img)
                st.synchronize()
                start.wait()
                dev.flood_fill(512, 768, 3, 0.0, zb.Connectivity.EIGHT, zb.FloodFillMode.SEED)
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
        assert sha(results[seed]) == sha(want[seed]), seed


def test_golden_fixtures(zb):
    gold = json.loads(GOLDEN.read_text())["cases"]
    for name, (_, (r, c), fill, th, conn, mode) in CASES.items():
        img = image(name)
        assert sha(img) == gold[name]["input_sha256"], name
        assert sha(_device(zb, img, r, c, fill, th, conn, mode)) == gold[name]["output_sha256"], name
