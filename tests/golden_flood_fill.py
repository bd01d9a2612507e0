"""Seeded Image.floodFill inputs and cases shared by the fixture generator (tests/golden/make_golden_flood_fill.py), the CPU tests of the
oracle (tests/test_flood_fill_host.py) and the GPU tests (tests/test_gpu_flood_fill.py).  Every image comes from numpy's PCG64 or a closed
form, so the fixtures only pin the oracle's output."""
import numpy as np

import flood_fill_oracle as zo

FORMATS = ("u8", "f32", "rgb8", "rgba8", "rgbaf32")
_SHAPE = {"u8": (), "f32": (), "rgb8": (3,), "rgba8": (4,), "rgbaf32": (4,)}
_DTYPE = {"u8": np.uint8, "f32": np.float32, "rgb8": np.uint8, "rgba8": np.uint8, "rgbaf32": np.float32}
PERCOLATION = {4: 0.5927, 8: 0.4073}   # site-percolation thresholds of the square lattice


def random_image(fmt, rows, cols, seed, levels=3):
    """Values on a coarse grid of `levels` steps (so that threshold 0 still forms regions), plus small noise in the float formats."""
    rng = np.random.default_rng(seed)
    shape = (rows, cols) + _SHAPE[fmt]
    q = rng.integers(0, levels, shape)
    if _DTYPE[fmt] == np.uint8:
        return (q * (255 // max(levels - 1, 1))).astype(np.uint8)
    img = q.astype(np.float32) / np.float32(max(levels - 1, 1))
    jitter = rng.random(shape) < 0.2
    return np.where(jitter, img + rng.normal(0, 0.05, shape).astype(np.float32), img).astype(np.float32)


def special_floats(rows, cols, seed, channels=None):
    """f32 values drawn from {0, -0, 1, NaN, inf, -inf, 0.5} (per channel when `channels`)."""
    rng = np.random.default_rng(seed)
    vals = np.array([0.0, -0.0, 1.0, np.nan, np.inf, -np.inf, 0.5], np.float32)
    shape = (rows, cols) if channels is None else (rows, cols, channels)
    return vals[rng.integers(0, vals.size, shape)]


def spiral(n, value=255):
    """A one-pixel-wide square spiral path (gap one pixel) from the top-left corner inwards: one 4-connected path over about half the
    pixels of an n x n u8 image."""
    img = np.zeros((n, n), np.uint8)
    lengths = [n - 1, n - 1, n - 1]
    k = n - 3
    while k > 0:
        lengths += [k, k]
        k -= 2
    r = c = 0
    img[0, 0] = value
    dirs = ((0, 1), (1, 0), (0, -1), (-1, 0))
    for i, ln in enumerate(lengths):
        dr, dc = dirs[i % 4]
        if dr:
            rs = np.arange(r + dr, r + dr * (ln + 1), dr)
            img[rs, c] = value
            r += dr * ln
        else:
            cs = np.arange(c + dc, c + dc * (ln + 1), dc)
            img[r, cs] = value
            c += dc * ln
    return img


def checkerboard(rows, cols, offset=0):
    """255 where (r + c + offset) is even: under 8-connectivity every connection is diagonal, including those across tile corners."""
    rr, cc = np.mgrid[0:rows, 0:cols]
    return np.where((rr + cc + offset) % 2 == 0, 255, 0).astype(np.uint8)


def diagonals(rows, cols):
    """The two diagonals r == c and r + c == cols - 1 of an otherwise empty u8 image (8-connected lines through tile corners)."""
    img = np.zeros((rows, cols), np.uint8)
    n = min(rows, cols)
    i = np.arange(n)
    img[i, i] = 255
    img[i, cols - 1 - i] = 255
    return img


def percolation(rows, cols, p, seed):
    """Sites 255 with probability p, else 0; the centre site is set, so a fill from it grows the cluster through the centre."""
    rng = np.random.default_rng(seed)
    img = np.where(rng.random((rows, cols)) < p, 255, 0).astype(np.uint8)
    img[rows // 2, cols // 2] = 255
    return img


def gradient_rgb(rows, cols):
    """A smooth Rgb(u8) ramp: neighbours differ by at most a few steps, far pixels by a lot (.neighbor fills much more than .seed)."""
    rr, cc = np.mgrid[0:rows, 0:cols]
    return np.stack([(rr * 3) % 256, (cc * 2) % 256, ((rr + cc) // 2) % 256], axis=2).astype(np.uint8)


# name -> (image builder, (start_row, start_col), fill_value, threshold, connectivity, mode)
CASES = {
    "u8_random_333x517_seed_c4": (lambda: random_image("u8", 333, 517, 1), (100, 200), 7, 0.0, 4, zo.SEED),
    "u8_random_333x517_neighbor_c8": (lambda: random_image("u8", 333, 517, 2, levels=4), (5, 9), 200, 85.0, 8, zo.NEIGHBOR),
    "f32_random_257x129_neighbor_c4": (lambda: random_image("f32", 257, 129, 3), (128, 64), -1.5, 0.06, 4, zo.NEIGHBOR),
    "f32_special_200x300_seed_c8": (lambda: special_floats(200, 300, 4), (0, 0), 9.0, np.inf, 8, zo.SEED),
    "rgb8_gradient_300x400_neighbor_c4": (lambda: gradient_rgb(300, 400), (150, 150), (255, 0, 0), 4.0, 4, zo.NEIGHBOR),
    "rgb8_gradient_300x400_seed_c8": (lambda: gradient_rgb(300, 400), (150, 150), (0, 255, 0), 40.0, 8, zo.SEED),
    "rgba8_random_199x301_seed_c4": (lambda: random_image("rgba8", 199, 301, 5, levels=2), (99, 150), (1, 2, 3, 4), 361.0, 4, zo.SEED),
    "rgbaf32_random_150x250_neighbor_c8": (lambda: random_image("rgbaf32", 150, 250, 6, levels=2), (75, 125), (0.25, 0.5, 0.75, 1.0), 1.1, 8,
                                           zo.NEIGHBOR),
    "u8_spiral_509_c4": (lambda: spiral(509), (0, 0), 128, 0.0, 4, zo.SEED),
    "u8_checkerboard_97x131_c8": (lambda: checkerboard(97, 131), (0, 0), 1, 0.0, 8, zo.SEED),
    "u8_percolation_512_c4": (lambda: percolation(512, 512, PERCOLATION[4], 7), (256, 256), 77, 0.0, 4, zo.SEED),
    "u8_percolation_512_c8": (lambda: percolation(512, 512, PERCOLATION[8], 8), (256, 256), 77, 0.0, 8, zo.NEIGHBOR),
}


def image(name):
    return CASES[name][0]()


def oracle(name, img=None):
    """The oracle's filled image for a case (a copy of the input)."""
    img = image(name) if img is None else img.copy()
    _, (r, c), fill, th, conn, mode = CASES[name]
    return zo.flood_fill(img, r, c, fill, th, conn, mode)
